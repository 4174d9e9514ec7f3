"""Pitch targets on the GPU against the host: B = 64 clips at 22050 Hz with lengths uniform in 1 ... 10 s (fixed seed;
voiced harmonic segments with vibrato, pauses and noise), turned into f0 by one ragged ``tacotron2_b200.pyin(y,
C2, C7, lengths=...)`` call, and per-symbol averages by one ``average_by_durations`` call.  Both go through the public
functions, argument checks and their host reads included.  The host arm is the numpy fp64 oracle
(``tests/pyin_oracle.py``, librosa 0.10's algorithm) on --host-clips of the clips, one clip at a time; its time per
second of audio gives the estimate for the whole batch.  Prints the median CUDA-event time of each GPU call over --reps
timed runs after --warmup untimed ones, the host medians, whether the GPU's voiced flags equal the oracle's on the host
clips, and the card's name and power limit, as one JSON line.

    python tools/pitch_timing.py [--reps 10] [--warmup 3] [--host-clips 4] [--out /tmp/pitch_timing.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import tacotron2_b200 as t2  # noqa: E402
from tests import pyin_oracle as PO  # noqa: E402

SR = 22050
C2, C7 = 65.40639132514966, 2093.004522404789


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def clip(n, g):
    """Voiced segments (a harmonic tone with vibrato at a random pitch), pauses, and a little noise."""
    y = 0.01 * torch.randn(n, generator=g)
    pos = 0
    while pos < n:
        seg = int(torch.randint(SR // 10, SR // 2, (1,), generator=g))
        if float(torch.rand(1, generator=g)) < 0.7:
            f = 80 + float(torch.rand(1, generator=g)) * 320
            tt = torch.arange(min(seg, n - pos)) / SR
            ph = 2 * np.pi * f * (tt + 0.004 * torch.sin(2 * np.pi * 5 * tt))
            y[pos:pos + len(tt)] += sum(0.3 / k * torch.sin(k * ph) for k in range(1, 5))
        pos += seg
    return y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-clips", type=int, default=4)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    g = torch.Generator().manual_seed(args.seed)
    lengths = torch.randint(SR, 10 * SR + 1, (args.B,), generator=g).tolist()
    n = max(lengths)
    y = torch.zeros(args.B, n)
    for b, L in enumerate(lengths):
        y[b, :L] = clip(L, g)
    y = y.cuda()
    ln = torch.tensor(lengths, device="cuda")
    F = 1 + n // 256
    T_text = 100
    d = torch.zeros(args.B, T_text, dtype=torch.int64)
    for b, L in enumerate(lengths):                       # each row's frames spread over its 100 symbols
        Fb = 1 + L // 256
        d[b] = Fb // T_text
        d[b, :Fb % T_text] += 1
    d = d.cuda()
    f0 = t2.pyin(y, C2, C7, lengths=ln)[0]
    runs = {"pyin": lambda: t2.pyin(y, C2, C7, lengths=ln),
            "average_by_durations": lambda: t2.average_by_durations(f0, d)}
    for fn in runs.values():
        for _ in range(args.warmup):
            fn()
    times = {k: [] for k in runs}
    for _ in range(args.reps):
        for k, fn in runs.items():
            times[k].append(timed(fn))
    med = {k: statistics.median(v) for k, v in times.items()}
    _, flag, _ = t2.pyin(y, C2, C7, lengths=ln)
    flag = flag.cpu().numpy()
    host, host_audio, agree = [], 0.0, True
    for b in range(min(args.host_clips, args.B)):
        x = y[b, :lengths[b]].cpu().numpy()
        t0 = time.perf_counter()
        _, oflag, _ = PO.pyin(x, C2, C7)
        host.append(time.perf_counter() - t0)
        host_audio += lengths[b] / SR
        agree = agree and bool(np.array_equal(oflag, flag[b, :1 + lengths[b] // 256]))
    audio = sum(lengths) / SR
    res = {"card": card(), "B": args.B, "seconds_of_audio": round(audio, 1), "frames_max": F, "reps": args.reps,
           "median_ms": {k: round(v, 3) for k, v in med.items()},
           "spread_ms": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
           "host_oracle": {"clips": len(host), "seconds_of_audio": round(host_audio, 1),
                           "median_s_per_clip": round(statistics.median(host), 3),
                           "s_per_audio_second": round(sum(host) / host_audio, 4),
                           "batch_estimate_s": round(sum(host) / host_audio * audio, 1)},
           "voiced_flags_equal_oracle_on_host_clips": agree}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
