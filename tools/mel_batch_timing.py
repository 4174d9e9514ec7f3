"""Ragged log-mel extraction against one call per clip: B = 64 clips at 22050 Hz with lengths uniform in 1 ... 10 s (fixed
seed), turned into mels by one ``TacotronSTFT.mel_spectrogram(y, lengths)`` call and by 64 ``mel_spectrogram(clip)``
calls.  Both go through the public method, range check included.  Prints the median CUDA-event time of each over --reps
timed runs after --warmup untimed ones, with the card's name and power limit, as one JSON line.

    python tools/mel_batch_timing.py [--reps 10] [--warmup 3] [--out /tmp/mel_timing.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import tacotron2_b200 as t2  # noqa: E402

SR = 22050


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    g = torch.Generator().manual_seed(args.seed)
    lengths = torch.randint(SR, 10 * SR + 1, (args.B,), generator=g).tolist()
    n = max(lengths)
    y = (0.3 * torch.randn(args.B, n, generator=g)).clamp(-1, 1)
    for b, L in enumerate(lengths):
        y[b, L:] = 0
    y = y.cuda()
    clips = [y[b:b + 1, :L] for b, L in enumerate(lengths)]
    stft = t2.TacotronSTFT().cuda()
    runs = {
        "ragged_one_call": lambda: stft.mel_spectrogram(y, lengths),
        "per_clip_calls": lambda: [stft.mel_spectrogram(c) for c in clips],
    }
    for fn in runs.values():
        for _ in range(args.warmup):
            fn()
    times = {k: [] for k in runs}
    for _ in range(args.reps):                          # alternate the two, so drift hits both alike
        for k, fn in runs.items():
            times[k].append(timed(fn))
    med = {k: statistics.median(v) for k, v in times.items()}
    res = {"card": card(), "B": args.B, "seconds_of_audio": round(sum(lengths) / SR, 1), "n_max": n, "reps": args.reps,
           "median_ms": {k: round(v, 3) for k, v in med.items()},
           "spread_ms": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
           "speedup": round(med["per_clip_calls"] / med["ragged_one_call"], 2)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
