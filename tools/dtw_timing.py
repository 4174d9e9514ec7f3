"""Objective evaluation on the GPU against the host: B = 64 pairs of log-mels of 100 ... 1000 frames (fixed seed).  x is
``TacotronSTFT.mel_spectrogram`` of seeded clips (harmonic segments with vibrato, pauses and noise, one ragged call);
y is each x warped by a seeded monotone frame map to 0.8 ... 1.25 times its length (at most 1000 frames) plus noise of
standard deviation 0.1.  Times ``tacotron2_b200.dtw`` on the mels (D = 80, fp32) and ``mel_cepstral_distortion``
(n_cep = 24), each a call through the public function with its argument checks, and ``dtw`` on the longest pair alone
(one CTA on one SM: what the batch cannot finish faster than).  The host arm is the numpy fp64 oracle
(``tests/dtw_oracle.py``) on --host-pairs of the pairs, one at a time.  Prints the median CUDA-event time of each GPU
call over --reps timed runs after --warmup untimed ones, the host medians, whether the GPU's cost and path equal the
oracle's on the host pairs, and the card's name and power limit, as one JSON line.

    python tools/dtw_timing.py [--reps 20] [--warmup 3] [--host-pairs 4] [--out /tmp/dtw_timing.json]"""
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
from tests import dtw_oracle as O  # noqa: E402

SR, HOP = 22050, 256


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
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-pairs", type=int, default=4)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    g = torch.Generator().manual_seed(args.seed)
    fx = torch.randint(100, 1001, (args.B,), generator=g)
    samples = (fx - 1) * HOP                                # 1 + samples // 256 frames
    audio = torch.zeros(args.B, int(samples.max()))
    for b, n in enumerate(samples.tolist()):
        audio[b, :n] = clip(n, g)
    mel_x = t2.TacotronSTFT().cuda().mel_spectrogram(audio.cuda(), samples.cuda())
    assert mel_x.shape[2] == int(fx.max())
    fy = torch.clamp((fx.double() * (0.8 + 0.45 * torch.rand(args.B, generator=g, dtype=torch.float64))).long(), 100,
                     1000)
    mel_y = torch.zeros(args.B, 80, int(fy.max()), device="cuda")
    for b in range(args.B):
        idx = torch.sort(torch.randint(0, int(fx[b]), (int(fy[b]),), generator=g)).values.cuda()
        mel_y[b, :, :fy[b]] = mel_x[b, :, idx] + 0.1 * torch.randn(80, int(fy[b]), generator=g).cuda()
    longest = int(torch.argmax(fx * fy))
    one_x, one_y = mel_x[longest:longest + 1, :, :fx[longest]].contiguous(), mel_y[longest:longest + 1, :, :fy[longest]]
    one_y = one_y.contiguous()
    xl, yl = fx.cuda(), fy.cuda()
    runs = {"dtw": lambda: t2.dtw(mel_x, mel_y, xl, yl),
            "mel_cepstral_distortion": lambda: t2.mel_cepstral_distortion(mel_x, mel_y, xl, yl),
            "dtw_longest_pair_alone": lambda: t2.dtw(one_x, one_y)}
    for fn in runs.values():
        for _ in range(args.warmup):
            fn()
    times = {k: [] for k in runs}
    for _ in range(args.reps):
        for k, fn in runs.items():
            times[k].append(timed(fn))
    med = {k: statistics.median(v) for k, v in times.items()}
    cost, path, n = (t.cpu() for t in t2.dtw(mel_x, mel_y, xl, yl))
    host, agree = [], True
    for b in range(min(args.host_pairs, args.B)):
        x, y = mel_x[b, :, :fx[b]].cpu().numpy(), mel_y[b, :, :fy[b]].cpu().numpy()
        t0 = time.perf_counter()
        c, p = O.dtw(x, y)
        host.append(time.perf_counter() - t0)
        agree = agree and float(cost[b]) == c and int(n[b]) == len(p) and np.array_equal(path[b, :len(p)].numpy(), p)
    cells = int((fx * fy).sum())
    host_cells = int((fx[:len(host)] * fy[:len(host)]).sum())
    res = {"card": card(), "B": args.B, "frames_x": [int(fx.min()), int(fx.max())],
           "frames_y": [int(fy.min()), int(fy.max())], "cells": cells,
           "longest_pair": [int(fx[longest]), int(fy[longest])], "reps": args.reps,
           "median_ms": {k: round(v, 3) for k, v in med.items()},
           "spread_ms": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
           "host_oracle": {"pairs": len(host), "median_s_per_pair": round(statistics.median(host), 3),
                           "s_per_million_cells": round(sum(host) / host_cells * 1e6, 3),
                           "batch_estimate_s": round(sum(host) / host_cells * cells, 1)},
           "cost_and_path_equal_oracle_on_host_pairs": agree}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
