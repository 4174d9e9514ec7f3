"""The cost of the attention window against the free run: B = 64 texts of 150 symbols (fixed seeds), every row running
800 decoder steps (gate threshold 1, max_decoder_steps 800).  Alternates a free ``Tacotron2.inference``, one with
``attention_window=(1, 3)`` and one with a window wide enough to mask nothing (both sides = the text length), all with
per-utterance seeds, and prints the median CUDA-event time of each over --reps timed rounds after --warmup untimed
ones, with the card's name and power limit and whether the wide window reproduced the free run bit for bit, as one JSON
line.  The windowed runs take the argmax pass on every step; the wide one isolates its cost, as it masks nothing.

    python tools/attention_window_timing.py [--reps 5] [--warmup 1] [--out /tmp/window_timing.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import tacotron2_b200 as t2  # noqa: E402


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
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--T", type=int, default=150)
    ap.add_argument("--steps", type=int, default=800)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    torch.manual_seed(0)
    model = t2.Tacotron2(t2.create_hparams()).cuda().eval()
    model.decoder.max_decoder_steps = args.steps
    model.decoder.gate_threshold = 1.0                   # every row runs all steps
    text = torch.randint(1, 148, (args.B, args.T), generator=torch.Generator().manual_seed(1)).cuda()
    seeds = [1000 + 7919 * b for b in range(args.B)]
    with torch.no_grad():
        runs = {
            "free": lambda: model.inference(text, seeds=seeds),
            "window_1_3": lambda: model.inference(text, seeds=seeds, attention_window=(1, 3)),
            "window_wide": lambda: model.inference(text, seeds=seeds, attention_window=(args.T, args.T)),
        }
        for fn in runs.values():
            for _ in range(args.warmup):
                fn()
        free = [o.clone() for o in runs["free"]()]
        times = {k: [] for k in runs}
        same = True
        for _ in range(args.reps):                       # alternate them, so drift hits all alike
            for k, fn in runs.items():
                ms, out = timed(fn)
                times[k].append(ms)
                if k == "window_wide":
                    same &= all(torch.equal(a, b) for a, b in zip(out, free))
    med = {k: statistics.median(v) for k, v in times.items()}
    res = {"card": card(), "B": args.B, "T_text": args.T, "steps": int(model.mel_lengths.max()), "reps": args.reps,
           "median_ms": {k: round(v, 2) for k, v in med.items()},
           "spread_ms": {k: [round(min(v), 2), round(max(v), 2)] for k, v in times.items()},
           "window_1_3_over_free": round(med["window_1_3"] / med["free"], 3),
           "window_wide_over_free": round(med["window_wide"] / med["free"], 3), "wide_window_reproduced_free": bool(same)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
