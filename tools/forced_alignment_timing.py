"""Forced-alignment synthesis against the free run it replays: B = 64 texts of 150 symbols (fixed seeds), every row
running 800 decoder steps (gate threshold 1, max_decoder_steps 800).  Alternates a free ``Tacotron2.inference`` with a
forced ``inference`` fed that run's own alignments and mel_lengths, both with per-utterance seeds, and prints the median
CUDA-event time of each over --reps timed pairs after --warmup untimed ones, with the card's name and power limit and
whether the forced run reproduced the free run's decoder outputs (mel, gate, alignments) bit for bit, as one JSON line.
The postnet outputs are not compared: the forced call runs every row's postnet on its own, the free one batched.

    python tools/forced_alignment_timing.py [--reps 5] [--warmup 1] [--out /tmp/forced_timing.json]"""
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
        free = [o.clone() for o in model.inference(text, seeds=seeds)]
        lengths = model.mel_lengths.clone()
        runs = {
            "free": lambda: model.inference(text, seeds=seeds),
            "forced": lambda: model.inference(text, seeds=seeds, alignments=free[3], alignment_lengths=lengths),
        }
        for fn in runs.values():
            for _ in range(args.warmup):
                fn()
        times = {k: [] for k in runs}
        same = True
        for _ in range(args.reps):                       # alternate the two, so drift hits both alike
            for k, fn in runs.items():
                ms, out = timed(fn)
                times[k].append(ms)
                if k == "forced":
                    same &= all(torch.equal(out[i], free[i]) for i in (0, 2, 3))     # mel, gate, alignments
    med = {k: statistics.median(v) for k, v in times.items()}
    res = {"card": card(), "B": args.B, "T_text": args.T, "steps": int(lengths.max()), "reps": args.reps,
           "median_ms": {k: round(v, 2) for k, v in med.items()},
           "spread_ms": {k: [round(min(v), 2), round(max(v), 2)] for k, v in times.items()},
           "forced_over_free": round(med["forced"] / med["free"], 3), "decoder_outputs_reproduced": bool(same)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
