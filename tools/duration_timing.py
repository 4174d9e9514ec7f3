"""Duration extraction from real free-run attention maps: for each shape (B texts x T symbols x steps frames; default
64 x 150 x 800 and 32 x 300 x 2000) a seeded free ``Tacotron2.inference`` with the default-initialised (synthetic)
weights runs every row for all its steps (gate threshold 1), and its alignments go through

- ``durations_from_alignments`` with method "mas" and "argmax" (median CUDA-event time over --reps calls after
  --warmup untimed ones);
- the host path a user has without it: copy the map to the host, then the numpy fp64 dynamic programme of
  tests/durations_oracle.py row by row (MAS), or numpy argmax + bincount (median wall time over --host-reps calls,
  each ending with its result on the host).

Prints one JSON line with the card's name and power limit, the times in ms, and how many rows of the GPU's MAS
durations differ from the host oracle's (a difference is allowed only for paths whose fp64 scores tie to 1e-12).

    python tools/duration_timing.py [--reps 20] [--warmup 3] [--host-reps 3] [--out /tmp/duration_timing.json]"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import tacotron2_b200 as t2  # noqa: E402
from tests import durations_oracle as DO  # noqa: E402
from tools.forced_alignment_timing import card, timed  # noqa: E402


def free_run_map(B, T, steps):
    torch.manual_seed(0)
    model = t2.Tacotron2(t2.create_hparams()).cuda().eval()
    model.decoder.max_decoder_steps = steps
    model.decoder.gate_threshold = 1.0                   # every row runs all steps
    text = torch.randint(1, 148, (B, T), generator=torch.Generator().manual_seed(1)).cuda()
    with torch.no_grad():
        align = model.inference(text, seeds=[1000 + 7919 * b for b in range(B)])[3].clone()
    lengths = model.mel_lengths.clone()
    del model
    return align, lengths


def host_mas(align):
    a = align.cpu().numpy()
    return np.stack([DO.mas(a[b]) for b in range(a.shape[0])])


def host_argmax(align):
    a = align.cpu().numpy()
    return np.stack([DO.argmax(a[b]) for b in range(a.shape[0])])


def wall(fn):
    t0 = time.perf_counter()
    out = fn()
    return 1e3 * (time.perf_counter() - t0), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="64x150x800,32x300x2000", help="BxTxsteps, comma separated")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    result = {"card": card(), "shapes": []}
    for shape in args.shapes.split(","):
        B, T, steps = (int(v) for v in shape.split("x"))
        align, lengths = free_run_map(B, T, steps)
        assert align.shape == (B, steps, T) and bool((lengths == steps).all())
        row = {"B": B, "T_text": T, "T_mel": steps}
        for method in ("mas", "argmax"):
            fn = lambda: t2.durations_from_alignments(align, None, lengths, method)  # noqa: E731
            for _ in range(args.warmup):
                fn()
            torch.cuda.synchronize()
            row["gpu_%s_ms" % method] = statistics.median(timed(fn)[0] for _ in range(args.reps))
        host = {"mas": host_mas, "argmax": host_argmax}
        outs = {}
        for method, fn in host.items():
            times = []
            for _ in range(args.host_reps):
                ms, outs[method] = wall(lambda: fn(align))
                times.append(ms)
            row["host_%s_ms" % method] = statistics.median(times)
        gpu = {m: t2.durations_from_alignments(align, None, lengths, m).cpu().numpy() for m in host}
        row["argmax_equal"] = bool(np.array_equal(gpu["argmax"], outs["argmax"]))
        a = align.cpu().numpy()
        differ = [b for b in range(B) if not np.array_equal(gpu["mas"][b], outs["mas"][b])]
        for b in differ:
            s, r = DO.path_score(a[b], gpu["mas"][b]), DO.path_score(a[b], outs["mas"][b])
            assert abs(s - r) <= 1e-12 * abs(r), (b, s, r)
        row["mas_rows_differing_by_a_tie"] = len(differ)
        result["shapes"].append(row)
        print(json.dumps(row), flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
