"""Throughput of a queue of utterances of very different lengths: static 64-row batches against continuous batching.

A seeded workload -- 512 requests, text lengths uniform in 20..200, frame counts uniform in 100..1000 -- runs on synthetic
weights.  The frame counts are imposed through each request's max_decoder_steps with gate_threshold = 1.0: the gates of
random weights fire on the first step otherwise (DESIGN section 7).  Timed, alternating, in one process, after one untimed
pass over every arm (which warms every shape):

  static/arrival   64-row batches in arrival order through inference(text, input_lengths), max_decoder_steps = the
                   batch's longest row
  static/sorted    the same after sorting the requests by frame count (what a static scheduler could do with an oracle)
  server/16,32,64  inference_server(slots=64) at chunk_steps 16 / 32 / 64

Per arm: wall time to the last result (host clock around work that ends in a synchronise), useful mel frames per second
(the sum of the requests' lengths over that time), slot occupancy = useful row-steps / (64 x decoder steps launched), a
count, and for the server the time per chunk outside the decoder kernel (admission, collect, postnet of finished rows,
host sync: wall time less the decoder launches' CUDA-event time, over the chunks).  One JSON line per arm, then a table.

    python tools/serve_throughput.py [--requests 512] [--rounds 3] [--out FILE]
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import tacotron2_b200 as t2  # noqa: E402
from tests.common import synth_state_dict  # noqa: E402

SLOTS = 64


def workload(n, seed):
    g = torch.Generator().manual_seed(seed)
    text_len = torch.randint(20, 201, (n,), generator=g).tolist()
    frames = torch.randint(100, 1001, (n,), generator=g).tolist()
    texts = [torch.randint(0, 148, (L,), generator=g) for L in text_len]
    return texts, frames


def static_batches(model, texts, frames, order):
    """Returns (useful frames, decoder steps launched)."""
    steps = 0
    for i in range(0, len(order), SLOTS):
        idx = order[i:i + SLOTS]
        lens = torch.tensor([texts[j].numel() for j in idx])
        pad = torch.zeros(len(idx), int(lens.max()), dtype=torch.int64)
        for r, j in enumerate(idx):
            pad[r, :lens[r]] = texts[j]
        cap = max(frames[j] for j in idx)
        model.decoder.max_decoder_steps = cap
        model.inference(pad.cuda(), input_lengths=lens)
        steps += cap
    torch.cuda.synchronize()
    return sum(frames), steps


def served(model, texts, frames, chunk):
    """Returns (useful frames, decoder steps launched, chunks, milliseconds inside the decoder launches)."""
    server = model.inference_server(slots=SLOTS, max_text_len=200, chunk_steps=chunk)
    events, launch = [], server.backend.launch

    def timed_launch(*a):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        launch(*a)
        e1.record()
        events.append((e0, e1))
    server.backend.launch = timed_launch
    for t, f in zip(texts, frames):
        server.submit(t, f)
    useful = sum(r["mel_length"] for r in server.run())
    torch.cuda.synchronize()
    return useful, server.row_steps // SLOTS, server.chunks, sum(a.elapsed_time(b) for a, b in events)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=2024)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    texts, frames = workload(args.requests, args.seed)
    if not torch.cuda.is_available():
        raise SystemExit("serve_throughput: no CUDA device; this measurement has no CPU fallback")
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                                    "-i", "0"]).decode().strip()
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(synth_state_dict(5, scale=2.0))
    model = model.cuda().eval()
    model.decoder.gate_threshold = 1.0
    arrival = list(range(len(texts)))
    by_frames = sorted(arrival, key=lambda j: frames[j])
    arms = [("static/arrival", lambda: static_batches(model, texts, frames, arrival)),
            ("static/sorted", lambda: static_batches(model, texts, frames, by_frames))]
    arms += [("server/%d" % c, (lambda c: lambda: served(model, texts, frames, c))(c)) for c in (16, 32, 64)]
    rows = {name: [] for name, _ in arms}
    with torch.no_grad():
        for rnd in range(args.rounds + 1):            # round 0 warms every shape
            for name, fn in arms:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                with contextlib.redirect_stdout(io.StringIO()):      # one max-steps warning per request
                    res = fn()
                dt = time.perf_counter() - t0
                if rnd:
                    rows[name].append((dt,) + tuple(res))
    useful_steps = sum(frames)
    out = []
    for name, _ in arms:
        r = rows[name]
        wall = sorted(x[0] for x in r)
        med = wall[len(wall) // 2]
        rec = dict(arm=name, card=card, requests=len(texts), rounds=len(r), wall_s=round(med, 4),
                   wall_s_min=round(wall[0], 4), wall_s_max=round(wall[-1], 4), useful_frames=r[0][1],
                   useful_frames_per_s=round(r[0][1] / med, 1), decoder_steps=r[0][2],
                   slot_occupancy=round(useful_steps / (SLOTS * r[0][2]), 4))
        if name.startswith("server"):
            pick = min(r, key=lambda x: abs(x[0] - med))
            rec.update(chunks=pick[3], ms_per_chunk_outside_decoder=round((pick[0] * 1e3 - pick[4]) / pick[3], 3),
                       decoder_ms=round(pick[4], 1))
        out.append(rec)
        print(json.dumps(rec))
    print("\n%s" % card)
    print("| arm | wall s (min..max) | useful frames/s | decoder steps | slot occupancy | ms/chunk outside the decoder |")
    print("|---|---|---|---|---|---|")
    for rec in out:
        print("| %s | %.3f (%.3f..%.3f) | %.0f | %d | %.1f %% | %s |" % (
            rec["arm"], rec["wall_s"], rec["wall_s_min"], rec["wall_s_max"], rec["useful_frames_per_s"], rec["decoder_steps"],
            100 * rec["slot_occupancy"], rec.get("ms_per_chunk_outside_decoder", "-")))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
