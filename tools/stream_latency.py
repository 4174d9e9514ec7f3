"""Time to first audio frames: Tacotron2.inference_stream against Tacotron2.inference on the same inputs.

    python tools/stream_latency.py [--reps 5] [--json OUT]

Cases: B = 1 and 64, T_text = 150, 800 decoder steps (gate_threshold = 1.0, so every row runs to the cap, as bench.py
does), chunk_steps = 8, 32, 128.  For each case: the time to the first item (host clock from the call to the first item
in hand; the item's tensors are on the device and complete, since every chunk ends in a host sync), the total time of the
stream, and inference() on the same inputs, as medians over --reps after one warm-up of each shape.  The card's name and
power limit are read in the same run."""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import tacotron2_b200 as t2  # noqa: E402
from tests.common import keep_mask, rand_text, synth_state_dict  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return name, q.split(",")[1].strip()
    except Exception as e:  # noqa: BLE001
        return name, "unknown (%s)" % e


def time_inference(model, text):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        out = model.inference(text)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def time_stream(model, text, chunk):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first, n_items = None, 0
    with contextlib.redirect_stdout(io.StringIO()):       # the max-steps warning of every run
        for item in model.inference_stream(text, chunk_steps=chunk):
            if first is None:
                first = time.perf_counter() - t0
            n_items += 1
    torch.cuda.synchronize()
    return first, time.perf_counter() - t0, n_items


def time_decoder(model, memory, chunk):
    """The decoder alone: inference() vs inference_stream(), to split the stream's extra time into the decoder's share
    (relaunch, state save / restore, one host sync per chunk) and the rest (postnet over the halo, item assembly)."""
    dec = model.decoder
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        if chunk is None:
            dec.inference(memory)
        else:
            for _ in dec.inference_stream(memory, chunk_steps=chunk):
                pass
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=800)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "stream_latency needs a GPU"
    name, power = card()
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(synth_state_dict(5))
    model = model.cuda().eval()
    model.decoder.max_decoder_steps = args.steps
    model.decoder.gate_threshold = 1.0
    rows = []
    with torch.no_grad():
        for B in (1, 64):
            text = rand_text(B, 150, 1).cuda()
            keep = keep_mask((args.steps, 2, B, 256), 0.5, 2).cuda()
            with t2.dropout_masks(prenet=keep):
                time_inference(model, text)
                inf = statistics.median(time_inference(model, text)[0] for _ in range(args.reps))
                memory = model._t2_engine().encoder(text=text)
                time_decoder(model, memory, None)
                dec_inf = statistics.median(time_decoder(model, memory, None) for _ in range(args.reps))
                for chunk in (8, 32, 128):
                    time_stream(model, text, chunk)
                    runs = [time_stream(model, text, chunk) for _ in range(args.reps)]
                    time_decoder(model, memory, chunk)
                    dec_stream = statistics.median(time_decoder(model, memory, chunk) for _ in range(args.reps))
                    first = statistics.median(r[0] for r in runs)
                    total = statistics.median(r[1] for r in runs)
                    row = dict(B=B, T_text=150, steps=args.steps, chunk_steps=chunk, items=runs[0][2],
                               first_item_ms=round(first * 1e3, 2), stream_total_ms=round(total * 1e3, 2),
                               inference_ms=round(inf * 1e3, 2), total_over_inference=round(total / inf - 1.0, 4),
                               decoder_stream_ms=round(dec_stream * 1e3, 2), decoder_inference_ms=round(dec_inf * 1e3, 2))
                    rows.append(row)
                    print(json.dumps(row), flush=True)
    res = dict(card=name, power_limit=power, reps=args.reps, rows=rows)
    print(json.dumps(dict(card=name, power_limit=power)))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
