"""Cost of per-utterance seeds: alternates seeded and unseeded runs of Tacotron2.inference (B = 64 x 800 decoder steps,
gate_threshold 1.0 so every row runs all steps) and of WaveGlow.infer (B = 64 x 800 frames, fp16 tier) and prints the
median CUDA-event time of each, with the card's name and power limit, as one JSON line.

    python tools/seeded_inference_timing.py [--reps 5] [--out /tmp/seeded_timing.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import tacotron2_b200 as t2  # noqa: E402
from tests.common import rand_text, synth_state_dict  # noqa: E402
from tests.waveglow_common import CONFIG, mel_input  # noqa: E402
from tests.waveglow_common import synth_state_dict as wg_state_dict  # noqa: E402


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
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--steps", type=int, default=800)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    B, S = args.B, args.steps
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(synth_state_dict(5))
    model = model.cuda().eval()
    model.decoder.max_decoder_steps, model.decoder.gate_threshold = S, 1.0
    text = rand_text(B, 150, 1).cuda()
    seeds = torch.arange(1, B + 1, dtype=torch.int64).cuda()
    glow = t2.WaveGlow(**CONFIG)
    glow.load_state_dict(wg_state_dict(7))
    glow = glow.cuda().half()
    mel = mel_input(B, S, 2).cuda().half()
    runs = {
        "inference_unseeded": lambda: model.inference(text),
        "inference_seeded": lambda: model.inference(text, seeds=seeds),
        "waveglow_unseeded": lambda: glow.infer(mel, 0.666),
        "waveglow_seeded": lambda: glow.infer(mel, 0.666, seeds=seeds),
    }
    times = {k: [] for k in runs}
    with torch.no_grad():
        for fn in runs.values():          # warm-up: modules, workspaces, packed weights
            fn()
        torch.cuda.synchronize()
        for _ in range(args.reps):        # alternate so drift hits both sides alike
            for k, fn in runs.items():
                times[k].append(timed(fn))
    res = dict(card=card(), B=B, steps_or_frames=S, reps=args.reps,
               median_ms={k: round(statistics.median(v), 3) for k, v in times.items()},
               min_ms={k: round(min(v), 3) for k, v in times.items()},
               max_ms={k: round(max(v), 3) for k, v in times.items()})
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
