"""Streaming text-to-audio latency: WaveGlow.infer_stream(Tacotron2.inference_stream(...)) against
Tacotron2.inference() followed by WaveGlow.infer() on the same inputs.

For every case it reports the median, after warm-up, of
  - base_ms:   inference() + infer(), ending in a device synchronise;
  - first_ms:  from the call to the first audio item whose samples are on the device;
  - total_ms:  the whole stream, ending in a device synchronise.
Cases: B = 1 and 64, T_text = 150, gate_threshold = 1.0 so every row runs max_decoder_steps = 800 steps, chunk_steps 32,
128 and 256, in the fp32 tier and in the notebook's .half() form.  Weights are the seeded synthetic ones of the tests
(the timing does not depend on their values).  The card's name and power limit are read in the same run.  Prints one
JSON line per case and a markdown table.

    python tools/audio_stream_latency.py [--batches 1,64] [--chunks 32,128,256] [--reps 3] [--warmup 1]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                      text=True).strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,64")
    ap.add_argument("--chunks", default="32,128,256")
    ap.add_argument("--tiers", default="fp32,fp16")
    ap.add_argument("--t-text", type=int, default=150)
    ap.add_argument("--steps", type=int, default=800)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sigma", type=float, default=0.666)
    args = ap.parse_args()

    import torch
    import tacotron2_b200 as t2
    from tests.common import rand_text, synth_state_dict
    from tests.waveglow_common import CONFIG, synth_state_dict as wg_state_dict
    if not torch.cuda.is_available():
        raise SystemExit("audio_stream_latency: needs a CUDA device")
    torch.cuda.set_device(0)
    name, limit = card()
    rows = []
    for tier in args.tiers.split(","):
        model = t2.Tacotron2(t2.create_hparams())
        model.load_state_dict(synth_state_dict(5, gate_bias=-10.0, scale=2.0))
        model = model.cuda().eval()
        glow = t2.WaveGlow(**CONFIG)
        glow.load_state_dict(wg_state_dict(7))
        glow = glow.cuda()
        if tier == "fp16":                 # the notebook: model.half(), waveglow.half() with convinv kept in fp32
            model = model.half()
            glow = glow.half()
            for k in glow.convinv:
                k.float()
        model.decoder.max_decoder_steps = args.steps
        model.decoder.gate_threshold = 1.0
        for B in [int(b) for b in args.batches.split(",")]:
            text = rand_text(B, args.t_text, 1).cuda()

            def base():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                with torch.no_grad():
                    post = model.inference(text)[1]
                    glow.infer(post, sigma=args.sigma, lengths=model.mel_lengths)
                torch.cuda.synchronize()
                return (time.perf_counter() - t0) * 1e3

            def stream(chunk):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                first = None
                n = 0
                for item in glow.infer_stream(model.inference_stream(text, chunk_steps=chunk), sigma=args.sigma):
                    n += 1
                    if first is None:
                        torch.cuda.synchronize()
                        first = (time.perf_counter() - t0) * 1e3
                torch.cuda.synchronize()
                return first, (time.perf_counter() - t0) * 1e3, n

            for _ in range(args.warmup):
                base()
            base_ms = statistics.median(base() for _ in range(args.reps))
            for chunk in [int(c) for c in args.chunks.split(",")]:
                for _ in range(args.warmup):
                    stream(chunk)
                runs = [stream(chunk) for _ in range(args.reps)]
                r = dict(tier=tier, B=B, T_text=args.t_text, steps=args.steps, chunk_steps=chunk, items=runs[0][2],
                         base_ms=round(base_ms, 1), first_ms=round(statistics.median(x[0] for x in runs), 1),
                         total_ms=round(statistics.median(x[1] for x in runs), 1), reps=args.reps, card=name,
                         power_limit=limit)
                print(json.dumps(r), flush=True)
                rows.append(r)
    print("\n%s, power limit %s; medians of %d runs after %d warm-up" % (name, limit, args.reps, args.warmup))
    print("| tier | B | chunk_steps | audio items | first audio (ms) | stream total (ms) | inference() + infer() (ms) |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %s | %d | %d | %d | %.1f | %.1f | %.1f |" % (r["tier"], r["B"], r["chunk_steps"], r["items"], r["first_ms"],
                                                        r["total_ms"], r["base_ms"]))


if __name__ == "__main__":
    main()
