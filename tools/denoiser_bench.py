"""Denoiser timing on the GPU.

Reports, as medians of CUDA-event timings after warm-up (the card's name and power limit are read in the same run):
  - Denoiser.forward at B = 1 and B = 64 x 204,800 samples (800 frames), and the same call through the eager fp32
    oracle restatement (oracle/denoiser_oracle.py: conv1d, atan2, conv_transpose1d, ...) on the same card, as context;
  - WaveGlow.infer at B = 64 x 800 frames in both tiers, and the share the denoiser adds to it;
  - Denoiser.stream over the items of WaveGlow.infer_stream (B = 64, 800 decoder steps) at chunk_steps 32 and 128,
    against the same WaveGlow stream alone.
Work: about 4.2 MFLOP per 256-sample block per transform pair (2 x 1024 x 1026 multiply-adds each), 0.22 TFLOP at
B = 64 x 800 blocks.  Weights are the seeded synthetic ones of the tests.  Prints one JSON line per measurement.

    python tools/denoiser_bench.py [--reps 5] [--warmup 2]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.audio_stream_latency import card  # noqa: E402


def timed(fn, reps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--samples", type=int, default=204800)
    args = ap.parse_args()

    import torch
    import tacotron2_b200 as t2
    from oracle import denoiser_oracle as D
    from tests.common import rand_text, synth_state_dict
    from tests.waveglow_common import CONFIG, mel_input, synth_state_dict as wg_state_dict
    if not torch.cuda.is_available():
        raise SystemExit("denoiser_bench: needs a CUDA device")
    torch.cuda.set_device(0)
    name, limit = card()
    ctx = dict(card=name, power_limit=limit, reps=args.reps)

    def emit(**r):
        r.update(ctx)
        print(json.dumps(r), flush=True)

    glows = {}
    for tier in ("fp32", "fp16"):
        g = t2.WaveGlow(**CONFIG)
        g.load_state_dict(wg_state_dict(7))
        g = g.cuda()
        if tier == "fp16":
            g = g.half()
            for k in g.convinv:
                k.float()
        glows[tier] = g
    den = t2.Denoiser(glows["fp32"])
    n = args.samples
    blocks = n // 256
    for B in (1, 64):
        y = (torch.randn(B, n, generator=torch.Generator().manual_seed(B)) * 0.3).cuda()
        ms = timed(lambda: den(y, 0.1), args.reps, args.warmup)
        flop = 2.0 * 2 * 1024 * 1026 * B * blocks
        emit(what="Denoiser.forward", B=B, samples=n, ms=round(ms, 3), tflops=round(flop / ms / 1e9, 1))
        ms_o = timed(lambda: D.denoise(y, den.bias_spec, 0.1, torch.float32), max(1, args.reps // 2), 1)
        emit(what="eager fp32 oracle", B=B, samples=n, ms=round(ms_o, 3))
        if B == 64:
            ms_den = ms
    mel = mel_input(64, blocks, 1).cuda()
    for tier, g in glows.items():
        m = mel.half() if tier == "fp16" else mel
        ms_w = timed(lambda: g.infer(m, sigma=0.666), max(1, args.reps // 2), 1)
        emit(what="WaveGlow.infer", tier=tier, B=64, frames=blocks, ms=round(ms_w, 1),
             denoiser_share_pct=round(100.0 * ms_den / ms_w, 3))
    # streams: the text-to-mel stream is collected first, so only the vocoder and the denoiser are timed
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(synth_state_dict(5, gate_bias=-10.0, scale=2.0))
    model = model.cuda().eval()
    model.decoder.max_decoder_steps = blocks
    model.decoder.gate_threshold = 1.0
    text = rand_text(64, 150, 1).cuda()
    g = glows["fp32"]
    for chunk in (32, 128):
        with torch.no_grad():
            mels = list(model.inference_stream(text, chunk_steps=chunk))
        ms_ws = timed(lambda: list(g.infer_stream(iter(mels), sigma=0.666)), 1, 1)
        audio_items = list(g.infer_stream(iter(mels), sigma=0.666))
        ms_ds = timed(lambda: list(den.stream(iter(audio_items), 0.1)), args.reps, args.warmup)
        emit(what="Denoiser.stream", B=64, steps=blocks, chunk_steps=chunk, audio_items=len(audio_items),
             stream_ms=round(ms_ds, 2), waveglow_stream_ms=round(ms_ws, 1),
             denoiser_share_pct=round(100.0 * ms_ds / ms_ws, 3))


if __name__ == "__main__":
    main()
