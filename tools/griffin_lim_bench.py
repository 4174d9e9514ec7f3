"""Griffin-Lim timing on the GPU.

Reports, as medians of CUDA-event timings after warm-up (the card's name and power limit are read in the same run):
  - the engine's Griffin-Lim (one t2_griffin_lim call from uploaded angles) at B = 1 and B = 64 x 800 frames, for
    n_iters 30 and 60, and the cost of one iteration from the difference;
  - the host draw of the initial angles (np.random.rand + np.angle(np.exp(...)), as the reference draws them) and their
    upload, timed on the host clock;
  - STFT.transform and STFT.inverse alone at the same sizes;
  - the same Griffin-Lim through the eager fp32 oracle (tests/griffin_lim_oracle.py: conv1d, atan2, conv_transpose1d, the
    reference's algorithm) on the same card, as context.
Work: about 4.2 MFLOP per frame per iteration (a forward and an inverse GEMM of 2 x 1024 x 1026 multiply-adds each).
The target is the magnitude of seeded noise.  Prints one JSON line per measurement.

    python tools/griffin_lim_bench.py [--reps 5] [--warmup 2] [--frames 800]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.audio_stream_latency import card  # noqa: E402
from tools.denoiser_bench import timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--frames", type=int, default=800)
    args = ap.parse_args()

    import numpy as np
    import torch
    import tacotron2_b200 as t2
    from tests import griffin_lim_oracle as G
    from tacotron2_b200.audio_processing import _griffin_lim
    if not torch.cuda.is_available():
        raise SystemExit("griffin_lim_bench: needs a CUDA device")
    torch.cuda.set_device(0)
    name, limit = card()
    ctx = dict(card=name, power_limit=limit, reps=args.reps)

    def emit(**r):
        r.update(ctx)
        print(json.dumps(r), flush=True)

    st = t2.TacotronSTFT().cuda().stft_fn
    F = args.frames
    n = 256 * (F - 1)
    for B in (1, 64):
        y = (torch.randn(B, n, generator=torch.Generator().manual_seed(B)) * 0.3).cuda()
        mag, _ = st.transform(y)
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            a = np.angle(np.exp(2j * np.pi * np.random.rand(*mag.shape))).astype(np.float32)
            ang = torch.from_numpy(a).cuda()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        emit(what="host angle draw + upload", B=B, frames=F, ms=round(statistics.median(ts), 3))
        ms = {}
        for it in (30, 60):
            ms[it] = timed(lambda: _griffin_lim(mag, ang, st, it), args.reps, args.warmup)
            emit(what="griffin_lim engine", B=B, frames=F, n_iters=it, launches=3 * it + 2, ms=round(ms[it], 3))
        per = (ms[60] - ms[30]) / 30
        flop = 2.0 * 2 * 1024 * 1026 * B * F
        emit(what="griffin_lim one iteration (from n_iters 60 - 30)", B=B, frames=F, ms=round(per, 4),
             tflops=round(flop / per / 1e9, 1))
        emit(what="STFT.transform", B=B, frames=F, ms=round(timed(lambda: st.transform(y), args.reps, args.warmup), 4))
        emit(what="STFT.inverse", B=B, frames=F,
             ms=round(timed(lambda: st.inverse(mag, ang), args.reps, args.warmup), 4))
        ms_o = timed(lambda: G.griffin_lim(mag, ang, 30, torch.float32), max(1, args.reps // 2), 1)
        emit(what="eager fp32 oracle griffin_lim", B=B, frames=F, n_iters=30, ms=round(ms_o, 2))


if __name__ == "__main__":
    main()
