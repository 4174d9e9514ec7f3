"""HiFi-GAN generator throughput on the GPU: V1, V2 and V3 in both tiers, with WaveGlow.infer and the generator in
eager torch (cuDNN, fp32 and fp16) on the same mels and the same card.

    python tools/hifigan_bench.py [--reps 5] [--warmup 2] [--T 800] [--B 1 64] [--no-eager] [--no-waveglow]
                                  [--out results/hifigan_bench.json]

Times with CUDA events after warm-up, median over repeats.  Algorithmic TFLOP/s uses the FLOP count computed here from
the layer shapes (flops_per_sample: V1 2.40, V2 0.150, V3 0.176 MFLOP per sample).  The card name and power limit are
read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import tacotron2_b200 as t2  # noqa: E402
from tacotron2_b200.hifigan import CONFIGS  # noqa: E402
from tests.hifigan_common import mel_input, model  # noqa: E402
from tests.waveglow_common import CONFIG as WG_CONFIG, synth_state_dict as wg_state_dict  # noqa: E402


def flops_per_sample(h):
    """Multiply-adds x 2 per audio sample of the generator, from the layer shapes."""
    c, rate = h["upsample_initial_channel"], 1.0 / 256
    mac = 80 * c * 7 * rate                                            # conv_pre
    nd = 3 if h["resblock"] == "1" else 2
    for u, k in zip(h["upsample_rates"], h["upsample_kernel_sizes"]):
        co = c // 2
        mac += c * co * k * rate                                       # each input frame scatters c x co x k
        rate *= u
        for kk in h["resblock_kernel_sizes"]:
            mac += (2 * nd if h["resblock"] == "1" else nd) * co * co * kk * rate
        c = co
    mac += c * 7                                                       # conv_post
    return 2 * mac


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def eager(G, x):
    """models.py's Generator.forward in eager torch on the module tree (cuDNN convolutions)."""
    lrelu = torch.nn.functional.leaky_relu
    x = G.conv_pre(x)
    for i in range(G.num_upsamples):
        x = G.ups[i](lrelu(x, 0.1))
        xs = None
        for j in range(G.num_kernels):
            rb = G.resblocks[i * G.num_kernels + j]
            y = x
            if hasattr(rb, "convs1"):
                for c1, c2 in zip(rb.convs1, rb.convs2):
                    y = c2(lrelu(c1(lrelu(y, 0.1)), 0.1)) + y
            else:
                for c in rb.convs:
                    y = c(lrelu(y, 0.1)) + y
            xs = y if xs is None else xs + y
        x = xs / G.num_kernels
    return torch.tanh(G.conv_post(lrelu(x)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--T", type=int, default=800)
    ap.add_argument("--B", type=int, nargs="+", default=[1, 64])
    ap.add_argument("--no-eager", action="store_true")
    ap.add_argument("--no-waveglow", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    res = dict(card=card(), T=a.T, reps=a.reps, warmup=a.warmup, rows=[])
    print("card:", res["card"])
    for B in a.B:
        mel = mel_input(B, a.T, 1).cuda()
        n = B * 256 * a.T
        for name in ("v1", "v2", "v3"):
            fl = flops_per_sample(CONFIGS[name])
            for tier in ("fp32", "fp16"):
                G = model(name).cuda().eval()
                if tier == "fp16":
                    G = G.half()
                x = mel.to(G.conv_pre.bias.dtype)
                with torch.no_grad():
                    ms = timed(lambda: G(x), a.reps, a.warmup)
                    row = dict(B=B, model=name, tier=tier, what="engine", ms=ms, samples_per_s=n / ms * 1e3,
                               tflops=fl * n / ms / 1e9, mflop_per_sample=fl / 1e6)
                    res["rows"].append(row)
                    print(json.dumps(row))
                    if not a.no_eager:
                        ms = timed(lambda: eager(G, x), a.reps, a.warmup)
                        row = dict(B=B, model=name, tier=tier, what="eager cuDNN", ms=ms, samples_per_s=n / ms * 1e3,
                                   tflops=fl * n / ms / 1e9, mflop_per_sample=fl / 1e6)
                        res["rows"].append(row)
                        print(json.dumps(row))
                del G
                torch.cuda.empty_cache()
        if not a.no_waveglow:
            for tier in ("fp32", "fp16"):
                W = t2.WaveGlow(**WG_CONFIG)
                W.load_state_dict(wg_state_dict(7))
                W = W.cuda()
                if tier == "fp16":
                    W = W.half()
                    for k in W.convinv:
                        k.float()
                x = mel.to(W.upsample.weight.dtype)
                with torch.no_grad():
                    ms = timed(lambda: W.infer(x), a.reps, a.warmup)
                row = dict(B=B, model="waveglow", tier=tier, what="WaveGlow.infer", ms=ms, samples_per_s=n / ms * 1e3)
                res["rows"].append(row)
                print(json.dumps(row))
                del W
                torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
