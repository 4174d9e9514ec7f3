"""WaveGlow.infer throughput / latency on the GPU, with the eager oracle (cuDNN) on the same card as context.

    python tools/waveglow_bench.py [--reps 5] [--warmup 2] [--channels 256 --layers 8 --flows 12] [--no-oracle]
                                   [--out results/waveglow_bench.json]
The default shape is the published model's; --channels / --layers / --flows pick another WN width, depth and flow count
(early outputs every 4 flows, 2 channels), with seeded weights.

Times with CUDA events after warm-up, median over repeats.  Achieved TFLOP/s uses the algorithmic count computed from
the shapes (flops_per_sample), against the H100 SXM data-sheet dense FP16 peak (989 TFLOP/s); the card name and power
limit are read in the same run.
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
from tests import waveglow_config_oracle as WO  # noqa: E402
from tests.waveglow_common import CONFIG, mel_input, noise, synth_state_dict  # noqa: E402

PEAK_FP16 = 989e12


def flops_per_sample(n_mel=80, n_ch=256, n_layers=8, n_flows=12, group=8):
    """Multiply-adds x 2 per audio sample of WaveGlow.infer, from the layer shapes."""
    cond = 2 * n_mel * group * 2 * n_ch * n_layers                      # cond_layer 640 -> 4096 per group column
    layers = n_layers * 2 * (3 * n_ch * 2 * n_ch) + (n_layers - 1) * 2 * n_ch * 2 * n_ch + 2 * n_ch * n_ch
    per_flow = cond + layers + 2 * 4 * n_ch * 2                          # + start / end (<= 4 / 8 channels)
    upsample = 2 * n_mel * n_mel * 4                                     # 4 frames x 80 x 80 per output sample
    return n_flows * per_flow / group + upsample


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--T", type=int, default=800)
    ap.add_argument("--oracle-fp32-rows", type=int, default=8)
    ap.add_argument("--channels", type=int, default=CONFIG["WN_config"]["n_channels"])
    ap.add_argument("--layers", type=int, default=CONFIG["WN_config"]["n_layers"])
    ap.add_argument("--flows", type=int, default=CONFIG["n_flows"])
    ap.add_argument("--no-oracle", action="store_true", help="time the engine only")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "waveglow_bench needs a GPU"
    cfg = dict(CONFIG, n_flows=a.flows, WN_config=dict(n_layers=a.layers, n_channels=a.channels, kernel_size=3))
    fpsamp = flops_per_sample(n_ch=a.channels, n_layers=a.layers, n_flows=a.flows)
    if cfg == CONFIG:
        sd = synth_state_dict(7)
    else:
        from tests.waveglow_configs import state_dict_for
        sd = state_dict_for(cfg, 7)
    res = {"card": card(), "config": dict(channels=a.channels, layers=a.layers, flows=a.flows), "flops_per_sample": fpsamp,
           "B": a.B, "T_mel": a.T}
    print("card:", res["card"], " algorithmic MFLOP per sample: %.2f" % (fpsamp / 1e6))

    def record(name, ms, B, T):
        n = B * 256 * T
        r = {"ms": ms, "samples_per_s": n / (ms / 1e3), "tflops": fpsamp * n / (ms / 1e3) / 1e12}
        r["share_of_fp16_peak"] = r["tflops"] * 1e12 / PEAK_FP16
        res[name] = r
        print("%-28s B=%-3d T=%-4d %10.2f ms  %12.0f samples/s  %7.1f TFLOP/s (%.1f%% of FP16 peak)" %
              (name, B, T, ms, r["samples_per_s"], r["tflops"], 100 * r["share_of_fp16_peak"]))

    for half in (True, False):
        m = t2.WaveGlow(**cfg)
        m.load_state_dict(sd)
        m = m.cuda()
        if half:
            m = m.half()
            for k in m.convinv:
                k.float()
        dt = torch.float16 if half else torch.float32
        tier = "fp16" if half else "fp32"
        mel = mel_input(a.B, a.T, 1).to("cuda", dt)
        record("engine_%s_B%d" % (tier, a.B), timed(lambda: m.infer(mel, sigma=0.666), a.reps, a.warmup), a.B, a.T)
        mel1 = mel[:1].contiguous()
        record("engine_%s_B1" % tier, timed(lambda: m.infer(mel1, sigma=0.666), a.reps, a.warmup), 1, a.T)
        del m
        torch.cuda.empty_cache()

    if a.no_oracle:
        if a.out:
            os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
            with open(a.out, "w") as f:
                json.dump(res, f, indent=1)
        return
    # eager oracle (cuDNN): fp16 at the full batch, fp32 with TF32 off on a slice of it
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sd16 = {k: (v.half() if not k.startswith("convinv") else v).cuda() for k, v in sd.items()}
    mel = mel_input(a.B, a.T, 1).cuda()
    z = noise(a.B, a.T, 2).cuda()
    with torch.no_grad():
        record("oracle_fp16_cudnn_B%d" % a.B,
               timed(lambda: WO.infer(sd16, mel.half(), 0.666, z.half(), torch.float16), max(1, a.reps // 2), 1), a.B, a.T)
        del sd16
        torch.cuda.empty_cache()
        b = a.oracle_fp32_rows
        sd32 = {k: v.cuda() for k, v in sd.items()}
        record("oracle_fp32_notf32_B%d" % b,
               timed(lambda: WO.infer(sd32, mel[:b], 0.666, z[:b], torch.float32), max(1, a.reps // 2), 1), b, a.T)
    res["speedup_fp16_vs_oracle_fp16"] = res["oracle_fp16_cudnn_B%d" % a.B]["ms"] / res["engine_fp16_B%d" % a.B]["ms"]
    print("engine fp16 tier vs eager fp16 oracle at B=%d: %.2fx" % (a.B, res["speedup_fp16_vs_oracle_fp16"]))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
