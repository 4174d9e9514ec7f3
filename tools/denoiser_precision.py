"""Where the denoiser's error against fp64 comes from.

The engine computes both transforms as GEMMs on split fp16 operands (x = hi + lo, hi * hi + lo * hi + hi * lo, fp32
accumulation in wgmma).  This tool rebuilds, in fp64 on the GPU, exactly the operands the kernels feed to the tensor
cores (the reflect-padded audio, the forward basis, the gated spectrum stored as X / 512, the inverse basis times 2^12,
each split into its fp16 hi and lo halves) and sums the three products exactly.  Then
  - split_err  = |emulation - fp64 oracle|: what rounding the operands to split fp16 costs;
  - accum_err  = |engine - emulation|: what the tensor cores' fp32 accumulation (and the fp32 epilogues) add;
  - ftz_err    = |engine - emulation with fp16 subnormals flushed to zero|: a check that the lo halves below fp16's
                 normal range are used, not flushed;
each as max |difference| / max |fp64 oracle|.  Also runs the amplitude cases: int16-scale audio (x 32767) and audio
just below the fp16 limit.  Prints one JSON line per case.

    python tools/denoiser_precision.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    import torch
    import tacotron2_b200 as t2
    from oracle import denoiser_oracle as D
    from tests.common import stft_inputs
    from tests.waveglow_common import CONFIG, synth_state_dict
    if not torch.cuda.is_available():
        raise SystemExit("denoiser_precision: needs a CUDA device")
    dev = torch.device("cuda")
    f64 = torch.float64
    glow = t2.WaveGlow(**CONFIG)
    glow.load_state_dict(synth_state_dict(7))
    den = t2.Denoiser(glow.cuda())
    bias = den.bias_spec.double()
    fwd = den.stft.forward_basis.float()
    inv = den.stft.inverse_basis.float() * 4096.0

    def split(x, ftz):
        hi = x.half().float()
        lo = (x - hi).half().float()
        if ftz:
            tiny = torch.finfo(torch.float16).tiny
            hi = torch.where(hi.abs() < tiny, torch.zeros_like(hi), hi)
            lo = torch.where(lo.abs() < tiny, torch.zeros_like(lo), lo)
        return hi.to(f64), lo.to(f64)

    def emulate(y, strength, ftz):
        x = torch.nn.functional.pad(y[:, None, None, :], (512, 512, 0, 0), mode="reflect")[:, 0]
        hx, lx = split(x, ftz)
        hw, lw = split(fwd, ftz)
        conv = torch.nn.functional.conv1d
        ft = conv(hx, hw, stride=256) + conv(lx, hw, stride=256) + conv(hx, lw, stride=256)
        re, im = ft[:, :513], ft[:, 513:]
        mag = torch.sqrt(re ** 2 + im ** 2)
        m = torch.clamp(mag - bias * strength, min=0.0)
        s = torch.where(mag > 0, m / torch.where(mag > 0, mag, torch.ones_like(mag)), torch.zeros_like(mag))
        spec = torch.cat([torch.where(mag > 0, re * s, m), im * s], 1).float() / 512.0
        hs, ls = split(spec, ftz)
        hi_, li_ = split(inv, ftz)
        ct = torch.nn.functional.conv_transpose1d
        out = ct(hs, hi_, stride=256) + ct(ls, hi_, stride=256) + ct(hs, li_, stride=256)
        out = out * (512.0 / 4096.0)
        env = torch.from_numpy(D.window_sumsquare(mag.shape[-1])).to(dev).to(f64)
        nz = env > torch.finfo(torch.float32).tiny
        out[:, :, nz] /= env[nz]
        return (out * 4.0)[:, :, 512:-512]

    sig = stft_inputs(3, 256 * 40 + 100)
    unit = sig / sig.abs().max()
    cases = [("stft_inputs, strength 0", sig, 0.0),
             ("stft_inputs, strength 0.1", sig, 0.1),
             ("randn 0.3, B=8 x 204800, strength 0.1",
              (torch.randn(8, 204800, generator=torch.Generator().manual_seed(1)) * 0.3).clamp(-1, 1), 0.1),
             ("int16 scale (max 32767), strength 0.1", unit * 32767.0, 0.1),
             ("near the fp16 limit (max 65000), strength 0.1", unit * 65000.0, 0.1)]
    for name, y, strength in cases:
        y = y.to(dev)
        got = den(y, strength=strength).double()
        ref = D.denoise(y, bias, strength, f64)
        scale = float(ref.abs().max())
        em, em_ftz = emulate(y.float(), strength, False), emulate(y.float(), strength, True)
        r = dict(case=name, max_abs_audio=float(y.abs().max()), finite=bool(torch.isfinite(got).all()),
                 engine_err=float((got - ref).abs().max()) / scale,
                 split_err=float((em - ref).abs().max()) / scale,
                 accum_err=float((got - em).abs().max()) / scale,
                 ftz_err=float((got - em_ftz).abs().max()) / scale,
                 card=torch.cuda.get_device_name(0))
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
