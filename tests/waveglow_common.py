"""Seeded WaveGlow weights, inputs and the host rebuild of the engine's Philox noise, shared by the WaveGlow tests,
the fixture generator, smoke() and tools/waveglow_bench.py."""
import math

import torch

from tests.philox_ref import philox4x32_10

CONFIG = dict(n_mel_channels=80, n_flows=12, n_group=8, n_early_every=4, n_early_size=2,
              WN_config=dict(n_layers=8, n_channels=256, kernel_size=3))
NOISE_TAG = 0x3c6ef372        # the fourth counter word of the engine's noise draws (waveglow.cu)


def n_remaining(k):
    return 8 if k < 4 else (6 if k < 8 else 4)


def state_dict_shapes():
    """(name, shape) of the 686 state_dict entries of WaveGlow(**CONFIG), in the reference's order."""
    s = [("upsample.weight", (80, 80, 1024)), ("upsample.bias", (80,))]
    for k in range(12):
        p, nh = "WN.%d." % k, n_remaining(k) // 2
        for i in range(8):
            q = p + "in_layers.%d." % i
            s += [(q + "bias", (512,)), (q + "weight_g", (512, 1, 1)), (q + "weight_v", (512, 256, 3))]
        for i in range(8):
            q, r = p + "res_skip_layers.%d." % i, (512 if i < 7 else 256)
            s += [(q + "bias", (r,)), (q + "weight_g", (r, 1, 1)), (q + "weight_v", (r, 256, 1))]
        s += [(p + "start.bias", (256,)), (p + "start.weight_g", (256, 1, 1)), (p + "start.weight_v", (256, nh, 1)),
              (p + "end.weight", (2 * nh, 256, 1)), (p + "end.bias", (2 * nh,)),
              (p + "cond_layer.bias", (4096,)), (p + "cond_layer.weight_g", (4096, 1, 1)),
              (p + "cond_layer.weight_v", (4096, 640, 1))]
    s += [("convinv.%d.conv.weight" % k, (n_remaining(k), n_remaining(k), 1)) for k in range(12)]
    return s


def synth_state_dict(seed=7):
    """Deterministic weights with a non-trivial coupling in every flow: the reference zeroes ``end`` (every coupling is
    then the identity), here end ~ U(+-1/16) and biases ~ U(+-0.05); weight_v ~ U(+-1/sqrt(fan_in)) with weight_g =
    ||v|| * U(0.5, 1.5) so the weight-norm fold matters; convinv an orthonormal, determinant +1 matrix."""
    g = torch.Generator().manual_seed(seed)
    u = lambda shape, b: (torch.rand(shape, generator=g) * 2 - 1) * b          # noqa: E731
    sd = {}
    for name, shape in state_dict_shapes():
        if name == "upsample.weight":
            sd[name] = u(shape, 1.0 / math.sqrt(4 * 80))
        elif name.endswith("weight_v"):
            sd[name] = u(shape, 1.0 / math.sqrt(shape[1] * shape[2]))
        elif name.endswith("weight_g"):
            sd[name] = None
        elif name.endswith("end.weight"):
            sd[name] = u(shape, 1.0 / 16)
        elif name.startswith("convinv"):
            c = shape[0]
            w = torch.linalg.qr(torch.randn(c, c, generator=g, dtype=torch.float64))[0]
            if torch.det(w) < 0:
                w[:, 0] = -w[:, 0]
            sd[name] = w.float().view(c, c, 1)
        else:
            sd[name] = u(shape, 0.05)
    # weight_g is listed before weight_v: fill it now that v exists
    for name, shape in state_dict_shapes():
        if name.endswith("weight_g"):
            v = sd[name[:-1] + "v"]
            sd[name] = v.flatten(1).norm(dim=1).view(-1, 1, 1) * (0.5 + torch.rand(shape, generator=g))
    return {n: sd[n] for n, _ in state_dict_shapes()}


def mel_input(B, T, seed):
    """A seeded (B, 80, T) spectrogram-like input."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 80, T, generator=g) * 0.5 - 1.0


def noise(B, T, seed):
    """Seeded standard-normal draws (B, 8, 32 T) for waveglow_noise."""
    return torch.randn(B, 8, 32 * T, generator=torch.Generator().manual_seed(seed))


def philox_noise(seed, B, T):
    """Host rebuild of the engine's in-kernel draws: z[b, c, t] from Philox4x32-10 with counter (t, b, c, NOISE_TAG)
    and key (seed lo, seed hi); Box-Muller on output words 0 and 1 in fp32 (waveglow.cu, philox_normal)."""
    L = 32 * T
    t = torch.arange(L, dtype=torch.int64).view(1, 1, L).expand(B, 8, L)
    b = torch.arange(B, dtype=torch.int64).view(B, 1, 1).expand(B, 8, L)
    c = torch.arange(8, dtype=torch.int64).view(1, 8, 1).expand(B, 8, L)
    o = philox4x32_10((t, b, c, torch.full_like(t, NOISE_TAG)), (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))
    u1 = ((o[0] >> 8) + 1).to(torch.float32) * (1.0 / 16777216.0)
    u2 = (o[1] >> 8).to(torch.float32) * (1.0 / 16777216.0)
    return torch.sqrt(-2.0 * torch.log(u1)) * torch.cos(6.283185307179586 * u2)
