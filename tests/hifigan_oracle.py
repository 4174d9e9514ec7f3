"""The HiFi-GAN generator's forward (jik876/hifi-gan, models.py) restated in torch fp64 with functional conv ops and
explicit weight-norm folding, from a state_dict and a configuration.

round16=True also rounds to fp16 wherever the engine's fp16 tier stores fp16: the folded weights of every GEMM
convolution, the input mels and every activation plane (each layer's lrelu input and each residual).  The MRF sum and
conv_post stay wide, as in the engine."""
import torch
import torch.nn.functional as F


def _f(h, name):
    return h[name] if isinstance(h, dict) else getattr(h, name)


def fold(sd, prefix):
    """The convolution's weight in fp64: g * v / ||v|| with the norm over every dim but 0, or the plain weight."""
    if prefix + ".weight_g" in sd:
        v = sd[prefix + ".weight_v"].double()
        g = sd[prefix + ".weight_g"].double()
        return g * v / v.norm(dim=tuple(range(1, v.dim())), keepdim=True)
    return sd[prefix + ".weight"].double()


def forward(sd, h, mel, round16=False):
    """mel (B, 80, T) -> audio (B, 1, 256 T), fp64 (on mel's device)."""
    sd = {k: v.to(mel.device) for k, v in sd.items()}
    r = (lambda t: t.half().double()) if round16 else (lambda t: t)

    def conv(x, p, dil=1, pad=None, rw=True):
        w = fold(sd, p)
        w = r(w) if rw else w
        k = w.shape[2]
        return F.conv1d(x, w, sd[p + ".bias"].double(), dilation=dil,
                        padding=(k * dil - dil) // 2 if pad is None else pad)

    lrelu = lambda t, s=0.1: F.leaky_relu(t, s)
    nk = len(_f(h, "resblock_kernel_sizes"))
    rb = str(_f(h, "resblock"))
    x = r(mel.double())
    x = r(lrelu(conv(x, "conv_pre", pad=3)))
    n_up = len(_f(h, "upsample_rates"))
    for i, (u, k) in enumerate(zip(_f(h, "upsample_rates"), _f(h, "upsample_kernel_sizes"))):
        p = "ups.%d" % i
        y = F.conv_transpose1d(x, r(fold(sd, p)), sd[p + ".bias"].double(), stride=u, padding=(k - u) // 2)
        Y, AY = r(y), r(lrelu(y))
        xs = None
        for j, (kk, ds) in enumerate(zip(_f(h, "resblock_kernel_sizes"), _f(h, "resblock_dilation_sizes"))):
            q = "resblocks.%d" % (i * nk + j)
            res, a = Y, AY
            ds = list(ds)[:3 if rb == "1" else 2]
            for m, d in enumerate(ds):
                if rb == "1":
                    t = r(lrelu(conv(a, "%s.convs1.%d" % (q, m), d)))
                    t = conv(t, "%s.convs2.%d" % (q, m), 1) + res
                else:
                    t = conv(a, "%s.convs.%d" % (q, m), d) + res
                if m < len(ds) - 1:
                    res, a = r(t), r(lrelu(t))
            xs = t if xs is None else xs + t
        x = xs / nk
        x = r(lrelu(x, 0.1 if i < n_up - 1 else 0.01))
    return torch.tanh(conv(x, "conv_post", pad=3, rw=False))
