"""Plain-torch restatement of WaveGlow.infer (waveglow/glow.py:251-293) over a state dict.

Dtype-generic: ``dtype=torch.float64`` is the truth the engine is measured against; ``dtype=torch.float16`` rounds where
the reference's half path does (module converted with ``.half()``, ``convinv`` kept in fp32 and its inverse computed in
fp32 then cast to half, glow.py:88-96).  The reference itself cannot run ``infer`` in fp64: Invertible1x1Conv computes
``W_inverse`` through ``.float()`` and casts it back only for CUDA half tensors (glow.py:91-94), so a double input meets
an fp32 weight in ``conv1d``.  The noise is an argument: ``z`` (B, n_group, L) in draw order (the initial channels,
then the early blocks of flow 8 and flow 4), where the reference draws ``torch.cuda.FloatTensor(...).normal_()``.
"""
import torch
import torch.nn.functional as F

N_FLOWS, N_GROUP, N_EARLY_EVERY, N_EARLY_SIZE, N_LAYERS, N_CH = 12, 8, 4, 2, 8, 256


def conv_weight(sd, prefix):
    """The effective weight of a (possibly weight-normed) conv: g * v / ||v|| over all but dim 0
    (torch.nn.utils.weight_norm with dim=0), or the plain weight after remove_weightnorm."""
    if prefix + "weight_v" in sd:
        v, g = sd[prefix + "weight_v"], sd[prefix + "weight_g"]
        return v * (g / v.flatten(1).norm(dim=1).view(-1, 1, 1))
    return sd[prefix + "weight"]


def _wn(sd, k, audio, spect, dt):
    """WN.forward (glow.py:153-175) for flow k."""
    p = "WN.%d." % k
    w = lambda n: conv_weight(sd, p + n).to(dt)                       # noqa: E731
    bias = lambda n: sd[p + n + "bias"].to(dt)                         # noqa: E731
    audio = F.conv1d(audio, w("start."), bias("start."))              # :155
    output = torch.zeros_like(audio)                                   # :156
    spect = F.conv1d(spect, w("cond_layer."), bias("cond_layer."))    # :159
    for i in range(N_LAYERS):                                          # :161-173
        d = 2 ** i
        x = F.conv1d(audio, w("in_layers.%d." % i), bias("in_layers.%d." % i), dilation=d, padding=d)
        x = x + spect[:, i * 2 * N_CH:(i + 1) * 2 * N_CH, :]
        acts = torch.tanh(x[:, :N_CH]) * torch.sigmoid(x[:, N_CH:])    # :34-40
        rs = F.conv1d(acts, w("res_skip_layers.%d." % i), bias("res_skip_layers.%d." % i))
        if i < N_LAYERS - 1:
            audio = audio + rs[:, :N_CH]
            output = output + rs[:, N_CH:]
        else:
            output = output + rs
    return F.conv1d(output, sd[p + "end.weight"].to(dt), sd[p + "end.bias"].to(dt))   # :175


def infer(sd, spect, sigma, z, dtype=torch.float64):
    """spect (B, 80, T) -> audio (B, 256 T) in `dtype`, on spect's device."""
    dev = spect.device
    sd = {k: v.to(dev) for k, v in sd.items()}
    dt = dtype
    spect = spect.to(dt)
    B = spect.shape[0]
    spect = F.conv_transpose1d(spect, sd["upsample.weight"].to(dt), sd["upsample.bias"].to(dt), stride=256)   # :252
    spect = spect[:, :, :-(1024 - 256)]                                                                      # :254-255
    spect = spect.unfold(2, N_GROUP, N_GROUP).permute(0, 2, 1, 3)                                            # :257
    spect = spect.contiguous().view(B, spect.size(1), -1).permute(0, 2, 1)                                    # :258
    L = spect.shape[2]
    z = z.to(device=dev, dtype=dt)
    assert tuple(z.shape) == (B, N_GROUP, L), (tuple(z.shape), (B, N_GROUP, L))
    n_rem = N_GROUP - N_EARLY_SIZE * ((N_FLOWS - 1) // N_EARLY_EVERY)
    zc = n_rem
    audio = sigma * z[:, :n_rem]                                                                             # :260-269
    for k in reversed(range(N_FLOWS)):                                                                       # :271
        n_half = audio.size(1) // 2
        a0, a1 = audio[:, :n_half], audio[:, n_half:]
        out = _wn(sd, k, a0, spect, dt)                                                                      # :276
        s, b = out[:, n_half:], out[:, :n_half]
        a1 = (a1 - b) / torch.exp(s)                                                                         # :280
        audio = torch.cat([a0, a1], 1)
        W = sd["convinv.%d.conv.weight" % k].squeeze()
        Winv = W.double().inverse() if dt == torch.float64 else W.float().inverse()                         # :91
        audio = F.conv1d(audio, Winv.to(dt)[..., None])                                                      # :96
        if k % N_EARLY_EVERY == 0 and k > 0:                                                                 # :285-290
            audio = torch.cat((sigma * z[:, zc:zc + N_EARLY_SIZE], audio), 1)
            zc += N_EARLY_SIZE
    return audio.permute(0, 2, 1).contiguous().view(B, -1)                                                   # :292
