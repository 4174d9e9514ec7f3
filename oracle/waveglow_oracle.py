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


def _w(sd, name, dt):
    return conv_weight(sd, name).to(dt)


def n_remaining(k):
    """Channels flow k's coupling acts on: the early outputs of flows 4 and 8 leave the later flows fewer."""
    return N_GROUP - N_EARLY_SIZE * (k // N_EARLY_EVERY)


def upsample_unfold(sd, mel):
    """mel (B, 80, T) -> the conditioning (B, 640, 32 T) in mel's dtype: upsample, trim, group (glow.py:252-258)."""
    dt, B = mel.dtype, mel.shape[0]
    spect = F.conv_transpose1d(mel, sd["upsample.weight"].to(dt), sd["upsample.bias"].to(dt), stride=256)     # :252
    spect = spect[:, :, :-(1024 - 256)]                                                                      # :254-255
    spect = spect.unfold(2, N_GROUP, N_GROUP).permute(0, 2, 1, 3)                                            # :257
    return spect.contiguous().view(B, spect.size(1), -1).permute(0, 2, 1)                                     # :258


def start(sd, k, aud):
    """h (B, 256, L) of flow k's WN from the first half of aud's channels (glow.py:155)."""
    p, a0 = "WN.%d.start." % k, aud[:, :aud.size(1) // 2]
    return F.conv1d(a0, _w(sd, p, aud.dtype), sd[p + "bias"].to(aud.dtype))


def cond_layer(sd, k, spect):
    """The conditioning of all 8 layers of flow k's WN, (B, 4096, L) (glow.py:159)."""
    p = "WN.%d.cond_layer." % k
    return F.conv1d(spect, _w(sd, p, spect.dtype), sd[p + "bias"].to(spect.dtype))


def gate(sd, k, l, h, spect, cond=None):
    """acts (B, 256, L) of layer l of flow k's WN (glow.py:161-166, 34-40).  `cond` is cond_layer(sd, k, spect) when the
    caller has it; without it only layer l's 512 rows of the conditioning are computed, from spect."""
    dt, p, d = h.dtype, "WN.%d.in_layers.%d." % (k, l), 2 ** l
    x = F.conv1d(h, _w(sd, p, dt), sd[p + "bias"].to(dt), dilation=d, padding=d)
    rows = slice(l * 2 * N_CH, (l + 1) * 2 * N_CH)
    if cond is None:
        c = "WN.%d.cond_layer." % k
        x = x + F.conv1d(spect, _w(sd, c, dt)[rows], sd[c + "bias"].to(dt)[rows])
    else:
        x = x + cond[:, rows, :]
    return torch.tanh(x[:, :N_CH]) * torch.sigmoid(x[:, N_CH:])


def res_skip(sd, k, l, acts, h, skip):
    """(h', skip') after layer l of flow k's WN (glow.py:168-173); the last layer has no residual half."""
    p = "WN.%d.res_skip_layers.%d." % (k, l)
    rs = F.conv1d(acts, _w(sd, p, acts.dtype), sd[p + "bias"].to(acts.dtype))
    if l < N_LAYERS - 1:
        return h + rs[:, :N_CH], skip + rs[:, N_CH:]
    return h, skip + rs


def flow_tail(sd, k, aud, skip, z, sigma):
    """aud after flow k: end, the affine coupling, the inverse 1x1 convolution and, after flows 8 and 4, the early
    noise in front (glow.py:175, 278-290).  z (B, 8, L) is in draw order."""
    dt, p = aud.dtype, "WN.%d.end." % k
    n_half = aud.size(1) // 2
    a0, a1 = aud[:, :n_half], aud[:, n_half:]
    out = F.conv1d(skip, sd[p + "weight"].to(dt), sd[p + "bias"].to(dt))                                     # :175
    s, b = out[:, n_half:], out[:, :n_half]
    a1 = (a1 - b) / torch.exp(s)                                                                             # :280
    aud = torch.cat([a0, a1], 1)
    W = sd["convinv.%d.conv.weight" % k].squeeze()
    Winv = W.double().inverse() if dt == torch.float64 else W.float().inverse()                             # :91
    aud = F.conv1d(aud, Winv.to(dt)[..., None])                                                              # :96
    if k % N_EARLY_EVERY == 0 and k > 0:                                                                     # :285-290
        zc = aud.size(1)
        aud = torch.cat((sigma * z[:, zc:zc + N_EARLY_SIZE], aud), 1)
    return aud


def infer(sd, spect, sigma, z, dtype=torch.float64):
    """spect (B, 80, T) -> audio (B, 256 T) in `dtype`, on spect's device."""
    dev = spect.device
    sd = {k: v.to(dev) for k, v in sd.items()}
    B = spect.shape[0]
    spect = upsample_unfold(sd, spect.to(dtype))
    L = spect.shape[2]
    z = z.to(device=dev, dtype=dtype)
    assert tuple(z.shape) == (B, N_GROUP, L), (tuple(z.shape), (B, N_GROUP, L))
    audio = sigma * z[:, :n_remaining(N_FLOWS - 1)]                                                          # :260-269
    for k in reversed(range(N_FLOWS)):                                                                       # :271
        h = start(sd, k, audio)
        skip = torch.zeros_like(h)                                                                           # :156
        cond = cond_layer(sd, k, spect)
        for l in range(N_LAYERS):
            acts = gate(sd, k, l, h, spect, cond)
            h, skip = res_skip(sd, k, l, acts, h, skip)
        audio = flow_tail(sd, k, audio, skip, z, sigma)
    return audio.permute(0, 2, 1).contiguous().view(B, -1)                                                   # :292
