"""WaveGlow.infer (waveglow/glow.py:251-293) in plain torch for any configuration: every shape -- flows, WN layers and
width, the early-output schedule -- is read from the state dict.

The stages that do not depend on the shape (the weight-norm fold, upsample / trim / unfold, start, cond_layer) are those
of oracle/waveglow_oracle.py, which states the published configuration; the gate, res/skip, the flow tail and the loop
over flows are restated here without its constants.  Dtype-generic as that oracle is: ``dtype=torch.float64`` is the
truth, ``torch.float16`` rounds where the reference's half path does.  ``z`` (B, 8, L) holds the draws in draw order:
the last flow's channels, then the early blocks from the last early flow down."""
import torch
import torch.nn.functional as F

from oracle.waveglow_oracle import N_GROUP, _w, cond_layer, start, upsample_unfold  # noqa: F401


def shape(sd):
    """dict(flows, layers, channels, n_rem=[channels flow k's coupling acts on]) of a WaveGlow state dict."""
    flows = sum(1 for k in sd if k.startswith("convinv.") and k.endswith(".conv.weight"))
    layers = sum(1 for k in sd if k.startswith("WN.0.in_layers.") and k.endswith(".bias"))
    return dict(flows=flows, layers=layers, channels=sd["WN.0.start.bias"].shape[0],
                n_rem=[sd["convinv.%d.conv.weight" % k].shape[0] for k in range(flows)])


def n_remaining(k, sd=None, n_early_every=4, n_early_size=2):
    """Channels flow k's coupling acts on: from the state dict when given, else from the early schedule (default: the
    published one)."""
    if sd is not None:
        return sd["convinv.%d.conv.weight" % k].shape[0]
    return N_GROUP - n_early_size * (k // n_early_every)


def gate(sd, k, l, h, cond):
    """acts (B, C, L) of layer l of flow k's WN (glow.py:161-166, 34-40), C = h's channels; cond = cond_layer(...)."""
    dt, p, d, n_ch = h.dtype, "WN.%d.in_layers.%d." % (k, l), 2 ** l, h.shape[1]
    x = F.conv1d(h, _w(sd, p, dt), sd[p + "bias"].to(dt), dilation=d, padding=d)
    x = x + cond[:, l * 2 * n_ch:(l + 1) * 2 * n_ch, :]
    return torch.tanh(x[:, :n_ch]) * torch.sigmoid(x[:, n_ch:])


def res_skip(sd, k, l, acts, h, skip):
    """(h', skip') after layer l of flow k's WN (glow.py:168-173); the last layer has no residual half."""
    p, n_ch = "WN.%d.res_skip_layers.%d." % (k, l), h.shape[1]
    rs = F.conv1d(acts, _w(sd, p, acts.dtype), sd[p + "bias"].to(acts.dtype))
    if rs.shape[1] == 2 * n_ch:
        return h + rs[:, :n_ch], skip + rs[:, n_ch:]
    return h, skip + rs


def flow_tail(sd, k, aud, skip, z, sigma):
    """aud after flow k: end, the affine coupling, the inverse 1x1 convolution and, where flow k - 1 acts on more
    channels, the early noise in front (glow.py:175, 278-290)."""
    dt, p = aud.dtype, "WN.%d.end." % k
    n_half = aud.size(1) // 2
    a0, a1 = aud[:, :n_half], aud[:, n_half:]
    out = F.conv1d(skip, sd[p + "weight"].to(dt), sd[p + "bias"].to(dt))                                     # :175
    s, b = out[:, n_half:], out[:, :n_half]
    a1 = (a1 - b) / torch.exp(s)                                                                             # :280
    aud = torch.cat([a0, a1], 1)
    W = sd["convinv.%d.conv.weight" % k].squeeze(-1)
    Winv = W.double().inverse() if dt == torch.float64 else W.float().inverse()                             # :91
    aud = F.conv1d(aud, Winv.to(dt)[..., None])                                                              # :96
    early = n_remaining(k - 1, sd) - aud.size(1) if k > 0 else 0
    if early > 0:                                                                                            # :285-290
        zc = aud.size(1)
        aud = torch.cat((sigma * z[:, zc:zc + early], aud), 1)
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
    shp = shape(sd)
    audio = sigma * z[:, :shp["n_rem"][-1]]                                                                  # :260-269
    for k in reversed(range(shp["flows"])):                                                                  # :271
        h = start(sd, k, audio)
        skip = torch.zeros_like(h)                                                                           # :156
        cond = cond_layer(sd, k, spect)
        for l in range(shp["layers"]):
            acts = gate(sd, k, l, h, cond)
            h, skip = res_skip(sd, k, l, acts, h, skip)
        audio = flow_tail(sd, k, audio, skip, z, sigma)
    return audio.permute(0, 2, 1).contiguous().view(B, -1)                                                   # :292
