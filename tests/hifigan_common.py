"""Shared inputs of the HiFi-GAN tests: synthetic weights that keep the signal alive through the generator, and mels."""
import torch

from tacotron2_b200.hifigan import CONFIGS, Generator

# weight_g per convolution so that each keeps roughly unit gain: v ~ N(0, 1) rows have norm g, so a Conv1d row of
# unit-variance inputs gives variance ~ g^2; lrelu halves it, so the first conv of a pair gets sqrt(2).  A
# ConvTranspose1d output reads 2 of its 2u taps per input channel, cin = 2 cout: variance ~ 2 g^2 / u.  The second conv
# of a residual pair is damped so that the residual sums do not grow through the stages (the tanh would saturate).
GAIN_PRE, GAIN_FIRST, GAIN_SECOND, GAIN_POST = 0.2, 1.4, 0.35, 0.6


def synth_state_dict(model, seed, removed=False):
    """A state_dict for `model`'s tree: v ~ N(0, 1), g from the gains above, biases ~ N(0, 0.05)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, v in model.state_dict().items():
        if k.endswith(".bias"):
            sd[k] = torch.randn(v.shape, generator=g, dtype=torch.float32) * 0.05
        elif k.endswith(".weight_v") or k.endswith(".weight"):
            sd[k] = torch.randn(v.shape, generator=g, dtype=torch.float32)
    for k in list(sd):
        if not k.endswith(".weight_v"):
            continue
        p = k[:-len(".weight_v")]
        if p == "conv_pre":
            gain = GAIN_PRE
        elif p == "conv_post":
            gain = GAIN_POST
        elif p.startswith("ups."):
            u = sd[k].shape[2] // 2
            gain = 1.4 * (u / 2) ** 0.5
        elif ".convs2." in p or (".convs." in p):
            gain = GAIN_SECOND if ".convs2." in p else 0.6
        else:
            gain = GAIN_FIRST
        sd[p + ".weight_g"] = torch.full(model.state_dict()[p + ".weight_g"].shape, gain)
    return {k: sd[k] for k in model.state_dict()}


def mel_input(B, T, seed):
    """Log-mel-like input: smooth in time around -5, within the range Tacotron2's mels take."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 80, T, generator=g)
    x = torch.nn.functional.avg_pool1d(x, 3, 1, 1) * 2.0 - 5.0
    return x.contiguous()


def model(name, seed=3):
    G = Generator(CONFIGS[name])
    G.load_state_dict(synth_state_dict(G, seed))
    return G
