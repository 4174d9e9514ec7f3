"""WaveGlow configurations beyond the published one: seeded weights for any of them, the reference fixture cases
(tools/make_golden.py waveglow_configs), and the SHA-256 digests that pin the published model's outputs
(tests/golden/waveglow_published_sha256.json)."""
import math

import torch

from tests.waveglow_common import CONFIG, mel_input, noise


def config(channels, layers, flows, early_every=4, early_size=2):
    return dict(CONFIG, n_flows=flows, n_early_every=early_every, n_early_size=early_size,
                WN_config=dict(n_layers=layers, n_channels=channels, kernel_size=3))


def name_of(cfg):
    w = cfg["WN_config"]
    return "c%d_l%d_f%d_e%d_s%d" % (w["n_channels"], w["n_layers"], cfg["n_flows"], cfg["n_early_every"],
                                    cfg["n_early_size"])


# The configurations the GPU tests run (each against the fp64 oracle); the first is the common wide retrain.
GPU_CONFIGS = [config(512, 8, 12), config(128, 4, 6), config(384, 10, 12), config(256, 8, 9, 3, 2)]

# Reference fixtures: (config, B, T_mel, sigma, weight seed, mel seed, noise seed).  Short mels keep the reference's
# CPU run quick; the 512-channel one and the early schedules (every flow outputs 2 channels; one 4-channel output)
# are the shapes the engine did not run before.
FIXTURE_CASES = [
    (config(512, 8, 12), 1, 6, 0.666, 11, 51, 52),
    (config(128, 4, 6, 2, 2), 2, 5, 0.666, 12, 53, 54),
    (config(384, 10, 12), 1, 4, 0.5, 13, 55, 56),
    (config(256, 8, 9, 3, 2), 1, 5, 0.666, 14, 57, 58),
    (config(128, 3, 4, 1, 2), 2, 6, 1.0, 15, 59, 60),
    (config(256, 2, 3, 2, 4), 1, 7, 0.666, 16, 61, 62),
]


def state_dict_for(cfg, seed):
    """Seeded fp32 weights of WaveGlow(**cfg), drawn as tests/waveglow_common.synth_state_dict draws the published
    ones: non-zero ``end``, weight_g off ||v||, orthonormal convinv with determinant +1."""
    import tacotron2_b200 as t2
    shapes = [(n, tuple(v.shape)) for n, v in t2.WaveGlow(**cfg).state_dict().items()]
    g = torch.Generator().manual_seed(seed)
    u = lambda shape, b: (torch.rand(shape, generator=g) * 2 - 1) * b          # noqa: E731
    sd = {}
    for name, shape in shapes:
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
    for name, shape in shapes:
        if name.endswith("weight_g"):
            v = sd[name[:-1] + "v"]
            sd[name] = v.flatten(1).norm(dim=1).view(-1, 1, 1) * (0.5 + torch.rand(shape, generator=g))
    return {n: sd[n] for n, _ in shapes}


def fixture_inputs(B, T, mseed, zseed):
    return mel_input(B, T, mseed), noise(B, T, zseed)


# ---- the published model's outputs, pinned by digest ---------------------------------------------------------------
def published_digests():
    """{case: tensor_digest} of the published configuration's outputs on the GPU: infer in both tiers (B = 1 and 3,
    seeded and with injected noise, ragged lengths), a 32-step infer_stream over a Tacotron2 stream, and
    Denoiser.forward.  The same code runs on the build that recorded the digests and on later builds."""
    import tacotron2_b200 as t2
    from tests.common import keep_mask, rand_text, tensor_digest
    from tests.test_gpu_streaming import make_model, set_decoder, weights
    from tests.waveglow_common import synth_state_dict

    sd = synth_state_dict(7)
    out = {}

    def vocoder(half):
        m = t2.WaveGlow(**CONFIG)
        m.load_state_dict(sd)
        m = m.cuda()
        if half:
            m = m.half()
            for k in m.convinv:
                k.float()
        return m

    for half in (False, True):
        tier = "fp16" if half else "fp32"
        m = vocoder(half)
        dt = torch.float16 if half else torch.float32
        mel1, mel3 = mel_input(1, 50, 41).cuda().to(dt), mel_input(3, 37, 43).cuda().to(dt)
        lengths = torch.tensor([37, 20, 9])
        out[tier + "/b1_seeded"] = tensor_digest(m.infer(mel1, sigma=0.666, seeds=[1234]))
        out[tier + "/b3_seeded_ragged"] = tensor_digest(m.infer(mel3, sigma=0.666, lengths=lengths,
                                                                seeds=[5, 2 ** 63 + 7, 99]))
        with t2.waveglow_noise(noise(1, 50, 42)):
            out[tier + "/b1_z"] = tensor_digest(m.infer(mel1, sigma=0.666))
        with t2.waveglow_noise(noise(3, 37, 44)):
            out[tier + "/b3_z_ragged"] = tensor_digest(m.infer(mel3, sigma=0.666, lengths=lengths))
        den = t2.Denoiser(m)
        out[tier + "/denoiser_bias"] = tensor_digest(den.bias_spec)
        y = m.infer(mel3, sigma=0.666, seeds=[1, 2, 3])
        out[tier + "/denoiser_forward"] = tensor_digest(den(y, strength=0.1))

    model = make_model("w7", weights())
    set_decoder(model, 120, 0.5)
    text, keep = rand_text(2, 23, 5), keep_mask((120, 2, 2, 256), 0.5, 6)
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        items = list(model.inference_stream(text.cuda(), chunk_steps=32))
    glow = vocoder(False)
    audio = [it["audio"] for it in glow.infer_stream(iter(items), sigma=0.666, seeds=[77, 78])]
    out["fp32/stream32_seeded"] = tensor_digest(torch.cat(audio, dim=1))
    torch.cuda.synchronize()
    return out
