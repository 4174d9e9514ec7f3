"""WaveGlow.infer for configurations beyond the published one, on the H100: against the fp64 oracle and the reference's
fixtures, each ragged row against its own B = 1 call, infer_stream against infer, the Denoiser, exact-size buffers, the
refusals, and the published model's outputs against the digests recorded before the engine was generalised.

Bars: the fp32-grade tier within 5e-5 of max |expected| (E64_BAR), the fp16 tier within twice the error of the oracle
that rounds where the reference's half path does, the reference's fixtures within 1e-4."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tacotron2_b200.glow import HOP
from tests import waveglow_config_oracle as WO
from tests.common import GOLDEN_DIR, keep_mask, rand_text, rel_err
from tests.test_gpu_streaming import make_model, set_decoder, weights
from tests.waveglow_common import mel_input, noise
from tests.waveglow_configs import FIXTURE_CASES, GPU_CONFIGS, config, name_of, published_digests, state_dict_for

pytestmark = pytest.mark.gpu

E64_BAR = 5e-5
REF_BAR = 1e-4
IDS = [name_of(c) for c in GPU_CONFIGS]
_SD = {}


def sd_of(cfg, seed=21):
    key = (name_of(cfg), seed)
    if key not in _SD:
        _SD[key] = state_dict_for(cfg, seed)
    return _SD[key]


def vocoder(cfg, half=False, seed=21):
    m = t2.WaveGlow(**cfg)
    m.load_state_dict(sd_of(cfg, seed))
    m = m.cuda()
    if half:                                   # the notebook's form: .half(), then convinv back to fp32
        m = m.half()
        for k in m.convinv:
            k.float()
    return m


def run(m, mel, sigma, z=None, **kw):
    with t2.waveglow_noise(z):
        out = m.infer(mel.cuda(), sigma=sigma, **kw)
    torch.cuda.synchronize()
    return out


def max_rel(got, want):
    return float((got.double() - want.double()).abs().max() / want.double().abs().max())


@pytest.mark.parametrize("cfg", GPU_CONFIGS, ids=IDS)
def test_fp32_tier_against_the_fp64_oracle(cfg):
    B, T, sigma = 2, 24, 0.666
    mel, z = mel_input(B, T, 31), noise(B, T, 32)
    out = run(vocoder(cfg), mel, sigma, z)
    assert out.dtype == torch.float32 and out.shape == (B, HOP * T)
    truth = WO.infer(sd_of(cfg), mel.cuda().double(), sigma, z.cuda().double())
    e = max_rel(out, truth)
    print("%s fp32 tier: max |engine - fp64| / max |fp64| = %.2e" % (name_of(cfg), e))
    assert e <= E64_BAR


@pytest.mark.parametrize("cfg", GPU_CONFIGS, ids=IDS)
def test_fp16_tier_within_the_fp16_rounding_yardstick(cfg):
    B, T, sigma = 2, 24, 0.666
    mel, z = mel_input(B, T, 33), noise(B, T, 34)
    out = run(vocoder(cfg, half=True), mel.half(), sigma, z)
    assert out.dtype == torch.float16
    sd = sd_of(cfg)
    sd16 = {k: (v.half().double() if not k.startswith("convinv") else v.double()) for k, v in sd.items()}
    truth = WO.infer(sd16, mel.half().cuda().double(), sigma, z.half().cuda().double())
    emul = WO.infer({k: (v.half() if not k.startswith("convinv") else v) for k, v in sd.items()},
                    mel.half().cuda(), sigma, z.half().cuda(), torch.float16)
    e_eng, e_ora = rel_err(out, truth), rel_err(emul, truth)
    print("%s fp16 tier: engine vs fp64 %.2e, fp16-emulating oracle vs fp64 %.2e (ratio %.2f)" %
          (name_of(cfg), e_eng, e_ora, e_eng / e_ora))
    assert e_eng <= 2.0 * e_ora


@pytest.mark.parametrize("case", FIXTURE_CASES, ids=[name_of(c[0]) for c in FIXTURE_CASES])
def test_reference_fixtures(case):
    cfg, B, T, sigma, wseed, mseed, zseed = case
    g = np.load(os.path.join(GOLDEN_DIR, "waveglow_configs.npz"))
    name = name_of(cfg)
    mel, z = torch.from_numpy(g[name + "/mel"]), torch.from_numpy(g[name + "/z"])
    out = run(vocoder(cfg, seed=wseed), mel, float(g[name + "/sigma"]), z)
    e = max_rel(out.cpu(), torch.from_numpy(g[name + "/audio"]))
    print("%s: max |engine - reference| / max |reference| = %.2e" % (name, e))
    assert e <= REF_BAR


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "fp16"])
@pytest.mark.parametrize("cfg", GPU_CONFIGS, ids=IDS)
def test_ragged_rows_equal_their_own_calls(cfg, half):
    lengths = [40, 23, 7]
    B, T, sigma = len(lengths), max(lengths), 0.666
    m = vocoder(cfg, half)
    dt = torch.float16 if half else torch.float32
    mel, z = mel_input(B, T, 35).to(dt), noise(B, T, 36)
    seeds = [11, 2 ** 64 - 5, 12345]
    rag_z = run(m, mel, sigma, z, lengths=torch.tensor(lengths))
    rag_s = run(m, mel, sigma, lengths=torch.tensor(lengths), seeds=seeds)
    rag_s2 = run(m, mel[[2, 0]], sigma, lengths=torch.tensor([lengths[2], lengths[0]]), seeds=[seeds[2], seeds[0]])
    for b, L in enumerate(lengths):
        own_z = run(m, mel[b:b + 1, :, :L], sigma, z[b:b + 1, :, :32 * L].contiguous())
        own_s = run(m, mel[b:b + 1, :, :L], sigma, seeds=[seeds[b]])
        assert torch.equal(rag_z[b, :HOP * L], own_z[0]), b
        assert torch.equal(rag_s[b, :HOP * L], own_s[0]), b
        assert not bool(rag_z[b, HOP * L:].any()) and not bool(rag_s[b, HOP * L:].any())
    assert torch.equal(rag_s2[0], rag_s[2]) and torch.equal(rag_s2[1], rag_s[0])


@pytest.mark.parametrize("cfg", GPU_CONFIGS, ids=IDS)
def test_stream_equals_infer(cfg):
    B, T_text, S = 2, 31, 480
    model = make_model("w7", weights())
    set_decoder(model, S, 0.5)
    text, keep = rand_text(B, T_text, 5), keep_mask((S, 2, B, 256), 0.5, 6)
    glow = vocoder(cfg)
    left, right = glow.window_halo()
    reach = cfg["n_flows"] * (2 ** cfg["WN_config"]["n_layers"] - 1)
    assert (left, right) == (-(-reach // 32) + 3, -(-reach // 32))
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        post = model.inference(text.cuda())[1].clone()
    lengths = model.mel_lengths.clone()
    seeds = [3, 4]
    ref = run(glow, post, 0.666, lengths=lengths, seeds=seeds)
    z = noise(B, S, 37)
    ref_z = run(glow, post, 0.666, z[:, :, :32 * post.shape[2]].contiguous(), lengths=lengths)
    print("%s: halos (%d, %d), mel lengths %s" % (name_of(cfg), left, right, lengths.tolist()))
    for chunk in (32, 128):
        with torch.no_grad(), t2.dropout_masks(prenet=keep):
            mels = list(model.inference_stream(text.cuda(), chunk_steps=chunk))
        items = list(glow.infer_stream(iter(mels), sigma=0.666, seeds=seeds))
        got = torch.cat([it["audio"] for it in items], dim=1)
        assert torch.equal(got, ref), (chunk, float((got - ref).abs().max()))
        a0 = 0
        for it, (s0, s1) in zip(items, [it["samples"] for it in items]):
            assert s0 == a0
            a0 = s1
        with t2.waveglow_noise(z):
            items = list(glow.infer_stream(iter(mels), sigma=0.666))
        assert torch.equal(torch.cat([it["audio"] for it in items], dim=1), ref_z), chunk


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "fp16"])
@pytest.mark.parametrize("cfg", GPU_CONFIGS, ids=IDS)
def test_denoiser_runs(cfg, half):
    m = vocoder(cfg, half)
    den = t2.Denoiser(m)
    assert den.bias_spec.shape == (1, 513, 1) and bool(torch.isfinite(den.bias_spec).all())
    y = run(m, mel_input(2, 20, 38).to(torch.float16 if half else torch.float32), 0.666, seeds=[1, 2])
    out = den(y, strength=0.1)
    torch.cuda.synchronize()
    assert out.shape == (2, 1, y.shape[1]) and bool(torch.isfinite(out.float()).all())


@pytest.mark.parametrize("cfg", GPU_CONFIGS, ids=IDS)
def test_infer_stays_inside_exact_size_buffers(cfg):
    """Workspace and audio of exactly the reported size, 256 bytes past a 512-byte boundary, between 64 KiB canaries."""
    canary = 64 * 1024
    B, T = 2, 30
    m = vocoder(cfg)
    mel, lengths = mel_input(B, T, 39).cuda(), torch.tensor([30, 17], dtype=torch.int32).cuda()
    ref = run(m, mel, 0.7, lengths=lengths.cpu(), seeds=[5, 6])
    seeds = torch.tensor([5, 6], dtype=torch.int64).cuda()
    gen = torch.Generator(device="cuda")

    def placed(n):
        raw = torch.randint(0, 256, (2 * canary + 256 + n,), generator=gen.manual_seed(n), dtype=torch.uint8, device="cuda")
        assert raw.data_ptr() % 512 == 0
        return raw, raw.clone(), raw[canary + 256:canary + 256 + n]

    L = _capi.lib()
    n_ws = int(L.t2_waveglow_workspace_bytes(m._t2.handle, B, T))
    n_audio = B * HOP * T * 4
    ws_raw, ws_copy, ws = placed(n_ws)
    au_raw, au_copy, au = placed(n_audio)
    a = _capi.T2WaveGlowArgs(mel.data_ptr(), B, T, lengths.data_ptr(), 0, 0.7, None, 0, au.data_ptr(), ws.data_ptr(),
                             n_ws, seeds.data_ptr())
    _capi.check(L.t2_waveglow_infer(m._t2.handle, C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    for raw, copy, n in ((ws_raw, ws_copy, n_ws), (au_raw, au_copy, n_audio)):
        lo = canary + 256
        assert torch.equal(raw[:lo], copy[:lo]) and torch.equal(raw[lo + n:], copy[lo + n:]), n
    assert torch.equal(au.view(torch.float32).view(B, -1), ref)


REFUSED = [config(64, 8, 12), config(320, 8, 12), config(256, 11, 12), config(256, 8, 17),
           dict(config(256, 8, 12), WN_config=dict(n_layers=8, n_channels=256, kernel_size=5))]


@pytest.mark.parametrize("cfg", REFUSED, ids=lambda c: name_of(c) + "_k%d" % c["WN_config"]["kernel_size"])
def test_unsupported_configurations_are_refused_before_any_launch(cfg):
    m = t2.WaveGlow(**cfg).cuda()
    L = _capi.lib()
    n0 = L.t2_kernel_launch_count()
    with pytest.raises(_capi.T2Error, match="configuration"):
        m.infer(mel_input(1, 4, 0).cuda())
    assert L.t2_kernel_launch_count() == n0


def test_published_model_outputs_are_unchanged():
    """Digests of the published model's outputs (infer in both tiers, B = 1 and 3, seeded and with injected noise,
    ragged lengths; a 32-step infer_stream; the Denoiser) recorded before the engine took other configurations."""
    with open(os.path.join(GOLDEN_DIR, "waveglow_published_sha256.json")) as f:
        want = json.load(f)["digests"]
    got = published_digests()
    assert sorted(got) == sorted(want)
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, bad
