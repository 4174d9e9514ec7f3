"""Denoiser on the GPU (denoiser.cu) against the reference's fixture, the fp64 oracle and its own full runs, bit for bit
where rows, windows and streams must reproduce them.

Each GEMM row of the two transforms is computed from its own operand rows in a fixed order wherever it sits in a tile,
so a row of a ragged batch, a window with its halos and a stream item all reproduce the full run's bits.  Against fp64
the split-fp16 GEMMs are held to 5e-5 of max |expected|: on an H100 they measured 2.1e-5 on the reference fixture,
2.2e-5 on the strength-0 round trip and 2.1e-5 at B=64 x 204,800.  tools/denoiser_precision.py traces that to the tensor
cores' fp32 accumulation over the long K: the exact sum of the same split operands is 1.3e-6 from fp64 (DESIGN.md 6.7)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import tacotron2_b200 as t2
from oracle import denoiser_oracle as D
from oracle import waveglow_oracle as WO
from tacotron2_b200 import _capi
from tests.common import GOLDEN_DIR, keep_mask, rand_text, rel_err, stft_inputs
from tests.test_gpu_streaming import make_model, set_decoder, stop_threshold, weights
from tests.test_gpu_waveglow_stream import mel_items, reference, sd7, vocoder

pytestmark = pytest.mark.gpu
HOP = 256


def fixture():
    return np.load(os.path.join(GOLDEN_DIR, "denoiser_b2.npz"))


_DEN = {}


def denoiser(half=False):
    key = "half" if half else "fp32"
    if key not in _DEN:
        _DEN[key] = t2.Denoiser(vocoder(half))
    return _DEN[key]


def injected(bias):
    """A denoiser whose bias_spec is replaced (the bias does not depend on anything else the tests vary)."""
    den = t2.Denoiser(vocoder())
    den.bias_spec.copy_(torch.as_tensor(bias).view(1, 513, 1).cuda())
    return den


def test_module_matches_the_reference_layout():
    g = fixture()
    den = denoiser()
    sd = den.state_dict()
    assert list(sd) == list(g["keys"])
    assert [",".join(str(x) for x in v.shape) for v in sd.values()] == list(g["shapes"])
    assert den.stft.filter_length == 1024 and den.stft.hop_length == 256 and den.stft.win_length == 1024


def test_stft_path_with_the_reference_bias():
    g = fixture()
    y = stft_inputs(int(g["seed"]), int(g["n"]))
    den = injected(g["bias_spec"])
    for s in g["strengths"]:
        got = den(y.cuda(), strength=float(s))
        ref = torch.from_numpy(g["out_%g" % s])
        o64 = D.denoise(y, torch.from_numpy(g["bias_spec"]), float(s), torch.float64)
        e_ref, e64 = rel_err(got, ref), rel_err(got, o64)
        print("strength %g: max |err| / max |expected| vs reference %.2e, vs fp64 oracle %.2e" % (s, e_ref, e64))
        assert got.shape == ref.shape and got.dtype == torch.float32
        assert e_ref <= 5e-5 and e64 <= 5e-5


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "fp16"])
def test_bias_from_the_engine(half):
    """bias_spec from the engine's WaveGlow.infer, and the audio denoised with it.  The fp32 tier is held to the
    reference's fixture at 1e-3.  The notebook's .half() form rounds the WaveGlow weights to fp16, which alone moves
    bias_spec 1.3e-3 from the fp32 reference (the fp64 oracle on the fp16-rounded weights against the fixture).  So it is
    held at 1e-3 to that oracle, and at 3e-3 to the fixture."""
    g = fixture()
    den = denoiser(half)
    y = stft_inputs(int(g["seed"]), int(g["n"])).cuda()
    fix_bias = torch.from_numpy(g["bias_spec"])
    fix_outs = [torch.from_numpy(g["out_%g" % s]) for s in g["strengths"]]
    outs = [den(y, strength=float(s)) for s in g["strengths"]]
    e_bias = rel_err(den.bias_spec, fix_bias)
    errs = [rel_err(o, r) for o, r in zip(outs, fix_outs)]
    print("%s WaveGlow vs the reference fixture: bias_spec rel err %.2e, denoised audio rel err %s" %
          ("fp16" if half else "fp32", e_bias, ["%.2e" % e for e in errs]))
    if not half:
        assert e_bias <= 1e-3 and max(errs) <= 1e-3
        return
    sd16 = {k: (v.half().double() if not k.startswith("convinv") else v.double()) for k, v in sd7().items()}
    audio = WO.infer(sd16, torch.zeros(1, 80, 88, dtype=torch.float64, device="cuda"), 0.0,
                     torch.zeros(1, 8, 88 * 32, dtype=torch.float64, device="cuda"))
    bias16 = D.bias_spec(audio)
    e16 = rel_err(den.bias_spec, bias16)
    errs16 = [rel_err(o, D.denoise(y, bias16, float(s), torch.float64)) for o, s in zip(outs, g["strengths"])]
    print("fp16 WaveGlow vs the fp64 oracle on fp16-rounded weights: bias_spec rel err %.2e, audio %s; that oracle's "
          "bias_spec vs the fixture %.2e" % (e16, ["%.2e" % e for e in errs16], rel_err(bias16, fix_bias)))
    assert e16 <= 1e-3 and max(errs16) <= 1e-3
    assert e_bias <= 3e-3 and max(errs) <= 3e-3


def test_round_trip_at_strength_zero():
    y = stft_inputs(11, 256 * 50 + 13).cuda()
    out = denoiser()(y, strength=0.0)
    err = rel_err(out[:, 0], y[:, :256 * 50])
    print("strength 0: max |out - in| / max |in| %.2e" % err)
    assert err <= 5e-5


def test_full_size_against_the_fp64_oracle():
    B, n = 64, 204800
    y = (torch.randn(B, n, generator=torch.Generator().manual_seed(12)) * 0.3).clamp(-1, 1).cuda()
    den = denoiser()
    got = den(y, strength=0.1)
    ref = D.denoise(y, den.bias_spec, 0.1, torch.float64)
    err = rel_err(got, ref)
    print("B=64 x 204800: rel err vs fp64 oracle %.2e" % err)
    assert got.shape == (B, 1, n) and err <= 5e-5


def test_fp16_input_is_converted_when_packed():
    y = stft_inputs(13, 256 * 20 + 50).half().cuda()
    den = denoiser()
    assert torch.equal(den(y, 0.1), den(y.float(), 0.1))


def test_ragged_rows_equal_their_own_calls():
    n = 256 * 40 + 100
    lengths = torch.tensor([n, 256 * 31, 256 * 17 + 5, 400, 513, 0])
    y = (torch.randn(len(lengths), n, generator=torch.Generator().manual_seed(14)) * 0.3).cuda()
    den = denoiser()
    out = den(y, strength=0.1, lengths=lengths)
    assert out.shape == (len(lengths), 1, 256 * 40)
    for b, L in enumerate(lengths.tolist()):
        k = HOP * (L // HOP)
        if L > 512:
            own = den(y[b:b + 1, :L].contiguous(), strength=0.1)
            assert torch.equal(out[b, 0, :k], own[0, 0]), b
        assert not bool(out[b, 0, k if L > 512 else 0:].any()), b
    ref = D.denoise(y, den.bias_spec, 0.1, torch.float64, lengths=lengths)
    assert rel_err(out, ref) <= 5e-5


@pytest.mark.parametrize("peak", [32767.0, 65000.0], ids=["int16_scale", "fp16_limit"])
def test_loud_audio_up_to_the_fp16_limit(peak):
    """Samples below 65504 in magnitude are supported: int16-scale audio and audio just below the limit stay finite and
    match the fp64 oracle as closely as audio in [-1, 1] does."""
    y = stft_inputs(20, 256 * 30 + 40)
    y = (y / y.abs().max() * peak).cuda()
    den = denoiser()
    out = den(y, strength=0.1)
    err = rel_err(out, D.denoise(y, den.bias_spec, 0.1, torch.float64))
    print("peak %g: finite %s, rel err vs fp64 oracle %.2e" % (peak, bool(torch.isfinite(out).all()), err))
    assert bool(torch.isfinite(out).all()) and err <= 5e-5


def test_bad_inputs_are_refused_before_any_launch():
    den = denoiser()
    L = _capi.lib()
    n0 = L.t2_kernel_launch_count()
    with pytest.raises(ValueError):
        den(torch.zeros(3, 2, 1000, device="cuda"))
    with pytest.raises(ValueError):
        den(torch.zeros(2, 512, device="cuda"))
    with pytest.raises(ValueError):
        den(torch.zeros(2, 1000, device="cuda"), lengths=torch.tensor([5]))
    with pytest.raises(TypeError):
        den(torch.zeros(2, 1000, device="cuda", dtype=torch.complex64))
    assert L.t2_kernel_launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------------
# windows against the full run
# ---------------------------------------------------------------------------------------------------------------------
def window(den, y, lengths, strength, s0, n, out0, out1, at_end, out=None):
    eng = den._engine()
    eng.ensure(den)
    x = y[:, s0:s0 + n].contiguous()
    win_len = (lengths - s0).clamp(min=0).to(torch.int32).cuda()
    B = y.shape[0]
    if out is None:
        out = torch.empty(B, HOP * (out1 - out0), device="cuda")
    a = eng.args(den, x, win_len, strength, out)
    w = _capi.T2DenoiserWindowArgs()
    w.dn, w.s0, w.out0, w.out1, w.at_end = a, s0, out0, out1, int(at_end)
    _capi.check(_capi.lib().t2_denoiser_run_window(eng.handle, C.byref(w), eng.stream()))
    torch.cuda.synchronize()
    return out


N_SEQ = 256 * 60 + 37
WINDOWS = [                                  # (s0, n, out0, out1, at_end) over an N_SEQ-sample sequence
    (0, 256 * 20, 0, 17, False),             # start: no left halo needed
    (0, 256 * 20, 5, 9, False),
    (256 * 10, 256 * 20, 3, 17, False),      # interior, exactly the halos
    (256 * 7, 256 * 30 + 11, 8, 20, False),
    (256 * 40, N_SEQ - 256 * 40, 3, 20, True),   # end
    (256 * 50, N_SEQ - 256 * 50, 3, 10, True),
    (0, N_SEQ, 0, 60, True),                 # the whole sequence
    (0, N_SEQ, 31, 32, True),
]


def test_windows_equal_the_full_run():
    lengths = torch.tensor([N_SEQ, N_SEQ - 300, 700])
    y = (torch.randn(3, N_SEQ, generator=torch.Generator().manual_seed(15)) * 0.3).cuda()
    den = denoiser()
    full = den(y, strength=0.1, lengths=lengths)[:, 0]
    for s0, n, out0, out1, at_end in WINDOWS:
        got = window(den, y, lengths, 0.1, s0, n, out0, out1, at_end)
        ref = full[:, s0 + HOP * out0:s0 + HOP * out1]
        assert got.shape == ref.shape
        assert torch.equal(got, ref), ((s0, n, out0, out1), float((got - ref).abs().max()))


def test_too_narrow_windows_are_refused_before_any_launch():
    lengths = torch.tensor([N_SEQ])
    y = torch.randn(1, N_SEQ, generator=torch.Generator().manual_seed(16)).cuda()
    den = denoiser()
    window(den, y, lengths, 0.1, 256 * 10, 256 * 20, 3, 17, False)        # exactly the halos: accepted
    L = _capi.lib()
    n0 = L.t2_kernel_launch_count()
    with pytest.raises(_capi.T2Error, match="left halo is 3 blocks"):
        window(den, y, lengths, 0.1, 256 * 10, 256 * 20, 2, 17, False)
    with pytest.raises(_capi.T2Error, match="right halo is 3 blocks"):
        window(den, y, lengths, 0.1, 256 * 10, 256 * 20, 3, 18, False)
    with pytest.raises(_capi.T2Error, match="right halo is 3 blocks"):
        window(den, y, lengths, 0.1, 0, 256 * 20, 0, 20, False)
    with pytest.raises(_capi.T2Error, match="multiple of 256"):
        window(den, y, lengths, 0.1, 100, 256 * 20, 3, 17, False)
    misaligned = torch.empty(HOP * 14 + 1, device="cuda")[1:].view(1, HOP * 14)
    with pytest.raises(_capi.T2Error, match="16-byte aligned"):
        window(den, y, lengths, 0.1, 256 * 10, 256 * 20, 3, 17, False, out=misaligned)
    assert L.t2_kernel_launch_count() == n0


@pytest.mark.parametrize("windowed", [False, True], ids=["run", "run_window"])
def test_stays_inside_exact_size_buffers(windowed):
    """Workspace and output of exactly the reported size, 256 bytes past a 512-byte boundary, between 64 KiB canaries."""
    canary = 64 * 1024
    B, n = 2, 256 * 30 + 70
    lengths = torch.tensor([n, 256 * 21 + 9])
    y = torch.randn(B, n, generator=torch.Generator().manual_seed(17)).cuda()
    den = denoiser()
    s0, nw, out0, out1, at_end = (256 * 5, 256 * 20, 3, 17, False) if windowed else (0, n, 0, n // HOP, True)
    ref = window(den, y, lengths, 0.2, s0, nw, out0, out1, at_end)
    gen = torch.Generator(device="cuda")

    def placed(nbytes):
        raw = torch.randint(0, 256, (2 * canary + 256 + nbytes,), generator=gen.manual_seed(nbytes), dtype=torch.uint8,
                            device="cuda")
        assert raw.data_ptr() % 512 == 0
        return raw, raw.clone(), raw[canary + 256:canary + 256 + nbytes]

    L = _capi.lib()
    eng = den._engine()
    n_ws = int(L.t2_denoiser_workspace_bytes(eng.handle, B, nw))
    n_out = B * HOP * (out1 - out0) * 4
    ws_raw, ws_copy, ws = placed(n_ws)
    o_raw, o_copy, o = placed(n_out)
    x = y[:, s0:s0 + nw].contiguous()
    win_len = (lengths - s0).clamp(min=0).to(torch.int32).cuda()
    a = _capi.T2DenoiserArgs()
    a.audio, a.B, a.n, a.lengths, a.io_half = x.data_ptr(), B, nw, win_len.data_ptr(), 0
    bias = den.bias_spec.contiguous()
    a.bias, a.strength, a.out, a.ws, a.ws_bytes = bias.data_ptr(), 0.2, o.data_ptr(), ws.data_ptr(), n_ws
    if windowed:
        w = _capi.T2DenoiserWindowArgs()
        w.dn, w.s0, w.out0, w.out1, w.at_end = a, s0, out0, out1, int(at_end)
        _capi.check(L.t2_denoiser_run_window(eng.handle, C.byref(w), eng.stream()))
    else:
        _capi.check(L.t2_denoiser_run(eng.handle, C.byref(a), eng.stream()))
    torch.cuda.synchronize()
    for raw, copy, nb in ((ws_raw, ws_copy, n_ws), (o_raw, o_copy, n_out)):
        lo = canary + 256
        assert torch.equal(raw[:lo], copy[:lo]) and torch.equal(raw[lo + nb:], copy[lo + nb:]), nb
    assert torch.equal(o.view(torch.float32).view(B, -1), ref)


def test_invalidate_weights_refreshes_the_denoiser(monkeypatch):
    """tacotron2_b200.invalidate_weights() makes the Denoiser re-pack its bases on its next call, as it does every other
    engine; the output keeps its bits."""
    den = t2.Denoiser(vocoder())
    y = stft_inputs(22, 256 * 16 + 30).cuda()
    before = den(y, strength=0.1)
    L, refreshed = _capi.lib(), []
    real = L.t2_denoiser_refresh

    def refresh(*args):
        refreshed.append(args[0])
        return real(*args)
    monkeypatch.setattr(L, "t2_denoiser_refresh", refresh)
    again = den(y, strength=0.1)
    assert refreshed == []                       # same bases, same key: nothing to re-pack
    t2.invalidate_weights()
    after = den(y, strength=0.1)
    assert len(refreshed) == 1
    assert torch.equal(again, before) and torch.equal(after, before)


def test_mode_normal_builds_and_denoises():
    torch.manual_seed(18)
    den = t2.Denoiser(vocoder(), mode='normal')
    assert den.bias_spec.shape == (1, 513, 1) and bool(torch.isfinite(den.bias_spec).all())
    y = stft_inputs(19, 256 * 12).cuda()
    out = den(y, strength=0.05)
    assert out.shape == (2, 1, 256 * 12) and bool(torch.isfinite(out).all())
    with pytest.raises(Exception, match="not supported"):
        t2.Denoiser(vocoder(), mode='uniform')


# ---------------------------------------------------------------------------------------------------------------------
# Denoiser.stream(WaveGlow.infer_stream(Tacotron2.inference_stream(...))) against the unstreamed chain
# ---------------------------------------------------------------------------------------------------------------------
def expected_blocks(audio_items):
    out, d0 = [], 0
    for it in audio_items:
        held, fin = it["samples"][1] // HOP, it["finished"]
        d1 = held if fin else max(d0, held - 3)
        if d1 > d0 or fin:
            out.append((d0, d1))
        d0 = d1
    return out


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "fp16"])
def test_stream_equals_the_unstreamed_chain(half):
    """Rows stop at different steps and one never stops (the fp32 model's lengths; the .half() model, under the same
    threshold, gives its own)."""
    B, T, S, strength = 3, 33, 230, 0.1
    text, keep = rand_text(B, T, 9), keep_mask((S, 2, B, 256), 0.5, 10)
    model = make_model("w7", weights())
    thr = stop_threshold(model, text, keep, S, lambda L: bool((L == S).any()) and int(L.min()) < S - 5)
    if half:
        model = t2.Tacotron2(t2.create_hparams())
        model.load_state_dict(weights())
        model = model.cuda().eval().half()
    set_decoder(model, S, thr)
    glow = vocoder(half)
    den = t2.Denoiser(glow)
    audio, lengths = reference(model, glow, text, keep, None, None, 21)
    ref = den(audio, strength, lengths=HOP * lengths)[:, 0]
    print("lengths %s" % lengths.tolist())
    for chunk in (8, 32, 128):
        mels = mel_items(model, text, keep, chunk)
        torch.manual_seed(21)
        audio_items = list(glow.infer_stream(iter(mels), sigma=0.666))
        items = list(den.stream(iter(audio_items), strength))
        assert [tuple(s // HOP for s in it["samples"]) for it in items] == expected_blocks(audio_items)
        assert [it["finished"] for it in items] == [False] * (len(items) - 1) + [True]
        got = torch.cat([it["audio"] for it in items], dim=1)
        assert got.shape == ref.shape and got.dtype == torch.float32
        assert torch.equal(got, ref), (chunk, float((got - ref).abs().max()))
        assert torch.equal(items[-1]["mel_lengths"], lengths.to(items[-1]["mel_lengths"].device))
        print("chunk %d: %d audio items -> %d denoised items" % (chunk, len(audio_items), len(items)))
