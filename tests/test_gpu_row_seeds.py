"""Per-utterance seeds: with ``seeds`` every row draws the random streams of a B = 1 call with its own seed, so a text
reproduces its mel, gate, alignments and audio bit for bit in any batch, 64-row slice, stream chunking or server slot.

* prenet keep bit of row b, its own step s, layer k, column j: ``philox_keep(seeds[b], 4 s + k, j, 0.5)``;
* WaveGlow noise of row b, channel c, group column t: ``philox_normal(seeds[b], 0, c, t)``.

At B = 1 these are the unseeded formulas, so ``seeds=[s]`` equals the unseeded call whose drawn seed was s."""
import ctypes

import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi, _engine
from tacotron2_b200 import glow as glow_mod
from tests import philox_ref as P
from tests.common import rand_text, synth_state_dict
from tests.waveglow_common import CONFIG, mel_input
from tests.waveglow_common import synth_state_dict as wg_state_dict

pytestmark = pytest.mark.gpu
CAP = 40
BIG = (1 << 64) - 5            # a seed whose top bit is set: the key takes all 64 bits
OUT = ("mel_outputs", "mel_outputs_postnet", "gate_outputs", "alignments")


def _model(impl=None, half=False, cap=CAP):
    # a gate this close to the threshold stops rows at different steps within the cap, and lets some run to it
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(synth_state_dict(77, gate_bias=0.09, scale=1.0, gate_sign=-4.0))
    model = model.cuda().eval()
    if half:
        model = model.half()
    model.decoder.max_decoder_steps = cap
    if impl is not None:
        model._t2_engine().impl = impl
    return model


def _run(model, text, **kw):
    with torch.no_grad():
        out = [o.clone() for o in model.inference(text.cuda(), **kw)]
    torch.cuda.synchronize()
    return out + [model.mel_lengths.clone()]


def _equal(a, b):
    bad = [i for i, (x, y) in enumerate(zip(a, b)) if not (x.shape == y.shape and torch.equal(x, y))]
    assert not bad, bad


def _seeds(n, base=1000):
    return [BIG if i == 1 else base + 7919 * i for i in range(n)]


def seeded_prenet_masks(seeds, cap):
    """dropout_masks(prenet=...) layout (cap, 2, B, 256): row b is a B = 1 mask drawn with seeds[b]."""
    return torch.stack([P.infer_prenet_masks(s, cap, 1)[:, :, 0] for s in seeds], 2).contiguous()


# ---- 1. the definition ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("impl", [_capi.IMPL_STEPWISE, _capi.IMPL_PERSISTENT])
@pytest.mark.parametrize("s", [12345, BIG])
def test_b1_seed_is_the_unseeded_call_with_that_engine_seed(impl, s, monkeypatch):
    model = _model(impl)
    text = rand_text(1, 29, 3)
    seeded = _run(model, text, seeds=[s])
    monkeypatch.setattr(_engine, "next_seed", lambda: s)
    _equal(seeded, _run(model, text))


@pytest.mark.parametrize("impl", [_capi.IMPL_STEPWISE, _capi.IMPL_PERSISTENT])
@pytest.mark.parametrize("half", [False, True], ids=["fp32", "half"])
def test_seeded_run_equals_host_rebuilt_per_row_masks(impl, half):
    """B = 67 (two 64-row slices on the persistent decoder): each row's masks rebuilt from its own seed."""
    model = _model(impl, half)
    B = 67
    text, seeds = rand_text(B, 29, 4), _seeds(B)
    seeded = _run(model, text, seeds=torch.tensor([s - (1 << 64) if s >= 1 << 63 else s for s in seeds]))
    with t2.dropout_masks(prenet=seeded_prenet_masks(seeds, CAP)):
        _equal(seeded, _run(model, text))


# ---- 2. a row of a batch equals its own B = 1 call ------------------------------------------------------------------

_batch = {}


def batch_case():
    """B = 130 (three 64-row slices), ragged texts, distinct seeds except rows 0 and 129 (same text and seed)."""
    if not _batch:
        model = _model(_capi.IMPL_PERSISTENT)
        B, T = 130, 60
        text = rand_text(B, T, 9)
        g = torch.Generator().manual_seed(9)
        lengths = torch.randint(1, T + 1, (B,), generator=g)
        lengths[0], lengths[1], lengths[64] = T, 1, T
        text[129], lengths[129] = text[0], lengths[0]
        seeds = _seeds(B)
        seeds[129] = seeds[0]
        out = _run(model, text, input_lengths=lengths, seeds=seeds)
        _batch.update(model=model, text=text, lengths=lengths, seeds=seeds, out=out)
    return _batch


def _alone(model, text, L, seed):
    return _run(model, text[None, :L], seeds=[seed])


def test_every_row_of_a_ragged_130_row_batch_equals_its_own_b1_call():
    c = batch_case()
    model, text, lengths, seeds, out = c["model"], c["text"], c["lengths"], c["seeds"], c["out"]
    mel, post, gate, align, mel_len = out
    stops = set()
    for b in range(text.shape[0]):
        L = int(lengths[b])
        one = _alone(model, text[b], L, seeds[b])
        n = one[0].shape[2]
        stops.add(int(one[4][0]))
        assert int(mel_len[b]) == int(one[4][0]), b
        assert torch.equal(mel[b, :, :n], one[0][0]), b
        assert torch.equal(post[b, :, :n], one[1][0]), b
        assert torch.equal(gate[b, :n], one[2][0]), b
        assert torch.equal(align[b, :n, :L], one[3][0]), b
    assert len(stops) > 3            # the rows stop at different steps


def test_same_text_and_seed_agree_and_other_seeds_differ():
    c = batch_case()
    mel, post, gate, align, mel_len = c["out"]
    # rows 0 and 129 run in different 64-row slices: gate and alignments past the row's length are its slice's
    n = int(mel_len[0])
    assert int(mel_len[129]) == n and torch.equal(mel[0], mel[129]) and torch.equal(post[0], post[129])
    assert torch.equal(gate[0, :n], gate[129, :n]) and torch.equal(align[0, :n], align[129, :n])
    # frame 0 is the prenet of the zero go frame whatever the mask: run to the cap so later frames are compared
    model = _model(_capi.IMPL_PERSISTENT)
    model.decoder.gate_threshold = 1.0
    L = int(c["lengths"][0])
    a = _alone(model, c["text"][0], L, c["seeds"][0])
    b = _alone(model, c["text"][0], L, c["seeds"][0] + 1)
    assert a[0].shape[2] == CAP and not torch.equal(a[0], b[0])


# ---- 3. streams ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("chunk", [1, 7, 32, 128])
def test_inference_stream_with_seeds_concatenates_to_inference(chunk):
    model = _model(_capi.IMPL_PERSISTENT)
    text = rand_text(5, 33, 5)
    lengths = torch.tensor([33, 4, 20, 33, 11])
    seeds = _seeds(5, 77)
    ref = _run(model, text, input_lengths=lengths, seeds=seeds)
    with torch.no_grad():
        items = list(model.inference_stream(text.cuda(), chunk, input_lengths=lengths, seeds=seeds))
    cat = [torch.cat([it[k] for it in items], 2 if k in ("mel_outputs", "mel_outputs_postnet") else 1)
           for k in ("mel_outputs", "mel_outputs_postnet", "gate_outputs", "alignments")]
    _equal(cat, ref[:4])
    assert torch.equal(items[-1]["mel_lengths"], ref[4])


# ---- 4. the server ---------------------------------------------------------------------------------------------------

_server = {}


def server_case():
    if not _server:
        model = _model(_capi.IMPL_PERSISTENT, cap=48)
        g = torch.Generator().manual_seed(11)
        n = 24
        lengths = [1, 150, 95, 94] + torch.randint(1, 151, (n - 4,), generator=g).tolist()
        texts = [rand_text(1, L, 300 + i)[0] for i, L in enumerate(lengths)]
        limits = [48 if i % 5 else 17 for i in range(n)]
        seeds = _seeds(n, 500)
        refs = []
        for x, lim, s in zip(texts, limits, seeds):
            model.decoder.max_decoder_steps = lim
            refs.append(_run(model, x[None], seeds=[s]))
        model.decoder.max_decoder_steps = 48
        _server.update(model=model, texts=texts, limits=limits, seeds=seeds, refs=refs)
    return _server


def _check_served(res, ref):
    mel, post, gate, align, ml = ref
    assert res["mel_length"] == int(ml[0])
    for name, o in zip(OUT, (mel, post, gate, align)):
        assert torch.equal(res[name], o), name


@pytest.mark.parametrize("slots,chunk,reverse", [(1, 7, False), (3, 1, True), (8, 7, False), (8, 32, True),
                                                 (70, 7, False)])
def test_every_seeded_request_equals_its_own_b1_inference(slots, chunk, reverse):
    c = server_case()
    n = 8 if slots == 1 else len(c["texts"])
    order = list(reversed(range(n))) if reverse else list(range(n))
    server = c["model"].inference_server(slots=slots, max_text_len=150, chunk_steps=chunk)
    ids = {server.submit(c["texts"][i], c["limits"][i], seed=c["seeds"][i]): i for i in order}
    with torch.no_grad():
        out = {ids[r["id"]]: r for r in server.run()}
    assert sorted(out) == sorted(order)
    for i in order:
        assert out[i]["seed"] == c["seeds"][i]
        _check_served(out[i], c["refs"][i])


def test_late_submissions_and_readmitted_slots_start_at_step_0():
    """Requests queued while others run: each one that enters a slot mid-session (a slot whose last occupant stopped)
    draws from its own step 0."""
    c = server_case()
    server = c["model"].inference_server(slots=3, max_text_len=150, chunk_steps=5)
    ids = {server.submit(c["texts"][i], c["limits"][i], seed=c["seeds"][i]): i for i in range(3)}
    out = {}
    with torch.no_grad():
        for k in range(3, 12):
            for r in server.step():
                out[ids[r["id"]]] = r
            ids[server.submit(c["texts"][k], c["limits"][k], seed=c["seeds"][k])] = k
        for r in server.run():
            out[ids[r["id"]]] = r
    assert sorted(out) == list(range(12))
    for i in range(12):
        _check_served(out[i], c["refs"][i])


def test_inference_many_with_seeds():
    c = server_case()
    res = c["model"].inference_many(c["texts"][:6], slots=4, max_decoder_steps=c["limits"][:6], seeds=c["seeds"][:6])
    for r, ref in zip(res, c["refs"][:6]):
        _check_served(r, ref)


# ---- 5. audio --------------------------------------------------------------------------------------------------------

def _glow(half=False):
    glow = t2.WaveGlow(**CONFIG)
    glow.load_state_dict(wg_state_dict(7))
    glow = glow.cuda()
    return glow.half() if half else glow


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "fp16"])
def test_waveglow_b1_seed_is_the_unseeded_call_with_that_seed(half, monkeypatch):
    glow = _glow(half)
    mel = mel_input(1, 30, 1).cuda()
    mel = mel.half() if half else mel
    with torch.no_grad():
        seeded = glow.infer(mel, 0.666, seeds=[BIG])
        monkeypatch.setattr(glow_mod._WaveGlowEngine, "_draw_seed", lambda self: BIG)
        plain = glow.infer(mel, 0.666)
    assert torch.equal(seeded, plain)


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "fp16"])
def test_waveglow_rows_equal_their_own_b1_calls_and_the_stream(half):
    glow = _glow(half)
    B, T = 5, 48
    mel = mel_input(B, T, 2).cuda()
    mel = mel.half() if half else mel
    lengths = torch.tensor([48, 3, 30, 48, 17])
    seeds = _seeds(B, 40)
    with torch.no_grad():
        audio = glow.infer(mel, 0.7, lengths=lengths, seeds=seeds)
        for b in range(B):
            L = int(lengths[b])
            one = glow.infer(mel[b:b + 1, :, :L].contiguous(), 0.7, seeds=[seeds[b]])
            assert torch.equal(audio[b, :256 * L], one[0]), b
            assert not bool(audio[b, 256 * L:].any())
        other = glow.infer(mel[:1], 0.7, seeds=[seeds[0] + 1])
        assert not torch.equal(other[0], audio[0])


def test_waveglow_stream_with_seeds_equals_infer():
    model = _model(_capi.IMPL_PERSISTENT, cap=300)
    model.decoder.gate_threshold = 1.0                 # every row runs to the cap: long enough for several windows
    glow = _glow()
    text = rand_text(3, 20, 6)
    seeds, wseeds = _seeds(3, 10), _seeds(3, 20)
    with torch.no_grad():
        ref_mel = model.inference(text.cuda(), seeds=seeds)
        ref = glow.infer(ref_mel[1], 0.6, lengths=model.mel_lengths, seeds=wseeds)
        items = list(glow.infer_stream(model.inference_stream(text.cuda(), 16, seeds=seeds), 0.6, seeds=wseeds))
    audio = torch.cat([it["audio"] for it in items], 1)
    assert len(items) > 2 and torch.equal(audio, ref)


def test_text_to_denoised_audio_of_one_row_equals_its_solo_pipeline():
    model = _model(_capi.IMPL_PERSISTENT)
    model.decoder.gate_threshold = 1.0                 # every row runs to the cap: enough samples to denoise
    glow = _glow()
    den = t2.Denoiser(glow)
    text = rand_text(4, 30, 8)
    lengths = torch.tensor([30, 12, 25, 7])
    seeds, wseeds = _seeds(4, 3), _seeds(4, 5)
    b = 2
    with torch.no_grad():
        out = model.inference(text.cuda(), input_lengths=lengths, seeds=seeds)
        ml = model.mel_lengths.clone()
        audio = glow.infer(out[1], 0.666, lengths=ml, seeds=wseeds)
        clean = den(audio, 0.05, lengths=(ml * 256).to(torch.int32))
        L = int(lengths[b])
        one = model.inference(text[b:b + 1, :L].cuda(), seeds=[seeds[b]])
        n = int(model.mel_lengths[0])
        one_audio = glow.infer(one[1], 0.666, seeds=[wseeds[b]])
        one_clean = den(one_audio, 0.05)
    assert int(ml[b]) == n
    assert torch.equal(audio[b, :256 * n], one_audio[0])
    assert torch.equal(clean[b, :256 * n], one_clean[0])


# ---- 6. refusals -----------------------------------------------------------------------------------------------------

def _refused(fn, err):
    L = _capi.lib()
    torch.cuda.synchronize()
    before = L.t2_kernel_launch_count()
    with pytest.raises(err):
        fn()
    assert L.t2_kernel_launch_count() == before


def test_bad_seeds_are_refused_before_any_launch():
    model = _model(_capi.IMPL_PERSISTENT)
    glow = _glow()
    text = rand_text(3, 10, 1).cuda()
    mel = mel_input(2, 8, 1).cuda()
    with torch.no_grad():
        _run(model, text, seeds=[1, 2, 3])                             # handles and workspaces exist
        glow.infer(mel, seeds=[1, 2])
        _refused(lambda: model.inference(text, seeds=[1, 2]), ValueError)
        _refused(lambda: model.inference(text, seeds=torch.ones(3, 1, dtype=torch.int64)), ValueError)
        _refused(lambda: model.inference(text, seeds=torch.ones(3)), TypeError)
        _refused(lambda: model.inference(text, seeds=[1, 2, -3]), ValueError)
        _refused(lambda: next(model.inference_stream(text, 4, seeds=[1.0, 2, 3])), TypeError)
        with t2.dropout_masks(prenet=torch.ones(CAP, 2, 3, 256, dtype=torch.uint8)):
            _refused(lambda: model.inference(text, seeds=[1, 2, 3]), ValueError)
        model.train()
        _refused(lambda: model.inference(text, seeds=[1, 2, 3]), ValueError)
        model.eval()
        _refused(lambda: glow.infer(mel, seeds=[1]), ValueError)
        _refused(lambda: glow.infer(mel, seeds=torch.ones(2, dtype=torch.float64)), TypeError)
        with t2.waveglow_noise(torch.zeros(2, 8, 32 * 8)):
            _refused(lambda: glow.infer(mel, seeds=[1, 2]), ValueError)


def test_library_refuses_row_seeds_with_injected_inputs():
    """The C entry points refuse row_seeds next to prenet_keep / training / z with T2_ERR_INVALID."""
    model = _model(_capi.IMPL_PERSISTENT)
    eng = model._t2_engine()
    memory = torch.zeros(2, 10, 512, device="cuda")
    rs = torch.tensor([1, 2], device="cuda")
    with torch.no_grad():
        model.inference(rand_text(2, 10, 1).cuda())
        with pytest.raises(_capi.T2Error, match="exclude"):
            eng.decoder(memory, _capi.MODE_INFER, 4, prenet_keep=torch.ones(4, 2, 2, 256, dtype=torch.uint8),
                        row_seeds=rs)
        with pytest.raises(_capi.T2Error, match="training"):
            eng.decoder(memory, _capi.MODE_INFER, 4, training=True, row_seeds=rs)
        glow = _glow()
        ge = glow._engine()
        ge.ensure(glow)
        mel = mel_input(2, 8, 1).cuda()
        audio = torch.empty(2, 256 * 8, device="cuda")
        a = ge._args(mel, None, torch.zeros(2, 8, 256, device="cuda"), 1.0, 0, audio, rs)
        with pytest.raises(_capi.T2Error, match="exclude"):
            ge._call(_capi.lib().t2_waveglow_infer, ctypes.byref(a))
