"""Constrained synthesis: ``inference(..., attention_window=(back, front), max_decoder_steps=caps)`` keeps each row's
attention near its last peak and stops each row at its own step limit, on the persistent decoder's limited
instantiation.

1. against the fp64 oracle loop with the window mask, in eval and training mode; the window is exact on the engine's
   own alignments;
2. a window that masks nothing is the free run bit for bit, across the kernel's T_enc regimes;
3. the (0, 1) window equals the forced run of its one-hot map;
4. every row of a ragged 130-row batch with a window and per-row caps equals its own B = 1 call (fp32 / half, masks /
   seeds);
5. caps alone: the uncapped bits, the step count and the per-row warning;
6. streams and 7. the server concatenate / equal inference() with the same limits;
8. refusals, and exact-size buffers."""
import pytest
import torch

import tacotron2_b200 as t2
from oracle import tacotron2_oracle as O
from tacotron2_b200 import _capi
from tests.common import keep_mask, rand_text, rel_err, synth_state_dict
from tests.test_attention_window_cpu import window_ranges
from tests.test_gpu_buffer_bounds import SEED, randn, same_both_ways

pytestmark = pytest.mark.gpu
TOL = 1e-3             # the decoder parity bar of tests/test_gpu_parity.py
CAP = 40
OUT = ("mel_outputs", "mel_outputs_postnet", "gate_outputs", "alignments")
WARNING = "Warning! Reached max decoder steps"


def _model(half=False, cap=CAP):
    # a gate close to its threshold: free runs stop at different steps within the cap
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(synth_state_dict(77, gate_bias=0.09, scale=1.0, gate_sign=-4.0))
    model = model.cuda().eval()
    if half:
        model = model.half()
    model.decoder.max_decoder_steps = cap
    model._t2_engine().impl = _capi.IMPL_PERSISTENT
    return model


def _run(model, text, **kw):
    with torch.no_grad():
        out = [o.clone() for o in model.inference(text.cuda(), **kw)]
    torch.cuda.synchronize()
    return out + [model.mel_lengths.clone()]


def _equal(a, b):
    bad = [i for i, (x, y) in enumerate(zip(a, b)) if not (x.shape == y.shape and torch.equal(x, y))]
    assert not bad, bad


def assert_windowed(align, lengths, window):
    """Exact, on the engine's own fp32 alignments (B, T_steps, T_text): at every step the weights outside the window
    around the first argmax of the step before are 0 and those inside are positive, i.e. the kernel used exactly that
    p_t.  Frames after the row's 64-row slice stopped are all zero and are only checked to be so."""
    lo, hi = window_ranges(align.cpu(), lengths, window)
    a = align.cpu()
    pos = torch.arange(a.shape[2])
    inside = (pos[None, None] >= lo[..., None]) & (pos[None, None] < hi[..., None])
    assert not bool(a[~inside].any())
    ran = a.sum(-1, keepdim=True) > 0
    assert bool((a[inside & ran] > 0).all())


# ---- 1. the fp64 oracle ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("training", [False, True])
@pytest.mark.parametrize("window", [(1, 3), (2, 6)])
def test_windowed_decoder_matches_the_fp64_oracle(window, training):
    B, T, S = 3, 37, 60
    sd = synth_state_dict(41, scale=2.0)
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    model = model.cuda().train(training)
    model.decoder.max_decoder_steps = S
    model.decoder.gate_threshold = 1.0               # no row stops: all S steps are compared
    mem_len = torch.tensor([37, 20, 29])
    memory = torch.randn(B, T, 512, generator=torch.Generator().manual_seed(5))
    keep = keep_mask((S, 2, B, 256), 0.5, 8)
    masks = dict(prenet=keep)
    if training:
        masks.update(att=keep_mask((S, B, 1024), 0.1, 9), dec=keep_mask((S, B, 1024), 0.1, 10))
    with torch.no_grad(), t2.dropout_masks(**masks):
        mel, gate, align = model.decoder.inference(memory.cuda(), memory_lengths=mem_len, attention_window=window)
    n = mel.shape[2]
    assert n == S
    assert_windowed(align, mem_len, window)
    # the oracle loop with the length mask OR the window mask; p_t taken from the engine's alignments, since random
    # weights make near-ties of the argmax likely
    lo, hi = window_ranges(align.float().cpu(), mem_len, window)
    pos = torch.arange(T)
    m64 = memory.double()
    st = O.init_decoder_state(sd64, m64)
    x = m64.new_zeros(B, 80)
    mels, gates, aligns = [], [], []
    for t in range(n):
        px = O.prenet(sd64, x, keep[t, 0], keep[t, 1])
        mask = (pos[None] >= mem_len[:, None]) | (pos[None] < lo[:, t, None]) | (pos[None] >= hi[:, t, None])
        ak = masks["att"][t] if training else None
        dk = masks["dec"][t] if training else None
        m, g, aw = O.decode_step(sd64, st, m64, px, mask, ak, dk)
        mels.append(m); gates.append(g); aligns.append(aw)
        x = m
    ref = torch.stack(mels, 2), torch.stack(gates, 1), torch.stack(aligns, 1)
    errs = [rel_err(mel, ref[0]), rel_err(gate[..., 0], ref[1][..., 0]), rel_err(align, ref[2])]
    assert max(errs) < TOL, errs


# ---- 2. a window that masks nothing ----------------------------------------------------------------------------------

@pytest.mark.parametrize("T", [37, 150, 281, 897, 1300])
def test_a_window_that_masks_nothing_is_the_free_run(T):
    """B = 1 across the regimes: pa tile precomputed (37, 150), pa after B2 (281), 3-stage ring (897, 1300)."""
    model = _model(cap=60)
    text = rand_text(1, T, T)
    free = _run(model, text, seeds=[T + 11])
    for window in ((T, T), (10 ** 12, 10 ** 12)):
        wide = _run(model, text, seeds=[T + 11], attention_window=window)
        _equal(wide, free)


# ---- 3. the (0, 1) window is a forced one-hot run --------------------------------------------------------------------

def test_window_0_1_equals_the_forced_one_hot_run():
    model = _model()
    B, T = 3, 30
    text = rand_text(B, T, 31)
    lengths = torch.tensor([30, 7, 19])
    seeds = [5, 6, 7]
    win = _run(model, text, input_lengths=lengths, seeds=seeds, attention_window=(0, 1))
    n = win[4]
    amap = torch.zeros(B, int(n.max()), T, device="cuda")
    amap[:, :, 0] = 1.0
    assert torch.equal(win[3], amap)                 # one-hot at position 0 at every step, also after a row has stopped
    for b in range(B):
        amap[b, int(n[b]):] = 0
    forced = _run(model, text, input_lengths=lengths, seeds=seeds, alignments=amap, alignment_lengths=n)
    assert torch.equal(forced[4], n) and forced[0].shape == win[0].shape
    for b in range(B):                               # a forced row past its steps attends to nothing: compare up to them
        k = int(n[b])
        assert torch.equal(forced[0][b], win[0][b]), b                  # zero past the row's length in both
        assert torch.equal(forced[1][b, :, :k], win[1][b, :, :k]), b
        assert torch.equal(forced[2][b, :k], win[2][b, :k]), b
        assert torch.equal(forced[3][b, :k], win[3][b, :k]), b


# ---- 4. per-row identity ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("half,source", [(False, "seeds"), (False, "masks"), (True, "seeds")])
def test_every_row_of_a_ragged_130_row_batch_equals_its_own_b1_call(half, source):
    model = _model(half=half)
    B, T, window = 130, 50, (1, 3)
    text = rand_text(B, T, 21)
    g = torch.Generator().manual_seed(21)
    lengths = torch.randint(1, T + 1, (B,), generator=g)
    caps = torch.randint(1, CAP + 1, (B,), generator=g)
    lengths[0], caps[0], caps[64], lengths[129], caps[100] = T, CAP, 1, 1, CAP + 7    # a cap above max_decoder_steps
    seeds = [9000 + 31 * b for b in range(B)]
    keep = keep_mask((CAP + 7, 2, B, 256), 0.5, 23)

    def call(txt, rows, **kw):
        kw.update(attention_window=window)
        if source == "seeds":
            return _run(model, txt, seeds=[seeds[b] for b in rows], **kw)
        with t2.dropout_masks(prenet=keep[:, :, rows].contiguous()):
            return _run(model, txt, **kw)

    out = call(text, list(range(B)), input_lengths=lengths, max_decoder_steps=caps.tolist())
    assert out[0].shape[2] == int(out[4].max()) and bool((out[4].cpu() <= caps).all())
    if not half:                                     # fp16 rounding of the returned weights can tie their maximum
        assert_windowed(out[3], lengths, window)
    try:
        for b in range(B):
            L, n = int(lengths[b]), int(out[4][b])
            model.decoder.max_decoder_steps = int(caps[b])
            one = call(text[b:b + 1, :L], [b])
            assert one[0].shape[2] == n and int(one[4][0]) == n, b
            assert torch.equal(out[0][b, :, :n], one[0][0]), b
            assert torch.equal(out[1][b, :, :n], one[1][0]), b
            assert torch.equal(out[2][b, :n], one[2][0]), b
            assert torch.equal(out[3][b, :n, :L], one[3][0]), b
    finally:
        model.decoder.max_decoder_steps = CAP


# ---- 5. caps alone ---------------------------------------------------------------------------------------------------

def test_caps_alone(capsys):
    model = _model()
    B, T = 8, 40
    text = rand_text(B, T, 41)
    lengths = torch.randint(5, T + 1, (B,), generator=torch.Generator().manual_seed(41))
    seeds = [300 + b for b in range(B)]
    free = _run(model, text, input_lengths=lengths, seeds=seeds)
    same = _run(model, text, input_lengths=lengths, seeds=seeds, max_decoder_steps=CAP)
    _equal(same, free)
    _equal(_run(model, text, input_lengths=lengths, seeds=seeds, max_decoder_steps=torch.full((B,), CAP).cuda()), free)
    n, gate = free[4].cpu(), free[2][..., 0].float().cpu()
    fired = torch.sigmoid(gate[torch.arange(B), n.long() - 1]) > model.decoder.gate_threshold
    rows = [b for b in range(B) if bool(fired[b]) and int(n[b]) >= 2]
    assert len(rows) >= 2, n
    sub = text[rows]
    sub_len, sub_seeds, sub_n = lengths[rows], [seeds[b] for b in rows], n[rows]
    # each row's cap at its own firing step: nothing is cut, no warning, and the run ends at the longest row
    capsys.readouterr()
    at = _run(model, sub, input_lengths=sub_len, seeds=sub_seeds, max_decoder_steps=sub_n.tolist())
    assert WARNING not in capsys.readouterr().out
    assert torch.equal(at[4].cpu(), sub_n) and at[0].shape[2] == int(sub_n.max())
    # one row cut a step before its gate fires: it stops there unfired, and the warning is printed once
    cut = sub_n.clone()
    cut[0] -= 1
    short = _run(model, sub, input_lengths=sub_len, seeds=sub_seeds, max_decoder_steps=cut.tolist())
    assert capsys.readouterr().out.count(WARNING) == 1
    assert torch.equal(short[4].cpu(), cut) and short[0].shape[2] == int(cut.max())
    k = int(cut[0])
    assert torch.equal(short[0][0, :, :k], at[0][0, :, :k]) and torch.equal(short[2][0, :k], at[2][0, :k])


# ---- 6. streams ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("chunk", [1, 7, 32, 128])
def test_limited_stream_concatenates_to_limited_inference(chunk, capsys):
    model = _model()
    text = rand_text(5, 33, 5)
    lengths = torch.tensor([33, 4, 20, 33, 11])
    caps = [50, 3, 27, 1, 44]
    seeds = [77 + 7919 * i for i in range(5)]
    kw = dict(input_lengths=lengths, seeds=seeds, attention_window=(1, 3), max_decoder_steps=caps)
    ref = _run(model, text, **kw)
    warned = capsys.readouterr().out.count(WARNING)
    with torch.no_grad():
        items = list(model.inference_stream(text.cuda(), chunk, **kw))
    cat = [torch.cat([it[k] for it in items], 2 if k in ("mel_outputs", "mel_outputs_postnet") else 1) for k in OUT]
    _equal(cat, ref[:4])
    assert torch.equal(items[-1]["mel_lengths"], ref[4])
    assert capsys.readouterr().out.count(WARNING) == warned
    with torch.no_grad():
        mem = torch.randn(5, 33, 512, generator=torch.Generator().manual_seed(6)).cuda()
        dref = [o.clone() for o in model.decoder.inference(mem, memory_lengths=lengths, seeds=seeds,
                                                           attention_window=(2, 2), max_decoder_steps=caps)]
        ditems = list(model.decoder.inference_stream(mem, chunk, memory_lengths=lengths, seeds=seeds,
                                                     attention_window=(2, 2), max_decoder_steps=caps))
    _equal([torch.cat([it[k] for it in ditems], 2 if k == "mel_outputs" else 1)
            for k in ("mel_outputs", "gate_outputs", "alignments")], dref)


# ---- 7. the server ---------------------------------------------------------------------------------------------------

def test_server_slots_take_the_window():
    """Five texts through two slots, so rows are admitted in the middle of a run: each result equals its own windowed
    B = 1 inference()."""
    model = _model()
    window = (1, 3)
    texts = [rand_text(1, L, 60 + L)[0] for L in (25, 6, 31, 12, 18)]
    seeds = [1000 + i for i in range(len(texts))]
    with torch.no_grad():
        res = model.inference_many(texts, slots=2, chunk_steps=8, seeds=seeds, attention_window=window)
    for x, s, r in zip(texts, seeds, res):
        one = _run(model, x[None], seeds=[s], attention_window=window)
        assert r["mel_length"] == int(one[4][0])
        _equal([r[k] for k in OUT], one[:4])


# ---- 8. refusals and buffers -----------------------------------------------------------------------------------------

def _refused(fn, err, match=None):
    L = _capi.lib()
    torch.cuda.synchronize()
    before = L.t2_kernel_launch_count()
    with pytest.raises(err, match=match):
        fn()
    assert L.t2_kernel_launch_count() == before


def test_bad_arguments_are_refused_before_any_launch():
    model = _model()
    text = rand_text(3, 10, 1).cuda()
    amap = torch.softmax(torch.randn(3, 8, 10), -1).cuda()
    with torch.no_grad():
        _run(model, text, attention_window=(1, 3))                       # handles and workspaces exist
        inf = model.inference
        _refused(lambda: inf(text, attention_window=(1, 3), alignments=amap), ValueError, "attention_window and alignments")
        _refused(lambda: inf(text, max_decoder_steps=5, alignments=amap), ValueError, "max_decoder_steps and alignments")
        _refused(lambda: inf(text, attention_window=(-1, 3)), ValueError, "attention_window")
        _refused(lambda: inf(text, attention_window=(1, 0)), ValueError, "attention_window")
        _refused(lambda: inf(text, attention_window=(1.5, 3)), TypeError, "attention_window")
        _refused(lambda: inf(text, max_decoder_steps=[1, 2]), ValueError, "max_decoder_steps")
        _refused(lambda: inf(text, max_decoder_steps=[1, 0, 2]), ValueError, "max_decoder_steps")
        _refused(lambda: inf(text, max_decoder_steps=torch.tensor([1.0, 2.0, 3.0])), TypeError, "max_decoder_steps")
        _refused(lambda: next(model.inference_stream(text, 4, attention_window=(0, 0))), ValueError, "attention_window")
        mem = torch.zeros(3, 10, 512, device="cuda")
        _refused(lambda: model.decoder.inference(mem, max_decoder_steps=0), ValueError, "max_decoder_steps")
        _refused(lambda: next(model.decoder.inference_stream(mem, 4, attention_window=(1, 3), alignments=amap)),
                 ValueError, "alignments")
        _refused(lambda: model.inference_many([text[0]], attention_window=(3,)), TypeError, "attention_window")
        model.train()
        model.decoder.inference(mem, attention_window=(1, 3))            # training-mode inference takes the window
        model.eval()


def test_library_refuses_invalid_limited_calls():
    """t2_decoder_run with limits: limits with forced_align, TEACHER, a negative window side or a back without a window ->
    T2_ERR_INVALID; the stepwise implementation, requested or chosen by AUTO -> T2_ERR_UNSUPPORTED.  The stream refuses
    the same, and admit refuses step limits."""
    model = _model()
    eng = model._t2_engine()
    B, T, cap = 2, 10, 4
    memory = torch.zeros(B, T, 512, device="cuda")
    caps = torch.full((B,), 3, dtype=torch.int32, device="cuda")
    fa = torch.zeros(B, cap, T, device="cuda")
    fl = torch.full((B,), cap, dtype=torch.int32, device="cuda")
    with torch.no_grad():
        model.inference(rand_text(B, T, 1).cuda())
        L = _capi.lib()
        before = L.t2_kernel_launch_count()
        with pytest.raises(_capi.T2Error, match="error -1: .*forced_align"):
            eng.decoder(memory, _capi.MODE_INFER, cap, window=(1, 3), forced_align=fa, forced_lengths=fl)
        with pytest.raises(_capi.T2Error, match="error -1: .*mode INFER"):
            eng.decoder(memory, _capi.MODE_TEACHER, cap, teacher_prenet=torch.zeros(cap, B, 256, device="cuda"),
                        max_steps=caps)
        with pytest.raises(_capi.T2Error, match="error -1: .*negative"):
            eng.decoder(memory, _capi.MODE_INFER, cap, window=(-1, 3))
        with pytest.raises(_capi.T2Error, match="error -1: .*negative"):
            eng.decoder(memory, _capi.MODE_INFER, cap, window=(1, -3))
        with pytest.raises(_capi.T2Error, match="error -1: .*without a window"):
            eng.decoder(memory, _capi.MODE_INFER, cap, window=(2, 0))
        with pytest.raises(_capi.T2Error, match="error -4: .*limits needs the persistent"):
            eng.decoder(memory, _capi.MODE_INFER, cap, impl=_capi.IMPL_STEPWISE, window=(1, 3))
        with pytest.raises(_capi.T2Error, match="error -4: .*limits needs the persistent"):
            eng.decoder(torch.zeros(1, 2400, 512, device="cuda"), _capi.MODE_INFER, cap, impl=_capi.IMPL_AUTO,
                        max_steps=caps[:1])
        with pytest.raises(_capi.T2Error, match="error -1: .*negative"):
            eng.decoder_stream(memory, cap, window=(1, -1))
        with pytest.raises(_capi.T2Error, match="error -1: .*forced_align"):
            eng.decoder_stream(memory, cap, max_steps=caps, forced_align=fa, forced_lengths=fl)
        assert L.t2_kernel_launch_count() == before
        lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
        st = eng.decoder_stream(memory, cap, memory_lengths=lens, gate_threshold=1.0, window=(1, 3), max_steps=caps)
        with pytest.raises(_capi.T2Error, match="error -1: .*max_steps"):
            st.admit([0])
        st.run(cap)
        torch.cuda.synchronize()
        assert st.mel_lengths.tolist() == [3, 3]
        served = eng.decoder_stream(memory, cap, memory_lengths=lens, window=(1, 3))
        served.admit([1])                                                 # a window alone goes with continuous batching


@pytest.mark.parametrize("Te", [95, 897])
def test_limited_run_stays_inside_its_buffers(Te):
    B = 65
    memory = randn(B, Te, 512, seed=Te + 1, scale=0.5)
    caps = torch.tensor([1 + b % 8 for b in range(B)], dtype=torch.int32, device="cuda")

    def run(eng):
        return list(eng.decoder(memory, _capi.MODE_INFER, 8, impl=_capi.IMPL_PERSISTENT, gate_threshold=0.5, seed=SEED,
                                window=(1, 3), max_steps=caps))
    same_both_ways(run)


def test_limited_stream_stays_inside_its_buffers():
    B, Te = 65, 95
    memory = randn(B, Te, 512, seed=19, scale=0.5)
    caps = torch.tensor([2 + b % 7 for b in range(B)], dtype=torch.int32, device="cuda")

    def run(eng):
        s = eng.decoder_stream(memory, 8, impl=_capi.IMPL_PERSISTENT, seed=SEED, window=(2, 2), max_steps=caps)
        for n in (3, 2, 4):
            s.run(n)
        return [s.mel, s.gate, s.align, s.mel_lengths, s.n_steps, s.status]
    same_both_ways(run)
