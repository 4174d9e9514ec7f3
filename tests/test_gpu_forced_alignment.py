"""Forced-alignment synthesis: ``inference(..., alignments=, alignment_lengths=)`` decodes with the given attention
weights (Mellotron's inference_noattention) on the persistent decoder's forced instantiation.

1. against a forced fp64 oracle loop, for soft and for one-hot maps;
2. a seeded free run fed its own alignments and mel_lengths comes out again bit for bit, across the kernel's T_enc
   regimes and over two 64-row slices;
3. every row of a ragged 130-row batch equals its own B = 1 forced call (fp32 / half, masks / seeds);
4. streams concatenate to the forced inference();
5. duration maps; 6. refusals before any launch."""
import pytest
import torch

import tacotron2_b200 as t2
from oracle import tacotron2_oracle as O
from tacotron2_b200 import _capi
from tests.common import keep_mask, rand_text, rel_err, synth_state_dict

pytestmark = pytest.mark.gpu
TOL = 1e-3             # the decoder parity bar of tests/test_gpu_parity.py
CAP = 40
OUT = ("mel_outputs", "mel_outputs_postnet", "gate_outputs", "alignments")


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


def soft_map(B, T_map, T, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.softmax(3.0 * torch.randn(B, T_map, T, generator=g), -1)


# ---- 1. the fp64 oracle ----------------------------------------------------------------------------------------------

def oracle_forced(sd64, memory, mem_len, amap, alen, keep, monkeypatch):
    """The reference decode loop (oracle decode_step) with the attention weights replaced by the given ones: zero past
    each row's text length and past its step count, as the contract says."""
    B, T_map, T = amap.shape
    used = amap.double().clone()
    for b in range(B):
        used[b, :, int(mem_len[b]):] = 0
        used[b, int(alen[b]):] = 0
    box = {}

    def given(sd, ah, mem, pm, aw_cat, mask, score_mask_value=-float("inf"), mm=None):
        w = box["w"]
        return torch.bmm(w.unsqueeze(1), mem).squeeze(1), w

    monkeypatch.setattr(O, "attention", given)
    memory = memory.double()
    st = O.init_decoder_state(sd64, memory)
    x = memory.new_zeros(B, 80)
    mels, gates, aligns = [], [], []
    with torch.no_grad():
        for t in range(int(max(alen))):
            px = O.prenet(sd64, x, keep[t, 0], keep[t, 1])
            box["w"] = used[:, t]
            mel, gate, aw = O.decode_step(sd64, st, memory, px)
            mels.append(mel); gates.append(gate); aligns.append(aw)
            x = mel
    monkeypatch.undo()
    return torch.stack(mels, 2), torch.stack(gates, 1), torch.stack(aligns, 1)


@pytest.mark.parametrize("kind", ["soft", "durations"])
def test_forced_decoder_matches_the_fp64_oracle(kind, monkeypatch):
    B, T, T_map = 3, 37, 60
    sd = synth_state_dict(41, scale=2.0)
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    model = model.cuda().eval()
    mem_len = torch.tensor([37, 20, 29])
    memory = torch.randn(B, T, 512, generator=torch.Generator().manual_seed(5))
    if kind == "soft":
        amap, alen = soft_map(B, T_map, T, 6), torch.tensor([60, 45, 52])
    else:
        g = torch.Generator().manual_seed(7)
        dur = torch.randint(0, 4, (B, T), generator=g)
        for b in range(B):
            dur[b, int(mem_len[b]):] = 0
        dur[0, 0] += T_map - int(dur[0].sum())           # the longest row fills the map
        amap, alen = t2.alignments_from_durations(dur)
        assert amap.shape[1] == T_map and int(alen.max()) == T_map and len(set(alen.tolist())) == 3
    keep = keep_mask((T_map, 2, B, 256), 0.5, 8)
    ref = oracle_forced(sd64, memory, mem_len, amap, alen, keep, monkeypatch)
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        mel, gate, align = model.decoder.inference(memory.cuda(), memory_lengths=mem_len, alignments=amap.cuda(),
                                                   alignment_lengths=alen)
    assert model.decoder.mel_lengths.cpu().tolist() == alen.tolist()
    errs = [rel_err(mel, ref[0]), rel_err(gate[..., 0], ref[1][..., 0]), rel_err(align, ref[2])]
    assert max(errs) < TOL, errs
    if kind == "durations":
        assert torch.equal(align.cpu(), amap)          # a one-hot map within the text comes back as it went in


# ---- 2. round trip ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("T", [37, 150, 281, 897, 1300])
def test_free_run_fed_its_own_alignments_comes_out_again(T):
    """B = 1 across the regimes: pa tile precomputed (37, 150), pa after B2 (281), 3-stage ring (897, 1300)."""
    model = _model(cap=60)
    text = rand_text(1, T, T)
    free = _run(model, text, seeds=[T + 11])
    n = int(free[4][0])
    forced = _run(model, text, seeds=[T + 11], alignments=free[3], alignment_lengths=free[4])
    assert int(forced[4][0]) == n and free[0].shape[2] == n
    _equal(forced[:4], free[:4])


def test_ragged_two_slice_round_trip():
    model = _model()
    B, T = 70, 48
    text = rand_text(B, T, 3)
    lengths = torch.randint(1, T + 1, (B,), generator=torch.Generator().manual_seed(3))
    lengths[0], lengths[65] = T, 2
    seeds = [500 + 13 * b for b in range(B)]
    free = _run(model, text, input_lengths=lengths, seeds=seeds)
    forced = _run(model, text, input_lengths=lengths, seeds=seeds, alignments=free[3], alignment_lengths=free[4])
    assert torch.equal(forced[4], free[4]) and len(set(free[4].tolist())) > 3
    for b in range(B):
        n = int(free[4][b])
        assert torch.equal(forced[0][b], free[0][b]), b                 # zero past the row's length in both
        assert torch.equal(forced[1][b, :, :n], free[1][b, :, :n]), b
        assert torch.equal(forced[2][b, :n], free[2][b, :n]), b
        assert torch.equal(forced[3][b, :n], free[3][b, :n]), b


# ---- 3. per-row identity ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("half,source", [(False, "seeds"), (False, "masks"), (True, "seeds")])
def test_every_row_of_a_ragged_130_row_batch_equals_its_own_b1_forced_call(half, source):
    model = _model(half=half)
    B, T, T_map = 130, 50, 36
    text = rand_text(B, T, 21)
    g = torch.Generator().manual_seed(21)
    lengths = torch.randint(1, T + 1, (B,), generator=g)
    alen = torch.randint(1, T_map + 1, (B,), generator=g)
    lengths[0], alen[0], alen[64], lengths[129] = T, T_map, 1, 1
    amap = soft_map(B, T_map, T, 22).cuda()
    if half:
        amap = amap.half()
    seeds = [9000 + 31 * b for b in range(B)]
    keep = keep_mask((T_map, 2, B, 256), 0.5, 23)

    def call(txt, a, n, rows, **kw):
        kw.update(alignments=a, alignment_lengths=n)
        if source == "seeds":
            return _run(model, txt, seeds=[seeds[b] for b in rows], **kw)
        with t2.dropout_masks(prenet=keep[:int(a.shape[1]), :, rows].contiguous()):
            return _run(model, txt, **kw)

    out = call(text, amap, alen, list(range(B)), input_lengths=lengths)
    assert torch.equal(out[4].cpu(), alen.to(torch.int32))
    for b in range(B):
        L, n = int(lengths[b]), int(alen[b])
        one = call(text[b:b + 1, :L], amap[b:b + 1, :n, :L], [n], [b])
        assert one[0].shape[2] == n and int(one[4][0]) == n
        assert torch.equal(out[0][b, :, :n], one[0][0]), b
        assert torch.equal(out[1][b, :, :n], one[1][0]), b
        assert torch.equal(out[2][b, :n], one[2][0]), b
        assert torch.equal(out[3][b, :n, :L], one[3][0]), b
        assert not bool(out[0][b, :, n:].any()) and not bool(out[1][b, :, n:].any()), b
        assert not bool(out[3][b, :, L:].any()) and not bool(out[3][b, n:].any()), b


# ---- 4. streams ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("chunk", [1, 7, 32, 128])
def test_forced_stream_concatenates_to_forced_inference(chunk):
    model = _model()
    text = rand_text(5, 33, 5)
    lengths = torch.tensor([33, 4, 20, 33, 11])
    alen = torch.tensor([50, 3, 27, 1, 44])
    amap = soft_map(5, 50, 33, 5).cuda()
    seeds = [77 + 7919 * i for i in range(5)]
    ref = _run(model, text, input_lengths=lengths, seeds=seeds, alignments=amap, alignment_lengths=alen)
    with torch.no_grad():
        items = list(model.inference_stream(text.cuda(), chunk, input_lengths=lengths, seeds=seeds, alignments=amap,
                                            alignment_lengths=alen))
    cat = [torch.cat([it[k] for it in items], 2 if k in ("mel_outputs", "mel_outputs_postnet") else 1) for k in OUT]
    _equal(cat, ref[:4])
    assert torch.equal(items[-1]["mel_lengths"], ref[4]) and torch.equal(ref[4].cpu(), alen.to(torch.int32))


# ---- 5. durations ----------------------------------------------------------------------------------------------------

def test_duration_maps_set_the_lengths_and_come_back_as_given():
    model = _model()
    B, T = 4, 12
    text = rand_text(B, T, 4)
    lengths = torch.tensor([12, 5, 9, 1])
    dur = torch.randint(0, 5, (B, T), generator=torch.Generator().manual_seed(4))
    for b in range(B):
        dur[b, int(lengths[b]):] = 0
    dur[:, 0] += 1                                          # every row has a frame
    amap, alen = t2.alignments_from_durations(dur)
    out = _run(model, text, input_lengths=lengths, alignments=amap.cuda(), alignment_lengths=alen)
    assert out[4].cpu().tolist() == dur.sum(1).tolist()
    assert torch.equal(out[3].cpu(), amap)


# ---- 6. refusals -----------------------------------------------------------------------------------------------------

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
    amap = soft_map(3, 8, 10, 1).cuda()
    with torch.no_grad():
        _run(model, text, alignments=amap)                                  # handles and workspaces exist
        inf = model.inference
        _refused(lambda: inf(text, alignment_lengths=[1, 2, 3]), ValueError, "alignment_lengths needs alignments")
        _refused(lambda: inf(text, alignments=amap[:2]), ValueError, "alignments must have shape")
        _refused(lambda: inf(text, alignments=amap[:, :, :9]), ValueError, "alignments must have shape")
        _refused(lambda: inf(text, alignments=amap.long()), TypeError, "alignments must be a float")
        _refused(lambda: inf(text, alignments=amap.cpu()), ValueError, "device")
        _refused(lambda: inf(text, alignments=amap, alignment_lengths=[1, 2, 9]), ValueError, "1..8")
        _refused(lambda: inf(text, alignments=amap, alignment_lengths=[0, 2, 3]), ValueError, "1..8")
        _refused(lambda: inf(text, alignments=amap, alignment_lengths=[1.0, 2, 3]), TypeError, "integers")
        _refused(lambda: inf(text, alignments=amap, alignment_lengths=[1, 2]), ValueError, "shape")
        _refused(lambda: next(model.inference_stream(text, 4, alignments=amap[:1])), ValueError, "shape")
        mem = torch.zeros(3, 10, 512, device="cuda")
        _refused(lambda: model.decoder.inference(mem, alignments=amap[:, :, :4]), ValueError, "shape")
        _refused(lambda: next(model.decoder.inference_stream(mem, 4, alignment_lengths=[1, 1, 1])), ValueError,
                 "needs alignments")
        model.train()
        _refused(lambda: inf(text, alignments=amap), ValueError, "eval mode")
        _refused(lambda: model.decoder.inference(mem, alignments=amap), ValueError, "eval mode")
        model.eval()


def test_library_refuses_invalid_forced_calls():
    """t2_decoder_run: only one of the two pointers, TEACHER, training = 1 -> T2_ERR_INVALID; the stepwise implementation
    -> T2_ERR_UNSUPPORTED.  The stream refuses the same, and continuous batching takes no map."""
    model = _model()
    eng = model._t2_engine()
    B, T, cap = 2, 10, 4
    memory = torch.zeros(B, T, 512, device="cuda")
    fa = torch.zeros(B, cap, T, device="cuda")
    fl = torch.full((B,), cap, dtype=torch.int32, device="cuda")
    with torch.no_grad():
        model.inference(rand_text(B, T, 1).cuda())
        L = _capi.lib()
        before = L.t2_kernel_launch_count()
        with pytest.raises(_capi.T2Error, match="error -1: .*go together"):
            eng.decoder(memory, _capi.MODE_INFER, cap, forced_align=fa)
        with pytest.raises(_capi.T2Error, match="error -1: .*go together"):
            eng.decoder(memory, _capi.MODE_INFER, cap, forced_lengths=fl)
        with pytest.raises(_capi.T2Error, match="error -1: .*mode INFER"):
            eng.decoder(memory, _capi.MODE_TEACHER, cap, teacher_prenet=torch.zeros(cap, B, 256, device="cuda"),
                        forced_align=fa, forced_lengths=fl)
        with pytest.raises(_capi.T2Error, match="error -1: .*training = 0"):
            eng.decoder(memory, _capi.MODE_INFER, cap, training=True, forced_align=fa, forced_lengths=fl)
        with pytest.raises(_capi.T2Error, match="error -4: .*persistent"):
            eng.decoder(memory, _capi.MODE_INFER, cap, impl=_capi.IMPL_STEPWISE, forced_align=fa, forced_lengths=fl)
        with pytest.raises(_capi.T2Error, match="error -1: .*go together"):
            eng.decoder_stream(memory, cap, forced_align=fa)
        assert L.t2_kernel_launch_count() == before
        lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
        st = eng.decoder_stream(memory, cap, memory_lengths=lens, forced_align=fa, forced_lengths=fl)
        with pytest.raises(_capi.T2Error, match="error -1: .*no forced alignment"):
            st.admit([0])
        st.run(cap)
        torch.cuda.synchronize()
        assert st.mel_lengths.tolist() == [cap, cap]
