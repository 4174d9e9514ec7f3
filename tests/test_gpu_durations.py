"""Durations from attention maps on the GPU (``durations_from_alignments``; DESIGN section 6.10):

1. MAS against the numpy fp64 oracle on softmax maps, exact-zero blocks and a ragged batch, on-chip and workspace bits;
2. argmax against torch's argmax + bincount, ties included;
3. the tie rule on uniform maps;
4. round trips through ``alignments_from_durations``;
5. each row of a ragged batch equals its own B = 1 call, fp16 maps give the fp32 result;
6. end to end on the model: free run -> durations -> forced run, a lengthened symbol, teacher-forced durations."""
import numpy as np
import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tests import durations_oracle as DO
from tests.common import rand_text, synth_state_dict

pytestmark = pytest.mark.gpu


def durations(a, il=None, ml=None, method="mas"):
    out = t2.durations_from_alignments(a, il, ml, method)
    torch.cuda.synchronize()
    assert out.dtype == torch.int64 and out.device == a.device and out.shape == (a.shape[0], a.shape[2])
    return out.cpu()


def softmax_maps(B, T_mel, T_text, temperature, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.softmax(torch.randn(B, T_mel, T_text, generator=g) * temperature, -1)


def ragged(B, T_mel, T_text, seed, pairs=()):
    """Per-row (L_text, L_mel) with L_mel >= L_text, the given pairs first, and a map that is a softmax over each row's
    own symbols, with large finite garbage outside the row."""
    g = torch.Generator().manual_seed(seed)
    lt = torch.randint(1, T_text + 1, (B,), generator=g)
    lm = torch.minimum(lt + torch.randint(0, T_mel, (B,), generator=g), torch.full((B,), T_mel))
    for b, (x, y) in enumerate(pairs):
        lt[b], lm[b] = x, y
    lt[len(pairs)], lm[len(pairs)] = T_text, T_mel
    a = torch.rand(B, T_mel, T_text, generator=g) * 1e3
    for b in range(B):
        a[b, :lm[b], :lt[b]] = torch.softmax(torch.randn(int(lm[b]), int(lt[b]), generator=g) * 3, -1)
    return a, lt, lm


def assert_mas_matches_oracle(a, lt, lm, got):
    """Durations equal the oracle's; where they differ, the two paths' fp64 scores must agree to 1e-12 relative (a tie
    under the rounding of fp64 log).  Returns the number of such rows."""
    ties = 0
    for b in range(a.shape[0]):
        x = a[b, :lm[b], :lt[b]].double().numpy()
        want, d = DO.mas(x), got[b, :lt[b]].numpy()
        assert not got[b, lt[b]:].any() and d.sum() == lm[b] and (d >= 1).all()
        if not np.array_equal(d, want):
            s, r = DO.path_score(x, d), DO.path_score(x, want)
            assert abs(s - r) <= 1e-12 * abs(r), (b, s, r)
            ties += 1
    return ties


# ---- 1. MAS against the fp64 oracle ----------------------------------------------------------------------------------

@pytest.mark.parametrize("temperature", [0.5, 3.0, 12.0])
@pytest.mark.parametrize("B,T_mel,T_text", [(6, 90, 17), (4, 400, 150), (3, 2600, 1000)])
def test_mas_matches_the_fp64_oracle_on_softmax_maps(B, T_mel, T_text, temperature):
    a = softmax_maps(B, T_mel, T_text, temperature, T_text)
    if T_text == 17:                                  # exact-zero blocks, as padding or attention_window leave
        a[:, 10:40, 3:12] = 0
        a[1] = 0
    got = durations(a.cuda())
    full = torch.full((B,), T_text), torch.full((B,), T_mel)
    assert assert_mas_matches_oracle(a, *full, got) <= 1


def test_mas_matches_the_fp64_oracle_on_a_ragged_batch():
    a, lt, lm = ragged(37, 2000, 300, 1, pairs=[(300, 300), (1, 2000), (1, 1), (57, 57), (1, 13), (299, 2000)])
    for il, ml in ((lt, lm), (lt.cuda(), lm.cuda()), (lt.tolist(), lm.int())):
        got = durations(a.cuda(), il, ml)
        assert assert_mas_matches_oracle(a, lt, lm, got) <= 2
    assert got[1, 0] == 2000 and got[2, 0] == 1 and got[0, :300].tolist() == [1] * 300


# ---- 2. argmax ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B,T_mel,T_text", [(5, 70, 9), (37, 2000, 300), (2, 300, 4096)])
def test_argmax_equals_torch_argmax_and_bincount(B, T_mel, T_text):
    g = torch.Generator().manual_seed(T_text)
    a = torch.floor(torch.rand(B, T_mel, T_text, generator=g) * 8) / 8     # coarse values: many tied maxima
    a[:, : T_mel // 3] = 0                                                  # all-zero frames go to symbol 0
    lt = torch.randint(1, T_text + 1, (B,), generator=g)
    lm = torch.randint(1, T_mel + 1, (B,), generator=g)
    got = durations(a.cuda(), lt, lm, "argmax")
    for b in range(B):
        x = a[b, :lm[b], :lt[b]]
        want = torch.bincount(x.argmax(1), minlength=T_text)
        assert torch.equal(got[b], want), b
        assert np.array_equal(got[b, :lt[b]].numpy(), DO.argmax(x.numpy()))
    assert torch.equal(got.sum(1), lm)


# ---- 3. the tie rule --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("T_mel,T_text", [(1, 1), (5, 5), (800, 150), (2000, 300), (3000, 1500), (4096, 4096)])
def test_a_uniform_map_advances_as_late_as_it_can(T_mel, T_text):
    a = torch.full((2, T_mel, T_text), 1.0 / T_text, device="cuda")
    a[1] = 0
    got = durations(a)
    want = [1] * (T_text - 1) + [T_mel - T_text + 1]
    assert got[0].tolist() == want and got[1].tolist() == want


# ---- 4. round trips ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B,T_text,hi", [(3, 1, 9), (16, 40, 6), (130, 150, 8), (2, 1500, 3)])
def test_durations_of_a_duration_map_come_back(B, T_text, hi):
    g = torch.Generator().manual_seed(B + T_text)
    d = torch.randint(1, hi, (B, T_text), generator=g)
    if T_text == 1500:
        d[:] = 2                                      # 3000 frames at several symbols per thread, bits in the workspace
    a, n = t2.alignments_from_durations(d.cuda())
    assert torch.equal(durations(a, None, n), d)
    z = torch.randint(0, hi, (B, T_text), generator=g)
    z[:, 0] += (z.sum(1) == 0).long()                 # argmax takes zeros, but not a row of 0 frames
    a, n = t2.alignments_from_durations(z.cuda())
    assert torch.equal(durations(a, None, n, "argmax"), z)


def test_ragged_round_trip_keeps_each_rows_own_symbols():
    g = torch.Generator().manual_seed(3)
    d = torch.randint(1, 5, (9, 60), generator=g)
    lt = torch.randint(1, 61, (9,), generator=g)
    d[torch.arange(60)[None, :] >= lt[:, None]] = 0
    a, n = t2.alignments_from_durations(d.cuda())
    assert torch.equal(durations(a, lt, n), d)
    assert torch.equal(durations(a, lt, n, "argmax"), d)


# ---- 5. ragged rows and fp16 ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("method", ["mas", "argmax"])
def test_every_row_of_a_ragged_batch_equals_its_own_b1_call(method):
    a, lt, lm = ragged(70, 600, 120, 4, pairs=[(120, 120), (1, 600), (1, 1)])
    a = a.cuda()
    got = durations(a, lt, lm, method)
    for b in range(a.shape[0]):
        one = durations(a[b:b + 1, :lm[b], :lt[b]].contiguous(), method=method)
        assert torch.equal(got[b, :lt[b]], one[0]) and not got[b, lt[b]:].any(), b
    h = a.half()
    assert torch.equal(durations(h, lt, lm, method), durations(h.float(), lt, lm, method))
    assert torch.equal(durations(a.double(), lt, lm, method), got)         # fp64 rounds to the same fp32 weights here


def test_a_map_that_requires_grad_is_taken():
    a = softmax_maps(2, 50, 10, 3.0, 0).cuda().requires_grad_()
    assert torch.equal(durations(a), durations(a.detach()))


def test_bad_arguments_are_refused_before_any_launch():
    a = softmax_maps(2, 6, 4, 1.0, 0)
    with pytest.raises(ValueError, match="CUDA device"):
        t2.durations_from_alignments(a)
    bad = a.cuda()
    bad[1, 2, 3] = float("nan")
    with pytest.raises(ValueError, match="finite"):
        t2.durations_from_alignments(bad)
    with pytest.raises(ValueError, match=r"rows \[1\]"):
        t2.durations_from_alignments(a.cuda(), [4, 4], torch.tensor([6, 3], device="cuda"))


def test_library_refuses_invalid_calls():
    L = _capi.lib()
    a = torch.rand(2, 6, 4, device="cuda")
    out = torch.empty(2, 4, dtype=torch.int64, device="cuda")
    need = L.t2_durations_workspace_bytes(2, 6, 4, _capi.DURATIONS_MAS)
    ws = _capi.byte_buffer(need, a.device)

    def rc(**kw):
        f = dict(alignments=a.data_ptr(), input_lengths=None, mel_lengths=None, B=2, T_mel=6, T_text=4,
                 method=_capi.DURATIONS_MAS, durations=out.data_ptr(), ws=ws.data_ptr(), ws_bytes=need)
        f.update(kw)
        args = _capi.T2DurationsArgs(**f)
        return L.t2_durations(args, torch.cuda.current_stream().cuda_stream)
    assert rc() == 0
    for kw in (dict(alignments=None), dict(durations=None), dict(ws=None), dict(B=0), dict(T_mel=0), dict(T_text=0),
               dict(T_text=4097), dict(method=2), dict(method=-1)):
        assert rc(**kw) == -1, kw
    assert rc(ws_bytes=need - 1) == -3
    assert L.t2_durations_workspace_bytes(2, 6, 4097, 0) == 0 and L.t2_durations_workspace_bytes(2, 6, 4, 7) == 0
    torch.cuda.synchronize()


def test_lengths_outside_the_map_are_clamped_by_the_library():
    L = _capi.lib()
    a = softmax_maps(2, 8, 5, 2.0, 1).cuda()
    out = torch.full((2, 5), -7, dtype=torch.int64, device="cuda")
    il = torch.tensor([9, -3], dtype=torch.int32, device="cuda")
    ml = torch.tensor([100, 0], dtype=torch.int32, device="cuda")
    for method in (_capi.DURATIONS_MAS, _capi.DURATIONS_ARGMAX):
        need = L.t2_durations_workspace_bytes(2, 8, 5, method)
        ws = _capi.byte_buffer(need, a.device)
        args = _capi.T2DurationsArgs(a.data_ptr(), il.data_ptr(), ml.data_ptr(), 2, 8, 5, method, out.data_ptr(),
                                     ws.data_ptr(), need)
        assert L.t2_durations(args, torch.cuda.current_stream().cuda_stream) == 0
        want = t2.durations_from_alignments(a, [5, 1], [8, 1], "mas" if method == 0 else "argmax")
        assert torch.equal(out, want)


# ---- 6. end to end on the model ---------------------------------------------------------------------------------------

def _model(cap=60):
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(synth_state_dict(5, gate_bias=-10.0, scale=2.0))
    model = model.cuda().eval()
    model.decoder.max_decoder_steps = cap
    return model


def test_free_run_durations_drive_a_forced_run():
    model = _model()
    text = rand_text(4, 19, 8).cuda()
    lengths = [19, 7, 12, 1]
    seeds = [11, 12, 13, 14]
    with torch.no_grad():
        out = model.inference(text, input_lengths=lengths, seeds=seeds, attention_window=(1, 3),
                              max_decoder_steps=[60, 25, 41, 9])
        align, mel_lengths = out[3].clone(), model.mel_lengths.clone()
        d = t2.durations_from_alignments(align, lengths, mel_lengths)
        assert torch.equal(d.sum(1), mel_lengths.long())
        assert mel_lengths.tolist() == [60, 25, 41, 9]
        amap, n = t2.alignments_from_durations(d)
        model.inference(text, input_lengths=lengths, seeds=seeds, alignments=amap, alignment_lengths=n)
        assert torch.equal(model.mel_lengths.long(), d.sum(1))
        # five more frames on one symbol of row 2 lengthen that row by exactly five
        e = d.clone()
        e[2, 4] += 5
        amap, n = t2.alignments_from_durations(e)
        model.inference(text, input_lengths=lengths, seeds=seeds, alignments=amap, alignment_lengths=n)
        got = model.mel_lengths.long().cpu()
    assert (got - d.sum(1).cpu()).tolist() == [0, 0, 5, 0]


def test_teacher_forced_alignments_give_durations_that_sum_to_the_output_lengths():
    model = _model()
    g = torch.Generator().manual_seed(2)
    B, T_text, T_mel = 6, 40, 120
    text = rand_text(B, T_text, 9)
    tl = torch.tensor([40, 33, 30, 17, 9, 2])
    ol = torch.tensor([120, 70, 101, 44, 9, 30])
    mels = torch.randn(B, 80, T_mel, generator=g)
    gate = torch.zeros(B, T_mel)
    x, _ = model.parse_batch((text, tl, mels, gate, ol))
    with torch.no_grad():
        out = model(x)
    align = out[3]
    assert align.shape == (B, T_mel, T_text)
    for method in ("mas", "argmax"):
        d = t2.durations_from_alignments(align, x[1], x[4], method)
        assert torch.equal(d.sum(1).cpu(), ol)
        assert not d.cpu()[torch.arange(T_text)[None, :] >= tl[:, None]].any()
