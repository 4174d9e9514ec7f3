"""The decoder across its encoder-length regimes and its 64-row batch slices, against the oracle in float64.

The persistent decoder sizes its shared memory from T_enc (``persistent_smem_bytes`` in decoder_persistent.cu, 227 KiB per
block on the H100):

    T_enc        ring     encoder-memory rows staged in the idle ring (the rest is read from L2)
    1 - 94       4 stages all of them
    95 - 896     4 stages rows 0-93
    897 - 2274   3 stages rows 0-57
    >= 2275      refused; T2_IMPL_AUTO falls back to the stepwise decoder, which itself stops at T_enc = 1282

and the decoder backward's attention kernel stops at T_enc = 408.  Batches of more than 64 rows run as independent 64-row
launches of the persistent kernel, each stopping when its own rows have fired.

Bar: max|a - b| / max|b| < 1e-4 on mel, gate and alignments over <= 12 steps (10x below the 1e-3 parity bar); gradients keep
the 1e-3 bar of tests/test_gpu_backward.py.  Every case prints its measured errors.  So that a kernel reading the wrong
encoder-memory row cannot hide in that bar, the synthetic memories scale the rows next to every layout edge by +-8 (row 0, the
last staged and first L2 row of both ring depths, the attention round / tile edges 63/64 and 127/128, row T_enc - 1), and
the CPU test ``test_marked_rows_make_a_one_row_context_slip_visible`` shows that dropping or double-counting any one of
those rows in the oracle's context moves the outputs by more than 10x the bar."""
import functools
import re

import pytest
import torch

import tacotron2_b200 as t2
from oracle import tacotron2_oracle as O
from tacotron2_b200 import _capi
from tests.common import keep_mask, rand_text, rel_err, synth_state_dict

TOL = 1e-4          # forward outputs over <= 12 steps vs the fp64 oracle
GRAD_TOL = 1e-3     # decoder backward (same bar as tests/test_gpu_backward.py)
STEPS = 8
IMPLS = [(_capi.IMPL_STEPWISE, "stepwise"), (_capi.IMPL_PERSISTENT, "persistent")]
STEPWISE_MAX_T_ENC = 1282        # stepwise_attention_smem(T_enc) <= 200 KiB
PERSISTENT_MAX_T_ENC = 2274      # persistent_smem_bytes(T_enc, 3 stages) <= 227 KiB
BACKWARD_MAX_T_ENC = 408         # att_bwd_smem(T_enc) <= 220 KiB
EDGE_ROWS = (0, 57, 58, 63, 64, 93, 94, 127, 128)


def as_fp64(sd):
    return {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}


def marked_rows(T):
    return sorted({r for r in EDGE_ROWS if r < T} | {T - 1})


@functools.lru_cache(maxsize=None)
def regime_weights():
    sd = synth_state_dict(41, scale=2.0)
    return sd, as_fp64(sd)


def regime_inputs(B, T):
    """Seeded encoder memory with the layout-edge rows scaled by +-8, and prenet keep masks for STEPS steps.  A scaled row
    saturates the tanh of its attention energy, which then is about v . sign(W_memory m) for any query; the sign is chosen
    to make that positive, so the attention does look at every marked row (with a negative one it may weigh ~1e-5)."""
    _, sd64 = regime_weights()
    wm = sd64["decoder.attention_layer.memory_layer.linear_layer.weight"].float()
    v = sd64["decoder.attention_layer.v.linear_layer.weight"][0].float()
    memory = torch.randn(B, T, 512, generator=torch.Generator().manual_seed(1000 * B + T))
    rows = marked_rows(T)
    memory[:, rows] *= 8.0 * torch.sign(torch.sign(memory[:, rows] @ wm.t()) @ v).unsqueeze(-1)
    return memory, keep_mask((STEPS, 2, B, 256), 0.5, T + 7)


def oracle_inference(sd64, memory, keep, steps, gate_threshold=1.0):
    with torch.no_grad():
        mel, gate, align, lengths = O.decoder_inference(sd64, memory.double(), keep, gate_threshold, steps)
    return (mel, gate, align), lengths


def output_errors(out, ref):
    return {k: rel_err(a, b) for k, a, b in zip(("mel", "gate", "align"), out, ref)}


_models = {}


def make_model(sd, key):
    if key not in _models:
        model = t2.Tacotron2(t2.create_hparams())
        model.load_state_dict(sd)
        _models[key] = model.cuda().eval()
    return _models[key]


def run_inference(model, memory, keep, impl, steps, gate_threshold=1.0):
    model._t2_engine().impl = impl
    model.decoder.max_decoder_steps = steps
    model.decoder.gate_threshold = gate_threshold
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        out = model.decoder.inference(memory.cuda())
    torch.cuda.synchronize()
    return [o.cpu() for o in out], model.decoder.mel_lengths.cpu()


def stages_seen(capfd):
    """Ring depths the persistent decoder reported (T2_VERBOSE=1), one per 64-row launch."""
    return [int(s) for s in re.findall(r"persistent decoder: .* stages=(\d+)", capfd.readouterr().err)]


# ---------------------------------------------------------------------------------------------------------------------
# the marked rows make a one-row slip in the context visible (CPU)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("factor", [0.0, 2.0], ids=["dropped", "doubled"])
@pytest.mark.parametrize("T", [896, 2274])
def test_marked_rows_make_a_one_row_context_slip_visible(T, factor, monkeypatch):
    """A mutant oracle whose context drops one marked memory row (or counts it twice) differs from the true oracle by more
    than 10x TOL, so the GPU cases below would catch a kernel making that mistake at any layout edge."""
    B = 3
    _, sd64 = regime_weights()
    memory, keep = regime_inputs(B, T)
    ref, _ = oracle_inference(sd64, memory, keep, STEPS)
    attention = O.attention

    def slipped(row):
        def att(sd, ah, mem, pm, aw_cat, mask, score_mask_value=-float("inf"), mm=None):
            _, aw = attention(sd, ah, mem, pm, aw_cat, mask, score_mask_value, mm)
            w = aw.clone()
            w[:, row] *= factor
            return torch.bmm(w.unsqueeze(1), mem).squeeze(1), aw
        return att

    moved = {}
    for row in marked_rows(T):
        monkeypatch.setattr(O, "attention", slipped(row))
        out, _ = oracle_inference(sd64, memory, keep, STEPS)
        moved[row] = max(output_errors(out, ref).values())
    monkeypatch.setattr(O, "attention", attention)
    print("T_enc=%d row %s: outputs move by %s" % (T, "dropped" if factor == 0 else "doubled",
                                                   ", ".join("%d: %.1e" % kv for kv in moved.items())))
    assert min(moved.values()) >= 10 * TOL, moved


# ---------------------------------------------------------------------------------------------------------------------
# 1. inference across the T_enc regimes
# ---------------------------------------------------------------------------------------------------------------------
REGIMES = [  # (T_enc, B, T2_STAGES, ring stages expected)
    (94, 3, None, 4),        # every row the context reads is staged
    (95, 3, None, 4),        # row 94: first row read from L2
    (896, 3, None, 4),       # longest 4-stage layout
    (897, 3, None, 3),       # shortest 3-stage layout
    (897, 64, None, 3),      # all 64 attention CTA pairs on the 3-stage layout
    (1282, 3, None, 3),      # longest the stepwise decoder takes
    (1283, 3, None, 3),      # persistent only
    (2274, 3, None, 3),      # longest the persistent decoder takes
    (58, 3, "3", 3),         # 3 stages forced: every row staged
    (59, 3, "3", 3),         # 3 stages forced: row 58 from L2
]


@pytest.mark.gpu
@pytest.mark.parametrize("T,B,force_stages,stages", REGIMES,
                         ids=["T%d-B%d%s" % (T, B, "-stages%s" % f if f else "") for T, B, f, _ in REGIMES])
def test_decoder_inference_across_encoder_length_regimes(T, B, force_stages, stages, monkeypatch, capfd):
    """Decoder.inference, every step live (gate_threshold = 1), persistent and (where it fits) stepwise vs the fp64 oracle;
    the persistent launch must report the ring depth the case is meant to cover."""
    sd, sd64 = regime_weights()
    model = make_model(sd, "regime")
    memory, keep = regime_inputs(B, T)
    ref, ref_lengths = oracle_inference(sd64, memory, keep, STEPS)
    monkeypatch.setenv("T2_VERBOSE", "1")
    if force_stages:
        monkeypatch.setenv("T2_STAGES", force_stages)
    else:
        monkeypatch.delenv("T2_STAGES", raising=False)
    impls = [(_capi.IMPL_PERSISTENT, "persistent")]
    if T <= STEPWISE_MAX_T_ENC:
        impls.append((_capi.IMPL_STEPWISE, "stepwise"))
    report, bad, outs = [], {}, {}
    for impl, name in impls:
        capfd.readouterr()
        out, lengths = run_inference(model, memory, keep, impl, STEPS)
        seen = stages_seen(capfd)
        if impl == _capi.IMPL_PERSISTENT:
            assert seen == [stages] * ((B + 63) // 64), seen
        assert lengths.tolist() == ref_lengths.tolist() == [STEPS] * B
        assert out[0].shape == (B, 80, STEPS) and out[2].shape == (B, STEPS, T)
        errs = output_errors(out, ref)
        row_sum = float((out[2].double().sum(-1) - 1).abs().max())
        report.append("%s %s, align row sums %.1e" % (name, ", ".join("%s %.2e" % kv for kv in errs.items()), row_sum))
        bad.update({(name, k): v for k, v in errs.items() if not v < TOL})
        if not row_sum < 1e-5:
            bad[(name, "align row sum")] = row_sum
        outs[name] = out
    if T == PERSISTENT_MAX_T_ENC:    # summation order is fixed: a rerun is bit-identical
        again, _ = run_inference(model, memory, keep, _capi.IMPL_PERSISTENT, STEPS)
        assert all(torch.equal(a, b) for a, b in zip(outs["persistent"], again))
    print("T_enc=%d B=%d stages=%d: %s" % (T, B, stages, "; ".join(report)))
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------------
# 2. end to end at a long text
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_tacotron2_inference_at_a_897_token_text(monkeypatch, capfd):
    """Encoder convs, persistent BiLSTM and the 3-stage decoder at T_text = 897 vs the fp64 oracle."""
    B, T, S = 2, 897, 6
    sd, sd64 = regime_weights()
    model = make_model(sd, "regime")
    text = rand_text(B, T, 97)
    keep = keep_mask((S, 2, B, 256), 0.5, 98)
    with torch.no_grad():
        ref = O.tacotron2_inference(sd64, text, keep, 1.0, S)
    model._t2_engine().impl = _capi.IMPL_AUTO
    model.decoder.max_decoder_steps = S
    model.decoder.gate_threshold = 1.0
    monkeypatch.setenv("T2_VERBOSE", "1")
    capfd.readouterr()
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        out = [o.cpu() for o in model.inference(text.cuda())]
    torch.cuda.synchronize()
    assert stages_seen(capfd) == [3]
    assert model.mel_lengths.cpu().tolist() == ref[4].tolist() == [S] * B
    errs = {k: rel_err(a, b) for k, a, b in zip(("mel", "mel_postnet", "gate", "align"), out, ref[:4])}
    print("T_text=%d B=%d: %s" % (T, B, ", ".join("%s %.2e" % kv for kv in errs.items())))
    assert all(v < TOL for v in errs.values()), errs


# ---------------------------------------------------------------------------------------------------------------------
# 3. refusals past the kernels' limits
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("T,impl", [(STEPWISE_MAX_T_ENC + 1, _capi.IMPL_STEPWISE),
                                    (PERSISTENT_MAX_T_ENC + 1, _capi.IMPL_PERSISTENT),
                                    (PERSISTENT_MAX_T_ENC + 1, _capi.IMPL_AUTO)],
                         ids=["stepwise-1283", "persistent-2275", "auto-2275"])
def test_decoder_refuses_encoder_lengths_past_its_kernels(T, impl):
    """An encoder memory too long for the requested implementation is refused on the host with an error naming T_enc, and
    the engine keeps working afterwards."""
    sd, sd64 = regime_weights()
    model = make_model(sd, "regime")
    memory = torch.randn(1, T, 512, generator=torch.Generator().manual_seed(T))
    keep = keep_mask((4, 2, 1, 256), 0.5, 3)
    with pytest.raises(_capi.T2Error, match=r"T_enc ?= ?%d\b" % T):
        run_inference(model, memory, keep, impl, 4)
    memory, keep = torch.randn(2, 40, 512, generator=torch.Generator().manual_seed(40)), keep_mask((4, 2, 2, 256), 0.5, 4)
    ref, _ = oracle_inference(sd64, memory, keep, 4)
    out, _ = run_inference(model, memory, keep, impl, 4)
    assert all(v < TOL for v in output_errors(out, ref).values())


# ---------------------------------------------------------------------------------------------------------------------
# 4. ragged stops across 64-row slices
# ---------------------------------------------------------------------------------------------------------------------
def choose_stop_bias(gate, S):
    """Gate logits (B, S) of a run in which no row stops (the gate is not fed back, so they do not depend on the threshold).
    Returns the logit t at which rows are made to stop -- the midpoint of the widest gap between the rows' running-maximum
    logits among the gaps that spread the stops over both slices -- with each row's frame count for that t.  The gate bias
    is then shifted by -t and the threshold kept at sigmoid(0) = 0.5."""
    B = gate.shape[0]
    running = torch.cummax(gate, dim=1).values
    vals = torch.unique(running.flatten())
    best = None
    for lo, hi in zip(vals[:-1].tolist(), vals[1:].tolist()):
        fired = running > (lo + hi) / 2
        lengths = torch.where(fired.any(1), fired.int().argmax(1) + 1, torch.full((B,), S))
        ends = [int(lengths[:64].max()), int(lengths[64:].max())]
        spread = len(set(lengths[fired.any(1)].tolist()))
        if ends[0] != ends[1] and spread >= 10 and not bool(fired.any(1).all()) and (best is None or hi - lo > best[0]):
            best = (hi - lo, (lo + hi) / 2)
    assert best is not None, "no stop threshold spreads the stops over both slices"
    return best[1]


@functools.lru_cache(maxsize=None)
def ragged_case():
    """B = 100 rows (launches of 64 + 36), T_enc = 41, 40 steps; stop points chosen from a first oracle run."""
    B, T, S = 100, 41, 40
    sd = synth_state_dict(31, gate_bias=0.0, gate_sign=10.0, scale=2.0)
    memory = torch.randn(B, T, 512, generator=torch.Generator().manual_seed(31))
    keep = keep_mask((S, 2, B, 256), 0.5, 32)
    (_, gate, _), _ = oracle_inference(as_fp64(sd), memory, keep, S)
    theta = choose_stop_bias(gate[:, :, 0], S)
    sd["decoder.gate_layer.linear_layer.bias"] = torch.tensor([-theta], dtype=torch.float32)
    theta = -float(sd["decoder.gate_layer.linear_layer.bias"])
    ref, lengths = oracle_inference(as_fp64(sd), memory, keep, S, gate_threshold=0.5)
    live = torch.arange(S)[None, :] < lengths[:, None].long()
    margin = float((gate[:, :, 0] - theta).abs()[live].min())     # of every stop decision the latch takes
    ends = [int(lengths[:64].max()), int(lengths[64:].max())]
    return dict(sd=sd, memory=memory, keep=keep, S=S, ref=ref, lengths=lengths, margin=margin, ends=ends)


def test_ragged_stop_case_spreads_stops_over_both_slices():
    c = ragged_case()
    lengths = c["lengths"]
    print("ragged case: stop logit margin %.3f, slices end at %s, %d distinct stops, %d rows never fire" % (
        c["margin"], c["ends"], len(set(lengths[lengths < c["S"]].tolist())), int((lengths == c["S"]).sum())))
    assert c["margin"] >= 1e-5
    assert c["ends"][0] != c["ends"][1]
    assert len(set(lengths.tolist())) >= 10 and bool((lengths == c["S"]).any())


@pytest.mark.gpu
@pytest.mark.parametrize("impl,impl_name", IMPLS)
def test_ragged_stops_across_64_row_slices(impl, impl_name):
    """Persistent: each 64-row launch stops when its own rows have fired; frames from its last step on stay exactly zero.
    Stepwise: one launch over all rows, every frame up to the batch's last step matches the oracle."""
    c = ragged_case()
    model = make_model(c["sd"], "ragged")
    (mel, gate, align), lengths = run_inference(model, c["memory"], c["keep"], impl, c["S"], gate_threshold=0.5)
    assert lengths.tolist() == c["lengths"].tolist()
    n = mel.shape[2]
    assert n == int(c["lengths"].max()) == gate.shape[1] == align.shape[1]
    rmel, rgate, ralign = (r[:, :, :n] if i == 0 else r[:, :n] for i, r in enumerate(c["ref"]))
    errs = []
    for s, (b0, b1) in enumerate([(0, 64), (64, 100)]):
        end = c["ends"][s] if impl == _capi.IMPL_PERSISTENT else n
        e = output_errors((mel[b0:b1, :, :end], gate[b0:b1, :end], align[b0:b1, :end]),
                          (rmel[b0:b1, :, :end], rgate[b0:b1, :end], ralign[b0:b1, :end]))
        errs.append("rows %d-%d to step %d: %s" % (b0, b1 - 1, end, ", ".join("%s %.2e" % kv for kv in e.items())))
        assert all(v < TOL for v in e.values()), (s, e)
        if end < n:
            assert float(mel[b0:b1, :, end:].abs().max()) == 0.0
            assert float(gate[b0:b1, end:].abs().max()) == 0.0
            assert float(align[b0:b1, end:].abs().max()) == 0.0
    print("ragged stops [%s]: %s" % (impl_name, "; ".join(errs)))


@pytest.mark.gpu
def test_tacotron2_inference_zeroes_frames_past_each_rows_length():
    """Tacotron2.inference at B = 100 with stops spread over both slices: mel and mel_postnet are zero from each row's
    length on and match the fp64 oracle before it."""
    B, T, S = 100, 41, 40
    sd = synth_state_dict(31, gate_bias=0.0, gate_sign=10.0, scale=2.0)
    text = rand_text(B, T, 31)
    keep = keep_mask((S, 2, B, 256), 0.5, 33)
    with torch.no_grad():
        gate = O.tacotron2_inference(as_fp64(sd), text, keep, 1.0, S)[2]
    sd["decoder.gate_layer.linear_layer.bias"] = torch.tensor([-choose_stop_bias(gate[:, :, 0], S)], dtype=torch.float32)
    with torch.no_grad():
        ref = O.tacotron2_inference(as_fp64(sd), text, keep, 0.5, S)
    model = make_model(sd, "ragged-text")
    model.decoder.max_decoder_steps = S
    model.decoder.gate_threshold = 0.5
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        mel, post, gate, align = [o.cpu() for o in model.inference(text.cuda())]
    lengths = model.mel_lengths.cpu()
    assert lengths.tolist() == ref[4].tolist()
    pad = torch.arange(mel.shape[2])[None, :] >= lengths[:, None].long()
    assert float(mel.masked_select(pad[:, None, :]).abs().max()) == 0.0
    assert float(post.masked_select(pad[:, None, :]).abs().max()) == 0.0
    errs = {"mel": rel_err(mel, ref[0]), "mel_postnet": rel_err(post, ref[1])}
    print("Tacotron2.inference B=%d, %d distinct lengths: %s" % (B, len(set(lengths.tolist())),
                                                              ", ".join("%s %.2e" % kv for kv in errs.items())))
    assert all(v < TOL for v in errs.values()), errs


# ---------------------------------------------------------------------------------------------------------------------
# 5. teacher forcing over two slices, and the backward near its limit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("impl,impl_name", IMPLS)
def test_teacher_forced_forward_over_two_slices(impl, impl_name):
    """No-grad Decoder.forward (validation) at B = 70 with ragged memory lengths in both slices, one of them 1."""
    B, Te, Tm = 70, 37, 8
    sd, sd64 = regime_weights()
    model = make_model(sd, "regime")
    model._t2_engine().impl = impl
    g = torch.Generator().manual_seed(70)
    memory = torch.randn(B, Te, 512, generator=g)
    mels = torch.randn(B, 80, Tm, generator=g)
    lens = torch.randint(1, Te + 1, (B,), generator=g)
    lens[[0, 64]] = Te
    lens[[5, 66]] = 1
    pk = keep_mask((Tm + 1, 2, B, 256), 0.5, 71)
    with torch.no_grad():
        ref = O.decoder_forward(sd64, memory.double(), mels.double(), lens, pk, training=False)
        with t2.dropout_masks(prenet=pk):
            out = [o.cpu() for o in model.decoder(memory.cuda(), mels.cuda(), lens.cuda())]
    errs = output_errors(out, ref)
    print("teacher forcing [%s] B=%d: %s" % (impl_name, B, ", ".join("%s %.2e" % kv for kv in errs.items())))
    assert all(v < TOL for v in errs.values()), errs
    for b in range(B):
        assert int(torch.count_nonzero(out[2][b, :, int(lens[b]):])) == 0, b


def decoder_backward_case(Te, seed):
    """B = 3, T_mel = 6, training dropout masks, ragged memory lengths."""
    from tests.test_gpu_backward import decoder_case
    return decoder_case(3, Te, 6, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("Te", [257, BACKWARD_MAX_T_ENC])
def test_decoder_backward_near_its_encoder_length_limit(Te):
    from tests.test_gpu_backward import oracle_decoder_grads
    sd, sd64 = regime_weights()
    memory, mels, lens, pk, ak, dk, d_mel, d_gate, d_align = decoder_backward_case(Te, 500 + Te)
    ref_out, ref_g, ref_dmem = oracle_decoder_grads(sd64, memory.double(), mels.double(), lens, pk, ak, dk, d_mel.double(),
                                                    d_gate.double(), d_align.double(), True)
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    dec = model.cuda().train(True).decoder
    mem = memory.cuda().requires_grad_(True)
    with t2.dropout_masks(prenet=pk, att=ak, dec=dk):
        mel, gate, align = dec(mem, mels.cuda(), lens.cuda())
        ((mel * d_mel.cuda()).sum() + (gate * d_gate.cuda()).sum() + (align * d_align.cuda()).sum()).backward()
    torch.cuda.synchronize()
    fwd = output_errors((mel, gate, align), ref_out)
    errs = {"d_memory": rel_err(mem.grad, ref_dmem)}
    for k, p in dec.named_parameters():
        assert p.grad is not None, k
        errs[k] = rel_err(p.grad, ref_g["decoder." + k])
    worst = max(errs, key=errs.get)
    print("decoder backward T_enc=%d: forward %s; worst gradient %s %.2e" % (
        Te, ", ".join("%s %.2e" % kv for kv in fwd.items()), worst, errs[worst]))
    assert all(v < TOL for v in fwd.values()), fwd
    bad = {k: v for k, v in errs.items() if not v < GRAD_TOL}
    assert not bad, bad


@pytest.mark.gpu
def test_decoder_backward_refuses_encoder_length_409():
    Te = BACKWARD_MAX_T_ENC + 1
    sd, _ = regime_weights()
    memory, mels, lens, pk, ak, dk, d_mel, d_gate, _ = decoder_backward_case(Te, 500 + Te)
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    dec = model.cuda().train(True).decoder
    mem = memory.cuda().requires_grad_(True)
    with t2.dropout_masks(prenet=pk, att=ak, dec=dk):
        mel, gate, _ = dec(mem, mels.cuda(), lens.cuda())
        with pytest.raises(_capi.T2Error, match=r"T_enc ?= ?%d\b" % Te):
            ((mel * d_mel.cuda()).sum() + (gate * d_gate.cuda()).sum()).backward()
    assert mem.grad is None
