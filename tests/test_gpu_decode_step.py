"""The decoder step API -- Decoder.initialize_decoder_states / decode, Attention.forward / get_alignment_energies,
LocationLayer.forward -- against the reference's fixtures, the fp64 oracle step by step, and the stepwise decoder's bits.

Step by step, the oracle starts every step from the engine's own state (widened to fp64), so the bar of
tests/test_gpu_decoder_regimes.py (1e-4 of the largest magnitude) holds for one step however long the loop runs."""
import functools
import hashlib
import json
import os

import pytest
import torch

import tacotron2_b200 as t2
from oracle import tacotron2_oracle as O
from tacotron2_b200 import _capi
from tacotron2_b200.utils import get_mask_from_lengths
from tests.common import keep_mask, rel_err, synth_state_dict
from tests.test_oracle_golden import infer_inputs, load

TOL = 1e-4                  # one step vs the fp64 oracle (tests/test_gpu_decoder_regimes.py)
FIXTURE_TOL = 1e-3          # a whole loop vs the reference's fixtures (tests/test_gpu_parity.py)
STEP_LAUNCHES = 7           # 2 x (LSTM GEMM + pointwise), attention, projection GEMM, mel / gate split
DIGESTS = os.path.join(os.path.dirname(__file__), "golden", "decoder_stepwise_sha256.json")
STATE = ("attention_hidden", "attention_cell", "decoder_hidden", "decoder_cell", "attention_weights",
         "attention_weights_cum", "attention_context")
ORACLE_KEY = dict(attention_hidden="ah", attention_cell="ac", decoder_hidden="dh", decoder_cell="dc",
                  attention_weights="aw", attention_weights_cum="awc", attention_context="ctx")


def as_fp64(sd):
    return {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}


@functools.lru_cache(maxsize=None)
def weights():
    sd = synth_state_dict(41, scale=2.0)
    return sd, as_fp64(sd)


_models = {}


def make_model(sd, key, impl=_capi.IMPL_STEPWISE):
    if key not in _models:
        model = t2.Tacotron2(t2.create_hparams())
        model.load_state_dict(sd)
        _models[key] = model.cuda().eval()
    model = _models[key]
    model._t2_engine().impl = impl
    return model


def memory_of(B, T, seed):
    return torch.randn(B, T, 512, generator=torch.Generator().manual_seed(seed)).cuda()


def prenet_step(dec, x, keep_t):
    with t2.dropout_masks(prenet=keep_t[None]):
        return dec.prenet(x)


def oracle_state(dec, sd64):
    st = {ORACLE_KEY[k]: getattr(dec, k).detach().double().cpu() for k in STATE}
    st["pm"] = O.init_decoder_state(sd64, dec.memory.detach().double().cpu())["pm"]
    return st


def check_step_against_oracle(dec, sd64, x, mask=None, ak=None, dk=None):
    """decode(x) vs the oracle's decode_step from the same state: (largest error, decode()'s mel)."""
    st = oracle_state(dec, sd64)
    mem64 = dec.memory.detach().double().cpu()
    m64 = None if mask is None else mask.cpu()
    rmel, rgate, raw = O.decode_step(sd64, st, mem64, x.double().cpu(), m64,
                                     None if ak is None else ak.cpu(), None if dk is None else dk.cpu(),
                                     score_mask_value=float(dec.attention_layer.score_mask_value))
    mel, gate, aw = dec.decode(x)
    errs = [rel_err(mel.cpu(), rmel), rel_err(gate.cpu(), rgate), rel_err(aw.cpu(), raw)]
    errs += [rel_err(getattr(dec, k).cpu(), st[ORACLE_KEY[k]]) for k in STATE]
    return max(errs), mel


# ---------------------------------------------------------------------------------------------------------------------
# 1. the reference's own loop on its fixtures
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["infer_b1_t50", "infer_b4_t24", "infer_b3_t37"])
def test_reference_loop_matches_fixture(name):
    g = load(name)
    sd, _, keep, _ = infer_inputs(g)
    dec = make_model(sd, name).decoder
    memory = torch.from_numpy(g["memory"]).cuda()
    S = int(g["mel"].shape[2])
    mels, gates, aligns = [], [], []
    with torch.no_grad():
        dec.initialize_decoder_states(memory, None)
        x = dec.get_go_frame(memory)
        for t in range(S):
            mel, gate, aw = dec.decode(prenet_step(dec, x, keep[t]))
            mels.append(mel); gates.append(gate); aligns.append(aw)
            x = mel
        mel, gate, align = dec.parse_decoder_outputs(mels, gates, aligns)
    errs = [rel_err(mel.cpu(), torch.from_numpy(g["mel"])), rel_err(gate.cpu(), torch.from_numpy(g["gate"])),
            rel_err(align.cpu(), torch.from_numpy(g["align"]))]
    print("%s: mel %.2e gate %.2e align %.2e" % ((name,) + tuple(errs)))
    assert max(errs) < FIXTURE_TOL, errs


# ---------------------------------------------------------------------------------------------------------------------
# 2. the fp64 oracle, step by step
# ---------------------------------------------------------------------------------------------------------------------
CASES = [(1, 37, 100), (3, 150, 100), (64, 897, 100), (130, 1282, 100)]


@pytest.mark.gpu
@pytest.mark.parametrize("training", [False, True], ids=["eval", "train"])
@pytest.mark.parametrize("B,T,S", CASES, ids=["B%d-T%d" % (B, T) for B, T, _ in CASES])
def test_each_step_matches_oracle(B, T, S, training):
    sd, sd64 = weights()
    dec = make_model(sd, "w41").decoder
    dec.train(training)
    memory = memory_of(B, T, 7 * B + T)
    keep = keep_mask((S, 2, B, 256), 0.5, B + T)
    ak, dk = keep_mask((S, B, 1024), 0.1, 3 + T), keep_mask((S, B, 1024), 0.1, 4 + T)
    worst = 0.0
    try:
        with torch.no_grad():
            dec.initialize_decoder_states(memory, None)
            x = dec.get_go_frame(memory)
            for t in range(S):
                px = prenet_step(dec, x, keep[t])
                if training:
                    with t2.dropout_masks(att=ak[t], dec=dk[t]):
                        err, x = check_step_against_oracle(dec, sd64, px, None, ak[t], dk[t])
                else:
                    err, x = check_step_against_oracle(dec, sd64, px)
                worst = max(worst, err)
    finally:
        dec.train(False)
    print("B=%d T_enc=%d %s, %d steps: worst one-step error %.2e" % (B, T, "train" if training else "eval", S, worst))
    assert worst < TOL


# ---------------------------------------------------------------------------------------------------------------------
# 3. bits: the stepwise decoder's loop is a loop of decode()
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("training", [False, True], ids=["eval", "train"])
def test_decode_loop_equals_teacher_run_bit_for_bit(training):
    sd, _ = weights()
    model = make_model(sd, "w41")
    dec, eng = model.decoder, model._t2_engine()
    B, T, S = 5, 61, 24
    memory = memory_of(B, T, 61)
    px = torch.randn(S, B, 256, generator=torch.Generator().manual_seed(62)).relu().cuda()
    ak, dk = keep_mask((S, B, 1024), 0.1, 63), keep_mask((S, B, 1024), 0.1, 64)
    with torch.no_grad():
        mel, gate, align, _, _ = eng.decoder(memory, _capi.MODE_TEACHER, S, teacher_prenet=px, training=training,
                                             att_keep=ak, dec_keep=dk, impl=_capi.IMPL_STEPWISE)
        dec.train(training)
        try:
            dec.initialize_decoder_states(memory, None)
            outs = []
            for t in range(S):
                with t2.dropout_masks(att=ak[t], dec=dk[t]):
                    outs.append(dec.decode(px[t]))
        finally:
            dec.train(False)
    assert torch.equal(torch.stack([o[0] for o in outs], 1), mel)
    assert torch.equal(torch.stack([o[1][:, 0] for o in outs], 1), gate)
    assert torch.equal(torch.stack([o[2] for o in outs], 1), align)


@pytest.mark.gpu
def test_free_loop_equals_decoder_inference_bit_for_bit():
    sd, _ = weights()
    model = make_model(sd, "w41")
    dec = model.decoder
    B, T, S = 4, 45, 30
    memory = memory_of(B, T, 45)
    keep = keep_mask((S, 2, B, 256), 0.5, 46)
    dec.max_decoder_steps, dec.gate_threshold = S, 1.0
    with torch.no_grad():
        with t2.dropout_masks(prenet=keep):
            mel, gate, align = dec.inference(memory)
        dec.initialize_decoder_states(memory, None)
        x = dec.get_go_frame(memory)
        mels, gates, aligns = [], [], []
        for t in range(S):
            m, g, a = dec.decode(prenet_step(dec, x, keep[t]))
            mels.append(m); gates.append(g); aligns.append(a)
            x = m
        lm, lg, la = dec.parse_decoder_outputs(mels, gates, aligns)
    dec.max_decoder_steps, dec.gate_threshold = 1000, 0.5
    assert torch.equal(lm, mel) and torch.equal(lg, gate) and torch.equal(la, align)


def stepwise_digests():
    """sha256 of decoder_run_stepwise's outputs on seeded inputs: INFER with ragged memory lengths, TEACHER in training
    mode with Philox hidden-state dropout.  tools/stepwise_digests.py records them for a build."""
    sd, _ = weights()
    model = make_model(sd, "w41")
    eng = model._t2_engine()
    B, T, S = 6, 53, 20
    memory = memory_of(B, T, 53)
    lens = torch.tensor([53, 1, 20, 53, 37, 52], dtype=torch.int32).cuda()
    keep = keep_mask((S, 2, B, 256), 0.5, 54)
    px = torch.randn(S, B, 256, generator=torch.Generator().manual_seed(55)).relu().cuda()
    out = {}
    with torch.no_grad():
        mel, gate, align, ml, n = eng.decoder(memory, _capi.MODE_INFER, S, memory_lengths=lens, prenet_keep=keep,
                                              gate_threshold=1.0, impl=_capi.IMPL_STEPWISE, seed=77)
        out["infer"] = [mel, gate, align, ml, n]
        mel, gate, align, _, _ = eng.decoder(memory, _capi.MODE_TEACHER, S, memory_lengths=lens, teacher_prenet=px,
                                             training=True, impl=_capi.IMPL_STEPWISE, seed=78)
        out["teacher_train"] = [mel, gate, align]
    torch.cuda.synchronize()
    return {k: [hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest() for t in v] for k, v in out.items()}


@pytest.mark.gpu
def test_stepwise_run_keeps_its_bits():
    """The stepwise decoder computes what it computed before its loop body became decoder_step."""
    with open(DIGESTS) as f:
        assert stepwise_digests() == json.load(f)


# ---------------------------------------------------------------------------------------------------------------------
# 4. masks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_length_mask_rows_equal_their_own_loops():
    sd, _ = weights()
    dec = make_model(sd, "w41").decoder
    B, T, S = 4, 40, 12
    memory = memory_of(B, T, 40)
    lengths = torch.tensor([40, 7, 23, 1]).cuda()
    px = torch.randn(S, B, 256, generator=torch.Generator().manual_seed(41)).relu().cuda()

    def loop(mem, mask, x):
        dec.initialize_decoder_states(mem, mask)
        return [dec.decode(x[t]) for t in range(S)]
    with torch.no_grad():
        full = loop(memory, ~get_mask_from_lengths(lengths), px)
        for b in range(B):
            L = int(lengths[b])
            own = loop(memory[b:b + 1, :L].contiguous(), None, px[:, b:b + 1].contiguous())
            for t in range(S):
                assert torch.equal(full[t][0][b:b + 1], own[t][0]), (b, t)
                assert torch.equal(full[t][1][b:b + 1], own[t][1]), (b, t)
                assert torch.equal(full[t][2][b:b + 1, :L], own[t][2]), (b, t)
                assert float(full[t][2][b, L:].abs().max()) == 0.0 if L < T else True


@pytest.mark.gpu
def test_non_suffix_mask_matches_oracle():
    sd, sd64 = weights()
    dec = make_model(sd, "w41").decoder
    B, T = 3, 50
    memory = memory_of(B, T, 50)
    mask = torch.zeros(B, T, dtype=torch.bool)
    mask[0, 5:9] = True
    mask[1, ::3] = True
    mask[2, :30] = True
    mask = mask.cuda()
    px = torch.randn(10, B, 256, generator=torch.Generator().manual_seed(51)).relu().cuda()
    with torch.no_grad():
        dec.initialize_decoder_states(memory, mask)
        worst = max(check_step_against_oracle(dec, sd64, px[t], mask)[0] for t in range(10))
        assert float(dec.attention_weights.masked_select(mask).abs().max()) == 0.0
    assert worst < TOL, worst


# ---------------------------------------------------------------------------------------------------------------------
# 5. state edits and aliasing
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_edits_between_steps_and_aliasing():
    sd, sd64 = weights()
    dec = make_model(sd, "w41").decoder
    B, T = 2, 33
    memory = memory_of(B, T, 33)
    px = torch.randn(4, B, 256, generator=torch.Generator().manual_seed(34)).relu().cuda()
    with torch.no_grad():
        dec.initialize_decoder_states(memory, None)
        cum = dec.attention_weights_cum
        mel0, gate0, aw0 = dec.decode(px[0])
        assert aw0 is dec.attention_weights and dec.attention_weights_cum is cum
        kept = [t.clone() for t in (mel0, gate0, aw0)]
        stored = {k: getattr(dec, k) for k in STATE}
        stored_vals = {k: v.clone() for k, v in stored.items() if k != "attention_weights_cum"}
        dec.decode(px[1])
        assert dec.attention_weights_cum is cum
        assert all(torch.equal(a, b) for a, b in zip((mel0, gate0, aw0), kept))
        assert all(torch.equal(stored[k], v) for k, v in stored_vals.items())
        # edits: steer the attention to position 20, replace the context
        dec.attention_weights_cum.zero_()
        dec.attention_weights_cum[:, 20] = 1.0
        dec.attention_context = torch.randn(B, 512, generator=torch.Generator().manual_seed(35)).cuda()
        err, _ = check_step_against_oracle(dec, sd64, px[2])
    assert err < TOL, err


# ---------------------------------------------------------------------------------------------------------------------
# 6. sub-module forwards and half models
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_attention_submodules_match_oracle_and_decode():
    sd, sd64 = weights()
    dec = make_model(sd, "w41").decoder
    att = dec.attention_layer
    B, T = 3, 70
    memory = memory_of(B, T, 70)
    g = torch.Generator().manual_seed(71)
    q = torch.randn(B, 1024, generator=g).cuda()
    cat = torch.rand(B, 2, T, generator=g).cuda()
    mask = torch.zeros(B, T, dtype=torch.bool).cuda()
    mask[1, 60:] = True
    with torch.no_grad():
        dec.initialize_decoder_states(memory, None)
        pm = dec.processed_memory
        pm64 = O.init_decoder_state(sd64, memory.double().cpu())["pm"]
        assert rel_err(pm.cpu(), pm64) < TOL
        loc = att.location_layer(cat)
        assert rel_err(loc.cpu(), O.location_layer(sd64, cat.double().cpu())) < TOL
        e = att.get_alignment_energies(q, pm, cat)
        assert rel_err(e.cpu(), O.alignment_energies(sd64, q.double().cpu(), pm64, cat.double().cpu())) < TOL
        ctx, w = att(q, memory, pm, cat, mask)
        rctx, rw = O.attention(sd64, q.double().cpu(), memory.double().cpu(), pm64, cat.double().cpu(), mask.cpu())
        assert rel_err(ctx.cpu(), rctx) < TOL and rel_err(w.cpu(), rw) < TOL
        # on decode()'s own inputs of a step: its weights and context, bit for bit
        dec.decode(torch.randn(B, 256, generator=g).relu().cuda())
        prev = torch.stack((dec.attention_weights, dec.attention_weights_cum.clone()), 1)
        x = torch.randn(B, 256, generator=g).relu().cuda()
        dec.decode(x)
        ctx, w = att(dec.attention_hidden, memory, pm, prev, None)
        assert torch.equal(w, dec.attention_weights) and torch.equal(ctx, dec.attention_context)


@pytest.mark.gpu
def test_half_model_returns_and_stores_half():
    sd, sd64 = weights()
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    dec = model.cuda().half().eval().decoder
    memory = memory_of(2, 30, 30).half()
    with torch.no_grad():
        dec.initialize_decoder_states(memory, None)
        cum = dec.attention_weights_cum
        x = dec.prenet(dec.get_go_frame(memory))
        mel, gate, aw = dec.decode(x)
    assert mel.dtype == gate.dtype == aw.dtype == torch.float16
    assert all(getattr(dec, k).dtype == torch.float16 for k in STATE) and dec.attention_weights_cum is cum
    assert float(cum.float().sum(1).sub(1).abs().max()) < 1e-2


# ---------------------------------------------------------------------------------------------------------------------
# 7. cost, buffers, refusals
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_launch_count_per_step_is_constant():
    sd, _ = weights()
    dec = make_model(sd, "w41").decoder
    L = _capi.lib()
    counts = []
    for B, T in ((1, 20), (64, 300), (130, 1282)):
        memory = memory_of(B, T, B)
        with torch.no_grad():
            dec.initialize_decoder_states(memory, None)
            x = torch.zeros(B, 256).cuda()
            for _ in range(3):
                n0 = L.t2_kernel_launch_count()
                dec.decode(x)
                counts.append(L.t2_kernel_launch_count() - n0)
    assert counts == [STEP_LAUNCHES] * len(counts), counts


def guarded(shapes, G=4096):
    """Views of the given shapes in one NaN-filled fp32 buffer: each ends exactly where a guard region of >= G floats
    begins, and each starts 16-byte aligned (the step's contract)."""
    starts, off = [], G
    for a, b in shapes:
        starts.append(off)
        off = -(-(off + a * b + G) // 4) * 4
    buf = torch.full((off,), float("nan"), device="cuda")
    return buf, [buf[o:o + a * b].view(a, b) for o, (a, b) in zip(starts, shapes)]


@pytest.mark.gpu
def test_step_writes_stay_inside_exact_size_buffers():
    """Every state and output array of t2_decoder_step sits between NaN guard regions; the step writes none of them."""
    sd, _ = weights()
    eng = make_model(sd, "w41")._t2_engine()
    B, T = 3, 29
    shapes = [(B, 1024)] * 4 + [(B, T), (B, T), (B, 512)]
    buf, views = guarded(shapes)
    inside = torch.zeros_like(buf, dtype=torch.bool)
    for v in views:
        v.zero_()
        o = (v.data_ptr() - buf.data_ptr()) // 4
        inside[o:o + v.numel()] = True
    memory = memory_of(B, T, 29)
    with torch.no_grad():
        pm = eng.processed_memory(memory)
        mel, gate = eng.decoder_step(memory, pm, None, views, torch.rand(B, 256).cuda(), False, None, None, 0,
                                     -float("inf"))
    torch.cuda.synchronize()
    assert bool(buf[~inside].isnan().all())
    assert not bool(buf[inside].isnan().any())
    assert mel.shape == (B, 80) and gate.shape == (B, 1)


@pytest.mark.gpu
def test_library_refusals_launch_nothing():
    sd, _ = weights()
    eng = make_model(sd, "w41")._t2_engine()
    L = _capi.lib()
    B = 2
    f = lambda *s: torch.zeros(*s, device="cuda")
    T = 1283
    state = [f(B, 1024)] * 4 + [f(B, T)] * 2 + [f(B, 512)]
    n0 = L.t2_kernel_launch_count()
    with pytest.raises(_capi.T2Error, match=r"error -4: .*T_enc=1283"):
        eng.decoder_step(f(B, T, 512), f(B, T, 128), None, state, f(B, 256), False, None, None, 0, -float("inf"))
    assert L.t2_kernel_launch_count() == n0
    state = [f(B, 1024)] * 4 + [f(B, 10)] * 2 + [f(B, 512)]
    odd = f(B * 256 + 1)[1:].view(B, 256)                  # 4 bytes past a 16-byte boundary
    with pytest.raises(_capi.T2Error, match="16-byte aligned"):
        eng.decoder_step(f(B, 10, 512), f(B, 10, 128), None, state, odd, False, None, None, 0, -float("inf"))
    assert L.t2_kernel_launch_count() == n0
    a = _capi.T2DecoderStepArgs()
    a.B, a.T_enc = 2, 0
    with pytest.raises(_capi.T2Error, match=r"error -1: .*T_enc=0"):
        _capi.call(L.t2_decoder_step, eng.device, eng.handle, C_byref(a))
    a.T_enc = 10
    with pytest.raises(_capi.T2Error, match="null tensor pointer"):
        _capi.call(L.t2_decoder_step, eng.device, eng.handle, C_byref(a))
    att = _capi.T2AttentionArgs()
    att.B, att.T_enc = 2, 10
    with pytest.raises(_capi.T2Error, match="attention"):
        _capi.call(L.t2_attention_forward, eng.device, eng.handle, C_byref(att))
    assert L.t2_kernel_launch_count() == n0


def C_byref(x):
    import ctypes
    return ctypes.byref(x)
