"""Streaming inference (Tacotron2.inference_stream / Decoder.inference_stream) against inference().

The persistent decoder runs in chunks that stop at a step boundary and resume from a per-stream state buffer; its dropout
is keyed by the absolute step.  So a stream must reproduce inference() bit for bit: mel, postnet, gate, alignments and
lengths, for any chunk size.  Each item must carry exactly the frames that are final at the end of its chunk: every
frame up to the steps run less 10 (the postnet's reach) while a row is live, and everything once every 64-row slice has
stopped (``expected_ranges``).  One small case is tied to the fp64 oracle as well."""
import ctypes
import functools

import pytest
import torch

import tacotron2_b200 as t2
from oracle import tacotron2_oracle as O
from tacotron2_b200 import _capi, _engine
from tests.common import keep_mask, rand_text, rel_err, synth_state_dict

HALO = 10
PERSISTENT_MAX_T_ENC = 2274


def expected_ranges(chunk, ends, halo):
    """Frame ranges of the items of a stream whose 64-row slices stop after ends[s] steps (their longest row, or the cap)."""
    ranges, t0, k = [], 0, 0
    while True:
        k += 1
        steps = k * chunk
        live = [e for e in ends if steps < e]
        t1 = max(ends) if not live else max(t0, steps - halo)
        if t1 > t0 or not live:
            ranges.append((t0, t1))
        if not live:
            return ranges
        t0 = t1


def test_expected_ranges_follow_the_finality_rule():
    assert expected_ranges(32, [800], HALO)[:2] == [(0, 22), (22, 54)]
    assert expected_ranges(7, [40], HALO) == [(0, 4), (4, 11), (11, 18), (18, 25), (25, 40)]
    assert expected_ranges(40, [40], HALO) == [(0, 40)]
    assert expected_ranges(5, [12, 30], HALO) == [(0, 5), (5, 10), (10, 15), (15, 30)]


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
_models = {}


def make_model(key, sd):
    if key not in _models:
        model = t2.Tacotron2(t2.create_hparams())
        model.load_state_dict(sd)
        _models[key] = model.cuda().eval()
    return _models[key]


@functools.lru_cache(maxsize=None)
def weights(seed=7, gate_sign=10.0):
    return synth_state_dict(seed, gate_bias=0.0, gate_sign=gate_sign, scale=2.0)


def set_decoder(model, steps, threshold, impl=_capi.IMPL_AUTO):
    model._t2_engine().impl = impl
    model.decoder.max_decoder_steps = steps
    model.decoder.gate_threshold = threshold


def run_inference(model, text, keep, seed_at=None):
    if seed_at is not None:
        _engine._seed_counter[0] = seed_at
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        out = [o.clone() for o in model.inference(text.cuda())]
    return out, model.mel_lengths.clone()


def run_stream(model, text, keep, chunk, seed_at=None):
    if seed_at is not None:
        _engine._seed_counter[0] = seed_at
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        items = list(model.inference_stream(text.cuda(), chunk_steps=chunk))
    return items


KEYS = ("mel_outputs", "mel_outputs_postnet", "gate_outputs", "alignments")
DIMS = (2, 2, 1, 1)


def check_stream(items, ref, ref_lengths, chunk, halo=HALO, keys=KEYS, dims=DIMS):
    """Bit-identical concatenation, the finality rule and the per-item lengths."""
    B = ref_lengths.shape[0]
    ends = [int(ref_lengths[b0:b0 + 64].max()) for b0 in range(0, B, 64)]
    assert [it["frames"] for it in items] == expected_ranges(chunk, ends, halo), ([it["frames"] for it in items], ends)
    assert [it["finished"] for it in items] == [False] * (len(items) - 1) + [True]
    for k, d, r in zip(keys, dims, ref):
        got = torch.cat([it[k] for it in items], dim=d)
        assert got.dtype == r.dtype and got.shape == r.shape, (k, got.shape, r.shape)
        assert torch.equal(got, r), (k, float((got.double() - r.double()).abs().max()))
    final = ref_lengths.cpu()
    for it in items:
        ml = it["mel_lengths"].cpu()
        assert ml.dtype == torch.int32 and it["mel_lengths"].is_cuda
        live = ml == -1
        assert torch.equal(ml[~live], final[~live])
        assert bool((final[live] > it["frames"][1]).all())
    assert torch.equal(items[-1]["mel_lengths"].cpu(), final)


def stop_threshold(model, text, keep, steps, want):
    """A gate threshold under which the rows' first firing steps satisfy want(lengths); found from the gate logits of a run
    in which no row stops (the gate is not fed back, so the logits do not depend on the threshold)."""
    set_decoder(model, steps, 1.0)
    (_, _, gate, _), _ = run_inference(model, text, keep)
    logits = gate[:, :, 0].double().cpu()
    running = torch.cummax(logits, dim=1).values
    vals = torch.unique(running.flatten()).tolist()
    for lo, hi in sorted(zip(vals[:-1], vals[1:]), key=lambda p: p[0] - p[1]):     # widest gaps first
        theta = (lo + hi) / 2
        fired = running > theta
        lengths = torch.where(fired.any(1), fired.int().argmax(1) + 1, torch.full((logits.shape[0],), steps))
        if want(lengths):
            return float(torch.sigmoid(torch.tensor(theta)))
    raise AssertionError("no threshold gives the wanted stops")


# ---------------------------------------------------------------------------------------------------------------------
# 1. every row live to the cap, across chunk sizes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,T", [(1, 50), (64, 37)], ids=["B1", "B64"])
@pytest.mark.parametrize("chunk", [1, 7, 32, 45], ids=["c1", "c7", "c32", "cap"])
def test_stream_equals_inference_when_no_row_fires(B, T, chunk, capsys):
    """gate_threshold = 1: every row runs to max_decoder_steps = 45 (not a multiple of 7 or 32); the warning is printed
    after the last item exactly as inference() prints it."""
    S = 45
    model = make_model("w7", weights())
    set_decoder(model, S, 1.0)
    text, keep = rand_text(B, T, B + T), keep_mask((S, 2, B, 256), 0.5, B)
    ref, ref_lengths = run_inference(model, text, keep)
    warned = capsys.readouterr().out.count("Reached max decoder steps")
    items = run_stream(model, text, keep, chunk)
    assert capsys.readouterr().out.count("Reached max decoder steps") == warned == 1
    check_stream(items, ref, ref_lengths, chunk)
    assert torch.equal(model.mel_lengths, ref_lengths) and ref_lengths.tolist() == [S] * B


# ---------------------------------------------------------------------------------------------------------------------
# 2. rows that stop at different steps; chunk boundaries at, before and after a stop
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def ragged_b3():
    B, T, S = 3, 41, 60
    model = make_model("w7", weights())
    text, keep = rand_text(B, T, 5), keep_mask((S, 2, B, 256), 0.5, 6)
    thr = stop_threshold(model, text, keep, S, lambda L: len(set(L.tolist())) == 3 and int(L.max()) < S and
                         int(L.min()) >= 12)
    set_decoder(model, S, thr)
    ref, lengths = run_inference(model, text, keep)
    return dict(S=S, text=text, keep=keep, thr=thr, ref=ref, lengths=lengths)


def ragged_chunks():
    # resolved lazily on the GPU: "first" = the earliest stop, "last" = the slice's end; +-1 around both
    return ["first-1", "first", "first+1", "last-1", "last", "last+1", 1, 7, 32, "cap"]


@pytest.mark.gpu
@pytest.mark.parametrize("chunk_spec", ragged_chunks(), ids=[str(c) for c in ragged_chunks()])
def test_stream_with_rows_stopping_at_different_steps(chunk_spec):
    c = ragged_b3()
    model = make_model("w7", weights())
    set_decoder(model, c["S"], c["thr"])
    L = sorted(c["lengths"].tolist())
    if isinstance(chunk_spec, int):
        chunk = chunk_spec
    elif chunk_spec == "cap":
        chunk = c["S"]
    else:
        base = L[0] if chunk_spec.startswith("first") else L[-1]
        chunk = base + (int(chunk_spec[-2:]) if chunk_spec[-2] in "+-" else 0)
    items = run_stream(model, c["text"], c["keep"], chunk)
    print("B=3 stops at %s, chunk %d: items %s" % (L, chunk, [it["frames"] for it in items]))
    check_stream(items, c["ref"], c["lengths"], chunk)


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [1, 7, 32, "end0", 60], ids=["c1", "c7", "c32", "slice0-end", "cap"])
def test_stream_over_two_slices_that_stop_at_different_steps(chunk, monkeypatch, capfd):
    """B = 65: rows 0-63 and row 64 run as two launches per chunk; the slice that stopped first is not launched again."""
    B, T, S = 65, 23, 60
    model = make_model("w7", weights())
    text, keep = rand_text(B, T, 65), keep_mask((S, 2, B, 256), 0.5, 66)
    thr = stop_threshold(model, text, keep, S, lambda L: int(L[64]) < S and min(int(L[:64].max()), int(L[64])) >= 15 and
                         abs(int(L[:64].max()) - int(L[64])) >= 3)
    set_decoder(model, S, thr)
    ref, lengths = run_inference(model, text, keep)
    ends = [int(lengths[:64].max()), int(lengths[64])]
    if chunk == "end0":
        chunk = ends[0]
    monkeypatch.setenv("T2_VERBOSE", "1")
    capfd.readouterr()
    items = run_stream(model, text, keep, chunk)
    err = capfd.readouterr().err
    launches = [err.count("persistent decoder: B=64 "), err.count("persistent decoder: B=1 ")]
    print("B=65 slices end at %s, chunk %d: %d items, decoder launches per slice %s" % (ends, chunk, len(items), launches))
    check_stream(items, ref, lengths, chunk)
    assert launches == [(e + chunk - 1) // chunk for e in ends]


@pytest.mark.gpu
def test_stream_with_a_row_that_never_fires_and_a_cap_off_the_chunk_grid(capsys):
    B, T, S = 3, 33, 47
    model = make_model("w7", weights())
    text, keep = rand_text(B, T, 9), keep_mask((S, 2, B, 256), 0.5, 10)
    thr = stop_threshold(model, text, keep, S, lambda L: bool((L == S).any()) and int(L.min()) < S - 5)
    set_decoder(model, S, thr)
    capsys.readouterr()
    ref, lengths = run_inference(model, text, keep)
    print("B=3, cap %d: lengths %s" % (S, lengths.tolist()))
    assert capsys.readouterr().out.count("Reached max decoder steps") == 1
    for chunk in (7, 32):
        items = run_stream(model, text, keep, chunk)
        assert capsys.readouterr().out.count("Reached max decoder steps") == 1
        check_stream(items, ref, lengths, chunk)
        assert torch.equal(model.mel_lengths, lengths)


# ---------------------------------------------------------------------------------------------------------------------
# 3. encoder lengths across the decoder's shared-memory regimes (Decoder.inference_stream)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("T", [94, 95, 900, PERSISTENT_MAX_T_ENC])
def test_decoder_stream_across_encoder_length_regimes(T):
    B, S, chunk = 2, 12, 5
    model = make_model("w7", weights())
    set_decoder(model, S, 1.0)
    memory = torch.randn(B, T, 512, generator=torch.Generator().manual_seed(T)).cuda()
    keep = keep_mask((S, 2, B, 256), 0.5, T)
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        ref = [o.clone() for o in model.decoder.inference(memory)]
        lengths = model.decoder.mel_lengths.clone()
        items = list(model.decoder.inference_stream(memory, chunk_steps=chunk))
    check_stream(items, ref, lengths, chunk, halo=0, keys=KEYS[:1] + KEYS[2:], dims=DIMS[:1] + DIMS[2:])
    assert [it["frames"] for it in items] == [(0, 5), (5, 10), (10, 12)]


# ---------------------------------------------------------------------------------------------------------------------
# 4. in-kernel Philox dropout, a .half() model
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_stream_with_in_kernel_philox_dropout():
    B, T, S, chunk = 3, 29, 40, 9
    model = make_model("w7", weights())
    set_decoder(model, S, 1.0)
    text = rand_text(B, T, 11)
    at = _engine._seed_counter[0] + 100
    ref, lengths = run_inference(model, text, None, seed_at=at)
    items = run_stream(model, text, None, chunk, seed_at=at)
    check_stream(items, ref, lengths, chunk)
    other = run_stream(model, text, None, chunk, seed_at=at + 50)      # another seed: other dropout, other frames
    assert not torch.equal(torch.cat([it["mel_outputs"] for it in other], 2), ref[0])


@pytest.mark.gpu
def test_stream_of_a_half_model():
    B, T, S, chunk = 2, 31, 30, 8
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(weights())
    model = model.cuda().eval().half()
    set_decoder(model, S, 1.0)
    text, keep = rand_text(B, T, 12), keep_mask((S, 2, B, 256), 0.5, 13)
    ref, lengths = run_inference(model, text, keep)
    assert ref[0].dtype == torch.float16
    items = run_stream(model, text, keep, chunk)
    check_stream(items, ref, lengths, chunk)


# ---------------------------------------------------------------------------------------------------------------------
# 5. independent streams
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_two_interleaved_streams_each_equal_their_own_inference():
    S, chunk = 50, 6
    model = make_model("w7", weights())
    set_decoder(model, S, 1.0)
    cases = [(rand_text(3, 27, 21), keep_mask((S, 2, 3, 256), 0.5, 22)),
             (rand_text(70, 19, 23), keep_mask((S, 2, 70, 256), 0.5, 24))]
    refs = [run_inference(model, text, keep) for text, keep in cases]
    gens, items = [], [[], []]
    for text, keep in cases:
        with t2.dropout_masks(prenet=keep):
            gens.append(model.inference_stream(text.cuda(), chunk_steps=chunk))
    with torch.no_grad():
        live = [0, 1]
        while live:
            for i in list(live):
                with t2.dropout_masks(prenet=cases[i][1]):
                    try:
                        items[i].append(next(gens[i]))
                    except StopIteration:
                        live.remove(i)
    for i in range(2):
        check_stream(items[i], refs[i][0], refs[i][1], chunk)


@pytest.mark.gpu
def test_abandoned_stream_leaves_the_model_clean():
    """A stream closed after two items: the next inference() is bit-identical to one on a fresh model."""
    S, B, T = 40, 4, 25
    sd = weights()
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    model = model.cuda().eval()
    set_decoder(model, S, 1.0)
    text, keep = rand_text(B, T, 31), keep_mask((S, 2, B, 256), 0.5, 32)
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        gen = model.inference_stream(rand_text(B, T, 33).cuda(), chunk_steps=16)
        assert not next(gen)["finished"] and not next(gen)["finished"]
        gen.close()
    out, lengths = run_inference(model, text, keep)
    fresh = t2.Tacotron2(t2.create_hparams())
    fresh.load_state_dict(sd)
    fresh = fresh.cuda().eval()
    set_decoder(fresh, S, 1.0)
    ref, ref_lengths = run_inference(fresh, text, keep)
    assert all(torch.equal(a, b) for a, b in zip(out, ref)) and torch.equal(lengths, ref_lengths)


# ---------------------------------------------------------------------------------------------------------------------
# 6. refusals
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_stream_refusals():
    model = make_model("w7", weights())
    set_decoder(model, 8, 1.0, impl=_capi.IMPL_STEPWISE)
    with torch.no_grad():
        with pytest.raises(_capi.T2Error, match="STEPWISE"):
            next(model.inference_stream(rand_text(1, 20, 1).cuda()))
        set_decoder(model, 8, 1.0)
        memory = torch.randn(1, PERSISTENT_MAX_T_ENC + 1, 512).cuda()
        with pytest.raises(_capi.T2Error, match=r"T_enc=%d\b" % (PERSISTENT_MAX_T_ENC + 1)):
            next(model.decoder.inference_stream(memory))
        with pytest.raises(ValueError):
            next(model.inference_stream(rand_text(1, 20, 1).cuda(), chunk_steps=0))
        model.train()
        try:
            with pytest.raises(RuntimeError, match="eval mode"):
                next(model.inference_stream(rand_text(1, 20, 1).cuda()))
        finally:
            model.eval()
        # the run call itself refuses the same way, whatever begin accepted
        eng = model._t2_engine()
        st = eng.decoder_stream(torch.randn(2, 30, 512).cuda(), 8)
        L = _capi.lib()
        st.args.dec.impl = _capi.IMPL_STEPWISE
        rc = L.t2_decoder_stream_run(eng.handle, ctypes.byref(st.args), 4, None, eng._stream())
        assert rc == -4 and b"STEPWISE" in L.t2_last_error()
        st.args.dec.impl = _capi.IMPL_AUTO
        st.args.dec.T_enc = PERSISTENT_MAX_T_ENC + 1
        rc = L.t2_decoder_stream_run(eng.handle, ctypes.byref(st.args), 4, None, eng._stream())
        assert rc == -4 and b"T_enc=%d" % (PERSISTENT_MAX_T_ENC + 1) in L.t2_last_error()
        st.args.dec.T_enc = 30
        assert st.run(8)[2]                       # still usable: 8 steps = the cap
    text, keep = rand_text(2, 20, 2), keep_mask((8, 2, 2, 256), 0.5, 3)
    ref, lengths = run_inference(model, text, keep)
    check_stream(run_stream(model, text, keep, 3), ref, lengths, 3)


# ---------------------------------------------------------------------------------------------------------------------
# 7. tied to the reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_stream_against_the_oracle():
    B, T, S, chunk = 2, 19, 24, 7
    sd = synth_state_dict(5, gate_bias=-10.0, scale=2.0)
    model = make_model("oracle", sd)
    set_decoder(model, S, 0.5)
    text, keep = rand_text(B, T, 3), keep_mask((S, 2, B, 256), 0.5, 4)
    with torch.no_grad():
        ref = O.tacotron2_inference(sd, text, keep, 0.5, S)
    items = run_stream(model, text, keep, chunk)
    out = [torch.cat([it[k] for it in items], dim=d) for k, d in zip(KEYS, DIMS)]
    errs = {k: rel_err(a, b) for k, a, b in zip(KEYS, out, ref[:4])}
    print("stream vs oracle: %s" % ", ".join("%s %.2e" % kv for kv in errs.items()))
    assert all(v < 1e-3 for v in errs.values()), errs
    assert model.mel_lengths.cpu().tolist() == ref[4].tolist()
