"""Batched inference over texts of different lengths (``input_lengths``): every row of a ragged batch equals, bit for bit,
the same model's inference on that row's text alone.

A row of length L inside a batch sized for T_text may run in another shared-memory regime of the persistent decoder than
its own B = 1 call (4 ring stages with every memory row staged up to T_enc = 94, rows 0-93 staged up to 896, a 3-stage
ring with rows 0-57 staged beyond), on other 64-row slices, and through the encoder's other BiLSTM kernel (B > 64).  The
checks below cover each of those, the .half() model, the stream and the host entry point, and compare the ragged batch
with the reference's own B = 1 inference (tests/golden/infer_ragged_b4_t40.npz, tools/make_golden.py ragged)."""
import os

import numpy as np
import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tests.common import GOLDEN_DIR, keep_mask, rand_text, rel_err, synth_state_dict

pytestmark = pytest.mark.gpu
HOP = 256


def make_model(sd, steps, threshold=0.5, half=False, impl=None):
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    model = model.cuda().eval()
    if half:
        model = model.half()
    model.decoder.max_decoder_steps = steps
    model.decoder.gate_threshold = threshold
    if impl is not None:
        model._t2_engine().impl = impl
    return model


def infer(model, text, keep, lengths=None):
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        out = [o.clone() for o in model.inference(text.cuda(), input_lengths=lengths)]
    return out, model.mel_lengths.clone()


def alone(model, text, keep, b, L):
    """Row b's text alone: inference(text[b:b+1, :L]) with its slice of the prenet masks."""
    return infer(model, text[b:b + 1, :L], keep[:, :, b:b + 1].contiguous())


def check_row(batch, batch_lengths, one, one_lengths, b, L):
    mel, post, gate, align = batch
    m1, p1, g1, a1 = one
    n1 = int(one_lengths[0])
    assert m1.shape[2] == n1 and int(batch_lengths[b]) == n1, (b, n1, int(batch_lengths[b]))
    assert torch.equal(mel[b, :, :n1], m1[0]), b
    assert torch.equal(post[b, :, :n1], p1[0]), b
    assert torch.equal(gate[b, :n1], g1[0]), b
    assert torch.equal(align[b, :n1, :L], a1[0, :, :L]), b
    assert not bool(mel[b, :, n1:].any()) and not bool(post[b, :, n1:].any())
    assert not bool(align[b, :, L:].any()), b


def threshold_for(model, text, keep, lengths, steps):
    """A gate threshold under which the rows stop at different steps: the median of the running maximum of the gate
    logits of a run in which no row stops (the gate is not fed back, so the logits do not depend on the threshold)."""
    model.decoder.gate_threshold = 1.0
    (_, _, gate, _), _ = infer(model, text, keep, lengths)
    running = torch.cummax(gate[:, :, 0].float().cpu(), dim=1).values
    return float(torch.sigmoid(running[:, steps // 2].median()))


def ragged_text(lengths, seed):
    """(B, max L) ids; the positions past each row's length hold other ids (garbage the engine must ignore)."""
    return rand_text(len(lengths), max(lengths), seed)


# ---------------------------------------------------------------------------------------------------------------------
# 1. per-row identity across the decoder's staging regimes, fp32 and .half()
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("half", [False, True], ids=["fp32", "half"])
def test_rows_equal_their_own_b1_runs(half):
    lengths = [95, 1, 150, 37, 94]                 # shuffled: no ordering is required
    S = 60
    text, keep = ragged_text(lengths, 11), keep_mask((S, 2, len(lengths), 256), 0.5, 12)
    model = make_model(synth_state_dict(7, gate_bias=0.0, gate_sign=10.0, scale=2.0), S, half=half)
    L = torch.tensor(lengths)
    model.decoder.gate_threshold = threshold_for(model, text, keep, L, S)
    batch, bl = infer(model, text, keep, L)
    print("half=%s lengths %s -> mel lengths %s" % (half, lengths, bl.tolist()))
    for b, Lb in enumerate(lengths):
        one, ol = alone(model, text, keep, b, Lb)
        check_row(batch, bl, one, ol, b, Lb)
    assert len(set(bl.tolist())) > 1


@pytest.mark.parametrize("lengths", [[50, 900, 94], [95, 2274, 60]], ids=["T900-3stage", "T2274"])
def test_short_rows_in_a_long_batch(lengths):
    """The longest row puts the batch in the 3-stage ring (rows 0-57 staged); the short rows run alone with 4 stages."""
    S = 12
    text, keep = ragged_text(lengths, 21), keep_mask((S, 2, len(lengths), 256), 0.5, 22)
    model = make_model(synth_state_dict(7, gate_bias=-30.0, scale=2.0), S)
    batch, bl = infer(model, text, keep, torch.tensor(lengths))
    for b, Lb in enumerate(lengths):
        if Lb != max(lengths):
            one, ol = alone(model, text, keep, b, Lb)
            check_row(batch, bl, one, ol, b, Lb)


def test_rows_across_64_row_slices():
    """B = 130: three decoder launches and the encoder's stepped BiLSTM; rows 0, 63, 64, 129 against their B = 1 runs."""
    B, S = 130, 10
    lengths = torch.randint(1, 81, (B,), generator=torch.Generator().manual_seed(3))
    lengths[[0, 63, 64, 129]] = torch.tensor([80, 7, 80, 41])
    text, keep = rand_text(B, 80, 31), keep_mask((S, 2, B, 256), 0.5, 32)
    model = make_model(synth_state_dict(7, gate_bias=0.0, gate_sign=10.0, scale=2.0), S)
    model.decoder.gate_threshold = threshold_for(model, text, keep, lengths, S)
    batch, bl = infer(model, text, keep, lengths.cuda())
    for b in (0, 63, 64, 129):
        one, ol = alone(model, text, keep, b, int(lengths[b]))
        check_row(batch, bl, one, ol, b, int(lengths[b]))


def test_stepwise_decoder_rows_equal_their_own_runs():
    """The stepwise implementation takes the same lengths; its softmax and context sum positions in a fixed order, so it
    is bit-exact per row too."""
    lengths, S = [33, 8, 20], 16
    text, keep = ragged_text(lengths, 41), keep_mask((S, 2, 3, 256), 0.5, 42)
    model = make_model(synth_state_dict(7, gate_bias=-30.0, scale=2.0), S, impl=_capi.IMPL_STEPWISE)
    batch, bl = infer(model, text, keep, torch.tensor(lengths))
    for b, Lb in enumerate(lengths):
        one, ol = alone(model, text, keep, b, Lb)
        check_row(batch, bl, one, ol, b, Lb)


def test_encoder_memory_is_zero_past_each_length():
    lengths = torch.tensor([5, 12, 1])
    model = make_model(synth_state_dict(7), 4)
    text = rand_text(3, 12, 51).cuda()
    with torch.no_grad():
        emb = model.embedding(text).transpose(1, 2)
        mem = model.encoder.inference(emb, input_lengths=lengths)
        for b, L in enumerate(lengths.tolist()):
            assert torch.equal(mem[b, :L], model.encoder.inference(emb[b:b + 1, :, :L])[0])
            assert not bool(mem[b, L:].any())


# ---------------------------------------------------------------------------------------------------------------------
# 2. no lengths, or every length = T_text: today's outputs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [40, 300], ids=["4stage-staged", "4stage-L2"])
def test_full_lengths_equal_no_lengths(T):
    B, S = 3, 20
    text, keep = rand_text(B, T, 61), keep_mask((S, 2, B, 256), 0.5, 62)
    model = make_model(synth_state_dict(7, gate_bias=0.0, gate_sign=10.0, scale=2.0), S)
    model.decoder.gate_threshold = threshold_for(model, text, keep, None, S)
    a, al = infer(model, text, keep)
    b, bl = infer(model, text, keep, torch.full((B,), T))
    assert torch.equal(al, bl)
    for k, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), k


# ---------------------------------------------------------------------------------------------------------------------
# 3. against the reference's own B = 1 inference
# ---------------------------------------------------------------------------------------------------------------------
def test_ragged_batch_matches_reference_b1_runs():
    g = np.load(os.path.join(GOLDEN_DIR, "infer_ragged_b4_t40.npz"))
    B, T, S = int(g["B"]), int(g["T_text"]), int(g["max_steps"])
    sd = synth_state_dict(int(g["wseed"]), gate_bias=float(g["gate_bias"]), scale=float(g["wscale"]),
                          gate_sign=float(g["gate_sign"]))
    text, keep = rand_text(B, T, int(g["tseed"])), keep_mask((S, 2, B, 256), 0.5, int(g["mseed"]))
    lengths = torch.from_numpy(g["input_lengths"])
    model = make_model(sd, S)
    (mel, post, gate, align), ml = infer(model, text, keep, lengths)
    assert ml.cpu().tolist() == g["mel_lengths"].tolist()                       # stop decisions bit-exact
    n = int(g["mel"].shape[2])
    assert mel.shape[2] == n
    live = torch.arange(n)[None, :] < torch.from_numpy(g["mel_lengths"]).long()[:, None]
    assert rel_err(mel, torch.from_numpy(g["mel"])) < 1e-3
    assert rel_err(post, torch.from_numpy(g["mel_post"])) < 1e-3
    assert rel_err(gate.cpu() * live[:, :, None], torch.from_numpy(g["gate"])) < 1e-3
    assert rel_err(align.cpu() * live[:, :, None], torch.from_numpy(g["align"])) < 1e-3


# ---------------------------------------------------------------------------------------------------------------------
# 4. streaming, and text to audio
# ---------------------------------------------------------------------------------------------------------------------
def stream(model, text, keep, lengths, chunk):
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        return list(model.inference_stream(text.cuda(), chunk_steps=chunk, input_lengths=lengths))


def test_stream_items_concatenate_to_the_batch_call():
    lengths, S = [70, 9, 130, 41], 48
    text, keep = ragged_text(lengths, 71), keep_mask((S, 2, 4, 256), 0.5, 72)
    model = make_model(synth_state_dict(7, gate_bias=0.0, gate_sign=10.0, scale=2.0), S)
    L = torch.tensor(lengths)
    model.decoder.gate_threshold = threshold_for(model, text, keep, L, S)
    ref, rl = infer(model, text, keep, L)
    for chunk in (1, 11, 32):
        items = stream(model, text, keep, L, chunk)
        for k, key in enumerate(("mel_outputs", "mel_outputs_postnet", "gate_outputs", "alignments")):
            got = torch.cat([it[key] for it in items], dim=2 if k < 2 else 1)
            assert torch.equal(got, ref[k]), (chunk, key)
        assert torch.equal(items[-1]["mel_lengths"], rl)


def test_stream_to_audio_equals_each_rows_own_text_to_audio():
    from tests.test_gpu_waveglow_stream import vocoder
    from tests.waveglow_common import noise
    lengths, S, strength = [12, 57], 40, 0.1
    text, keep = ragged_text(lengths, 81), keep_mask((S, 2, 2, 256), 0.5, 82)
    model = make_model(synth_state_dict(7, gate_bias=0.0, gate_sign=10.0, scale=2.0), S)
    L = torch.tensor(lengths)
    model.decoder.gate_threshold = threshold_for(model, text, keep, L, S)
    glow = vocoder()
    den = t2.Denoiser(glow)
    z = noise(2, S, 83).cuda()
    mels = stream(model, text, keep, L, 16)
    with t2.waveglow_noise(z):
        audio_items = list(glow.infer_stream(iter(mels), sigma=0.666))
    got = torch.cat([it["audio"] for it in den.stream(iter(audio_items), strength)], dim=1)
    print("lengths %s -> mel lengths %s, audio %s" % (lengths, model.mel_lengths.tolist(), tuple(got.shape)))
    for b, Lb in enumerate(lengths):
        (_, post, _, _), ol = alone(model, text, keep, b, Lb)
        n1 = int(ol[0])
        with t2.waveglow_noise(z[b:b + 1, :, :32 * n1].contiguous()):
            a1 = glow.infer(post, sigma=0.666)
        ref = den(a1, strength)[:, 0]
        assert torch.equal(got[b, :HOP * n1], ref[0]), b
        assert not bool(got[b, HOP * n1:].any()), b


# ---------------------------------------------------------------------------------------------------------------------
# 5. the host entry point and the refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_infer_host_lengths_equals_inference():
    """t2_infer_host_lengths takes a Philox seed rather than masks: inference() draws one seed per call it makes (encoder,
    decoder, postnet), so with the counter reset the decoder's is the second."""
    from tacotron2_b200 import _engine
    lengths, S = [30, 3, 17], 24
    text = ragged_text(lengths, 91)
    model = make_model(synth_state_dict(7, gate_bias=-2.0, scale=2.0), S)
    c0 = _engine._seed_counter[0]
    with torch.no_grad():
        ref = model.inference(text.cuda(), input_lengths=torch.tensor(lengths))[1].clone()
    ref_len = model.mel_lengths.clone()
    seed = (torch.initial_seed() * 1000003 + c0 + 2) & 0xFFFFFFFFFFFFFFFF
    mel_h, len_h, ns_h = model._t2_engine().infer_host(
        text.to(torch.int64).contiguous().pin_memory(), S, 0.5, seed=seed,
        input_lengths_host=torch.tensor(lengths, dtype=torch.int64).pin_memory())
    n = int(ns_h[0])
    print("lengths %s -> mel lengths %s, %d steps" % (lengths, len_h.tolist(), n))
    assert n == ref.shape[2] and torch.equal(len_h, ref_len.cpu())
    assert torch.equal(mel_h[:, :, :n], ref.cpu()) and not bool(mel_h[:, :, n:].any())


def test_bad_lengths_are_refused_before_any_launch():
    model = make_model(synth_state_dict(7), 4)
    text = rand_text(3, 10, 1).cuda()
    eng = model._t2_engine()                       # weights packed here, not inside the count
    before = _capi.lib().t2_kernel_launch_count()
    with torch.no_grad():
        for bad, err in [(torch.tensor([3, 0, 5]), ValueError), (torch.tensor([3, 11, 5]), ValueError),
                         (torch.tensor([3, 5]), ValueError), (torch.tensor([[3, 4, 5]]), ValueError),
                         (torch.tensor([3.0, 4.0, 5.0]), TypeError)]:
            with pytest.raises(err):
                model.inference(text, input_lengths=bad)
            with pytest.raises(err):
                next(model.inference_stream(text, input_lengths=bad))
    assert _capi.lib().t2_kernel_launch_count() == before
    mel = torch.empty(3, 80, 4).pin_memory()
    out = (mel, torch.empty(3, dtype=torch.int32).pin_memory(), torch.empty(1, dtype=torch.int32).pin_memory())
    with pytest.raises(_capi.T2Error, match="outside"):
        eng.infer_host(text.cpu().pin_memory(), 4, out_host=out, input_lengths_host=torch.tensor([3, 0, 5]).pin_memory())
    assert _capi.lib().t2_kernel_launch_count() == before
