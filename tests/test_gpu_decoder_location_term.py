"""The decoder's location term across step, chunk and slot boundaries.

In inference the persistent decoder computes the location term pa of step t+1 (the fused location conv + dense applied to
the attention weights of step t) while it waits for x2 at the end of step t, into a per-row buffer that a resumable
stream keeps across chunks and that a re-admitted row starts from zero.  That only holds where the whole tile fits the
ring (T_enc <= 280 at 4 stages); longer memories and the 3-stage ring compute it after the q barrier as before.  Every case
equals one-launch inference() bit for bit, and the fp64 oracle under the bar of tests/test_gpu_decoder_regimes.py."""
import functools

import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tests.common import keep_mask, rand_text, synth_state_dict
from tests.test_gpu_decoder_regimes import (STEPS, TOL, make_model, oracle_inference, output_errors, regime_inputs,
                                            regime_weights, run_inference)

pytestmark = pytest.mark.gpu
PA_MAX_T_ENC = 280       # longest T_enc whose pa tile fits the 4-stage ring


def stream_outputs(model, memory, keep, cap, chunks, memory_lengths=None):
    """Decoder stream over `memory`, advanced by each of `chunks` steps in turn: (mel, gate, align) as inference() shapes
    them, and the lengths."""
    eng = model._t2_engine()
    with torch.no_grad():
        st = eng.decoder_stream(memory.cuda(), cap, prenet_keep=keep, gate_threshold=1.0,
                                memory_lengths=memory_lengths)
        for n in chunks:
            st.run(n)
        torch.cuda.synchronize()
    return [st.mel.transpose(1, 2).cpu(), st.gate.unsqueeze(-1).cpu(), st.align.cpu()], st.mel_lengths.cpu()


def assert_same_bits(got, ref):
    for name, a, b in zip(("mel", "gate", "align"), got, ref):
        assert a.shape == b.shape and torch.equal(a, b), (name, float((a.double() - b.double()).abs().max()))


@pytest.mark.parametrize("ragged", [False, True], ids=["full", "ragged"])
def test_pa_is_carried_across_chunk_boundaries_at_steps_1_2_and_33(ragged):
    B, T, S = 5, 150, 40
    sd, _ = regime_weights()
    model = make_model(sd, "regime")
    memory = torch.randn(B, T, 512, generator=torch.Generator().manual_seed(150))
    keep = keep_mask((S, 2, B, 256), 0.5, 151)
    lengths = torch.tensor([150, 95, 94, 1, 37], dtype=torch.int32) if ragged else None
    model._t2_engine().impl = _capi.IMPL_PERSISTENT
    model.decoder.max_decoder_steps, model.decoder.gate_threshold = S, 1.0
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        ref = [o.cpu() for o in model.decoder.inference(memory.cuda(), memory_lengths=lengths)]
    ref_lengths = model.decoder.mel_lengths.cpu()
    got, got_lengths = stream_outputs(model, memory, keep, S, (1, 1, 31, S - 33),
                                      None if lengths is None else lengths.cuda())
    assert_same_bits(got, ref)
    assert got_lengths.tolist() == ref_lengths.tolist() == [S] * B
    if ragged:                       # every row equals its own run on its own slice of the memory
        for b, L in enumerate(lengths.tolist()):
            one, _ = run_inference(model, memory[b:b + 1, :L], keep[:, :, b:b + 1].contiguous(), _capi.IMPL_PERSISTENT, S)
            assert_same_bits([o[0] for o in one], [ref[0][b], ref[1][b], ref[2][b, :, :L]])


@pytest.mark.parametrize("T,force_stages", [(PA_MAX_T_ENC, None), (PA_MAX_T_ENC + 1, None), (897, None), (150, "3")],
                         ids=["T280-pa-tile", "T281-no-tile", "T897-3-stages", "T150-3-stages-forced"])
def test_pa_tile_and_its_fallback_against_the_oracle(T, force_stages, monkeypatch):
    """Either side of the longest tile, the 3-stage regime, and a tile beside a forced 3-stage ring: vs the fp64 oracle,
    and a stream chunked at steps 1 and 2 equals the one-launch run bit for bit."""
    B = 3
    sd, sd64 = regime_weights()
    model = make_model(sd, "regime")
    memory, keep = regime_inputs(B, T)
    if force_stages:
        monkeypatch.setenv("T2_STAGES", force_stages)
    else:
        monkeypatch.delenv("T2_STAGES", raising=False)
    ref, ref_lengths = oracle_inference(sd64, memory, keep, STEPS)
    out, lengths = run_inference(model, memory, keep, _capi.IMPL_PERSISTENT, STEPS)
    errs = output_errors(out, ref)
    print("T_enc=%d stages=%s: %s" % (T, force_stages or "auto", ", ".join("%s %.2e" % kv for kv in errs.items())))
    assert lengths.tolist() == ref_lengths.tolist() == [STEPS] * B
    assert all(v < TOL for v in errs.values()), errs
    got, _ = stream_outputs(model, memory, keep, STEPS, (1, 1, STEPS - 2))
    assert_same_bits(got, out)


@functools.lru_cache(maxsize=None)
def served_model():
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(synth_state_dict(7, gate_bias=0.0, gate_sign=10.0, scale=2.0))
    model = model.cuda().eval()
    model.decoder.gate_threshold = 1.0          # nothing fires: every request runs to its own limit
    return model


def test_a_row_readmitted_mid_stream_starts_from_a_zero_location_term():
    """Two slots, chunks of 5 steps: slot 1 runs a 7-step request, then takes a 150-symbol text at step 10 while slot 0 is
    mid-flight; every request equals its own B = 1 inference()."""
    S, T_CAP = 24, 150
    model = served_model()
    reqs = [(rand_text(1, T_CAP, 11)[0], S, keep_mask((S, 2, 256), 0.5, 12)),
            (rand_text(1, 60, 13)[0], 7, keep_mask((S, 2, 256), 0.5, 14)),
            (rand_text(1, T_CAP, 15)[0], 12, keep_mask((S, 2, 256), 0.5, 16))]
    server = model.inference_server(slots=2, max_text_len=T_CAP, chunk_steps=5)
    ids = [server.submit(text, limit, prenet_keep=k) for text, limit, k in reqs]
    with torch.no_grad():
        out = {r["id"]: r for r in server.run()}
    for i, (text, limit, k) in zip(ids, reqs):
        model.decoder.max_decoder_steps = limit
        with torch.no_grad(), t2.dropout_masks(prenet=k[:limit, :, None].contiguous()):
            one = [o.clone() for o in model.inference(text[None].cuda())]
        r = out[i]
        assert r["mel_length"] == limit == int(model.mel_lengths[0])
        for name, o in zip(("mel_outputs", "mel_outputs_postnet", "gate_outputs", "alignments"), one):
            assert torch.equal(r[name], o), (i, name)
