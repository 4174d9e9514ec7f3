"""The decoder step API's host side: parse_decoder_outputs against the reference's stacking, and the refusals that need
no GPU (tests/test_gpu_decode_step.py runs the steps)."""
import pytest
import torch

import tacotron2_b200 as t2


def decoder():
    return t2.Tacotron2(t2.create_hparams()).decoder


def reference_parse(mel_outputs, gate_outputs, alignments, n_mel):
    """model.py:311-338 as written there."""
    alignments = torch.stack(alignments).transpose(0, 1)
    gate_outputs = torch.stack(gate_outputs).transpose(0, 1)
    gate_outputs = gate_outputs.contiguous()
    mel_outputs = torch.stack(mel_outputs).transpose(0, 1).contiguous()
    mel_outputs = mel_outputs.view(mel_outputs.size(0), -1, n_mel)
    mel_outputs = mel_outputs.transpose(1, 2)
    return mel_outputs, gate_outputs, alignments


@pytest.mark.parametrize("B,T,S", [(1, 5, 1), (3, 17, 9), (4, 2, 30)])
def test_parse_decoder_outputs_equals_reference(B, T, S):
    g = torch.Generator().manual_seed(B * 100 + S)
    mels = [torch.randn(B, 80, generator=g) for _ in range(S)]
    gates = [torch.randn(B, 1, generator=g) for _ in range(S)]
    aligns = [torch.rand(B, T, generator=g) for _ in range(S)]
    out = decoder().parse_decoder_outputs(mels, gates, aligns)
    ref = reference_parse(mels, gates, aligns, 80)
    for a, b in zip(out, ref):
        assert a.shape == b.shape and torch.equal(a, b)


def test_refuses_under_autograd():
    dec = decoder()
    mem = torch.zeros(1, 4, 512)
    cat = torch.zeros(1, 2, 4)
    for call in (lambda: dec.initialize_decoder_states(mem, None), lambda: dec.decode(torch.zeros(1, 256)),
                 lambda: dec.attention_layer(torch.zeros(1, 1024), mem, torch.zeros(1, 4, 128), cat, None),
                 lambda: dec.attention_layer.get_alignment_energies(torch.zeros(1, 1024), torch.zeros(1, 4, 128), cat),
                 lambda: dec.attention_layer.location_layer(cat)):
        with pytest.raises(NotImplementedError, match="no autograd node"):
            call()


def test_refuses_cpu_tensors():
    dec = decoder()
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="no CPU path"):
            dec.initialize_decoder_states(torch.zeros(1, 4, 512), None)
        with pytest.raises(RuntimeError, match="no CPU path"):
            dec.attention_layer.location_layer(torch.zeros(1, 2, 4))


def test_decode_needs_initialized_states():
    with torch.no_grad(), pytest.raises(RuntimeError, match="initialize_decoder_states"):
        decoder().decode(torch.zeros(1, 256))


def test_stand_alone_attention_is_refused():
    att = decoder().attention_layer.__class__(1024, 512, 128, 32, 31)
    with torch.no_grad(), pytest.raises(RuntimeError, match="part of a Decoder"):
        att.location_layer._t2_engine()


@pytest.mark.parametrize("memory,mask,match", [
    (torch.zeros(2, 4), None, "memory must be"),
    (torch.zeros(2, 4, 256), None, r"shape \(2, 4, 512\)"),
    (torch.zeros(2, 4, 512, dtype=torch.int32), None, "float tensor"),
    (torch.zeros(2, 4, 512), torch.zeros(2, 4, dtype=torch.uint8), "bool tensor"),
    (torch.zeros(2, 4, 512), torch.zeros(2, 5, dtype=torch.bool), r"mask must have shape \(2, 4\)"),
    (torch.zeros(2, 4, 512), torch.zeros(4, dtype=torch.bool), r"mask must have shape \(2, 4\)"),
])
def test_refuses_bad_shapes_and_dtypes(memory, mask, match, monkeypatch):
    dec = decoder()
    monkeypatch.setattr(type(dec), "_t2_device", lambda self: torch.device("cpu"))
    with torch.no_grad(), pytest.raises((TypeError, ValueError), match=match):
        dec.initialize_decoder_states(memory, mask)


def test_refuses_bad_decoder_input_and_t_enc_1283(monkeypatch):
    dec = decoder()
    monkeypatch.setattr(type(dec), "_t2_device", lambda self: torch.device("cpu"))
    with torch.no_grad():
        with pytest.raises(ValueError, match=r"T_enc=1283"):
            dec.initialize_decoder_states(torch.zeros(1, 1283, 512), None)
        dec.memory = torch.zeros(2, 4, 512)
        with pytest.raises(ValueError, match=r"decoder_input must have shape \(2, 256\)"):
            dec.decode(torch.zeros(2, 80))
