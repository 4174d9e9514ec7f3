"""CPU: the ragged-inference boundary -- the header declares the entry points, and bad per-row lengths are refused by the
public API before the engine (or CUDA) is touched."""
import os

import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tests.common import ROOT


def test_host_entry_points_are_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "t2b200.h")).read()
    for name in ("t2_encoder_infer", "t2_infer_workspace_bytes", "t2_infer_host"):
        assert name + "(" in header and name in _capi.EXPORTS
    # one host-buffer entry point: texts of different lengths go through T2InferArgs.input_lengths_host
    assert "int    t2_infer_host(T2Model* m, const T2InferArgs* a, void* stream);" in header
    assert "#define T2_ABI_VERSION 2" in header


BAD = [(torch.tensor([3, 0, 5]), ValueError, "1..10"),
       (torch.tensor([3, 11, 5]), ValueError, "1..10"),
       (torch.tensor([3, 5]), ValueError, "shape"),
       (torch.tensor([[3, 4, 5]]), ValueError, "shape"),
       (torch.tensor([3.0, 4.0, 5.0]), TypeError, "integers"),
       (torch.tensor([True, True, True]), TypeError, "integers")]


@pytest.mark.parametrize("bad,err,match", BAD, ids=["zero", "too-long", "short", "2d", "float", "bool"])
def test_bad_lengths_raise_before_the_engine(bad, err, match):
    """Checked before anything else: on a CPU-only host the engine would raise about CUDA instead."""
    model = t2.Tacotron2(t2.create_hparams()).eval()
    text = torch.zeros(3, 10, dtype=torch.long)
    with torch.no_grad():
        with pytest.raises(err, match=match):
            model.inference(text, input_lengths=bad)
        with pytest.raises(err, match=match):
            next(model.inference_stream(text, input_lengths=bad))
        with pytest.raises(err, match=match):
            model.decoder.inference(torch.zeros(3, 10, 512), memory_lengths=bad)
        with pytest.raises(err, match=match):
            model.encoder.inference(torch.zeros(3, 512, 10), input_lengths=bad)
    assert "_t2_engine_obj" not in model.__dict__


def test_lengths_may_be_a_list_in_any_order():
    model = t2.Tacotron2(t2.create_hparams()).eval()
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA"):     # validated, then refused for want of a GPU
        model.inference(torch.zeros(3, 10, dtype=torch.long), input_lengths=[4, 10, 1])
