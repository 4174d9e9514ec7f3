"""CPU: the ragged-inference boundary -- the T2InferArgs mirror matches the C layout, the header declares the new entry
points, and bad per-row lengths are refused by the public API before the engine (or CUDA) is touched."""
import ctypes
import os
import subprocess

import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tests.common import ROOT


def test_infer_args_struct_matches_c_layout(tmp_path):
    fields = ["text_host", "input_lengths_host", "B", "T_text", "max_steps", "gate_threshold", "seed", "impl",
              "mel_post_host", "mel_lengths_host", "n_steps_host", "ws", "ws_bytes"]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "t2b200.h"', 'int main(void){',
             'printf("size %zu\\n", sizeof(T2InferArgs));']
    lines += ['printf("%s %%zu\\n", offsetof(T2InferArgs, %s));' % (f, f) for f in fields]
    lines.append('return 0;}')
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    assert int(out["size"]) == ctypes.sizeof(_capi.T2InferArgs)
    for f in fields:
        assert int(out[f]) == getattr(_capi.T2InferArgs, f).offset, f


def test_new_entry_points_are_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "t2b200.h")).read()
    for name in ("t2_encoder_infer", "t2_infer_lengths_workspace_bytes", "t2_infer_host_lengths"):
        assert name + "(" in header and name in _capi.EXPORTS
    # the existing entry points and the ABI version are unchanged
    assert "int    t2_infer_host(T2Model* m, const int64_t* text_host, int32_t B, int32_t T_text," in header
    assert "#define T2_ABI_VERSION 1" in header


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
