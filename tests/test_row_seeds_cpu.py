"""Per-utterance seeds without a GPU: the C layout of the new ABI fields, the parsing of ``seeds`` and the scheduler's
per-slot seed / step hand-over (tacotron2_b200/serving.py) over a fake engine side."""
import ctypes
import os
import subprocess

import pytest
import torch

from tacotron2_b200 import _capi, _engine
from tacotron2_b200.serving import InferenceServer
from tests.common import ROOT
from tests.test_serving_cpu import FakeStream

FIELDS = {
    "T2DecoderArgs": ["stash_bytes", "row_seeds"],
    "T2DecoderStreamArgs": ["dec", "state", "state_bytes", "status", "row_step0"],
    "T2WaveGlowArgs": ["mel", "B", "T_mel", "lengths", "io_half", "sigma", "z", "seed", "audio", "ws", "ws_bytes",
                       "row_seeds"],
    "T2WaveGlowWindowArgs": ["wg", "frame0", "out0", "out1", "z_frames", "at_end"],
    "T2InferArgs": ["text_host", "input_lengths_host", "B", "T_text", "max_steps", "gate_threshold", "seed", "impl",
                    "mel_post_host", "mel_lengths_host", "n_steps_host", "ws", "ws_bytes", "row_seeds_host"],
}


def test_new_abi_fields_match_c_layout(tmp_path):
    """sizeof / offsetof of the structs that gained row_seeds / row_step0, as gcc sees the header == the ctypes mirror;
    the fields that existed before keep their offsets (the new ones are appended)."""
    src = tmp_path / "layout.c"
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "t2b200.h"', 'int main(void){']
    for s, fs in FIELDS.items():
        lines.append('printf("%s %%zu\\n", sizeof(%s));' % (s, s))
        for f in fs:
            lines.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (s, f, s, f))
    lines.append('return 0;}')
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(line.split() for line in subprocess.check_output([str(exe)]).decode().splitlines())
    for s, fs in FIELDS.items():
        cls = getattr(_capi, s)
        assert int(out[s]) == ctypes.sizeof(cls), s
        for f in fs:
            assert int(out["%s.%s" % (s, f)]) == getattr(cls, f).offset, (s, f)
    # appended last: every earlier field is where it was
    assert _capi.T2DecoderArgs.row_seeds.offset == _capi.T2DecoderArgs.stash_bytes.offset + 8
    assert _capi.T2WaveGlowArgs.row_seeds.offset == _capi.T2WaveGlowArgs.ws_bytes.offset + 8
    assert _capi.T2InferArgs.row_seeds_host.offset == _capi.T2InferArgs.ws_bytes.offset + 8


def test_seeds_are_taken_as_64_bit_patterns():
    cpu = torch.device("cpu")
    top = (1 << 64) - 1
    out = _engine.row_seeds([0, 5, 1 << 63, top], 4, cpu, "t")
    assert out.dtype == torch.int64 and out.tolist() == [0, 5, -(1 << 63), -1]
    t = torch.tensor([3, -1], dtype=torch.int64)                 # int64: its bit pattern, -1 = 2**64 - 1
    assert _engine.row_seeds(t, 2, cpu, "t").tolist() == [3, -1]
    assert _engine.row_seeds(torch.tensor([7, 9], dtype=torch.int32), 2, cpu, "t").tolist() == [7, 9]
    assert _engine.row_seeds(torch.tensor([7, 255], dtype=torch.uint8), 2, cpu, "t").tolist() == [7, 255]
    assert _engine.row_seeds(None, 3, cpu, "t") is None


@pytest.mark.parametrize("seeds,err", [
    ([1, 2], ValueError),                                        # wrong count
    ([1, 2, 1 << 64], ValueError),                               # out of range
    ([1, 2, -1], ValueError),
    ([1, 2, 3.0], TypeError),                                    # not an integer
    ([1, 2, True], TypeError),
    (torch.zeros(3), TypeError),                                 # float tensor
    (torch.zeros(3, dtype=torch.bool), TypeError),
    (torch.zeros(3, 1, dtype=torch.int64), ValueError),          # wrong shape
    (torch.tensor([1, -2, 3], dtype=torch.int32), ValueError),   # negative narrow integers
])
def test_bad_seeds_are_refused(seeds, err):
    with pytest.raises(err):
        _engine.row_seeds(seeds, 3, torch.device("cpu"), "t")


class SeedStream(FakeStream):
    def launch(self, n, chunk_index, keep, slots, row_seeds=None):
        super().launch(n, chunk_index, keep, slots)
        self.calls[-1] = self.calls[-1] + (row_seeds,)


def test_server_hands_every_slot_its_seed_and_its_requests_step_count():
    """Two slots, chunks of 4: request 0 fires at its step 5 (local step 1 of its second chunk), request 2 then takes
    its slot at step 0 while request 1 carries on from step 8."""
    server = InferenceServer(SeedStream(2, {0: 5}), 2, 8, 4, 100)
    for rid, seed in enumerate([11, (1 << 64) - 1, 7]):
        server.submit(torch.arange(3), seed=seed)
    launches = []
    for _ in range(3):
        server.step()
        launches.append([c for c in server.backend.calls if c[0] == "launch"][-1][-1])
    assert launches[0] == ([11, (1 << 64) - 1], [0, 0])
    assert launches[1] == ([11, (1 << 64) - 1], [4, 4])
    assert launches[2] == ([7, (1 << 64) - 1], [0, 8])


def test_server_seed_rules():
    server = InferenceServer(SeedStream(2), 2, 8, 4, 100)
    server.submit(torch.arange(3), seed=1)
    with pytest.raises(ValueError, match="seed for every request or for none"):
        server.submit(torch.arange(3))
    with pytest.raises(ValueError):
        server.submit(torch.arange(3), seed=1 << 64)
    with pytest.raises(TypeError):
        server.submit(torch.arange(3), seed=1.5)
    with pytest.raises(ValueError, match="exclude each other"):
        server.submit(torch.arange(3), prenet_keep=torch.ones(100, 2, 256, dtype=torch.uint8), seed=2)
    plain = InferenceServer(SeedStream(2), 2, 8, 4, 100)
    plain.submit(torch.arange(3))
    with pytest.raises(ValueError, match="seed for every request or for none"):
        plain.submit(torch.arange(3), seed=3)
    plain.step()
    assert [c for c in plain.backend.calls if c[0] == "launch"][0][-1] is None      # unseeded: no per-slot keys
