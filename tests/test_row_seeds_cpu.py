"""Per-utterance seeds without a GPU: the parsing of ``seeds`` and the scheduler's
per-slot seed / step hand-over (tacotron2_b200/serving.py) over a fake engine side."""
import pytest
import torch

from tacotron2_b200 import _engine
from tacotron2_b200.serving import InferenceServer
from tests.test_serving_cpu import FakeStream

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
