"""The continuous-batching scheduler (tacotron2_b200/serving.py) without a GPU, over a fake of the engine side that
records every call and plays back a script of firing steps."""
import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200.serving import InferenceServer, chunk_seed
from tests.common import keep_mask


class FakeStream:
    """Stands in for EngineBackend / DecoderStream.  fire_at: request id -> the request's own step (0-based) at which its
    gate fires; a request without an entry never fires."""

    def __init__(self, slots, fire_at=()):
        self.slots, self.fire_at, self.calls = slots, dict(fire_at), []
        self.masks = []

    def admit(self, pairs):
        self.calls.append(("admit", [(slot, r.id) for slot, r in pairs]))

    def launch(self, n, chunk_index, keep, slots):
        self.calls.append(("launch", n, chunk_index, list(slots)))
        self.masks.append(keep)
        self.n = n

    def collect(self, entries):
        self.calls.append(("collect", [(slot, r.id, s, cnt) for slot, r, s, cnt in entries]))
        self.entries = entries

    def read(self):
        fired = [-1] * self.slots
        for slot, r, s, _ in self.entries:
            f = self.fire_at.get(r.id)
            if f is not None and s <= f < s + self.n:
                fired[slot] = f - s + 1
        n_slices = (self.slots + 63) // 64
        ran = []
        for i in range(n_slices):           # a slice whose occupied rows have all fired stops at the last firing step
            rows = [fired[slot] for slot, _, _, _ in self.entries if slot // 64 == i]
            full = len(rows) == min(64, self.slots - 64 * i)
            ran.append(max(rows) if rows and full and all(f > 0 for f in rows) else self.n)
        self.calls.append(("read",))
        return fired, ran

    def finish(self, requests):
        self.calls.append(("finish", [r.id for r in requests]))
        return [dict(id=r.id, mel_length=r.length, hit_max_steps=r.hit_max_steps) for r in requests]


def server(slots, chunk, fire_at=(), limit=1000, max_text_len=8):
    return InferenceServer(FakeStream(slots, fire_at), slots, max_text_len, chunk, limit)


TEXT = torch.arange(5)


def test_fifo_admission_one_request_per_idle_slot_and_slots_are_reused():
    s = server(2, 4, {0: 1, 1: 9, 2: 2, 3: 0, 4: 3})
    ids = [s.submit(TEXT) for _ in range(5)]
    assert ids == [0, 1, 2, 3, 4]
    done = s.step()
    assert [r["id"] for r in done] == [0] and done[0]["mel_length"] == 2
    assert s.backend.calls[0] == ("admit", [(0, 0), (1, 1)])
    done = s.step()                                      # request 2 takes slot 0; request 1 is mid-flight in slot 1
    assert ("admit", [(0, 2)]) in s.backend.calls
    assert [r["id"] for r in done] == [2] and done[0]["mel_length"] == 3
    done = s.step()                                      # 3 into slot 0; 1 fires at its step 9 = local step 1
    assert [(r["id"], r["mel_length"]) for r in done] == [(3, 1), (1, 10)]
    done = s.step()
    assert [(r["id"], r["mel_length"]) for r in done] == [(4, 4)]
    assert s.idle() and s.step() == []
    admits = [c[1] for c in s.backend.calls if c[0] == "admit"]
    assert admits == [[(0, 0), (1, 1)], [(0, 2)], [(0, 3)], [(0, 4)]]    # FIFO, lowest idle slot first


def test_run_ends_exactly_when_queue_and_slots_are_empty():
    s = server(3, 5, {i: 3 * i for i in range(7)})
    for _ in range(7):
        s.submit(TEXT)
    got = list(s.run())
    assert sorted(r["id"] for r in got) == list(range(7))
    assert {r["id"]: r["mel_length"] for r in got} == {i: 3 * i + 1 for i in range(7)}
    assert s.idle()
    n_launch = sum(c[0] == "launch" for c in s.backend.calls)
    assert list(s.run()) == [] and sum(c[0] == "launch" for c in s.backend.calls) == n_launch
    assert s.backend.calls[-1][0] == "finish"            # nothing ran after the last request had left


def test_step_accounting_across_chunk_boundaries_and_the_requests_own_limit():
    s = server(2, 4, {0: 9})
    s.submit(TEXT, max_decoder_steps=20)
    s.submit(TEXT, max_decoder_steps=6)                  # never fires: leaves at its limit, inside the second chunk
    assert s.step() == []
    assert s.backend.calls[-2] == ("collect", [(0, 0, 0, 4), (1, 1, 0, 4)])
    done = s.step()
    assert s.backend.calls[-3] == ("collect", [(0, 0, 4, 4), (1, 1, 4, 2)])     # 2 frames are left of request 1
    assert done == [dict(id=1, mel_length=6, hit_max_steps=True)]
    done = s.step()
    assert s.backend.calls[-3] == ("collect", [(0, 0, 8, 4)])
    assert done == [dict(id=0, mel_length=10, hit_max_steps=False)]


def test_a_gate_that_fires_past_the_limit_does_not_count():
    s = server(1, 8, {0: 5, 1: 2})
    s.submit(TEXT, max_decoder_steps=3)                  # fires at its step 5, but only 3 steps are its own
    s.submit(TEXT, max_decoder_steps=3)                  # fires at step 2: length 3, the limit, and not a miss
    assert [list(r.values()) for r in s.run()] == [[0, 3, True], [1, 3, False]]


def test_one_warning_per_request_that_hit_its_limit(capsys):
    s = server(2, 3)
    for _ in range(3):
        s.submit(TEXT, max_decoder_steps=4)
    assert all(r["hit_max_steps"] for r in s.run())
    assert capsys.readouterr().out.count("Warning! Reached max decoder steps") == 3


def test_chunk_mask_holds_each_requests_mask_at_its_own_step_offset():
    s = server(3, 4, {0: 100, 1: 1, 2: 100})
    masks = [keep_mask((12, 2, 256), 0.5, 10 + i) for i in range(3)]
    for m in masks:
        s.submit(TEXT, max_decoder_steps=12, prenet_keep=m)
    s.step()
    k = s.backend.masks[0]
    assert k.shape == (5, 2, 3, 256) and k.dtype == torch.uint8
    for slot in range(3):
        assert torch.equal(k[:, :, slot], masks[slot][0:5])
    s.submit(TEXT, max_decoder_steps=12, prenet_keep=masks[1])      # id 3 -> slot 1 at its step 0; the others at step 4
    s.step()
    k = s.backend.masks[1]
    assert torch.equal(k[:, :, 0], masks[0][4:9]) and torch.equal(k[:, :, 2], masks[2][4:9])
    assert torch.equal(k[:, :, 1], masks[1][0:5])
    s.step()                                              # steps 8..12 of a 12-row mask: the row past it is ones
    k = s.backend.masks[2]
    assert torch.equal(k[:4, :, 0], masks[0][8:12]) and bool((k[4, :, 0] == 1).all())


def test_without_masks_no_mask_is_assembled_and_chunk_seeds_differ():
    s = server(1, 2, {0: 3})
    s.submit(TEXT)
    list(s.run())
    assert s.backend.masks == [None, None]
    assert [c[2] for c in s.backend.calls if c[0] == "launch"] == [0, 1]
    assert len({chunk_seed(7, i) for i in range(1000)}) == 1000 and chunk_seed(7, 0) != 7


def test_submit_refusals_come_before_any_engine_call():
    s = server(2, 4, max_text_len=8)
    with pytest.raises(ValueError, match="longer than"):
        s.submit(torch.arange(9))
    with pytest.raises(ValueError, match="empty"):
        s.submit(torch.zeros(0, dtype=torch.long))
    with pytest.raises(TypeError, match="integers"):
        s.submit(torch.zeros(3))
    with pytest.raises(ValueError, match="max_decoder_steps"):
        s.submit(TEXT, max_decoder_steps=0)
    with pytest.raises(ValueError, match="1-D"):
        s.submit(torch.zeros(1, 3, dtype=torch.long))
    with pytest.raises(ValueError, match="prenet_keep"):
        s.submit(TEXT, max_decoder_steps=5, prenet_keep=keep_mask((4, 2, 256), 0.5, 1))
    s.submit(TEXT)
    with pytest.raises(ValueError, match="every request or for none"):
        s.submit(TEXT, max_decoder_steps=5, prenet_keep=keep_mask((5, 2, 256), 0.5, 1))
    assert s.backend.calls == [] and len(s.queue) == 1
    for bad in (dict(slots=0), dict(max_text_len=0), dict(chunk_steps=0)):
        kw = dict(slots=1, max_text_len=1, chunk_steps=1)
        kw.update(bad)
        with pytest.raises(ValueError):
            InferenceServer(None, max_decoder_steps=10, **kw)


def test_submit_between_steps_and_more_slots_than_requests():
    s = server(4, 2, {0: 5, 1: 0})
    s.submit(TEXT)
    assert s.step() == []
    assert s.backend.calls[1] == ("launch", 2, 0, [0])   # three slots stay idle
    s.submit(TEXT)
    done = s.step()                                      # request 1 joins slot 1 while request 0 is at its step 2
    assert ("admit", [(1, 1)]) in s.backend.calls
    assert s.backend.calls[-3] == ("collect", [(0, 0, 2, 2), (1, 1, 0, 2)])
    assert done == [dict(id=1, mel_length=1, hit_max_steps=False)]
    assert [r["id"] for r in s.run()] == [0]


def test_row_steps_counts_slots_times_steps_of_the_slices_that_ran():
    s = server(70, 4, {i: 1 for i in range(64)})         # the first slice is full and stops after 2 steps
    for _ in range(65):
        s.submit(TEXT, max_decoder_steps=4)
    s.step()
    assert s.row_steps == 64 * 2 + 6 * 4 and s.chunks == 1


def test_servers_need_cuda_and_eval_mode():
    m = t2.Tacotron2(t2.create_hparams())
    with pytest.raises(RuntimeError, match="eval mode"):
        m.train().inference_server()
    with pytest.raises(RuntimeError, match="CUDA"):
        m.eval().inference_server(slots=2, max_text_len=4, chunk_steps=2)
