"""Forced-alignment synthesis without a GPU: the host-side checks of ``alignments`` / ``alignment_lengths`` and the
``alignments_from_durations`` helper."""
import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _engine

CPU = torch.device("cpu")


def check(alignments, lengths=None, B=2, T=5, training=False):
    return _engine.forced_alignment(alignments, lengths, B, T, CPU, training, "t")


def test_valid_maps_are_taken_as_fp32_with_int32_lengths():
    a = torch.rand(2, 7, 5, dtype=torch.float16)
    fa, fl = check(a)
    assert fa.dtype == torch.float32 and fa.is_contiguous() and torch.equal(fa, a.float())
    assert fl.dtype == torch.int32 and fl.tolist() == [7, 7]
    for lengths in ([3, 7], torch.tensor([1, 7]), torch.tensor([2, 4], dtype=torch.int16)):
        _, fl = check(a, lengths)
        assert fl.dtype == torch.int32 and fl.tolist() == torch.as_tensor(lengths).tolist()
    assert check(None) == (None, None)


@pytest.mark.parametrize("alignments,lengths,training,err,match", [
    (None, [1, 2], False, ValueError, "alignment_lengths needs alignments"),
    (torch.rand(2, 4, 5), None, True, ValueError, "alignments need eval mode"),
    ([[0.0]], None, False, TypeError, "alignments must be a tensor"),
    (torch.ones(2, 4, 5, dtype=torch.int64), None, False, TypeError, "alignments must be a float"),
    (torch.ones(2, 4, 5, dtype=torch.bool), None, False, TypeError, "alignments must be a float"),
    (torch.rand(2, 4), None, False, ValueError, "alignments must have shape"),
    (torch.rand(3, 4, 5), None, False, ValueError, "alignments must have shape"),
    (torch.rand(2, 4, 6), None, False, ValueError, "alignments must have shape"),          # T_text mismatch
    (torch.rand(2, 0, 5), None, False, ValueError, "alignments must have shape"),
    (torch.rand(2, 4, 5), [1.0, 2.0], False, TypeError, "alignment_lengths must hold integers"),
    (torch.rand(2, 4, 5), torch.ones(2, dtype=torch.bool), False, TypeError, "alignment_lengths must hold integers"),
    (torch.rand(2, 4, 5), [1, 2, 3], False, ValueError, "alignment_lengths must have shape"),
    (torch.rand(2, 4, 5), [0, 2], False, ValueError, "alignment_lengths must lie in 1..4"),
    (torch.rand(2, 4, 5), [1, 5], False, ValueError, "alignment_lengths must lie in 1..4"),
])
def test_bad_arguments_are_refused(alignments, lengths, training, err, match):
    with pytest.raises(err, match=match):
        check(alignments, lengths, training=training)


def test_durations_give_a_one_hot_map():
    d = torch.tensor([[2, 0, 1, 3], [0, 1, 0, 0], [1, 1, 1, 1]])
    a, n = t2.alignments_from_durations(d)
    assert n.tolist() == [6, 1, 4] and torch.equal(n, d.sum(1))
    assert a.shape == (3, 6, 4) and a.dtype == torch.float32
    expect = [[0, 0, 2, 3, 3, 3], [1], [0, 1, 2, 3]]
    for b, syms in enumerate(expect):
        assert a[b, :len(syms)].argmax(1).tolist() == syms
        assert torch.equal(a[b, :len(syms)].sum(1), torch.ones(len(syms)))
        assert not bool(a[b, len(syms):].any())                 # steps past the row's length are empty
    a2, n2 = t2.alignments_from_durations([[2, 0, 1, 3], [0, 1, 0, 0], [1, 1, 1, 1]])
    assert torch.equal(a2, a) and torch.equal(n2, n)


@pytest.mark.parametrize("durations,err", [
    (torch.tensor([[1, 0], [0, 0]]), ValueError),                # a row of 0 frames
    (torch.tensor([[1, -1]]), ValueError),
    (torch.tensor([[1.0, 2.0]]), TypeError),
    (torch.tensor([1, 2]), ValueError),                          # not (B, T_text)
])
def test_bad_durations_are_refused(durations, err):
    with pytest.raises(err):
        t2.alignments_from_durations(durations)
