"""Constrained synthesis without a GPU: the host-side checks of ``attention_window`` / ``max_decoder_steps``, how they
reach the decoder's arguments, and ``window_ranges``, the reference of the window that the GPU tests
(tests/test_gpu_attention_window.py) check the engine's alignments against."""
import pytest
import torch

from tacotron2_b200 import _engine

CPU = torch.device("cpu")


def window_ranges(align, lengths, window):
    """The positions each step of a windowed run may attend to: (lo, hi) (B, T_steps) int64, step t of row b allowed
    [lo, hi).  align (B, T_steps, T_text): the run's attention weights; lengths (B,): text lengths; window (back, front).
    p_t is the first position of the largest weight of step t - 1 below the row's length (0 at step 0)."""
    B, S, T = align.shape
    back, front = window
    lengths = torch.as_tensor(lengths).long().cpu()
    prev = torch.cat([torch.zeros(B, 1, T, dtype=align.dtype), align.cpu()[:, :-1]], 1)
    pos = torch.arange(T)
    prev = prev.masked_fill(pos[None, None, :] >= lengths[:, None, None], -1.0)
    p = prev.argmax(-1)                                       # torch.argmax returns the first maximal index
    return (p - back).clamp(min=0), torch.minimum(p + front, lengths[:, None])


def check(window=None, caps=None, B=3, forced=False):
    amap = torch.zeros(B, 2, 4) if forced else None
    opts = _engine.inference_options("t", B, 4, CPU, alignments=amap, attention_window=window, max_decoder_steps=caps)
    return opts.window, opts.max_steps, None if opts.max_steps is None else opts.cap


def test_builder_takes_valid_limits_as_the_decoder_wants_them():
    assert check() == (None, None, None)
    assert check((1, 3)) == ((1, 3), None, None)
    assert check([0, 1])[0] == (0, 1)
    assert check(torch.tensor([2, 6]))[0] == (2, 6)
    for caps, want in ((7, [7, 7, 7]), ([5, 9, 1], [5, 9, 1]), (torch.tensor([4, 2, 8]), [4, 2, 8]),
                       (torch.tensor([3, 3, 6], dtype=torch.int16), [3, 3, 6])):
        window, got, longest = check(None, caps)
        assert window is None and got.dtype == torch.int32 and got.is_contiguous() and got.tolist() == want
        assert longest == max(want)
    caps = torch.tensor([3, 4], dtype=torch.int32)
    a = _engine.decoder_args(window=(2, 5), max_steps=caps)
    assert (a.window_back, a.window_front, a.max_steps) == (2, 5, caps.data_ptr())
    a = _engine.decoder_args(window=None, max_steps=caps[:1])
    assert (a.window_back, a.window_front) == (0, 0) and a.max_steps
    a = _engine.decoder_args(window=None, max_steps=None)
    assert (a.window_back, a.window_front, a.max_steps) == (0, 0, None)      # zeroed: no limits


@pytest.mark.parametrize("window,caps,forced,err,match", [
    ((1, 3), None, True, ValueError, "attention_window and alignments"),
    (None, 10, True, ValueError, "max_decoder_steps and alignments"),
    ((1,), None, False, TypeError, "two integers"),
    ((1, 2, 3), None, False, TypeError, "two integers"),
    ((1.0, 3), None, False, TypeError, "two integers"),
    ((True, 3), None, False, TypeError, "two integers"),
    (3, None, False, TypeError, "two integers"),
    ((-1, 3), None, False, ValueError, "back >= 0 and front >= 1"),
    ((1, 0), None, False, ValueError, "back >= 0 and front >= 1"),
    (None, 0, False, ValueError, "max_decoder_steps must lie in"),
    (None, -4, False, ValueError, "max_decoder_steps must lie in"),
    (None, [4, 0, 2], False, ValueError, "max_decoder_steps must lie in"),
    (None, [4, 2], False, ValueError, r"max_decoder_steps must be one integer or have shape \(3,\)"),
    (None, torch.ones(3, 1, dtype=torch.int32), False, ValueError, "shape"),
    (None, [4.0, 2.0, 1.0], False, TypeError, "max_decoder_steps must hold integers"),
    (None, 4.0, False, TypeError, "max_decoder_steps must hold integers"),
    (None, torch.ones(3, dtype=torch.bool), False, TypeError, "max_decoder_steps must hold integers"),
])
def test_builder_refuses_bad_limits(window, caps, forced, err, match):
    with pytest.raises(err, match=match):
        check(window, caps, forced=forced)


def test_window_ranges():
    a = torch.zeros(2, 4, 6)
    a[0, 0, 2] = 1.0                         # step 1 of row 0 centres on 2
    a[0, 1, 1] = a[0, 1, 4] = 0.5            # a tie: the first position wins
    a[0, 2, 5] = 0.9                         # past row 0's length 5: ignored, all below are 0 -> p = 0
    a[1, 0, 3] = 0.7
    lo, hi = window_ranges(a, [5, 6], (1, 3))
    assert lo.tolist() == [[0, 1, 0, 0], [0, 2, 0, 0]]
    assert hi.tolist() == [[3, 5, 4, 3], [3, 6, 3, 3]]
    lo, hi = window_ranges(a, [5, 6], (6, 6))       # both sides at least the length: everything is allowed
    assert not bool(lo.any()) and hi.tolist() == [[5] * 4, [6] * 4]
