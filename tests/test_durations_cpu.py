"""Durations from attention maps without a GPU: the host-side checks of ``durations_from_alignments`` (through its
validation helper, on CPU tensors), and the numpy fp64 oracles the GPU tests compare against -- MAS against brute-force
enumeration of every monotonic path, with its tie rule, and argmax on hand-made ties."""
import itertools

import numpy as np
import pytest
import torch

from tacotron2_b200 import _capi, _engine
from tests import durations_oracle as DO


def check(alignments, input_lengths=None, mel_lengths=None, method="mas", device_type="cpu"):
    return _engine.duration_inputs(alignments, input_lengths, mel_lengths, method, device_type)


def test_valid_arguments_are_taken_as_fp32_with_int32_lengths():
    a = torch.rand(2, 7, 5, dtype=torch.float16)
    fa, il, ml, code = check(a)
    assert fa.dtype == torch.float32 and fa.is_contiguous() and torch.equal(fa, a.float())
    assert il is None and ml is None and code == _capi.DURATIONS_MAS
    for lengths in ([3, 5], torch.tensor([1, 5]), torch.tensor([2, 4], dtype=torch.int16)):
        _, il, ml, _ = check(a, lengths, [7, 6])
        assert il.dtype == ml.dtype == torch.int32 and il.tolist() == torch.as_tensor(lengths).tolist()
        assert ml.tolist() == [7, 6]
    assert check(a, method="argmax")[3] == _capi.DURATIONS_ARGMAX
    g = torch.rand(1, 3, 2, requires_grad=True)
    assert not check(g)[0].requires_grad
    # exact zeros (padding, a window) are valid weights; argmax takes rows with fewer frames than symbols
    check(torch.zeros(2, 3, 5), method="argmax")
    check(torch.rand(2, 3, 5), [3, 2], [3, 2])


@pytest.mark.parametrize("alignments,input_lengths,mel_lengths,method,err,match", [
    ([[[0.5]]], None, None, "mas", TypeError, "alignments must be a tensor"),
    (torch.ones(2, 4, 5, dtype=torch.int64), None, None, "mas", TypeError, "alignments must be a float"),
    (torch.ones(2, 4, 5, dtype=torch.bool), None, None, "mas", TypeError, "alignments must be a float"),
    (torch.rand(4, 5), None, None, "mas", ValueError, "alignments must have shape"),
    (torch.rand(1, 2, 4, 5), None, None, "mas", ValueError, "alignments must have shape"),
    (torch.rand(0, 4, 5), None, None, "mas", ValueError, "alignments must have shape"),
    (torch.rand(2, 0, 5), None, None, "mas", ValueError, "alignments must have shape"),
    (torch.rand(2, 4, 0), None, None, "mas", ValueError, "alignments must have shape"),
    (torch.rand(1, 1, 4097), None, None, "argmax", ValueError, "T_text must be at most 4096"),
    (torch.tensor([[[0.5, float("nan")]]]), None, None, "mas", ValueError, "finite and >= 0"),
    (torch.tensor([[[0.5, float("inf")]]]), None, None, "argmax", ValueError, "finite and >= 0"),
    (torch.tensor([[[0.5, -float("inf")]]]), None, None, "mas", ValueError, "finite and >= 0"),
    (torch.tensor([[[0.5, -1e-30]]]), None, None, "argmax", ValueError, "finite and >= 0"),
    (torch.tensor([[[0.5, 1e300]]], dtype=torch.float64), None, None, "mas", ValueError, "finite and >= 0"),
    (torch.rand(2, 4, 5), [1.0, 2.0], None, "mas", TypeError, "input_lengths must hold integers"),
    (torch.rand(2, 4, 5), None, torch.ones(2, dtype=torch.bool), "mas", TypeError, "mel_lengths must hold integers"),
    (torch.rand(2, 4, 5), [1, 2, 3], None, "mas", ValueError, r"input_lengths must have shape \(2,\)"),
    (torch.rand(2, 4, 5), None, torch.tensor([[4, 4]]), "mas", ValueError, r"mel_lengths must have shape \(2,\)"),
    (torch.rand(2, 4, 5), [0, 2], None, "mas", ValueError, "input_lengths must lie in 1..5"),
    (torch.rand(2, 4, 5), [1, 6], None, "argmax", ValueError, "input_lengths must lie in 1..5"),
    (torch.rand(2, 4, 5), None, [0, 4], "mas", ValueError, "mel_lengths must lie in 1..4"),
    (torch.rand(2, 4, 5), None, [4, 5], "argmax", ValueError, "mel_lengths must lie in 1..4"),
    (torch.rand(2, 4, 5), None, None, "mas", ValueError, r"rows \[0, 1\] have fewer frames than symbols"),
    (torch.rand(3, 6, 5), [5, 2, 4], [6, 1, 3], "mas", ValueError, r"rows \[1, 2\] have fewer frames than symbols"),
    (torch.rand(2, 4, 5), None, None, "viterbi", ValueError, "method must be one of"),
    (torch.rand(2, 4, 5), None, None, None, ValueError, "method must be one of"),
])
def test_bad_arguments_are_refused(alignments, input_lengths, mel_lengths, method, err, match):
    with pytest.raises(err, match=match):
        check(alignments, input_lengths, mel_lengths, method)


def test_a_cpu_map_is_refused():
    with pytest.raises(ValueError, match="must be on a CUDA device"):
        _engine.duration_inputs(torch.rand(1, 4, 3), None, None, "mas", "cuda")


# ---- the MAS oracle against every monotonic path ---------------------------------------------------------------------

def brute_force(a):
    """Every monotonic path through (T, N) as durations, with its fp64 score; the best score and the path MAS must
    return among those that reach it: the one that, read from the last frame back, stays on each symbol longest."""
    T, N = a.shape
    paths = []
    for adv in itertools.combinations(range(1, T), N - 1):           # the frames at which the path advances
        cuts = (0,) + adv + (T,)
        d = np.diff(cuts)
        paths.append((DO.path_score(a, d), d))
    best = max(s for s, _ in paths)
    tied = [d for s, d in paths if s == best]

    def backward_symbols(d):
        return tuple(np.repeat(np.arange(N), d)[::-1])
    return best, tied, max(tied, key=backward_symbols)


def small_maps():
    rng = np.random.default_rng(5)
    for T in range(1, 10):
        for N in range(1, min(T, 5) + 1):
            yield "uniform", np.full((T, N), 0.25, dtype=np.float32)
            yield "random", rng.random((T, N), dtype=np.float32)
            yield "softmax", torch.softmax(torch.from_numpy(rng.standard_normal((T, N)).astype(np.float32)) * 4, -1).numpy()
            # 0 / 1 entries: cells are 0 or log(FLT_MIN) exactly, so many paths tie exactly
            yield "binary", (rng.random((T, N)) < 0.5).astype(np.float32)
            z = rng.random((T, N), dtype=np.float32)
            z[rng.random((T, N)) < 0.4] = 0.0                        # exact-zero blocks
            yield "zeros", z


@pytest.mark.parametrize("kind", ["uniform", "random", "softmax", "binary", "zeros"])
def test_mas_oracle_takes_the_best_path_with_the_tie_rule(kind):
    n = 0
    for k, a in small_maps():
        if k != kind:
            continue
        best, tied, pick = brute_force(a)
        d = DO.mas(a)
        assert d.sum() == a.shape[0] and (d >= 1).all()
        assert DO.path_score(a, d) == best
        if kind in ("uniform", "binary"):                            # exact ties: the rule decides
            assert d.tolist() == pick.tolist(), (a, d, pick)
        elif len(tied) == 1:
            assert d.tolist() == tied[0].tolist()
        n += 1
    assert n == 35


@pytest.mark.parametrize("T,N", [(1, 1), (4, 1), (5, 5), (9, 3), (200, 7)])
def test_mas_oracle_on_a_uniform_map_advances_as_late_as_it_can(T, N):
    assert DO.mas(np.full((T, N), 1.0 / N)).tolist() == [1] * (N - 1) + [T - N + 1]
    assert DO.mas(np.zeros((T, N))).tolist() == [1] * (N - 1) + [T - N + 1]


def test_argmax_oracle_takes_the_first_of_tied_maxima():
    a = np.array([[0.2, 0.4, 0.4, 0.0],
                  [0.5, 0.1, 0.5, 0.5],
                  [0.0, 0.0, 0.0, 0.0],
                  [0.1, 0.2, 0.3, 0.3],
                  [0.0, 0.7, 0.1, 0.7]], dtype=np.float32)
    assert DO.argmax(a).tolist() == [2, 2, 1, 0]
    assert DO.argmax(a[:, :1]).tolist() == [5]
