"""Dynamic time warping, MCD and f0 frame errors without a GPU: the numpy fp64 oracle (``tests/dtw_oracle.py``) on
hand-worked cases and against brute-force enumeration of every warping path with its tie rule, the DCT table against
scipy, the pitch measures' torch arithmetic against the oracle, and every host-side refusal of ``dtw``,
``mel_cepstral_distortion`` and ``pitch_errors`` (through their validation helpers, on CPU tensors)."""
import math

import numpy as np
import pytest
import scipy.fft
import torch

from tacotron2_b200 import _capi, evaluation as E
from tests import dtw_oracle as O


def seq(*v):
    return np.array([v], np.float64)                   # one feature, D = 1


# ---- the oracle on hand-worked cases ---------------------------------------------------------------------------------

def test_hand_worked_3x4_with_a_tie_between_diagonal_and_up():
    # C = |x_i - y_j| = [[0 0 1 1], [1 1 0 0], [0 0 1 1]].  D row 0: 0 0 1 2; row 1: 1 1 0 0; row 2: 1 1 1 1.
    # D[2, 3] = C + min(D[1, 2] = 0 (diagonal), D[2, 2] = 1, D[1, 3] = 0): the diagonal wins the tie with up.
    cost, path = O.dtw(seq(0, 1, 0), seq(0, 0, 1, 1))
    assert cost == 1.0
    assert path.tolist() == [[0, 0], [0, 1], [1, 2], [2, 3]]


def test_hand_worked_4x3_with_a_tie_between_left_and_up():
    # C = |x_i - y_j| = [[1 2 0], [1 2 0], [1 2 0], [1 0 2]];  D = [[1 3 3], [2 3 3], [3 4 3], [4 3 5]].
    # D[3, 2] = C + min(D[2, 1] = 4 (diagonal), D[3, 1] = 3 (left), D[2, 2] = 3 (up)): left wins the tie with up;
    # D[3, 1] = C + min(D[2, 0] = 3, D[3, 0] = 4, D[2, 1] = 4): diagonal; then up along column 0.
    cost, path = O.dtw(seq(0, 0, 0, 2), seq(1, 2, 0))
    assert cost == 5.0
    assert path.tolist() == [[0, 0], [1, 0], [2, 0], [3, 1], [3, 2]]


def all_paths(Lx, Ly):
    """Every warping path from (0, 0) to (Lx - 1, Ly - 1), each with its backward step codes."""
    out = []

    def walk(i, j, cells, steps):
        if i == 0 and j == 0:
            out.append((cells[::-1], tuple(steps)))
            return
        for code, (di, dj) in ((O.DIAG, (1, 1)), (O.LEFT, (0, 1)), (O.UP, (1, 0))):
            if i - di >= 0 and j - dj >= 0:
                walk(i - di, j - dj, cells + [(i - di, j - dj)], steps + [code])
    walk(Lx - 1, Ly - 1, [(Lx - 1, Ly - 1)], [])
    return out


@pytest.mark.parametrize("Lx,Ly", [(1, 1), (1, 4), (4, 1), (2, 2), (3, 4), (4, 3), (5, 5)])
def test_oracle_takes_the_cheapest_path_and_breaks_ties_diagonal_left_up(Lx, Ly):
    """Integer-valued frames with D = 1 make every distance and every sum exact, so tied paths tie exactly.  Among the
    cheapest paths the rule picks, walking back from the end, the first step that differs as diagonal before left
    before up."""
    rng = np.random.default_rng(Lx * 10 + Ly)
    paths = all_paths(Lx, Ly)
    ties = 0
    for _ in range(40):
        x, y = rng.integers(0, 4, (1, Lx)).astype(np.float64), rng.integers(0, 4, (1, Ly)).astype(np.float64)
        C = O.distances(x, y)
        cost, path = O.dtw(x, y)
        costs = [sum(C[i, j] for i, j in cells) for cells, _ in paths]
        best = min(costs)
        tied = [p for p, c in zip(paths, costs) if c == best]
        pick = min(tied, key=lambda p: p[1])
        assert cost == best
        assert path.tolist() == [list(c) for c in pick[0]]
        ties += len(tied) > 1
    assert min(Lx, Ly) < 2 or ties > 0


def test_identical_sequences_cost_zero_on_the_diagonal():
    x = np.random.default_rng(0).standard_normal((80, 37))
    cost, path = O.dtw(x, x)
    assert cost == 0.0 and path.tolist() == [[t, t] for t in range(37)]


def test_frames_repeated_by_a_monotone_map_cost_zero():
    rng = np.random.default_rng(1)
    x = rng.standard_normal((5, 30))
    idx = np.sort(np.concatenate([np.arange(30), rng.integers(0, 30, 25)]))    # every frame at least once
    cost, path = O.dtw(x, x[:, idx])
    assert cost == 0.0
    assert all(np.array_equal(x[:, i], x[:, idx[j]]) for i, j in path)


@pytest.mark.parametrize("Lx,Ly", [(1, 1), (1, 9), (9, 1), (13, 40), (40, 13), (64, 64)])
def test_path_is_a_warping_path_of_bounded_length(Lx, Ly):
    rng = np.random.default_rng(Lx + 100 * Ly)
    cost, path = O.dtw(rng.standard_normal((3, Lx)), rng.standard_normal((3, Ly)))
    assert max(Lx, Ly) <= len(path) <= Lx + Ly - 1
    assert path[0].tolist() == [0, 0] and path[-1].tolist() == [Lx - 1, Ly - 1]
    steps = np.diff(path, axis=0)
    assert set(map(tuple, steps.tolist())) <= {(1, 1), (0, 1), (1, 0)}


def test_distances_sum_sequentially_over_d():
    rng = np.random.default_rng(2)
    x, y = rng.standard_normal((80, 4)), rng.standard_normal((80, 3))
    C = O.distances(x, y)
    for i in range(4):
        for j in range(3):
            s = 0.0
            for d in range(80):
                s = s + (x[d, i] - y[d, j]) * (x[d, i] - y[d, j])
            assert C[i, j] == math.sqrt(s)


# ---- cepstra and MCD -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n_mel,n_cep", [(80, 24), (80, 79), (2, 1), (128, 40)])
def test_dct_table_is_scipys_orthonormal_dct(n_mel, n_cep):
    assert np.array_equal(E.dct_table(n_mel, n_cep), O.dct_table(n_mel, n_cep))
    mel = np.log(np.maximum(np.random.default_rng(n_mel).random((n_mel, 17)), 1e-5))
    want = scipy.fft.dct(mel, type=2, norm="ortho", axis=0)[1:n_cep + 1]
    np.testing.assert_allclose(O.cepstra(mel, n_cep), want, rtol=0, atol=1e-12 * np.abs(want).max())


def test_mcd_of_a_mel_with_itself_is_zero_and_scales_by_the_path_length():
    mel = np.log(np.maximum(np.random.default_rng(3).random((80, 50)), 1e-5))
    assert O.mcd(mel, mel)[0] == 0.0
    other = mel + 0.1
    m, path = O.mcd(mel, other)                        # a level shift changes c_0 only
    assert abs(m) < 1e-12
    cost, _ = O.dtw(O.cepstra(mel, 24), O.cepstra(mel[:, ::-1].copy(), 24))
    m, path = O.mcd(mel, mel[:, ::-1].copy())
    assert m == O.MCD_SCALE * cost / len(path) and E.MCD_SCALE == O.MCD_SCALE


# ---- pitch errors ----------------------------------------------------------------------------------------------------

def hand_tracks():
    """Six path pairs: both voiced within 20 % (2), both voiced off by more than 20 % (1), voicing differs (2),
    both unvoiced (1)."""
    f0_x = np.array([100.0, 110.0, 200.0, 150.0, np.nan, np.nan])
    v_x = np.array([True, True, True, True, False, False])
    f0_y = np.array([100.0, 100.0, 150.0, np.nan, 120.0, np.nan])
    v_y = np.array([True, True, True, False, True, False])
    path = np.array([[t, t] for t in range(6)])
    return f0_x, v_x, f0_y, v_y, path


def test_pitch_error_definitions_on_hand_made_flags():
    got = O.pitch_errors(*hand_tracks())
    cents = 1200 * np.log2(np.array([1.0, 1.1, 200 / 150]))
    assert got["gpe"] == 1 / 3 and got["vde"] == 2 / 6 and got["ffe"] == 3 / 6
    assert got["f0_rmse_cents"] == pytest.approx(math.sqrt(np.mean(cents ** 2)), rel=1e-14)
    # no pair voiced in both: GPE and the RMSE are NaN, VDE and FFE are not
    f0_x, v_x, f0_y, v_y, path = hand_tracks()
    got = O.pitch_errors(f0_x, v_x, f0_y, ~v_x, path)
    assert math.isnan(got["gpe"]) and math.isnan(got["f0_rmse_cents"]) and got["vde"] == 1.0 and got["ffe"] == 1.0


def test_frame_errors_match_the_oracle_along_ragged_paths():
    f0_x, v_x, f0_y, v_y, path = hand_tracks()
    rng = np.random.default_rng(4)
    B, F = 3, 40
    fx = rng.uniform(80, 300, (B, F))
    fy = fx * rng.uniform(0.7, 1.3, (B, F))
    vx, vy = rng.random((B, F)) < 0.7, rng.random((B, F)) < 0.7
    fx[~vx] = np.nan
    fy[~vy] = np.nan
    paths = [O.dtw(rng.standard_normal((2, F)), rng.standard_normal((2, F)))[1] for _ in range(B - 1)] + [path]
    fx[2, :6], vx[2, :6], fy[2, :6], vy[2, :6] = f0_x, v_x, f0_y, v_y
    P = 2 * F - 1
    pt = torch.full((B, P, 2), -1, dtype=torch.int64)
    for b, p in enumerate(paths):
        pt[b, :len(p)] = torch.from_numpy(p)
    n = torch.tensor([len(p) for p in paths])
    args = [torch.from_numpy(a) for a in (fx, vx, fy, vy)]
    p, n = E.pitch_inputs(*args, pt, n, device_type="cpu")
    got = E.frame_errors(*args, p, n)
    for b in range(B):
        want = O.pitch_errors(fx[b], vx[b], fy[b], vy[b], paths[b])
        for k in ("gpe", "vde", "ffe"):
            assert float(got[k][b]) == want[k], (b, k)
        assert float(got["f0_rmse_cents"][b]) == pytest.approx(want["f0_rmse_cents"], rel=1e-12)


# ---- refusals --------------------------------------------------------------------------------------------------------

def check_dtw(x, y, xl=None, yl=None):
    return E.dtw_inputs(x, y, xl, yl, device_type="cpu")


def test_valid_dtw_arguments_are_taken_as_they_are():
    x, y = torch.rand(2, 3, 7), torch.rand(2, 3, 5)
    a, b, xl, yl, code = check_dtw(x, y)
    assert a.data_ptr() == x.data_ptr() and b.data_ptr() == y.data_ptr() and xl is None and yl is None and code == _capi.DTW_F32
    _, _, xl, yl, code = check_dtw(x.double(), y.double(), [7, 1], torch.tensor([5, 2], dtype=torch.int16))
    assert code == _capi.DTW_F64 and xl.dtype == yl.dtype == torch.int32 and xl.tolist() == [7, 1]
    a = check_dtw(x.transpose(1, 2).contiguous().transpose(1, 2), y)[0]
    assert a.is_contiguous() and torch.equal(a, x)
    check_dtw(torch.rand(1, 1024, 1), torch.rand(1, 1024, 8192))


@pytest.mark.parametrize("x,y,xl,yl,err,match", [
    ([[[0.5]]], torch.rand(1, 1, 1), None, None, TypeError, "x must be a tensor"),
    (torch.rand(1, 1, 1), None, None, None, TypeError, "y must be a tensor"),
    (torch.rand(1, 2, 3).half(), torch.rand(1, 2, 3).half(), None, None, TypeError, "x must be float32 or float64"),
    (torch.rand(1, 2, 3), torch.ones(1, 2, 3, dtype=torch.int64), None, None, TypeError, "y must be float32 or float64"),
    (torch.rand(1, 2, 3), torch.rand(1, 2, 3).double(), None, None, TypeError, "the same dtype"),
    (torch.rand(2, 3), torch.rand(1, 2, 3), None, None, ValueError, r"x must have shape \(B, D, T\)"),
    (torch.rand(1, 2, 3), torch.rand(1, 2, 3, 1), None, None, ValueError, r"y must have shape \(B, D, T\)"),
    (torch.rand(0, 2, 3), torch.rand(0, 2, 3), None, None, ValueError, "x must have shape"),
    (torch.rand(1, 0, 3), torch.rand(1, 0, 3), None, None, ValueError, "x must have shape"),
    (torch.rand(1, 2, 3), torch.rand(1, 2, 0), None, None, ValueError, "y must have shape"),
    (torch.rand(1, 2, 3), torch.rand(2, 2, 3), None, None, ValueError, "must agree in B and D"),
    (torch.rand(1, 2, 3), torch.rand(1, 3, 3), None, None, ValueError, "must agree in B and D"),
    (torch.rand(1, 1025, 1), torch.rand(1, 1025, 1), None, None, ValueError, "D must be at most 1024"),
    (torch.rand(1, 1, 8193), torch.rand(1, 1, 1), None, None, ValueError, "T_x and T_y must be at most 8192"),
    (torch.rand(1, 1, 1), torch.rand(1, 1, 8193), None, None, ValueError, "T_x and T_y must be at most 8192"),
    (torch.rand(2, 2, 3), torch.rand(2, 2, 4), [1.0, 2.0], None, TypeError, "x_lengths must hold integers"),
    (torch.rand(2, 2, 3), torch.rand(2, 2, 4), None, torch.ones(2, dtype=torch.bool), TypeError,
     "y_lengths must hold integers"),
    (torch.rand(2, 2, 3), torch.rand(2, 2, 4), [1, 2, 3], None, ValueError, r"x_lengths must have shape \(2,\)"),
    (torch.rand(2, 2, 3), torch.rand(2, 2, 4), [0, 3], None, ValueError, "x_lengths must lie in 1..3"),
    (torch.rand(2, 2, 3), torch.rand(2, 2, 4), [1, 4], None, ValueError, "x_lengths must lie in 1..3"),
    (torch.rand(2, 2, 3), torch.rand(2, 2, 4), None, [4, 5], ValueError, "y_lengths must lie in 1..4"),
    (torch.rand(2, 2, 3), torch.rand(2, 2, 4), None, [0, 1], ValueError, "y_lengths must lie in 1..4"),
])
def test_bad_dtw_arguments_are_refused(x, y, xl, yl, err, match):
    with pytest.raises(err, match=match):
        check_dtw(x, y, xl, yl)


def test_cpu_tensors_are_refused():
    with pytest.raises(ValueError, match="x must be on a CUDA device"):
        E.dtw_inputs(torch.rand(1, 2, 3), torch.rand(1, 2, 3))
    with pytest.raises(ValueError, match="mel_cepstral_distortion: x must be on a CUDA device"):
        E.mcd_inputs(torch.rand(1, 80, 3), torch.rand(1, 80, 3))
    f0, v = torch.rand(1, 5), torch.ones(1, 5, dtype=torch.bool)
    with pytest.raises(ValueError, match="f0_x must be on a CUDA device"):
        E.pitch_inputs(f0, v, f0, v, torch.zeros(1, 9, 2, dtype=torch.int64), [1])


@pytest.mark.parametrize("n_mel,n_cep,err,match", [
    (80, 0, ValueError, r"n_cep must lie in 1..n_mel - 1 = 79"),
    (80, 80, ValueError, r"n_cep must lie in 1..n_mel - 1 = 79"),
    (1, 1, ValueError, r"n_cep must lie in 1..n_mel - 1 = 0"),
    (80, 24.0, TypeError, "n_cep must be an integer"),
    (80, True, TypeError, "n_cep must be an integer"),
])
def test_bad_n_cep_is_refused(n_mel, n_cep, err, match):
    with pytest.raises(err, match=match):
        E.mcd_inputs(torch.rand(1, n_mel, 3), torch.rand(1, n_mel, 4), n_cep=n_cep, device_type="cpu")
    E.mcd_inputs(torch.rand(1, 80, 3), torch.rand(1, 80, 4), n_cep=79, device_type="cpu")


def test_mcd_refuses_what_dtw_refuses_under_its_own_name():
    with pytest.raises(ValueError, match="mel_cepstral_distortion: B must be at most 65535"):
        E.mcd_inputs(torch.rand(65536, 2, 1), torch.rand(65536, 2, 1), n_cep=1, device_type="cpu")
    with pytest.raises(ValueError, match="mel_cepstral_distortion: x .* must agree in B and D"):
        E.mcd_inputs(torch.rand(1, 80, 3), torch.rand(1, 40, 3), device_type="cpu")
    with pytest.raises(TypeError, match="mel_cepstral_distortion: x must be float32 or float64"):
        E.mcd_inputs(torch.rand(1, 80, 3).half(), torch.rand(1, 80, 3).half(), device_type="cpu")


def pitch_args(**kw):
    f0, v = torch.rand(2, 5) + 1, torch.ones(2, 5, dtype=torch.bool)
    path = torch.zeros(2, 9, 2, dtype=torch.int64)
    a = dict(f0_x=f0, voiced_x=v, f0_y=torch.rand(2, 6) + 1, voiced_y=torch.ones(2, 6, dtype=torch.bool), path=path,
             path_lengths=torch.tensor([1, 9]))
    a.update(kw)
    return a


@pytest.mark.parametrize("kw,err,match", [
    (dict(f0_x=[[1.0]]), TypeError, "f0_x must be a float tensor"),
    (dict(f0_y=torch.ones(2, 6, dtype=torch.int64)), TypeError, "f0_y must be a float tensor"),
    (dict(f0_x=torch.rand(10)), ValueError, r"f0_x must have shape \(B, F\)"),
    (dict(voiced_x=torch.ones(2, 5)), TypeError, "voiced_x must be a bool tensor"),
    (dict(voiced_y=torch.ones(2, 5, dtype=torch.bool)), ValueError, "voiced_y must have f0_y's shape"),
    (dict(f0_y=torch.rand(3, 6), voiced_y=torch.ones(3, 6, dtype=torch.bool)), ValueError, "f0_y must have f0_x's B"),
    (dict(path=torch.zeros(2, 9, 2)), TypeError, "path must hold integers"),
    (dict(path=torch.zeros(2, 9, 3, dtype=torch.int64)), ValueError, r"path must have shape \(2, P >= 1, 2\)"),
    (dict(path=torch.zeros(2, 0, 2, dtype=torch.int64)), ValueError, r"path must have shape"),
    (dict(path_lengths=[1, 2, 3]), ValueError, r"path_lengths must have shape \(2,\)"),
    (dict(path_lengths=[1.0, 2.0]), TypeError, "path_lengths must hold integers"),
    (dict(path_lengths=[0, 2]), ValueError, "path_lengths must lie in 1..9"),
    (dict(path_lengths=[1, 10]), ValueError, "path_lengths must lie in 1..9"),
    (dict(path=torch.tensor([[[0, 0]] * 8 + [[5, 0]]] * 2)), ValueError, r"frames must lie in \[0, 5\) x \[0, 6\)"),
    (dict(path=torch.tensor([[[0, 0]] * 8 + [[0, 6]]] * 2)), ValueError, r"frames must lie in"),
    (dict(path=torch.tensor([[[0, 0]] * 8 + [[-1, 0]]] * 2)), ValueError, r"frames must lie in"),
])
def test_bad_pitch_arguments_are_refused(kw, err, match):
    with pytest.raises(err, match=match):
        E.pitch_inputs(**pitch_args(**kw), device_type="cpu")


def test_padding_past_the_path_length_is_not_checked():
    path = torch.full((2, 9, 2), -1, dtype=torch.int64)
    path[:, 0] = 0
    E.pitch_inputs(**pitch_args(path=path, path_lengths=[1, 1]), device_type="cpu")
