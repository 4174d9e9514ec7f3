"""pYIN and per-symbol averaging without a GPU (DESIGN section 6.11): the numpy fp64 oracle ``tests/pyin_oracle.py``
that the GPU tests compare against -- its difference function against the time-domain sums, its Viterbi against
brute-force enumeration, the banded Viterbi the kernel runs against the dense one, the transition matrix, decoded
tones and silence -- the host tables of ``tacotron2_b200.pitch`` against the oracle's, and every host-side refusal."""
import itertools
import math

import numpy as np
import pytest
import torch

from tacotron2_b200 import pitch
from tests import pyin_oracle as PO

C2, C7 = 65.40639132514966, 2093.004522404789
SR = 22050


def test_difference_function_equals_the_time_domain_sums():
    rng = np.random.default_rng(0)
    y = np.sin(2 * np.pi * 180 * np.arange(4000) / SR) + 0.1 * rng.standard_normal(4000)
    frames = PO.frame(y, 1024, 256)
    assert frames.shape == (1 + 4000 // 256, 1024)
    mp = PO.periods(SR, C2, C7, 1024, 512)[1]
    d = PO.difference(frames, 1024, 512, mp)
    ref = PO.difference_direct(frames, 512, mp)
    assert np.abs(d - ref).max() <= 1e-10 * np.abs(ref).max()


def brute_force(log_prob, log_trans, log_init):
    """Among the best-scoring state sequences, the one whose reversed sequence is lexicographically smallest (the dense
    Viterbi's tie rule: the smallest final state, then at every step back the smallest predecessor)."""
    n_steps, n_states = log_prob.shape
    best, best_key = -np.inf, None
    for path in itertools.product(range(n_states), repeat=n_steps):
        s = log_prob[0, path[0]] + log_init[path[0]]
        for t in range(1, n_steps):
            s = log_prob[t, path[t]] + (s + log_trans[path[t - 1], path[t]])
        key = tuple(reversed(path))
        if s > best or (s == best and key < best_key):
            best, best_key = s, key
    return np.array(list(reversed(best_key)))


@pytest.mark.parametrize("seed", range(12))
def test_viterbi_equals_brute_force_with_ties_and_tiny_moves(seed):
    """Small integer logs make every sum exact, so ties are real; -708 entries stand for log(tiny)."""
    rng = np.random.default_rng(seed)
    n_states, n_steps = (4, 5) if seed % 2 else (3, 6)
    lp = rng.integers(-3, 1, (n_steps, n_states)).astype(float)
    lt = rng.integers(-2, 1, (n_states, n_states)).astype(float)
    lt[rng.random((n_states, n_states)) < 0.4] = -708.0
    lp[rng.random((n_steps, n_states)) < 0.3] = -708.0
    li = rng.integers(-1, 1, n_states).astype(float)
    got, gaps = PO.viterbi(lp, lt, li, gaps=True)
    assert np.array_equal(got, brute_force(lp, lt, li))
    assert np.array_equal(got, PO.viterbi(lp, lt, li))
    assert (gaps >= 0).all()


def banded_viterbi(log_prob, band, h, log_tiny, log_init):
    """The kernel's Viterbi restated in numpy: band[s][k][j] is the transition from bin j - h + k to bin j within
    (s = 0) or across (s = 1) the two halves; everything else is log_tiny.  Out-of-band maxima come from first-index
    prefix / suffix scans of v + log_tiny per half, and the pieces are visited in index order with a strict >."""
    n_steps, S = log_prob.shape
    nb = S // 2
    v = log_prob[0] + log_init
    ptr = np.zeros((n_steps, S), dtype=np.int64)

    def scan(vals, idx, reverse):
        out_v, out_i = vals.copy(), idx.copy()
        rng = range(nb - 2, -1, -1) if reverse else range(1, nb)
        for k in rng:
            o = k + 1 if reverse else k - 1
            if out_v[o] > out_v[k] or (out_v[o] == out_v[k] and out_i[o] < out_i[k]):
                out_v[k], out_i[k] = out_v[o], out_i[o]
        return out_v, out_i

    for t in range(1, n_steps):
        s = v + log_tiny
        pre = [scan(s[hs * nb:(hs + 1) * nb], np.arange(hs * nb, (hs + 1) * nb), False) for hs in range(2)]
        suf = [scan(s[hs * nb:(hs + 1) * nb], np.arange(hs * nb, (hs + 1) * nb), True) for hs in range(2)]
        nv = np.empty(S)
        for j in range(S):
            hj, jb = divmod(j, nb)
            lo, hi = jb - h, jb + h
            bv, bi = -np.inf, S
            for hs in range(2):
                if lo > 0:
                    c = (pre[hs][0][lo - 1], pre[hs][1][lo - 1])
                    if c[0] > bv or (c[0] == bv and c[1] < bi):
                        bv, bi = c
                for k in range(max(0, -lo), min(2 * h + 1, nb - lo)):
                    val = v[hs * nb + lo + k] + band[int(hs != hj), k, jb]
                    if val > bv:
                        bv, bi = val, hs * nb + lo + k
                if hi < nb - 1:
                    c = (suf[hs][0][hi + 1], suf[hs][1][hi + 1])
                    if c[0] > bv or (c[0] == bv and c[1] < bi):
                        bv, bi = c
            nv[j] = log_prob[t, j] + bv
            ptr[t, j] = bi
        v = nv
    state = np.zeros(n_steps, dtype=np.int64)
    state[-1] = np.argmax(v)
    for t in range(n_steps - 2, -1, -1):
        state[t] = ptr[t + 1, state[t + 1]]
    return state


@pytest.mark.parametrize("seed", range(8))
def test_banded_viterbi_equals_the_dense_one(seed):
    """Degenerate frames included: voiced_prob == 1 (unvoiced states at log(tiny)), voiced observations all zero,
    exact ties, and moves that only an out-of-band transition makes."""
    rng = np.random.default_rng(100 + seed)
    nb, width, steps = 9, (3, 5)[seed % 2], 12
    h = width // 2
    dense = PO.transition(nb, width, (0.01, 0.3)[seed % 2 == 0])
    log_tiny = np.log(PO.TINY)
    lt = np.log(dense + PO.TINY)
    band = np.full((2, 2 * h + 1, nb), log_tiny)
    for s in range(2):
        for k in range(2 * h + 1):
            for j in range(nb):
                i = j - h + k
                if 0 <= i < nb:
                    band[s, k, j] = lt[i + s * nb if s else i, j]
    obs = np.zeros((steps, 2 * nb))
    for t in range(steps):
        kind = rng.integers(0, 4)
        if kind == 0:                        # all voiced observations zero
            obs[t, nb:] = 1.0 / nb
        elif kind == 1:                      # voiced_prob == 1: one far bin, unvoiced 0
            obs[t, rng.integers(0, nb)] = 1.0
        else:
            bins = rng.choice(nb, 2, replace=False)
            obs[t, bins] = [0.25, 0.25] if kind == 2 else rng.random(2) * 0.5
            obs[t, nb:] = (1 - obs[t, :nb].sum()) / nb
    p_init = np.zeros(2 * nb)
    p_init[nb:] = 1 / nb
    lp, li = np.log(obs + PO.TINY), np.log(p_init + PO.TINY)
    assert np.array_equal(banded_viterbi(lp, band, h, log_tiny, li), PO.viterbi(lp, lt, li))


def test_transition_matrix_rows_sum_to_one_and_the_band_is_51_wide():
    assert PO.transition_width(SR, 256, 35.92, 0.1) == 51
    assert PO.n_pitch_bins(C2, C7) == 601
    T = PO.transition_local(601, 51)
    assert np.allclose(T.sum(1), 1, atol=1e-12)
    i, j = np.nonzero(T)
    assert np.abs(i - j).max() == 25
    assert all(np.count_nonzero(T[r]) == 51 for r in range(25, 576))
    K = PO.transition(601, 51, 0.01)
    assert K.shape == (1202, 1202) and np.allclose(K.sum(1), 1, atol=1e-12)
    assert np.allclose(K[:601, 601:], 0.01 * T) and np.allclose(K[601:, 601:], 0.99 * T)


@pytest.mark.parametrize("params", [dict(), dict(switch_prob=0.1, resolution=0.05, n_thresholds=37, no_trough_prob=0.2,
                                                 boltzmann_parameter=1.5, beta_parameters=(1, 10)),
                                    dict(frame_length=2048, fmin=40.0, fmax=1000.0)])
def test_host_tables_equal_the_oracle(params):
    args = dict(sr=SR, fmin=C2, fmax=C7, frame_length=1024)
    args.update(params)
    p = pitch.pyin_params(**args)
    t = pitch.pyin_tables(p)
    fl, wl, hop = p["frame_length"], p["win_length"], p["hop_length"]
    thr, beta, nb, w = PO.tables(SR, p["fmin"], args["fmax"], fl, wl, hop, p["n_thresholds"], p["beta"],
                                 p["boltzmann_parameter"], args.get("resolution", 0.1), 35.92, p["switch_prob"])
    assert (nb, w) == (p["n_bins"], p["width"])
    assert np.array_equal(t["thresholds"], thr[1:]) and np.array_equal(t["beta_probs"], beta)
    assert all(t["beta_prefix"][m] == np.sum(beta[:m]) for m in range(len(beta) + 1))
    lt = np.log(PO.transition(nb, w, p["switch_prob"]) + PO.TINY)
    h = w // 2
    for s in range(2):
        for k in range(2 * h + 1):
            j = np.arange(nb)
            i = j - h + k
            ok = (i >= 0) & (i < nb)
            assert np.array_equal(t["log_trans"][s, k, ok], lt[i[ok] + s * nb, j[ok]])
    i, j = np.meshgrid(np.arange(nb), np.arange(nb), indexing="ij")
    assert (lt[:nb, :nb][np.abs(i - j) > h] == t["log_tiny"]).all()
    assert (lt[nb:, :nb][np.abs(i - j) > h] == t["log_tiny"]).all()
    n_max = (p["max_period"] - p["min_period"] + 2) // 2
    for N in (1, 2, 7, n_max):
        import scipy.stats
        assert np.array_equal(t["boltzmann"][N * (N - 1) // 2:N * (N + 1) // 2],
                              scipy.stats.boltzmann.pmf(np.arange(N), p["boltzmann_parameter"], N))
    assert len(t["boltzmann"]) == n_max * (n_max + 1) // 2
    assert t["log_init_unvoiced"] == np.log(1 / nb + PO.TINY)


def tone(f, seconds=0.6, harmonics=1, amp=0.5):
    tt = np.arange(int(SR * seconds)) / SR
    return (amp * sum(np.sin(2 * np.pi * f * k * tt) / k for k in range(1, harmonics + 1))).astype(np.float32)


@pytest.mark.parametrize("f", [80.0, 220.0, 900.0])
@pytest.mark.parametrize("harmonics", [1, 4])
def test_tones_decode_voiced_at_their_bin(f, harmonics):
    f0, voiced, prob = PO.pyin(tone(f, harmonics=harmonics), C2, C7)
    mid = slice(4, len(f0) - 4)
    assert voiced[mid].all() and (prob[mid] > 0.5).all()
    want = 120 * np.log2(f / C2)
    assert np.abs(120 * np.log2(f0[mid] / C2) - want).max() <= 1.0 + 1e-9


def test_silence_decodes_unvoiced():
    f0, voiced, prob = PO.pyin(np.zeros(5000, dtype=np.float32), C2, C7)
    assert not voiced.any() and np.isnan(f0).all() and (prob == 0).all()
    f0, voiced, _ = PO.pyin(np.zeros(5000, dtype=np.float32), C2, C7, fill_na=0.0)
    assert (f0 == 0).all()


def test_average_pitch_oracle():
    v = np.array([0, 100, np.nan, 200, 0, 0, 300, 301])
    got = PO.average_pitch(v, [2, 3, 1, 2, 0])
    assert np.array_equal(got, [100.0, 200.0, 0.0, 300.5, 0.0])


# ---- host-side refusals ----------------------------------------------------------------------------------------------
def params(**kw):
    a = dict(sr=SR, fmin=C2, fmax=C7)
    a.update(kw)
    return pitch.pyin_params(**a)


def test_valid_parameters_derive_librosas_quantities():
    p = params()
    assert (p["min_period"], p["max_period"], p["n_bins"], p["width"]) == (10, 338, 601, 51)
    assert (p["win_length"], p["hop_length"], p["bins_per_semitone"]) == (512, 256, 10)
    p = params(frame_length=2048, resolution=0.05)
    assert (p["win_length"], p["hop_length"], p["n_bins"], p["width"]) == (1024, 512, 1201, 201)


@pytest.mark.parametrize("kw,err,match", [
    (dict(center=False), ValueError, "center must be True"),
    (dict(pad_mode="reflect"), ValueError, "pad_mode must be 'constant'"),
    (dict(fmin=500.0, fmax=400.0), ValueError, "fmin .* must be below fmax"),
    (dict(fmin=400.0, fmax=400.0), ValueError, "fmin .* must be below fmax"),
    (dict(fmax=12000.0), ValueError, r"fmax .* must be at most sr / 2"),
    (dict(frame_length=4096), ValueError, "frame_length must lie in"),
    (dict(frame_length=1024.0), TypeError, "frame_length must be an integer"),
    (dict(frame_length=16), ValueError, "max_period .* must exceed min_period"),
    (dict(win_length=1024), ValueError, "win_length must lie in"),
    (dict(hop_length=0), ValueError, "hop_length must lie in"),
    (dict(sr=0), ValueError, "sr must lie in"),
    (dict(fmin=float("nan")), ValueError, "fmin must lie in"),
    (dict(fmin=-1.0), ValueError, "fmin must lie in"),
    (dict(fmin=20.0, fmax=11000.0, resolution=0.05), ValueError, "pitch bins .* exceed 1536"),
    (dict(n_thresholds=0), ValueError, "n_thresholds must lie in"),
    (dict(beta_parameters=(2,)), TypeError, "beta_parameters must be a pair"),
    (dict(beta_parameters=(2, -1)), ValueError, "beta_parameters must lie in"),
    (dict(boltzmann_parameter=0), ValueError, "boltzmann_parameter must lie in"),
    (dict(resolution=0), ValueError, "resolution must lie in"),
    (dict(switch_prob=1.5), ValueError, "switch_prob must lie in"),
    (dict(no_trough_prob=-0.1), ValueError, "no_trough_prob must lie in"),
    (dict(max_transition_rate=-1), ValueError, "max_transition_rate must lie in"),
    (dict(max_transition_rate=1e4), ValueError, "transition width .* exceeds"),
    (dict(fill_na="nan"), TypeError, "fill_na must be a real number"),
])
def test_parameter_refusals(kw, err, match):
    with pytest.raises(err, match=match):
        params(**kw)


def test_valid_inputs_are_taken_as_fp32_with_int32_lengths():
    y = torch.rand(3, 700, dtype=torch.float16)
    x, ln, one = pitch.pyin_inputs(y, [700, 1, 350], "cpu")
    assert x.dtype == torch.float32 and torch.equal(x, y.float()) and ln.dtype == torch.int32 and not one
    x, ln, one = pitch.pyin_inputs(torch.rand(50), None, "cpu")
    assert x.shape == (1, 50) and ln is None and one


@pytest.mark.parametrize("y,lengths,err,match", [
    ([0.0, 1.0], None, TypeError, "y must be a tensor"),
    (torch.ones(2, 10, dtype=torch.int32), None, TypeError, "y must be a float tensor"),
    (torch.ones(2, 3, 10), None, ValueError, "y must have shape"),
    (torch.ones(2, 0), None, ValueError, "y must have shape"),
    (torch.tensor([0.0, float("nan")]), None, ValueError, "y must be finite"),
    (torch.tensor([[0.0, float("inf")]]), None, ValueError, "y must be finite"),
    (torch.ones(2, 10), [10], ValueError, r"lengths must have shape \(2,\)"),
    (torch.ones(2, 10), [0, 10], ValueError, "lengths must lie in 1..10"),
    (torch.ones(2, 10), [3, 11], ValueError, "lengths must lie in 1..10"),
    (torch.ones(2, 10), [3.0, 4.0], TypeError, "lengths must hold integers"),
    (torch.ones(10), [3], ValueError, "lengths needs y of shape"),
])
def test_input_refusals(y, lengths, err, match):
    with pytest.raises(err, match=match):
        pitch.pyin_inputs(y, lengths, "cpu")


def test_cpu_tensors_are_refused():
    with pytest.raises(ValueError, match="y must be on a CUDA device"):
        pitch.pyin(torch.zeros(1000), C2, C7)
    with pytest.raises(ValueError, match="values must be on a CUDA device"):
        pitch.average_by_durations(torch.zeros(2, 5), torch.ones(2, 3, dtype=torch.int64))


@pytest.mark.parametrize("values,durations,err,match", [
    ([[1.0]], [[1]], TypeError, "values must be a tensor"),
    (torch.ones(2, 5, dtype=torch.int64), torch.ones(2, 3, dtype=torch.int64), TypeError, "values must be a float"),
    (torch.ones(5), torch.ones(2, 3, dtype=torch.int64), ValueError, "values must have shape"),
    (torch.ones(2, 5), torch.ones(2, 3), TypeError, "durations must hold integers"),
    (torch.ones(2, 5), torch.ones(3, 3, dtype=torch.int64), ValueError, r"durations must have shape \(2, T_text"),
    (torch.ones(2, 5), torch.ones(2, dtype=torch.int64), ValueError, r"durations must have shape \(2, T_text"),
    (torch.ones(2, 5), torch.tensor([[1, -1, 2], [0, 0, 0]]), ValueError, "durations must be >= 0"),
    (torch.ones(2, 5), torch.tensor([[1, 1, 2], [3, 3, 0]]), ValueError, r"rows \[1\] sum to more than the 5 frames"),
])
def test_average_refusals(values, durations, err, match):
    with pytest.raises(err, match=match):
        pitch.average_inputs(values, durations, "cpu")


def test_average_inputs_take_fp64_and_int64():
    v, d = pitch.average_inputs(torch.ones(2, 5, dtype=torch.float16), torch.tensor([[1, 4], [5, 0]],
                                                                                     dtype=torch.int32), "cpu")
    assert v.dtype == torch.float64 and d.dtype == torch.int64 and not math.isnan(float(v.sum()))
