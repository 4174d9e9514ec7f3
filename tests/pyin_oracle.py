"""numpy fp64 oracle of ``tacotron2_b200.pyin`` (DESIGN section 6.11): librosa 0.10's ``pyin`` with ``center=True,
pad_mode="constant"``, restated step by step with librosa's names, for one clip at a time.  librosa itself is not a
dependency, so parity with it stays unpinned; this file is the contract the GPU is tested against.

Also ``average_pitch``: FastPitch's per-symbol average of the non-zero (and non-NaN) frame values over durations."""
import math

import numpy as np
import scipy.stats

TINY = np.finfo(np.float64).tiny


def frame(y, frame_length, hop_length):
    """Zero-pad by frame_length // 2 on both sides, then frames (n_frames, frame_length): 1 + len(y) // hop frames."""
    y = np.asarray(y, dtype=np.float64)
    pad = frame_length // 2
    yp = np.pad(y, (pad, pad), mode="constant")
    n = 1 + (len(yp) - frame_length) // hop_length
    idx = np.arange(frame_length)[None, :] + hop_length * np.arange(n)[:, None]
    return yp[idx]


def periods(sr, fmin, fmax, frame_length, win_length):
    return int(np.floor(sr / fmax)), min(int(np.ceil(sr / fmin)), frame_length - win_length - 1)


def difference(frames, frame_length, win_length, max_period):
    """librosa's FFT form: acf[tau] = sum_{j=1..W} x[j] x[j+tau] and e[tau] = sum_{j=tau+1..tau+W} x[j]^2 (a difference of
    cumulative sums), each zeroed where |.| < 1e-6; returns d[tau] = e[0] + e[tau] - 2 acf[tau] for tau in 0..max_period."""
    W = win_length
    a = np.fft.rfft(frames, frame_length, axis=-1)
    b = np.fft.rfft(frames[:, W:0:-1], frame_length, axis=-1)
    acf = np.fft.irfft(a * b, frame_length, axis=-1)[:, W:]
    acf[np.abs(acf) < 1e-6] = 0
    energy = np.cumsum(frames ** 2, axis=-1)
    energy = energy[:, W:] - energy[:, :-W]
    energy[np.abs(energy) < 1e-6] = 0
    d = energy[:, :1] + energy - 2 * acf
    return d[:, :max_period + 1]


def difference_direct(frames, win_length, max_period):
    """The same d from the time-domain sums, without zeroing (the test's statement of what the FFT form computes)."""
    W = win_length
    x = np.asarray(frames, dtype=np.float64)
    acf = np.stack([np.sum(x[:, 1:W + 1] * x[:, 1 + t:W + 1 + t], axis=1) for t in range(max_period + 1)], 1)
    e = np.stack([np.sum(x[:, t + 1:t + W + 1] ** 2, axis=1) for t in range(max_period + 1)], 1)
    return e[:, :1] + e - 2 * acf


def cmnd(d, min_period, max_period):
    """yin[tau] = d[tau] / (mean(d[1..tau]) + tiny) for tau in min_period..max_period: (n_frames, n_lags)."""
    cm = np.cumsum(d[:, 1:max_period + 1], axis=-1) / np.arange(1, max_period + 1)
    return d[:, min_period:max_period + 1] / (cm[:, min_period - 1:max_period] + TINY)


def parabolic_shifts(yin):
    """librosa 0.10's __parabolic_interpolation over the lag axis; the first and last shifts are 0."""
    s = np.zeros_like(yin)
    a = yin[:, 2:] + yin[:, :-2] - 2 * yin[:, 1:-1]
    b = (yin[:, 2:] - yin[:, :-2]) / 2
    with np.errstate(divide="ignore", invalid="ignore"):
        s[:, 1:-1] = np.where(np.abs(b) >= np.abs(a), 0.0, -b / a)
    return s


def troughs(frame_yin):
    """Strict left, non-strict right local minima; lag 0 if below lag 1; the last lag if below its left neighbour."""
    y = frame_yin
    t = np.zeros(len(y), dtype=bool)
    t[1:-1] = (y[1:-1] < y[:-2]) & (y[1:-1] <= y[2:])
    t[0] = y[0] < y[1]
    t[-1] = y[-1] < y[-2]
    return np.nonzero(t)[0]


def n_bins_per_semitone(resolution):
    return int(np.ceil(1.0 / resolution))


def n_pitch_bins(fmin, fmax, resolution=0.1):
    return int(np.floor(12 * n_bins_per_semitone(resolution) * np.log2(fmax / fmin))) + 1


def transition_width(sr, hop_length, max_transition_rate, resolution):
    return round(max_transition_rate * 12 * hop_length / sr) * n_bins_per_semitone(resolution) + 1


def triang(M):
    """scipy.signal.windows.triang(M, sym=True)."""
    n = np.arange(1, (M + 1) // 2 + 1)
    if M % 2 == 0:
        w = (2 * n - 1.0) / M
        return np.r_[w, w[::-1]]
    w = 2 * n / (M + 1.0)
    return np.r_[w, w[-2::-1]]


def transition_local(n_states, width):
    """librosa.sequence.transition_local(n_states, width, window="triangle", wrap=False)."""
    T = np.zeros((n_states, n_states), dtype=np.float64)
    win = triang(width)
    for i in range(n_states):
        row = np.zeros(n_states)
        lpad = (n_states - width) // 2
        row[lpad:lpad + width] = win
        row = np.roll(row, n_states // 2 + i + 1)
        row[min(n_states, i + width // 2 + 1):] = 0
        row[:max(0, i - width // 2)] = 0
        T[i] = row
    T /= T.sum(axis=1, keepdims=True)
    return T


def transition_loop(n_states, prob):
    """librosa.sequence.transition_loop(n_states, prob) for a scalar prob."""
    T = np.empty((n_states, n_states), dtype=np.float64)
    for i in range(n_states):
        T[i] = (1.0 - prob) / (n_states - 1)
        T[i, i] = prob
    return T


def transition(n_bins, width, switch_prob):
    return np.kron(transition_loop(2, 1 - switch_prob), transition_local(n_bins, width))


def viterbi(log_prob, log_trans, log_p_init, gaps=False):
    """librosa.sequence.viterbi on logs: log_prob (n_steps, n_states).  Ties go to the smallest index.  With gaps, also
    returns the gap between the best and the runner-up predecessor of every state on the path (and of the final argmax):
    the margin by which the path's discrete decisions were made."""
    n_steps, n_states = log_prob.shape
    value = log_prob[0] + log_p_init
    ptr = np.zeros((n_steps, n_states), dtype=np.int64)
    top2 = np.zeros((n_steps, n_states))
    for t in range(1, n_steps):
        trans_out = value[:, None] + log_trans            # [i, j]: from i to j
        ptr[t] = np.argmax(trans_out, axis=0)
        best = trans_out[ptr[t], np.arange(n_states)]
        if gaps:
            two = np.partition(trans_out, -2, axis=0)
            top2[t] = two[-1] - two[-2]
        value = log_prob[t] + best
    state = np.zeros(n_steps, dtype=np.int64)
    state[-1] = np.argmax(value)
    for t in range(n_steps - 2, -1, -1):
        state[t] = ptr[t + 1, state[t + 1]]
    if not gaps:
        return state
    srt = np.sort(value)
    g = [srt[-1] - srt[-2]] + [top2[t, state[t]] for t in range(1, n_steps)]
    return state, np.array(g)


def tables(sr, fmin, fmax, frame_length, win_length, hop_length, n_thresholds, beta_parameters, boltzmann_parameter,
           resolution, max_transition_rate, switch_prob):
    """The parameters' derived quantities, as the helper below uses them."""
    thresholds = np.linspace(0, 1, n_thresholds + 1)
    beta_probs = np.diff(scipy.stats.beta.cdf(thresholds, beta_parameters[0], beta_parameters[1]))
    nb = n_pitch_bins(fmin, fmax, resolution)
    w = transition_width(sr, hop_length, max_transition_rate, resolution)
    return thresholds, beta_probs, nb, w


def observations(yin, shifts, sr, fmin, min_period, thresholds, beta_probs, boltzmann_parameter, no_trough_prob, nb,
                 bps):
    """librosa 0.10's __pyin_helper: (observation probabilities (n_frames, 2 nb), voiced_prob (n_frames,))."""
    n_frames, n_lags = yin.shape
    yin_probs = np.zeros_like(yin)
    for i in range(n_frames):
        y = yin[i]
        idx = troughs(y)
        if len(idx) == 0:
            continue
        heights = y[idx]
        below = np.less.outer(heights, thresholds[1:])
        positions = np.cumsum(below, axis=0) - 1
        n_troughs = np.count_nonzero(below, axis=0)
        with np.errstate(divide="ignore", invalid="ignore"):
            prior = scipy.stats.boltzmann.pmf(positions, boltzmann_parameter, n_troughs)
        prior[~below] = 0
        probs = prior.dot(beta_probs)
        gmin = np.argmin(heights)
        n_below_min = np.count_nonzero(~below[gmin, :])
        probs[gmin] += no_trough_prob * np.sum(beta_probs[:n_below_min])
        yin_probs[i, idx] = probs
    frame_index, lag = np.nonzero(yin_probs)                 # frame-major: per frame, lags ascending
    period = min_period + lag
    period = period + shifts[frame_index, lag]
    f0 = sr / period
    bin_index = 12 * bps * np.log2(f0 / fmin)
    bin_index = np.clip(np.round(bin_index), 0, nb).astype(int)
    obs = np.zeros((2 * nb, n_frames))
    obs[bin_index, frame_index] = yin_probs[frame_index, lag]  # per frame, the largest lag wins a shared bin
    voiced_prob = np.clip(np.sum(obs[:nb, :], axis=0), 0, 1)
    obs[nb:, :] = (1 - voiced_prob) / nb
    return obs.T, voiced_prob


def pyin(y, fmin, fmax, sr=22050, frame_length=1024, win_length=None, hop_length=None, n_thresholds=100,
         beta_parameters=(2, 18), boltzmann_parameter=2, resolution=0.1, max_transition_rate=35.92, switch_prob=0.01,
         no_trough_prob=0.01, fill_na=np.nan, gaps=False):
    """(f0, voiced_flag, voiced_prob) of one clip, fp64; with gaps, also the decoded states and the Viterbi margins."""
    win_length = frame_length // 2 if win_length is None else win_length
    hop_length = frame_length // 4 if hop_length is None else hop_length
    frames = frame(y, frame_length, hop_length)
    min_period, max_period = periods(sr, fmin, fmax, frame_length, win_length)
    yin = cmnd(difference(frames, frame_length, win_length, max_period), min_period, max_period)
    shifts = parabolic_shifts(yin)
    thresholds, beta_probs, nb, w = tables(sr, fmin, fmax, frame_length, win_length, hop_length, n_thresholds,
                                           beta_parameters, boltzmann_parameter, resolution, max_transition_rate,
                                           switch_prob)
    bps = n_bins_per_semitone(resolution)
    obs, voiced_prob = observations(yin, shifts, sr, fmin, min_period, thresholds, beta_probs, boltzmann_parameter,
                                    no_trough_prob, nb, bps)
    p_init = np.zeros(2 * nb)
    p_init[nb:] = 1 / nb
    res = viterbi(np.log(obs + TINY), np.log(transition(nb, w, switch_prob) + TINY), np.log(p_init + TINY), gaps)
    states = res[0] if gaps else res
    freqs = fmin * 2 ** (np.arange(nb) / (12 * bps))
    f0 = freqs[states % nb]
    voiced = states < nb
    f0[~voiced] = fill_na
    if gaps:
        return f0, voiced, voiced_prob, states, res[1]
    return f0, voiced, voiced_prob


def average_pitch(values, durations):
    """values (F,), durations (T,) -> (T,) fp64: per span [cum_j, cum_{j+1}) the mean of the values that are neither 0
    nor NaN, summed in frame order; 0 for a span without any."""
    out = np.zeros(len(durations))
    start = 0
    for j, d in enumerate(durations):
        s, n = 0.0, 0
        for v in values[start:start + int(d)]:
            if v != 0 and not math.isnan(v):
                s += float(v)
                n += 1
        out[j] = s / n if n else 0.0
        start += int(d)
    return out
