"""numpy fp64 oracles of durations_from_alignments (DESIGN section 6.10), one row at a time, and the score of a path."""
import numpy as np

FLT_MIN = 2.0 ** -126


def cells(a):
    """The MAS cell scores c[t, j] = log(max(a, FLT_MIN)) of a (L_mel, L_text) map, in fp64."""
    return np.log(np.maximum(np.asarray(a, dtype=np.float64), FLT_MIN))


def mas(a):
    """Monotonic alignment search on one row's own (L_mel, L_text) map: its durations (L_text,) int64."""
    c = cells(a)
    T, N = c.shape
    if T < N:
        raise ValueError("no monotonic path: %d frames < %d symbols" % (T, N))
    S = np.full((T, N), -np.inf)
    S[0, 0] = c[0, 0]
    for t in range(1, T):
        left = np.concatenate(([-np.inf], S[t - 1, :-1]))
        S[t] = c[t] + np.maximum(S[t - 1], left)
    d = np.zeros(N, dtype=np.int64)
    j = N - 1
    for t in range(T - 1, -1, -1):
        d[j] += 1
        if t > 0 and j > 0 and (j == t or S[t - 1, j - 1] > S[t - 1, j]):
            j -= 1
    return d


def argmax(a):
    """FastPitch's rule on one row's own (L_mel, L_text) map: frames per first-index argmax symbol."""
    a = np.asarray(a)
    return np.bincount(a.argmax(1), minlength=a.shape[1]).astype(np.int64)


def path_score(a, d):
    """The fp64 score of the monotonic path with durations d (every d >= 1) through the map a, summed in frame order
    (the order the recurrence adds in)."""
    c = cells(a)
    sym = np.repeat(np.arange(len(d)), d)
    s = 0.0
    for t, j in enumerate(sym):
        s += c[t, j]
    return s
