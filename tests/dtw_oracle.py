"""numpy fp64 restatement of tacotron2_b200.dtw, mel_cepstral_distortion and pitch_errors (DESIGN section 6.12): the
contract the GPU tests compare against bit for bit.

- distance: C[i, j] = sqrt(s) with s = 0, then s = s + (x_d - y_d) * (x_d - y_d) for d = 0 .. D - 1, every operation
  rounded on its own;
- DP: D[0, 0] = C[0, 0], D[0, j] = C + D[0, j - 1], D[i, 0] = C + D[i - 1, 0], otherwise best = D[i - 1, j - 1], then
  `left < best` takes D[i, j - 1], then `up < best` takes D[i - 1, j] (ties: diagonal, then left, then up);
- cepstra: c_k = sum_m table[k - 1, m] mel[m] in the order m = 0 .. n_mel - 1, table the orthonormal DCT-II rows;
- MCD = (10 sqrt(2) / ln 10) cost / path length."""
import math

import numpy as np

MCD_SCALE = 10.0 * math.sqrt(2.0) / math.log(10.0)
DIAG, LEFT, UP = 0, 1, 2


def distances(x, y):
    """x (D, L_x), y (D, L_y) -> C (L_x, L_y) fp64, summed sequentially over d (in blocks of rows of x)."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    D, Lx = x.shape
    C = np.empty((Lx, y.shape[1]))
    for r in range(0, Lx, 512):
        s = np.zeros((min(512, Lx - r), y.shape[1]))
        for d in range(D):
            diff = x[d, r:r + 512, None] - y[d, None, :]
            s = s + diff * diff
        C[r:r + 512] = np.sqrt(s)
    return C


def dtw_matrix(C):
    """(cost, path (N, 2) int64, predecessor codes (L_x, L_y) int8) of the DP over C, swept by anti-diagonals."""
    Lx, Ly = C.shape
    inf = np.inf
    prev1, prev2 = np.full(Lx, inf), np.full(Lx, inf)          # D on diagonals k - 1 and k - 2, indexed by i
    code = np.zeros((Lx, Ly), np.int8)
    for k in range(Lx + Ly - 1):
        lo, hi = max(0, k - Ly + 1), min(k, Lx - 1)
        i = np.arange(lo, hi + 1)
        j = k - i
        dist = C[i, j]
        left = prev1[i]                                         # D[i, j - 1]
        up = prev1[np.maximum(i - 1, 0)]                       # D[i - 1, j]
        diag = prev2[np.maximum(i - 1, 0)]                     # D[i - 1, j - 1]
        best, c = diag.copy(), np.zeros(len(i), np.int8)
        m = left < best
        best[m], c[m] = left[m], LEFT
        m = up < best
        best[m], c[m] = up[m], UP
        e = i == 0
        best[e], c[e] = left[e], LEFT
        e = j == 0
        best[e], c[e] = up[e], UP
        v = dist + best
        v[(i == 0) & (j == 0)] = dist[(i == 0) & (j == 0)]
        code[i, j] = c
        cur = np.full(Lx, inf)
        cur[i] = v
        prev2, prev1 = prev1, cur
    cost = float(prev1[Lx - 1])
    i, j, path = Lx - 1, Ly - 1, []
    while True:
        path.append((i, j))
        if i == 0 and j == 0:
            break
        c = code[i, j]
        if c != LEFT:
            i -= 1
        if c != UP:
            j -= 1
    return cost, np.array(path[::-1], np.int64), code


def dtw(x, y):
    """x (D, L_x), y (D, L_y) -> (cost, path (N, 2) int64)."""
    cost, path, _ = dtw_matrix(distances(x, y))
    return cost, path


def dct_table(n_mel, n_cep):
    m = np.arange(n_mel)
    k = np.arange(1, n_cep + 1)[:, None]
    return np.sqrt(2.0 / n_mel) * np.cos(np.pi * k * (2 * m + 1) / (2 * n_mel))


def cepstra(mel, n_cep):
    """mel (n_mel, L) -> (n_cep, L) fp64, summed sequentially over the bands."""
    mel = np.asarray(mel, np.float64)
    tab = dct_table(mel.shape[0], n_cep)
    s = np.zeros((n_cep, mel.shape[1]))
    for m in range(mel.shape[0]):
        s = s + tab[:, m, None] * mel[m, None, :]
    return s


def mcd(mel_x, mel_y, n_cep=24):
    """(mcd, path) of one pair of natural-log mels (n_mel, L_x), (n_mel, L_y)."""
    cost, path = dtw(cepstra(mel_x, n_cep), cepstra(mel_y, n_cep))
    return MCD_SCALE * cost / float(len(path)), path


def pitch_errors(f0_x, voiced_x, f0_y, voiced_y, path):
    """The four f0 measures of one pair along path (N, 2), as floats (NaN for an empty denominator)."""
    i, j = path[:, 0], path[:, 1]
    fx, fy = np.asarray(f0_x, np.float64)[i], np.asarray(f0_y, np.float64)[j]
    vx, vy = np.asarray(voiced_x, bool)[i], np.asarray(voiced_y, bool)[j]
    both = vx & vy
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = fx / fy
        gross = both & (np.abs(ratio - 1.0) > 0.2)
        n, nb, ng, nd = float(len(path)), float(both.sum()), float(gross.sum()), float((vx != vy).sum())
        cents = 1200.0 * np.log2(ratio[both])
        return {"gpe": ng / nb if nb else math.nan, "vde": nd / n, "ffe": (ng + nd) / n,
                "f0_rmse_cents": math.sqrt(float(np.sum(cents * cents)) / nb) if nb else math.nan}
