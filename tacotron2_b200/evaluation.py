"""Objective evaluation of synthesized speech against recordings on the GPU: ``dtw`` -- dynamic time warping of two
batches of frame sequences of different lengths --, ``mel_cepstral_distortion`` (MCD-DTW) on natural-log mels, and
``pitch_errors`` (GPE, VDE, FFE and the f0 RMSE in cents) of two ``pyin`` outputs along a warping path.  See DESIGN
section 6.12.  The contract is the numpy fp64 oracle ``tests/dtw_oracle.py``."""
import ctypes as C
import math

import numpy as np
import torch

from . import _capi
from ._engine import _cached_table, _float_tensor, _integer_tensor, _number, row_lengths

_DTW = "tacotron2_b200.dtw"
_MCD = "tacotron2_b200.mel_cepstral_distortion"
_PITCH = "tacotron2_b200.pitch_errors"
MCD_SCALE = 10.0 * math.sqrt(2.0) / math.log(10.0)     # dB per unit of Euclidean cepstral distance
_DTYPES = {torch.float32: _capi.DTW_F32, torch.float64: _capi.DTW_F64}


def dtw_inputs(x, y, x_lengths=None, y_lengths=None, what=_DTW, device_type="cuda"):
    """The arguments of dtw checked and put in the library's form: (x, y contiguous, x_lengths and y_lengths as (B,)
    int32 on their device or None, the dtype code).  Reads a device-side lengths tensor back once.  Raises TypeError /
    ValueError before anything is launched."""
    _float_tensor(x, "x", what, "(B, D, T)", (3,), device_type, _DTYPES)
    _float_tensor(y, "y", what, "(B, D, T)", (3,), device_type, _DTYPES)
    if x.dtype != y.dtype:
        raise TypeError("%s: x and y must have the same dtype (got %s and %s)" % (what, x.dtype, y.dtype))
    if x.device != y.device:
        raise ValueError("%s: x and y must be on the same device (got %s and %s)" % (what, x.device, y.device))
    (B, D, T_x), (B_y, D_y, T_y) = (tuple(int(s) for s in t.shape) for t in (x, y))
    if B_y != B or D_y != D:
        raise ValueError("%s: x (B, D, T_x) and y (B, D, T_y) must agree in B and D (got %s and %s)"
                         % (what, tuple(x.shape), tuple(y.shape)))
    if D > _capi.DTW_MAX_DIM:
        raise ValueError("%s: D must be at most %d (got %d)" % (what, _capi.DTW_MAX_DIM, D))
    if max(T_x, T_y) > _capi.DTW_MAX_FRAMES:
        raise ValueError("%s: T_x and T_y must be at most %d (got %d and %d)" % (what, _capi.DTW_MAX_FRAMES, T_x, T_y))
    xl, _ = row_lengths(x_lengths, B, T_x, "x_lengths", x.device)
    yl, _ = row_lengths(y_lengths, B, T_y, "y_lengths", x.device)
    return x.detach().contiguous(), y.detach().contiguous(), xl, yl, _DTYPES[x.dtype]


def _dtw_call(x, y, xl, yl, code):
    B, D, T_x = (int(s) for s in x.shape)
    T_y = int(y.shape[2])
    dev = x.device
    cost = torch.empty(B, dtype=torch.float64, device=dev)
    path = torch.empty(B, T_x + T_y - 1, 2, dtype=torch.int64, device=dev)
    path_lengths = torch.empty(B, dtype=torch.int64, device=dev)
    L = _capi.lib()
    ws = _capi.byte_buffer(L.t2_dtw_workspace_bytes(B, D, T_x, T_y, code), dev)
    args = _capi.T2DtwArgs(x.data_ptr(), y.data_ptr(), None if xl is None else xl.data_ptr(),
                           None if yl is None else yl.data_ptr(), B, D, T_x, T_y, code, cost.data_ptr(),
                           path.data_ptr(), path_lengths.data_ptr(), ws.data_ptr(), ws.numel())
    _capi.call(L.t2_dtw, dev, C.byref(args))
    return cost, path, path_lengths


def dtw(x, y, x_lengths=None, y_lengths=None):
    """Dynamic time warping of two batches of frame sequences.

    x: (B, D, T_x) and y: (B, D, T_y) tensors of one dtype, float32 or float64, on one CUDA device -- the (B, n_mel, T)
    layout of ``Tacotron2.inference`` and ``TacotronSTFT.mel_spectrogram``, so mels go in as they are; D <= 1024,
    T_x, T_y <= 8192.  x_lengths / y_lengths: None (T_x / T_y for every row) or B integers in 1..T_x / 1..T_y, as a
    list, a host or a device tensor.  Row b reads only x[b, :, :x_lengths[b]] and y[b, :, :y_lengths[b]].

    The frame distance is the Euclidean C[i, j] = sqrt(sum_d (x_d - y_d)^2), in fp64 with the sum taken in the order
    d = 0 .. D - 1; the path from (0, 0) to (L_x - 1, L_y - 1) takes steps (1, 1), (0, 1), (1, 0) with unit weights
    and minimises the summed distance, ties going to the diagonal, then to (i, j - 1), then to (i - 1, j).

    Returns (cost (B,) fp64, the summed distance along the path; path (B, T_x + T_y - 1, 2) int64, the (i, j) pairs
    from (0, 0) on, padded with -1; path_lengths (B,) int64), on x's device.  Each row equals its own B = 1 call."""
    return _dtw_call(*dtw_inputs(x, y, x_lengths, y_lengths))


def dct_table(n_mel, n_cep):
    """Rows 1 .. n_cep of the orthonormal DCT-II over n_mel bands, (n_cep, n_mel) fp64: c_k = sum_m table[k - 1, m]
    mel[m] is scipy.fft.dct(mel, type=2, norm="ortho")[k]."""
    m = np.arange(n_mel)
    k = np.arange(1, n_cep + 1)[:, None]
    return np.sqrt(2.0 / n_mel) * np.cos(np.pi * k * (2 * m + 1) / (2 * n_mel))


def _device_table(n_mel, n_cep, device):
    key = ("dct", n_mel, n_cep, str(device))
    return _cached_table(key, lambda: torch.from_numpy(dct_table(n_mel, n_cep)).to(device))


def mcd_inputs(mel_x, mel_y, x_lengths=None, y_lengths=None, n_cep=24, device_type="cuda"):
    """The arguments of mel_cepstral_distortion checked: dtw_inputs' tuple and n_cep.  Raises TypeError / ValueError
    before anything is launched."""
    n_cep = _number(n_cep, "n_cep", _MCD, integer=True)
    args = dtw_inputs(mel_x, mel_y, x_lengths, y_lengths, _MCD, device_type)
    B, n_mel = (int(s) for s in args[0].shape[:2])
    if B > 65535:
        raise ValueError("%s: B must be at most 65535 (got %d)" % (_MCD, B))
    if not 1 <= n_cep <= n_mel - 1:
        raise ValueError("%s: n_cep must lie in 1..n_mel - 1 = %d (got %d)" % (_MCD, n_mel - 1, n_cep))
    return args, n_cep


def mel_cepstral_distortion(mel_x, mel_y, x_lengths=None, y_lengths=None, n_cep=24):
    """Mel-cepstral distortion after dynamic time warping (MCD-DTW), in dB.

    mel_x: (B, n_mel, T_x) and mel_y: (B, n_mel, T_y) natural-log mels (what ``Tacotron2.inference`` and
    ``TacotronSTFT.mel_spectrogram`` return), float32 or float64, on one CUDA device, B <= 65535; lengths as for
    ``dtw``.  Each frame's cepstrum is the orthonormal DCT-II over the bands, computed on the device in fp64 with a
    fixed summation order; c_1 .. c_n_cep are kept (c_0, the level, is dropped), 1 <= n_cep < n_mel.

    Returns (mcd (B,) fp64, path, path_lengths): ``dtw`` on the cepstra, and mcd_b = (10 sqrt(2) / ln 10)
    cost_b / path_lengths_b, the distortion averaged over the warping path.  The path aligns anything else on the
    frame grid, e.g. ``pyin`` outputs for ``pitch_errors``."""
    (x, y, xl, yl, code), n_cep = mcd_inputs(mel_x, mel_y, x_lengths, y_lengths, n_cep)
    B, n_mel, T_x = (int(s) for s in x.shape)
    T_y = int(y.shape[2])
    dev = x.device
    table = _device_table(n_mel, n_cep, dev)
    L = _capi.lib()
    ceps = []
    for t, ln, T in ((x, xl, T_x), (y, yl, T_y)):
        cep = torch.empty(B, n_cep, T, dtype=torch.float64, device=dev)
        _capi.call(L.t2_mel_cepstra, dev, t.data_ptr(), code, None if ln is None else ln.data_ptr(), B, n_mel, T,
                   table.data_ptr(), n_cep, cep.data_ptr())
        ceps.append(cep)
    cost, path, path_lengths = _dtw_call(ceps[0], ceps[1], xl, yl, _capi.DTW_F64)
    return MCD_SCALE * cost / path_lengths.to(torch.float64), path, path_lengths


def _pitch_track(f0, voiced, name, device_type):
    if not torch.is_tensor(f0):
        raise TypeError("%s: f0_%s must be a float tensor (got %s)" % (_PITCH, name, type(f0).__name__))
    _float_tensor(f0, "f0_" + name, _PITCH, "(B, F)", (2,), device_type)
    if not torch.is_tensor(voiced) or voiced.dtype != torch.bool:
        raise TypeError("%s: voiced_%s must be a bool tensor (got %s)"
                        % (_PITCH, name, voiced.dtype if torch.is_tensor(voiced) else type(voiced).__name__))
    if voiced.shape != f0.shape or voiced.device != f0.device:
        raise ValueError("%s: voiced_%s must have f0_%s's shape %s and device %s (got %s on %s)"
                         % (_PITCH, name, name, tuple(f0.shape), f0.device, tuple(voiced.shape), voiced.device))


def pitch_inputs(f0_x, voiced_x, f0_y, voiced_y, path, path_lengths, device_type="cuda"):
    """The arguments of pitch_errors checked: (path (B, P, 2) int64, path_lengths (B,) int64), both on f0_x's device.
    Reads the device back once for the lengths' and indices' ranges.  Raises TypeError / ValueError before anything
    reads the tracks."""
    _pitch_track(f0_x, voiced_x, "x", device_type)
    _pitch_track(f0_y, voiced_y, "y", device_type)
    dev = f0_x.device
    B, F_x = (int(s) for s in f0_x.shape)
    F_y = int(f0_y.shape[1])
    if f0_y.device != dev or int(f0_y.shape[0]) != B:
        raise ValueError("%s: f0_y must have f0_x's B = %d and device %s (got %s on %s)"
                         % (_PITCH, B, dev, tuple(f0_y.shape), f0_y.device))
    p = _integer_tensor(path, "path", _PITCH)
    if p.dim() != 3 or p.shape[0] != B or p.shape[1] < 1 or p.shape[2] != 2:
        raise ValueError("%s: path must have shape (%d, P >= 1, 2) (got %s)" % (_PITCH, B, tuple(p.shape)))
    n = _integer_tensor(path_lengths, "path_lengths", _PITCH)
    if tuple(n.shape) != (B,):
        raise ValueError("%s: path_lengths must have shape (%d,) (got %s)" % (_PITCH, B, tuple(n.shape)))
    p = p.to(device=dev, dtype=torch.int64)
    n = n.to(device=dev, dtype=torch.int64)
    P = int(p.shape[1])
    valid = torch.arange(P, device=dev)[None, :] < n[:, None]
    i, j = (torch.where(valid, p[..., c], 0) for c in (0, 1))
    lo_n, hi_n, lo, hi_i, hi_j = torch.stack((n.min(), n.max(), torch.minimum(i.min(), j.min()), i.max(),
                                              j.max())).tolist()           # the one host read
    if lo_n < 1 or hi_n > P:
        raise ValueError("%s: path_lengths must lie in 1..%d (got %d..%d)" % (_PITCH, P, lo_n, hi_n))
    if lo < 0 or hi_i >= F_x or hi_j >= F_y:
        raise ValueError("%s: the path's frames must lie in [0, %d) x [0, %d) (got i up to %d, j up to %d, min %d)"
                         % (_PITCH, F_x, F_y, hi_i, hi_j, lo))
    return p, n


def pitch_errors(f0_x, voiced_x, f0_y, voiced_y, path, path_lengths):
    """F0 frame errors of x against y along a warping path (``dtw`` / ``mel_cepstral_distortion``).

    f0_x, voiced_x: (B, F_x) float and bool tensors on a CUDA device (``pyin``'s f0 and voiced_flag on the mel frame
    grid, ``frame_length=1024``); f0_y, voiced_y: (B, F_y) likewise.  path (B, P, 2) and path_lengths (B,): integers,
    the first path_lengths[b] pairs (i, j) of row b in [0, F_x) x [0, F_y).

    Returns a dict of (B,) fp64 tensors over the N = path_lengths[b] pairs, "both voiced" meaning voiced in x and in y:
    ``gpe`` (gross pitch error) = #(both voiced and |f0_x / f0_y - 1| > 0.2) / #(both voiced); ``vde`` (voicing
    decision error) = #(voicing differs) / N; ``ffe`` (f0 frame error) = (#gross errors + #voicing differences) / N;
    ``f0_rmse_cents`` = sqrt(mean over both voiced of (1200 log2(f0_x / f0_y))^2).  A ratio with an empty denominator
    is NaN."""
    p, n = pitch_inputs(f0_x, voiced_x, f0_y, voiced_y, path, path_lengths)
    return frame_errors(f0_x, voiced_x, f0_y, voiced_y, p, n)


def frame_errors(f0_x, voiced_x, f0_y, voiced_y, path, path_lengths):
    """pitch_errors' measures on checked arguments (path (B, P, 2) and path_lengths (B,) int64 on the tracks' device,
    every index in range), on any device."""
    dev = f0_x.device
    valid = torch.arange(path.shape[1], device=dev)[None, :] < path_lengths[:, None]
    i, j = (torch.where(valid, path[..., c], 0) for c in (0, 1))
    fx = torch.gather(f0_x.detach().to(torch.float64), 1, i)
    fy = torch.gather(f0_y.detach().to(torch.float64), 1, j)
    vx = torch.gather(voiced_x, 1, i) & valid
    vy = torch.gather(voiced_y, 1, j) & valid
    both = vx & vy
    ratio = fx / fy
    gross = both & ((ratio - 1.0).abs() > 0.2)
    n_both, n_gross = both.sum(1).to(torch.float64), gross.sum(1).to(torch.float64)
    n_diff, N = (vx != vy).sum(1).to(torch.float64), path_lengths.to(torch.float64)
    cents = torch.where(both, 1200.0 * torch.log2(ratio), 0.0)
    return {"gpe": n_gross / n_both, "vde": n_diff / N, "ffe": (n_gross + n_diff) / N,
            "f0_rmse_cents": torch.sqrt((cents * cents).sum(1) / n_both)}
