"""Pitch targets for non-autoregressive TTS data preparation (FastPitch): ``pyin`` -- librosa 0.10's probabilistic YIN
over a ragged batch of clips on the GPU -- and ``average_by_durations`` -- a per-frame target (f0, energy) averaged
over each symbol's frames, with the durations of ``durations_from_alignments``.  See DESIGN section 6.11.

The host turns librosa's parameters into small fp64 tables (beta probabilities, Boltzmann pmf, the transition band,
the bin frequencies) exactly as ``tests/pyin_oracle.py`` computes them, and the kernels of ``pitch.cu`` only read them."""
import ctypes as C
import numbers

import numpy as np
import torch

from . import _capi
from ._engine import _cached_table, _float_tensor, _integer_tensor, _number, row_lengths

TINY = np.finfo(np.float64).tiny
_PYIN = "tacotron2_b200.pyin"
_AVG = "tacotron2_b200.average_by_durations"


def _transition_local(n, width):
    """librosa.sequence.transition_local(n, width, window="triangle", wrap=False), row-normalised."""
    m = np.arange(1, (width + 1) // 2 + 1)
    if width % 2 == 0:
        w = (2 * m - 1.0) / width
        win = np.r_[w, w[::-1]]
    else:
        w = 2 * m / (width + 1.0)
        win = np.r_[w, w[-2::-1]]
    T = np.zeros((n, n))
    lpad = (n - width) // 2
    for i in range(n):
        row = np.zeros(n)
        row[lpad:lpad + width] = win
        row = np.roll(row, n // 2 + i + 1)
        row[min(n, i + width // 2 + 1):] = 0
        row[:max(0, i - width // 2)] = 0
        T[i] = row
    T /= T.sum(axis=1, keepdims=True)
    return T


def pyin_params(sr, fmin, fmax, frame_length=1024, win_length=None, hop_length=None, n_thresholds=100,
                beta_parameters=(2, 18), boltzmann_parameter=2, resolution=0.1, max_transition_rate=35.92,
                switch_prob=0.01, no_trough_prob=0.01, fill_na=float("nan"), center=True, pad_mode="constant"):
    """librosa's parameters checked and derived: a dict of the C call's scalar fields.  Raises TypeError / ValueError
    naming the argument."""
    if center is not True:
        raise ValueError("%s: center must be True (frames are centred on multiples of hop_length; got %r)"
                         % (_PYIN, center))
    if pad_mode != "constant":
        raise ValueError("%s: pad_mode must be 'constant' (zero padding; got %r)" % (_PYIN, pad_mode))
    sr = _number(sr, "sr", _PYIN, 0, None, True, integer=True)
    frame_length = _number(frame_length, "frame_length", _PYIN, 2, _capi.PYIN_MAX_FRAME, integer=True)
    win_length = frame_length // 2 if win_length is None else _number(win_length, "win_length", _PYIN, 1,
                                                                       frame_length - 1, integer=True)
    hop_length = frame_length // 4 if hop_length is None else _number(hop_length, "hop_length", _PYIN, 1, None,
                                                                       integer=True)
    if hop_length < 1:
        raise ValueError("%s: hop_length must be at least 1 (frame_length %d)" % (_PYIN, frame_length))
    fmin = _number(fmin, "fmin", _PYIN, 0, None, True)
    fmax = _number(fmax, "fmax", _PYIN, 0, None, True)
    if fmin >= fmax:
        raise ValueError("%s: fmin (%r) must be below fmax (%r)" % (_PYIN, fmin, fmax))
    if fmax > sr / 2:
        raise ValueError("%s: fmax (%r) must be at most sr / 2 (%r)" % (_PYIN, fmax, sr / 2))
    min_period = int(np.floor(sr / fmax))
    max_period = min(int(np.ceil(sr / fmin)), frame_length - win_length - 1)
    if max_period <= min_period:
        raise ValueError("%s: max_period = min(ceil(sr / fmin), frame_length - win_length - 1) = %d must exceed "
                         "min_period = floor(sr / fmax) = %d: lower fmin or raise frame_length / fmax"
                         % (_PYIN, max_period, min_period))
    n_thresholds = _number(n_thresholds, "n_thresholds", _PYIN, 1, _capi.PYIN_MAX_THRESHOLDS, integer=True)
    if not isinstance(beta_parameters, (tuple, list)) or len(beta_parameters) != 2:
        raise TypeError("%s: beta_parameters must be a pair (got %r)" % (_PYIN, beta_parameters))
    beta = tuple(_number(p, "beta_parameters", _PYIN, 0, None, True) for p in beta_parameters)
    boltzmann_parameter = _number(boltzmann_parameter, "boltzmann_parameter", _PYIN, 0, None, True)
    resolution = _number(resolution, "resolution", _PYIN, 0, 1, True)
    max_transition_rate = _number(max_transition_rate, "max_transition_rate", _PYIN, 0)
    switch_prob = _number(switch_prob, "switch_prob", _PYIN, 0, 1)
    no_trough_prob = _number(no_trough_prob, "no_trough_prob", _PYIN, 0, 1)
    if isinstance(fill_na, bool) or not isinstance(fill_na, numbers.Real):
        raise TypeError("%s: fill_na must be a real number (got %r)" % (_PYIN, fill_na))
    bps = int(np.ceil(1.0 / resolution))
    n_bins = int(np.floor(12 * bps * np.log2(fmax / fmin))) + 1
    if n_bins > _capi.PYIN_MAX_BINS:
        raise ValueError("%s: %d pitch bins (12 ceil(1 / resolution) log2(fmax / fmin) + 1) exceed %d, the most one "
                         "CTA's shared memory holds: narrow [fmin, fmax] or coarsen resolution"
                         % (_PYIN, n_bins, _capi.PYIN_MAX_BINS))
    width = round(max_transition_rate * 12 * hop_length / sr) * bps + 1
    if width > n_bins:
        raise ValueError("%s: the transition width %d (round(max_transition_rate 12 hop_length / sr) ceil(1 / resolution)"
                         " + 1) exceeds the %d pitch bins: lower max_transition_rate" % (_PYIN, width, n_bins))
    return dict(sr=sr, fmin=fmin, frame_length=frame_length, win_length=win_length, hop_length=hop_length,
                min_period=min_period, max_period=max_period, n_thresholds=n_thresholds, n_bins=n_bins,
                bins_per_semitone=bps, width=width, no_trough_prob=no_trough_prob, fill_na=float(fill_na),
                beta=beta, boltzmann_parameter=boltzmann_parameter, switch_prob=switch_prob)


def pyin_tables(p):
    """The fp64 host tables of t2_pyin for the derived parameters p (include/t2b200.h), as numpy arrays."""
    import scipy.stats
    thresholds = np.linspace(0, 1, p["n_thresholds"] + 1)
    beta_probs = np.diff(scipy.stats.beta.cdf(thresholds, p["beta"][0], p["beta"][1]))
    beta_prefix = np.array([np.sum(beta_probs[:m]) for m in range(p["n_thresholds"] + 1)])
    n_max = (p["max_period"] - p["min_period"] + 2) // 2
    N = np.repeat(np.arange(1, n_max + 1), np.arange(1, n_max + 1))
    pos = np.arange(len(N)) - N * (N - 1) // 2
    boltzmann = scipy.stats.boltzmann.pmf(pos, p["boltzmann_parameter"], N)
    nb, h = p["n_bins"], p["width"] // 2
    loop = 1 - p["switch_prob"]
    stay, switch = loop, (1.0 - loop) / 1
    Tl = _transition_local(nb, p["width"])
    log_tiny = np.log(TINY)
    band = np.full((2, 2 * h + 1, nb), log_tiny)
    j = np.arange(nb)
    for s, scale in enumerate((stay, switch)):
        M = np.log(scale * Tl + TINY)
        for k in range(2 * h + 1):
            i = j - h + k
            ok = (i >= 0) & (i < nb)
            band[s, k, ok] = M[i[ok], j[ok]]
    freqs = p["fmin"] * 2 ** (np.arange(nb) / (12 * p["bins_per_semitone"]))
    p_init = np.log(1 / nb + TINY)
    return dict(thresholds=thresholds[1:].copy(), beta_probs=beta_probs, beta_prefix=beta_prefix, boltzmann=boltzmann,
                log_trans=band, freqs=freqs, log_tiny=float(log_tiny), log_init_unvoiced=float(p_init))


def _device_tables(p, device):
    """pyin_tables(p) on `device`, cached per parameter set and device (built outside any graph capture)."""
    def build():
        return {k: (torch.from_numpy(np.ascontiguousarray(v)).to(device) if isinstance(v, np.ndarray) else v)
                for k, v in pyin_tables(p).items()}
    key = ("pyin", tuple(sorted((k, v) for k, v in p.items() if k != "fill_na")), str(device))
    return _cached_table(key, build)


def pyin_inputs(y, lengths, device_type="cuda"):
    """y and lengths checked and put in the library's form: (y (B, n) fp32 contiguous, lengths (B,) int32 on y's device
    or None, whether y was 1-D).  Reads the device back once for the samples' finiteness (and once for device-side
    lengths).  Raises TypeError / ValueError before anything is launched."""
    _float_tensor(y, "y", _PYIN, "(n,) or (B, n)", (1, 2), device_type)
    one = y.dim() == 1
    x = y.detach().reshape(1, -1) if one else y.detach()
    B, n = (int(s) for s in x.shape)
    if one and lengths is not None:
        raise ValueError("%s: lengths needs y of shape (B, n)" % _PYIN)
    ln, _ = row_lengths(lengths, B, n, "lengths", x.device)
    x = x.to(torch.float32).contiguous()
    if not bool(torch.isfinite(x).all()):                         # the one host read of the samples
        raise ValueError("%s: y must be finite" % _PYIN)
    return x, ln, one


def _pyin_call(x, ln, p, t, device):
    """(ctypes args, outputs, workspace) of one t2_pyin call on checked inputs; the caller keeps all of them alive."""
    B, n = (int(s) for s in x.shape)
    F = 1 + n // p["hop_length"]
    f0 = torch.empty(B, F, dtype=torch.float64, device=device)
    flag = torch.empty(B, F, dtype=torch.bool, device=device)
    prob = torch.empty(B, F, dtype=torch.float64, device=device)
    args = _capi.T2PyinArgs(
        x.data_ptr(), None if ln is None else ln.data_ptr(), B, n, p["sr"], p["frame_length"], p["win_length"],
        p["hop_length"], p["min_period"], p["max_period"], p["n_thresholds"], p["n_bins"], p["bins_per_semitone"],
        p["width"], p["fmin"], p["no_trough_prob"], p["fill_na"], t["log_tiny"], t["log_init_unvoiced"],
        t["thresholds"].data_ptr(), t["beta_probs"].data_ptr(), t["beta_prefix"].data_ptr(), t["boltzmann"].data_ptr(),
        t["log_trans"].data_ptr(), t["freqs"].data_ptr(), f0.data_ptr(), flag.data_ptr(), prob.data_ptr(), None, 0)
    L = _capi.lib()
    ws = _capi.byte_buffer(L.t2_pyin_workspace_bytes(C.byref(args)), device)
    args.ws, args.ws_bytes = ws.data_ptr(), ws.numel()
    return args, (f0, flag, prob), ws


def pyin(y, fmin, fmax, sr=22050, frame_length=1024, win_length=None, hop_length=None, n_thresholds=100,
         beta_parameters=(2, 18), boltzmann_parameter=2, resolution=0.1, max_transition_rate=35.92, switch_prob=0.01,
         no_trough_prob=0.01, fill_na=float("nan"), center=True, pad_mode="constant", lengths=None):
    """librosa 0.10's ``pyin`` (center=True, pad_mode="constant") on the GPU, for a batch of clips at once.

    y: (n,) or (B, n) float tensor on a CUDA device, finite, read as fp32 and computed in fp64.  lengths: None (n for
    every row) or B integers in 1..n (list, host or device tensor): row b is y[b, :lengths[b]] and has
    1 + lengths[b] // hop_length frames; its later frames get f0 0, voiced_flag False and voiced_prob 0, and it equals
    its own B = 1 call.  The other arguments are librosa's, with frame_length defaulting to 1024 (FastPitch's; with
    hop_length = frame_length // 4 = 256 the frames are those of ``TacotronSTFT.mel_spectrogram``); frame_length
    <= 2048 and at most 1536 pitch bins (601 for C2..C7 at resolution 0.1).

    Returns (f0 fp64, voiced_flag bool, voiced_prob fp64), each (B, F) -- (F,) for 1-D y -- with F = 1 + n //
    hop_length, on y's device; f0 is fill_na on unvoiced frames.  See DESIGN section 6.11."""
    p = pyin_params(sr, fmin, fmax, frame_length, win_length, hop_length, n_thresholds, beta_parameters,
                    boltzmann_parameter, resolution, max_transition_rate, switch_prob, no_trough_prob, fill_na, center,
                    pad_mode)
    x, ln, one = pyin_inputs(y, lengths)
    t = _device_tables(p, x.device)
    args, out, ws = _pyin_call(x, ln, p, t, x.device)
    _capi.call(_capi.lib().t2_pyin, x.device, C.byref(args))
    return tuple(o[0] for o in out) if one else out


def average_inputs(values, durations, device_type="cuda"):
    """values and durations checked and put in the library's form: (values (B, F) fp64 contiguous, durations (B, T)
    int64 contiguous).  Reads the device back once.  Raises TypeError / ValueError before anything is launched."""
    _float_tensor(values, "values", _AVG, "(B, F)", (2,), device_type)
    d = _integer_tensor(durations, "durations", _AVG)
    B, F = (int(s) for s in values.shape)
    if d.dim() != 2 or d.shape[0] != B or d.shape[1] < 1:
        raise ValueError("%s: durations must have shape (%d, T_text >= 1) (got %s)" % (_AVG, B, tuple(d.shape)))
    if d.device != values.device:
        raise ValueError("%s: durations must be on values' device %s (got %s)" % (_AVG, values.device, d.device))
    d = d.to(torch.int64).contiguous()
    lo, hi = torch.stack((d.min(), d.sum(1).max())).tolist()     # the one host read
    if lo < 0:
        raise ValueError("%s: durations must be >= 0 (got %d)" % (_AVG, lo))
    if hi > F:
        rows = [b for b, s in enumerate(d.sum(1).tolist()) if s > F]
        raise ValueError("%s: the durations of rows %s sum to more than the %d frames of values" % (_AVG, rows, F))
    return values.detach().to(torch.float64).contiguous(), d


def average_by_durations(values, durations):
    """Per-symbol averages of a per-frame target: FastPitch's ``average_pitch`` (after its NaN -> 0).

    values: (B, F) float tensor on a CUDA device (f0 from ``pyin``, energy, ...), read as fp64.  durations: (B, T_text)
    integers >= 0 on the same device (``durations_from_alignments``' output), each row summing to at most F.

    Returns (B, T_text) fp32: for symbol j of row b the mean of the values[b, f] that are neither 0 nor NaN over its
    frames [sum(durations[b, :j]), sum(durations[b, :j + 1])), summed in fp64 in frame order; 0 where there is none."""
    v, d = average_inputs(values, durations)
    B, F = (int(s) for s in v.shape)
    T = int(d.shape[1])
    out = torch.empty(B, T, dtype=torch.float32, device=v.device)
    _capi.call(_capi.lib().t2_average_by_durations, v.device, v.data_ptr(), d.data_ptr(), B, F, T, out.data_ptr())
    return out
