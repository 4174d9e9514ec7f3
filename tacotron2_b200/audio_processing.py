"""audio_processing.py of the reference: Griffin-Lim on the sm_90a engine, and the small helpers around it.

``griffin_lim(magnitudes, stft_fn, n_iters)`` draws its initial angles on the host exactly as the reference does (so
``np.random.seed(s)`` gives the reference's starting phase), uploads them and runs the whole loop as one library call
(``t2_griffin_lim``) on the bases ``stft_fn`` holds.  ``window_sumsquare`` and the dynamic-range helpers are plain
numpy / torch restatements; they are not on the hot path.
"""
import ctypes

import numpy as np
import torch

from . import _capi


def window_sumsquare(window, n_frames, hop_length=200, win_length=800, n_fft=800, dtype=np.float32, norm=None):
    """The sum-square envelope of a window at a hop (audio_processing.py:7-56, from librosa 0.6):
    (n_fft + hop_length (n_frames - 1),), the squared window added one frame at a time.  window: 'hann' (periodic) or
    an array of win_length values; norm None only (the reference's callers pass none)."""
    if norm is not None:
        raise ValueError("window_sumsquare: only norm=None is supported")
    if win_length is None:
        win_length = n_fft
    n = n_fft + hop_length * (n_frames - 1)
    x = np.zeros(n, dtype=dtype)
    if isinstance(window, str):
        if window not in ("hann", "hanning"):
            raise ValueError("window_sumsquare: only the Hann window is supported by name, got %r" % (window,))
        win = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(win_length) / win_length)
    else:
        win = np.asarray(window, dtype=np.float64)
        if win.shape != (win_length,):
            raise ValueError("window_sumsquare: the window must hold win_length = %d values" % win_length)
    win_sq = np.zeros(n_fft)
    lpad = (n_fft - win_length) // 2
    win_sq[lpad:lpad + win_length] = win ** 2
    for i in range(n_frames):
        sample = i * hop_length
        x[sample:min(n, sample + n_fft)] += win_sq[:max(0, min(n_fft, n - sample))]
    return x


def griffin_lim(magnitudes, stft_fn, n_iters=30, lengths=None):
    """audio_processing.py:59-75: magnitudes (B, 513, F) on the GPU, F >= 4 -> audio (B, 256 (F - 1)) fp32.

    stft_fn: a tacotron2_b200 STFT on the same device (``TacotronSTFT().cuda().stft_fn``).  The initial angles are
    ``np.angle(np.exp(2j pi np.random.rand(B, 513, F)))`` as float32, drawn on the host as in the reference.
    lengths (B) in frames, optional (``model.mel_lengths``): row b equals, bit for bit, the call on its first
    lengths[b] frames alone with the same angles, and its samples from 256 (lengths[b] - 1) on are zero; a value
    outside [0, F] counts as F, and a row of fewer than 4 frames gives zeros.  Magnitudes of any scale are supported."""
    stft_fn._check_spectrum("griffin_lim", magnitudes, lengths, n_iters)
    angles = np.angle(np.exp(2j * np.pi * np.random.rand(*magnitudes.size())))
    angles = torch.from_numpy(angles.astype(np.float32)).to(magnitudes.device)
    return _griffin_lim(magnitudes, angles, stft_fn, n_iters, lengths)


def _griffin_lim(magnitudes, angles, stft_fn, n_iters, lengths=None):
    """griffin_lim from the given initial angles (B, 513, F) on the GPU: one t2_griffin_lim call."""
    a, out, eng, _held = stft_fn._spectrum_args("griffin_lim", magnitudes, angles, lengths, n_iters)
    eng._call(_capi.lib().t2_griffin_lim, ctypes.byref(a))
    return out


def dynamic_range_compression(x, C=1, clip_val=1e-5):
    """audio_processing.py:78-84: log(clamp(x, clip_val) C)."""
    return torch.log(torch.clamp(x, min=clip_val) * C)


def dynamic_range_decompression(x, C=1):
    """audio_processing.py:87-93: exp(x) / C."""
    return torch.exp(x) / C
