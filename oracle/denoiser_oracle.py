"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

Plain-torch restatement of the WaveGlow denoiser, next to the forward transform of stft_oracle.py:

    stft.py:44-66            the windowed bases: forward (stft_oracle.stft_forward_basis) and inverse = the
                             pseudo-inverse of (filter_length / hop) * the unwindowed forward basis, transposed, windowed
    stft.py:69-94            transform: reflect-pad by n/2, conv1d at stride hop, magnitude and atan2 phase
    stft.py:96-136           inverse: [mag cos(phase); mag sin(phase)], conv_transpose1d at stride hop, divide by
                             window_sumsquare where it exceeds float32 tiny, multiply by filter_length / hop, trim n/2
                             samples at each end
    audio_processing.py:7-56 window_sumsquare: a float32 envelope, the squared window added one frame at a time
    waveglow/denoiser.py:10-45  bias_spec = magnitude of frame 0 of the bias audio; forward: magnitudes minus
                             strength * bias_spec, clamped at 0, phase kept

Pinning: tests/test_denoiser_cpu.py against tests/golden/denoiser_b2.npz, which the reference's own
waveglow/denoiser.py wrote on the CPU (tools/make_golden.py denoiser).
"""
import functools

import numpy as np
import torch

from oracle.stft_oracle import hann_periodic, stft_forward_basis


@functools.lru_cache(maxsize=None)
def stft_inverse_basis(filter_length=1024, hop_length=256, win_length=1024):
    """(filter_length + 2, filter_length) float32: stft.py:44-66.  Cached: callers must not modify it."""
    n, cutoff = filter_length, filter_length // 2 + 1
    ang = 2.0 * np.pi * np.arange(cutoff)[:, None] * np.arange(n)[None, :] / n
    fourier = np.concatenate([np.cos(ang), -np.sin(ang)], axis=0)
    win = np.zeros(n)
    lpad = (n - win_length) // 2
    win[lpad:lpad + win_length] = hann_periodic(win_length)
    inv = np.linalg.pinv((n / hop_length) * fourier).T.astype(np.float32)
    return (inv * win.astype(np.float32)[None, :]).astype(np.float32)


@functools.lru_cache(maxsize=None)
def window_sumsquare(n_frames, hop_length=256, win_length=1024, n_fft=1024):
    """audio_processing.py:7-56 with norm=None: float32 (n_fft + hop (n_frames - 1),).  Cached: callers must not
    modify it."""
    n = n_fft + hop_length * (n_frames - 1)
    x = np.zeros(n, dtype=np.float32)
    win_sq = np.zeros(n_fft)
    lpad = (n_fft - win_length) // 2
    win_sq[lpad:lpad + win_length] = hann_periodic(win_length) ** 2
    for i in range(n_frames):
        s = i * hop_length
        x[s:min(n, s + n_fft)] += win_sq[:max(0, min(n_fft, n - s))]
    return x


def transform(y, dtype=torch.float64, filter_length=1024, hop_length=256, win_length=1024):
    """stft.py:69-94: y (B, n) -> (magnitude, phase), each (B, n/2 + 1, 1 + n // hop), in dtype."""
    basis = torch.from_numpy(stft_forward_basis(filter_length, win_length)).to(dtype=dtype, device=y.device)[:, None, :]
    x = torch.nn.functional.pad(y.to(dtype)[:, None, None, :], (filter_length // 2, filter_length // 2, 0, 0),
                                mode="reflect")[:, 0]
    ft = torch.nn.functional.conv1d(x, basis, stride=hop_length)
    cutoff = filter_length // 2 + 1
    re, im = ft[:, :cutoff], ft[:, cutoff:]
    return torch.sqrt(re ** 2 + im ** 2), torch.atan2(im, re)


def inverse(mag, phase, filter_length=1024, hop_length=256, win_length=1024):
    """stft.py:96-136 in mag's dtype and on its device: -> (B, 1, hop (frames - 1))."""
    dtype, dev = mag.dtype, mag.device
    basis = torch.from_numpy(stft_inverse_basis(filter_length, hop_length, win_length)).to(dtype=dtype, device=dev)[:, None, :]
    x = torch.cat([mag * torch.cos(phase), mag * torch.sin(phase)], dim=1)
    y = torch.nn.functional.conv_transpose1d(x, basis, stride=hop_length)
    wss = window_sumsquare(mag.shape[-1], hop_length, win_length, filter_length)
    nz = torch.from_numpy(np.where(wss > np.finfo(np.float32).tiny)[0]).to(dev)
    y[:, :, nz] /= torch.from_numpy(wss).to(dtype=dtype, device=dev)[nz]
    y *= float(filter_length) / hop_length
    return y[:, :, filter_length // 2:-(filter_length // 2)]


def bias_spec(bias_audio, dtype=torch.float64):
    """waveglow/denoiser.py:36-38: (1, n/2 + 1, 1)."""
    mag, _ = transform(bias_audio, dtype)
    return mag[:, :, 0][:, :, None]


def denoise(y, bias, strength, dtype=torch.float64, lengths=None):
    """Denoiser.forward (waveglow/denoiser.py:40-45) in dtype, on y's device: y (B, n) -> (B, 1, 256 (n // 256)).  With lengths (B)
    each row is denoised on its own first lengths[b] samples, the rest of its output zero (rows of <= 512 samples give
    zeros)."""
    B, n = y.shape
    if lengths is None:
        mag, phase = transform(y, dtype)
        mag = torch.clamp(mag - bias.to(dtype=dtype, device=y.device) * strength, 0.0)
        return inverse(mag, phase)
    out = torch.zeros(B, 1, 256 * (n // 256), dtype=dtype, device=y.device)
    for b in range(B):
        L = min(max(int(lengths[b]), 0), n)
        if L > 512:
            out[b:b + 1, :, :256 * (L // 256)] = denoise(y[b:b + 1, :L], bias, strength, dtype)
    return out
