"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

Plain-torch restatement of the reference's Griffin-Lim (audio_processing.py:59-75) over the STFT transform and inverse
of oracle/denoiser_oracle.py (stft.py:69-136), in any dtype: the inverse from the initial angles, then n_iters times the
inverse of the target magnitudes on the phase of the transform of the signal.

Pinning: tests/test_griffin_lim_cpu.py against tests/golden/griffin_lim_b2.npz, which the reference's own
audio_processing.griffin_lim wrote on the CPU (tools/make_golden.py griffin_lim).
"""
import torch

from oracle.denoiser_oracle import inverse, transform


def griffin_lim(mag, angles, n_iters, dtype=torch.float64, lengths=None):
    """audio_processing.py:59-75 in dtype, on mag's device, from the given initial angles: mag, angles (B, n/2 + 1, F)
    -> (B, hop (F - 1)).  With lengths (B) in frames each row runs on its own first lengths[b] frames (a value outside
    [0, F] counts as F), the rest of its output zero; rows of fewer than 4 frames give zeros."""
    B, _, F = mag.shape
    if lengths is None:
        mag = mag.to(dtype)
        signal = inverse(mag, angles.to(dtype)).squeeze(1)
        for _ in range(n_iters):
            _, phase = transform(signal, dtype)
            signal = inverse(mag, phase).squeeze(1)
        return signal
    out = torch.zeros(B, 256 * (F - 1), dtype=dtype, device=mag.device)
    for b in range(B):
        L = int(lengths[b])
        L = L if 0 <= L <= F else F
        if L >= 4:
            out[b, :256 * (L - 1)] = griffin_lim(mag[b:b + 1, :, :L], angles[b:b + 1, :, :L], n_iters, dtype)[0]
    return out


def spectral_convergence(mag, signal, dtype=torch.float64):
    """|| S - |STFT(signal)| || / || S ||, per row (B,): how far a Griffin-Lim signal is from the target magnitudes."""
    got, _ = transform(signal, dtype)
    S = mag.to(dtype)
    return (S - got).flatten(1).norm(dim=1) / S.flatten(1).norm(dim=1)
