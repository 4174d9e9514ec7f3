"""The reference's STFT module (stft.py) on the sm_90a engine.

``STFT(filter_length, hop_length, win_length)`` has the reference's constructor, buffers and ``state_dict`` keys, and
its ``transform`` / ``inverse`` / ``forward``.  The transforms run in libt2b200 (denoiser.cu) on the same two GEMMs the
Denoiser uses, with the bases packed once per module in a ``T2Denoiser`` handle that the module owns: there is no CPU
path and no fallback.  Only the reference configuration (filter_length 1024, hop 256, win_length 1024, periodic Hann)
has kernels; other configurations construct and hold their bases, and their transforms raise.  CUDA tensors only.
"""
import ctypes as C
import functools

import numpy as np
import torch

from . import _capi
from . import _engine

HOP = 256
SUPPORTED = (1024, 256, 1024)      # (filter_length, hop_length, win_length) the kernels are built for
MIN_FRAMES = 4                     # 256 (F - 1) > 512 samples: what the reflect padding of the next transform needs


def _windowed_fourier_basis(filter_length, win_length):
    """Rows 0 .. n/2 = real part, rows n/2+1 .. n+1 = imaginary part of the first n/2 + 1 DFT bins (exp(-2 pi i k t / n)),
    each multiplied by the periodic hann window zero-padded symmetrically to filter_length (stft.py:44-63)."""
    n, cutoff = int(filter_length), int(filter_length) // 2 + 1
    if win_length > n:
        raise ValueError("win_length must not exceed filter_length (stft.py:56)")
    phase = (2.0 * np.pi / n) * np.outer(np.arange(cutoff), np.arange(n))
    window = np.zeros(n)
    left = (n - win_length) // 2
    window[left:left + win_length] = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(win_length) / win_length)
    basis = np.vstack((np.cos(phase), -np.sin(phase))).astype(np.float32)
    return torch.from_numpy(basis * window.astype(np.float32))


@functools.lru_cache(maxsize=None)
def _bases(filter_length, hop_length, win_length):
    """(forward, inverse) windowed bases, fp32 (filter_length + 2, 1, filter_length) (stft.py:44-66): the forward basis
    is the real, then the imaginary rows of the first n/2 + 1 DFT bins; the inverse basis is the pseudo-inverse of the
    unwindowed forward basis scaled by filter_length / hop_length, transposed.  Both are multiplied by the periodic Hann
    window.  The pseudo-inverse is computed once per configuration."""
    n, cutoff = filter_length, filter_length // 2 + 1
    phase = (2.0 * np.pi / n) * np.outer(np.arange(cutoff), np.arange(n))
    fourier = np.vstack((np.cos(phase), -np.sin(phase)))
    window = np.zeros(n)
    left = (n - win_length) // 2
    window[left:left + win_length] = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(win_length) / win_length)
    inverse = torch.from_numpy(np.linalg.pinv((n / hop_length) * fourier).T.astype(np.float32))
    inverse = inverse * torch.from_numpy(window.astype(np.float32))
    forward = _windowed_fourier_basis(filter_length, win_length)
    return forward[:, None, :].contiguous(), inverse[:, None, :].contiguous()


def _lengths(lengths, B, device, what):
    """Per-row lengths as int32 on the device, shape-checked (None stays None)."""
    if lengths is None:
        return None
    t = torch.as_tensor(lengths)
    if tuple(t.shape) != (B,):
        raise ValueError("%s: lengths must have shape (%d,), got %s" % (what, B, tuple(t.shape)))
    return None if device is None else _engine._i32(t, device)


class STFT(torch.nn.Module):
    """stft.py:41-141: the windowed bases as buffers, ``transform``, ``inverse`` and ``forward``."""

    def __init__(self, filter_length=800, hop_length=200, win_length=800, window='hann'):
        super().__init__()
        self.filter_length, self.hop_length, self.win_length, self.window = filter_length, hop_length, win_length, window
        if window != 'hann':
            raise ValueError("tacotron2_b200.STFT: only the Hann window is supported, got %r" % (window,))
        if win_length > filter_length:
            raise ValueError("win_length must not exceed filter_length (stft.py:56)")
        forward, inverse = _bases(int(filter_length), int(hop_length), int(win_length))
        self.register_buffer('forward_basis', forward.clone())
        self.register_buffer('inverse_basis', inverse.clone())
        self._t2 = None

    def __getstate__(self):
        # the engine handle is per-instance runtime state: a pickled module rebuilds it on first use
        state = self.__dict__.copy()
        state["_t2"] = None
        return state

    def _engine(self):
        if self._t2 is None:
            self._t2 = _StftEngine(self)
        return self._t2

    def _check_config(self, what):
        cfg = (int(self.filter_length), int(self.hop_length), int(self.win_length))
        if cfg != SUPPORTED:
            raise ValueError("%s: the sm_90a kernels are built for filter_length 1024, hop_length 256 and win_length "
                             "1024 only (this STFT has %d / %d / %d)" % ((what,) + cfg))

    def _device(self, what, *tensors):
        """The CUDA device of the module's bases, which every tensor argument must share."""
        dev = self.forward_basis.device
        for t in (self.forward_basis,) + tensors:
            if not t.is_cuda:
                raise RuntimeError("%s: CUDA tensors only (move the module and its inputs to the GPU)" % what)
        return dev

    @torch.no_grad()
    def transform(self, input_data, lengths=None):
        """input_data (B, n) -> (magnitude, phase), each (B, 513, n // 256 + 1) fp32 (stft.py:69-94).

        lengths (B) in samples, optional: row b is transformed as ``input_data[b, :lengths[b]]`` alone, bit for bit,
        and its frames from lengths[b] // 256 + 1 on are zero; a value outside [0, n] counts as n, and a row of at most
        512 samples gives zeros.  Without lengths n must exceed 512, as in the reference.  Any scale of input is
        supported (each row is scaled by a power of two on the device and the magnitude scaled back)."""
        what = "STFT.transform"
        self._check_config(what)
        x = _real_2d(input_data, what)
        B, n = int(x.shape[0]), int(x.shape[1])
        _lengths(lengths, B, None, what)
        if lengths is None and n <= 512:
            raise ValueError("%s: %d samples cannot be reflect-padded by 512 (the reference needs n > 512)" % (what, n))
        dev = self._device(what, x)
        len32 = _lengths(lengths, B, dev, what)
        self.num_samples = n
        eng = self._engine()
        eng.ensure(self)
        x = x.to(device=dev, dtype=torch.float32).contiguous()
        F = n // HOP + 1
        mag = torch.empty(B, SUPPORTED[0] // 2 + 1, F, device=dev, dtype=torch.float32)
        phase = torch.empty_like(mag)
        ws = eng._ws.get("transform", _capi.lib().t2_stft_transform_workspace_bytes(eng.handle, B, n), dev)
        a = _capi.T2StftTransformArgs(x.data_ptr(), B, n, _engine._ptr(len32), mag.data_ptr(), phase.data_ptr(),
                                      ws.data_ptr(), ws.numel())
        eng._call(_capi.lib().t2_stft_transform, C.byref(a))
        return mag, phase

    @torch.no_grad()
    def inverse(self, magnitude, phase, lengths=None):
        """magnitude, phase (B, 513, F) -> (B, 1, 256 (F - 1)) fp32 (stft.py:96-136); F >= 4.

        lengths (B) in frames, optional (``model.mel_lengths``): row b is the inverse of its first lengths[b] frames
        alone, bit for bit, and its samples from 256 (lengths[b] - 1) on are zero; a value outside [0, F] counts as F,
        and a row of fewer than 4 frames gives zeros."""
        a, out, eng, _held = self._spectrum_args("STFT.inverse", magnitude, phase, lengths)
        eng._call(_capi.lib().t2_stft_inverse, C.byref(a))
        return out[:, None, :]

    def forward(self, input_data):
        """stft.py:138-141: transform, keep magnitude and phase as attributes, and invert them."""
        self.magnitude, self.phase = self.transform(input_data)
        return self.inverse(self.magnitude, self.phase)

    def _check_spectrum(self, what, magnitude, lengths, n_iters=None):
        """Everything about a (B, 513, F) magnitude, its lengths and n_iters that can be refused before a GPU is touched;
        -> (B, F)."""
        self._check_config(what)
        if not isinstance(magnitude, torch.Tensor) or magnitude.dim() != 3 or magnitude.shape[1] != SUPPORTED[0] // 2 + 1:
            raise ValueError("%s: magnitudes must be a (B, 513, F) tensor, got %s" %
                             (what, tuple(getattr(magnitude, "shape", ()))))
        if magnitude.dtype == torch.bool or magnitude.is_complex():
            raise TypeError("%s: magnitudes must be real-valued, got %s" % (what, magnitude.dtype))
        B, F = int(magnitude.shape[0]), int(magnitude.shape[2])
        if B == 0:
            raise ValueError("%s: empty batch" % what)
        if F < MIN_FRAMES:
            raise ValueError("%s: %d frames give %d samples, which cannot be reflect-padded by 512 (at least %d frames "
                             "are needed)" % (what, F, HOP * (F - 1), MIN_FRAMES))
        _lengths(lengths, B, None, what)
        if n_iters is not None and int(n_iters) < 0:
            raise ValueError("%s: n_iters must be >= 0, got %d" % (what, n_iters))
        self._device(what, magnitude)
        return B, F

    def _spectrum_args(self, what, magnitude, phase, lengths, n_iters=None):
        """T2StftInverseArgs (T2GriffinLimArgs with n_iters) over (B, 513, F) inputs on the device;
        -> (args, out, engine, the tensors the args point to)."""
        B, F = self._check_spectrum(what, magnitude, lengths, n_iters)
        if not isinstance(phase, torch.Tensor) or phase.shape != magnitude.shape:
            raise ValueError("%s: phase must have the magnitudes' shape %s, got %s" %
                             (what, tuple(magnitude.shape), tuple(getattr(phase, "shape", ()))))
        if phase.dtype == torch.bool or phase.is_complex():
            raise TypeError("%s: phase must be real-valued, got %s" % (what, phase.dtype))
        dev = self._device(what, magnitude, phase)
        len32 = _lengths(lengths, B, dev, what)
        eng = self._engine()
        eng.ensure(self)
        m = magnitude.to(device=dev, dtype=torch.float32).contiguous()
        p = phase.to(device=dev, dtype=torch.float32).contiguous()
        out = torch.empty(B, HOP * (F - 1), device=dev, dtype=torch.float32)
        L = _capi.lib()
        if n_iters is None:
            ws = eng._ws.get("inverse", L.t2_stft_inverse_workspace_bytes(eng.handle, B, F), dev)
        else:
            ws = eng._ws.get("griffin_lim", L.t2_griffin_lim_workspace_bytes(eng.handle, B, F), dev)
        a = _capi.T2StftInverseArgs(m.data_ptr(), p.data_ptr(), B, F, _engine._ptr(len32), out.data_ptr(),
                                    ws.data_ptr(), ws.numel())
        if n_iters is not None:
            a = _capi.T2GriffinLimArgs(a, int(n_iters))
        return a, out, eng, (m, p, len32)


def _real_2d(x, what):
    if not isinstance(x, torch.Tensor) or x.dim() != 2:
        raise ValueError("%s: input must be a (B, n) tensor, got %s" % (what, tuple(getattr(x, "shape", ()))))
    if x.dtype == torch.bool or x.is_complex():
        raise TypeError("%s: input must be real-valued, got %s" % (what, x.dtype))
    if x.shape[0] == 0 or x.shape[1] == 0:
        raise ValueError("%s: input is empty, shape %s" % (what, tuple(x.shape)))
    return x


class _StftEngine(_engine._Handle):
    """One T2Denoiser handle (an STFT module's packed bases on one device) + cached workspaces.  The module's
    transforms, Griffin-Lim and the Denoiser holding the module all run on it."""

    kind, what = "denoiser", "tacotron2_b200.STFT"
    stream = _engine._Handle._stream      # the name callers of the window entry points use

    def __init__(self, stft):
        super().__init__()
        self.cfg = (int(stft.filter_length), int(stft.hop_length), int(stft.win_length))

    def ensure(self, module):
        """module: the STFT, or a module holding it as ``stft`` (the Denoiser)."""
        st = getattr(module, "stft", module)
        self._ensure(st.forward_basis.device, (st.forward_basis, st.inverse_basis))

    def _pack(self, bases, dev):
        f, i = (b.detach().to(device=dev, dtype=torch.float32).contiguous() for b in bases)
        return (f, i), (f.data_ptr(), i.data_ptr())

    def _config(self):
        return _capi.T2DenoiserConfig(*self.cfg, 0)

    # -- the Denoiser's entry points ------------------------------------------------------------------------------
    def audio(self, audio, what):
        """audio (B, n) on the device: fp16 stays fp16 (converted as it is packed), any other real dtype becomes fp32."""
        _real_2d(audio, what)
        dt = torch.float16 if audio.dtype == torch.float16 else torch.float32
        return audio.to(device=self.device, dtype=dt).contiguous()

    def bias(self, module, bias_audio):
        """bias_spec (513,) of bias_audio (1, n) fp32: the magnitude of its frame 0 (t2_denoiser_bias)."""
        self.ensure(module)
        x = bias_audio.to(device=self.device, dtype=torch.float32).contiguous()
        out = torch.empty(module.stft.filter_length // 2 + 1, device=self.device, dtype=torch.float32)
        self._call(_capi.lib().t2_denoiser_bias, x.data_ptr(), int(x.shape[-1]), out.data_ptr())
        return out

    def args(self, module, audio, len32, strength, out):
        """T2DenoiserArgs over audio (B, n) on the device, with a workspace of the engine's cache."""
        B, n = int(audio.shape[0]), int(audio.shape[1])
        bias = module.bias_spec
        if bias.numel() != module.stft.filter_length // 2 + 1 or bias.device != self.device:
            raise ValueError("Denoiser: bias_spec must hold %d values on %s" % (module.stft.filter_length // 2 + 1,
                                                                               self.device))
        self._bias = bias.detach().to(torch.float32).contiguous()
        ws = self._ws.get("run", _capi.lib().t2_denoiser_workspace_bytes(self.handle, B, n), self.device)
        return _capi.T2DenoiserArgs(audio.data_ptr(), B, n, _engine._ptr(len32), int(audio.dtype == torch.float16),
                                    self._bias.data_ptr(), float(strength), out.data_ptr(), ws.data_ptr(), ws.numel())
