"""The WaveGlow denoiser (waveglow/denoiser.py of the reference) on the sm_90a engine.

``Denoiser(waveglow)`` has the reference's constructor, ``stft`` submodule, buffers and ``state_dict`` keys.  Its
``bias_spec`` comes from the engine's own ``WaveGlow.infer`` and ``forward`` runs entirely in libt2b200 (denoiser.cu):
there is no CPU path and no fallback.  ``forward`` also takes per-row ``lengths``, and ``stream`` denoises the items of
``WaveGlow.infer_stream`` as they arrive.
"""
import ctypes as C
import functools

import numpy as np
import torch

from . import _capi
from . import _engine
from ._stream import FinalWindow
from .layers import _windowed_fourier_basis

HOP = 256


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


class STFT(torch.nn.Module):
    """Holds the reference STFT's configuration and its two windowed bases (stft.py:41-66).  The transforms themselves
    run only inside ``Denoiser.forward``."""

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


class Denoiser(torch.nn.Module):
    """Removes model bias from audio produced with WaveGlow (waveglow/denoiser.py)."""

    def __init__(self, waveglow, filter_length=1024, n_overlap=4, win_length=1024, mode='zeros'):
        super().__init__()
        dev, dt = waveglow.upsample.weight.device, waveglow.upsample.weight.dtype
        self.stft = STFT(filter_length=filter_length, hop_length=int(filter_length / n_overlap),
                         win_length=win_length).to(dev)
        if mode == 'zeros':
            mel_input = torch.zeros((1, 80, 88), dtype=dt, device=dev)
        elif mode == 'normal':
            mel_input = torch.randn((1, 80, 88), dtype=dt, device=dev)
        else:
            raise Exception("Mode {} if not supported".format(mode))
        self._t2 = None
        with torch.no_grad():
            bias_audio = waveglow.infer(mel_input, sigma=0.0).float()
            bias_spec = self._engine().bias(self, bias_audio)
        self.register_buffer('bias_spec', bias_spec.view(1, -1, 1))

    def __getstate__(self):
        # the engine handle is per-instance runtime state: a pickled module rebuilds it on first use
        state = self.__dict__.copy()
        state["_t2"] = None
        return state

    def _engine(self):
        if self._t2 is None:
            self._t2 = _DenoiserEngine(self.stft)
        return self._t2

    @torch.no_grad()
    def forward(self, audio, strength=0.1, lengths=None):
        """audio (B, n) -> denoised audio (B, 1, 256 floor(n / 256)) fp32 (denoiser.py:40-45).

        lengths (B) in samples, optional: row b is denoised as ``audio[b, :lengths[b]]`` alone, bit for bit, and its
        samples from 256 floor(lengths[b] / 256) on are zero; a value outside [0, n] counts as n.  A row of at most 512
        samples cannot be reflect-padded and gives zeros.  Without lengths, n must exceed 512, as in the reference.
        The transforms run on split fp16 operands: samples must stay below 65504 in magnitude (int16-scale audio, up to
        32767, is fine) and strength must be >= 0, or the output holds inf / NaN."""
        eng = self._engine()
        eng.ensure(self)
        audio = eng.audio(audio, "Denoiser.forward")
        B, n = int(audio.shape[0]), int(audio.shape[1])
        if lengths is None and n <= 512:
            raise ValueError("Denoiser.forward: %d samples cannot be reflect-padded by 512 (the reference needs n > 512)" % n)
        len32 = None
        if lengths is not None:
            len32 = _engine._i32(torch.as_tensor(lengths), eng.device)
            if tuple(len32.shape) != (B,):
                raise ValueError("Denoiser.forward: lengths must have shape (%d,), got %s" % (B, tuple(len32.shape)))
        out = torch.empty(B, 1, HOP * (n // HOP), device=eng.device, dtype=torch.float32)
        if n // HOP == 0:
            return out
        eng._call(_capi.lib().t2_denoiser_run, C.byref(eng.args(self, audio, len32, strength, out)))
        return out

    @torch.no_grad()
    def stream(self, items, strength=0.1):
        """forward() over the items of ``WaveGlow.infer_stream(...)``, as a generator that hands out denoised audio as
        soon as no later sample can change it.

        Each item is a dict: ``samples`` = (d0, d1), the same for every row; ``audio`` (B, d1 - d0) fp32; ``mel_lengths``
        and ``finished`` of the audio item it came from.  An output block of 256 samples depends on the 3 blocks of
        audio before it and the 3 after it (``denoiser_halo()``), so while a row is live an item holds every block up to
        the final audio less 3 blocks, and the last item (``finished``) holds the rest; audio items that make no block
        final yield nothing.  Concatenated along time the items are bit-identical to
        ``forward(waveglow.infer(mel_outputs_postnet, sigma, lengths=model.mel_lengths), strength,
        lengths=256 * model.mel_lengths)[:, 0]``.  The stream keeps only the audio later windows can still need: the
        two halos plus one item.  It shares the module's workspace with forward, so both enqueue on the same CUDA
        stream (torch's current stream)."""
        eng = self._engine()
        win = FinalWindow("Denoiser.stream: audio items", "samples", 1, *denoiser_halo(), unit=HOP)
        for item in items:
            win.check(item)
            x = item["audio"]
            if win.kept is None:
                eng.ensure(self)
                x = eng.audio(x, "Denoiser.stream")
            span = win.add(item, x)
            if span is None:
                continue
            (d0, d1), finished, kept = span, bool(item["finished"]), win.kept
            out = torch.empty(int(kept.shape[0]), HOP * (d1 - d0), device=eng.device, dtype=torch.float32)
            if d1 > d0:                # the window is every kept sample; -1: a row that does not end in it goes on
                a = eng.args(self, kept.contiguous(), win.lengths(item["mel_lengths"], -1), strength, out)
                w = _capi.T2DenoiserWindowArgs(a, win.base, d0 - win.base // HOP, d1 - win.base // HOP, int(finished))
                eng._call(_capi.lib().t2_denoiser_run_window, C.byref(w))
            yield dict(samples=(HOP * d0, HOP * d1), audio=out, mel_lengths=item["mel_lengths"], finished=finished)
            if finished:
                return


class _DenoiserEngine(_engine._Handle):
    """One T2Denoiser handle (packed bases on one device) + a cached workspace."""

    kind, what = "denoiser", "tacotron2_b200.Denoiser"
    stream = _engine._Handle._stream      # the name callers of the window entry points use

    def __init__(self, stft):
        super().__init__()
        self.cfg = (int(stft.filter_length), int(stft.hop_length), int(stft.win_length))

    def ensure(self, module):
        st = module.stft
        self._ensure(st.forward_basis.device, (st.forward_basis, st.inverse_basis))

    def _pack(self, bases, dev):
        f, i = (b.detach().to(device=dev, dtype=torch.float32).contiguous() for b in bases)
        return (f, i), (f.data_ptr(), i.data_ptr())

    def _config(self):
        return _capi.T2DenoiserConfig(*self.cfg, 0)

    def audio(self, audio, what):
        """audio (B, n) on the device: fp16 stays fp16 (converted as it is packed), any other real dtype becomes fp32."""
        if not isinstance(audio, torch.Tensor) or audio.dim() != 2:
            raise ValueError("%s: audio must be a (B, n) tensor, got %s" % (what, tuple(getattr(audio, "shape", ()))))
        if audio.dtype == torch.bool or audio.is_complex():
            raise TypeError("%s: audio must be real-valued, got %s" % (what, audio.dtype))
        if audio.shape[0] == 0 or audio.shape[1] == 0:
            raise ValueError("%s: audio is empty, shape %s" % (what, tuple(audio.shape)))
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


def denoiser_halo():
    """(left, right): the 256-sample blocks of audio before and after an output block that it depends on
    (t2_denoiser_window_halo)."""
    left, right = C.c_int32(), C.c_int32()
    _capi.lib().t2_denoiser_window_halo(C.byref(left), C.byref(right))
    return left.value, right.value
