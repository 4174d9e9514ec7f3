"""The WaveGlow denoiser (waveglow/denoiser.py of the reference) on the sm_90a engine.

``Denoiser(waveglow)`` has the reference's constructor, ``stft`` submodule, buffers and ``state_dict`` keys.  Its
``bias_spec`` comes from the engine's own ``WaveGlow.infer`` and ``forward`` runs entirely in libt2b200 (denoiser.cu),
on the engine handle of its ``stft`` (tacotron2_b200.stft.STFT, also importable from here): there is no CPU path and
no fallback.  ``forward`` also takes per-row ``lengths``, and ``stream`` denoises the items of
``WaveGlow.infer_stream`` as they arrive.
"""
import ctypes as C

import torch

from . import _capi
from . import _engine
from ._stream import FinalWindow
from .stft import STFT

HOP = 256


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
        with torch.no_grad():
            bias_audio = waveglow.infer(mel_input, sigma=0.0).float()
            bias_spec = self._engine().bias(self, bias_audio)
        self.register_buffer('bias_spec', bias_spec.view(1, -1, 1))

    def _engine(self):
        # the handle holding the packed bases belongs to the stft submodule
        return self.stft._engine()

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


def denoiser_halo():
    """(left, right): the 256-sample blocks of audio before and after an output block that it depends on
    (t2_denoiser_window_halo)."""
    left, right = C.c_int32(), C.c_int32()
    _capi.lib().t2_denoiser_window_halo(C.byref(left), C.byref(right))
    return left.value, right.value
