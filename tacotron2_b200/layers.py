"""LinearNorm / ConvNorm with the reference's parameter names and initialisation (layers.py:8-39).
They only *hold* parameters (``linear_layer.weight``, ``conv.weight`` ... are the state_dict keys the
published checkpoints use); the arithmetic of the hot path is done by libt2b200.so.
TacotronSTFT (layers.py:42-80): the log-mel extraction of the data path, on the GPU through ``t2_mel_spectrogram``, and
its ``stft_fn``, the STFT that ``audio_processing.griffin_lim`` takes."""
import ctypes as C

import torch

from . import _capi
from .stft import STFT, _lengths, _windowed_fourier_basis  # noqa: F401  (layers.py re-exports STFT, as the reference's does)


class LinearNorm(torch.nn.Module):
    def __init__(self, in_dim, out_dim, bias=True, w_init_gain='linear'):
        super(LinearNorm, self).__init__()
        self.linear_layer = torch.nn.Linear(in_dim, out_dim, bias=bias)
        torch.nn.init.xavier_uniform_(
            self.linear_layer.weight, gain=torch.nn.init.calculate_gain(w_init_gain))

    def forward(self, x):
        # not on the engine's hot path (the fused kernels read linear_layer.weight directly); kept so
        # the module stays usable stand-alone
        return self.linear_layer(x)


class ConvNorm(torch.nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size=1, stride=1, padding=None,
                 dilation=1, bias=True, w_init_gain='linear'):
        super(ConvNorm, self).__init__()
        if padding is None:
            assert kernel_size % 2 == 1
            padding = int(dilation * (kernel_size - 1) / 2)
        self.conv = torch.nn.Conv1d(in_channels, out_channels, kernel_size=kernel_size, stride=stride,
                                    padding=padding, dilation=dilation, bias=bias)
        torch.nn.init.xavier_uniform_(self.conv.weight, gain=torch.nn.init.calculate_gain(w_init_gain))

    def forward(self, signal):
        return self.conv(signal)


# ---- TacotronSTFT: log-mel extraction on the GPU (layers.py:42-80, stft.py:44-94) -----------------------------------
def _slaney_mel_filterbank(sampling_rate, n_fft, n_mels, fmin, fmax):
    """The filterbank the reference takes from librosa 0.6.0 (``librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax)``,
    layers.py:50-51; librosa is a dependency outside the reference tree): triangular filters on the Slaney mel scale
    (linear below 1 kHz, logarithmic above), each normalised to unit area in Hz."""
    import numpy as np
    lin_step, knee_hz = 200.0 / 3.0, 1000.0
    knee_mel, log_step = knee_hz / lin_step, np.log(6.4) / 27.0

    def to_mel(hz):
        hz = np.asarray(hz, dtype=np.float64)
        return np.where(hz < knee_hz, hz / lin_step, knee_mel + np.log(np.maximum(hz, 1e-12) / knee_hz) / log_step)

    def to_hz(mel):
        mel = np.asarray(mel, dtype=np.float64)
        return np.where(mel < knee_mel, mel * lin_step, knee_hz * np.exp((mel - knee_mel) * log_step))
    top = sampling_rate / 2.0 if fmax is None else fmax
    edges = to_hz(np.linspace(to_mel(fmin), to_mel(top), n_mels + 2))              # n_mels + 2 band edges in Hz
    bins = np.linspace(0.0, sampling_rate / 2.0, n_fft // 2 + 1)
    rising = (bins[None, :] - edges[:-2, None]) / (edges[1:-1] - edges[:-2])[:, None]
    falling = (edges[2:, None] - bins[None, :]) / (edges[2:] - edges[1:-1])[:, None]
    bank = np.clip(np.minimum(rising, falling), 0.0, None) * (2.0 / (edges[2:] - edges[:-2]))[:, None]
    return torch.from_numpy(bank.astype(np.float32))


class TacotronSTFT(torch.nn.Module):
    """layers.py:42-80 with the same constructor, the ``mel_basis`` buffer and ``mel_spectrogram(y)``; the transform
    itself (reflect padding, windowed DFT as a tensor-core GEMM over overlapping frames, magnitude, mel projection, log
    compression) is ``t2_mel_spectrogram`` of libt2b200.  ``stft_fn`` is the reference's STFT submodule (its
    ``transform`` / ``inverse`` and Griffin-Lim run on the denoiser's GEMMs).  CUDA tensors only."""

    def __init__(self, filter_length=1024, hop_length=256, win_length=1024, n_mel_channels=80, sampling_rate=22050,
                 mel_fmin=0.0, mel_fmax=8000.0):
        super(TacotronSTFT, self).__init__()
        self.n_mel_channels, self.sampling_rate = n_mel_channels, sampling_rate
        self.filter_length, self.hop_length, self.win_length = filter_length, hop_length, win_length
        self.stft_fn = STFT(filter_length, hop_length, win_length)
        self.register_buffer("mel_basis", _slaney_mel_filterbank(sampling_rate, filter_length, n_mel_channels, mel_fmin, mel_fmax))
        self.register_buffer("forward_basis", _windowed_fourier_basis(filter_length, win_length))
        self._ws = _capi.Workspace()

    def spectral_normalize(self, magnitudes):
        return torch.log(torch.clamp(magnitudes, min=1e-5))             # audio_processing.py:78-84, C = 1

    def spectral_de_normalize(self, magnitudes):
        return torch.exp(magnitudes)                                    # audio_processing.py:87-93

    def mel_spectrogram(self, y, lengths=None):
        """y (B, T) in [-1, 1] -> (B, n_mel_channels, T // hop_length + 1).

        lengths (B) in samples, optional (a list, a host or a device integer tensor): row b is the log-mel of
        ``y[b, :lengths[b]]`` alone, bit for bit the B = 1 call on those samples, with its frames from
        lengths[b] // hop_length + 1 on zero; the samples past a row's length are never read and the range check covers
        each row's own samples only.  Each length must lie in [filter_length // 2 + 1, T].  Without lengths, the rows
        of a batch share each frame's operand scale (see DESIGN section 6.9), so a row can differ in its last bits from
        its own B = 1 call."""
        if not y.is_cuda or not self.mel_basis.is_cuda:
            raise RuntimeError("tacotron2_b200.TacotronSTFT: CUDA tensors only (move the module and the audio to the GPU)")
        if lengths is None:
            assert torch.min(y.data) >= -1                              # layers.py:74-75
            assert torch.max(y.data) <= 1
        else:
            if y.dim() != 2:
                raise ValueError("TacotronSTFT.mel_spectrogram: y must be (B, T) with lengths, got %s" % (tuple(y.shape),))
            host = _sample_lengths(lengths, int(y.shape[0]), int(y.shape[1]), self.filter_length)
            len32 = torch.tensor(host, dtype=torch.int32).to(y.device, non_blocking=True)
            own = torch.where(torch.arange(y.shape[1], device=y.device)[None, :] < len32[:, None], y.data, 0)
            assert torch.min(own) >= -1                                 # layers.py:74-75, each row's own samples
            assert torch.max(own) <= 1
        L = _capi.lib()
        y32 = y.detach().to(torch.float32).contiguous()
        B, n = int(y32.shape[0]), int(y32.shape[1])
        frames = int(L.t2_mel_spectrogram_frames(n, self.hop_length))
        out = torch.empty(B, self.n_mel_channels, frames, device=y.device, dtype=torch.float32)
        query = L.t2_mel_spectrogram_workspace_bytes if lengths is None else L.t2_mel_spectrogram_workspace_bytes_lengths
        ws = self._ws.get("mel", query(B, n, self.filter_length, self.hop_length, self.n_mel_channels), y.device)
        a = _capi.T2MelSpecArgs(y32.data_ptr(), B, n, self.filter_length, self.hop_length, self.n_mel_channels,
                                self.forward_basis.data_ptr(), self.mel_basis.data_ptr(), 1e-5, out.data_ptr(),
                                ws.data_ptr(), ws.numel(), None if lengths is None else len32.data_ptr())
        _capi.call(L.t2_mel_spectrogram, y.device, C.byref(a))
        return out


def _sample_lengths(lengths, B, n, filter_length):
    """Per-row sample counts as a host list of ints: B integers in [filter_length // 2 + 1, n] (what reflect padding by
    filter_length // 2 needs), from a list or a host / device integer tensor.  Raises TypeError / ValueError."""
    what = "TacotronSTFT.mel_spectrogram"
    _lengths(lengths, B, None, what)
    t = torch.as_tensor(lengths)
    if t.dtype == torch.bool or t.dtype.is_floating_point or t.dtype.is_complex:
        raise TypeError("%s: lengths must hold integers (got %s)" % (what, t.dtype))
    lo = filter_length // 2 + 1
    vals = [int(v) for v in t.tolist()]
    for b, v in enumerate(vals):
        if not lo <= v <= n:
            raise ValueError("%s: length %d of row %d lies outside [%d, %d] (reflect padding by %d needs more than %d "
                             "samples, and a row holds at most the %d columns of y)" % (what, v, b, lo, n, lo - 1, lo - 1, n))
    return vals
