"""WaveGlow (waveglow/glow.py of the reference) with inference on the sm_90a engine.

The module tree, parameter names, registration order and seeded initialisation are those of the reference, so its
checkpoints load unchanged and ``torch.manual_seed`` gives the same weights.  ``WaveGlow.infer`` runs entirely in
libt2b200 (waveglow.cu): there is no CPU path and no fallback.  Training (``forward``) is not implemented.
"""
import contextlib
import ctypes as C
import threading
import warnings

import torch

from . import _capi
from . import _engine

N_MEL, N_FLOWS, N_GROUP, N_EARLY_EVERY, N_EARLY_SIZE = 80, 12, 8, 4, 2
WN_CONFIG = dict(n_layers=8, n_channels=256, kernel_size=3)
HOP = 256


def _weight_norm(conv):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", FutureWarning)
        return torch.nn.utils.weight_norm(conv, name="weight")


def _remove_weight_norm(conv):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", FutureWarning)
        return torch.nn.utils.remove_weight_norm(conv)


class Invertible1x1Conv(torch.nn.Module):
    """1x1 convolution with a random orthonormal, determinant +1 weight (glow.py:62-80).  Inference applies its
    inverse, which the engine computes once when it packs the weights."""

    def __init__(self, c):
        super().__init__()
        self.conv = torch.nn.Conv1d(c, c, kernel_size=1, stride=1, padding=0, bias=False)
        w = torch.linalg.qr(torch.FloatTensor(c, c).normal_(), mode="reduced")[0]
        if torch.det(w) < 0:
            w[:, 0] = -1 * w[:, 0]
        self.conv.weight.data = w.view(c, c, 1)


class WN(torch.nn.Module):
    """The non-causal WaveNet of each affine coupling (glow.py:105-151): start, n_layers dilated gated layers with
    residual / skip outputs, end (zero-initialised)."""

    def __init__(self, n_in_channels, n_mel_channels, n_layers, n_channels, kernel_size):
        super().__init__()
        assert kernel_size % 2 == 1 and n_channels % 2 == 0
        self.n_layers = n_layers
        self.n_channels = n_channels
        self.in_layers = torch.nn.ModuleList()
        self.res_skip_layers = torch.nn.ModuleList()
        self.start = _weight_norm(torch.nn.Conv1d(n_in_channels, n_channels, 1))
        end = torch.nn.Conv1d(n_channels, 2 * n_in_channels, 1)
        end.weight.data.zero_()
        end.bias.data.zero_()
        self.end = end
        self.cond_layer = _weight_norm(torch.nn.Conv1d(n_mel_channels, 2 * n_channels * n_layers, 1))
        for i in range(n_layers):
            dilation = 2 ** i
            padding = (kernel_size * dilation - dilation) // 2
            self.in_layers.append(_weight_norm(torch.nn.Conv1d(n_channels, 2 * n_channels, kernel_size,
                                                               dilation=dilation, padding=padding)))
            res_skip = 2 * n_channels if i < n_layers - 1 else n_channels
            self.res_skip_layers.append(_weight_norm(torch.nn.Conv1d(n_channels, res_skip, 1)))

    def forward(self, forward_input):
        raise NotImplementedError("tacotron2_b200.WN runs only inside WaveGlow.infer (the engine's kernels)")


# ---- injected noise (tests feed the same z to the engine and the oracle) ----------------------------------
_tls = threading.local()


@contextlib.contextmanager
def waveglow_noise(z):
    """Standard-normal draws for the next ``WaveGlow.infer`` calls: (B, n_group, 32 T_mel), channels in draw order
    (the n_remaining_channels initial ones, then the early blocks of flow 8 and flow 4).  None => in-kernel Philox."""
    prev = getattr(_tls, "z", None)
    _tls.z = z
    try:
        yield
    finally:
        _tls.z = prev


def noise_channel_order(n_flows=N_FLOWS, n_group=N_GROUP, n_early_every=N_EARLY_EVERY, n_early_size=N_EARLY_SIZE):
    """[(flow or None, n channels)] in the order infer draws them: None = the initial draw."""
    n_rem = n_group - n_early_size * ((n_flows - 1) // n_early_every)
    out = [(None, n_rem)]
    for k in reversed(range(n_flows)):
        if k % n_early_every == 0 and k > 0:
            out.append((k, n_early_size))
    return out


class WaveGlow(torch.nn.Module):
    def __init__(self, n_mel_channels, n_flows, n_group, n_early_every, n_early_size, WN_config):
        super().__init__()
        self.upsample = torch.nn.ConvTranspose1d(n_mel_channels, n_mel_channels, 1024, stride=256)
        assert n_group % 2 == 0
        self.n_flows = n_flows
        self.n_group = n_group
        self.n_early_every = n_early_every
        self.n_early_size = n_early_size
        self.WN = torch.nn.ModuleList()
        self.convinv = torch.nn.ModuleList()
        n_half = n_group // 2
        n_remaining_channels = n_group
        for k in range(n_flows):
            if k % n_early_every == 0 and k > 0:
                n_half = n_half - n_early_size // 2
                n_remaining_channels = n_remaining_channels - n_early_size
            self.convinv.append(Invertible1x1Conv(n_remaining_channels))
            self.WN.append(WN(n_half, n_mel_channels * n_group, **WN_config))
        self.n_remaining_channels = n_remaining_channels
        self._cfg = (n_mel_channels, n_flows, n_group, n_early_every, n_early_size, WN_config.get("n_layers"),
                     WN_config.get("kernel_size"), WN_config.get("n_channels"))
        self._t2 = None

    def forward(self, forward_input):
        raise NotImplementedError("tacotron2_b200.WaveGlow implements inference only (WaveGlow.infer); training "
                                  "(forward / WaveGlowLoss) is not supported")

    @staticmethod
    def remove_weightnorm(model):
        for wn in model.WN:
            wn.start = _remove_weight_norm(wn.start)
            wn.in_layers = torch.nn.ModuleList([_remove_weight_norm(c) for c in wn.in_layers])
            wn.cond_layer = _remove_weight_norm(wn.cond_layer)
            wn.res_skip_layers = torch.nn.ModuleList([_remove_weight_norm(c) for c in wn.res_skip_layers])
        return model

    def __getstate__(self):
        # the engine handle is per-instance runtime state: a pickled module rebuilds it on first use
        state = self.__dict__.copy()
        state["_t2"] = None
        return state

    def invalidate_weights(self):
        """Re-pack the engine's weights on the next call (after writes through ``.data`` that torch does not count)."""
        if self._t2 is not None:
            self._t2.key = None

    def _weight_table(self):
        """(tensor or None) x 686 in the engine's table order: the reference state_dict order with weight-normed
        convolutions as (bias, weight_g, weight_v); plain weights (after remove_weightnorm) go in the weight_v slot."""
        def conv(m):
            if hasattr(m, "weight_v"):
                return [m.bias, m.weight_g, m.weight_v]
            return [m.bias, None, m.weight]
        t = [self.upsample.weight, self.upsample.bias]
        for wn in self.WN:
            for c in wn.in_layers:
                t += conv(c)
            for c in wn.res_skip_layers:
                t += conv(c)
            t += conv(wn.start) + [wn.end.weight, wn.end.bias] + conv(wn.cond_layer)
        t += [c.conv.weight for c in self.convinv]
        return t

    def _engine(self):
        if self._t2 is None:
            self._t2 = _WaveGlowEngine(self._cfg)
        return self._t2

    @torch.no_grad()
    def infer(self, spect, sigma=1.0, lengths=None):
        """mel spectrogram (B, n_mel, T_mel) -> audio (B, 256 T_mel) in the spectrogram's dtype (glow.py:251-293).
        lengths (B) in mel frames, optional: row b's samples [0, 256 lengths[b]) are what infer gives for that row's
        first lengths[b] frames alone; later samples are zero."""
        return self._engine().infer(self, spect, sigma, lengths, getattr(_tls, "z", None))


class _WaveGlowEngine:
    """One T2WaveGlow handle (packed weights on one device) + a cached workspace."""

    def __init__(self, cfg):
        self.cfg = cfg
        self.handle = None
        self.key = None
        self.held = None
        self.device = None
        self.fp16 = None
        self._ws = None
        self.last_seed = None

    def ensure(self, module):
        table = module._weight_table()
        dev = module.upsample.weight.device
        if dev.type != "cuda":
            raise RuntimeError("tacotron2_b200.WaveGlow must live on a CUDA device (H100); there is no CPU path -- "
                               "call .cuda() first")
        fp16 = module.upsample.weight.dtype == torch.float16
        key = (_engine._weights_generation[0], fp16) + tuple(
            None if t is None else (t.data_ptr(), t._version, t.dtype) for t in table)
        if self.handle is not None and key == self.key and dev == self.device:
            return
        n_conv = _capi.T2_WAVEGLOW_NUM_WEIGHTS - len(module.convinv)
        want = torch.float16 if fp16 else torch.float32
        held, ptrs = [], (C.c_void_p * _capi.T2_WAVEGLOW_NUM_WEIGHTS)()
        for i, t in enumerate(table[:_capi.T2_WAVEGLOW_NUM_WEIGHTS]):
            if t is None:
                ptrs[i] = None
                continue
            t = t.detach()
            dt = torch.float32 if i >= n_conv else want     # convinv: always fp32 (the notebook keeps it so)
            if t.dtype != dt or not t.is_contiguous():
                t = t.to(dt).contiguous()
            held.append(t)
            ptrs[i] = t.data_ptr()
        L = _capi.lib()
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        with torch.cuda.device(dev):
            if self.handle is None or dev != self.device or fp16 != self.fp16:
                self.close()
                cfg = _capi.T2WaveGlowConfig(*[int(x) if x is not None else -1 for x in self.cfg], int(fp16))
                h = C.c_void_p()
                _capi.check(L.t2_waveglow_create(C.byref(h), C.byref(cfg), ptrs, _capi.T2_WAVEGLOW_NUM_WEIGHTS, stream))
                self.handle = h
            else:
                _capi.check(L.t2_waveglow_refresh(self.handle, ptrs, _capi.T2_WAVEGLOW_NUM_WEIGHTS, stream))
        self.key, self.held, self.device, self.fp16 = key, held, dev, fp16

    def close(self):
        if self.handle is not None:
            _capi.lib().t2_waveglow_destroy(self.handle)
            self.handle = None
            self.key = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def infer(self, module, spect, sigma, lengths, z):
        self.ensure(module)
        if spect.dim() != 3 or spect.shape[1] != self.cfg[0]:
            raise ValueError("WaveGlow.infer: spect must be (B, %d, T_mel), got %s" % (self.cfg[0], tuple(spect.shape)))
        if spect.dtype not in (torch.float32, torch.float16):
            raise TypeError("WaveGlow.infer: spect must be float32 or float16, got %s" % spect.dtype)
        dev = self.device
        spect = spect.to(dev).contiguous()
        B, T = int(spect.shape[0]), int(spect.shape[2])
        L = _capi.lib()
        audio = torch.empty(B, HOP * T, device=dev, dtype=spect.dtype)
        a = _capi.T2WaveGlowArgs()
        a.mel, a.B, a.T_mel, a.io_half = spect.data_ptr(), B, T, int(spect.dtype == torch.float16)
        len32 = None
        if lengths is not None:
            len32 = torch.as_tensor(lengths).to(device=dev, dtype=torch.int32).contiguous()
            if tuple(len32.shape) != (B,):
                raise ValueError("WaveGlow.infer: lengths must have shape (%d,)" % B)
            a.lengths = len32.data_ptr()
        zt = None
        if z is not None:
            zt = z.to(device=dev, dtype=torch.float32).contiguous()
            if tuple(zt.shape) != (B, N_GROUP, 32 * T):
                raise ValueError("waveglow_noise: z must be (%d, %d, %d), got %s" % (B, N_GROUP, 32 * T, tuple(z.shape)))
            a.z = zt.data_ptr()
        a.sigma = float(sigma)
        # Philox seed drawn from torch's default generator: reproducible under torch.manual_seed, fresh on every call
        a.seed = int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64).item())
        self.last_seed = a.seed
        nbytes = int(L.t2_waveglow_workspace_bytes(self.handle, B, T))
        if self._ws is None or self._ws.numel() < nbytes or self._ws.device != dev:
            self._ws = None
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        a.audio, a.ws, a.ws_bytes = audio.data_ptr(), self._ws.data_ptr(), self._ws.numel()
        with torch.cuda.device(dev):
            _capi.check(L.t2_waveglow_infer(self.handle, C.byref(a), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        return audio
