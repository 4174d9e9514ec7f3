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
from ._stream import FinalWindow

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
    (``noise_channel_order``: the n_remaining_channels initial ones, then each early block from the last early flow
    down; published: 4, then flows 8 and 4).  None => in-kernel Philox."""
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
            self._t2.invalidate()

    def window_halo(self):
        """(left, right): the mel frames before and after a frame that this model's audio depends on
        (t2_waveglow_window_halo_config); (99, 96) for the published configuration."""
        return config_halo(self._cfg)

    def _weight_table(self):
        """(tensor or None) x t2_waveglow_num_weights in the engine's table order: the reference state_dict order with
        weight-normed convolutions as (bias, weight_g, weight_v); plain weights (after remove_weightnorm) go in the
        weight_v slot."""
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
    def infer(self, spect, sigma=1.0, lengths=None, seeds=None):
        """mel spectrogram (B, n_mel, T_mel) -> audio (B, 256 T_mel) in the spectrogram's dtype (glow.py:251-293).
        lengths (B) in mel frames, optional: row b's samples [0, 256 lengths[b]) are what infer gives for that row's
        first lengths[b] frames alone; later samples are zero.

        seeds: one noise seed per row, B integers in [0, 2**64) as a list, a host tensor or a device tensor (int64 values
        are taken as their 64-bit pattern).  Row b then draws the noise of ``infer(spect[b:b+1], sigma, seeds=[seeds[b]])``
        and equals that call bit for bit in any batch; a B = 1 call with seeds=[s] is the unseeded call whose drawn seed
        was s.  Not together with ``waveglow_noise``.  None: one seed per call from torch's generator, as before."""
        return self._engine().infer(self, spect, sigma, lengths, getattr(_tls, "z", None), seeds)

    def infer_stream(self, items, sigma=1.0, seeds=None):
        """infer() over the items of ``Tacotron2.inference_stream(...)``, as a generator that hands out audio as soon as
        no later mel frame can change it.

        Each item is a dict: ``samples`` = (s0, s1), the same for every row; ``audio`` (B, s1 - s0) in the mel's dtype;
        ``mel_lengths`` and ``finished`` of the mel item it came from.  The audio of frame t depends on the mel frames
        t - 99 ... t + 96 (``window_halo()``), so while a row is live an item holds the audio of every frame up to the
        final mel frames less 96, and the last item (``finished``) holds the rest; mel items that make no audio final
        yield nothing.  (99 and 96 are the published configuration's halos; another configuration's are
        ``self.window_halo()``.)  Each item runs one windowed inference over the frames its audio depends on.  Concatenated along
        time the audio is bit-identical to ``infer(mel_outputs_postnet, sigma, lengths=model.mel_lengths)`` after
        ``model.inference(...)``, with the same weights and inputs and the same injected noise (``waveglow_noise``, read
        when infer_stream is called) or torch seed: the stream draws its Philox seed from torch's generator once, at its
        first mel item.  A stopped row's samples past 256 * mel_lengths are zero.

        The stream keeps on the device only the final mel frames later windows can still need (at most the two halos and
        one item's frames).  Several streams, and infer, can be used on one WaveGlow at a time: each stream has its own
        frames, noise seed and position, and they share the module's workspace, so all of them must enqueue on the same
        CUDA stream (torch's current stream), as successive infer calls do.  seeds: as for infer(); the stream then
        equals ``infer(..., seeds=seeds)``."""
        return self._engine().stream(self, items, sigma, getattr(_tls, "z", None), seeds)


class _WaveGlowEngine(_engine._Handle):
    """One T2WaveGlow handle (packed weights on one device) + a cached workspace."""

    kind, what = "waveglow", "tacotron2_b200.WaveGlow"

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        self.last_seed = None

    def ensure(self, module):
        w = module.upsample.weight
        self._ensure(w.device, module._weight_table(), (w.dtype == torch.float16,))

    def _pack(self, table, dev, fp16):
        n = num_weights(self.cfg) or len(table)    # an unsupported configuration: t2_waveglow_create refuses it
        n_conv = n - self.cfg[1]                   # the table ends with one convinv weight per flow
        held, ptrs = [], (C.c_void_p * n)()
        for i, t in enumerate(table[:n]):
            if t is None:
                continue
            t = t.detach()
            dt = torch.float32 if i >= n_conv or not fp16 else torch.float16    # convinv: always fp32 (as the notebook)
            if t.dtype != dt or not t.is_contiguous():
                t = t.to(dt).contiguous()
            held.append(t)
            ptrs[i] = t.data_ptr()
        return held, (ptrs, n)

    def _config(self, fp16):
        return _config_struct(self.cfg, fp16)

    def _spect(self, spect, what):
        if spect.dim() != 3 or spect.shape[1] != self.cfg[0]:
            raise ValueError("%s: spect must be (B, %d, T_mel), got %s" % (what, self.cfg[0], tuple(spect.shape)))
        if spect.dtype not in (torch.float32, torch.float16):
            raise TypeError("%s: spect must be float32 or float16, got %s" % (what, spect.dtype))
        return spect.to(self.device).contiguous()

    def _z(self, z, B, T):
        """Injected noise as fp32 on the device, (B, n_group, 32 T') with T' >= T frames; returns (tensor, T')."""
        zt = z.to(device=self.device, dtype=torch.float32).contiguous()
        if zt.dim() != 3 or tuple(zt.shape[:2]) != (B, N_GROUP) or zt.shape[2] % 32 or zt.shape[2] < 32 * T:
            raise ValueError("waveglow_noise: z must be (%d, %d, 32 T_mel) with T_mel >= %d, got %s" %
                             (B, N_GROUP, T, tuple(z.shape)))
        return zt, zt.shape[2] // 32

    def _draw_seed(self):
        # Philox seed drawn from torch's default generator: reproducible under torch.manual_seed, fresh on every call
        seed = int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64).item())
        self.last_seed = seed
        return seed

    def _args(self, spect, len32, zt, sigma, seed, audio, row_seeds=None):
        """T2WaveGlowArgs over spect (B, n_mel, T) on the device, with a workspace of the engine's cache."""
        B, T = int(spect.shape[0]), int(spect.shape[2])
        ws = self._ws.get("infer", _capi.lib().t2_waveglow_workspace_bytes(self.handle, B, T), self.device)
        return _capi.T2WaveGlowArgs(spect.data_ptr(), B, T, _engine._ptr(len32), int(spect.dtype == torch.float16),
                                    float(sigma), _engine._ptr(zt), seed, audio.data_ptr(), ws.data_ptr(), ws.numel(),
                                    _engine._ptr(row_seeds))

    def _row_seeds(self, seeds, z, B, what):
        """seeds as (B,) int64 bit patterns on the device, or None; refused together with injected noise."""
        if seeds is None:
            return None
        if z is not None:
            raise ValueError("%s: seeds and waveglow_noise exclude each other" % what)
        return _engine.row_seeds(seeds, B, self.device, what)

    def infer(self, module, spect, sigma, lengths, z, seeds=None):
        self.ensure(module)
        spect = self._spect(spect, "WaveGlow.infer")
        dev = self.device
        B, T = int(spect.shape[0]), int(spect.shape[2])
        row_seeds = self._row_seeds(seeds, z, B, "WaveGlow.infer")
        audio = torch.empty(B, HOP * T, device=dev, dtype=spect.dtype)
        len32 = None
        if lengths is not None:
            len32 = _engine._i32(torch.as_tensor(lengths), dev)
            if tuple(len32.shape) != (B,):
                raise ValueError("WaveGlow.infer: lengths must have shape (%d,)" % B)
        zt = None
        if z is not None:
            zt = z.to(device=dev, dtype=torch.float32).contiguous()
            if tuple(zt.shape) != (B, N_GROUP, 32 * T):
                raise ValueError("waveglow_noise: z must be (%d, %d, %d), got %s" % (B, N_GROUP, 32 * T, tuple(z.shape)))
        # a seeded call draws nothing from torch's generator
        a = self._args(spect, len32, zt, sigma, 0 if row_seeds is not None else self._draw_seed(), audio, row_seeds)
        self._call(_capi.lib().t2_waveglow_infer, C.byref(a))
        return audio

    def infer_window(self, spect, len32, zt, z_frames, sigma, seed, frame0, out0, out1, at_end, row_seeds=None):
        """Audio (B, 256 (out1 - out0)) of the window-relative frames [out0, out1) of spect, which holds the frames
        [frame0, frame0 + T) of a sequence (t2_waveglow_infer_window).  Call ensure() first."""
        audio = torch.empty(int(spect.shape[0]), HOP * (out1 - out0), device=self.device, dtype=spect.dtype)
        w = _capi.T2WaveGlowWindowArgs(self._args(spect, len32, zt, sigma, seed, audio, row_seeds), frame0, out0, out1,
                                       z_frames if zt is not None else 0, int(at_end))
        self._call(_capi.lib().t2_waveglow_infer_window, C.byref(w))
        return audio

    @torch.no_grad()
    def stream(self, module, items, sigma, z, seeds=None):
        """The generator behind WaveGlow.infer_stream."""
        win = FinalWindow("WaveGlow.infer_stream: mel items", "frames", 2, *config_halo(self.cfg))
        zt = z_frames = seed = row_seeds = None
        for item in items:
            win.check(item)
            post = item["mel_outputs_postnet"]
            if win.kept is None:       # the first item: weights, the noise seed (one draw, as infer)
                self.ensure(module)
                post = self._spect(post, "WaveGlow.infer_stream")
                if z is not None:
                    zt, z_frames = self._z(z, int(post.shape[0]), item["frames"][1])
                row_seeds = self._row_seeds(seeds, z, int(post.shape[0]), "WaveGlow.infer_stream")
                seed = 0 if row_seeds is not None else self._draw_seed()
            span = win.add(item, post)
            if span is None:
                continue
            (a0, a1), finished, kept = span, bool(item["finished"]), win.kept
            audio = kept.new_empty(kept.shape[0], 0)
            if a1 > a0:                # the window is every kept frame; a row that does not end in it ends at its end
                audio = self.infer_window(kept.contiguous(), win.lengths(item["mel_lengths"], win.held - win.base), zt,
                                          z_frames, sigma, seed, win.base, a0 - win.base, a1 - win.base, finished,
                                          row_seeds)
            yield dict(samples=(HOP * a0, HOP * a1), audio=audio, mel_lengths=item["mel_lengths"], finished=finished)
            if finished:
                return


def window_halo():
    """(left, right): the mel frames before and after a frame that the published WaveGlow's audio depends on
    (t2_waveglow_window_halo); ``WaveGlow.window_halo()`` gives a model's own."""
    left, right = C.c_int32(), C.c_int32()
    _capi.lib().t2_waveglow_window_halo(C.byref(left), C.byref(right))
    return left.value, right.value


def _config_struct(cfg, fp16=0):
    return _capi.T2WaveGlowConfig(*[int(x) if x is not None else -1 for x in cfg], int(fp16))


def num_weights(cfg):
    """Length of the engine's weight table for the configuration tuple ``cfg`` (WaveGlow._cfg); 0 if unsupported."""
    return int(_capi.lib().t2_waveglow_num_weights(C.byref(_config_struct(cfg))))


def config_halo(cfg):
    """(left, right) halos of the configuration tuple ``cfg`` (t2_waveglow_window_halo_config)."""
    left, right = C.c_int32(), C.c_int32()
    _capi.check(_capi.lib().t2_waveglow_window_halo_config(C.byref(_config_struct(cfg)), C.byref(left), C.byref(right)))
    return left.value, right.value
