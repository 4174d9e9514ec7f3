"""The HiFi-GAN generator (jik876/hifi-gan, models.py: Generator, ResBlock1, ResBlock2) with inference on the sm_90a
engine.

The module tree, parameter names, registration order and seeded initialisation are those of models.py, so a published
generator checkpoint loads unchanged: ``G.load_state_dict(torch.load(ckpt)["generator"])``.  ``Generator.forward`` runs
entirely in libt2b200 (hifigan.cu): there is no CPU path and no fallback, and no backward.

It reads the mels Tacotron2 makes (80 Slaney bands, 22050 Hz, hop 256, log of the clamped magnitude), so text to audio
is ``G(model.inference(text, lengths)[1], lengths=model.mel_lengths)``.
"""
import ctypes as C
import warnings

import torch

from . import _capi
from . import _engine

N_MEL = 80
HOP = 256
LRELU_SLOPE = 0.1

CONFIGS = {
    "v1": dict(resblock="1", upsample_rates=[8, 8, 2, 2], upsample_kernel_sizes=[16, 16, 4, 4],
               upsample_initial_channel=512, resblock_kernel_sizes=[3, 7, 11],
               resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]]),
    "v2": dict(resblock="1", upsample_rates=[8, 8, 2, 2], upsample_kernel_sizes=[16, 16, 4, 4],
               upsample_initial_channel=128, resblock_kernel_sizes=[3, 7, 11],
               resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]]),
    "v3": dict(resblock="2", upsample_rates=[8, 8, 4], upsample_kernel_sizes=[16, 16, 8],
               upsample_initial_channel=256, resblock_kernel_sizes=[3, 5, 7],
               resblock_dilation_sizes=[[1, 2], [2, 6], [3, 12]]),
}
MAX_STAGES, MAX_KERNELS, MAX_PAD = 8, 8, 64      # T2_HIFIGAN_MAX_STAGES / _KERNELS / _PAD


def get_padding(kernel_size, dilation=1):
    return int((kernel_size * dilation - dilation) / 2)


def init_weights(m, mean=0.0, std=0.01):
    """models.py's initialiser.  Applied after weight_norm, as there, it draws into the module's computed ``weight``;
    weight_g and weight_v keep torch's default initialisation, and the draws advance torch's generator."""
    if m.__class__.__name__.find("Conv") != -1:
        m.weight.data.normal_(mean, std)


def _weight_norm(conv):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", FutureWarning)
        return torch.nn.utils.weight_norm(conv)


def _remove_weight_norm(conv):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", FutureWarning)
        torch.nn.utils.remove_weight_norm(conv)


def _field(h, name):
    return h[name] if isinstance(h, dict) else getattr(h, name)


class ResBlock1(torch.nn.Module):
    def __init__(self, h, channels, kernel_size=3, dilation=(1, 3, 5)):
        super().__init__()
        self.h = h
        self.convs1 = torch.nn.ModuleList([
            _weight_norm(torch.nn.Conv1d(channels, channels, kernel_size, 1, dilation=d,
                                         padding=get_padding(kernel_size, d))) for d in dilation[:3]])
        self.convs1.apply(init_weights)
        self.convs2 = torch.nn.ModuleList([
            _weight_norm(torch.nn.Conv1d(channels, channels, kernel_size, 1, dilation=1,
                                         padding=get_padding(kernel_size, 1))) for _ in range(3)])
        self.convs2.apply(init_weights)

    def forward(self, x):
        raise NotImplementedError("tacotron2_b200.hifigan.ResBlock1 runs only inside Generator.forward (the engine)")

    def remove_weight_norm(self):
        for c in self.convs1:
            _remove_weight_norm(c)
        for c in self.convs2:
            _remove_weight_norm(c)


class ResBlock2(torch.nn.Module):
    def __init__(self, h, channels, kernel_size=3, dilation=(1, 3)):
        super().__init__()
        self.h = h
        self.convs = torch.nn.ModuleList([
            _weight_norm(torch.nn.Conv1d(channels, channels, kernel_size, 1, dilation=d,
                                         padding=get_padding(kernel_size, d))) for d in dilation[:2]])
        self.convs.apply(init_weights)

    def forward(self, x):
        raise NotImplementedError("tacotron2_b200.hifigan.ResBlock2 runs only inside Generator.forward (the engine)")

    def remove_weight_norm(self):
        for c in self.convs:
            _remove_weight_norm(c)


def check_config(h):
    """Refuses, naming the field, a configuration the sm_90a kernels do not implement (ValueError)."""
    rb = str(_field(h, "resblock"))
    rates, kernels = list(_field(h, "upsample_rates")), list(_field(h, "upsample_kernel_sizes"))
    c0 = int(_field(h, "upsample_initial_channel"))
    rks, rds = list(_field(h, "resblock_kernel_sizes")), [list(d) for d in _field(h, "resblock_dilation_sizes")]
    what = "tacotron2_b200.HiFiGAN"
    if rb not in ("1", "2"):
        raise ValueError('%s: resblock must be "1" or "2" (got %r)' % (what, rb))
    if not 1 <= len(rates) <= MAX_STAGES or len(kernels) != len(rates):
        raise ValueError("%s: upsample_rates and upsample_kernel_sizes must have the same 1 ... %d entries" % (what, MAX_STAGES))
    if any(u < 2 or u % 2 for u in rates):
        raise ValueError("%s: upsample_rates must be even (got %s)" % (what, rates))
    prod = 1
    for u in rates:
        prod *= u
    if prod != HOP:
        raise ValueError("%s: the product of upsample_rates must be %d, the hop length (got %d)" % (what, HOP, prod))
    if any(k != 2 * u for u, k in zip(rates, kernels)):
        raise ValueError("%s: upsample_kernel_sizes must be twice upsample_rates (got %s for %s)" % (what, kernels, rates))
    for i in range(-1, len(rates)):
        ch = c0 >> (i + 1)
        if ch < 8 or ch > 512 or ch % 8 or ch << (i + 1) != c0:
            raise ValueError("%s: upsample_initial_channel %d gives stage %d %d channels; every stage needs a multiple "
                             "of 8 in 8 ... 512" % (what, c0, i + 1, c0 / 2 ** (i + 1)))
    if not 1 <= len(rks) <= MAX_KERNELS or len(rds) != len(rks):
        raise ValueError("%s: resblock_kernel_sizes and resblock_dilation_sizes must have the same 1 ... %d entries"
                         % (what, MAX_KERNELS))
    nd = 3 if rb == "1" else 2
    for k, ds in zip(rks, rds):
        if k < 1 or k > 15 or k % 2 == 0:
            raise ValueError("%s: resblock_kernel_sizes must be odd and at most 15 (got %d)" % (what, k))
        if len(ds) < nd:
            raise ValueError("%s: resblock_dilation_sizes needs %d dilations per kernel for resblock %s (got %s)"
                             % (what, nd, rb, ds))
        for d in ds[:nd]:
            if d < 1 or get_padding(k, d) > MAX_PAD:
                raise ValueError("%s: resblock_dilation_sizes: kernel %d with dilation %d pads %d rows; the guard rows "
                                 "allow dilations >= 1 with at most %d" % (what, k, d, get_padding(k, d), MAX_PAD))


class Generator(torch.nn.Module):
    def __init__(self, h):
        super().__init__()
        self.h = h
        self.num_kernels = len(_field(h, "resblock_kernel_sizes"))
        self.num_upsamples = len(_field(h, "upsample_rates"))
        c0 = _field(h, "upsample_initial_channel")
        self.conv_pre = _weight_norm(torch.nn.Conv1d(N_MEL, c0, 7, 1, padding=3))
        resblock = ResBlock1 if str(_field(h, "resblock")) == "1" else ResBlock2
        self.ups = torch.nn.ModuleList()
        for i, (u, k) in enumerate(zip(_field(h, "upsample_rates"), _field(h, "upsample_kernel_sizes"))):
            self.ups.append(_weight_norm(torch.nn.ConvTranspose1d(c0 // (2 ** i), c0 // (2 ** (i + 1)), k, u,
                                                                  padding=(k - u) // 2)))
        self.resblocks = torch.nn.ModuleList()
        for i in range(len(self.ups)):
            ch = c0 // (2 ** (i + 1))
            for k, d in zip(_field(h, "resblock_kernel_sizes"), _field(h, "resblock_dilation_sizes")):
                self.resblocks.append(resblock(h, ch, k, d))
        self.conv_post = _weight_norm(torch.nn.Conv1d(ch, 1, 7, 1, padding=3))
        self.ups.apply(init_weights)
        self.conv_post.apply(init_weights)
        self._t2 = None

    def remove_weight_norm(self):
        for c in self.ups:
            _remove_weight_norm(c)
        for r in self.resblocks:
            r.remove_weight_norm()
        _remove_weight_norm(self.conv_pre)
        _remove_weight_norm(self.conv_post)

    def __getstate__(self):
        # the engine handle is per-instance runtime state: a pickled module rebuilds it on first use
        state = self.__dict__.copy()
        state["_t2"] = None
        return state

    def invalidate_weights(self):
        """Re-pack the engine's weights on the next call (after writes through ``.data`` that torch does not count)."""
        if self._t2 is not None:
            self._t2.invalidate()

    def convs(self):
        """Every convolution in state_dict order: conv_pre, ups, resblocks (ResBlock1: convs1, then convs2), conv_post."""
        out = [self.conv_pre] + list(self.ups)
        for r in self.resblocks:
            out += list(r.convs1) + list(r.convs2) if isinstance(r, ResBlock1) else list(r.convs)
        return out + [self.conv_post]

    def _weight_table(self):
        """(tensor or None) x t2_hifigan_num_weights: (bias, weight_g, weight_v) of every convolution in state_dict
        order; after remove_weight_norm, (bias, None, weight)."""
        t = []
        for c in self.convs():
            t += [c.bias, c.weight_g, c.weight_v] if hasattr(c, "weight_v") else [c.bias, None, c.weight]
        return t

    def forward(self, x, lengths=None):
        """mel spectrogram x (B, 80, T_mel) -> audio (B, 1, 256 T_mel) in the module's dtype.  lengths (B,) in mel
        frames, optional (e.g. ``model.mel_lengths``): row b's samples [0, 256 lengths[b]) equal
        ``G(x[b:b+1, :, :lengths[b]])`` bit for bit; later samples are zero."""
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("tacotron2_b200.HiFiGAN implements inference only: there is no backward.  Run it "
                                      "under torch.no_grad() / torch.inference_mode() or with requires_grad_(False)")
        if self._t2 is None:
            self._t2 = _HiFiGANEngine()
        with torch.no_grad():
            return self._t2.infer(self, x, lengths)


HiFiGAN = Generator


def config_struct(h, fp16=0):
    """T2HiFiGANConfig of the configuration ``h`` (no checks: the library refuses what it does not implement)."""
    c = _capi.T2HiFiGANConfig()
    c.n_mel_channels = N_MEL
    c.resblock = int(str(_field(h, "resblock")))
    rates, kernels = list(_field(h, "upsample_rates")), list(_field(h, "upsample_kernel_sizes"))
    c.n_upsamples = len(rates)
    for i, (u, k) in enumerate(zip(rates[:MAX_STAGES], kernels[:MAX_STAGES])):
        c.upsample_rates[i], c.upsample_kernel_sizes[i] = int(u), int(k)
    c.upsample_initial_channel = int(_field(h, "upsample_initial_channel"))
    rks, rds = list(_field(h, "resblock_kernel_sizes")), list(_field(h, "resblock_dilation_sizes"))
    c.n_kernels = len(rks)
    for j, (k, ds) in enumerate(zip(rks[:MAX_KERNELS], rds[:MAX_KERNELS])):
        c.resblock_kernel_sizes[j] = int(k)
        for m, d in enumerate(list(ds)[:3]):
            c.resblock_dilation_sizes[j][m] = int(d)
    c.fp16 = int(fp16)
    return c


def num_weights(h):
    """Length of the engine's weight table for the configuration ``h``; 0 if unsupported."""
    return int(_capi.lib().t2_hifigan_num_weights(C.byref(config_struct(h))))


def guard_rows(h):
    """The zero rows the engine keeps around each sequence: the widest resblock padding, at least 4."""
    nd = 3 if str(_field(h, "resblock")) == "1" else 2
    pads = [get_padding(k, d) for k, ds in zip(_field(h, "resblock_kernel_sizes"), _field(h, "resblock_dilation_sizes"))
            for d in list(ds)[:nd]]
    return max([4] + pads)


class _HiFiGANEngine(_engine._Handle):
    """One T2HiFiGAN handle (packed weights on one device) + a cached workspace."""

    kind, what = "hifigan", "tacotron2_b200.HiFiGAN"

    def _pack(self, table, dev, fp16):
        dt = torch.float16 if fp16 else torch.float32
        held, ptrs = [], (C.c_void_p * len(table))()
        for i, t in enumerate(table):
            if t is None:
                continue
            t = t.detach()
            if t.dtype != dt or not t.is_contiguous():
                t = t.to(dt).contiguous()
            held.append(t)
            ptrs[i] = t.data_ptr()
        return held, (ptrs, len(table))

    def _config(self, fp16):
        return config_struct(self.h, fp16)

    def infer(self, module, x, lengths):
        what = "tacotron2_b200.HiFiGAN"
        check_config(module.h)
        if not isinstance(x, torch.Tensor):
            raise TypeError("%s: x must be a tensor (B, %d, T_mel)" % (what, N_MEL))
        if x.dim() != 3 or x.shape[1] != N_MEL or x.shape[0] < 1 or x.shape[2] < 1:
            raise ValueError("%s: x must be (B, %d, T_mel) with B, T_mel >= 1, got %s" % (what, N_MEL, tuple(x.shape)))
        if x.dtype not in (torch.float32, torch.float16):
            raise TypeError("%s: x must be float32 or float16, got %s" % (what, x.dtype))
        B, T = int(x.shape[0]), int(x.shape[2])
        if B * (HOP * T + guard_rows(module.h)) >= 1 << 30:
            raise ValueError("%s: x of %d rows x %d frames is too large: B * (256 T_mel + %d) must stay below 2^30"
                             % (what, B, T, guard_rows(module.h)))
        w = module.conv_pre.bias
        dev = w.device
        len32, _ = _engine.row_lengths(lengths, B, T, "lengths", dev)
        if dev.type != "cuda":
            raise RuntimeError("%s must live on a CUDA device (H100); there is no CPU path -- call .cuda() first" % what)
        self.h = module.h
        fp16 = w.dtype == torch.float16
        self._ensure(dev, module._weight_table(), (fp16,))
        x = x.to(device=dev, dtype=w.dtype).contiguous()
        audio = torch.empty(B, 1, HOP * T, device=dev, dtype=w.dtype)
        ws = self._ws.get("infer", _capi.lib().t2_hifigan_workspace_bytes(self.handle, B, T), dev)
        a = _capi.T2HiFiGANArgs(x.data_ptr(), B, T, _engine._ptr(len32), int(fp16), audio.data_ptr(), ws.data_ptr(),
                                ws.numel())
        self._call(_capi.lib().t2_hifigan_infer, C.byref(a))
        return audio
