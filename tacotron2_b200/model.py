"""The reference's nn.Module surface (model.py) over the H100 engine.

Same class names, constructor signatures, attribute names, parameter registration order (hence the
same ``state_dict`` keys AND the same random initialisation under a given torch seed) as
NVIDIA/tacotron2 ``model.py`` -- so ``train.py`` / ``inference.ipynb`` / published checkpoints work
unchanged -- but ``forward`` / ``inference`` run hand-written sm_90a kernels through libt2b200.so:

    Tacotron2.inference  (model.py:517-529)  -> encoder kernels -> persistent decoder kernel -> postnet
    Tacotron2.forward    (model.py:499-515)  -> encoder -> teacher-forced decoder -> postnet -> parse_output
    Decoder.inference    (model.py:418-454)  -> t2_decoder_run(INFER): batched, per-row stop latch
    Decoder.forward      (model.py:381-416)  -> t2_prenet_forward + t2_decoder_run(TEACHER)
    Encoder.forward/.inference (:173-201), Postnet.forward (:141-146)

There is no CPU path: calling these on CPU tensors raises.
"""
import weakref
from math import sqrt

import torch
from torch import nn

from . import _capi
from . import _engine as _engine_mod
from ._engine import Engine, current_masks, next_seed
from .layers import ConvNorm, LinearNorm
from .utils import get_mask_from_lengths, to_gpu


class _EngineOwner(object):
    """Mixin: finds (or lazily creates) the Engine for this module.  Sub-modules of a Tacotron2 share
    the root's engine; a stand-alone Encoder / Decoder / Postnet builds its own (the weight-table
    entries it does not have are filled with zeros)."""

    _t2_prefix = ""

    def _t2_root(self):
        ref = self.__dict__.get("_t2_root_ref")
        root = ref() if ref is not None else None
        return root if root is not None else self

    def _t2_link(self):
        """(Re-)point the children at this module as their engine owner.  The links are weak references kept out of
        copies / pickles (__getstate__ below), so they are rebuilt lazily: a deepcopy of a Tacotron2 must resolve ITS OWN
        parameters, not the original's."""
        ref = None
        for child in self._t2_children():
            cur = child.__dict__.get("_t2_root_ref")
            if cur is None or cur() is not self:
                if ref is None:
                    ref = weakref.ref(self)
                child.__dict__["_t2_root_ref"] = ref

    def _t2_children(self):
        return ()

    def __getstate__(self):
        # copy.deepcopy / pickle / torch.save(model): the engine (a ctypes handle + device workspaces) and the weak
        # back-references are per-instance runtime state; the copy builds its own on first use
        state = dict(super().__getstate__())       # nn.Module.__getstate__ (the mixin precedes nn.Module in the MRO)
        state.pop("_t2_root_ref", None)
        state.pop("_t2_engine_obj", None)
        return state

    def invalidate_weights(self):
        """Call after writing parameters / buffers in a way torch's version counter does not see (``p.data.copy_()``,
        ``p.data.mul_()``, raw pointer writes): the packed device-side operand images are rebuilt on the next call."""
        eng = self._t2_root().__dict__.get("_t2_engine_obj")
        if eng is not None:
            eng.invalidate()

    def _t2_engine(self):
        root = self._t2_root()
        root._t2_link()
        if "_t2_hparams" not in root.__dict__:
            raise RuntimeError("tacotron2_b200: %s must be used as part of a Decoder / Tacotron2" % type(self).__name__)
        eng = root.__dict__.get("_t2_engine_obj")
        if eng is None:
            eng = Engine(root._t2_hparams)
            root.__dict__["_t2_engine_obj"] = eng
        prefix = root._t2_prefix
        named = {}
        for k, v in root.named_parameters():
            named[prefix + k] = v
        for k, v in root.named_buffers():
            named[prefix + k] = v
        # under autograd in training mode the parameters change every step (possibly through .data, which the version
        # counter does not see): always re-pack there; otherwise the (pointer, version, dtype) key decides
        # ... once per top-level call: the modules Tacotron2.forward calls in turn (embedding + encoder, decoder, postnet)
        # share the packing done at its start (root._t2_packed_in_call), they do not repeat it
        force = (root.training and torch.is_grad_enabled() and not root.__dict__.get("_t2_packed_in_call", False) and
                 any(p_.requires_grad for p_ in root.parameters()))
        eng.ensure(named, force=force)
        return eng

    def _t2_device(self):
        """The device of the module's parameters, the one its engine runs on (known without building the engine)."""
        for p_ in self._t2_root().parameters():
            return p_.device
        return torch.device("cpu")

    def _t2_out_dtype(self):
        for p_ in self.parameters():
            return p_.dtype
        return torch.float32


def _invalidate_after_load(module, incompatible_keys):
    """load_state_dict copies into the parameters through .data-like paths: re-pack on the next call."""
    module.invalidate_weights()


def _require_no_grad(module, what, why="the prenet's backward is part of Decoder.forward's, model.py:396-399"):
    if torch.is_grad_enabled() and any(p_.requires_grad for p_ in module.parameters()):
        raise NotImplementedError(
            "tacotron2_b200: %s on its own has no autograd node (%s); call it through Decoder.forward / "
            "Tacotron2.forward or under torch.no_grad()" % (what, why))


_STEP_NO_GRAD = "the step API has no per-step backward; training goes through Decoder.forward"
STEP_MAX_T_ENC = 1282      # the stepwise attention kernel's shared memory (t2_decoder_step)


def _f32(t):
    """t as a contiguous fp32 tensor (itself when it already is one)."""
    return t.detach().to(torch.float32).contiguous()


def _step_tensor(t, name, shape, device, what):
    """A float tensor of the given shape on `device`; TypeError / ValueError naming it otherwise."""
    if not torch.is_tensor(t):
        raise TypeError("tacotron2_b200: %s: %s must be a tensor (got %s)" % (what, name, type(t).__name__))
    if not t.dtype.is_floating_point:
        raise TypeError("tacotron2_b200: %s: %s must be a float tensor (got %s)" % (what, name, t.dtype))
    if tuple(t.shape) != tuple(shape):
        raise ValueError("tacotron2_b200: %s: %s must have shape %s (got %s)" % (what, name, tuple(shape), tuple(t.shape)))
    if t.device != device:
        raise ValueError("tacotron2_b200: %s: %s must be on the model's device %s (got %s); there is no CPU path"
                         % (what, name, device, t.device))
    return t


def _step_mask(mask, B, T, device, what):
    """The reference's mask (None, or bool (B, T_enc), True = padding) as the library's uint8 (B, T_enc), or None."""
    if mask is None:
        return None
    if not torch.is_tensor(mask) or mask.dtype != torch.bool:
        raise TypeError("tacotron2_b200: %s: mask must be None or a bool tensor, True at padded positions (got %s)"
                        % (what, mask.dtype if torch.is_tensor(mask) else type(mask).__name__))
    if tuple(mask.shape) != (B, T):
        raise ValueError("tacotron2_b200: %s: mask must have shape %s (got %s)" % (what, (B, T), tuple(mask.shape)))
    if mask.device != device:
        raise ValueError("tacotron2_b200: %s: mask must be on the model's device %s (got %s)" % (what, device, mask.device))
    return mask.contiguous().view(torch.uint8)


def _step_t_enc(T, what):
    if T > STEP_MAX_T_ENC:
        raise ValueError("tacotron2_b200: %s: T_enc=%d is longer than the step API takes (at most %d)"
                         % (what, T, STEP_MAX_T_ENC))


def _wants_grad(module, *tensors):
    return torch.is_grad_enabled() and (any(t is not None and t.requires_grad for t in tensors) or
                                        any(p_.requires_grad for p_ in module.parameters()))


def _require_no_grad_with_lengths(module, what):
    if torch.is_grad_enabled() and any(p_.requires_grad for p_ in module.parameters()):
        raise NotImplementedError("tacotron2_b200: %s with per-row lengths has no autograd node; call it under "
                                  "torch.no_grad()" % what)


class LocationLayer(_EngineOwner, nn.Module):
    """model.py:10-26.  Evaluated inside the decoder kernels; forward() runs as part of a Decoder / Tacotron2."""
    _t2_prefix = "decoder.attention_layer.location_layer."

    def __init__(self, attention_n_filters, attention_kernel_size, attention_dim):
        super(LocationLayer, self).__init__()
        padding = int((attention_kernel_size - 1) / 2)
        self.location_conv = ConvNorm(2, attention_n_filters, kernel_size=attention_kernel_size,
                                      padding=padding, bias=False, stride=1, dilation=1)
        self.location_dense = LinearNorm(attention_n_filters, attention_dim, bias=False, w_init_gain='tanh')

    def forward(self, attention_weights_cat):
        """model.py:22-26: attention_weights_cat (B, 2, T_enc) -> the location term (B, T_enc, attention_dim), on the
        step API's attention kernel (T_enc <= 1282)."""
        what = "LocationLayer.forward"
        _require_no_grad(self, what, _STEP_NO_GRAD)
        cat = _attention_cat(attention_weights_cat, self._t2_device(), what)
        B, T = int(cat.shape[0]), int(cat.shape[2])
        eng = self._t2_engine()
        loc, = eng.attention(B, T, _f32(cat), location=True)
        return loc.to(attention_weights_cat.dtype)


def _attention_cat(cat, device, what):
    if not torch.is_tensor(cat) or cat.dim() != 3 or cat.shape[1] != 2 or cat.shape[0] < 1 or cat.shape[2] < 1:
        raise ValueError("tacotron2_b200: %s: attention_weights_cat must be a (B, 2, T_enc) tensor (got %s)"
                         % (what, tuple(cat.shape) if torch.is_tensor(cat) else type(cat).__name__))
    _step_tensor(cat, "attention_weights_cat", cat.shape, device, what)
    _step_t_enc(int(cat.shape[2]), what)
    return cat


class Attention(_EngineOwner, nn.Module):
    """model.py:29-86 (score_mask_value, which train.py:76 overwrites from outside, is read at every call).  Its
    forwards run as part of a Decoder / Tacotron2."""
    _t2_prefix = "decoder.attention_layer."

    def __init__(self, attention_rnn_dim, embedding_dim, attention_dim, attention_location_n_filters,
                 attention_location_kernel_size):
        super(Attention, self).__init__()
        self.query_layer = LinearNorm(attention_rnn_dim, attention_dim, bias=False, w_init_gain='tanh')
        self.memory_layer = LinearNorm(embedding_dim, attention_dim, bias=False, w_init_gain='tanh')
        self.v = LinearNorm(attention_dim, 1, bias=False)
        self.location_layer = LocationLayer(attention_location_n_filters, attention_location_kernel_size,
                                            attention_dim)
        self.score_mask_value = -float("inf")

    def _inputs(self, what, query, processed_memory, attention_weights_cat, memory=None, mask=None):
        _require_no_grad(self, what, _STEP_NO_GRAD)
        dev = self._t2_device()
        cat = _attention_cat(attention_weights_cat, dev, what)
        B, T = int(cat.shape[0]), int(cat.shape[2])
        _step_tensor(query, "query", (B, self.query_layer.linear_layer.in_features), dev, what)
        _step_tensor(processed_memory, "processed_memory", (B, T, self.query_layer.linear_layer.out_features), dev, what)
        if memory is not None:
            _step_tensor(memory, "memory", (B, T, self.memory_layer.linear_layer.in_features), dev, what)
        return B, T, dict(weights_cat=_f32(cat), query=_f32(query), pm=_f32(processed_memory),
                          memory=None if memory is None else _f32(memory), mask=_step_mask(mask, B, T, dev, what),
                          score_mask_value=float(self.score_mask_value))

    def get_alignment_energies(self, query, processed_memory, attention_weights_cat):
        """model.py:43-63: query (B, attention_rnn_dim), processed_memory (B, T_enc, attention_dim),
        attention_weights_cat (B, 2, T_enc) -> energies (B, T_enc), before any mask."""
        B, T, kw = self._inputs("Attention.get_alignment_energies", query, processed_memory, attention_weights_cat)
        energies, = self._t2_engine().attention(B, T, energies=True, **kw)
        return energies.to(processed_memory.dtype)

    def forward(self, attention_hidden_state, memory, processed_memory, attention_weights_cat, mask):
        """model.py:65-86 -> (attention_context (B, 512), attention_weights (B, T_enc)) in memory's dtype.  mask: None or
        bool (B, T_enc), True at padded positions, which get score_mask_value before the softmax.  Nothing cumulative is
        updated.  On decode()'s inputs of a step it gives that step's weights and context bit for bit."""
        B, T, kw = self._inputs("Attention.forward", attention_hidden_state, processed_memory, attention_weights_cat,
                                memory, mask)
        weights, context = self._t2_engine().attention(B, T, weights=True, context=True, **kw)
        return context.to(memory.dtype), weights.to(memory.dtype)


class _EncoderFn(torch.autograd.Function):
    """Encoder.forward (model.py:173-190) [+ the embedding lookup of model.py:503 when `text` is given] as one autograd
    node: forward = fp32 conv stack + persistent BiLSTM with a stash, backward = t2_encoder_backward."""

    @staticmethod
    def forward(ctx, owner, prefix_params, text, embedded, lengths, training, *params):
        eng = owner._t2_engine()
        keep = current_masks()["enc"]
        seed = next_seed()
        src = text if text is not None else embedded
        B, T = int(src.shape[0]), int(src.shape[1])
        stash = eng.stash_buffer("encoder", B, T)
        emb32 = None
        if embedded is not None:
            emb32 = embedded.detach().to(dtype=torch.float32).contiguous()
        memory = eng.encoder(text=text, embedded=emb32, lengths=lengths, training=training, keep=keep, stash=stash, seed=seed)
        if training and not owner._t2_root().__dict__.get("_t2_packed_in_call", False):
            eng.invalidate()              # running statistics changed under the packed copies (see Tacotron2._forward_packed)
        ctx.saved = dict(eng=eng, text=text, embedded=emb32, lengths=lengths, training=training, keep=keep, seed=seed,
                         stash=stash, names=prefix_params, params=params,
                         emb_dtype=embedded.dtype if embedded is not None else None)
        return memory

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_memory):
        sv = ctx.saved
        f32 = dict(device=d_memory.device, dtype=torch.float32)
        grads = {n: torch.empty(p_.shape, **f32) for n, p_ in zip(sv["names"], sv["params"])}
        d_emb = sv["eng"].encoder_backward(sv["text"], sv["embedded"], sv["lengths"], sv["training"], sv["keep"], sv["seed"],
                                           sv["stash"], d_memory, sv["embedded"] is not None, grads)
        ctx.saved = None
        if d_emb is not None:
            d_emb = d_emb.to(sv["emb_dtype"])
        return (None, None, None, d_emb, None, None) + tuple(grads[n].to(p_.dtype) for n, p_ in zip(sv["names"], sv["params"]))


class _PostnetFn(torch.autograd.Function):
    """Postnet.forward (model.py:141-146) [+ the residual of model.py:511 when add_residual] as one autograd node."""

    @staticmethod
    def forward(ctx, owner, names, mel_btc, add_residual, training, wgrad_lengths, *params):
        eng = owner._t2_engine()
        keep = current_masks()["post"]
        seed = next_seed()
        x = mel_btc.detach()
        if x.dtype != torch.float32 or x.stride(2) != 1 or x.stride(1) != x.shape[2]:
            x = x.float().contiguous()
        B, T = int(x.shape[0]), int(x.shape[1])
        stash = eng.stash_buffer("postnet", B, T)
        out = eng.postnet(x, None, add_residual, training, keep, stash=stash, seed=seed)
        if training and not owner._t2_root().__dict__.get("_t2_packed_in_call", False):
            eng.invalidate()
        ctx.saved = dict(eng=eng, B=B, T=T, add_residual=add_residual, training=training, keep=keep, seed=seed, stash=stash,
                         names=names, params=params, in_dtype=mel_btc.dtype, wgrad_lengths=wgrad_lengths)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_out):
        sv = ctx.saved
        f32 = dict(device=d_out.device, dtype=torch.float32)
        grads = {n: torch.empty(p_.shape, **f32) for n, p_ in zip(sv["names"], sv["params"])}
        d_mel = sv["eng"].postnet_backward(sv["B"], sv["T"], sv["training"], sv["add_residual"], sv["keep"], sv["seed"],
                                           sv["stash"], d_out, grads, sv["wgrad_lengths"])
        ctx.saved = None
        return (None, None, d_mel.to(sv["in_dtype"]), None, None, None) + tuple(grads[n].to(p_.dtype) for n, p_ in
                                                                          zip(sv["names"], sv["params"]))


class Prenet(_EngineOwner, nn.Module):
    """model.py:89-100.  Dropout(0.5) is always on, as in the reference (model.py:99)."""
    _t2_prefix = "decoder.prenet."

    def __init__(self, in_dim, sizes):
        super(Prenet, self).__init__()
        in_sizes = [in_dim] + sizes[:-1]
        self.layers = nn.ModuleList(
            [LinearNorm(in_size, out_size, bias=False) for (in_size, out_size) in zip(in_sizes, sizes)])

    def forward(self, x):
        _require_no_grad(self, "Prenet.forward")
        eng = self._t2_engine()
        shp = x.shape
        keep = current_masks()["prenet"]
        if keep is not None:   # (steps, 2, B, 256) -> (2, steps*B, 256)
            keep = keep.permute(1, 0, 2, 3).reshape(2, -1, keep.shape[-1])
        out = eng.prenet(x.reshape(-1, shp[-1]), keep)
        return out.reshape(*shp[:-1], out.shape[-1]).to(x.dtype)


class Postnet(_EngineOwner, nn.Module):
    """model.py:103-146: five conv1d(k=5) + BatchNorm1d, tanh on the first four."""
    _t2_prefix = "postnet."

    def __init__(self, hparams):
        super(Postnet, self).__init__()
        self.__dict__["_t2_hparams"] = hparams
        self.convolutions = nn.ModuleList()
        self.convolutions.append(
            nn.Sequential(
                ConvNorm(hparams.n_mel_channels, hparams.postnet_embedding_dim,
                         kernel_size=hparams.postnet_kernel_size, stride=1,
                         padding=int((hparams.postnet_kernel_size - 1) / 2), dilation=1, w_init_gain='tanh'),
                nn.BatchNorm1d(hparams.postnet_embedding_dim)))
        for i in range(1, hparams.postnet_n_convolutions - 1):
            self.convolutions.append(
                nn.Sequential(
                    ConvNorm(hparams.postnet_embedding_dim, hparams.postnet_embedding_dim,
                             kernel_size=hparams.postnet_kernel_size, stride=1,
                             padding=int((hparams.postnet_kernel_size - 1) / 2), dilation=1, w_init_gain='tanh'),
                    nn.BatchNorm1d(hparams.postnet_embedding_dim)))
        self.convolutions.append(
            nn.Sequential(
                ConvNorm(hparams.postnet_embedding_dim, hparams.n_mel_channels,
                         kernel_size=hparams.postnet_kernel_size, stride=1,
                         padding=int((hparams.postnet_kernel_size - 1) / 2), dilation=1, w_init_gain='linear'),
                nn.BatchNorm1d(hparams.n_mel_channels)))

    def _run(self, x, lengths, add_residual):
        xt = x.transpose(1, 2)                       # (B, T, 80): the decoder's native storage
        if lengths is None and _wants_grad(self, x):
            named = [("postnet." + k, p_) for k, p_ in self.named_parameters()]
            return _PostnetFn.apply(self, [n for n, _ in named], xt, add_residual, self.training, None,
                                    *[p_ for _, p_ in named]).to(x.dtype)
        eng = self._t2_engine()
        if xt.dtype != torch.float32 or xt.stride(2) != 1 or xt.stride(1) != xt.shape[2]:
            xt = xt.float().contiguous()
        return eng.postnet(xt.detach(), lengths, add_residual, self.training, current_masks()["post"]).to(x.dtype)

    def forward(self, x):
        """x (B, n_mel, T) -> postnet(x) (B, n_mel, T); the caller adds the residual (model.py:511)."""
        return self._run(x, None, False)


class Encoder(_EngineOwner, nn.Module):
    """model.py:149-201: 3 x (conv1d k5 + BatchNorm1d + ReLU [+dropout]) then a BiLSTM."""
    _t2_prefix = "encoder."

    def __init__(self, hparams):
        super(Encoder, self).__init__()
        self.__dict__["_t2_hparams"] = hparams
        convolutions = []
        for _ in range(hparams.encoder_n_convolutions):
            conv_layer = nn.Sequential(
                ConvNorm(hparams.encoder_embedding_dim, hparams.encoder_embedding_dim,
                         kernel_size=hparams.encoder_kernel_size, stride=1,
                         padding=int((hparams.encoder_kernel_size - 1) / 2), dilation=1, w_init_gain='relu'),
                nn.BatchNorm1d(hparams.encoder_embedding_dim))
            convolutions.append(conv_layer)
        self.convolutions = nn.ModuleList(convolutions)
        self.lstm = nn.LSTM(hparams.encoder_embedding_dim, int(hparams.encoder_embedding_dim / 2), 1,
                            batch_first=True, bidirectional=True)

    def _run(self, x, lengths):
        emb = x.transpose(1, 2)                      # (B, T, 512) -- contiguous when x came from the embedding
        if _wants_grad(self, x):
            named = [("encoder." + k, p_) for k, p_ in self.named_parameters()]
            return _EncoderFn.apply(self, [n for n, _ in named], None, emb, lengths, self.training,
                                    *[p_ for _, p_ in named]).to(x.dtype)
        eng = self._t2_engine()
        out = eng.encoder(embedded=emb.detach(), lengths=lengths, training=self.training, keep=current_masks()["enc"])
        return out.to(x.dtype)

    def forward(self, x, input_lengths):
        """x (B, 512, T) embedded text, input_lengths sorted descending (pack_padded_sequence
        semantics, model.py:180-188) -> (B, T, 512)."""
        return self._run(x, input_lengths)

    def inference(self, x, input_lengths=None):
        """x (B, 512, T) embedded text -> (B, T, 512).  input_lengths (B,) integers in 1..T, any order: row b is encoded
        as x[b:b+1, :, :input_lengths[b]] alone, bit for bit (the columns past it are ignored), and its memory past
        input_lengths[b] is zero, as pad_packed_sequence leaves it."""
        if input_lengths is None:
            return self._run(x, None)
        lengths, _ = _engine_mod.row_lengths(input_lengths, x.size(0), x.size(2), "input_lengths", self._t2_device())
        _require_no_grad_with_lengths(self, "Encoder.inference")
        eng = self._t2_engine()
        out = eng.encoder(embedded=x.transpose(1, 2).detach(), lengths=lengths, training=False, per_row=True)
        return out.to(x.dtype)


class Decoder(_EngineOwner, nn.Module):
    """model.py:204-454."""
    _t2_prefix = "decoder."

    def __init__(self, hparams):
        super(Decoder, self).__init__()
        self.__dict__["_t2_hparams"] = hparams
        self.n_mel_channels = hparams.n_mel_channels
        self.n_frames_per_step = hparams.n_frames_per_step
        self.encoder_embedding_dim = hparams.encoder_embedding_dim
        self.attention_rnn_dim = hparams.attention_rnn_dim
        self.decoder_rnn_dim = hparams.decoder_rnn_dim
        self.prenet_dim = hparams.prenet_dim
        self.max_decoder_steps = hparams.max_decoder_steps
        self.gate_threshold = hparams.gate_threshold
        self.p_attention_dropout = hparams.p_attention_dropout
        self.p_decoder_dropout = hparams.p_decoder_dropout

        self.prenet = Prenet(hparams.n_mel_channels * hparams.n_frames_per_step,
                             [hparams.prenet_dim, hparams.prenet_dim])
        self.attention_rnn = nn.LSTMCell(hparams.prenet_dim + hparams.encoder_embedding_dim,
                                         hparams.attention_rnn_dim)
        self.attention_layer = Attention(hparams.attention_rnn_dim, hparams.encoder_embedding_dim,
                                         hparams.attention_dim, hparams.attention_location_n_filters,
                                         hparams.attention_location_kernel_size)
        self.decoder_rnn = nn.LSTMCell(hparams.attention_rnn_dim + hparams.encoder_embedding_dim,
                                       hparams.decoder_rnn_dim, 1)
        self.linear_projection = LinearNorm(hparams.decoder_rnn_dim + hparams.encoder_embedding_dim,
                                            hparams.n_mel_channels * hparams.n_frames_per_step)
        self.gate_layer = LinearNorm(hparams.decoder_rnn_dim + hparams.encoder_embedding_dim, 1,
                                     bias=True, w_init_gain='sigmoid')
        self.mel_lengths = None        # (B,) int32 after inference(): frames per row (stop latch)
        self._t2_link()

    def _t2_children(self):
        return (self.prenet, self.attention_layer, self.attention_layer.location_layer)

    def get_go_frame(self, memory):
        """model.py:243-256."""
        return memory.new_zeros(memory.size(0), self.n_mel_channels * self.n_frames_per_step)

    def parse_decoder_inputs(self, decoder_inputs):
        """model.py:291-309: (B, n_mel, T_out) -> (T_out, B, n_mel)."""
        decoder_inputs = decoder_inputs.transpose(1, 2)
        decoder_inputs = decoder_inputs.view(decoder_inputs.size(0),
                                             int(decoder_inputs.size(1) / self.n_frames_per_step), -1)
        return decoder_inputs.transpose(0, 1)

    def parse_decoder_outputs(self, mel_outputs, gate_outputs, alignments):
        """model.py:311-338: lists of per-step (B, n_mel), (B, 1) / (B,), (B, T_enc) -> mel (B, n_mel, T_out), gate
        (B, T_out[, 1]), alignments (B, T_out, T_enc)."""
        alignments = torch.stack(alignments).transpose(0, 1)
        gate_outputs = torch.stack(gate_outputs).transpose(0, 1)
        gate_outputs = gate_outputs.contiguous()
        mel_outputs = torch.stack(mel_outputs).transpose(0, 1).contiguous()
        mel_outputs = mel_outputs.view(mel_outputs.size(0), -1, self.n_mel_channels)
        mel_outputs = mel_outputs.transpose(1, 2)
        return mel_outputs, gate_outputs, alignments

    # -- the step API: the reference's own decoder loop, one library call per step (README "custom decoder loops") ----
    _STATE = ("attention_hidden", "attention_cell", "decoder_hidden", "decoder_cell", "attention_weights",
              "attention_weights_cum", "attention_context")

    def initialize_decoder_states(self, memory, mask):
        """model.py:258-289: the seven recurrent states as zeros of the reference's shapes in memory's dtype, memory,
        processed_memory = memory_layer(memory) (on the engine) and mask (None, or bool (B, T_enc), True at padded
        positions).  T_enc is at most 1282 (the stepwise attention kernel's limit)."""
        what = "Decoder.initialize_decoder_states"
        _require_no_grad(self, what, _STEP_NO_GRAD)
        dev = self._t2_device()
        if not torch.is_tensor(memory) or memory.dim() != 3:
            raise ValueError("tacotron2_b200: %s: memory must be a (B, T_enc, %d) tensor" % (what, self.encoder_embedding_dim))
        B, T = int(memory.shape[0]), int(memory.shape[1])
        if B < 1 or T < 1:
            raise ValueError("tacotron2_b200: %s: memory must not be empty (got %s)" % (what, tuple(memory.shape)))
        _step_tensor(memory, "memory", (B, T, self.encoder_embedding_dim), dev, what)
        _step_t_enc(T, what)
        _step_mask(mask, B, T, dev, what)
        eng = self._t2_engine()
        z = dict(device=memory.device, dtype=memory.dtype)
        self.attention_hidden = torch.zeros(B, self.attention_rnn_dim, **z)
        self.attention_cell = torch.zeros(B, self.attention_rnn_dim, **z)
        self.decoder_hidden = torch.zeros(B, self.decoder_rnn_dim, **z)
        self.decoder_cell = torch.zeros(B, self.decoder_rnn_dim, **z)
        self.attention_weights = torch.zeros(B, T, **z)
        self.attention_weights_cum = torch.zeros(B, T, **z)
        self.attention_context = torch.zeros(B, self.encoder_embedding_dim, **z)
        self.memory = memory
        self.processed_memory = eng.processed_memory(_f32(memory)).to(memory.dtype)
        self.mask = mask

    def decode(self, decoder_input):
        """model.py:340-379: one decoder step on the states the attributes hold at the call.  decoder_input (B, 256) is
        the prenet output.  Returns (decoder_output (B, n_mel), gate_prediction (B, 1), attention_weights (B, T_enc)) in
        memory's dtype.  As in the reference the six other states get new tensors, attention_weights_cum is updated in
        place and the returned weights are the new attention_weights; nothing returned or stored by one call is changed
        by the next.  Training mode applies the attention / decoder dropout with keys from a seed drawn per call
        (injected att / dec masks of one step, (B, 1024), take precedence); score_mask_value is read at every call."""
        what = "Decoder.decode"
        _require_no_grad(self, what, _STEP_NO_GRAD)
        memory = self.__dict__.get("memory")
        if memory is None:
            raise RuntimeError("tacotron2_b200: %s: call initialize_decoder_states(memory, mask) first" % what)
        dev = self._t2_device()
        B, T = int(memory.shape[0]), int(memory.shape[1])
        _step_tensor(memory, "memory", (B, T, self.encoder_embedding_dim), dev, what)
        _step_t_enc(T, what)
        _step_tensor(decoder_input, "decoder_input", (B, self.prenet_dim), dev, what)
        shapes = dict(attention_hidden=(B, self.attention_rnn_dim), attention_cell=(B, self.attention_rnn_dim),
                      decoder_hidden=(B, self.decoder_rnn_dim), decoder_cell=(B, self.decoder_rnn_dim),
                      attention_weights=(B, T), attention_weights_cum=(B, T),
                      attention_context=(B, self.encoder_embedding_dim))
        st = {k: _step_tensor(self.__dict__.get(k), k, shapes[k], dev, what) for k in self._STATE}
        pm = _step_tensor(self.__dict__.get("processed_memory"), "processed_memory",
                          (B, T, self.attention_layer.memory_layer.linear_layer.out_features), dev, what)
        mask = _step_mask(self.__dict__.get("mask"), B, T, dev, what)
        keys = dict(att=None, dec=None)
        seed = 0
        if self.training:
            masks = current_masks()
            for k, n in (("att", self.attention_rnn_dim), ("dec", self.decoder_rnn_dim)):
                if masks[k] is not None:
                    keys[k] = _engine_mod._u8(masks[k], dev).reshape(-1)
                    if keys[k].numel() != B * n:
                        raise ValueError("tacotron2_b200: %s: injected %s masks must hold one step, (B, %d) (got %s)"
                                         % (what, k, n, tuple(masks[k].shape)))
            seed = next_seed()
        eng = self._t2_engine()
        # the six states that get new tensors, copied into one fresh fp32 buffer the step updates in place
        new = ("attention_hidden", "attention_cell", "decoder_hidden", "decoder_cell", "attention_context",
               "attention_weights")
        buf = torch.cat([st[k].detach().reshape(-1) for k in new]).to(torch.float32)
        views, off = {}, 0
        for k in new:
            n = shapes[k][0] * shapes[k][1]
            views[k] = buf[off:off + n].view(shapes[k])
            off += n
        cum = st["attention_weights_cum"]
        cum32 = cum if (cum.dtype == torch.float32 and cum.is_contiguous()) else _f32(cum)
        mel, gate = eng.decoder_step(
            _f32(memory), _f32(pm), mask,
            [views[k] for k in ("attention_hidden", "attention_cell", "decoder_hidden", "decoder_cell",
                                "attention_weights")] + [cum32, views["attention_context"]],
            _f32(decoder_input), self.training, keys["att"], keys["dec"], seed, float(self.attention_layer.score_mask_value))
        if cum32 is not cum:
            with torch.no_grad():
                cum.copy_(cum32)
        dt = memory.dtype
        for k in new:
            setattr(self, k, views[k] if dt == torch.float32 else views[k].to(dt))
        return mel.to(dt), gate.to(dt), self.attention_weights

    def _teacher_forward(self, memory, decoder_inputs, memory_lengths, keep_stash):
        """Shared by the no-grad path and _DecoderFn.forward.  Returns (mel (B,T,80), gate, align, saved)."""
        eng = self._t2_engine()
        masks = current_masks()
        go = self.get_go_frame(memory).unsqueeze(0)
        frames = torch.cat((go.float(), self.parse_decoder_inputs(decoder_inputs).float()), dim=0)   # (T+1, B, 80)
        T_mel = frames.size(0) - 1
        pk = masks["prenet"]
        if pk is not None:
            pk = pk.permute(1, 0, 2, 3).reshape(2, -1, pk.shape[-1])
        frames2d = frames.reshape(-1, frames.size(-1))
        pre_seed, dec_seed = next_seed(), next_seed()
        px = eng.prenet(frames2d, pk, seed=pre_seed)                                                 # model.py:399
        smv = float(self.attention_layer.score_mask_value)
        mem32 = memory.detach().to(dtype=torch.float32).contiguous()
        stash = eng.decoder_stash(mem32.size(0), mem32.size(1), T_mel) if keep_stash else None
        mel, gate, align, _, _ = eng.decoder(
            mem32, _capi.MODE_TEACHER, T_mel, memory_lengths=memory_lengths, teacher_prenet=px,
            training=self.training, att_keep=masks["att"], dec_keep=masks["dec"], score_mask_value=smv,
            stash=stash, seed=dec_seed)
        saved = dict(eng=eng, memory=mem32, memory_lengths=memory_lengths, frames=frames2d, pk=pk, px=px, align=align,
                     stash=stash, pre_seed=pre_seed, dec_seed=dec_seed, training=self.training, att_keep=masks["att"],
                     dec_keep=masks["dec"], smv=smv)
        return mel, gate, align, saved

    def forward(self, memory, decoder_inputs, memory_lengths):
        """Teacher-forced pass (model.py:381-416).  Returns mel (B, n_mel, T), gate (B, T),
        alignments (B, T, T_enc).  Under autograd the backward pass is libt2b200's hand-written reverse
        recurrence (t2_decoder_backward / t2_prenet_backward)."""
        dt = memory.dtype
        params = [p_ for p_ in self.parameters()]
        if torch.is_grad_enabled() and (memory.requires_grad or any(p_.requires_grad for p_ in params)):
            mel, gate, align = _DecoderFn.apply(self, memory, decoder_inputs, memory_lengths, *params)
        else:
            mel, gate, align, _ = self._teacher_forward(memory, decoder_inputs, memory_lengths, False)
        return mel.transpose(1, 2).to(dt), gate.to(dt), align.to(dt)

    def _warn_max_steps(self, lengths, gate, n, caps):
        """model.py:445-447 after a free run of n steps: the warning, once, if a row stopped at its step limit without its
        gate firing at that step.  Without caps the limit is max_decoder_steps (the reference's B = 1 rule over the whole
        batch); with caps (B,) it is each row's own, so row b warns as its own B = 1 call would."""
        if caps is None:
            if n != self.max_decoder_steps or not bool((lengths >= n).any()):
                return
            fired = torch.sigmoid(gate[:, n - 1]) > self.gate_threshold
            if not bool(fired.all()):
                print("Warning! Reached max decoder steps")                                         # model.py:446
            return
        fired = torch.sigmoid(gate.gather(1, caps.long()[:, None] - 1)[:, 0]) > self.gate_threshold
        if bool(((lengths == caps) & ~fired).any()):
            print("Warning! Reached max decoder steps")                                             # model.py:446

    def inference(self, memory, memory_lengths=None, seeds=None, alignments=None, alignment_lengths=None,
                  attention_window=None, max_decoder_steps=None):
        """Free-running pass (model.py:418-454), batched: per-row stop latch, see README "batched
        inference".  Returns mel (B, n_mel, T), gate (B, T, 1), alignments (B, T, T_enc); T = steps
        until every row has fired (or max_decoder_steps); ``self.mel_lengths`` holds per-row lengths.  In training mode
        the attention / decoder hidden states take their dropout as in the reference's decode() (model.py:355-356,
        370-371); injected att / dec masks are (max_decoder_steps, B, 1024).  memory_lengths (B,) integers in 1..T_enc,
        any order: row b attends to memory[b, :memory_lengths[b]] only and its outputs equal those of a call on that
        slice alone, bit for bit; its alignments past memory_lengths[b] are zero.  seeds: B integers in [0, 2**64) (list,
        host or device tensor), eval mode only: row b draws the prenet dropout of a B = 1 call seeded seeds[b], so its
        outputs equal that call's bit for bit in any batch.

        alignments (B, T_map, T_enc), any float dtype (read as fp32), on the model's device, eval mode only: a forced run
        (Mellotron's inference_noattention).  Row b runs alignment_lengths[b] steps (B integers in 1..T_map; default
        T_map) and at step t takes the context sum_j alignments[b, t, j] memory[b, j] over j < memory_lengths[b], with
        the weights as given; its gate is computed but stops nothing, and max_decoder_steps plays no part.  The returned
        alignments are the weights used (zero past memory_lengths[b] and past the row's steps); injected prenet masks
        are (T_map, 2, B, 256).  Row b equals its own B = 1 forced call bit for bit, and a seeded free run fed its own
        alignments and mel_lengths comes out again bit for bit.

        attention_window (back, front), integers with back >= 0 and front >= 1 (README "robust synthesis"; also in
        training mode): at step t row b may only attend to [p - back, p + front) within its length, p being the first
        position of its largest attention weight of step t - 1 (0 at step 0); the energies outside get score_mask_value
        before the softmax, so those weights are exactly 0.  Everything else is the free run's.  max_decoder_steps: one
        integer or B integers >= 1 (list, host or device tensor): row b stops at its first gate firing or after
        max_decoder_steps[b] steps, whichever comes first, and the run ends when every row has stopped (injected masks are
        (max of them, 2, B, 256)); None: self.max_decoder_steps for every row.  Row b equals bit for bit its own B = 1
        call with self.max_decoder_steps = max_decoder_steps[b] and the same window.  Neither goes with alignments."""
        opts = self._options("Decoder.inference", memory, "memory_lengths", memory_lengths, seeds, alignments,
                             alignment_lengths, attention_window, max_decoder_steps)
        return self._inference(memory, opts)

    def _options(self, what, x, lengths_name, lengths, seeds, alignments, alignment_lengths, attention_window,
                 max_decoder_steps):
        """The options of an inference call over x (B, T_enc, ...) checked once, in the engine's form."""
        return _engine_mod.inference_options(
            what, x.size(0), x.size(1), self._t2_device(), training=self.training,
            prenet_masks=current_masks()["prenet"] is not None, lengths=lengths, lengths_name=lengths_name, seeds=seeds,
            alignments=alignments, alignment_lengths=alignment_lengths, attention_window=attention_window,
            max_decoder_steps=max_decoder_steps)

    def _inference(self, memory, opts):
        """inference() with its options already in the engine's form (an _engine.InferenceOptions)."""
        eng = self._t2_engine()
        masks = current_masks()
        mel, gate, align, lengths, n_steps = eng.decoder(
            memory, _capi.MODE_INFER, opts.cap or self.max_decoder_steps, training=self.training,
            prenet_keep=masks["prenet"], att_keep=masks["att"], dec_keep=masks["dec"], gate_threshold=self.gate_threshold,
            **opts.decoder_kwargs())
        n = int(n_steps.item())                      # the one host sync of the whole loop (model.py:443 syncs every step)
        self.mel_lengths = lengths
        if opts.forced_align is None:
            self._warn_max_steps(lengths, gate, n, opts.max_steps)
        dt = memory.dtype
        return (mel[:, :n].transpose(1, 2).to(dt), gate[:, :n].unsqueeze(-1).to(dt), align[:, :n].to(dt))

    def _stream_chunks(self, memory, chunk_steps, halo, opts):
        """The persistent decoder in chunks of chunk_steps steps.  Yields (t0, t1, finished, stream): frames [t0, t1) are
        the new ones that every row has produced and that no frame within `halo` steps of them can still change, i.e. all
        frames up to the steps run less `halo` while any row is live, and all of them once every 64-row slice has
        stopped.  Before the last tuple, self.mel_lengths and the max-steps warning are set as by inference().  opts: the
        run's options in the engine's form (an _engine.InferenceOptions)."""
        chunk_steps = int(chunk_steps)
        if chunk_steps < 1:
            raise ValueError("tacotron2_b200: chunk_steps must be >= 1 (got %d)" % chunk_steps)
        eng = self._t2_engine()
        st = eng.decoder_stream(memory, opts.cap or self.max_decoder_steps, prenet_keep=current_masks()["prenet"],
                                gate_threshold=self.gate_threshold, **opts.decoder_kwargs())
        t0 = 0
        while True:
            live_steps, n, finished = st.run(chunk_steps)
            t1 = n if finished else max(t0, live_steps - halo)
            if finished:
                self.mel_lengths = st.mel_lengths
                if opts.forced_align is None:                                                   # as inference()
                    self._warn_max_steps(st.mel_lengths, st.gate, n, opts.max_steps)
            if t1 > t0 or finished:
                yield t0, t1, finished, st
            if finished:
                return
            t0 = t1

    def inference_stream(self, memory, chunk_steps=32, memory_lengths=None, seeds=None, alignments=None,
                         alignment_lengths=None, attention_window=None, max_decoder_steps=None):
        """inference() in chunks of ``chunk_steps`` decoder steps, as a generator: one item per chunk that produced
        frames, a dict with ``frames`` = (t0, t1) (the same for every row), ``mel_outputs`` (B, n_mel, t1-t0),
        ``gate_outputs`` (B, t1-t0, 1), ``alignments`` (B, t1-t0, T_enc), ``mel_lengths`` (B,) int32 on the device with -1
        for rows that are still live, and ``finished``.  A decoder frame is handed out as soon as every row has produced
        it; concatenated along time the items are bit-identical to inference() (same weights, memory, memory_lengths,
        masks / seed / seeds / alignments / attention_window / max_decoder_steps).  Evaluation mode only: the resumable decoder applies no hidden-state dropout,
        which inference() does in training mode."""
        if self.training:
            raise RuntimeError("tacotron2_b200: Decoder.inference_stream needs eval mode (in training mode inference() "
                               "applies the attention / decoder dropout, which the resumable decoder does not)")
        opts = self._options("Decoder.inference_stream", memory, "memory_lengths", memory_lengths, seeds, alignments,
                             alignment_lengths, attention_window, max_decoder_steps)
        dt = memory.dtype
        for t0, t1, finished, st in self._stream_chunks(memory, chunk_steps, 0, opts):
            yield dict(frames=(t0, t1), mel_outputs=st.mel[:, t0:t1].transpose(1, 2).to(dt),
                       gate_outputs=st.gate[:, t0:t1].unsqueeze(-1).to(dt), alignments=st.align[:, t0:t1].to(dt),
                       mel_lengths=st.mel_lengths.clone(), finished=finished)


class _DecoderFn(torch.autograd.Function):
    """Decoder.forward (model.py:381-416) as one autograd node: forward = the persistent teacher-forced kernel with
    its training stash, backward = t2_decoder_backward + t2_prenet_backward."""

    @staticmethod
    def forward(ctx, dec, memory, decoder_inputs, memory_lengths, *params):
        mel, gate, align, saved = dec._teacher_forward(memory, decoder_inputs, memory_lengths, True)
        ctx.dec, ctx.saved = dec, saved
        ctx.mem_dtype = memory.dtype
        ctx.set_materialize_grads(False)
        return mel, gate, align

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_mel, d_gate, d_align):
        sv, dec = ctx.saved, ctx.dec
        eng = sv["eng"]
        align = sv["align"]
        B, T = align.shape[0], align.shape[1]
        f32 = dict(device=align.device, dtype=torch.float32)
        if d_mel is None:
            d_mel = torch.zeros(B, T, dec.n_mel_channels, **f32)
        if d_gate is None:
            d_gate = torch.zeros(B, T, **f32)
        named = [("decoder." + k, p_) for k, p_ in dec.named_parameters()]
        grads = {n: torch.empty(p_.shape, **f32) for n, p_ in named}
        d_memory, d_px = eng.decoder_backward(
            sv["memory"], sv["memory_lengths"], sv["px"], align, sv["stash"], sv["dec_seed"], sv["training"],
            sv["att_keep"], sv["dec_keep"], sv["smv"], d_mel, d_gate, d_align, grads)
        # the prenet ran over T+1 frames (model.py:396-399); the last frame's output is unused (model.py:405)
        d_out = torch.cat((d_px.reshape(-1, d_px.shape[-1]), torch.zeros(B, d_px.shape[-1], **f32)), 0)
        eng.prenet_backward(sv["frames"], sv["pk"], sv["pre_seed"], d_out, grads)
        ctx.saved = None
        return (None, d_memory.to(ctx.mem_dtype), None, None) + tuple(grads[n].to(p_.dtype) for n, p_ in named)


class Tacotron2(_EngineOwner, nn.Module):
    """model.py:457-529."""

    def __init__(self, hparams):
        super(Tacotron2, self).__init__()
        self.__dict__["_t2_hparams"] = hparams
        self.mask_padding = hparams.mask_padding
        self.fp16_run = hparams.fp16_run
        self.n_mel_channels = hparams.n_mel_channels
        self.n_frames_per_step = hparams.n_frames_per_step
        self.embedding = nn.Embedding(hparams.n_symbols, hparams.symbols_embedding_dim)
        std = sqrt(2.0 / (hparams.n_symbols + hparams.symbols_embedding_dim))
        val = sqrt(3.0) * std  # uniform bounds for std
        self.embedding.weight.data.uniform_(-val, val)
        self.encoder = Encoder(hparams)
        self.decoder = Decoder(hparams)
        self.postnet = Postnet(hparams)
        self.mel_lengths = None
        self.register_load_state_dict_post_hook(_invalidate_after_load)
        self._t2_link()

    def _t2_children(self):
        return (self.encoder, self.decoder, self.postnet, self.decoder.prenet, self.decoder.attention_layer,
                self.decoder.attention_layer.location_layer)

    def parse_batch(self, batch):
        """model.py:473-485."""
        text_padded, input_lengths, mel_padded, gate_padded, output_lengths = batch
        # the reference reads max_len back from the GPU copy (a device sync, model.py:478); the collate function hands over
        # host tensors, so take it there and let the (pinned, non_blocking) copies overlap
        max_len = torch.max(input_lengths.data).item()
        text_padded = to_gpu(text_padded).long()
        input_lengths = to_gpu(input_lengths).long()
        mel_padded = to_gpu(mel_padded).float()
        gate_padded = to_gpu(gate_padded).float()
        output_lengths = to_gpu(output_lengths).long()
        return ((text_padded, input_lengths, mel_padded, max_len, output_lengths), (mel_padded, gate_padded))

    def parse_output(self, outputs, output_lengths=None):
        """model.py:487-497: zero mel / mel_postnet and set gate to 1e3 beyond each row's length."""
        if self.mask_padding and output_lengths is not None:
            mask = ~get_mask_from_lengths(output_lengths, outputs[0].size(2))
            mask = mask.expand(self.n_mel_channels, mask.size(0), mask.size(1))
            mask = mask.permute(1, 0, 2)
            outputs[0].data.masked_fill_(mask, 0.0)
            outputs[1].data.masked_fill_(mask, 0.0)
            outputs[2].data.masked_fill_(mask[:, 0, :], 1e3)  # gate energies
        return outputs

    def forward(self, inputs):
        """model.py:499-515."""
        text_inputs, text_lengths, mels, max_len, output_lengths = inputs
        text_lengths, output_lengths = text_lengths.data, output_lengths.data
        eng = self._t2_engine()                       # (re-)packs the weights once for the whole forward pass
        self.__dict__["_t2_packed_in_call"] = True
        try:
            return self._forward_packed(eng, text_inputs, text_lengths, mels, output_lengths)
        finally:
            self.__dict__["_t2_packed_in_call"] = False

    def _forward_packed(self, eng, text_inputs, text_lengths, mels, output_lengths):
        masks = current_masks()
        grad = _wants_grad(self)
        if grad:   # embedding lookup + encoder as one node (the embedding gradient comes out of t2_encoder_backward)
            named = [("embedding.weight", self.embedding.weight)] + [("encoder." + k, p_) for k, p_ in self.encoder.named_parameters()]
            memory = _EncoderFn.apply(self, [n for n, _ in named], text_inputs, None, text_lengths, self.training,
                                      *[p_ for _, p_ in named])
        else:
            memory = eng.encoder(text=text_inputs, lengths=text_lengths, training=self.training, keep=masks["enc"])
        memory = memory.to(self._t2_out_dtype())
        mel_outputs, gate_outputs, alignments = self.decoder(memory, mels, memory_lengths=text_lengths)
        mel_btc = mel_outputs.transpose(1, 2)
        if grad:
            named = [("postnet." + k, p_) for k, p_ in self.postnet.named_parameters()]
            # parse_output below zeroes the padded frames of mel_outputs in place (model.py:492); in the reference that
            # tensor is what the first postnet conv saved for its weight gradient -> reproduce (wgrad_lengths)
            wl = output_lengths if self.mask_padding else None
            mel_outputs_postnet = _PostnetFn.apply(self, [n for n, _ in named], mel_btc, True, self.training, wl,
                                                   *[p_ for _, p_ in named]).to(mel_outputs.dtype)
        else:
            if mel_btc.dtype != torch.float32 or not mel_btc.is_contiguous():
                mel_btc = mel_btc.float().contiguous()
            mel_outputs_postnet = eng.postnet(mel_btc, None, True, self.training, masks["post"]).to(mel_outputs.dtype)
        if self.training:
            for mod in self.modules():
                if isinstance(mod, nn.BatchNorm1d) and mod.num_batches_tracked is not None:
                    mod.num_batches_tracked += 1
            # the kernels updated the BatchNorm running statistics through raw pointers (no torch version bump); the
            # BN-folded inference images must not outlive them: next call re-packs
            eng.invalidate()
        outputs = [mel_outputs, mel_outputs_postnet, gate_outputs, alignments]
        cast = self.__dict__.get("_t2_cast_outputs")     # amp.initialize(opt_level="O2"): outputs in fp32 for the loss
        if cast is not None:
            outputs = [o.to(cast) for o in outputs]
        return self.parse_output(outputs, output_lengths)

    def inference(self, inputs, input_lengths=None, seeds=None, alignments=None, alignment_lengths=None,
                  attention_window=None, max_decoder_steps=None):
        """model.py:517-529, batched.  For B > 1 frames at t >= mel_lengths[b] of mel_outputs and
        mel_outputs_postnet are zero (same convention as parse_output); ``self.mel_lengths`` holds
        the per-row lengths.  B == 1 is exactly the reference.

        input_lengths (B,) integers in 1..T_text, on the host or the device, in any order: texts of different lengths in
        one batch.  Row b then computes what ``inference(inputs[b:b+1, :input_lengths[b]])`` computes, bit for bit (its
        frames up to the batch's step count, alignments[b, :, :input_lengths[b]], mel_lengths[b]); the ids past its length
        are ignored and alignments[b, :, input_lengths[b]:] is zero.  None: every row is T_text long.

        seeds: one seed per utterance, B integers in [0, 2**64) as a list, a host tensor or a device tensor (int64 values
        are taken as their 64-bit pattern); eval mode only, not together with injected prenet masks.  Row b then draws the
        prenet dropout that ``inference(inputs[b:b+1, :input_lengths[b]], seeds=[seeds[b]])`` draws, so it reproduces that
        call bit for bit in any batch, slice, stream or server slot.  A B = 1 call with seeds=[s] is the unseeded call
        whose engine seed was s.  None: one seed per call (the next engine seed), as before.

        alignments (B, T_map, T_text), alignment_lengths (B,): a forced run with the given attention weights, eval mode
        only (README "timing control"; Decoder.inference has the contract).  Row b runs alignment_lengths[b] steps
        (default T_map), mel_lengths = alignment_lengths, and every row's postnet is its own B = 1 postnet, so row b
        equals ``inference(inputs[b:b+1, :L_b], alignments=alignments[b:b+1, :alignment_lengths[b], :L_b])`` bit for bit
        (L_b = input_lengths[b]).  ``alignments_from_durations`` turns per-symbol frame counts into such a map.

        attention_window (back, front) and max_decoder_steps (one integer or B): guards for free runs on long or
        out-of-domain text (README "robust synthesis"; Decoder.inference has the contract).  Row b then equals
        ``inference(inputs[b:b+1, :L_b], attention_window=w)`` with ``decoder.max_decoder_steps = max_decoder_steps[b]``
        bit for bit.  Neither goes with alignments."""
        opts = self.decoder._options("Tacotron2.inference", inputs, "input_lengths", input_lengths, seeds, alignments,
                                     alignment_lengths, attention_window, max_decoder_steps)
        eng = self._t2_engine()
        memory = eng.encoder(text=inputs, lengths=opts.lengths, training=self.training, keep=current_masks()["enc"],
                             per_row=opts.lengths is not None)
        memory = memory.to(self._t2_out_dtype())     # a .half() model hands half tensors between its modules (ipynb:89-90)
        mel_outputs, gate_outputs, alignments = self.decoder._inference(memory, opts)
        lengths = self.decoder.mel_lengths
        self.mel_lengths = lengths
        mel_btc = mel_outputs.transpose(1, 2)
        if mel_btc.dtype != torch.float32:
            mel_btc = mel_btc.float().contiguous()
        multi = inputs.size(0) > 1
        # a forced run knows its lengths before it runs: every row's postnet is its own, as for a ragged batch
        mel_outputs_postnet = eng.postnet(mel_btc, lengths if multi else None, True, self.training,
                                          current_masks()["post"],
                                          per_row=opts.ragged or (opts.forced_align is not None and multi)
                                          ).to(mel_outputs.dtype)
        if multi:
            pad = ~get_mask_from_lengths(lengths.long(), mel_outputs.size(2))
            mel_outputs = mel_outputs.masked_fill(pad.unsqueeze(1), 0.0)
        return self.parse_output([mel_outputs, mel_outputs_postnet, gate_outputs, alignments])

    def inference_stream(self, inputs, chunk_steps=32, input_lengths=None, seeds=None, alignments=None,
                         alignment_lengths=None, attention_window=None, max_decoder_steps=None):
        """inference() as a generator that hands out frames while the decoder runs (README "streaming inference").

        The encoder runs once; the decoder runs in chunks of ``chunk_steps`` steps.  Each item is a dict describing frames
        [t0, t1) (``frames``, the same for every row): ``mel_outputs`` and ``mel_outputs_postnet`` (B, n_mel, t1-t0),
        ``gate_outputs`` (B, t1-t0, 1), ``alignments`` (B, t1-t0, T_enc), ``mel_lengths`` (B,) int32 on the device with -1
        for rows that are still live, and ``finished``.  The postnet's five k=5 convolutions see +-10 frames, so frame t is
        handed out once the decoder has run step t+10 or every row has stopped; it is never revised.  Concatenated along
        time the items are bit-identical to inference() with the same weights, inputs and dropout masks / seed.  After the
        last item ``self.mel_lengths`` and the max-steps warning are as after inference().  input_lengths: as for
        inference(), whose output the items then concatenate to.  seeds, alignments, alignment_lengths,
        attention_window, max_decoder_steps: as for inference().  Evaluation mode only: in
        training mode BatchNorm normalises over the whole sequence, so no frame is final before the last one."""
        if self.training:
            raise RuntimeError("tacotron2_b200: inference_stream needs eval mode (training-mode BatchNorm uses the statistics "
                               "of the whole sequence, so no postnet frame is final before the decoder ends)")
        opts = self.decoder._options("Tacotron2.inference_stream", inputs, "input_lengths", input_lengths, seeds,
                                     alignments, alignment_lengths, attention_window, max_decoder_steps)
        eng = self._t2_engine()
        memory = eng.encoder(text=inputs, lengths=opts.lengths, training=False, keep=current_masks()["enc"],
                             per_row=opts.lengths is not None)
        dt = self._t2_out_dtype()
        memory = memory.to(dt)
        multi = inputs.size(0) > 1
        ragged = opts.ragged or (opts.forced_align is not None and multi)     # as inference()
        halo = POSTNET_HALO
        for t0, t1, finished, st in self.decoder._stream_chunks(memory, chunk_steps, halo, opts):
            if finished:
                self.mel_lengths = st.mel_lengths
            lengths = st.mel_lengths
            # postnet over input frames [w0, w1): its zero padding reaches only output frames outside [t0, t1)
            w0, w1 = max(0, t0 - halo), (t1 if finished else t1 + halo)
            mel_btc = st.mel[:, w0:w1]
            if dt != torch.float32:                    # inference() feeds the postnet the model-dtype mel (ipynb:89-90)
                mel_btc = mel_btc.to(dt)
            if mel_btc.dtype != torch.float32:
                mel_btc = mel_btc.float().contiguous()
            win_len = None
            if multi:                                  # frames at t >= length count as zero; live rows have none
                win_len = torch.where(lengths < 0, torch.full_like(lengths, w1 - w0), (lengths - w0).clamp(min=0))
            post = eng.postnet(mel_btc, win_len, True, False, None, per_row=ragged)[:, :, t0 - w0:t1 - w0].to(dt)
            mel_outputs = st.mel[:, t0:t1].transpose(1, 2).to(dt)
            if multi:
                t = torch.arange(t0, t1, device=lengths.device)
                pad = (lengths[:, None] >= 0) & (t[None, :] >= lengths[:, None])
                mel_outputs = mel_outputs.masked_fill(pad.unsqueeze(1), 0.0)
            yield dict(frames=(t0, t1), mel_outputs=mel_outputs, mel_outputs_postnet=post,
                       gate_outputs=st.gate[:, t0:t1].unsqueeze(-1).to(dt), alignments=st.align[:, t0:t1].to(dt),
                       mel_lengths=lengths.clone(), finished=finished)

    def inference_server(self, slots=64, max_text_len=200, chunk_steps=32, seed=None, attention_window=None):
        """Continuous batching (README "serving a queue"): an ``InferenceServer`` that keeps ``slots`` decoder rows in
        flight and refills a row with the next queued text as soon as its request has stopped.

            server = model.inference_server(slots=64, max_text_len=200, chunk_steps=32)
            rid = server.submit(text_ids, max_decoder_steps=None)      # 1-D integer tensor of 1..max_text_len ids
            for result in server.run(): ...                            # or server.step(), one chunk at a time

        A result is a dict: ``id``, ``mel_outputs`` / ``mel_outputs_postnet`` (1, n_mel, L), ``gate_outputs`` (1, L, 1),
        ``alignments`` (1, L, T_text), ``mel_length`` and ``hit_max_steps`` -- the names and shapes inference() returns for
        that text alone.  With injected prenet masks it equals that call bit for bit (serving.py).  Evaluation mode and the
        persistent decoder only, as inference_stream.  The server owns its decoder state: several servers, streams and
        inference() calls can be alive on one model.  seed: the session's Philox seed (default: the next engine seed).
        attention_window: (back, front) for every request of the server, as for inference(); a result then equals
        ``inference(text[None], attention_window=attention_window)`` under its own limit."""
        from .serving import EngineBackend, InferenceServer
        if self.training:
            raise RuntimeError("tacotron2_b200: inference_server needs eval mode (training-mode BatchNorm uses the statistics "
                               "of the whole sequence, so no postnet frame is final before the decoder ends)")
        window = _engine_mod.inference_options("inference_server", 1, 1, torch.device("cpu"),
                                               attention_window=attention_window).window
        server = InferenceServer(None, slots, max_text_len, chunk_steps, self.decoder.max_decoder_steps)
        server.backend = EngineBackend(self, server.slots, server.max_text_len, server.chunk_steps, seed, window)
        return server

    def inference_many(self, texts, slots=64, max_text_len=None, chunk_steps=32, max_decoder_steps=None, seeds=None,
                       attention_window=None):
        """Every text of ``texts`` (1-D integer tensors) through an inference_server; returns the results in input order.
        max_text_len: default the longest text; max_decoder_steps: one limit for all, or one per text.  seeds: one per text
        (as for inference()); result i then equals ``inference(texts[i][None], seeds=[seeds[i]])`` bit for bit.
        attention_window: one window for every text (see inference_server)."""
        texts = list(texts)
        opts = _engine_mod.inference_options("inference_many", len(texts), 1, torch.device("cpu"), seeds=seeds,
                                             attention_window=attention_window)
        if not texts:
            return []
        if max_text_len is None:
            max_text_len = max(int(torch.as_tensor(t).numel()) for t in texts)
        limits = max_decoder_steps if isinstance(max_decoder_steps, (list, tuple)) else [max_decoder_steps] * len(texts)
        per_text = [None] * len(texts)
        if opts.row_seeds is not None:      # the server takes each as a Python int
            per_text = [int(v) & 0xFFFFFFFFFFFFFFFF for v in opts.row_seeds.tolist()]
        server = self.inference_server(min(int(slots), len(texts)), max(1, max_text_len), chunk_steps,
                                       attention_window=opts.window)
        ids = [server.submit(t, limit, seed=sd) for t, limit, sd in zip(texts, limits, per_text)]
        results = {r["id"]: r for r in server.run()}
        return [results[i] for i in ids]


POSTNET_HALO = 10     # frames each side a postnet output depends on: 5 convolutions with k = 5 (model.py:103-146)
