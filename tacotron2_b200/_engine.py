"""Host-side glue between the nn.Module boundary and libt2b200.so: weight table, handle cache,
workspaces, dropout-mask injection.  All arithmetic happens in the shared library."""
import contextlib
import ctypes as C
import threading

import torch

from . import _capi


def weight_table_spec(hp):
    """(name, shape) of the 84 state_dict entries in the reference's order (SURVEY.md 8(b1))."""
    E, K = hp.encoder_embedding_dim, hp.encoder_kernel_size
    s = [("embedding.weight", (hp.n_symbols, hp.symbols_embedding_dim))]

    def bn(p, c):
        return [(p + "weight", (c,)), (p + "bias", (c,)), (p + "running_mean", (c,)),
                (p + "running_var", (c,)), (p + "num_batches_tracked", ())]
    for i in range(hp.encoder_n_convolutions):
        p = "encoder.convolutions.%d." % i
        s += [(p + "0.conv.weight", (E, E, K)), (p + "0.conv.bias", (E,))] + bn(p + "1.", E)
    H = E // 2
    for suf in ("", "_reverse"):
        s += [("encoder.lstm.weight_ih_l0" + suf, (4 * H, E)), ("encoder.lstm.weight_hh_l0" + suf, (4 * H, H)),
              ("encoder.lstm.bias_ih_l0" + suf, (4 * H,)), ("encoder.lstm.bias_hh_l0" + suf, (4 * H,))]
    d = "decoder."
    nm = hp.n_mel_channels * hp.n_frames_per_step
    A, D, P = hp.attention_rnn_dim, hp.decoder_rnn_dim, hp.prenet_dim
    s += [(d + "prenet.layers.0.linear_layer.weight", (P, nm)), (d + "prenet.layers.1.linear_layer.weight", (P, P)),
          (d + "attention_rnn.weight_ih", (4 * A, P + E)), (d + "attention_rnn.weight_hh", (4 * A, A)),
          (d + "attention_rnn.bias_ih", (4 * A,)), (d + "attention_rnn.bias_hh", (4 * A,))]
    a = d + "attention_layer."
    s += [(a + "query_layer.linear_layer.weight", (hp.attention_dim, A)),
          (a + "memory_layer.linear_layer.weight", (hp.attention_dim, E)),
          (a + "v.linear_layer.weight", (1, hp.attention_dim)),
          (a + "location_layer.location_conv.conv.weight",
           (hp.attention_location_n_filters, 2, hp.attention_location_kernel_size)),
          (a + "location_layer.location_dense.linear_layer.weight", (hp.attention_dim, hp.attention_location_n_filters))]
    s += [(d + "decoder_rnn.weight_ih", (4 * D, A + E)), (d + "decoder_rnn.weight_hh", (4 * D, D)),
          (d + "decoder_rnn.bias_ih", (4 * D,)), (d + "decoder_rnn.bias_hh", (4 * D,)),
          (d + "linear_projection.linear_layer.weight", (nm, D + E)), (d + "linear_projection.linear_layer.bias", (nm,)),
          (d + "gate_layer.linear_layer.weight", (1, D + E)), (d + "gate_layer.linear_layer.bias", (1,))]
    PD, PK, n = hp.postnet_embedding_dim, hp.postnet_kernel_size, hp.postnet_n_convolutions
    for i in range(n):
        ci = hp.n_mel_channels if i == 0 else PD
        co = hp.n_mel_channels if i == n - 1 else PD
        p = "postnet.convolutions.%d." % i
        s += [(p + "0.conv.weight", (co, ci, PK)), (p + "0.conv.bias", (co,))] + bn(p + "1.", co)
    return s


# ---- dropout mask injection (parity tests feed the SAME Bernoulli masks to oracle and engine) ----
_tls = threading.local()


@contextlib.contextmanager
def dropout_masks(prenet=None, att=None, dec=None, enc=None, post=None):
    """uint8 keep masks (1 = keep).  prenet: (steps, 2, B, 256) [Decoder.forward: steps = T_mel+1];
    att / dec: (T_mel, B, 1024) [training-mode inference: (max_decoder_steps, B, 1024)]; enc: (3, B, 512, T_text); post: list/tuple of 5 masks in the
    reference layout [(B,512,T)]*4 + [(B,80,T)] (training only).  None => in-kernel Philox."""
    prev = getattr(_tls, "masks", None)
    _tls.masks = dict(prenet=prenet, att=att, dec=dec, enc=enc, post=post)
    try:
        yield
    finally:
        _tls.masks = prev


def current_masks():
    return getattr(_tls, "masks", None) or dict(prenet=None, att=None, dec=None, enc=None, post=None)


# Bumped by code that updates parameters in place without going through torch (the fused optimizer): part of the
# handle-cache key, so the packed device-side copies are rebuilt.
_weights_generation = [0]


def bump_weights_generation():
    _weights_generation[0] += 1


def invalidate_weights():
    """Public: every engine re-packs its device-side weight copies on its next call (use after in-place parameter writes
    that bypass torch's version counter, e.g. ``p.data.copy_()`` for EMA / SWA / weight surgery)."""
    bump_weights_generation()


_seed_counter = [0]


def next_seed():
    """Philox seed for one engine call: torch's global seed + a call counter."""
    _seed_counter[0] += 1
    return (torch.initial_seed() * 1000003 + _seed_counter[0]) & 0xFFFFFFFFFFFFFFFF


def _i32(x, device):
    """Per-row lengths as contiguous int32 on the device (None stays None)."""
    return None if x is None else x.to(device=device, dtype=torch.int32).contiguous()


def _u8(mask, device):
    """A keep mask as contiguous uint8 on the device; a list / tuple of masks is concatenated flat, in order."""
    if mask is None:
        return None
    if isinstance(mask, (list, tuple)):
        mask = torch.cat([k.to(torch.uint8).reshape(-1) for k in mask])
    return mask.to(device=device, dtype=torch.uint8).contiguous()


def _ptr(t):
    return None if t is None else t.data_ptr()


def _source(text, embedded, device):
    """The encoder's input on the device: (text int64, None) or (None, embedded fp32)."""
    if text is not None:
        return text.to(device=device, dtype=torch.int64).contiguous(), None
    return None, embedded.to(device=device, dtype=torch.float32).contiguous()


class _Handle:
    """One library object (t2_<kind>_create / _refresh / _destroy) holding packed copies of a module's tensors on one
    device, and its cached workspaces.  The copies are keyed on the global weights generation and each tensor's pointer,
    torch version counter and dtype: the first call creates the object, a call with another key refreshes it, and one on
    another device, or with other `extra` key parts, replaces it.  Subclasses supply ``_pack`` and ``_config``."""

    kind = what = None      # the library object; the module named in the error for a module that is not on a GPU

    def __init__(self):
        self.handle = self.key = self.held = self.device = self.extra = None
        self._ws = _capi.Workspace()

    def invalidate(self):
        """Forget the cache key: the next call re-packs every device-side copy from the live tensors."""
        self.key = None

    def _ensure(self, dev, tensors, extra=(), force=False):
        """tensors: the module's tensors in table order (None: absent); extra: key parts the object is created with."""
        if dev is None or dev.type != "cuda":
            raise RuntimeError("%s must live on a CUDA device (H100); there is no CPU path -- call .cuda() first" % self.what)
        key = (_weights_generation[0],) + tuple(extra) + tuple(
            None if t is None else (t.data_ptr(), t._version, t.dtype) for t in tensors)
        if self.handle is not None and key == self.key and dev == self.device and not force:
            return
        held, args = self._pack(tensors, dev, *extra)
        L = _capi.lib()
        if self.handle is None or (dev, extra) != (self.device, self.extra):
            self.close()
            cfg, h = self._config(*extra), C.c_void_p()
            _capi.call(getattr(L, "t2_%s_create" % self.kind), dev, C.byref(h), C.byref(cfg), *args)
            self.handle = h
        else:
            _capi.call(getattr(L, "t2_%s_refresh" % self.kind), dev, self.handle, *args)
        self.key, self.held, self.device, self.extra = key, held, dev, extra

    def close(self):
        if self.handle is not None:
            getattr(_capi.lib(), "t2_%s_destroy" % self.kind)(self.handle)
            self.handle = self.key = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _call(self, fn, *args):
        """A library entry point on this object (the handle goes first, the stream last)."""
        _capi.call(fn, self.device, self.handle, *args)


class Engine(_Handle):
    """One T2Model handle (packed weights on one device) + cached workspaces."""

    kind, what = "model", "tacotron2_b200: the model"

    def __init__(self, hp):
        super().__init__()
        self.hp = hp
        self.spec = weight_table_spec(hp)
        self.impl = _capi.IMPL_AUTO

    # -- weights ---------------------------------------------------------------------------------
    def ensure(self, named, force=False):
        """named: dict full-name -> tensor (missing entries are replaced by zeros).  The packed copies are rebuilt when the
        key (global generation, per-tensor pointer / torch version counter / dtype) changed or when `force` is set.
        Writes through ``.data`` do not move torch's version counter: callers doing that use
        ``model.invalidate_weights()`` / ``tacotron2_b200.invalidate_weights()``."""
        dev = next((t.device for t in named.values() if t.is_cuda), None)
        self._ensure(dev, [named.get(n) for n, _ in self.spec], force=force)

    def _pack(self, tensors, dev):
        held, ptrs = [], (C.c_void_p * _capi.T2_NUM_WEIGHTS)()
        for i, ((n, shape), t) in enumerate(zip(self.spec, tensors)):
            if n.endswith("num_batches_tracked"):
                continue
            if t is None:
                t = torch.zeros(shape, device=dev, dtype=torch.float32)
                if n.endswith("running_var"):
                    t.fill_(1.0)
            else:
                if tuple(t.shape) != tuple(shape):
                    raise RuntimeError("tacotron2_b200: %s has shape %s, expected %s" % (n, tuple(t.shape), shape))
                t = t.detach()
                if t.dtype != torch.float32 or not t.is_contiguous():
                    t = t.float().contiguous()
            held.append(t)
            ptrs[i] = t.data_ptr()
        return held, (ptrs, _capi.T2_NUM_WEIGHTS)

    def _config(self):
        hp = self.hp
        if hp.n_frames_per_step != 1:
            raise RuntimeError("n_frames_per_step != 1 is not supported (hparams.py:56)")
        return _capi.T2Config(
            hp.n_mel_channels, hp.n_symbols, hp.symbols_embedding_dim, hp.encoder_kernel_size,
            hp.encoder_n_convolutions, hp.encoder_embedding_dim, hp.attention_rnn_dim,
            hp.decoder_rnn_dim, hp.prenet_dim, hp.attention_dim, hp.attention_location_n_filters,
            hp.attention_location_kernel_size, hp.postnet_embedding_dim, hp.postnet_kernel_size,
            hp.postnet_n_convolutions, hp.p_attention_dropout, hp.p_decoder_dropout, 1e-5)

    def _workspace(self, tag, nbytes):
        return self._ws.get(tag, nbytes, self.device)

    # -- encoder ---------------------------------------------------------------------------------
    def encoder(self, text=None, embedded=None, lengths=None, training=False, keep=None, stash=None, seed=None,
                per_row=False):
        """per_row: t2_encoder_infer -- row b is encoded as its first lengths[b] positions alone (lengths in any order);
        otherwise lengths has Encoder.forward's packed-sequence meaning (t2_encoder_forward)."""
        L = _capi.lib()
        text, embedded = _source(text, embedded, self.device)
        src = text if text is not None else embedded
        B, T = int(src.shape[0]), int(src.shape[1])
        memory = torch.empty(B, T, self.hp.encoder_embedding_dim, device=self.device, dtype=torch.float32)
        ws = self._workspace("enc", L.t2_encoder_workspace_bytes(self.handle, B, T))
        len32, keep = _i32(lengths, self.device), _u8(keep, self.device)
        a = _capi.T2EncoderArgs(_ptr(text), _ptr(embedded), _ptr(len32), B, T, int(bool(training)), _ptr(keep),
                                next_seed() if seed is None else seed, memory.data_ptr(), ws.data_ptr(), ws.numel(),
                                _ptr(stash), 0 if stash is None else stash.numel())
        self._call(L.t2_encoder_infer if per_row else L.t2_encoder_forward, C.byref(a))
        return memory

    def stash_buffer(self, kind, *dims):
        return _capi.byte_buffer(getattr(_capi.lib(), "t2_%s_stash_bytes" % kind)(self.handle, *dims), self.device)

    def encoder_backward(self, text, embedded, lengths, training, keep, seed, stash, d_memory, want_d_embedded, named_grads):
        L = _capi.lib()
        B, T = int(d_memory.shape[0]), int(d_memory.shape[1])
        f32 = dict(device=self.device, dtype=torch.float32)
        text, embedded = _source(text, embedded, self.device)
        len32, keep = _i32(lengths, self.device), _u8(keep, self.device)
        d_memory = d_memory.to(**f32).contiguous()
        d_emb = torch.empty(B, T, self.hp.encoder_embedding_dim, **f32) if want_d_embedded else None
        ws = self._workspace("enc_bwd", L.t2_encoder_backward_workspace_bytes(self.handle, B, T))
        a = _capi.T2EncoderBwdArgs(_ptr(text), _ptr(embedded), _ptr(len32), B, T, int(bool(training)), _ptr(keep), seed,
                                   stash.data_ptr(), stash.numel(), d_memory.data_ptr(), _ptr(d_emb),
                                   self.grad_table(named_grads), _capi.T2_NUM_WEIGHTS, ws.data_ptr(), ws.numel())
        self._call(L.t2_encoder_backward, C.byref(a))
        return d_emb

    def postnet_backward(self, B, T, training, add_residual, keep, seed, stash, d_mel_post, named_grads, wgrad_lengths=None):
        """d_mel_post (B, 80, T) -> d_mel (B, T, 80)."""
        L = _capi.lib()
        f32 = dict(device=self.device, dtype=torch.float32)
        keep, wl32 = _u8(keep, self.device), _i32(wgrad_lengths, self.device)
        d_mel_post = d_mel_post.to(**f32).contiguous()
        d_mel = torch.empty(B, T, self.hp.n_mel_channels, **f32)
        ws = self._workspace("post_bwd", L.t2_postnet_backward_workspace_bytes(self.handle, B, T))
        a = _capi.T2PostnetBwdArgs(B, T, int(bool(training)), int(bool(add_residual)), _ptr(keep), seed, _ptr(wl32),
                                   stash.data_ptr(), stash.numel(), d_mel_post.data_ptr(), d_mel.data_ptr(),
                                   self.grad_table(named_grads), _capi.T2_NUM_WEIGHTS, ws.data_ptr(), ws.numel())
        self._call(L.t2_postnet_backward, C.byref(a))
        return d_mel

    # -- decoder ---------------------------------------------------------------------------------
    def decoder(self, memory, mode, n_steps_cap, memory_lengths=None, teacher_prenet=None, training=False,
                prenet_keep=None, att_keep=None, dec_keep=None, gate_threshold=0.5,
                score_mask_value=-float("inf"), impl=None, stash=None, seed=None):
        L = _capi.lib()
        memory = memory.to(device=self.device, dtype=torch.float32).contiguous()
        B, T = int(memory.shape[0]), int(memory.shape[1])
        cap = int(n_steps_cap)
        # zero-initialised: batches of more than 64 rows run as independent 64-row launches that may stop at
        # different steps; frames past a launch's last step stay zero
        mel = torch.zeros(B, cap, self.hp.n_mel_channels, device=self.device, dtype=torch.float32)
        gate = torch.zeros(B, cap, device=self.device, dtype=torch.float32)
        align = torch.zeros(B, cap, T, device=self.device, dtype=torch.float32)
        mel_lengths = torch.zeros(B, device=self.device, dtype=torch.int32)
        n_steps = torch.zeros(1, device=self.device, dtype=torch.int32)
        ws = self._workspace("dec", L.t2_decoder_workspace_bytes(self.handle, B, T, cap))
        len32 = _i32(memory_lengths, self.device)
        if teacher_prenet is not None:
            teacher_prenet = teacher_prenet.contiguous()
        pk, ak, dk = _u8(prenet_keep, self.device), _u8(att_keep, self.device), _u8(dec_keep, self.device)
        a = _capi.T2DecoderArgs(mode, self.impl if impl is None else impl, int(bool(training)), memory.data_ptr(),
                                _ptr(len32), B, T, cap, _ptr(teacher_prenet), _ptr(pk), _ptr(ak), _ptr(dk),
                                next_seed() if seed is None else seed, float(gate_threshold), float(score_mask_value),
                                mel.data_ptr(), gate.data_ptr(), align.data_ptr(), mel_lengths.data_ptr(),
                                n_steps.data_ptr(), ws.data_ptr(), ws.numel(),
                                _ptr(stash), 0 if stash is None else stash.numel())
        self._call(L.t2_decoder_run, C.byref(a))
        self._last_decoder_args = (a, memory, len32, teacher_prenet, pk, ak, dk, ws, mel, gate, align, mel_lengths, n_steps)
        return mel, gate, align, mel_lengths, n_steps

    def decoder_stream(self, memory, n_steps_cap, prenet_keep=None, gate_threshold=0.5, score_mask_value=-float("inf"),
                       impl=None, seed=None, memory_lengths=None):
        """Begins a resumable INFER run of the persistent decoder (t2_decoder_stream_begin); see DecoderStream."""
        return DecoderStream(self, memory, n_steps_cap, prenet_keep, gate_threshold, score_mask_value,
                             self.impl if impl is None else impl, next_seed() if seed is None else seed, memory_lengths)

    def decoder_profile(self):
        """Per-phase SM cycles of the last persistent decoder run: dict phase -> [cta0, cta60, cta100]."""
        a = self._last_decoder_args[0]
        out = (C.c_int64 * 72)()
        _capi.check(_capi.lib().t2_decoder_profile(C.byref(a), out))
        names = ["E0 x2->att gemm", "E0 epilogue(ah)", "B1", "E1 ah->dec/att/q gemm", "B2", "attention", "B3",
                 "E2 ctx gemm", "E2 epilogue(dh)", "B4", "E3 dh gemm", "E3 epilogue(mel/x1)", "B5", "E4 x1 gemm+epi", "B6",
                 "att:im2col", "att:mma", "att:energies", "att:softmax", "att:context"]
        return {names[i]: [int(out[s * 24 + i]) for s in range(3)] for i in range(len(names))}

    def grad_table(self, named_grads):
        """ctypes pointer array of T2_NUM_WEIGHTS entries: named_grads maps full state_dict names to the contiguous fp32
        tensors the library overwrites with that parameter's gradient."""
        return (C.c_void_p * _capi.T2_NUM_WEIGHTS)(*[_ptr(named_grads.get(n)) for n, _ in self.spec])

    def decoder_stash(self, B, T_enc, T_mel):
        return self.stash_buffer("decoder", B, T_enc, T_mel)

    def decoder_backward(self, memory, memory_lengths, teacher_prenet, align, stash, seed, training, att_keep, dec_keep,
                         score_mask_value, d_mel, d_gate, d_align, named_grads):
        """Backward of the teacher-forced decoder run that filled `stash`.  d_mel (B, T, 80), d_gate (B, T), d_align
        (B, T, T_enc) or None.  Returns (d_memory (B, T_enc, 512), d_prenet (T, B, 256))."""
        L = _capi.lib()
        B, Te = int(memory.shape[0]), int(memory.shape[1])
        T = int(align.shape[1])
        f32 = dict(device=self.device, dtype=torch.float32)
        d_memory = torch.empty(B, Te, self.hp.encoder_embedding_dim, **f32)
        d_prenet = torch.empty(T, B, self.hp.prenet_dim, **f32)
        ws = self._workspace("dec_bwd", L.t2_decoder_backward_workspace_bytes(self.handle, B, Te, T))
        memory, len32 = memory.contiguous(), _i32(memory_lengths, self.device)
        ak, dk = _u8(att_keep, self.device), _u8(dec_keep, self.device)
        d_mel, d_gate = d_mel.to(**f32).contiguous(), d_gate.to(**f32).contiguous()
        if d_align is not None:
            d_align = d_align.to(**f32).contiguous()
        a = _capi.T2DecoderBwdArgs(memory.data_ptr(), _ptr(len32), B, Te, T, int(bool(training)), teacher_prenet.data_ptr(),
                                   _ptr(ak), _ptr(dk), seed, float(score_mask_value), align.data_ptr(),
                                   stash.data_ptr(), stash.numel(), d_mel.data_ptr(), d_gate.data_ptr(), _ptr(d_align),
                                   d_memory.data_ptr(), d_prenet.data_ptr(), self.grad_table(named_grads),
                                   _capi.T2_NUM_WEIGHTS, ws.data_ptr(), ws.numel())
        self._call(L.t2_decoder_backward, C.byref(a))
        return d_memory, d_prenet

    def prenet_backward(self, frames, keep, seed, d_out, named_grads):
        L = _capi.lib()
        frames = frames.to(device=self.device, dtype=torch.float32).contiguous()
        M = int(frames.shape[0])
        d_out, keep = d_out.contiguous(), _u8(keep, self.device)
        ws = self._workspace("pre_bwd", L.t2_prenet_backward_workspace_bytes(self.handle, M))
        a = _capi.T2PrenetBwdArgs(frames.data_ptr(), M, _ptr(keep), seed, d_out.data_ptr(), self.grad_table(named_grads),
                                  _capi.T2_NUM_WEIGHTS, ws.data_ptr(), ws.numel())
        self._call(L.t2_prenet_backward, C.byref(a))

    def prenet(self, frames, keep=None, seed=None):
        """frames (M, 80) -> (M, 256); keep (2, M, 256) uint8 or None."""
        frames = frames.to(device=self.device, dtype=torch.float32).contiguous()
        M = int(frames.shape[0])
        out = torch.empty(M, self.hp.prenet_dim, device=self.device, dtype=torch.float32)
        ws = self._workspace("pre", M * self.hp.prenet_dim * 4)
        keep = _u8(keep, self.device)
        self._call(_capi.lib().t2_prenet_forward, frames.data_ptr(), M, _ptr(keep), next_seed() if seed is None else seed,
                   out.data_ptr(), ws.data_ptr(), ws.numel())
        return out

    # -- postnet ---------------------------------------------------------------------------------
    def postnet(self, mel_btc, lengths=None, add_residual=True, training=False, keep=None, stash=None, seed=None,
                per_row=False):
        """mel_btc: (B, T, 80) time-major rows (batch stride may exceed T*80).  Returns (B, 80, T).  per_row
        (t2_postnet_infer): row b is computed as its first lengths[b] frames alone."""
        L = _capi.lib()
        # a single frame (T = 1) may carry any time stride: torch calls such a tensor contiguous and keeps it as it is
        assert mel_btc.dtype == torch.float32 and mel_btc.stride(2) == 1 and (mel_btc.stride(1) == mel_btc.shape[2] or mel_btc.shape[1] == 1)
        B, T = int(mel_btc.shape[0]), int(mel_btc.shape[1])
        out = torch.empty(B, self.hp.n_mel_channels, T, device=self.device, dtype=torch.float32)
        ws = self._workspace("post", L.t2_postnet_workspace_bytes(self.handle, B, T))
        len32, keep = _i32(lengths, self.device), _u8(keep, self.device)
        a = _capi.T2PostnetArgs(mel_btc.data_ptr(), int(mel_btc.stride(0)), _ptr(len32), B, T, int(bool(training)),
                                _ptr(keep), next_seed() if seed is None else seed, int(bool(add_residual)),
                                out.data_ptr(), ws.data_ptr(), ws.numel(), _ptr(stash), 0 if stash is None else stash.numel())
        self._call(L.t2_postnet_infer if per_row else L.t2_postnet_forward, C.byref(a))
        return out

    # -- end to end with host buffers (bench e2e leg) ------------------------------------------------
    def infer_host(self, text_host, max_steps, gate_threshold=0.5, impl=None, out_host=None, seed=None, input_lengths_host=None):
        """text_host: pinned int64 (B, T).  Returns (mel_post_host (B,80,max_steps), lengths, n_steps).  seed: the
        Philox seed of the decoder's prenet dropout (default: next_seed()).  input_lengths_host: pinned int64 (B) or None;
        given, t2_infer_host_lengths runs each row as its first input_lengths_host[b] symbols alone."""
        L = _capi.lib()
        B, T = int(text_host.shape[0]), int(text_host.shape[1])
        if out_host is None:
            out_host = (torch.empty(B, self.hp.n_mel_channels, max_steps, dtype=torch.float32).pin_memory(),
                        torch.empty(B, dtype=torch.int32).pin_memory(), torch.empty(1, dtype=torch.int32).pin_memory())
        mel, lens, ns = out_host
        seed = next_seed() if seed is None else seed
        impl = self.impl if impl is None else impl
        if input_lengths_host is not None:
            ws = self._workspace("e2e", L.t2_infer_lengths_workspace_bytes(self.handle, B, T, max_steps))
            a = _capi.T2InferArgs(text_host.data_ptr(), input_lengths_host.data_ptr(), B, T, int(max_steps),
                                  float(gate_threshold), seed, impl, mel.data_ptr(), lens.data_ptr(), ns.data_ptr(),
                                  ws.data_ptr(), ws.numel())
            self._call(L.t2_infer_host_lengths, C.byref(a))
            return mel, lens, ns
        ws = self._workspace("e2e", L.t2_infer_workspace_bytes(self.handle, B, T, max_steps))
        self._call(L.t2_infer_host, text_host.data_ptr(), B, T, int(max_steps), float(gate_threshold), seed, impl,
                   mel.data_ptr(), lens.data_ptr(), ns.data_ptr(), ws.data_ptr(), ws.numel())
        return mel, lens, ns


def f32_buffer(device, *shape):
    """A zeroed fp32 tensor over a byte buffer of exactly its size (the allocation the buffer-bounds tests place)."""
    n = 1
    for d in shape:
        n *= int(d)
    return _capi.byte_buffer(4 * n, device).view(torch.float32).zero_().view(*shape)


class DecoderStream:
    """One resumable decoder run: full-size output buffers (mel (B, cap, 80), gate (B, cap), align (B, cap, T_enc),
    mel_lengths (B,) with -1 for live rows) and the per-stream state buffer that carries everything across a chunk
    boundary.  ``run(n)`` advances every live 64-row slice by up to n steps and takes the one host sync of the chunk.

    Continuous batching (serving.py) uses the rows as slots: ``cap`` is the chunk length + 1, the buffers hold one chunk,
    ``chunk`` runs local steps [0, n), ``admit`` resets rows for new texts and ``collect`` hands a chunk's frames to the
    requests' own buffers.  ``memory``, ``len32`` and ``keep`` are the tensors the kernel reads: such a session rewrites
    their rows in place between chunks."""

    def __init__(self, eng, memory, cap, prenet_keep, gate_threshold, score_mask_value, impl, seed, memory_lengths=None):
        L = _capi.lib()
        dev = eng.device
        self.eng = eng
        self.memory = memory.to(device=dev, dtype=torch.float32).contiguous()
        B, T = int(self.memory.shape[0]), int(self.memory.shape[1])
        self.B, self.T_enc, self.cap = B, T, int(cap)
        f32 = dict(device=dev, dtype=torch.float32)
        self.mel = f32_buffer(dev, B, self.cap, eng.hp.n_mel_channels)
        self.gate = f32_buffer(dev, B, self.cap)
        self.align = f32_buffer(dev, B, self.cap, T)
        self.n_steps = torch.zeros(1, device=dev, dtype=torch.int32)
        self.n_slices = (B + 63) // 64
        # mel_lengths | status in one tensor: what the host reads back after a chunk is one copy
        self.readback = torch.zeros(B + 2 * self.n_slices, device=dev, dtype=torch.int32)
        self.mel_lengths, self.status = self.readback[:B], self.readback[B:]
        self.status_host = None                      # the caller's copy of `status` after the last run
        self.state = _capi.byte_buffer(L.t2_decoder_stream_state_bytes(eng.handle, B, T), dev)
        self.keep, self.len32 = _u8(prenet_keep, dev), _i32(memory_lengths, dev)
        d = _capi.T2DecoderArgs(_capi.MODE_INFER, impl, 0, self.memory.data_ptr(), _ptr(self.len32), B, T, self.cap,
                                None, _ptr(self.keep), None, None, seed, float(gate_threshold), float(score_mask_value),
                                self.mel.data_ptr(), self.gate.data_ptr(), self.align.data_ptr(),
                                self.mel_lengths.data_ptr(), self.n_steps.data_ptr())
        self.args = _capi.T2DecoderStreamArgs(d, self.state.data_ptr(), self.state.numel(), self.status.data_ptr())
        eng._call(L.t2_decoder_stream_begin, C.byref(self.args))

    def run(self, n):
        """Advance by up to n steps.  Returns (live_steps, n_total, finished): the steps run by the slices that are still
        live (None when none is), the most steps any slice has run, and whether every slice has stopped."""
        self.eng._call(_capi.lib().t2_decoder_stream_run, C.byref(self.args), int(n), _ptr(self.status_host))
        self.status_host = self.status.cpu()         # the one host sync of the chunk
        steps = self.status_host[0::2].tolist()
        stopped = self.status_host[1::2].tolist()
        live = [s for s, x in zip(steps, stopped) if not x]
        return (min(live) if live else None), max(steps), not live

    # -- continuous batching ------------------------------------------------------------------------
    def admit(self, rows):
        """rows (ascending ints): back to the state begin gives them, processed memory from memory[row] / len32[row]."""
        arr = (C.c_int32 * len(rows))(*rows)
        self.eng._call(_capi.lib().t2_decoder_stream_admit, C.byref(self.args), arr, len(rows))

    def launch_chunk(self, n, seed, skip_slices=()):
        """Enqueue local steps [0, n) of every 64-row slice not in skip_slices (n < cap) under the Philox seed `seed`."""
        assert 1 <= n < self.cap
        self.args.dec.seed = seed
        host = torch.tensor([[0, int(i in skip_slices)] for i in range(self.n_slices)], dtype=torch.int32)
        self.eng._call(_capi.lib().t2_decoder_stream_run, C.byref(self.args), int(n), host.data_ptr())

    def collect(self, entries):
        """entries: (row, n_frames, T_text, mel, gate, align) -- the chunk's first n_frames frames of `row` go to the fp32
        tensors mel (n_frames, 80), gate (n_frames,), align (n_frames, T_text) (views at the request's own step offset)."""
        arr = (_capi.T2CollectRow * len(entries))(*[
            _capi.T2CollectRow(r, n, T, 0, mel.data_ptr(), gate.data_ptr(), align.data_ptr())
            for r, n, T, mel, gate, align in entries])
        self.eng._call(_capi.lib().t2_decoder_stream_collect, C.byref(self.args), arr, len(entries))

    def read_chunk(self):
        """The one host sync of a chunk: (mel_lengths per row: local firing step + 1 or -1, steps run per slice)."""
        host = self.readback.cpu().tolist()
        return host[:self.B], host[self.B::2]
