"""Host-side glue between the nn.Module boundary and libt2b200.so: weight table, handle cache,
workspaces, dropout-mask injection.  All arithmetic happens in the shared library."""
import contextlib
import ctypes as C
import math
import numbers
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


def seed_pattern(v, what):
    """One seed, an integer in [0, 2**64), as its 64-bit pattern in int64 range; raises ValueError outside."""
    v = int(v)
    if not 0 <= v < 1 << 64:
        raise ValueError("%s: seed %d is outside [0, 2**64)" % (what, v))
    return v - (1 << 64) if v >= 1 << 63 else v


def row_seeds(seeds, B, device, what):
    """Per-utterance seeds as B 64-bit Philox keys, an int64 tensor on `device` holding each key's bit pattern (None
    stays None).  seeds: B integers in [0, 2**64), as a list, a host tensor or a device tensor; int64 / uint64 values are
    taken as their 64-bit pattern, narrower integer dtypes must be >= 0.  Raises TypeError / ValueError before anything
    runs."""
    if seeds is None:
        return None
    if torch.is_tensor(seeds):
        t = seeds
        if t.dtype == torch.bool or t.dtype.is_floating_point or t.dtype.is_complex:
            raise TypeError("%s: seeds must hold integers (got %s)" % (what, t.dtype))
        if t.dim() != 1 or t.shape[0] != B:
            raise ValueError("%s: seeds must have shape (%d,) (got %s)" % (what, B, tuple(t.shape)))
        if t.dtype == torch.uint64:
            t = t.contiguous().view(torch.int64)
        elif t.dtype != torch.int64:
            if t.dtype.is_signed and bool((t < 0).any()):
                raise ValueError("%s: seeds must lie in [0, 2**64)" % what)
            t = t.to(torch.int64)
        return t.to(device=device).contiguous()
    vals = list(seeds)
    if len(vals) != B:
        raise ValueError("%s: seeds must hold %d values (got %d)" % (what, B, len(vals)))
    for v in vals:
        if isinstance(v, bool) or not isinstance(v, numbers.Integral):
            raise TypeError("%s: seeds must be integers (got %r)" % (what, v))
    return torch.tensor([seed_pattern(v, what) for v in vals], dtype=torch.int64).to(device)


def _integer_tensor(x, name, what):
    """x (a tensor, or anything torch.as_tensor takes) as a tensor of integers; TypeError otherwise."""
    t = x if torch.is_tensor(x) else torch.as_tensor(x)
    if t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool:
        raise TypeError("%s: %s must hold integers (got %s)" % (what, name, t.dtype))
    return t


def _float_tensor(t, name, what, shape, dims, device_type, dtypes=None):
    """Refuses t as argument `name` of `what` unless it is a tensor of a floating dtype (one of `dtypes` if given) with
    a number of dims in `dims` (the allowed shapes written as `shape`), no extent 0, on a device of type `device_type`:
    TypeError / ValueError."""
    if not torch.is_tensor(t):
        raise TypeError("%s: %s must be a tensor (got %s)" % (what, name, type(t).__name__))
    if dtypes is None and not t.dtype.is_floating_point:
        raise TypeError("%s: %s must be a float tensor (got %s)" % (what, name, t.dtype))
    if dtypes is not None and t.dtype not in dtypes:
        names = " or ".join(str(d).replace("torch.", "") for d in dtypes)
        raise TypeError("%s: %s must be %s (got %s)" % (what, name, names, t.dtype))
    if t.dim() not in dims or min(t.shape) < 1:
        raise ValueError("%s: %s must have shape %s, none of them 0 (got %s)" % (what, name, shape, tuple(t.shape)))
    if t.device.type != device_type:
        raise ValueError("%s: %s must be on a %s device (got %s); there is no CPU path"
                         % (what, name, device_type.upper(), t.device))


def _number(x, name, what, lo=None, hi=None, lo_open=False, integer=False):
    """x as argument `name` of `what`: a real number (an integer if `integer`), finite and in [lo, hi] ((lo, hi] if
    lo_open), as a float (int); TypeError / ValueError otherwise."""
    if isinstance(x, bool) or not isinstance(x, numbers.Real) or (integer and not isinstance(x, numbers.Integral)):
        raise TypeError("%s: %s must be %s (got %r)" % (what, name, "an integer" if integer else "a real number", x))
    x = int(x) if integer else float(x)
    if (not integer and not math.isfinite(x)) or (lo is not None and (x <= lo if lo_open else x < lo)) or \
            (hi is not None and x > hi):
        rng = "%s%s, %s]" % ("(" if lo_open else "[", lo if lo is not None else "-inf", hi if hi is not None else "inf")
        raise ValueError("%s: %s must lie in %s (got %r)" % (what, name, rng, x))
    return x


_TABLES = {}
_TABLES_LOCK = threading.Lock()


def _cached_table(key, build):
    """build() -- host tables put on a device -- cached under `key`; a 17th key drops the 16 cached ones."""
    with _TABLES_LOCK:
        t = _TABLES.get(key)
        if t is None:
            t = build()
            if len(_TABLES) >= 16:
                _TABLES.clear()
            _TABLES[key] = t
        return t


def row_lengths(lengths, B, T, name, device):
    """Per-row lengths of a ragged inference batch: (B,) integers, each in 1..T, as a list, a host or a device tensor.
    Returns (lengths as int32 on `device`, whether some row is shorter than T), reading a device tensor back once;
    (None, False) for None.  Raises TypeError / ValueError before anything is launched."""
    if lengths is None:
        return None, False
    t = _integer_tensor(lengths, name, "tacotron2_b200")
    if tuple(t.shape) != (B,):
        raise ValueError("tacotron2_b200: %s must have shape (%d,) (got %s)" % (name, B, tuple(t.shape)))
    host = t.cpu()
    lo, hi = int(host.min()), int(host.max())
    if lo < 1 or hi > T:
        raise ValueError("tacotron2_b200: %s must lie in 1..%d (got %d..%d)" % (name, T, lo, hi))
    return t.to(device=device, dtype=torch.int32).contiguous(), lo < T


def forced_alignment(alignments, alignment_lengths, B, T_text, device, training, what):
    """The forced-alignment part of inference_options: given attention weights as the engine takes them, (map (B, T_map,
    T_text) fp32 contiguous, lengths (B,) int32), both on `device`; (None, None) without a map."""
    if alignments is None:
        if alignment_lengths is not None:
            raise ValueError("%s: alignment_lengths needs alignments" % what)
        return None, None
    if training:
        raise ValueError("%s: alignments need eval mode (a forced run is an inference; training-mode inference applies "
                         "the hidden-state dropout, which a forced run does not take)" % what)
    if not torch.is_tensor(alignments):
        raise TypeError("%s: alignments must be a tensor (got %s)" % (what, type(alignments).__name__))
    if not alignments.dtype.is_floating_point:
        raise TypeError("%s: alignments must be a float tensor (got %s)" % (what, alignments.dtype))
    if alignments.dim() != 3 or alignments.shape[0] != B or alignments.shape[1] < 1 or alignments.shape[2] != T_text:
        raise ValueError("%s: alignments must have shape (%d, T_map >= 1, %d) (got %s)" % (what, B, T_text,
                                                                                          tuple(alignments.shape)))
    if alignments.device != torch.device(device):
        raise ValueError("%s: alignments must be on the model's device %s (got %s)" % (what, device, alignments.device))
    T_map = int(alignments.shape[1])
    if alignment_lengths is None:
        lengths = torch.full((B,), T_map, dtype=torch.int32, device=device)
    else:
        lengths = _integer_tensor(alignment_lengths, "alignment_lengths", what)
        if tuple(lengths.shape) != (B,):
            raise ValueError("%s: alignment_lengths must have shape (%d,) (got %s)" % (what, B, tuple(lengths.shape)))
        host = lengths.cpu()
        lo, hi = int(host.min()), int(host.max())
        if lo < 1 or hi > T_map:
            raise ValueError("%s: alignment_lengths must lie in 1..%d (got %d..%d)" % (what, T_map, lo, hi))
        lengths = lengths.to(device=device, dtype=torch.int32).contiguous()
    return alignments.to(dtype=torch.float32).contiguous(), lengths


def _integral(v):
    return isinstance(v, numbers.Integral) and not isinstance(v, bool)


def _limits(attention_window, max_decoder_steps, B, device, forced, what):
    """The limits of a free run as the engine takes them: (window, caps, longest) -- window None or (back, front) ints,
    caps None or (B,) int32 contiguous on `device`, longest None or max(caps) (see inference_options)."""
    if forced and attention_window is not None:
        raise ValueError("%s: attention_window and alignments exclude each other (a forced run computes no energies)" % what)
    if forced and max_decoder_steps is not None:
        raise ValueError("%s: max_decoder_steps and alignments exclude each other (the map decides the steps)" % what)
    window = None
    if attention_window is not None:
        w = attention_window.tolist() if torch.is_tensor(attention_window) else attention_window
        if not isinstance(w, (tuple, list)) or len(w) != 2 or not all(_integral(v) for v in w):
            raise TypeError("%s: attention_window must be two integers (back, front) (got %r)" % (what, attention_window))
        back, front = int(w[0]), int(w[1])
        if back < 0 or front < 1:
            raise ValueError("%s: attention_window needs back >= 0 and front >= 1 (got (%d, %d))" % (what, back, front))
        window = (min(back, 2 ** 31 - 1), min(front, 2 ** 31 - 1))
    if max_decoder_steps is None:
        return window, None, None
    if _integral(max_decoder_steps):
        caps = host = torch.full((B,), int(max_decoder_steps), dtype=torch.int64)
    else:
        caps = _integer_tensor(max_decoder_steps, "max_decoder_steps", what)
        if tuple(caps.shape) != (B,):
            raise ValueError("%s: max_decoder_steps must be one integer or have shape (%d,) (got %s)"
                             % (what, B, tuple(caps.shape)))
        host = caps.cpu().to(torch.int64)
    lo, hi = int(host.min()), int(host.max())
    if lo < 1 or hi > 2 ** 31 - 1:
        raise ValueError("%s: max_decoder_steps must lie in 1..2**31-1 (got %d..%d)" % (what, lo, hi))
    return window, caps.to(device=device, dtype=torch.int32).contiguous(), hi


class InferenceOptions:
    """The per-row options of one inference call in the engine's form (inference_options()).

    lengths: (B,) int32 on the device or None; ragged: some row is shorter than T_enc; row_seeds: (B,) int64 key
    patterns on the device or None; forced_align / forced_lengths: a forced run's map (B, T_map, T_enc) fp32 and steps
    (B,) int32, or None; window: (back, front) or None; max_steps: (B,) int32 step limits or None; cap: the run's
    n_steps_cap when the options fix it (T_map, or the largest limit), else None."""

    def __init__(self, lengths, ragged, row_seeds, forced, limits):
        self.lengths, self.ragged, self.row_seeds = lengths, ragged, row_seeds
        self.forced_align, self.forced_lengths = forced
        self.window, self.max_steps, longest = limits
        self.cap = self.forced_align.size(1) if self.forced_align is not None else longest

    def decoder_kwargs(self):
        """The keyword arguments of Engine.decoder / Engine.decoder_stream these options set."""
        return dict(memory_lengths=self.lengths, row_seeds=self.row_seeds, forced_align=self.forced_align,
                    forced_lengths=self.forced_lengths, window=self.window, max_steps=self.max_steps)


def inference_options(what, B, T_enc, device, training=False, prenet_masks=False, lengths=None,
                      lengths_name="memory_lengths", seeds=None, alignments=None, alignment_lengths=None,
                      attention_window=None, max_decoder_steps=None):
    """The user-facing options of one inference call (``what``, e.g. "Tacotron2.inference") checked once and turned into
    the engine's form, an InferenceOptions.  Each device tensor among them is read back to the host at most once.

    lengths (named ``lengths_name``): None or B integers in 1..T_enc (see row_lengths).  seeds: None or B integers in
    [0, 2**64) (see row_seeds); they need eval mode (training False) and no injected prenet masks (prenet_masks False).
    alignments: None or a float tensor (B, T_map, T_enc) on `device`, eval mode only; alignment_lengths: None (T_map for
    every row) or B integers in 1..T_map.  attention_window: None or two integers (back >= 0, front >= 1);
    max_decoder_steps: None, one integer or B integers >= 1; neither goes with alignments.  Raises TypeError /
    ValueError naming the argument before anything runs."""
    lengths, ragged = row_lengths(lengths, B, T_enc, lengths_name, device)
    what = "tacotron2_b200: " + what
    if seeds is not None:
        if training:
            raise ValueError("%s: seeds need eval mode (training-mode BatchNorm mixes the rows and the hidden-state dropout "
                             "is not keyed per row)" % what)
        if prenet_masks:
            raise ValueError("%s: seeds and injected prenet masks exclude each other" % what)
    keys = row_seeds(seeds, B, device, what)
    forced = forced_alignment(alignments, alignment_lengths, B, T_enc, device, training, what)
    limits = _limits(attention_window, max_decoder_steps, B, device, forced[0] is not None, what)
    return InferenceOptions(lengths, ragged, keys, forced, limits)


def alignments_from_durations(durations):
    """Durations (B, T_text) of non-negative integer frame counts -> (alignments, alignment_lengths) for a forced
    ``Tacotron2.inference``: a one-hot map (B, T_map, T_text) fp32 in which symbol j of row b is attended for
    durations[b, j] consecutive steps, and the steps of each row, durations.sum(1) (int64), both on durations' device;
    T_map is the longest row.  Rows whose counts sum to 0 are refused."""
    d = durations if torch.is_tensor(durations) else torch.as_tensor(durations)
    if d.dtype.is_floating_point or d.dtype.is_complex or d.dtype == torch.bool:
        raise TypeError("tacotron2_b200: durations must hold integers (got %s)" % d.dtype)
    if d.dim() != 2 or d.shape[1] < 1:
        raise ValueError("tacotron2_b200: durations must have shape (B, T_text) (got %s)" % (tuple(d.shape),))
    d = d.long()
    if bool((d < 0).any()):
        raise ValueError("tacotron2_b200: durations must be >= 0")
    lengths = d.sum(1)
    empty = (lengths == 0).nonzero().flatten().tolist()
    if empty:
        raise ValueError("tacotron2_b200: durations of rows %s sum to 0 frames" % empty)
    B, T = d.shape
    total = int(lengths.sum())
    dev = d.device
    sym = torch.repeat_interleave(torch.arange(T, device=dev).repeat(B), d.reshape(-1))            # symbol of each step
    row = torch.repeat_interleave(torch.arange(B, device=dev), lengths)
    step = torch.arange(total, device=dev) - torch.repeat_interleave(lengths.cumsum(0) - lengths, lengths)
    out = torch.zeros(B, int(lengths.max()), T, dtype=torch.float32, device=dev)
    out[row, step, sym] = 1.0
    return out, lengths


_DURATION_METHODS = {"mas": _capi.DURATIONS_MAS, "argmax": _capi.DURATIONS_ARGMAX}


def duration_inputs(alignments, input_lengths, mel_lengths, method, device_type="cuda"):
    """The arguments of durations_from_alignments checked and put in the library's form: (alignments fp32 contiguous,
    input_lengths and mel_lengths as (B,) int32 on its device or None, the method's code).  The map must live on a
    device of type `device_type`.  Reads the device back once for the weights' range (and, for MAS, the rows without a
    path) and once per device-side lengths tensor.  Raises TypeError / ValueError before anything is launched."""
    what = "tacotron2_b200.durations_from_alignments"
    if method not in _DURATION_METHODS:
        raise ValueError("%s: method must be one of %s (got %r)" % (what, sorted(_DURATION_METHODS), method))
    _float_tensor(alignments, "alignments", what, "(B, T_mel, T_text)", (3,), device_type)
    B, T_mel, T_text = (int(s) for s in alignments.shape)
    if T_text > _capi.DURATIONS_MAX_TEXT:
        raise ValueError("%s: T_text must be at most %d (got %d)" % (what, _capi.DURATIONS_MAX_TEXT, T_text))
    dev = alignments.device
    il, _ = row_lengths(input_lengths, B, T_text, "input_lengths", dev)
    ml, _ = row_lengths(mel_lengths, B, T_mel, "mel_lengths", dev)
    a = alignments.detach().to(torch.float32).contiguous()
    probe = torch.stack(torch.aminmax(a)).double()
    if method == "mas":
        n_text = il if il is not None else torch.full((B,), T_text, dtype=torch.int32, device=dev)
        n_mel = ml if ml is not None else torch.full((B,), T_mel, dtype=torch.int32, device=dev)
        probe = torch.cat((probe, (n_mel < n_text).double()))
    host = probe.tolist()                                       # the one host read of the weights
    if not (math.isfinite(host[0]) and math.isfinite(host[1]) and host[0] >= 0):
        raise ValueError("%s: alignments must be finite and >= 0 (got values in [%r, %r])" % (what, host[0], host[1]))
    short = [b for b, v in enumerate(host[2:]) if v]
    if short:
        raise ValueError("%s: rows %s have fewer frames than symbols, so no monotonic path gives every symbol a frame "
                         "(method='mas')" % (what, short))
    return a, il, ml, _DURATION_METHODS[method]


def durations_from_alignments(alignments, input_lengths=None, mel_lengths=None, method="mas"):
    """Attention maps -> per-symbol frame counts: the inverse of alignments_from_durations.

    alignments: (B, T_mel, T_text) float tensor of any float dtype on a CUDA device, finite and >= 0 (what
    Tacotron2.inference, Decoder.inference and Tacotron2.forward return), read as fp32; T_text <= 4096.
    input_lengths / mel_lengths: None (T_text / T_mel for every row) or B integers in 1..T_text / 1..T_mel, as a list, a
    host or a device tensor (``model.mel_lengths`` after inference; ``input_lengths`` / ``output_lengths`` from
    ``parse_batch`` for a teacher-forced batch).

    Returns (B, T_text) int64 on the alignments' device.  Row b sums to mel_lengths[b], is zero from input_lengths[b]
    on, and depends only on alignments[b, :mel_lengths[b], :input_lengths[b]], so it equals its own B = 1 call on that
    slice.

    method "mas" (monotonic alignment search): the path from (0, 0) to (L_mel - 1, L_text - 1) that stays on its symbol
    or advances by one per frame and maximises the sum of log(max(a, 2**-126)), in fp64; every symbol gets at least one
    frame, and where paths tie the later advance wins (a uniform map gives [1, ..., 1, L_mel - L_text + 1]).  Rows with
    mel_lengths[b] < input_lengths[b] have no such path and are refused.  method "argmax": each frame goes to the first
    symbol holding its maximum; a symbol may get 0 frames.  See DESIGN section 6.10."""
    a, il, ml, code = duration_inputs(alignments, input_lengths, mel_lengths, method)
    B, T_mel, T_text = (int(s) for s in a.shape)
    L = _capi.lib()
    out = torch.empty(B, T_text, dtype=torch.int64, device=a.device)
    ws = _capi.byte_buffer(L.t2_durations_workspace_bytes(B, T_mel, T_text, code), a.device)
    args = _capi.T2DurationsArgs(a.data_ptr(), _ptr(il), _ptr(ml), B, T_mel, T_text, code, out.data_ptr(),
                                 ws.data_ptr(), ws.numel())
    _capi.call(L.t2_durations, a.device, C.byref(args))
    return out


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
                score_mask_value=-float("inf"), impl=None, stash=None, seed=None, row_seeds=None, forced_align=None,
                forced_lengths=None, window=None, max_steps=None):
        """row_seeds: None or (B,) int64 on the device (see row_seeds()): per-row prenet keys.  forced_align /
        forced_lengths: None, or the given attention weights (B, n_steps_cap, T_enc) fp32 and each row's step count (B,)
        int32, both contiguous on the device.  window / max_steps: None, or the attention window (back, front) and each
        row's step limit (B,) int32 on the device (see InferenceOptions)."""
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
        a = decoder_args(mode=mode, impl=self.impl if impl is None else impl, training=int(bool(training)), memory=memory,
                         memory_lengths=len32, B=B, T_enc=T, n_steps_cap=cap, teacher_prenet=teacher_prenet,
                         prenet_keep=pk, att_keep=ak, dec_keep=dk, seed=next_seed() if seed is None else seed,
                         gate_threshold=float(gate_threshold), score_mask_value=float(score_mask_value), mel=mel,
                         gate=gate, align=align, mel_lengths=mel_lengths, n_steps=n_steps, ws=ws, ws_bytes=ws.numel(),
                         stash=stash, stash_bytes=0 if stash is None else stash.numel(), row_seeds=row_seeds,
                         forced_align=forced_align, forced_lengths=forced_lengths, window=window, max_steps=max_steps)
        self._call(L.t2_decoder_run, C.byref(a))
        self._last_decoder_args = (a, memory, len32, teacher_prenet, pk, ak, dk, ws, mel, gate, align, mel_lengths, n_steps,
                                   row_seeds, forced_align, forced_lengths, max_steps)
        return mel, gate, align, mel_lengths, n_steps

    # -- the step API (Decoder.initialize_decoder_states / decode, Attention / LocationLayer forwards) ----------------
    def processed_memory(self, memory):
        """memory (B, T_enc, 512) fp32 contiguous on the device -> memory_layer(memory) (B, T_enc, 128) fp32."""
        B, T = int(memory.shape[0]), int(memory.shape[1])
        out = torch.empty(B, T, self.hp.attention_dim, device=self.device, dtype=torch.float32)
        self._call(_capi.lib().t2_processed_memory, memory.data_ptr(), B, T, out.data_ptr())
        return out

    def decoder_step(self, memory, pm, mask, state, x, training, att_keep, dec_keep, seed, score_mask_value):
        """One t2_decoder_step.  memory / pm fp32 contiguous, mask None or (B, T_enc) uint8, state: the seven fp32
        contiguous arrays (ah, ac, dh, dc, aw, awc, ctx), updated in place; x (B, 256) fp32.  Returns mel (B, 80) and
        gate (B, 1), fp32."""
        L = _capi.lib()
        B, T = int(memory.shape[0]), int(memory.shape[1])
        mel = torch.empty(B, self.hp.n_mel_channels, device=self.device, dtype=torch.float32)
        gate = torch.empty(B, 1, device=self.device, dtype=torch.float32)
        ws = self._workspace("step", L.t2_decoder_step_workspace_bytes(self.handle, B))
        ah, ac, dh, dc, aw, awc, ctx = state
        a = _capi.T2DecoderStepArgs(B, T, memory.data_ptr(), pm.data_ptr(), _ptr(mask), ah.data_ptr(), ac.data_ptr(),
                                    dh.data_ptr(), dc.data_ptr(), aw.data_ptr(), awc.data_ptr(), ctx.data_ptr(),
                                    x.data_ptr(), mel.data_ptr(), gate.data_ptr(), int(bool(training)), _ptr(att_keep),
                                    _ptr(dec_keep), seed, float(score_mask_value), ws.data_ptr(), ws.numel())
        self._call(L.t2_decoder_step, C.byref(a))
        return mel, gate

    def attention(self, B, T, weights_cat, query=None, memory=None, pm=None, mask=None, score_mask_value=-float("inf"),
                  energies=False, location=False, weights=False, context=False):
        """One t2_attention_forward over fp32 contiguous inputs; returns the requested outputs (fp32) in the order
        energies, location, weights, context."""
        f32 = dict(device=self.device, dtype=torch.float32)
        outs = dict(energies=torch.empty(B, T, **f32) if energies else None,
                    location=torch.empty(B, T, self.hp.attention_dim, **f32) if location else None,
                    weights=torch.empty(B, T, **f32) if weights else None,
                    context=torch.empty(B, self.hp.encoder_embedding_dim, **f32) if context else None)
        a = _capi.T2AttentionArgs(B, T, _ptr(query), _ptr(memory), _ptr(pm), weights_cat.data_ptr(), _ptr(mask),
                                  float(score_mask_value), *[_ptr(outs[k]) for k in ("energies", "location", "weights",
                                                                                     "context")])
        self._call(_capi.lib().t2_attention_forward, C.byref(a))
        return [v for v in outs.values() if v is not None]

    def decoder_stream(self, memory, n_steps_cap, prenet_keep=None, gate_threshold=0.5, score_mask_value=-float("inf"),
                       impl=None, seed=None, memory_lengths=None, row_seeds=None, forced_align=None, forced_lengths=None,
                       window=None, max_steps=None):
        """Begins a resumable INFER run of the persistent decoder (t2_decoder_stream_begin); see DecoderStream."""
        return DecoderStream(self, memory, n_steps_cap, prenet_keep, gate_threshold, score_mask_value,
                             self.impl if impl is None else impl, next_seed() if seed is None else seed, memory_lengths,
                             row_seeds, forced_align, forced_lengths, window, max_steps)

    def decoder_profile(self):
        """Per-phase SM cycles of the last persistent decoder run: dict phase -> [cta0, cta60, cta100]."""
        a = self._last_decoder_args[0]
        out = (C.c_int64 * 72)()
        _capi.check(_capi.lib().t2_decoder_profile(C.byref(a), out))
        names = ["E0 x2->att gemm", "E0 epilogue(ah)", "B1", "E1 ah->dec/att/q gemm", "B2", "attention", "B3",
                 "E2 ctx gemm", "E2 epilogue(dh)", "B4", "E3 dh gemm", "E3 epilogue(mel/x1)", "B5", "E4 x1 gemm+epi", "B6",
                 "att:before B2 (pa copy or round 0)", "att:pa rounds 1+ or tile wait", "att:energies", "att:softmax",
                 "att:context", "att:next step's pa (in B6)", "Ed deferred ah->att' gemm (lower CTAs)"]
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
    def infer_host(self, text_host, max_steps, gate_threshold=0.5, impl=None, out_host=None, seed=None, input_lengths_host=None,
                   row_seeds_host=None):
        """text_host: pinned int64 (B, T).  Returns (mel_post_host (B,80,max_steps), lengths, n_steps).  seed: the
        Philox seed of the decoder's prenet dropout (default: next_seed()).  input_lengths_host: pinned int64 (B) or None;
        given, each row runs as its first input_lengths_host[b] symbols alone.  row_seeds_host: int64 (B) host tensor of
        per-row seeds (needs input_lengths_host): row b then equals its B = 1 call with that seed."""
        L = _capi.lib()
        B, T = int(text_host.shape[0]), int(text_host.shape[1])
        if out_host is None:
            out_host = (torch.empty(B, self.hp.n_mel_channels, max_steps, dtype=torch.float32).pin_memory(),
                        torch.empty(B, dtype=torch.int32).pin_memory(), torch.empty(1, dtype=torch.int32).pin_memory())
        mel, lens, ns = out_host
        ws = self._workspace("e2e", L.t2_infer_workspace_bytes(self.handle, B, T, max_steps))
        a = _capi.T2InferArgs(text_host.data_ptr(), _ptr(input_lengths_host), B, T, int(max_steps), float(gate_threshold),
                              next_seed() if seed is None else seed, self.impl if impl is None else impl, mel.data_ptr(),
                              lens.data_ptr(), ns.data_ptr(), ws.data_ptr(), ws.numel(), _ptr(row_seeds_host))
        self._call(L.t2_infer_host, C.byref(a))
        return mel, lens, ns


def decoder_args(window=None, **fields):
    """A T2DecoderArgs from its fields by name: tensors by their data pointer, None as NULL, fields not given zero.
    window: None (no window) or (back, front)."""
    a = _capi.T2DecoderArgs()
    if window is not None:
        a.window_back, a.window_front = window
    for name, v in fields.items():
        setattr(a, name, v.data_ptr() if torch.is_tensor(v) else v)
    return a


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

    def __init__(self, eng, memory, cap, prenet_keep, gate_threshold, score_mask_value, impl, seed, memory_lengths=None,
                 row_seeds=None, forced_align=None, forced_lengths=None, window=None, max_steps=None):
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
        self.row_seeds = row_seeds      # (B,) int64 bit patterns on the device or None; a session may rewrite them
        self.held = (forced_align, forced_lengths, max_steps)     # the kernel reads them in every chunk
        d = decoder_args(mode=_capi.MODE_INFER, impl=impl, memory=self.memory, memory_lengths=self.len32, B=B, T_enc=T,
                         n_steps_cap=self.cap, prenet_keep=self.keep, seed=seed, gate_threshold=float(gate_threshold),
                         score_mask_value=float(score_mask_value), mel=self.mel, gate=self.gate, align=self.align,
                         mel_lengths=self.mel_lengths, n_steps=self.n_steps, row_seeds=row_seeds,
                         forced_align=forced_align, forced_lengths=forced_lengths, window=window, max_steps=max_steps)
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

    def launch_chunk(self, n, seed, skip_slices=(), row_step0=None):
        """Enqueue local steps [0, n) of every 64-row slice not in skip_slices (n < cap) under the Philox seed `seed`.
        row_step0: with row seeds, (B,) int32 on the device -- the steps each row's request ran before this chunk."""
        assert 1 <= n < self.cap
        self.args.dec.seed = seed
        self.args.row_step0 = _ptr(row_step0)
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
