"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY.

A plain-tensor fp32 restatement of the NVIDIA/tacotron2 hot path (``model.py``), written
from the reference's *behaviour*: no ``nn.Module`` is used, every function takes a flat
``state_dict``-style mapping of weights plus explicit state and cites the reference
``file:line`` it follows.  It is the checker for the CUDA path and the ``cpu_baseline``
("port") leg of ``bench.py``; the product package ``tacotron2_b200`` never imports it.

Parity pinning: the reference ships no tests / golden vectors (SURVEY.md section 4), so this
oracle is pinned by executing the unmodified reference ``model.py`` (``oracle/ref_import.py``):
``tools/make_golden.py`` stores what the reference computed under ``tests/golden``, and
``tests/test_oracle_vs_reference.py`` / ``tests/test_oracle_golden.py`` compare the oracle with it.

All arithmetic is done by torch CPU fp32 tensor ops (matmul / conv1d); an optional
``mm`` hook lets precision studies swap the matmul (tools/precision_study.py).
"""
import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------------------
# primitives
# --------------------------------------------------------------------------------------


def _mm(x, w, mm=None):
    """x (.., K) @ w (N, K)^T.  (torch.nn.Linear semantics, layers.py:17-18)."""
    if mm is not None:
        return mm(x, w)
    return x @ w.t()


def dropout_with_mask(x, keep_mask, p):
    """F.dropout for a given Bernoulli keep-mask: x * keep / (1-p)  (model.py:99, 355, 370)."""
    if keep_mask is None:
        return x
    return x * keep_mask.to(x.dtype) * (1.0 / (1.0 - p))


def lstm_cell(x, h, c, w_ih, w_hh, b_ih, b_hh, mm=None):
    """torch.nn.LSTMCell (model.py:222-224, 231-233): gate order i, f, g, o."""
    gates = _mm(x, w_ih, mm) + b_ih + _mm(h, w_hh, mm) + b_hh
    H = h.shape[-1]
    i = torch.sigmoid(gates[..., 0 * H:1 * H])
    f = torch.sigmoid(gates[..., 1 * H:2 * H])
    g = torch.tanh(gates[..., 2 * H:3 * H])
    o = torch.sigmoid(gates[..., 3 * H:4 * H])
    c_new = f * c + i * g
    h_new = o * torch.tanh(c_new)
    return h_new, c_new


def get_mask_from_lengths(lengths, max_len=None):
    """utils.py:6-10 (device agnostic): True where position < length."""
    if max_len is None:
        max_len = int(lengths.max().item())
    ids = torch.arange(max_len, device=lengths.device)
    return ids.unsqueeze(0) < lengths.unsqueeze(1)


# --------------------------------------------------------------------------------------
# decoder
# --------------------------------------------------------------------------------------

P = "decoder."


def prenet(sd, x, keep1, keep2, mm=None):
    """Prenet.forward model.py:97-100: dropout(p=0.5) is ALWAYS on (training=True hard coded)."""
    w1 = sd[P + "prenet.layers.0.linear_layer.weight"]
    w2 = sd[P + "prenet.layers.1.linear_layer.weight"]
    x = dropout_with_mask(torch.relu(_mm(x, w1, mm)), keep1, 0.5)
    x = dropout_with_mask(torch.relu(_mm(x, w2, mm)), keep2, 0.5)
    return x


def location_layer(sd, aw_cat, mm=None):
    """LocationLayer.forward model.py:22-26: conv1d(2->32, k=31, pad=15, no bias), transpose,
    dense 32->128 (no bias).  aw_cat (B, 2, T) channel 0 = previous weights, 1 = cumulative
    (model.py:358-360)."""
    wc = sd[P + "attention_layer.location_layer.location_conv.conv.weight"]
    wd = sd[P + "attention_layer.location_layer.location_dense.linear_layer.weight"]
    pad = (wc.shape[-1] - 1) // 2
    loc = F.conv1d(aw_cat, wc, padding=pad)            # (B, 32, T)
    return _mm(loc.transpose(1, 2), wd, mm)           # (B, T, 128)


def alignment_energies(sd, query, processed_memory, aw_cat, mm=None):
    """Attention.get_alignment_energies model.py:43-63."""
    wq = sd[P + "attention_layer.query_layer.linear_layer.weight"]
    v = sd[P + "attention_layer.v.linear_layer.weight"]
    pq = _mm(query.unsqueeze(1), wq, mm)                       # (B, 1, 128)
    pa = location_layer(sd, aw_cat, mm)                        # (B, T, 128)
    e = _mm(torch.tanh(pq + pa + processed_memory), v)         # (B, T, 1)
    return e.squeeze(-1)


def attention(sd, ah, memory, processed_memory, aw_cat, mask, score_mask_value=-float("inf"),
              mm=None):
    """Attention.forward model.py:65-86.  ``mask`` True at PADDED positions."""
    e = alignment_energies(sd, ah, processed_memory, aw_cat, mm)
    if mask is not None:
        e = e.masked_fill(mask, score_mask_value)
    aw = torch.softmax(e, dim=1)
    ctx = torch.bmm(aw.unsqueeze(1), memory).squeeze(1)
    return ctx, aw


def init_decoder_state(sd, memory, mm=None):
    """Decoder.initialize_decoder_states model.py:258-289 (+ get_go_frame :243-256)."""
    B, T, _ = memory.shape
    z = lambda n: memory.new_zeros(B, n)
    wm = sd[P + "attention_layer.memory_layer.linear_layer.weight"]
    return dict(ah=z(sd[P + "attention_rnn.weight_hh"].shape[1]),
                ac=z(sd[P + "attention_rnn.weight_hh"].shape[1]),
                dh=z(sd[P + "decoder_rnn.weight_hh"].shape[1]),
                dc=z(sd[P + "decoder_rnn.weight_hh"].shape[1]),
                aw=z(T), awc=z(T), ctx=z(memory.shape[2]),
                pm=_mm(memory, wm, mm))


def decode_step(sd, st, memory, x, mask=None, att_keep=None, dec_keep=None,
                p_att=0.1, p_dec=0.1, score_mask_value=-float("inf"), mm=None):
    """Decoder.decode model.py:340-379.  ``x`` is the prenet output (B, 256); ``st`` is mutated.
    att_keep / dec_keep: training-mode dropout keep masks for the two hidden states (the
    DROPPED hidden state is what recurs, model.py:353-356, 368-371)."""
    ar, dr = P + "attention_rnn.", P + "decoder_rnn."
    cell_in = torch.cat((x, st["ctx"]), -1)                                  # :352
    st["ah"], st["ac"] = lstm_cell(cell_in, st["ah"], st["ac"], sd[ar + "weight_ih"],
                                   sd[ar + "weight_hh"], sd[ar + "bias_ih"],
                                   sd[ar + "bias_hh"], mm)                   # :353-354
    st["ah"] = dropout_with_mask(st["ah"], att_keep, p_att)                  # :355-356
    aw_cat = torch.stack((st["aw"], st["awc"]), dim=1)                       # :358-360
    st["ctx"], st["aw"] = attention(sd, st["ah"], memory, st["pm"], aw_cat, mask,
                                    score_mask_value, mm)                    # :361-363
    st["awc"] = st["awc"] + st["aw"]                                         # :365
    dec_in = torch.cat((st["ah"], st["ctx"]), -1)                            # :366-367
    st["dh"], st["dc"] = lstm_cell(dec_in, st["dh"], st["dc"], sd[dr + "weight_ih"],
                                   sd[dr + "weight_hh"], sd[dr + "bias_ih"],
                                   sd[dr + "bias_hh"], mm)                   # :368-369
    st["dh"] = dropout_with_mask(st["dh"], dec_keep, p_dec)                  # :370-371
    dhc = torch.cat((st["dh"], st["ctx"]), dim=1)                            # :373-374
    mel = _mm(dhc, sd[P + "linear_projection.linear_layer.weight"], mm) + \
        sd[P + "linear_projection.linear_layer.bias"]                        # :375-376
    gate = _mm(dhc, sd[P + "gate_layer.linear_layer.weight"]) + \
        sd[P + "gate_layer.linear_layer.bias"]                               # :378
    return mel, gate, st["aw"]


def decoder_inference(sd, memory, prenet_keep, gate_threshold=0.5, max_decoder_steps=1000,
                      mm=None, return_states=False, att_keep=None, dec_keep=None, training=False):
    """Decoder.inference model.py:418-454, generalised to B>1 with a per-row stop latch
    (SURVEY.md section 8(a) row A9):

      done[b] |= sigmoid(gate[b]) > gate_threshold      (same predicate as model.py:443)
      mel_lengths[b] = index of the first firing step + 1 (the firing frame is included)
      the loop ends when every row has fired or after max_decoder_steps steps; rows that
      fired keep decoding (their later frames are present in the raw outputs).

    For B == 1 this is exactly the reference loop.  ``prenet_keep``: uint8/bool tensor
    (n_steps_cap, 2, B, prenet_dim) of keep masks (step t consumes [t,0] then [t,1]).
    att_keep / dec_keep (n_steps_cap, B, 1024): the hidden-state dropout of decode() (model.py:355-356,
    370-371), applied only when ``training`` (a module in train() mode runs inference with it).
    Returns mel (B, 80, T), gate (B, T, 1), align (B, T, T_enc), mel_lengths (B) int32.
    """
    B = memory.shape[0]
    st = init_decoder_state(sd, memory, mm)
    x = memory.new_zeros(B, sd[P + "prenet.layers.0.linear_layer.weight"].shape[1])
    done = torch.zeros(B, dtype=torch.bool, device=memory.device)
    lengths = torch.zeros(B, dtype=torch.int32, device=memory.device)
    mels, gates, aligns, states = [], [], [], []
    while True:
        t = len(mels)
        px = prenet(sd, x, prenet_keep[t, 0], prenet_keep[t, 1], mm)             # :436
        ak = att_keep[t] if (training and att_keep is not None) else None
        dk = dec_keep[t] if (training and dec_keep is not None) else None
        mel, gate, aw = decode_step(sd, st, memory, px, None, ak, dk, mm=mm)     # :437
        mels.append(mel); gates.append(gate); aligns.append(aw)
        if return_states:
            states.append({k: v.clone() for k, v in st.items() if k != "pm"})
        fire = (torch.sigmoid(gate[:, 0]) > gate_threshold) & ~done              # :443
        lengths[fire] = t + 1
        done |= fire
        if bool(done.all()):
            break
        if len(mels) == max_decoder_steps:                                       # :445-447
            break
        x = mel                                                                  # :449
    lengths[~done] = len(mels)
    mel_o = torch.stack(mels).transpose(0, 1).transpose(1, 2)                    # :311-338
    gate_o = torch.stack(gates).transpose(0, 1).contiguous()
    align_o = torch.stack(aligns).transpose(0, 1)
    if return_states:
        return mel_o, gate_o, align_o, lengths, states
    return mel_o, gate_o, align_o, lengths


def decoder_forward(sd, memory, mels_in, memory_lengths, prenet_keep=None, att_keep=None,
                    dec_keep=None, training=True, score_mask_value=-float("inf"), mm=None):
    """Decoder.forward model.py:381-416 (teacher forcing).  mels_in (B, 80, T_mel).
    prenet_keep (T_mel+1, 2, B, 256) (the prenet runs over go-frame + all T_mel frames at once,
    :396-399; the last frame's output is unused, :405).  att_keep / dec_keep (T_mel, B, 1024)
    are only applied when ``training``."""
    B, n_mel, T_mel = mels_in.shape
    go = memory.new_zeros(1, B, n_mel)                                           # :396
    di = torch.cat((go, mels_in.permute(2, 0, 1)), 0)                            # :397-398
    w1 = sd[P + "prenet.layers.0.linear_layer.weight"]
    w2 = sd[P + "prenet.layers.1.linear_layer.weight"]
    k1 = prenet_keep[:, 0] if prenet_keep is not None else None
    k2 = prenet_keep[:, 1] if prenet_keep is not None else None
    px = dropout_with_mask(torch.relu(_mm(di, w1, mm)), k1, 0.5)
    px = dropout_with_mask(torch.relu(_mm(px, w2, mm)), k2, 0.5)                 # :399
    st = init_decoder_state(sd, memory, mm)
    mask = ~get_mask_from_lengths(memory_lengths, memory.shape[1])               # :401-402
    mels, gates, aligns = [], [], []
    for t in range(T_mel):                                                       # :405
        ak = att_keep[t] if (training and att_keep is not None) else None
        dk = dec_keep[t] if (training and dec_keep is not None) else None
        mel, gate, aw = decode_step(sd, st, memory, px[t], mask, ak, dk,
                                    score_mask_value=score_mask_value, mm=mm)
        mels.append(mel); gates.append(gate[:, 0]); aligns.append(aw)
    mel_o = torch.stack(mels).transpose(0, 1).transpose(1, 2)
    gate_o = torch.stack(gates).transpose(0, 1).contiguous()
    align_o = torch.stack(aligns).transpose(0, 1)
    return mel_o, gate_o, align_o


# --------------------------------------------------------------------------------------
# encoder / postnet / wrapper
# --------------------------------------------------------------------------------------


def batchnorm1d(x, sd, prefix, training, eps=1e-5):
    """nn.BatchNorm1d over (B, C, T).  Eval: running stats.  Training: biased batch statistics
    over (B, T) INCLUDING padded positions (the reference does not mask them)."""
    w, b = sd[prefix + "weight"], sd[prefix + "bias"]
    if training:
        mean = x.mean(dim=(0, 2))
        var = x.var(dim=(0, 2), unbiased=False)
    else:
        mean, var = sd[prefix + "running_mean"], sd[prefix + "running_var"]
    xh = (x - mean[None, :, None]) / torch.sqrt(var[None, :, None] + eps)
    return xh * w[None, :, None] + b[None, :, None]


def conv_bn(x, sd, prefix, training, wgrad_x=None):
    """ConvNorm (layers.py:21-39) + BatchNorm1d as built at model.py:112-139, 157-167.
    wgrad_x: if given, the WEIGHT gradient of the conv is taken with this tensor as its input while the
    value and the input gradient use x (see tacotron2_forward: a side effect of model.py:492)."""
    w, b = sd[prefix + "0.conv.weight"], sd[prefix + "0.conv.bias"]
    pad = (w.shape[-1] - 1) // 2
    if wgrad_x is None:
        y = F.conv1d(x, w, b, padding=pad)
    else:
        yw = F.conv1d(wgrad_x.detach(), w, None, padding=pad)
        y = F.conv1d(x, w.detach(), b, padding=pad) + (yw - yw.detach())
    return batchnorm1d(y, sd, prefix + "1.", training)


def lstm_direction(x, lengths, w_ih, w_hh, b_ih, b_hh, reverse):
    """One direction of nn.LSTM over a padded batch with pack_padded_sequence semantics
    (model.py:180-188): each row runs over its own valid prefix; the reverse direction starts at
    the row's own last valid token; outputs at padded positions are zero."""
    B, T, _ = x.shape
    H = w_hh.shape[1]
    h = x.new_zeros(B, H); c = x.new_zeros(B, H)
    out = x.new_zeros(B, T, H)
    steps = range(T - 1, -1, -1) if reverse else range(T)
    for t in steps:
        valid = (t < lengths).unsqueeze(1)
        hn, cn = lstm_cell(x[:, t], h, c, w_ih, w_hh, b_ih, b_hh)
        h = torch.where(valid, hn, h); c = torch.where(valid, cn, c)
        out[:, t] = torch.where(valid, hn, torch.zeros_like(hn))
    return out


def encoder(sd, x, lengths=None, training=False, keep=None):
    """Encoder.forward model.py:173-190 (lengths given, packed semantics) /
    Encoder.inference :192-201 (lengths None).  x (B, 512, T).  ``keep``: list of 3 dropout keep
    masks (B, 512, T) applied when training (p=0.5)."""
    n = 0
    while ("encoder.convolutions.%d.0.conv.weight" % n) in sd:
        n += 1
    for i in range(n):
        x = torch.relu(conv_bn(x, sd, "encoder.convolutions.%d." % i, training))
        if training and keep is not None:
            x = dropout_with_mask(x, keep[i], 0.5)
    x = x.transpose(1, 2)
    B, T, _ = x.shape
    if lengths is None:
        lengths = torch.full((B,), T, dtype=torch.long, device=x.device)
    l = "encoder.lstm."
    fw = lstm_direction(x, lengths, sd[l + "weight_ih_l0"], sd[l + "weight_hh_l0"],
                        sd[l + "bias_ih_l0"], sd[l + "bias_hh_l0"], False)
    bw = lstm_direction(x, lengths, sd[l + "weight_ih_l0_reverse"],
                        sd[l + "weight_hh_l0_reverse"], sd[l + "bias_ih_l0_reverse"],
                        sd[l + "bias_hh_l0_reverse"], True)
    return torch.cat((fw, bw), -1)


def postnet(sd, x, training=False, keep=None, wgrad_x0=None):
    """Postnet.forward model.py:141-146: tanh on the first n-1 layers, dropout(0.5) when training."""
    n = 0
    while ("postnet.convolutions.%d.0.conv.weight" % n) in sd:
        n += 1
    for i in range(n):
        x = conv_bn(x, sd, "postnet.convolutions.%d." % i, training, wgrad_x0 if i == 0 else None)
        if i < n - 1:
            x = torch.tanh(x)
        if training and keep is not None:
            x = dropout_with_mask(x, keep[i], 0.5)
    return x


def tacotron2_inference(sd, text, prenet_keep, gate_threshold=0.5, max_decoder_steps=1000,
                        training=False, enc_keep=None, att_keep=None, dec_keep=None, post_keep=None):
    """Tacotron2.inference model.py:517-529 (+ batched stop latch, see decoder_inference).
    For B > 1 decoder frames at t >= mel_lengths[b] are zeroed BEFORE the postnet (the same
    convention parse_output uses for training, model.py:487-497); B == 1 is the reference.
    ``training``: the model is in train() mode -- batch statistics in every BatchNorm and the
    encoder / decoder / postnet dropout with the given keep masks (post_keep at the decoded length)."""
    emb = sd["embedding.weight"][text].transpose(1, 2)                           # :518
    memory = encoder(sd, emb, None, training, enc_keep)                          # :519
    mel, gate, align, lengths = decoder_inference(sd, memory, prenet_keep, gate_threshold,
                                                  max_decoder_steps, att_keep=att_keep,
                                                  dec_keep=dec_keep, training=training)  # :520-521
    if mel.shape[0] > 1:
        pad = ~get_mask_from_lengths(lengths.long(), mel.shape[2])
        mel = mel.masked_fill(pad.unsqueeze(1), 0.0)
    post = mel + postnet(sd, mel, training, post_keep)                           # :523-524
    if mel.shape[0] > 1:
        post = post.masked_fill(pad.unsqueeze(1), 0.0)
    return mel, post, gate, align, lengths


def tacotron2_forward(sd, text, text_lengths, mels, output_lengths, prenet_keep=None,
                      att_keep=None, dec_keep=None, enc_keep=None, post_keep=None,
                      training=True, mask_padding=True, score_mask_value=-float("inf")):
    """Tacotron2.forward model.py:499-515 + parse_output :487-497."""
    emb = sd["embedding.weight"][text].transpose(1, 2)                           # :503
    memory = encoder(sd, emb, text_lengths, training, enc_keep)                  # :505
    mel, gate, align = decoder_forward(sd, memory, mels, text_lengths, prenet_keep, att_keep,
                                       dec_keep, training, score_mask_value)     # :507-508
    wgrad_x0 = None
    if mask_padding and output_lengths is not None and torch.is_grad_enabled():
        # Side effect of model.py:492 that the reference's gradients contain: parse_output zeroes the padded frames of
        # mel_outputs IN PLACE through .data after the postnet ran, and that tensor is the input the first postnet
        # conv saved for its backward pass -- autograd therefore computes THAT conv's weight gradient from the masked
        # frames (values and all other gradients are unaffected).  Pinned by tests/golden/grad_*.npz.
        wgrad_x0 = mel.masked_fill((~get_mask_from_lengths(output_lengths, mel.shape[2])).unsqueeze(1), 0.0)
    post = mel + postnet(sd, mel, training, post_keep, wgrad_x0)                 # :510-511
    if mask_padding and output_lengths is not None:                              # :488-495
        pad = ~get_mask_from_lengths(output_lengths, mel.shape[2])
        mel = mel.masked_fill(pad.unsqueeze(1), 0.0)
        post = post.masked_fill(pad.unsqueeze(1), 0.0)
        gate = gate.masked_fill(pad, 1e3)
    return mel, post, gate, align


def tacotron2_loss(mel, post, gate, mel_target, gate_target):
    """Tacotron2Loss.forward loss_function.py:8-19."""
    return F.mse_loss(mel, mel_target) + F.mse_loss(post, mel_target) + \
        F.binary_cross_entropy_with_logits(gate.reshape(-1, 1), gate_target.reshape(-1, 1))
