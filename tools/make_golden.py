"""Generates tests/golden/*.npz by executing the UNMODIFIED reference model.py (needs a checkout of
NVIDIA/tacotron2).  Run:  T2_REFERENCE_DIR=<reference checkout> python tools/make_golden.py [stft|full|grads|live|waveglow|waveglow_configs|denoiser|ragged]

Every file holds the inputs' seeds, the reference outputs and a checksum of the synthetic weights
(tests/common.synth_state_dict) so a drift of the generator is detected instead of silently
mis-comparing.  The reference ships no golden vectors of its own (SURVEY.md section 4); these files
are outputs of the reference itself and are what pins oracle/ and the CUDA path.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.ref_import import (REFERENCE_DIR, MaskInjector, default_hparams, import_reference_model,  # noqa: E402
                               injected_dropout)
from tests.common import (GOLDEN_DIR, keep_mask, rand_text, sample_index, stft_inputs,  # noqa: E402
                          synth_state_dict, tensor_digest, weights_checksum)

torch.set_num_threads(8)
ref = import_reference_model()


def build(sd, training=False):
    model = ref.Tacotron2(default_hparams())
    model.load_state_dict(sd)
    return model.train(training)


def ref_batched_inference(model, text, keep, thr, max_steps):
    """Reference modules driven by a loop that mirrors model.py:435-449 row-wise (the reference's
    own Decoder.inference raises for B > 1, SURVEY.md section 3.1)."""
    dec = model.decoder
    B = text.shape[0]
    masks = [keep[t, l].bool() for t in range(max_steps) for l in range(2)]
    with torch.no_grad(), injected_dropout(ref, MaskInjector(masks)):
        emb = model.embedding(text).transpose(1, 2)
        memory = model.encoder.inference(emb)
        x = dec.get_go_frame(memory)
        dec.initialize_decoder_states(memory, mask=None)
        mels, gates, aligns = [], [], []
        done = torch.zeros(B, dtype=torch.bool); lengths = torch.zeros(B, dtype=torch.int32)
        while True:
            x = dec.prenet(x)
            mel, gate, aw = dec.decode(x)
            mels.append(mel); gates.append(gate); aligns.append(aw)
            fire = (torch.sigmoid(gate.data[:, 0]) > thr) & ~done
            lengths[fire] = len(mels); done |= fire
            if bool(done.all()) or len(mels) == max_steps:
                break
            x = mel
        lengths[~done] = len(mels)
        mel, gate, align = dec.parse_decoder_outputs(mels, gates, aligns)
        mel_masked = mel.clone()
        if B > 1:
            pad = torch.arange(mel.shape[2])[None, :] >= lengths[:, None]
            mel_masked = mel.masked_fill(pad[:, None, :], 0.0)
        post = mel_masked + model.postnet(mel_masked)
        if B > 1:
            post = post.masked_fill(pad[:, None, :], 0.0)
    return memory, mel, mel_masked, post, gate, align, lengths


def calibrate_gate(sd, text, keep, steps, quantile):
    """Pick the gate weight sign and bias so rows stop at different, non-trivial steps: the sign
    makes the gate trend upwards over time, the bias puts the threshold at ``quantile`` of the
    gate values seen after the first 4 steps."""
    sd = dict(sd); sd["decoder.gate_layer.linear_layer.bias"] = torch.zeros(1)
    model = build(sd)
    _, _, _, _, gate, _, _ = ref_batched_inference(model, text, keep, 2.0, steps)
    g = gate[:, :, 0]
    sign = 1.0 if float(g[:, steps // 2:].mean()) > float(g[:, :4].mean()) else -1.0
    g = g * sign
    return sign, -float(torch.quantile(g[:, 4:].flatten(), quantile))


def save(name, **arrays):
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    out = {}
    for k, v in arrays.items():
        out[k] = v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v)
    path = os.path.join(GOLDEN_DIR, name + ".npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


def infer_case(name, B, T_text, max_steps, quantile, wseed, tseed, mseed, wscale=2.0):
    sd = synth_state_dict(wseed, scale=wscale)
    text = rand_text(B, T_text, tseed)
    keep = keep_mask((max_steps, 2, B, 256), 0.5, mseed)
    best = None
    for qq in (quantile, quantile - 0.03, quantile + 0.02, quantile - 0.06, quantile + 0.04):
        sign, bias = calibrate_gate(sd, text, keep, max_steps, qq)
        sd_q = synth_state_dict(wseed, gate_bias=bias, scale=wscale, gate_sign=sign)
        r = ref_batched_inference(build(sd_q), text, keep, 0.5, max_steps)
        lengths, gate = r[6], r[4]
        live = torch.arange(gate.shape[1])[None, :] < lengths[:, None]     # decisions that matter
        margin = float((torch.sigmoid(gate[:, :, 0]) - 0.5).abs()[live].min())
        varied = len(set(lengths.tolist())) > 1 or B == 1
        score = margin if (varied and int(lengths.min()) > 2) else margin * 1e-3
        if best is None or score > best[0]:
            best = (score, sign, bias, sd_q, r, margin)
    _, sign, bias, sd, (memory, mel, mel_masked, post, gate, align, lengths), margin = best
    model = build(sd)
    if B == 1:   # cross-check against the reference's OWN inference() entry point
        model.decoder.max_decoder_steps = max_steps
        masks = [keep[t, l].bool() for t in range(max_steps) for l in range(2)]
        with torch.no_grad(), injected_dropout(ref, MaskInjector(masks)):
            o = model.inference(text)
        assert torch.equal(o[0], mel) and torch.equal(o[1], post) and torch.equal(o[3], align)
        assert torch.equal(o[2], gate)
    print(name, "lengths", lengths.tolist(), "steps", mel.shape[2], "gate margin", margin)
    save(name, B=B, T_text=T_text, max_steps=max_steps, wseed=wseed, wscale=wscale, tseed=tseed, mseed=mseed,
         gate_bias=bias, gate_sign=sign, wsum=weights_checksum(sd), memory=memory, mel=mel, mel_masked=mel_masked,
         mel_post=post, gate=gate, align=align, mel_lengths=lengths, gate_margin=margin)


def ragged_case(name="infer_ragged_b4_t40", lengths=(23, 40, 7, 31), max_steps=40, quantiles=(0.97, 0.95, 0.93, 0.9),
                wseed=1234, tseed=81, mseed=82, wscale=2.0):
    """Texts of different lengths, each run ALONE through the reference's own Tacotron2.inference (B = 1 on
    text[b, :lengths[b]] with the prenet masks keep[:, :, b]).  The engine runs them as one ragged batch
    (input_lengths); the ids past each row's length in `text` are padding it must ignore.  Outputs are stored
    zero-padded to the longest run: mel / mel_post (B, 80, S), gate (B, S, 1), align (B, S, T_text)."""
    B, T_text = len(lengths), max(lengths)
    text = rand_text(B, T_text, tseed)
    keep = keep_mask((max_steps, 2, B, 256), 0.5, mseed)
    bl = int(np.argmax(lengths))

    def run(sd):
        model = build(sd)
        model.decoder.max_decoder_steps = max_steps
        rows = []
        for b, L in enumerate(lengths):
            masks = [keep[t, l, b:b + 1].bool() for t in range(max_steps) for l in range(2)]
            with torch.no_grad(), injected_dropout(ref, MaskInjector(masks)):
                rows.append(model.inference(text[b:b + 1, :L]))
        n = [int(r[0].shape[2]) for r in rows]
        margin = min(float((torch.sigmoid(r[2][0, :, 0]) - 0.5).abs().min()) for r in rows)
        return rows, n, margin

    best = None
    for q in quantiles:
        sign, bias = calibrate_gate(synth_state_dict(wseed, scale=wscale), text[bl:bl + 1, :lengths[bl]],
                                    keep[:, :, bl:bl + 1], max_steps, q)
        sd = synth_state_dict(wseed, gate_bias=bias, scale=wscale, gate_sign=sign)
        rows, n, margin = run(sd)
        score = margin if (len(set(n)) > 2 and min(n) > 2) else margin * 1e-3
        if best is None or score > best[0]:
            best = (score, sign, bias, sd, rows, n, margin)
    _, sign, bias, sd, rows, n, margin = best
    S = max(n)
    mel = torch.zeros(B, 80, S); post = torch.zeros(B, 80, S); gate = torch.zeros(B, S, 1); align = torch.zeros(B, S, T_text)
    for b, (r, nb) in enumerate(zip(rows, n)):
        mel[b, :, :nb] = r[0][0]; post[b, :, :nb] = r[1][0]; gate[b, :nb] = r[2][0]; align[b, :nb, :lengths[b]] = r[3][0]
    print(name, "input lengths", list(lengths), "mel lengths", n, "gate margin", margin)
    save(name, B=B, T_text=T_text, max_steps=max_steps, wseed=wseed, wscale=wscale, tseed=tseed, mseed=mseed,
         gate_bias=bias, gate_sign=sign, wsum=weights_checksum(sd), input_lengths=np.array(lengths), mel=mel,
         mel_post=post, gate=gate, align=align, mel_lengths=np.array(n, dtype=np.int32), gate_margin=margin)


def ref_free_running(model, text, keep, steps):
    """The reference's own prenet / decode modules for exactly `steps` steps, no stop test (rows are independent,
    so the trajectory of a row does not depend on when other rows stop): (memory, mel (B,80,S), gate (B,S), align)."""
    dec = model.decoder
    masks = [keep[t, l].bool() for t in range(steps) for l in range(2)]
    with torch.no_grad(), injected_dropout(ref, MaskInjector(masks)):
        emb = model.embedding(text).transpose(1, 2)
        memory = model.encoder.inference(emb)
        x = dec.get_go_frame(memory)
        dec.initialize_decoder_states(memory, mask=None)
        mels, gates, aligns = [], [], []
        for _ in range(steps):
            x = dec.prenet(x)
            mel, gate, aw = dec.decode(x)
            mels.append(mel); gates.append(gate); aligns.append(aw)
            x = mel
        mel, gate, align = dec.parse_decoder_outputs(mels, gates, aligns)
    return memory, mel, gate[:, :, 0], align


def pick_gate(gate, S):
    """Gate sign and bias (applied to decoder.gate_layer; the gate is not fed back, so the mel trajectory does not depend
    on them) such that rows stop at many different steps, at least one row never fires (the run keeps all S steps) and the
    smallest |gate pre-activation| over the live decisions -- the distance of a stop decision from flipping -- is as
    large as possible.  Only the running maxima of a row matter (a row fires at the first step whose gate exceeds the
    level), so the optimum is the midpoint of the widest gap between consecutive record values that satisfies the
    constraints: exact search, no grid."""
    best = None
    B = gate.shape[0]
    for sign in (1.0, -1.0):
        g = gate.double() * sign
        cm = torch.cummax(g, dim=1)[0]
        rec = torch.unique(cm.flatten())                       # sorted record values of all rows
        gaps = rec[1:] - rec[:-1]
        for j in torch.argsort(gaps, descending=True)[:2000].tolist():
            level = 0.5 * float(rec[j] + rec[j + 1])
            fired = cm > level
            never = ~fired.any(1)
            lengths = torch.where(never, torch.full((B,), S), fired.float().argmax(1) + 1)
            n_never = int(never.sum())
            if n_never < 1 or n_never > B // 4 or int(lengths.min()) < 8 or len(set(lengths.tolist())) < B // 2:
                continue
            live = torch.arange(S)[None, :] < lengths[:, None]
            margin = float((g - level).abs()[live].min())
            if best is None or margin > best[0]:
                best = (margin, sign, -level, lengths.to(torch.int32))
            break                                              # gaps are sorted: the first feasible one is the widest
    assert best is not None, "no gate calibration found"
    return best


FULL_STRIDE, FULL_TAIL, FULL_ALIGN_STRIDE = 25, 8, 100


def full_frame_index(S):
    return sorted(set(range(0, S, FULL_STRIDE)) | set(range(S - FULL_TAIL, S)))


def full_infer_case(name, B, T_text, S, wseed, tseed, mseed, wscale):
    """The configuration a number is QUOTED on (BASELINE.json configs[1] / configs[4] per GPU), all S steps through the
    reference's own modules.  Stored: every 25th frame + the last 8 of mel / mel_postnet, all gates, all mel_lengths,
    the alignment argmax of every step and the alignment rows of every 100th step."""
    sd0 = synth_state_dict(wseed, gate_bias=0.0, scale=wscale)
    text = rand_text(B, T_text, tseed)
    keep = keep_mask((S, 2, B, 256), 0.5, mseed)
    memory, mel, gate0, align = ref_free_running(build(sd0), text, keep, S)
    margin, sign, bias, lengths = pick_gate(gate0, S)
    sd = synth_state_dict(wseed, gate_bias=bias, scale=wscale, gate_sign=sign)
    model = build(sd)
    with torch.no_grad():
        gate = model.decoder.gate_layer.linear_layer.bias + sign * gate0        # what the calibrated reference outputs
        pad = torch.arange(S)[None, :] >= lengths[:, None]
        mel_masked = mel.masked_fill(pad[:, None, :], 0.0)
        post = (mel_masked + model.postnet(mel_masked)).masked_fill(pad[:, None, :], 0.0)
    if B <= 8 or os.environ.get("T2_GOLDEN_VERIFY", "1") == "1":   # the calibrated model, stop test on, gives the same thing
        r = ref_batched_inference(model, text, keep, 0.5, S)
        assert r[6].tolist() == lengths.tolist(), (r[6].tolist(), lengths.tolist())
        assert torch.equal(r[1], mel) and torch.equal(r[3], post) and torch.allclose(r[4][:, :, 0], gate, atol=1e-6)
        gate = r[4][:, :, 0]
    idx = torch.tensor(full_frame_index(S))
    aidx = torch.arange(0, S, FULL_ALIGN_STRIDE)
    print(name, "lengths min/max", int(lengths.min()), int(lengths.max()), "distinct", len(set(lengths.tolist())),
          "gate pre-activation margin %.3e" % margin)
    save(name, B=B, T_text=T_text, max_steps=S, wseed=wseed, wscale=wscale, tseed=tseed, mseed=mseed, gate_bias=bias,
         gate_sign=sign, wsum=weights_checksum(sd), frame_index=idx, align_index=aidx, mel_masked=mel_masked[:, :, idx],
         mel_raw=mel[:, :, idx], mel_post=post[:, :, idx], gate=gate, mel_lengths=lengths, gate_margin=margin,
         align_argmax=align.argmax(-1).to(torch.int16), align_max=align.max(-1)[0], align_rows=align[:, aidx],
         memory_abs_sum=memory.double().abs().sum())


def forward_case(name, training, B, T_text, T_mel, wseed, seed, wscale=2.0):
    sd = synth_state_dict(wseed, scale=wscale)
    g = torch.Generator().manual_seed(seed)
    text = rand_text(B, T_text, seed + 1)
    tl = torch.sort(torch.randint(T_text // 3, T_text + 1, (B,), generator=g), descending=True)[0]
    tl[0] = T_text
    ol = torch.randint(T_mel // 3, T_mel + 1, (B,), generator=g); ol[1] = T_mel
    mels = torch.randn(B, 80, T_mel, generator=g)
    pk = keep_mask((T_mel + 1, 2, B, 256), 0.5, seed + 2)
    ak = keep_mask((T_mel, B, 1024), 0.1, seed + 3)
    dk = keep_mask((T_mel, B, 1024), 0.1, seed + 4)
    ek = keep_mask((3, B, 512, T_text), 0.5, seed + 5)
    qk4 = keep_mask((4, B, 512, T_mel), 0.5, seed + 6)
    qk1 = keep_mask((B, 80, T_mel), 0.5, seed + 7)
    model = build(sd, training)
    if training:
        masks = [ek[i].bool() for i in range(3)] + [pk[:, 0].bool(), pk[:, 1].bool()]
        for t in range(T_mel):
            masks += [ak[t].bool(), dk[t].bool()]
        masks += [qk4[i].bool() for i in range(4)] + [qk1.bool()]
    else:
        masks = [pk[:, 0].bool(), pk[:, 1].bool()]
    with torch.no_grad(), injected_dropout(ref, MaskInjector(masks)) as inj:
        emb = model.embedding(text).transpose(1, 2)
    with torch.no_grad(), injected_dropout(ref, MaskInjector(masks)) as inj:
        out = model((text, tl, mels, int(tl.max()), ol))
        assert inj.calls == len(masks)
    sd_after = model.state_dict()
    save(name, training=int(training), B=B, T_text=T_text, T_mel=T_mel, wseed=wseed, seed=seed, wscale=wscale,
         wsum=weights_checksum(sd), text_lengths=tl, output_lengths=ol, mels_in=mels,
         mel=out[0], mel_post=out[1], gate=out[2], align=out[3],
         bn0_running_mean=sd_after["encoder.convolutions.0.1.running_mean"],
         bn0_running_var=sd_after["encoder.convolutions.0.1.running_var"])


def grad_sample_index(name, numel, n=96):
    """Deterministic flat indices at which the gradient of parameter `name` is stored in the fixture."""
    h = 0
    for ch in name:
        h = (h * 131 + ord(ch)) % 2147483647
    g = torch.Generator().manual_seed(h)
    return torch.randint(0, numel, (min(n, numel),), generator=g)


def gate_targets(ol, T_mel):
    """data_utils.py:105-107: gate_padded[i, len_i - 1:] = 1."""
    gt = torch.zeros(len(ol), T_mel)
    for i, n in enumerate(ol.tolist()):
        gt[i, n - 1:] = 1.0
    return gt


def import_reference_loss():
    import importlib.util
    spec = importlib.util.spec_from_file_location("ref_loss_function", os.path.join(REFERENCE_DIR, "loss_function.py"))
    lf = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(lf)
    return lf


def grad_case(name, training, B, T_text, T_mel, wseed, seed, wscale=2.0, n_samples=96, keep_outputs=True,
              ref64=False):
    """Full training step of the REFERENCE (forward + Tacotron2Loss + backward, autograd) with injected dropout
    masks; the fixture keeps the loss and, per parameter, sum / abs-sum / max of the gradient plus 96 sampled entries."""
    import importlib.util
    lf = import_reference_loss()
    sd = synth_state_dict(wseed, scale=wscale)
    g = torch.Generator().manual_seed(seed)
    text = rand_text(B, T_text, seed + 1)
    tl = torch.sort(torch.randint(T_text // 3, T_text + 1, (B,), generator=g), descending=True)[0]
    tl[0] = T_text
    ol = torch.randint(T_mel // 3, T_mel + 1, (B,), generator=g); ol[1] = T_mel
    mels = torch.randn(B, 80, T_mel, generator=g)
    for i, n in enumerate(ol.tolist()):
        mels[i, :, n:] = 0.0                                    # TextMelCollate zero-pads (data_utils.py:97-104)
    pk = keep_mask((T_mel + 1, 2, B, 256), 0.5, seed + 2)
    ak = keep_mask((T_mel, B, 1024), 0.1, seed + 3)
    dk = keep_mask((T_mel, B, 1024), 0.1, seed + 4)
    ek = keep_mask((3, B, 512, T_text), 0.5, seed + 5)
    qk4 = keep_mask((4, B, 512, T_mel), 0.5, seed + 6)
    qk1 = keep_mask((B, 80, T_mel), 0.5, seed + 7)
    model = build(sd, training)
    if training:
        masks = [ek[i].bool() for i in range(3)] + [pk[:, 0].bool(), pk[:, 1].bool()]
        for t in range(T_mel):
            masks += [ak[t].bool(), dk[t].bool()]
        masks += [qk4[i].bool() for i in range(4)] + [qk1.bool()]
    else:
        masks = [pk[:, 0].bool(), pk[:, 1].bool()]
    gt = gate_targets(ol, T_mel)
    with injected_dropout(ref, MaskInjector(masks)) as inj:
        out = model((text, tl, mels, int(tl.max()), ol))
        assert inj.calls == len(masks)
    loss = lf.Tacotron2Loss()(out, (mels, gt))
    loss.backward()
    arrays = dict(training=int(training), B=B, T_text=T_text, T_mel=T_mel, wseed=wseed, seed=seed, wscale=wscale,
                  wsum=weights_checksum(sd), text_lengths=tl, output_lengths=ol, mels_in=mels, gate_target=gt,
                  loss=loss.detach(), mel=out[0].detach(), mel_post=out[1].detach(), n_samples=n_samples)
    if not keep_outputs:      # full-size case: the inputs are regenerated from the seeds, outputs sub-sampled in time
        idx = torch.tensor(full_frame_index(T_mel))
        arrays.update(mel=out[0].detach()[:, :, idx], mel_post=out[1].detach()[:, :, idx], frame_index=idx, gate=out[2].detach())
        del arrays["mels_in"], arrays["gate_target"]
    for k, p_ in model.named_parameters():
        gr = p_.grad.detach().double().reshape(-1)
        idx = grad_sample_index(k, gr.numel(), n_samples)
        arrays["g/" + k] = torch.cat((torch.stack((gr.sum(), gr.abs().sum(), gr.abs().max())), gr[idx]))
    if ref64:
        # The same step through the reference in DOUBLE precision (model.double()): at B=64 / T_mel=800 the reference's
        # fp32 autograd is itself 1e-3 ... 1e-2 (relative to the gradient's maximum) away from this for the parameters
        # behind the training-mode BatchNorms (DESIGN.md section 2), so the fp64 values are what an fp32-grade
        # implementation is held to, with the fp32 reference's own deviation as the yardstick.
        model64 = build(sd, training).double()
        with injected_dropout(ref, MaskInjector(masks)) as inj:
            out64 = model64((text, tl, mels.double(), int(tl.max()), ol))
        loss64 = lf.Tacotron2Loss()(out64, (mels.double(), gt.double()))
        loss64.backward()
        arrays["loss64"] = loss64.detach()
        worst = {}
        for k, p_ in model64.named_parameters():
            gr = p_.grad.detach().reshape(-1)
            idx = grad_sample_index(k, gr.numel(), n_samples)
            arrays["g64/" + k] = torch.cat((torch.stack((gr.sum(), gr.abs().sum(), gr.abs().max())), gr[idx]))
            gmax = float(gr.abs().max())
            if gmax > 1e-5:
                worst[k] = float((torch.as_tensor(arrays["g/" + k])[3:] - gr[idx]).abs().max()) / gmax
        top = sorted(worst.items(), key=lambda kv: -kv[1])[:8]
        print(name, "fp32 reference vs fp64 reference, largest sampled deviations / max|g|:",
              ", ".join("%s %.1e" % kv for kv in top))
    print(name, "loss", float(loss))
    save(name, **arrays)


def import_reference_stft():
    """The reference's stft.py with functional stand-ins for the two librosa.util helpers it imports (librosa itself is
    not in this image): pad_center = symmetric zero padding, tiny = smallest normal float32."""
    import importlib.util
    import types

    def pad_center(data, size, axis=-1, **kw):
        n = data.shape[axis]
        lpad = int((size - n) // 2)
        lengths = [(0, 0)] * data.ndim
        lengths[axis] = (lpad, int(size - n - lpad))
        return np.pad(data, lengths, mode="constant")
    saved = {k: sys.modules.get(k) for k in ("librosa", "librosa.util", "librosa.filters", "audio_processing", "stft")}
    lib, lu, lf = types.ModuleType("librosa"), types.ModuleType("librosa.util"), types.ModuleType("librosa.filters")
    lu.pad_center, lu.tiny, lf.mel = pad_center, (lambda x: np.finfo(np.float32).tiny), None
    lib.util, lib.filters = lu, lf
    sys.modules.update({"librosa": lib, "librosa.util": lu, "librosa.filters": lf})
    sys.path.insert(0, REFERENCE_DIR)
    try:
        spec = importlib.util.spec_from_file_location("t2_reference_stft", os.path.join(REFERENCE_DIR, "stft.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        sys.path.remove(REFERENCE_DIR)
        for k, v in saved.items():
            sys.modules.pop(k, None)
            if v is not None:
                sys.modules[k] = v
    return mod


def stft_case():
    """STFT magnitudes of the reference's own stft.STFT(1024, 256, 1024) (stft.py:69-94) for a seeded 2-row signal."""
    mod = import_reference_stft()
    ref_stft = mod.STFT(1024, 256, 1024)
    y = stft_inputs()
    mag, _ = ref_stft.transform(y)
    save("stft_mag", y=y, mag=mag, basis_abs_sum=ref_stft.forward_basis.double().abs().sum())


def import_reference_data_utils():
    """The reference's data_utils.py with empty stand-ins for the modules only its dataset class needs."""
    import importlib.util
    import types
    saved = {k: sys.modules.get(k) for k in ("layers", "utils", "text", "librosa", "librosa.filters", "librosa.util",
                                             "stft", "audio_processing")}
    try:
        for k in ("layers", "utils", "text"):
            sys.modules[k] = types.ModuleType(k)
        sys.modules["utils"].load_wav_to_torch = sys.modules["utils"].load_filepaths_and_text = None
        sys.modules["text"].text_to_sequence = None
        spec = importlib.util.spec_from_file_location("t2_reference_data_utils", os.path.join(REFERENCE_DIR, "data_utils.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        for k, v in saved.items():
            sys.modules.pop(k, None)
            if v is not None:
                sys.modules[k] = v
    return mod


def collate_batches(nfs_list=(1, 2), trials=20):
    """The text / mel batches of tests/test_boundary_cpu.py::test_text_mel_collate_matches_reference_semantics, in order:
    per n_frames_per_step the fixed 5-row batch, then `trials` random ragged batches (ties in the text lengths included)."""
    g = torch.Generator().manual_seed(0)
    fixed = [(torch.randint(1, 148, (n_text,), generator=g), torch.randn(80, n_mel, generator=g))
             for n_text, n_mel in [(7, 13), (12, 5), (3, 21), (12, 9), (1, 1)]]
    out = []
    for nfs in nfs_list:
        out.append((nfs, fixed))
        for _ in range(trials):
            n = int(torch.randint(1, 9, (1,), generator=g))
            out.append((nfs, [(torch.randint(1, 148, (int(torch.randint(1, 12, (1,), generator=g)),), generator=g),
                               torch.randn(80, int(torch.randint(1, 30, (1,), generator=g)), generator=g)) for _ in range(n)]))
    return out


def reference_live_case():
    """What tests/test_oracle_vs_reference.py and the collate test compare against, computed by the reference itself:
    batched inference (B=1, 12 steps), the state_dict layout and seeded initialisation, a full training step's loss / gradients (sum, abs-sum, max,
    sum of squares and 96 sampled entries per parameter), stft.STFT bases (sampled) and magnitudes for three filter / hop
    settings, and TextMelCollate on the batches of collate_batches()."""
    arrays = {}
    # inference, B=1: model.inference with injected prenet masks
    sd = synth_state_dict(5, gate_bias=-10.0, scale=2.0)
    model = build(sd)
    model.decoder.max_decoder_steps = 12
    text = rand_text(1, 19, 3)
    keep = keep_mask((12, 2, 1, 256), 0.5, 4)
    masks = [keep[t, l].bool() for t in range(12) for l in range(2)]
    with torch.no_grad(), injected_dropout(ref, MaskInjector(masks)):
        r = model.inference(text)
    for k, v in zip(("mel", "post", "gate", "align"), r):
        arrays["infer/" + k] = v
    # state_dict layout, and the initialisation under torch.manual_seed(1234) as SHA-256 digests of every tensor's bytes
    torch.manual_seed(1234)
    sdr = ref.Tacotron2(default_hparams()).state_dict()
    arrays["init1234/digest"] = np.array([tensor_digest(v) for v in sdr.values()])
    arrays["sd/keys"] = np.array(list(sdr.keys()))
    arrays["sd/shapes"] = np.array([list(v.shape) + [0] * (4 - v.dim()) for v in sdr.values()], dtype=np.int64)
    # training step (tests/test_oracle_vs_reference.py::test_reference_training_step_gradients_live)
    lf = import_reference_loss()
    B, T, Tm, seed = 3, 15, 8, 91
    sd = synth_state_dict(4321, scale=2.0)
    g = torch.Generator().manual_seed(seed)
    text = rand_text(B, T, seed + 1)
    tl = torch.sort(torch.randint(T // 3, T + 1, (B,), generator=g), descending=True)[0]
    tl[0] = T
    ol = torch.randint(Tm // 3, Tm + 1, (B,), generator=g)
    ol[1] = Tm
    mels = torch.randn(B, 80, Tm, generator=g)
    gt = torch.zeros(B, Tm)
    for i, n in enumerate(ol.tolist()):
        mels[i, :, n:] = 0.0
        gt[i, n - 1:] = 1.0
    m = dict(pk=keep_mask((Tm + 1, 2, B, 256), 0.5, seed + 2), ak=keep_mask((Tm, B, 1024), 0.1, seed + 3),
             dk=keep_mask((Tm, B, 1024), 0.1, seed + 4), ek=keep_mask((3, B, 512, T), 0.5, seed + 5),
             qk4=keep_mask((4, B, 512, Tm), 0.5, seed + 6), qk1=keep_mask((B, 80, Tm), 0.5, seed + 7))
    model = build(sd, True)
    masks = [m["ek"][i].bool() for i in range(3)] + [m["pk"][:, 0].bool(), m["pk"][:, 1].bool()]
    for t in range(Tm):
        masks += [m["ak"][t].bool(), m["dk"][t].bool()]
    masks += [m["qk4"][i].bool() for i in range(4)] + [m["qk1"].bool()]
    with injected_dropout(ref, MaskInjector(masks)):
        out = model((text, tl, mels, int(tl.max()), ol))
    loss = lf.Tacotron2Loss()(out, (mels, gt))
    loss.backward()
    arrays["train/loss"] = loss.detach()
    for k, p_ in model.named_parameters():
        gr = p_.grad.detach().double().reshape(-1)
        idx = grad_sample_index(k, gr.numel())
        arrays["train/g/" + k] = torch.cat((torch.stack((gr.sum(), gr.abs().sum(), gr.abs().max(), (gr * gr).sum())), gr[idx]))
    # stft.STFT
    mod = import_reference_stft()
    for fl, hop, win in ((1024, 256, 1024), (800, 200, 800), (512, 128, 400)):
        st = mod.STFT(fl, hop, win)
        y = stft_inputs(seed=fl, n=5000)
        mag, _ = st.transform(y)
        for name, v in (("basis", st.forward_basis[:, 0, :]), ("mag", mag)):
            v = v.detach().double().reshape(-1)
            arrays["stft/%d/%s_shape" % (fl, name)] = np.array((st.forward_basis[:, 0, :] if name == "basis" else mag).shape)
            arrays["stft/%d/%s_sample" % (fl, name)] = v[sample_index(v.numel(), 2048, fl)]
            arrays["stft/%d/%s_stats" % (fl, name)] = torch.stack((v.sum(), v.abs().sum(), (v * v).sum(), v.abs().max()))
    # TextMelCollate
    du = import_reference_data_utils()
    arrays["collate/digest"] = np.array([[tensor_digest(v) for v in du.TextMelCollate(nfs)(batch)]
                                         for nfs, batch in collate_batches()])
    save("reference_live", **arrays)


# ---- WaveGlow (waveglow/glow.py, run on the CPU with the noise injected) ----------------------------------------
def import_reference_glow(z_queue):
    """The reference's glow.py with one shim: ``torch.cuda.FloatTensor(*size).normal_()`` (glow.py:265, 289) returns
    the next injected draw from ``z_queue`` instead of touching CUDA."""
    import importlib.util
    import types
    spec = importlib.util.spec_from_file_location("t2_reference_glow", os.path.join(REFERENCE_DIR, "waveglow", "glow.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)

    class _Draw:
        def __init__(self, *size):
            self.size = tuple(size)

        def normal_(self):
            z = z_queue.pop(0)
            assert tuple(z.shape) == self.size, (tuple(z.shape), self.size)
            return z.clone()

    class _TorchProxy(types.ModuleType):
        def __getattr__(self, name):
            return getattr(torch, name)

    proxy = _TorchProxy("torch")
    proxy.cuda = types.SimpleNamespace(FloatTensor=_Draw, HalfTensor=_Draw)
    mod.torch = proxy
    return mod


def reference_waveglow_infer(sd, mel, sigma, z):
    """Reference WaveGlow.infer with z (B, 8, L) split into its three draws in draw order."""
    from tests.waveglow_common import CONFIG
    queue = [z[:, 0:4].contiguous(), z[:, 4:6].contiguous(), z[:, 6:8].contiguous()]
    glow = import_reference_glow(queue)
    model = glow.WaveGlow(**CONFIG)
    model.load_state_dict(sd)
    with torch.no_grad():
        out = model.infer(mel, sigma=sigma)
    assert not queue
    return out


def waveglow_init_case():
    from tests.waveglow_common import CONFIG
    glow = import_reference_glow([])
    torch.manual_seed(1234)
    model = glow.WaveGlow(**CONFIG)
    sd = model.state_dict()
    keys = list(sd)
    shapes = [",".join(str(x) for x in sd[k].shape) for k in keys]
    digests = [tensor_digest(sd[k]) for k in keys]
    model = glow.WaveGlow.remove_weightnorm(model)
    sd2 = model.state_dict()
    save("waveglow_init", keys=np.array(keys), shapes=np.array(shapes), digests=np.array(digests),
         removed_keys=np.array(list(sd2)), removed_digests=np.array([tensor_digest(sd2[k]) for k in sd2]))


def waveglow_infer_case(name, B, T, sigma, wseed, mseed, zseed):
    from tests.waveglow_common import mel_input, noise, synth_state_dict
    sd = synth_state_dict(wseed)
    mel, z = mel_input(B, T, mseed), noise(B, T, zseed)
    audio = reference_waveglow_infer(sd, mel, sigma, z)
    save(name, mel=mel, z=z, audio=audio, sigma=sigma, wseed=wseed, checksum=weights_checksum(sd))


def waveglow_full_case(name, B, T, sigma, wseed, mseed, zseed, n_samples=4096):
    """Large fixture: inputs regenerated from their seeds, outputs as seeded sample entries + full-tensor statistics."""
    from tests.waveglow_common import mel_input, noise, synth_state_dict
    sd = synth_state_dict(wseed)
    mel, z = mel_input(B, T, mseed), noise(B, T, zseed)
    audio = reference_waveglow_infer(sd, mel, sigma, z)
    idx = sample_index(audio.numel(), n_samples, 5)
    a = audio.double()
    save(name, B=B, T=T, sigma=sigma, wseed=wseed, mseed=mseed, zseed=zseed, checksum=weights_checksum(sd),
         mel_digest=tensor_digest(mel), z_digest=tensor_digest(z), idx=idx, samples=audio.reshape(-1)[idx],
         stats=np.array([float(a.mean()), float(a.std()), float(a.abs().max()), float(a.abs().mean())]))


def waveglow_configs_case():
    """The reference's WaveGlow.infer for the configurations of tests/waveglow_configs.FIXTURE_CASES, one npz: per case
    ``<name>/mel``, ``/z`` (draw order), ``/audio``, ``/sigma``, ``/wseed`` and ``/checksum``."""
    from tacotron2_b200.glow import noise_channel_order
    from tests.waveglow_configs import FIXTURE_CASES, fixture_inputs, name_of, state_dict_for
    arrays = {}
    for cfg, B, T, sigma, wseed, mseed, zseed in FIXTURE_CASES:
        sd = state_dict_for(cfg, wseed)
        mel, z = fixture_inputs(B, T, mseed, zseed)
        queue, c0 = [], 0
        for _, n in noise_channel_order(cfg["n_flows"], cfg["n_group"], cfg["n_early_every"], cfg["n_early_size"]):
            queue.append(z[:, c0:c0 + n].contiguous())
            c0 += n
        glow = import_reference_glow(queue)
        model = glow.WaveGlow(**cfg)
        model.load_state_dict(sd)
        with torch.no_grad():
            audio = model.infer(mel, sigma=sigma)
        assert not queue
        name = name_of(cfg)
        print(name, tuple(audio.shape), float(audio.abs().max()))
        arrays.update({name + "/mel": mel, name + "/z": z, name + "/audio": audio, name + "/sigma": sigma,
                       name + "/wseed": wseed, name + "/checksum": weights_checksum(sd)})
    save("waveglow_configs", **arrays)


def waveglow_cases():
    waveglow_init_case()
    waveglow_infer_case("waveglow_b1_t50_s0", 1, 50, 0.0, 7, 41, 42)
    waveglow_infer_case("waveglow_b3_t37_s666", 3, 37, 0.666, 7, 43, 44)
    waveglow_full_case("waveglow_full_b2_t800", 2, 800, 0.666, 7, 45, 46)


def denoiser_case(seed=3, n=256 * 40 + 100, strengths=(0.01, 0.1, 3.0), n_samples=4096):
    """The reference's own waveglow/denoiser.py on the CPU: bias_spec of the reference WaveGlow with
    synth_state_dict(7) (fp32, mode 'zeros'), both bases, and the denoised seeded 2-row signal stft_inputs(seed, n) at
    three strengths.  Shims: the librosa stand-ins of import_reference_stft plus normalize, the noise shim of
    import_reference_glow (sigma = 0, so the draws are zeros), and .cuda() as a no-op while the fixture is made."""
    import importlib.util
    import types
    from tests.waveglow_common import CONFIG, synth_state_dict

    def pad_center(data, size, axis=-1, **kw):
        n_ = data.shape[axis]
        lpad = int((size - n_) // 2)
        lengths = [(0, 0)] * data.ndim
        lengths[axis] = (lpad, int(size - n_ - lpad))
        return np.pad(data, lengths, mode="constant")

    def normalize(S, norm=np.inf, **kw):       # audio_processing.py:48 calls it with norm=None: no normalisation
        assert norm is None
        return S
    names = ("librosa", "librosa.util", "librosa.filters", "audio_processing", "stft", "layers")
    saved = {k: sys.modules.get(k) for k in names}
    lib, lu, lf = types.ModuleType("librosa"), types.ModuleType("librosa.util"), types.ModuleType("librosa.filters")
    lu.pad_center, lu.tiny, lu.normalize, lf.mel = pad_center, (lambda x: np.finfo(np.float32).tiny), normalize, None
    lib.util, lib.filters = lu, lf
    sys.modules.update({"librosa": lib, "librosa.util": lu, "librosa.filters": lf})
    for k in ("audio_processing", "stft", "layers"):
        sys.modules.pop(k, None)
    module_cuda, tensor_cuda = torch.nn.Module.cuda, torch.Tensor.cuda
    torch.nn.Module.cuda = lambda self, *a, **kw: self
    torch.Tensor.cuda = lambda self, *a, **kw: self
    sys.path.insert(0, REFERENCE_DIR)
    try:
        spec = importlib.util.spec_from_file_location("t2_reference_denoiser",
                                                      os.path.join(REFERENCE_DIR, "waveglow", "denoiser.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        L = 88 * 32
        glow = import_reference_glow([torch.zeros(1, 4, L), torch.zeros(1, 2, L), torch.zeros(1, 2, L)])
        sd = synth_state_dict(7)
        model = glow.WaveGlow(**CONFIG)
        model.load_state_dict(sd)
        den = mod.Denoiser(model)
        y = stft_inputs(seed, n)
        with torch.no_grad():
            outs = {"out_%g" % s: den(y, strength=s) for s in strengths}
        sdict = den.state_dict()
    finally:
        torch.nn.Module.cuda, torch.Tensor.cuda = module_cuda, tensor_cuda
        sys.path.remove(REFERENCE_DIR)
        for k, v in saved.items():
            sys.modules.pop(k, None)
            if v is not None:
                sys.modules[k] = v
    fb, ib = sdict["stft.forward_basis"], sdict["stft.inverse_basis"]
    idx = sample_index(fb.numel(), n_samples, 7)
    stats = lambda t: np.array([float(t.double().sum()), float(t.double().abs().sum()), float(t.double().abs().max())])  # noqa: E731
    for s in strengths:
        mag = den.stft.transform(y)[0]
        print("strength %g: %.1f %% of the bins clamp to 0" % (s, 100.0 * float((mag - den.bias_spec * s <= 0).double().mean())))
    save("denoiser_b2", seed=seed, n=n, strengths=np.array(strengths), wseed=7, checksum=weights_checksum(sd),
         keys=np.array(list(sdict)), shapes=np.array([",".join(str(x) for x in sdict[k].shape) for k in sdict]),
         bias_spec=sdict["bias_spec"], basis_idx=idx, forward_samples=fb.reshape(-1)[idx],
         inverse_samples=ib.reshape(-1)[idx], forward_stats=stats(fb), inverse_stats=stats(ib), **outs)


def griffin_lim_case(seed=5, n=256 * 24 + 100, np_seed=1234, iters=(0, 1, 30)):
    """The reference's own audio_processing.griffin_lim over its stft.STFT(1024, 256, 1024) on the CPU: the target is
    the magnitude of the seeded 2-row signal stft_inputs(seed, n); before each call np.random.seed(np_seed), so every
    run starts from the same angles.  Shims: the librosa stand-ins of denoiser_case."""
    import importlib.util
    import types

    def pad_center(data, size, axis=-1, **kw):
        n_ = data.shape[axis]
        lpad = int((size - n_) // 2)
        lengths = [(0, 0)] * data.ndim
        lengths[axis] = (lpad, int(size - n_ - lpad))
        return np.pad(data, lengths, mode="constant")

    def normalize(S, norm=np.inf, **kw):       # audio_processing.py:48 calls it with norm=None: no normalisation
        assert norm is None
        return S
    names = ("librosa", "librosa.util", "librosa.filters", "audio_processing", "stft")
    saved = {k: sys.modules.get(k) for k in names}
    lib, lu, lf = types.ModuleType("librosa"), types.ModuleType("librosa.util"), types.ModuleType("librosa.filters")
    lu.pad_center, lu.tiny, lu.normalize, lf.mel = pad_center, (lambda x: np.finfo(np.float32).tiny), normalize, None
    lib.util, lib.filters = lu, lf
    sys.modules.update({"librosa": lib, "librosa.util": lu, "librosa.filters": lf})
    for k in ("audio_processing", "stft"):
        sys.modules.pop(k, None)
    sys.path.insert(0, REFERENCE_DIR)
    try:
        spec = importlib.util.spec_from_file_location("audio_processing", os.path.join(REFERENCE_DIR, "audio_processing.py"))
        ap = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(ap)
        sys.modules["audio_processing"] = ap
        spec = importlib.util.spec_from_file_location("t2_reference_stft", os.path.join(REFERENCE_DIR, "stft.py"))
        st = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(st)
        stft_fn = st.STFT(1024, 256, 1024)
        y = stft_inputs(seed, n)
        with torch.no_grad():
            mag, _ = stft_fn.transform(y)
            outs = {}
            for k in iters:
                np.random.seed(np_seed)
                outs["out_%d" % k] = ap.griffin_lim(mag, stft_fn, n_iters=k)
    finally:
        sys.path.remove(REFERENCE_DIR)
        for k, v in saved.items():
            sys.modules.pop(k, None)
            if v is not None:
                sys.modules[k] = v
    save("griffin_lim_b2", seed=seed, n=n, np_seed=np_seed, iters=np.array(iters), mag=mag, **outs)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "ragged":
        ragged_case()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "denoiser":
        denoiser_case()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "griffin_lim":
        griffin_lim_case()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "waveglow":
        waveglow_cases()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "waveglow_configs":
        waveglow_configs_case()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "live":
        reference_live_case()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "stft":
        stft_case()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "full":        # the configurations the benchmark numbers are quoted on
        which = sys.argv[2:] or ["infer64", "infer32", "grad64"]
        if "infer64" in which:   # BASELINE.json configs[1]: B=64, T_text=150, 800 steps, the bench weights (scale 1.0)
            full_infer_case("full_infer_b64_t150_s800", 64, 150, 800, 1234, 101, 102, 1.0)
        if "infer32" in which:   # configs[4] per GPU: B=32, T_text=300, 2000 steps
            full_infer_case("full_infer_b32_t300_s2000", 32, 300, 2000, 1234, 111, 112, 1.0)
        if "grad64" in which:    # configs[2]: teacher-forced training step B=64, T_mel=800
            grad_case("full_grad_train_b64_t150_m800", True, 64, 150, 800, 1234, 160, wscale=1.0, n_samples=1024,
                      keep_outputs=False, ref64=True)
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "grads":
        grad_case("grad_train_b4", True, 4, 24, 12, 1234, 60)
        grad_case("grad_eval_b3", False, 3, 17, 9, 77, 70)
        sys.exit(0)
    infer_case("infer_b1_t50", 1, 50, 40, 0.95, 1234, 11, 12)
    infer_case("infer_b4_t24", 4, 24, 32, 0.93, 1234, 21, 22)
    infer_case("infer_b3_t37", 3, 37, 16, 0.90, 77, 31, 32, wscale=1.0)
    forward_case("forward_train_b4", True, 4, 24, 12, 1234, 40)
    forward_case("forward_eval_b4", False, 4, 24, 12, 1234, 50)
