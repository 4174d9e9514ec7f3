"""The training backward across gradient scales, zero-gradient channels, its K-split regimes and the inference conv tiles,
against the oracle in float64; the training-mode conv stack forward without autograd.

Every gradient comes from three split-fp16 engines: gemm_tc (the LSTM products and the forward convs), wgrad_tc (the decoder
LSTM and the conv weight gradients) and wg_gemm with its conv epilogue (the conv input gradients, through conv_tc).  Each
scales its fp32 operands by powers of two before splitting them into fp16 hi / lo halves, so:

* A backward is linear in its upstream gradient and every scale is a power of two: multiplying the seeds by 2^k must
  multiply every gradient by exactly 2^k (bit for bit), at any magnitude and with channels whose gradient is all zero (a
  dead ReLU, a BatchNorm gamma of 0).  Real upstream gradients are small: Tacotron2Loss is a mean over B x 80 x T_mel
  elements, and the full-size training step prints the gradients at the BatchNorm inputs (max |G_z| per layer).
* wgrad_tc splits its K dimension (decoder steps, or 64-row chunks of the conv's padded rows) into segments of
  wgrad_seg(n) = 100 chunks, 150 once there would be more than 15 segments; the cases below land on full, partial and
  single-chunk last segments and on both sides of the switch.
* wg_gemm runs a conv on 128-row tiles of the padded rows, in clusters of 2 (an odd tile count adds a padding tile).

Bars: 1e-3 relative (max |a - b| / max |b|) on gradients, as tests/test_gpu_backward.py; 1e-4 on Encoder and Postnet
outputs, as tests/test_gpu_parity.py.  Every case prints its worst error."""
import contextlib
import math

import pytest
import torch

import tacotron2_b200 as t2
from oracle import tacotron2_oracle as O
from tests.common import keep_mask, rand_text, rel_err, synth_state_dict
from tests.test_oracle_golden import grad_inputs, load, oracle_train_step

pytestmark = pytest.mark.gpu
TOL = 1e-3
INFER_TOL = 1e-4
ZC = 5                      # the channel forced to an all-zero gradient
ZERO_LAYER = {"encoder": "encoder.convolutions.1.", "postnet": "postnet.convolutions.2."}


def weights(zero=None):
    """Synthetic weights; zero = "encoder": beta = -50 on one channel of encoder conv layer 1, so its ReLU is dead over the
    batch; "postnet": gamma = 0 on one channel of postnet layer 2.  Either gives that channel an all-zero G_z (the gradient
    at the BatchNorm input)."""
    sd = {k: v.clone() for k, v in synth_state_dict(seed=33, scale=2.0).items()}
    if zero == "encoder":
        sd[ZERO_LAYER["encoder"] + "1.bias"][ZC] = -50.0
    elif zero == "postnet":
        sd[ZERO_LAYER["postnet"] + "1.weight"][ZC] = 0.0
    return sd


def engine_model(sd, training):
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    return model.cuda().train(training)


@contextlib.contextmanager
def pre_bn_grad_max():
    """Records max |G_z| of every oracle conv layer (the gradient at its BatchNorm input) during a backward."""
    rec = {}
    orig = O.batchnorm1d

    def bn(x, sd, prefix, training, eps=1e-5):
        if x.requires_grad:
            x.register_hook(lambda g, p=prefix[:-3]: rec.__setitem__(p, float(g.abs().max())))   # "<module>.convolutions.<i>"
        return orig(x, sd, prefix, training, eps)

    O.batchnorm1d = bn
    try:
        yield rec
    finally:
        O.batchnorm1d = orig


def to64(sd, device):
    return {k: (v.to(device=device, dtype=torch.float64) if v.is_floating_point() else v.to(device)) for k, v in sd.items()}


# ---- Encoder / Postnet under autograd ---------------------------------------------------------------------------------
def module_case(module, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    C = 512 if module == "encoder" else 80
    x = torch.randn(B, C, T, generator=g)
    lens = torch.sort(torch.randint(max(1, T // 2), T + 1, (B,), generator=g), descending=True)[0]
    lens[0] = T
    if module == "encoder":
        keep = keep_mask((3, B, 512, T), 0.5, seed + 1)
        seed_grad = torch.randn(B, T, 512, generator=g)
    else:
        keep = [keep_mask((B, 512, T), 0.5, seed + 1 + i) for i in range(4)] + [keep_mask((B, 80, T), 0.5, seed + 5)]
        seed_grad = torch.randn(B, 80, T, generator=g)
    return x, lens, keep, seed_grad


def engine_module_grads(model, module, x, lens, keep, seed_grad):
    """Gradients of <module>'s parameters and of its input (d_input) for the upstream gradient seed_grad."""
    mod = getattr(model, module)
    for p in mod.parameters():
        p.grad = None
    xe = x.cuda().requires_grad_(True)
    if module == "encoder":
        with t2.dropout_masks(enc=keep):
            out = mod(xe, lens.cuda())
    else:
        with t2.dropout_masks(post=keep):
            out = mod(xe)
    out.backward(seed_grad.cuda())
    torch.cuda.synchronize()
    grads = {module + "." + k: p.grad.detach().clone() for k, p in mod.named_parameters()}
    grads["d_input"] = xe.grad.detach().clone()
    return grads


def oracle_module_grads(module, sd, training, x, lens, keep, seed_grad, device="cpu"):
    """The same gradients from the oracle's autograd in float64; also max |G_z| per conv layer."""
    sdx = to64(sd, device)
    names = [k for k, v in sdx.items() if k.startswith(module + ".") and v.is_floating_point() and "running" not in k]
    for k in names:
        sdx[k] = sdx[k].clone().requires_grad_(True)
    xo = x.to(device=device, dtype=torch.float64).requires_grad_(True)
    kp = None
    if training:
        kp = keep.to(device) if module == "encoder" else [k_.to(device) for k_ in keep]
    with pre_bn_grad_max() as gz:
        if module == "encoder":
            out = O.encoder(sdx, xo, lens.to(device), training, kp)
        else:
            out = O.postnet(sdx, xo, training, kp)
        out.backward(seed_grad.to(device=device, dtype=torch.float64))
    grads = {k: sdx[k].grad for k in names}
    grads["d_input"] = xo.grad
    return grads, gz


def grad_errors(got, ref, training, scale=1.0):
    """rel_err of every gradient; conv biases in front of a training-mode BatchNorm have an exactly-zero gradient, where both
    sides hold rounding noise: those only have to be tiny next to the BatchNorm beta gradient."""
    errs = {}
    for k, r in ref.items():
        g = got[k].double().cpu()
        r = r.double().cpu() * scale
        if training and k.endswith("0.conv.bias"):
            beta = float(ref[k.replace("0.conv.bias", "1.bias")].abs().max()) * scale
            assert float(g.abs().max()) < 1e-3 * beta, k
            continue
        errs[k] = rel_err(g, r)
    return errs


def check_errors(errs, label):
    worst = max(errs, key=errs.get)
    print("%s: worst %.2e (%s)" % (label, errs[worst], worst))
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, bad


# ---- A1: bitwise scale equivariance --------------------------------------------------------------------------------
SCALES = (-24, -12, 12)


def decoder_case(B, Te, T, seed):
    g = torch.Generator().manual_seed(seed)
    memory = torch.randn(B, Te, 512, generator=g)
    mels = torch.randn(B, 80, T, generator=g)
    lens = torch.full((B,), Te, dtype=torch.long)
    if B > 1:
        lens[1:] = torch.randint(max(1, Te // 2), Te + 1, (B - 1,), generator=g)
        lens, _ = torch.sort(lens, descending=True)
    masks = dict(prenet=keep_mask((T + 1, 2, B, 256), 0.5, seed + 1), att=keep_mask((T, B, 1024), 0.1, seed + 2),
                 dec=keep_mask((T, B, 1024), 0.1, seed + 3))
    seeds = (torch.randn(B, 80, T, generator=g), torch.randn(B, T, generator=g), torch.randn(B, T, Te, generator=g))
    return memory, mels, lens, masks, seeds


def engine_decoder_grads(model, memory, mels, lens, masks, seeds, use_align=True):
    dec = model.decoder
    for p in dec.parameters():
        p.grad = None
    mem = memory.cuda().requires_grad_(True)
    with t2.dropout_masks(**masks):
        mel, gate, align = dec(mem, mels.cuda(), lens.cuda())
        loss = (mel * seeds[0].cuda()).sum() + (gate * seeds[1].cuda()).sum()
        if use_align:
            loss = loss + (align * seeds[2].cuda()).sum()
        loss.backward()
    torch.cuda.synchronize()
    grads = {"decoder." + k: p.grad.detach().clone() for k, p in dec.named_parameters()}
    grads["d_memory"] = mem.grad.detach().clone()
    return grads


def check_equivariant(run, label):
    base = run(1.0)
    for k in SCALES:
        got = run(2.0 ** k)
        diff = {n: rel_err(got[n], base[n] * 2.0 ** k) for n in base if not torch.equal(got[n], base[n] * 2.0 ** k)}
        print("%s, seeds x 2^%d: %d of %d gradients bit-identical to 2^%d x the unit-seed ones" %
              (label, k, len(base) - len(diff), len(base), k))
        assert not diff, (k, diff)


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("module,zero", [("encoder", False), ("encoder", True), ("postnet", False), ("postnet", True)])
def test_conv_module_backward_is_exactly_scale_equivariant(module, zero, training):
    """Encoder (with lengths) / Postnet backward: seeds x 2^k -> every parameter gradient and the input gradient x 2^k exactly,
    also with one channel's G_z all zero (the conv input gradient's pre-scale must come from the largest live channel)."""
    sd = weights(module if zero else None)
    model = engine_model(sd, training)
    x, lens, keep, seed_grad = module_case(module, 3, 21, seed=7)
    got = engine_module_grads(model, module, x, lens, keep, seed_grad)
    if zero:    # the forced channel's G_z really is all zero: its rows of the conv weight gradient are exactly 0
        assert not bool(got[ZERO_LAYER[module] + "0.conv.weight"][ZC].any())
    check_equivariant(lambda s: engine_module_grads(model, module, x, lens, keep, seed_grad * s),
                      "%s %s%s" % (module, "train" if training else "eval", " zero-channel" if zero else ""))


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_decoder_backward_is_exactly_scale_equivariant(training):
    sd = weights()
    model = engine_model(sd, training)
    memory, mels, lens, masks, seeds = decoder_case(3, 19, 7, seed=11)
    check_equivariant(lambda s: engine_decoder_grads(model, memory, mels, lens, masks, tuple(v * s for v in seeds)),
                      "decoder %s" % ("train" if training else "eval"))


# ---- A2: zero-gradient channels at a realistic gradient magnitude, vs fp64 ---------------------------------------------
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("module", ["encoder", "postnet"])
def test_zero_channel_backward_at_small_gradients_vs_fp64(module, training):
    """Seeds scaled by a power of two so that max |G_z| of the layer with the all-zero channel is about 1e-6."""
    sd = weights(module)
    x, lens, keep, seed_grad = module_case(module, 3, 21, seed=7)
    ref, gz = oracle_module_grads(module, sd, training, x, lens, keep, seed_grad)
    gz0 = gz[ZERO_LAYER[module][:-1]]
    s = 2.0 ** round(math.log2(1e-6 / gz0))
    got = engine_module_grads(engine_model(sd, training), module, x, lens, keep, seed_grad * s)
    errs = grad_errors(got, ref, training, s)
    check_errors(errs, "%s %s zero-channel, max|G_z| %.2e" % (module, "train" if training else "eval", gz0 * s))


def test_full_train_step_with_a_zero_gamma_encoder_channel_vs_fp64():
    """Tacotron2 + Tacotron2Loss at the golden b4 inputs with one encoder gamma zeroed, against the oracle in float64."""
    g = load("grad_train_b4")
    sd, text, tl, ol, mels, gt, m = grad_inputs(g)
    sd = {k: v.clone() for k, v in sd.items()}
    sd[ZERO_LAYER["encoder"] + "1.weight"][ZC] = 0.0
    with pre_bn_grad_max() as gz:
        _, _, ref = oracle_train_step(sd, text, tl, ol, mels, gt, m, True, dtype=torch.float64)
    model = engine_model(sd, True)
    post_keep = [m["qk4"][i] for i in range(4)] + [m["qk1"]]
    with t2.dropout_masks(prenet=m["pk"], att=m["ak"], dec=m["dk"], enc=m["ek"], post=post_keep):
        out = model((text.cuda(), tl.cuda(), mels.cuda(), int(tl.max()), ol.cuda()))
        t2.Tacotron2Loss()(out, (mels.cuda(), gt.cuda())).backward()
    torch.cuda.synchronize()
    errs = grad_errors({k: p.grad for k, p in model.named_parameters()}, ref, True)
    print("max|G_z| per conv layer: " + ", ".join("%s %.1e" % (k.replace("convolutions.", ""), v) for k, v in sorted(gz.items())))
    check_errors(errs, "train step b4, encoder gamma zeroed")


def test_pre_batchnorm_gradient_magnitude_of_the_full_size_training_step():
    """At the benchmark's training shape (B=64, T_text=150, T_mel=800) the gradients at every BatchNorm input are far below
    0.5: the regime in which an all-zero channel used to decide the conv input gradient's pre-scale."""
    g = load("full_grad_train_b64_t150_m800")
    from tests.test_oracle_golden import full_grad_inputs
    sd, text, tl, ol, mels, gt, m = full_grad_inputs(g)
    sdc = {k: v.cuda() for k, v in sd.items()}
    mc = {k: v.cuda() for k, v in m.items()}
    with pre_bn_grad_max() as gz:
        oracle_train_step(sdc, text.cuda(), tl.cuda(), ol.cuda(), mels.cuda(), gt.cuda(), mc, True)
    print("full-size training step, max|G_z| per conv layer (fp32 oracle): " +
          ", ".join("%s %.1e" % (k.replace("convolutions.", ""), v) for k, v in sorted(gz.items())))
    assert len(gz) == 8 and max(gz.values()) < 0.5


# ---- B: K-split and tile regimes vs fp64 ----------------------------------------------------------------------------
def oracle_decoder_grads(sd, memory, mels, lens, masks, seeds, training, device):
    sdx = to64(sd, device)
    names = [k for k in sdx if k.startswith("decoder.")]
    for k in names:
        sdx[k] = sdx[k].clone().requires_grad_(True)
    mem = memory.to(device=device, dtype=torch.float64).requires_grad_(True)
    mel, gate, align = O.decoder_forward(sdx, mem, mels.to(device=device, dtype=torch.float64), lens.to(device),
                                         masks["prenet"].to(device), masks["att"].to(device), masks["dec"].to(device),
                                         training=training)
    loss = (mel * seeds[0].to(device=device, dtype=torch.float64)).sum() + (gate * seeds[1].to(device=device, dtype=torch.float64)).sum()
    loss.backward()
    grads = {k: sdx[k].grad for k in names}
    grads["d_memory"] = mem.grad
    return grads


# (B, T_mel, oracle device): wgrad_seg(T_mel) segments of the time-batched LSTM weight gradients
#   100 -> 1 x 100;  101 -> 100 + 1;  250 -> 2 x 100 + 50;  1500 -> 15 x 100;  1501 -> seg 150: 10 x 150 + 1
@pytest.mark.parametrize("B,T,device", [(3, 100, "cpu"), (3, 101, "cpu"), (3, 250, "cpu"), (2, 1500, "cuda"), (2, 1501, "cuda"),
                                        (64, 101, "cuda")])
def test_decoder_lstm_weight_gradient_k_splits_vs_fp64(B, T, device):
    # weights of the reference's initialisation scale: with twice that, teacher forcing over 1500 random frames makes the
    # backward recurrence grow d_memory to ~1e3 and fp32 rounding alone moves the gradients by ~1e-2
    sd = synth_state_dict(seed=33)
    memory, mels, lens, masks, seeds = decoder_case(B, 20, T, seed=300 + B)
    ref = oracle_decoder_grads(sd, memory, mels, lens, masks, seeds, True, device)
    got = engine_decoder_grads(engine_model(sd, True), memory, mels, lens, masks, seeds, use_align=False)
    check_errors(grad_errors(got, ref, True), "decoder backward B=%d T_mel=%d" % (B, T))


# (B, T) -> B (T + 4) padded rows -> nch = ceil(rows / 64) K chunks of the conv weight gradients:
#   (1, 60) 64 -> 1;  (1, 61) 65 -> 2;  (64, 96) 6400 -> 100;  (64, 97) 6464 -> 101;  (64, 1496) 96000 -> 1500 (15 x 100);
#   (64, 1497) 96064 -> 1501 (seg 150: 10 x 150 + 1)
@pytest.mark.parametrize("module,B,T", [("postnet", 1, 60), ("postnet", 1, 61), ("postnet", 64, 96), ("postnet", 64, 97),
                                        ("postnet", 64, 1496), ("postnet", 64, 1497), ("encoder", 64, 97), ("encoder", 1, 61)])
def test_conv_weight_gradient_k_splits_vs_fp64(module, B, T):
    sd = weights()
    x, lens, keep, seed_grad = module_case(module, B, T, seed=B * 10000 + T)
    ref, _ = oracle_module_grads(module, sd, True, x, lens, keep, seed_grad, device="cpu" if B == 1 else "cuda")
    got = engine_module_grads(engine_model(sd, True), module, x, lens, keep, seed_grad)
    check_errors(grad_errors(got, ref, True), "%s backward B=%d T=%d" % (module, B, T))


# B (T + 4) padded rows in 128-row tiles, clusters of 2: (1, 124) one tile, (1, 125) one row past it, (2, 60) one tile,
# (3, 81) and (64, 2) odd tile counts (+ the cluster's padding tile), (1, 1) a single frame
@pytest.mark.parametrize("B,T", [(1, 1), (1, 124), (1, 125), (2, 60), (3, 81), (64, 2)])
def test_inference_conv_tiles_vs_fp64(B, T):
    sd = synth_state_dict(9, scale=1.5)         # the weights and embedded-text inputs of test_gpu_parity's module test
    model = engine_model(sd, False)
    emb = sd["embedding.weight"][rand_text(B, T, B * 1000 + T)].transpose(1, 2).contiguous()
    mel = torch.randn(B, 80, T, generator=torch.Generator().manual_seed(B * 1000 + T))
    sd64 = to64(sd, "cpu")
    with torch.no_grad():
        ref_mem = O.encoder(sd64, emb.double(), None, False)
        ref_post = O.postnet(sd64, mel.double(), False)
        mem = model.encoder.inference(emb.cuda())
        post = model.postnet(mel.cuda())
    torch.cuda.synchronize()
    e_mem, e_post = rel_err(mem, ref_mem), rel_err(post, ref_post)
    print("inference convs B=%d T=%d: encoder %.2e, postnet %.2e" % (B, T, e_mem, e_post))
    assert e_mem < INFER_TOL and e_post < INFER_TOL


# ---- training-mode forwards outside autograd ------------------------------------------------------------------------
def training_forward(sd, module, x, lens, keep, grad):
    """A training-mode <module>.forward on a fresh model, with or without autograd: its output and the BatchNorm running
    statistics it left."""
    mod = getattr(engine_model(sd, True), module)
    masks = dict(enc=keep) if module == "encoder" else dict(post=keep)
    with torch.set_grad_enabled(grad), t2.dropout_masks(**masks):
        out = mod(x.cuda(), lens.cuda()) if module == "encoder" else mod(x.cuda())
    torch.cuda.synchronize()
    return out.detach(), {k: v.clone() for k, v in mod.state_dict().items() if "running" in k}


@pytest.mark.parametrize("module,B,T", [("encoder", 5, 33), ("encoder", 64, 40), ("postnet", 3, 41), ("postnet", 2, 1)])
def test_training_forward_without_autograd_equals_autograd_forward(module, B, T):
    """Both run the training conv stack (under autograd with a stash for the backward pass), so the output and the updated
    BatchNorm running statistics are the same bits.  Fresh models from one state dict, the same injected dropout masks."""
    sd = weights()
    x, lens, keep, _ = module_case(module, B, T, seed=B * 1000 + T)
    out_ng, run_ng = training_forward(sd, module, x, lens, keep, False)
    out_ag, run_ag = training_forward(sd, module, x, lens, keep, True)
    assert torch.equal(out_ng, out_ag)
    bad = [k for k in run_ng if not torch.equal(run_ng[k], run_ag[k])]
    assert not bad, bad


def test_training_postnet_with_lengths_vs_fp64():
    """The training-mode postnet with per-row lengths, as Tacotron2.inference on a training-mode model runs it for B > 1:
    input frames at t >= lengths[b] hold real values but count as zero, and the output there is zero.  The rows sit in a
    wider buffer (batch stride > T * 80), like the decoder's output."""
    B, T = 4, 37
    sd = weights()
    g = torch.Generator().manual_seed(5)
    rows = torch.randn(B, T + 6, 80, generator=g).cuda()[:, :T]
    lens = torch.tensor([T, 20, 1, 9], dtype=torch.int32)
    keep = [keep_mask((B, 512, T), 0.5, 60 + i) for i in range(4)] + [keep_mask((B, 80, T), 0.5, 64)]
    with torch.no_grad():
        got = engine_model(sd, True)._t2_engine().postnet(rows, lens.cuda(), True, True, keep).cpu()
    past = torch.arange(T)[None, :] >= lens[:, None].long()                    # (B, T)
    x = rows.cpu().double().transpose(1, 2).masked_fill(past[:, None, :], 0.0)
    ref = (O.postnet(to64(sd, "cpu"), x, True, keep) + x).masked_fill(past[:, None, :], 0.0)
    err = rel_err(got, ref)
    print("training postnet with lengths %s: %.2e" % (lens.tolist(), err))
    assert err < INFER_TOL
    assert not bool(got.masked_select(past[:, None, :]).any())


# ---- C: shape changes on one model ----------------------------------------------------------------------------------
def train_inputs(B, Tt, Tm, seed):
    g = torch.Generator().manual_seed(seed)
    text = rand_text(B, Tt, seed)
    tl = torch.sort(torch.randint(max(1, Tt // 2), Tt + 1, (B,), generator=g), descending=True)[0]
    tl[0] = Tt
    ol = torch.randint(max(1, Tm // 2), Tm + 1, (B,), generator=g)
    ol[0] = Tm
    mels = torch.randn(B, 80, Tm, generator=g)
    gt = torch.zeros(B, Tm)
    for i, n in enumerate(ol.tolist()):
        mels[i, :, n:] = 0
        gt[i, n - 1:] = 1
    masks = dict(prenet=keep_mask((Tm + 1, 2, B, 256), 0.5, seed + 1), att=keep_mask((Tm, B, 1024), 0.1, seed + 2),
                 dec=keep_mask((Tm, B, 1024), 0.1, seed + 3), enc=keep_mask((3, B, 512, Tt), 0.5, seed + 4),
                 post=[keep_mask((B, 512, Tm), 0.5, seed + 5 + i) for i in range(4)] + [keep_mask((B, 80, Tm), 0.5, seed + 9)])
    return (text, tl, mels, ol, gt), masks


def train_step(model, inputs, masks):
    text, tl, mels, ol, gt = inputs
    model.zero_grad(set_to_none=True)
    with t2.dropout_masks(**masks):
        out = model((text.cuda(), tl.cuda(), mels.cuda(), int(tl.max()), ol.cuda()))
        loss = t2.Tacotron2Loss()(out, (mels.cuda(), gt.cuda()))
        loss.backward()
    torch.cuda.synchronize()
    res = {"loss": loss.detach().clone(), "mel_post": out[1].detach().clone()}
    res.update({k: p.grad.detach().clone() for k, p in model.named_parameters()})
    return res


def test_training_steps_across_shape_changes_match_a_fresh_model():
    """One model runs (8, 60, 120), (3, 20, 37), (8, 60, 120): each step equals a fresh model's step at that shape bit for
    bit, so the cached workspaces, the input-gradient weight images and their staging buffer carry nothing between calls."""
    sd = weights()
    model = engine_model(sd, True)
    for B, Tt, Tm in [(8, 60, 120), (3, 20, 37), (8, 60, 120)]:
        inputs, masks = train_inputs(B, Tt, Tm, seed=B * 100 + Tt)
        got = train_step(model, inputs, masks)
        want = train_step(engine_model(sd, True), inputs, masks)
        diff = [k for k in want if not torch.equal(got[k], want[k])]
        print("shape (%d, %d, %d) on a reused model: %d of %d tensors bit-identical to a fresh model's" %
              (B, Tt, Tm, len(want) - len(diff), len(want)))
        assert not diff, diff
