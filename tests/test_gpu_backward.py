"""GPU (H100): gradients of the CUDA training path vs torch autograd through the CPU oracle (the oracle's
autograd is pinned against the reference's own autograd in tests/test_oracle_vs_reference.py and by
tests/golden/grad_*.npz).  Same weights, inputs and dropout masks on both sides.

Tolerance: max|g - g_ref| / max|g_ref| < 1e-3 for every parameter gradient and for d_memory."""
import pytest
import torch

import tacotron2_b200 as t2
from oracle import tacotron2_oracle as O
from tests.common import keep_mask, rel_err, synth_state_dict
from tests.test_oracle_golden import (GRADS, check_grads_vs_fixture, check_grads_vs_fp64_fixture, full_grad_inputs,
                                      grad_inputs, load, oracle_train_step)
from tests.test_gpu_train_regimes import to64

pytestmark = pytest.mark.gpu
TOL = 1e-3


def decoder_case(B, Te, T, seed, ragged=True):
    g = torch.Generator().manual_seed(seed)
    memory = torch.randn(B, Te, 512, generator=g)
    mels = torch.randn(B, 80, T, generator=g)
    lens = torch.full((B,), Te, dtype=torch.long)
    if ragged and B > 1:
        lens[1:] = torch.randint(max(1, Te // 2), Te + 1, (B - 1,), generator=g)
        lens, _ = torch.sort(lens, descending=True)
    pk = keep_mask((T + 1, 2, B, 256), 0.5, seed + 1)
    ak = keep_mask((T, B, 1024), 0.1, seed + 2)
    dk = keep_mask((T, B, 1024), 0.1, seed + 3)
    d_mel = torch.randn(B, 80, T, generator=g)
    d_gate = torch.randn(B, T, generator=g)
    d_align = torch.randn(B, T, Te, generator=g)
    return memory, mels, lens, pk, ak, dk, d_mel, d_gate, d_align


def oracle_decoder_grads(sd, memory, mels, lens, pk, ak, dk, d_mel, d_gate, d_align, training):
    names = [k for k in sd if k.startswith("decoder.")]
    sdg = dict(sd)
    for k in names:
        sdg[k] = sd[k].clone().requires_grad_(True)
    mem = memory.clone().requires_grad_(True)
    mel, gate, align = O.decoder_forward(sdg, mem, mels, lens, pk.float(), ak.float(), dk.float(), training=training)
    loss = (mel * d_mel).sum() + (gate * d_gate).sum()
    if d_align is not None:
        loss = loss + (align * d_align).sum()
    loss.backward()
    return (mel.detach(), gate.detach(), align.detach()), {k: sdg[k].grad for k in names}, mem.grad


@pytest.mark.parametrize("B,Te,T,training,use_align", [(3, 19, 7, True, False), (5, 40, 12, True, True),
                                                       (4, 150, 9, False, False), (64, 33, 5, True, False)])
def test_decoder_backward_vs_oracle_autograd(B, Te, T, training, use_align):
    """The reverse recurrence's skinny GEMMs and the time-batched LSTM weight gradients on the wgmma split-fp16 engines."""
    sd = synth_state_dict(seed=21, scale=2.0)
    memory, mels, lens, pk, ak, dk, d_mel, d_gate, d_align = decoder_case(B, Te, T, seed=100 + B)
    if not use_align:
        d_align = None
    ref_out, ref_g, ref_dmem = oracle_decoder_grads(sd, memory, mels, lens, pk, ak, dk, d_mel, d_gate, d_align, training)

    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    model = model.cuda().train(training)
    dec = model.decoder
    mem = memory.cuda().requires_grad_(True)
    with t2.dropout_masks(prenet=pk, att=ak, dec=dk):
        mel, gate, align = dec(mem, mels.cuda(), lens.cuda())
        loss = (mel * d_mel.cuda()).sum() + (gate * d_gate.cuda()).sum()
        if d_align is not None:
            loss = loss + (align * d_align.cuda()).sum()
        loss.backward()
    torch.cuda.synchronize()
    assert rel_err(mel, ref_out[0]) < TOL and rel_err(gate, ref_out[1]) < TOL and rel_err(align, ref_out[2]) < TOL
    errs = {"d_memory": rel_err(mem.grad, ref_dmem)}
    for k, p in dec.named_parameters():
        assert p.grad is not None, k
        errs[k] = rel_err(p.grad, ref_g["decoder." + k])
    bad = {k: v for k, v in errs.items() if not v < TOL}
    print("decoder backward B=%d Te=%d T=%d: worst %.2e" % (B, Te, T, max(errs.values())))
    assert not bad, bad


@pytest.mark.parametrize("name", GRADS)
def test_full_train_step_matches_reference_gradient_golden(name):
    """Tacotron2.forward + Tacotron2Loss + backward through the CUDA path vs (a) the gradients the reference's own
    autograd produced (tests/golden/grad_*.npz) and (b) the oracle's autograd, every parameter, full tensors."""
    g = load(name)
    training = bool(int(g["training"]))
    sd, text, tl, ol, mels, gt, m = grad_inputs(g)
    ref_loss, _, ref_g = oracle_train_step(sd, text, tl, ol, mels, gt, m, training)
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    model = model.cuda().train(training)
    post_keep = [m["qk4"][i] for i in range(4)] + [m["qk1"]]
    with t2.dropout_masks(prenet=m["pk"], att=m["ak"], dec=m["dk"], enc=m["ek"], post=post_keep):
        out = model((text.cuda(), tl.cuda(), mels.cuda(), int(tl.max()), ol.cuda()))
        loss = t2.Tacotron2Loss()(out, (mels.cuda(), gt.cuda()))
        loss.backward()
    torch.cuda.synchronize()
    assert abs(float(loss) - float(g["loss"])) < 1e-4 * abs(float(g["loss"]))
    assert rel_err(out[0], torch.from_numpy(g["mel"])) < TOL and rel_err(out[1], torch.from_numpy(g["mel_post"])) < TOL
    grads = {k: p.grad for k, p in model.named_parameters()}
    assert all(v is not None for v in grads.values())
    check_grads_vs_fixture(grads, g, TOL)
    errs = {}
    for k, v in grads.items():
        if float(ref_g[k].abs().max()) < 1e-5:
            continue
        errs[k] = rel_err(v, ref_g[k])
    print("train step %s: loss %.6f (ref %.6f), worst gradient error %.2e" % (name, float(loss), float(ref_loss), max(errs.values())))
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, bad


def test_full_size_train_step_matches_reference_gradient_golden():
    """BASELINE.json configs[2]: the teacher-forced training step at B=64, T_text=150, T_mel=800 against the gradients
    the REFERENCE's own autograd produced at that size (tools/make_golden.py full grad64: per parameter sum / abs-sum /
    max + 1024 sampled entries, loss, sub-sampled outputs), in fp32 AND in fp64.  The forward outputs and the loss are
    held to the fp32 reference at 1e-3 / 1e-4; the gradients to the fp64 reference at max(1e-3, 4 x the deviation of the
    reference's own fp32 autograd from it) -- that deviation is 1e-3 ... 1e-2 for the encoder convolutions, the
    embedding and the prenet at this size (printed below)."""
    g = load("full_grad_train_b64_t150_m800")
    sd, text, tl, ol, mels, gt, m = full_grad_inputs(g)
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    model = model.cuda().train()
    post_keep = [m["qk4"][i] for i in range(4)] + [m["qk1"]]
    with t2.dropout_masks(prenet=m["pk"], att=m["ak"], dec=m["dk"], enc=m["ek"], post=post_keep):
        out = model((text.cuda(), tl.cuda(), mels.cuda(), int(tl.max()), ol.cuda()))
        loss = t2.Tacotron2Loss()(out, (mels.cuda(), gt.cuda()))
        loss.backward()
    torch.cuda.synchronize()
    idx = torch.from_numpy(g["frame_index"]).long()
    e_mel = rel_err(out[0][:, :, idx], torch.from_numpy(g["mel"]))
    e_post = rel_err(out[1][:, :, idx], torch.from_numpy(g["mel_post"]))
    e_gate = rel_err(out[2], torch.from_numpy(g["gate"]))
    print("full-size train step: loss %.6f (reference %.6f), mel %.2e post %.2e gate %.2e" %
          (float(loss), float(g["loss"]), e_mel, e_post, e_gate))
    assert abs(float(loss) - float(g["loss"])) < 1e-4 * abs(float(g["loss"]))
    assert e_mel < TOL and e_post < TOL and e_gate < TOL
    grads = {k: p.grad for k, p in model.named_parameters()}
    assert all(v is not None for v in grads.values())
    rep = check_grads_vs_fp64_fixture(grads, g, TOL)
    worst = sorted(rep.items(), key=lambda kv: -kv[1][0])[:10]
    print("full-size gradients vs the fp64 reference (engine error, fp32 reference's own error):")
    for k, (e_eng, e_ref) in worst:
        print("   %-66s %.2e  %.2e" % (k, e_eng, e_ref))
    n_better = sum(1 for e_eng, e_ref in rep.values() if e_eng <= e_ref)
    print("   engine closer to fp64 than the fp32 reference for %d of %d parameters" % (n_better, len(rep)))


@pytest.mark.parametrize("B,T", [(3, 21), (5, 64)])
def test_postnet_and_encoder_modules_backward_vs_oracle(B, T):
    """The Encoder and Postnet nn.Modules on their own under autograd (training mode, injected masks)."""
    sd = synth_state_dict(seed=33, scale=2.0)
    g = torch.Generator().manual_seed(B * 100 + T)
    x = torch.randn(B, 80, T, generator=g)
    emb = torch.randn(B, 512, T, generator=g)
    lens = torch.sort(torch.randint(max(1, T // 2), T + 1, (B,), generator=g), descending=True)[0]
    lens[0] = T
    post_keep = [keep_mask((B, 512, T), 0.5, 7 + i) for i in range(4)] + [keep_mask((B, 80, T), 0.5, 11)]
    ek = keep_mask((3, B, 512, T), 0.5, 12)
    d_post = torch.randn(B, 80, T, generator=g)
    d_mem = torch.randn(B, T, 512, generator=g)
    # oracle
    names = [k for k, v in sd.items() if v.dtype.is_floating_point and "running" not in k and not k.startswith("decoder.")]
    sdg = dict(sd)
    for k in names:
        sdg[k] = sd[k].clone().requires_grad_(True)
    xo, eo = x.clone().requires_grad_(True), emb.clone().requires_grad_(True)
    (O.postnet(sdg, xo, True, post_keep) * d_post).sum().backward()
    (O.encoder(sdg, eo, lens, True, ek) * d_mem).sum().backward()
    # engine
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    model = model.cuda().train()
    xe, ee = x.cuda().requires_grad_(True), emb.cuda().requires_grad_(True)
    with t2.dropout_masks(enc=ek, post=post_keep):
        (model.postnet(xe) * d_post.cuda()).sum().backward()
        (model.encoder(ee, lens.cuda()) * d_mem.cuda()).sum().backward()
    torch.cuda.synchronize()
    errs = {"d_x": rel_err(xe.grad, xo.grad), "d_emb": rel_err(ee.grad, eo.grad)}
    for k, p in model.named_parameters():
        if k.startswith("postnet.") or k.startswith("encoder."):
            assert p.grad is not None, k
            if k.endswith("conv.bias"):
                # a bias in front of a training-mode BatchNorm has an exactly-zero gradient; both sides hold rounding noise
                scale = float(sdg[k.replace("0.conv.bias", "1.bias")].grad.abs().max())
                assert float(sdg[k].grad.abs().max()) < 1e-3 * scale and float(p.grad.abs().max()) < 1e-3 * scale, k
                continue
            errs[k] = rel_err(p.grad, sdg[k].grad)
    print("encoder/postnet backward B=%d T=%d: worst %.2e" % (B, T, max(errs.values())))
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, bad


def test_full_size_backward_vs_fp64_and_determinism():
    """B=64, T_enc=150 (the benchmark shape), 24 teacher-forced steps, injected dropout masks: two runs are bit-identical,
    and d_memory and every decoder parameter gradient are within 1e-4 of the oracle's autograd in float64 (or 4 x the fp32
    oracle's own deviation from float64 where that exceeds 2.5e-5, the yardstick of DESIGN section 2)."""
    torch.manual_seed(7)
    model = t2.Tacotron2(t2.create_hparams()).cuda().train()
    dec = model.decoder
    B, Te, T = 64, 150, 24
    g = torch.Generator().manual_seed(3)
    memory = torch.randn(B, Te, 512, generator=g)
    mels = torch.randn(B, 80, T, generator=g)
    lens = torch.sort(torch.randint(75, Te + 1, (B,), generator=g), descending=True)[0]
    lens[0] = Te
    d_mel = torch.randn(B, 80, T, generator=g)
    d_gate = torch.randn(B, T, generator=g)
    pk = keep_mask((T + 1, 2, B, 256), 0.5, 1)
    ak, dk = keep_mask((T, B, 1024), 0.1, 2), keep_mask((T, B, 1024), 0.1, 3)

    def run():
        for p in dec.parameters():
            p.grad = None
        mem = memory.cuda().requires_grad_(True)
        with t2.dropout_masks(prenet=pk, att=ak, dec=dk):
            mel, gate, _ = dec(mem, mels.cuda(), lens.cuda())
            ((mel * d_mel.cuda()).sum() + (gate * d_gate.cuda()).sum()).backward()
        torch.cuda.synchronize()
        return [mem.grad.clone()] + [p.grad.clone() for p in dec.parameters()]

    a, b = run(), run()
    names = ["d_memory"] + [k for k, _ in dec.named_parameters()]
    diff = {n: rel_err(x, y) for n, x, y in zip(names, a, b) if not torch.equal(x, y)}
    assert not diff, "backward is not bit-reproducible: %s" % diff

    sd = {k: v.cpu() for k, v in model.state_dict().items()}
    _, ref32, ref32_dmem = oracle_decoder_grads(sd, memory, mels, lens, pk, ak, dk, d_mel, d_gate, None, True)
    _, ref64, ref64_dmem = oracle_decoder_grads(to64(sd, "cpu"), memory.double(), mels.double(), lens, pk, ak, dk, d_mel.double(),
                                                d_gate.double(), None, True)
    ref32["d_memory"], ref64["d_memory"] = ref32_dmem, ref64_dmem
    errs, bars = {}, {}
    for n, x in zip(names, a):
        k = n if n == "d_memory" else "decoder." + n
        errs[n] = rel_err(x, ref64[k])
        bars[n] = max(1e-4, 4.0 * rel_err(ref32[k], ref64[k]))
    worst = max(errs, key=errs.get)
    print("full-size backward vs fp64: worst %.2e (%s, bar %.2e)" % (errs[worst], worst, bars[worst]))
    bad = {n: (e, bars[n]) for n, e in errs.items() if not e < bars[n]}
    assert not bad, bad


def test_fused_clip_adam_matches_torch():
    """t2.FusedClipAdam.step(max_norm) == clip_grad_norm_ + torch.optim.Adam.step (train.py:229-236), 4 steps, odd sizes,
    clipping active in some steps and not in others; the engine notices the in-place parameter update."""
    g = torch.Generator().manual_seed(5)
    shapes = [(7,), (129, 3), (4096, 33), (1,), (65537,), (80, 512, 5)]
    ref_p = [torch.nn.Parameter(torch.randn(s, generator=g).cuda()) for s in shapes]
    our_p = [torch.nn.Parameter(p.detach().clone()) for p in ref_p]
    ref_opt = torch.optim.Adam(ref_p, lr=1e-3, weight_decay=1e-6)
    our_opt = t2.FusedClipAdam(our_p, lr=1e-3, weight_decay=1e-6)
    for it in range(4):
        scale = [5.0, 1e-3, 0.3, 50.0][it]
        for a, b in zip(ref_p, our_p):
            gr = torch.randn(a.shape, generator=g).cuda() * scale
            a.grad, b.grad = gr.clone(), gr.clone()
        n_ref = torch.nn.utils.clip_grad_norm_(ref_p, 1.0)
        ref_opt.step()
        n_our = our_opt.step(max_norm=1.0)
        assert abs(float(n_ref) - float(n_our)) < 1e-5 * float(n_ref)
        for a, b in zip(ref_p, our_p):
            assert rel_err(b, a) < 2e-6 and rel_err(b.grad, a.grad) < 2e-6
    sd_ref, sd_our = ref_opt.state_dict(), our_opt.state_dict()
    for k in sd_ref["state"]:
        assert rel_err(sd_our["state"][k]["exp_avg"], sd_ref["state"][k]["exp_avg"]) < 2e-6
        assert rel_err(sd_our["state"][k]["exp_avg_sq"], sd_ref["state"][k]["exp_avg_sq"]) < 2e-6
        assert float(sd_our["state"][k]["step"]) == float(sd_ref["state"][k]["step"])
    # in-place update through the library -> the next forward uses the new weights
    model = t2.Tacotron2(t2.create_hparams()).cuda().eval()
    opt = t2.FusedClipAdam(model.parameters(), lr=1e-2)
    text = torch.randint(0, 148, (2, 9)).cuda()
    model.decoder.max_decoder_steps = 4
    with torch.no_grad():
        before = model.inference(text)[0].clone()
    for p in model.parameters():
        p.grad = torch.ones_like(p)
    opt.step()
    with torch.no_grad():
        after = model.inference(text)[0]
    assert not torch.equal(before, after)


def test_checkpoint_round_trip_like_train_py(tmp_path):
    """train.py:99-113: save {'state_dict', 'optimizer'} after a few steps, load into fresh objects, and the next step is
    bit-identical (fused optimizer state included)."""
    import tacotron2_b200._engine as E
    hp = t2.create_hparams()
    g = torch.Generator().manual_seed(1)
    text = torch.randint(0, 148, (4, 12), generator=g).cuda()
    tl = torch.tensor([12, 11, 9, 7]).cuda()
    ol = torch.tensor([10, 14, 8, 14]).cuda()
    mels = torch.randn(4, 80, 14, generator=g).cuda()
    gt = torch.zeros(4, 14).cuda()
    for i, n in enumerate(ol.tolist()):
        mels[i, :, n:] = 0
        gt[i, n - 1:] = 1
    x, y = (text, tl, mels, 12, ol), (mels, gt)
    crit = t2.Tacotron2Loss()

    def step(model, opt):
        model.zero_grad()
        loss = crit(model(x), y)
        loss.backward()
        opt.step(max_norm=hp.grad_clip_thresh)
        return loss.item()

    torch.manual_seed(3)
    model = t2.Tacotron2(hp).cuda().train()
    opt = t2.FusedClipAdam(model.parameters(), lr=hp.learning_rate, weight_decay=hp.weight_decay)
    E._seed_counter[0] = 0
    losses = [step(model, opt) for _ in range(3)]
    assert losses[2] < losses[0]
    path = str(tmp_path / "ckpt")
    torch.save({"iteration": 3, "state_dict": model.state_dict(), "optimizer": opt.state_dict(), "learning_rate": hp.learning_rate}, path)
    counter = E._seed_counter[0]
    a = step(model, opt)
    ck = torch.load(path, map_location="cpu")
    model2 = t2.Tacotron2(hp).cuda().train()
    model2.load_state_dict(ck["state_dict"])
    opt2 = t2.FusedClipAdam(model2.parameters(), lr=hp.learning_rate, weight_decay=hp.weight_decay)
    opt2.load_state_dict(ck["optimizer"])
    E._seed_counter[0] = counter                      # same Philox dropout streams as the original's 4th step
    b = step(model2, opt2)
    assert a == b
    for p1, p2 in zip(model.parameters(), model2.parameters()):
        assert torch.equal(p1, p2)


@pytest.mark.parametrize("B,Tt,Tm", [(1, 1, 1), (1, 3, 2), (2, 5, 1), (3, 2, 6)])
def test_train_step_minimal_shapes_vs_oracle_autograd(B, Tt, Tm):
    """Degenerate sizes: one utterance, one symbol, one frame -- full training step vs the oracle's autograd."""
    from tests.common import rand_text
    sd = synth_state_dict(seed=41, scale=2.0)
    g = torch.Generator().manual_seed(B * 100 + Tt * 10 + Tm)
    text = rand_text(B, Tt, 3)
    tl = torch.sort(torch.randint(1, Tt + 1, (B,), generator=g), descending=True)[0]
    tl[0] = Tt
    ol = torch.randint(1, Tm + 1, (B,), generator=g)
    ol[0] = Tm
    mels = torch.randn(B, 80, Tm, generator=g)
    gt = torch.zeros(B, Tm)
    for i, n in enumerate(ol.tolist()):
        mels[i, :, n:] = 0
        gt[i, n - 1:] = 1
    m = dict(pk=keep_mask((Tm + 1, 2, B, 256), 0.5, 1), ak=keep_mask((Tm, B, 1024), 0.1, 2), dk=keep_mask((Tm, B, 1024), 0.1, 3),
             ek=keep_mask((3, B, 512, Tt), 0.5, 4), qk4=keep_mask((4, B, 512, Tm), 0.5, 5), qk1=keep_mask((B, 80, Tm), 0.5, 6))
    ref_loss32, _, ref_g32 = oracle_train_step(sd, text, tl, ol, mels, gt, m, True)
    ref_loss, _, ref_g = oracle_train_step(sd, text, tl, ol, mels, gt, m, True, dtype=torch.float64)
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    model = model.cuda().train()
    post_keep = [m["qk4"][i] for i in range(4)] + [m["qk1"]]
    with t2.dropout_masks(prenet=m["pk"], att=m["ak"], dec=m["dk"], enc=m["ek"], post=post_keep):
        out = model((text.cuda(), tl.cuda(), mels.cuda(), int(tl.max()), ol.cuda()))
        loss = t2.Tacotron2Loss()(out, (mels.cuda(), gt.cuda()))
        loss.backward()
    torch.cuda.synchronize()
    # the loss too: five stacked BatchNorms over 1-2 frames per channel move it by 2e-4 between fp32 and fp64 alone
    loss_yard = abs(float(ref_loss32) - float(ref_loss)) / abs(float(ref_loss))
    assert abs(loss.item() - float(ref_loss)) < max(1e-4, 8.0 * loss_yard) * abs(float(ref_loss)), (loss.item(), float(ref_loss), loss_yard)
    gmax = max(float(v.abs().max()) for v in ref_g.values())
    errs, yard = {}, {}
    for k, p in model.named_parameters():
        # tiny batches make BatchNorm statistics (1-6 samples per channel) badly conditioned (rstd up to 1/sqrt(eps) = 316 per
        # layer amplifies rounding differences): the truth is the oracle in DOUBLE precision, errors are relative to the
        # largest gradient of the model, and the yardstick is how far the fp32 oracle itself lands from the fp64 one
        errs[k] = float((p.grad.detach().cpu().double() - ref_g[k]).abs().max()) / gmax
        yard[k] = float((ref_g32[k].double() - ref_g[k]).abs().max()) / gmax
    print("minimal train step B=%d T_text=%d T_mel=%d: loss %.5f, worst gradient error / max gradient %.2e (fp32 oracle vs fp64 "
          "oracle: %.2e)" % (B, Tt, Tm, loss.item(), max(errs.values()), max(yard.values())))
    bad = {k: (v, yard[k]) for k, v in errs.items() if not v < max(1e-3, 8.0 * yard[k])}
    assert not bad, bad


@pytest.mark.parametrize("B,T", [(1, 1), (3, 37), (64, 800)])
def test_fused_loss_and_gradient_seeds_vs_oracle(B, T):
    """t2_tacotron2_loss (SURVEY 8(f) item 3): Tacotron2Loss + its gradient seeds in one pass vs oracle.tacotron2_loss and
    torch autograd; and the in-place parse_output mask (model.py:487-497) when output_lengths is handed to the kernel."""
    import ctypes as C
    from tacotron2_b200 import _capi
    g = torch.Generator().manual_seed(B * 1000 + T)
    mel, post = torch.randn(B, 80, T, generator=g), torch.randn(B, 80, T, generator=g)
    gate = torch.randn(B, T, generator=g) * 3
    tgt = torch.randn(B, 80, T, generator=g)
    gt = (torch.rand(B, T, generator=g) > 0.7).float()
    lens = torch.randint(1, T + 1, (B,), generator=g); lens[0] = T
    # (a) through the nn.Module: loss value and gradients
    leaves = [x.clone().requires_grad_(True) for x in (mel, post, gate)]
    ref = O.tacotron2_loss(leaves[0], leaves[1], leaves[2], tgt, gt)
    ref.backward()
    dev = [x.clone().cuda().requires_grad_(True) for x in (mel, post, gate)]
    loss = t2.Tacotron2Loss()([dev[0], dev[1], dev[2], None], (tgt.cuda(), gt.cuda()))
    (loss * 3.0).backward()
    assert abs(float(loss) - float(ref)) < 2e-6 * abs(float(ref))
    for a, b in zip(dev, leaves):
        assert rel_err(a.grad, 3.0 * b.grad) < 1e-5
    # (b) the C entry point with output_lengths: masks in place, then the same loss as masking first
    pad = torch.arange(T)[None, :] >= lens[:, None]
    ref_m = O.tacotron2_loss(mel.masked_fill(pad[:, None, :], 0.0), post.masked_fill(pad[:, None, :], 0.0),
                             gate.masked_fill(pad, 1e3), tgt, gt)
    L = _capi.lib()
    m_d, p_d, g_d, t_d, gt_d = (x.clone().cuda().contiguous() for x in (mel, post, gate, tgt, gt))
    l32 = lens.to(torch.int32).cuda()
    out = torch.empty(4, device="cuda")
    ws = torch.empty(int(L.t2_loss_workspace_bytes()), dtype=torch.uint8, device="cuda")
    a = _capi.T2LossArgs()
    a.mel, a.mel_post, a.gate, a.mel_target, a.gate_target = (x.data_ptr() for x in (m_d, p_d, g_d, t_d, gt_d))
    a.output_lengths, a.B, a.C, a.T, a.loss = l32.data_ptr(), B, 80, T, out.data_ptr()
    a.ws, a.ws_bytes = ws.data_ptr(), ws.numel()
    _capi.check(L.t2_tacotron2_loss(C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert abs(float(out[0]) - float(ref_m)) < 2e-6 * abs(float(ref_m))
    assert torch.equal(m_d.cpu(), mel.masked_fill(pad[:, None, :], 0.0)) and torch.equal(g_d.cpu(), gate.masked_fill(pad, 1e3))


def test_running_statistics_updated_by_a_training_forward_reach_the_next_inference():
    """The training-mode kernels update the BatchNorm running statistics through raw pointers (torch's version counters do not
    move); the BN-folded inference images must be rebuilt before the next eval-mode call even when no optimizer step happened in
    between."""
    sd = synth_state_dict(seed=3, gate_bias=-10.0, scale=2.0)
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    model = model.cuda()
    g = torch.Generator().manual_seed(0)
    text = torch.randint(0, 148, (3, 17), generator=g).cuda()
    keep = keep_mask((6, 2, 3, 256), 0.5, 1)
    model.decoder.max_decoder_steps = 6
    model.eval()
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        before = model.inference(text)[1].clone()
    model.train()
    tl = torch.tensor([17, 12, 9]).cuda(); ol = torch.tensor([5, 4, 3]).cuda()
    mels = torch.randn(3, 80, 5, generator=g).cuda()
    with torch.no_grad():
        model((text, tl, mels, 17, ol))                       # updates running_mean / running_var (momentum 0.1), nothing else
    model.eval()
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        after = model.inference(text)[1].clone()
    fresh = t2.Tacotron2(t2.create_hparams())
    fresh.load_state_dict(model.state_dict())
    fresh = fresh.cuda().eval()
    fresh.decoder.max_decoder_steps = 6
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        want = fresh.inference(text)[1]
    assert rel_err(after, want) < 1e-6 and rel_err(before, want) > 1e-4
