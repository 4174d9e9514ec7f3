"""GPU (H100): the mixed-precision training flow (BASELINE.json configs[2] / [3] say "fp16": the reference trains through
Apex AMP O2, train.py:173-176, 222-236) -- tacotron2_b200.amp + AmpFusedClipAdam (t2_amp_adam_step).

(1) the optimizer step alone against torch: unscale -> clip_grad_norm_ on fp32 master gradients -> torch.optim.Adam ->
    fp16 write-back, with an overflow step in the middle (skip, scale / 2) and scale growth;
(2) a whole O2-shaped training step of the model against the CPU oracle run in fp32 WITH THE SAME ROUNDING POINTS: fp16
    parameter storage (BatchNorm fp32), fp16 tensors between encoder / decoder / postnet and for the outputs, fp32 loss,
    loss scale, fp16 gradients, fp32 masters."""
import re

import pytest
import torch

import tacotron2_b200 as t2
from oracle import tacotron2_oracle as O
from tests.common import rel_err
from tests.test_oracle_golden import grad_inputs, load

pytestmark = pytest.mark.gpu


def test_amp_adam_step_matches_torch_adam_on_masters_with_overflow_and_growth():
    g = torch.Generator().manual_seed(0)
    shapes = [(257, 33), (4096,), (5, 7, 3), (1,)]
    halfs = [True, True, False, True]                       # an fp32 tensor among them (BatchNorm under O2)
    w0 = [torch.randn(s, generator=g) * 0.1 for s in shapes]
    params = [torch.nn.Parameter((w.half() if h else w.clone()).cuda()) for w, h in zip(w0, halfs)]
    opt = t2.AmpFusedClipAdam(params, lr=1e-2, weight_decay=1e-3, init_scale=1024.0, growth_interval=2)
    masters = [torch.nn.Parameter(p.detach().float().cpu().clone()) for p in params]     # apex: masters start from the model copies
    ref = torch.optim.Adam(masters, lr=1e-2, weight_decay=1e-3)
    scale, good = 1024.0, 0
    for it in range(6):
        grads = [torch.randn(s, generator=g) * (10.0 ** -(it % 3)) for s in shapes]
        overflow = it == 2
        for p, gr, h in zip(params, grads, halfs):
            sg = gr * scale
            if overflow and p is params[1]:
                sg = sg.clone(); sg.view(-1)[17] = float("inf")
            p.grad = (sg.half() if h else sg).cuda()
        norm = opt.step(max_norm=0.5)
        # ---- the same step in torch on the masters ----
        un = [(p.grad.float().cpu() / scale) for p in params]
        total = torch.sqrt(sum((u.double() ** 2).sum() for u in un)).float()
        if not torch.isfinite(total):
            assert opt.last_step_skipped()
            scale, good = max(scale * 0.5, 1.0), 0
        else:
            assert not opt.last_step_skipped()
            assert abs(float(norm) - float(total)) < 1e-5 * float(total)
            for mp, u in zip(masters, un):
                mp.grad = u.clone()
            torch.nn.utils.clip_grad_norm_(masters, 0.5)
            ref.step()
            good += 1
            if good >= 2:
                scale, good = scale * 2.0, 0
        assert float(opt.loss_scale()) == scale, (it, float(opt.loss_scale()), scale)
        for p, mp, h in zip(params, masters, halfs):
            m_eng = opt.state[p]["master"].cpu()
            assert rel_err(m_eng, mp.data) < 2e-6, it
            assert torch.equal(p.detach().cpu(), m_eng.half() if h else m_eng)            # model copy = rounded master
    assert opt.steps_taken() == 5                                                        # the overflow step does not count
    sd = opt.state_dict()
    assert sd["amp_scaler"][0] == scale and float(sd["state"][0]["step"]) == 5.0


class _Round16(torch.autograd.Function):
    """fp16 rounding point with the engine's gradient behaviour: values AND gradients pass through fp16."""

    @staticmethod
    def forward(ctx, x):
        return x.half().float()

    @staticmethod
    def backward(ctx, g):
        return g.half().float()


class _Round16Jitter(torch.autograd.Function):
    """_Round16 whose GRADIENT is perturbed by 2.5e-4 relative noise before the fp16 rounding: two implementations that agree
    to 2.5e-4 before a rounding point land on different fp16 neighbours about half of the time.  Running the emulation with
    and without it measures how strongly a parameter gradient depends on those coin flips."""

    @staticmethod
    def forward(ctx, x):
        return x.half().float()

    @staticmethod
    def backward(ctx, g):
        gen = torch.Generator().manual_seed(1234)
        return (g * (1.0 + 2.5e-4 * torch.randn(g.shape, generator=gen))).half().float()


def test_o2_training_step_matches_oracle_with_the_same_rounding_points():
    gfix = load("grad_train_b4")
    sd, text, tl, ol, mels, gt, m = grad_inputs(gfix)
    S = 4096.0
    smv = float(torch.finfo(torch.float16).min)                                  # train.py:75-76
    lr, wd, max_norm = 1e-3, 1e-6, 1.0
    # ---- engine: the train.py flow with tacotron2_b200.amp in place of apex.amp ----
    model = t2.Tacotron2(t2.create_hparams("fp16_run=True"))
    model.load_state_dict(sd)
    model = model.cuda().train()
    model.decoder.attention_layer.score_mask_value = smv
    optimizer = torch.optim.Adam(model.parameters(), lr=lr, weight_decay=wd)
    model, optimizer = t2.amp.initialize(model, optimizer, opt_level="O2", loss_scale=S)
    assert model.embedding.weight.dtype == torch.float16 and model.postnet.convolutions[0][1].weight.dtype == torch.float32
    post_keep = [m["qk4"][i] for i in range(4)] + [m["qk1"]]
    with t2.dropout_masks(prenet=m["pk"], att=m["ak"], dec=m["dk"], enc=m["ek"], post=post_keep):
        out = model((text.cuda(), tl.cuda(), mels.cuda(), int(tl.max()), ol.cuda()))
        assert all(o.dtype == torch.float32 for o in out)
        loss = t2.Tacotron2Loss()(out, (mels.cuda(), gt.cuda()))
        with t2.amp.scale_loss(loss, optimizer) as scaled_loss:
            scaled_loss.backward()
    grads_eng = {k: p.grad.detach().float().cpu() for k, p in model.named_parameters()}
    assert model.decoder.attention_rnn.weight_ih.grad.dtype == torch.float16
    norm = optimizer.step(max_norm=max_norm)
    torch.cuda.synchronize()
    assert not optimizer.last_step_skipped()

    # ---- oracle, fp32, same rounding points ----
    is_bn = lambda k: re.search(r"convolutions\.\d+\.1\.", k) is not None     # Sequential(ConvNorm, BatchNorm1d)[1]
    w16 = {k: (v if (not v.dtype.is_floating_point or is_bn(k)) else v.half().float()) for k, v in sd.items()}
    names = [k for k, v in w16.items() if v.dtype.is_floating_point and "running" not in k]
    R = _Round16.apply

    def emulate(round_memory):
        sdg = dict(w16)
        for k in names:
            sdg[k] = w16[k].clone().requires_grad_(True)
        emb = sdg["embedding.weight"][text].transpose(1, 2)
        memory = round_memory(O.encoder(sdg, emb, tl, True, m["ek"]))
        mel, gate, align = O.decoder_forward(sdg, memory, mels, tl, m["pk"], m["ak"], m["dk"], True, smv)
        mel, gate = R(mel), R(gate)
        pad = ~O.get_mask_from_lengths(ol, mel.shape[2])
        wgrad_x0 = mel.masked_fill(pad.unsqueeze(1), 0.0)
        post = R(mel + O.postnet(sdg, mel, True, post_keep, wgrad_x0))
        mel_m, post_m = mel.masked_fill(pad.unsqueeze(1), 0.0), post.masked_fill(pad.unsqueeze(1), 0.0)
        gate_m = gate.masked_fill(pad, 1e3)
        ref_loss = O.tacotron2_loss(mel_m, post_m, gate_m, mels, gt)
        (ref_loss * S).backward()
        g16 = {k: (sdg[k].grad if is_bn(k) else sdg[k].grad.half().float()) for k in names}     # fp16 gradient storage
        return ref_loss.detach(), mel_m.detach(), post_m.detach(), g16

    ref_loss, mel_m, post_m, g16 = emulate(R)
    # how much of a gradient is decided by fp16 coin flips at the encoder / decoder boundary: the encoder's conv-stack
    # gradients pass through three training-mode BatchNorm backward passes (mean subtraction = cancellation) after d_memory
    # was rounded to fp16 -- at this size (96 samples per channel) that moves them by several per cent, in Apex as here
    _, _, _, g16_j = emulate(_Round16Jitter.apply)
    assert abs(float(loss) - float(ref_loss)) < 2e-4 * abs(float(ref_loss))
    assert rel_err(out[0], mel_m) < 1e-3 and rel_err(out[1], post_m) < 1e-3
    errs = {}
    for k in names:
        gmax = float(g16[k].abs().max())
        if gmax / S < 1e-5:
            continue
        errs[k] = float((grads_eng[k] - g16[k]).abs().max()) / gmax
    worst = max(errs.values())
    print("O2 fp16 gradients, largest deviations:", ", ".join("%s %.1e" % kv for kv in sorted(errs.items(), key=lambda kv: -kv[1])[:8]))
    yard = {k: float((g16_j[k] - g16[k]).abs().max()) / float(g16[k].abs().max()) for k in errs}
    print("   sensitivity of the same gradients to fp16 rounding coin flips at the memory boundary:",
          ", ".join("%s %.1e" % (k, yard[k]) for k, _ in sorted(errs.items(), key=lambda kv: -kv[1])[:8]))
    # both sides round to fp16 (2^-11 relative on top of the 1e-3 bar); parameters whose gradient hinges on the coin flips are
    # held to 4x the measured sensitivity instead
    bad = {k: (v, yard[k]) for k, v in errs.items() if not v < max(2e-3, 4.0 * yard[k])}
    assert not bad, bad
    # the optimizer half of the step, from the gradients the engine produced (their agreement with the oracle is settled above)
    un = {k: grads_eng[k] / S for k in names}
    total = float(torch.sqrt(sum((u.double() ** 2).sum() for u in un.values())))
    total_ref = float(torch.sqrt(sum(((g16[k] / S).double() ** 2).sum() for k in names)))
    assert abs(float(norm) - total) < 1e-5 * total and abs(total - total_ref) < 2e-2 * total_ref
    coef = min(1.0, max_norm / (total + 1e-6))
    for k, p in model.named_parameters():
        st = optimizer.state[p]
        ref_m = (1 - 0.9) * (un[k] * coef + wd * w16[k])                                    # exp_avg after step 1
        if float(ref_m.abs().max()) > 1e-7:
            assert rel_err(st["exp_avg"], ref_m) < 1e-5, k
        delta = st["master"].cpu() - w16[k]
        assert float(delta.abs().max()) <= lr * 1.0001 and float(delta.abs().max()) > 0        # Adam's first step: |delta| <= lr
        assert torch.equal(p.detach().cpu(), st["master"].cpu().to(p.dtype))                 # model copy = rounded master
    print("O2 step: loss %.6f (oracle %.6f), worst fp16-gradient deviation %.2e, grad norm %.5f (oracle %.5f)" %
          (float(loss), float(ref_loss), worst, float(norm), total))
