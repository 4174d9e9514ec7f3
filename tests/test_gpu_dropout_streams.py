"""The production dropout path: masks drawn inside the kernels from Philox4x32-10, keyed by (seed, site, element).

Every other oracle comparison injects its masks (``t2.dropout_masks``), so by itself it cannot see a kernel that draws
a different mask than the reference layout says, nor a forward and a backward kernel of the same layer that disagree
on a site, an index or a scale.  Here ``tests/philox_ref.py`` rebuilds every mask a Philox run drew, from the seed each
engine call used (recorded by the ``seed_log`` fixture), and

* the same call with the rebuilt masks injected must be bit-identical to the Philox run: the kernels consume an
  injected mask and their own draw through the same arithmetic, so any difference is a different mask;
* the Philox run must match the fp64 oracle fed the rebuilt masks: that pins the forward AND the backward of each layer
  to the mask the reference layout defines.

The CPU tests check the rebuild itself (Random123 known answers, the threshold rule) and the statistics of the masks at
the production shapes.  The tests marked ``gpu`` need an H100."""
import contextlib

import pytest
import torch

import tacotron2_b200 as t2
from oracle import tacotron2_oracle as O
from tacotron2_b200 import _capi, _engine
from tacotron2_b200._engine import Engine
from tests import philox_ref as P
from tests.common import rand_text, rel_err, synth_state_dict
from tests.test_oracle_golden import grad_inputs, load, oracle_train_step

gpu = pytest.mark.gpu
HP = t2.create_hparams()
P_ATT, P_DEC = HP.p_attention_dropout, HP.p_decoder_dropout


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the host rebuild and the statistics of the streams
# ---------------------------------------------------------------------------------------------------------------------

def test_philox_reproduces_random123_known_answers():
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        assert [int(w) for w in P.philox4x32_10(ctr, key)] == list(want)


def test_keep_decision_at_the_threshold_is_u_ge_p():
    seed, site = 0x0123456789abcdef, 0xA1
    idx = torch.arange(4096)
    u = P.uniform(seed, site, idx)
    assert u.dtype == torch.float32 and float(u.min()) >= 0.0 and float(u.max()) < 1.0
    assert torch.equal(u * 16777216.0, (u * 16777216.0).round())          # 24-bit grid: (o >> 8) * 2^-24
    i = int(torch.argmin((u - 0.5).abs()))
    at = float(u[i])
    above = float(torch.nextafter(torch.tensor(at), torch.tensor(2.0)))
    assert bool(P.keep(seed, site, idx[i:i + 1], at)[0])                   # u == p: kept
    assert not bool(P.keep(seed, site, idx[i:i + 1], above)[0])            # p one fp32 ulp above u: dropped
    # the bulk builders use the same rule and the same lane order as the per-element path
    assert torch.equal(P._stream(seed, [site], 4096, at, "cpu")[0].bool(), u >= at)


def test_the_64_bit_seed_and_block_index_reach_the_key_and_counter():
    idx = torch.tensor([5, 5 + (1 << 34)])                                  # same lane, block differs only in its high word
    u = P.uniform(7, 3, idx)
    assert float(u[0]) != float(u[1])
    assert float(P.uniform(7, 3, idx[:1])[0]) != float(P.uniform(7 + (1 << 32), 3, idx[:1])[0])


def _rate(a, b=None):
    """(fraction kept) or (fraction of elements on which a and b agree), and the number of elements."""
    a = a.reshape(-1)
    if b is None:
        return int(a.sum()) / a.numel(), a.numel()
    return int((a == b.reshape(-1)).sum()) / a.numel(), a.numel()


def _within_6_sigma(rate, n, expect):
    sigma = (expect * (1 - expect) / n) ** 0.5
    return abs(rate - expect) < 6 * sigma


@pytest.fixture(scope="module")
def production_masks():
    """Every stream of one training step (B=64, T_text=150, T_mel=800) and one inference (cap 1000), distinct seeds."""
    B, Tt, Tm, cap = 64, 150, 800, 1000
    return dict(enc=P.encoder_masks(11, B, Tt), post=P.postnet_masks(12, B, Tm), pk=P.teacher_prenet_masks(13, Tm, B),
                ak=P.lstm_masks(14, Tm, B, "att", P_ATT), dk=P.lstm_masks(14, Tm, B, "dec", P_DEC),
                ik=P.infer_prenet_masks(15, cap, B))


def test_mask_keep_rates_at_production_shapes(production_masks):
    m = production_masks
    cases = [("enc", m["enc"], 0.5), ("pk", m["pk"], 0.5), ("ik", m["ik"], 0.5), ("ak", m["ak"], 1 - P_ATT),
             ("dk", m["dk"], 1 - P_DEC)] + [("post%d" % i, k, 0.5) for i, k in enumerate(m["post"])]
    for name, k, q in cases:
        rate, n = _rate(k)
        assert _within_6_sigma(rate, n, q), (name, rate, q, n)


def test_mask_streams_are_independent_at_production_shapes(production_masks):
    """Pairs that a wrong site or index would correlate agree only at chance level, p^2 + (1-p)^2."""
    m = production_masks
    half = 0.5
    pairs = [
        ("teacher prenet layer 0 / 1", m["pk"][:, 0], m["pk"][:, 1], half),
        ("inference prenet layer 0 / 1", m["ik"][:, 0], m["ik"][:, 1], half),
        ("teacher prenet consecutive steps", m["pk"][:-1], m["pk"][1:], half),
        ("inference prenet consecutive steps", m["ik"][:-1], m["ik"][1:], half),
        ("attention LSTM consecutive steps", m["ak"][:-1], m["ak"][1:], P_ATT),
        ("decoder LSTM consecutive steps", m["dk"][:-1], m["dk"][1:], P_DEC),
        ("attention / decoder LSTM of one step", m["ak"], m["dk"], P_ATT),
        ("attention LSTM neighbouring rows", m["ak"][:, :-1], m["ak"][:, 1:], P_ATT),
        ("inference prenet neighbouring rows", m["ik"][:, :, :-1], m["ik"][:, :, 1:], half),
        ("encoder neighbouring rows", m["enc"][:, :-1], m["enc"][:, 1:], half),
        ("encoder conv i / i+1", m["enc"][:-1], m["enc"][1:], half),
        ("postnet conv i / i+1", torch.stack(m["post"][:3]), torch.stack(m["post"][1:4]), half),
    ]
    # the 4 lanes of one Philox block: consecutive elements of the flat (element-index-ordered) streams
    for name, k, p in (("attention LSTM", m["ak"], P_ATT), ("inference prenet", m["ik"], half)):
        lanes = k.reshape(-1, 4)
        for a in range(4):
            for b in range(a + 1, 4):
                pairs.append(("%s lanes %d / %d" % (name, a, b), lanes[:, a], lanes[:, b], p))
    enc_lanes = m["enc"].permute(0, 1, 3, 2).reshape(-1, 4)                  # element index (b*T + t)*512 + c
    pairs += [("encoder lanes 0 / %d" % b, enc_lanes[:, 0], enc_lanes[:, b], half) for b in (1, 2, 3)]
    bad = []
    for name, a, b, p in pairs:
        expect = p * p + (1 - p) * (1 - p)
        rate, n = _rate(a, b)
        if not _within_6_sigma(rate, n, expect):
            bad.append((name, rate, expect))
    assert not bad, bad


def test_distinct_seeds_are_what_keeps_decoder_and_encoder_sites_apart():
    """Decoder site t*4+k reaches the encoder's 1000+i at t = 250: under one seed those streams would be the same bits."""
    assert 250 * 4 + 0 == 1000 and 250 * 4 + 2 == 1002
    enc = P.encoder_masks(99, 2, 256)[0].permute(0, 2, 1).reshape(-1)[:256 * 2]      # site 1000, elements 0..511
    ik = P.infer_prenet_masks(99, 251, 2)[250, 0].reshape(-1)                        # site 250*4+0, elements 0..511
    assert torch.equal(enc, ik)
    assert not torch.equal(enc, P.infer_prenet_masks(100, 251, 2)[250, 0].reshape(-1))


def test_decoder_inference_stream_refuses_training_mode():
    """Training-mode inference() applies the hidden-state dropout; the resumable decoder does not, so it refuses."""
    model = t2.Tacotron2(HP).train()
    with pytest.raises(RuntimeError, match="eval mode"):
        next(model.decoder.inference_stream(torch.zeros(1, 5, 512)))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: Philox runs against host-rebuilt masks and the fp64 oracle
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture
def seed_log(monkeypatch):
    """Records (engine call, seed) for every dropout-capable engine call.  A call made without a seed draws next_seed()
    here and passes it on, so the log holds the seed of every call whatever the caller's order."""
    log = []

    def wrap(name):
        orig = getattr(Engine, name)

        def call(self, *args, seed=None, **kw):
            if seed is None:
                seed = _engine.next_seed()
            log.append((name, seed))
            return orig(self, *args, seed=seed, **kw)
        monkeypatch.setattr(Engine, name, call)

    for name in ("encoder", "prenet", "decoder", "decoder_stream", "postnet", "infer_host"):
        wrap(name)
    return log


def _seed_of(log, name):
    seeds = [s for n, s in log if n == name]
    assert len(seeds) == 1, (name, log)
    return seeds[0]


def _model(sd, training, half=False, cap=None, impl=None):
    model = t2.Tacotron2(HP)
    model.load_state_dict(sd)
    model = model.cuda().train(training)
    if half:
        model = model.half()
    if cap is not None:
        model.decoder.max_decoder_steps = cap
    if impl is not None:
        model._t2_engine().impl = impl
    return model


def _masked(masks):
    return t2.dropout_masks(**masks) if masks is not None else contextlib.nullcontext()


def _infer(model, text, masks=None):
    with torch.no_grad(), _masked(masks):
        out = model.inference(text.cuda())
    torch.cuda.synchronize()
    return [o.cpu() for o in out] + [model.mel_lengths.cpu()]


def _rebuild_inference_masks(log, B, cap, n, training):
    """dropout_masks kwargs for the Tacotron2.inference call that `log` recorded (n = frames it returned)."""
    s_dec = _seed_of(log, "decoder")
    masks = dict(prenet=P.infer_prenet_masks(s_dec, cap, B))
    if training:
        masks.update(att=P.lstm_masks(s_dec, cap, B, "att", P_ATT), dec=P.lstm_masks(s_dec, cap, B, "dec", P_DEC),
                     post=P.postnet_masks(_seed_of(log, "postnet"), B, n))
    return masks


def _assert_all_equal(a, b, names):
    bad = [nm for x, y, nm in zip(a, b, names) if not (x.shape == y.shape and torch.equal(x, y))]
    assert not bad, bad


INFER_OUT = ["mel", "mel_postnet", "gate", "alignments", "mel_lengths"]
CAP = 24


def _infer_case(B, seed=3):
    # a gate this close to the threshold stops rows at different steps within the cap (and lets some run to it); at
    # B=65 the second 64-row slice stops several steps before the first, leaving frames its launch never writes
    return synth_state_dict(77, gate_bias=0.09, scale=1.0, gate_sign=-4.0), rand_text(B, 29, seed)


@gpu
@pytest.mark.parametrize("impl", [_capi.IMPL_STEPWISE, _capi.IMPL_PERSISTENT])
@pytest.mark.parametrize("B,half", [(1, False), (3, False), (64, False), (65, False), (3, True)])
def test_inference_philox_equals_rebuilt_masks(B, half, impl, seed_log):
    """Tacotron2.inference (eval: only the prenet dropout, model.py:99): the Philox run vs the same call with the rebuilt
    masks.  At B=65 the persistent decoder runs two 64-row slices; the second draws its bits at absolute rows 64+."""
    sd, text = _infer_case(B)
    model = _model(sd, False, half=half, cap=CAP, impl=impl)
    ph = _infer(model, text)
    masks = _rebuild_inference_masks(seed_log, B, CAP, ph[0].shape[2], False)
    inj = _infer(model, text, masks)
    _assert_all_equal(ph, inj, INFER_OUT)
    print("inference B=%d impl=%d half=%s: lengths %s" % (B, impl, half, ph[4].tolist()[:8]))


@gpu
@pytest.mark.parametrize("impl", [_capi.IMPL_STEPWISE, _capi.IMPL_PERSISTENT])
def test_training_mode_inference_matches_fp64_oracle_and_rebuilt_masks(impl, seed_log):
    """A model in train() mode runs inference with batch-statistics BatchNorm and every dropout of the reference,
    including the attention / decoder hidden-state dropout of decode() (model.py:355-356, 370-371)."""
    sd = synth_state_dict(5, gate_bias=-10.0, scale=2.0)
    text = rand_text(1, 19, 3)
    cap = 16
    model = _model(sd, True, cap=cap, impl=impl)
    ph = _infer(model, text)
    n = ph[0].shape[2]
    masks = _rebuild_inference_masks(seed_log, 1, cap, n, True)
    masks["enc"] = P.encoder_masks(_seed_of(seed_log, "encoder"), 1, text.shape[1])
    sd64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in sd.items()}
    ref = O.tacotron2_inference(sd64, text, masks["prenet"], 0.5, cap, training=True, enc_keep=masks["enc"],
                                att_keep=masks["att"], dec_keep=masks["dec"], post_keep=masks["post"])
    errs = [rel_err(ph[0], ref[0]), rel_err(ph[1], ref[1]), rel_err(ph[2].squeeze(-1), ref[2].squeeze(-1)),
            rel_err(ph[3], ref[3])]
    print("training-mode inference impl=%d: rel err mel %.2e post %.2e gate %.2e align %.2e" % (impl, *errs))
    assert ph[4].tolist() == ref[4].tolist()
    assert max(errs) < 1e-3, errs
    inj = _infer(model, text, masks)
    _assert_all_equal(ph, inj, INFER_OUT)


@gpu
def test_eval_inference_matches_fp64_oracle_with_rebuilt_prenet_masks(seed_log):
    sd = synth_state_dict(5, gate_bias=-10.0, scale=2.0)
    text = rand_text(1, 19, 3)
    cap = 16
    ph = _infer(_model(sd, False, cap=cap), text)
    pk = P.infer_prenet_masks(_seed_of(seed_log, "decoder"), cap, 1)
    sd64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in sd.items()}
    ref = O.tacotron2_inference(sd64, text, pk, 0.5, cap)
    errs = [rel_err(ph[0], ref[0]), rel_err(ph[1], ref[1]), rel_err(ph[3], ref[3])]
    print("eval inference: rel err mel %.2e post %.2e align %.2e" % tuple(errs))
    assert ph[4].tolist() == ref[4].tolist() and max(errs) < 1e-3, errs


@gpu
@pytest.mark.parametrize("B", [3, 65])
def test_infer_host_equals_inference_and_never_reads_unwritten_frames(B, seed_log):
    """t2_infer_host (host buffers, explicit seed) vs Tacotron2.inference with the prenet masks rebuilt from that seed.
    Its workspace is not cleared between calls, and the decoder leaves every frame past a row's stop unwritten; the
    postnet's length mask must keep those out.  The second call runs on a workspace whose every byte is 0xFF (every
    fp32 word a NaN) and must give the same bits."""
    sd, text = _infer_case(B)
    model = _model(sd, False, cap=CAP)
    eng = model._t2_engine()
    seed = 0x5eed0000 + B
    text_h = text.pin_memory()

    def host_run():
        mel_post, lens, ns = eng.infer_host(text_h, CAP, model.decoder.gate_threshold, seed=seed)
        return mel_post.clone(), lens.clone(), int(ns[0])

    mel_post, lens, n = host_run()
    ref = _infer(model, text, dict(prenet=P.infer_prenet_masks(seed, CAP, B)))
    assert n == ref[0].shape[2]
    assert torch.equal(lens, ref[4])
    assert torch.equal(mel_post[:, :, :n], ref[1])
    t = torch.arange(CAP)
    beyond = t[None, :] >= lens[:, None].long()
    assert torch.isfinite(mel_post).all()
    assert bool((mel_post.masked_select(beyond.unsqueeze(1)) == 0).all())         # frames past each row's length
    print("infer_host B=%d: n_steps %d, rows stopping before the cap: %d" % (B, n, int((lens < CAP).sum())))
    eng._ws["e2e"].fill_(0xFF)
    mel_post2, lens2, n2 = host_run()
    assert n2 == n and torch.equal(lens2, lens) and torch.equal(mel_post2, mel_post)


def _ragged_case(B=64, Tt=40, Tm=60, seed=7):
    g = torch.Generator().manual_seed(seed)
    tl = torch.randint(Tt // 2, Tt + 1, (B,), generator=g)
    tl[0] = Tt
    tl, _ = torch.sort(tl, descending=True)
    ol = torch.randint(Tm // 2, Tm + 1, (B,), generator=g)
    ol[B // 2] = Tm
    mels = torch.randn(B, 80, Tm, generator=g) * 0.5
    gt = (torch.arange(Tm)[None, :] >= ol[:, None] - 1).float()
    return synth_state_dict(1234, scale=2.0), rand_text(B, Tt, seed + 1), tl, ol, mels, gt


def _forward_masks(log, B, Tt, Tm, training):
    """dropout_masks kwargs for the Tacotron2.forward call that `log` recorded."""
    masks = dict(prenet=P.teacher_prenet_masks(_seed_of(log, "prenet"), Tm, B))
    if training:
        s_dec = _seed_of(log, "decoder")
        masks.update(enc=P.encoder_masks(_seed_of(log, "encoder"), B, Tt), att=P.lstm_masks(s_dec, Tm, B, "att", P_ATT),
                     dec=P.lstm_masks(s_dec, Tm, B, "dec", P_DEC), post=P.postnet_masks(_seed_of(log, "postnet"), B, Tm))
    return masks


def _train_step(sd, text, tl, ol, mels, gt, masks=None):
    model = _model(sd, True)
    with _masked(masks):
        out = model((text.cuda(), tl.cuda(), mels.cuda(), int(tl.max()), ol.cuda()))
        loss = t2.Tacotron2Loss()(out, (mels.cuda(), gt.cuda()))
        loss.backward()
    torch.cuda.synchronize()
    return loss.detach().cpu(), [o.detach().cpu() for o in out], {k: p.grad.cpu() for k, p in model.named_parameters()}


@gpu
@pytest.mark.parametrize("training", [False, True])
def test_teacher_forced_forward_without_grad_philox_equals_rebuilt_masks(training, seed_log):
    """In training mode under no_grad the encoder and postnet run the training conv stack without a stash (its
    bn_act_kernel draws the dropout masks) rather than with the autograd stash; in eval mode only the prenet dropout is
    active."""
    sd, text, tl, ol, mels, gt = _ragged_case(8, 30, 20, seed=9)
    outs = []
    for masks in (None, "rebuilt"):
        if masks == "rebuilt":
            masks = _forward_masks(seed_log, 8, 30, 20, training)
        model = _model(sd, training)
        with torch.no_grad(), _masked(masks):
            out = model((text.cuda(), tl.cuda(), mels.cuda(), int(tl.max()), ol.cuda()))
        outs.append([o.cpu() for o in out])
    _assert_all_equal(outs[0], outs[1], ["mel", "mel_postnet", "gate", "alignments"])


def _train_case(name):
    if name == "grad_train_b4":
        sd, text, tl, ol, mels, gt, _ = grad_inputs(load("grad_train_b4"))
        return sd, text, tl, ol, mels, gt
    return _ragged_case()


@gpu
@pytest.mark.parametrize("case", ["grad_train_b4", "ragged_b64"])
def test_training_step_philox_equals_rebuilt_masks(case, seed_log):
    """Tacotron2 + Tacotron2Loss + backward: loss, every output and every parameter gradient bit-identical.  In the
    Philox run each backward kernel redraws the mask of its forward; with injected masks both read the same tensor."""
    sd, text, tl, ol, mels, gt = _train_case(case)
    B, Tt, Tm = text.shape[0], text.shape[1], mels.shape[2]
    ph = _train_step(sd, text, tl, ol, mels, gt)
    inj = _train_step(sd, text, tl, ol, mels, gt, _forward_masks(seed_log, B, Tt, Tm, True))
    assert torch.equal(ph[0], inj[0])
    _assert_all_equal(ph[1], inj[1], ["mel", "mel_postnet", "gate", "alignments"])
    bad = [k for k in ph[2] if not torch.equal(ph[2][k], inj[2][k])]
    assert not bad, bad


@gpu
def test_training_step_philox_matches_fp64_oracle_with_rebuilt_masks(seed_log):
    """The production-mode step at the grad_train_b4 inputs against the fp64 oracle fed the masks the kernels drew, at
    the bars of test_full_train_step_matches_reference_gradient_golden (loss 1e-4, outputs and gradients 1e-3)."""
    sd, text, tl, ol, mels, gt = _train_case("grad_train_b4")
    B, Tt, Tm = text.shape[0], text.shape[1], mels.shape[2]
    loss, out, grads = _train_step(sd, text, tl, ol, mels, gt)
    mk = _forward_masks(seed_log, B, Tt, Tm, True)
    m = dict(pk=mk["prenet"], ak=mk["att"], dk=mk["dec"], ek=mk["enc"], qk4=torch.stack(mk["post"][:4]), qk1=mk["post"][4])
    ref_loss, ref_out, ref_g = oracle_train_step(sd, text, tl, ol, mels, gt, m, True, dtype=torch.float64)
    assert abs(float(loss) - float(ref_loss)) < 1e-4 * abs(float(ref_loss))
    assert rel_err(out[0], ref_out[0]) < 1e-3 and rel_err(out[1], ref_out[1]) < 1e-3
    errs = {k: rel_err(v, ref_g[k]) for k, v in grads.items() if float(ref_g[k].abs().max()) >= 1e-5}
    print("Philox train step vs fp64 oracle: loss %.6f (oracle %.6f), worst gradient error %.2e (%s)" %
          (float(loss), float(ref_loss), max(errs.values()), max(errs, key=errs.get)))
    bad = {k: v for k, v in errs.items() if not v < 1e-3}
    assert not bad, bad


@gpu
def test_amp_o2_step_philox_equals_rebuilt_masks(seed_log):
    """One AMP O2 step (tacotron2_b200.amp + AmpFusedClipAdam): master weights, loss scale and the skip decision."""
    sd, text, tl, ol, mels, gt = _train_case("grad_train_b4")
    B, Tt, Tm = text.shape[0], text.shape[1], mels.shape[2]

    def step(masks):
        model = t2.Tacotron2(t2.create_hparams("fp16_run=True"))
        model.load_state_dict(sd)
        model = model.cuda().train()
        model.decoder.attention_layer.score_mask_value = float(torch.finfo(torch.float16).min)
        optimizer = torch.optim.Adam(model.parameters(), lr=1e-3, weight_decay=1e-6)
        model, optimizer = t2.amp.initialize(model, optimizer, opt_level="O2", loss_scale="dynamic")
        with _masked(masks):
            out = model((text.cuda(), tl.cuda(), mels.cuda(), int(tl.max()), ol.cuda()))
            loss = t2.Tacotron2Loss()(out, (mels.cuda(), gt.cuda()))
            with t2.amp.scale_loss(loss, optimizer) as scaled_loss:
                scaled_loss.backward()
        optimizer.step(max_norm=1.0)
        torch.cuda.synchronize()
        masters = {k: optimizer.state[p]["master"].cpu() for k, p in model.named_parameters()}
        return float(loss), masters, float(optimizer.loss_scale()), optimizer.last_step_skipped()

    ph = step(None)
    inj = step(_forward_masks(seed_log, B, Tt, Tm, True))
    assert ph[0] == inj[0] and ph[2] == inj[2] and ph[3] == inj[3]
    bad = [k for k in ph[1] if not torch.equal(ph[1][k], inj[1][k])]
    assert not bad, bad


@gpu
def test_every_engine_call_of_a_step_and_an_inference_has_its_own_seed(seed_log):
    sd, text, tl, ol, mels, gt = _train_case("grad_train_b4")
    _train_step(sd, text, tl, ol, mels, gt)
    _infer(_model(sd, True, cap=8), text)
    names = sorted(n for n, _ in seed_log)
    assert names == sorted(["encoder", "prenet", "decoder", "postnet"] + ["encoder", "decoder", "postnet"]), names
    seeds = [s for _, s in seed_log]
    assert len(set(seeds)) == len(seeds), seed_log
