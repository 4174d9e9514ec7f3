"""GPU (H100): the CUDA path through the public nn.Module API / C-ABI vs (a) the golden vectors
produced by the reference model.py and (b) the CPU oracle on fresh seeded inputs.

Tolerance (north_star): mel frames within 1e-3 relative fp32 -- measured as max|a-b| / max|b| --
and stop decisions (mel_lengths) bit-exact.  The engine is expected to land ~1e-5."""
import ctypes as C

import pytest
import torch

import tacotron2_b200 as t2
from oracle import tacotron2_oracle as O
from tacotron2_b200 import _capi
from tests.common import keep_mask, rand_text, rel_err, synth_state_dict
from tests.test_oracle_golden import FULL_INFER, INFER, check_full_inference, forward_inputs, infer_inputs, load

pytestmark = pytest.mark.gpu
TOL = 1e-3
IMPLS = [(_capi.IMPL_STEPWISE, "stepwise"), (_capi.IMPL_PERSISTENT, "persistent")]


def make_model(sd, max_steps=None, impl=None, training=False):
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    model = model.cuda().train(training)
    if max_steps is not None:
        model.decoder.max_decoder_steps = max_steps
    if impl is not None:
        model._t2_engine().impl = impl
    return model


def test_native_library_is_loaded():
    L = _capi.lib()
    info = (C.c_int32 * 5)()
    _capi.check(L.t2_device_info(info))
    assert (info[1], info[2]) == (9, 0), "sm_90 device expected, got sm_%d%d" % (info[1], info[2])


@pytest.mark.parametrize("passes,tol", [(3, 2e-5), (1, 2e-3)])
@pytest.mark.parametrize("N,K", [(32, 256), (8, 64), (64, 1024), (80, 192), (48, 1024)])
def test_umma_split_gemm_selftest(N, K, passes, tol):
    """wgmma engine of the persistent decoder: C = 2 * A (64xK) . W (NxK)^T (two accumulating runs)."""
    g = torch.Generator().manual_seed(N * 1000 + K)
    A = torch.randn(64, K, generator=g).cuda()
    W = (torch.randn(N, K, generator=g) / K ** 0.5).cuda()
    Cd = torch.full((64, N), float("nan"), device="cuda")
    _capi.check_selftest(_capi.selftest_lib().t2_selftest_umma(A.data_ptr(), W.data_ptr(), N, K, passes, Cd.data_ptr(),
                                             C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    ref = 2.0 * (A.double() @ W.double().t())
    assert rel_err(Cd, ref) < tol


@pytest.mark.parametrize("impl,impl_name", IMPLS)
@pytest.mark.parametrize("name", INFER)
def test_inference_matches_reference_golden(name, impl, impl_name):
    g = load(name)
    sd, text, keep, S = infer_inputs(g)
    model = make_model(sd, S, impl)
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        mel, post, gate, align = model.inference(text.cuda())
    torch.cuda.synchronize()
    assert model.mel_lengths.cpu().tolist() == g["mel_lengths"].tolist()           # bit-exact stop decisions
    n = int(g["mel"].shape[2])
    assert mel.shape[2] == n and gate.shape == (text.shape[0], n, 1)
    assert rel_err(mel, torch.from_numpy(g["mel_masked"])) < TOL
    assert rel_err(post, torch.from_numpy(g["mel_post"])) < TOL
    assert rel_err(gate, torch.from_numpy(g["gate"])) < TOL
    assert rel_err(align, torch.from_numpy(g["align"])) < TOL
    live = torch.arange(n)[None, :] < torch.from_numpy(g["mel_lengths"])[:, None]
    dec_e = (torch.sigmoid(gate[:, :, 0].cpu()) > 0.5)[live]
    dec_g = (torch.sigmoid(torch.from_numpy(g["gate"])[:, :, 0]) > 0.5)[live]
    assert torch.equal(dec_e, dec_g)


@pytest.mark.parametrize("impl,impl_name", IMPLS)
@pytest.mark.parametrize("name,training", [("forward_eval_b4", False), ("forward_train_b4", True)])
def test_teacher_forced_forward_matches_reference_golden(name, training, impl, impl_name):
    g = load(name)
    sd, text, tl, ol, mels, m = forward_inputs(g)
    model = make_model(sd, impl=impl, training=training)
    post_keep = [m["qk4"][i] for i in range(4)] + [m["qk1"]]
    with torch.no_grad(), t2.dropout_masks(prenet=m["pk"], att=m["ak"], dec=m["dk"], enc=m["ek"], post=post_keep):
        out = model((text.cuda(), tl.cuda(), mels.cuda(), int(tl.max()), ol.cuda()))
    torch.cuda.synchronize()
    for a, k in zip(out, ("mel", "mel_post", "gate", "align")):
        assert rel_err(a, torch.from_numpy(g[k])) < TOL, k
    if training:   # BatchNorm running statistics were updated like nn.BatchNorm1d does
        sd_after = model.state_dict()
        assert rel_err(sd_after["encoder.convolutions.0.1.running_mean"], torch.from_numpy(g["bn0_running_mean"])) < 1e-4
        assert rel_err(sd_after["encoder.convolutions.0.1.running_var"], torch.from_numpy(g["bn0_running_var"])) < 1e-4


@pytest.mark.parametrize("conv_path", ["tc", "train"])
@pytest.mark.parametrize("B,T", [(5, 33), (12, 140)])
def test_encoder_and_postnet_modules_vs_oracle(B, T, conv_path):
    """Encoder (conv stack + packed BiLSTM) and Postnet as stand-alone modules on both conv paths: tc = evaluation mode
    (wgmma implicit-GEMM convs); train = training mode without autograd (the training conv stack: batch statistics and
    injected dropout masks)."""
    training = conv_path == "train"
    sd = synth_state_dict(9, scale=1.5)
    model = make_model(sd, training=training)
    g = torch.Generator().manual_seed(0)
    text = rand_text(B, T, 2)
    lengths = torch.sort(torch.randint(1, T + 1, (B,), generator=g), descending=True)[0]
    lengths[0] = T; lengths[-1] = 1
    emb = sd["embedding.weight"][text].transpose(1, 2)
    x = torch.randn(max(B // 2, 1), 80, T + 8, generator=g)
    enc_keep = post_keep = None
    if training:
        enc_keep = keep_mask((3, B, 512, T), 0.5, 10)
        post_keep = [keep_mask((x.shape[0], 512, x.shape[2]), 0.5, 11 + i) for i in range(4)] + \
                    [keep_mask((x.shape[0], 80, x.shape[2]), 0.5, 15)]
    with torch.no_grad():
        ref_inf = O.encoder(sd, emb, None, training, enc_keep)
        ref_fwd = O.encoder(sd, emb, lengths, training, enc_keep)
        with t2.dropout_masks(enc=enc_keep):
            got_inf = model.encoder.inference(emb.cuda())
            got_fwd = model.encoder(emb.cuda(), lengths.cuda())
        assert rel_err(got_inf, ref_inf) < 1e-4 and rel_err(got_fwd, ref_fwd) < 1e-4
        assert float(got_fwd[-1, 1:].abs().max()) == 0.0                       # zeros at padded positions
        with t2.dropout_masks(post=post_keep):
            got_post = model.postnet(x.cuda())
        assert rel_err(got_post, O.postnet(sd, x, training, post_keep)) < 1e-4


@pytest.mark.parametrize("impl,impl_name", IMPLS)
def test_fresh_inputs_vs_oracle_edge_shapes(impl, impl_name):
    """Ragged / minimal shapes: B=1 T_text=1, odd T_text, B not a multiple of anything."""
    for (B, T, S, seed) in [(1, 1, 5, 1), (7, 13, 9, 2), (2, 150, 6, 3), (70, 11, 4, 4), (3, 300, 3, 5), (2, 270, 3, 6),
                            (2, 129, 4, 7), (2, 160, 3, 8)]:
        sd = synth_state_dict(100 + seed, gate_bias=-10.0, scale=2.0)
        model = make_model(sd, S, impl)
        text = rand_text(B, T, seed)
        keep = keep_mask((S, 2, B, 256), 0.5, seed + 50)
        with torch.no_grad():
            ref = O.tacotron2_inference(sd, text, keep, 0.5, S)
            with t2.dropout_masks(prenet=keep):
                out = model.inference(text.cuda())
        assert model.mel_lengths.cpu().tolist() == ref[4].tolist()
        for a, b in zip(out, (ref[0], ref[1], ref[2], ref[3])):
            assert rel_err(a, b) < TOL, (B, T, impl_name)


def test_full_size_persistent_vs_stepwise_and_oracle_prefix():
    """BASELINE config 2 shape (B=64, T_text=150): the two CUDA implementations agree over 200 steps
    and match the CPU oracle on the first 24 (the oracle costs ~8 ms per step at this size)."""
    B, T, S = 64, 150, 200
    sd = synth_state_dict(1234, gate_bias=-10.0, scale=2.0)
    text = rand_text(B, T, 7)
    keep = keep_mask((S, 2, B, 256), 0.5, 8)
    outs = {}
    for impl, nm in IMPLS:
        model = make_model(sd, S, impl)
        with torch.no_grad(), t2.dropout_masks(prenet=keep):
            outs[nm] = [o.cpu() for o in model.inference(text.cuda())]
        assert model.mel_lengths.cpu().tolist() == [S] * B
    for a, b in zip(outs["persistent"], outs["stepwise"]):
        assert rel_err(a, b) < TOL
    with torch.no_grad():
        memory = O.encoder(sd, sd["embedding.weight"][text].transpose(1, 2))
        ref = O.decoder_inference(sd, memory, keep, 0.5, 24)
    assert rel_err(outs["persistent"][0][:, :, :24], ref[0]) < TOL
    assert rel_err(outs["persistent"][3][:, :24], ref[2]) < TOL
    # size-independent properties: attention rows are probability vectors, alignments non-negative
    al = outs["persistent"][3]
    assert float((al.sum(-1) - 1).abs().max()) < 1e-4 and float(al.min()) >= 0.0


@pytest.mark.parametrize("name", FULL_INFER)
def test_quoted_configs_match_reference_golden_every_step(name):
    """The configurations the benchmark numbers are quoted on, ALL steps, against fixtures produced by the reference's
    own modules (tools/make_golden.py full): B=64 / T_text=150 / 800 steps with the bench weights (BASELINE.json
    configs[1]) and the config-5 per-GPU shape B=32 / T_text=300 / 2000 steps.  1e-3 on mel / mel_postnet / gate /
    alignments, stop decisions (mel_lengths and every live per-step decision) bit-exact; the measured drift of the
    split-fp16 path at the end of the autoregressive run is printed (DESIGN.md section 2)."""
    g = load(name)
    sd, text, keep, S = infer_inputs(g)
    model = make_model(sd, S, _capi.IMPL_PERSISTENT)
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        mel, post, gate, align = model.inference(text.cuda())
    torch.cuda.synchronize()
    assert mel.shape[2] == S
    errs = check_full_inference(g, mel, post, gate[:, :, 0], align, model.mel_lengths, TOL)
    print("quoted config %s: %s (gate pre-activation margin of the fixture %.2e, max |gate| %.3f)" % (
        name, ", ".join("%s %.2e" % kv for kv in errs.items()), float(g["gate_margin"]), float(abs(g["gate"]).max())))


def test_philox_mode_is_deterministic_and_statistically_sane():
    """Production dropout (no injected masks): same seed -> same output on both implementations."""
    sd = synth_state_dict(77, gate_bias=-10.0, scale=2.0)
    text = rand_text(3, 21, 5).cuda()
    res = []
    for impl, nm in IMPLS:
        model = make_model(sd, 10, impl)
        import tacotron2_b200._engine as E
        E._seed_counter[0] = 1000
        torch.manual_seed(5)
        with torch.no_grad():
            res.append(model.inference(text)[0].cpu())
    assert rel_err(res[0], res[1]) < TOL


def test_persistent_decoder_is_bit_reproducible():
    """Two runs with the same inputs and masks give bit-identical mel / gate / alignments at the benchmark shape (the
    attention energies are summed in a fixed order: no shared-memory atomics) -- stop decisions cannot flip run to run."""
    torch.manual_seed(11)
    model = t2.Tacotron2(t2.create_hparams()).cuda().eval()
    model._t2_engine().impl = _capi.IMPL_PERSISTENT
    model.decoder.max_decoder_steps = 20
    model.decoder.gate_threshold = 1.0
    g = torch.Generator().manual_seed(3)
    memory = torch.randn(64, 150, 512, generator=g).cuda()
    keep = keep_mask((20, 2, 64, 256), 0.5, 9)
    outs = []
    for _ in range(3):
        with torch.no_grad(), t2.dropout_masks(prenet=keep):
            outs.append([x.clone() for x in model.decoder.inference(memory)])
    for o in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(outs[0], o))


def test_half_model_inference_like_the_notebook():
    """inference.ipynb:89-90 does model.cuda().eval().half(): tensors crossing the nn.Module boundaries (embedding, encoder
    output, mel) are half like in the reference, the kernels compute in their fp32-grade mode from the half-rounded weights.
    Outputs are half tensors within half-precision distance of the float model holding the same rounded weights."""
    sd = synth_state_dict(9, gate_bias=-10.0, scale=2.0)
    sd_r = {k: (v.half().float() if v.dtype.is_floating_point else v) for k, v in sd.items()}
    text = rand_text(2, 17, 4).cuda()
    keep = keep_mask((8, 2, 2, 256), 0.5, 6)
    outs = []
    for half in (False, True):
        model = make_model(sd_r if not half else sd, 8)
        if half:
            model = model.half()
        with torch.no_grad(), t2.dropout_masks(prenet=keep):
            o = model.inference(text)
        outs.append(o)
        assert all(x.dtype == (torch.float16 if half else torch.float32) for x in o)
    for a, b in zip(outs[0], outs[1]):
        assert a.shape == b.shape and rel_err(b.float(), a) < 2e-2


GEMM_CASES = [
    # ta, tb, M, N, K, lda_pad, ldb_pad, ldc_pad, beta, batch, scaleA, scaleB
    (0, 1, 300, 128, 512, 0, 0, 0, 0.0, 1, 1.0, 1.0),            # x . W^T (processed memory / queries)
    (0, 0, 257, 1536, 81, 0, 0, 0, 0.0, 1, 1e-6, 1.0),           # ld = 81: unaligned rows, K not a multiple of 64
    (1, 0, 80, 1024, 5000, 1, 0, 512, 0.0, 1, 1e-8, 1.0),        # time-batched weight gradient: small tile, split K
    (1, 0, 1, 512, 3000, 80, 0, 0, 0.0, 1, 1e-5, 1.0),           # single output row (the gate layer)
    (0, 0, 1, 4096, 2000, 0, 0, 0, 0.0, 1, 1.0, 1e-7),           # ones . X  (column sums through the GEMM)
    (1, 0, 128, 64, 70000, 0, 0, 0, 1.0, 1, 1e-4, 1.0),          # location filter gradient chunk: huge K, beta = 1
    (0, 0, 150, 512, 37, 0, 0, 0, 1.0, 3, 1.0, 1e-3),            # strided batch (d_memory += aw^T . g_ctx), beta = 1
    (0, 1, 130, 70, 64, 3, 5, 7, 0.5, 1, 1.0, 1.0),              # padded leading dimensions, fractional beta
]


@pytest.mark.parametrize("case", GEMM_CASES)
def test_training_path_tensor_core_gemm_vs_fp64(case):
    """gemm_tc.cu (the wgmma split-fp16 GEMM that replaced every cuBLAS sgemm of the training path) against torch fp64:
    fp32-grade accuracy (error <= 2e-5 of the result's maximum; cuBLAS fp32 lands at ~1e-6) for gradient-like operands
    many orders of magnitude below 1, rows of wildly different magnitude, unaligned / padded leading dimensions."""
    ta, tb, M, N, K, pa, pb, pc, beta, batch, sa, sb = case
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    a_rows, a_cols = (K, M) if ta else (M, K)
    b_rows, b_cols = (N, K) if tb else (K, N)
    lda, ldb, ldc = a_cols + pa, b_cols + pb, N + pc
    A = torch.randn(batch, a_rows, lda, generator=g) * sa
    B = torch.randn(batch, b_rows, ldb, generator=g) * sb
    # rows of op(A) spanning 6 orders of magnitude (per-row operand scales must cope)
    rs = torch.logspace(0, -6, M).view(1, -1, 1) if not ta else torch.logspace(0, -6, M).view(1, 1, -1)
    A[:, :, :a_cols] *= rs
    C0 = torch.randn(batch, M, ldc, generator=g) * (sa * sb)
    Ad, Bd, Cd = A.cuda(), B.cuda(), C0.clone().cuda()
    L = _capi.selftest_lib()
    _capi.check_selftest(L.t2_selftest_gemm_tc(ta, tb, M, N, K, Ad.data_ptr(), lda, Bd.data_ptr(), ldb, Cd.data_ptr(), ldc, beta,
                                               batch, a_rows * lda, b_rows * ldb, M * ldc,
                                               C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    opA = A[:, :, :a_cols].double().transpose(1, 2) if ta else A[:, :, :a_cols].double()
    opB = B[:, :, :b_cols].double().transpose(1, 2) if tb else B[:, :, :b_cols].double()
    ref = opA @ opB + beta * C0[:, :, :N].double()
    got = Cd.cpu()[:, :, :N].double()
    # per output row (rows differ by orders of magnitude): error relative to the row's maximum
    den = ref.abs().amax(dim=2, keepdim=True).clamp_min(1e-300)
    err = float(((got - ref).abs() / den).max())
    assert err < 2e-5, err
    if pc:   # padding columns of C untouched
        assert torch.equal(Cd.cpu()[:, :, N:], C0[:, :, N:])


def test_column_sums_kernel():
    g = torch.Generator().manual_seed(0)
    X = (torch.randn(5000, 90, generator=g) * 1e-4).cuda()
    out = torch.empty(81, device="cuda")
    _capi.check_selftest(_capi.selftest_lib().t2_selftest_colsum(X.data_ptr(), 90, 5000, 81, out.data_ptr(),
                                                                 C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    ref = X[:, :81].double().sum(0)
    assert rel_err(out, ref) < 1e-6


@pytest.mark.parametrize("B,n,cfg", [(2, 6000, (1024, 256, 1024, 80)), (5, 22050 * 3 + 17, (1024, 256, 1024, 80)), (3, 4000, (800, 200, 800, 40))])
def test_mel_spectrogram_vs_oracle(B, n, cfg):
    """TacotronSTFT.mel_spectrogram on the GPU (t2_mel_spectrogram: reflect pad, windowed DFT as a strided-batch tensor-core
    GEMM over overlapping frames, magnitude, mel projection, log) vs oracle/stft_oracle.py, whose STFT half is pinned by the
    reference's own stft.STFT (tests/golden/stft_mag.npz); layers.py:63-80."""
    from oracle import stft_oracle as S
    fl, hop, win, n_mel = cfg
    if (B, n) == (2, 6000):
        y = torch.from_numpy(load("stft_mag")["y"])
    else:
        g = torch.Generator().manual_seed(n)
        t = torch.arange(n) / 22050.0
        y = torch.stack([(0.4 * torch.sin(2 * 3.14159265 * (110.0 * (b + 1)) * t) + 0.1 * torch.randn(n, generator=g)).clamp(-1, 1) for b in range(B)])
    stft = t2.TacotronSTFT(fl, hop, win, n_mel_channels=n_mel).cuda()
    got = stft.mel_spectrogram(y.cuda())
    ref = S.mel_spectrogram(y, fl, hop, win, n_mel_channels=n_mel)
    assert got.shape == ref.shape == (B, n_mel, n // hop + 1)
    assert float((got.cpu() - ref).abs().max()) < 1e-3                      # log-mel, absolute
    assert rel_err(torch.exp(got), torch.exp(ref)) < 1e-4                     # linear mel energies, relative to the maximum
    with pytest.raises(AssertionError):
        stft.mel_spectrogram((y * 3).cuda())                                  # layers.py:74-75 range check


def test_device_collate_matches_host_collate():
    """t2_collate (DeviceTextMelCollate) == the host TextMelCollate -- itself checked against the reference's collate function
    in tests/test_boundary_cpu.py -- on ragged batches (distinct text lengths: ties are ordered by input position on the
    device, by torch.sort on the host)."""
    from tacotron2_b200.data_utils import DeviceTextMelCollate, TextMelCollate
    g = torch.Generator().manual_seed(5)
    for B, nfs in [(1, 1), (7, 1), (64, 2)]:
        tls = torch.randperm(200, generator=g)[:B] + 1
        batch = [(torch.randint(1, 148, (int(tls[i]),), generator=g), torch.randn(80, int(torch.randint(1, 300, (1,), generator=g)), generator=g))
                 for i in range(B)]
        ref = TextMelCollate(nfs)(batch)
        got = DeviceTextMelCollate(nfs)([(t.cuda(), m.cuda()) for t, m in batch])
        torch.cuda.synchronize()
        for a, b in zip(got, ref):
            assert a.dtype == b.dtype and torch.equal(a.cpu(), b)
    # ties: stable by input position
    batch = [(torch.full((5,), i + 1), torch.randn(80, 3 + i, generator=g)) for i in range(4)]
    got = DeviceTextMelCollate(1)([(t.cuda(), m.cuda()) for t, m in batch])
    assert got[0][:, 0].cpu().tolist() == [1, 2, 3, 4] and got[4].cpu().tolist() == [3, 4, 5, 6]
