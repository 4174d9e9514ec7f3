"""The public STFT and Griffin-Lim on the GPU (denoiser.cu) against the reference's fixture and the fp64 oracle, and
against their own runs bit for bit where rows and scales must reproduce them.

Both transforms are the denoiser's split-fp16 GEMMs, so each is held to the denoiser's 5e-5 of max |expected| against
fp64.  Griffin-Lim after 30 iterations is held to 1e-3 against the fp64 oracle started from the same angles; the
measured errors are printed and recorded in DESIGN.md 6.8."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import tacotron2_b200 as t2
from oracle import denoiser_oracle as D
from tests import griffin_lim_oracle as G
from tacotron2_b200 import _capi
from tacotron2_b200.audio_processing import _griffin_lim
from tests.common import GOLDEN_DIR, rel_err, stft_inputs

pytestmark = pytest.mark.gpu
HOP = 256
BAR = 5e-5


def fixture():
    return np.load(os.path.join(GOLDEN_DIR, "griffin_lim_b2.npz"))


def ref_angles(shape, seed):
    np.random.seed(seed)
    return torch.from_numpy(np.angle(np.exp(2j * np.pi * np.random.rand(*shape))).astype(np.float32))


_ST = {}


def stft():
    if "st" not in _ST:
        _ST["st"] = t2.TacotronSTFT().cuda().stft_fn
    return _ST["st"]


def unit_case(B=2, n=256 * 40, seed=30):
    """A target magnitude of a real signal (B, 513, n / 256 + 1) and random angles of its shape, on the CPU."""
    y = stft_inputs(seed, n)[:B] if B <= 2 else (torch.randn(B, n, generator=torch.Generator().manual_seed(seed)) * 0.3)
    mag, _ = D.transform(y, torch.float32)
    ang = (torch.rand(mag.shape, generator=torch.Generator().manual_seed(seed + 1)) * 2 - 1) * np.pi
    return y, mag.float(), ang.float()


def phase_err(got_phase, ref_phase, ref_mag):
    """max |wrapped phase difference| over the bins whose magnitude exceeds 1e-3 of their row's max."""
    d = torch.remainder(got_phase.double().cpu() - ref_phase.double().cpu() + np.pi, 2 * np.pi) - np.pi
    keep = ref_mag.cpu() > 1e-3 * ref_mag.cpu().flatten(1).max(dim=1).values[:, None, None]
    return float(d.abs()[keep].max())


# ---------------------------------------------------------------------------------------------------------------------
# transform / inverse / forward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("amp", [1.0, 1e-3, 3e4], ids=["unit", "quiet", "loud"])
def test_transform_against_fp64(amp):
    y = stft_inputs(31, 256 * 40 + 77) * amp
    mag, phase = stft().transform(y.cuda())
    m64, p64 = D.transform(y, torch.float64)
    e_mag, e_ph = rel_err(mag, m64), phase_err(phase, p64, m64)
    print("amplitude %g: magnitude rel err %.2e, phase max |err| %.2e rad" % (amp, e_mag, e_ph))
    assert mag.shape == phase.shape == (2, 513, 41) and mag.dtype == phase.dtype == torch.float32
    assert stft().num_samples == y.shape[1]
    assert e_mag <= BAR and e_ph <= 1e-2


def test_inverse_and_forward_against_fp64():
    y, mag, ang = unit_case()
    out = stft().inverse(mag.cuda(), ang.cuda())
    ref = D.inverse(mag.double(), ang.double())
    e_inv = rel_err(out, ref)
    rec = stft()(y.cuda())
    e_rt = rel_err(rec[:, 0], y[:, :rec.shape[-1]])
    print("inverse rel err %.2e; forward round trip rel err %.2e" % (e_inv, e_rt))
    assert out.shape == (2, 1, 256 * 40) and e_inv <= BAR
    assert rec.shape == (2, 1, 256 * 40) and e_rt <= BAR
    assert torch.equal(stft().magnitude, stft().transform(y.cuda())[0])


# ---------------------------------------------------------------------------------------------------------------------
# Griffin-Lim
# ---------------------------------------------------------------------------------------------------------------------
def test_one_iteration_against_the_fp64_projection():
    """GL(1) against one fp64 step (transform, keep the phase, inverse with the target) from the engine's own GL(0)."""
    _, mag, ang = unit_case()
    x0 = _griffin_lim(mag.cuda(), ang.cuda(), stft(), 0)
    x1 = _griffin_lim(mag.cuda(), ang.cuda(), stft(), 1)
    _, ph = D.transform(x0.double().cpu(), torch.float64)
    ref = D.inverse(mag.double(), ph)[:, 0]
    err = rel_err(x1, ref)
    print("one iteration from the engine's own signal: rel err vs the fp64 step %.2e" % err)
    assert err <= BAR


def test_end_to_end_against_the_reference_and_fp64():
    g = fixture()
    mag, seed = torch.from_numpy(g["mag"]), int(g["np_seed"])
    ang = ref_angles(mag.shape, seed)
    st = stft()
    for n_iters in (0, 1, 30):
        np.random.seed(seed)
        got = t2.griffin_lim(mag.cuda(), st, n_iters=n_iters)
        ref = torch.from_numpy(g["out_%d" % n_iters])
        o64 = G.griffin_lim(mag.double(), ang.double(), n_iters)
        e_ref, e64 = rel_err(got, ref), rel_err(got, o64)
        sc, sc64 = G.spectral_convergence(mag, got.cpu()), G.spectral_convergence(mag, o64)
        print("n_iters %d: rel err vs reference %.2e, vs fp64 oracle %.2e; spectral convergence %s (fp64 %s)"
              % (n_iters, e_ref, e64, ["%.6f" % v for v in sc.tolist()], ["%.6f" % v for v in sc64.tolist()]))
        assert got.shape == ref.shape and got.dtype == torch.float32
        assert e64 <= (BAR if n_iters <= 1 else 1e-3) and e_ref <= (BAR if n_iters <= 1 else 1e-3)
        if n_iters == 30:
            assert bool(((sc - sc64).abs() <= 0.01 * sc64).all())


def test_spectral_convergence_does_not_increase():
    """Griffin-Lim never moves away from the target: ||S - |STFT(x_k)||| / ||S|| is non-increasing in k (up to the
    transforms' own error)."""
    _, mag, ang = unit_case()
    errs = [G.spectral_convergence(mag, _griffin_lim(mag.cuda(), ang.cuda(), stft(), k).cpu()) for k in range(0, 13)]
    print("spectral convergence:", ["%.5f" % float(e.max()) for e in errs])
    for k, (e0, e1) in enumerate(zip(errs, errs[1:])):
        assert bool((e1 <= e0 + 1e-5).all()), (k, e0, e1)


def test_launches_and_rejections():
    """3 n_iters + 2 launches; a refused call launches nothing."""
    _, mag, ang = unit_case()
    st = stft()
    L = _capi.lib()
    for n_iters in (0, 1, 4):
        _griffin_lim(mag.cuda(), ang.cuda(), st, n_iters)
        n0 = L.t2_kernel_launch_count()
        _griffin_lim(mag.cuda(), ang.cuda(), st, n_iters)
        assert L.t2_kernel_launch_count() - n0 == 3 * n_iters + 2
    a, out, eng, held = st._spectrum_args("test", mag.cuda(), ang.cuda(), None, 2)
    n0 = L.t2_kernel_launch_count()
    for field, value, msg in (("F", 3, "at least 4 frames"), ("B", 0, "empty batch"), ("ws_bytes", 100, "too small")):
        bad = _capi.T2GriffinLimArgs.from_buffer_copy(a)
        setattr(bad.inv, field, value)
        with pytest.raises(_capi.T2Error, match=msg):
            _capi.check(L.t2_griffin_lim(eng.handle, C.byref(bad), eng.stream()))
    bad = _capi.T2GriffinLimArgs.from_buffer_copy(a)
    bad.inv.out = out.data_ptr() + 4
    with pytest.raises(_capi.T2Error, match="16-byte aligned"):
        _capi.check(L.t2_griffin_lim(eng.handle, C.byref(bad), eng.stream()))
    bad = _capi.T2GriffinLimArgs.from_buffer_copy(a)
    bad.n_iters = -1
    with pytest.raises(_capi.T2Error, match="negative"):
        _capi.check(L.t2_griffin_lim(eng.handle, C.byref(bad), eng.stream()))
    assert L.t2_kernel_launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------------
# ragged rows and scales: bit for bit
# ---------------------------------------------------------------------------------------------------------------------
def test_ragged_griffin_lim_rows_equal_their_own_calls():
    _, mag, ang = unit_case(B=4, n=256 * 30)
    F = mag.shape[-1]
    lengths = torch.tensor([F, 17, 4, 3])
    out = _griffin_lim(mag.cuda(), ang.cuda(), stft(), 5, lengths=lengths)
    assert out.shape == (4, 256 * (F - 1))
    for b, L in enumerate(lengths.tolist()):
        k = 256 * (L - 1) if L >= 4 else 0
        if L >= 4:
            own = _griffin_lim(mag[b:b + 1, :, :L].contiguous().cuda(), ang[b:b + 1, :, :L].contiguous().cuda(), stft(), 5)
            assert torch.equal(out[b, :k], own[0]), b
        assert not bool(out[b, k:].any()), b
    inv = stft().inverse(mag.cuda(), ang.cuda(), lengths=lengths)
    assert torch.equal(inv[1, 0, :256 * 16], stft().inverse(mag[1:2, :, :17].cuda(), ang[1:2, :, :17].cuda())[0, 0])
    assert not bool(inv[1, 0, 256 * 16:].any()) and not bool(inv[3].any())
    ref = G.griffin_lim(mag.double(), ang.double(), 5, lengths=lengths)
    assert rel_err(out, ref) <= 1e-3


def test_ragged_transform_rows_equal_their_own_calls():
    n = 256 * 30 + 40
    y = torch.randn(4, n, generator=torch.Generator().manual_seed(33)) * 0.3
    y[2] *= 1e-3
    lengths = torch.tensor([n, 256 * 17 + 5, 2000, 400])
    mag, phase = stft().transform(y.cuda(), lengths=lengths)
    for b, L in enumerate(lengths.tolist()):
        f = L // 256 + 1 if L > 512 else 0
        if f:
            m1, p1 = stft().transform(y[b:b + 1, :L].cuda())
            assert torch.equal(mag[b, :, :f], m1[0]) and torch.equal(phase[b, :, :f], p1[0]), b
        assert not bool(mag[b, :, f:].any()) and not bool(phase[b, :, f:].any()), b


@pytest.mark.parametrize("scale", [2.0 ** -20, 2.0 ** 10, 1e-4, 1e4], ids=["2^-20", "2^10", "1e-4", "1e4"])
def test_target_scale(scale):
    """Every scale meets the unit case's bars; a power-of-two scale scales the output bit for bit."""
    _, mag, ang = unit_case()
    st = stft()
    unit = _griffin_lim(mag.cuda(), ang.cuda(), st, 3)
    got = _griffin_lim((mag * scale).cuda(), ang.cuda(), st, 3)
    err = rel_err(got, G.griffin_lim(mag.double() * scale, ang.double(), 3))
    inv = st.inverse((mag * scale).cuda(), ang.cuda())
    e_inv = rel_err(inv, D.inverse(mag.double() * scale, ang.double()))
    print("target x %g: 3 iterations rel err vs fp64 %.2e, inverse %.2e" % (scale, err, e_inv))
    assert bool(torch.isfinite(got).all()) and err <= 1e-3 and e_inv <= BAR
    if float(np.log2(scale)).is_integer():
        assert torch.equal(got, unit * scale)
        assert torch.equal(inv, st.inverse(mag.cuda(), ang.cuda()) * scale)


def test_transform_power_of_two_scale_is_exact():
    y = stft_inputs(34, 256 * 20 + 9).cuda()
    m1, p1 = stft().transform(y)
    for k in (-30, -7, 12):
        mk, pk = stft().transform(y * 2.0 ** k)
        assert torch.equal(mk, m1 * 2.0 ** k) and torch.equal(pk, p1), k


# ---------------------------------------------------------------------------------------------------------------------
# workspace and output bounds
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("entry", ["griffin_lim", "inverse", "transform"])
def test_stays_inside_exact_size_buffers(entry):
    """Workspace and outputs of exactly the reported size, 256 bytes past a 512-byte boundary, between 64 KiB
    canaries."""
    canary = 64 * 1024
    y, mag, ang = unit_case(B=2, n=256 * 21)
    B, F = mag.shape[0], mag.shape[-1]
    lengths = torch.tensor([F, 9], dtype=torch.int32).cuda()
    st = stft()
    eng = st._engine()
    eng.ensure(st)
    L = _capi.lib()
    gen = torch.Generator(device="cuda")

    def placed(nbytes):
        raw = torch.randint(0, 256, (2 * canary + 256 + nbytes,), generator=gen.manual_seed(nbytes), dtype=torch.uint8,
                            device="cuda")
        assert raw.data_ptr() % 512 == 0
        return raw, raw.clone(), raw[canary + 256:canary + 256 + nbytes]

    m, a_ = mag.cuda(), ang.cuda()
    if entry == "transform":
        x = y.cuda()
        n = x.shape[1]
        sample_len = torch.tensor([n, 256 * 9 + 7], dtype=torch.int32).cuda()
        n_ws = int(L.t2_stft_transform_workspace_bytes(eng.handle, B, n))
        n_out = [B * 513 * (n // HOP + 1) * 4] * 2
        ref = st.transform(x, lengths=sample_len)
    else:
        nbytes = L.t2_griffin_lim_workspace_bytes if entry == "griffin_lim" else L.t2_stft_inverse_workspace_bytes
        n_ws = int(nbytes(eng.handle, B, F))
        n_out = [B * HOP * (F - 1) * 4]
        ref = (_griffin_lim(m, a_, st, 3, lengths=lengths),) if entry == "griffin_lim" else \
            (st.inverse(m, a_, lengths=lengths)[:, 0],)
    bufs = [placed(n_ws)] + [placed(nb) for nb in n_out]
    ws, outs = bufs[0][2], [b[2] for b in bufs[1:]]
    if entry == "transform":
        a = _capi.T2StftTransformArgs(x.data_ptr(), B, n, sample_len.data_ptr(), outs[0].data_ptr(), outs[1].data_ptr(),
                                      ws.data_ptr(), n_ws)
        _capi.check(L.t2_stft_transform(eng.handle, C.byref(a), eng.stream()))
    else:
        a = _capi.T2StftInverseArgs(m.data_ptr(), a_.data_ptr(), B, F, lengths.data_ptr(), outs[0].data_ptr(),
                                    ws.data_ptr(), n_ws)
        if entry == "griffin_lim":
            _capi.check(L.t2_griffin_lim(eng.handle, C.byref(_capi.T2GriffinLimArgs(a, 3)), eng.stream()))
        else:
            _capi.check(L.t2_stft_inverse(eng.handle, C.byref(a), eng.stream()))
    torch.cuda.synchronize()
    for (raw, copy, _), nb in zip(bufs, [n_ws] + n_out):
        lo = canary + 256
        assert torch.equal(raw[:lo], copy[:lo]) and torch.equal(raw[lo + nb:], copy[lo + nb:]), nb
    for o, r in zip(outs, ref):
        assert torch.equal(o.view(torch.float32).view(r.shape), r)
