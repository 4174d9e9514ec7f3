"""Dynamic time warping, MCD and f0 frame errors on the GPU (``dtw``, ``mel_cepstral_distortion``, ``pitch_errors``;
DESIGN section 6.12):

1. cost and path bit for bit against the numpy fp64 oracle on ragged batches: 1 x 1, 1 x N and N x 1 rows, D = 1, 80
   and 1024, fp32 and fp64, predecessor maps on both sides of the on-chip / workspace boundary, one 8192 x 8192 pair;
2. every row equals its own B = 1 call, with NaN written past each row's lengths (which are never read);
3. MCD: a mel with itself is 0; free-run mels of the default-initialised model against ``mel_spectrogram`` of seeded
   audio equal the oracle bit for bit;
4. ``pitch_errors`` on ``pyin`` outputs of two seeded clips against the oracle;
5. output and workspace buffers of exactly the queried size, between canaries, are never overrun; the C refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tests import dtw_oracle as O
from tests.common import rand_text
from tests.test_gpu_buffer_bounds import Placed

pytestmark = pytest.mark.gpu
NAN = float("nan")


def batch(lx, ly, D, dtype, seed, T_x=None, T_y=None):
    """x (B, D, T_x), y (B, D, T_y) with row b's frames random up to lx[b] / ly[b] and NaN after; y is a noisy,
    time-warped copy of x where the lengths allow, so paths are not trivial."""
    g = torch.Generator().manual_seed(seed)
    B = len(lx)
    T_x, T_y = T_x or max(lx), T_y or max(ly)
    x = torch.full((B, D, T_x), NAN, dtype=torch.float64)
    y = torch.full((B, D, T_y), NAN, dtype=torch.float64)
    for b in range(B):
        xb = torch.randn(D, lx[b], generator=g).cumsum(1) * 0.3
        idx = torch.sort(torch.randint(0, lx[b], (ly[b],), generator=g)).values
        x[b, :, :lx[b]] = xb
        y[b, :, :ly[b]] = xb[:, idx] + 0.2 * torch.randn(D, ly[b], generator=g)
    return x.to(dtype), y.to(dtype)


def run(x, y, xl=None, yl=None):
    cost, path, n = t2.dtw(x.cuda(), y.cuda(), xl, yl)
    torch.cuda.synchronize()
    B, P = x.shape[0], x.shape[2] + y.shape[2] - 1
    assert cost.dtype == torch.float64 and cost.shape == (B,)
    assert path.dtype == torch.int64 and path.shape == (B, P, 2) and n.dtype == torch.int64 and n.shape == (B,)
    return cost.cpu(), path.cpu(), n.cpu()


def assert_matches_oracle(x, y, lx, ly, got):
    cost, path, n = got
    for b in range(x.shape[0]):
        want_cost, want_path = O.dtw(x[b, :, :lx[b]].double().numpy(), y[b, :, :ly[b]].double().numpy())
        N = len(want_path)
        assert float(cost[b]) == want_cost, (b, float(cost[b]), want_cost)
        assert int(n[b]) == N and torch.equal(path[b, :N], torch.from_numpy(want_path)), b
        assert bool((path[b, N:] == -1).all()), b


def plan_on_chip(T_x, T_y):
    """Whether the predecessor map stays in shared memory (dtw.cu's dtw_plan)."""
    words = min((T_x + 31) // 32, (min(T_x, T_y) + 31) // 32 + 1)
    return (T_x + T_y - 1) * words * 8 <= 96 * 1024


# ---- 1. bit for bit against the oracle -------------------------------------------------------------------------------

CASES = {
    "edges_d1": ([1, 1, 40, 17, 40, 3], [1, 40, 1, 17, 40, 39], 1),
    "d80": ([200, 1, 120, 200, 77], [150, 150, 1, 90, 150], 80),
    "d1024": ([60, 1, 33, 60], [50, 50, 1, 17], 1024),
    "k2_long_x": ([900, 1, 900, 250], [1, 300, 300, 120], 16),
    "on_chip_edge": ([430, 200], [430, 430], 8),
    "workspace_edge": ([440, 200], [440, 440], 8),
}


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_cost_and_path_equal_the_oracle_bit_for_bit(case, dtype):
    lx, ly, D = CASES[case]
    x, y = batch(lx, ly, D, dtype, seed=len(case) + D)
    if case == "on_chip_edge":
        assert plan_on_chip(x.shape[2], y.shape[2])
    if case == "workspace_edge":
        assert not plan_on_chip(x.shape[2], y.shape[2])
    assert_matches_oracle(x, y, lx, ly, run(x, y, lx, ly))


def test_one_pair_at_the_frame_limit():
    n = _capi.DTW_MAX_FRAMES
    x, y = batch([n], [n], 2, torch.float32, seed=8192)
    got = run(x, y)
    assert_matches_oracle(x, y, [n], [n], got)
    assert int(got[2][0]) >= n


def test_identical_and_repeated_frames_cost_zero():
    x, _ = batch([300, 5], [300, 5], 80, torch.float32, seed=3)
    x = torch.nan_to_num(x, nan=0.0)
    cost, path, n = run(x, x.clone(), [300, 5], [300, 5])
    assert cost.tolist() == [0.0, 0.0] and n.tolist() == [300, 5]
    assert torch.equal(path[0, :300], torch.arange(300)[:, None].expand(300, 2))
    extra = torch.randint(0, 300, (200,), generator=torch.Generator().manual_seed(1))
    idx = torch.sort(torch.cat([torch.arange(300), extra])).values                    # every frame, some repeated
    cost, path, n = run(x[:1], x[:1, :, idx])
    assert float(cost[0]) == 0.0 and 500 <= int(n[0]) <= 799


# ---- 2. rows against their own B = 1 calls ---------------------------------------------------------------------------

@pytest.mark.parametrize("lengths_as", ["list", "host", "device"])
def test_each_row_equals_its_own_b1_call(lengths_as):
    g = torch.Generator().manual_seed(11)
    B = 24
    lx = torch.randint(1, 700, (B,), generator=g)
    ly = torch.randint(1, 500, (B,), generator=g)
    lx[0], ly[0], lx[1], ly[1] = 1, 1, 699, 499
    x, y = batch(lx.tolist(), ly.tolist(), 80, torch.float32, seed=12, T_x=700, T_y=500)
    xl, yl = {"list": (lx.tolist(), ly.tolist()), "host": (lx, ly), "device": (lx.cuda(), ly.cuda())}[lengths_as]
    cost, path, n = run(x, y, xl, yl)
    for b in range(B):
        c1, p1, n1 = run(x[b:b + 1, :, :lx[b]], y[b:b + 1, :, :ly[b]])
        N = int(n1[0])
        assert int(n[b]) == N and float(cost[b]) == float(c1[0]) and torch.equal(path[b, :N], p1[0, :N]), b
        assert bool((path[b, N:] == -1).all())


# ---- 3. mel-cepstral distortion --------------------------------------------------------------------------------------

def test_mcd_of_a_mel_with_itself_is_exactly_zero():
    mel = torch.log(torch.rand(3, 80, 120, generator=torch.Generator().manual_seed(5)).clamp(min=1e-5)).cuda()
    mcd, path, n = t2.mel_cepstral_distortion(mel, mel, [120, 7, 1], [120, 7, 1])
    assert mcd.tolist() == [0.0, 0.0, 0.0] and n.tolist() == [120, 7, 1]


def test_mcd_of_free_run_mels_against_recorded_mels_equals_the_oracle():
    torch.manual_seed(0)
    model = t2.Tacotron2(t2.create_hparams()).cuda().eval()
    text, tl = rand_text(3, 40, 21), [40, 23, 9]
    with torch.no_grad():
        mel_x = model.inference(text.cuda(), input_lengths=tl, seeds=[1, 2, 3], max_decoder_steps=180)[1].clone()
    lx = model.mel_lengths.clone()
    g = torch.Generator().manual_seed(22)
    ly = [22050, 14000, 3000]
    audio = torch.zeros(3, max(ly))
    for b, L in enumerate(ly):
        t = torch.arange(L) / 22050
        audio[b, :L] = 0.3 * torch.sin(2 * np.pi * (120 + 40 * b) * t) + 0.02 * torch.randn(L, generator=g)
    sample_lengths = torch.tensor(ly)
    mel_y = t2.TacotronSTFT().cuda().mel_spectrogram(audio.cuda(), sample_lengths)
    fy = [L // 256 + 1 for L in ly]
    mel_x[torch.arange(mel_x.shape[2], device="cuda")[None, None, :].expand_as(mel_x) >= lx[:, None, None]] = NAN
    mcd, path, n = t2.mel_cepstral_distortion(mel_x, mel_y, lx, fy)
    torch.cuda.synchronize()
    for b in range(3):
        want, want_path = O.mcd(mel_x[b, :, :lx[b]].cpu().numpy(), mel_y[b, :, :fy[b]].cpu().numpy())
        assert float(mcd[b]) == want, (b, float(mcd[b]), want)
        N = len(want_path)
        assert int(n[b]) == N and torch.equal(path[b, :N].cpu(), torch.from_numpy(want_path))
    assert bool((mcd > 0).all())
    mcd16, _, _ = t2.mel_cepstral_distortion(mel_x, mel_y, lx, fy, n_cep=16)
    for b in range(3):
        assert float(mcd16[b]) == O.mcd(mel_x[b, :, :lx[b]].cpu().numpy(), mel_y[b, :, :fy[b]].cpu().numpy(), 16)[0]


# ---- 4. f0 frame errors ----------------------------------------------------------------------------------------------

def test_pitch_errors_on_pyin_outputs_equal_the_oracle():
    g = torch.Generator().manual_seed(31)
    sr, L = 22050, [33075, 30000]
    audio = torch.zeros(2, max(L))
    for b, n in enumerate(L):
        t = torch.arange(n) / sr
        f = (140 + 30 * b) * (1 + 0.1 * torch.sin(2 * np.pi * (1.5 + b) * t))
        ph = 2 * np.pi * torch.cumsum(f, 0) / sr
        gate = (torch.sin(2 * np.pi * (2 + b) * t) > -0.3).float()            # voiced stretches and pauses
        audio[b, :n] = gate * sum(0.3 / k * torch.sin(k * ph) for k in range(1, 4)) + 0.005 * torch.randn(n, generator=g)
    audio = audio.cuda()
    ln = torch.tensor(L)
    f0, voiced, _ = t2.pyin(audio, 65.41, 2093.0, lengths=ln)
    mel = t2.TacotronSTFT().cuda().mel_spectrogram(audio, ln)
    F = [n // 256 + 1 for n in L]
    _, path, n = t2.mel_cepstral_distortion(mel[:1], mel[1:], F[:1], F[1:])
    got = t2.pitch_errors(f0[:1], voiced[:1], f0[1:], voiced[1:], path, n)
    N = int(n[0])
    want = O.pitch_errors(f0[0].cpu().numpy(), voiced[0].cpu().numpy(), f0[1].cpu().numpy(), voiced[1].cpu().numpy(),
                          path[0, :N].cpu().numpy())
    for k in ("gpe", "vde", "ffe"):
        assert float(got[k][0]) == want[k], k
    assert float(got["f0_rmse_cents"][0]) == pytest.approx(want["f0_rmse_cents"], rel=1e-12)
    assert 0 < want["vde"] < 1 and want["gpe"] == want["gpe"]           # some voicing differs, some frames both voiced
    # a track against itself along its own diagonal: no errors
    same = t2.pitch_errors(f0, voiced, f0, voiced, torch.arange(F[0], device="cuda")[None, :, None].expand(2, F[0], 2),
                           torch.tensor(F))
    assert [float(same[k][b]) for k in ("gpe", "vde", "ffe", "f0_rmse_cents") for b in range(2)] == [0.0] * 8


# ---- 5. exact-size buffers and the C refusals ------------------------------------------------------------------------

def c_call(x, y, xl, yl, bufs, ws_bytes=None):
    B, D, T_x = x.shape
    T_y = y.shape[2]
    code = _capi.DTW_F32 if x.dtype == torch.float32 else _capi.DTW_F64
    L = _capi.lib()
    need = L.t2_dtw_workspace_bytes(B, D, T_x, T_y, code)
    cost, path, n, ws = (bufs(k) for k in (B * 8, B * (T_x + T_y - 1) * 16, B * 8, need if ws_bytes is None else ws_bytes))
    args = _capi.T2DtwArgs(x.data_ptr(), y.data_ptr(), None if xl is None else xl.data_ptr(),
                           None if yl is None else yl.data_ptr(), B, D, T_x, T_y, code, cost.data_ptr(),
                           path.data_ptr(), n.data_ptr(), ws.data_ptr(), ws.numel())
    rc = L.t2_dtw(C.byref(args), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    return rc, cost.view(torch.float64), path.view(torch.int64).view(B, -1, 2), n.view(torch.int64)


@pytest.mark.parametrize("lx,ly,D", [([1], [1], 1), ([430, 3], [430, 430], 8), ([440, 1], [440, 17], 8),
                                     ([600, 599], [33, 64], 80), ([3000, 2], [1, 2500], 4)])
def test_exact_size_buffers_are_not_overrun(lx, ly, D):
    x, y = batch(lx, ly, D, torch.float32, seed=sum(lx))
    x, y = x.cuda(), y.cuda()
    xl, yl = torch.tensor(lx, dtype=torch.int32).cuda(), torch.tensor(ly, dtype=torch.int32).cuda()
    ref = t2.dtw(x, y, xl, yl)
    placed = Placed()
    rc, *got = c_call(x, y, xl, yl, placed.empty)
    assert rc == 0
    placed.check()
    for a, b in zip(got, ref):
        assert torch.equal(a, b)
    # the cepstra: an exact-size output, and frames past the lengths written as 0
    mel = torch.log(torch.rand(2, 80, 50, device="cuda").clamp(min=1e-5))
    mel[1, :, 20:] = NAN
    table = torch.from_numpy(O.dct_table(80, 24)).cuda()
    out = placed.empty(2 * 24 * 50 * 8)
    rc = _capi.lib().t2_mel_cepstra(mel.data_ptr(), _capi.DTW_F32, torch.tensor([50, 20], dtype=torch.int32).cuda()
                                    .data_ptr(), 2, 80, 50, table.data_ptr(), 24, out.data_ptr(),
                                    C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    placed.check()
    cep = out.view(torch.float64).view(2, 24, 50).cpu()
    assert torch.equal(cep[0], torch.from_numpy(O.cepstra(mel[0].cpu().numpy(), 24)))
    assert torch.equal(cep[1, :, :20], torch.from_numpy(O.cepstra(mel[1, :, :20].cpu().numpy(), 24)))
    assert not bool(cep[1, :, 20:].any())


def test_device_lengths_are_clamped_into_range():
    x, y = batch([50, 50], [40, 40], 3, torch.float64, seed=4)
    x, y = x.cuda(), y.cuda()
    rc, cost, path, n = c_call(x, y, torch.tensor([0, 10 ** 6], dtype=torch.int32).cuda(),
                               torch.tensor([-5, 40], dtype=torch.int32).cuda(),
                               lambda k: torch.empty(k, dtype=torch.uint8, device="cuda"))
    assert rc == 0
    one = t2.dtw(x[:1, :, :1], y[:1, :, :1])
    full = t2.dtw(x[1:], y[1:])
    assert float(cost[0]) == float(one[0][0]) and int(n[0]) == 1
    assert float(cost[1]) == float(full[0][0]) and torch.equal(path[1], full[1][0])


def test_the_library_refuses_bad_sizes_before_any_launch():
    L = _capi.lib()
    x = torch.zeros(2, 4, 16, device="cuda")

    def rc(**kw):
        a = dict(x=x, y=x, xl=None, yl=None)
        a.update(kw)
        return c_call(a["x"], a["y"], a["xl"], a["yl"], lambda k: torch.empty(max(k, 1), dtype=torch.uint8, device="cuda"),
                      kw.get("ws_bytes"))[0]
    assert L.t2_dtw_workspace_bytes(1, 1025, 4, 4, 0) == 0 and L.t2_dtw_workspace_bytes(1, 4, 8193, 4, 0) == 0
    assert L.t2_dtw_workspace_bytes(0, 4, 4, 4, 0) == 0 and L.t2_dtw_workspace_bytes(1, 4, 4, 4, 2) == 0
    assert L.t2_dtw_workspace_bytes(1, 1024, 8192, 8192, 1) > 0
    assert rc(x=torch.zeros(1, 1025, 2, device="cuda"), y=torch.zeros(1, 1025, 2, device="cuda")) == -4
    assert rc(x=torch.zeros(1, 1, 8193, device="cuda"), y=torch.zeros(1, 1, 3, device="cuda")) == -4
    assert rc(ws_bytes=1) == -3
    args = _capi.T2DtwArgs(x.data_ptr(), None, None, None, 2, 4, 16, 16, 0, x.data_ptr(), x.data_ptr(), x.data_ptr(),
                           x.data_ptr(), 1 << 20)
    assert L.t2_dtw(C.byref(args), None) == -1
    args.y, args.dtype = x.data_ptr(), 7
    assert L.t2_dtw(C.byref(args), None) == -1
    assert L.t2_mel_cepstra(x.data_ptr(), 0, None, 2, 4, 16, x.data_ptr(), 4, x.data_ptr(), None) == -1
    assert L.t2_mel_cepstra(x.data_ptr(), 0, None, 2, 1025, 16, x.data_ptr(), 4, x.data_ptr(), None) == -4
