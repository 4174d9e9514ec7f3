"""Ragged log-mel extraction: ``TacotronSTFT.mel_spectrogram(y, lengths)`` (t2_mel_spectrogram with T2MelSpecArgs.lengths).

Row b of a ragged call must be bit for bit the B = 1 call on ``y[b, :lengths[b]]``, zero past its own frames, whatever
its tail holds and whatever it is batched with; it must match the CPU oracle of that clip alone; bad lengths refuse
before any launch; the call stays inside its exact-size buffers and replays from a CUDA graph; and
``DeviceTextMelCollate(k, stft)`` over audio gives what the collation of per-clip mels gives."""
import ctypes as C
import math

import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tacotron2_b200.data_utils import DeviceTextMelCollate
from tests.common import rel_err

pytestmark = pytest.mark.gpu
SR, HOP = 22050, 256
LENGTHS = [513, 1024, 1025, 256 * 40, SR + 17, 3 * SR, 3 * SR + 1000]     # the minimum ... n_max
N_MAX = max(LENGTHS)


def clips(lengths, n, seed, tail=float("nan")):
    """(B, n) in [-1, 1] up to each row's length: tones plus noise; every row's tail holds `tail` (NaN, or a value
    outside [-1, 1] on odd rows)."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n) / SR
    rows = []
    for b, L in enumerate(lengths):
        x = 0.4 * torch.sin(2 * math.pi * (110.0 * (b + 1)) * t) + 0.1 * torch.randn(n, generator=g)
        x = x.clamp(-1, 1)
        x[L:] = tail if b % 2 == 0 else 7.5
        rows.append(x)
    return torch.stack(rows)


def frames(L):
    return L // HOP + 1


@pytest.fixture(scope="module")
def stft():
    return t2.TacotronSTFT().cuda()


def check_rows(stft, y, lengths, out):
    """out (B, 80, n // 256 + 1): every row == its own B = 1 call on its own samples, zeros after."""
    assert out.shape == (y.shape[0], 80, y.shape[1] // HOP + 1)
    for b, L in enumerate(lengths):
        one = stft.mel_spectrogram(y[b:b + 1, :L])[0]
        F = frames(L)
        assert torch.equal(out[b, :, :F], one), "row %d (length %d) differs from its own B = 1 call" % (b, L)
        assert not bool(out[b, :, F:].any()), "row %d has non-zero frames past its %d" % (b, F)


def test_each_row_is_its_own_b1_call(stft):
    y = clips(LENGTHS, N_MAX, seed=1).cuda()
    L = _capi.lib()
    n0 = L.t2_kernel_launch_count()
    out = stft.mel_spectrogram(y, LENGTHS)
    assert L.t2_kernel_launch_count() - n0 == 9                 # pad, 3 per product, magnitude, log: whatever B
    check_rows(stft, y, LENGTHS, out)
    # the lengths as a host tensor and as a device tensor give the same bits
    for lens in (torch.tensor(LENGTHS), torch.tensor(LENGTHS, dtype=torch.int32).cuda()):
        assert torch.equal(stft.mel_spectrogram(y, lens), out)
    # permuted rows, and the rows split over two calls
    perm = [4, 0, 6, 2, 5, 1, 3]
    outp = stft.mel_spectrogram(y[perm], [LENGTHS[i] for i in perm])
    assert torch.equal(outp, out[perm])
    for part in (slice(0, 3), slice(3, 7)):
        sub = stft.mel_spectrogram(y[part], LENGTHS[part])
        assert torch.equal(sub, out[part])


def test_full_length_rows(stft):
    """Every length equal to n: each row is still its own B = 1 call (the unlengthed batch need not be)."""
    n = SR + 300
    y = clips([n] * 5, n, seed=2).cuda()
    check_rows(stft, y, [n] * 5, stft.mel_spectrogram(y, [n] * 5))


def test_a_long_batch_of_short_and_long_rows(stft):
    """64 rows from 1 to 10 s: K-split regimes of both products from 4 splits (short rows) to none."""
    g = torch.Generator().manual_seed(3)
    lengths = torch.randint(SR, 10 * SR + 1, (64,), generator=g).tolist()
    lengths[:3] = [513, 128 * 11 * HOP - 1, 128 * 12 * HOP]          # 1408 frames: 11 tiles, 2 splits
    n = max(lengths)
    y = clips(lengths, n, seed=4).cuda()
    out = stft.mel_spectrogram(y, lengths)
    check_rows(stft, y, lengths, out)


def test_rows_match_the_oracle(stft):
    from oracle import stft_oracle as S
    y = clips(LENGTHS, N_MAX, seed=5)
    out = stft.mel_spectrogram(y.cuda(), LENGTHS).cpu()
    for b, L in enumerate(LENGTHS):
        ref = S.mel_spectrogram(y[b:b + 1, :L])[0]
        got = out[b, :, :frames(L)]
        assert got.shape == ref.shape
        assert float((got - ref).abs().max()) < 1e-3, b                    # log-mel, absolute
        assert rel_err(torch.exp(got), torch.exp(ref)) < 1e-4, b             # linear mel energies


@pytest.mark.parametrize("lengths,err", [
    ([512, 1000, 1000], ValueError),                 # below filter_length / 2 + 1
    ([1000, 2001, 1000], ValueError),                # past n
    ([1000, 1000], ValueError),                      # wrong count
    (torch.tensor([[1000, 1000, 1000]]), ValueError),  # wrong shape
    (torch.tensor([1000.0, 1000.0, 1000.0]), TypeError),
    ([1000, 1000.0, 1000], TypeError),
])
def test_bad_lengths_refuse_before_any_launch(stft, lengths, err):
    y = clips([2000] * 3, 2000, seed=6).cuda()
    L = _capi.lib()
    torch.cuda.synchronize()
    n0 = L.t2_kernel_launch_count()
    with pytest.raises(err):
        stft.mel_spectrogram(y, lengths)
    assert L.t2_kernel_launch_count() == n0


def test_range_check_covers_each_rows_own_samples(stft):
    y = clips([1500, 2000], 2000, seed=7).cuda()
    stft.mel_spectrogram(y, [1500, 2000])                      # the NaN past row 0's end is not checked
    y[1, 1999] = 1.5
    L = _capi.lib()
    torch.cuda.synchronize()
    n0 = L.t2_kernel_launch_count()
    with pytest.raises(AssertionError):
        stft.mel_spectrogram(y, [1500, 2000])
    assert L.t2_kernel_launch_count() == n0


# ---- the library call: exact-size buffers and graph capture -----------------------------------------------------------
CANARY = 64 * 1024


def pattern(n):
    g = torch.Generator(device="cuda").manual_seed(91)
    return torch.randint(0, 256, (n,), generator=g, dtype=torch.uint8, device="cuda")


def library_call(stft, y, len32, out, ws):
    B, n = y.shape
    a = _capi.T2MelSpecArgs(y.data_ptr(), B, n, stft.filter_length, stft.hop_length, stft.n_mel_channels,
                            stft.forward_basis.data_ptr(), stft.mel_basis.data_ptr(), 1e-5, out.data_ptr(), ws.data_ptr(),
                            ws.numel(), len32.data_ptr())
    _capi.call(_capi.lib().t2_mel_spectrogram, y.device, C.byref(a))
    return out


def test_exact_size_buffers_and_graph_replay(stft):
    lengths = [513, 4000, 9001]
    y = clips(lengths, 9001, seed=8).cuda()
    len32 = torch.tensor(lengths, dtype=torch.int32).cuda()
    B, n = y.shape
    L = _capi.lib()
    ref = stft.mel_spectrogram(y, lengths)
    ws_bytes = L.t2_mel_spectrogram_workspace_bytes_lengths(B, n, 1024, HOP, 80)
    out_bytes = ref.numel() * 4
    raws = []

    def placed(nbytes):                       # 256 bytes past a 512-byte boundary, between canaries
        raw = pattern(2 * CANARY + 256 + nbytes)
        assert raw.data_ptr() % 512 == 0
        raws.append((raw, nbytes))
        return raw[CANARY + 256:CANARY + 256 + nbytes]
    ws = placed(ws_bytes)
    out = placed(out_bytes).view(torch.float32).view(ref.shape)
    library_call(stft, y, len32, out, ws)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    for raw, nbytes in raws:
        exp, lo = pattern(raw.numel()), CANARY + 256
        assert torch.equal(raw[:lo], exp[:lo]) and torch.equal(raw[lo + nbytes:], exp[lo + nbytes:]), nbytes
    # one byte short is refused
    with pytest.raises(_capi.T2Error, match="workspace"):
        library_call(stft, y, len32, out, ws[:-1])
    # capture: the replay writes the eager bits
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        library_call(stft, y, len32, out, ws)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


# ---- collate ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 2])
def test_collate_over_audio_equals_collate_over_per_clip_mels(stft, k):
    g = torch.Generator().manual_seed(9)
    lengths = [SR + 17, 600, 2 * SR, 256 * 30, 513]
    texts = [torch.randint(1, 148, (int(t),), generator=g).cuda() for t in (17, 40, 9, 40, 23)]
    y = clips(lengths, max(lengths), seed=10)
    audio = [y[b, :L].cuda() for b, L in enumerate(lengths)]
    got = DeviceTextMelCollate(k, stft)([(t, a) for t, a in zip(texts, audio)])
    mels = [stft.mel_spectrogram(a[None])[0] for a in audio]
    ref = DeviceTextMelCollate(k)([(t, m) for t, m in zip(texts, mels)])
    assert len(got) == len(ref) == 5
    for a, b in zip(got, ref):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
