"""pYIN and per-symbol averaging on the GPU (``tacotron2_b200.pyin`` / ``average_by_durations``; DESIGN section 6.11):

1. every frame's voiced flag and decoded state, f0 bit for bit and voiced_prob to 1e-12 against the numpy fp64 oracle
   ``tests/pyin_oracle.py``, on tones, chirps, vibrato, tones in noise, silence and near-silence at the 1e-6 edges and
   three segments of a real speech clip (``tests/golden/demo.wav``, 4.5 s at 22050 Hz), after checking that the
   oracle's path was not decided by a margin below 1e-9 (the clip as a whole has margins of a few ulps, so segments of
   it without them stand in for it);
2. ragged batches (B = 64 of 1-10 s, B = 130) equal to their rows' B = 1 calls bit for bit, zeros past each row;
3. frame_length 2048, non-default switch_prob / resolution / no_trough_prob, fill_na, fp16 input;
4. average_by_durations against a numpy fp64 statement, on durations_from_alignments output, all-unvoiced spans;
5. a CUDA-graph capture of both calls, and the library's refusals."""
import os

import numpy as np
import pytest
import scipy.io.wavfile
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi, pitch
from tests import pyin_oracle as PO

pytestmark = pytest.mark.gpu

C2, C7 = 65.40639132514966, 2093.004522404789
SR = 22050
HERE = os.path.dirname(os.path.abspath(__file__))


def speech():
    sr, x = scipy.io.wavfile.read(os.path.join(HERE, "golden", "demo.wav"))
    assert sr == SR
    return x.astype(np.float32)


SPEECH_SEGMENTS = ((0, 24000), (36000, 56000), (70000, 92000))   # samples; oracle paths without a near-tie


def tone(f, seconds=0.5, harmonics=1, amp=0.5):
    tt = np.arange(int(SR * seconds)) / SR
    return amp * sum(np.sin(2 * np.pi * f * k * tt) / k for k in range(1, harmonics + 1))


def chirp(f0, f1, seconds):
    tt = np.arange(int(SR * seconds)) / SR
    k = np.log(f1 / f0) / seconds
    return 0.5 * np.sin(2 * np.pi * f0 * (np.exp(k * tt) - 1) / k)


def vibrato(f, seconds=0.6, depth=1.0, rate=5.5):
    tt = np.arange(int(SR * seconds)) / SR
    inst = f * 2 ** (depth / 12 * np.sin(2 * np.pi * rate * tt))
    return 0.4 * np.sin(2 * np.pi * np.cumsum(inst) / SR)


def signals():
    rng = np.random.default_rng(7)
    out = {
        "tone80": tone(80.0, harmonics=3), "tone220": tone(220.0), "tone900": tone(900.0, harmonics=2),
        "chirp": chirp(70.0, 2000.0, 1.0), "vibrato": vibrato(330.0),
        "noisy_tone": tone(150.0, harmonics=4) + 0.15 * rng.standard_normal(int(SR * 0.5)),
        "silence": np.zeros(6000), "near_silence": tone(200.0, 0.3, amp=1e-4),
        "below_edge": tone(200.0, 0.3, amp=3e-5) + 1e-5 * rng.standard_normal(int(SR * 0.3)),
    }
    return {k: v.astype(np.float32) for k, v in out.items()}


def assert_equals_oracle(y, f0, flag, prob, **kw):
    """One clip's GPU outputs against the oracle: the path's margins first, then every frame."""
    of0, oflag, oprob, _, gaps = PO.pyin(y, kw.pop("fmin", C2), kw.pop("fmax", C7), gaps=True, **kw)
    close = (gaps > 0) & (gaps < 1e-9)
    assert not close.any(), "the oracle's path has a near-tie at frames %s" % np.nonzero(close)[0][:8]
    assert f0.shape == of0.shape
    assert np.array_equal(flag, oflag), np.nonzero(flag != oflag)[0][:8]
    assert np.array_equal(f0, of0, equal_nan=True), np.nonzero(~((f0 == of0) | (np.isnan(f0) & np.isnan(of0))))[0][:8]
    assert np.abs(prob - oprob).max() <= 1e-12
    return int(oflag.sum())


def run(ys, lengths=None, **kw):
    out = t2.pyin(ys, kw.pop("fmin", C2), kw.pop("fmax", C7), lengths=lengths, **kw)
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in out]


def test_signals_and_speech_in_one_ragged_call_equal_the_oracle():
    sig = signals()
    for a, b in SPEECH_SEGMENTS:
        sig["speech%d" % a] = speech()[a:b]
    names = list(sig)
    n = max(len(v) for v in sig.values())
    y = torch.zeros(len(names), n)
    for b, k in enumerate(names):
        y[b, :len(sig[k])] = torch.from_numpy(sig[k])
        y[b, len(sig[k]):] = 0.3                           # garbage past each row's end: never read
    lengths = [len(sig[k]) for k in names]
    f0, flag, prob = run(y.cuda(), lengths)
    voiced = {}
    for b, k in enumerate(names):
        F = 1 + lengths[b] // 256
        voiced[k] = assert_equals_oracle(sig[k], f0[b, :F], flag[b, :F], prob[b, :F])
        assert (f0[b, F:] == 0).all() and not flag[b, F:].any() and (prob[b, F:] == 0).all()
    assert voiced["silence"] == 0 and voiced["tone220"] > 0, voiced
    assert min(voiced["speech%d" % a] for a, _ in SPEECH_SEGMENTS) > 30, voiced


def bits(x):
    return x.contiguous().view(torch.int64) if x.dtype == torch.float64 else x


@pytest.mark.parametrize("B,lo,hi", [(64, 1.0, 10.0), (130, 0.05, 1.0)])
def test_ragged_rows_equal_their_own_calls(B, lo, hi):
    g = torch.Generator().manual_seed(B)
    lengths = (torch.rand(B, generator=g) * (hi - lo) * SR + lo * SR).long()
    n = int(lengths.max())
    tt = torch.arange(n) / SR
    f = 80 + torch.rand(B, 1, generator=g) * 600
    y = 0.4 * torch.sin(2 * np.pi * f * tt * (1 + 0.05 * torch.sin(2 * np.pi * 3 * tt))) \
        + 0.05 * torch.randn(B, n, generator=g)
    y[:, ::7] *= (torch.rand(B, 1, generator=g) > 0.3).float()
    y[B // 2:B // 2 + 2] = 0                                  # silent rows
    yc = y.cuda()
    out = t2.pyin(yc, C2, C7, lengths=lengths.cuda())
    F = 1 + n // 256
    assert all(o.shape == (B, F) for o in out)
    for b in range(B):
        L = int(lengths[b])
        one = t2.pyin(yc[b, :L].contiguous(), C2, C7)
        Fb = 1 + L // 256
        for o, r in zip(out, one):
            assert torch.equal(bits(o[b, :Fb]), bits(r)), b
        assert not out[0][b, Fb:].any() and not out[1][b, Fb:].any() and not out[2][b, Fb:].any()


@pytest.mark.parametrize("kw", [
    dict(frame_length=2048),
    dict(switch_prob=0.1, resolution=0.05, no_trough_prob=0.2),
    dict(fill_na=0.0, n_thresholds=37, boltzmann_parameter=1.5, beta_parameters=(1.5, 12)),
    dict(fmin=50.0, fmax=1000.0, fill_na=-1.0, max_transition_rate=20.0),
])
def test_parameters_equal_the_oracle(kw):
    sig = signals()
    names = ["tone220", "chirp", "noisy_tone", "silence"]
    n = max(len(sig[k]) for k in names)
    y = torch.zeros(len(names), n)
    for b, k in enumerate(names):
        y[b, :len(sig[k])] = torch.from_numpy(sig[k])
    lengths = [len(sig[k]) for k in names]
    f0, flag, prob = run(y.cuda(), lengths, **dict(kw))
    hop = kw.get("frame_length", 1024) // 4
    for b, k in enumerate(names):
        F = 1 + lengths[b] // hop
        assert_equals_oracle(sig[k], f0[b, :F], flag[b, :F], prob[b, :F], **dict(kw))


def test_fp16_input_is_read_as_fp32():
    y = torch.from_numpy(signals()["vibrato"]).half()
    got = [o.cpu() for o in t2.pyin(y.cuda(), C2, C7)]
    want = [o.cpu() for o in t2.pyin(y.float().cuda(), C2, C7)]
    assert all(torch.equal(bits(a), bits(b)) for a, b in zip(got, want))
    assert_equals_oracle(y.float().numpy(), *[o.numpy() for o in got])


def test_average_by_durations_equals_the_numpy_statement():
    g = torch.Generator().manual_seed(3)
    B, F, T = 5, 200, 40
    v = torch.rand(B, F, generator=g, dtype=torch.float64) * 300
    v[torch.rand(B, F, generator=g) < 0.3] = 0
    v[torch.rand(B, F, generator=g) < 0.1] = float("nan")
    v[1, :] = float("nan")                                     # all-unvoiced row
    d = torch.randint(0, 9, (B, T), generator=g)
    d[d.sum(1) > F] = 1
    d[2, 3:9] = 0
    got = t2.average_by_durations(v.cuda(), d.cuda()).cpu()
    assert got.dtype == torch.float32 and got.shape == (B, T)
    for b in range(B):
        want = PO.average_pitch(v[b].numpy(), d[b].numpy()).astype(np.float32)
        assert np.array_equal(got[b].numpy(), want), b
    assert (got[1] == 0).all()
    f32 = t2.average_by_durations(v.float().cuda(), d.cuda()).cpu()
    for b in range(B):
        assert np.array_equal(f32[b].numpy(), PO.average_pitch(v[b].float().double().numpy(), d[b].numpy())
                              .astype(np.float32))


def test_pitch_per_symbol_end_to_end_on_durations_from_alignments():
    """mel frames of a clip, MAS durations from an attention map over those frames, pyin, then per-symbol pitch."""
    y = torch.from_numpy(speech())
    F = 1 + len(y) // 256
    mel = t2.TacotronSTFT().cuda().mel_spectrogram(y[None].cuda())
    assert mel.shape[-1] == F
    T_text = 60
    g = torch.Generator().manual_seed(11)
    a = torch.softmax(torch.randn(1, F, T_text, generator=g) * 3, -1).cuda()
    d = t2.durations_from_alignments(a)
    assert int(d.sum()) == F
    f0, flag, _ = t2.pyin(y[None].cuda(), C2, C7)
    got = t2.average_by_durations(f0, d).cpu()
    want = PO.average_pitch(f0[0].cpu().numpy(), d[0].cpu().numpy()).astype(np.float32)
    assert np.array_equal(got[0].numpy(), want)
    spans = np.split(flag[0].cpu().numpy(), np.cumsum(d[0].cpu().numpy())[:-1])
    for j, s in enumerate(spans):
        assert (got[0, j] == 0) == (not s.any()), j              # a span of unvoiced frames gives 0


def test_cuda_graph_capture_of_both_calls():
    sig = signals()
    y = torch.zeros(3, 12000)
    for b, k in enumerate(["tone220", "chirp", "noisy_tone"]):
        y[b, :len(sig[k][:12000])] = torch.from_numpy(sig[k][:12000])
    y = y.cuda()
    lengths = torch.tensor([11025, 12000, 5000], dtype=torch.int32, device="cuda")
    p = pitch.pyin_params(SR, C2, C7)
    t = pitch._device_tables(p, y.device)
    args, out, ws = pitch._pyin_call(y, lengths, p, t, y.device)
    d = torch.full((3, 8), 5, dtype=torch.int64, device="cuda")
    avg = torch.empty(3, 8, dtype=torch.float32, device="cuda")
    L = _capi.lib()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            _capi.call(L.t2_pyin, y.device, args)
            _capi.call(L.t2_average_by_durations, y.device, out[0].data_ptr(), d.data_ptr(), 3, out[0].shape[1], 8,
                       avg.data_ptr())
    graph.replay()
    torch.cuda.synchronize()
    want = t2.pyin(y, C2, C7, lengths=lengths)
    assert all(torch.equal(bits(a), bits(b)) for a, b in zip(out, want))
    assert torch.equal(avg, t2.average_by_durations(want[0], d))
    y[0].mul_(0.5)                                            # a replay reads the buffers anew
    graph.replay()
    want = t2.pyin(y, C2, C7, lengths=lengths)
    torch.cuda.synchronize()
    assert all(torch.equal(bits(a), bits(b)) for a, b in zip(out, want))


def test_library_refuses_invalid_calls():
    y = torch.from_numpy(signals()["tone220"])[None].cuda()
    p = pitch.pyin_params(SR, C2, C7)
    t = pitch._device_tables(p, y.device)
    args, out, ws = pitch._pyin_call(y, None, p, t, y.device)
    L = _capi.lib()
    stream = torch.cuda.current_stream().cuda_stream
    need = args.ws_bytes

    def rc(**kw):
        a = _capi.T2PyinArgs.from_buffer_copy(args)
        for k, v in kw.items():
            setattr(a, k, v)
        return L.t2_pyin(a, stream)
    assert rc() == 0
    for kw in (dict(y=None), dict(f0=None), dict(voiced_flag=None), dict(voiced_prob=None), dict(ws=None),
               dict(log_trans=None), dict(boltzmann=None), dict(B=0), dict(n=0), dict(frame_length=4096),
               dict(win_length=1024), dict(hop_length=0), dict(max_period=10), dict(max_period=600),
               dict(n_bins=1537), dict(n_bins=0), dict(n_thresholds=0), dict(n_thresholds=4097), dict(width=0),
               dict(bins_per_semitone=0), dict(sr=0), dict(fmin=0.0)):
        assert rc(**kw) == -1, kw
        assert L.t2_pyin_workspace_bytes(_capi.T2PyinArgs.from_buffer_copy(args)) == need
    assert rc(ws_bytes=need - 1) == -3
    v = torch.zeros(2, 5, dtype=torch.float64, device="cuda")
    d = torch.ones(2, 3, dtype=torch.int64, device="cuda")
    o = torch.empty(2, 3, dtype=torch.float32, device="cuda")
    assert L.t2_average_by_durations(v.data_ptr(), d.data_ptr(), 2, 5, 3, o.data_ptr(), stream) == 0
    for B, F, T in ((0, 5, 3), (2, 0, 3), (2, 5, 0)):
        assert L.t2_average_by_durations(v.data_ptr(), d.data_ptr(), B, F, T, o.data_ptr(), stream) == -1
    assert L.t2_average_by_durations(None, d.data_ptr(), 2, 5, 3, o.data_ptr(), stream) == -1
    torch.cuda.synchronize()


def test_device_lengths_are_clamped_by_the_library():
    y = torch.from_numpy(signals()["tone220"][:4000])[None].repeat(2, 1).cuda()
    p = pitch.pyin_params(SR, C2, C7)
    t = pitch._device_tables(p, y.device)
    lengths = torch.tensor([0, 99999], dtype=torch.int32, device="cuda")
    args, out, ws = pitch._pyin_call(y, lengths, p, t, y.device)
    _capi.call(_capi.lib().t2_pyin, y.device, args)
    one = t2.pyin(y[:1, :1].contiguous(), C2, C7)
    full = t2.pyin(y[1:].contiguous(), C2, C7)
    torch.cuda.synchronize()
    assert torch.equal(bits(out[0][0, :1]), bits(one[0][0])) and not out[1][0, 1:].any()
    assert all(torch.equal(bits(o[1]), bits(f[0])) for o, f in zip(out, full))
