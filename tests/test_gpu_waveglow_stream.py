"""Windowed WaveGlow inference (t2_waveglow_infer_window) and WaveGlow.infer_stream against WaveGlow.infer, bit for bit.

A window holds frames [frame0, frame0 + T) of a sequence.  Its noise is keyed by absolute columns, every flow computes
only the columns later flows still need, and every GEMM row computes the same bits wherever it sits in a tile, so the
audio of its output frames equals the same samples of infer over the whole sequence exactly (the halos are pinned on
the CPU in test_waveglow_window_cpu.py).  The stream runs one window per mel item and must hand out every sample once,
in order, as soon as it is final."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tacotron2_b200.glow import HOP
from tests.common import GOLDEN_DIR, keep_mask, rand_text, sample_index, tensor_digest
from tests.test_gpu_streaming import make_model, set_decoder, stop_threshold, weights
from tests.waveglow_common import CONFIG, mel_input, noise, synth_state_dict

pytestmark = pytest.mark.gpu
LEFT, RIGHT = 99, 96
_SD = {}


def sd7():
    if "sd" not in _SD:
        _SD["sd"] = synth_state_dict(7)
    return _SD["sd"]


def vocoder(half=False):
    m = t2.WaveGlow(**CONFIG)
    m.load_state_dict(sd7())
    m = m.cuda()
    if half:                                   # the notebook's form: .half(), then convinv back to fp32
        m = m.half()
        for k in m.convinv:
            k.float()
    return m


def test_library_reports_the_halo():
    assert t2.window_halo() == (LEFT, RIGHT)


# ---------------------------------------------------------------------------------------------------------------------
# windows against infer
# ---------------------------------------------------------------------------------------------------------------------
def window(m, mel, lengths, z, sigma, seed, frame0, T, out0, out1, at_end):
    eng = m._engine()
    eng.ensure(m)
    spect = mel[:, :, frame0:frame0 + T].contiguous()
    win_len = (lengths - frame0).clamp(min=0, max=T).to(torch.int32).cuda()
    zt = z_frames = None
    if z is not None:
        zt, z_frames = z.cuda().contiguous(), z.shape[2] // 32
    out = eng.infer_window(spect, win_len, zt, z_frames, sigma, seed, frame0, out0, out1, at_end)
    torch.cuda.synchronize()
    return out


WINDOWS = [                      # (frame0, T, out0, out1, at_end) over a 400-frame sequence
    (0, 200, 0, 104, False),     # start: no left halo needed
    (0, 200, 17, 31, False),
    (100, 260, 99, 164, False),  # interior, exactly the halos
    (37, 330, 120, 200, False),
    (250, 150, 99, 150, True),   # end
    (300, 100, 99, 100, True),
    (0, 400, 0, 400, True),      # the whole sequence
    (0, 400, 150, 151, True),
]


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "fp16"])
@pytest.mark.parametrize("philox", [False, True], ids=["z", "philox"])
def test_windows_equal_infer(half, philox):
    B, T, sigma = 3, 400, 0.666
    lengths = torch.tensor([400, 351, 123])
    m = vocoder(half)
    mel = mel_input(B, T, 21).cuda()
    mel = mel.half() if half else mel
    z = None if philox else noise(B, T, 22)
    torch.manual_seed(5)
    with t2.waveglow_noise(z):
        full = m.infer(mel, sigma=sigma, lengths=lengths)
    seed = m._t2.last_seed
    for frame0, Tw, out0, out1, at_end in WINDOWS:
        got = window(m, mel, lengths, z, sigma, seed, frame0, Tw, out0, out1, at_end)
        ref = full[:, HOP * (frame0 + out0):HOP * (frame0 + out1)]
        assert got.dtype == ref.dtype and got.shape == ref.shape
        assert torch.equal(got, ref), ((frame0, Tw, out0, out1), float((got.double() - ref.double()).abs().max()))


def test_too_narrow_windows_are_refused_before_any_launch():
    B, T = 1, 300
    m = vocoder()
    mel, lengths = mel_input(B, T, 31).cuda(), torch.tensor([T])
    window(m, mel, lengths, None, 1.0, 1, 10, 250, 99, 154, False)        # exactly the halos: accepted
    L = _capi.lib()
    n0 = L.t2_kernel_launch_count()
    with pytest.raises(_capi.T2Error, match="left halo is 99 frames"):
        window(m, mel, lengths, None, 1.0, 1, 10, 250, 98, 154, False)
    with pytest.raises(_capi.T2Error, match="right halo is 96 frames"):
        window(m, mel, lengths, None, 1.0, 1, 10, 250, 99, 155, False)
    with pytest.raises(_capi.T2Error, match="right halo is 96 frames"):
        window(m, mel, lengths, None, 1.0, 1, 0, 250, 0, 250, False)
    with pytest.raises(_capi.T2Error, match="z holds"):
        window(m, mel, lengths, noise(B, 200, 1), 1.0, 1, 10, 250, 99, 154, False)
    assert L.t2_kernel_launch_count() == n0


def test_window_stays_inside_exact_size_buffers():
    """Workspace and audio of exactly the reported size, 256 bytes past a 512-byte boundary, between 64 KiB canaries."""
    canary = 64 * 1024
    B, T, frame0, Tw, out0, out1 = 2, 300, 20, 230, 99, 134
    m = vocoder()
    mel, lengths = mel_input(B, T, 41).cuda(), torch.tensor([300, 150])
    ref = window(m, mel, lengths, None, 0.7, 99, frame0, Tw, out0, out1, False)
    gen = torch.Generator(device="cuda")

    def placed(n):
        raw = torch.randint(0, 256, (2 * canary + 256 + n,), generator=gen.manual_seed(n), dtype=torch.uint8, device="cuda")
        assert raw.data_ptr() % 512 == 0
        return raw, raw.clone(), raw[canary + 256:canary + 256 + n]

    L = _capi.lib()
    n_ws = int(L.t2_waveglow_workspace_bytes(m._t2.handle, B, Tw))
    n_audio = B * HOP * (out1 - out0) * 4
    ws_raw, ws_copy, ws = placed(n_ws)
    au_raw, au_copy, au = placed(n_audio)
    spect = mel[:, :, frame0:frame0 + Tw].contiguous()
    win_len = (lengths - frame0).clamp(min=0, max=Tw).to(torch.int32).cuda()
    w = _capi.T2WaveGlowWindowArgs()
    w.wg.mel, w.wg.B, w.wg.T_mel, w.wg.lengths, w.wg.io_half = spect.data_ptr(), B, Tw, win_len.data_ptr(), 0
    w.wg.sigma, w.wg.seed, w.wg.audio, w.wg.ws, w.wg.ws_bytes = 0.7, 99, au.data_ptr(), ws.data_ptr(), n_ws
    w.frame0, w.out0, w.out1, w.at_end = frame0, out0, out1, 0
    _capi.check(L.t2_waveglow_infer_window(m._t2.handle, C.byref(w), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    for raw, copy, n in ((ws_raw, ws_copy, n_ws), (au_raw, au_copy, n_audio)):
        lo = canary + 256
        assert torch.equal(raw[:lo], copy[:lo]) and torch.equal(raw[lo + n:], copy[lo + n:]), n
    assert torch.equal(au.view(torch.float32).view(B, -1), ref)


# ---------------------------------------------------------------------------------------------------------------------
# infer_stream(inference_stream(...)) against infer(inference(...))
# ---------------------------------------------------------------------------------------------------------------------
def mel_items(model, text, keep, chunk):
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        items = list(model.inference_stream(text.cuda(), chunk_steps=chunk))
    return items


def reference(model, glow, text, keep, z, sigma, seed):
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        post = model.inference(text.cuda())[1].clone()
    lengths = model.mel_lengths.clone()
    zz = None if z is None else z[:, :, :32 * post.shape[2]]
    torch.manual_seed(seed)
    with t2.waveglow_noise(zz):
        audio = glow.infer(post, sigma=0.666 if sigma is None else sigma, lengths=lengths)
    return audio, lengths


def expected_ranges(frames):
    """Audio frame ranges the finality rule gives for mel items [(t0, t1, finished)]."""
    out, a0 = [], 0
    for _, t1, fin in frames:
        a1 = t1 if fin else max(a0, t1 - RIGHT)
        if a1 > a0 or fin:
            out.append((a0, a1))
        a0 = a1
    return out


def check_audio_stream(items, mels, ref, ref_lengths):
    frames = [(it["frames"][0], it["frames"][1], it["finished"]) for it in mels]
    assert [tuple(s // HOP for s in it["samples"]) for it in items] == expected_ranges(frames)
    assert [it["finished"] for it in items] == [False] * (len(items) - 1) + [True]
    got = torch.cat([it["audio"] for it in items], dim=1)
    assert got.dtype == ref.dtype and got.shape == ref.shape, (got.shape, ref.shape)
    assert torch.equal(got, ref), float((got.double() - ref.double()).abs().max())
    assert torch.equal(items[-1]["mel_lengths"], ref_lengths.to(items[-1]["mel_lengths"].device))


def run_case(model, glow, text, keep, chunks, z_seed=None, seed=9, sigma=0.666):
    S = model.decoder.max_decoder_steps
    z = None if z_seed is None else noise(text.shape[0], S, z_seed)
    ref, lengths = reference(model, glow, text, keep, z, sigma, seed)
    print("B=%d, cap %d: lengths %s" % (text.shape[0], S, lengths.tolist()[:8]))
    for chunk in chunks:
        mels = mel_items(model, text, keep, chunk)
        torch.manual_seed(seed)
        with t2.waveglow_noise(z):
            gen = glow.infer_stream(iter(mels), sigma=sigma)
        items = list(gen)
        print("chunk %d: %d mel items -> audio frames %s" % (chunk, len(mels), [tuple(s // HOP for s in it["samples"])
                                                                               for it in items]))
        check_audio_stream(items, mels, ref, lengths)
    return ref


@pytest.mark.parametrize("noise_kind", ["z", "philox"])
def test_stream_with_rows_stopping_at_different_steps(noise_kind):
    B, T, S = 3, 41, 300
    model = make_model("w7", weights())
    text, keep = rand_text(B, T, 5), keep_mask((S, 2, B, 256), 0.5, 6)
    thr = stop_threshold(model, text, keep, S, lambda L: len(set(L.tolist())) == 3 and int(L.max()) < S)
    set_decoder(model, S, thr)
    run_case(model, vocoder(), text, keep, [1, 7, 32, 128, S + 1], z_seed=3 if noise_kind == "z" else None)


def test_stream_with_a_row_that_never_fires():
    B, T, S = 3, 33, 230
    model = make_model("w7", weights())
    text, keep = rand_text(B, T, 9), keep_mask((S, 2, B, 256), 0.5, 10)
    thr = stop_threshold(model, text, keep, S, lambda L: bool((L == S).any()) and int(L.min()) < S - 5)
    set_decoder(model, S, thr)
    run_case(model, vocoder(), text, keep, [32, 128])


def test_stream_over_two_64_row_slices():
    B, T, S = 65, 23, 200
    model = make_model("w7", weights())
    text, keep = rand_text(B, T, 65), keep_mask((S, 2, B, 256), 0.5, 66)
    thr = stop_threshold(model, text, keep, S, lambda L: int(L[64]) < S and abs(int(L[:64].max()) - int(L[64])) >= 3)
    set_decoder(model, S, thr)
    run_case(model, vocoder(), text, keep, [32, 128], z_seed=4)


def test_stream_of_a_half_model_and_vocoder():
    B, T, S = 2, 31, 240
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(weights())
    model = model.cuda().eval().half()
    set_decoder(model, S, 1.0)
    text, keep = rand_text(B, T, 12), keep_mask((S, 2, B, 256), 0.5, 13)
    ref = run_case(model, vocoder(half=True), text, keep, [32, 128])
    assert ref.dtype == torch.float16


def test_two_interleaved_streams_and_an_abandoned_one():
    S = 220
    model = make_model("w7", weights())
    set_decoder(model, S, 1.0)
    glow = vocoder()
    cases = []
    for i, (B, T) in enumerate([(1, 30), (2, 44)]):
        text, keep = rand_text(B, T, 70 + i), keep_mask((S, 2, B, 256), 0.5, 80 + i)
        ref, lengths = reference(model, glow, text, keep, None, None, 100 + i)
        cases.append((mel_items(model, text, keep, 32), ref, lengths))
    gens = []
    for i, (mels, _, _) in enumerate(cases):
        torch.manual_seed(100 + i)
        gen = glow.infer_stream(iter(mels), sigma=0.666)
        gens.append((gen, [next(gen)]))               # the seed is drawn at the first item
    done = False
    while not done:
        done = True
        for gen, got in gens:
            if not got[-1]["finished"]:
                got.append(next(gen))
                done = False
    for (mels, ref, lengths), (_, got) in zip(cases, gens):
        check_audio_stream(got, mels, ref, lengths)
    # an abandoned stream leaves the next infer unchanged
    mel, z = mel_input(2, 150, 90), noise(2, 150, 91)
    with t2.waveglow_noise(z):
        before = glow.infer(mel.cuda(), sigma=0.5)
    gen = glow.infer_stream(iter(cases[1][0]), sigma=0.666)
    next(gen)
    del gen
    with t2.waveglow_noise(z):
        after = glow.infer(mel.cuda(), sigma=0.5)
    assert torch.equal(before, after)


# ---------------------------------------------------------------------------------------------------------------------
# infer itself: the bits of the build before windows existed
# ---------------------------------------------------------------------------------------------------------------------
BITS_FIXTURE = "waveglow_infer_bits_b64_t800"
BITS_SAMPLES = 4096


def bits_cases():
    """(name, half, philox): infer at B=64 x 800 in both tiers, with injected noise and with Philox noise and ragged
    lengths."""
    return [("%s_%s" % ("fp16" if half else "fp32", "philox" if philox else "z"), half, philox)
            for half in (False, True) for philox in (False, True)]


def bits_outputs(half, philox):
    """WaveGlow.infer on the seeded B=64 x 800 inputs of one case (whatever build tacotron2_b200 loads)."""
    B, T = 64, 800
    m = vocoder(half)
    mel = mel_input(B, T, 101).cuda()
    mel = mel.half() if half else mel
    with torch.no_grad():
        if philox:
            lengths = torch.randint(1, T + 1, (B,), generator=torch.Generator().manual_seed(102))
            lengths[0] = T
            torch.manual_seed(103)
            out = m.infer(mel, sigma=0.666, lengths=lengths)
        else:
            with t2.waveglow_noise(noise(B, T, 104)):
                out = m.infer(mel, sigma=0.666)
    return out.cpu()


def bits_sample(out):
    flat = out.reshape(-1)
    return flat[sample_index(flat.numel(), BITS_SAMPLES, 105)]


@pytest.mark.parametrize("name,half,philox", bits_cases(), ids=[c[0] for c in bits_cases()])
def test_infer_is_bit_identical_to_the_build_before_windows(name, half, philox):
    """The fixture holds the SHA-256 digest of the whole output and 4096 sampled samples of infer from the build before
    t2_waveglow_infer became the window call (tools/make_waveglow_bits.py); the outputs themselves are 26-52 MB each."""
    g = np.load(os.path.join(GOLDEN_DIR, BITS_FIXTURE + ".npz"))
    out = bits_outputs(half, philox)
    ref = torch.from_numpy(g[name + "_samples"]).to(out.dtype)
    got = bits_sample(out)
    assert torch.equal(got, ref), float((got.double() - ref.double()).abs().max())
    assert tensor_digest(out) == str(g[name + "_digest"])
