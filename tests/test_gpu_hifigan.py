"""HiFi-GAN on the H100 against the fp64 oracle (tests/hifigan_oracle.py): V1, V2 and V3, both tiers, ragged batches,
weight handling, exact-size buffers and the library's refusals.

BAR: max|engine - oracle| / max|oracle| of the fp32-grade tier.  The fp16 tier is held to twice the error of an oracle
that rounds to fp16 wherever that tier stores fp16."""
import ctypes as C

import pytest
import torch

from tests import hifigan_oracle as HO
from tests.hifigan_common import mel_input, model, synth_state_dict

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tacotron2_b200.hifigan import CONFIGS, config_struct

pytestmark = pytest.mark.gpu

BAR = 1e-4


def rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


def oracle(G, mel, round16=False, rows=8):
    """The fp64 oracle on the GPU, a few rows at a time."""
    sd = {k: v.detach() for k, v in G.state_dict().items()}
    return torch.cat([HO.forward(sd, G.h, mel[i:i + rows].cuda(), round16) for i in range(0, mel.shape[0], rows)])


def run(G, mel, lengths=None):
    with torch.no_grad():
        out = G(mel.cuda(), lengths=lengths)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("name", ["v1", "v2", "v3"])
@pytest.mark.parametrize("B,T", [(2, 24), (64, 800)])
def test_fp32_tier_against_the_fp64_oracle(name, B, T):
    G = model(name).cuda().eval()
    mel = mel_input(B, T, 11)
    out = run(G, mel)
    assert out.dtype == torch.float32 and tuple(out.shape) == (B, 1, 256 * T)
    ref = oracle(G, mel)
    e = rel(out, ref)
    print("hifigan %s B=%d T=%d fp32 tier: rel err %.2e, output std %.3f, max |y| %.3f"
          % (name, B, T, e, ref.std().item(), ref.abs().max().item()))
    assert 0.05 < ref.std().item() and ref.abs().max().item() < 0.999    # the tanh is neither idle nor saturated
    assert e < BAR


@pytest.mark.parametrize("name", ["v1", "v2", "v3"])
def test_fp16_tier_within_twice_an_fp16_storing_oracle(name):
    G = model(name).cuda().eval().half()
    mel = mel_input(2, 24, 12).half()
    out = run(G, mel)
    assert out.dtype == torch.float16 and tuple(out.shape) == (2, 1, 256 * 24)
    ref = oracle(G, mel)
    ref16 = oracle(G, mel, round16=True)
    e, e16 = rel(out, ref), rel(ref16, ref)
    print("hifigan %s fp16 tier: rel err %.2e; the fp16-storing oracle's %.2e" % (name, e, e16))
    assert e <= 2 * e16


@pytest.mark.parametrize("half", [False, True])
def test_ragged_rows_equal_their_own_b1_calls_bit_for_bit(half):
    G = model("v2").cuda().eval()
    if half:
        G = G.half()
    B, T = 130, 24
    g = torch.Generator().manual_seed(3)
    lengths = torch.randint(1, T + 1, (B,), generator=g)
    lengths[0], lengths[1] = T, 1
    mel = mel_input(B, T, 13).to(G.conv_pre.bias.dtype)
    mel_dirty = mel.clone()
    for b in range(B):       # frames past a row's length must not matter
        mel_dirty[b, :, int(lengths[b]):] = 1e3
    out = run(G, mel_dirty, lengths=lengths.cuda())
    for b in range(B):
        n = int(lengths[b])
        one = run(G, mel[b:b + 1, :, :n])
        assert torch.equal(out[b, :, :256 * n], one[0]), b
        assert not out[b, :, 256 * n:].any(), b


def test_remove_weight_norm_and_load_state_dict_repack():
    G = model("v3").cuda().eval()
    mel = mel_input(2, 24, 14)
    before = run(G, mel)
    G.remove_weight_norm()
    after = run(G, mel)
    assert rel(after, before) < BAR
    assert rel(after, oracle(G, mel)) < BAR
    G2 = model("v3", seed=3).cuda().eval()
    sd = synth_state_dict(G2, 9)
    G2.load_state_dict({k: v.cuda() for k, v in sd.items()})
    out = run(G2, mel)
    assert rel(out, before) > 1e-2
    assert rel(out, oracle(G2, mel)) < BAR


def _handle(G):
    G(torch.zeros(1, 80, 2, device="cuda", dtype=G.conv_pre.bias.dtype))
    return G._t2.handle


def test_exact_size_output_and_workspace_buffers():
    G = model("v3").cuda().eval()
    with torch.no_grad():
        h = _handle(G)
    L = _capi.lib()
    B, T = 3, 17
    mel = mel_input(B, T, 15).cuda()
    n_ws = L.t2_hifigan_workspace_bytes(h, B, T)
    canary = 4096
    ws = torch.full((n_ws + canary,), 0x5A, dtype=torch.uint8, device="cuda")
    audio = torch.full((B * 256 * T + canary,), 7.0, device="cuda")
    lengths = torch.tensor([17, 5, 9], dtype=torch.int32, device="cuda")
    a = _capi.T2HiFiGANArgs(mel.data_ptr(), B, T, lengths.data_ptr(), 0, audio.data_ptr(), ws.data_ptr(), n_ws)
    _capi.call(L.t2_hifigan_infer, torch.device("cuda"), h, C.byref(a))
    torch.cuda.synchronize()
    assert bool((ws[n_ws:] == 0x5A).all())
    assert bool((audio[B * 256 * T:] == 7.0).all())
    with torch.no_grad():
        ref = G(mel, lengths=lengths)
    assert torch.equal(audio[:B * 256 * T].view(B, 1, 256 * T), ref)
    # device lengths are clamped: past T acts as T, below 0 as 0
    wild = torch.tensor([1000, -4, 9], dtype=torch.int32, device="cuda")
    a.lengths = wild.data_ptr()
    _capi.call(L.t2_hifigan_infer, torch.device("cuda"), h, C.byref(a))
    torch.cuda.synchronize()
    got = audio[:B * 256 * T].view(B, 1, 256 * T)
    with torch.no_grad():
        full = G(mel)
    assert torch.equal(got[0], full[0]) and not got[1].any() and torch.equal(got[2], ref[2])


def test_library_refusals():
    L = _capi.lib()
    assert L.t2_hifigan_num_weights(C.byref(config_struct(CONFIGS["v1"]))) == 234
    assert L.t2_hifigan_num_weights(C.byref(config_struct(CONFIGS["v3"]))) == 69
    bad = dict(CONFIGS["v1"], upsample_rates=[8, 8, 2, 4], upsample_kernel_sizes=[16, 16, 4, 8])
    assert L.t2_hifigan_num_weights(C.byref(config_struct(bad))) == 0
    assert L.t2_hifigan_num_weights(None) == 0
    G = model("v3").cuda().eval()
    tab = G._weight_table()
    ptrs = (C.c_void_p * len(tab))(*[t.data_ptr() if t is not None else None for t in tab])
    h = C.c_void_p()
    for cfg in (bad, dict(CONFIGS["v3"], resblock_kernel_sizes=[3, 5, 8]),
                dict(CONFIGS["v3"], upsample_initial_channel=252)):
        assert L.t2_hifigan_create(C.byref(h), C.byref(config_struct(cfg)), ptrs, len(tab), None) == -4
        assert b"upsample" in L.t2_last_error() or b"resblock" in L.t2_last_error() or b"channel" in L.t2_last_error()
    assert L.t2_hifigan_create(C.byref(h), C.byref(config_struct(CONFIGS["v3"])), ptrs, len(tab) - 1, None) == -1
    ptrs0 = (C.c_void_p * len(tab))(*[t.data_ptr() if t is not None else None for t in tab])
    ptrs0[2] = None
    assert L.t2_hifigan_create(C.byref(h), C.byref(config_struct(CONFIGS["v3"])), ptrs0, len(tab), None) == -1
    with torch.no_grad():
        h = _handle(G)
    mel = torch.zeros(2, 80, 5, device="cuda")
    audio = torch.zeros(2, 256 * 5, device="cuda")
    n_ws = L.t2_hifigan_workspace_bytes(h, 2, 5)
    ws = torch.zeros(n_ws, dtype=torch.uint8, device="cuda")
    count = L.t2_kernel_launch_count()
    for B, T, n, rc in ((0, 5, n_ws, -1), (2, 0, n_ws, -1), (2, 5, n_ws - 1, -3), (64, 70000, n_ws, -1)):
        a = _capi.T2HiFiGANArgs(mel.data_ptr(), B, T, None, 0, audio.data_ptr(), ws.data_ptr(), n)
        assert L.t2_hifigan_infer(h, C.byref(a), None) == rc
    a = _capi.T2HiFiGANArgs(None, 2, 5, None, 0, audio.data_ptr(), ws.data_ptr(), n_ws)
    assert L.t2_hifigan_infer(h, C.byref(a), None) == -1
    a = _capi.T2HiFiGANArgs(mel.data_ptr(), 2, 5, None, 2, audio.data_ptr(), ws.data_ptr(), n_ws)
    assert L.t2_hifigan_infer(h, C.byref(a), None) == -1
    assert L.t2_kernel_launch_count() == count
    assert L.t2_hifigan_workspace_bytes(h, 0, 5) == 0


def test_text_to_audio_on_tacotron2_mels():
    from tests.common import rand_text, synth_state_dict as t2_sd
    model_t2 = t2.Tacotron2(t2.create_hparams())
    model_t2.load_state_dict(t2_sd(5, gate_bias=-10.0, scale=2.0))
    model_t2 = model_t2.cuda().eval()
    model_t2.decoder.max_decoder_steps = 20
    G = model("v2").cuda().eval()
    text = rand_text(3, 19, 3).cuda()
    with torch.no_grad():
        mel = model_t2.inference(text, input_lengths=[19, 12, 7])[1]
        audio = G(mel, lengths=model_t2.mel_lengths)
    lens = model_t2.mel_lengths.cpu()
    assert tuple(audio.shape) == (3, 1, 256 * mel.shape[2])
    for b in range(3):
        n = int(lens[b])
        with torch.no_grad():
            one = G(mel[b:b + 1, :, :n])
        assert torch.equal(audio[b, :, :256 * n], one[0])
