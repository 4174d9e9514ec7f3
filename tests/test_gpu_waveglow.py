"""WaveGlow.infer on the H100 against the reference's fixtures (bar: 1e-3 relative) and the fp64 oracle.

E64_BAR: the fp32-grade tier's audio against the fp64 oracle measures 0.9e-5 ... 1.3e-5 on an H100 over these cases;
the bar is about 4 x that.  (tests/test_gpu_waveglow_stages.py holds each of the 207 launches to its own bar.)"""
import os

import numpy as np
import pytest
import torch

from oracle import waveglow_oracle as WO
from tests.common import GOLDEN_DIR, rel_err, sample_index, tensor_digest
from tests.waveglow_common import CONFIG, mel_input, noise, philox_noise, synth_state_dict

import tacotron2_b200 as t2
from tacotron2_b200 import _capi

pytestmark = pytest.mark.gpu

E64_BAR = 5e-5

_SD = {}


def sd7():
    if "sd" not in _SD:
        _SD["sd"] = synth_state_dict(7)
    return _SD["sd"]


def model(half=False):
    m = t2.WaveGlow(**CONFIG)
    m.load_state_dict(sd7())
    m = m.cuda()
    if half:                                   # the notebook's form: .half(), then convinv back to fp32
        m = m.half()
        for k in m.convinv:
            k.float()
    return m


def load(name):
    return np.load(os.path.join(GOLDEN_DIR, name + ".npz"))


def run(m, mel, sigma, z=None, lengths=None):
    with t2.waveglow_noise(z):
        out = m.infer(mel.cuda(), sigma=sigma, lengths=lengths)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("name", ["waveglow_b1_t50_s0", "waveglow_b3_t37_s666"])
def test_fp32_tier_matches_reference_and_fp64_oracle(name):
    g = load(name)
    mel, z, sigma = torch.from_numpy(g["mel"]), torch.from_numpy(g["z"]), float(g["sigma"])
    out = run(model(), mel, sigma, z)
    assert out.dtype == torch.float32 and out.shape == (mel.shape[0], 256 * mel.shape[2])
    truth = WO.infer(sd7(), mel.cuda().double(), sigma, z.cuda().double())
    e_ref, e64 = rel_err(out, torch.from_numpy(g["audio"])), rel_err(out, truth)
    print("%s: engine vs reference %.2e, vs fp64 oracle %.2e" % (name, e_ref, e64))
    assert e_ref <= 1e-3 and e64 <= E64_BAR


def test_ragged_rows_are_bit_identical_to_their_own_runs():
    lens = [50, 37, 11, 1]
    B, T = len(lens), max(lens)
    mel, z = mel_input(B, T, 51), noise(B, T, 52)
    m = model()
    out = run(m, mel, 0.666, z, lengths=torch.tensor(lens))
    for b, n in enumerate(lens):
        one = run(m, mel[b:b + 1, :, :n], 0.666, z[b:b + 1, :, :32 * n])
        assert torch.equal(out[b, :256 * n], one[0]), b
        assert float(out[b, 256 * n:].abs().max()) == 0.0 if n < T else True
    truth = WO.infer(sd7(), mel[:1].cuda().double(), 0.666, z[:1].cuda().double())
    e = rel_err(out[0], truth[0])
    print("ragged: full-length row vs fp64 oracle %.2e" % e)
    assert e <= E64_BAR


def test_philox_noise_matches_host_rebuild_and_is_reproducible():
    B, T = 2, 23
    mel = mel_input(B, T, 61)
    m = model()
    torch.manual_seed(11)
    a = run(m, mel, 0.666)
    seed = m._t2.last_seed
    torch.manual_seed(11)
    b = run(m, mel, 0.666)
    assert torch.equal(a, b)
    truth = WO.infer(sd7(), mel.cuda().double(), 0.666, philox_noise(seed, B, T).cuda().double())
    e = rel_err(a, truth)
    print("philox: engine vs fp64 oracle on the host-rebuilt noise %.2e" % e)
    assert e <= E64_BAR
    c = run(m, mel, 0.666)                     # the next call draws fresh noise
    assert not torch.equal(a, c)


def test_fp16_tier_notebook_form_within_the_fp16_rounding_yardstick():
    B, T, sigma = 2, 40, 0.666
    mel, z = mel_input(B, T, 71), noise(B, T, 72)
    m = model(half=True)
    out = run(m, mel.half(), sigma, z)
    assert out.dtype == torch.float16
    # truth: fp64 on the fp16-rounded weights and input; yardstick: the oracle rounding where the reference's half path does
    sd16 = {k: (v.half().double() if not k.startswith("convinv") else v.double()) for k, v in sd7().items()}
    mel16 = mel.half()
    truth = WO.infer(sd16, mel16.cuda().double(), sigma, z.half().cuda().double())
    emul = WO.infer({k: (v.half() if not k.startswith("convinv") else v) for k, v in sd7().items()},
                    mel16.cuda(), sigma, z.half().cuda(), torch.float16)
    e_eng, e_ora = rel_err(out, truth), rel_err(emul, truth)
    print("fp16 tier: engine vs fp64 %.2e, fp16-emulating oracle vs fp64 %.2e (ratio %.2f)" % (e_eng, e_ora, e_eng / e_ora))
    assert e_eng <= 2.0 * e_ora


def test_full_length_batch_matches_the_800_frame_fixture():
    g = load("waveglow_full_b2_t800")
    T, sigma = int(g["T"]), float(g["sigma"])
    mel2, z2 = mel_input(2, T, int(g["mseed"])), noise(2, T, int(g["zseed"]))
    assert tensor_digest(mel2) == str(g["mel_digest"]) and tensor_digest(z2) == str(g["z_digest"])
    mel = torch.cat([mel2, mel_input(62, T, 81)])
    z = torch.cat([z2, noise(62, T, 82)])
    out = run(model(), mel, sigma, z)[:2].double().cpu()
    idx = torch.from_numpy(g["idx"])
    ref = torch.from_numpy(g["samples"]).double()
    e = rel_err(out.reshape(-1)[idx], ref)
    st = g["stats"]
    e_stats = max(abs(float(out.mean()) - st[0]), abs(float(out.std()) - st[1]), abs(float(out.abs().max()) - st[2]),
                  abs(float(out.abs().mean()) - st[3])) / st[2]
    print("B=64 x 800: rows 0-1 vs fixture samples %.2e, statistics %.2e" % (e, e_stats))
    assert e <= 1e-3 and e_stats <= 1e-3


def test_weight_cache_repacks_after_invalidate_and_load_state_dict():
    mel, z = mel_input(1, 12, 91), noise(1, 12, 92)
    m = model()
    a = run(m, mel, 0.5, z)
    m.WN[5].end.weight.data.mul_(0.5)          # .data writes do not move torch's version counter
    m.invalidate_weights()
    b = run(m, mel, 0.5, z)
    assert not torch.equal(a, b)
    m.load_state_dict(sd7())
    c = run(m, mel, 0.5, z)
    assert torch.equal(a, c)
    t2.WaveGlow.remove_weightnorm(m)           # plain weights: the same function
    d = run(m, mel, 0.5, z)
    assert rel_err(d, a) <= 1e-5


def test_unsupported_configuration_raises_before_any_launch():
    cfg = dict(CONFIG, WN_config=dict(n_layers=2, n_channels=64, kernel_size=3))
    m = t2.WaveGlow(**cfg).cuda()
    L = _capi.lib()
    n0 = L.t2_kernel_launch_count()
    with pytest.raises(_capi.T2Error, match="configuration"):
        m.infer(mel_input(1, 4, 0).cuda())
    assert L.t2_kernel_launch_count() == n0
