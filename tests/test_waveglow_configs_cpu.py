"""WaveGlow configurations beyond the published one, without a GPU: the shape-generic fp64 oracle against the
reference's own infer for each fixture configuration, the window halos each configuration implies against
t2_waveglow_window_halo_config, the weight table's length and order, and the host-side refusals."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tacotron2_b200.glow import _config_struct, config_halo, num_weights
from tests import waveglow_config_oracle as WO
from tests.common import GOLDEN_DIR, weights_checksum
from tests.waveglow_common import CONFIG, mel_input, noise
from tests.waveglow_configs import FIXTURE_CASES, GPU_CONFIGS, config, name_of, state_dict_for

T2_ERR_UNSUPPORTED = -4


def cfg_tuple(cfg):
    w = cfg["WN_config"]
    return (cfg["n_mel_channels"], cfg["n_flows"], cfg["n_group"], cfg["n_early_every"], cfg["n_early_size"],
            w["n_layers"], w["kernel_size"], w["n_channels"])


@pytest.fixture(scope="module")
def fixtures():
    return np.load(os.path.join(GOLDEN_DIR, "waveglow_configs.npz"))


@pytest.mark.parametrize("case", FIXTURE_CASES, ids=[name_of(c[0]) for c in FIXTURE_CASES])
def test_oracle_matches_the_reference_for_every_fixture_configuration(fixtures, case):
    cfg, B, T, sigma, wseed, mseed, zseed = case
    name = name_of(cfg)
    sd = state_dict_for(cfg, wseed)
    assert float(fixtures[name + "/checksum"]) == weights_checksum(sd)
    mel, z = torch.from_numpy(fixtures[name + "/mel"]), torch.from_numpy(fixtures[name + "/z"])
    assert torch.equal(mel, mel_input(B, T, mseed)) and torch.equal(z, noise(B, T, zseed))
    ref = torch.from_numpy(fixtures[name + "/audio"]).double()
    got = WO.infer(sd, mel.double(), float(fixtures[name + "/sigma"]), z.double())
    assert got.shape == ref.shape == (B, 256 * T)
    err = float((got - ref).abs().max() / ref.abs().max())
    print("%s: max |oracle - reference| / max |reference| = %.2e" % (name, err))
    assert err <= 1e-5


def test_the_published_configuration_keeps_its_constants():
    assert num_weights(cfg_tuple(CONFIG)) == _capi.T2_WAVEGLOW_NUM_WEIGHTS == 686
    assert config_halo(cfg_tuple(CONFIG)) == t2.window_halo() == (99, 96)


# ---- halos, pinned by autograd through the fp64 oracle at a narrow width ---------------------------------------------
HALO_CASES = sorted({(c["WN_config"]["n_layers"], c["n_flows"]) for c in GPU_CONFIGS} | {(1, 1), (3, 4)})


@pytest.mark.parametrize("layers,flows", HALO_CASES, ids=["l%d_f%d" % c for c in HALO_CASES])
def test_halos_are_the_receptive_field_of_the_configuration(layers, flows):
    """The halos are the noise's receptive field rounded out to whole frames: the audio of frames [t0, t1) depends on
    noise columns 32 t0 - reach and 32 t1 - 1 + reach, reach = n_flows (2^n_layers - 1), and on none further out.  The
    mel reaches one column less (a WN layer's conditioning is a 1x1 convolution, so the last layer's dilation is not
    spent on it), and the upsample adds the 3 frames before; every frame it reaches lies inside the halos.  The
    receptive field does not depend on the WN width, so a 16-channel WN keeps the fp64 run short."""
    narrow = config(16, layers, flows)
    left, right = config_halo(cfg_tuple(config(128, layers, flows)))
    reach = flows * (2 ** layers - 1)
    assert right == -(-reach // 32) and left == right + 3
    t0, t1 = left + 5, left + 25
    T = t1 + right + 5
    sd = {k: v.double() for k, v in state_dict_for(narrow, 3).items()}
    mel = mel_input(1, T, 4).double().requires_grad_()
    z = noise(1, T, 5).double().requires_grad_()
    WO.infer(sd, mel, 0.666, z)[:, 256 * t0:256 * t1].sum().backward()
    gm = mel.grad.abs().amax(dim=(0, 1))
    gz = z.grad.abs().amax(dim=(0, 1))
    z_lo, z_hi = 32 * t0 - reach, 32 * t1 + reach      # noise columns [z_lo, z_hi) matter
    assert float(gz[:z_lo].max()) == 0.0 and float(gz[z_hi:].max()) == 0.0
    assert float(gz[z_lo]) > 0.0 and float(gz[z_hi - 1]) > 0.0
    m_lo, m_hi = (z_lo + 1) // 32 - 3, (z_hi - 2) // 32      # the mel frames [m_lo, m_hi] matter
    print("l%d f%d: halos (%d, %d); mel frames [%d, %d] of [%d, %d]: %.3e, %.3e" %
          (layers, flows, left, right, m_lo, m_hi, t0 - left, t1 + right - 1, gm[m_lo], gm[m_hi]))
    assert float(gm[:m_lo].max()) == 0.0 and float(gm[m_hi + 1:].max()) == 0.0
    assert float(gm[m_lo]) > 0.0 and float(gm[m_hi]) > 0.0
    assert t0 - left <= m_lo and m_hi <= t1 + right - 1
    # the halos are tight: one frame less on either side misses a noise column the audio depends on
    assert z_lo < 32 * (t0 - right + 1) and z_hi > 32 * (t1 + right - 1)


# ---- weight table ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", GPU_CONFIGS + [c[0] for c in FIXTURE_CASES], ids=lambda c: name_of(c))
def test_weight_table_length_and_order_follow_the_state_dict(cfg):
    m = t2.WaveGlow(**cfg)
    sd = m.state_dict(keep_vars=True)
    table = m._weight_table()
    L, F = cfg["WN_config"]["n_layers"], cfg["n_flows"]
    assert len(table) == len(sd) == num_weights(cfg_tuple(cfg)) == 2 + F * (6 * L + 9)
    assert all(a is b for a, b in zip(table, sd.values()))
    assert [n for n in sd][-F:] == ["convinv.%d.conv.weight" % k for k in range(F)]
    for k in range(F):
        n_rem = m.convinv[k].conv.weight.shape[0]
        assert n_rem == WO.n_remaining(k, n_early_every=cfg["n_early_every"], n_early_size=cfg["n_early_size"])
        assert n_rem == WO.n_remaining(k, sd)


# ---- refusals -------------------------------------------------------------------------------------------------------
REFUSED = [
    dict(CONFIG, WN_config=dict(n_layers=8, n_channels=64, kernel_size=3)),
    dict(CONFIG, WN_config=dict(n_layers=8, n_channels=320, kernel_size=3)),
    dict(CONFIG, WN_config=dict(n_layers=8, n_channels=640, kernel_size=3)),
    dict(CONFIG, WN_config=dict(n_layers=11, n_channels=256, kernel_size=3)),
    dict(CONFIG, WN_config=dict(n_layers=0, n_channels=256, kernel_size=3)),
    dict(CONFIG, WN_config=dict(n_layers=8, n_channels=256, kernel_size=5)),
    dict(CONFIG, n_flows=17),
    dict(CONFIG, n_flows=0),
    dict(CONFIG, n_group=4),
    dict(CONFIG, n_mel_channels=40),
    dict(CONFIG, n_early_size=3),
    dict(CONFIG, n_flows=16, n_early_every=2, n_early_size=2),     # 8 - 2 * 7 channels left
]


@pytest.mark.parametrize("cfg", REFUSED, ids=lambda c: name_of(c) + "_g%d_m%d" % (c["n_group"], c["n_mel_channels"]) +
                         "_k%d" % c["WN_config"]["kernel_size"])
def test_configurations_outside_the_table_are_refused_on_the_host(cfg):
    L = _capi.lib()
    c = _config_struct(cfg_tuple(cfg))
    assert L.t2_waveglow_num_weights(C.byref(c)) == 0
    left, right = C.c_int32(-1), C.c_int32(-1)
    assert L.t2_waveglow_window_halo_config(C.byref(c), C.byref(left), C.byref(right)) == T2_ERR_UNSUPPORTED
    assert (left.value, right.value) == (-1, -1)
    assert b"configuration" in L.t2_last_error() or b"must" in L.t2_last_error()
    # create refuses before it looks for a device or reads a weight
    ptrs = (C.c_void_p * 1)()
    h = C.c_void_p()
    assert L.t2_waveglow_create(C.byref(h), C.byref(c), ptrs, 1, None) == T2_ERR_UNSUPPORTED
    assert not h.value


@pytest.mark.parametrize("cfg", GPU_CONFIGS, ids=lambda c: name_of(c))
def test_supported_configurations_are_accepted_on_the_host(cfg):
    L = _capi.lib()
    c = _config_struct(cfg_tuple(cfg))
    left, right = C.c_int32(), C.c_int32()
    assert L.t2_waveglow_window_halo_config(C.byref(c), C.byref(left), C.byref(right)) == 0
    assert L.t2_waveglow_num_weights(C.byref(c)) == len(t2.WaveGlow(**cfg).state_dict())
