"""The receptive field behind windowed WaveGlow inference (t2_waveglow_infer_window), pinned on the CPU with the fp64
oracle, and the C layout of its argument struct.

The audio of mel frames [t0, t1) is fixed by the frames [t0 - 99, t1 + 96): twelve flows of a WN whose dilated k = 3
layers reach +-255 group columns give +-3060 columns (96 frames of 32 columns, rounded out), and the upsample gives a
column of frame f the frames f-3 ... f.  A window with these halos must reproduce the full run's samples, and the
audio must depend on the frames at both edges of the halo and on none beyond them.  The receptive field does not
depend on the WN width, so a 16-channel WN keeps the fp64 runs short (the published 256 channels take minutes at 250
frames)."""
import math
from unittest import mock

import pytest
import torch

import tacotron2_b200 as t2
from oracle import waveglow_oracle as WO
from tests.waveglow_common import CONFIG, mel_input, noise

HALO_LEFT, HALO_RIGHT = 99, 96
WIDTH = 16


def narrow_state_dict(width, seed):
    """Seeded weights of a WaveGlow whose WN has ``width`` channels, drawn as tests/waveglow_common.synth_state_dict
    draws the published ones (non-zero ``end``, weight_g off ||v||, orthonormal convinv with determinant +1)."""
    m = t2.WaveGlow(**dict(CONFIG, WN_config=dict(n_layers=8, n_channels=width, kernel_size=3)))
    g = torch.Generator().manual_seed(seed)
    u = lambda shape, b: (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) * b      # noqa: E731
    sd = {}
    for name, v in m.state_dict().items():
        shape = tuple(v.shape)
        if name == "upsample.weight":
            sd[name] = u(shape, 1.0 / math.sqrt(4 * 80))
        elif name.endswith("weight_v"):
            sd[name] = u(shape, 1.0 / math.sqrt(shape[1] * shape[2]))
        elif name.endswith("weight_g"):
            sd[name] = None
        elif name.endswith("end.weight"):
            sd[name] = u(shape, 1.0 / 16)
        elif name.startswith("convinv"):
            c = shape[0]
            w = torch.linalg.qr(torch.randn(c, c, generator=g, dtype=torch.float64))[0]
            if torch.det(w) < 0:
                w[:, 0] = -w[:, 0]
            sd[name] = w.view(c, c, 1)
        else:
            sd[name] = u(shape, 0.05)
    for name in sd:
        if name.endswith("weight_g"):
            v = sd[name[:-1] + "v"]
            sd[name] = v.flatten(1).norm(dim=1).view(-1, 1, 1) * (0.5 + torch.rand(v.shape[0], 1, 1, generator=g,
                                                                                      dtype=torch.float64))
    return sd


def oracle_infer(sd, mel, sigma, z):
    """The fp64 oracle at the narrow width.  oracle/waveglow_oracle.py states the published WN width (256) as the module
    constant N_CH, which it uses only to split the gate channels; it is replaced for the duration of the call."""
    assert sd["WN.0.start.weight_v"].shape[0] == WIDTH
    with mock.patch.object(WO, "N_CH", WIDTH):
        return WO.infer(sd, mel, sigma, z)


@pytest.fixture(scope="module")
def narrow():
    T, sigma = 250, 0.666
    sd = narrow_state_dict(WIDTH, 3)
    mel, z = mel_input(1, T, 4).double(), noise(1, T, 5).double()
    return dict(T=T, sigma=sigma, sd=sd, mel=mel, z=z, full=oracle_infer(sd, mel, sigma, z))


def window_audio(c, w0, w1, t0, t1):
    """Oracle audio of frames [t0, t1) from a run over the frames [w0, w1) alone, with the noise of those columns."""
    out = oracle_infer(c["sd"], c["mel"][:, :, w0:w1], c["sigma"], c["z"][:, :, 32 * w0:32 * w1])
    return out[:, 256 * (t0 - w0):256 * (t1 - w0)]


def test_halo_is_sufficient(narrow):
    """The halos suffice: the windowed run reproduces the full one.  (Shorter windows do too, to fp64 rounding: the
    dependence at the halo's edge is far below it; test_halo_is_tight shows the halos are also needed.)"""
    c = narrow
    t0, t1 = 110, 140
    ref = c["full"][:, 256 * t0:256 * t1]
    assert float(ref.abs().max()) > 0.1
    d = float((window_audio(c, t0 - HALO_LEFT, t1 + HALO_RIGHT, t0, t1) - ref).abs().max())
    print("frames [%d, %d) from the window [%d, %d): max |diff| %.3e" % (t0, t1, t0 - HALO_LEFT, t1 + HALO_RIGHT, d))
    assert d <= 1e-12


def test_halo_is_tight(narrow):
    """The audio of frames [t0, t1) depends on mel frames t0 - 99 and t1 + 95 and on noise columns 32 t0 - 3060 and
    32 t1 - 1 + 3060, and on nothing further out.  The dependence at the edge passes through twelve flows of eight layers
    at full dilation reach, so its size (printed) lies far below fp64 rounding of the audio: a window one frame short
    gives the same fp64 samples.  Autograd measures it exactly instead; outside the receptive field the sensitivity is
    exactly zero."""
    c = narrow
    t0, t1 = 110, 140
    mel, z = c["mel"].clone().requires_grad_(), c["z"].clone().requires_grad_()
    oracle_infer(c["sd"], mel, c["sigma"], z)[:, 256 * t0:256 * t1].sum().backward()
    gm = mel.grad.abs().amax(dim=(0, 1))                # per frame
    gz = z.grad.abs().amax(dim=(0, 1))                  # per group column
    lo, hi = t0 - HALO_LEFT, t1 + HALO_RIGHT            # the frames [lo, hi) matter
    print("sensitivity to mel frame %d: %.3e, %d: %.3e; frame %d: %.3e, %d: %.3e" %
          (lo - 1, gm[lo - 1], lo, gm[lo], hi - 1, gm[hi - 1], hi, gm[hi]))
    assert float(gm[:lo].abs().max()) == 0.0 and float(gm[hi:].abs().max()) == 0.0
    assert float(gm[lo]) > 0.0 and float(gm[hi - 1]) > 0.0
    reach = 12 * 255
    z_lo, z_hi = 32 * t0 - reach, 32 * t1 + reach      # noise columns [z_lo, z_hi) matter
    print("sensitivity to noise column %d: %.3e, %d: %.3e; column %d: %.3e, %d: %.3e" %
          (z_lo - 1, gz[z_lo - 1], z_lo, gz[z_lo], z_hi - 1, gz[z_hi - 1], z_hi, gz[z_hi]))
    assert float(gz[:z_lo].max()) == 0.0 and float(gz[z_hi:].max()) == 0.0
    assert float(gz[z_lo]) > 0.0 and float(gz[z_hi - 1]) > 0.0
    # the stated halos are the receptive field rounded out to whole frames
    assert HALO_RIGHT == -(-reach // 32) and HALO_LEFT == HALO_RIGHT + 3


def test_windows_at_the_sequence_edges_need_no_halo_there(narrow):
    c = narrow
    T = c["T"]
    for (w0, w1, t0, t1) in [(0, 30 + HALO_RIGHT, 0, 30), (T - 30 - HALO_LEFT, T, T - 30, T)]:
        got = window_audio(c, w0, w1, t0, t1)
        d = float((got - c["full"][:, 256 * t0:256 * t1]).abs().max())
        print("window [%d, %d) -> frames [%d, %d): max |diff| %.3e" % (w0, w1, t0, t1, d))
        assert d <= 1e-12
