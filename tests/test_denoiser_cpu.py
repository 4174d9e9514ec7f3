"""The denoiser's oracle (oracle/denoiser_oracle.py) against the reference's own waveglow/denoiser.py, and the facts the
engine's windows rely on, on the CPU.

tests/golden/denoiser_b2.npz was written by the reference (tools/make_golden.py denoiser): its bias_spec for the fp32
WaveGlow of synth_state_dict(7) in mode 'zeros', samples and sums of both bases, and the denoised stft_inputs(3, 10340)
at strengths 0.01, 0.1 and 3 (where 42 % of the bins clamp to zero)."""
import os

import numpy as np
import pytest
import torch

from oracle import denoiser_oracle as D
from oracle import waveglow_oracle as WO
from tests.common import GOLDEN_DIR, stft_inputs
from tests.waveglow_common import synth_state_dict

FIXTURE = os.path.join(GOLDEN_DIR, "denoiser_b2.npz")


def fixture():
    return np.load(FIXTURE)


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max())


def test_oracle_output_matches_the_reference():
    g = fixture()
    y, bias = stft_inputs(int(g["seed"]), int(g["n"])), torch.from_numpy(g["bias_spec"])
    for s in g["strengths"]:
        ref = torch.from_numpy(g["out_%g" % s])
        got = D.denoise(y, bias, float(s), torch.float32)
        assert got.shape == ref.shape == (2, 1, 256 * 40)
        assert rel(got, ref) <= 1e-6, s
        assert rel(D.denoise(y, bias, float(s), torch.float64), ref) <= 1e-5, s


def test_oracle_bases_match_the_reference():
    g = fixture()
    idx = torch.from_numpy(g["basis_idx"])
    for basis, name in ((D.stft_forward_basis(1024, 1024), "forward"), (D.stft_inverse_basis(), "inverse")):
        t = torch.from_numpy(basis)
        assert rel(t.reshape(-1)[idx], g[name + "_samples"]) <= 1e-6
        st = g[name + "_stats"]
        assert abs(float(t.double().abs().sum()) - st[1]) <= 1e-6 * st[1]
        assert abs(float(t.double().abs().max()) - st[2]) <= 1e-6 * st[2]


def test_oracle_bias_matches_the_reference():
    """bias_spec from the fp32 WaveGlow oracle (sigma = 0, so no noise) and the oracle's transform."""
    g = fixture()
    audio = WO.infer(synth_state_dict(int(g["wseed"])), torch.zeros(1, 80, 88), 0.0, torch.zeros(1, 8, 88 * 32))
    assert rel(D.bias_spec(audio, torch.float32), g["bias_spec"]) <= 1e-6


def test_engine_stft_bases_and_keys_match_the_reference():
    from tacotron2_b200.denoiser import STFT
    g = fixture()
    st = STFT(1024, 256, 1024)
    idx = torch.from_numpy(g["basis_idx"])
    for name in ("forward", "inverse"):
        b = getattr(st, name + "_basis")
        assert tuple(b.shape) == (1026, 1, 1024) and b.dtype == torch.float32
        assert rel(b.reshape(-1)[idx], g[name + "_samples"]) <= 1e-6
    assert list(g["keys"]) == ["bias_spec", "stft.forward_basis", "stft.inverse_basis"]
    assert list(g["shapes"]) == ["1,513,1", "1026,1,1024", "1026,1,1024"]
    assert ["stft." + k for k in st.state_dict()] == list(g["keys"])[1:]


def test_round_trip_at_strength_zero():
    y = stft_inputs(4, 256 * 30 + 77).double()
    out = D.denoise(y, torch.zeros(1, 513, 1), 0.0, torch.float64)
    assert rel(out[:, 0], y[:, :256 * 30]) <= 1e-6


@pytest.mark.parametrize("n", [256 * 12, 256 * 12 + 100])
def test_output_length(n):
    out = D.denoise(stft_inputs(5, n), torch.zeros(1, 513, 1), 0.1, torch.float64)
    assert out.shape == (2, 1, 256 * (n // 256))


def reach(n, j, bias):
    """Output samples of an fp64 denoise that change when input sample j is perturbed."""
    y = stft_inputs(6, n)[:1].double()
    base = D.denoise(y, bias, 0.1, torch.float64)[0, 0]
    y2 = y.clone()
    y2[0, j] += 1e-3
    d = (D.denoise(y2, bias, 0.1, torch.float64)[0, 0] - base).abs()
    return torch.nonzero(d > 1e-13).flatten()


def test_reach_is_three_blocks_each_way():
    """An input sample reaches the output samples of the frames that hold it, all within +-1023 samples; in 256-sample
    blocks, input block k reaches output blocks k - 3 ... k + 3 and no further.  Near the end the reflection folds the
    input back, so the last input sample reaches three blocks back as well."""
    bias = torch.from_numpy(fixture()["bias_spec"]).double()
    n = 256 * 24
    blocks = set()
    for j in (256 * 11, 256 * 11 + 1, 256 * 11 + 100, 256 * 12 - 1):
        ch = reach(n, j, bias)
        assert int(ch.min()) >= j - 1023 and int(ch.max()) <= j + 1023, j
        blocks |= set((ch // 256).tolist())
    assert blocks == set(range(11 - 3, 11 + 4))
    ch = reach(n, n - 1, bias)
    assert int(ch.min()) >= n - 1 - 1023 and int(ch.min()) // 256 == 24 - 1 - 3 and int(ch.max()) == n - 1


def test_library_reports_the_halo():
    from tacotron2_b200.denoiser import denoiser_halo
    assert denoiser_halo() == (3, 3)
