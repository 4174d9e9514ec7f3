"""Griffin-Lim and the public STFT on the CPU: the oracle (tests/griffin_lim_oracle.py) against the reference's own
audio_processing.griffin_lim, the C ABI's struct layout, the module surface the reference's notebook imports, and the
arguments refused before anything touches a GPU.

tests/golden/griffin_lim_b2.npz was written by the reference (tools/make_golden.py griffin_lim): the magnitude of
stft_inputs(5, 6244) through its stft.STFT(1024, 256, 1024) (2 rows x 25 frames), the numpy seed, and
griffin_lim(magnitude, stft, n_iters) for n_iters 0, 1 and 30, each started under np.random.seed(seed)."""
import os

import numpy as np
import pytest
import torch

from oracle import denoiser_oracle as D
from tests import griffin_lim_oracle as G
from tests.common import GOLDEN_DIR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def fixture():
    return np.load(os.path.join(GOLDEN_DIR, "griffin_lim_b2.npz"))


def angles(g):
    """The reference's initial angles (audio_processing.py:68) under the fixture's seed."""
    np.random.seed(int(g["np_seed"]))
    a = np.angle(np.exp(2j * np.pi * np.random.rand(*g["mag"].shape)))
    return torch.from_numpy(a.astype(np.float32))


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("n_iters", [0, 1, 30])
def test_oracle_matches_the_reference(n_iters):
    """The fp32 oracle computes what the reference computed (it is bit-identical on this fixture); the fp64 oracle
    stays within 2e-5 of it (measured 4.4e-7, 7.0e-7 and 4.1e-6 at 0, 1 and 30 iterations)."""
    g = fixture()
    mag, ref = torch.from_numpy(g["mag"]), torch.from_numpy(g["out_%d" % n_iters])
    a = angles(g)
    assert ref.shape == (2, 256 * (mag.shape[-1] - 1))
    assert rel(G.griffin_lim(mag, a, n_iters, torch.float32), ref) <= 1e-6
    assert rel(G.griffin_lim(mag, a, n_iters, torch.float64), ref) <= 2e-5


def test_oracle_spectral_convergence_does_not_increase():
    g = fixture()
    mag, a = torch.from_numpy(g["mag"]).double(), angles(g)
    errs = [G.spectral_convergence(mag, G.griffin_lim(mag, a, k)) for k in range(6)]
    for e0, e1 in zip(errs, errs[1:]):
        assert bool((e1 <= e0 * (1 + 1e-9)).all()), (e0, e1)


def test_oracle_ragged_rows_are_their_own_runs():
    g = fixture()
    mag, a = torch.from_numpy(g["mag"]).double(), angles(g)
    out = G.griffin_lim(mag, a, 2, lengths=torch.tensor([17, 3]))
    assert torch.equal(out[0, :256 * 16], G.griffin_lim(mag[:1, :, :17], a[:1, :, :17], 2)[0])
    assert not bool(out[0, 256 * 16:].any()) and not bool(out[1].any())


def test_the_notebook_imports_resolve():
    """inference.ipynb: ``from layers import TacotronSTFT, STFT`` and ``from audio_processing import griffin_lim``."""
    import tacotron2_b200 as t2
    from tacotron2_b200.audio_processing import griffin_lim
    from tacotron2_b200.denoiser import STFT as DenoiserSTFT
    from tacotron2_b200.layers import STFT, TacotronSTFT
    assert STFT is DenoiserSTFT is t2.STFT and griffin_lim is t2.griffin_lim and TacotronSTFT is t2.TacotronSTFT


def test_tacotron_stft_state_dict_has_the_reference_keys():
    """The reference's TacotronSTFT (layers.py:42-53) holds mel_basis and the stft_fn submodule's two bases."""
    import tacotron2_b200 as t2
    from tacotron2_b200.stft import STFT
    m = t2.TacotronSTFT()
    sd = m.state_dict()
    for k in ("mel_basis", "stft_fn.forward_basis", "stft_fn.inverse_basis"):
        assert k in sd, k
    assert isinstance(m.stft_fn, STFT)
    assert (m.stft_fn.filter_length, m.stft_fn.hop_length, m.stft_fn.win_length) == (1024, 256, 1024)
    assert torch.equal(sd["stft_fn.forward_basis"][:, 0], sd["forward_basis"])
    assert rel(sd["stft_fn.inverse_basis"][:, 0], D.stft_inverse_basis()) <= 1e-6


def test_window_sumsquare_and_dynamic_range():
    from tacotron2_b200 import audio_processing as A
    for frames in (1, 4, 25):
        assert np.array_equal(A.window_sumsquare('hann', frames, 256, 1024, 1024), D.window_sumsquare(frames))
    x = torch.tensor([0.0, 1e-6, 0.5, 3.0])
    assert torch.equal(A.dynamic_range_compression(x), torch.log(torch.clamp(x, min=1e-5)))
    assert torch.allclose(A.dynamic_range_decompression(A.dynamic_range_compression(x[2:])), x[2:])


def test_bad_arguments_are_refused_before_the_gpu():
    """Refused in Python, before a library call: too few frames, a configuration without kernels, CPU tensors, lengths
    of the wrong shape."""
    import tacotron2_b200 as t2
    st = t2.STFT(1024, 256, 1024)
    mag = torch.ones(2, 513, 10)
    with pytest.raises(ValueError, match="at least 4 frames"):
        t2.griffin_lim(torch.ones(1, 513, 3), st, 2)
    with pytest.raises(ValueError, match="at least 4 frames"):
        st.inverse(torch.ones(1, 513, 3), torch.zeros(1, 513, 3))
    with pytest.raises(ValueError, match="built for filter_length 1024"):
        t2.griffin_lim(mag, t2.STFT(), 2)                  # the reference's STFT default: 800 / 200 / 800
    with pytest.raises(ValueError, match="built for filter_length 1024"):
        t2.STFT(1024, 200, 800).transform(torch.zeros(1, 4000))
    with pytest.raises(ValueError, match="lengths must have shape"):
        t2.griffin_lim(mag, st, 2, lengths=torch.tensor([5, 6, 7]))
    with pytest.raises(ValueError, match="lengths must have shape"):
        st.transform(torch.zeros(2, 4000), lengths=[4000])
    with pytest.raises(ValueError, match="cannot be reflect-padded"):
        st.transform(torch.zeros(2, 512))
    with pytest.raises(ValueError, match="n_iters"):
        t2.griffin_lim(mag, st, -1)
    with pytest.raises(RuntimeError, match="CUDA"):
        t2.griffin_lim(mag, st, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        st.transform(torch.zeros(2, 4000))
    with pytest.raises(RuntimeError, match="CUDA"):
        st.inverse(mag, torch.zeros_like(mag))
    state = np.random.get_state()[1].copy()
    with pytest.raises(ValueError):
        t2.griffin_lim(torch.ones(1, 513, 3), st, 2)
    assert np.array_equal(np.random.get_state()[1], state)      # a refused call draws no angles
