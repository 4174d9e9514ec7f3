"""WaveGlow without a GPU: module surface and seeded initialisation against the reference's, the plain-torch oracle
against the reference's own infer, the host rebuild of the engine's noise, and the C ABI struct layouts."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import waveglow_oracle as WO
from tests.common import GOLDEN_DIR, ROOT, rel_err, tensor_digest, weights_checksum
from tests.waveglow_common import CONFIG, mel_input, noise, philox_noise, state_dict_shapes, synth_state_dict

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tacotron2_b200.glow import noise_channel_order


def load(name):
    return np.load(os.path.join(GOLDEN_DIR, name + ".npz"))


def test_state_dict_keys_shapes_and_order_match_the_reference():
    g = load("waveglow_init")
    m = t2.WaveGlow(**CONFIG)
    sd = m.state_dict()
    assert len(sd) == 686
    assert list(sd) == [str(k) for k in g["keys"]]
    assert [",".join(str(x) for x in v.shape) for v in sd.values()] == [str(s) for s in g["shapes"]]
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == state_dict_shapes()


def test_seeded_initialisation_is_bit_identical_before_and_after_remove_weightnorm():
    g = load("waveglow_init")
    torch.manual_seed(1234)
    m = t2.WaveGlow(**CONFIG)
    assert [tensor_digest(v) for v in m.state_dict().values()] == [str(d) for d in g["digests"]]
    assert all(float(v.abs().max()) == 0.0 for k, v in m.state_dict().items() if ".end." in k)   # the reference's zeroed end
    m = t2.WaveGlow.remove_weightnorm(m)
    sd = m.state_dict()
    assert list(sd) == [str(k) for k in g["removed_keys"]]
    assert [tensor_digest(v) for v in sd.values()] == [str(d) for d in g["removed_digests"]]


def test_state_dicts_from_before_and_after_removal_load():
    sd = synth_state_dict(7)
    m = t2.WaveGlow(**CONFIG)
    m.load_state_dict(sd)
    removed = t2.WaveGlow.remove_weightnorm(m).state_dict()
    m2 = t2.WaveGlow.remove_weightnorm(t2.WaveGlow(**CONFIG))
    m2.load_state_dict(removed)
    assert len(m2._weight_table()) == 686


@pytest.mark.parametrize("name", ["waveglow_b1_t50_s0", "waveglow_b3_t37_s666"])
def test_oracle_matches_reference_infer(name):
    g = load(name)
    sd = synth_state_dict(int(g["wseed"]))
    assert abs(weights_checksum(sd) - float(g["checksum"])) < 1e-6 * float(g["checksum"])
    mel, z, sigma = torch.from_numpy(g["mel"]), torch.from_numpy(g["z"]), float(g["sigma"])
    ref = torch.from_numpy(g["audio"])
    out32 = WO.infer(sd, mel, sigma, z, torch.float32)
    out64 = WO.infer(sd, mel, sigma, z, torch.float64)
    e32, e64 = rel_err(out32, ref), rel_err(ref, out64)
    print("%s: oracle fp32 vs reference %.2e, reference vs oracle fp64 %.2e" % (name, e32, e64))
    assert e32 <= 1e-5 and e64 <= 1e-5
    assert float(ref.abs().max()) > 0.1                       # the couplings are not the identity


def test_host_noise_rebuild_is_standard_normal_and_keyed_per_row():
    z = philox_noise(0x1234_5678_9abc, 3, 40)
    assert z.shape == (3, 8, 1280) and z.dtype == torch.float32
    assert abs(float(z.mean())) < 0.02 and abs(float(z.std()) - 1.0) < 0.02
    assert torch.equal(philox_noise(0x1234_5678_9abc, 2, 40)[1], z[1])         # independent of B
    assert torch.equal(philox_noise(0x1234_5678_9abc, 3, 20)[2], z[2, :, :640])  # and of the padded length
    assert not torch.equal(philox_noise(0x1234_5678_9abd, 3, 40), z)


def test_noise_draw_order():
    assert noise_channel_order() == [(None, 4), (8, 2), (4, 2)]


def test_forward_is_not_implemented_and_infer_needs_cuda():
    m = t2.WaveGlow(**CONFIG)
    with pytest.raises(NotImplementedError):
        m((torch.zeros(1, 80, 4), torch.zeros(1, 1024)))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.infer(mel_input(1, 4, 0))


def test_oracle_fp64_is_consistent_across_rows():
    """Rows of a batch are independent in the oracle (what the engine's ragged test relies on)."""
    sd = synth_state_dict(7)
    mel, z = mel_input(2, 6, 3), noise(2, 6, 4)
    both = WO.infer(sd, mel, 0.5, z)
    one = WO.infer(sd, mel[1:], 0.5, z[1:])
    assert rel_err(both[1:], one) < 1e-12


def test_oracle_steps_compose_to_infer_bit_for_bit():
    """infer is the composition of the oracle's named steps.  Its fp64 and fp16-emulating outputs on a seeded case are
    the bits recorded before infer was split into steps (tests/golden/waveglow_oracle_b2_t3.npz, one CPU thread), and the
    steps called one by one -- as the per-launch GPU tests call them, each gate computing its own slice of the
    conditioning -- give the same audio."""
    g = load("waveglow_oracle_b2_t3")
    sd = synth_state_dict(7)
    sd16 = {k: (v.half() if not k.startswith("convinv") else v) for k, v in sd.items()}
    mel, z, sigma = mel_input(2, 3, 101), noise(2, 3, 102), 0.666

    def by_steps(sd, mel, z):
        spect = WO.upsample_unfold(sd, mel)
        aud = sigma * z[:, :WO.n_remaining(11)]
        for k in reversed(range(12)):
            h = WO.start(sd, k, aud)
            skip = torch.zeros_like(h)
            for l in range(8):
                acts = WO.gate(sd, k, l, h, spect)
                h, skip = WO.res_skip(sd, k, l, acts, h, skip)
            aud = WO.flow_tail(sd, k, aud, skip, z, sigma)
        return aud.permute(0, 2, 1).contiguous().view(mel.shape[0], -1)

    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        a64 = WO.infer(sd, mel, sigma, z)
        a16 = WO.infer(sd16, mel.half(), sigma, z.half(), torch.float16)
        s64, s16 = by_steps(sd, mel.double(), z.double()), by_steps(sd16, mel.half(), z.half())
    finally:
        torch.set_num_threads(threads)
    assert a64.dtype == torch.float64 and a16.dtype == torch.float16
    assert np.array_equal(a64.numpy(), g["a64"]) and np.array_equal(a16.numpy(), g["a16"])
    assert torch.equal(s64, a64) and torch.equal(s16, a16)
    assert [WO.n_remaining(k) for k in (11, 8, 7, 4, 3, 0)] == [4, 4, 6, 6, 8, 8]


def test_waveglow_ctypes_structs_match_c_layout(tmp_path):
    src = tmp_path / "layout.c"
    fields = {
        "T2WaveGlowConfig": ["n_mel_channels", "n_flows", "n_group", "n_early_every", "n_early_size", "wn_n_layers",
                             "wn_kernel_size", "wn_n_channels", "fp16"],
        "T2WaveGlowArgs": ["mel", "B", "T_mel", "lengths", "io_half", "sigma", "z", "seed", "audio", "ws", "ws_bytes"],
    }
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "t2b200.h"', 'int main(void){',
             'printf("NUM %d\\n", T2_WAVEGLOW_NUM_WEIGHTS);']
    for s, fs in fields.items():
        lines.append('printf("%s %%zu\\n", sizeof(%s));' % (s, s))
        for f in fs:
            lines.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (s, f, s, f))
    lines.append('return 0;}')
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    assert int(out["NUM"]) == _capi.T2_WAVEGLOW_NUM_WEIGHTS == 686
    for s, fs in fields.items():
        cls = getattr(_capi, s)
        assert int(out[s]) == ctypes.sizeof(cls), s
        for f in fs:
            assert int(out["%s.%s" % (s, f)]) == getattr(cls, f).offset, (s, f)
