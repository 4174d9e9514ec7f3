"""CPU: the oracle against what the unmodified reference (NVIDIA/tacotron2) computed for the same inputs, stored in
tests/golden/reference_live.npz by tools/make_golden.py (``live``): batched inference, the state_dict layout, a full
training step's gradients and stft.STFT."""
import os

import numpy as np
import torch

from oracle import tacotron2_oracle as O
from tests.common import GOLDEN_DIR, keep_mask, rand_text, rel_err, synth_state_dict

_golden = None


def golden():
    global _golden
    if _golden is None:
        _golden = dict(np.load(os.path.join(GOLDEN_DIR, "reference_live.npz")))
    return _golden


def test_reference_inference_b1_live():
    g = golden()
    sd = synth_state_dict(5, gate_bias=-10.0, scale=2.0)
    text = rand_text(1, 19, 3); keep = keep_mask((12, 2, 1, 256), 0.5, 4)
    r = [torch.from_numpy(g["infer/" + k]) for k in ("mel", "post", "gate", "align")]
    with torch.no_grad():
        mel, post, gate, align, lengths = O.tacotron2_inference(sd, text, keep, 0.5, 12)
    assert int(lengths[0]) == r[0].shape[2] == 12
    for a, b in zip((mel, post, gate, align), r):
        assert rel_err(a, b) < 2e-5


def test_reference_state_dict_layout():
    """The 84 keys / shapes the boundary must reproduce (SURVEY.md section 8(b1))."""
    from tests.common import state_dict_shapes
    g = golden()
    keys = [str(k) for k in g["sd/keys"]]
    want = state_dict_shapes()
    assert keys == list(want.keys())
    for k, shp in zip(keys, g["sd/shapes"]):
        assert tuple(int(x) for x in shp if x) == tuple(want[k]), k


def test_reference_training_step_gradients_live():
    """Full training step (forward + Tacotron2Loss + backward) of the unmodified reference vs torch autograd through
    the oracle: every parameter gradient (sum, abs-sum, max, sum of squares and 96 sampled entries of the reference's)."""
    from tests.test_oracle_golden import grad_sample_index, oracle_train_step
    g = golden()
    B, T, Tm, seed = 3, 15, 8, 91
    sd = synth_state_dict(4321, scale=2.0)
    gen = torch.Generator().manual_seed(seed)
    text = rand_text(B, T, seed + 1)
    tl = torch.sort(torch.randint(T // 3, T + 1, (B,), generator=gen), descending=True)[0]
    tl[0] = T
    ol = torch.randint(Tm // 3, Tm + 1, (B,), generator=gen)
    ol[1] = Tm
    mels = torch.randn(B, 80, Tm, generator=gen)
    gt = torch.zeros(B, Tm)
    for i, n in enumerate(ol.tolist()):
        mels[i, :, n:] = 0.0
        gt[i, n - 1:] = 1.0
    m = dict(pk=keep_mask((Tm + 1, 2, B, 256), 0.5, seed + 2), ak=keep_mask((Tm, B, 1024), 0.1, seed + 3),
             dk=keep_mask((Tm, B, 1024), 0.1, seed + 4), ek=keep_mask((3, B, 512, T), 0.5, seed + 5),
             qk4=keep_mask((4, B, 512, Tm), 0.5, seed + 6), qk1=keep_mask((B, 80, Tm), 0.5, seed + 7))
    loss = float(g["train/loss"])
    o_loss, _, o_grads = oracle_train_step(sd, text, tl, ol, mels, gt, m, True)
    assert abs(loss - float(o_loss)) < 1e-5 * abs(loss)
    names = [k[len("train/g/"):] for k in g if k.startswith("train/g/")]
    assert sorted(names) == sorted(o_grads.keys())
    for k in names:
        ref = torch.from_numpy(g["train/g/" + k])
        gsum, gabs, gmax, gsq, sample = ref[0], ref[1], float(ref[2]), ref[3], ref[4:]
        og = o_grads[k].detach().double().reshape(-1)
        if gmax < 1e-5:      # conv biases in front of a training-mode BatchNorm: rounding noise
            assert float(og.abs().max()) < 1e-4
            continue
        idx = grad_sample_index(k, og.numel())
        assert float((og[idx] - sample).abs().max()) / gmax < 1e-4, k
        assert abs(float(og.abs().max()) - gmax) / gmax < 1e-4, k
        assert abs(float(og.sum()) - float(gsum)) / float(gabs) < 1e-4, k
        assert abs(float(og.abs().sum()) - float(gabs)) / float(gabs) < 1e-4, k
        assert abs(float((og * og).sum()) ** 0.5 - float(gsq) ** 0.5) / float(gsq) ** 0.5 < 1e-4, k


def test_stft_oracle_vs_reference_stft_live():
    """oracle/stft_oracle.py against the reference's own stft.STFT (run with functional stand-ins for the two
    librosa.util helpers stft.py imports): the windowed Fourier basis and the magnitudes for three filter / hop settings,
    2048 sampled entries each and the full tensors' sum, abs-sum, sum of squares and maximum."""
    from oracle import stft_oracle as S
    from tests.common import sample_index, stft_inputs
    g = golden()
    for fl, hop, win in ((1024, 256, 1024), (800, 200, 800), (512, 128, 400)):
        y = stft_inputs(seed=fl, n=5000)
        for name, v in (("basis", torch.from_numpy(S.stft_forward_basis(fl, win))), ("mag", S.stft_magnitude(y, fl, hop, win))):
            key = "stft/%d/%s_" % (fl, name)
            assert tuple(v.shape) == tuple(int(x) for x in g[key + "shape"]), (fl, name)
            v = v.detach().double().reshape(-1)
            total, abs_total, sq, vmax = (float(x) for x in g[key + "stats"])
            ref = torch.from_numpy(g[key + "sample"])
            assert float((v[sample_index(v.numel(), 2048, fl)] - ref).abs().max()) / vmax < 1e-6, (fl, name)
            assert abs(float(v.abs().max()) - vmax) / vmax < 1e-6, (fl, name)
            assert abs(float(v.sum()) - total) / abs_total < 1e-6, (fl, name)
            assert abs(float(v.abs().sum()) - abs_total) / abs_total < 1e-6, (fl, name)
            assert abs(float((v * v).sum()) - sq) / sq < 1e-6, (fl, name)
