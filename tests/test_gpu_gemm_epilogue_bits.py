"""Bit-exactness of every wg_gemm instantiation that tests/golden/waveglow_published_sha256.json does not pin (that
file covers WaveGlow and the denoiser): the Tacotron2 conv epilogue in inference and training, HiFi-GAN's in both
tiers and all three column tilings, the public STFT transform and Griffin-Lim's projection.

The digests in tests/golden/gemm_epilogue_sha256.json were recorded with tools/gemm_epilogue_digests.py on the build
before the GEMM epilogues moved out of wg_gemm.cuh into their callers' files; a later build must reproduce them bit for
bit."""
import json
import os

import numpy as np
import pytest
import torch

from tests.common import GOLDEN_DIR, keep_mask, rand_text, stft_inputs, synth_state_dict, tensor_digest

pytestmark = pytest.mark.gpu


def digests():
    """{case: tensor_digest} of outputs that reach each instantiation.  The same code runs on the build that recorded
    the digests and on later builds."""
    import tacotron2_b200 as t2
    from tacotron2_b200.audio_processing import _griffin_lim
    from oracle import denoiser_oracle as D
    from tests.hifigan_common import mel_input, model
    from tests.test_oracle_golden import grad_inputs, load

    out = {}
    # Tacotron2 encoder and postnet in inference, ragged: conv k5 (128 x 2), the LSTM input projection (128 x 2) and
    # the postnet's last conv (80 x 1)
    hp = t2.create_hparams()
    m = t2.Tacotron2(hp)
    m.load_state_dict(synth_state_dict(5, gate_bias=-10.0, scale=2.0))
    m = m.cuda().eval()
    m.decoder.max_decoder_steps = 40
    text, lengths = rand_text(3, 37, 21), [37, 20, 6]
    with torch.no_grad():
        emb = m.embedding(text.cuda()).transpose(1, 2)
        out["t2/encoder_ragged"] = tensor_digest(m.encoder.inference(emb, torch.tensor(lengths)))
        with t2.dropout_masks(prenet=keep_mask((40, 2, 3, 256), 0.5, 22)):
            res = m.inference(text.cuda(), input_lengths=lengths)
        out["t2/inference_ragged_mel_postnet"] = tensor_digest(res[1])
        out["t2/inference_ragged_mel_lengths"] = tensor_digest(m.mel_lengths)

    # a teacher-forced training step: encoder and postnet forwards on the training conv stack, and their conv input
    # gradients
    sd, text, tl, ol, mels, gt, mk = grad_inputs(load("grad_train_b4"))
    m = t2.Tacotron2(hp)
    m.load_state_dict(sd)
    m = m.cuda().train()
    post_keep = [mk["qk4"][i] for i in range(4)] + [mk["qk1"]]
    with t2.dropout_masks(prenet=mk["pk"], att=mk["ak"], dec=mk["dk"], enc=mk["ek"], post=post_keep):
        res = m((text.cuda(), tl.cuda(), mels.cuda(), int(tl.max()), ol.cuda()))
        t2.Tacotron2Loss()(res, (mels.cuda(), gt.cuda())).backward()
    for k, p in m.named_parameters():
        if k.startswith(("embedding.", "encoder.convolutions.", "postnet.")):
            out["t2/train_grad/" + k] = tensor_digest(p.grad)
    out["t2/train_mel_postnet"] = tensor_digest(res[1])

    # HiFi-GAN V1 (128 x 2), V2 (64 x 1 and 128 x 1) and V3 in both tiers, ragged
    with torch.no_grad():
        for name in ("v1", "v2", "v3"):
            for half in (False, True):
                G = model(name).cuda().eval()
                if half:
                    G = G.half()
                mel = mel_input(3, 40, 23).to(G.conv_pre.bias.dtype).cuda()
                y = G(mel, lengths=torch.tensor([40, 23, 7]).cuda())
                out["hifigan/%s_%s_ragged" % (name, "fp16" if half else "fp32")] = tensor_digest(y)

    # STFT.transform (magnitude and phase) and a few Griffin-Lim iterations (the projection), ragged
    st = t2.TacotronSTFT().cuda().stft_fn
    n = 256 * 30 + 40
    y = torch.randn(3, n, generator=torch.Generator().manual_seed(24)) * 0.3
    mag, phase = st.transform(y.cuda(), lengths=torch.tensor([n, 256 * 17 + 5, 2000]))
    out["stft/transform_mag"] = tensor_digest(mag)
    out["stft/transform_phase"] = tensor_digest(phase)
    target, _ = D.transform(stft_inputs(25, 256 * 30), torch.float32)
    target = target.float()
    ang = (torch.rand(target.shape, generator=torch.Generator().manual_seed(26)) * 2 - 1) * np.pi
    F = target.shape[-1]
    audio = _griffin_lim(target.cuda(), ang.float().cuda(), st, 4, lengths=torch.tensor([F, 17]))
    out["griffin_lim/4_iters_ragged"] = tensor_digest(audio)
    torch.cuda.synchronize()
    return out


def test_gemm_epilogue_outputs_are_unchanged():
    with open(os.path.join(GOLDEN_DIR, "gemm_epilogue_sha256.json")) as f:
        want = json.load(f)["digests"]
    got = digests()
    assert sorted(got) == sorted(want)
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, bad
