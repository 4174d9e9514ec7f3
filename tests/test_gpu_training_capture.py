"""The training calls allocate nothing, never wait on the host and keep no process-wide state.

Each training entry point -- the encoder and postnet forwards in training mode with a stash, the encoder, postnet, decoder
and prenet backward, and t2_mel_spectrogram -- is captured into a CUDA graph after one eager warm-up call, and the replay
must reproduce the eager outputs bit for bit (every output is zeroed between capture and replay; stashes and gradient
tables start zeroed, so bytes a call does not write compare equal).  A call that allocated, synchronised or copied from
pageable host memory would be refused by the capture.

With two devices, a backward pass and a mel spectrogram on cuda:1 after the same calls on cuda:0 in one process must equal
the same calls on cuda:1 in a process that never touched cuda:0."""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tacotron2_b200._engine import Engine
from tests.common import rand_text, synth_state_dict

pytestmark = pytest.mark.gpu
SEED = 0x5EED
HP = t2.create_hparams()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def engine(device="cuda"):
    eng = Engine(HP)
    eng.ensure({k: v.to(device) for k, v in synth_state_dict(seed=3, scale=2.0).items()})
    return eng


def randn(*shape, seed, scale=1.0, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(device)


def grad_table(eng, prefix):
    return {n: torch.zeros(shape, device=eng.device) for n, shape in eng.spec
            if n.startswith(prefix) and not n.endswith(("running_mean", "running_var", "num_batches_tracked"))}


def stash(eng, kind, *dims):
    return eng.stash_buffer(kind, *dims).zero_()


def replay_equals_eager(run):
    """run() enqueues one library call and returns the tensors it writes."""
    ref = [t.clone() for t in run()]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = run()
    for t in out:
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert len(out) == len(ref)
    for i, (a, b) in enumerate(zip(out, ref)):
        assert torch.equal(a, b), "output %d of the replay differs from the eager call" % i


# ---- calls ------------------------------------------------------------------------------------------------------------

def encoder_step(eng, text, d_memory):
    """Training forward with stash + backward; returns (memory, stash, grads)."""
    st = stash(eng, "encoder", *text.shape)
    memory = eng.encoder(text=text, training=True, stash=st, seed=SEED)
    grads = grad_table(eng, "encoder.")
    grads["embedding.weight"] = torch.zeros(148, 512, device=eng.device)
    eng.encoder_backward(text, None, None, True, None, SEED, st, d_memory, False, grads)
    return memory, st, grads


def mel_spectrogram(stft, y, out, ws):
    B, n = y.shape
    a = _capi.T2MelSpecArgs(y.data_ptr(), B, n, stft.filter_length, stft.hop_length, stft.n_mel_channels,
                            stft.forward_basis.data_ptr(), stft.mel_basis.data_ptr(), 1e-5, out.data_ptr(), ws.data_ptr(),
                            ws.numel())
    _capi.call(_capi.lib().t2_mel_spectrogram, y.device, C.byref(a))
    return out


def mel_buffers(stft, y):
    B, n = y.shape
    L = _capi.lib()
    out = torch.empty(B, stft.n_mel_channels, int(L.t2_mel_spectrogram_frames(n, stft.hop_length)), device=y.device)
    ws = _capi.byte_buffer(L.t2_mel_spectrogram_workspace_bytes(B, n, stft.filter_length, stft.hop_length,
                                                                stft.n_mel_channels), y.device)
    return out, ws


# ---- capture ----------------------------------------------------------------------------------------------------------

def test_encoder_forward_training_with_stash():
    eng, text = engine(), rand_text(3, 37, seed=1).cuda()
    st = stash(eng, "encoder", 3, 37)
    replay_equals_eager(lambda: [eng.encoder(text=text, training=True, stash=st, seed=SEED), st])


def test_postnet_forward_training_with_stash():
    eng, mel = engine(), randn(3, 37, 80, seed=2)
    st = stash(eng, "postnet", 3, 37)
    replay_equals_eager(lambda: [eng.postnet(mel, training=True, stash=st, seed=SEED), st])


def test_encoder_backward():
    eng, text, d_memory = engine(), rand_text(3, 37, seed=3).cuda(), randn(3, 37, 512, seed=4)
    _, st, grads = encoder_step(eng, text, d_memory)

    def run():
        d_emb = eng.encoder_backward(text, None, None, True, None, SEED, st, d_memory, True, grads)
        return [d_emb] + list(grads.values())
    replay_equals_eager(run)


def test_postnet_backward():
    eng, B, T = engine(), 3, 37
    mel, d_out = randn(B, T, 80, seed=5), randn(B, 80, T, seed=6)
    st = stash(eng, "postnet", B, T)
    eng.postnet(mel, training=True, stash=st, seed=SEED)
    grads = grad_table(eng, "postnet.")
    replay_equals_eager(lambda: [eng.postnet_backward(B, T, True, True, None, SEED, st, d_out, grads)] + list(grads.values()))


def test_decoder_backward():
    eng, B, Te, T = engine(), 3, 41, 6
    memory = randn(B, Te, 512, seed=7, scale=0.5)
    prenet = torch.relu(randn((T + 1) * B, 256, seed=8))
    d_mel, d_gate, d_align = randn(B, T, 80, seed=9), randn(B, T, seed=10), randn(B, T, Te, seed=11)
    st = stash(eng, "decoder", B, Te, T)
    _, _, align, _, _ = eng.decoder(memory, _capi.MODE_TEACHER, T, teacher_prenet=prenet, training=True,
                                    impl=_capi.IMPL_PERSISTENT, stash=st, seed=SEED)
    grads = grad_table(eng, "decoder.")

    def run():
        d_memory, d_prenet = eng.decoder_backward(memory, None, prenet, align, st, SEED, True, None, None, -float("inf"),
                                                  d_mel, d_gate, d_align, grads)
        return [d_memory, d_prenet] + list(grads.values())
    replay_equals_eager(run)


def test_prenet_backward():
    eng, M = engine(), 64 * 3
    frames, d_out = randn(M, 80, seed=12), randn(M, 256, seed=13)
    grads = grad_table(eng, "decoder.prenet.")
    replay_equals_eager(lambda: eng.prenet_backward(frames, None, SEED, d_out, grads) or list(grads.values()))


def test_mel_spectrogram():
    stft = t2.TacotronSTFT().cuda()
    y = torch.rand(2, 6000, generator=torch.Generator().manual_seed(14)).cuda() * 2 - 1
    out, ws = mel_buffers(stft, y)
    replay_equals_eager(lambda: [mel_spectrogram(stft, y, out, ws)])


# ---- two devices in one process -------------------------------------------------------------------------------------

def two_device_outputs(devices, path):
    """The encoder step and a mel spectrogram on each of `devices` in turn; saves the last device's outputs."""
    for dev in devices:
        torch.cuda.set_device(dev)
        eng = engine(dev)
        memory, _, grads = encoder_step(eng, rand_text(3, 37, seed=15).to(dev), randn(3, 37, 512, seed=16, device=dev))
        stft = t2.TacotronSTFT().to(dev)
        y = (torch.rand(2, 6000, generator=torch.Generator().manual_seed(17)) * 2 - 1).to(dev)
        mel = stft.mel_spectrogram(y)
        torch.cuda.synchronize(dev)
    torch.save([memory.cpu(), mel.cpu()] + [g.cpu() for g in grads.values()], path)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_second_device_equals_a_process_that_only_used_it(tmp_path):
    def run(devices, name):
        path = str(tmp_path / name)
        code = "from tests.test_gpu_training_capture import two_device_outputs; two_device_outputs(%r, %r)" % (devices, path)
        subprocess.run([sys.executable, "-c", code], cwd=ROOT, check=True)
        return torch.load(path)
    both, alone = run(["cuda:0", "cuda:1"], "both.pt"), run(["cuda:1"], "alone.pt")
    assert len(both) == len(alone)
    for i, (a, b) in enumerate(zip(both, alone)):
        assert torch.equal(a, b), "output %d on cuda:1 depends on the earlier calls on cuda:0" % i
