"""Every entry point that takes a caller buffer (workspace, stash, stream state) stays inside the byte count its size query
reports, whatever the buffer's alignment.

Each case runs twice on the same inputs: once with the buffers the engine allocates itself, once with every such buffer
sized exactly as its query reports and placed 256 bytes past a 512-byte boundary, between 64 KiB canaries of a seeded
byte pattern (the buffer itself starts out filled with the pattern too).  The canaries must be intact afterwards and the
outputs bit-identical to the first run.  The cases sit on the layout edges: one row / one frame, more than 64 rows, the
decoder's shared-memory regimes (T_enc 94 / 95, 896 / 897, 2274), the stepwise decoder's longest memory, the backward
passes."""
import contextlib
from unittest import mock

import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tacotron2_b200._engine import Engine
from tests.common import rand_text, synth_state_dict

pytestmark = pytest.mark.gpu
CANARY = 64 * 1024
SEED = 0x5EED
HP = t2.create_hparams()


def pattern(n):
    g = torch.Generator(device="cuda").manual_seed(77)
    return torch.randint(0, 256, (n,), generator=g, dtype=torch.uint8, device="cuda")


class Placed:
    """Hands out exact-size buffers at 256 mod 512 between canaries, and checks the canaries."""

    def __init__(self):
        self.raw = []

    def empty(self, n):
        raw = pattern(2 * CANARY + 256 + n)
        assert raw.data_ptr() % 512 == 0
        self.raw.append((raw, n))
        return raw[CANARY + 256:CANARY + 256 + n]

    def check(self):
        torch.cuda.synchronize()
        assert self.raw, "no caller buffer was placed"
        for raw, n in self.raw:
            ref, lo = pattern(raw.numel()), CANARY + 256
            assert torch.equal(raw[:lo], ref[:lo]), "canary before a %d-byte buffer overwritten" % n
            assert torch.equal(raw[lo + n:], ref[lo + n:]), "canary after a %d-byte buffer overwritten" % n


@contextlib.contextmanager
def placed_buffers():
    """Routes the library's byte buffers (torch.empty(n, dtype=uint8, device=...) in the engine, the optimizers, the loss and
    the STFT) through Placed, and stops the engine from reusing a larger cached workspace."""
    p, real = Placed(), torch.empty

    def empty(*size, dtype=None, device=None, **kw):
        if dtype is torch.uint8 and device is not None and len(size) == 1 and isinstance(size[0], int) and not kw:
            return p.empty(size[0])
        return real(*size, dtype=dtype, device=device, **kw)

    with mock.patch.object(torch, "empty", empty), \
            mock.patch.object(Engine, "_workspace", lambda self, tag, n: torch.empty(int(n), dtype=torch.uint8, device=self.device)):
        yield p
    p.check()


def engine():
    """A fresh handle on fresh weight copies: training forwards update the BatchNorm running statistics in place."""
    eng = Engine(HP)
    eng.ensure({k: v.cuda() for k, v in synth_state_dict(seed=3, scale=2.0).items()})
    return eng


def same_both_ways(run):
    ref = [t.clone() for t in run(engine())]
    torch.cuda.synchronize()
    with placed_buffers():
        out = run(engine())
        torch.cuda.synchronize()
    assert len(out) == len(ref)
    for i, (a, b) in enumerate(zip(out, ref)):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), "output %d differs" % i


def randn(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


def grad_table(eng, prefix):
    return {n: torch.zeros(shape, device="cuda") for n, shape in eng.spec
            if n.startswith(prefix) and not n.endswith(("running_mean", "running_var", "num_batches_tracked"))}


# ---- forward passes ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["infer", "train", "stash"])
@pytest.mark.parametrize("B,T", [(1, 1), (3, 37), (64, 150), (65, 150)])
def test_encoder(B, T, mode):
    if mode == "stash" and B > 64:
        pytest.skip("the training stash takes at most 64 rows")
    text = rand_text(B, T, seed=B * 1000 + T).cuda()

    def run(eng):
        stash = eng.stash_buffer("encoder", B, T) if mode == "stash" else None
        return [eng.encoder(text=text, training=mode != "infer", stash=stash, seed=SEED)]
    same_both_ways(run)


@pytest.mark.parametrize("mode", ["infer", "train", "stash"])
@pytest.mark.parametrize("B,T", [(1, 1), (3, 1), (3, 37), (64, 150), (65, 150)])
def test_postnet(B, T, mode):
    if mode == "stash" and B > 64:
        pytest.skip("the training stash takes at most 64 rows")
    mel = randn(B, T, 80, seed=B * 1000 + T)

    def run(eng):
        stash = eng.stash_buffer("postnet", B, T) if mode == "stash" else None
        return [eng.postnet(mel, training=mode != "infer", stash=stash, seed=SEED)]
    same_both_ways(run)


@pytest.mark.parametrize("impl,Te", [(_capi.IMPL_PERSISTENT, 94), (_capi.IMPL_PERSISTENT, 95), (_capi.IMPL_PERSISTENT, 896),
                                     (_capi.IMPL_PERSISTENT, 897), (_capi.IMPL_PERSISTENT, 2274), (_capi.IMPL_STEPWISE, 1282)])
@pytest.mark.parametrize("B", [1, 65])
def test_decoder_inference(B, Te, impl):
    memory = randn(B, Te, 512, seed=Te, scale=0.5)

    def run(eng):
        return list(eng.decoder(memory, _capi.MODE_INFER, 4, impl=impl, gate_threshold=0.5, seed=SEED))
    same_both_ways(run)


def test_decoder_stream():
    B, Te = 65, 95
    memory = randn(B, Te, 512, seed=9, scale=0.5)

    def run(eng):
        s = eng.decoder_stream(memory, 8, impl=_capi.IMPL_PERSISTENT, seed=SEED)
        for n in (3, 2, 4):
            s.run(n)
        return [s.mel, s.gate, s.align, s.mel_lengths, s.n_steps, s.status]
    same_both_ways(run)


def test_infer_host():
    text = rand_text(3, 23, seed=5).pin_memory()

    def run(eng):
        return [t.clone() for t in eng.infer_host(text, 6, seed=SEED)]
    same_both_ways(run)


# ---- backward passes --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("Te", [95, 408])
def test_decoder_teacher_stash_and_backward(Te):
    B, T = 64, 5
    memory = randn(B, Te, 512, seed=Te, scale=0.5)
    prenet = torch.relu(randn((T + 1) * B, 256, seed=Te + 1))
    d_mel, d_gate, d_align = randn(B, T, 80, seed=1), randn(B, T, seed=2), randn(B, T, Te, seed=3)

    def run(eng):
        stash = eng.decoder_stash(B, Te, T)
        mel, gate, align, lens, n = eng.decoder(memory, _capi.MODE_TEACHER, T, teacher_prenet=prenet, training=True,
                                                impl=_capi.IMPL_PERSISTENT, stash=stash, seed=SEED)
        grads = grad_table(eng, "decoder.")
        d_memory, d_prenet = eng.decoder_backward(memory, None, prenet, align, stash, SEED, True, None, None, -float("inf"),
                                                  d_mel, d_gate, d_align, grads)
        return [mel, gate, align, lens, n, d_memory, d_prenet] + list(grads.values())
    same_both_ways(run)


def test_encoder_backward():
    B, T = 64, 37
    text = rand_text(B, T, seed=11).cuda()
    d_memory = randn(B, T, 512, seed=12)

    def run(eng):
        stash = eng.stash_buffer("encoder", B, T)
        memory = eng.encoder(text=text, training=True, stash=stash, seed=SEED)
        grads = grad_table(eng, "encoder.")
        grads["embedding.weight"] = torch.zeros(148, 512, device="cuda")
        d_emb = eng.encoder_backward(text, None, None, True, None, SEED, stash, d_memory, False, grads)
        assert d_emb is None
        return [memory] + list(grads.values())
    same_both_ways(run)


def test_postnet_backward():
    B, T = 64, 37
    mel = randn(B, T, 80, seed=13)
    d_out = randn(B, 80, T, seed=14)

    def run(eng):
        stash = eng.stash_buffer("postnet", B, T)
        out = eng.postnet(mel, training=True, stash=stash, seed=SEED)
        grads = grad_table(eng, "postnet.")
        d_mel = eng.postnet_backward(B, T, True, True, None, SEED, stash, d_out, grads)
        return [out, d_mel] + list(grads.values())
    same_both_ways(run)


def test_prenet_backward():
    M = 64 * 6
    frames, d_out = randn(M, 80, seed=15), randn(M, 256, seed=16)

    def run(eng):
        grads = grad_table(eng, "decoder.prenet.")
        eng.prenet_backward(frames, None, SEED, d_out, grads)
        return list(grads.values())
    same_both_ways(run)


# ---- optimizers, loss, mel spectrogram --------------------------------------------------------------------------------

def test_clip_adam():
    shapes = [(7,), (129, 3), (65537,), (80, 512, 5)]

    def run(_):
        params = [torch.nn.Parameter(randn(*s, seed=i)) for i, s in enumerate(shapes)]
        opt = t2.FusedClipAdam(params, lr=1e-3, weight_decay=1e-6)
        norms = []
        for it in range(2):
            for i, p in enumerate(params):
                p.grad = randn(*p.shape, seed=100 * it + i)
            norms.append(torch.tensor([float(opt.step(max_norm=1.0))]))
        return [p.detach() for p in params] + norms
    same_both_ways(run)


def test_amp_adam():
    shapes, halfs = [(257, 33), (4096,), (5, 7, 3)], [True, False, True]

    def run(_):
        params = [torch.nn.Parameter(randn(*s, seed=i, scale=0.1).to(torch.half if h else torch.float))
                  for i, (s, h) in enumerate(zip(shapes, halfs))]
        opt = t2.AmpFusedClipAdam(params, lr=1e-2, init_scale=1024.0)
        for it in range(2):
            for i, p in enumerate(params):
                p.grad = (randn(*p.shape, seed=100 * it + i) * 1024.0).to(p.dtype)
            opt.step(max_norm=0.5)
        return [p.detach() for p in params] + [m.detach() for m in opt.master_params()]
    same_both_ways(run)


def test_loss():
    B, T = 5, 41

    def run(_):
        mel, post = randn(B, 80, T, seed=1).requires_grad_(), randn(B, 80, T, seed=2).requires_grad_()
        gate = randn(B, T, seed=3).requires_grad_()
        loss = t2.Tacotron2Loss()((mel, post, gate, None), (randn(B, 80, T, seed=4), (randn(B, T, seed=5) > 0).float()))
        loss.backward()
        return [loss.detach(), mel.grad, post.grad, gate.grad]
    same_both_ways(run)


def test_mel_spectrogram():
    y = torch.rand(2, 6000, generator=torch.Generator().manual_seed(6)).cuda() * 2 - 1

    def run(_):
        return [t2.TacotronSTFT().cuda().mel_spectrogram(y)]
    same_both_ways(run)
