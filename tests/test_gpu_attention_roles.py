"""The persistent decoder's CTA roles: CTA b + 64 runs the attention of batch row b (energies, softmax, alignment row, all 512
context columns) while CTA b streams the deferred W_hh^a . ah products of both CTAs (event Ed) and hands its partner's sums
over through a per-slice buffer.

The split moves work between SMs but keeps every sum in its order, so the outputs are bit-identical to those of the layout
in which both CTAs of a pair ran the attention and split the context.  Each case is checked twice:
  - against the float64 oracle (max|a - b| / max|b| < 1e-4 on mel, gate and alignments; the backward's gradients keep the
    1e-3 bar of tests/test_gpu_backward.py);
  - against the SHA-256 digest of the same outputs from the earlier layout, in tests/golden/attention_roles_sha256.json.

Cases: B = 1, 37 and 64 (below 64 rows some CTA pairs have no row, but their lower CTA still runs Ed for its partner's
units), the 3-stage ring (T_enc = 897), a stream resumed every 3 steps, and a teacher-forced training forward whose stash
(which carries the context of every step) feeds the backward."""
import functools
import hashlib
import json
import os

import pytest
import torch

import tacotron2_b200 as t2
from oracle import tacotron2_oracle as O
from tests.common import keep_mask, rel_err, synth_state_dict

pytestmark = pytest.mark.gpu

TOL = 1e-4
GRAD_TOL = 1e-3
STEPS = 7
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "attention_roles_sha256.json")

INFER_CASES = {  # name: (B, T_enc)
    "free_B1_T37": (1, 37),
    "free_B37_T150": (37, 150),
    "free_B64_T150": (64, 150),
    "free_B3_T897_3stages": (3, 897),
}
STREAM_CASE = ("stream_B37_T150_chunk3", 37, 150, 3)
TEACHER_CASE = ("teacher_B4_T40", 4, 40, 6)


@functools.lru_cache(maxsize=None)
def weights():
    sd = synth_state_dict(41, scale=2.0)
    return sd, {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}


_models = {}


def model(train=False):
    if train not in _models:
        m = t2.Tacotron2(t2.create_hparams())
        m.load_state_dict(weights()[0])
        _models[train] = m.cuda().train() if train else m.cuda().eval()
    return _models[train]


def inputs(B, T):
    g = torch.Generator().manual_seed(7 * B + T)
    return torch.randn(B, T, 512, generator=g), keep_mask((STEPS, 2, B, 256), 0.5, B + T)


def digest(tensors):
    h = hashlib.sha256()
    for x in tensors:
        h.update(x.detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()


def golden(name):
    with open(GOLDEN) as f:
        return json.load(f)[name]


def infer_outputs(B, T):
    dec = model().decoder
    dec.max_decoder_steps, dec.gate_threshold = STEPS, 1.0
    memory, keep = inputs(B, T)
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        mel, gate, align = dec.inference(memory.cuda())
    torch.cuda.synchronize()
    return [mel.cpu(), gate.cpu(), align.cpu(), dec.mel_lengths.cpu()]


def stream_outputs(B, T, chunk):
    dec = model().decoder
    dec.max_decoder_steps, dec.gate_threshold = STEPS, 1.0
    memory, keep = inputs(B, T)
    items = []
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        for it in dec.inference_stream(memory.cuda(), chunk_steps=chunk):
            items.append({k: (v.cpu() if torch.is_tensor(v) else v) for k, v in it.items()})
    torch.cuda.synchronize()
    assert len(items) > 1 and items[-1]["finished"]
    return [torch.cat([it["mel_outputs"] for it in items], 2), torch.cat([it["gate_outputs"] for it in items], 1),
            torch.cat([it["alignments"] for it in items], 1), items[-1]["mel_lengths"]]


def teacher_case(B, Te, T):
    g = torch.Generator().manual_seed(11)
    memory = torch.randn(B, Te, 512, generator=g)
    mels = torch.randn(B, 80, T, generator=g)
    lens = torch.tensor([Te] + [Te - 3 * i for i in range(1, B)])
    d_mel, d_gate = torch.randn(B, 80, T, generator=g), torch.randn(B, T, generator=g)
    pk = keep_mask((T + 1, 2, B, 256), 0.5, 1)
    ak, dk = keep_mask((T, B, 1024), 0.1, 2), keep_mask((T, B, 1024), 0.1, 3)
    return memory, mels, lens, d_mel, d_gate, pk, ak, dk


def teacher_outputs(B, Te, T):
    dec = model(train=True).decoder
    memory, mels, lens, d_mel, d_gate, pk, ak, dk = teacher_case(B, Te, T)
    for p in dec.parameters():
        p.grad = None
    mem = memory.cuda().requires_grad_(True)
    with t2.dropout_masks(prenet=pk, att=ak, dec=dk):
        mel, gate, align = dec(mem, mels.cuda(), lens.cuda())
        ((mel * d_mel.cuda()).sum() + (gate * d_gate.cuda()).sum()).backward()
    torch.cuda.synchronize()
    return [mel.detach().cpu(), gate.detach().cpu(), align.detach().cpu(), mem.grad.cpu()] + \
        [p.grad.cpu() for p in dec.parameters()]


def oracle_infer(B, T):
    memory, keep = inputs(B, T)
    with torch.no_grad():
        mel, gate, align, lengths = O.decoder_inference(weights()[1], memory.double(), keep, 1.0, STEPS)
    return (mel, gate, align), lengths


def all_digests():
    """Every case's digest; tests/golden/attention_roles_sha256.json holds these from the earlier layout."""
    out = {name: digest(infer_outputs(B, T)) for name, (B, T) in INFER_CASES.items()}
    name, B, T, chunk = STREAM_CASE
    out[name] = digest(stream_outputs(B, T, chunk))
    name, B, Te, T = TEACHER_CASE
    out[name] = digest(teacher_outputs(B, Te, T))
    return out


@pytest.mark.parametrize("name", list(INFER_CASES))
def test_inference_matches_oracle_and_earlier_layout(name):
    B, T = INFER_CASES[name]
    out = infer_outputs(B, T)
    ref, ref_lengths = oracle_infer(B, T)
    errs = {k: rel_err(a, b) for k, a, b in zip(("mel", "gate", "align"), out[:3], ref)}
    print("%s: %s" % (name, ", ".join("%s %.2e" % kv for kv in errs.items())))
    assert out[3].tolist() == ref_lengths.tolist() == [STEPS] * B
    assert max(errs.values()) < TOL, errs
    assert digest(out) == golden(name)


def test_resumed_stream_matches_whole_run_and_earlier_layout():
    name, B, T, chunk = STREAM_CASE
    out = stream_outputs(B, T, chunk)
    whole = infer_outputs(B, T)
    assert all(torch.equal(a.reshape(b.shape), b) for a, b in zip(out[:3], whole[:3]))
    assert out[3].tolist() == whole[3].tolist()
    assert digest(out) == golden(name)


def test_teacher_stash_backward_matches_oracle_and_earlier_layout():
    from tests.test_gpu_backward import oracle_decoder_grads
    from tests.test_gpu_train_regimes import to64
    name, B, Te, T = TEACHER_CASE
    out = teacher_outputs(B, Te, T)
    memory, mels, lens, d_mel, d_gate, pk, ak, dk = teacher_case(B, Te, T)
    sd = {k: v.cpu() for k, v in model(train=True).state_dict().items()}
    _, ref, ref_dmem = oracle_decoder_grads(to64(sd, "cpu"), memory.double(), mels.double(), lens, pk, ak, dk,
                                            d_mel.double(), d_gate.double(), None, True)
    names = [k for k, _ in model(train=True).decoder.named_parameters()]
    errs = {"d_memory": rel_err(out[3], ref_dmem)}
    errs.update({n: rel_err(g, ref["decoder." + n]) for n, g in zip(names, out[4:])})
    worst = max(errs, key=errs.get)
    print("%s: worst gradient error %.2e (%s)" % (name, errs[worst], worst))
    assert errs[worst] < GRAD_TOL, errs
    assert digest(out) == golden(name)
