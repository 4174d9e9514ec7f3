"""Continuous batching (``Tacotron2.inference_server``): with injected prenet masks every served request equals, bit for
bit, the same model's ``inference(text[None])`` under the request's own step limit and masks -- whatever the slot count,
the chunk size, the order of submission, what shared the batch with it and at which step it was admitted."""
import pytest
import torch

import tacotron2_b200 as t2
from oracle import tacotron2_oracle as O
from tacotron2_b200 import _engine
from tests.common import keep_mask, rand_text, rel_err, synth_state_dict, tensor_digest
from tests.test_gpu_buffer_bounds import placed_buffers
from tests.test_oracle_golden import infer_inputs, load

pytestmark = pytest.mark.gpu
S = 48              # the longest step limit of a request
T_CAP = 150         # max_text_len: spans the decoder's staging regimes (94 / 95)
NAMES = ("mel_outputs", "mel_outputs_postnet", "gate_outputs", "alignments")


def make_model(sd, threshold=0.5, half=False):
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    model = model.cuda().eval()
    if half:
        model = model.half()
    model.decoder.gate_threshold = threshold
    return model


class Req:
    def __init__(self, i, length, limit):
        self.text = rand_text(1, length, 1000 + i)[0]
        self.keep = keep_mask((S, 2, 256), 0.5, 2000 + i)
        self.limit = limit


def requests(n=40):
    lengths = [1, T_CAP, 95, 94, 37, 3, 120, 60]
    g = torch.Generator().manual_seed(5)
    lengths += torch.randint(1, T_CAP + 1, (max(0, n - len(lengths)),), generator=g).tolist()
    return [Req(i, lengths[i], (5, 17)[i // 5 % 2] if i % 5 == 4 else S) for i in range(n)]


def alone(model, r):
    """inference(text[None]) under the request's own limit and masks: (outputs, length)."""
    model.decoder.max_decoder_steps = r.limit
    with torch.no_grad(), t2.dropout_masks(prenet=r.keep[:r.limit, :, None].contiguous()):
        out = [o.clone() for o in model.inference(r.text[None].cuda())]
    return out, int(model.mel_lengths[0])


def pick_threshold(model, reqs):
    """A gate threshold under which the requests stop at different steps (the gate is not fed back, so the logits of a run
    in which nothing stops do not depend on it): the median of the running maximum of the logits at a third of S."""
    model.decoder.gate_threshold = 1.0
    peak = []
    for r in reqs[:12]:
        (_, _, gate, _), _ = alone(model, _with_limit(r, S))
        peak.append(float(torch.cummax(gate[0, :, 0].float().cpu(), 0).values[S // 3]))
    return float(torch.sigmoid(torch.tensor(peak).median()))


def _with_limit(r, limit):
    c = Req.__new__(Req)
    c.text, c.keep, c.limit = r.text, r.keep, limit
    return c


def serve(model, reqs, slots, chunk, order=None, masks=True, **kw):
    server = model.inference_server(slots=slots, max_text_len=T_CAP, chunk_steps=chunk, **kw)
    order = list(range(len(reqs))) if order is None else order
    ids = {server.submit(reqs[i].text, reqs[i].limit, prenet_keep=reqs[i].keep if masks else None): i for i in order}
    with torch.no_grad():
        out = {ids[res["id"]]: res for res in server.run()}
    assert sorted(out) == sorted(order) and server.idle()
    return out, server


def check(res, ref, T_text):
    out, L = ref
    assert res["mel_length"] == L
    for name, o in zip(NAMES, out):
        assert res[name].dtype == o.dtype and res[name].shape == o.shape, name
        assert torch.equal(res[name], o), name
    assert res["alignments"].shape == (1, L, T_text) and res["gate_outputs"].shape == (1, L, 1)


_cache = {}


def fixture(half):
    """(model, requests, their B = 1 references), built once per dtype."""
    if half not in _cache:
        model = make_model(synth_state_dict(7, gate_bias=0.0, gate_sign=10.0, scale=2.0), half=half)
        reqs = requests()
        thr = pick_threshold(model, reqs)
        model.decoder.gate_threshold = thr
        refs = [alone(model, r) for r in reqs]
        print("half=%s threshold %.4f lengths %s" % (half, thr, [L for _, L in refs]))
        assert len({L for _, L in refs}) > 5 and min(L for _, L in refs) < S
        _cache[half] = (model, reqs, refs)
    return _cache[half]


@pytest.mark.parametrize("chunk", [1, 7, 32])
@pytest.mark.parametrize("half", [False, True], ids=["fp32", "half"])
def test_every_request_equals_its_own_b1_inference(half, chunk):
    model, reqs, refs = fixture(half)
    out, server = serve(model, reqs, 8, chunk)
    for i, r in enumerate(reqs):
        check(out[i], refs[i], r.text.numel())
        assert out[i]["hit_max_steps"] == (refs[i][1] == r.limit and
                                           not bool(torch.sigmoid(refs[i][0][2][0, -1, 0].float()) > model.decoder.gate_threshold))
    assert server.row_steps >= sum(L for _, L in refs)


@pytest.mark.parametrize("slots", [1, 8, 70])
def test_other_submission_order_and_slot_counts_give_the_same_bits(slots):
    model, reqs, refs = fixture(False)
    n = 12 if slots == 1 else len(reqs)
    order = list(reversed(range(n)))
    out, _ = serve(model, reqs, slots, 7, order)
    for i in order:
        check(out[i], refs[i], reqs[i].text.numel())


def test_a_refilled_slot_is_reset_completely_and_its_neighbours_are_untouched():
    """Slot 1's first occupant is the longest text and runs to its limit; the one-symbol text that follows it there, and
    the neighbours that were mid-flight while the slot was reset, equal their own runs."""
    model, reqs, refs = fixture(False)
    thr = model.decoder.gate_threshold
    try:
        model.decoder.gate_threshold = 1.0                  # nothing fires: the lengths are the limits
        long_, short, left, right = (_with_limit(reqs[1], 20), _with_limit(reqs[0], 9), _with_limit(reqs[2], 33),
                                     _with_limit(reqs[6], 31))
        rs = [left, long_, right, short]
        server = model.inference_server(slots=3, max_text_len=T_CAP, chunk_steps=5)
        for r in rs:
            server.submit(r.text, r.limit, prenet_keep=r.keep)
        out = {}
        with torch.no_grad():
            while not server.idle():
                for res in server.step():
                    out[res["id"]] = res
                if 3 not in out and server.chunks == 5:     # after chunk 4 the long request has left slot 1
                    assert server.table[1] is not None and server.table[1].id == 3
                    assert server.table[0].id == 0 and server.table[2].id == 2
        for i, r in enumerate(rs):
            check(out[i], alone(model, r), r.text.numel())
            assert out[i]["hit_max_steps"]
    finally:
        model.decoder.gate_threshold = thr


def test_a_requests_own_limit_and_its_one_warning(capsys):
    model, reqs, _ = fixture(False)
    thr = model.decoder.gate_threshold
    try:
        model.decoder.gate_threshold = 1.0
        rs = [_with_limit(reqs[4], 11), _with_limit(reqs[5], 4)]
        refs = [alone(model, r) for r in rs]
        capsys.readouterr()
        out, _ = serve(model, rs, 2, 8)
        assert capsys.readouterr().out.count("Warning! Reached max decoder steps") == 2
        for i, r in enumerate(rs):
            check(out[i], refs[i], r.text.numel())
            assert out[i]["hit_max_steps"] and out[i]["mel_length"] == r.limit
    finally:
        model.decoder.gate_threshold = thr


def test_first_step_firing_late_submission_and_more_slots_than_requests():
    model = make_model(synth_state_dict(9, gate_bias=10.0, scale=2.0))      # every gate fires on the first step
    reqs = requests(6)
    refs = [alone(model, r) for r in reqs]
    assert all(L == 1 for _, L in refs)
    out, server = serve(model, reqs[:3], 8, 4)
    for i in range(3):
        check(out[i], refs[i], reqs[i].text.numel())
        assert not out[i]["hit_max_steps"]
    assert server.chunks == 1
    # a request submitted while others are mid-flight
    model2, reqs2, refs2 = fixture(False)
    server = model2.inference_server(slots=4, max_text_len=T_CAP, chunk_steps=3)
    ids = {server.submit(reqs2[i].text, reqs2[i].limit, prenet_keep=reqs2[i].keep): i for i in (6, 7)}
    got = {}
    with torch.no_grad():
        got.update({ids[r["id"]]: r for r in server.step()})
        ids[server.submit(reqs2[0].text, reqs2[0].limit, prenet_keep=reqs2[0].keep)] = 0
        got.update({ids[r["id"]]: r for r in server.step()})
        ids[server.submit(reqs2[3].text, reqs2[3].limit, prenet_keep=reqs2[3].keep)] = 3
        got.update({ids[r["id"]]: r for r in server.run()})
    for i in (6, 7, 0, 3):
        check(got[i], refs2[i], reqs2[i].text.numel())


def test_two_servers_and_a_stream_interleaved_on_one_model():
    model, reqs, refs = fixture(False)
    a = model.inference_server(slots=3, max_text_len=T_CAP, chunk_steps=4)
    b = model.inference_server(slots=2, max_text_len=T_CAP, chunk_steps=9)
    ia = {a.submit(reqs[i].text, reqs[i].limit, prenet_keep=reqs[i].keep): i for i in range(0, 8)}
    ib = {b.submit(reqs[i].text, reqs[i].limit, prenet_keep=reqs[i].keep): i for i in range(8, 14)}
    text, keep = rand_text(2, 30, 77), keep_mask((S, 2, 2, 256), 0.5, 78)
    model.decoder.max_decoder_steps = S
    with torch.no_grad(), t2.dropout_masks(prenet=keep):
        whole = [o.clone() for o in model.inference(text.cuda())]
    ga, gb, items = {}, {}, []
    with torch.no_grad():
        with t2.dropout_masks(prenet=keep):
            stream = model.inference_stream(text.cuda(), chunk_steps=5)
            while not (a.idle() and b.idle() and stream is None):
                ga.update({ia[r["id"]]: r for r in a.step()})
                if stream is not None:
                    item = next(stream, None)
                    if item is None:
                        stream = None
                    else:
                        items.append(item)
                gb.update({ib[r["id"]]: r for r in b.step()})
    for i in range(0, 8):
        check(ga[i], refs[i], reqs[i].text.numel())
    for i in range(8, 14):
        check(gb[i], refs[i], reqs[i].text.numel())
    for k, name in enumerate(NAMES):
        assert torch.equal(torch.cat([it[name] for it in items], dim=1 if k >= 2 else 2), whole[k]), name


def test_inference_is_unchanged_by_a_server_on_the_same_model():
    g = load("infer_b4_t24")
    sd, text, keep, steps = infer_inputs(g)
    model = make_model(sd)
    model.decoder.max_decoder_steps = steps

    def digests():
        with torch.no_grad(), t2.dropout_masks(prenet=keep):
            out = model.inference(text.cuda())
        return [tensor_digest(o) for o in out] + [tensor_digest(model.mel_lengths)]
    before = digests()
    reqs = requests(10)
    serve(model, reqs, 4, 6)
    model.decoder.max_decoder_steps = steps
    assert digests() == before


def test_guard_bands_around_state_chunk_and_output_buffers():
    model, reqs, refs = fixture(False)
    with placed_buffers():
        out, _ = serve(model, reqs[:20], 70, 7)
        out = {i: {k: (v.clone() if torch.is_tensor(v) else v) for k, v in r.items()} for i, r in out.items()}
        torch.cuda.synchronize()
    for i in range(20):
        check(out[i], refs[i], reqs[i].text.numel())


def test_bad_rows_are_refused_before_any_launch():
    model, reqs, _ = fixture(False)
    server = model.inference_server(slots=3, max_text_len=T_CAP, chunk_steps=4)
    st = server.backend.stream
    launches = t2._capi.lib().t2_kernel_launch_count()
    for rows in ([3], [-1], [1, 1], [2, 0]):
        with pytest.raises(t2._capi.T2Error, match="admit"):
            st.admit(rows)
    buf = torch.zeros(5 * 80, device="cuda")
    for entry in ((3, 1, 4, buf, buf, buf), (0, 6, 4, buf, buf, buf), (0, 1, T_CAP + 1, buf, buf, buf), (0, 1, 0, buf, buf, buf)):
        with pytest.raises(t2._capi.T2Error, match="collect"):
            st.collect([entry])
    assert t2._capi.lib().t2_kernel_launch_count() == launches


def test_one_served_request_against_the_fp64_oracle():
    sd = synth_state_dict(105, gate_bias=-10.0, scale=2.0)
    model = make_model(sd)
    r = Req(3, 37, 9)
    with torch.no_grad():
        ref = O.tacotron2_inference(sd, r.text[None], r.keep[:9, :, None].contiguous(), 0.5, 9)
    out, _ = serve(model, [r, Req(4, 20, 6)], 2, 4)
    assert out[0]["mel_length"] == int(ref[4][0])
    for name, b in zip(NAMES, ref[:4]):
        assert rel_err(out[0][name], b) < 1e-3, name


def test_philox_path_runs_and_repeats_under_the_same_seed():
    model, reqs, _ = fixture(False)

    def run():
        torch.manual_seed(31)
        _engine._seed_counter[0] = 500
        out, _ = serve(model, reqs[:12], 5, 6, masks=False)
        return out
    a, b = run(), run()
    for i in range(12):
        L = a[i]["mel_length"]
        assert 1 <= L <= reqs[i].limit
        for name in NAMES:
            assert bool(torch.isfinite(a[i][name]).all()) and torch.equal(a[i][name], b[i][name]), name
    other, _ = serve(model, reqs[:12], 5, 6, masks=False, seed=12345)
    assert any(other[i]["mel_outputs"].shape != a[i]["mel_outputs"].shape or
               not torch.equal(other[i]["mel_outputs"], a[i]["mel_outputs"]) for i in range(12))      # another seed, other masks
