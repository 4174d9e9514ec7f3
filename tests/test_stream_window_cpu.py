"""FinalWindow, the finality window behind WaveGlow.infer_stream and Denoiser.stream, on synthetic item sequences:
spans, windows, window-relative row ends and the kept input against the two loops those streams ran before they shared
it, restated here in their own units (mel frames; samples in 256-sample blocks)."""
import random

import pytest
import torch

from tacotron2_b200._stream import FinalWindow

HOP = 256
B = 3


def waveglow_loop(items, left, right):
    """WaveGlow.infer_stream's loop in mel frames: per yielded item its span, kept frames and (window, row ends)."""
    out, kept, base, held, a0 = [], None, 0, 0, 0
    for it in items:
        f0, f1 = it["frames"]
        assert f0 == held
        kept = it["x"] if kept is None else torch.cat((kept, it["x"]), 2)
        held, finished = f1, it["finished"]
        a1 = held if finished else max(a0, held - right)
        if a1 == a0 and not finished:
            continue
        rec = dict(span=(a0, a1), kept=kept, window=None)
        if a1 > a0:
            w0, w1, lengths = base, held, it["mel_lengths"]
            win_len = torch.where(lengths < 0, torch.full_like(lengths, w1 - w0),
                                  (lengths - w0).clamp(min=0, max=w1 - w0)).to(torch.int32)
            rec["window"] = ((w0, a0 - w0, a1 - w0), win_len)
        out.append(rec)
        a0 = a1
        if finished:
            break
        drop = max(0, a0 - left) - base
        kept, base = kept[:, :, drop:], base + drop
    return out


def denoiser_loop(items, left, right):
    """Denoiser.stream's loop in samples, final in 256-sample blocks; same records as waveglow_loop."""
    out, kept, base, held, d0 = [], None, 0, 0, 0
    for it in items:
        s0, s1 = it["samples"]
        assert s0 == held
        kept = it["x"] if kept is None else torch.cat((kept, it["x"]), 1)
        held, finished = s1, it["finished"]
        d1 = held // HOP if finished else max(d0, held // HOP - right)
        if d1 == d0 and not finished:
            continue
        rec = dict(span=(d0, d1), kept=kept, window=None)
        if d1 > d0:
            lengths = it["mel_lengths"]
            win_len = torch.where(lengths < 0, torch.full_like(lengths, -1),
                                  (HOP * lengths - base).clamp(min=0)).to(torch.int32)
            rec["window"] = ((base, d0 - base // HOP, d1 - base // HOP), win_len)
        out.append(rec)
        d0 = d1
        if finished:
            break
        drop = HOP * max(0, d0 - left) - base
        kept, base = kept[:, drop:], base + drop
    return out


def window_loop(items, key, axis, left, right, unit, open_end):
    """The same records from FinalWindow, and the most input elements it kept after an item beyond the two halos."""
    win, out, over = FinalWindow("test items", key, axis, left, right, unit), [], []
    for it in items:
        win.check(it)
        span = win.add(it, it["x"])
        over.append(win.kept.shape[axis] - (left + right) * unit - it["x"].shape[axis])
        assert win.kept.shape[axis] == win.held - win.base
        if span is None:
            continue
        rec = dict(span=span, kept=win.kept, window=None)
        if span[1] > span[0]:
            rec["window"] = ((win.base, span[0] - win.base // unit, span[1] - win.base // unit),
                             win.lengths(it["mel_lengths"], open_end(win)))
        out.append(rec)
        if it["finished"]:
            break
    return out, max(over)


def make_items(sizes, key, unit, axis):
    """Consecutive items of sizes[i] units; the last one finishes the stream.  Row 0 stays live to the end, row 1 stops
    a third of the way in and reports it once half of that is held, row 2 reports its stop from the start (it can lie
    past the input held so far)."""
    total = sum(sizes)
    seq = torch.arange(B * 2 * total * unit, dtype=torch.float32).view(B, 2, total * unit)
    if axis == 1:
        seq = seq[:, 0]
    items, held = [], 0
    for i, n in enumerate(sizes):
        finished = i == len(sizes) - 1
        s0, held = held, held + n
        lengths = torch.tensor([total if finished else -1, total // 3 if held >= total // 6 or finished else -1,
                                total - 1 if total > 1 else total], dtype=torch.int32)
        items.append({key: (s0 * unit, held * unit), "x": seq.narrow(axis, s0 * unit, n * unit), "finished": finished,
                      "mel_lengths": lengths})
    return items, seq, total


def chunkings():
    rng = random.Random(5)
    for total in (1, 6, 96, 97, 99, 195, 196, 300, 431):
        for c in range(1, 41):
            sizes = [c] * (total // c) + ([total % c] if total % c else [])
            yield sizes
            yield sizes + [0]                        # a last item with no new input, as a stream that stops on a boundary
        sizes, n = [], total
        while n > 0:
            sizes.append(min(n, rng.randint(1, 40)))
            n -= sizes[-1]
        yield sizes


CASES = [("waveglow", (99, 96)), ("waveglow", (3, 3)), ("denoiser", (3, 3)), ("denoiser", (99, 96))]


@pytest.mark.parametrize("stage,halo", CASES, ids=["%s-%d-%d" % (s, *h) for s, h in CASES])
def test_final_window_matches_the_streams_loops(stage, halo):
    left, right = halo
    if stage == "waveglow":
        key, axis, unit, old = "frames", 2, 1, waveglow_loop
        open_end = lambda w: w.held - w.base
    else:
        key, axis, unit, old = "samples", 1, HOP, denoiser_loop
        open_end = lambda w: -1
    for sizes in chunkings():
        items, seq, total = make_items(sizes, key, unit, axis)
        got, over = window_loop(items, key, axis, left, right, unit, open_end)
        ref = old(items, left, right)
        assert [r["span"] for r in got] == [r["span"] for r in ref], sizes
        # the spans are consecutive, cover [0, total) and only the last item finishes
        assert got[0]["span"][0] == 0 and got[-1]["span"][1] == total
        assert all(a["span"][1] == b["span"][0] for a, b in zip(got, got[1:]))
        # the stream keeps at most the two halos plus one item
        assert over <= 0, (sizes, over)
        for g, r in zip(got, ref):
            assert torch.equal(g["kept"], r["kept"]), sizes
            assert (g["window"] is None) == (r["window"] is None)
            if g["window"] is None:
                continue
            assert g["window"][0] == r["window"][0], sizes
            ends, old_ends = g["window"][1], r["window"][1]
            n = g["kept"].shape[axis]
            if stage == "waveglow":
                assert torch.equal(ends, old_ends)
            else:                                    # a row that ends past the window runs through it: -1 or > n alike
                assert torch.equal(ends, torch.where(old_ends > n, torch.full_like(old_ends, -1), old_ends))


@pytest.mark.parametrize("left,right", [(99, 96), (3, 3)])
def test_no_span_passes_the_held_input_less_the_right_halo(left, right):
    for sizes in chunkings():
        items, _, _ = make_items(sizes, "frames", 1, 2)
        win = FinalWindow("test items", "frames", 2, left, right)
        for it in items:
            win.check(it)
            span = win.add(it, it["x"])
            if span is not None and not it["finished"]:
                assert span[0] < span[1] <= win.held - right, (sizes, span, win.held)


def test_items_must_be_consecutive():
    items, _, _ = make_items([4, 4, 4], "samples", HOP, 1)
    win = FinalWindow("Denoiser.stream: audio items", "samples", 1, 3, 3, HOP)
    win.check(items[0])
    win.add(items[0], items[0]["x"])
    with pytest.raises(ValueError, match=r"Denoiser.stream: audio items must be consecutive \(samples \(2048, 3072\) "
                                         r"after 1024\)"):
        win.check(items[2])
