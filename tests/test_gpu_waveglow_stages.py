"""Every launch of WaveGlow inference against an fp64 restatement of that one launch, in both precision tiers.

t2_selftest_waveglow_state runs t2_waveglow_infer_window's own launch sequence, stops after n launches and hands out
the workspace (spect, h, acts, skip, aud) as fp32.  For launch n + 1 the oracle step (oracle/waveglow_oracle.py) is
applied in fp64 to the state the engine itself held after n launches -- exactly the operands the kernel read -- and
compared with the state after n + 1.  What is left in that difference is one launch's arithmetic: the split-operand
products, the fp32 accumulation, tanhf / expf, and the rounding of the output (2^-22 into split planes, 2^-11 into
fp16 planes, none into the fp32 skip / aud buffers), so the bars are per output kind and far below the 1e-3 of the
end-to-end tests.  The reference weights are folded from the state dict, never read back from the packed images, so
packing, row permutation, tap order, cond slice and bias sums are under test as well.

Launch order (207): mel to planes, upsample GEMM, initial tail, then per flow 11 ... 0: 8 x (gate GEMM, res/skip GEMM)
and a tail.  Rows: q = b * span + t, span = 32 T_mel + 128, in tiles of 128."""
import ctypes as C

import pytest
import torch

from oracle import waveglow_oracle as WO
from tacotron2_b200 import _capi
from tests.waveglow_common import CONFIG, mel_input, noise, state_dict_shapes, synth_state_dict

pytestmark = pytest.mark.gpu

GUARD, TILE, N_LAUNCHES, SIGMA = 128, 128, 207, 0.666
DEV = "cuda"
FLOW_REACH = 255           # columns one flow's eight dilated layers reach to either side (1 + 2 + ... + 128)
TIERS = ["fp32", "fp16"]

# max |engine - truth| / max |truth| per stage output; about 4 x the largest value seen on an H100 (80GB HBM3, 700 W)
# over all the cases below (DESIGN.md 6.6 has the values), and never above 2e-5 (fp32-grade tier, and the fp32 skip /
# aud buffers of the fp16 tier) or 1e-3 (outputs stored as fp16 planes: they measure 3e-4 ... 4.7e-4, fp16's half ulp
# relative to the maximum).
BARS = {
    "fp32": dict(upsample=1e-5, start=1e-6, gate=2e-5, res=2e-6, skip=6e-6, tail=1.5e-6),
    "fp16": dict(upsample=1e-3, start=1e-3, gate=1e-3, res=1e-3, skip=3e-6, tail=1.5e-6),
}

_CACHE = {}


def cached(key, make):
    if key not in _CACHE:
        _CACHE[key] = make()
    return _CACHE[key]


def sd7():
    return cached("sd", lambda: synth_state_dict(7))


class Engine:
    """A T2WaveGlow handle of the self-test library over the seeded weights, in one tier."""

    def __init__(self, tier):
        self.L, self.fp16 = _capi.selftest_lib(), tier == "fp16"
        self.held = []
        names = [n for n, _ in state_dict_shapes()]
        assert len(names) == _capi.T2_WAVEGLOW_NUM_WEIGHTS
        ptrs = (C.c_void_p * len(names))()
        for i, n in enumerate(names):
            half = self.fp16 and not n.startswith("convinv")      # convinv stays fp32, as in the notebook's half model
            t = sd7()[n].to(device=DEV, dtype=torch.float16 if half else torch.float32).contiguous()
            self.held.append(t)
            ptrs[i] = t.data_ptr()
        w = CONFIG["WN_config"]
        cfg = _capi.T2WaveGlowConfig(80, 12, 8, 4, 2, w["n_layers"], w["kernel_size"], w["n_channels"], int(self.fp16))
        h = C.c_void_p()
        _capi.check_selftest(self.L.t2_waveglow_create(C.byref(h), C.byref(cfg), ptrs, len(names), None))
        torch.cuda.synchronize()
        self.handle = h

    def state(self, n, mel, z, lengths=None, frame0=0, out=None, at_end=True):
        """The workspace after n launches as fp32 tensors (rows, C), and the audio buffer (written by launch 207)."""
        B, T = mel.shape[0], mel.shape[2]
        out0, out1 = out if out is not None else (0, T)
        span = 32 * T + GUARD
        rows = (B * span + TILE - 1) // TILE * TILE
        key = ("ws", B, T)
        ws = cached(key, lambda: torch.zeros(self.L.t2_waveglow_workspace_bytes(None, B, T), dtype=torch.uint8, device=DEV))
        audio = torch.zeros(B, 256 * (out1 - out0), device=DEV)
        a = _capi.T2WaveGlowArgs(mel.data_ptr(), B, T, lengths.data_ptr() if lengths is not None else None, 0, SIGMA,
                                 z.data_ptr(), 0, audio.data_ptr(), ws.data_ptr(), ws.numel())
        w = _capi.T2WaveGlowWindowArgs(a, frame0, out0, out1, z.shape[2] // 32, int(at_end))
        s = {k: torch.empty(rows, c, device=DEV) for k, c in (("spect", 640), ("h", 256), ("acts", 256), ("skip", 256),
                                                                 ("aud", 8))}
        _capi.check_selftest(self.L.t2_selftest_waveglow_state(self.handle, C.byref(w), n, *[s[k].data_ptr() for k in
                                                               ("spect", "h", "acts", "skip", "aud")], None))
        torch.cuda.synchronize()
        s["audio"] = audio
        return s


def engine(tier):
    return cached(("engine", tier), lambda: Engine(tier))


def engine_fold(v, g):
    """v * (g / sqrt(sum v^2)) in fp32 in the order of waveglow.cu's wn_scale, for fp16-valued v and g: 256 threads
    each add the squares of their elements i, i + 256, ... in turn (exact products: 11-bit operands), a 32-lane
    butterfly adds lanes 16, 8, 4, 2, 1 apart, and thread 0 adds the 8 warp sums in turn from zero."""
    x = v.float().flatten(1)
    sq = torch.nn.functional.pad(x * x, (0, -x.shape[1] % 256)).view(x.shape[0], -1, 256)
    ss = sq[:, 0]
    for j in range(1, sq.shape[1]):
        ss = ss + sq[:, j]
    ss = ss.view(-1, 8, 32)
    for o in (16, 8, 4, 2, 1):
        ss = ss[..., :o] + ss[..., o:2 * o]
    tot = torch.zeros_like(ss[:, 0, 0])
    for w in range(8):
        tot = tot + ss[:, w, 0]
    return v.float() * (g.float().view(-1) / tot.sqrt()).view(-1, 1, 1)


def truth_weights(tier):
    """The state dict the fp64 steps use, with the weight norm folded: plain `weight` entries, as after
    remove_weightnorm.  fp32-grade tier: everything in fp64.  fp16 tier: the engine is given fp16 tensors and keeps only
    the fp16 hi plane of each folded GEMM weight, so the entries are rounded to fp16 first and the folded GEMM weights
    again; start and end stay fp32 on the CUDA cores.  A weight folded in fp64 that lies within the engine's fp32 fold
    error of an fp16 rounding boundary rounds to the other neighbour -- about 16 weights of a 512 x 256 matrix, each one
    fp16 ulp off, which alone puts 2e-5 ... 5e-5 into skip -- so the GEMM weights are folded as the engine folds them
    (engine_fold) and the fp16 image is reproduced exactly."""
    def make():
        sd, out = sd7(), {}
        for n, v in sd.items():
            v = v.to(DEV)
            if tier == "fp16" and not n.startswith("convinv"):
                v = v.half()
            if n.endswith("weight_g"):
                continue
            if n.endswith("weight_v"):
                p, g = n[:-len("weight_v")], sd[n[:-1] + "g"].to(DEV)
                gemm = ".start." not in n
                if tier == "fp16" and gemm:
                    v = engine_fold(v, g.half()).half()
                else:
                    g, v = (g.half() if tier == "fp16" else g).double(), v.double()
                    v = v * (g / v.flatten(1).norm(dim=1).view(-1, 1, 1))
                out[p + "weight"] = v.double()
            else:
                out[n] = v.double()
        return out
    return cached(("truth", tier), make)


def operand_rounding(x, tier):
    """What the planes hold of an fp32 input: hi + lo of the split in the fp32-grade tier, the fp16 value in the fp16 tier."""
    hi = x.half()
    if tier == "fp16":
        return hi.double()
    return hi.double() + (x - hi.float()).half().double()


def launch_of(k, l=None, res=False):
    """1-based index of flow k's gate (l, res False), res/skip (l, res True) or tail (l None) launch."""
    base = 3 + (11 - k) * 17
    return base + 17 if l is None else base + 2 * l + 1 + int(res)


def stage_of(n):
    """(kind, k, l) of launch n (1-based)."""
    if n <= 3:
        return (("mel", "upsample", "init")[n - 1], None, None)
    k, r = 11 - (n - 4) // 17, (n - 4) % 17
    return ("tail", k, None) if r == 16 else (("gate", "res")[r % 2], k, r // 2)


def needed(k_after, T, out):
    """Columns [lo, hi) a launch must compute when k_after flows follow it (`widen` in waveglow.cu): the output columns
    widened by one flow's reach per flow still to run, clipped to the window."""
    return max(0, 32 * out[0] - FLOW_REACH * k_after), min(32 * T, 32 * out[1] + FLOW_REACH * k_after)


class Case:
    def __init__(self, name, T, lengths, launches=None, window=None, scale=None, seed=0):
        self.name, self.T, self.lengths, self.window = name, T, lengths, window
        self.B = len(lengths)
        self.launches = list(range(2, N_LAUNCHES + 1)) if launches is None else launches   # launch 1 writes no state read here
        self.frame0, self.out, self.at_end = window if window else (0, (0, T), True)
        self.scale, self.seed, self.span = scale, seed, 32 * T + GUARD
        self._inputs = None

    def inputs(self):
        """(mel, z, lengths or None) on the device; made on first use, so that collecting the tests needs no GPU."""
        if self._inputs is None:
            mel, z = mel_input(self.B, self.T, 500 + self.seed), noise(self.B, self.frame0 + self.T, 600 + self.seed)
            if self.scale is not None:
                s = torch.tensor(self.scale).view(-1, 1, 1)
                mel, z = mel * s, z * s
            ragged = any(n != self.T for n in self.lengths)
            len32 = torch.tensor(self.lengths, dtype=torch.int32, device=DEV) if ragged else None
            self._inputs = (mel.to(DEV).contiguous(), z.to(DEV).contiguous(), len32)
        return self._inputs

    mel = property(lambda self: self.inputs()[0])
    z = property(lambda self: self.inputs()[1])

    def state(self, tier, n):
        return engine(tier).state(n, *self.inputs(), self.frame0, self.out if self.window else None,
                                  self.at_end)

    def seqs(self, x):
        """(rows, C) -> (B, C, 32 T) fp64: the data columns of each sequence."""
        return x[:self.B * self.span].view(self.B, self.span, -1)[:, :32 * self.T].permute(0, 2, 1).double()

    def valid(self):
        """(B, 1, 32 T) bool: columns inside each row's own length."""
        t = torch.arange(32 * self.T, device=DEV).view(1, 1, -1)
        return t < 32 * torch.tensor(self.lengths, device=DEV).view(-1, 1, 1)

    def padding_rows(self):
        """(rows) bool over a dump: rows that are not data of any sequence (past a row's length, the guard rows between
        sequences, the rest of the last tile)."""
        rows = (self.B * self.span + TILE - 1) // TILE * TILE
        q = torch.arange(rows, device=DEV)
        b, t = q // self.span, q % self.span
        lens = torch.tensor(self.lengths + [0], device=DEV)
        return t >= 32 * lens[b.clamp(max=self.B)]


EARLY = [launch_of(8), launch_of(4)]                  # the tails that put the early noise in front
SUBSET = sorted({2, 3, launch_of(11, 0), launch_of(11, 0, True), launch_of(11, 7), launch_of(11, 7, True), launch_of(11),
                 *EARLY, launch_of(0, 0), launch_of(0, 0, True), launch_of(0, 7), launch_of(0, 7, True), launch_of(0)})
FLOW11 = list(range(2, launch_of(11) + 1))            # the upsample, the initial tail and all of flow 11

CASES = [
    # 32 columns: every dilation >= 32 reads nothing but guard rows
    Case("T1_B1", 1, [1], seed=1),
    Case("T1_B3", 1, [1, 1, 1], seed=2),
    # span 224: the three sequences sit at three different offsets in their 128-row tiles, and straddle them
    Case("T3_ragged", 3, [3, 1, 2], seed=3),
    # span 256: every sequence starts exactly on a tile boundary
    Case("T4_B2", 4, [4, 4], seed=4),
    # 3 M tiles: the odd tile count runs the cluster's padding tile, which streams tile 0 and discards
    Case("T8_B1", 8, [8], seed=5),
    # frame domain of the upsample GEMM: T + 4 = 128 is exactly one tile, 129 is one row past it
    Case("T124_B1", 124, [124], launches=FLOW11, seed=6),
    Case("T125_B1", 125, [125], launches=FLOW11, seed=7),
    # the ragged shape of the end-to-end tests, every launch
    Case("T37_ragged", 37, [37, 11, 1], seed=8),
    # a window inside a sequence: frames [10, 240), audio of window frames [110, 120); the first flows skip the tiles
    # before column 32 * 110 - 12 * 255 = 460 and after 32 * 120 + 12 * 255 = 6900, later flows skip more
    Case("window_T230", 230, [230], launches=SUBSET, window=(10, (110, 120), False), seed=9),
]


def check(errs, kind, got, want, mask, where):
    """Record max |got - want| / max |want| over the masked entries under `kind`."""
    mask = mask.expand_as(want)
    den = float(want[mask].abs().max())
    e = float((got - want)[mask].abs().max()) / (den if den > 0 else 1.0)
    assert e == e, "%s: not a number at %s" % (kind, where)
    if e > errs.get(kind, (-1.0, None))[0]:
        errs[kind] = (e, where)


def one_step(case, tier, n, before, after, errs):
    """Compare launch n: the fp64 step on `before` (the state after n - 1 launches) against `after`."""
    sd, (kind, k, l) = truth_weights(tier), stage_of(n)
    where = "launch %d (%s%s%s)" % (n, kind, "" if k is None else " flow %d" % k, "" if l is None else " layer %d" % l)
    T, S = case.T, case.seqs
    valid = case.valid()
    cols = torch.arange(32 * T, device=DEV).view(1, 1, -1)

    def rng(k_after):                       # the columns this launch must have computed
        lo, hi = needed(k_after, T, case.out)
        return (cols >= lo) & (cols < hi)
    if kind == "upsample":
        mel = operand_rounding(case.mel, tier)
        mel = mel * (torch.arange(T, device=DEV).view(1, 1, -1) < torch.tensor(case.lengths, device=DEV).view(-1, 1, 1))
        check(errs, "upsample", S(after["spect"]), WO.upsample_unfold(sd, mel), cols >= 0, where)
    elif kind == "init":
        z = case.z[:, :, 32 * case.frame0:].double()
        m = valid & rng(12)
        want = torch.cat([SIGMA * z[:, :4], torch.zeros_like(z[:, :4])], 1) * valid
        got = S(after["aud"])
        check(errs, "tail", got, want, m, where)
        check(errs, "start", S(after["h"]), WO.start(sd, 11, got[:, :4]) * valid, m, where)
    elif kind == "gate":
        want = WO.gate(sd, k, l, S(before["h"]), S(before["spect"])) * valid
        check(errs, "gate", S(after["acts"]), want, rng(k + 1), where)
    elif kind == "res":
        h, skip = S(before["h"]), S(before["skip"])
        h2, skip2 = WO.res_skip(sd, k, l, S(before["acts"]), h, torch.zeros_like(skip) if l == 0 else skip)
        check(errs, "res", S(after["h"]), h2 * valid, rng(k + 1), where)
        check(errs, "skip", S(after["skip"]), skip2, valid & rng(k + 1), where)
    elif kind == "tail":
        nr = WO.n_remaining(k)
        z = case.z[:, :, 32 * case.frame0:].double()
        m = valid & rng(k)
        want = WO.flow_tail(sd, k, S(before["aud"])[:, :nr], S(before["skip"]), z, SIGMA)
        if k > 0:
            got, nn = S(after["aud"]), WO.n_remaining(k - 1)
            assert want.shape[1] == nn
            check(errs, "tail", got[:, :nn], want, m, where)
            assert not bool((got[:, nn:] != 0).any()), where
            check(errs, "start", S(after["h"]), WO.start(sd, k - 1, got[:, :nn]) * valid, m, where)
        else:                               # the last tail writes the audio: (B, 8 columns) of the output frames
            lo, hi = 32 * case.out[0], 32 * case.out[1]
            got = after["audio"].view(case.B, hi - lo, 8).permute(0, 2, 1).double()
            check(errs, "tail", got, (want * valid)[:, :, lo:hi], cols[:, :, lo:hi] >= 0, where)
    if case.window is None and n >= 2:
        # what the next launches read as zero padding is zero: exactly, and after every launch
        pad = case.padding_rows()
        assert not bool((after["h"][pad] != 0).any()) and not bool((after["acts"][pad] != 0).any()), where
        if kind in ("init", "tail") and k != 0:
            assert not bool((after["aud"][pad] != 0).any()), where


@pytest.mark.parametrize("tier", TIERS)
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_each_launch_matches_the_fp64_step_on_its_own_operands(case, tier):
    errs, states = {}, {}
    for n in case.launches:
        for i in (n - 1, n):
            if i not in states:
                states[i] = case.state(tier, i)
        one_step(case, tier, n, states[n - 1], states[n], errs)
        states.pop(n - 1)
    bars = BARS[tier]
    print("\n%s %s (%d launches):" % (case.name, tier, len(case.launches)), "  ".join(
        "%s %.2e / %.0e" % (kd, errs[kd][0], bars[kd]) for kd in ("upsample", "start", "gate", "res", "skip", "tail") if kd in errs))
    for kd, (e, where) in errs.items():
        assert e <= bars[kd], "%s: %.3e > %.0e at %s" % (kd, e, bars[kd], where)


@pytest.mark.parametrize("tier", TIERS)
def test_a_short_row_between_two_large_ones_keeps_the_bits_of_its_own_run(tier):
    """T_mel = 1: 32 columns, so the taps of dilation 32, 64 and 128 land in the guard rows -- or, were a shift or a
    guard wrong, in the neighbouring sequence.  The neighbours are 1000 times larger, so any leak shows; the middle row
    must have the bits of its own B = 1 run after every launch."""
    three = Case("scaled", 1, [1, 1, 1], scale=[1e3, 1.0, 1e3], seed=11)
    alone = Case("alone", 1, [1], seed=11)
    alone._inputs = (three.mel[1:2].contiguous(), three.z[1:2].contiguous(), None)
    for n in range(2, N_LAUNCHES + 1):
        a, b = three.state(tier, n), alone.state(tier, n)
        for key in ("spect", "h", "acts", "skip", "aud"):
            if key == "skip" and n < launch_of(11, 0, True):
                continue                    # not written yet: skip is not cleared
            if key == "aud" and n < 3:
                continue
            got, want = a[key][three.span:three.span + 32], b[key][:32]
            assert torch.equal(got, want), (n, stage_of(n), key)
        if n == N_LAUNCHES:
            assert torch.equal(a["audio"][1], b["audio"][0])
        pad = three.padding_rows()
        assert not bool((a["h"][pad] != 0).any()) and not bool((a["acts"][pad] != 0).any()), n
