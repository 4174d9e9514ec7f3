"""GPU (H100): the streaming-event engine (run_event in event_engine.cuh) shared by the persistent decoder and the
backward skinny GEMMs, on every consumer plan they use, through t2_selftest_event (the skinny GEMM kernel, one CTA).

A plan is a list of consumers (1-3, of 16 or 32 weight rows); MMA warpgroup 1 + c multiplies consumer c's [W_hi; W_lo]
rows with both split-fp16 activation planes.  The result C = A . W^T is compared with fp64, and two runs of the same
plan must be bitwise equal."""
import ctypes as C

import pytest
import torch

from tacotron2_b200 import _capi
from tests.common import rel_err

pytestmark = pytest.mark.gpu

PLANS = [
    (32,),          # E0 (attention gates <- x2); E3 (decoder gates <- dh) on most CTAs
    (32, 32),       # E1 / E2 (both LSTMs' gates); backward tile of 64 columns
    (32, 32, 16),   # E1 with q, E2 with the projection; backward tile of 80 columns
    (32, 16),       # E3 with the projection
    (16,),          # E4 (prenet layer 2)
]


def run_event(cons, A, W):
    n = sum(cons)
    arr = (C.c_int32 * len(cons))(*cons)
    Cd = torch.full((64, n), float("nan"), device="cuda")
    _capi.check_selftest(_capi.selftest_lib().t2_selftest_event(A.data_ptr(), W.data_ptr(), arr, len(cons), A.shape[1],
                                                                Cd.data_ptr(),
                                                                C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return Cd


@pytest.mark.parametrize("K", [64, 192, 256, 1024])
@pytest.mark.parametrize("cons", PLANS, ids=lambda c: "x".join(map(str, c)))
def test_event_plan_matches_fp64_and_is_bitwise_reproducible(cons, K):
    n = sum(cons)
    g = torch.Generator().manual_seed(n * 1000 + K + len(cons))
    A = torch.randn(64, K, generator=g).cuda()
    W = (torch.randn(n, K, generator=g) / K ** 0.5).cuda()
    C1 = run_event(cons, A, W)
    ref = A.double() @ W.double().t()
    assert rel_err(C1, ref) < 2e-5
    C2 = run_event(cons, A, W)
    assert torch.equal(C1, C2)


@pytest.mark.parametrize("cons", [(40,), (32, 32, 32, 8), (12,), (), (8,), (24,), (32, 8)])
def test_event_rejects_plans_the_warpgroups_cannot_take(cons):
    A = torch.zeros(64, 64, device="cuda")
    W = torch.zeros(max(sum(cons), 8), 64, device="cuda")
    with pytest.raises(_capi.T2Error, match="consumers"):
        run_event(cons, A, W)
