import ctypes as C, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tacotron2_b200 import _capi
torch.zeros(1).cuda()
L = _capi.selftest_lib()
out = (C.c_int64 * 2)()
for M in (64,):
    for N in (32, 64, 128):
        for alt in (0, 1):
            for reps in (8, 64, 256):
                _capi.check_selftest(L.t2_selftest_mma_rate(M, N, reps, alt, out))
                print("M=%3d N=%3d alt=%d reps=%3d  issue %6d clk (%.1f/mma)  total %7d clk (%.1f/mma)" % (M, N, alt, reps, out[0], out[0]/reps, out[1], out[1]/reps))

print("groups of G MMAs + commit + wait (one K chunk of a streaming event), cycles per group / per MMA:")
for M in (64,):
    for N in (32, 64, 128):
        for G in (1, 2, 4, 8, 16):
            _capi.check_selftest(L.t2_selftest_mma_group(M, N, G, 64, out))
            print("M=%3d N=%3d group=%2d  %7.1f clk / group  %6.1f clk / MMA" % (M, N, G, out[0] / 64, out[0] / 64 / G))
