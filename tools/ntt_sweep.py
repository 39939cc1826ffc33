"""Sweep the column-group size of the 2^20 NTT and of the cfg2-shaped LDE (run on the H100): small groups keep the
intermediate of the two passes in the 50 MB L2, large groups give full waves. The group counts transforms per launch:
the rate-1/8 LDE runs a group of g as g/8 columns x 8 cosets."""
import ctypes as C, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from plonky2_b200 import _native as N
L = N.lib()
dev = torch.device("cuda", 0)
stream = torch.cuda.Stream(device=dev)
ctx = N.Context(0, stream=stream.cuda_stream)
ctx.set_profiling(True)
log_n, cols = 20, 64
n = 1 << log_n
with torch.cuda.stream(stream):
    buf = torch.randint(0, 2**63 - 1, (cols, n), dtype=torch.int64, device=dev)
    big = torch.randint(0, 2**63 - 1, (234, n), dtype=torch.int64, device=dev)
    for grp in (4, 8, 16, 32, 64):
        ctx.set_ntt_group(grp)
        for _ in range(3):
            N.check(L.gl_ntt(ctx.h, C.c_void_p(buf.data_ptr()), log_n, cols, n, 0, 0, 1, N.MEM_DEVICE), ctx.h)
        torch.cuda.synchronize()
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        for _ in range(10):
            N.check(L.gl_ntt(ctx.h, C.c_void_p(buf.data_ptr()), log_n, cols, n, 0, 0, 1, N.MEM_DEVICE), ctx.h)
        e.record(stream); torch.cuda.synchronize()
        ms = a.elapsed_time(e) / 10
        # one cfg2 commitment: phase times of the iNTT and the LDE
        for rep in range(2):
            ctx.reset_phases()
            h = N.vp()
            N.check(L.gl_commit_create(ctx.h, C.c_void_p(big.data_ptr()), n, 234, log_n, 3, 4, None, 0, N.MEM_DEVICE, C.byref(h)), ctx.h)
            torch.cuda.synchronize()
            ph = ctx.phase_ms()
            L.gl_commit_destroy(h)
        print("group=%3d : NTT 64x2^20 %.3f ms (%.0f GB/s alg, frac %.3f) | cfg2 iNTT %.2f ms, LDE %.2f ms" % (
            grp, ms, 16.0 * n * cols / ms / 1e6, 16.0 * n * cols / ms / 1e6 / 3350.0, ph["intt"][0], ph["lde"][0]), flush=True)
