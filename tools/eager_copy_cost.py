"""Cost of a SOURCE-COMPATIBLE drop-in for cfg2: after from_values, copy back every public field of the reference's
PolynomialBatch (polynomials, merkle_tree.leaves as row-major rows, merkle_tree.digests, cap) into host memory.
Run on the H100; prints one line."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import plonky2_b200 as pb
from plonky2_b200 import _native as N
from conftest import synth

B, log_n, r, h = 234, 20, 3, 4
vals = synth(0x02, (B, 1 << log_n))
ctx = pb.default_context(0)
for rep in range(2):
    t0 = time.perf_counter()
    c = pb.PolynomialBatch.from_values(vals, r, False, h)
    cap = c.merkle_tree.cap
    t1 = time.perf_counter()
    coeffs = c.polynomials
    t2 = time.perf_counter()
    rows = 1 << (log_n + r)
    leaves = np.empty((rows, B), dtype=np.uint64)
    step = 1 << 20
    for r0 in range(0, rows, step):
        N.check(N.lib().gl_commit_leaves(c.h, r0, step, N.vp(leaves[r0:r0 + step].ctypes.data), N.MEM_HOST), ctx.h)
    t3 = time.perf_counter()
    dig = c.merkle_tree.digests
    t4 = time.perf_counter()
    c.close()
print("cfg2 eager copy-back (pageable host buffers): commit + cap %.3f s | polynomials (1.96 GB) %.3f s | leaves as rows "
      "(15.7 GB, device transpose + D2H) %.3f s | digests (0.54 GB) %.3f s | total extra %.3f s"
      % (t1 - t0, t2 - t1, t3 - t2, t4 - t3, t4 - t1))
