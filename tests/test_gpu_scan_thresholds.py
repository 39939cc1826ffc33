"""Both single-CTA scans of the library past their one-chunk-per-thread threshold (run with `-m gpu` on an H100).

Two running sums are three-phase scans over chunks of 2048 items whose second phase runs in one CTA of 1024 threads;
each thread takes several chunk totals only once there are more than 1024 chunks, i.e. more than 2^21 items:
  - k_mscan_phase2: the running product of gl_partial_products_and_zs (n rows x M partial-product chunks per row).
    Circuits with 80 routed wires, degree 8 and 2^18..2^20 rows are above the threshold.
  - k_scan_phase2: the suffix sums of divide_by_linear in gl_fri_begin (n coefficients per opening batch), above the
    threshold from 2^22 rows.
"""
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from conftest import P, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pb():
    import torch

    if not torch.cuda.is_available():
        if os.environ.get("GL_REQUIRE_GPU") == "1":
            raise AssertionError("GPU tests need a CUDA device")
        pytest.skip("no CUDA device (gpu-marked tests run on an H100)")
    import plonky2_b200 as p

    p.default_context()
    return p


# (R routed wires, degree, log_n): M = ceil(R / degree) chunks per row, n * M / 2048 scan chunks
@pytest.mark.parametrize("R,deg,log_n", [(64, 2, 15),    # 512 scan chunks
                                         (64, 2, 16),    # exactly 1024, M = 32 (the most a row may have)
                                         (80, 8, 18),    # 1280, not a multiple of 1024
                                         (80, 8, 19),    # 2560
                                         (63, 2, 17)])   # 2048, the last row chunk short
def test_partial_products_past_one_cta(pb, oracle, R, deg, log_n):
    from plonky2_b200.prover import wires_permutation_partial_products_and_zs as gpu_pp

    n = 1 << log_n
    w, sg, k = synth(0x7600 + R, (R, n)), synth(0x7601 + R, (R, n)), synth(0x7602, (R,))
    beta, gamma = int(synth(0x7603, (1,))[0]), int(synth(0x7604, (1,))[0])
    got = gpu_pp(w, sg, k, beta, gamma, deg)
    want = oracle.partial_products_and_zs(w, sg, k, beta, gamma, deg)
    bad = np.argwhere(got != want)
    assert not bad.size, "R=%d degree=%d log_n=%d: first wrong (column, row) %s of %d" % (R, deg, log_n, bad[0], len(bad))


def test_partial_products_chunk_limit(pb, oracle):
    """32 chunks per row work; 33 are refused before the kernel, whose per-thread arrays hold 32."""
    from plonky2_b200.prover import wires_permutation_partial_products_and_zs as gpu_pp

    n = 1 << 4
    for R, ok in ((64, True), (65, False), (66, False)):
        w, sg, k = synth(0x7610 + R, (R, n)), synth(0x7611 + R, (R, n)), synth(0x7612, (R,))
        if ok:
            assert np.array_equal(gpu_pp(w, sg, k, 3, 5, 2), oracle.partial_products_and_zs(w, sg, k, 3, 5, 2))
        else:
            with pytest.raises(pb.NativeError, match="native error 4: more than 32 partial-product chunks"):
                gpu_pp(w, sg, k, 3, 5, 2)


# ----------------------------------------------------------------------------- FRI: divide_by_linear of gl_fri_begin
def e2_mul(x, y):
    return (x[0] * y[0] + 7 * x[1] * y[1]) % P, (x[0] * y[1] + x[1] * y[0]) % P


def e2_inv(x):
    d = pow((x[0] * x[0] - 7 * x[1] * x[1]) % P, P - 2, P)
    return x[0] * d % P, (P - x[1]) * d % P


def e2_pow(x, e):
    r = (1, 0)
    for _ in range(e):
        r = e2_mul(r, x)
    return r


@pytest.mark.parametrize("log_n", [21, 22])  # 1024 and 2048 scan chunks
@pytest.mark.parametrize("points", ["ext_and_base", "zero_and_ext"])
def test_fri_begin_past_one_cta(pb, oracle, log_n, points):
    """gl_fri_begin with two oracles and two opening points, read back with gl_fri_coeffs, satisfies the defining
    identity  c(x) = sum_b alpha^{k_b} (F_b(x) - F_b(z_b)) / (x - z_b),  F_b = sum_j alpha^j f_{b,j}, k_b = the number of
    polynomials in the later batches, at 3 random points x of F_{p^2} (Horner over the commitments' coefficients).
    Points: a generic z in F_{p^2} and a z with c1 = 0, or z = 0 (the division by X branch) and a generic z."""
    from plonky2_b200 import _native as N

    n = 1 << log_n
    r = [int(v) for v in synth(0x7700 + log_n, (12,))]
    zs = {"ext_and_base": [(r[0], r[1]), (r[2], 0)], "zero_and_ext": [(0, 0), (r[3], r[4])]}[points]
    alpha = (r[5], r[6])
    xs = [(r[7], r[8]), (r[9], r[10]), (r[11], 1)]
    coeffs = [synth(0x7710 + log_n, (2, n)), synth(0x7720 + log_n, (3, n))]
    # batch 0 at zs[0]: oracle 0 polys 0, 1 and oracle 1 poly 2; batch 1 at zs[1]: oracle 1 polys 0, 1
    refs = [[(0, 0), (0, 1), (1, 2)], [(1, 0), (1, 1)]]
    commits = [pb.PolynomialBatch.from_coeffs(c, 1, False, 2) for c in coeffs]
    ctx = pb.default_context()
    barr = (N.FriBatch * 2)()
    keep = []
    for i, (z, rr) in enumerate(zip(zs, refs)):
        oi = np.array([o for o, _ in rr], dtype=np.uint32)
        pi = np.array([j for _, j in rr], dtype=np.uint32)
        keep += [oi, pi]
        barr[i].point[0], barr[i].point[1] = z
        barr[i].num_polys = len(rr)
        barr[i].oracle_index = oi.ctypes.data_as(N.u32p)
        barr[i].poly_index = pi.ctypes.data_as(N.u32p)
    handles = (N.vp * 2)(*[c.h for c in commits])
    al = np.array(alpha, dtype=np.uint64)
    h = N.vp()
    try:
        N.check(N.lib().gl_fri_begin(ctx.h, handles, 2, barr, 2, N.np_ptr(al), 1, 2, C.byref(h)), ctx.h)
        got = np.empty((n, 2), dtype=np.uint64)
        N.check(N.lib().gl_fri_coeffs(h, N.np_ptr(got)), ctx.h)
    finally:
        if h:
            N.lib().gl_fri_destroy(h)
        for c in commits:
            c.close()
    assert int(got[n - 1, 0]) == 0 and int(got[n - 1, 1]) == 0, "the quotient has degree < n - 1"
    c0, c1 = np.ascontiguousarray(got[:, 0]), np.ascontiguousarray(got[:, 1])
    pts = xs + list(zs)
    polys = [(o, j) for rr in refs for o, j in rr]
    with ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 1)) as ex:
        ev = dict(zip([(pt, p) for pt in pts for p in polys],
                      ex.map(lambda a: oracle.eval_poly_base_at_ext(coeffs[a[1][0]][a[1][1]], a[0]),
                             [(pt, p) for pt in pts for p in polys])))
        cx = list(ex.map(lambda x: (oracle.eval_poly_base_at_ext(c0, x), oracle.eval_poly_base_at_ext(c1, x)), xs))
    counts = [len(rr) for rr in refs]
    for x, (a, b) in zip(xs, cx):
        want = (0, 0)
        for bi, (z, rr) in enumerate(zip(zs, refs)):
            Fx, Fz = (0, 0), (0, 0)
            for j, p in enumerate(rr):
                aj = e2_pow(alpha, j)
                Fx = tuple(map(sum, zip(Fx, e2_mul(aj, ev[(x, p)]))))
                Fz = tuple(map(sum, zip(Fz, e2_mul(aj, ev[(z, p)]))))
            q = e2_mul(((Fx[0] - Fz[0]) % P, (Fx[1] - Fz[1]) % P), e2_inv(((x[0] - z[0]) % P, (x[1] - z[1]) % P)))
            q = e2_mul(e2_pow(alpha, sum(counts[bi + 1:])), q)
            want = ((want[0] + q[0]) % P, (want[1] + q[1]) % P)
        # c(x) = C0(x) + w * C1(x) with w^2 = 7
        gx = ((a[0] + 7 * b[1]) % P, (a[1] + b[0]) % P)
        assert gx == want, "log_n=%d points=%s x=%s: c(x) = %s, want %s" % (log_n, points, x, gx, want)
