"""Every NTT pass plan and both kernel bodies against exact references (run with `-m gpu` on an H100).

A transform of n = 2^log_n runs as up to three passes (gl_ntt.cuh, ntt_plan): a1 and a2 are strided column passes
(k_ntt_col<LOG>), b is the contiguous row pass (k_ntt_row<LOG, MODE>, natural-order stores for fft / ifft, bit-reversed
stores for the coset LDE of a commitment). Each pass length is its own template instantiation with its own thread
shape, and even lengths have a second, shared-body kernel (k_ntt_*_shared) that runs unless bit 31 of
gl_ctx_set_ntt_group selects the two-copy kernels. Every test here runs both: variant 0 is the default context
setting, variant 1 sets bit 31.

    log_n    a1  a2   b          log_n    a1  a2   b
    1..10     -   -  log_n       21        7   7   7
    11        5   -   6          22        7   7   8
    12        6   -   6          23        7   8   8
    13        6   -   7          24        8   8   8
    14        7   -   7          25        8   8   9
    15        7   -   8          26        8   9   9
    16        8   -   8          27        9   9   9
    17        8   -   9
    18        9   -   9
    19        9   -  10
    20       10   -  10

So log_n 1..22 reach every column length 5..10 and every row length 1..10, in natural order (fft and ifft) and
bit-reversed order (from_coeffs), under both variants; log_n 23..27 reach the remaining three-pass shapes.

The inputs push the lazy 3-word butterflies (gl_lazy.cuh) of the first pass, which see the caller's raw words, to
their largest magnitudes: all 2^64 - 1, all p - 1, and square waves of 0 / 2^64 - 1 whose period matches a level of a
pass. Every mismatch names (log_n, plan, variant, mode, input class, column, index).
"""
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from conftest import EDGE, P, synth

pytestmark = pytest.mark.gpu

M64 = 2**64 - 1
VARIANT_BIT = 0x80000000
# coset shifts: a random one, a small one, -1, p + 1 (= 1: must take the plain path) and the non-canonical 2^64 - 1
SHIFTS = [("random", int(synth(0x7A1, (1,))[0]) | 1), ("7", 7), ("p-1", P - 1), ("p+1", P + 1), ("2^64-1", M64)]


def ntt_plan(log_n):
    """(a1, a2, b): the restatement of gl_ntt.cuh's ntt_plan that the table above lists."""
    if log_n <= 10:
        return 0, 0, log_n
    if log_n <= 20:
        b = (log_n + 1) // 2
        return log_n - b, 0, b
    b = (log_n + 2) // 3
    a2 = (log_n - b + 1) // 2
    return log_n - b - a2, a2, b


def test_plan_table_reaches_every_pass_length():
    plans = {k: ntt_plan(k) for k in range(1, 28)}
    cols = {a for k in range(1, 23) for a in plans[k][:2] if a}
    rows = {plans[k][2] for k in range(1, 23)}
    assert cols == set(range(5, 11)) and rows == set(range(1, 11))
    assert {plans[k] for k in range(21, 28)} == {(7, 7, 7), (7, 7, 8), (7, 8, 8), (8, 8, 8), (8, 8, 9), (8, 9, 9), (9, 9, 9)}
    assert [k for k in range(1, 28) if 9 in plans[k][:2]] == [18, 19, 26, 27]


PLAN_PRINTER = r"""
#include <cstdio>
#include "gl_ntt.cuh"
int main() {
    for (int k = 1; k <= 30; k++) {
        const gl::NttPlan p = gl::ntt_plan(k);
        printf("%d %d %d %d\n", k, p.a1, p.a2, p.b);
    }
    return 0;
}
"""


def test_plan_restatement_matches_the_library(tmp_path):
    """ntt_plan above and the docstring table are what gl_ntt.cuh's ntt_plan computes (host build of the header), so
    the coverage this module claims follows the library's planner."""
    import re
    import subprocess

    src, exe = tmp_path / "plans.cpp", str(tmp_path / "plans")
    src.write_text(PLAN_PRINTER)
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "plonky2_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", csrc, "-o", exe, str(src)])
    lib = {int(k): (int(a1), int(a2), int(b))
           for k, a1, a2, b in (line.split() for line in subprocess.check_output([exe], text=True).splitlines())}
    assert lib == {k: ntt_plan(k) for k in range(1, 31)}
    table = {int(k): (0 if a1 == "-" else int(a1), 0 if a2 == "-" else int(a2), int(b))
             for k, a1, a2, b in re.findall(r"(\d+)\s+(\d+|-)\s+(\d+|-)\s+(\d+)", __doc__)}
    assert len(table) == 17 and all(lib[k] == v for k, v in table.items()), table


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


@pytest.fixture(scope="module")
def variants(pb):
    """Private contexts: variant 0 (default kernels) and variant 1 (two-copy kernels for even pass lengths)."""
    ctxs = [pb.Context(0), pb.Context(0)]
    ctxs[1].set_ntt_group(VARIANT_BIT)
    yield ctxs
    for c in ctxs:
        c.close()


@pytest.fixture(scope="module")
def grouped(pb):
    """Private contexts with 8-column groups: 13 columns run as two groups, the second one short."""
    ctxs = [pb.Context(0), pb.Context(0)]
    ctxs[0].set_ntt_group(8)
    ctxs[1].set_ntt_group(8 | VARIANT_BIT)
    yield ctxs
    for c in ctxs:
        c.close()


def _pool():
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    return ThreadPoolExecutor(max_workers=max(1, min(n, 32)))  # the oracle's ctypes calls release the GIL


def _pmap(fn, items):
    with _pool() as ex:
        return list(ex.map(fn, items))


def square(n, k):
    """0 / 2^64 - 1 square wave of period 2^k (first half of each period 0)."""
    j = np.arange(n, dtype=np.uint64)
    return np.where((j >> np.uint64(k - 1)) & np.uint64(1), np.uint64(M64), np.uint64(0))


def square_periods(log_n):
    """log2 of the square-wave periods that alternate the inputs of each level of the first pass's step 1 (the
    radix-E lazy DFT over the high index bits q, input stride 2^(s + r2)), plus 2 and 2^LOG of every pass."""
    a1, a2, b = ntt_plan(log_n)
    first = a1 or b
    s = log_n - first
    r1, r2 = first - first // 2, first // 2
    ks = {1, s + r2 + 1, s + r2 + r1} | {L for L in (a1, a2, b) if L}
    return sorted(k for k in ks if 1 <= k <= log_n)


def input_classes(log_n, seed):
    n = 1 << log_n
    out = [("random non-canonical", synth(seed, (n,), canonical=False)),
           ("all 2^64-1", np.full(n, M64, dtype=np.uint64)),
           ("all p-1", np.full(n, P - 1, dtype=np.uint64))]
    out += [("square 2^%d" % k, square(n, k)) for k in square_periods(log_n)]
    imp = np.zeros(n, dtype=np.uint64)
    imp[n - 1] = M64
    out += [("impulse at n-1", imp), ("EDGE tiled", np.resize(np.array(EDGE, dtype=np.uint64), n))]
    return out


def assert_same(got, want, tag, names):
    """Bit-exact comparison of (columns, n) arrays; the message names the first wrong column and index."""
    got, want = np.atleast_2d(got), np.atleast_2d(want)
    assert got.shape == want.shape, (tag, got.shape, want.shape)
    bad = np.nonzero(got != want)
    if bad[0].size:
        c, i = int(bad[0][0]), int(bad[1][0])
        raise AssertionError("%s, input class=%s, column=%d, index=%d: got %#x want %#x (%d wrong words)"
                             % (tag, names[c], c, i, int(got[c, i]), int(want[c, i]), bad[0].size))


def run_mode(pb, ctx, x, mode, shift):
    if mode == "fft":
        return pb.fft(x, ctx=ctx)
    if mode == "ifft":
        return pb.ifft(x, ctx=ctx)
    if mode == "coset_fft":
        return pb.coset_fft(x, shift, ctx=ctx)
    return pb.coset_ifft(x, shift, ctx=ctx)


def oracle_mode(oracle, mode, shift):
    return {"fft": oracle.fft, "ifft": oracle.ifft,
            "coset_fft": lambda c: oracle.coset_fft(c, shift),
            "coset_ifft": lambda c: oracle.coset_ifft(c, shift)}[mode]


# ----------------------------------------------------------------------------- 1. every plan, log_n 1..22
@pytest.mark.parametrize("log_n", range(1, 23))
def test_ntt_plan_matches_oracle(pb, oracle, variants, log_n):
    classes = input_classes(log_n, 0x7000 + log_n)
    names = [c[0] for c in classes]
    x = np.stack([c[1] for c in classes])
    plan = ntt_plan(log_n)
    xc = x % np.uint64(P)
    cases = [("fft", "1", 1), ("ifft", "1", 1)]
    cases += [(m, sname, s) for sname, s in SHIFTS for m in ("coset_fft", "coset_ifft")]
    plain = {}
    for mode, sname, shift in cases:
        if sname == "p+1":  # shift = 1 (mod p): the plain transform, already computed
            want = plain["fft" if mode == "coset_fft" else "ifft"]
        else:
            want = np.stack(_pmap(oracle_mode(oracle, mode, shift), list(x)))
        if shift == 1:
            plain[mode] = want
        if log_n <= 10:  # the oracle's NTT is not the only reference: plain O(n^2) evaluation on the coset
            for c in range(len(x)):
                tag = "log_n=%d plan=%s naive, mode=%s shift=%s" % (log_n, plan, mode, sname)
                if mode.endswith("ifft"):
                    assert_same(oracle.naive_coset_eval(want[c], shift), xc[c], tag, names[c:])
                else:
                    assert_same(want[c], oracle.naive_coset_eval(x[c], shift), tag, names[c:])
        for v, ctx in enumerate(variants):
            got = run_mode(pb, ctx, x, mode, shift)
            assert_same(got, want, "log_n=%d plan=%s variant=%d mode=%s shift=%s" % (log_n, plan, v, mode, sname), names)


# ----------------------------------------------------------------------------- 2. three-pass plans up to 2^27
def spot_indices(log_n, seed):
    """k = 0, 1, n/2, n-1 and indices in different row blocks of every pass (output k = k1 + R*k2)."""
    n = 1 << log_n
    a1, a2, b = ntt_plan(log_n)
    R = 1 << (log_n - b)
    rng = np.random.default_rng(seed)
    ks = {0, 1, n // 2, n - 1, R - 1, R + 1, n - R, (1 << a1) + 3, int(rng.integers(0, n))}
    return sorted(ks)


@pytest.mark.parametrize("log_n", [23, 24, 25, 26, 27])
def test_ntt_large_plans(pb, oracle, variants, log_n):
    """One column per transform. Values are spot-checked by Horner evaluation of the input at shift * w_n^k; the
    constant column is checked at every index (fft of c is (n*c, 0, ..., 0)), and inverse(forward(x)) == x."""
    n = 1 << log_n
    plan = ntt_plan(log_n)
    w = int(oracle.lib().glo_primitive_root_of_unity(log_n))
    shift = SHIFTS[0][1]
    ks = spot_indices(log_n, log_n)
    for cname, x in [("random non-canonical", synth(0x7100 + log_n, (n,), canonical=False)),
                     ("square 2^%d" % (log_n - plan[0] + plan[0] // 2 + 1), square(n, log_n - plan[0] + plan[0] // 2 + 1)),
                     ("all 2^64-1", np.full(n, M64, dtype=np.uint64))]:
        xc = x % np.uint64(P)
        want = {}
        if cname.startswith("all"):
            want["fft"] = np.zeros(n, dtype=np.uint64)
            want["fft"][0] = n * M64 % P
        else:
            pts = [(s, k) for s in (1, shift) for k in ks]
            vals = _pmap(lambda sk: oracle.eval_poly_base_at_ext(xc, (sk[0] * pow(w, sk[1], P) % P, 0))[0], pts)
            want["spot"] = dict(zip(pts, vals))
        for v, ctx in enumerate(variants):
            names = [cname]
            for mode, s in (("fft", 1), ("coset_fft", shift)):
                got = run_mode(pb, ctx, x, mode, s)
                tag = "log_n=%d plan=%s variant=%d mode=%s" % (log_n, plan, v, mode)
                if mode == "fft" and "fft" in want:
                    assert_same(got, want["fft"], tag, names)
                if "spot" in want:
                    for k in ks:
                        assert int(got[k]) == want["spot"][(s, k)], "%s, input class=%s, column=0, index=%d" % (tag, cname, k)
                back = run_mode(pb, ctx, got, "ifft" if s == 1 else "coset_ifft", s)
                assert_same(back, xc, tag + " round trip", names)
                del got, back


# ----------------------------------------------------------------------------- 3. groups of columns
def _to_dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64).copy()).cuda()


def _to_np(t):
    return t.cpu().numpy().view(np.uint64)


def _leaf_ref(oracle, coeffs, rate_bits, rows, full=None):
    """Leaf rows of a commitment of `coeffs`: leaf j, column k = P_k(g * w_N^bitrev(j)), i.e. the natural-order coset
    fft of the zero-padded coefficients at the bit-reversed position. `full`: compute the whole coset fft instead of
    Horner evaluations at the rows."""
    B, n = coeffs.shape
    logN = int(np.log2(n)) + rate_bits
    N = 1 << logN
    g = int(oracle.lib().glo_coset_shift())
    cc = coeffs % np.uint64(P)
    br = [int(oracle.lib().glo_reverse_bits(int(j), logN)) for j in rows]
    if full:
        pad = np.zeros((B, N), dtype=np.uint64)
        pad[:, :n] = cc
        lde = np.stack(_pmap(lambda c: oracle.coset_fft(c, g), list(pad)))
        return lde[:, br].T.copy()
    wN = int(oracle.lib().glo_primitive_root_of_unity(logN))
    pts = [(k, b) for b in br for k in range(B)]
    vals = _pmap(lambda kb: oracle.eval_poly_base_at_ext(cc[kb[0]], (g * pow(wN, kb[1], P) % P, 0))[0], pts)
    return np.array(vals, dtype=np.uint64).reshape(len(rows), B)


@pytest.mark.parametrize("log_n", [11, 13, 19, 21, 24])
def test_ntt_groups(pb, oracle, grouped, log_n):
    """13 columns on 8-column groups (the second group short): gl_ntt on device columns with a stride > n, gl_ntt_bcast
    to 3 destinations, and from_values / from_coeffs."""
    from plonky2_b200 import _native as N

    n, B, pad = 1 << log_n, 13, 24
    stride = n + pad
    plan = ntt_plan(log_n)
    names = ["column %d" % b for b in range(B)]
    x = synth(0x7200 + log_n, (B, stride), canonical=False)
    x[3, :n] = M64
    x[11, :n] = square(n, 1)
    shift = 7
    want_fwd = np.stack(_pmap(lambda c: oracle.coset_fft(c[:n], shift), list(x)))
    want_inv = np.stack(_pmap(lambda c: oracle.ifft(c[:n]), list(x)))
    rows = sorted({0, 1, n - 1, n, n + 1, 2 * n - 1})
    vals = np.ascontiguousarray(x[:, :n])
    coeffs = {"values": want_inv, "coeffs": vals % np.uint64(P)}
    leaf_ref = {k: _leaf_ref(oracle, coeffs[k], 1, rows) for k in coeffs} if log_n > 13 else {}
    for v, ctx in enumerate(grouped):
        tag = "log_n=%d plan=%s variant=%d" % (log_n, plan, v)
        d = _to_dev(x)
        N.check(N.lib().gl_ntt(ctx.h, N.vp(d.data_ptr()), log_n, B, stride, 0, 0, shift, N.MEM_DEVICE), ctx.h)
        ctx.synchronize()
        got = _to_np(d)
        assert_same(got[:, :n], want_fwd, tag + " mode=coset_fft (gl_ntt, device, stride n+%d)" % pad, names)
        assert_same(got[:, n:], x[:, n:], tag + " padding", names)
        del d
        # gl_ntt_bcast: 3 destinations, column b at row b + 1 of each
        import torch

        src = _to_dev(x)
        dests = [torch.zeros((B + 2, stride), dtype=torch.int64, device="cuda") for _ in range(3)]
        torch.cuda.synchronize()
        outs = (N.vp * 3)(*[N.vp(dd[1:].data_ptr()) for dd in dests])
        N.check(N.lib().gl_ntt_bcast(ctx.h, N.vp(src.data_ptr()), stride, log_n, B, 1, outs, 3, stride), ctx.h)
        ctx.synchronize()
        for i, dd in enumerate(dests):
            gd = _to_np(dd)
            assert_same(gd[1:B + 1, :n], want_inv, tag + " mode=ifft (gl_ntt_bcast destination %d)" % i, names)
            assert not gd[0].any() and not gd[B + 1].any() and not gd[1:B + 1, n:].any(), tag + " bcast wrote outside"
        assert np.array_equal(_to_np(src), x), tag + " bcast changed its input"
        del src, dests
        # commitments
        for kind in ("values", "coeffs"):
            mk = pb.PolynomialBatch.from_values if kind == "values" else pb.PolynomialBatch.from_coeffs
            c = mk(vals, 1, False, 2, ctx=ctx)
            try:
                assert_same(c.polynomials, coeffs[kind], tag + " from_%s coefficients" % kind, names)
                if log_n <= 13:
                    o = oracle.Commit(vals, 1, 2, is_coeffs=kind == "coeffs")
                    leaves = c.merkle_tree.leaves
                    bad = np.nonzero(leaves != o.leaves)
                    assert not bad[0].size, "%s from_%s leaf %d column %d" % (tag, kind, bad[0][0], bad[1][0])
                    assert np.array_equal(c.merkle_tree.cap.hashes, o.cap), tag + " cap"
                else:
                    ref = leaf_ref[kind]
                    for i, r in enumerate(rows):
                        got_r = c.merkle_tree.get_rows(r, 1)[0]
                        bad = np.nonzero(got_r != ref[i])[0]
                        assert not bad.size, "%s from_%s leaf %d column %d" % (tag, kind, r, bad[0])
            finally:
                c.close()


# ----------------------------------------------------------------------------- 4. coset LDE (bit-reversed row pass) for every plan
@pytest.mark.parametrize("log_n", range(1, 23))
def test_lde_every_plan(pb, oracle, variants, log_n):
    """from_coeffs at rate_bits 1 and 3: every coset block (the row pass's bit-reversed stores at offset row0)
    against the zero-padded coset fft of the coefficients at bit-reversed positions."""
    n = 1 << log_n
    plan = ntt_plan(log_n)
    cols = np.stack([synth(0x7300 + log_n, (n,), canonical=False), np.full(n, M64, dtype=np.uint64),
                     np.resize(np.array(EDGE, dtype=np.uint64), n)])
    names = ["random non-canonical", "all 2^64-1", "EDGE tiled"]
    for r in (1, 3):
        N = n << r
        if N <= 1 << 16:
            rows = list(range(N))
        else:  # a few rows of every coset block c (leaf rows c*n .. c*n + n - 1)
            rng = np.random.default_rng(log_n * 8 + r)
            rows = sorted({c * n + j for c in range(1 << r) for j in (0, 1, n - 1, int(rng.integers(0, n)))})
        ref = _leaf_ref(oracle, cols, r, rows, full=N <= 1 << 18)
        for v, ctx in enumerate(variants):
            tag = "log_n=%d plan=%s variant=%d mode=lde rate_bits=%d" % (log_n, plan, v, r)
            c = pb.PolynomialBatch.from_coeffs(cols, r, False, min(2, log_n + r), ctx=ctx)
            try:
                assert_same(c.polynomials, cols % np.uint64(P), tag + " coefficients", names)
                got = c.merkle_tree.get_rows(0, N) if len(rows) == N else np.stack([c.merkle_tree.get_rows(j, 1)[0] for j in rows])
                bad = np.nonzero(got != ref)
                if bad[0].size:
                    i, k = int(bad[0][0]), int(bad[1][0])
                    raise AssertionError("%s, input class=%s, column=%d, index=leaf %d (coset block %d): got %#x want %#x"
                                         % (tag, names[k], k, rows[i], rows[i] // n, int(got[i, k]), int(ref[i, k])))
            finally:
                c.close()


# ----------------------------------------------------------------------------- 5. more columns than gridDim.y allows
@pytest.mark.parametrize("log_n", [1, 2])
@pytest.mark.parametrize("batch", [65535, 65536])
def test_coset_ifft_more_columns_than_grid_y(pb, oracle, log_n, batch):
    """The coset-inverse scaling runs one column per blockIdx.y (at most 65535): wider batches are launched in
    chunks, so every column of a 65536-column coset_ifft is right."""
    n = 1 << log_n
    x = synth(0x7400 + log_n, (batch, n), canonical=False)
    shift = 7
    got = pb.coset_ifft(x, shift)
    want = np.stack([oracle.coset_ifft(c, shift) for c in x])
    assert_same(got, want, "log_n=%d batch=%d mode=coset_ifft" % (log_n, batch), ["column"] * batch)
    assert np.array_equal(pb.coset_fft(got, shift), x % np.uint64(P))


def test_sharded_commit_more_columns_than_grid_y(pb, oracle):
    """A row-block shard smaller than n restricts the polynomials to its coset first (k_fold_coeffs, one column per
    blockIdx.y): 65536 device columns of degree 2 in one call, on 2 shards, rate_bits 0."""
    from plonky2_b200 import _native as N

    B, n = 65536, 2
    vals = synth(0x7500, (B, n))
    o = oracle.Commit(vals, 0, 1, is_coeffs=True)
    d = _to_dev(vals)
    ctx = pb.default_context()
    for g in range(2):
        h = N.vp()
        N.check(N.lib().gl_commit_create_sharded(ctx.h, N.vp(d.data_ptr()), n, B, 1, 0, 1, None, 1, N.MEM_DEVICE, g, 2,
                                                 C.byref(h)), ctx.h)
        c = pb.PolynomialBatch(h, ctx, B, 1, 0, 1, False, shard=(g, 2))
        try:
            assert np.array_equal(c.merkle_tree.get_rows(0, 1)[0], o.leaves[g]), g
        finally:
            c.close()
