"""FRI's opening composition in both domains, and the batch-FRI mix, against an exact evaluator.

The first codeword of every FRI proof is, at the LDE leaf j with x_j = g * w_N^{bitrev(j)} (oracle.rs:186-220,
reducing.rs:83-106),
    c(x_j) = sum_b alpha^{k_b} (F_b(x_j) - F_b(z_b)) / (x_j - z_b),   F_b = sum_i alpha^i f_{b,i},
with k_b the number of polynomials in the batches after b. The library builds it twice: gl_fri_begin composes the
coefficients, divides by (X - z_b) with a three-phase suffix scan (k_div_by_x for z_b = 0) and takes the coset LDE;
gl_fri_begin_values evaluates the formula at each leaf from the commitments' LDE rows, shard by shard. `compose` below
is the formula in exact arithmetic (tests/gl_numpy.py), reading f_{b,i}(x_j) by Horner from the coefficients or from
the oracle's LDE rows. The CPU test pins it to the oracle's prove_openings; the gpu tests (run with `-m gpu` on an
H100) compare both device codewords with it and with each other: every size to 2^17 leaves, 1..9 batches, batches of
up to 234 polynomials with repeated references, every kind of point and of commitment handle, row-block shards at every
G through the FRI rounds, the benchmarked cfg2 and cfg5 shapes, and gl_fri_mix from 2^1 to 2^25 elements.
"""
import ctypes as C
import os

import numpy as np
import pytest

import gl_numpy as G
from conftest import P, synth

SHIFT = 14293326489335486720                # MULTIPLICATIVE_GROUP_GENERATOR (goldilocks_field.rs), the LDE coset's shift
TWO_ADIC_ROOT = 7277203076849721926         # POWER_OF_TWO_GENERATOR: a primitive 2^32-th root of unity
XTAB = 4096                                 # the device's w^i = hi[i >> 12] * lo[i & 4095] table split


def root(log):
    return pow(TWO_ADIC_ROOT, 1 << (32 - log), P)


# ----------------------------------------------------------------------------- F_{p^2} = F_p[X] / (X^2 - 7), scalars
def e2_add(x, y):
    return (x[0] + y[0]) % P, (x[1] + y[1]) % P


def e2_mul(x, y):
    return (x[0] * y[0] + 7 * x[1] * y[1]) % P, (x[0] * y[1] + x[1] * y[0]) % P


def e2_pow(x, e):
    r = (1, 0)
    while e:
        if e & 1:
            r = e2_mul(r, x)
        x = e2_mul(x, x)
        e >>= 1
    return r


# ----------------------------------------------------------------------------- the exact evaluator
def leaf_points(leaves, log_N):
    """x_j = g * w_N^{bitrev(j)} for the leaf indices j (the LDE row of leaf j is reverse_bits(j), oracle.rs:142-147)."""
    i = G.brev(np.asarray(leaves, dtype=np.uint64), log_N)
    out, sq = np.ones(len(i), dtype=np.uint64), root(log_N)
    for k in range(log_N):
        bit = ((i >> np.uint64(k)) & np.uint64(1)).astype(bool)
        out = np.where(bit, G.mul(out, np.uint64(sq)), out)
        sq = sq * sq % P
    return G.mul(out, np.uint64(SHIFT))


def horner_columns(coeffs, x):
    """f(x) for every coefficient row of `coeffs` (num_polys, n) at every base-field x: (num_polys, len(x))."""
    out = np.zeros((coeffs.shape[0], len(x)), dtype=np.uint64)
    for k in range(coeffs.shape[1] - 1, -1, -1):
        out = G.add(G.mul(out, x[None, :]), coeffs[:, k:k + 1])
    return out


def compose(leaves, log_N, batches, alpha, opened, f_at):
    """(c0, c1) arrays: the composed codeword at `leaves`. batches = [(z_b, [(oracle, poly), ...])], opened[b][i] =
    f_{b,i}(z_b) in F_{p^2}, f_at(oracle, poly) = that polynomial's values at `leaves` (base field)."""
    x = leaf_points(leaves, log_N)
    zero = np.zeros(len(x), dtype=np.uint64)
    acc0, acc1 = zero, zero
    for (z, refs), ys in zip(batches, opened):
        # F_b(x) and F_b(z_b) with alpha^i, i counted from 0 in every batch (reduce_polys_base, reducing.rs:83-95)
        s0, s1, y, a = zero, zero, (0, 0), (1, 0)
        for (o, p), yv in zip(refs, ys):
            f = f_at(o, p)
            s0, s1 = G.add(s0, G.mul(f, np.uint64(a[0]))), G.add(s1, G.mul(f, np.uint64(a[1])))
            y = e2_add(y, e2_mul(a, (int(yv[0]), int(yv[1]))))
            a = e2_mul(a, alpha)
        # the quotient (F_b(x) - F_b(z_b)) / (x - z_b): times (d0 - d1 X) / (d0^2 - 7 d1^2) with d = x - z_b
        d0, d1 = G.sub(x, np.uint64(z[0] % P)), (P - z[1] % P) % P
        norm = G.sub(G.mul(d0, d0), np.uint64(7 * d1 * d1 % P))
        assert not np.any(norm == 0), "an opening point lies on the LDE coset"
        inv = G.pow_scalar(norm, P - 2)
        n0, n1 = G.sub(s0, np.uint64(y[0])), G.sub(s1, np.uint64(y[1]))
        q0 = G.mul(G.sub(G.mul(n0, d0), G.mul(n1, np.uint64(7 * d1 % P))), inv)
        q1 = G.mul(G.sub(G.mul(n1, d0), G.mul(n0, np.uint64(d1))), inv)
        # alpha.shift_poly(&mut final_poly); final_poly += quotient (reducing.rs:102-106): acc * alpha^{|batch|} + q
        sh = e2_pow(alpha, len(refs))
        m0, m1 = G.ext_mul((acc0, acc1), (np.uint64(sh[0]), np.uint64(sh[1])))
        acc0, acc1 = G.add(m0, q0), G.add(m1, q1)
    return acc0, acc1


def openings(coeffs, batches, oracle):
    """opened[b][i] = f_{b,i}(z_b), Horner in F_{p^2} by the CPU oracle. coeffs[o] = (num_polys, n)."""
    return [np.array([oracle.eval_poly_base_at_ext(coeffs[o][p], z) for o, p in refs], dtype=np.uint64).reshape(-1, 2)
            for z, refs in batches]


def point_kinds(log_n, seed):
    """The opening points the prover meets, and the ones it might: F_{p^2}, F_p, zeta * w_n, 0 and a point of H (off the
    shifted LDE coset)."""
    r = [int(v) for v in synth(seed, (6,))]
    zeta = (r[0], r[1])
    return {"ext": zeta, "base": (r[2], 0), "zeta_w": e2_mul(zeta, (root(log_n), 0)), "zero": (0, 0),
            "H": (pow(root(log_n), r[3] % (1 << log_n), P), 0), "ext2": (r[4], r[5])}


def sample_leaves(log_N, seed, shards=(1, 2, 4, 8, 16), count=4096):
    """`count` seeded leaves, the first and last leaf of every shard of each G, and the leaves whose LDE index i is
    on either side of a multiple of 4096 (where the device's w^i table steps to its next high entry)."""
    N = 1 << log_N
    rng = np.random.default_rng(seed)
    picks = [rng.integers(0, N, size=min(count, N), dtype=np.uint64)]
    for g_count in shards:
        if g_count <= N:
            edges = np.arange(g_count, dtype=np.uint64) * np.uint64(N // g_count)
            picks += [edges, edges + np.uint64(N // g_count - 1)]
    m = np.arange(0, N, XTAB, dtype=np.uint64)
    picks += [G.brev(m, log_N), G.brev(np.maximum(m, np.uint64(1)) - np.uint64(1), log_N)]
    return np.unique(np.concatenate(picks))


def as_pairs(c0, c1):
    return np.stack([c0, c1], axis=1)


# ----------------------------------------------------------------------------- CPU: the evaluator against the oracle
@pytest.mark.parametrize("log_n,r,kinds", [(0, 1, ("ext",)), (2, 1, ("ext", "zeta_w")), (3, 2, ("zero", "base", "ext")),
                                           (4, 3, ("H", "ext", "zero")), (5, 1, ("ext", "base", "zeta_w", "H"))])
def test_evaluator_matches_oracle_prove_openings(oracle, log_n, r, kinds):
    """The evaluator's value at every leaf equals the oracle's composed polynomial (its prove_openings final_poly tap,
    the coefficients before the LDE) evaluated at that leaf's point; the f_{b,i} are read by Horner and from the oracle's
    LDE rows, with repeated references inside and across batches."""
    n, N = 1 << log_n, 1 << (log_n + r)
    coeffs = [synth(0x5C00 + log_n, (3, n)), synth(0x5C10 + log_n, (2, n))]
    pts = point_kinds(log_n, 0x5C20 + log_n)
    refs = [[(0, 0), (1, 1), (0, 2), (0, 0)], [(1, 0), (0, 2)], [(0, 1)], [(1, 1), (1, 1), (0, 0)]]
    batches = [(pts[k], refs[b % len(refs)]) for b, k in enumerate(kinds)]
    commits = [oracle.Commit(c, r, 0, is_coeffs=True) for c in coeffs]
    ch = oracle.Challenger()
    ch.observe_elements(synth(0x5C30, (8,)))
    alpha = ch.clone().get_extension_challenge()
    _, taps = oracle.prove_openings(commits, batches, ch, oracle.make_params(r, 0, 0, 2, []), taps=True)
    final = taps["final_poly"]
    leaves = np.arange(N, dtype=np.uint64)
    x = leaf_points(leaves, log_n + r)
    want0, want1 = [horner_columns(np.ascontiguousarray(final[:, k])[None, :], x)[0] for k in (0, 1)]
    opened = openings(coeffs, batches, oracle)
    by_horner = [horner_columns(c, x) for c in coeffs]
    lde = [c.leaves for c in commits]
    for f_at in (lambda o, p: by_horner[o][p], lambda o, p: lde[o][:, p]):
        got0, got1 = compose(leaves, log_n + r, batches, alpha, opened, f_at)
        assert np.array_equal(got0, want0) and np.array_equal(got1, want1)


def test_sample_leaves_cover_the_table_steps_and_shard_edges():
    log_N = 17
    s = set(int(v) for v in sample_leaves(log_N, 1))
    N = 1 << log_N
    for g_count in (2, 16):
        for g in range(g_count):
            assert g * N // g_count in s and (g + 1) * N // g_count - 1 in s
    for m in (XTAB, 5 * XTAB, N - XTAB):
        for i in (m - 1, m):
            assert int(G.brev(np.array([i], dtype=np.uint64), log_N)[0]) in s


# ----------------------------------------------------------------------------- device helpers
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


def _batch_array(batches):
    from plonky2_b200 import _native as N

    barr = (N.FriBatch * len(batches))()
    keep = []
    for i, (z, refs) in enumerate(batches):
        oi = np.array([o for o, _ in refs], dtype=np.uint32)
        pi = np.array([p for _, p in refs], dtype=np.uint32)
        keep += [oi, pi]
        barr[i].point[0], barr[i].point[1] = z[0] % P, z[1] % P
        barr[i].num_polys = len(refs)
        barr[i].oracle_index = oi.ctypes.data_as(N.u32p)
        barr[i].poly_index = pi.ctypes.data_as(N.u32p)
    return barr, keep


class Fri:
    """One gl_fri handle, destroyed on close."""

    def __init__(self, h, ctx):
        self.h, self.ctx = h, ctx

    def _read(self):
        from plonky2_b200 import _native as N

        L = N.lib()
        size = 2
        while True:  # the local length is 2^(log_cur - shard_log); grow the buffer until it fits
            buf = np.empty(2 * size, dtype=np.uint64)
            ln = C.c_size_t()
            rc = L.gl_fri_values_local(self.h, N.np_ptr(buf), buf.size, C.byref(ln))
            if rc == N.GL_OK:
                return buf[:2 * ln.value].reshape(-1, 2)
            msg = L.gl_last_error(self.ctx.h)
            if b"too small" not in (msg or b""):
                N.check(rc, self.ctx.h)
            size *= 2

    def close(self):
        from plonky2_b200 import _native as N

        if self.h:
            N.lib().gl_fri_destroy(self.h)
            self.h = None


def begin_values(pb, commits, batches, alpha, opened, cap_height=0):
    from plonky2_b200 import _native as N

    ctx = commits[0].ctx
    barr, keep = _batch_array(batches)  # keep: the index arrays barr points into
    handles = (N.vp * len(commits))(*[c.h for c in commits])
    op = np.ascontiguousarray(np.concatenate([np.asarray(o, dtype=np.uint64).reshape(-1, 2) for o in opened]).reshape(-1))
    al = np.array([alpha[0], alpha[1]], dtype=np.uint64)
    h = N.vp()
    N.check(N.lib().gl_fri_begin_values(ctx.h, handles, len(commits), barr, len(batches), N.np_ptr(op), N.np_ptr(al),
                                        cap_height, C.byref(h)), ctx.h)
    return Fri(h, ctx)


def begin_coeffs(pb, commits, batches, alpha, rate_bits, cap_height=0):
    from plonky2_b200 import _native as N

    ctx = commits[0].ctx
    barr, keep = _batch_array(batches)  # keep: the index arrays barr points into
    handles = (N.vp * len(commits))(*[c.h for c in commits])
    al = np.array([alpha[0], alpha[1]], dtype=np.uint64)
    h = N.vp()
    N.check(N.lib().gl_fri_begin(ctx.h, handles, len(commits), barr, len(batches), N.np_ptr(al), rate_bits, cap_height,
                                 C.byref(h)), ctx.h)
    return Fri(h, ctx)


def both_codewords(pb, commits, batches, alpha, opened, rate_bits, cap_height=0):
    """(value-domain codeword, coefficient-domain codeword), each (N, 2) in leaf order."""
    out = []
    for make in (lambda: begin_values(pb, commits, batches, alpha, opened, cap_height),
                 lambda: begin_coeffs(pb, commits, batches, alpha, rate_bits, cap_height)):
        f = make()
        try:
            out.append(f._read())
        finally:
            f.close()
    return out


def first_diff(got, want):
    bad = np.argwhere(np.any(got != want, axis=1))
    return "first wrong leaf %d of %d (%d wrong)" % (int(bad[0][0]), len(want), len(bad)) if bad.size else "equal"


def check_case(pb, oracle, coeffs, batches, alpha, rate_bits, commits=None, leaves=None, cap_height=0):
    """Both device codewords of the instance against each other and the evaluator (every leaf unless `leaves`).
    coeffs[o] = (num_polys, n) host coefficients; commits default to from_coeffs handles of them."""
    log_n = int(coeffs[0].shape[1]).bit_length() - 1
    log_N = log_n + rate_bits
    own = commits is None
    if own:
        commits = [pb.PolynomialBatch.from_coeffs(c, rate_bits, False, cap_height) for c in coeffs]
    try:
        opened = openings(coeffs, batches, oracle)
        vals, co = both_codewords(pb, commits, batches, alpha, opened, rate_bits, cap_height)
    finally:
        if own:
            for c in commits:
                c.close()
    assert np.array_equal(vals, co), "value vs coefficient domain: " + first_diff(vals, co)
    leaves = np.arange(1 << log_N, dtype=np.uint64) if leaves is None else leaves
    if (1 << log_n) * len(leaves) <= 1 << 16:
        x = leaf_points(leaves, log_N)
        cols = [horner_columns(c, x) for c in coeffs]
        f_at = lambda o, p: cols[o][p]  # noqa: E731
    else:
        rows = [oracle.Commit(c, rate_bits, 0, is_coeffs=True).leaf_rows(leaves) for c in coeffs]
        f_at = lambda o, p: rows[o][:, p]  # noqa: E731
    want = as_pairs(*compose(leaves, log_N, batches, alpha, opened, f_at))
    got = vals[leaves.astype(np.int64)]
    assert np.array_equal(got, want), "device vs evaluator: " + first_diff(got, want)
    return vals


# ----------------------------------------------------------------------------- every size, batch count and width
@pytest.mark.gpu
@pytest.mark.parametrize("rate_bits", [1, 2, 3])
@pytest.mark.parametrize("log_n", list(range(15)))
def test_every_size(pb, oracle, log_n, rate_bits):
    """log_n 0..14 at rates 1..3: codewords of 2 .. 2^17 leaves, across the 2^12 and 2^13 steps of the w^i table;
    a plonky2-shaped instance (everything at zeta, two columns at zeta * w_n), every leaf."""
    n = 1 << log_n
    coeffs = [synth(0x5D00 + log_n, (3, n)), synth(0x5D20 + log_n, (2, n))]
    pts = point_kinds(log_n, 0x5D40 + log_n)
    batches = [(pts["ext"], [(0, 0), (0, 1), (0, 2), (1, 0), (1, 1)]), (pts["zeta_w"], [(0, 1), (1, 0)])]
    alpha = tuple(int(v) for v in synth(0x5D60 + log_n, (2,)))
    check_case(pb, oracle, coeffs, batches, alpha, rate_bits)


def _spread(count, widths, seed):
    """`count` (oracle, poly) references over oracles of the given widths, with repeats."""
    rng = np.random.default_rng(seed)
    o = rng.integers(0, len(widths), size=count)
    return [(int(a), int(rng.integers(0, widths[a]))) for a in o]


@pytest.mark.gpu
@pytest.mark.parametrize("n_batches", list(range(1, 10)))
def test_batch_counts(pb, oracle, n_batches):
    """1..8 batches, each at another kind of point, over 4 oracles with references repeated inside and across batches,
    on a codeword of 2^13 leaves; 9 batches are refused by the value domain (its kernel holds 8) and still composed
    by the coefficient domain."""
    from plonky2_b200 import _native as N

    log_n, r = 11, 2
    widths = (3, 5, 2, 4)
    coeffs = [synth(0x5E00 + k, (w, 1 << log_n)) for k, w in enumerate(widths)]
    pts = point_kinds(log_n, 0x5E10 + n_batches)
    kinds = ["ext", "base", "zeta_w", "zero", "H", "ext2", "ext", "base", "zeta_w"]
    batches = [(pts[kinds[b]], _spread(1 + (3 * b) % 7, widths, 0x5E20 + 16 * n_batches + b)) for b in range(n_batches)]
    batches[0] = (batches[0][0], batches[0][1] + [batches[0][1][0]])  # a repeat inside a batch
    alpha = tuple(int(v) for v in synth(0x5E30 + n_batches, (2,)))
    if n_batches <= 8:
        check_case(pb, oracle, coeffs, batches, alpha, r)
        return
    commits = [pb.PolynomialBatch.from_coeffs(c, r, False, 0) for c in coeffs]
    try:
        opened = openings(coeffs, batches, oracle)
        with pytest.raises(N.NativeError, match="native error 4: more than 8 opening batches"):
            begin_values(pb, commits, batches, alpha, opened)
        f = begin_coeffs(pb, commits, batches, alpha, r)
        try:
            co = f._read()
        finally:
            f.close()
    finally:
        for c in commits:
            c.close()
    leaves = sample_leaves(log_n + r, 0x5E40, count=512)
    rows = [oracle.Commit(c, r, 0, is_coeffs=True).leaf_rows(leaves) for c in coeffs]
    want = as_pairs(*compose(leaves, log_n + r, batches, alpha, opened, lambda o, p: rows[o][:, p]))
    assert np.array_equal(co[leaves.astype(np.int64)], want), first_diff(co[leaves.astype(np.int64)], want)


@pytest.mark.gpu
@pytest.mark.parametrize("width", [1, 2, 135, 234])
def test_batch_widths(pb, oracle, width):
    """Batches of 1, 2, 135 and 234 polynomials (the benchmarked circuits' widths) over 4 oracles, repeated
    references inside a batch and across the two batches, a codeword of 2^13 leaves."""
    log_n, r = 10, 3
    widths = (70, 64, 60, 40)
    coeffs = [synth(0x5F00 + k, (w, 1 << log_n)) for k, w in enumerate(widths)]
    pts = point_kinds(log_n, 0x5F10 + width)
    first = _spread(width, widths, 0x5F20 + width)
    batches = [(pts["ext"], first), (pts["zeta_w"], first[:2] + _spread(max(1, width // 3), widths, 0x5F30 + width))]
    alpha = tuple(int(v) for v in synth(0x5F40 + width, (2,)))
    check_case(pb, oracle, coeffs, batches, alpha, r, leaves=sample_leaves(log_n + r, 0x5F50 + width))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ext", "base", "zeta_w", "zero", "H"])
def test_point_kinds(pb, oracle, kind):
    """Each kind of point alone and next to a generic one, every leaf of a 2^14-leaf codeword."""
    log_n, r = 12, 2
    coeffs = [synth(0x6000, (4, 1 << log_n))]
    pts = point_kinds(log_n, 0x6010)
    alpha = tuple(int(v) for v in synth(0x6020, (2,)))
    check_case(pb, oracle, coeffs, [(pts[kind], [(0, 0), (0, 3), (0, 1)])], alpha, r)
    check_case(pb, oracle, coeffs, [(pts["ext2"], [(0, 2)]), (pts[kind], [(0, 1), (0, 2)])], alpha, r)


@pytest.mark.gpu
def test_point_on_the_lde_coset_is_refused(pb, oracle):
    """A point x_j of the LDE coset divides by zero at leaf j: the value domain refuses it."""
    log_n, r = 6, 2
    coeffs = [synth(0x6100, (2, 1 << log_n))]
    z = (int(leaf_points(np.array([37], dtype=np.uint64), log_n + r)[0]), 0)
    commits = [pb.PolynomialBatch.from_coeffs(coeffs[0], r, False, 0)]
    try:
        batches = [(z, [(0, 0), (0, 1)])]
        with pytest.raises(ZeroDivisionError, match="Opening point is in the LDE domain"):
            begin_values(pb, commits, batches, (3, 5), openings(coeffs, batches, oracle))
    finally:
        commits[0].close()


# ----------------------------------------------------------------------------- every kind of handle
@pytest.mark.gpu
@pytest.mark.parametrize("handle", ["from_values", "from_coeffs", "incremental", "keyed", "salted"])
def test_handle_kinds(pb, oracle, handle):
    """Commitments made every way, on a 2^14-leaf codeword: the salted ones have leaf width B + 4, and their salt
    columns neither enter the sum nor can be referenced."""
    from plonky2_b200 import _native as N

    log_n, r, h = 12, 2, 3
    n = 1 << log_n
    vals = [synth(0x6200 + k, (w, n)) for k, w in enumerate((5, 3))]
    coeffs = [oracle.Commit(v, 0, 0).coeffs for v in vals]
    ctx = pb.default_context()

    def make(k):
        v = vals[k]
        if handle == "from_values":
            return pb.PolynomialBatch.from_values(v, r, False, h)
        if handle == "from_coeffs":
            return pb.PolynomialBatch.from_coeffs(coeffs[k], r, False, h)
        if handle == "keyed":
            return pb.PolynomialBatch.from_values(v, r, True, h, salt_key=bytes(range(k, 32 + k)))
        if handle == "salted":
            return pb.PolynomialBatch.from_values(v, r, True, h, salt=synth(0x6210 + k, (4, n << r)))

        def add_columns(hh):  # one column at a time, values then coefficients
            for j in range(v.shape[0]):
                src = np.ascontiguousarray(v[j:j + 1] if j % 2 else coeffs[k][j:j + 1])
                N.check(N.lib().gl_commit_add_columns(hh, j, 1, N.np_ptr(src), n,
                                                      N.COLS_VALUES if j % 2 else N.COLS_COEFFS, N.MEM_HOST), ctx.h)
        return pb.PolynomialBatch._from_device(ctx, v.shape[0], log_n, r, h, add_columns)

    commits = [make(0), make(1)]
    try:
        if handle in ("keyed", "salted"):
            assert all(c.leaf_width == c.num_polys + 4 for c in commits)
        pts = point_kinds(log_n, 0x6220)
        batches = [(pts["ext"], [(0, j) for j in range(5)] + [(1, j) for j in range(3)]),
                   (pts["zeta_w"], [(0, 4), (1, 2)])]
        alpha = tuple(int(v) for v in synth(0x6230, (2,)))
        check_case(pb, oracle, coeffs, batches, alpha, r, commits=commits, cap_height=h)
        bad = [(pts["ext"], [(0, 0), (1, 3)])]
        for call in (lambda: begin_values(pb, commits, bad, alpha, [np.zeros((2, 2), dtype=np.uint64)], h),
                     lambda: begin_coeffs(pb, commits, bad, alpha, r, h)):
            with pytest.raises(N.NativeError, match="native error 5: bad polynomial reference"):
                call()
    finally:
        for c in commits:
            c.close()


@pytest.mark.gpu
def test_non_resident_handles(pb, oracle):
    """A non-resident commitment (lde_blocks) has no LDE rows: the value domain refuses it, the coefficient domain
    composes it to the resident commitment's codeword."""
    from plonky2_b200 import _native as N

    log_n, r, h = 12, 2, 4
    vals = synth(0x6300, (4, 1 << log_n))
    res = pb.PolynomialBatch.from_values(vals, r, False, h)
    blk = pb.PolynomialBatch.from_values(vals, r, False, h, lde_blocks=4)
    try:
        pts = point_kinds(log_n, 0x6310)
        batches = [(pts["ext"], [(0, 0), (0, 1), (0, 2), (0, 3)]), (pts["zeta_w"], [(0, 1)])]
        alpha = tuple(int(v) for v in synth(0x6320, (2,)))
        coeffs = [oracle.Commit(vals, 0, 0).coeffs]
        opened = openings(coeffs, batches, oracle)
        with pytest.raises(N.NativeError, match="native error 5: a non-resident commitment has no LDE to read"):
            begin_values(pb, [blk], batches, alpha, opened, h)
        got = []
        for c in (res, blk):
            f = begin_coeffs(pb, [c], batches, alpha, r, h)
            try:
                got.append(f._read())
            finally:
                f.close()
        assert np.array_equal(got[0], got[1])
        vals_res = check_case(pb, oracle, coeffs, batches, alpha, r, commits=[res], cap_height=h,
                              leaves=sample_leaves(log_n + r, 0x6330))
        assert np.array_equal(vals_res, got[1])
    finally:
        res.close()
        blk.close()


# ----------------------------------------------------------------------------- row-block shards through the rounds
def _gather(states):
    return np.concatenate([s._read() for s in states])


@pytest.mark.gpu
@pytest.mark.parametrize("shards", [1, 2, 4, 8, 16])
def test_row_block_shards_through_the_rounds(pb, oracle, shards):
    """Value-domain states over G row-block shards at cap height 4 and 2^17 leaves (every shard reads several w^i
    table entries): the local blocks in shard order are the unsharded codeword word for word, and stay so after each
    commit (whose cap entries in shard order are the unsharded cap) and fold; the final polynomials agree."""
    from plonky2_b200 import _native as N
    from plonky2_b200 import fri as F

    log_n, r, h = 15, 2, 4
    arities = [3, 3, 3]
    n = 1 << log_n
    vals = [synth(0x6400, (3, n)), synth(0x6401, (2, n))]
    coeffs = [oracle.Commit(v, 0, 0).coeffs for v in vals]
    pts = point_kinds(log_n, 0x6410)
    batches = [(pts["ext"], [(0, 0), (0, 1), (0, 2), (1, 0), (1, 1)]), (pts["zeta_w"], [(1, 1), (0, 2)])]
    alpha = tuple(int(v) for v in synth(0x6420, (2,)))
    opened = openings(coeffs, batches, oracle)
    whole = [pb.PolynomialBatch.from_values(v, r, False, h) for v in vals]
    parts = [[pb.PolynomialBatch.from_values(v, r, False, h, shard=(g, shards)) for v in vals] for g in range(shards)]
    ref = begin_coeffs(pb, whole, batches, alpha, r, h)
    states = [begin_values(pb, parts[g], batches, alpha, opened, h) for g in range(shards)]
    L, ctx = N.lib(), ref.ctx
    betas = synth(0x6430, (len(arities), 2))
    try:
        want = ref._read()
        got = _gather(states)
        assert np.array_equal(got, want), first_diff(got, want)
        leaves = sample_leaves(log_n + r, 0x6440)
        rows = [oracle.Commit(c, r, 0, is_coeffs=True).leaf_rows(leaves) for c in coeffs]
        ev = as_pairs(*compose(leaves, log_n + r, batches, alpha, opened, lambda o, p: rows[o][:, p]))
        assert np.array_equal(want[leaves.astype(np.int64)], ev)
        for rnd, ab in enumerate(arities):
            cap = np.empty(4 << h, dtype=np.uint64)
            N.check(L.gl_fri_commit_round(ref.h, ab, N.np_ptr(cap)), ctx.h)
            locs = []
            for st in states:
                loc = np.empty((4 << h) // shards, dtype=np.uint64)
                N.check(L.gl_fri_commit_round(st.h, ab, N.np_ptr(loc)), ctx.h)
                locs.append(loc)
            assert np.array_equal(np.concatenate(locs), cap), rnd
            for st in [ref] + states:
                N.check(L.gl_fri_fold(st.h, N.np_ptr(np.ascontiguousarray(betas[rnd]))), ctx.h)
            want, got = ref._read(), _gather(states)
            assert np.array_equal(got, want), "round %d: %s" % (rnd, first_diff(got, want))
        log_last = log_n + r - sum(arities)
        shift = pow(SHIFT, 1 << sum(arities), P)
        coeffs_last = F._final_poly_from_values(_gather(states), log_last, shift, r, ctx)
        buf = np.empty(2 << log_last, dtype=np.uint64)
        for st in [ref] + (states if shards == 1 else []):  # one shard is an ordinary state with its own final poly
            ln = C.c_size_t()
            N.check(L.gl_fri_final_poly(st.h, N.np_ptr(buf), buf.size, C.byref(ln)), ctx.h)
            assert ln.value == 1 << (log_last - r)
            assert np.array_equal(coeffs_last.reshape(-1), buf[:2 * ln.value])
    finally:
        for st in [ref] + states:
            st.close()
        for b in whole + [x for p in parts for x in p]:
            b.close()


# ----------------------------------------------------------------------------- the benchmarked sizes
def _dev_view(ptr, words):
    import torch

    class View:
        __cuda_array_interface__ = {"shape": (words,), "typestr": "<i8", "data": (ptr, False), "version": 2}

    return torch.as_tensor(View(), device="cuda")


def _lde_rows(commit, leaves):
    """(num_polys, len(leaves)) LDE values of a resident commitment at `leaves`, gathered on the device."""
    import torch

    from plonky2_b200 import _native as N

    stride = C.c_size_t()
    ptr = N.lib().gl_commit_dev_lde(commit.h, C.byref(stride))
    lde = _dev_view(ptr, commit.num_polys * stride.value).view(commit.num_polys, stride.value)
    idx = torch.as_tensor(leaves.astype(np.int64), device="cuda")
    commit.ctx.synchronize()
    return lde[:, idx].cpu().numpy().view(np.uint64)


def _device_commit(pb, src, log_n, r, h, shard=(0, 1)):
    """A commitment of the rows of the device tensor `src` as coefficients."""
    from plonky2_b200 import _native as N

    ctx = pb.default_context()
    ctx.after_caller()

    def add_columns(hh):
        N.check(N.lib().gl_commit_add_columns(hh, 0, src.shape[0], N.vp(src.data_ptr()), 1 << log_n, N.COLS_COEFFS,
                                              N.MEM_DEVICE), ctx.h)

    return pb.PolynomialBatch._from_device(ctx, src.shape[0], log_n, r, h, add_columns, shard=shard)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["cfg2", "cfg5"])
def test_benchmarked_sizes(pb, cfg):
    """cfg2 (234 x 2^20, rate 3) and cfg5 (64 x 2^24, rate 1: a 2^25-leaf codeword, and 8192 scan chunks, past the
    single-CTA scan's 1024), cap height 4, with a plonky2-like instance (every column at zeta, two at zeta * w_n) and
    a starky-like one (every column at zeta, the first half at zeta * w_n): both domains word for word, the evaluator at
    the sampled leaves, and for cfg5 the blocks of 2 and 4 row-block shards."""
    import torch

    B, log_n, r = {"cfg2": (234, 20, 3), "cfg5": (64, 24, 1)}[cfg]
    h, n = 4, 1 << log_n
    need = B * n * 8 * (2 + (1 << r)) + (4 << 30)  # source, coefficients, LDE, and room for the FRI buffers
    free, _ = torch.cuda.mem_get_info()
    in_use, _ = pb.default_context().device_bytes()
    if free < need:
        pytest.skip("%s needs about %.1f GiB of device memory, %.1f GiB free (%.1f GiB held by the library)"
                    % (cfg, need / 2**30, free / 2**30, in_use / 2**30))
    gen = torch.Generator(device="cuda").manual_seed(0x6500 + B)
    src = torch.randint(0, 1 << 62, (B, n), dtype=torch.int64, device="cuda", generator=gen)
    pts = point_kinds(log_n, 0x6510 + B)
    instances = {"plonky2": [(pts["ext"], [(0, j) for j in range(B)]), (pts["zeta_w"], [(0, 0), (0, 1)])],
                 "starky": [(pts["ext"], [(0, j) for j in range(B)]), (pts["zeta_w"], [(0, j) for j in range(B // 2)])]}
    alpha = tuple(int(v) for v in synth(0x6520 + B, (2,)))
    leaves = sample_leaves(log_n + r, 0x6530 + B)
    whole = _device_commit(pb, src, log_n, r, h)
    codewords = {}
    try:
        rows = _lde_rows(whole, leaves)
        for name, batches in instances.items():
            ev = pb.eval_commitments([(whole, z) for z, _ in batches])
            opened = [np.array([ev[b][p] for _, p in refs], dtype=np.uint64) for b, (_, refs) in enumerate(batches)]
            vals, co = both_codewords(pb, [whole], batches, alpha, opened, r, h)
            assert np.array_equal(vals, co), "%s %s: value vs coefficient domain: %s" % (cfg, name, first_diff(vals, co))
            want = as_pairs(*compose(leaves, log_n + r, batches, alpha, opened, lambda o, p: rows[p]))
            got = vals[leaves.astype(np.int64)]
            assert np.array_equal(got, want), "%s %s: device vs evaluator: %s" % (cfg, name, first_diff(got, want))
            codewords[name] = (vals, opened)
            del co
    finally:
        whole.close()
    if cfg != "cfg5":
        return
    n_leaves = n << r
    for shards in (2, 4):
        for g in range(shards):
            part = _device_commit(pb, src, log_n, r, h, shard=(g, shards))
            try:
                for name, batches in instances.items():
                    vals, opened = codewords[name]
                    f = begin_values(pb, [part], batches, alpha, opened, h)
                    try:
                        loc = f._read()
                    finally:
                        f.close()
                    blk = vals[g * n_leaves // shards:(g + 1) * n_leaves // shards]
                    assert np.array_equal(loc, blk), "%s shard %d of %d: %s" % (name, g, shards, first_diff(loc, blk))
            finally:
                part.close()


# ----------------------------------------------------------------------------- gl_fri_mix
def _from_coeffs_state(pb, coeffs_ext, log_n, rate_bits, cap_height=0):
    from plonky2_b200 import _native as N

    ctx = pb.default_context()
    h = N.vp()
    N.check(N.lib().gl_fri_begin_from_coeffs(ctx.h, N.np_ptr(np.ascontiguousarray(coeffs_ext.reshape(-1))), log_n,
                                             rate_bits, cap_height, C.byref(h)), ctx.h)
    return Fri(h, ctx)


def _mix(f, other, beta):
    from plonky2_b200 import _native as N

    N.check(N.lib().gl_fri_mix(f.h, other.h, N.np_ptr(np.array(beta, dtype=np.uint64))), f.ctx.h)


def _mix_want(v, w, beta):
    m0, m1 = G.ext_mul((v[:, 0], v[:, 1]), (np.uint64(beta[0]), np.uint64(beta[1])))
    return as_pairs(G.add(m0, w[:, 0]), G.add(m1, w[:, 1]))


@pytest.mark.gpu
def test_fri_mix_every_length(pb):
    """values <- values * beta + other's, element by element, on codewords of 2^1 .. 2^25 elements; codewords of
    different lengths are refused."""
    for log_len in range(1, 26):
        log_n = log_len - 1
        a = _from_coeffs_state(pb, synth(0x6600 + log_len, (1 << log_n, 2)), log_n, 1)
        b = _from_coeffs_state(pb, synth(0x6640 + log_len, (1 << log_n, 2)), log_n, 1)
        try:
            v, w = a._read(), b._read()
            beta = tuple(int(x) for x in synth(0x6680 + log_len, (2,)))
            _mix(a, b, beta)
            got, want = a._read(), _mix_want(v, w, beta)
            assert np.array_equal(got, want), "2^%d: %s" % (log_len, first_diff(got, want))
            assert np.array_equal(b._read(), w)
        finally:
            a.close()
            b.close()
    a = _from_coeffs_state(pb, synth(0x66C0, (32, 2)), 5, 1)
    b = _from_coeffs_state(pb, synth(0x66C1, (16, 2)), 4, 1)
    try:
        with pytest.raises(ValueError, match="codeword lengths differ: 2\\^6 vs 2\\^5"):
            _mix(a, b, (1, 2))
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("shards", [2, 8])
def test_fri_mix_row_block_shards(pb, oracle, shards):
    """Row-block sharded value-domain states mix their local blocks: shard by shard, the mixed blocks in shard order are
    the unsharded mix. Two states sharded differently (another shard, or another number of shards) are refused."""
    from plonky2_b200 import _native as N

    log_n, r, h = 12, 2, 4
    n = 1 << log_n
    vals = [synth(0x6700, (3, n)), synth(0x6701, (2, n))]
    coeffs = [oracle.Commit(v, 0, 0).coeffs for v in vals]
    pts = point_kinds(log_n, 0x6710)
    inst = [[(pts["ext"], [(0, 0), (0, 1), (0, 2)]), (pts["zeta_w"], [(0, 1)])],
            [(pts["base"], [(1, 0), (1, 1)]), (pts["ext2"], [(1, 1), (0, 2)])]]
    alphas = [tuple(int(v) for v in synth(0x6720 + k, (2,))) for k in range(2)]
    beta = tuple(int(v) for v in synth(0x6730, (2,)))
    opened = [openings(coeffs, b, oracle) for b in inst]
    whole = [pb.PolynomialBatch.from_values(v, r, False, h) for v in vals]
    parts = [[pb.PolynomialBatch.from_values(v, r, False, h, shard=(g, shards)) for v in vals] for g in range(shards)]
    ref = [begin_values(pb, whole, inst[k], alphas[k], opened[k], h) for k in range(2)]
    st = [[begin_values(pb, parts[g], inst[k], alphas[k], opened[k], h) for k in range(2)] for g in range(shards)]
    try:
        v, w = ref[0]._read(), ref[1]._read()
        _mix(ref[0], ref[1], beta)
        want = ref[0]._read()
        assert np.array_equal(want, _mix_want(v, w, beta))
        with pytest.raises(N.NativeError, match="native error 5: this FRI state is row-block sharded 0 of %d, the other "
                                                "1 of %d" % (shards, shards)):
            _mix(st[0][0], st[1][1], beta)
        with pytest.raises(N.NativeError, match="native error 5: this FRI state is row-block sharded 0 of 1, the other "
                                                "0 of %d" % shards):
            _mix(ref[1], st[0][1], beta)
        for g in range(shards):
            _mix(st[g][0], st[g][1], beta)
        got = _gather([s[0] for s in st])
        assert np.array_equal(got, want), first_diff(got, want)
        assert np.array_equal(_gather([s[1] for s in st]), w)
    finally:
        for f in ref + [x for s in st for x in s]:
            f.close()
        for b in whole + [x for p in parts for x in p]:
            b.close()
