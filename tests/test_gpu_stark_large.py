"""starky's device columns, STARK quotient and FRI at the row counts the project benchmarks (2^22 to 2^25 points),
checked exactly on every row or coset point against identities that need no field inversion.

The references are vectorised exact Goldilocks arithmetic (tests/gl_numpy.py), pinned here against Python integers.
Every device column is pinned by an identity that defines it uniquely once no denominator is zero:
  - a logUp helper column h over looking columns J with filters phi: h * prod_J (f_j + gamma) ==
    sum_j phi_j * prod_{j' != j} (f_j' + gamma); Z: Z[0] == 0 and (Z[i+1] - Z[i] - sum_k h_k[i]) (t[i] + gamma) + m[i]
    == 0 (at the last row with Z[n] = 0 when the lookup is honest);
  - a CTL helper column: the same with combine_j = gamma + sum_k beta^k v_{j,k}; Z[i] - Z[i+1] == sum_k h_k[i] (one
    entry: (Z[i] - Z[i+1]) combine[i] == filter[i]) with Z[n] = 0;
  - the quotient q at every coset point x: q(x) Z_H(x) D(x) == sum_c alpha-weight_c C_c(x) S_c(x), D(x) = n (x - 1)
    (x - last), S_c the constraint's selector multiplied through by D.
At these sizes the additive three-phase scan gives each thread of its middle phase more than one chunk total, and the
factored power tables read hi entries past the 4096-entry minimum.

CPU: the numpy field against Python integers; the vectorised range-check trace generator against the test one; the
2^12 edge-operand traces (values p - 1, 2^32, 2^63, ..., denominators of exactly 1 and p - 1, filters that are not
0/1) through the host run of the row code, the restatements and the identities.

GPU (-m gpu): logUp columns at 2^22 and 2^24 rows; CTL columns at 2^22 (and 2^24 for one table) through a permuted
zs_index; the quotient at 2^21 and 2^25 coset points (and through the auxiliary entry point); whole proofs at 2^20 and
2^22 rows accepted by the restated verifiers and rejected when tampered; FRI over a 64 x 2^22 commitment against the
oracle verifier (64 x 2^24 with GL_LARGE_FRI_24=1)."""
import copy
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import gl_numpy as G
import stark_twin as T
from conftest import EDGE, P, synth
from plonky2_b200 import _native as N
from plonky2_b200 import cross_table_lookup as X
from plonky2_b200 import field as E
from plonky2_b200 import stark as S
from plonky2_b200.lookup import GrandProductChallenge
from test_gpu_field_lazy import EDGE_SET
from test_stark_ctl import _emu as _ctl_emu
from test_stark_ctl import _restated_table_aux, _wide_ctls, system_ctls
from test_stark_lookups import (A0, A1, B, E_, MA, MB, SEL, SEL2, TABLE, NextRowLookupStark, RangeCheckStark,
                                RangeCheckStark4)
from test_stark_lookups import G as G_
from test_stark_lookups import _emu_helpers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = 2**64 - 1
# the looked, table and frequency values of the edge-operand traces
EDGE_VALUES = [0, 1, P - 1, P - 2, 2**32 - 1, 2**32, P - 2**32, 2**63]


# ------------------------------------------------------------------------------------------------ numpy references
def col_rows(column, trace):
    """Column::eval_table on every row (the next row of the last row is row 0), as canonical uint64."""
    n = trace.shape[1]
    acc = np.full(n, column.constant, dtype=np.uint64)
    for terms, rows in ((column.linear_combination, lambda c: trace[c]),
                        (column.next_row_linear_combination, lambda c: np.roll(trace[c], -1))):
        for c, f in terms:
            v = rows(c)
            acc = G.add(acc, v if f == 1 else G.mul(v, np.uint64(f)))
    return acc


def filter_rows(filt, trace):
    """Filter::eval_table on every row."""
    acc = np.zeros(trace.shape[1], dtype=np.uint64)
    for a, b in filt.products:
        acc = G.add(acc, G.mul(col_rows(a, trace), col_rows(b, trace)))
    for c in filt.constants:
        acc = G.add(acc, col_rows(c, trace))
    return acc


def _first_bad(got, want):
    bad = np.nonzero(got != want)[0]
    return None if len(bad) == 0 else int(bad[0])


def assert_rows_equal(got, want, what):
    i = _first_bad(got, want)
    assert i is None, "%s: first differing row %d of %d" % (what, i, len(got))


def assert_helper(h, dens, filters, what):
    """h * prod_j dens_j == sum_j filters_j * prod_{j' != j} dens_j'."""
    lhs = h
    for d in dens:
        lhs = G.mul(lhs, d)
    rhs = np.zeros(len(h), dtype=np.uint64)
    for j, f in enumerate(filters):
        t = f
        for k, d in enumerate(dens):
            if k != j:
                t = G.mul(t, d)
        rhs = G.add(rhs, t)
    assert_rows_equal(lhs, rhs, what)


def chunk_size(degree):
    return degree - 1 if degree > 1 else 1


def check_lookup_columns(stark, trace, challenges, aux, honest):
    """Every logUp helper and Z column of aux ((num_aux, n) uint64, prover.rs's order: every lookup, every challenge,
    h_k then Z) against the identities, on every row. honest: Z closes at the wrap (Z[n] = 0)."""
    chunk = chunk_size(stark.constraint_degree())
    pos = 0
    for li, lookup in enumerate(stark.lookups()):
        f = [col_rows(c, trace) for c in lookup.columns]
        phi = [filter_rows(fl, trace) for fl in lookup.filter_columns]
        t, m = col_rows(lookup.table_column, trace), col_rows(lookup.frequencies_column, trace)
        for ci, gamma in enumerate(challenges):
            g = np.uint64(int(gamma) % P)
            dens = [G.add(v, g) for v in f]
            td = G.add(t, g)
            assert all(d.all() for d in dens) and td.all(), "a zero denominator: the identities would not pin the columns"
            hsum = np.zeros(trace.shape[1], dtype=np.uint64)
            for k in range(0, len(f), chunk):
                h = aux[pos]
                assert_helper(h, dens[k:k + chunk], phi[k:k + chunk], "lookup %d challenge %d h_%d" % (li, ci, k // chunk))
                hsum = G.add(hsum, h)
                pos += 1
            z = aux[pos]
            pos += 1
            assert int(z[0]) == 0
            zn = np.roll(z, -1)
            zn[-1] = 0
            lhs = G.add(G.mul(G.sub(G.sub(zn, z), hsum), td), m)
            rows = slice(None) if honest else slice(0, -1)
            assert_rows_equal(lhs[rows], np.zeros_like(lhs[rows]), "lookup %d challenge %d Z" % (li, ci))
    assert pos == len(aux)


def combine_rows(columns, trace, beta, gamma):
    """GrandProductChallenge::combine on every row: gamma + sum_k beta^k v_k, by Horner from the last value."""
    acc = np.zeros(trace.shape[1], dtype=np.uint64)
    for col in reversed(columns):
        acc = G.add(G.mul(acc, np.uint64(beta)), col_rows(col, trace))
    return G.add(acc, np.uint64(gamma))


def check_ctl_columns(trace, groups, pairs, degree, zs_index, out):
    """The table's CTL columns `out` ((helpers + Zs, n) uint64) for zs_index (g * len(pairs) + c -> Z position; the
    helper columns of the Z positions in order, then the Zs) against the identities, on every row."""
    nch, chunk = len(pairs), chunk_size(degree)
    at = {int(z): k for k, z in enumerate(zs_index)}
    num_h = [-(-len(entries) // chunk) if len(entries) > 1 else 0 for _, entries in groups]
    nh = sum(num_h) * nch
    assert out.shape[0] == nh + len(zs_index)
    hpos = 0
    for z in range(len(zs_index)):
        g, c = divmod(at[z], nch)
        beta, gamma = (int(v) % P for v in pairs[c])
        entries = groups[g][1]
        dens = [combine_rows(t.columns, trace, beta, gamma) for t in entries]
        phi = [filter_rows(t.filter, trace) for t in entries]
        assert all(d.all() for d in dens), "a zero combine: the identities would not pin the columns"
        zc = out[nh + z]
        zn = np.roll(zc, -1)
        zn[-1] = 0
        what = "group %d challenge %d" % (g, c)
        if num_h[g] == 0:
            assert_rows_equal(G.mul(G.sub(zc, zn), dens[0]), phi[0], what + " Z")
        else:
            hsum = np.zeros(trace.shape[1], dtype=np.uint64)
            for k in range(num_h[g]):
                h = out[hpos + k]
                assert_helper(h, dens[k * chunk:(k + 1) * chunk], phi[k * chunk:(k + 1) * chunk], what + " h_%d" % k)
                hsum = G.add(hsum, h)
            assert_rows_equal(G.sub(zc, zn), hsum, what + " Z")
        hpos += num_h[g]
    assert hpos == nh


def range_check_trace(log_n, seed=7, table_bits=16, count_combination=True):
    """RangeCheckStark.generate_trace, vectorised (the same draws, E written with numpy field arithmetic)."""
    n = 1 << log_n
    T_ = min(n, 1 << table_bits)
    rng = np.random.default_rng(seed)
    u = lambda: rng.integers(0, T_, n).astype(np.uint64)  # noqa: E731
    junk = np.uint64(1 << 40) + np.arange(n, dtype=np.uint64)
    tr = np.zeros((10, n), dtype=np.uint64)
    s, s2 = rng.integers(0, 2, n).astype(np.uint64), rng.integers(0, 2, n).astype(np.uint64)
    s[n - 1] = s2[n - 1] = 1
    tr[SEL], tr[SEL2] = s, s2
    tr[A0] = np.where(s == 1, u(), junk)
    tr[A1] = u()
    both = (s * s2) == 1
    target = np.where(both, u(), junk + np.uint64(1 << 20))
    tr[G_] = u()
    tr[E_] = G.sub(G.sub(target, np.roll(tr[G_], -1)), np.uint64(3))
    tr[B] = np.where(s2 == 1, u(), junk)
    tr[TABLE] = np.arange(n, dtype=np.uint64) % np.uint64(T_)
    looked = [tr[A0][s == 1], tr[A1]] + ([target[both]] if count_combination else [])
    tr[MA, :T_] = np.bincount(np.concatenate(looked).astype(np.int64), minlength=T_)
    tr[MB, :T_] = np.bincount(tr[B][s2 == 1].astype(np.int64), minlength=T_)
    return tr


def edge_range_trace(log_n=12, seed=0xE0):
    """RangeCheckStark's columns with looked, table and frequency values from EDGE_VALUES and selectors that are
    arbitrary field elements (edge values and random ones): no honest lookup, every operand an edge."""
    n = 1 << log_n
    rng = np.random.default_rng(seed)
    ev = np.array(EDGE_VALUES, dtype=np.uint64)
    tr = ev[rng.integers(0, len(ev), (10, n))]
    sel = np.concatenate([ev, synth(seed, (n,))])
    tr[SEL] = sel[rng.integers(0, len(sel), n)]
    tr[SEL2] = sel[rng.integers(0, len(sel), n)]
    return tr


def pick_gammas(values, forbidden=()):
    """Challenges gamma with some value + gamma == 1 and some value + gamma == p - 1 while no value (nor any of
    `forbidden`) + gamma is 0: one gamma doing both if there is one, else one for each."""
    vals = sorted({int(v) % P for v in values})
    bad = {int(v) % P for v in vals} | {int(v) % P for v in forbidden}

    def ok(g):
        return (-g) % P not in bad

    for e in vals:                               # e + g = 1 and (e - 2) + g = p - 1
        g = (1 - e) % P
        if ok(g) and (e - 2) % P in bad:
            return [g]
    one = next((1 - e) % P for e in vals if ok((1 - e) % P))
    minus_one = next((P - 1 - e) % P for e in vals if ok((P - 1 - e) % P))
    return [one, minus_one]


def _lookup_values(stark, trace):
    out = []
    for lookup in stark.lookups():
        out += [col_rows(c, trace) for c in lookup.columns] + [col_rows(lookup.table_column, trace)]
    return np.concatenate(out)


def edge_ctl_traces(log_n=12, seed=0xE1):
    n = 1 << log_n
    rng = np.random.default_rng(seed)
    ev = np.array(EDGE_VALUES, dtype=np.uint64)
    return [ev[rng.integers(0, len(ev), (8, n))] for _ in range(2)]


def edge_ctl_pairs(traces, ctls, beta=2**32):
    """(beta, gamma) pairs for the wide CTLs over edge traces: some combine equal to 1 and to p - 1, none 0."""
    base = []
    for t in range(2):
        for _, entries in X.table_groups(ctls, t):
            base += [combine_rows(e.columns, traces[t], beta, 0) for e in entries]
    return [(beta, g) for g in pick_gammas(np.concatenate(base))]


def _hits(dens):
    d = np.concatenate(dens)
    return bool((d == 1).any()), bool((d == np.uint64(P - 1)).any())


# ----------------------------------------------------------------------------------------------------------- CPU
def test_numpy_field_matches_python_integers():
    """add, sub, mul, canon, F_{p^2} mul and powers on every pair of edge words and 2^20 random pairs (a quarter near
    2^64 - 1, a quarter near p, inputs not reduced), against Python integers."""
    edges = sorted(set(EDGE) | set(EDGE_SET) | {M64, M64 - 1, P + 2**32 - 2})
    ea, eb = np.meshgrid(np.array(edges, dtype=np.uint64), np.array(edges, dtype=np.uint64))
    rng = np.random.default_rng(0xF1E1D)
    q = 1 << 18
    near = lambda c: (np.uint64(c) - rng.integers(0, 1 << 33, q, dtype=np.uint64)).astype(np.uint64)  # noqa: E731
    near_p = (np.uint64(P) + rng.integers(-(1 << 32), 1 << 32, q).astype(np.int64).astype(np.uint64))
    rand = lambda k: rng.integers(0, 2**64, k, dtype=np.uint64)  # noqa: E731
    a = np.concatenate([ea.reshape(-1), near(M64), near_p, rand(2 * q)])
    b = np.concatenate([eb.reshape(-1), rng.permutation(np.concatenate([near(M64), near_p])), rand(2 * q)])
    ao, bo = a.astype(object), b.astype(object)

    def same(got, want, what):
        assert got.dtype == np.uint64 and (got < np.uint64(P)).all(), what
        assert np.array_equal(got.astype(object), want % P), what

    same(G.add(a, b), ao + bo, "add")
    same(G.sub(a, b), ao - bo, "sub")
    same(G.mul(a, b), ao * bo, "mul")
    same(G.canon(a), ao, "canon")
    same(G.neg(a), -ao, "neg")
    same(G.mul(a, np.uint64(M64)), ao * M64, "mul by a scalar")
    # F_{p^2}: (a0 + a1 X)(b0 + b1 X) = a0 b0 + 7 a1 b1 + (a0 b1 + a1 b0) X
    a1, b1 = np.roll(a, 1), np.roll(b, 7)
    c0, c1 = G.ext_mul((a, a1), (b, b1))
    a1o, b1o = a1.astype(object), b1.astype(object)
    same(c0, ao * bo + 7 * a1o * b1o, "ext_mul c0")
    same(c1, ao * b1o + a1o * bo, "ext_mul c1")
    # powers: every entry of short runs, sampled entries of a long one, and a root of unity closing its subgroup
    for base in edges[:8] + [int(v) for v in synth(0xF1, (4,), canonical=False)]:
        pw = G.powers(base, 1000)
        assert [int(v) for v in pw] == [pow(base, k, P) for k in range(1000)], base
    w = E.primitive_root_of_unity(20)
    pw = G.powers(w, 1 << 20)
    idx = rng.integers(0, 1 << 20, 2000)
    assert all(int(pw[k]) == pow(w, int(k), P) for k in idx)
    assert int(G.mul(pw[-1], np.uint64(w))) == 1 and len(set(pw[:4096].tolist())) == 4096
    assert [int(v) for v in G.pow_scalar(np.array(edges[:6], dtype=np.uint64), 12345)] == \
        [pow(v, 12345, P) for v in edges[:6]]
    assert [int(v) for v in G.brev(np.arange(8), 3)] == [0, 4, 2, 6, 1, 5, 3, 7]


def test_vectorised_range_check_trace_equals_the_generator():
    for log_n, cc in [(8, True), (10, False)]:
        assert np.array_equal(range_check_trace(log_n, seed=log_n, count_combination=cc),
                              RangeCheckStark.generate_trace(log_n, seed=log_n, count_combination=cc))


def test_identities_reject_a_wrong_column():
    """The identity checks fail on a helper or Z column with one word changed, at the first and last rows."""
    stark, trace = RangeCheckStark(), range_check_trace(8)
    challenges = [int(v) for v in synth(0xE10, (2,))]
    aux, _ = T.aux_columns(stark, trace, challenges)
    check_lookup_columns(stark, trace, challenges, aux, honest=True)
    for col, row in [(0, 0), (2, 255), (3, 17), (4, 255), (9, 1)]:
        bad = aux.copy()
        bad[col, row] = (bad[col, row] + np.uint64(1)) % np.uint64(P)
        with pytest.raises(AssertionError):
            check_lookup_columns(stark, trace, challenges, bad, honest=True)
    ctls = _wide_ctls()
    traces = [synth(0xE11, (8, 64)), synth(0xE12, (8, 64))]
    pairs = [tuple(int(v) for v in synth(0xE13, (2,)))]
    groups = X.table_groups(ctls, 0)
    zs_index, _, _ = X.zs_layout(groups, 1, 3)
    out = _restated_table_aux(traces[0], groups, pairs, 3)
    check_ctl_columns(traces[0], groups, pairs, 3, zs_index, out)
    for row in range(out.shape[0]):
        bad = out.copy()
        bad[row, 63] ^= np.uint64(1)
        with pytest.raises(AssertionError):
            check_ctl_columns(traces[0], groups, pairs, 3, zs_index, bad)


@pytest.fixture(scope="module")
def logup_emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("logup_emu_large") / "liblogup_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DGL_FORCE_32BIT_PATH", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "emu", "logup_emu.cpp")])
    L = C.CDLL(out)
    L.emu_stark_lookup_helpers.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                           C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    return L


@pytest.fixture(scope="module")
def ctl_emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ctl_emu_large") / "libctl_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DGL_FORCE_32BIT_PATH", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "emu", "ctl_emu.cpp")])
    L = C.CDLL(out)
    L.emu_stark_ctl_helpers.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                        C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    return L


def _edge_lookup_case():
    stark, trace = RangeCheckStark(), edge_range_trace()
    challenges = pick_gammas(_lookup_values(stark, trace)) + [int(synth(0xE14, (1,))[0])]
    return stark, trace, challenges


def test_edge_operand_lookup_columns_on_host(logup_emu):
    """Edge looked, table and frequency values, non-boolean filters, denominators of exactly 1 and p - 1: the row code
    on the host equals the restatement element for element, and both satisfy the identities."""
    stark, trace, challenges = _edge_lookup_case()
    f = _lookup_values(stark, trace)
    assert _hits([G.add(f, np.uint64(g)) for g in challenges]) == (True, True)
    assert not np.isin(trace[SEL], [0, 1]).all()
    want, wraps = T.aux_columns(stark, trace, challenges)
    rc, got = _emu_helpers(logup_emu, stark, trace, challenges)
    assert rc == 0 and np.array_equal(got, want)
    check_lookup_columns(stark, trace, challenges, want, honest=False)
    assert any(w != 0 for w in wraps)


def _edge_ctl_case():
    ctls, traces = _wide_ctls(), edge_ctl_traces()
    return ctls, traces, edge_ctl_pairs(traces, ctls)


@pytest.mark.parametrize("degree", [3, 4])
def test_edge_operand_ctl_columns_on_host(ctl_emu, degree):
    ctls, traces, pairs = _edge_ctl_case()
    dens = []
    for t in range(2):
        groups = X.table_groups(ctls, t)
        want = _restated_table_aux(traces[t], groups, pairs, degree)
        rc, got = _ctl_emu(ctl_emu, traces[t], groups, pairs, degree)
        assert rc == 0 and np.array_equal(got, want), t
        zs_index, _, _ = X.zs_layout(groups, len(pairs), degree)
        check_ctl_columns(traces[t], groups, pairs, degree, zs_index, want)
        dens += [combine_rows(e.columns, traces[t], *pr) for _, es in groups for e in es for pr in pairs]
    assert _hits(dens) == (True, True)


# ----------------------------------------------------------------------------------------------------------- GPU
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


def _to_device(trace):
    import torch

    dev = torch.from_numpy(np.ascontiguousarray(trace).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return dev


def _to_host(t):
    return t.cpu().numpy().view(np.uint64)


LOOKUP_CASES = ["range_22_c1", "range_22_c4", "range_24_c2", "range4_22_c2", "next_row_22_c4", "edge_12_c3"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", LOOKUP_CASES)
def test_device_lookup_columns_satisfy_the_identities(pb, case):
    """compute_lookup_helper_columns on a torch trace; every helper and Z column checked on every row. From 2^22 rows
    the additive scan's middle phase gives each thread more than one chunk total."""
    kind, log_n, nch = case.rsplit("_", 2)[0], int(case.rsplit("_", 2)[1]), int(case[-1])
    honest = True
    if kind == "range":
        stark, trace = RangeCheckStark(), range_check_trace(log_n, seed=log_n)
    elif kind == "range4":
        stark, trace = RangeCheckStark4(), range_check_trace(log_n, seed=log_n, count_combination=False)
    elif kind == "next_row":
        stark, trace, honest = NextRowLookupStark(), synth(0xE20, (7, 1 << log_n)), False
    else:
        stark, trace, challenges = _edge_lookup_case()
        honest = False
    if kind != "edge":
        challenges = [int(v) for v in synth(0xE30 + log_n, (nch,))]
    got = _to_host(S.compute_lookup_helper_columns(stark, _to_device(trace), challenges, pb.default_context()))
    assert got.shape == (stark._helper_columns_per_challenge() * len(challenges), 1 << log_n)
    check_lookup_columns(stark, trace, challenges, got, honest)
    if kind == "edge":
        assert np.array_equal(got, T.aux_columns(stark, trace, challenges)[0])


CTL_CASES = ["wide_22_d3_c4", "wide_22_d4_c1", "system_22_d3_c4", "system_22_d3_c1", "wide_24_d3_c1",
             "edge_12_d3_c2", "edge_12_d4_c2"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CTL_CASES)
def test_device_ctl_columns_satisfy_the_identities(pb, case):
    """gl_stark_ctl_helpers with a zs_index that is not the identity permutation; every helper and Z column checked on
    every row, in the order zs_index asks for. wide_24: the looking table only."""
    import torch

    kind, log_n, degree, nch = case.split("_")
    log_n, degree, nch = int(log_n), int(degree[1:]), int(nch[1:])
    if kind == "system":
        ctls = system_ctls()
        traces = [synth(0xE40 + k, (w, 1 << log_n)) for k, w in enumerate((9, 6, 4))]
    elif kind == "wide":
        ctls = _wide_ctls()
        traces = [synth(0xE50, (8, 1 << log_n)), synth(0xE51, (8, 1 << log_n))]
    else:
        ctls, traces, pairs = _edge_ctl_case()
    if kind != "edge":
        pairs = [tuple(int(v) for v in synth(0xE60 + c, (2,))) for c in range(nch)]
    nch = len(pairs)
    ctx = pb.default_context()
    L = N.lib()
    tables = [0] if log_n == 24 else range(len(traces))
    rng = np.random.default_rng(log_n * 10 + degree)
    for t in tables:
        groups = X.table_groups(ctls, t)
        prog, offsets, consts = X.ctl_row_programs(groups, traces[t].shape[0])
        _, _, nh = X.zs_layout(groups, nch, degree)
        n_zs = len(groups) * nch
        zs_index = rng.permutation(n_zs).astype(np.uint32)
        if n_zs > 1 and (zs_index == np.arange(n_zs)).all():
            zs_index = np.roll(zs_index, 1)
        dev = _to_device(traces[t])
        out = torch.empty((nh + n_zs, traces[t].shape[1]), dtype=torch.int64, device="cuda")
        ch = np.array([int(v) % P for pr in pairs for v in pr], dtype=np.uint64)
        consts = consts if len(consts) else np.zeros(1, dtype=np.uint64)
        N.check(L.gl_stark_ctl_helpers(ctx.h, N.vp(dev.data_ptr()), traces[t].shape[1], traces[t].shape[0], log_n,
                                       prog, offsets.ctypes.data_as(N.u32p), len(offsets) - 1, N.np_ptr(consts),
                                       len(consts), N.np_ptr(ch), nch, degree, zs_index.ctypes.data_as(N.u32p),
                                       N.vp(out.data_ptr())), ctx.h)
        ctx.synchronize()
        got = _to_host(out)
        del out, dev
        check_ctl_columns(traces[t], groups, pairs, degree, zs_index, got)
        if kind == "edge":          # the product's own zs_index order against the restatement
            want = _restated_table_aux(traces[t], groups, pairs, degree)
            dev = _to_device(traces[t])
            out = torch.empty(want.shape, dtype=torch.int64, device="cuda")
            X.compute_ctl_helper_columns(dev, groups, [GrandProductChallenge(*pr) for pr in pairs], degree, ctx, out)
            assert np.array_equal(_to_host(out), want), t


# ------------------------------------------------------------------------------------------------ STARK quotient
class AllOpsStark(S.Stark):
    """Four columns, one public input; every opcode (local, next, public input and program constants, add, sub, mul)
    and every emit kind. The declared degree sets the quotient degree factor; the kernel does not depend on the
    constraints' actual degree, so any trace does."""
    COLUMNS, PUBLIC_INPUTS = 4, 1

    def __init__(self, degree):
        self.degree = degree

    def eval(self, v, y):
        a, b, c, d = (v.local(k) for k in range(4))
        y.constraint(a * b - c + 5)
        y.constraint_transition(v.next(0) - a * d)
        y.constraint_first_row(b - v.public_input(0))
        y.constraint_last_row(c * d + v.next(3) - 11)

    def constraint_degree(self):
        return self.degree


def quotient_program(stark, num_aux=0):
    """The Stark's constraint program; with num_aux, two more constraints reading the auxiliary columns on the local
    and next rows."""
    b = S.ConstraintBuilder(stark.COLUMNS, stark.PUBLIC_INPUTS, num_aux)
    stark.eval(b, b)
    if num_aux:
        b.constraint_transition(b.aux_next(0) - b.aux_local(1) * b.local(2))
        b.constraint(b.aux_local(0) * b.aux_next(1) - b.next(1))
    return b


def eval_program_on_coset(b, consts, trace_vals, aux_vals, step, alphas, sel):
    """The program at every coset point in numpy: LOCAL / NEXT read the coset values of the point and of the point
    `step` further on; each emit's constraint times its selector sel[kind] is folded into every alpha by Horner.
    Values are dropped after their last use."""
    last_use = {}
    for k, (op, a, c) in enumerate(b.instrs):
        if op in (S.OP_ADD, S.OP_SUB, S.OP_MUL):
            last_use[a] = last_use[c] = k
        elif op == S.OP_EMIT:
            last_use[a] = k
    size = trace_vals.shape[1]
    acc = [np.zeros(size, dtype=np.uint64) for _ in alphas]
    v = {}
    for k, (op, a, c) in enumerate(b.instrs):
        r = None
        if op == S.OP_LOCAL:
            r = trace_vals[a]
        elif op == S.OP_NEXT:
            r = np.roll(trace_vals[a], -step)
        elif op == S.OP_AUX_LOCAL:
            r = aux_vals[a]
        elif op == S.OP_AUX_NEXT:
            r = np.roll(aux_vals[a], -step)
        elif op == S.OP_CONST:
            r = np.uint64(consts[a])
        elif op == S.OP_ADD:
            r = G.add(v[a], v[c])
        elif op == S.OP_SUB:
            r = G.sub(v[a], v[c])
        elif op == S.OP_MUL:
            r = G.mul(v[a], v[c])
        else:
            e = G.mul(v[a], sel[c])
            acc = [G.add(G.mul(s, np.uint64(al)), e) for s, al in zip(acc, alphas)]
        if r is not None and k in last_use:
            v[k] = r
        for j in [j for j in v if last_use[j] <= k]:
            del v[j]
    return acc


def check_quotient_values(b, consts, alphas, q, tv, av, log_n, qd_bits):
    """q ((alphas, size) values on the coset shift * <w_size>, natural order) against
    q(x) Z_H(x) D(x) == sum_c alpha^(E-1-c) C_c(x) S_c(x) at every point, C_c evaluated on the trace and auxiliary
    coset values tv, av (natural order); Z_H from Python integers on the 2^qd_bits cosets of the trace subgroup."""
    n, size = 1 << log_n, 1 << (log_n + qd_bits)
    shift = E.coset_shift()
    w = E.primitive_root_of_unity(log_n + qd_bits)
    last = pow(E.primitive_root_of_unity(log_n), n - 1, P)
    x = G.mul(G.powers(w, size), np.uint64(shift))
    zh_cosets = np.array([(pow(shift * pow(w, j, P), n, P) - 1) % P for j in range(1 << qd_bits)], dtype=np.uint64)
    zh = zh_cosets[np.arange(size) & ((1 << qd_bits) - 1)]
    xm1, xl = G.sub(x, np.uint64(1)), G.sub(x, np.uint64(last))
    del x
    d = G.mul(G.mul(xm1, xl), np.uint64(n % P))
    sel = {S.KIND_CONSTRAINT: d, S.KIND_TRANSITION: G.mul(xl, d), S.KIND_FIRST_ROW: G.mul(zh, xl),
           S.KIND_LAST_ROW: G.mul(G.mul(zh, xm1), np.uint64(last))}
    del xm1, xl
    rhs = eval_program_on_coset(b, consts, tv, av, 1 << qd_bits, alphas, sel)
    del sel
    zd = G.mul(zh, d)
    for a in range(len(alphas)):
        assert_rows_equal(G.mul(q[a], zd), rhs[a], "alpha %d" % a)


@pytest.mark.parametrize("qdf,num_aux,n_alphas", [(2, 0, 4), (8, 2, 1), (2, 2, 2)])
def test_quotient_identity_pins_the_quotient(oracle, qdf, num_aux, n_alphas):
    """check_quotient_values accepts the quotient computed point by point with Python integers (the selectors with
    their divisions, then division by Z_H) on a 2^5-row trace, and rejects it with any one value changed."""
    log_n, n = 5, 32
    qd_bits = (qdf - 1).bit_length()
    size = n << qd_bits
    stark = AllOpsStark(qdf + 1)
    b = quotient_program(stark, num_aux)
    consts = [int(synth(0xE74, (1,))[0])] + b.consts[b.num_bound:]
    alphas = [int(v) for v in synth(0xE75, (n_alphas,))]
    shift = E.coset_shift()

    def coset_values(vals):
        pad = np.zeros((vals.shape[0], size), dtype=np.uint64)
        pad[:, :n] = [oracle.ifft(v) for v in vals]
        return np.stack([oracle.coset_fft(v, shift) for v in pad])

    tv = coset_values(synth(0xE76, (4, n)))
    av = coset_values(synth(0xE77, (num_aux, n))) if num_aux else None
    w, g = E.primitive_root_of_unity(log_n + qd_bits), E.primitive_root_of_unity(log_n)
    last = E.inverse(g)
    q = np.zeros((n_alphas, size), dtype=np.uint64)
    for i in range(size):
        x = shift * pow(w, i, P) % P
        zh = (pow(x, n, P) - 1) % P
        sel = {S.KIND_CONSTRAINT: 1, S.KIND_TRANSITION: (x - last) % P,
               S.KIND_FIRST_ROW: zh * E.inverse(n * (x - 1) % P) % P,
               S.KIND_LAST_ROW: zh * E.inverse(n * (g * x - 1) % P) % P}
        v, acc = [], [0] * n_alphas
        for op, a, c in b.instrs:
            r = 0
            if op in (S.OP_LOCAL, S.OP_NEXT):
                r = int(tv[a, (i + (op == S.OP_NEXT) * (1 << qd_bits)) % size])
            elif op in (S.OP_AUX_LOCAL, S.OP_AUX_NEXT):
                r = int(av[a, (i + (op == S.OP_AUX_NEXT) * (1 << qd_bits)) % size])
            elif op == S.OP_CONST:
                r = consts[a]
            elif op == S.OP_ADD:
                r = (v[a] + v[c]) % P
            elif op == S.OP_SUB:
                r = (v[a] - v[c]) % P
            elif op == S.OP_MUL:
                r = v[a] * v[c] % P
            else:
                acc = [(s * al + v[a] * sel[c]) % P for s, al in zip(acc, alphas)]
            v.append(r)
        for k in range(n_alphas):
            q[k, i] = acc[k] * E.inverse(zh) % P
    check_quotient_values(b, consts, alphas, q, tv, av, log_n, qd_bits)
    for k, i in [(0, 0), (n_alphas - 1, size - 1), (0, 1), (n_alphas // 2, size // 2 + 3)]:
        bad = q.copy()
        bad[k, i] = (bad[k, i] + np.uint64(1)) % np.uint64(P)
        with pytest.raises(AssertionError):
            check_quotient_values(b, consts, alphas, bad, tv, av, log_n, qd_bits)


QUOTIENT_CASES = ["plain_20_r1_a4", "plain_22_r3_a1", "aux_20_r1_a2"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", QUOTIENT_CASES)
def test_stark_quotient_at_every_coset_point(pb, case):
    """gl_stark_quotient[_aux]'s values, recovered from its coefficients by the coset FFT, satisfy
    q(x) Z_H(x) D(x) == sum_c alpha^(E-1-c) C_c(x) S_c(x) at every point of the coset (plain_22_r3: 2^25 points, quotient
    degree factor 8, past the 2^24 points where the power tables' hi part grows beyond its minimum)."""
    import torch

    from plonky2_b200.fft import coset_fft, ifft

    kind, log_n, rate, na = case.split("_")
    log_n, rate_bits, n_alphas = int(log_n), int(rate[1:]), int(na[1:])
    qdf = 8 if rate_bits == 3 else 2
    stark = AllOpsStark(qdf + 1)
    qd_bits = (qdf - 1).bit_length()
    n, size = 1 << log_n, 1 << (log_n + qd_bits)
    num_aux = 2 if kind == "aux" else 0
    b = quotient_program(stark, num_aux)
    used = {op for op, _, _ in b.instrs} | {S.OP_EMIT * 16 + c for op, _, c in b.instrs if op == S.OP_EMIT}
    assert {S.OP_LOCAL, S.OP_NEXT, S.OP_CONST, S.OP_ADD, S.OP_SUB, S.OP_MUL} <= used
    assert {S.OP_EMIT * 16 + k for k in range(4)} <= used
    pis = [int(synth(0xE70, (1,))[0])]
    consts = np.array(pis + b.consts[b.num_bound:], dtype=np.uint64)
    alphas = [int(v) for v in synth(0xE71 + log_n, (n_alphas,))]
    trace = synth(0xE72, (stark.COLUMNS, n))
    ctx = pb.default_context()
    tc = pb.PolynomialBatch.from_values(trace, rate_bits, False, 4)
    aux = aux_vals_host = None
    if num_aux:
        aux_vals_host = synth(0xE73, (num_aux, n))
        aux = pb.PolynomialBatch.from_values(aux_vals_host, rate_bits, False, 4)
    out = torch.empty((n_alphas, size), dtype=torch.int64, device="cuda")
    al = np.array(alphas, dtype=np.uint64)
    L = N.lib()
    if aux is None:
        rc = L.gl_stark_quotient(ctx.h, tc.h, b.program(), len(b.instrs), N.np_ptr(consts), len(consts), N.np_ptr(al),
                                 n_alphas, qdf, N.vp(out.data_ptr()))
    else:
        rc = L.gl_stark_quotient_aux(ctx.h, tc.h, aux.h, b.program(), len(b.instrs), N.np_ptr(consts), len(consts),
                                     N.np_ptr(al), n_alphas, qdf, N.vp(out.data_ptr()))
    N.check(rc, ctx.h)
    ctx.synchronize()
    coeffs = _to_host(out)
    del out
    tc.close()
    if aux is not None:
        aux.close()
    shift = E.coset_shift()
    q = coset_fft(coeffs, shift)
    del coeffs

    def coset_values(vals):            # the columns' values on the quotient coset, natural order
        pad = np.zeros((vals.shape[0], size), dtype=np.uint64)
        pad[:, :n] = ifft(vals)
        return coset_fft(pad, shift)

    check_quotient_values(b, consts, alphas, q, coset_values(trace), coset_values(aux_vals_host) if num_aux else None,
                          log_n, qd_bits)


# ------------------------------------------------------------------------------------------------ whole proofs
def replay_challenges(oracle, stark, config, proof, lookups):
    """The transcript up to zeta on the oracle's challenger, from the proof's caps and public inputs."""
    p = proof.proof
    degree_bits = p.recover_degree_bits(config)
    ch = oracle.Challenger()
    ch.observe_elements(list(proof.public_inputs))
    T.observe_config(ch, config)
    ch.observe_cap(p.trace_cap.hashes)
    pairs = betas = None
    num_aux = 0
    if lookups:
        pairs = T._draw_lookup_challenges(ch, config.num_challenges)
        betas = [bt for bt, _ in pairs]
        ch.observe_cap(p.auxiliary_polys_cap.hashes)
        num_aux = len(p.openings.auxiliary_polys)
    alphas = T.bind_constraints(ch, stark, list(proof.public_inputs), config.num_challenges, degree_bits, betas,
                                num_aux)
    ch.observe_cap(p.quotient_polys_cap.hashes)
    return pairs, alphas, ch.get_extension_challenge()


class _FriBytes:
    """A FRI proof whose bytes are given: what a verifier reads of a proof with one byte changed."""

    def __init__(self, fp, data):
        self._fp, self._data = fp, data

    def to_bytes(self):
        return self._data

    def __getattr__(self, k):
        return getattr(self._fp, k)


def _fri_byte_changed(proof):
    bad = copy.copy(proof)
    bad.proof = copy.copy(proof.proof)
    data = bytearray(proof.proof.opening_proof.to_bytes())
    data[len(data) // 2] ^= 4
    bad.proof.opening_proof = _FriBytes(proof.proof.opening_proof, bytes(data))
    return bad


def _opening_changed(proof, field):
    bad = copy.deepcopy(proof)
    getattr(bad.proof.openings, field)[0, 1] ^= np.uint64(1)
    return bad


def _check_replay(oracle, stark, config, proof, lookups):
    pairs, alphas, zeta = replay_challenges(oracle, stark, config, proof, lookups)
    ch = proof.get_challenges(stark, config)
    if lookups:
        assert [(c.beta, c.gamma) for c in ch["lookup_challenge_set"]] == pairs
    assert ch["stark_alphas"] == alphas and ch["stark_zeta"] == zeta


@pytest.mark.gpu
def test_prove_range_check_2_20_from_a_torch_trace(pb, oracle):
    stark, config = RangeCheckStark(), S.StarkConfig.standard_fast_config()
    trace = range_check_trace(20, seed=20)
    proof = S.prove(stark, config, _to_device(trace), [0])
    assert T.verify(oracle, stark, config, proof) is None
    _check_replay(oracle, stark, config, proof, True)
    assert T.verify(oracle, stark, config, _opening_changed(proof, "auxiliary_polys")) is not None
    assert T.verify(oracle, stark, config, _fri_byte_changed(proof)) is not None
    trace[MA, 5] += np.uint64(1)
    assert T.verify(oracle, stark, config, S.prove(stark, config, _to_device(trace), [0])) == (
        "Mismatch between evaluation and opening of quotient polynomial")


def _fibonacci_pairs():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import stark_prove_cost
    finally:
        sys.path.remove(os.path.join(ROOT, "tools"))
    return stark_prove_cost.FibonacciPairsStark(), stark_prove_cost.fibonacci_pairs_trace


@pytest.mark.gpu
def test_prove_fibonacci_pairs_2_22(pb, oracle):
    """64 columns x 2^22 rows at standard_fast_config, the trace written on the device."""
    stark, gen = _fibonacci_pairs()
    config = S.StarkConfig.standard_fast_config()
    trace = gen(22)
    proof = S.prove(stark, config, trace, [])
    assert T.verify(oracle, stark, config, proof) is None
    _check_replay(oracle, stark, config, proof, False)
    assert T.verify(oracle, stark, config, _opening_changed(proof, "local_values")) is not None
    assert T.verify(oracle, stark, config, _fri_byte_changed(proof)) is not None
    trace[3, 1000] += 1
    assert T.verify(oracle, stark, config, S.prove(stark, config, trace, [])) is not None


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", [22, pytest.param(24, marks=pytest.mark.skipif(
    os.environ.get("GL_LARGE_FRI_24") != "1", reason="64 x 2^24 FRI: set GL_LARGE_FRI_24=1 (its CPU side takes tens "
                                                     "of seconds)"))])
def test_fri_at_the_benchmarked_shape(pb, oracle, log_n):
    """A 64 x 2^log_n commitment at starky's standard_fast_config (rate 1/2, cap 4, arity 16, 84 queries): the FRI
    proof is accepted by the oracle's verifier, a copy with one byte changed is rejected, the openings match Horner on
    the CPU at two polynomials, and the value-domain begin gives a byte-identical proof."""
    from plonky2_b200 import fri as F

    B = 64
    vals = synth(0x05, (B, 1 << log_n))
    cfg = pb.starky_standard_fast_fri_config()
    r, h = cfg.rate_bits, cfg.cap_height
    params = cfg.fri_params(log_n, False)
    c = pb.PolynomialBatch.from_values(vals, r, False, h)
    del vals
    try:
        cap = c.merkle_tree.cap
        zeta = (0x1122334455667788 % P, 0x99AABBCCDDEEFF00 % P)
        gz = E.ext_mul(zeta, (E.primitive_root_of_unity(log_n), 0))
        inst = pb.FriInstanceInfo([pb.FriOracleInfo(B, False)],
                                  [pb.FriBatchInfo(zeta, [pb.FriPolynomialInfo(0, i) for i in range(B)]),
                                   pb.FriBatchInfo(gz, [pb.FriPolynomialInfo(0, 0), pb.FriPolynomialInfo(0, 1)])])
        ev_z, ev_gz = c.eval_commitment(zeta), c.eval_commitment(gz)
        ch = pb.Challenger()
        ch.observe_cap(cap)
        pbytes = pb.prove_openings(inst, [c], ch, params).to_bytes()
        co = c.polynomials
        assert tuple(int(v) for v in ev_z[3]) == oracle.eval_poly_base_at_ext(co[3], zeta)
        assert tuple(int(v) for v in ev_gz[1]) == oracle.eval_poly_base_at_ext(co[1], gz)
        del co
        opened = np.concatenate([ev_z.reshape(-1), ev_gz[:2].reshape(-1)])
        obatches = [(bt.point, [(p.oracle_index, p.polynomial_index) for p in bt.polynomials]) for bt in inst.batches]
        oparams = oracle.make_params(r, h, cfg.proof_of_work_bits, cfg.num_query_rounds, params.reduction_arity_bits)

        def verify(data):
            och = oracle.Challenger()
            och.observe_cap(cap.hashes)
            return oracle.verify_fri_proof([cap.hashes], [B], [B], obatches, opened, log_n, och, oparams, data)

        assert verify(pbytes) == 0
        bad = bytearray(pbytes)
        bad[len(bad) // 2] ^= 4
        assert verify(bytes(bad)) != 0
        ch2 = pb.Challenger()
        ch2.observe_cap(cap)
        st = F._begin_values(inst, [c], ch2.get_extension_challenge(), [ev_z, ev_gz[:2]], params)
        try:
            caps, final = F.fri_committed_trees(st, ch2, params)
            poww = F.fri_proof_of_work(ch2, params.config, st.ctx)
            rounds, _ = F.fri_prover_query_rounds([c], st, ch2, params.lde_size(), params)
            assert F.FriProof(caps, rounds, final, poww).to_bytes() == pbytes
        finally:
            st.close()
    finally:
        c.close()


def system_traces_equal_heights(log_n, seed=5):
    """Honest traces of test_stark_ctl.py's three-table system, every table 2^log_n rows, written with numpy: selectors
    on about one row in eight, so that the looked table has room for every looking tuple."""
    from test_stark_ctl import FREQ, LF, LF2, LK, LV, MG, MP, MQ, MR, MT, MW, RV, S0, S1, TBL, X0, X1, Y0, Y1

    rng = np.random.default_rng(seed)
    n = 1 << log_n
    cpu, mem, looked = (np.zeros((w, n), dtype=np.uint64) for w in (9, 6, 4))
    cpu[S0], cpu[S1], mem[MG] = ((rng.random(n) < 0.125).astype(np.uint64) for _ in range(3))
    for c in (X0, Y0, X1, Y1):
        cpu[c] = rng.integers(0, 1 << 40, n)
    for c in (MP, MQ, MR):
        mem[c] = rng.integers(0, 1 << 40, n)
    cpu[RV] = rng.integers(0, n, n)
    cpu[TBL] = np.arange(n)
    cpu[FREQ] = np.bincount(cpu[RV].astype(np.int64), minlength=n)
    mg = mem[MG] == 1
    keys = np.concatenate([cpu[X0][cpu[S0] == 1], cpu[X1][cpu[S1] == 1],
                           G.add(G.mul(mem[MP], np.uint64(2)), G.add(np.roll(mem[MQ], -1), np.uint64(5)))[mg]])
    vals = np.concatenate([cpu[Y0][cpu[S0] == 1], cpu[Y1][cpu[S1] == 1], mem[MR][mg]])
    assert len(keys) <= n // 2
    order = rng.permutation(n)[:len(keys)]
    looked[LK] = rng.integers(0, 1 << 40, n) + (1 << 50)
    looked[LV] = rng.integers(0, 1 << 40, n)
    looked[LK, order], looked[LV, order], looked[LF, order] = keys, vals, 1
    f2 = np.sort(rng.permutation(n)[:n // 2])
    looked[LF2, f2] = 1
    mem[MT, :len(f2)] = 1
    mem[MW, :len(f2)] = looked[LV, f2]
    mem[MW, len(f2):] = rng.integers(0, 1 << 40, n - len(f2))
    return [cpu, mem, looked], [[], [], [int(looked[LK, 0])]]


def test_equal_height_system_traces_satisfy_the_ctls():
    traces, _ = system_traces_equal_heights(8)
    X.check_ctls(traces, system_ctls())


@pytest.mark.gpu
def test_prove_with_ctls_2_18(pb, oracle):
    """The three-table system at 2^18 rows per table: accepted by the restated verifier; with one looking tuple moved
    where its filter is on, every table still proves and the cross-table check rejects."""
    from test_stark_ctl import MG, MR, system

    starks, config, ctls = system()
    traces, pis = system_traces_equal_heights(18)
    X.check_ctls(traces, ctls)
    mp = X.prove_with_ctls(starks, config, traces, ctls, pis)
    assert T.verify_with_ctls(oracle, starks, config, ctls, mp) is None
    on = int(np.nonzero(traces[1][MG])[0][0])
    traces[1][MR, on] += np.uint64(1)
    mp = X.prove_with_ctls(starks, config, traces, ctls, pis)
    assert T.verify_with_ctls(oracle, starks, config, ctls, mp) == "Cross-table lookup 0 verification failed."
