"""starky's cross-table lookups (cross_table_lookup.py, gl_stark_ctl_helpers, the CTL constraints in the STARK quotient,
prove_with_ctls).

The test system has three tables of different heights, all with num_challenges = 2:
- CpuTable (2^5 rows, degree 3) looks twice into CTL 0 (two consecutive entries: one helper column per challenge at
  degree 3), and has its own logUp range check, whose betas come from the CTL challenges.
- MemTable (2^4 rows, no CTL helper columns) looks into CTL 0 with the tuple (2 p + q(next row) + 5, r) and is
  the looked table of CTL 1.
- LookedTable (2^6 rows, degree 3) is CTL 0's looked table and looks into CTL 1.

CPU: the restatement (tests/stark_twin.py) pinned by the CTL invariant and every column identity; the CTL terms of
eval_vanishing_poly against hand-written formulas; the device row arithmetic run on the host (tests/emu/ctl_emu.cpp)
against the restatement; prove_with_ctls's host logic with the oracle standing in for the device calls (field-for-field
equal to the twin, accepted by the restated verifier, its transcript replayed by MultiStarkProof.get_challenges,
tampering rejected); every shape error.

GPU (-m gpu): device CTL columns against the restatement, one table at 2^16 rows; prove_with_ctls against the twin from
host and torch device traces; a mismatched system; extra looking sums; gl_stark_ctl_helpers's error codes."""
import copy
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import stark_twin as T
from conftest import P, synth
from plonky2_b200 import _native as N
from plonky2_b200 import cross_table_lookup as X
from plonky2_b200 import field as E
from plonky2_b200 import stark as S
from plonky2_b200.cross_table_lookup import CrossTableLookup, TableWithColumns, check_ctls
from plonky2_b200.lookup import Column, Filter, GrandProductChallenge, Lookup

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

X0, Y0, S0, X1, Y1, S1, RV, TBL, FREQ = range(9)         # CpuTable
MP, MQ, MR, MG, MW, MT = range(6)                        # MemTable
LK, LV, LF, LF2 = range(4)                               # LookedTable


class CpuTable(S.Stark):
    COLUMNS, PUBLIC_INPUTS = 9, 0

    def eval(self, v, y):
        for s in (S0, S1):
            y.constraint(v.local(s) * v.local(s) - v.local(s))

    def constraint_degree(self):
        return 3

    def lookups(self):
        return [Lookup([Column.single(RV)], Column.single(TBL), Column.single(FREQ), [Filter.default()])]

    def requires_ctls(self):
        return True


class MemTable(S.Stark):
    COLUMNS, PUBLIC_INPUTS = 6, 0

    def eval(self, v, y):
        y.constraint(v.local(MG) * v.local(MG) - v.local(MG))

    def constraint_degree(self):
        # a CTL's Z checks are combine * Z (degree 2) under a row filter: degree 3, whatever the table's own degree
        return 3

    def requires_ctls(self):
        return True


class LookedTable(S.Stark):
    COLUMNS, PUBLIC_INPUTS = 4, 1

    def eval(self, v, y):
        y.constraint(v.local(LF) * v.local(LF) - v.local(LF))
        y.constraint_first_row(v.local(LK) - v.public_input(0))

    def constraint_degree(self):
        return 3

    def requires_ctls(self):
        return True


MEM_TUPLE = [Column.linear_combination_and_next_row_with_constant([(MP, 2)], [(MQ, 1)], 5), Column.single(MR)]


def system_ctls():
    ctl0 = CrossTableLookup([TableWithColumns(0, Column.singles([X0, Y0]), Filter.new_simple(Column.single(S0))),
                             TableWithColumns(0, Column.singles([X1, Y1]), Filter.new_simple(Column.single(S1))),
                             TableWithColumns(1, MEM_TUPLE, Filter.new_simple(Column.single(MG)))],
                            TableWithColumns(2, Column.singles([LK, LV]), Filter.new_simple(Column.single(LF))))
    ctl1 = CrossTableLookup([TableWithColumns(2, [Column.single(LV)], Filter.new_simple(Column.single(LF2)))],
                            TableWithColumns(1, [Column.single(MW)], Filter.new_simple(Column.single(MT))))
    return [ctl0, ctl1]


def system_traces(log_cpu=5, log_mem=4, log_looked=6, seed=3):
    """Traces satisfying both CTLs; the looked table's public input is its first k."""
    rng = np.random.default_rng(seed)
    nc, nm, nl = 1 << log_cpu, 1 << log_mem, 1 << log_looked
    cpu = np.zeros((9, nc), dtype=np.uint64)
    mem = np.zeros((6, nm), dtype=np.uint64)
    looked = np.zeros((4, nl), dtype=np.uint64)
    budget = nl // 2
    cpu[S0] = rng.integers(0, 2, nc)
    cpu[S1] = rng.integers(0, 2, nc)
    mem[MG] = rng.integers(0, 2, nm)
    while int(cpu[S0].sum() + cpu[S1].sum() + mem[MG].sum()) > budget:
        cpu[S1, int(np.nonzero(cpu[S1])[0][0])] = 0
    for c in (X0, Y0, X1, Y1):
        cpu[c] = rng.integers(0, 1 << 40, nc)
    for c in (MP, MQ, MR):
        mem[c] = rng.integers(0, 1 << 40, nm)
    cpu[RV] = rng.integers(0, nc, nc)
    cpu[TBL] = np.arange(nc)
    cpu[FREQ] = np.bincount(cpu[RV].astype(np.int64), minlength=nc)
    rows = [(int(cpu[X0, i]), int(cpu[Y0, i])) for i in range(nc) if cpu[S0, i]]
    rows += [(int(cpu[X1, i]), int(cpu[Y1, i])) for i in range(nc) if cpu[S1, i]]
    rows += [((2 * int(mem[MP, i]) + int(mem[MQ, (i + 1) % nm]) + 5) % P, int(mem[MR, i])) for i in range(nm) if mem[MG, i]]
    order = rng.permutation(nl)[:len(rows)]
    looked[LK] = rng.integers(0, 1 << 40, nl) + (1 << 50)
    looked[LV] = rng.integers(0, 1 << 40, nl)
    for r, (k, v) in zip(order, rows):
        looked[LK, r], looked[LV, r], looked[LF, r] = k, v, 1
    f2 = rng.permutation(nl)[:nm // 2]
    looked[LF2, f2] = 1
    mem[MT, :len(f2)] = 1
    mem[MW, :len(f2)] = looked[LV, np.sort(f2)]
    mem[MW, len(f2):] = rng.integers(0, 1 << 40, nm - len(f2))
    return [cpu, mem, looked], [[], [], [int(looked[LK, 0])]]


def system():
    return [CpuTable(), MemTable(), LookedTable()], S.StarkConfig.standard_fast_config(), system_ctls()


def _pairs(seed):
    v = [int(x) for x in synth(seed, (4,))]
    return [(v[0], v[1]), (v[2], v[3])]


# ----------------------------------------------------------------------------------------------------------- CPU
def test_ctl_invariant_pins_the_restatement():
    """Sum over distinct looking tables of Z[0] equals the looked table's Z[0] exactly when check_ctls accepts; every
    Z and helper column satisfies its transition and last-row identity on every row."""
    starks, _, ctls = system()
    traces, _ = system_traces()
    check_ctls(traces, ctls)
    pairs = _pairs(0xA00)
    data = T.cross_table_lookup_data(traces, ctls, pairs, 3)
    assert [len(d) for d in data] == [2, 4, 4]
    firsts = [[int(z["z"][0]) for z in d] for d in data]
    # CTL 0: table 0 (group), table 1, looked table 2; CTL 1: table 2 looking, table 1 looked
    assert [len(z["helpers"]) for z in data[0]] == [1, 1]
    for c in range(2):
        assert (firsts[0][c] + firsts[1][c]) % P == firsts[2][c]
        assert firsts[2][2 + c] == firsts[1][2 + c]
    for t, d in enumerate(data):
        for z in d:
            beta, gamma = z["challenge"]
            h = [np.array(x, dtype=object) for x in z["helpers"]]
            zz = np.array(z["z"], dtype=object)
            tr = traces[t]
            if h:
                row = sum(h, np.zeros(len(zz), dtype=object)) % P
                for k, hk in enumerate(h):      # chunk k of two entries: h * c0 * c1 = f0 c1 + f1 c0
                    ents = list(zip(z["columns"], z["filter"]))[2 * k:2 * k + 2]
                    cs = [T.combine_rows(cols, tr, beta, gamma) for cols, _ in ents]
                    fs = [T.filter_eval_table(f, tr) for _, f in ents]
                    assert all(v % P == 0 for v in (hk * cs[0] * cs[1] - fs[0] * cs[1] - fs[1] * cs[0]))
            else:
                c0 = T.combine_rows(z["columns"][0], tr, beta, gamma)
                row = T._inv_each(c0) * T.filter_eval_table(z["filter"][0], tr) % P
            assert zz[-1] == row[-1]
            assert all((zz[:-1] - zz[1:] - row[:-1]) % P == 0)
    # a tuple moved where its filter is on breaks the check and the sums; one moved where it is off does not
    bad = [t.copy() for t in traces]
    on = int(np.nonzero(bad[1][MG])[0][0])
    bad[1][MR, on] += np.uint64(1)
    with pytest.raises(ValueError, match="Cross-table lookup 0"):
        check_ctls(bad, ctls)
    d = T.cross_table_lookup_data(bad, ctls, pairs, 3)
    assert all((int(d[0][c]["z"][0]) + int(d[1][c]["z"][0])) % P != int(d[2][c]["z"][0]) for c in range(2))
    off = [t.copy() for t in traces]
    o = int(np.nonzero(off[1][MG] == 0)[0][0])
    off[1][MR, o] += np.uint64(1)
    check_ctls(off, ctls)
    d = T.cross_table_lookup_data(off, ctls, pairs, 3)
    assert all((int(d[0][c]["z"][0]) + int(d[1][c]["z"][0])) % P == int(d[2][c]["z"][0]) for c in range(2))
    # extra looking values: a looked row nobody looks up
    extra = [t.copy() for t in traces]
    free = int(np.nonzero(extra[2][LF] == 0)[0][0])
    extra[2][LF, free] = 1
    with pytest.raises(ValueError):
        check_ctls(extra, ctls)
    check_ctls(extra, ctls, {0: [(int(extra[2][LK, free]), int(extra[2][LV, free]))]})


class _Ctl0(S.Stark):
    """A Stark without constraints of its own, for the CTL terms alone."""
    COLUMNS, PUBLIC_INPUTS = 4, 0

    def eval(self, v, y):
        pass

    def constraint_degree(self):
        return 3

    def requires_ctls(self):
        return True


def test_eval_vanishing_poly_ctl_terms_match_hand_written_formulas():
    """The helper case (Z - sum h on the last row, Z - Z' - sum h as a transition, h c0 c1 - f0 c1 - f1 c0), the
    single-entry case and the two-entry case without helper columns, at a random point."""
    log_n = 4
    x = tuple(int(v) for v in synth(0xA10, (2,)))
    loc = [tuple(int(v) for v in synth(0xA11 + k, (2,))) for k in range(4)]
    nxt = [tuple(int(v) for v in synth(0xA21 + k, (2,))) for k in range(4)]
    h, z, zn = [tuple(int(v) for v in synth(0xA31 + k, (2,))) for k in range(3)]
    ch = GrandProductChallenge(*[int(v) for v in synth(0xA40, (2,))])
    alpha = int(synth(0xA41, (1,))[0])
    l0, llast = S.eval_l_0_and_l_last(log_n, x)
    zlast = E.ext_sub(x, (E.inverse(E.primitive_root_of_unity(log_n)), 0))
    add, sub, mul = E.ext_add, E.ext_sub, E.ext_mul
    b = lambda v: (v % P, 0)  # noqa: E731
    cols_a = [Column.single(0), Column.linear_combination_and_next_row_with_constant([(1, 3)], [(2, 1)], 7)]
    cols_b = [Column.single(3), Column.single_next_row(0)]
    fa, fb = Filter.new_simple(Column.single(2)), Filter.new([(Column.single(1), Column.single_next_row(3))], [])

    def comb(vals):
        acc = (0, 0)
        for v in reversed(vals):
            acc = add(mul(acc, b(ch.beta)), v)
        return add(acc, b(ch.gamma))

    va = [loc[0], add(add(mul(loc[1], b(3)), nxt[2]), b(7))]
    vb = [loc[3], nxt[0]]
    ffa, ffb = loc[2], mul(loc[1], nxt[3])
    ca, cb = comb(va), comb(vb)

    def fold(cs):
        acc = (0, 0)
        for c in cs:
            acc = add(mul(acc, b(alpha)), c)
        return acc

    def run(vars_):
        return S.eval_vanishing_poly(_Ctl0(), loc, nxt, [], [alpha], x, log_n, [], [], ctl_vars=vars_)[0]

    with_h = X.CtlCheckVars([h], z, zn, ch, [cols_a, cols_b], [fa, fb])
    hsum = h
    want = [sub(sub(mul(mul(cb, ca), h), mul(ffa, cb)), mul(ffb, ca)), mul(sub(z, hsum), llast),
            mul(sub(sub(z, zn), hsum), zlast)]
    assert run([with_h]) == fold(want)
    one = X.CtlCheckVars([], z, zn, ch, [cols_a], [fa])
    want1 = [mul(sub(mul(ca, z), ffa), llast), mul(sub(mul(ca, sub(z, zn)), ffa), zlast)]
    assert run([one]) == fold(want1)
    two = X.CtlCheckVars([], z, zn, ch, [cols_a, cols_b], [fa, fb])
    t = lambda zz: sub(sub(mul(mul(ca, cb), zz), mul(ffa, cb)), mul(ffb, ca))  # noqa: E731
    want2 = [mul(t(z), llast), mul(t(sub(z, zn)), zlast)]
    assert run([two]) == fold(want2)
    assert run([with_h, one]) == fold(want + want1)


@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ctl_emu") / "libctl_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DGL_FORCE_32BIT_PATH", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "emu", "ctl_emu.cpp")])
    L = C.CDLL(out)
    L.emu_stark_ctl_helpers.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                        C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    return L


def _groups_and_aux(traces, ctls, t, pairs, degree):
    groups = X.table_groups(ctls, t)
    want = T.ctl_aux(T.cross_table_lookup_data(traces, ctls, pairs, degree)[t], traces[t].shape[1])
    return groups, want


def _emu(L, trace, groups, pairs, degree):
    trace = np.ascontiguousarray(trace, dtype=np.uint64)
    n = trace.shape[1]
    prog, offsets, consts = X.ctl_row_programs(groups, trace.shape[0])
    zs_index, _, nh = X.zs_layout(groups, len(pairs), degree)
    ch = np.array([v for pr in pairs for v in pr], dtype=np.uint64)
    out = np.zeros((nh + len(zs_index), n), dtype=np.uint64)
    consts = consts if len(consts) else np.zeros(1, dtype=np.uint64)
    rc = L.emu_stark_ctl_helpers(trace.ctypes.data, n, n.bit_length() - 1, C.addressof(prog), offsets.ctypes.data,
                                 len(offsets) - 1, consts.ctypes.data, ch.ctypes.data, len(pairs), degree,
                                 zs_index.ctypes.data, out.ctypes.data)
    return rc, out


def _wide_ctls():
    """1, 2 and 3 entries of three-column tuples with next-row terms and constants, table 0 looking into table 1."""
    tup = lambda a: [Column.single(a), Column.linear_combination_and_next_row_with_constant([(a + 1, 5)], [(a, 1)], 11),  # noqa: E731
                     Column.constant(9)]
    f = lambda c: Filter.new([(Column.single(c), Column.single_next_row(c))], [Column.single(c + 1)])  # noqa: E731
    looked = TableWithColumns(1, tup(0), f(3))
    return [CrossTableLookup([TableWithColumns(0, tup(0), f(6))], looked),
            CrossTableLookup([TableWithColumns(0, tup(1), f(6)), TableWithColumns(0, tup(2), Filter.default())], looked),
            CrossTableLookup([TableWithColumns(0, tup(k), f(k + 3)) for k in range(3)], looked)]


@pytest.mark.parametrize("degree", [3, 4])
def test_ctl_rows_on_host_match_restatement(emu_lib, degree):
    """The kernel's row source on the host equals the restatement bit for bit: the test system's tables, and groups of
    1, 2 and 3 entries with three-column tuples, next-row terms and constants (degree 4: one chunk of three)."""
    pairs = _pairs(0xA50)
    if degree == 3:
        traces, _ = system_traces()
        ctls = system_ctls()
        for t in range(3):
            groups, want = _groups_and_aux(traces, ctls, t, pairs, 3)
            rc, got = _emu(emu_lib, traces[t], groups, pairs, 3)
            assert rc == 0 and np.array_equal(got, want), t
    traces = [synth(0xA60, (8, 32)), synth(0xA61, (8, 32))]
    ctls = _wide_ctls()
    for t in range(2):
        groups, want = _groups_and_aux(traces, ctls, t, pairs, degree)
        rc, got = _emu(emu_lib, traces[t], groups, pairs, degree)
        assert rc == 0 and np.array_equal(got, want), t
    # a challenge making one row's combine vanish: the batch inversion meets zero
    groups = X.table_groups(ctls, 1)
    v = [int(traces[1][0, 0]), (int(traces[1][1, 0]) * 5 + int(traces[1][0, 1]) + 11) % P, 9]
    beta = 3
    gamma = (-(v[0] + beta * v[1] + beta * beta * v[2])) % P
    rc, _ = _emu(emu_lib, traces[1], groups, [(beta, gamma)], degree)
    assert rc == 1


def _cpu_ctl_backends(monkeypatch, oracle, calls):
    from test_stark_lookups import _cpu_lookup_backends

    logs, ctx = _cpu_lookup_backends(monkeypatch, oracle, CpuTable(), calls)

    def lookup_helpers(stark_, trace, challenges, ctx_, out=None):
        calls.append(("helpers", [int(c) for c in challenges]))
        cols = T.aux_columns(stark_, np.asarray(trace), challenges)[0]
        if out is None:
            return cols
        out[...] = cols
        return out

    def ctl_helpers(trace, groups, ctl_challenges, degree, ctx_, out):
        calls.append(("ctl", len(groups)))
        pairs = [(c.beta, c.gamma) for c in ctl_challenges]
        out[...] = _restated_table_aux(np.asarray(trace), groups, pairs, degree)

    def quotient(stark_, tc, pis, alphas, auxiliary_polys_commitment=None, lookup_challenges=None, ctl_vars=None):
        aux = auxiliary_polys_commitment.o.coeffs if auxiliary_polys_commitment is not None else None
        return T.host_quotient(oracle, stark_, tc.o.coeffs, pis, alphas, aux, lookup_challenges or [], ctl_vars or [])

    import plonky2_b200.fri as fri_mod

    oracle_fri = fri_mod.prove_openings

    def prove_openings(instance, oracles, challenger, fri_params, final_poly_coeff_len=None, max_num_query_steps=None):
        """The oracle's FRI proof; the product's challenger then takes FRI's transcript from the proof (as the device
        prover's does), since the next table continues on it."""
        fp = oracle_fri(instance, oracles, challenger, fri_params, final_poly_coeff_len, max_num_query_steps)
        fri_mod.fri_challenges(challenger, fp.commit_phase_merkle_caps, fp.final_poly, fp.pow_witness,
                               fri_params.degree_bits, fri_params.config, final_poly_coeff_len, max_num_query_steps)
        return fp

    monkeypatch.setattr(fri_mod, "prove_openings", prove_openings)
    monkeypatch.setattr(S, "compute_lookup_helper_columns", lookup_helpers)
    monkeypatch.setattr(X, "compute_ctl_helper_columns", ctl_helpers)
    monkeypatch.setattr(X, "_alloc_auxiliary", lambda rows, n, trace: np.zeros((rows, n), dtype=np.uint64))
    monkeypatch.setattr(S, "compute_quotient_polys", quotient)
    return logs, ctx


def _restated_table_aux(trace, groups, pairs, degree):
    """The restatement's CTL columns of one table from its groups: per CTL, per challenge, per group partial_sums."""
    helpers, zs = [], []
    for i in sorted({c for c, _ in groups}):
        for pr in pairs:
            for c, entries in groups:
                if c == i:
                    cols = T.partial_sums(trace, [(t.columns, t.filter) for t in entries], pr, degree)
                    helpers += cols[:-1]
                    zs.append(cols[-1])
    return np.stack(helpers + zs)


def _tampered(mp, what):
    bad = copy.deepcopy(mp)
    if what == "ctl_zs_first":
        bad.stark_proofs[2].proof.openings.ctl_zs_first[0] ^= np.uint64(1)
    elif what == "ctl_z_opening":
        bad.stark_proofs[0].proof.openings.auxiliary_polys[-1, 0] ^= np.uint64(1)
    else:
        bad.stark_proofs[0], bad.stark_proofs[1] = bad.stark_proofs[1], bad.stark_proofs[0]
    return bad


def test_prove_with_ctls_host_logic_with_cpu_backends(oracle, monkeypatch):
    starks, config, ctls = system()
    traces, pis = system_traces()
    twin = T.twin_prove_with_ctls(oracle, starks, config, traces, ctls, pis)
    calls = []
    logs, ctx = _cpu_ctl_backends(monkeypatch, oracle, calls)
    mp = X.prove_with_ctls(starks, config, traces, ctls, pis, ctx=ctx)
    T.assert_matches_twin(mp, twin)
    assert T.verify_with_ctls(oracle, starks, config, ctls, mp) is None
    betas = [b for b, _ in twin["ctl_challenges"]]
    assert [c for c in calls if isinstance(c, tuple) and c[0] == "helpers"] == [("helpers", betas)]
    assert [c for c in calls if isinstance(c, tuple) and c[0] == "ctl"] == [("ctl", 1), ("ctl", 2), ("ctl", 2)]
    assert calls.count("close") == 9
    ch = mp.get_challenges(starks, config, ctls)
    assert [(c.beta, c.gamma) for c in ch["ctl_challenges"]] == twin["ctl_challenges"]
    for got, t in zip(ch["stark_challenges"], twin["tables"]):
        assert got["stark_alphas"] == t["alphas"] and got["stark_zeta"] == t["zeta"]
    prover_draws = [v for kind, v in logs[0] if kind == "challenge"]
    replay_draws = [v for kind, v in logs[1] if kind == "challenge"]
    assert replay_draws[:len(prover_draws)] == prover_draws
    for what in ("ctl_zs_first", "ctl_z_opening", "swapped"):
        assert T.verify_with_ctls(oracle, starks, config, ctls, _tampered(mp, what)) is not None, what
    assert T.verify_with_ctls(oracle, starks, config, ctls, _tampered(mp, "ctl_zs_first")).startswith("table 2")


class _Deg1(MemTable):
    def constraint_degree(self):
        return 1


class _NoCtl(MemTable):
    def requires_ctls(self):
        return False


class _Cpu2(CpuTable):
    def constraint_degree(self):
        return 2


def test_shape_errors(oracle, monkeypatch):
    starks, config, ctls = system()
    traces, pis = system_traces()
    calls = []
    _, ctx = _cpu_ctl_backends(monkeypatch, oracle, calls)

    def refused(match, starks_=starks, traces_=traces, ctls_=ctls, pis_=pis):
        with pytest.raises(N.ShapeError, match=match):
            X.prove_with_ctls(starks_, config, traces_, ctls_, pis_, ctx=ctx)

    refused("expected 3 traces", traces_=traces[:2])
    refused("public-input lists", pis_=pis[:2])
    refused("COLUMNS", traces_=[traces[1], traces[0], traces[2]])
    refused("public inputs", pis_=[[], [], []])
    bad_idx = system_ctls() + [CrossTableLookup([TableWithColumns(5, [Column.single(0)], Filter.default())],
                                                TableWithColumns(1, [Column.single(MW)], Filter.default()))]
    refused("names table 5", ctls_=bad_idx)
    refused("requires_ctls", starks_=[starks[0], _NoCtl(), starks[2]])
    refused("takes no part", starks_=starks + [CpuTable()], traces_=traces + [traces[0]], pis_=pis + [[]])
    # degree 1 with CTL helper columns: table 0 looks twice at degree 1 (all tables degree <= 1)
    c0 = system_ctls()[0]
    refused("divide by zero", starks_=[_Deg1(), _Deg1()], traces_=[traces[1], traces[1]], pis_=[[], []],
            ctls_=[CrossTableLookup([TableWithColumns(0, MEM_TUPLE, Filter.default()),
                                     TableWithColumns(0, MEM_TUPLE, Filter.default())],
                                    TableWithColumns(1, MEM_TUPLE, Filter.default()))])
    three = CrossTableLookup(c0.looking_tables[:2] + [c0.looking_tables[0]] + c0.looking_tables[2:], c0.looked_table)
    from test_stark_lookups import T_config_rate2

    with pytest.raises(N.ShapeError, match="Allow other constraint degrees"):
        class Cpu4(CpuTable):
            def constraint_degree(self):
                return 4

            def lookups(self):
                return []
        X.prove_with_ctls([Cpu4(), starks[1], starks[2]], T_config_rate2(), traces, [three], pis, ctx=ctx)
    split = CrossTableLookup([c0.looking_tables[0], c0.looking_tables[2], c0.looking_tables[1]], c0.looked_table)
    refused("not consecutive", ctls_=[split, system_ctls()[1]])
    both = CrossTableLookup(c0.looking_tables + [TableWithColumns(2, Column.singles([LK, LV]), Filter.default())],
                            c0.looked_table)
    refused("both looked and looking", ctls_=[both, system_ctls()[1]])
    refused("constraint degree 2, not the system's 3", starks_=[_Cpu2(), starks[1], starks[2]])
    with pytest.raises(N.ShapeError, match="width"):
        CrossTableLookup([TableWithColumns(0, [Column.single(0)], Filter.default())], c0.looked_table)
    assert not [c for c in calls if c == "close" or isinstance(c, tuple)]
    assert CrossTableLookup.num_ctl_helpers_zs_all(ctls, 0, 2, 3) == (2, 2, [1, 0])
    assert CrossTableLookup.num_ctl_helpers_zs_all(ctls, 2, 2, 3) == (0, 4, [0, 0])


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

    return torch.from_numpy(np.ascontiguousarray(trace).view(np.int64)).cuda()


def _device_ctl(trace, groups, pairs, degree):
    import torch

    dev = _to_device(trace)
    zs_index, _, nh = X.zs_layout(groups, len(pairs), degree)
    out = torch.empty((nh + len(zs_index), trace.shape[1]), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    X.compute_ctl_helper_columns(dev, groups, [GrandProductChallenge(*p) for p in pairs], degree,
                                 N.default_context(), out)
    return out.cpu().numpy().view(np.uint64)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["system", "wide_3", "wide_4", "wide_16"])
def test_device_ctl_columns_equal_restatement(pb, case):
    pairs = _pairs(0xA70)
    if case == "system":
        traces, _ = system_traces()
        ctls, tables, degree = system_ctls(), range(3), 3
    else:
        log_n = 16 if case == "wide_16" else 6
        degree = 4 if case == "wide_4" else 3
        traces = [synth(0xA80, (8, 1 << log_n)), synth(0xA81, (8, 1 << log_n))]
        ctls, tables = _wide_ctls(), range(2)
    for t in tables:
        groups = X.table_groups(ctls, t)
        if case == "wide_16":
            want = _restated_table_aux(traces[t], groups, pairs, degree)
        else:
            _, want = _groups_and_aux(traces, ctls, t, pairs, degree)
        got = _device_ctl(traces[t], groups, pairs, degree)
        assert np.array_equal(got, want), (case, t)


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["host", "device"])
def test_prove_with_ctls_on_device_equals_cpu_twin(pb, oracle, source):
    import torch

    starks, config, ctls = system()
    traces, pis = system_traces()
    arg = traces if source == "host" else [_to_device(t) for t in traces]
    torch.cuda.synchronize()
    mp = X.prove_with_ctls(starks, config, arg, ctls, pis)
    twin = T.twin_prove_with_ctls(oracle, starks, config, traces, ctls, pis)
    T.assert_matches_twin(mp, twin)
    assert T.verify_with_ctls(oracle, starks, config, ctls, mp) is None
    ch = mp.get_challenges(starks, config, ctls)
    assert [(c.beta, c.gamma) for c in ch["ctl_challenges"]] == twin["ctl_challenges"]
    for got, t in zip(ch["stark_challenges"], twin["tables"]):
        assert got["stark_alphas"] == t["alphas"] and got["stark_zeta"] == t["zeta"]


@pytest.mark.gpu
def test_mismatched_system_proves_and_the_ctl_check_rejects(pb, oracle):
    """A looking tuple absent from the looked table: every table's STARK check passes (its Z columns are honest), and
    verify_cross_table_lookups rejects."""
    starks, config, ctls = system()
    traces, pis = system_traces()
    on = int(np.nonzero(traces[1][MG])[0][0])
    traces[1][MR, on] += np.uint64(1)
    with pytest.raises(ValueError):
        check_ctls(traces, ctls)
    mp = X.prove_with_ctls(starks, config, traces, ctls, pis)
    assert T.verify_with_ctls(oracle, starks, config, ctls, mp) == "Cross-table lookup 0 verification failed."


@pytest.mark.gpu
def test_extra_looking_sums(pb, oracle):
    """A looked row no table looks up: accepted with that row as an extra looking value, rejected without."""
    starks, config, ctls = system()
    traces, pis = system_traces()
    free = int(np.nonzero(traces[2][LF] == 0)[0][1])
    traces[2][LF, free] = 1
    row = (int(traces[2][LK, free]), int(traces[2][LV, free]))
    check_ctls(traces, ctls, {0: [row]})
    mp = X.prove_with_ctls(starks, config, traces, ctls, pis)
    ch = mp.get_challenges(starks, config, ctls)["ctl_challenges"]
    sums = [(pow((row[0] + c.beta * row[1] + c.gamma) % P, P - 2, P)) for c in ch]
    assert T.verify_with_ctls(oracle, starks, config, ctls, mp, {0: sums}) is None
    assert T.verify_with_ctls(oracle, starks, config, ctls, mp) == "Cross-table lookup 0 verification failed."


@pytest.mark.gpu
def test_entry_point_errors(pb):
    """gl_stark_ctl_helpers: a crafted challenge making a combine vanish -> GL_ERR_DIV_ZERO ("Tried to invert zero");
    the limits -> GL_ERR_UNSUPPORTED; an invalid program or zs_index -> GL_ERR_BAD_ARG; degree 1 with helper columns
    -> GL_ERR_BAD_SHAPE."""
    import torch

    ctx = pb.default_context()
    L = N.lib()
    trace = synth(0xA90, (8, 32))
    dev = _to_device(trace)
    out = torch.empty((64, 32), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    ctls = _wide_ctls()
    groups = X.table_groups(ctls, 0)
    prog, offsets, consts = X.ctl_row_programs(groups, 8)

    def call(pairs, degree=3, program=prog, offs=offsets, zs=None, cols=8):
        ch = np.array([v for p in pairs for v in p], dtype=np.uint64)
        zs = X.zs_layout(groups, len(pairs), 3)[0] if zs is None else zs   # positions do not depend on the degree
        return L.gl_stark_ctl_helpers(ctx.h, N.vp(dev.data_ptr()), 32, cols, 5, program, offs.ctypes.data_as(N.u32p),
                                      len(offs) - 1, N.np_ptr(consts), len(consts), N.np_ptr(ch), len(pairs), degree,
                                      zs.ctypes.data_as(N.u32p), N.vp(out.data_ptr()))

    assert call([(3, 4), (5, 6)]) == N.GL_OK
    v = [int(trace[0, 0]), (int(trace[1, 0]) * 5 + int(trace[0, 1]) + 11) % P, 9]
    zero = (-(v[0] + 3 * v[1] + 9 * v[2])) % P
    assert call([(3, zero)]) == N.GL_ERR_DIV_ZERO
    assert b"Tried to invert zero" in L.gl_last_error(ctx.h)
    assert call([(1, 2)] * 5) == N.GL_ERR_UNSUPPORTED
    assert call([(3, 4)], degree=1) == N.GL_ERR_BAD_SHAPE
    many = X.ctl_row_programs([(0, [TableWithColumns(0, [Column.single(0)], Filter.default())] * 9)], 8)
    assert call([(3, 4)], program=many[0], offs=many[1], zs=np.zeros(1, dtype=np.uint32)) == N.GL_ERR_UNSUPPORTED
    wide = X.ctl_row_programs([(0, [TableWithColumns(0, [Column.single(0)] * 33, Filter.default())])], 8)
    assert call([(3, 4)], program=wide[0], offs=wide[1], zs=np.zeros(1, dtype=np.uint32)) == N.GL_ERR_UNSUPPORTED
    ngroups = X.ctl_row_programs([(0, [TableWithColumns(0, [Column.single(0)], Filter.default())])] * 17, 8)
    assert call([(3, 4)], program=ngroups[0], offs=ngroups[1], zs=np.arange(17, dtype=np.uint32)) == N.GL_ERR_UNSUPPORTED
    long = np.zeros((257, 4), dtype=np.uint16)                        # LOCAL 0 ..., then one value and its filter
    long[-2:, 0], long[-2:, 2] = S.OP_EMIT, [X.CTL_VALUE, X.CTL_FILTER]
    one = np.zeros(1, dtype=np.uint32)
    assert call([(3, 4)], program=long[1:].ctypes.data, offs=np.array([0, 256], dtype=np.uint32), zs=one) == N.GL_OK
    before = ctx.launch_count
    assert call([(3, 4)], program=long.ctypes.data, offs=np.array([0, 257], dtype=np.uint32),
                zs=one) == N.GL_ERR_UNSUPPORTED
    assert b"CTL group 0: row program of 1..256 instructions" in L.gl_last_error(ctx.h) and ctx.launch_count == before
    assert call([(3, 4)], cols=2) == N.GL_ERR_BAD_ARG                 # a program reads column 7 of a 2-column trace
    assert call([(3, 4)], zs=np.zeros(3, dtype=np.uint32)) == N.GL_ERR_BAD_ARG
    assert b"permutation" in L.gl_last_error(ctx.h)
    open_entry = (S.StarkInstr * 2)()
    open_entry[0].op, open_entry[0].a = S.OP_LOCAL, 0
    open_entry[1].op, open_entry[1].a, open_entry[1].b = S.OP_EMIT, 0, X.CTL_VALUE
    assert call([(3, 4)], program=open_entry, offs=np.array([0, 2], dtype=np.uint32),
                zs=np.zeros(1, dtype=np.uint32)) == N.GL_ERR_BAD_ARG
