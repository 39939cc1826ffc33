"""starky's logUp lookups (lookup.py, gl_stark_lookup_helpers, gl_stark_quotient_aux, stark.prove with an auxiliary
commitment).

Two test STARKs: the reference's PermutationStark (permutation_stark.rs: constraint degree 0, so no quotient and the
lookup constraints are never checked, but the proof carries the auxiliary cap and openings), and RangeCheckStark, of
degree 3, whose quotient does constrain its helper columns: two lookups share one table column; the first has three
looking columns (chunks of 2 + 1), one of them a linear combination with a next-row term, a new_simple filter and a
product filter; the generator writes the frequencies and puts out-of-range values wherever a filter is off.

CPU: eval_vanishing_poly's lookup terms against hand-written formulas; the device row arithmetic run on the host
(tests/emu/logup_emu.cpp) bit-exact against the restatement of lookup_helper_columns (tests/stark_twin.py),
wrap-around next-row terms included; the logUp invariant pinning that restatement; prove's host logic with the oracle
standing in for the device calls (accepted by the restated verifier, field-for-field equal to the CPU twin, transcript
replayed by get_challenges, tampering rejected); every shape error.

GPU (-m gpu): device helper columns against the restatement at 2^10 and 2^20 rows; stark.prove against the twin for
both STARKs, from host columns and a torch device trace; a wrong frequency; the entry points' error codes; a lookup-free
proof through the same prove."""
import copy
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import stark_twin as T
from conftest import P, synth
from plonky2_b200 import _native as N
from plonky2_b200 import field as E
from plonky2_b200 import stark as S
from plonky2_b200.lookup import Column, Filter, Lookup, row_programs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class PermutationStark(S.Stark):
    """permutation_stark.rs: columns (i, j, frequency), column 0 looked up in column 1; no constraints of its own."""
    COLUMNS, PUBLIC_INPUTS = 3, 1

    def __init__(self, num_rows):
        self.num_rows = num_rows

    def generate_trace(self, x0):
        """permutation_stark.rs:38-51: rows (x0 + i, x0 + i + 1, 1), the last row's column 1 set to x0."""
        n = self.num_rows
        tr = np.empty((3, n), dtype=np.uint64)
        tr[0] = (np.arange(n, dtype=np.uint64) + np.uint64(x0))
        tr[1] = tr[0] + np.uint64(1)
        tr[2] = 1
        tr[1, n - 1] = x0
        return tr

    def eval(self, v, y):
        pass

    def constraint_degree(self):
        return 0

    def lookups(self):
        return [Lookup([Column.single(0)], Column.single(1), Column.single(2), [Filter.default()])]


A0, A1, E_, G, B, SEL, SEL2, TABLE, MA, MB = range(10)


class RangeCheckStark(S.Stark):
    """Limbs A0, A1, the combination E + G(next row) + 3 and B range-checked against TABLE (0, 1, ..., T - 1 repeated)
    with the frequency columns MA, MB; SEL and SEL2 are boolean selectors, TABLE starts at the public input."""
    COLUMNS, PUBLIC_INPUTS = 10, 1

    def __init__(self, degree=3):
        self.degree = degree

    def eval(self, v, y):
        s, s2 = v.local(SEL), v.local(SEL2)
        y.constraint(s * s - s)
        y.constraint(s2 * s2 - s2)
        y.constraint_first_row(v.local(TABLE) - v.public_input(0))

    def constraint_degree(self):
        return self.degree

    def lookups(self):
        combo = Column.linear_combination_and_next_row_with_constant([(E_, 1)], [(G, 1)], 3)
        return [Lookup([Column.single(A0), Column.single(A1), combo], Column.single(TABLE), Column.single(MA),
                       [Filter.new_simple(Column.single(SEL)), Filter.default(),
                        Filter.new([(Column.single(SEL), Column.single(SEL2))], [])]),
                Lookup([Column.single(B)], Column.single(TABLE), Column.single(MB),
                       [Filter.new_simple(Column.single(SEL2))])]

    @staticmethod
    def generate_trace(log_n, seed=7, table_bits=16, count_combination=True):
        n = 1 << log_n
        T_ = min(n, 1 << table_bits)
        rng = np.random.default_rng(seed)
        u = lambda: rng.integers(0, T_, n).astype(np.uint64)  # noqa: E731
        junk = np.uint64(1 << 40) + np.arange(n, dtype=np.uint64)     # out of range where a filter is off
        tr = np.zeros((10, n), dtype=np.uint64)
        s, s2 = rng.integers(0, 2, n).astype(np.uint64), rng.integers(0, 2, n).astype(np.uint64)
        s[n - 1] = s2[n - 1] = 1          # the last row's combination (which reads row 0) is looked up: the wrap counts
        tr[SEL], tr[SEL2] = s, s2
        tr[A0] = np.where(s == 1, u(), junk)
        tr[A1] = u()
        both = (s * s2) == 1
        target = np.where(both, u(), junk + np.uint64(1 << 20))
        tr[G] = u()
        tr[E_] = [(int(t) - int(g) - 3) % P for t, g in zip(target, np.roll(tr[G], -1))]
        tr[B] = np.where(s2 == 1, u(), junk)
        tr[TABLE] = np.arange(n, dtype=np.uint64) % np.uint64(T_)
        looked = [tr[A0][s == 1], tr[A1]] + ([target[both]] if count_combination else [])
        tr[MA, :T_] = np.bincount(np.concatenate(looked).astype(np.int64), minlength=T_)
        tr[MB, :T_] = np.bincount(tr[B][s2 == 1].astype(np.int64), minlength=T_)
        return tr


class RangeCheckStark4(RangeCheckStark):
    """RangeCheckStark at constraint degree 4 (rate 1/4) without the combination column: quotient degree factor 3, so
    the quotient's top chunk must vanish (at degree 3 the factor is 2 and the reference's trim cannot fail); its
    lookups keep to two looking columns, the longest chunk eval_helper_columns handles."""

    def __init__(self):
        super().__init__(degree=4)

    def lookups(self):
        a, b = super().lookups()
        return [Lookup(a.columns[:2], a.table_column, a.frequencies_column, a.filter_columns[:2]), b]


NL_F, NL_T, NL_TN, NL_M, NL_MN, NL_FA, NL_FB = range(7)


class NextRowLookupStark(S.Stark):
    """One lookup whose table, frequencies and first filter all have next-row terms: the helper columns read them
    (eval_table), the constraints read the table and frequencies on the local row only (Column::eval) and the filters
    on both rows (eval_with_next), as the reference does (lookup.rs:292-335,851-856). The looking columns are F and F on
    the next row. No constraints of its own; degree 3, so one chunk of two looking columns."""
    COLUMNS, PUBLIC_INPUTS = 7, 0

    def eval(self, v, y):
        pass

    def constraint_degree(self):
        return 3

    def lookups(self):
        table = Column.linear_combination_and_next_row_with_constant([(NL_T, 1)], [(NL_TN, 1)], 5)
        freq = Column.linear_combination_and_next_row_with_constant([(NL_M, 1)], [(NL_MN, 2)], 0)
        filt = Filter.new([(Column.single(NL_FA), Column.single_next_row(NL_FA))], [Column.single_next_row(NL_FB)])
        return [Lookup([Column.single(NL_F), Column.single_next_row(NL_F)], table, freq, [filt, Filter.default()])]


def _range_case(log_n):
    return RangeCheckStark(), S.StarkConfig.standard_fast_config(), RangeCheckStark.generate_trace(log_n), [0]


def _perm_case(log_n=5):
    stark = PermutationStark(1 << log_n)
    return stark, S.StarkConfig.standard_fast_config(), stark.generate_trace(0), [0]


# ----------------------------------------------------------------------------------------------------------- CPU
def test_eval_vanishing_poly_with_lookups_matches_hand_written_formulas():
    log_n, n = 6, 64
    stark = RangeCheckStark()
    g = E.primitive_root_of_unity(log_n)
    last = E.inverse(g)
    x = tuple(int(v) for v in synth(0x8A0, (2,)))
    loc = [tuple(int(w) for w in synth(0x8A1 + k, (2,))) for k in range(10)]
    nxt = [tuple(int(w) for w in synth(0x8B1 + k, (2,))) for k in range(10)]
    na = stark.num_lookup_helper_columns(S.StarkConfig.standard_fast_config())
    assert na == (3 + 2) * 2
    aux = [tuple(int(w) for w in synth(0x8C1 + k, (2,))) for k in range(na)]
    aux_n = [tuple(int(w) for w in synth(0x8D1 + k, (2,))) for k in range(na)]
    alphas = [int(a) for a in synth(0x8E0, (2,))]
    betas = [int(a) for a in synth(0x8E1, (2,))]
    pi = [11]
    l_0, l_last = S.eval_l_0_and_l_last(log_n, x)
    add, sub, mul = E.ext_add, E.ext_sub, E.ext_mul

    def c(v):
        return (v % P, 0)

    cons = [sub(mul(loc[SEL], loc[SEL]), loc[SEL]), sub(mul(loc[SEL2], loc[SEL2]), loc[SEL2]),
            mul(sub(loc[TABLE], c(pi[0])), l_0)]
    start = 0
    for lookup_idx in range(2):
        for beta in betas:
            gam = c(beta)
            t = add(loc[TABLE], gam)
            if lookup_idx == 0:
                f0, f1 = add(loc[A0], gam), add(loc[A1], gam)
                f2 = add(add(add(loc[E_], nxt[G]), c(3)), gam)
                h0, h1, z, zn = aux[start], aux[start + 1], aux[start + 2], aux_n[start + 2]
                cons.append(sub(sub(mul(mul(f1, f0), h0), mul(loc[SEL], f1)), mul(c(1), f0)))   # chunk of 2
                cons.append(sub(mul(f2, h1), mul(loc[SEL], loc[SEL2])))                         # chunk of 1
                hs, m, nh = add(h0, h1), loc[MA], 3
            else:
                f0 = add(loc[B], gam)
                h0, z, zn = aux[start], aux[start + 1], aux_n[start + 1]
                cons.append(sub(mul(f0, h0), loc[SEL2]))
                hs, m, nh = h0, loc[MB], 2
            cons.append(mul(z, l_0))
            cons.append(sub(mul(sub(zn, z), t), sub(mul(hs, t), m)))
            start += nh

    def fold(cs):
        out = []
        for al in alphas:
            acc = (0, 0)
            for v in cs:
                acc = add(mul(acc, (al, 0)), v)
            out.append(acc)
        return out

    got = S.eval_vanishing_poly(stark, loc, nxt, pi, alphas, x, log_n, aux, aux_n, betas)
    assert got == fold(cons)
    assert last == E.inverse(g)
    with pytest.raises(N.ShapeError):
        S.eval_vanishing_poly(stark, loc, nxt, pi, alphas, x, log_n)
    with pytest.raises(N.ShapeError):
        S.eval_vanishing_poly(stark, loc, nxt, pi, alphas, x, log_n, aux[:-1], aux_n[:-1], betas)
    # PermutationStark: no constraints of its own; chunk of 1 (degree 0), Z
    perm = PermutationStark(n)
    a4 = [tuple(int(w) for w in synth(0x8F1 + k, (2,))) for k in range(4)]
    a4n = [tuple(int(w) for w in synth(0x8F5 + k, (2,))) for k in range(4)]
    cons = []
    for k, beta in enumerate(betas):
        h, z, zn = a4[2 * k], a4[2 * k + 1], a4n[2 * k + 1]
        t = add(loc[1], c(beta))
        cons += [sub(mul(add(loc[0], c(beta)), h), c(1)), mul(z, l_0), sub(mul(sub(zn, z), t), sub(mul(h, t), loc[2]))]
    assert S.eval_vanishing_poly(perm, loc[:3], nxt[:3], [0], alphas, x, log_n, a4, a4n, betas) == fold(cons)
    # next-row terms: ignored in the table and frequencies (Column::eval), read in the filter (eval_with_next)
    nl = NextRowLookupStark()

    def next_row_cons(with_next_table):
        out = []
        for k, beta in enumerate(betas):
            gam = c(beta)
            h, z, zn = a4[2 * k], a4[2 * k + 1], a4n[2 * k + 1]
            c0, c1 = add(loc[NL_F], gam), add(nxt[NL_F], gam)
            f0 = add(mul(loc[NL_FA], nxt[NL_FA]), nxt[NL_FB])
            t = add(add(loc[NL_T], c(5)), gam)
            m = loc[NL_M]
            if with_next_table:
                t, m = add(t, nxt[NL_TN]), add(m, mul(c(2), nxt[NL_MN]))
            out += [sub(sub(mul(mul(c1, c0), h), mul(f0, c1)), mul(c(1), c0)), mul(z, l_0),
                    sub(mul(sub(zn, z), t), sub(mul(h, t), m))]
        return out

    got = S.eval_vanishing_poly(nl, loc[:7], nxt[:7], [], alphas, x, log_n, a4, a4n, betas)
    assert got == fold(next_row_cons(False)) and got != fold(next_row_cons(True))


@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("logup_emu") / "liblogup_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DGL_FORCE_32BIT_PATH", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "emu", "logup_emu.cpp")])
    L = C.CDLL(out)
    L.emu_stark_lookup_helpers.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                           C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    return L


def _emu_helpers(L, stark, trace, challenges):
    trace = np.ascontiguousarray(trace, dtype=np.uint64)
    n = trace.shape[1]
    prog, offsets, consts = row_programs(stark.lookups(), stark.COLUMNS)
    ch = np.array(challenges, dtype=np.uint64)
    out = np.zeros((stark._helper_columns_per_challenge() * len(ch), n), dtype=np.uint64)
    consts = consts if len(consts) else np.zeros(1, dtype=np.uint64)
    rc = L.emu_stark_lookup_helpers(trace.ctypes.data, n, n.bit_length() - 1, C.addressof(prog), offsets.ctypes.data,
                                    len(offsets) - 1, consts.ctypes.data, ch.ctypes.data, len(ch),
                                    stark.constraint_degree(), out.ctypes.data)
    return rc, out


@pytest.mark.parametrize("case", ["permutation_5", "range_3", "range_8"])
def test_helper_rows_on_host_match_restatement(emu_lib, case):
    """The kernel's row source on the host equals the restatement bit for bit; the range-check STARK's third looking
    column reads row 0 from the last row (the wrap of Column::eval_table), where its filter is on."""
    if case.startswith("permutation"):
        stark, _, trace, _ = _perm_case(5)
    else:
        stark, _, trace, _ = _range_case(int(case.split("_")[1]))
        assert trace[SEL, -1] == 1 and trace[SEL2, -1] == 1
    challenges = [int(v) for v in synth(0x900, (2,))]
    rc, got = _emu_helpers(emu_lib, stark, trace, challenges)
    want, wraps = T.aux_columns(stark, trace, challenges)
    assert rc == 0 and np.array_equal(got, want)
    assert wraps == [0] * len(wraps)
    if not case.startswith("permutation"):
        # row 0 of G feeds the last row's h of the chunk holding the combination, for every challenge
        moved = trace.copy()
        moved[G, 0] += np.uint64(1)
        rc, got_moved = _emu_helpers(emu_lib, stark, moved, challenges)
        n = trace.shape[1]
        for k in range(len(challenges)):
            col = 3 * k + 1
            assert got_moved[col, n - 1] != got[col, n - 1]
            assert np.array_equal(got_moved[col, :n - 1], got[col, :n - 1])
    # one challenge equal to minus a looked value: the row's batch inversion meets zero
    rc, _ = _emu_helpers(emu_lib, stark, trace, [(P - int(trace[0, 3])) % P])
    assert rc == 1


def test_next_row_terms_on_host_match_restatement(emu_lib):
    """Table, frequencies and filter with next-row terms: the row source reads them all (eval_table, wrapping to row 0
    on the last row), like the restatement; changing any next-row column changes the helper columns."""
    stark = NextRowLookupStark()
    trace = synth(0x940, (7, 64))
    challenges = [int(v) for v in synth(0x941, (2,))]
    rc, got = _emu_helpers(emu_lib, stark, trace, challenges)
    want, _ = T.aux_columns(stark, trace, challenges)
    assert rc == 0 and np.array_equal(got, want)
    # a next-row term read at row r belongs to row r - 1: the table and frequencies enter Z's step from row r - 1 to
    # r, so Z first differs at row r; the filter enters h at row r - 1 (row 0: at the last row, the wrap)
    for col, row, aux_cols, first in [(NL_TN, 5, [1, 3], 5), (NL_MN, 9, [1, 3], 9), (NL_FB, 0, [0, 2], 63)]:
        moved = trace.copy()
        moved[col, row] = (moved[col, row] + np.uint64(1)) % np.uint64(P)
        rc, got_moved = _emu_helpers(emu_lib, stark, moved, challenges)
        assert rc == 0 and np.array_equal(got_moved, T.aux_columns(stark, moved, challenges)[0])
        for a in aux_cols:
            assert np.array_equal(got_moved[a, :first], got[a, :first]), col
            assert got_moved[a, first] != got[a, first], col


def test_logup_invariant_pins_the_restatement():
    """Z closes to 0 at the wrap exactly when the frequencies match the filtered looked multiset."""
    challenges = [int(v) for v in synth(0x910, (2,))]
    for stark, trace in [(_perm_case(5)[0], _perm_case(5)[2]), (RangeCheckStark(), RangeCheckStark.generate_trace(6))]:
        _, wraps = T.aux_columns(stark, trace, challenges)
        assert wraps == [0] * len(wraps)
        bad = trace.copy()
        fcol = 2 if isinstance(stark, PermutationStark) else MB
        bad[fcol, 1] += np.uint64(1)
        _, wraps = T.aux_columns(stark, bad, challenges)
        assert all(w != 0 for w in wraps[-len(challenges):])
    # a looked value moved where its filter is off does not matter; where it is on, it does
    trace = RangeCheckStark.generate_trace(6)
    off = int(np.nonzero(trace[SEL] == 0)[0][0])
    on = int(np.nonzero(trace[SEL] == 1)[0][0])
    moved = trace.copy()
    moved[A0, off] = np.uint64(12345678901)
    assert T.aux_columns(RangeCheckStark(), moved, challenges)[1] == [0] * 4
    moved[A0, on] = np.uint64(12345678901)
    assert T.aux_columns(RangeCheckStark(), moved, challenges)[1][:2] != [0, 0]


def _cpu_lookup_backends(monkeypatch, oracle, stark, calls):
    from test_stark_prove import _cpu_backends

    logs, ctx = _cpu_backends(monkeypatch, oracle, stark, calls)

    def helpers(stark_, trace, challenges, ctx_):
        calls.append(("helpers", [int(c) for c in challenges]))
        return T.aux_columns(stark_, np.asarray(trace), challenges)[0]

    def quotient(stark_, tc, pis, alphas, auxiliary_polys_commitment=None, lookup_challenges=None):
        return T.host_quotient(oracle, stark_, tc.o.coeffs, pis, alphas, auxiliary_polys_commitment.o.coeffs,
                               lookup_challenges)

    monkeypatch.setattr(S, "_device_trace", lambda trace, ctx_: np.asarray(trace))
    monkeypatch.setattr(S, "compute_lookup_helper_columns", helpers)
    monkeypatch.setattr(S, "commit_auxiliary_polys",
                        lambda cols, rate_bits, cap_height, ctx_: S.PolynomialBatch.from_values(cols, rate_bits, False,
                                                                                                cap_height))
    monkeypatch.setattr(S, "compute_quotient_polys", quotient)
    return logs, ctx


def _tampered(proof, what):
    bad = copy.deepcopy(proof)
    if what == "aux_opening":
        bad.proof.openings.auxiliary_polys[0, 1] ^= np.uint64(1)
    elif what == "aux_next_opening":
        bad.proof.openings.auxiliary_polys_next[-1, 0] ^= np.uint64(1)
    elif what == "aux_cap":
        bad.proof.auxiliary_polys_cap.hashes[0, 0] ^= np.uint64(1)
    else:   # the auxiliary cap dropped
        bad.proof.auxiliary_polys_cap = None
    return bad


@pytest.mark.parametrize("case", ["permutation", "range_check"])
def test_prove_host_logic_with_cpu_backends(oracle, monkeypatch, case):
    stark, config, trace, pi = _perm_case(5) if case == "permutation" else _range_case(5)
    twin = T.twin_prove(oracle, stark, config, trace, pi)
    calls = []
    logs, ctx = _cpu_lookup_backends(monkeypatch, oracle, stark, calls)
    proof = S.prove(stark, config, trace, pi, ctx=ctx)
    assert calls.count("close") == (2 if case == "permutation" else 3)
    T.assert_matches_twin(proof, twin)
    assert T.verify(oracle, stark, config, proof) is None
    nq = stark.num_quotient_polys(config)
    assert len(proof.proof.opening_proof.query_round_proofs[0].initial_trees_proof.evals_proofs) == (3 if nq else 2)
    helpers = [c for c in calls if isinstance(c, tuple) and c[0] == "helpers"]
    assert helpers == [("helpers", [b for b, _ in twin["lookup_challenge_set"]])]
    ch = proof.get_challenges(stark, config)
    prover_draws = [v for kind, v in logs[0] if kind == "challenge"]
    replay_draws = [v for kind, v in logs[1] if kind == "challenge"]
    assert replay_draws[:len(prover_draws)] == prover_draws
    assert [(c.beta, c.gamma) for c in ch["lookup_challenge_set"]] == twin["lookup_challenge_set"]
    assert ch["stark_alphas"] == twin["alphas"] and ch["stark_zeta"] == twin["zeta"]
    for what in ["aux_opening", "aux_next_opening", "aux_cap", "dropped_aux_cap"]:
        assert T.verify(oracle, stark, config, _tampered(proof, what)) is not None, what
    assert T.verify(oracle, stark, config, _tampered(proof, "dropped")) == "Missing auxiliary_polys_cap"
    with pytest.raises(N.ShapeError, match="Missing auxiliary_polys_cap"):
        _tampered(proof, "dropped").get_challenges(stark, config)


def test_shape_errors(oracle, monkeypatch):
    """The reference's panics: constraint degree 1 divides by zero in num_helper_columns; a chunk of three looking
    columns is its todo!; one filter per looking column; duplicate columns. All raised before any commitment."""
    with pytest.raises(N.ShapeError, match="divide by zero"):
        Lookup([Column.single(0)], Column.single(1), Column.single(2), [Filter.default()]).num_helper_columns(1)
    with pytest.raises(N.ShapeError, match="one filter per looking column"):
        Lookup([Column.single(0)], Column.single(1), Column.single(2), [])
    with pytest.raises(N.ShapeError, match="Duplicate columns"):
        Column.linear_combination([(0, 1), (0, 2)])
    with pytest.raises(N.ShapeError):
        Column.linear_combination_and_next_row_with_constant([], [], 1)
    assert Lookup([Column.single(0)] * 3, Column.single(1), Column.single(2),
                  [Filter.default()] * 3).num_helper_columns(0) == 4
    calls = []
    _, _, trace, pi = _range_case(5)
    _, ctx = _cpu_lookup_backends(monkeypatch, oracle, RangeCheckStark(), calls)
    with pytest.raises(N.ShapeError, match="divide by zero"):
        S.prove(RangeCheckStark(degree=1), S.StarkConfig.standard_fast_config(), trace, pi, ctx=ctx)
    with pytest.raises(N.ShapeError, match="Allow other constraint degrees"):
        S.prove(RangeCheckStark(degree=4), T_config_rate2(), trace, pi, ctx=ctx)
    with pytest.raises(N.ShapeError, match="Allow other constraint degrees"):
        RangeCheckStark(degree=4).constraint_program(2)
    assert not [c for c in calls if c == "close" or (isinstance(c, tuple) and c[0] == "helpers")]
    # Column / Filter algebra on the host row program
    assert Column.le_bits([3, 4]).linear_combination == [(3, 1), (4, 2)]
    assert Column.le_bytes([3, 4]).linear_combination == [(3, 1), (4, 256)]
    assert Column.sum([1, 2]).linear_combination == [(1, 1), (2, 1)]
    assert Column.le_bits_with_constant([5], 9).constant == 9
    assert [c.next_row_linear_combination for c in Column.singles_next_row([1, 2])] == [[(1, 1)], [(2, 1)]]
    assert Column.zero().constant == 0 and Column.one().constant == 1


def T_config_rate2():
    from plonky2_b200.fri import FriConfig

    return S.StarkConfig(100, 2, FriConfig(rate_bits=2, cap_height=2, proof_of_work_bits=8,
                                           reduction_strategy=("ConstantArityBits", 2, 3), num_query_rounds=20))


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


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["range_10", "range_20", "next_row_10"])
def test_device_helper_columns_equal_restatement(pb, case):
    import torch

    log_n = int(case.split("_")[-1])
    if case.startswith("range"):
        stark, trace = RangeCheckStark(), RangeCheckStark.generate_trace(log_n, seed=log_n)
    else:
        stark, trace = NextRowLookupStark(), synth(0x950, (7, 1 << log_n))
    challenges = [int(v) for v in synth(0x920 + log_n, (2,))]
    dev = _to_device(trace)
    torch.cuda.synchronize()
    got = S.compute_lookup_helper_columns(stark, dev, challenges, pb.default_context()).cpu().numpy().view(np.uint64)
    want, wraps = T.aux_columns(stark, trace, challenges)
    assert np.array_equal(got, want)
    if case.startswith("range"):
        assert wraps == [0] * 4


def _gpu_case(name):
    if name.startswith("permutation"):
        return _perm_case(5)
    return _range_case(int(name.split("_")[1]))


@pytest.mark.gpu
@pytest.mark.parametrize("name,source", [("permutation_5", "host"), ("range_5", "host"), ("range_10", "host"),
                                         ("range_10", "device"), ("range_16", "host"), ("range_16", "device")])
def test_prove_on_device_equals_cpu_twin(pb, oracle, name, source):
    import torch

    stark, config, trace, pi = _gpu_case(name)
    arg = trace
    if source == "device":
        arg = _to_device(trace)
        torch.cuda.synchronize()
    proof = S.prove(stark, config, arg, pi)
    twin = T.twin_prove(oracle, stark, config, trace, pi)
    T.assert_matches_twin(proof, twin)
    assert T.verify(oracle, stark, config, proof) is None
    ch = proof.get_challenges(stark, config)
    assert [(c.beta, c.gamma) for c in ch["lookup_challenge_set"]] == twin["lookup_challenge_set"]
    assert ch["stark_alphas"] == twin["alphas"] and ch["stark_zeta"] == twin["zeta"]


@pytest.mark.gpu
def test_prove_on_device_with_a_wrong_frequency(pb, oracle):
    """One wrong frequency: Z no longer closes, so the unfiltered step constraint fails on the last row. At constraint
    degree 3 the quotient has two chunks per challenge and the reference's trim cannot fail: the proof is made and the
    restated verifier rejects it at zeta. At degree 4 (three chunks) prove raises "Quotient has failed"."""
    stark, config, trace, pi = _range_case(10)
    trace[MA, 5] += np.uint64(1)
    assert T.verify(oracle, stark, config, S.prove(stark, config, trace, pi)) == (
        "Mismatch between evaluation and opening of quotient polynomial")
    stark4, config4 = RangeCheckStark4(), T_config_rate2()
    trace = RangeCheckStark.generate_trace(10, count_combination=False)
    assert T.verify(oracle, stark4, config4, S.prove(stark4, config4, trace, pi)) is None
    trace[MA, 5] += np.uint64(1)
    with pytest.raises(pb.NativeError, match="Quotient has failed"):
        S.prove(stark4, config4, trace, pi)


@pytest.mark.gpu
def test_entry_point_errors(pb):
    """gl_stark_lookup_helpers: gamma = p - (a looked value) -> GL_ERR_DIV_ZERO; the limits -> GL_ERR_UNSUPPORTED;
    constraint degree 1 -> GL_ERR_BAD_SHAPE. gl_stark_quotient_aux rejects an auxiliary commitment of another degree or
    rate, a sharded one and an unfinished one, with the message on the calling context even when the auxiliary
    commitment belongs to another context."""
    import torch

    ctx = pb.default_context()
    L = N.lib()
    stark, _, trace, _ = _perm_case(5)
    dev = _to_device(trace)
    out = torch.empty((8, 32), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    prog, offsets, consts = row_programs(stark.lookups(), 3)

    def call(challenges, degree=0, offs=offsets, program=prog, cols=3):
        ch = np.array(challenges, dtype=np.uint64)
        return L.gl_stark_lookup_helpers(ctx.h, N.vp(dev.data_ptr()), 32, cols, 5, program, offs.ctypes.data_as(N.u32p),
                                         len(offs) - 1, N.np_ptr(consts), len(consts), N.np_ptr(ch), len(ch), degree,
                                         N.vp(out.data_ptr()))

    assert call([5, 6]) == N.GL_OK
    assert call([5, (P - int(trace[0, 7])) % P]) == N.GL_ERR_DIV_ZERO
    assert b"Tried to invert zero" in L.gl_last_error(ctx.h)
    assert call([1, 2, 3, 4, 5]) == N.GL_ERR_UNSUPPORTED
    assert call([5], degree=1) == N.GL_ERR_BAD_SHAPE
    wide = Lookup([Column.single(0)] * 17, Column.single(1), Column.single(2), [Filter.default()] * 17)
    wprog, woffs, _ = row_programs([wide], 3)
    assert call([5], offs=woffs, program=wprog) == N.GL_ERR_UNSUPPORTED
    assert call([5], cols=2) == N.GL_ERR_BAD_ARG                      # the program reads column 2 of a 2-column trace

    def long_lookup(n_instr):                                         # LOCAL 0 ..., then one emit of each role
        p = np.zeros((n_instr, 4), dtype=np.uint16)
        p[-4:, 0], p[-4:, 2] = S.OP_EMIT, [0, 1, 2, 3]
        return p

    lp = long_lookup(256)
    assert call([5], offs=np.array([0, 256], dtype=np.uint32), program=lp.ctypes.data) == N.GL_OK
    lp = long_lookup(257)
    before = ctx.launch_count
    assert call([5], offs=np.array([0, 257], dtype=np.uint32), program=lp.ctypes.data) == N.GL_ERR_UNSUPPORTED
    assert b"lookup 0: row program of 1..256 instructions" in L.gl_last_error(ctx.h) and ctx.launch_count == before
    cfg = S.StarkConfig.standard_fast_config().fri_config
    rs, rtrace, _ = RangeCheckStark(), RangeCheckStark.generate_trace(5), None
    tc = pb.PolynomialBatch.from_values(rtrace, cfg.rate_bits, False, cfg.cap_height)
    other = pb.PolynomialBatch.from_values(synth(0x930, (2, 64)), cfg.rate_bits, False, cfg.cap_height)
    b = rs.constraint_program(2)
    cs = np.array([0, 1, 2] + b.consts[b.num_bound:], dtype=np.uint64)
    al = np.array([3, 4], dtype=np.uint64)
    q = torch.empty((2, 64), dtype=torch.int64, device="cuda")
    rc = L.gl_stark_quotient_aux(ctx.h, tc.h, other.h, b.program(), len(b.instrs), N.np_ptr(cs), len(cs), N.np_ptr(al),
                                 2, 2, N.vp(q.data_ptr()))
    assert rc == N.GL_ERR_BAD_SHAPE and b"degree or rate" in L.gl_last_error(ctx.h)

    def quotient_aux(aux_h):
        return L.gl_stark_quotient_aux(ctx.h, tc.h, aux_h, b.program(), len(b.instrs), N.np_ptr(cs), len(cs),
                                       N.np_ptr(al), 2, 2, N.vp(q.data_ptr()))

    aux_cols = synth(0x931, (10, 32))
    other_rate = pb.PolynomialBatch.from_values(aux_cols, cfg.rate_bits + 1, False, cfg.cap_height)
    assert quotient_aux(other_rate.h) == N.GL_ERR_BAD_SHAPE
    sharded = pb.PolynomialBatch.from_values(aux_cols, cfg.rate_bits, False, cfg.cap_height, shard=(0, 2))
    assert quotient_aux(sharded.h) == N.GL_ERR_UNSUPPORTED
    assert b"whole auxiliary LDE" in L.gl_last_error(ctx.h)
    ctx2 = N.Context(0)
    h = N.vp()
    N.check(L.gl_commit_begin(ctx2.h, 10, 5, cfg.rate_bits, cfg.cap_height, 0, 0, 1, None, C.byref(h)), ctx2.h)
    assert quotient_aux(h) == N.GL_ERR_BAD_ARG
    assert b"not been called on the auxiliary commitment" in L.gl_last_error(ctx.h)
    L.gl_commit_destroy(h)
    other_rate.close()
    sharded.close()
    ctx2.close()
    rc = L.gl_stark_quotient(ctx.h, tc.h, b.program(), len(b.instrs), N.np_ptr(cs), len(cs), N.np_ptr(al), 2, 2,
                             N.vp(q.data_ptr()))
    assert rc == N.GL_ERR_BAD_ARG                                      # auxiliary reads without an auxiliary commitment
    # 513 instructions; a quotient degree factor of 9 at rate_bits 4 (2^4 points per row, more than 8): refused before
    # any launch
    long = np.zeros((513, 4), dtype=np.uint16)
    long[-1, 0] = S.OP_EMIT
    before = ctx.launch_count
    rc = L.gl_stark_quotient(ctx.h, tc.h, long.ctypes.data, 513, N.np_ptr(cs), len(cs), N.np_ptr(al), 2, 2,
                             N.vp(q.data_ptr()))
    assert rc == N.GL_ERR_UNSUPPORTED and ctx.launch_count == before
    assert b"program of 513 instructions (max 512)" in L.gl_last_error(ctx.h)
    tc4 = pb.PolynomialBatch.from_values(rtrace, 4, False, cfg.cap_height)
    before = ctx.launch_count
    rc = L.gl_stark_quotient(ctx.h, tc4.h, b.program(), len(b.instrs), N.np_ptr(cs), len(cs), N.np_ptr(al), 2, 9,
                             N.vp(q.data_ptr()))
    assert rc == N.GL_ERR_UNSUPPORTED and ctx.launch_count == before
    assert b"quotient degree factor too large" in L.gl_last_error(ctx.h)
    tc4.close()
    tc.close()
    other.close()


@pytest.mark.gpu
def test_lookup_free_proof_through_the_same_prove(pb, oracle):
    """FibonacciStark through the prove that now also handles lookups: the proof test_stark_prove.py checks, no
    auxiliary cap or openings."""
    from test_stark_prove import _fib_case

    stark, config, trace, pi = _fib_case(10)
    proof = S.prove(stark, config, trace, pi)
    T.assert_matches_twin(proof, T.twin_prove(oracle, stark, config, trace, pi))
    assert proof.proof.auxiliary_polys_cap is None
    assert proof.proof.openings.auxiliary_polys is None and proof.proof.openings.auxiliary_polys_next is None
    assert T.verify(oracle, stark, config, proof) is None
    assert proof.get_challenges(stark, config)["lookup_challenge_set"] is None
