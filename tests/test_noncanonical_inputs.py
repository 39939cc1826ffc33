"""Inputs may be non-canonical; outputs are canonical (the Conventions of include/plonky2_b200.h). The reference's
GoldilocksField does not reduce its results (an add can return a word in [p, 2^64)), so witness values, trace cells,
challenges and opened values reach the library in that form, and a proof must not depend on how its inputs are
represented.

A word x < 2^32 - 1 has exactly one other representation, its twin x + p; larger words have none. Every case here calls
an entry point once with canonical inputs and once with every eligible word replaced by its twin (0 -> p, 1 -> p + 1,
2^32 - 2 -> 2^64 - 1 among them), and checks that
  1. the outputs are bit-identical (an error case: the same status and message),
  2. every output word is below p,
  3. the canonical call matches the oracle or the exact restatement (where another file's test already checks that call
     at the same shape, that test is named instead).
Inputs are built with many small words so that most of them have a twin.

CPU: a static map over include/plonky2_b200.h: every gl_ entry point with a uint64_t input argument is in COVERED (the
test here that runs it with twins) or in NOT_NEEDED (why none is needed). The host layer (Challenger, eval_vanishing_poly,
Column / Filter, check_ctls, ProofWithPublicInputs) with twin values against the canonical ones.

GPU (-m gpu): the entry-point sweep, and whole proofs (starky with and without lookups, host columns and torch tensors,
a non-resident LDE, cross-table lookups; plonky2 with and without lookups, and with zero knowledge) from twin traces,
witnesses and public inputs: field for field the canonical input's proof, accepted by the restated verifier."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import P, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "plonky2_b200.h")
TWIN_BELOW = 2**32 - 1   # words below this have a twin x + p

# entry points with a uint64_t field input and the test here that gives them twins
COVERED = {
    "gl_partial_products_and_zs": "test_partial_products_and_zs",
    "gl_lookup_polys": "test_lookup_polys",
    "gl_stark_lookup_helpers": "test_stark_lookup_helpers",
    "gl_stark_ctl_helpers": "test_stark_ctl_helpers",
    "gl_stark_quotient": "test_stark_quotients",
    "gl_stark_quotient_aux": "test_stark_quotients",
    "gl_stark_quotient_shard": "test_stark_quotients",
    "gl_stark_quotient_from_shards": "test_stark_quotients",
    "gl_plonk_quotient": "test_plonk_quotients",
    "gl_plonk_quotient_shard": "test_plonk_quotients",
    "gl_sigma_polys": "test_sigma_polys",
    "gl_openings": "test_openings",
    "gl_openings_shard": "test_openings",
    "gl_commit_eval_ext": "test_openings",
    "gl_fri_begin": "test_fri_begin",
    "gl_fri_begin_values": "test_fri_begin_values",
    "gl_fri_fold": "test_fri_fold_and_mix",
    "gl_fri_mix": "test_fri_fold_and_mix",
    "gl_fri_pow": "test_fri_pow",
    "gl_commit_finish": "test_commit_salt",
    "gl_commit_create": "test_commit_salt",
    "gl_commit_finish_prefixed": "test_commit_finish_prefixed",
    "gl_merkle_build": "test_narrow_leaves",
    "gl_commit_add_columns": "test_narrow_leaves",
}
# entry points with a uint64_t input that need no case here, and why
NOT_NEEDED = {
    "gl_ctx_device_bytes": "its uint64_t pointers are outputs",
    "gl_ctx_phase_ms": "its uint64_t pointer is an output",
    "gl_ntt": "covered by synth(..., canonical=False) in test_gpu_parity.py and test_gpu_ntt_plans.py",
    "gl_ntt_bcast": "the NTT passes of gl_ntt, covered by test_gpu_ntt_plans.py's non-canonical inputs",
    "gl_bcast": "copies words; no field arithmetic",
    "gl_commit_create_sharded": "gl_commit_create's begin / add_columns / finish, which test_commit_salt covers",
    "gl_commit_begin": "coeff_storage is an output buffer; no field input",
    "gl_commit_begin_blocked": "coeff_storage is an output buffer; no field input",
    "gl_commit_cap": "an output buffer",
    "gl_commit_coeffs": "an output buffer",
    "gl_commit_leaves": "an output buffer; the leaves it reads are checked by test_commit_salt",
    "gl_commit_digests": "an output buffer",
    "gl_commit_get_lde_values": "an output buffer",
    "gl_commit_open": "leaf indices, not field elements; its leaves are checked by test_commit_salt",
    "gl_random_field_elements": "no field input (a key, a column and positions)",
    "gl_poseidon_permute_host": "covered by test_gpu_poseidon.py's non-canonical states",
    "gl_poseidon_permute_many": "covered by test_gpu_poseidon.py's non-canonical states",
    "gl_poseidon_hash_many": "covered by test_gpu_poseidon.py's non-canonical inputs (W <= 4 by test_narrow_leaves)",
    "gl_poseidon_hash_no_pad_many": "covered by test_gpu_poseidon.py's non-canonical inputs",
    "gl_poseidon_two_to_one_many": "covered by test_gpu_poseidon.py's non-canonical inputs",
    "gl_merkle_cap": "an output buffer",
    "gl_merkle_digests": "an output buffer",
    "gl_merkle_open": "leaf indices, not field elements; its leaves are checked by test_narrow_leaves",
    "gl_fri_values_local": "an output buffer",
    "gl_fri_begin_from_coeffs": "covered by test_gpu_host_buffers.py's non-canonical coefficients",
    "gl_fri_coeffs": "an output buffer",
    "gl_fri_commit_round": "an output buffer",
    "gl_fri_commit_round_sharded": "an output buffer",
    "gl_fri_final_poly": "an output buffer",
    "gl_fri_open": "leaf indices, not field elements",
}


# ----------------------------------------------------------------------------------------------------------- helpers
def twin(a):
    """Every word below 2^32 - 1 replaced by its twin x + p; other words as they are. Arrays (uint64) or ints."""
    if isinstance(a, (int, np.integer)):
        return int(a) + P if int(a) < TWIN_BELOW else int(a)
    a = np.asarray(a, dtype=np.uint64)
    return np.where(a < np.uint64(TWIN_BELOW), a + np.uint64(P), a)


def small_words(seed, shape):
    """Canonical words, about half of them below 2^32 - 1 (with twins), and 0, 1 and 2^32 - 2 always among them."""
    rng = np.random.default_rng(seed)
    v = synth(seed, shape).reshape(-1).copy()
    small = rng.random(v.size) < 0.5
    v[small] = rng.integers(0, TWIN_BELOW, int(small.sum()), dtype=np.uint64)
    v[:3] = [0, 1, 2**32 - 2][:v.size]
    return v.reshape(shape)


def _example(canon, lifted):
    """(canonical word, its twin) for the first lifted word of an input, for the failure messages."""
    c, t = np.asarray(canon, dtype=np.uint64).reshape(-1), np.asarray(lifted, dtype=np.uint64).reshape(-1)
    k = np.flatnonzero(c != t)
    return (int(c[k[0]]), int(t[k[0]])) if len(k) else None


def _outcome(run):
    from plonky2_b200 import _native as N

    try:
        return "ok", run()
    except (ZeroDivisionError, MemoryError, N.ShapeError, N.NativeError) as e:
        return type(e).__name__, str(e)


def _arrays(out):
    if isinstance(out, (list, tuple)):
        return [np.asarray(o, dtype=np.uint64) for o in out]
    return [np.asarray(out, dtype=np.uint64)]


def invariant(entry, what, run, canon_args, twin_args):
    """run(*canon_args) and run(*twin_args) must give the same outputs, all canonical, or the same error. Returns the
    canonical call's outcome (("ok", outputs) or (error type, message)). `what` names the twinned inputs; the message
    of a failure gives the entry point, an input word and the first differing output."""
    ex = next((e for e in (_example(c, t) for c, t in zip(canon_args, twin_args)
                           if isinstance(c, (np.ndarray, list, tuple, int))) if e), None)
    where = "%s [%s] with non-canonical words (e.g. input word %s for %s)" % (entry, what, ex[1] if ex else "-",
                                                                               ex[0] if ex else "-")
    a, b = _outcome(lambda: run(*canon_args)), _outcome(lambda: run(*twin_args))
    if a[0] != "ok" or b[0] != "ok":
        assert a[0] == b[0] and (a[0] == "ok" or a[1] == b[1]), "%s: canonical inputs give %s, non-canonical %s" % (
            where, a if a[0] != "ok" else "a result", b if b[0] != "ok" else "a result")
        return a
    for k, (x, y) in enumerate(zip(_arrays(a[1]), _arrays(b[1]))):
        assert x.shape == y.shape, (where, k, x.shape, y.shape)
        bad = np.argwhere(x != y)
        assert len(bad) == 0, "%s: output %d: %d of %d words differ; first at %s: %d, canonical inputs give %d" % (
            where, k, len(bad), x.size, tuple(int(i) for i in bad[0]), y[tuple(bad[0])], x[tuple(bad[0])])
        hi = np.argwhere(x >= np.uint64(P))
        assert len(hi) == 0, "%s: output %d word %s = %d is not canonical" % (
            where, k, tuple(int(i) for i in hi[0]), x[tuple(hi[0])])
    return a


# ----------------------------------------------------------------------------------------------------------- CPU
def field_input_entry_points(header):
    """Every gl_ function declared in the header with a uint64_t argument: an input (const, by value, or read and
    written in place like gl_ntt's data) or an output buffer; NOT_NEEDED says which of them only write."""
    out = set()
    for m in re.finditer(r"^(?:int|void|uint32_t|uint64_t|const\s+\w+\*)\s*(gl_\w+)\s*\(([^)]*)\)\s*;", header, re.M):
        args = [a.strip() for a in m.group(2).split(",")]
        if any(re.match(r"(const\s+)?uint64_t\b", a) for a in args):
            out.add(m.group(1))
    return out


def test_every_field_input_entry_point_is_covered_or_listed():
    with open(HEADER) as f:
        src = f.read()
    found = field_input_entry_points(src)
    assert not set(COVERED) & set(NOT_NEEDED), "an entry point listed twice"
    listed = set(COVERED) | set(NOT_NEEDED)
    assert sorted(found - listed) == [], "entry points with a uint64_t input that no test here covers or classifies"
    assert sorted(listed - found) == [], "listed entry points that the header no longer declares with a uint64_t input"
    assert all(name in globals() for name in COVERED.values())
    assert all(reason.strip() for reason in NOT_NEEDED.values())


def test_the_static_map_reads_multi_line_declarations():
    src = """
int gl_a(gl_ctx* ctx, const uint64_t* in,
         size_t n);
void gl_b(gl_ctx* ctx);
uint32_t gl_c(const gl_commit* c);
int gl_d(gl_ctx* ctx, uint64_t beta, uint32_t k);
int gl_e(gl_ctx* ctx, const uint64_t point[2], uint64_t* out);
"""
    assert field_input_entry_points(src) == {"gl_a", "gl_d", "gl_e"}


def test_twins():
    a = np.array([0, 1, 2**32 - 2, 2**32 - 1, P - 1, 5], dtype=np.uint64)
    assert twin(a).tolist() == [P, P + 1, 2**64 - 1, 2**32 - 1, P - 1, P + 5]
    assert twin(7) == P + 7 and twin(2**40) == 2**40
    w = small_words(3, (100,))
    assert w[:3].tolist() == [0, 1, 2**32 - 2] and (w < P).all() and (w < TWIN_BELOW).sum() > 30


def test_challenger_observes_residues():
    """Challenger.observe_element / _elements / _extension_element(s) / _hash: the same challenges from twins."""
    from plonky2_b200.challenger import Challenger

    words = [int(x) for x in small_words(0x6100, (21,))]
    out = []
    for vals in (words, [twin(x) for x in words]):
        ch = Challenger()
        ch.observe_element(vals[0])
        ch.observe_elements(vals[1:5])
        ch.observe_extension_element((vals[5], vals[6]))
        ch.observe_extension_elements([(vals[7], vals[8]), (vals[9], vals[10])])
        ch.observe_hash(vals[11:15])
        a = ch.get_n_challenges(3)
        ch.observe_elements(vals[15:])
        out.append(a + ch.get_n_challenges(5))
    assert out[0] == out[1] and all(v < P for v in out[0])


def test_eval_vanishing_poly_of_twins():
    """stark.eval_vanishing_poly with twin row values, public inputs, alphas and point; with lookups also the auxiliary
    values and lookup challenges: the same F_{p^2} values, canonical."""
    from plonky2_b200 import stark as S
    from test_stark_lookups import RangeCheckStark

    log_n = 6

    def ext_twin(v):
        return [(twin(a), twin(b)) for a, b in v]

    w = [int(x) for x in small_words(0x6200, (40,))]
    vals = [(w[2 * k], w[2 * k + 1]) for k in range(20)]
    x, alphas = vals[0], [w[3], w[4]]
    fib = S.FibonacciStark(1 << log_n)
    pi = [w[5], w[6], w[7]]
    want = S.eval_vanishing_poly(fib, vals[1:3], vals[3:5], pi, alphas, x, log_n)
    got = S.eval_vanishing_poly(fib, ext_twin(vals[1:3]), ext_twin(vals[3:5]), [twin(v) for v in pi],
                                [twin(a) for a in alphas], (twin(x[0]), twin(x[1])), log_n)
    assert got == want and all(0 <= c < P for v in want for c in v)
    rc = RangeCheckStark()
    nc, naux = rc.COLUMNS, rc._helper_columns_per_challenge() * 2
    loc, nxt = vals[:nc], vals[1:nc + 1]
    aux, auxn = vals[2:2 + naux], vals[3:3 + naux]
    lc = [w[8], w[9]]
    want = S.eval_vanishing_poly(rc, loc, nxt, [0] * rc.PUBLIC_INPUTS, alphas, x, log_n, aux, auxn, lc)
    got = S.eval_vanishing_poly(rc, ext_twin(loc), ext_twin(nxt), [P] * rc.PUBLIC_INPUTS, [twin(a) for a in alphas],
                                (twin(x[0]), twin(x[1])), log_n, ext_twin(aux), ext_twin(auxn), [twin(c) for c in lc])
    assert got == want


def test_columns_filters_and_check_ctls_of_twins():
    """lookup.Column coefficients and constants, and cross_table_lookup.check_ctls (Column::eval_table,
    Filter::eval_table) on twin traces: the same residues; a filter given as p + 1 is the binary 1, and one that is
    2 in any representation is refused."""
    from plonky2_b200 import cross_table_lookup as X
    from plonky2_b200.lookup import Column
    from test_stark_ctl import system_ctls, system_traces

    a = Column([(0, 3), (2, P + 5)], [(1, 2**64 - 1)], P + 1)
    b = Column([(0, 3), (2, 5)], [(1, 2**32 - 2)], 1)
    assert (a.linear_combination, a.next_row_linear_combination, a.constant) == (
        b.linear_combination, b.next_row_linear_combination, b.constant)
    traces, _ = system_traces()
    ctls = system_ctls()
    X.check_ctls(traces, ctls)
    X.check_ctls([twin(t) for t in traces], ctls)
    rows = [X._column_rows(c, t) for t in traces for c in (b, Column.single(0))]
    rows_t = [X._column_rows(c, twin(t)) for t in traces for c in (a, Column.single(0))]
    assert all(list(r) == list(s) for r, s in zip(rows, rows_t))
    bad = [t.copy() for t in traces]
    from test_stark_ctl import S0
    bad[0][S0, 0] = 2
    with pytest.raises(ValueError, match="Non-binary filter"):
        X.check_ctls([twin(t) for t in bad], ctls)


def test_proof_with_public_inputs_writes_canonical_words():
    """ProofWithPublicInputs (plonky2) and StarkProofWithPublicInputs keep twin public inputs as their residues, and
    to_bytes writes canonical words."""
    from plonky2_b200 import plonk
    from plonky2_b200 import stark as S

    pis = [0, 1, 2**32 - 2, 7, P - 1]

    class _Empty:
        def to_bytes(self):
            return b""

    a = plonk.ProofWithPublicInputs(_Empty(), pis)
    b = plonk.ProofWithPublicInputs(_Empty(), [twin(v) for v in pis])
    assert a.to_bytes() == b.to_bytes()
    assert np.frombuffer(b.to_bytes(), dtype="<u8").tolist() == [len(pis)] + pis
    assert S.StarkProofWithPublicInputs(None, [twin(v) for v in pis]).public_inputs == pis


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


def _dev(a):
    import torch

    t = torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64).copy()).cuda()
    torch.cuda.synchronize()
    return t


def _host(t):
    import torch

    torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint64)


def _u64(vals):
    return np.ascontiguousarray(np.array([int(v) for v in vals], dtype=np.uint64))


@pytest.mark.gpu
@pytest.mark.parametrize("mem", ["host", "device"])
def test_partial_products_and_zs(pb, oracle, mem):
    """gl_partial_products_and_zs with twin wires, sigmas, k_is, beta and gamma: host and device memory. A row whose
    denominator w + beta * sigma + gamma is the word p is refused as the word 0 is."""
    import torch

    from plonky2_b200 import _native as N

    R, log_n, deg = 9, 8, 4
    n = 1 << log_n
    w, sg, k = small_words(0x6300, (R, n)), small_words(0x6301, (R, n)), small_words(0x6302, (R,))
    k[0] = 1
    beta, gamma = 0x9E37, 0x79B9
    ctx, L = pb.default_context(), N.lib()
    M = (R + deg - 1) // deg

    def run(w, sg, k, beta, gamma):
        k = np.ascontiguousarray(k, dtype=np.uint64)
        if mem == "host":
            out = np.empty((M, n), dtype=np.uint64)
            N.check(L.gl_partial_products_and_zs(ctx.h, N.np_ptr(np.ascontiguousarray(w)), N.np_ptr(np.ascontiguousarray(sg)),
                                                 N.np_ptr(k), log_n, R, beta, gamma, deg, N.np_ptr(out), N.MEM_HOST), ctx.h)
            return out
        dw, ds = _dev(w), _dev(sg)
        out = torch.empty((M, n), dtype=torch.int64, device="cuda")
        N.check(L.gl_partial_products_and_zs(ctx.h, N.vp(dw.data_ptr()), N.vp(ds.data_ptr()), N.np_ptr(k), log_n, R,
                                             beta, gamma, deg, N.vp(out.data_ptr()), N.MEM_DEVICE), ctx.h)
        return _host(out)

    args = (w, sg, k, beta, gamma)
    targs = (twin(w), twin(sg), twin(k), twin(beta), twin(gamma))
    res = invariant("gl_partial_products_and_zs", "wires, sigmas, k_is, beta, gamma", run, args, targs)
    assert res[0] == "ok" and np.array_equal(res[1], oracle.partial_products_and_zs(w, sg, k, beta, gamma, deg))
    # row 5 of wire 2: w = 0, sigma = 0, gamma = 0 -> the denominator is 0; its twin adds p + p * beta + p
    w0, s0 = w.copy(), sg.copy()
    w0[2, 5], s0[2, 5] = 0, 0
    res = invariant("gl_partial_products_and_zs", "a zero denominator", run, (w0, s0, k, beta, 0),
                    (twin(w0), twin(s0), twin(k), twin(beta), P))
    assert res[0] == "ZeroDivisionError" and "invert zero" in res[1]
    # the denominator is exactly the word p: w = p, beta * sigma = 0 (sigma = 0), gamma = 0
    w1 = w0.copy()
    w1[2, 5] = P
    res = invariant("gl_partial_products_and_zs", "a denominator of exactly the word p", run, (w0, s0, k, beta, 0),
                    (w1, s0, k, beta, 0))
    assert res[0] == "ZeroDivisionError"


@pytest.mark.gpu
def test_lookup_polys(pb, oracle):
    """gl_lookup_polys with twin wires and challenges (A, B, alpha, delta); a looked slot whose denominator
    alpha - (inp + A * out) is zero only in non-canonical form is refused as the canonical zero is."""
    from plonky2_b200 import _native as N

    routed, qdf, log_n, rows = 12, 4, 8, [(10, 40, 60)]
    n = 1 << log_n
    wires = small_words(0x6400, (routed, n))
    deltas = [0x1234567, 0xABCDEF, 0x5555, 0x7777]
    ctx, L = pb.default_context(), N.lib()
    lr = np.array(rows, dtype=np.uint32).reshape(-1)
    need = max(3 * (routed // 3), 2 * (routed // 2))
    nP = -(-(routed // 2) // (qdf - 1))

    def run(wires, deltas):
        out = np.empty((nP + 1, n), dtype=np.uint64)
        d = np.ascontiguousarray(deltas, dtype=np.uint64)
        N.check(L.gl_lookup_polys(ctx.h, N.np_ptr(np.ascontiguousarray(wires[:need])), log_n, routed, qdf, N.np_ptr(d),
                                  lr.ctypes.data_as(N.u32p), 1, N.np_ptr(out), N.MEM_HOST), ctx.h)
        return out

    res = invariant("gl_lookup_polys", "wires, deltas", run, (wires, _u64(deltas)), (twin(wires), twin(_u64(deltas))))
    assert res[0] == "ok" and np.array_equal(res[1], oracle.lookup_polys(wires, routed, qdf, deltas, rows))
    # alpha = inp + A * out at the first looked slot of row 60: inp = out = 0 and alpha = 0, given as p
    w0 = wires.copy()
    w0[0, 60] = w0[1, 60] = 0
    bad = _u64([deltas[0], deltas[1], 0, deltas[3]])
    res = invariant("gl_lookup_polys", "a zero denominator", run, (w0, bad), (twin(w0), twin(bad)))
    assert res[0] == "ZeroDivisionError"


@pytest.mark.gpu
def test_stark_lookup_helpers(pb):
    """gl_stark_lookup_helpers with a twin trace (values, table, frequencies, filters as p / p + 1), twin challenges
    and twin program constants, against the restated helper columns; a zero denominator f + gamma given as p + p."""
    import stark_twin as T
    import torch

    from plonky2_b200 import _native as N
    from plonky2_b200 import field as F
    from plonky2_b200.lookup import row_programs
    from test_stark_lookups import RangeCheckStark

    log_n = 8
    n = 1 << log_n
    stark, trace = RangeCheckStark(), RangeCheckStark.generate_trace(log_n, seed=5)
    assert (trace < TWIN_BELOW).mean() > 0.5
    prog, offsets, consts = row_programs(stark.lookups(), stark.COLUMNS)
    challenges = _u64([0x31415, 0x27182])
    shape = (stark._helper_columns_per_challenge() * 2, n)
    ctx, L = pb.default_context(), N.lib()

    def run(trace, consts, ch):
        dt = _dev(trace)
        out = torch.empty(shape, dtype=torch.int64, device="cuda")
        c = np.ascontiguousarray(consts, dtype=np.uint64)
        N.check(L.gl_stark_lookup_helpers(ctx.h, N.vp(dt.data_ptr()), n, stark.COLUMNS, log_n, prog,
                                          offsets.ctypes.data_as(N.u32p), len(offsets) - 1,
                                          N.np_ptr(c) if len(c) else None, len(c), N.np_ptr(ch), len(ch),
                                          stark.constraint_degree(), N.vp(out.data_ptr())), ctx.h)
        return _host(out)

    res = invariant("gl_stark_lookup_helpers", "trace, constants, challenges", run, (trace, consts, challenges),
                    (twin(trace), twin(consts), twin(challenges)))
    assert res[0] == "ok" and np.array_equal(res[1], T.aux_columns(stark, trace, [int(c) for c in challenges])[0])
    # gamma = -(table value at row 0) makes t + gamma zero; the table value 0 with gamma 0 given as p
    lk = stark.lookups()[0]
    tcol = lk.table_column.linear_combination[0][0]
    t0 = trace.copy()
    t0[tcol, 0] = 0
    zero = _u64([0, challenges[1]])
    res = invariant("gl_stark_lookup_helpers", "a zero denominator", run, (t0, consts, zero),
                    (twin(t0), twin(consts), twin(zero)))
    assert res[0] == "ZeroDivisionError" and F.ORDER == P


@pytest.mark.gpu
def test_stark_ctl_helpers(pb):
    """gl_stark_ctl_helpers on each table of the three-table CTL system with twin traces (filters 0 / 1 as p / p + 1),
    twin (beta, gamma) pairs and twin program constants, against the restated CTL columns; a combine that is zero only
    in non-canonical form (a selected all-zero tuple, gamma 0 given as p) is refused as the canonical zero is."""
    import torch

    from plonky2_b200 import _native as N
    from plonky2_b200 import cross_table_lookup as X
    from test_stark_ctl import _groups_and_aux, system, system_traces

    starks, config, ctls = system()
    traces, _ = system_traces()
    pairs = [(0x1357, 0x2468), (0xACE, 0xBDF)]
    degree = 3
    ctx, L = pb.default_context(), N.lib()
    for t, trace in enumerate(traces):
        groups, want = _groups_and_aux(traces, ctls, t, pairs, degree)
        cols, n = trace.shape
        prog, offsets, consts = X.ctl_row_programs(groups, cols)
        zs_index, _, num_helpers = X.zs_layout(groups, len(pairs), degree)

        def run(trace, consts, ch):
            dt = _dev(trace)
            out = torch.empty((num_helpers + len(zs_index), n), dtype=torch.int64, device="cuda")
            c = np.ascontiguousarray(consts, dtype=np.uint64)
            N.check(L.gl_stark_ctl_helpers(ctx.h, N.vp(dt.data_ptr()), n, cols, (n - 1).bit_length(), prog,
                                           offsets.ctypes.data_as(N.u32p), len(offsets) - 1,
                                           N.np_ptr(c) if len(c) else None, len(c), N.np_ptr(ch), len(pairs), degree,
                                           zs_index.ctypes.data_as(N.u32p), N.vp(out.data_ptr())), ctx.h)
            return _host(out)

        ch = _u64([v for pr in pairs for v in pr])
        res = invariant("gl_stark_ctl_helpers", "table %d trace, constants, challenges" % t, run, (trace, consts, ch),
                        (twin(trace), twin(consts), twin(ch)))
        assert res[0] == "ok" and np.array_equal(res[1], want), t
    # the looked table of the second CTL (table 1, column MW with filter MT): MW = 0 at a row, gamma = 0
    from test_stark_ctl import MW
    t0 = traces[1].copy()
    t0[MW, 0] = 0
    groups, _ = _groups_and_aux(traces, ctls, 1, pairs, degree)
    cols, n = t0.shape
    prog, offsets, consts = X.ctl_row_programs(groups, cols)
    zs_index, _, num_helpers = X.zs_layout(groups, len(pairs), degree)
    zero = _u64([pairs[0][0], 0, pairs[1][0], 0])
    res = invariant("gl_stark_ctl_helpers", "a zero combine", run, (t0, consts, zero), (twin(t0), twin(consts), twin(zero)))
    assert res[0] == "ZeroDivisionError"


@pytest.mark.gpu
def test_stark_quotients(pb, oracle):
    """gl_stark_quotient (FibonacciStark) and gl_stark_quotient_aux (a logUp STARK) with twin public inputs and program
    constants in `consts` and twin alphas, against the restated quotient; gl_stark_quotient_shard (shard 0 of 1) the
    same, and gl_stark_quotient_from_shards from the gathered shard values given as twins."""
    import stark_twin as T
    import torch

    from plonky2_b200 import _native as N
    from plonky2_b200 import stark as S
    from test_stark_prove import _fib_case

    ctx, L = pb.default_context(), N.lib()
    stark, config, trace, pi = _fib_case(8)
    f = config.fri_config
    tc = S._commit_trace(_dev(trace), f.rate_bits, f.cap_height, ctx)
    try:
        alphas = _u64([0xC0FFEE, 1])
        b, consts, _ = S.quotient_program(stark, pi, [int(a) for a in alphas])
        prog, qdf = b.program(), stark.quotient_degree_factor()
        want = T.quotient(oracle, stark, oracle.Commit(trace, f.rate_bits, f.cap_height), pi, [int(a) for a in alphas])
        size = want.shape[1]

        def run(consts, al):
            out = torch.empty((len(al), size), dtype=torch.int64, device="cuda")
            N.check(L.gl_stark_quotient(ctx.h, tc.h, prog, len(b.instrs), N.np_ptr(consts), len(consts), N.np_ptr(al),
                                        len(al), qdf, N.vp(out.data_ptr())), ctx.h)
            return _host(out)

        res = invariant("gl_stark_quotient", "public inputs, constants, alphas", run, (consts, alphas),
                        (twin(consts), twin(alphas)))
        assert res[0] == "ok" and np.array_equal(res[1], want)

        def run_shard(consts, al):
            out = torch.empty((len(al), size), dtype=torch.int64, device="cuda")
            N.check(L.gl_stark_quotient_shard(ctx.h, tc.h, None, prog, len(b.instrs), N.np_ptr(consts), len(consts),
                                              N.np_ptr(al), len(al), qdf, N.vp(out.data_ptr())), ctx.h)
            return _host(out)

        res = invariant("gl_stark_quotient_shard", "public inputs, constants, alphas", run_shard, (consts, alphas),
                        (twin(consts), twin(alphas)))
        assert res[0] == "ok"

        def run_from(values):
            dv = _dev(values)
            out = torch.empty((2, size), dtype=torch.int64, device="cuda")
            N.check(L.gl_stark_quotient_from_shards(ctx.h, N.vp(dv.data_ptr()), 1, 2, tc.degree_log, qdf,
                                                    N.vp(out.data_ptr())), ctx.h)
            return _host(out)

        res = invariant("gl_stark_quotient_from_shards", "shard values", run_from, (res[1],), (twin(res[1]),))
        assert res[0] == "ok" and np.array_equal(res[1], want)
        vals = small_words(0x6501, (2, size))
        invariant("gl_stark_quotient_from_shards", "small shard values", run_from, (vals,), (twin(vals),))
    finally:
        tc.close()

    # gl_stark_quotient_aux: the range-check logUp STARK, lookup challenges bound in consts
    from test_stark_lookups import RangeCheckStark

    stark = RangeCheckStark()
    trace = RangeCheckStark.generate_trace(7, seed=2)
    ch = [0x4242, 0x1717]
    aux = T.aux_columns(stark, trace, ch)[0]
    tc = S._commit_trace(_dev(trace), f.rate_bits, f.cap_height, ctx)
    ac = S._commit_trace(_dev(aux), f.rate_bits, f.cap_height, ctx)
    try:
        alphas = _u64([5, 0x10001])
        b, consts, _ = S.quotient_program(stark, [0] * stark.PUBLIC_INPUTS, [int(a) for a in alphas], ac, ch)
        prog, qdf = b.program(), stark.quotient_degree_factor()
        want = T.quotient(oracle, stark, oracle.Commit(trace, f.rate_bits, f.cap_height), [0] * stark.PUBLIC_INPUTS,
                          [int(a) for a in alphas], aux_coeffs=oracle.Commit(aux, f.rate_bits, f.cap_height).coeffs,
                          lookup_challenges=ch)
        size = want.shape[1]

        def run_aux(consts, al):
            out = torch.empty((len(al), size), dtype=torch.int64, device="cuda")
            N.check(L.gl_stark_quotient_aux(ctx.h, tc.h, ac.h, prog, len(b.instrs), N.np_ptr(consts), len(consts),
                                            N.np_ptr(al), len(al), qdf, N.vp(out.data_ptr())), ctx.h)
            return _host(out)

        res = invariant("gl_stark_quotient_aux", "public inputs, challenges, constants, alphas", run_aux,
                        (consts, alphas), (twin(consts), twin(alphas)))
        assert res[0] == "ok" and np.array_equal(res[1], want)
    finally:
        tc.close()
        ac.close()


@pytest.mark.gpu
def test_plonk_quotients(pb):
    """gl_plonk_quotient and gl_plonk_quotient_shard (shard 0 of 1) with the challenges and program constants bound
    into `consts` and the alphas given as twins. The canonical call is plonk.compute_quotient_polys's, which
    test_plonk_quotient.py checks against the oracle at this shape."""
    import torch

    import plonk_circuits as PC
    from plonky2_b200 import _native as N
    from plonky2_b200 import plonk
    from plonky2_b200.prover import commit_zs_partial_products

    c = PC.shape_circuit(PC.SHAPES[0], cap_height=1)
    cfg, cd = c.config, c.common
    nr, nc = cfg.num_routed_wires, cfg.num_challenges
    betas, gammas, alphas = [0x11, 0x2222][:nc], [0x333, 1][:nc], [0x4444, 0][:nc]
    ctx, L = pb.default_context(), N.lib()
    cs = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height)
    w = pb.PolynomialBatch.from_values(c.wires, cfg.rate_bits, False, cfg.cap_height)
    z = commit_zs_partial_products(_dev(c.wires[:nr]), _dev(c.sigmas), cd.k_is, betas, gammas, cd.quotient_degree_factor,
                                   cfg.rate_bits, cfg.cap_height)
    try:
        commits = [cs, w, z]
        prog, consts, al = plonk.quotient_program(cd, commits, c.public_inputs_hash, betas, gammas, alphas)
        handles = (C.c_void_p * 3)(*[x.h for x in commits])
        qdf = cd.quotient_degree_factor
        size = (1 << cd.degree_bits) << (qdf - 1).bit_length()
        want = _host(plonk.compute_quotient_polys(cd, cs, c.public_inputs_hash, w, z, betas, gammas, alphas))

        for fn in ("gl_plonk_quotient", "gl_plonk_quotient_shard"):
            def run(consts, al):
                out = torch.empty((nc, size), dtype=torch.int64, device="cuda")
                N.check(getattr(L, fn)(ctx.h, handles, 3, prog, len(prog), N.np_ptr(consts), len(consts), N.np_ptr(al),
                                       nc, cd.num_vanishing_terms(), qdf, N.vp(out.data_ptr())), ctx.h)
                return _host(out)

            res = invariant(fn, "challenges, constants, alphas", run, (consts, al), (twin(consts), twin(al)))
            assert res[0] == "ok"
            if fn == "gl_plonk_quotient":
                assert np.array_equal(res[1], want)
    finally:
        for x in (cs, w, z):
            x.close()


@pytest.mark.gpu
def test_sigma_polys(pb):
    """gl_sigma_polys with twin k_is (host k_is, host and device outputs): the identity sigmas of the restatement."""
    import torch

    from plonky2_b200 import _native as N
    from plonky2_b200 import plonk
    from test_circuit_data import _want

    cfg, db = plonk.CircuitConfig(num_wires=12, num_routed_wires=8), 9
    n, nr = 1 << db, cfg.num_routed_wires
    ctx, L = pb.default_context(), N.lib()
    k = _u64(plonk.get_unique_coset_shifts(nr))

    def run(k):
        out = torch.zeros((nr, n), dtype=torch.int64, device="cuda")
        N.check(L.gl_sigma_polys(ctx.h, None, 0, N.MEM_HOST, cfg.num_wires, nr, db, 0, N.np_ptr(k), N.vp(out.data_ptr()),
                                 N.MEM_DEVICE), ctx.h)
        host = np.empty((nr, n), dtype=np.uint64)
        N.check(L.gl_sigma_polys(ctx.h, None, 0, N.MEM_HOST, cfg.num_wires, nr, db, 0, N.np_ptr(k), N.np_ptr(host),
                                 N.MEM_HOST), ctx.h)
        return [_host(out), host]

    res = invariant("gl_sigma_polys", "k_is", run, (k,), (twin(k),))
    want = _want(cfg, db, np.zeros((0, 2), dtype=np.int64), literal=True)
    assert res[0] == "ok" and np.array_equal(res[1][0], want) and np.array_equal(res[1][1], want)
    # k_is that are small words themselves (k_0 = 1 is the only small coset shift)
    ks = small_words(0x6600, (nr,))
    invariant("gl_sigma_polys", "small k_is", run, (ks,), (twin(ks),))


# points of F_{p^2}: zero, one, a coordinate 2^32 - 2 (twin 2^64 - 1), small, and mixed large/small
POINTS = [(0, 0), (1, 0), (2**32 - 2, 5), (7, 2**32 - 2), (0x123456789ABCDEF, 3), (11, 0)]


@pytest.mark.gpu
def test_openings(pb, oracle):
    """gl_openings (host and device out), gl_openings_shard (2 shards, summed) and gl_commit_eval_ext with twin points,
    among them (p, p) for zero and a coordinate 2^64 - 1, against Horner evaluation of the coefficients."""
    import torch

    from plonky2_b200 import _native as N

    ctx, L = pb.default_context(), N.lib()
    batches = [pb.PolynomialBatch.from_values(synth(0x6700 + i, (B, 1 << lg)), 1, False, 1)
               for i, (B, lg) in enumerate([(3, 6), (5, 8)])]
    try:
        handles = (N.vp * 2)(*[b.h for b in batches])
        reqs = [(0, 0), (1, 0), (0, 1), (1, 2), (0, 3), (1, 4), (1, 5)]   # (commitment, point)
        hs = (N.vp * len(reqs))(*[batches[i].h for i, _ in reqs])
        pidx = np.array([p for _, p in reqs], dtype=np.uint32)
        total = sum(batches[i].num_polys for i, _ in reqs)
        pts = _u64([v for p in POINTS for v in p])

        def run(points):
            out = np.empty((total, 2), dtype=np.uint64)
            N.check(L.gl_openings(ctx.h, hs, pidx.ctypes.data_as(N.u32p), len(reqs), N.np_ptr(points), len(POINTS),
                                  N.np_ptr(out), N.MEM_HOST), ctx.h)
            dout = torch.empty((total, 2), dtype=torch.int64, device="cuda")
            N.check(L.gl_openings(ctx.h, hs, pidx.ctypes.data_as(N.u32p), len(reqs), N.np_ptr(points), len(POINTS),
                                  N.vp(dout.data_ptr()), N.MEM_DEVICE), ctx.h)
            parts = []
            for g in range(2):
                part = np.empty((total, 2), dtype=np.uint64)
                N.check(L.gl_openings_shard(ctx.h, hs, pidx.ctypes.data_as(N.u32p), len(reqs), N.np_ptr(points),
                                            len(POINTS), g, 2, N.np_ptr(part), N.MEM_HOST), ctx.h)
                parts.append(part)
            ev = []
            for i, p in reqs:
                e = np.empty((batches[i].num_polys, 2), dtype=np.uint64)
                N.check(L.gl_commit_eval_ext(batches[i].h, N.np_ptr(points[2 * p:2 * p + 2].copy()), N.np_ptr(e)), ctx.h)
                ev.append(e)
            return [out, _host(dout)] + parts + [np.concatenate(ev)]

        res = invariant("gl_openings / gl_openings_shard / gl_commit_eval_ext", "points", run, (pts,), (twin(pts),))
        assert res[0] == "ok"
        out, dout, s0, s1, ev = res[1]
        want = np.array([oracle.eval_poly_base_at_ext(batches[i].polynomials[b], POINTS[p])
                         for i, p in reqs for b in range(batches[i].num_polys)], dtype=np.uint64)
        assert np.array_equal(out, want) and np.array_equal(dout, want) and np.array_equal(ev, want)
        summed = (s0.astype(object) + s1.astype(object)) % P
        assert np.array_equal(summed.astype(np.uint64), want)
        # the point (p, p) is zero: every value is the constant coefficient
        zero = _u64([P, P] * len(POINTS))
        res_z = _outcome(lambda: run(zero))
        assert res_z[0] == "ok" and np.array_equal(res_z[1][0], run(_u64([0, 0] * len(POINTS)))[0])
    finally:
        for b in batches:
            b.close()


def _fri_instance(pb, seed):
    """Two resident commitments (degree 2^7, rate 2) and two opening batches."""
    import ctypes

    from plonky2_b200 import _native as N

    a = pb.PolynomialBatch.from_values(synth(seed, (4, 1 << 7)), 2, False, 2)
    b = pb.PolynomialBatch.from_values(synth(seed + 1, (3, 1 << 7)), 2, False, 2)
    polys = [[(0, 0), (0, 1), (1, 2), (0, 3)], [(1, 0), (0, 2)]]
    keep = []

    def batches(points):
        arr = (N.FriBatch * len(polys))()
        for i, ps in enumerate(polys):
            oi = np.array([o for o, _ in ps], dtype=np.uint32)
            pi = np.array([p for _, p in ps], dtype=np.uint32)
            keep.extend([oi, pi])
            arr[i].point[0], arr[i].point[1] = int(points[2 * i]), int(points[2 * i + 1])
            arr[i].num_polys = len(ps)
            arr[i].oracle_index = oi.ctypes.data_as(N.u32p)
            arr[i].poly_index = pi.ctypes.data_as(N.u32p)
        return arr

    return [a, b], polys, batches, (ctypes.c_void_p * 2)(a.h, b.h)


def _fri_read(pb, f, n_coeffs=None):
    """(coefficients if any, first-round values) of a FRI state."""
    from plonky2_b200 import _native as N

    L = N.lib()
    ln = C.c_size_t()
    vals = np.empty(2 << 12, dtype=np.uint64)
    N.check(L.gl_fri_values_local(f, N.np_ptr(vals), vals.size, C.byref(ln)))
    out = [vals[:2 * ln.value].copy()]
    if n_coeffs:
        co = np.empty(2 * n_coeffs, dtype=np.uint64)
        N.check(L.gl_fri_coeffs(f, N.np_ptr(co)))
        out.insert(0, co)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("z", ["small", "zero"])
def test_fri_begin(pb, z):
    """gl_fri_begin with twin alpha and batch points. The point (p, p) is zero: it takes the k_div_by_x branch and gives
    (0, 0)'s result. The canonical call is the one test_gpu_parity.py's prove_openings checks against the oracle."""
    from plonky2_b200 import _native as N

    ctx, L = pb.default_context(), N.lib()
    oracles, _, batches, handles = _fri_instance(pb, 0x6800)
    try:
        pts = _u64([0x1234, 2**32 - 2, 0, 1] if z == "small" else [0, 0, 3, 2**32 - 2])
        alpha = _u64([0xBEEF, 0])

        def run(points, alpha):
            f = N.vp()
            N.check(L.gl_fri_begin(ctx.h, handles, 2, batches(points), 2, N.np_ptr(alpha), 2, 2, C.byref(f)), ctx.h)
            try:
                return _fri_read(pb, f, 1 << 7)
            finally:
                L.gl_fri_destroy(f)

        res = invariant("gl_fri_begin", "points, alpha", run, (pts, alpha), (twin(pts), twin(alpha)))
        assert res[0] == "ok"
        if z == "zero":
            pz = pts.copy()
            pz[:2] = P
            res2 = invariant("gl_fri_begin", "the point (p, p)", run, (pts, alpha), (pz, alpha))
            assert res2[0] == "ok"
    finally:
        for o in oracles:
            o.close()


@pytest.mark.gpu
def test_fri_begin_values(pb):
    """gl_fri_begin_values with twin opened values, alpha and points: the same first-round codeword as gl_fri_begin (in
    the value domain the quotients are exact). A point of the LDE domain given as (x, p) is refused as (x, 0) is."""
    from plonky2_b200 import _native as N
    from plonky2_b200.field import coset_shift

    ctx, L = pb.default_context(), N.lib()
    oracles, polys, batches, handles = _fri_instance(pb, 0x6900)
    try:
        pts = _u64([0x1234, 2**32 - 2, 5, 1])
        alpha = _u64([0xBEEF, 1])
        opened = []
        for i, ps in enumerate(polys):
            for o, p in ps:
                e = np.empty(oracles[o].num_polys * 2, dtype=np.uint64)
                N.check(L.gl_commit_eval_ext(oracles[o].h, N.np_ptr(pts[2 * i:2 * i + 2].copy()), N.np_ptr(e)), ctx.h)
                opened += list(e[2 * p:2 * p + 2])
        opened = _u64(opened)
        opened_small = opened.copy()
        opened_small[::3] = opened_small[::3] & np.uint64(0xFFFF)   # the codeword changes; the invariance must hold

        def run(points, opened, alpha):
            f = N.vp()
            N.check(L.gl_fri_begin_values(ctx.h, handles, 2, batches(points), 2, N.np_ptr(opened), N.np_ptr(alpha), 2,
                                          C.byref(f)), ctx.h)
            try:
                return _fri_read(pb, f)
            finally:
                L.gl_fri_destroy(f)

        res = invariant("gl_fri_begin_values", "points, opened values, alpha", run, (pts, opened, alpha),
                        (twin(pts), twin(opened), twin(alpha)))
        assert res[0] == "ok"
        f = N.vp()
        N.check(L.gl_fri_begin(ctx.h, handles, 2, batches(pts), 2, N.np_ptr(alpha), 2, 2, C.byref(f)), ctx.h)
        try:
            assert np.array_equal(_fri_read(pb, f)[0], res[1][0])
        finally:
            L.gl_fri_destroy(f)
        invariant("gl_fri_begin_values", "opened values", run, (pts, opened_small, alpha),
                  (twin(pts), twin(opened_small), twin(alpha)))
        lde = pts.copy()
        lde[0], lde[1] = coset_shift(), 0
        res = invariant("gl_fri_begin_values", "an LDE-domain point", run, (lde, opened, alpha),
                        (twin(lde), opened, alpha))
        assert res[0] == "ZeroDivisionError" and "LDE domain" in res[1]
    finally:
        for o in oracles:
            o.close()


@pytest.mark.gpu
def test_fri_fold_and_mix(pb):
    """gl_fri_fold and gl_fri_mix with twin beta (among them (p, p + 1) and (2^64 - 1, 0)): the same codeword, and
    the same final polynomial."""
    from plonky2_b200 import _native as N

    ctx, L = pb.default_context(), N.lib()
    big = synth(0x6A00, (1 << 8, 2))
    small = synth(0x6A01, (1 << 6, 2))

    def run(b1, b2):
        fs = []
        try:
            for co, lg in ((big, 8), (small, 6)):
                f = N.vp()
                N.check(L.gl_fri_begin_from_coeffs(ctx.h, N.np_ptr(np.ascontiguousarray(co)), lg, 1, 1, C.byref(f)), ctx.h)
                fs.append(f)
            cap = np.empty(8, dtype=np.uint64)
            N.check(L.gl_fri_commit_round(fs[0], 2, N.np_ptr(cap)), ctx.h)
            N.check(L.gl_fri_fold(fs[0], N.np_ptr(b1)), ctx.h)
            N.check(L.gl_fri_mix(fs[0], fs[1], N.np_ptr(b1)), ctx.h)
            N.check(L.gl_fri_commit_round(fs[0], 1, N.np_ptr(cap)), ctx.h)
            N.check(L.gl_fri_fold(fs[0], N.np_ptr(b2)), ctx.h)
            vals = _fri_read(pb, fs[0])[0]
            buf = np.empty(2 << 6, dtype=np.uint64)
            ln = C.c_size_t()
            N.check(L.gl_fri_final_poly(fs[0], N.np_ptr(buf), buf.size, C.byref(ln)), ctx.h)
            return [vals, buf[:2 * ln.value].copy()]
        finally:
            for f in fs:
                L.gl_fri_destroy(f)

    for b1, b2 in (([0, 1], [2**32 - 2, 0]), ([0x1234, 0x5678], [7, 2**40])):
        b1, b2 = _u64(b1), _u64(b2)
        res = invariant("gl_fri_fold / gl_fri_mix", "beta", run, (b1, b2), (twin(b1), twin(b2)))
        assert res[0] == "ok"


@pytest.mark.gpu
def test_fri_pow(pb):
    """gl_fri_pow from a twin duplex state: the canonical state's smallest nonce, which meets the bound."""
    from plonky2_b200 import _native as N
    from plonky2_b200.hash import PoseidonPermutation

    ctx, L = pb.default_context(), N.lib()
    state = small_words(0x6B00, (12,))
    bits = 12

    def run(st):
        nonce = np.zeros(1, dtype=np.uint64)
        N.check(L.gl_fri_pow(ctx.h, N.np_ptr(np.ascontiguousarray(st)), 3, bits, N.np_ptr(nonce)), ctx.h)
        return nonce

    res = invariant("gl_fri_pow", "state", run, (state,), (twin(state),))
    assert res[0] == "ok"
    nonce = int(res[1][0])
    st = state.copy()
    st[3] = nonce
    perm = PoseidonPermutation()
    perm.set_from_iter([int(v) for v in st], 0)
    perm.permute()
    assert 64 - int(perm.state[7]).bit_length() >= bits


@pytest.mark.gpu
@pytest.mark.parametrize("mem", ["host", "device"])
def test_commit_salt(pb, oracle, mem):
    """gl_commit_finish with a twin salt (host and device memory) and gl_commit_create with twin columns and salt: cap,
    digests, every leaf (gl_commit_leaves) and opened leaves (gl_commit_open) equal the canonical-salt commitment's,
    canonical, and the oracle's."""
    from plonky2_b200 import _native as N

    log_n, r, h, B = 8, 1, 2, 3
    n, NN = 1 << log_n, 1 << (log_n + r)
    vals, salt = small_words(0x6C00, (B, n)), small_words(0x6C01, (4, NN))
    ctx, L = pb.default_context(), N.lib()
    idx = np.array([0, 1, 77, NN - 1], dtype=np.uint64)

    def read(hnd):
        cap = np.empty((1 << h, 4), dtype=np.uint64)
        N.check(L.gl_commit_cap(hnd, N.np_ptr(cap), N.MEM_HOST), ctx.h)
        dig = np.empty((2 * (NN - (1 << h)), 4), dtype=np.uint64)
        N.check(L.gl_commit_digests(hnd, N.np_ptr(dig), N.MEM_HOST), ctx.h)
        lv = np.empty((NN, B + 4), dtype=np.uint64)
        N.check(L.gl_commit_leaves(hnd, 0, NN, N.np_ptr(lv), N.MEM_HOST), ctx.h)
        ol = np.empty((len(idx), B + 4), dtype=np.uint64)
        paths = np.empty((len(idx), log_n + r - h, 4), dtype=np.uint64)
        N.check(L.gl_commit_open(hnd, N.np_ptr(idx), len(idx), N.np_ptr(ol), N.np_ptr(paths)), ctx.h)
        return [cap, dig, lv, ol, paths]

    def run_finish(salt):
        hnd = N.vp()
        N.check(L.gl_commit_begin(ctx.h, B, log_n, r, h, 1, 0, 1, None, C.byref(hnd)), ctx.h)
        try:
            N.check(L.gl_commit_add_columns(hnd, 0, B, N.np_ptr(vals), n, N.COLS_VALUES, N.MEM_HOST), ctx.h)
            if mem == "host":
                N.check(L.gl_commit_finish(hnd, N.np_ptr(np.ascontiguousarray(salt)), N.MEM_HOST), ctx.h)
            else:
                ds = _dev(salt)
                N.check(L.gl_commit_finish(hnd, N.vp(ds.data_ptr()), N.MEM_DEVICE), ctx.h)
                ctx.synchronize()
            return read(hnd)
        finally:
            L.gl_commit_destroy(hnd)

    res = invariant("gl_commit_finish", "salt (%s memory)" % mem, run_finish, (salt,), (twin(salt),))
    o = oracle.Commit(vals, r, h, salt=salt)
    assert res[0] == "ok"
    cap, dig, lv, ol, _ = res[1]
    assert np.array_equal(cap, o.cap) and np.array_equal(dig, o.digests) and np.array_equal(lv, o.leaves)
    assert np.array_equal(ol, o.leaves[idx.astype(np.int64)])

    def run_create(vals, salt):
        hnd = N.vp()
        if mem == "host":
            N.check(L.gl_commit_create(ctx.h, N.np_ptr(np.ascontiguousarray(vals)), n, B, log_n, r, h,
                                       N.np_ptr(np.ascontiguousarray(salt)), 0, N.MEM_HOST, C.byref(hnd)), ctx.h)
        else:
            dv, ds = _dev(vals), _dev(salt)
            N.check(L.gl_commit_create(ctx.h, N.vp(dv.data_ptr()), n, B, log_n, r, h, N.vp(ds.data_ptr()), 0,
                                       N.MEM_DEVICE, C.byref(hnd)), ctx.h)
            ctx.synchronize()
        try:
            return read(hnd)
        finally:
            L.gl_commit_destroy(hnd)

    res = invariant("gl_commit_create", "columns and salt (%s memory)" % mem, run_create, (vals, salt),
                    (twin(vals), twin(salt)))
    assert res[0] == "ok" and np.array_equal(res[1][0], o.cap)


@pytest.mark.gpu
def test_commit_finish_prefixed(pb, oracle):
    """gl_commit_finish_prefixed with a twin prefix cap in device memory: the same cap and digests, and gl_commit_open's
    prefixed leaves canonical -- the leaves `prefix || row` of the oracle's tree."""
    from plonky2_b200 import _native as N

    log_n, r, h, B = 6, 1, 3, 3
    n, NN = 1 << log_n, 1 << (log_n + r)
    vals = small_words(0x6D00, (B, n))
    prefix = small_words(0x6D01, (NN, 4))
    ctx, L = pb.default_context(), N.lib()
    idx = np.array([0, 5, NN - 1], dtype=np.uint64)
    layers = log_n + r - h

    def run(prefix):
        hnd = N.vp()
        N.check(L.gl_commit_begin(ctx.h, B, log_n, r, h, 0, 0, 1, None, C.byref(hnd)), ctx.h)
        try:
            N.check(L.gl_commit_add_columns(hnd, 0, B, N.np_ptr(vals), n, N.COLS_VALUES, N.MEM_HOST), ctx.h)
            dp = _dev(prefix)
            N.check(L.gl_commit_finish_prefixed(hnd, N.vp(dp.data_ptr())), ctx.h)
            ctx.synchronize()
            cap = np.empty((1 << h, 4), dtype=np.uint64)
            N.check(L.gl_commit_cap(hnd, N.np_ptr(cap), N.MEM_HOST), ctx.h)
            ol = np.empty((len(idx), B + 4), dtype=np.uint64)
            paths = np.empty((len(idx), layers, 4), dtype=np.uint64)
            N.check(L.gl_commit_open(hnd, N.np_ptr(idx), len(idx), N.np_ptr(ol), N.np_ptr(paths)), ctx.h)
            return [cap, ol, paths]
        finally:
            L.gl_commit_destroy(hnd)

    res = invariant("gl_commit_finish_prefixed", "prefix", run, (prefix,), (twin(prefix),))
    assert res[0] == "ok"
    o = oracle.Commit(vals, r, h)
    leaves = np.concatenate([prefix, o.leaves], axis=1)
    digests, cap = oracle.merkle_build(leaves, h)
    assert np.array_equal(res[1][0], cap.reshape(-1, 4)) and np.array_equal(res[1][1], leaves[idx.astype(np.int64)])


@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 2, 3, 4])
def test_narrow_leaves(pb, oracle, W):
    """Leaves of 1 to 4 words, whose digest is the leaf itself (hash_or_noop): gl_merkle_build from twin leaves in host
    and device memory, and a commitment from twin coefficient columns (gl_commit_add_columns GL_COLS_COEFFS, host and
    device): cap, digests, opened leaves and paths canonical and equal to the canonical leaves'."""
    from plonky2_b200 import _native as N

    ctx, L = pb.default_context(), N.lib()
    NN, h = 1 << 8, 2
    leaves = small_words(0x6E00 + W, (NN, W))
    idx = np.array([0, 3, NN - 1], dtype=np.uint64)

    def run_tree(leaves, mem):
        m = N.vp()
        d = _dev(leaves) if mem == N.MEM_DEVICE else None
        src = N.vp(d.data_ptr()) if d is not None else N.np_ptr(np.ascontiguousarray(leaves))
        N.check(L.gl_merkle_build(ctx.h, src, NN, W, h, mem, C.byref(m)), ctx.h)
        try:
            cap = np.empty((1 << h, 4), dtype=np.uint64)
            N.check(L.gl_merkle_cap(m, N.np_ptr(cap), N.MEM_HOST), ctx.h)
            dig = np.empty((2 * (NN - (1 << h)), 4), dtype=np.uint64)
            N.check(L.gl_merkle_digests(m, N.np_ptr(dig), N.MEM_HOST), ctx.h)
            ol = np.empty((len(idx), W), dtype=np.uint64)
            paths = np.empty((len(idx), 8 - h, 4), dtype=np.uint64)
            N.check(L.gl_merkle_open(m, N.np_ptr(idx), len(idx), N.np_ptr(ol), N.np_ptr(paths)), ctx.h)
            return [cap, dig, ol, paths]
        finally:
            L.gl_merkle_destroy(m)

    for mem in (N.MEM_HOST, N.MEM_DEVICE):
        res = invariant("gl_merkle_build", "leaves of width %d (mem %d)" % (W, mem),
                        lambda lv: run_tree(lv, mem), (leaves,), (twin(leaves),))
        digests, cap = oracle.merkle_build(leaves, h)
        assert res[0] == "ok" and np.array_equal(res[1][0], cap.reshape(-1, 4))
        assert np.array_equal(res[1][1].reshape(-1), digests.reshape(-1))
        assert np.array_equal(res[1][2], leaves[idx.astype(np.int64)])

    coeffs = small_words(0x6F00 + W, (W, 1 << 6))

    def run_commit(cols, mem):
        hnd = N.vp()
        N.check(L.gl_commit_begin(ctx.h, W, 6, 2, h, 0, 0, 1, None, C.byref(hnd)), ctx.h)
        try:
            d = _dev(cols) if mem == N.MEM_DEVICE else None
            src = N.vp(d.data_ptr()) if d is not None else N.np_ptr(np.ascontiguousarray(cols))
            N.check(L.gl_commit_add_columns(hnd, 0, W, src, 1 << 6, N.COLS_COEFFS, mem), ctx.h)
            N.check(L.gl_commit_finish(hnd, None, N.MEM_HOST), ctx.h)
            cap = np.empty((1 << h, 4), dtype=np.uint64)
            N.check(L.gl_commit_cap(hnd, N.np_ptr(cap), N.MEM_HOST), ctx.h)
            co = np.empty((W, 1 << 6), dtype=np.uint64)
            N.check(L.gl_commit_coeffs(hnd, N.np_ptr(co), N.MEM_HOST), ctx.h)
            ol = np.empty((len(idx), W), dtype=np.uint64)
            paths = np.empty((len(idx), 8 - h, 4), dtype=np.uint64)
            N.check(L.gl_commit_open(hnd, N.np_ptr(idx), len(idx), N.np_ptr(ol), N.np_ptr(paths)), ctx.h)
            return [cap, co, ol, paths]
        finally:
            L.gl_commit_destroy(hnd)

    o = oracle.Commit(coeffs, 2, h, is_coeffs=True)
    for mem in (N.MEM_HOST, N.MEM_DEVICE):
        res = invariant("gl_commit_add_columns", "coefficient columns, width %d (mem %d)" % (W, mem),
                        lambda c: run_commit(c, mem), (coeffs,), (twin(coeffs),))
        assert res[0] == "ok" and np.array_equal(res[1][0], o.cap) and np.array_equal(res[1][1], coeffs)


# ------------------------------------------------------------------------------------------------ GPU: whole proofs
def _proof_arrays(obj, path=""):
    """[(path, array)] of every array in a proof object, recursively."""
    if isinstance(obj, np.ndarray):
        return [(path, obj)]
    if isinstance(obj, (list, tuple)):
        return [f for k, v in enumerate(obj) for f in _proof_arrays(v, "%s[%d]" % (path, k))]
    if isinstance(obj, dict):
        return [f for k in sorted(obj) for f in _proof_arrays(obj[k], "%s.%s" % (path, k))]
    if hasattr(obj, "__dict__"):
        return _proof_arrays(vars(obj), path)
    return []


def same_proofs(what, a, b):
    """a and b equal field for field, and every word of them canonical."""
    import stark_twin as T

    diff = T.proof_diff(a, b)
    assert not diff, "%s: the proof from non-canonical inputs differs at %s" % (what, diff)
    for p, x in _proof_arrays(a):
        assert all(int(v) < P for v in x.reshape(-1)), "%s: %s holds a non-canonical word" % (what, p)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fibonacci-host", "fibonacci-tensor", "range-host", "range-tensor",
                                  "range-blocked"])
def test_stark_proofs_of_twin_traces(pb, oracle, case):
    """stark.prove from a trace and from its twin (host columns or a torch CUDA tensor; the range-check case also with
    a non-resident LDE in 2 blocks), public inputs given as twins: equal proofs, accepted by the restated verifier."""
    import stark_twin as T

    from plonky2_b200 import stark as S
    from test_stark_lookups import _range_case
    from test_stark_prove import _fib_case

    name, source = case.split("-")
    stark, config, trace, pi = _fib_case(6) if name == "fibonacci" else _range_case(8)
    assert (trace < TWIN_BELOW).any()
    kw = dict(lde_blocks=2) if source == "blocked" else {}

    def arg(t):
        return _dev(t) if source == "tensor" else t

    a = S.prove(stark, config, arg(trace), pi, **kw)
    b = S.prove(stark, config, arg(twin(trace)), [twin(v) for v in pi], **kw)
    same_proofs("stark.prove(%s)" % case, a, b)
    assert T.verify(oracle, stark, config, b) is None


@pytest.mark.gpu
def test_ctl_proof_of_twin_traces(pb, oracle):
    """cross_table_lookup.prove_with_ctls on the three-table system from twin traces and public inputs: the proof of the
    canonical traces, accepted by the restated verifier."""
    import stark_twin as T

    from plonky2_b200 import cross_table_lookup as X
    from test_stark_ctl import system, system_traces

    starks, config, ctls = system()
    traces, pis = system_traces()
    a = X.prove_with_ctls(starks, config, traces, ctls, pis)
    b = X.prove_with_ctls(starks, config, [twin(t) for t in traces], ctls, [[twin(v) for v in p] for p in pis])
    same_proofs("prove_with_ctls", a, b)
    assert T.verify_with_ctls(oracle, starks, config, ctls, b) is None


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["plain", "lookup", "zk"])
def test_plonk_proofs_of_twin_witnesses(pb, oracle, shape):
    """plonk.prove_with_witness from a witness and from its twin (public inputs as twins too): the same to_bytes(), the
    canonical one equal to the CPU prover's, and the restated verifier accepts the proof read back from the twin's
    bytes. The zero-knowledge case uses fixed salt keys."""
    import plonk_circuits as PC
    from plonky2_b200 import plonk

    if shape == "zk":
        cfg = plonk.standard_recursion_zk_config()
        c, _ = PC.zk_circuit(plonk, cfg, PC.quick_fri_config(cfg))
        keys = PC.KEYS
    else:
        c = PC.shape_circuit(PC.SHAPES[0] if shape == "plain" else PC.LOOKUP_64, cap_height=1, public_inputs=[3, 1, 4, 1, 5])
        keys = None
    cfg, cd = c.config, c.common
    digest = [int(x) for x in synth(0x592, (4,))]
    fri_cfg = PC.quick_fri_config(cfg)
    fri_params = fri_cfg.fri_params(cd.degree_bits, keys is not None)
    assert (c.wires < TWIN_BELOW).any()
    cs = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height)
    try:
        prover_data = plonk.ProverOnlyCircuitData(cs, c.sigmas, digest, fri_params)
        kw = dict(salt_keys=keys) if keys else {}
        a = plonk.prove_with_witness(prover_data, cd, c.wires, c.public_inputs, **kw).to_bytes()
        b = plonk.prove_with_witness(prover_data, cd, twin(c.wires), [twin(v) for v in c.public_inputs], **kw).to_bytes()
        assert a == b, "prove_with_witness(%s): the bytes from a non-canonical witness differ" % shape
        want, _ = PC.oracle_prove(oracle, c, digest, fri_cfg, c.public_inputs, **(dict(salts=PC.salts(c)) if keys else {}))
        assert a == want
        proof = plonk.ProofWithPublicInputs.from_bytes(b, cd, fri_params)
        assert PC.oracle_verify(oracle, plonk, c, digest, fri_cfg, PC.parts_of(proof, cs.merkle_tree.cap.hashes)) is None
    finally:
        cs.close()
