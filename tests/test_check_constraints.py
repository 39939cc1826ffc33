"""check_constraints on the device: gl_stark_check_rows (k_stark_check_rows, gl_stark_rows.cuh) and gl_plonk_check_rows
(k_plonk_check_rows, gl_vanishing.cuh), stark.check_constraints / plonk.check_constraints and the provers'
check_constraints=True.

Every result is compared as the exact list of failing (row, index) pairs, in (row, index) order, with an evaluator
written here from the entry points' contract: each GL_STARK_EMIT filtered by [always] / [row != n - 1] / [row = 0] /
[row = n - 1], each GL_VP_TERM on its own with x = w_n^row and L_0 = [row = 0], on the commitments' values on H (the
oracle's FFT of their coefficients).

The two contracts of include/plonky2_b200.h that tests/test_gpu_host_buffers.py and tests/test_noncanonical_inputs.py
check for its entry points are checked here for those of include/plonky2_b200_check.h: host inputs (the program and
its constants) are read when a call returns, from page-locked buffers overwritten on return; non-canonical constants
give the same reports.

CPU: the binding, the refusals that need no device, ConstraintError's message, and the host build of both row functions
(tests/emu/check_rows_emu.cpp) on random programs at the limits.
GPU (-m gpu): random programs at the limits, report truncation, non-canonical constants, page-locked inputs, every
handle kind, holding and broken STARKs (lookups, CTLs, degree 0) and circuits, the provers' flag, and agreement with the
reference's alpha-combined check."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import gl_numpy as G
import stark_twin as T
from conftest import P, synth
from plonky2_b200 import _native as N
from plonky2_b200 import field as E
from plonky2_b200 import stark as S
from test_gpu_programs import SALT, STARK_MAX_INSTR, VP_CONSTS, VP_MAX_COMMITS, stark_program, vp_program

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VP_LOCAL, VP_NEXT, VP_CONST, VP_X, VP_L0, VP_ADD, VP_SUB, VP_MUL, VP_TERM, VP_ADDC, VP_MULC = range(11)


# ------------------------------------------------------------------------------------------------------ evaluators
def _pairs(fails, index_of):
    """(row, index) pairs in (row, index) order from [(index, bool array over rows)]."""
    rows, idx = [], []
    for k, f in fails:
        r = np.nonzero(f)[0]
        rows.append(r)
        idx.append(np.full(len(r), index_of(k), dtype=np.int64))
    if not rows:
        return []
    rows, idx = np.concatenate(rows), np.concatenate(idx)
    order = np.lexsort((idx, rows))
    return list(zip(rows[order].tolist(), idx[order].tolist()))


def stark_expected(prog, trace, aux, consts):
    """gl_stark_check_rows' failing (row, EMIT ordinal) pairs. prog: (n_instr, 4) uint16; trace, aux: values on H."""
    n = trace.shape[1]
    row = np.arange(n)
    on = {S.KIND_CONSTRAINT: np.ones(n, bool), S.KIND_TRANSITION: row != n - 1, S.KIND_FIRST_ROW: row == 0,
          S.KIND_LAST_ROW: row == n - 1}
    v, fails = {}, []
    for k, (op, a, b, _) in enumerate(np.asarray(prog).tolist()):
        if op in (S.OP_LOCAL, S.OP_NEXT, S.OP_AUX_LOCAL, S.OP_AUX_NEXT):
            col = (trace if op in (S.OP_LOCAL, S.OP_NEXT) else aux)[a]
            v[k] = col if op in (S.OP_LOCAL, S.OP_AUX_LOCAL) else np.roll(col, -1)
        elif op == S.OP_CONST:
            v[k] = np.full(n, consts[a], dtype=np.uint64)
        elif op == S.OP_ADD:
            v[k] = G.add(v[a], v[b])
        elif op == S.OP_SUB:
            v[k] = G.sub(v[a], v[b])
        elif op == S.OP_MUL:
            v[k] = G.mul(v[a], v[b])
        else:
            fails.append((len(fails), (G.canon(v[a]) != 0) & on[b]))
    return _pairs(fails, lambda e: e)


def vp_expected(prog, values, consts, log_n):
    """gl_plonk_check_rows' failing (row, term number) pairs. values[c]: commitment c's (B, n) values on H."""
    n = 1 << log_n
    x = G.powers(np.uint64(E.primitive_root_of_unity(log_n)), n)
    l0 = np.zeros(n, dtype=np.uint64)
    l0[0] = 1
    r, fails = {}, []
    for op, dst, a, b in np.asarray(prog).tolist():
        if op == VP_LOCAL:
            v = values[a][b]
        elif op == VP_NEXT:
            v = np.roll(values[a][b], -1)
        elif op == VP_CONST:
            v = np.full(n, consts[a | b << 16], dtype=np.uint64)
        elif op == VP_X:
            v = x
        elif op == VP_L0:
            v = l0
        elif op == VP_ADD:
            v = G.add(r[a], r[b])
        elif op == VP_SUB:
            v = G.sub(r[a], r[b])
        elif op == VP_MUL:
            v = G.mul(r[a], r[b])
        elif op == VP_ADDC:
            v = G.add(r[a], np.uint64(consts[b]))
        elif op == VP_MULC:
            v = G.mul(r[a], np.uint64(consts[b]))
        else:
            fails.append((b, G.canon(r[a]) != 0))
            continue
        r[dst] = v
    return _pairs(fails, lambda t: t)


def _stark_prog(b):
    return np.array([(op, a, c, 0) for op, a, c in b.instrs], dtype=np.uint16).reshape(-1, 4)


def _vp_prog(arr):
    return np.frombuffer(bytes(arr), dtype=np.uint16).reshape(-1, 4)


def _twin(a):
    """Every word below 2^32 - 1 replaced by its non-canonical twin x + p: the reports must not change."""
    return np.where(a < np.uint64(2**32 - 1), a + np.uint64(P), a)


def _sparse(seed, shape, density=0.6):
    """Values of which about `density` of the rows are zero in every column: random programs then hold on some rows
    and fail on others (a constant still reaches a zero row; the evaluator decides)."""
    v = synth(seed, shape)
    rows = np.random.default_rng(seed).random(shape[-1]) < density
    v[..., rows] = 0
    return v


# ------------------------------------------------------------------------------------------------------ CPU
def test_binding_matches_the_header():
    """Both entry points of include/plonky2_b200_check.h are exported and bound with the header's parameter count;
    ConstraintError is a ValueError."""
    import re

    with open(os.path.join(ROOT, "include", "plonky2_b200_check.h")) as f:
        header = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    assert sorted(re.findall(r"\b(gl_[a-z0-9_]+)\s*\(", header)) == sorted(N.CHECK_EXPORTS)
    for name, nargs in (("gl_stark_check_rows", 11), ("gl_plonk_check_rows", 12)):
        assert name in N.CHECK_EXPORTS
        decl = re.search(r"int %s\(([^;]*)\);" % name, header).group(1)
        assert decl.count(",") + 1 == nargs
        assert len(getattr(N.lib(), name).argtypes) == nargs
    assert issubclass(N.ConstraintError, ValueError)


def test_refusals_without_a_device():
    """A NULL context is refused before anything else touches the device; max_report outside 0..65536 is refused by
    the binding."""
    L = N.lib()
    f, r = C.c_uint64(), C.c_uint32()
    assert L.gl_stark_check_rows(None, None, None, None, 1, None, 0, 0, C.byref(f), None, C.byref(r)) == N.GL_ERR_BAD_ARG
    assert L.gl_last_error(None) == b"null argument"
    assert L.gl_plonk_check_rows(None, None, 1, None, 1, None, 0, 1, 0, C.byref(f), None, C.byref(r)) == N.GL_ERR_BAD_ARG
    for bad in (-1, N.MAX_REPORT + 1):
        with pytest.raises(ValueError, match="max_report"):
            N.check_rows(L.gl_stark_check_rows, None, (), bad)


def test_constraint_error_messages(monkeypatch):
    """The provers' message: the reference's "Constraint failed in {Stark} at row {row}", the first label, the total."""
    from plonky2_b200 import plonk

    report = N.ConstraintReport(3, [(5, 1, "constraint 1 (transition)"), (5, 2, "constraint 2 (transition)")])
    monkeypatch.setattr(S, "check_constraints", lambda *a, **k: report)
    with pytest.raises(N.ConstraintError) as e:
        S._raise_on_failure(S.FibonacciStark(8), None, [0, 1, 2])
    assert str(e.value) == ("Constraint failed in FibonacciStark at row 5: constraint 1 (transition); 3 failing "
                            "(row, constraint) pairs in all")
    assert e.value.report is report
    monkeypatch.setattr(plonk, "check_constraints", lambda *a, **k: N.ConstraintReport(1, [(7, 9, "gate constraint 0 of X")]))
    with pytest.raises(N.ConstraintError, match="Constraint failed in the circuit at row 7: gate constraint 0 of X; 1 "):
        plonk._raise_on_failure(None)
    monkeypatch.setattr(S, "check_constraints", lambda *a, **k: N.ConstraintReport(0, []))
    S._raise_on_failure(S.FibonacciStark(8), None, [0, 1, 2])


def test_labels_cover_every_emit():
    """ConstraintBuilder labels every EMIT: the Stark's own constraints by number and kind, then each lookup's checks
    by lookup and challenge."""
    from test_stark_lookups import RangeCheckStark

    b = S.FibonacciStark(8).constraint_program()
    assert b.labels == ["constraint 0 (first row)", "constraint 1 (first row)", "constraint 2 (last row)",
                        "constraint 3 (transition)", "constraint 4 (transition)"]
    b = RangeCheckStark().constraint_program(2)
    assert len(b.labels) == sum(op == S.OP_EMIT for op, _, _ in b.instrs)
    assert b.labels[:3] == ["constraint 0 (every row)", "constraint 1 (every row)", "constraint 2 (first row)"]
    assert b.labels[3].startswith("lookup 0, challenge 0, check 0") and "lookup 1, challenge 1, check" in b.labels[-1]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("gl_check_emu") / "libgl_check_rows_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DGL_FORCE_32BIT_PATH", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "emu", "check_rows_emu.cpp")])
    L = C.CDLL(out)
    for f in (L.emu_stark_check_rows, L.emu_plonk_check_rows):
        f.restype = C.c_uint64
    return L


def _emu_run(fn, *args, n):
    """Both passes of a host row check: the per-row counts, then every pair, rows in order."""
    counts = np.zeros(n, dtype=np.uint32)
    total = fn(*args, counts.ctypes.data_as(N.u32p), None)
    pairs = np.zeros(2 * max(total, 1), dtype=np.uint32)
    assert fn(*args, counts.ctypes.data_as(N.u32p), pairs.ctypes.data_as(N.u32p)) == total == counts.sum()
    got = pairs[:2 * total].reshape(-1, 2).tolist()
    return sorted(map(tuple, got))    # a row's failures come in program order


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_stark_row_function_on_host(emu, seed):
    """512 instructions of every opcode and filter, auxiliary columns, on 2^6 rows of which some are zero."""
    log_n, n_cols, n_aux, n_consts = 6, 5, 3, 7
    prog = stark_program(0x7A0 + seed, STARK_MAX_INSTR, n_cols, n_consts, n_aux)
    trace, aux = _sparse(0x7B0 + seed, (n_cols, 1 << log_n)), _sparse(0x7C0 + seed, (n_aux, 1 << log_n))
    consts = synth(0x7D0 + seed, (n_consts,))
    consts[::2] = 0
    got = _emu_run(emu.emu_stark_check_rows, N.np_ptr(trace), N.np_ptr(aux), log_n, prog.ctypes.data_as(N.vp),
                   len(prog), N.np_ptr(consts), n=1 << log_n)
    want = stark_expected(prog, trace, aux, consts)
    assert 0 < len(want) < (1 << log_n) * (prog[:, 0] == S.OP_EMIT).sum()
    assert got == want


@pytest.mark.parametrize("seed", [1, 2])
def test_plonk_row_function_on_host(emu, seed):
    """256 registers, 4 commitments, constants past 65 535, repeated terms, on 2^5 rows of which some are zero."""
    log_n, widths, n_terms = 5, [3, 6, 2, 4], 300
    prog = vp_program(0x7E0 + seed, 1500, widths, VP_CONSTS, n_terms, salted=-1)
    values = [_sparse(0x7F0 + seed + 16 * c, (w, 1 << log_n)) for c, w in enumerate(widths)]
    consts = synth(0x800 + seed, (VP_CONSTS,))
    consts[::3] = 0
    ptrs = (N.vp * VP_MAX_COMMITS)(*[v.ctypes.data for v in values])
    got = _emu_run(emu.emu_plonk_check_rows, ptrs, len(values), log_n, prog.ctypes.data_as(N.vp), len(prog),
                   N.np_ptr(consts), n=1 << log_n)
    want = vp_expected(prog, values, consts, log_n)
    assert 0 < len(want)
    assert got == want


# ------------------------------------------------------------------------------------------------------ GPU
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


def _on_h(oracle, batch):
    return np.stack([oracle.fft(c) for c in batch.polynomials])


def _stark_device(ctx, tc, ac, prog, consts, max_report):
    return N.check_rows(N.lib().gl_stark_check_rows, ctx, (tc.h, ac.h if ac is not None else None,
                                                           prog.ctypes.data_as(N.vp), len(prog), N.np_ptr(consts),
                                                           len(consts)), max_report)


@pytest.mark.gpu
def test_stark_random_programs_and_truncation(pb, oracle):
    """512 instructions with auxiliary reads on 2^7 rows: the whole list (max_report 65536), a truncated one whose
    total exceeds it (the first pairs in order, the straddling row cut mid-row), max_report 0, and the same list from
    non-canonical constants."""
    ctx = pb.default_context()
    log_n, n_cols, n_aux, n_consts = 7, 5, 2, 6
    prog = stark_program(0x810, STARK_MAX_INSTR, n_cols, n_consts, n_aux)
    tv, av = _sparse(0x811, (n_cols, 1 << log_n)), _sparse(0x812, (n_aux, 1 << log_n))
    consts = synth(0x813, (n_consts,))
    consts[::2] = 0
    tc, ac = pb.PolynomialBatch.from_values(tv, 1, False, 2), pb.PolynomialBatch.from_values(av, 1, False, 2)
    try:
        want = stark_expected(prog, tv, av, consts)
        assert len(want) > 100
        total, got = _stark_device(ctx, tc, ac, prog, consts, N.MAX_REPORT)
        assert total == len(want) and got == want
        for k in (1, 7, len(want) // 2 + 3):
            total, got = _stark_device(ctx, tc, ac, prog, consts, k)
            assert total == len(want) and got == want[:k]
        assert _stark_device(ctx, tc, ac, prog, _twin(consts), N.MAX_REPORT) == (len(want), want)
        assert _stark_device(ctx, tc, ac, prog, consts, 0) == (len(want), [])
    finally:
        tc.close(), ac.close()


@pytest.mark.gpu
@pytest.mark.parametrize("host", ["pinned", "pageable"])
def test_host_inputs_are_read_before_returning(pb, host):
    """The program and constants of both checks in a page-locked (or pageable) buffer that is overwritten the moment
    the call returns, with the library's stream held behind 0.2 s of spinning: the reports are the evaluator's for the
    original inputs (both calls end in a synchronising read-back)."""
    from test_gpu_host_buffers import _hold, _host_buffer, _overwrite

    ctx = pb.default_context()
    log_n, n_cols, n_consts = 6, 4, 5
    prog = stark_program(0x860, 200, n_cols, n_consts)
    tv = _sparse(0x861, (n_cols, 1 << log_n))
    consts = synth(0x862, (n_consts,))
    want = stark_expected(prog, tv, None, consts)
    tc = pb.PolynomialBatch.from_values(tv, 1, False, 2)
    try:
        pbuf, cbuf = _host_buffer(prog.view(np.uint64), host), _host_buffer(consts, host)
        _hold(ctx)
        got = N.check_rows(N.lib().gl_stark_check_rows, ctx, (tc.h, None, N.np_ptr(pbuf), len(prog), N.np_ptr(cbuf),
                                                               n_consts), N.MAX_REPORT)
        _overwrite(pbuf, cbuf)
        assert got == (len(want), want)
        vprog = vp_program(0x863, 400, [n_cols], VP_CONSTS, 50, salted=-1)
        vconsts = synth(0x864, (VP_CONSTS,))
        vwant = vp_expected(vprog, [tv], vconsts, log_n)
        pbuf, cbuf = _host_buffer(vprog.view(np.uint64), host), _host_buffer(vconsts, host)
        handles = (N.vp * 1)(tc.h)
        _hold(ctx)
        got = N.check_rows(N.lib().gl_plonk_check_rows, ctx, (handles, 1, N.np_ptr(pbuf), len(vprog), N.np_ptr(cbuf),
                                                              VP_CONSTS, 50), N.MAX_REPORT)
        _overwrite(pbuf, cbuf)
        assert got == (len(vwant), vwant)
    finally:
        tc.close()


@pytest.mark.gpu
def test_stark_handle_kinds_agree(pb, oracle):
    """Resident, non-resident (4 LDE blocks) and 2-shard handles give the same report; so does a degree-0 program."""
    ctx = pb.default_context()
    log_n, n_cols, n_aux, n_consts = 8, 4, 2, 5
    prog = stark_program(0x820, 300, n_cols, n_consts, n_aux)
    tv, av = _sparse(0x821, (n_cols, 1 << log_n)), _sparse(0x822, (n_aux, 1 << log_n))
    consts = synth(0x823, (n_consts,))
    want = stark_expected(prog, tv, av, consts)
    for kw in ({}, dict(lde_blocks=4), dict(shard=(0, 2)), dict(shard=(1, 2))):
        tc, ac = (pb.PolynomialBatch.from_values(v, 2, False, 2, **kw) for v in (tv, av))
        try:
            assert _stark_device(ctx, tc, ac, prog, consts, 500) == (len(want), want[:500]), kw
        finally:
            tc.close(), ac.close()


@pytest.mark.gpu
def test_plonk_random_programs_salted_and_truncated(pb, oracle):
    """256 registers, 4 commitments (one salted: LOCAL / NEXT are bounded by B), constants past 65 535, on 2^6 rows;
    truncated, max_report 0, and from non-canonical constants."""
    ctx = pb.default_context()
    log_n, widths, n_terms = 6, [3, 6, 2, 4], 4000
    prog = vp_program(0x830, 3000, widths, VP_CONSTS, n_terms, salted=-1)
    values = [_sparse(0x831 + c, (w, 1 << log_n)) for c, w in enumerate(widths)]
    consts = synth(0x835, (VP_CONSTS,))
    consts[::3] = 0
    batches = [pb.PolynomialBatch.from_values(v, 1, c == 1, 2) for c, v in enumerate(values)]
    assert N.lib().gl_commit_leaf_width(batches[1].h) == widths[1] + SALT
    try:
        want = vp_expected(prog, values, consts, log_n)
        handles = (N.vp * 4)(*[b.h for b in batches])

        def run(k):
            return N.check_rows(N.lib().gl_plonk_check_rows, ctx, (handles, 4, prog.ctypes.data_as(N.vp), len(prog),
                                                                   N.np_ptr(consts), len(consts), n_terms), k)
        assert run(N.MAX_REPORT) == (len(want), want)
        assert run(5) == (len(want), want[:5])
        consts[:] = _twin(consts)
        assert run(N.MAX_REPORT) == (len(want), want)
        assert run(0) == (len(want), [])
    finally:
        for b in batches:
            b.close()


@pytest.mark.gpu
def test_refusals_before_any_launch(pb):
    """NULL arguments, an unfinished handle, different degrees, another context, max_report > 65536, and the quotient's
    program errors with its messages; nothing is launched."""
    ctx = pb.default_context()
    L = N.lib()
    a = pb.PolynomialBatch.from_values(synth(0x840, (2, 16)), 1, False, 1)
    b = pb.PolynomialBatch.from_values(synth(0x841, (2, 32)), 1, False, 1)
    other = pb.Context(0)
    c = pb.PolynomialBatch.from_values(synth(0x842, (2, 16)), 1, False, 1, ctx=other)
    unfinished = N.vp()
    N.check(L.gl_commit_begin(ctx.h, 2, 4, 1, 1, 0, 0, 1, None, C.byref(unfinished)), ctx.h)
    prog = np.array([(S.OP_LOCAL, 0, 0, 0), (S.OP_EMIT, 0, 0, 0)], dtype=np.uint16)
    f, r, pairs = C.c_uint64(), C.c_uint32(), np.zeros(2, dtype=np.uint32)
    u32 = pairs.ctypes.data_as(N.u32p)

    def call(trace, aux, p=prog, max_report=1, out=u32, n_instr=None):
        rc = L.gl_stark_check_rows(ctx.h, trace, aux, p.ctypes.data_as(N.vp), len(p) if n_instr is None else n_instr,
                                   None, 0, max_report, C.byref(f), out, C.byref(r))
        return rc, L.gl_last_error(ctx.h).decode()
    try:
        before = ctx.launch_count
        assert call(a.h, None, out=None) == (N.GL_ERR_BAD_ARG, "null argument")
        assert call(None, None) == (N.GL_ERR_BAD_ARG, "null argument")
        assert call(unfinished, None) == (N.GL_ERR_BAD_ARG,
                                          "gl_commit_finish has not been called on the trace commitment")
        assert call(a.h, b.h)[0] == N.GL_ERR_BAD_SHAPE
        assert call(a.h, c.h) == (N.GL_ERR_BAD_ARG, "the auxiliary commitment belongs to another context")
        assert call(a.h, None, max_report=N.MAX_REPORT + 1) == (N.GL_ERR_BAD_ARG, "max_report 65537 > 65536")
        assert call(a.h, None, n_instr=STARK_MAX_INSTR + 1)[0] == N.GL_ERR_UNSUPPORTED
        bad = np.array([(S.OP_LOCAL, 2, 0, 0), (S.OP_EMIT, 0, 0, 0)], dtype=np.uint16)   # column 2 of 2
        assert call(a.h, None, p=bad) == (N.GL_ERR_BAD_ARG, "constraint program: bad instruction 0")
        aux_read = np.array([(S.OP_AUX_LOCAL, 0, 0, 0), (S.OP_EMIT, 0, 0, 0)], dtype=np.uint16)
        assert call(a.h, None, p=aux_read) == (N.GL_ERR_BAD_ARG, "constraint program: bad instruction 0")
        vp = np.array([(VP_LOCAL, 0, 0, 2), (VP_TERM, 0, 0, 0)], dtype=np.uint16)   # column 2 of 2
        for handles, want in (([a.h, b.h], N.GL_ERR_BAD_SHAPE), ([a.h, c.h], N.GL_ERR_BAD_ARG),
                              ([a.h, unfinished], N.GL_ERR_BAD_ARG), ([a.h], N.GL_ERR_BAD_ARG)):
            hs = (N.vp * len(handles))(*handles)
            rc = L.gl_plonk_check_rows(ctx.h, hs, len(handles), vp.ctypes.data_as(N.vp), 2, None, 0, 1, 1, C.byref(f),
                                       u32, C.byref(r))
            assert rc == want
        assert L.gl_last_error(ctx.h).decode() == "vanishing program: bad instruction 0"
        assert ctx.launch_count == before
    finally:
        for x in (a, b, c):
            x.close()
        L.gl_commit_destroy(unfinished)


# ---- real STARKs through the provers, every check recorded against the evaluator
def _record_stark_checks(monkeypatch, oracle):
    """Wrap stark.check_constraints: every check a prover runs is recorded with its whole report and the evaluator's
    pairs, and still decides whether the prover raises."""
    real, log = S.check_constraints, []

    def rec(stark, trace_commitment, public_inputs, auxiliary_polys_commitment=None, lookup_challenges=None,
            ctl_vars=None, max_report=64):
        report = real(stark, trace_commitment, public_inputs, auxiliary_polys_commitment, lookup_challenges, ctl_vars,
                      max_report=N.MAX_REPORT)
        b, consts, _ = S.quotient_program(stark, public_inputs, [], auxiliary_polys_commitment, lookup_challenges,
                                          ctl_vars)
        aux = _on_h(oracle, auxiliary_polys_commitment) if auxiliary_polys_commitment is not None else None
        log.append((type(stark).__name__, report, stark_expected(_stark_prog(b), _on_h(oracle, trace_commitment), aux,
                                                                 consts)))
        return report
    monkeypatch.setattr(S, "check_constraints", rec)
    return log


def _assert_log(log):
    for name, report, want in log:
        assert report.failures == len(want), name
        assert [(r, e) for r, e, _ in report.entries] == want, name


def _stark_cases():
    from test_stark_lookups import PermutationStark, RangeCheckStark, RangeCheckStark4

    fib = S.FibonacciStark(1 << 8)
    rc, rc4, perm = RangeCheckStark(), RangeCheckStark4(), PermutationStark(1 << 7)
    fib_trace = fib.generate_trace(0, 1)
    return {     # (stark, trace, public inputs); RangeCheckStark's TABLE starts at 0
        "fibonacci": (fib, fib_trace, [0, 1, int(fib_trace[1, -1])]),
        "range_check": (rc, RangeCheckStark.generate_trace(8), [0]),
        "range_check4": (rc4, RangeCheckStark.generate_trace(8, count_combination=False), [0]),
        "permutation": (perm, perm.generate_trace(3), [3]),
    }


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fibonacci", "range_check", "range_check4", "permutation"])
def test_holding_starks_report_nothing_and_prove_the_same(pb, oracle, monkeypatch, name):
    """FibonacciStark, RangeCheckStark(4) (lookups) and PermutationStark (degree 0, no quotient): 0 failures, and the
    proof with check_constraints=True equals the proof without, field for field."""
    from test_stark_lookups import T_config_rate2

    stark, trace, pis = _stark_cases()[name]
    config = T_config_rate2() if name == "range_check4" else S.StarkConfig.standard_fast_config()
    log = _record_stark_checks(monkeypatch, oracle)
    checked = S.prove(stark, config, trace, pis, check_constraints=True)
    assert len(log) == 1 and log[0][1].failures == 0
    _assert_log(log)
    assert not T.proof_diff(checked, S.prove(stark, config, trace, pis))
    assert len(log) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [(0,), (1,), (-1,), (0, 1, -1)])
def test_fibonacci_cells_changed_at_the_edges(pb, oracle, monkeypatch, rows):
    """One cell changed at rows 0, 1, n - 1 (and all three): the first-row, transition and last-row filters at the
    edges; the transition out of row n - 1 (which wraps to row 0) is never checked."""
    stark = S.FibonacciStark(1 << 6)
    trace = stark.generate_trace(0, 1)
    pis = [0, 1, int(trace[1, -1])]
    for r in rows:
        trace[1, r] = (int(trace[1, r]) + 1) % P
    log = _record_stark_checks(monkeypatch, oracle)
    with pytest.raises(N.ConstraintError) as e:
        S.prove(stark, S.StarkConfig.standard_fast_config(), trace, pis, check_constraints=True)
    _assert_log(log)
    first_row, _, first_label = log[0][1].entries[0]
    assert str(e.value).startswith("Constraint failed in FibonacciStark at row %d: %s; " % (first_row, first_label))
    got = {(r, e) for r, e, _ in log[0][1].entries}
    n = 1 << 6
    if rows == (0,):          # x1 at row 0: its first-row constraint, and both transitions out of row 0
        assert got == {(0, 1), (0, 3), (0, 4)}
    if rows == (-1,):         # x1 at row n - 1: the last-row constraint and the transitions into it, none out of it
        assert got == {(n - 2, 4), (n - 1, 2)}


@pytest.mark.gpu
def test_broken_lookup_multiplicity(pb, oracle, monkeypatch):
    """RangeCheckStark with one frequency off by one: the lookup's Z check fails and the label names the lookup."""
    from test_stark_lookups import MA, RangeCheckStark

    trace = RangeCheckStark.generate_trace(7)
    trace[MA, 5] += np.uint64(1)
    log = _record_stark_checks(monkeypatch, oracle)
    with pytest.raises(N.ConstraintError, match="Constraint failed in RangeCheckStark at row") as e:
        S.prove(RangeCheckStark(), S.StarkConfig.standard_fast_config(), trace, [int(trace[7, 0])],
                check_constraints=True)
    _assert_log(log)
    assert all(label.startswith("lookup 0, challenge") for _, _, label in e.value.report.entries)


@pytest.mark.gpu
def test_ctl_system_holds_and_a_broken_value_is_named(pb, oracle, monkeypatch):
    """Every table of the CTL system of test_stark_ctl.py reports 0 failures and proves the same with the flag; one
    value of the looked table's last CTL Z column changed breaks its transitions into and out of that row, and the
    labels name the CTL Z."""
    from plonky2_b200 import cross_table_lookup as X
    from test_stark_ctl import system, system_traces

    starks, config, ctls = system()
    traces, pis = system_traces()
    log = _record_stark_checks(monkeypatch, oracle)
    checked = X.prove_with_ctls(starks, config, traces, ctls, pis, check_constraints=True)
    assert [name for name, _, _ in log] == ["CpuTable", "MemTable", "LookedTable"]
    assert all(r.failures == 0 for _, r, _ in log)
    _assert_log(log)
    plain = X.prove_with_ctls(starks, config, traces, ctls, pis)
    assert not T.proof_diff(checked, plain)
    log.clear()
    real = X.cross_table_lookup_data

    def broken(*a, **k):                              # the looked table's last CTL Z, one value changed at row 5
        data = real(*a, **k)
        data[2].auxiliary[-1, 5] = 12345
        return data
    monkeypatch.setattr(X, "cross_table_lookup_data", broken)
    with pytest.raises(N.ConstraintError, match="Constraint failed in LookedTable at row 4: CTL Z") as e:
        X.prove_with_ctls(starks, config, traces, ctls, pis, check_constraints=True)
    _assert_log(log)
    assert {r for r, _, _ in e.value.report.entries} == {4, 5}
    assert all("CTL Z" in label for _, _, label in e.value.report.entries)


@pytest.mark.gpu
def test_alpha_combination_fails_exactly_on_the_reported_rows(pb, oracle):
    """The reference's semantics: the rows where the alpha-combined ConstraintConsumer accumulator is nonzero are the
    rows with a reported failure (random 512-instruction program, aux reads, random alphas)."""
    ctx = pb.default_context()
    log_n, n_cols, n_aux, n_consts = 7, 4, 2, 5
    prog = stark_program(0x850, STARK_MAX_INSTR, n_cols, n_consts, n_aux)
    tv, av = _sparse(0x851, (n_cols, 1 << log_n), 0.8), _sparse(0x852, (n_aux, 1 << log_n), 0.8)
    consts = synth(0x853, (n_consts,))
    consts[:] = 0
    n = 1 << log_n
    row = np.arange(n)
    w = E.primitive_root_of_unity(log_n)
    x = G.powers(np.uint64(w), n)
    sel = {S.KIND_CONSTRAINT: np.ones(n, dtype=np.uint64), S.KIND_TRANSITION: G.sub(x, np.uint64(pow(w, P - 2, P))),
           S.KIND_FIRST_ROW: (row == 0).astype(np.uint64), S.KIND_LAST_ROW: (row == n - 1).astype(np.uint64)}
    acc = np.zeros(n, dtype=np.uint64)
    alpha = np.uint64(int(synth(0x854, (1,))[0]))
    v = {}
    for k, (op, a, b, _) in enumerate(prog.tolist()):
        if op in (S.OP_LOCAL, S.OP_NEXT, S.OP_AUX_LOCAL, S.OP_AUX_NEXT):
            col = (tv if op in (S.OP_LOCAL, S.OP_NEXT) else av)[a]
            v[k] = col if op in (S.OP_LOCAL, S.OP_AUX_LOCAL) else np.roll(col, -1)
        elif op == S.OP_CONST:
            v[k] = np.full(n, consts[a], dtype=np.uint64)
        elif op in (S.OP_ADD, S.OP_SUB, S.OP_MUL):
            v[k] = {S.OP_ADD: G.add, S.OP_SUB: G.sub, S.OP_MUL: G.mul}[op](v[a], v[b])
        else:
            acc = G.add(G.mul(acc, alpha), G.mul(v[a], sel[b]))
    tc, ac = pb.PolynomialBatch.from_values(tv, 1, False, 2), pb.PolynomialBatch.from_values(av, 1, False, 2)
    try:
        total, pairs = _stark_device(ctx, tc, ac, prog, consts, N.MAX_REPORT)
    finally:
        tc.close(), ac.close()
    assert total == len(pairs) > 0
    assert {r for r, _ in pairs} == set(np.nonzero(G.canon(acc))[0].tolist())
    assert len({r for r, _ in pairs}) < n


# ---- plonky2
def _record_plonk_checks(monkeypatch, oracle):
    from plonky2_b200 import plonk

    real, log = plonk.check_constraints, []

    def rec(cd, cs, pih, w, z, betas, gammas, deltas=(), max_report=64):
        report = real(cd, cs, pih, w, z, betas, gammas, deltas, max_report=N.MAX_REPORT)
        prog, consts, _ = plonk.quotient_program(cd, [cs, w, z], pih, betas, gammas, betas, deltas)
        values = [_on_h(oracle, c) for c in (cs, w, z)]
        log.append((report, vp_expected(_vp_prog(prog), values, consts, cd.degree_bits)))
        return report
    monkeypatch.setattr(plonk, "check_constraints", rec)
    return log


def _prove_circuit(pb, c, digest, wires=None, check=False, salt_keys=None):
    from plonky2_b200 import plonk
    from plonky2_b200.fri import standard_recursion_fri_config

    cfg, cd = c.config, c.common
    fri_params = standard_recursion_fri_config().fri_params(cd.degree_bits, cfg.zero_knowledge)
    cs = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height)
    try:
        prover_data = plonk.ProverOnlyCircuitData(cs, c.sigmas, digest, fri_params)
        kw = dict(salt_keys=salt_keys) if salt_keys else {}
        return plonk.prove_with_witness(prover_data, cd, c.wires if wires is None else wires, c.public_inputs,
                                        check_constraints=check, **kw).to_bytes()
    finally:
        cs.close()


DIGEST = [int(x) for x in synth(0x6190, (4,))]


@pytest.mark.gpu
@pytest.mark.parametrize("zk", [False, True])
def test_holding_circuit_reports_nothing_and_proves_the_same(pb, oracle, monkeypatch, zk):
    """LargeCircuit at 2^13 gates with lookups (and with zero knowledge: salted commitments): 0 failures, and the proof
    with check_constraints=True is byte for byte the proof without."""
    import plonk_large as PL

    c = PL.large_circuit(13, public_inputs=[3, 1, 4])
    c.config.zero_knowledge = zk                      # salted wires, Z and quotient commitments; the witness holds
    log = _record_plonk_checks(monkeypatch, oracle)
    keys = [bytes([k]) * 32 for k in (1, 2, 3)] if zk else None
    checked = _prove_circuit(pb, c, DIGEST, check=True, salt_keys=keys)
    assert len(log) == 1 and log[0][0].failures == 0 and log[0][1] == []
    assert checked == _prove_circuit(pb, c, DIGEST, salt_keys=keys)


@pytest.mark.gpu
def test_bad_witness_at_qdf_8_now_raises(pb, oracle, monkeypatch):
    """The qdf-8 circuit of test_a_bad_witness_past_row_4096_is_rejected (no quotient tail to check): the flag raises
    ConstraintError at c.broken_row, naming the arithmetic gate's constraint."""
    import plonk_large as PL

    c = PL.large_circuit(13, qdf=8, break_arith=5000, public_inputs=[3, 1, 4, 1, 5, 9, 2, 6])
    log = _record_plonk_checks(monkeypatch, oracle)
    with pytest.raises(N.ConstraintError, match="at row %d: gate constraint \\d+ of ArithmeticGate" % c.broken_row) as e:
        _prove_circuit(pb, c, DIGEST, check=True)
    report, want = log[0]
    assert [(r, t) for r, t, _ in report.entries] == want and report.failures == len(want)
    assert {r for r, _, _ in e.value.report.entries if r != c.n - 1} == {c.broken_row}


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["copy", "lookup"])
def test_broken_copy_constraint_and_looking_pair(pb, oracle, monkeypatch, what):
    """A wire of a copy cycle changed: the last partial-product check fails at row n - 1 and says so. A looking pair
    changed to one not in its table: a lookup term fails. Both as exact sets against the evaluator."""
    import plonk_large as PL

    c = PL.large_circuit(10, public_inputs=[2, 7])
    wires = c.wires.copy()
    if what == "copy":
        (row, col) = c.partition()[1][2]
        wires[col, row] = (int(wires[col, row]) + 1) % P
    else:
        last_lu = c.lookup_rows[0][0]
        wires[1, last_lu] = (int(wires[1, last_lu]) + 12345) % P
    log = _record_plonk_checks(monkeypatch, oracle)
    with pytest.raises(N.ConstraintError) as e:
        _prove_circuit(pb, c, DIGEST, wires=wires, check=True)
    report, want = log[-1]
    assert [(r, t) for r, t, _ in report.entries] == want and report.failures == len(want)
    labels = [label for _, _, label in report.entries]
    if what == "copy":
        assert any(r == c.n - 1 and "copy constraint" in label for r, _, label in report.entries)
    else:
        assert any(label.startswith("lookup term") for label in labels)
