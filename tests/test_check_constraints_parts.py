"""check_constraints in parts of H: gl_stark_check_rows_part / gl_plonk_check_rows_part (k_stark_check_rows /
k_plonk_check_rows with part addressing), _native.merge_reports, the parts= and placement= of stark.check_constraints /
plonk.check_constraints, and the provers' check_constraints=True on non-resident (lde_blocks=G) and distributed proofs.

Part g of G is the rows i = g (mod G). Every part's report is compared, as the exact list of (row, index) pairs, with
the whole-H evaluators of tests/test_check_constraints.py restricted to those rows; the merged parts with the whole
check (gl_*_check_rows), truncation included.

CPU: the binding, the NULL-context refusals, the parts= refusal, merge_reports against the sorted whole on random
per-part reports, and the host build of both row functions with part addressing (tests/emu/check_rows_parts_emu.cpp)
on part values folded and evaluated in numpy from the coefficients, every part of G = 1 ... 16 and G = n.
GPU (-m gpu): every part of G = 1 ... 16 on every handle kind, the (0, 1) call against the whole check, refusals,
page-locked and non-canonical host inputs, the scratch high-water mark, and the provers with lde_blocks=G. torchrun
(tests/mgpu_check_constraints_check.py): the three distributed provers with check_constraints=True."""
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
from ranks import run_ranks
from test_check_constraints import _sparse, _stark_cases, _twin, stark_expected, vp_expected
from test_gpu_programs import STARK_MAX_INSTR, VP_CONSTS, VP_MAX_COMMITS, stark_program, vp_program

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PARTS = [1, 2, 4, 8, 16]


def _restrict(pairs, g, parts):
    return [(r, i) for r, i in pairs if r % parts == g]


# ------------------------------------------------------------------------------------------------------ CPU
def test_binding_matches_the_header():
    """Both _part entry points are declared in include/plonky2_b200_check.h, exported and bound with 13 and 14
    parameters: their counterparts' plus (part, parts) before max_report."""
    import re

    with open(os.path.join(ROOT, "include", "plonky2_b200_check.h")) as f:
        header = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    for name, nargs in (("gl_stark_check_rows_part", 13), ("gl_plonk_check_rows_part", 14)):
        assert name in N.CHECK_EXPORTS
        decl = re.search(r"int %s\(([^;]*)\);" % name, header).group(1)
        assert decl.count(",") + 1 == nargs
        assert "uint32_t part, uint32_t parts, uint32_t max_report" in " ".join(decl.split())
        assert len(getattr(N.lib(), name).argtypes) == nargs


def test_null_context_refusals():
    L = N.lib()
    f, r = C.c_uint64(), C.c_uint32()
    assert L.gl_stark_check_rows_part(None, None, None, None, 1, None, 0, 0, 1, 0, C.byref(f), None,
                                      C.byref(r)) == N.GL_ERR_BAD_ARG
    assert L.gl_last_error(None) == b"null argument"
    assert L.gl_plonk_check_rows_part(None, None, 1, None, 1, None, 0, 1, 0, 1, 0, C.byref(f), None,
                                      C.byref(r)) == N.GL_ERR_BAD_ARG
    assert L.gl_last_error(None) == b"null argument"


@pytest.mark.parametrize("parts", [0, -2, 3, 6, 12, 2.0, "4"])
def test_parts_must_be_a_positive_power_of_two(parts):
    """Refused by both check_constraints before anything reads the commitments."""
    from plonky2_b200 import plonk

    with pytest.raises(N.ShapeError, match="not a positive power of two"):
        S.check_constraints(S.FibonacciStark(8), None, [0, 1, 2], parts=parts)
    with pytest.raises(N.ShapeError, match="not a positive power of two"):
        plonk.check_constraints(None, None, None, None, None, [], [], parts=parts)
    with pytest.raises(N.ShapeError):
        N.check_parts(parts)


@pytest.mark.parametrize("seed", range(6))
def test_merge_reports_is_the_sorted_whole(seed):
    """Random failing pairs over 64 rows, split into the parts of G = 1 ... 32 and each part truncated to max_report
    as a part's check truncates it: the merge is the whole list's first max_report, for max_report 0, 1, one that cuts
    inside a row whose pairs straddle it, and one above the total; parts without failures are included."""
    rng = np.random.default_rng(0xC40 + seed)
    n = 64
    rows = rng.choice(n, size=12 + seed, replace=False)       # most rows hold: empty parts at large G
    whole = sorted({(int(r), int(i)) for r in rows for i in rng.choice(40, size=rng.integers(1, 6), replace=False)})
    straddle = next(k for k in range(1, len(whole)) if whole[k][0] == whole[k - 1][0])
    for parts in (1, 2, 4, 8, 16, 32):
        for max_report in (0, 1, straddle, len(whole) // 2, len(whole) + 5):
            reports = []
            for g in range(parts):
                mine = _restrict(whole, g, parts)
                reports.append((len(mine), mine[:max_report]))
            order = rng.permutation(parts)                     # the merge does not depend on the parts' order
            got = N.merge_reports([reports[k] for k in order], max_report)
            assert got == (len(whole), whole[:max_report]), (parts, max_report)
    assert N.merge_reports([], 5) == (0, [])
    assert N.merge_reports([(0, []), (0, [])], 0) == (0, [])


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("gl_check_parts_emu") / "libgl_check_rows_parts_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DGL_FORCE_32BIT_PATH", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "emu", "check_rows_parts_emu.cpp")])
    L = C.CDLL(out)
    for f in (L.emu_stark_check_rows_part, L.emu_plonk_check_rows_part):
        f.restype = C.c_uint64
    return L


def _coeffs(values):
    """Each row of `values` (a polynomial's values on H, natural order) interpolated: its coefficients, by the exact
    O(n^2) inverse DFT."""
    n = values.shape[-1]
    log_n = n.bit_length() - 1
    winv = pow(E.primitive_root_of_unity(log_n), P - 2, P)
    ninv = np.uint64(pow(n, P - 2, P))
    out = np.zeros_like(values)
    for k in range(n):
        xk = G.powers(np.uint64(pow(winv, k, P)), n)          # w^-jk over j
        acc = np.zeros(values.shape[0], dtype=np.uint64)
        for j in range(n):
            acc = G.add(acc, G.mul(values[:, j], np.uint64(int(xk[j]))))
        out[:, k] = G.mul(acc, ninv)
    return out


def _values_on_part(coeffs, e, parts):
    """The polynomials' values at w_n^e w_M^j, j < M = n / parts, from their coefficients as the device computes them:
    folded mod X^M - w_n^(e M), then evaluated at the M points (Horner)."""
    n = coeffs.shape[-1]
    log_n, M = n.bit_length() - 1, n // parts
    shift = pow(E.primitive_root_of_unity(log_n), e, P)
    sM = np.uint64(pow(shift, M, P))
    folded = np.zeros((coeffs.shape[0], M), dtype=np.uint64)
    for k1 in reversed(range(parts)):
        folded = G.add(G.mul(folded, sM), coeffs[:, k1 * M:(k1 + 1) * M])
    x = G.mul(G.powers(np.uint64(E.primitive_root_of_unity(log_n - (parts.bit_length() - 1))), M), np.uint64(shift))
    out = np.zeros((coeffs.shape[0], M), dtype=np.uint64)
    for k in reversed(range(M)):
        out = G.add(G.mul(out, x[None, :]), folded[:, k:k + 1])
    return np.ascontiguousarray(G.canon(out))


def _emu_part(fn, *args, rows):
    counts = np.zeros(rows, dtype=np.uint32)
    total = fn(*args, counts.ctypes.data_as(N.u32p), None)
    pairs = np.zeros(2 * max(total, 1), dtype=np.uint32)
    assert fn(*args, counts.ctypes.data_as(N.u32p), pairs.ctypes.data_as(N.u32p)) == total == counts.sum()
    got = [tuple(p) for p in pairs[:2 * total].reshape(-1, 2).tolist()]
    rows = [r for r, _ in got]
    assert rows == sorted(rows)                                 # global rows in order
    return sorted(got)                                          # a row's failures come in program order


@pytest.mark.parametrize("seed", [1, 2])
def test_stark_row_function_on_parts(emu, seed):
    """512 instructions of every opcode and filter with auxiliary reads on 2^6 rows: every part of G = 1, 2, 4, 8, 16
    and 64 (one row per part) gives the whole-H evaluator's pairs on its rows, and their union is the whole list."""
    log_n, n_cols, n_aux, n_consts = 6, 5, 3, 7
    n = 1 << log_n
    prog = stark_program(0xC10 + seed, STARK_MAX_INSTR, n_cols, n_consts, n_aux)
    trace, aux = _sparse(0xC20 + seed, (n_cols, n)), _sparse(0xC30 + seed, (n_aux, n))
    consts = synth(0xC50 + seed, (n_consts,))
    consts[::2] = 0
    want = stark_expected(prog, trace, aux, consts)
    assert 0 < len(want)
    tco, aco = _coeffs(trace), _coeffs(aux)
    for parts in PARTS + [n]:
        s = parts.bit_length() - 1
        union = []
        for g in range(parts):
            tl, al = _values_on_part(tco, g, parts), _values_on_part(aco, g, parts)
            tn = _values_on_part(tco, g + 1, parts) if parts > 1 else None
            an = _values_on_part(aco, g + 1, parts) if parts > 1 else None
            got = _emu_part(emu.emu_stark_check_rows_part, N.np_ptr(tl), tn.ctypes.data_as(N.vp) if tn is not None
                            else None, N.np_ptr(al), an.ctypes.data_as(N.vp) if an is not None else None, log_n, g, s,
                            prog.ctypes.data_as(N.vp), len(prog), N.np_ptr(consts), rows=n // parts)
            assert got == _restrict(want, g, parts), (parts, g)
            union += got
        assert sorted(union) == want, parts


@pytest.mark.parametrize("seed", [1, 2])
def test_plonk_row_function_on_parts(emu, seed):
    """256 registers, 4 commitments, constants past 65 535, X and L_0 at the global row, on 2^5 rows: every part of
    G = 1, 2, 4, 8, 16 and 32 against the whole-H evaluator, and their union is the whole list."""
    log_n, widths, n_terms = 5, [3, 6, 2, 4], 300
    n = 1 << log_n
    prog = vp_program(0xC60 + seed, 1500, widths, VP_CONSTS, n_terms, salted=-1)
    values = [_sparse(0xC70 + seed + 16 * c, (w, n)) for c, w in enumerate(widths)]
    consts = synth(0xC90 + seed, (VP_CONSTS,))
    consts[::3] = 0
    want = vp_expected(prog, values, consts, log_n)
    assert 0 < len(want)
    coeffs = [_coeffs(v) for v in values]
    for parts in PARTS + [n]:
        s = parts.bit_length() - 1
        union = []
        for g in range(parts):
            loc = [_values_on_part(c, g, parts) for c in coeffs]
            nxt = [_values_on_part(c, g + 1, parts) for c in coeffs] if parts > 1 else None
            lp = (N.vp * VP_MAX_COMMITS)(*[v.ctypes.data for v in loc])
            np_ = (N.vp * VP_MAX_COMMITS)(*[v.ctypes.data for v in nxt]) if nxt else None
            got = _emu_part(emu.emu_plonk_check_rows_part, lp, np_, len(loc), log_n, g, s, prog.ctypes.data_as(N.vp),
                            len(prog), N.np_ptr(consts), rows=n // parts)
            assert got == _restrict(want, g, parts), (parts, g)
            union += got
        assert sorted(union) == want, parts


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


def _stark_args(tc, ac, prog, consts):
    return (tc.h, ac.h if ac is not None else None, prog.ctypes.data_as(N.vp), len(prog), N.np_ptr(consts),
            len(consts))


def _check_all_parts(ctx, whole_fn, part_fn, args, want, parts_list):
    """Every part of every G: the restricted evaluator word for word; the merged parts equal the whole check at every
    truncation; the (0, 1) call equals the whole check bit for bit."""
    def whole(k):
        return N.check_rows(whole_fn, ctx, args, k)

    def part(g, parts, k):
        return N.check_rows(part_fn, ctx, args + (g, parts), k)
    cuts = (0, 1, 7, len(want) // 2 + 3, N.MAX_REPORT)
    for k in cuts:
        assert whole(k) == (len(want), want[:k]) == part(0, 1, k), k
    for parts in parts_list:
        for g in range(parts):
            mine = _restrict(want, g, parts)
            assert part(g, parts, N.MAX_REPORT) == (len(mine), mine), (parts, g)
        for k in cuts[:-1]:
            assert N.merge_reports([part(g, parts, k) for g in range(parts)], k) == whole(k), (parts, k)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["resident", "blocked", "shard0", "shard1"])
def test_stark_parts_on_every_handle_kind(pb, kind):
    """512 instructions with auxiliary reads on 2^7 rows, on resident, non-resident (4 LDE blocks) and both 2-shard
    handles: every part of G = 1 ... 16 (and 128, one row each) and every merge, from canonical and non-canonical
    constants."""
    ctx = pb.default_context()
    log_n, n_cols, n_aux, n_consts = 7, 5, 2, 6
    prog = stark_program(0xCA0, STARK_MAX_INSTR, n_cols, n_consts, n_aux)
    tv, av = _sparse(0xCA1, (n_cols, 1 << log_n)), _sparse(0xCA2, (n_aux, 1 << log_n))
    consts = synth(0xCA3, (n_consts,))
    consts[::2] = 0
    want = stark_expected(prog, tv, av, consts)
    assert len(want) > 100
    kw = {"resident": {}, "blocked": dict(lde_blocks=4), "shard0": dict(shard=(0, 2)), "shard1": dict(shard=(1, 2))}[kind]
    tc, ac = (pb.PolynomialBatch.from_values(v, 2, False, 2, **kw) for v in (tv, av))
    L = N.lib()
    try:
        for cs in (consts, _twin(consts)):
            _check_all_parts(ctx, L.gl_stark_check_rows, L.gl_stark_check_rows_part, _stark_args(tc, ac, prog, cs),
                             want, PARTS + ([1 << log_n] if cs is consts else []))
    finally:
        tc.close(), ac.close()


@pytest.mark.gpu
def test_plonk_parts_salted_and_truncated(pb):
    """256 registers, 4 commitments (one salted), constants past 65 535, on 2^6 rows: every part of G = 1 ... 16 and
    64, every merge, from canonical and non-canonical constants."""
    ctx = pb.default_context()
    log_n, widths, n_terms = 6, [3, 6, 2, 4], 4000
    prog = vp_program(0xCB0, 3000, widths, VP_CONSTS, n_terms, salted=-1)
    values = [_sparse(0xCB1 + c, (w, 1 << log_n)) for c, w in enumerate(widths)]
    consts = synth(0xCB5, (VP_CONSTS,))
    consts[::3] = 0
    batches = [pb.PolynomialBatch.from_values(v, 1, c == 1, 2) for c, v in enumerate(values)]
    L = N.lib()
    try:
        want = vp_expected(prog, values, consts, log_n)
        handles = (N.vp * 4)(*[b.h for b in batches])
        for cs in (consts, _twin(consts)):
            args = (handles, 4, prog.ctypes.data_as(N.vp), len(prog), N.np_ptr(cs), len(cs), n_terms)
            _check_all_parts(ctx, L.gl_plonk_check_rows, L.gl_plonk_check_rows_part, args, want,
                             PARTS + ([1 << log_n] if cs is consts else []))
    finally:
        for b in batches:
            b.close()


@pytest.mark.gpu
def test_part_refusals_before_any_launch(pb):
    """parts not a power of two or above n, part >= parts; the whole check's refusals keep their messages on the _part
    entry points; nothing is launched."""
    from test_check_constraints import VP_LOCAL, VP_TERM

    ctx = pb.default_context()
    L = N.lib()
    a = pb.PolynomialBatch.from_values(synth(0xCC0, (2, 16)), 1, False, 1)
    prog = np.array([(S.OP_LOCAL, 0, 0, 0), (S.OP_EMIT, 0, 0, 0)], dtype=np.uint16)
    vprog = np.array([(VP_LOCAL, 0, 0, 1), (VP_TERM, 0, 0, 0)], dtype=np.uint16)
    f, r, pairs = C.c_uint64(), C.c_uint32(), np.zeros(2, dtype=np.uint32)
    u32 = pairs.ctypes.data_as(N.u32p)
    hs = (N.vp * 1)(a.h)

    def stark(part, parts, p=prog, max_report=1):
        rc = L.gl_stark_check_rows_part(ctx.h, a.h, None, p.ctypes.data_as(N.vp), len(p), None, 0, part, parts,
                                        max_report, C.byref(f), u32, C.byref(r))
        return rc, L.gl_last_error(ctx.h).decode()

    def plonk(part, parts, p=vprog):
        rc = L.gl_plonk_check_rows_part(ctx.h, hs, 1, p.ctypes.data_as(N.vp), len(p), None, 0, 1, part, parts, 1,
                                        C.byref(f), u32, C.byref(r))
        return rc, L.gl_last_error(ctx.h).decode()
    try:
        before = ctx.launch_count
        for call in (stark, plonk):
            assert call(0, 3) == (N.GL_ERR_BAD_SHAPE, "parts 3 is not a power of two")
            assert call(0, 0) == (N.GL_ERR_BAD_SHAPE, "parts 0 is not a power of two")
            assert call(0, 32) == (N.GL_ERR_BAD_SHAPE, "parts 32 > the 16 rows of H")
            assert call(4, 4) == (N.GL_ERR_BAD_ARG, "part 4 >= parts 4")
            assert call(7, 3)[0] == N.GL_ERR_BAD_SHAPE
        assert stark(0, 2, max_report=N.MAX_REPORT + 1) == (N.GL_ERR_BAD_ARG, "max_report 65537 > 65536")
        bad = np.array([(S.OP_LOCAL, 2, 0, 0), (S.OP_EMIT, 0, 0, 0)], dtype=np.uint16)
        assert stark(0, 2, p=bad) == (N.GL_ERR_BAD_ARG, "constraint program: bad instruction 0")
        vbad = np.array([(VP_LOCAL, 0, 0, 2), (VP_TERM, 0, 0, 0)], dtype=np.uint16)
        assert plonk(0, 2, p=vbad) == (N.GL_ERR_BAD_ARG, "vanishing program: bad instruction 0")
        assert ctx.launch_count == before
        assert stark(15, 16)[0] == N.GL_OK and plonk(15, 16)[0] == N.GL_OK    # G = n: one row per part
    finally:
        a.close()


@pytest.mark.gpu
@pytest.mark.parametrize("host", ["pinned", "pageable"])
def test_part_host_inputs_are_read_before_returning(pb, host):
    """The program and constants of both _part calls in a page-locked (or pageable) buffer overwritten the moment the
    call returns, behind 0.2 s of spinning: each part's report is the evaluator's for the original inputs."""
    from test_gpu_host_buffers import _hold, _host_buffer, _overwrite

    ctx = pb.default_context()
    log_n, n_cols, n_consts, parts = 6, 4, 5, 4
    prog = stark_program(0xCD0, 200, n_cols, n_consts)
    tv = _sparse(0xCD1, (n_cols, 1 << log_n))
    consts = synth(0xCD2, (n_consts,))
    want = stark_expected(prog, tv, None, consts)
    vprog = vp_program(0xCD3, 400, [n_cols], VP_CONSTS, 50, salted=-1)
    vconsts = synth(0xCD4, (VP_CONSTS,))
    vwant = vp_expected(vprog, [tv], vconsts, log_n)
    tc = pb.PolynomialBatch.from_values(tv, 1, False, 2)
    handles = (N.vp * 1)(tc.h)
    try:
        for g in (1, 3):
            pbuf, cbuf = _host_buffer(prog.view(np.uint64), host), _host_buffer(consts, host)
            _hold(ctx)
            got = N.check_rows(N.lib().gl_stark_check_rows_part, ctx, (tc.h, None, N.np_ptr(pbuf), len(prog),
                                                                       N.np_ptr(cbuf), n_consts, g, parts), N.MAX_REPORT)
            _overwrite(pbuf, cbuf)
            mine = _restrict(want, g, parts)
            assert got == (len(mine), mine)
            pbuf, cbuf = _host_buffer(vprog.view(np.uint64), host), _host_buffer(vconsts, host)
            _hold(ctx)
            got = N.check_rows(N.lib().gl_plonk_check_rows_part, ctx, (handles, 1, N.np_ptr(pbuf), len(vprog),
                                                                       N.np_ptr(cbuf), VP_CONSTS, 50, g, parts),
                               N.MAX_REPORT)
            _overwrite(pbuf, cbuf)
            mine = _restrict(vwant, g, parts)
            assert got == (len(mine), mine)
    finally:
        tc.close()


@pytest.mark.gpu
def test_scratch_shrinks_with_the_parts(pb):
    """A 300-instruction program reading the next row of 32 columns of 2^16 rows: checked with parts=16 it gives the
    whole check's report, and its high-water mark above the handle is at most a quarter of the whole check's (the
    values on H, 16 MiB, against two buffers of 1/16 of them for the local and next rows)."""
    ctx = pb.default_context()
    log_n, n_cols, n_consts = 16, 32, 5
    prog = stark_program(0xCF0, 300, n_cols, n_consts)
    assert (prog[:, 0] == S.OP_NEXT).any()
    tv = _sparse(0xCF1, (n_cols, 1 << log_n))
    consts = synth(0xCF2, (n_consts,))
    tc = pb.PolynomialBatch.from_values(tv, 1, False, 4, ctx=ctx)
    L = N.lib()
    try:
        marks, reports = {}, {}
        for parts in (1, 16, 1):
            in_use, _ = ctx.device_bytes(reset_high=True)
            reports[parts] = N.check_rows_in_parts(L.gl_stark_check_rows, L.gl_stark_check_rows_part, ctx,
                                                   _stark_args(tc, None, prog, consts), 64, log_n, parts)
            marks[parts] = ctx.device_bytes()[1] - in_use
        assert reports[16] == reports[1] and reports[1][0] > 0
        assert 0 < marks[16] <= marks[1] // 4, marks
    finally:
        tc.close()


# ---- the provers with lde_blocks=G
def _error(fn):
    with pytest.raises(N.ConstraintError) as e:
        fn()
    return str(e.value), e.value.report.failures, e.value.report.entries


def _record_parts(monkeypatch, module):
    """Wrap module.check_constraints: the parts= every prover's check ran with."""
    real, seen = module.check_constraints, []

    def rec(*a, **k):
        seen.append(k.get("parts", 1))
        return real(*a, **k)
    monkeypatch.setattr(module, "check_constraints", rec)
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fibonacci", "range_check", "permutation"])
def test_blocked_starks_hold_and_prove_the_same(pb, monkeypatch, name):
    """FibonacciStark, RangeCheckStark (lookups) and PermutationStark (degree 0): with lde_blocks=4 and 16 the check
    runs in that many parts, finds nothing, and the proof equals the proof without the flag."""
    stark, trace, pis = _stark_cases()[name]
    config = S.StarkConfig.standard_fast_config()
    seen = _record_parts(monkeypatch, S)
    for G_ in (4, 16):
        checked = S.prove(stark, config, trace, pis, lde_blocks=G_, check_constraints=True)
        assert not T.proof_diff(checked, S.prove(stark, config, trace, pis, lde_blocks=G_))
    assert seen == [4, 16]


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [(0,), (-1,), (0, 1, -1)])
def test_blocked_broken_fibonacci_raises_the_resident_error(pb, rows):
    stark = S.FibonacciStark(1 << 8)
    trace = stark.generate_trace(0, 1)
    pis = [0, 1, int(trace[1, -1])]
    for r in rows:
        trace[1, r] = (int(trace[1, r]) + 1) % P
    config = S.StarkConfig.standard_fast_config()
    want = _error(lambda: S.prove(stark, config, trace, pis, check_constraints=True))
    for G_ in (2, 16):
        assert _error(lambda: S.prove(stark, config, trace, pis, lde_blocks=G_, check_constraints=True)) == want


@pytest.mark.gpu
def test_blocked_broken_lookup_raises_the_resident_error(pb):
    from test_stark_lookups import MA, RangeCheckStark

    trace = RangeCheckStark.generate_trace(7)
    trace[MA, 5] += np.uint64(1)
    config = S.StarkConfig.standard_fast_config()
    pis = [int(trace[7, 0])]
    want = _error(lambda: S.prove(RangeCheckStark(), config, trace, pis, check_constraints=True))
    assert want[0].startswith("Constraint failed in RangeCheckStark at row")
    assert _error(lambda: S.prove(RangeCheckStark(), config, trace, pis, lde_blocks=8, check_constraints=True)) == want


@pytest.mark.gpu
def test_blocked_ctl_system_holds_and_a_broken_value_raises_the_resident_error(pb, monkeypatch):
    """The CTL system of test_stark_ctl.py with lde_blocks=4: every table checked in 4 parts, the proofs equal those
    without the flag; one CTL Z value changed raises the resident run's ConstraintError."""
    from plonky2_b200 import cross_table_lookup as X
    from test_stark_ctl import system, system_traces

    starks, config, ctls = system()
    traces, pis = system_traces()
    seen = _record_parts(monkeypatch, S)
    checked = X.prove_with_ctls(starks, config, traces, ctls, pis, lde_blocks=4, check_constraints=True)
    assert seen == [4, 4, 4]
    assert not T.proof_diff(checked, X.prove_with_ctls(starks, config, traces, ctls, pis, lde_blocks=4))
    real = X.cross_table_lookup_data

    def broken(*a, **k):                              # the looked table's last CTL Z, one value changed at row 5
        data = real(*a, **k)
        data[2].auxiliary[-1, 5] = 12345
        return data
    monkeypatch.setattr(X, "cross_table_lookup_data", broken)
    want = _error(lambda: X.prove_with_ctls(starks, config, traces, ctls, pis, check_constraints=True))
    assert want[0].startswith("Constraint failed in LookedTable at row 4: CTL Z")
    assert _error(lambda: X.prove_with_ctls(starks, config, traces, ctls, pis, lde_blocks=4,
                                            check_constraints=True)) == want


def _prove_circuit(pb, c, G_=None, wires=None, check=False):
    from plonky2_b200 import plonk
    from plonky2_b200.fri import standard_recursion_fri_config

    cfg, cd = c.config, c.common
    fri_params = standard_recursion_fri_config().fri_params(cd.degree_bits, False)
    cs = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height, lde_blocks=G_)
    try:
        prover_data = plonk.ProverOnlyCircuitData(cs, c.sigmas, [int(x) for x in synth(0xCE0, (4,))], fri_params)
        return plonk.prove_with_witness(prover_data, cd, c.wires if wires is None else wires, c.public_inputs,
                                        check_constraints=check, lde_blocks=G_).to_bytes()
    finally:
        cs.close()


@pytest.mark.gpu
def test_blocked_circuit_holds_and_proves_the_same(pb, monkeypatch):
    """LargeCircuit at 2^13 gates with lookups, lde_blocks=2 and 16: the check runs in G parts and the bytes equal the
    proof's without the flag."""
    import plonk_large as PL
    from plonky2_b200 import plonk

    c = PL.large_circuit(13, public_inputs=[3, 1, 4])
    seen = _record_parts(monkeypatch, plonk)
    for G_ in (2, 16):
        assert _prove_circuit(pb, c, G_, check=True) == _prove_circuit(pb, c, G_), G_
    assert seen == [2, 16]


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["arith", "copy", "lookup"])
def test_blocked_broken_witness_raises_the_resident_error(pb, what):
    """A broken gate (qdf 8), a broken copy constraint and a broken looking pair: lde_blocks=4 and 16 raise the resident
    run's ConstraintError, message and report."""
    import plonk_large as PL

    if what == "arith":
        c = PL.large_circuit(13, qdf=8, break_arith=5000, public_inputs=[3, 1, 4, 1, 5, 9, 2, 6])
        wires = c.wires
    else:
        c = PL.large_circuit(10, public_inputs=[2, 7])
        wires = c.wires.copy()
        if what == "copy":
            (row, col) = c.partition()[1][2]
            wires[col, row] = (int(wires[col, row]) + 1) % P
        else:
            wires[1, c.lookup_rows[0][0]] = (int(wires[1, c.lookup_rows[0][0]]) + 12345) % P
    want = _error(lambda: _prove_circuit(pb, c, wires=wires, check=True))
    for G_ in (4, 16):
        assert _error(lambda: _prove_circuit(pb, c, G_, wires=wires, check=True)) == want, G_


# ---- the distributed provers
@pytest.mark.gpu
def test_distributed_provers_check_constraints(pb):
    """torchrun, one rank per GPU (2, or 4 with four GPUs; the ranks share GPU 0 over gloo on a single-GPU machine):
    distributed.prove_stark, prove_with_ctls and prove_plonk with check_constraints=True (tests/mgpu_check_constraints_
    check.py)."""
    run_ranks("mgpu_check_constraints_check.py", "MGPU_CHECK_CONSTRAINTS OK", timeout=900)
