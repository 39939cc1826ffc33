"""Non-resident commitments (gl_commit_begin_blocked / lde_blocks=G): a PolynomialBatch that keeps its coefficients,
digests and cap but never its LDE, and the starky provers on them.

CPU: every refusal of lde_blocks (not a positive power of two, more blocks than cap entries or than a table's quotient
coset, combined with blinding, a salt, shards or a prefix) is a ShapeError raised before any device work; the ABI
binding; Placement(num_shards > 1, lde_blocks) is refused.

GPU (-m gpu): for G = 1 ... 16 the non-resident batch equals the resident one in cap, digests, leaves (ranges across
block boundaries), Merkle openings of the first and last leaf of every block (paths verified against the cap),
get_lde_values and eval_commitment -- from values and coefficients, host and device columns, log n 4 ... 20, rates 1 ... 3,
widths 1 ... 135, including blocks smaller than the trace (the restriction branch). gl_stark_quotient[_aux] on
non-resident handles equals the resident call bit for bit, and a broken trace fails the same way. Proofs with
lde_blocks equal the resident proofs field for field and the restated verifier accepts them (FibonacciStark,
RangeCheckStark, the CTL system of tests/test_stark_ctl.py, whose tables' quotients are in their proofs). The library's
high-water mark during a blocked proof at 64 columns x 2^22 rows is lower than the resident proof's by at least half of
the summed LDE bytes, and no proof leaks device memory."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

import stark_twin as T
from conftest import synth
from plonky2_b200 import _native as N
from plonky2_b200 import cross_table_lookup as X
from plonky2_b200 import distributed as D
from plonky2_b200 import stark as S
from plonky2_b200.field import ORDER
from plonky2_b200.fri import FriConfig
from plonky2_b200.polynomial_batch import PolynomialBatch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAP_HEIGHT = 4
BLOCKS = [1, 2, 4, 8, 16]


# ----------------------------------------------------------------------------------------------------------- CPU
def test_refusals_before_device_work():
    """On a machine without a device each of these raises ShapeError, not the NativeError of context creation."""
    vals = np.zeros((2, 16), dtype=np.uint64)
    for G in (0, -4, 3, 6):
        with pytest.raises(N.ShapeError, match="positive power of two"):
            PolynomialBatch.from_values(vals, 1, False, CAP_HEIGHT, lde_blocks=G)
    with pytest.raises(N.ShapeError, match="exceeds the 16 cap entries"):
        PolynomialBatch.from_coeffs(vals, 1, False, CAP_HEIGHT, lde_blocks=32)
    with pytest.raises(N.ShapeError, match="cannot be blinded"):
        PolynomialBatch.from_values(vals, 1, True, CAP_HEIGHT, lde_blocks=2)
    with pytest.raises(N.ShapeError, match="cannot be blinded"):
        PolynomialBatch.from_values(vals, 1, False, CAP_HEIGHT, salt=np.zeros((4, 32), dtype=np.uint64), lde_blocks=2)
    with pytest.raises(N.ShapeError, match="cannot be blinded"):
        PolynomialBatch.from_values(vals, 1, True, CAP_HEIGHT, salt_key=bytes(32), lde_blocks=2)
    with pytest.raises(N.ShapeError, match="shard="):
        PolynomialBatch.from_values(vals, 1, False, CAP_HEIGHT, shard=(0, 2), lde_blocks=2)
    with pytest.raises(N.ShapeError, match="prefix="):
        PolynomialBatch._from_device(None, 2, 4, 1, CAP_HEIGHT, None, prefix=object(), lde_blocks=2)
    with pytest.raises(N.ShapeError, match="positive power of two"):
        PolynomialBatch._from_coeff_chunks(None, 2, 4, 1, CAP_HEIGHT, lde_blocks=5)

    config = S.StarkConfig.standard_fast_config()
    stark = S.FibonacciStark(16)
    trace = stark.generate_trace(0, 1)
    pis = [0, 1, int(trace[1, -1])]
    for G in (0, 3, 32):
        with pytest.raises(N.ShapeError, match="lde_blocks"):
            S.prove(stark, config, trace, pis, lde_blocks=G)
    # 16 blocks <= 2^cap_height, but more than the 8 points of FibonacciStark(8)'s quotient coset
    small = S.StarkConfig(100, 2, FriConfig(rate_bits=1, cap_height=4, proof_of_work_bits=0,
                                            reduction_strategy=("ConstantArityBits", 1, 3), num_query_rounds=2))
    stark8 = S.FibonacciStark(8)
    trace8 = stark8.generate_trace(0, 1)
    with pytest.raises(N.ShapeError, match="quotient coset"):
        S.prove(stark8, small, trace8, [0, 1, int(trace8[1, -1])], lde_blocks=16)

    from test_stark_ctl import system, system_traces

    starks, config, ctls = system()
    traces, cpis = system_traces()
    for G in (0, 3, 32):
        with pytest.raises(N.ShapeError, match="lde_blocks"):
            X.prove_with_ctls(starks, config, traces, ctls, cpis, lde_blocks=G)


def test_placement():
    with pytest.raises(N.ShapeError, match="one device"):
        D.Placement(num_shards=2, lde_blocks=4)
    assert D.Placement(lde_blocks=4).commit_kwargs == dict(lde_blocks=4)
    assert D.Placement(lde_blocks=4).step_kwargs == {}
    assert D.Placement().commit_kwargs == {}
    assert D.Placement(1, 2).commit_kwargs == dict(shard=(1, 2))


def test_abi_binding():
    import plonky2_b200.build as b

    b.build()
    L = N.lib()
    for name in ("gl_commit_begin_blocked", "gl_commit_lde_blocks", "gl_ctx_device_bytes"):
        assert name in N.EXPORTS
        assert getattr(L, name).argtypes is not None, name
    assert L.gl_commit_lde_blocks.restype == C.c_uint32


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


def _columns(seed, width, log_n):
    return (synth(seed, (width, 1 << log_n)) % np.uint64(ORDER)).astype(np.uint64)


def _batch(ctx, cols, rate_bits, is_coeffs, source, lde_blocks=None):
    """A batch of the host columns `cols`, from host memory or from a torch CUDA tensor (_from_device)."""
    import torch

    if source == "host":
        make = PolynomialBatch.from_coeffs if is_coeffs else PolynomialBatch.from_values
        return make(cols, rate_bits, False, CAP_HEIGHT, ctx=ctx, lde_blocks=lde_blocks)
    dev = torch.from_numpy(np.ascontiguousarray(cols).view(np.int64)).cuda()
    torch.cuda.synchronize()
    B, n = cols.shape
    kind = N.COLS_COEFFS if is_coeffs else N.COLS_VALUES

    def add_columns(h):
        N.check(N.lib().gl_commit_add_columns(h, 0, B, N.vp(dev.data_ptr()), n, kind, N.MEM_DEVICE), ctx.h)

    return PolynomialBatch._from_device(ctx, B, n.bit_length() - 1, rate_bits, CAP_HEIGHT, add_columns,
                                        lde_blocks=lde_blocks)


# (log n, rate_bits, width, coefficients?, source): every value of each axis; G = 16 restricts the trace to blocks of
# fewer than n points wherever 16 > 2^rate_bits
CASES = [(4, 1, 1, False, "host"), (4, 3, 9, True, "device"), (10, 2, 8, False, "device"), (10, 1, 135, True, "host"),
         (10, 3, 135, False, "host"), (16, 3, 9, False, "host"), (16, 1, 8, True, "device"), (20, 1, 8, False, "device"),
         (20, 2, 1, True, "host")]


@pytest.mark.gpu
@pytest.mark.parametrize("log_n,rate_bits,width,is_coeffs,source", CASES)
def test_blocked_batch_equals_resident(pb, log_n, rate_bits, width, is_coeffs, source):
    from plonky2_b200.hash import MerkleProof, verify_merkle_proof_to_cap

    ctx = pb.default_context()
    cols = _columns(0xB10C + 7 * log_n + width, width, log_n)
    whole = _batch(ctx, cols, rate_bits, is_coeffs, source)
    N_ = whole.lde_size
    z = (int(synth(0xE7A1, (1,))[0]) % ORDER, 5)
    try:
        assert whole.lde_blocks == 0
        cap, digests = whole.merkle_tree.cap.hashes, whole.merkle_tree.digests
        leaves = whole.merkle_tree.leaves if N_ * width <= 1 << 22 else None
        polys, ev = whole.polynomials, whole.eval_commitment(z)
        for G in BLOCKS:
            blk = _batch(ctx, cols, rate_bits, is_coeffs, source, lde_blocks=G)
            try:
                assert blk.lde_blocks == G and N.lib().gl_commit_lde_blocks(blk.h) == G
                assert N.lib().gl_commit_dev_lde(blk.h, None) is None
                assert np.array_equal(blk.merkle_tree.cap.hashes, cap), G
                assert np.array_equal(blk.merkle_tree.digests, digests), G
                assert np.array_equal(blk.polynomials, polys), G
                assert np.array_equal(blk.eval_commitment(z), ev), G
                Nb = N_ // G
                if leaves is not None:
                    assert np.array_equal(blk.merkle_tree.leaves, leaves), G
                for b in range(1, G):  # rows on both sides of every block boundary, in one call
                    lo, hi = max(0, b * Nb - 3), min(N_, b * Nb + 3)
                    assert np.array_equal(blk.merkle_tree.get_rows(lo, hi - lo), whole.merkle_tree.get_rows(lo, hi - lo))
                ends = sorted({i for b in range(G) for i in (b * Nb, (b + 1) * Nb - 1)})
                lv, pt = blk.merkle_tree.open_many(ends)
                wl, wp = whole.merkle_tree.open_many(ends)
                assert np.array_equal(lv, wl) and np.array_equal(pt, wp), G
                if G == BLOCKS[-1]:
                    for k, i in enumerate(ends):
                        verify_merkle_proof_to_cap(lv[k], i, blk.merkle_tree.cap, MerkleProof(pt[k]), ctx)
                for i in (0, 1, N_ // 2 + 1, N_ - 1):
                    assert np.array_equal(blk.get_lde_values(i, 1), whole.get_lde_values(i, 1)), (G, i)
            finally:
                blk.close()
    finally:
        whole.close()


@pytest.mark.gpu
def test_entry_point_errors(pb):
    """begin_blocked's shape refusals; keyed and prefixed finishes, the value-domain FRI start and the shard and plonky2
    quotients refuse a non-resident handle; mixing resident and non-resident handles in one quotient is refused; a
    non-resident cap still serves as another commitment's prefix."""
    import torch

    from test_gpu_stark_sharded import _stark_case, _to_device

    ctx = pb.default_context()
    L = N.lib()
    h = N.vp()
    for G in (0, 3, 32):
        assert L.gl_commit_begin_blocked(ctx.h, 2, 6, 1, CAP_HEIGHT, G, None, C.byref(h)) == N.GL_ERR_BAD_SHAPE, G
    assert L.gl_commit_begin_blocked(ctx.h, 2, 6, 1, CAP_HEIGHT, 4, None, C.byref(h)) == N.GL_OK
    prefix = np.zeros(4 << 7, dtype=np.uint64)  # refused before it is read
    assert L.gl_commit_finish_prefixed(h, N.np_ptr(prefix)) == N.GL_ERR_BAD_ARG
    assert L.gl_commit_finish_keyed(h, bytes(32)) == N.GL_ERR_BAD_ARG
    salt = np.zeros(4 << 7, dtype=np.uint64)
    assert L.gl_commit_finish(h, N.np_ptr(salt), N.MEM_HOST) == N.GL_ERR_BAD_ARG
    L.gl_commit_destroy(h)

    stark, trace, pis, challenges = _stark_case("range", 10)
    alphas = [3, 4]
    dev = _to_device(trace)
    helpers = S.compute_lookup_helper_columns(stark, dev, challenges, ctx)
    t_res = S._commit_trace(dev, 1, CAP_HEIGHT, ctx)
    t_blk = S._commit_trace(dev, 1, CAP_HEIGHT, ctx, lde_blocks=4)
    a_res = S.commit_auxiliary_polys(helpers, 1, CAP_HEIGHT, ctx)
    a_blk = S.commit_auxiliary_polys(helpers, 1, CAP_HEIGHT, ctx, lde_blocks=4)
    made = [t_res, t_blk, a_res, a_blk]
    try:
        b, consts, al = S.quotient_program(stark, pis, alphas, a_res, challenges)
        out = torch.empty((2, 2 << 10), dtype=torch.int64, device="cuda")

        def quotient_aux(t, a, fn=L.gl_stark_quotient_aux):
            return fn(ctx.h, t.h, a.h, b.program(), len(b.instrs), N.np_ptr(consts), len(consts), N.np_ptr(al), len(al),
                      stark.quotient_degree_factor(), N.vp(out.data_ptr()))

        for t, a in ((t_res, a_blk), (t_blk, a_res)):
            assert quotient_aux(t, a) == N.GL_ERR_BAD_ARG
            assert b"both be resident or both not" in L.gl_last_error(ctx.h)
        assert quotient_aux(t_blk, a_blk) == N.GL_OK
        assert quotient_aux(t_blk, a_blk, L.gl_stark_quotient_shard) == N.GL_ERR_BAD_ARG
        assert b"resident trace" in L.gl_last_error(ctx.h)

        one = np.zeros(1, dtype=np.uint32)
        batch = N.FriBatch((C.c_uint64 * 2)(3, 4), 1, one.ctypes.data_as(N.u32p), one.ctypes.data_as(N.u32p))
        opened = np.zeros(2, dtype=np.uint64)
        alpha = np.array([5, 6], dtype=np.uint64)
        f = N.vp()
        assert L.gl_fri_begin_values(ctx.h, (N.vp * 1)(t_blk.h), 1, C.byref(batch), 1, N.np_ptr(opened),
                                     N.np_ptr(alpha), CAP_HEIGHT, C.byref(f)) == N.GL_ERR_BAD_ARG
        assert b"non-resident" in L.gl_last_error(ctx.h)

        instr = np.zeros(4, dtype=np.uint16)  # one instruction; the commitment check comes first
        assert L.gl_plonk_quotient(ctx.h, (N.vp * 1)(t_blk.h), 1, instr.ctypes.data_as(N.vp), 1, None, 0,
                                   N.np_ptr(alpha), 1, 1, 1, N.vp(out.data_ptr())) == N.GL_ERR_BAD_ARG
        assert b"not resident" in L.gl_last_error(ctx.h)
        assert L.gl_plonk_quotient_shard(ctx.h, (N.vp * 1)(t_blk.h), 1, instr.ctypes.data_as(N.vp), 1, None, 0,
                                         N.np_ptr(alpha), 1, 1, 1, N.vp(out.data_ptr())) == N.GL_ERR_BAD_ARG

        # the prefix of a batch Merkle tree's next stage is the cap alone: 16 cap entries, 16 leaves of the next stage
        nxt = _columns(0xF1E, 3, 3)
        prefixed = []
        for prefix in (t_res, t_blk):
            prefixed.append(PolynomialBatch._from_device(
                ctx, 3, 3, 1, CAP_HEIGHT,
                lambda hh: N.check(L.gl_commit_add_columns(hh, 0, 3, N.np_ptr(nxt), 8, N.COLS_VALUES, N.MEM_HOST), ctx.h),
                prefix=prefix))
        made += prefixed
        assert np.array_equal(prefixed[0].merkle_tree.cap.hashes, prefixed[1].merkle_tree.cap.hashes)
    finally:
        for c in made:
            c.close()


def _quotients(pb, stark, trace, pis, challenges, rate_bits, alphas, blocks):
    """compute_quotient_polys on resident commitments, then on non-resident ones of each G in blocks."""
    ctx = pb.default_context()
    from test_gpu_stark_sharded import _to_device

    dev = _to_device(trace)
    helpers = S.compute_lookup_helper_columns(stark, dev, challenges, ctx) if challenges is not None else None
    out = []
    for G in [None] + list(blocks):
        t = S._commit_trace(dev, rate_bits, CAP_HEIGHT, ctx, **({} if G is None else dict(lde_blocks=G)))
        a = None
        try:
            if helpers is not None:
                a = S.commit_auxiliary_polys(helpers, rate_bits, CAP_HEIGHT, ctx,
                                             **({} if G is None else dict(lde_blocks=G)))
            args = dict(auxiliary_polys_commitment=a, lookup_challenges=challenges) if helpers is not None else {}
            try:
                out.append(S.compute_quotient_polys(stark, t, pis, alphas, **args))
            except N.NativeError as e:
                out.append(str(e))
        finally:
            t.close()
            if a is not None:
                a.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kind,log_n,rate_bits", [("fib", 10, 1), ("fib", 13, 2), ("fib", 16, 3), ("range", 10, 1),
                                                  ("range", 12, 2), ("range", 14, 3), ("range4", 11, 2)])
def test_blocked_quotient_equals_resident(pb, kind, log_n, rate_bits):
    """FibonacciStark (quotient coset smaller than the LDE coset; the next row leaves every part when G > 1; parts smaller
    than the trace from G = 2 on), RangeCheckStark (quotient degree 2: coset equal to the LDE coset at rate 1, smaller at
    rates 2 and 3), RangeCheckStark4 (quotient degree 4, the next row inside the part up to G = 4)."""
    import torch

    from test_gpu_stark_sharded import _stark_case

    stark, trace, pis, challenges = _stark_case(kind, log_n)
    alphas = [int(v) for v in synth(0xB5B0 + log_n, (2,))]
    want, *got = _quotients(pb, stark, trace, pis, challenges, rate_bits, alphas, BLOCKS)
    for G, g in zip(BLOCKS, got):
        assert torch.equal(g, want), G


@pytest.mark.gpu
def test_blocked_quotient_of_a_broken_trace(pb):
    """A trace that breaks a constraint fails the trim check with the resident call's message, at every G."""
    from test_gpu_stark_sharded import _stark_case
    from test_stark_lookups import SEL2

    stark, trace, pis, challenges = _stark_case("range4", 10)
    trace[SEL2, 9] = 2
    want, *got = _quotients(pb, stark, trace, pis, challenges, 2, [3, 4], [1, 4, 16])
    assert isinstance(want, str) and "Quotient has failed" in want
    assert got == [want] * 3


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["fib", "range"])
@pytest.mark.parametrize("source", ["host", "device"])
def test_prove_blocked_equals_resident(pb, oracle, kind, source):
    from test_gpu_stark_sharded import _stark_case, _to_device

    stark, trace, pis, _ = _stark_case(kind, 10)
    config = S.StarkConfig.standard_fast_config()
    arg = trace if source == "host" else _to_device(trace)
    want = S.prove(stark, config, arg, pis)
    assert T.verify(oracle, stark, config, want) is None
    for G in (1, 4, 16):
        got = S.prove(stark, config, arg, pis, lde_blocks=G)
        assert not T.proof_diff(got, want)
        assert T.verify(oracle, stark, config, got) is None


@pytest.mark.gpu
def test_prove_with_ctls_blocked_equals_resident(pb, oracle):
    from test_stark_ctl import system, system_traces

    starks, config, ctls = system()
    traces, pis = system_traces()
    want = X.prove_with_ctls(starks, config, traces, ctls, pis)
    got = X.prove_with_ctls(starks, config, traces, ctls, pis, lde_blocks=4)
    assert not T.proof_diff(got, want)
    assert T.verify_with_ctls(oracle, starks, config, ctls, got) is None


def _pairs_module():
    spec = importlib.util.spec_from_file_location("stark_prove_cost", os.path.join(ROOT, "tools", "stark_prove_cost.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.mark.gpu
def test_blocked_proof_lowers_the_high_water_mark(pb):
    """64 Fibonacci-pair columns x 2^22 rows at rate 1/2: the trace and quotient LDEs sum to over 4 GiB, 4x the NTT
    group scratch. Each proof runs once unmeasured first, so that the context's cached tables and scratch exist."""
    m = _pairs_module()
    stark, config = m.FibonacciPairsStark(), S.StarkConfig.standard_fast_config()
    log_n = 22
    trace = m.fibonacci_pairs_trace(log_n)
    rate_bits = config.fri_config.rate_bits
    lde_words = (stark.COLUMNS + stark.num_quotient_polys(config)) << (log_n + rate_bits)
    ctx = pb.default_context()
    proofs, highs = {}, {}
    for G in (None, 8):
        S.prove(stark, config, trace, [], ctx=ctx, lde_blocks=G)
        before, _ = ctx.device_bytes(reset_high=True)
        proofs[G] = S.prove(stark, config, trace, [], ctx=ctx, lde_blocks=G)
        after, highs[G] = ctx.device_bytes()
        assert after == before, (G, before, after)
    assert not T.proof_diff(proofs[8], proofs[None])
    assert highs[None] - highs[8] >= lde_words * 8 // 2, (highs, lde_words * 8)
