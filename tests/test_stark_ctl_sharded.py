"""A multi-STARK proof with cross-table lookups across several GPUs (distributed.prove_with_ctls), and the openings split
between the ranks that it, prove_stark and prove_plonk share (gl_openings_shard, Placement.openings_from_shards).

CPU: the coefficient blocks B_g(n) = [g*n/G, (g+1)*n/G) tile [0, n) for every n and G (n < G included) and the oracle's
partial sums over them add up to the whole evaluation; two gloo ranks with the native call stubbed add up their partial
openings in rank order and raise together when one rank fails; check_prove_with_ctls's refusals.
GPU (-m gpu): every shard's gl_openings_shard output, summed mod p, equals gl_openings bit for bit -- commitments of
several degrees in one call, the points zeta, g*zeta, 1 and 0, repeated points, host and device output, and one
2^22-coefficient commitment at G = 8; shard (0, 1) is gl_openings byte for byte; bad shard arguments return
GL_ERR_BAD_ARG. prove_with_ctls on one rank is cross_table_lookup.prove_with_ctls; on 2 (4 with four GPUs) torchrun
ranks (tests/mgpu_ctl_check.py) every rank's proof equals it and the restated verifier accepts it."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import P, synth
from plonky2_b200 import _native as N
from plonky2_b200 import distributed as D
from plonky2_b200 import stark as S
from ranks import run_ranks, spawn_ranks


def block(n, g, G):
    """B_g(n), the coefficients shard g of G sums (include/plonky2_b200.h, gl_openings_shard)."""
    return g * n // G, (g + 1) * n // G


# ----------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("log_n", [0, 1, 2, 3, 5, 10])
@pytest.mark.parametrize("G", [1, 2, 4, 8, 16])
def test_blocks_tile_the_coefficients_and_partials_add_up(oracle, log_n, G):
    n = 1 << log_n
    blocks = [block(n, g, G) for g in range(G)]
    assert blocks[0][0] == 0 and blocks[-1][1] == n
    assert all(blocks[g][1] == blocks[g + 1][0] for g in range(G - 1))
    assert sum(hi - lo for lo, hi in blocks) == n
    coeffs = synth(0x0C10 + log_n, (n,))
    z = (int(synth(0x0C11, (1,))[0]), int(synth(0x0C12, (1,))[0]))
    total = [0, 0]
    for lo, hi in blocks:
        part = np.zeros(n, dtype=np.uint64)
        part[lo:hi] = coeffs[lo:hi]
        v = oracle.eval_poly_base_at_ext(part, z)
        if lo == hi:
            assert v == (0, 0)
        total = [(total[0] + v[0]) % P, (total[1] + v[1]) % P]
    assert tuple(total) == oracle.eval_poly_base_at_ext(coeffs, z)


def test_add_mod_p_wraps_like_the_field():
    a = np.array([0, 1, P - 1, P - 1, 2**63, P - 2**32], dtype=np.uint64)
    b = np.array([0, P - 1, P - 1, 1, 2**63, P - 1], dtype=np.uint64)
    got = D._add_mod_p(a, b)
    assert [int(v) for v in got] == [(int(x) + int(y)) % P for x, y in zip(a, b)]


def _partials(rank, total):
    """Rank `rank`'s stand-in partial sums: canonical values, with p - 1 in places so that the sum wraps."""
    v = synth(0x0C20 + rank, (total, 2))
    v[::3] = np.uint64(P - 1)
    return v


class _Batch:
    h, ctx = None, None

    def __init__(self, num_polys):
        self.num_polys = num_polys


class _Ctx:
    h, device = None, 0


def _openings_worker(rank, world, fail_rank):
    from plonky2_b200 import _native as N_
    from plonky2_b200 import distributed as D_
    from plonky2_b200 import proof as proof_mod

    class Stub:
        """The library, with gl_openings_shard writing this rank's stand-in partials (or failing on fail_rank)."""

        def gl_openings_shard(self, ctx, handles, pidx, n_evals, points, n_points, g, G, out, mem):
            assert (g, G) == (rank, world) and mem == N_.MEM_HOST and n_evals == 3 and n_points == 2
            if rank == fail_rank:
                return N_.GL_ERR_BAD_ARG
            dst = np.ctypeslib.as_array(C.cast(out, C.POINTER(C.c_uint64)), (11 * 2,))
            dst[:] = _partials(rank, 11).reshape(-1)
            return N_.GL_OK

        def gl_last_error(self, ctx):
            return b"stub failure"

    N_._lib = Stub()
    batches = [_Batch(3), _Batch(4)]
    for b in batches:
        b.ctx = _Ctx()
    placement = D_.Placement(rank, world, None)
    try:
        res = proof_mod.eval_commitments([(batches[0], (5, 7)), (batches[1], (5, 7)), (batches[1], (1, 0))],
                                         placement=placement)
        return rank, "ok", [r.tolist() for r in res]
    except Exception as e:
        return rank, "%s: %s" % (type(e).__name__, e), None


def _run_two_ranks(fail_rank):
    return spawn_ranks(_openings_worker, 2, (fail_rank,), timeout=180)


def test_openings_gathered_and_summed_on_two_ranks():
    """eval_commitments on a Placement of two gloo ranks: each rank's (stubbed) gl_openings_shard partials are
    all-gathered and added up mod p in rank order; both ranks return the same arrays, split by request."""
    res = _run_two_ranks(fail_rank=None)
    want = [[(int(a) + int(b)) % P for a, b in zip(r0, r1)]
            for r0, r1 in zip(_partials(0, 11).tolist(), _partials(1, 11).tolist())]
    flat = lambda parts: [row for part in parts for row in part]  # noqa: E731
    assert [r[1] for r in res] == ["ok", "ok"]
    assert flat(res[0][2]) == flat(res[1][2]) == want
    assert [len(p) for p in res[0][2]] == [3, 4, 4]


def test_openings_failure_on_one_rank_raises_on_every_rank():
    res = _run_two_ranks(fail_rank=1)
    assert res[0][:2] == (0, "NativeError: the openings failed on rank 1")
    assert res[1][0] == 1 and res[1][1].startswith("NativeError: plonky2_b200 native error 5: stub failure")


def test_check_prove_with_ctls_refusals():
    from test_stark_ctl import system, system_traces

    starks, config, ctls = system()
    traces, pis = system_traces()
    for world in (1, 2, 4, 8, 16):
        D.check_prove_with_ctls(starks, config, traces, ctls, pis, world)
    with pytest.raises(N.ShapeError, match="power-of-two number of ranks, got 3"):
        D.check_prove_with_ctls(starks, config, traces, ctls, pis, 3)
    with pytest.raises(N.ShapeError, match="32 ranks exceed the 16 cap entries"):
        D.check_prove_with_ctls(starks, config, traces, ctls, pis, 32)
    # what prove_with_ctls refuses, refused here with its messages
    with pytest.raises(N.ShapeError, match="expected 3 traces"):
        D.check_prove_with_ctls(starks, config, traces[:2], ctls, pis, 2)
    with pytest.raises(N.ShapeError, match="public-input lists"):
        D.check_prove_with_ctls(starks, config, traces, ctls, pis[:2], 2)
    with pytest.raises(N.ShapeError, match="COLUMNS"):
        D.check_prove_with_ctls(starks, config, [traces[1], traces[0], traces[2]], ctls, pis, 2)
    with pytest.raises(N.ShapeError, match="names table 5"):
        from plonky2_b200.cross_table_lookup import CrossTableLookup, TableWithColumns
        from plonky2_b200.lookup import Column, Filter

        bad = ctls + [CrossTableLookup([TableWithColumns(5, [Column.single(0)], Filter.default())],
                                       TableWithColumns(1, [Column.single(0)], Filter.default()))]
        D.check_prove_with_ctls(starks, config, traces, bad, pis, 2)
    # a small table whose quotient degree bits (0) are fewer than rate_bits (1): its quotient coset is n = 8 points,
    # enough for 8 ranks and too few for 16, although 16 ranks fit the cap
    fib = S.FibonacciStark(8)
    trace = fib.generate_trace(0, 1)
    fib_pis = [[0, 1, int(trace[1, -1])]]
    D.check_prove_with_ctls([fib], config, [trace], [], fib_pis, 8)
    with pytest.raises(N.ShapeError, match="table 0's quotient coset has 8 points, fewer than the 16 ranks"):
        D.check_prove_with_ctls([fib], config, [trace], [], fib_pis, 16)


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


def _call(fn, ctx, batches, point_index, points, out, mem, *shard):
    handles = (N.vp * len(batches))(*[b.h for b in batches])
    pidx = np.array(point_index, dtype=np.uint32)
    pts = np.array(points, dtype=np.uint64).reshape(-1)
    return fn(ctx.h, handles, pidx.ctypes.data_as(N.u32p), len(batches), N.np_ptr(pts), len(points), *shard,
              N.vp(out.data_ptr() if hasattr(out, "data_ptr") else out.ctypes.data), mem)


def _shard_sum_case(pb, batches, point_index, points, Gs):
    import torch

    L, ctx = N.lib(), pb.default_context()
    total = sum(b.num_polys for b in batches)
    whole = np.empty((total, 2), dtype=np.uint64)
    N.check(_call(L.gl_openings, ctx, batches, point_index, points, whole, N.MEM_HOST), ctx.h)
    one = np.empty_like(whole)
    N.check(_call(L.gl_openings_shard, ctx, batches, point_index, points, one, N.MEM_HOST, 0, 1), ctx.h)
    assert one.tobytes() == whole.tobytes()
    for G in Gs:
        acc = np.zeros_like(whole)
        for g in range(G):
            if g % 2:  # device output on odd shards
                dev = torch.empty((total, 2), dtype=torch.int64, device="cuda:%d" % ctx.device)
                N.check(_call(L.gl_openings_shard, ctx, batches, point_index, points, dev, N.MEM_DEVICE, g, G), ctx.h)
                ctx.synchronize()
                part = dev.cpu().numpy().view(np.uint64)
            else:
                part = np.empty_like(whole)
                N.check(_call(L.gl_openings_shard, ctx, batches, point_index, points, part, N.MEM_HOST, g, G), ctx.h)
            assert (part < np.uint64(P)).all()
            acc = D._add_mod_p(acc, part)
        assert np.array_equal(acc, whole), G
    return whole


@pytest.mark.gpu
def test_shard_sums_equal_gl_openings(pb, oracle):
    """Commitments of 2^0 .. 2^12 coefficients in one call (n_c < G for the smallest), at zeta, g*zeta, 1 and 0, with
    points repeated between requests; every G in {1, 2, 4, 8, 16}; each shard's value is also the oracle's sum over its
    block."""
    logs = [12, 0, 3, 9, 1]
    data = [synth(0x0C30 + i, (2 + i, 1 << lg)) for i, lg in enumerate(logs)]
    batches = [pb.PolynomialBatch.from_values(d, 1, False, 0) for d in data]
    try:
        zeta = (int(synth(0x0C40, (1,))[0]), int(synth(0x0C41, (1,))[0]))
        gz = pb.field.ext_mul((pb.field.primitive_root_of_unity(12), 0), zeta)
        points = [zeta, gz, (1, 0), (0, 0)]
        point_index = [0, 1, 2, 3, 0]
        req = batches + [batches[0], batches[3], batches[1]]
        pidx = point_index + [2, 0, 1]
        whole = _shard_sum_case(pb, req, pidx, points, [1, 2, 4, 8, 16])
        # the oracle's block sums for shard 3 of 16 of every request
        L, ctx = N.lib(), pb.default_context()
        part = np.empty_like(whole)
        N.check(_call(L.gl_openings_shard, ctx, req, pidx, points, part, N.MEM_HOST, 3, 16), ctx.h)
        row = 0
        for b, p in zip(req, pidx):
            coeffs = b.polynomials
            lo, hi = block(coeffs.shape[1], 3, 16)
            for k in range(b.num_polys):
                masked = np.zeros_like(coeffs[k])
                masked[lo:hi] = coeffs[k, lo:hi]
                assert tuple(int(v) for v in part[row]) == oracle.eval_poly_base_at_ext(masked, points[p])
                row += 1
    finally:
        for b in batches:
            b.close()


@pytest.mark.gpu
def test_shard_sums_at_2_22_coefficients(pb):
    import torch

    vals = torch.from_numpy(synth(0x0C50, (3, 1 << 22)).view(np.int64)).cuda()
    torch.cuda.synchronize()
    c = S._commit_trace(vals, 1, 4, pb.default_context())
    try:
        zeta = (int(synth(0x0C51, (1,))[0]), int(synth(0x0C52, (1,))[0]))
        _shard_sum_case(pb, [c, c], [0, 1], [zeta, (1, 0)], [8])
    finally:
        c.close()


@pytest.mark.gpu
def test_bad_shard_arguments(pb):
    L, ctx = N.lib(), pb.default_context()
    c = pb.PolynomialBatch.from_values(synth(0x0C60, (2, 16)), 1, False, 0)
    try:
        out = np.empty((2, 2), dtype=np.uint64)
        for g, G in ((0, 0), (4, 4), (5, 2)):
            assert _call(L.gl_openings_shard, ctx, [c], [0], [(3, 4)], out, N.MEM_HOST, g, G) == N.GL_ERR_BAD_ARG
            assert "shard" in L.gl_last_error(ctx.h).decode()
        assert _call(L.gl_openings_shard, ctx, [c], [1], [(3, 4)], out, N.MEM_HOST, 0, 2) == N.GL_ERR_BAD_ARG
        assert _call(L.gl_openings_shard, ctx, [c], [0], [(3, 4)], out, N.MEM_HOST, 1, 2) == N.GL_OK
    finally:
        c.close()


@pytest.mark.gpu
def test_prove_with_ctls_on_one_rank_is_prove_with_ctls(pb):
    """Without a process group distributed.prove_with_ctls is cross_table_lookup.prove_with_ctls: the same proof, table
    by table, field for field."""
    import stark_twin as T
    from plonky2_b200 import cross_table_lookup as X
    from test_stark_ctl import system, system_traces

    starks, config, ctls = system()
    traces, pis = system_traces()
    assert not T.proof_diff(D.prove_with_ctls(starks, config, traces, ctls, pis),
                            X.prove_with_ctls(starks, config, traces, ctls, pis))


@pytest.mark.gpu
def test_prove_with_ctls_across_ranks(pb):
    """torchrun, one rank per GPU (2, or 4 with four GPUs; the ranks share GPU 0 over gloo on a single-GPU machine):
    every rank's MultiStarkProof equals prove_with_ctls's and the restated verifier accepts it; refusals on every
    rank."""
    run_ranks("mgpu_ctl_check.py", "MGPU_CTL_CHECK OK", timeout=900)
