"""One STARK proved across ranks: the sharded quotient (gl_stark_quotient_shard + gl_stark_quotient_from_shards) and
distributed.prove_stark.

CPU: prove_stark's refusals (world size not a power of two or above 2^cap_height, a Stark with CTLs), raised before any
device work.

GPU (-m gpu): every shard of the trace (and auxiliary) commitment built in one process, each shard's values from
gl_stark_quotient_shard, concatenated and interpolated by gl_stark_quotient_from_shards: bit for bit gl_stark_quotient's
coefficients, for G = 1 ... 16 shards, FibonacciStark and the lookup RangeCheckStark of tests/test_stark_lookups.py, the
local values read in place (quotient coset = LDE coset) or computed (rate above the quotient degree), the next row in
the same shard or computed, shards smaller than the trace (the restriction branch) and larger. The entry points' errors;
a broken trace failing the trim check after the gather. prove_stark on one rank is stark.prove; on 2 (4 with four GPUs)
torchrun ranks (tests/mgpu_stark_check.py) every rank's proof equals stark.prove's and the restated verifiers accept
it."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import synth
from plonky2_b200 import _native as N
from plonky2_b200 import distributed as D
from plonky2_b200 import stark as S
from ranks import run_ranks

CAP_HEIGHT = 4


class _CtlStark(S.FibonacciStark):
    def requires_ctls(self):
        return True


# ----------------------------------------------------------------------------------------------------------- CPU
def test_prove_stark_refusals_before_device_work():
    config = S.StarkConfig.standard_fast_config()
    assert config.fri_config.cap_height == CAP_HEIGHT
    stark = S.FibonacciStark(16)
    for world in (1, 2, 4, 8, 16):
        D.check_prove_stark(stark, config, world)
    for world in (0, 3, 6, 12):
        with pytest.raises(N.ShapeError, match="power-of-two"):
            D.check_prove_stark(stark, config, world)
    with pytest.raises(N.ShapeError, match="exceed the 16 cap entries"):
        D.check_prove_stark(stark, config, 32)
    with pytest.raises(N.ShapeError, match="cross-table lookups"):
        D.check_prove_stark(_CtlStark(16), config, 2)
    # without a process group prove_stark is one rank; it refuses before it looks for a device
    trace = np.zeros((2, 16), dtype=np.uint64)
    with pytest.raises(N.ShapeError, match="cross-table lookups"):
        D.prove_stark(_CtlStark(16), config, trace, [0, 0, 0])


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


def _stark_case(kind, log_n):
    """(stark, host trace, public inputs, lookup challenges or None)."""
    from test_stark_lookups import RangeCheckStark, RangeCheckStark4

    if kind == "fib":
        stark = S.FibonacciStark(1 << log_n)
        trace = stark.generate_trace(0, 1)
        return stark, trace, [0, 1, int(trace[1, -1])], None
    challenges = [int(v) for v in synth(0x5C0 + log_n, (2,))]
    if kind == "range":
        return RangeCheckStark(), RangeCheckStark.generate_trace(log_n, seed=log_n), [0], challenges
    return RangeCheckStark4(), RangeCheckStark.generate_trace(log_n, seed=log_n, count_combination=False), [0], challenges


def _to_device(trace):
    import torch

    dev = torch.from_numpy(np.ascontiguousarray(trace).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return dev


class _Shards:
    """Every shard g < G of the trace (and auxiliary) commitment of one Stark, built in this process."""

    def __init__(self, ctx, stark, dev_trace, helpers, rate_bits, G):
        self.commits = []
        for g in range(G):
            t = S._commit_trace(dev_trace, rate_bits, CAP_HEIGHT, ctx, shard=(g, G))
            a = S.commit_auxiliary_polys(helpers, rate_bits, CAP_HEIGHT, ctx, shard=(g, G)) if helpers is not None else None
            self.commits.append((t, a))

    def close(self):
        for t, a in self.commits:
            t.close()
            if a is not None:
                a.close()


def _shard_values(ctx, stark, trace_c, aux_c, program, alphas, out):
    b, consts, al = program
    return N.lib().gl_stark_quotient_shard(ctx.h, trace_c.h, aux_c.h if aux_c is not None else None, b.program(),
                                           len(b.instrs), N.np_ptr(consts), len(consts), N.np_ptr(al), len(al),
                                           stark.quotient_degree_factor(), N.vp(out.data_ptr()))


def _from_shards(ctx, values, G, n_alphas, degree_bits, qdf, out):
    return N.lib().gl_stark_quotient_from_shards(ctx.h, N.vp(values.data_ptr()), G, n_alphas, degree_bits, qdf,
                                                 N.vp(out.data_ptr()))


def _sharded_quotient(pb, stark, trace, pis, challenges, rate_bits, G, alphas):
    """(the shards' quotient through gl_stark_quotient_from_shards, gl_stark_quotient's) as int64 CUDA tensors."""
    import torch

    ctx = pb.default_context()
    dev = _to_device(trace)
    helpers = S.compute_lookup_helper_columns(stark, dev, challenges, ctx) if challenges is not None else None
    log_n = dev.shape[1].bit_length() - 1
    whole_t = S._commit_trace(dev, rate_bits, CAP_HEIGHT, ctx)
    whole_a = S.commit_auxiliary_polys(helpers, rate_bits, CAP_HEIGHT, ctx) if helpers is not None else None
    args = dict(auxiliary_polys_commitment=whole_a, lookup_challenges=challenges) if helpers is not None else {}
    want = S.compute_quotient_polys(stark, whole_t, pis, alphas, **args)
    program = S.quotient_program(stark, pis, alphas, whole_a, challenges)
    qdf = stark.quotient_degree_factor()
    size = (1 << log_n) << (qdf - 1).bit_length()
    shards = _Shards(ctx, stark, dev, helpers, rate_bits, G)
    try:
        values = torch.empty((G, len(alphas), size // G), dtype=torch.int64, device="cuda")
        for g, (t, a) in enumerate(shards.commits):
            assert _shard_values(ctx, stark, t, a, program, alphas, values[g]) == N.GL_OK, N.lib().gl_last_error(ctx.h)
        got = torch.empty((len(alphas), size), dtype=torch.int64, device="cuda")
        rc = _from_shards(ctx, values, G, len(alphas), log_n, qdf, got)
        assert rc == N.GL_OK, N.lib().gl_last_error(ctx.h)
        ctx.synchronize()
    finally:
        shards.close()
        whole_t.close()
        if whole_a is not None:
            whole_a.close()
    return got, want


# (stark, log2 rows, rate_bits): FibonacciStark (quotient degree 1) computes its local values on every shard, and with
# G > 1 restricts the trace to shards smaller than n; RangeCheckStark (degree 3, quotient degree 2) reads them in place at
# rate 1 and computes them at rates 2 and 3; RangeCheckStark4 (quotient degree 4 at rate 2) reads both rows in place up
# to G = 4.
SHAPES = [("fib", 10, 1), ("fib", 13, 2), ("fib", 16, 3), ("range", 10, 1), ("range", 12, 2), ("range", 14, 3),
          ("range", 16, 1), ("range4", 11, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 2, 4, 8, 16])
@pytest.mark.parametrize("kind,log_n,rate_bits", SHAPES)
def test_sharded_quotient_equals_whole(pb, kind, log_n, rate_bits, G):
    import torch

    stark, trace, pis, challenges = _stark_case(kind, log_n)
    alphas = [int(v) for v in synth(0x5B0 + log_n, (2,))]
    got, want = _sharded_quotient(pb, stark, trace, pis, challenges, rate_bits, G, alphas)
    assert torch.equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,G", [("range", 8), ("fib", 4)])
def test_sharded_quotient_equals_whole_at_2_20(pb, kind, G):
    import torch

    stark, trace, pis, challenges = _stark_case(kind, 20)
    alphas = [int(v) for v in synth(0x5B1, (2,))]
    got, want = _sharded_quotient(pb, stark, trace, pis, challenges, 1, G, alphas)
    assert torch.equal(got, want)


@pytest.mark.gpu
def test_entry_point_errors(pb):
    """Trace and auxiliary shards that differ in index or count, unfinished handles, a shard count that is not a power
    of two: GL_ERR_BAD_ARG; too many challenges: GL_ERR_UNSUPPORTED. A broken trace passes gl_stark_quotient_shard on
    every shard and fails the trim check in gl_stark_quotient_from_shards, with gl_stark_quotient's message."""
    import torch

    from test_stark_lookups import SEL2

    ctx = pb.default_context()
    L = N.lib()
    stark, trace, pis, challenges = _stark_case("range", 10)
    alphas = [3, 4]
    dev = _to_device(trace)
    helpers = S.compute_lookup_helper_columns(stark, dev, challenges, ctx)
    t0 = S._commit_trace(dev, 1, CAP_HEIGHT, ctx, shard=(0, 2))
    program = S.quotient_program(stark, pis, alphas, t0, challenges)
    out = torch.empty((2, 1 << 10), dtype=torch.int64, device="cuda")
    made = [t0]
    for shard in [(1, 2), (0, 4), (0, 1)]:
        a = S.commit_auxiliary_polys(helpers, 1, CAP_HEIGHT, ctx, shard=shard)
        made.append(a)
        assert _shard_values(ctx, stark, t0, a, program, alphas, out) == N.GL_ERR_BAD_ARG, shard
        assert b"the auxiliary commitment is shard" in L.gl_last_error(ctx.h)
    a0 = S.commit_auxiliary_polys(helpers, 1, CAP_HEIGHT, ctx, shard=(0, 2))
    made.append(a0)
    assert _shard_values(ctx, stark, t0, a0, program, alphas, out) == N.GL_OK
    unfinished = []
    for B in (stark.COLUMNS, helpers.shape[0]):
        h = N.vp()
        N.check(L.gl_commit_begin(ctx.h, B, 10, 1, CAP_HEIGHT, 0, 0, 2, None, C.byref(h)), ctx.h)
        unfinished.append(h)

    class _H:
        def __init__(self, h):
            self.h = h

    assert _shard_values(ctx, stark, _H(unfinished[0]), a0, program, alphas, out) == N.GL_ERR_BAD_ARG
    assert b"not been called on the trace commitment" in L.gl_last_error(ctx.h)
    assert _shard_values(ctx, stark, t0, _H(unfinished[1]), program, alphas, out) == N.GL_ERR_BAD_ARG
    assert b"not been called on the auxiliary commitment" in L.gl_last_error(ctx.h)
    for h in unfinished:
        L.gl_commit_destroy(h)
    b, consts, _ = program
    five = np.arange(1, 6, dtype=np.uint64)
    assert L.gl_stark_quotient_shard(ctx.h, t0.h, a0.h, b.program(), len(b.instrs), N.np_ptr(consts), len(consts),
                                     N.np_ptr(five), 5, 2, N.vp(out.data_ptr())) == N.GL_ERR_UNSUPPORTED
    values = torch.zeros((2, 2, 1 << 10), dtype=torch.int64, device="cuda")
    whole = torch.empty((2, 1 << 11), dtype=torch.int64, device="cuda")
    assert _from_shards(ctx, values, 3, 2, 10, 2, whole) == N.GL_ERR_BAD_ARG
    assert _from_shards(ctx, values, 2, 0, 10, 2, whole) == N.GL_ERR_UNSUPPORTED
    assert _from_shards(ctx, values, 2, 2, 10, 0, whole) == N.GL_ERR_BAD_ARG
    for c in made:
        c.close()

    # RangeCheckStark4: quotient degree factor 3 on a coset of 4n points, so the top chunk must vanish
    stark4, trace4, pis4, challenges4 = _stark_case("range4", 10)
    trace4[SEL2, 9] = 2                                         # not boolean on row 9
    dev4 = _to_device(trace4)
    helpers4 = S.compute_lookup_helper_columns(stark4, dev4, challenges4, ctx)
    G = 4
    shards = _Shards(ctx, stark4, dev4, helpers4, 2, G)
    try:
        program4 = S.quotient_program(stark4, pis4, alphas, shards.commits[0][1], challenges4)
        values = torch.empty((G, 2, (4 << 10) // G), dtype=torch.int64, device="cuda")
        for g, (t, a) in enumerate(shards.commits):
            assert _shard_values(ctx, stark4, t, a, program4, alphas, values[g]) == N.GL_OK
        whole = torch.empty((2, 4 << 10), dtype=torch.int64, device="cuda")
        assert _from_shards(ctx, values, G, 2, 10, 3, whole) == N.GL_ERR_BAD_ARG
        assert b"Quotient has failed" in L.gl_last_error(ctx.h)
    finally:
        shards.close()


@pytest.mark.gpu
def test_prove_stark_on_one_rank_is_prove(pb):
    """Without a process group prove_stark is stark.prove: the same proof, field for field."""
    import stark_twin as T
    from test_stark_prove import _fib_case

    stark, config, trace, pi = _fib_case(10)
    assert not T.proof_diff(D.prove_stark(stark, config, trace, pi), S.prove(stark, config, trace, pi))


@pytest.mark.gpu
def test_prove_stark_across_ranks(pb):
    """torchrun, one rank per GPU (2, or 4 with four GPUs; the ranks share GPU 0 over gloo on a single-GPU machine):
    every rank's proof equals stark.prove's and the restated verifiers accept it; refusals on every rank."""
    run_ranks("mgpu_stark_check.py", "MGPU_STARK_CHECK OK", timeout=900)
