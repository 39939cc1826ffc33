"""The boundary where a caller's torch CUDA tensors meet the library: the library's context runs on its own stream, so
every function that hands a torch tensor to it -- to read, or to write into memory torch allocated -- first orders that
stream after torch's current stream (Context.after_caller).

CPU: a static check over plonky2_b200/*.py: every function that passes a data_ptr() to the library calls after_caller
before its first library call (an explicit allowlist names the exceptions, each with its reason); the check itself
flags a function that omits the call or makes it too late.

GPU (-m gpu): a delayed producer. The destination starts out holding another well-formed input; torch's current stream
then spins for about 0.2 s (torch.cuda._sleep) before it copies the real input in, and the entry point is called at
once, with no synchronisation. The spin is asserted to be still pending when the call starts, and the result is compared
bit for bit with the CPU reference: a library that read before the copy landed would prove or compute the other input.
Cases: stark.prove (FibonacciStark; the logUp STARK; a transposed, non-contiguous trace; the producer on a side stream),
prove_with_ctls, the lookup and CTL helper columns, the auxiliary and quotient-chunk commitments, the sigma polynomials
from device pairs, and write-after-read on an `out=` tensor and on a block the allocator hands back."""
import ast
import glob
import os

import numpy as np
import pytest

import stark_twin as T
from conftest import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# about 0.2 s of SM clock cycles at the H100's 1.98 GHz boost clock: longer than any entry point's host-side prelude
SLEEP_CYCLES = 400_000_000

# functions that pass a data_ptr() to the library without after_caller, and why that is right
ALLOWLIST = {
    "distributed.PipelinedCommitter.commit": "its context must run on the torch stream current at commit() (checked by "
                                             "_check_stream), and it orders its copy and side streams with events",
}


# ----------------------------------------------------------------------------------------------------------- CPU
def _functions(tree):
    """(qualified name, node) of every module-level function and method; nested functions belong to their outer one."""
    for node in tree.body:
        if isinstance(node, ast.FunctionDef):
            yield node.name, node
        elif isinstance(node, ast.ClassDef):
            for m in node.body:
                if isinstance(m, ast.FunctionDef):
                    yield "%s.%s" % (node.name, m.name), m


def _is_lib_call(call):
    f = call.func
    return (isinstance(f, ast.Attribute) and f.attr == "lib" and isinstance(f.value, ast.Name) and f.value.id == "N") or (
        isinstance(f, ast.Name) and f.id == "lib")


def _attr_calls(fn, attr):
    return [n for n in ast.walk(fn) if isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute) and n.func.attr == attr]


def unordered_entry_points(source, module):
    """The functions of `source` that call .data_ptr() but do not call .after_caller() before their first N.lib() call
    (in source order, nested functions included), as 'module.function' names."""
    out = []
    for name, fn in _functions(ast.parse(source)):
        if not _attr_calls(fn, "data_ptr"):
            continue
        pos = lambda n: (n.lineno, n.col_offset)  # noqa: E731
        libs = [pos(n) for n in ast.walk(fn) if isinstance(n, ast.Call) and _is_lib_call(n)]
        waits = [pos(n) for n in _attr_calls(fn, "after_caller")]
        if not waits or (libs and min(waits) > min(libs)):
            out.append("%s.%s" % (module, name))
    return out


def _package_sources():
    for path in sorted(glob.glob(os.path.join(ROOT, "plonky2_b200", "*.py"))):
        with open(path) as f:
            yield os.path.splitext(os.path.basename(path))[0], f.read()


def test_every_tensor_entry_point_orders_after_the_caller():
    flagged = [name for module, src in _package_sources() for name in unordered_entry_points(src, module)]
    assert sorted(set(flagged) - set(ALLOWLIST)) == []
    # every allowlisted function still exists and still hands a pointer to the library
    assert sorted(set(ALLOWLIST) - set(flagged)) == []


def test_the_static_check_flags_a_missing_or_late_wait():
    src = '''
def missing(t, ctx):
    N.check(N.lib().gl_x(ctx.h, N.vp(t.data_ptr())))

def late(t, ctx):
    N.check(N.lib().gl_x(ctx.h, N.vp(t.data_ptr())))
    ctx.after_caller()

def in_closure(t, ctx):
    def add(h):
        N.check(N.lib().gl_y(h, N.vp(t.data_ptr())))
    ctx.after_caller()
    return run(add)

def ordered(t, ctx):
    ctx.after_caller()
    def add(h):
        N.check(N.lib().gl_y(h, N.vp(t.data_ptr())))
    return run(add)

class K:
    def method(self, t):
        L = N.lib()
        self.ctx.after_caller()
        L.gl_z(N.vp(t.data_ptr()))

def host_only(a, ctx):
    N.check(N.lib().gl_x(ctx.h, N.np_ptr(a)))
'''
    assert unordered_entry_points(src, "m") == ["m.missing", "m.late", "m.in_closure", "m.K.method"]


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
    """A host uint64 array as a torch int64 CUDA tensor, complete on return."""
    import torch

    t = torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


def _host(t):
    return t.cpu().numpy().view(np.uint64)


def _delayed(*copies):
    """Queue on torch's current stream a spin of SLEEP_CYCLES, then dst.copy_(src) for every (dst, src); assert that
    the stream is still busy, so that the call that follows starts while the copies are pending."""
    import torch

    torch.cuda.synchronize()              # the destinations' earlier contents are complete: a stale read is well formed
    torch.cuda._sleep(SLEEP_CYCLES)
    for dst, src in copies:
        dst.copy_(src)
    assert not torch.cuda.current_stream().query(), "the producer finished before the entry point was called"


def _fib():
    from test_stark_prove import _fib_case

    return _fib_case(10)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["contiguous", "transposed", "side_stream"])
def test_prove_reads_a_trace_still_in_production(pb, oracle, layout):
    """stark.prove on FibonacciStark from a torch trace whose copy is still queued: equal to the CPU twin field for
    field and accepted by the restated verifier. transposed: the trace is a (COLUMNS, n) view of an (n, COLUMNS)
    tensor, so prove's own .contiguous() copy is queued on the caller's stream too. side_stream: the producer and the
    call run under `with torch.cuda.stream(s)`, so ordering after the default stream would not be enough."""
    import torch

    from plonky2_b200 import stark as S

    stark, config, _, _ = _fib()
    x0, x1 = {"contiguous": (0, 1), "transposed": (5, 8), "side_stream": (13, 21)}[layout]
    trace = stark.generate_trace(x0, x1)       # a trace of its own: no block another case freed holds it
    pi = [x0, x1, int(trace[1, -1])]
    stale = stark.generate_trace(2, 3)
    decoy = None
    if layout == "transposed":
        src, buf = _dev(trace.T), _dev(stale.T)
        arg = buf.t()
        assert not arg.is_contiguous()
        # a stale trace in the layout prove's .contiguous() copy writes, freed below so that the copy likely gets its
        # block; making it also loads torch's transposing copy kernel, whose first launch could block the host
        decoy = buf.t().contiguous()
    else:
        src, buf = _dev(trace), _dev(stale)
        arg = buf
    s = torch.cuda.Stream() if layout == "side_stream" else torch.cuda.current_stream()
    with torch.cuda.stream(s):
        _delayed((buf, src))
        del decoy
        proof = S.prove(stark, config, arg, pi)
    T.assert_matches_twin(proof, T.twin_prove(oracle, stark, config, trace, pi))
    assert T.verify(oracle, stark, config, proof) is None


@pytest.mark.gpu
def test_prove_with_lookups_reads_a_trace_still_in_production(pb, oracle):
    """stark.prove for the logUp range-check STARK from a torch trace still being copied: _device_trace, the lookup
    helper columns and the auxiliary commitment all read it; equal to the CPU twin and accepted."""
    from test_stark_lookups import RangeCheckStark, _range_case

    from plonky2_b200 import stark as S

    stark, config, trace, pi = _range_case(10)
    src, buf = _dev(trace), _dev(RangeCheckStark.generate_trace(10, seed=8))
    _delayed((buf, src))
    proof = S.prove(stark, config, buf, pi)
    T.assert_matches_twin(proof, T.twin_prove(oracle, stark, config, trace, pi))
    assert T.verify(oracle, stark, config, proof) is None


@pytest.mark.gpu
def test_prove_with_ctls_reads_traces_still_in_production(pb, oracle):
    """prove_with_ctls with every table's trace a torch tensor still being copied: equal to the multi-STARK twin and
    accepted by the restated verifier."""
    from test_stark_ctl import system, system_traces

    from plonky2_b200 import cross_table_lookup as X

    starks, config, ctls = system()
    traces, pis = system_traces()
    stale, _ = system_traces(seed=4)
    srcs, bufs = [_dev(t) for t in traces], [_dev(t) for t in stale]
    _delayed(*zip(bufs, srcs))
    mp = X.prove_with_ctls(starks, config, bufs, ctls, pis)
    T.assert_matches_twin(mp, T.twin_prove_with_ctls(oracle, starks, config, traces, ctls, pis))
    assert T.verify_with_ctls(oracle, starks, config, ctls, mp) is None


@pytest.mark.gpu
def test_helper_columns_read_a_trace_still_in_production(pb):
    """compute_lookup_helper_columns and compute_ctl_helper_columns from a trace still being copied, against the
    restatements of lookup_helper_columns and cross_table_lookup_data."""
    import torch

    from test_stark_ctl import _groups_and_aux, _pairs, system_ctls, system_traces
    from test_stark_lookups import RangeCheckStark

    from plonky2_b200 import cross_table_lookup as X
    from plonky2_b200 import stark as S
    from plonky2_b200.lookup import GrandProductChallenge

    ctx = pb.default_context()
    stark, trace = RangeCheckStark(), RangeCheckStark.generate_trace(10, seed=10)
    challenges = [int(v) for v in synth(0x9A0, (2,))]
    src, buf = _dev(trace), _dev(RangeCheckStark.generate_trace(10, seed=11))
    _delayed((buf, src))
    got = S.compute_lookup_helper_columns(stark, buf, challenges, ctx)
    assert np.array_equal(_host(got), T.aux_columns(stark, trace, challenges)[0])

    traces, _ = system_traces()
    stale, _ = system_traces(seed=4)
    ctls, pairs = system_ctls(), _pairs(0x9A1)
    groups, want = _groups_and_aux(traces, ctls, 0, pairs, 3)
    src, buf = _dev(traces[0]), _dev(stale[0])
    out = torch.empty(want.shape, dtype=torch.int64, device="cuda")
    _delayed((buf, src))
    X.compute_ctl_helper_columns(buf, groups, [GrandProductChallenge(*p) for p in pairs], 3, ctx, out)
    assert np.array_equal(_host(out), want)


@pytest.mark.gpu
def test_commitments_read_columns_still_in_production(pb, oracle):
    """commit_auxiliary_polys (value columns) and PolynomialBatch._from_coeff_chunks (rows cut into coefficient chunks)
    from tensors still being copied: the caps and coefficients equal the oracle's commitment of the same columns."""
    from plonky2_b200 import stark as S
    from plonky2_b200.polynomial_batch import PolynomialBatch

    ctx = pb.default_context()
    values = synth(0x9B0, (6, 1 << 10))
    src, buf = _dev(values), _dev(synth(0x9B1, (6, 1 << 10)))
    _delayed((buf, src))
    c = S.commit_auxiliary_polys(buf, 1, 4, ctx)
    try:
        o = oracle.Commit(values, 1, 4)
        assert np.array_equal(c.merkle_tree.cap.hashes, o.cap) and np.array_equal(c.polynomials, o.coeffs)
    finally:
        c.close()

    chunks, n = 3, 1 << 9
    polys = synth(0x9B2, (2, chunks * n))
    src, buf = _dev(polys), _dev(synth(0x9B3, (2, chunks * n)))
    _delayed((buf, src))
    c = PolynomialBatch._from_coeff_chunks(buf, chunks, 9, 2, 3, ctx)
    try:
        o = oracle.Commit(polys.reshape(2 * chunks, n), 2, 3, is_coeffs=True)
        assert np.array_equal(c.merkle_tree.cap.hashes, o.cap) and np.array_equal(c.polynomials, o.coeffs)
    finally:
        c.close()


@pytest.mark.gpu
def test_sigma_polys_read_pairs_still_in_production(pb):
    """plonk.sigma_polys from device copy-constraint pairs still being copied, against the literal restatement."""
    from test_circuit_data import _want, random_pairs

    from plonky2_b200 import plonk

    cfg, db = plonk.CircuitConfig(num_wires=12, num_routed_wires=8), 6
    pairs = random_pairs(np.random.default_rng(0), 12, 8, db, 40, 200)
    stale = random_pairs(np.random.default_rng(1), 12, 8, db, 40, 200)
    src, buf = _dev(pairs.astype(np.uint64)), _dev(stale.astype(np.uint64))
    _delayed((buf, src))
    got = plonk.sigma_polys(cfg, db, buf, 40)
    assert np.array_equal(_host(got), _want(cfg, db, pairs, 40, literal=True))


@pytest.mark.gpu
def test_out_tensor_is_written_after_the_callers_reads(pb):
    """Write after read: `out` holds old values that a copy queued behind the spin still has to read; the lookup helper
    columns written into it must land after that read. The snapshot keeps the old values, `out` the new ones."""
    import torch

    from test_stark_lookups import RangeCheckStark

    from plonky2_b200 import stark as S

    ctx = pb.default_context()
    stark, trace = RangeCheckStark(), RangeCheckStark.generate_trace(10, seed=12)
    challenges = [int(v) for v in synth(0x9C0, (2,))]
    want = T.aux_columns(stark, trace, challenges)[0]
    dev = _dev(trace)
    old = synth(0x9C1, want.shape)
    out, snapshot = _dev(old), _dev(np.zeros_like(old))
    _delayed((snapshot, out))
    S.compute_lookup_helper_columns(stark, dev, challenges, ctx, out=out)
    assert np.array_equal(_host(snapshot), old)
    assert np.array_equal(_host(out), want)


@pytest.mark.gpu
def test_reused_block_is_written_after_the_callers_reads(pb, oracle):
    """Write after read on memory the library's caller allocates: a tensor of the quotient's shape is freed with a read
    still queued on it, and compute_quotient_polys's output takes its block from torch's caching allocator. The
    queued read still sees the old values and the quotient equals the oracle's."""
    import torch

    from plonky2_b200 import stark as S

    ctx = pb.default_context()
    stark, config, trace, pi = _fib()
    f = config.fri_config
    tc = S._commit_trace(_dev(trace), f.rate_bits, f.cap_height, ctx)
    try:
        alphas = [int(v) for v in synth(0x9D0, (config.num_challenges,))]
        want = T.quotient(oracle, stark, oracle.Commit(trace, f.rate_bits, f.cap_height), pi, alphas)
        old = synth(0x9D1, want.shape)
        victim, snapshot = _dev(old), _dev(np.zeros_like(old))
        _delayed((snapshot, victim))
        block = victim.data_ptr()
        del victim
        q = S.compute_quotient_polys(stark, tc, pi, alphas)
        reused = q.data_ptr() == block
        assert np.array_equal(_host(snapshot), old)
        assert np.array_equal(_host(q), want)
    finally:
        tc.close()
    if not reused:
        pytest.skip("the caching allocator did not hand the freed block to the quotient")
