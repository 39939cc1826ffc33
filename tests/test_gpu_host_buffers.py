"""Where a caller's host buffers meet the library: an entry point that takes a GL_MEM_HOST input has read it when it
returns, whether the buffer is pageable or page-locked, so the caller may refill it at once. A copy from
page-locked memory is fully asynchronous (the DMA reads the buffer when the stream reaches the copy), so the entry
points that queue one and return without a synchronising read-back wait for that copy before they return (HostReads in
csrc/plonky2_b200.cu).

CPU: a static check over plonky2_b200/csrc/plonky2_b200.cu: every `int gl_...(` whose body copies host memory to the
device (device_in, h2d, upload_program, a HostToDevice copy, or a call to a function that does) is in COVERED, the
entry points this file runs from an overwritten page-locked buffer; or in SYNCHRONISED, whose bodies end in a
synchronising read-back (d2h, flag_status); or in LIBRARY_OWNED, whose copies read only the library's own memory.

GPU (-m gpu): torch's current stream spins for about 0.2 s and the library's stream is ordered after it
(Context.after_caller), so every copy the call queues waits behind the spin. The input sits in a page-locked buffer (a
numpy view of a pinned torch tensor) that is overwritten with its bitwise complement the moment the call returns; after
a synchronise the outputs are compared with the oracle's for the original input. Every case also runs from a pageable
copy of the same input. Cases: gl_commit_add_columns at 1 ... 73 columns per call (the single copy, the 8-column first
chunk, the 32-column chunks, a short last chunk) with device columns before them, padded strides, every column kind,
external coefficient storage, a pinned salt, 4 row-block shards and a non-resident handle; gl_commit_create_sharded at
the benchmarked 234 x 2^20 shape against its golden cap; gl_commit_create and gl_commit_finish with a pinned salt;
gl_merkle_build; gl_fri_begin_from_coeffs; gl_sigma_polys with pinned k_is and a device output;
PolynomialBatch.from_values / from_coeffs with a pinned salt and MerkleTree; and gl_ntt, gl_stark_quotient and
gl_poseidon_hash_many, which synchronise before they return."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

from conftest import P, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CU = os.path.join(ROOT, "plonky2_b200", "csrc", "plonky2_b200.cu")

# about 0.2 s of SM clock cycles at the H100's 1.98 GHz boost clock, as in tests/test_gpu_stream_order.py
SLEEP_CYCLES = 400_000_000

# entry points run here from a page-locked buffer overwritten on return, and the test that does it
COVERED = {
    "gl_commit_add_columns": "test_add_columns_reads_host_columns_before_returning",
    "gl_commit_create_sharded": "test_create_sharded_at_the_benchmarked_shape",
    "gl_commit_create": "test_create_and_finish_read_the_salt_before_returning",
    "gl_commit_finish": "test_create_and_finish_read_the_salt_before_returning",
    "gl_merkle_build": "test_merkle_build_reads_leaves_before_returning",
    "gl_fri_begin_from_coeffs": "test_fri_begin_from_coeffs_reads_coefficients_before_returning",
    "gl_sigma_polys": "test_sigma_polys_reads_k_is_before_returning",
    "gl_ntt": "test_synchronising_entry_points",
    "gl_stark_quotient": "test_synchronising_entry_points",
    "gl_poseidon_hash_many": "test_synchronising_entry_points",
}
# entry points whose host inputs are copied before a synchronising read-back (d2h or flag_status) in their own body or
# a helper's: the stream has passed the copies when they return
SYNCHRONISED = {
    "gl_poseidon_hash_no_pad_many": "hash_many_impl: d2h of the digests",
    "gl_poseidon_two_to_one_many": "hash_many_impl: d2h of the digests",
    "gl_poseidon_permute_many": "d2h of the permuted states",
    "gl_partial_products_and_zs": "flag_status after the k_is copy",
    "gl_lookup_polys": "flag_status",
    "gl_stark_quotient_aux": "stark_quotient: flag_status",
    "gl_stark_quotient_shard": "stark_quotient: flag_status",
    "gl_stark_lookup_helpers": "flag_status after the program upload",
    "gl_stark_ctl_helpers": "flag_status after the program upload",
    "gl_plonk_quotient": "plonk_quotient: run_quotient's flag_status",
    "gl_plonk_quotient_shard": "plonk_quotient: run_quotient's flag_status",
}
# entry points whose host-to-device copies read only memory the library owns
LIBRARY_OWNED = {
    "gl_commit_finish_keyed": "commit_finish copies no salt: it is drawn on the device",
    "gl_commit_finish_prefixed": "commit_finish copies no salt; the prefix is device memory",
    "gl_commit_open": "tree_open copies the leaf indices into the context's own pinned staging after a synchronise",
    "gl_merkle_open": "tree_open copies the leaf indices into the context's own pinned staging after a synchronise",
    "gl_fri_open": "tree_open copies the leaf indices into the context's own pinned staging after a synchronise",
    "gl_fri_begin": "the std::vector of PolyRef built in the call: pageable, staged before the copy returns",
    "gl_fri_begin_values": "the std::vector of ValRef built in the call: pageable, staged before the copy returns",
}

DIRECT_COPY = re.compile(r"\bdevice_in\(|\bh2d\(|\bupload_program\(|HostToDevice")
SYNC = re.compile(r"\bd2h\(|\bflag_status\(")


# ----------------------------------------------------------------------------------------------------------- CPU
def function_bodies(src):
    """{name: body} of every top-level `int name(...) {...}` / `static int name(...) {...}` definition."""
    out = {}
    for m in re.finditer(r"^(?:static\s+)?int\s+(\w+)\s*\(", src, re.M):
        brace = src.find("{", m.end())
        if brace < 0 or ";" in src[m.end():brace]:
            continue  # a declaration
        depth = 0
        for j in range(brace, len(src)):
            depth += {"{": 1, "}": -1}.get(src[j], 0)
            if depth == 0:
                out[m.group(1)] = src[brace:j + 1]
                break
    return out


def _reaching(bodies, pattern):
    """The functions whose body matches `pattern` or calls, directly or through others, one that does."""
    hit = {n for n, b in bodies.items() if pattern.search(b)}
    while True:
        more = {n for n, b in bodies.items() if n not in hit and any(re.search(r"\b%s\(" % h, b) for h in hit)}
        if not more:
            return hit
        hit |= more


def host_copying_entry_points(src):
    return sorted(n for n in _reaching(function_bodies(src), DIRECT_COPY) if n.startswith("gl_"))


def test_every_host_input_entry_point_is_covered_or_listed():
    with open(CU) as f:
        src = f.read()
    found = host_copying_entry_points(src)
    listed = set(COVERED) | set(SYNCHRONISED) | set(LIBRARY_OWNED)
    assert len(listed) == len(COVERED) + len(SYNCHRONISED) + len(LIBRARY_OWNED), "an entry point listed twice"
    assert sorted(set(found) - listed) == [], "a host-input entry point that no test here covers"
    assert sorted(listed - set(found)) == [], "a listed entry point that no longer copies from the host"
    syncing = _reaching(function_bodies(src), SYNC)
    assert sorted(n for n in SYNCHRONISED if n not in syncing) == []
    assert all(name in globals() for name in COVERED.values())


def test_the_static_check_follows_helpers():
    src = """
static int helper(gl_ctx* ctx, const u64* in) {
    if (x) { return h2d(ctx, d, in, 4); }
    return GL_OK;
}
static int indirect(gl_ctx* ctx) { return helper(ctx, nullptr); }
int gl_a(gl_ctx* ctx) { return indirect(ctx); }
int gl_b(gl_ctx* ctx, const u64* p) { CK(ctx, cudaMemcpyAsync(d, p, 8, cudaMemcpyHostToDevice, s)); return GL_OK; }
int gl_c(gl_ctx* ctx) { return gl_b(ctx, nullptr); }
int gl_d(gl_ctx* ctx);
int gl_e(gl_ctx* ctx) { return d2h(ctx, out, dev, 4); }
"""
    assert host_copying_entry_points(src) == ["gl_a", "gl_b", "gl_c"]


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


HOST = ["pinned", "pageable"]


def _host_buffer(a, host):
    """A host copy of `a` as uint64: a numpy view of a page-locked torch tensor, or a plain (pageable) numpy array."""
    import torch

    a = np.ascontiguousarray(a, dtype=np.uint64)
    if host == "pageable":
        return a.copy()
    t = torch.empty(a.shape, dtype=torch.int64, pin_memory=True)
    assert t.is_pinned()
    v = t.numpy().view(np.uint64)  # the view keeps the tensor alive
    v[...] = a
    return v


def _hold(ctx):
    """Queue about 0.2 s of spinning on torch's current stream and order the library's stream after it: the copies the
    next call queues wait behind the spin."""
    import torch

    torch.cuda.synchronize()
    torch.cuda._sleep(SLEEP_CYCLES)
    ctx.after_caller()
    assert not torch.cuda.current_stream().query(), "the spin finished before the entry point was called"


def _same(got, want, what):
    """Equal arrays, or an error naming the first differing element and how many differ."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.argwhere(got != want)
    assert len(bad) == 0, "%s: %d of %d elements differ; first at %s: %d, want %d" % (
        what, len(bad), want.size, tuple(bad[0]), got[tuple(bad[0])], want[tuple(bad[0])])


def _overwrite(*bufs):
    for b in bufs:
        np.bitwise_not(b, out=b)


def _dev(a):
    import torch

    t = torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


def _noncanonical(a):
    """The same residues with every element below 2^32 - 1 lifted by p (so >= p)."""
    return np.where(a < np.uint64(2**32 - 1), a + np.uint64(P), a)


def _read(fn, h, shape, *args):
    from plonky2_b200 import _native as N

    out = np.empty(shape, dtype=np.uint64)
    N.check(fn(h, *args, N.np_ptr(out), N.MEM_HOST), None)
    return out


# (count of host columns in the call, device columns before them, stride padding, kind, layout)
ADD_CASES = [
    (1, 0, 0, "values", "resident"),
    (8, 3, 0, "coeffs", "external"),
    (9, 0, 5, "canonical", "blocked"),
    (32, 2, 0, "values", "blinded"),
    (33, 0, 3, "coeffs", "sharded"),
    (40, 5, 0, "canonical", "resident"),
    (41, 1, 7, "values", "blocked"),
    (73, 4, 9, "coeffs", "blinded"),
    (73, 0, 2, "canonical", "external"),
    (41, 6, 0, "values", "sharded"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("host", HOST)
@pytest.mark.parametrize("count,first,pad,kind,layout", ADD_CASES,
                         ids=["%d-%d-%d-%s-%s" % c for c in ADD_CASES])
def test_add_columns_reads_host_columns_before_returning(pb, oracle, host, count, first, pad, kind, layout):
    """gl_commit_begin (or _begin_blocked with G = 4, or one handle per row-block shard of 4), columns [0, first) as
    canonical coefficients from the device, then columns [first, first + count) from a host buffer with row stride
    n + pad, overwritten on return; with blinding, gl_commit_finish from a pinned salt overwritten on return too. The
    coefficients, cap, digests and every leaf row (for shards: concatenated) equal the oracle's commitment."""
    import torch

    from plonky2_b200 import _native as N

    log_n, r, h, G = 10, 2, 4, 4
    n, B = 1 << log_n, first + count
    seed = 0x4B00 + count * 16 + first
    host_cols = synth(seed, (count, n))
    if kind == "values":
        coeffs = np.stack([oracle.ifft(c) for c in host_cols])
        arg, code = host_cols, N.COLS_VALUES
    else:
        coeffs = host_cols
        arg = _noncanonical(host_cols) if kind == "coeffs" else host_cols
        code = N.COLS_COEFFS if kind == "coeffs" else N.COLS_COEFFS_CANONICAL
    dev_coeffs = synth(seed + 1, (first, n))
    all_coeffs = np.concatenate([dev_coeffs, coeffs])
    padded = np.zeros((count, n + pad), dtype=np.uint64)
    padded[:, :n] = arg
    padded[:, n:] = synth(seed + 2, (count, pad))
    salt = synth(seed + 3, (4, n << r)) if layout == "blinded" else None
    o = oracle.Commit(all_coeffs, r, h, salt=salt, is_coeffs=True)

    ctx, L = pb.default_context(), N.lib()
    dev = _dev(dev_coeffs) if first else None
    storage = torch.zeros((B, n), dtype=torch.int64, device="cuda") if layout == "external" else None
    shards = range(G) if layout == "sharded" else [0]
    handles, caps, leaves = [], [], []
    try:
        for g in shards:
            hnd = N.vp()
            if layout == "blocked":
                N.check(L.gl_commit_begin_blocked(ctx.h, B, log_n, r, h, G, None, C.byref(hnd)), ctx.h)
            else:
                N.check(L.gl_commit_begin(ctx.h, B, log_n, r, h, int(salt is not None), g, len(shards),
                                          N.vp(storage.data_ptr()) if storage is not None else None, C.byref(hnd)),
                        ctx.h)
            handles.append(hnd)
            if first:
                N.check(L.gl_commit_add_columns(hnd, 0, first, N.vp(dev.data_ptr()), n, N.COLS_COEFFS_CANONICAL,
                                                N.MEM_DEVICE), ctx.h)
            buf = _host_buffer(padded, host)
            _hold(ctx)
            N.check(L.gl_commit_add_columns(hnd, first, count, N.np_ptr(buf), n + pad, code, N.MEM_HOST), ctx.h)
            _overwrite(buf)
            if salt is not None:
                sbuf = _host_buffer(salt, host)
                _hold(ctx)
                N.check(L.gl_commit_finish(hnd, N.np_ptr(sbuf), N.MEM_HOST), ctx.h)
                _overwrite(sbuf)
            else:
                N.check(L.gl_commit_finish(hnd, None, N.MEM_HOST), ctx.h)
            ctx.synchronize()
            rows = (n << r) // len(shards)
            caps.append(_read(L.gl_commit_cap, hnd, ((1 << h) // len(shards), 4)))
            leaves.append(_read(L.gl_commit_leaves, hnd, (rows, o.W), 0, rows))
            _same(_read(L.gl_commit_coeffs, hnd, (B, n)), o.coeffs, "coefficients")
        _same(np.concatenate(caps), o.cap, "cap")
        _same(np.concatenate(leaves), o.leaves, "leaves")
        if layout != "sharded":
            _same(_read(L.gl_commit_digests, handles[0], o.digests.shape), o.digests, "digests")
            # a block of leaf rows across the first row-block boundary, read on its own (rebuilt when non-resident)
            q = (n << r) // G
            _same(_read(L.gl_commit_leaves, handles[0], (16, o.W), q - 8, 16), o.leaves[q - 8:q + 8],
                  "leaves across the first row-block boundary")
        if storage is not None:
            _same(storage.cpu().numpy().view(np.uint64), o.coeffs, "external coefficient storage")
    finally:
        for hnd in handles:
            L.gl_commit_destroy(hnd)


@pytest.fixture(scope="module")
def cfg2():
    with open(os.path.join(ROOT, "tests", "golden", "fullscale_cfg2.json")) as f:
        fx = json.load(f)
    cfg = fx["config"]
    return cfg, synth(cfg["seed"], (cfg["columns"], 1 << cfg["log_n"])), np.array(fx["cap"], dtype=np.uint64)


@pytest.mark.gpu
@pytest.mark.parametrize("host", HOST)
def test_create_sharded_at_the_benchmarked_shape(pb, cfg2, host):
    """gl_commit_create_sharded(shard 0 of 1) from host columns of 234 x 2^20 overwritten on return, as bench.py's e2e
    key commits them: the cap equals the golden cap the CPU oracle computed for the original columns."""
    from plonky2_b200 import _native as N

    cfg, vals, cap = cfg2
    B, log_n, r, h = cfg["columns"], cfg["log_n"], cfg["rate_bits"], cfg["cap_height"]
    ctx, L = pb.default_context(), N.lib()
    buf = _host_buffer(vals, host)
    hnd = N.vp()
    _hold(ctx)
    N.check(L.gl_commit_create_sharded(ctx.h, N.np_ptr(buf), 1 << log_n, B, log_n, r, h, None, 0, N.MEM_HOST, 0, 1,
                                       C.byref(hnd)), ctx.h)
    try:
        _overwrite(buf)
        _same(_read(L.gl_commit_cap, hnd, cap.shape), cap, "cap")
    finally:
        L.gl_commit_destroy(hnd)


@pytest.mark.gpu
@pytest.mark.parametrize("host", HOST)
def test_create_and_finish_read_the_salt_before_returning(pb, oracle, host):
    """gl_commit_finish on its own: a blinded handle whose columns came from the device, finished from a host salt
    overwritten on return; and gl_commit_create from host columns and salt, both overwritten on return. Cap, digests
    and leaves equal the oracle's salted commitment."""
    from plonky2_b200 import _native as N

    log_n, r, h, B = 11, 1, 3, 5
    n = 1 << log_n
    vals, salt = synth(0x4C00, (B, n)), synth(0x4C01, (4, n << r))
    o = oracle.Commit(vals, r, h, salt=salt)
    ctx, L = pb.default_context(), N.lib()
    dev = _dev(vals)
    hnds = []
    try:
        hnd = N.vp()
        N.check(L.gl_commit_begin(ctx.h, B, log_n, r, h, 1, 0, 1, None, C.byref(hnd)), ctx.h)
        hnds.append(hnd)
        N.check(L.gl_commit_add_columns(hnd, 0, B, N.vp(dev.data_ptr()), n, N.COLS_VALUES, N.MEM_DEVICE), ctx.h)
        sbuf = _host_buffer(salt, host)
        _hold(ctx)
        N.check(L.gl_commit_finish(hnd, N.np_ptr(sbuf), N.MEM_HOST), ctx.h)
        _overwrite(sbuf)

        cbuf, sbuf = _host_buffer(vals, host), _host_buffer(salt, host)
        hnd = N.vp()
        _hold(ctx)
        N.check(L.gl_commit_create(ctx.h, N.np_ptr(cbuf), n, B, log_n, r, h, N.np_ptr(sbuf), 0, N.MEM_HOST,
                                   C.byref(hnd)), ctx.h)
        hnds.append(hnd)
        _overwrite(cbuf, sbuf)
        for hnd in hnds:
            _same(_read(L.gl_commit_cap, hnd, o.cap.shape), o.cap, "cap")
            _same(_read(L.gl_commit_digests, hnd, o.digests.shape), o.digests, "digests")
            _same(_read(L.gl_commit_leaves, hnd, o.leaves.shape, 0, n << r), o.leaves, "leaves")
    finally:
        for hnd in hnds:
            L.gl_commit_destroy(hnd)


@pytest.mark.gpu
@pytest.mark.parametrize("host", HOST)
def test_merkle_build_reads_leaves_before_returning(pb, oracle, host):
    """gl_merkle_build from host leaves overwritten on return: cap and digests equal the oracle's tree."""
    from plonky2_b200 import _native as N

    leaves = synth(0x4D00, (1 << 12, 9))
    digests, cap = oracle.merkle_build(leaves, 3)
    ctx, L = pb.default_context(), N.lib()
    buf = _host_buffer(leaves, host)
    m = N.vp()
    _hold(ctx)
    N.check(L.gl_merkle_build(ctx.h, N.np_ptr(buf), len(leaves), 9, 3, N.MEM_HOST, C.byref(m)), ctx.h)
    try:
        _overwrite(buf)
        _same(_read(L.gl_merkle_cap, m, cap.shape), cap, "cap")
        _same(_read(L.gl_merkle_digests, m, digests.shape), digests, "digests")
    finally:
        L.gl_merkle_destroy(m)


@pytest.mark.gpu
@pytest.mark.parametrize("host", HOST)
def test_fri_begin_from_coeffs_reads_coefficients_before_returning(pb, oracle, host):
    """gl_fri_begin_from_coeffs from host F_{p^2} coefficients (non-canonical words among them) overwritten on return:
    gl_fri_coeffs gives them back canonical, and the first round's values are the oracle's coset LDE of them (each
    component on its own, shifted by the multiplicative group generator), in bit-reversed order."""
    from plonky2_b200 import _native as N
    from plonky2_b200.field import coset_shift, reverse_bits

    log_n, r, h = 10, 2, 3
    n, NN = 1 << log_n, 1 << (log_n + r)
    coeffs = synth(0x4E00, (n, 2))
    ctx, L = pb.default_context(), N.lib()
    buf = _host_buffer(_noncanonical(coeffs), host)
    f = N.vp()
    _hold(ctx)
    N.check(L.gl_fri_begin_from_coeffs(ctx.h, N.np_ptr(buf), log_n, r, h, C.byref(f)), ctx.h)
    try:
        _overwrite(buf)
        got = np.empty(2 * n, dtype=np.uint64)
        N.check(L.gl_fri_coeffs(f, N.np_ptr(got)), ctx.h)
        _same(got.reshape(n, 2), coeffs, "coefficients")
        vals = np.empty(2 * NN, dtype=np.uint64)
        ln = C.c_size_t()
        N.check(L.gl_fri_values_local(f, N.np_ptr(vals), vals.size, C.byref(ln)), ctx.h)
        assert ln.value == NN
        pad = np.zeros((2, NN), dtype=np.uint64)
        pad[:, :n] = coeffs.T
        nat = np.stack([oracle.coset_fft(pad[k], coset_shift()) for k in range(2)], axis=1)
        want = nat[[reverse_bits(j, log_n + r) for j in range(NN)]]
        _same(vals.reshape(NN, 2), want, "first-round values")
    finally:
        L.gl_fri_destroy(f)


@pytest.mark.gpu
@pytest.mark.parametrize("host", HOST)
def test_sigma_polys_reads_k_is_before_returning(pb, host):
    """gl_sigma_polys with no copy constraints (so no flag read-back synchronises the call), k_is in a host buffer
    overwritten on return and the output on the device: the identity sigmas k_is[c] * w^r of the restatement."""
    import torch

    from plonky2_b200 import _native as N
    from plonky2_b200 import plonk
    from plonky2_b200.plonk import get_unique_coset_shifts
    from test_circuit_data import _want

    cfg, db = plonk.CircuitConfig(num_wires=12, num_routed_wires=8), 11
    n, nr = 1 << db, cfg.num_routed_wires
    ctx, L = pb.default_context(), N.lib()
    k = _host_buffer(np.array(get_unique_coset_shifts(nr), dtype=np.uint64), host)
    out = torch.zeros((nr, n), dtype=torch.int64, device="cuda")
    _hold(ctx)
    N.check(L.gl_sigma_polys(ctx.h, None, 0, N.MEM_HOST, cfg.num_wires, nr, db, 0, N.np_ptr(k),
                             N.vp(out.data_ptr()), N.MEM_DEVICE), ctx.h)
    _overwrite(k)
    ctx.synchronize()
    _same(out.cpu().numpy().view(np.uint64), _want(cfg, db, np.zeros((0, 2), dtype=np.int64), literal=True), "sigmas")


@pytest.mark.gpu
@pytest.mark.parametrize("host", HOST)
def test_python_batches_and_trees_read_host_arrays_before_returning(pb, oracle, host):
    """PolynomialBatch.from_values and from_coeffs (which skip the wait on the library's stream) with host columns and
    salt, and MerkleTree, from buffers overwritten on return: equal to the oracle's commitments and tree."""
    log_n, r, h, B = 10, 3, 4, 6
    n = 1 << log_n
    ctx = pb.default_context()
    for is_coeffs in (False, True):
        vals, salt = synth(0x4F00 + is_coeffs, (B, n)), synth(0x4F10 + is_coeffs, (4, n << r))
        o = oracle.Commit(vals, r, h, salt=salt, is_coeffs=is_coeffs)
        cbuf, sbuf = _host_buffer(vals, host), _host_buffer(salt, host)
        make = pb.PolynomialBatch.from_coeffs if is_coeffs else pb.PolynomialBatch.from_values
        _hold(ctx)
        c = make(cbuf, r, True, h, salt=sbuf, ctx=ctx)
        _overwrite(cbuf, sbuf)
        try:
            _same(c.merkle_tree.cap.hashes, o.cap, ("cap", is_coeffs))
            _same(c.polynomials, o.coeffs, ("coefficients", is_coeffs))
            _same(c.merkle_tree.leaves, o.leaves, ("leaves", is_coeffs))
        finally:
            c.close()

    leaves = synth(0x4F20, (1 << 11, 7))
    digests, cap = oracle.merkle_build(leaves, 2)
    buf = _host_buffer(leaves, host)
    _hold(ctx)
    t = pb.MerkleTree(buf, 2, ctx)
    _overwrite(buf)
    try:
        _same(t.cap.hashes, cap, "cap")
        _same(t.digests, digests.reshape(t.digests.shape), "digests")
        _same(t.leaves, leaves, "leaves")  # the tree's own leaves, not the caller's refilled buffer
    finally:
        t.close()


@pytest.mark.gpu
@pytest.mark.parametrize("host", HOST)
def test_synchronising_entry_points(pb, oracle, host):
    """Entry points that end in a synchronising read-back, with page-locked inputs overwritten on return: gl_ntt on a
    host buffer (in and out: its contents on return are the oracle's inverse transform), gl_stark_quotient with the
    program's constants (the public inputs among them) in a host buffer, gl_poseidon_hash_many from host rows."""
    import stark_twin as T

    from plonky2_b200 import _native as N
    from plonky2_b200 import stark as S

    ctx, L = pb.default_context(), N.lib()
    x = synth(0x5000, (3, 1 << 11))
    buf = _host_buffer(x, host)
    _hold(ctx)
    N.check(L.gl_ntt(ctx.h, N.np_ptr(buf), 11, 3, 1 << 11, 1, 0, 1, N.MEM_HOST), ctx.h)
    got = buf.copy()
    _overwrite(buf)
    _same(got, np.stack([oracle.ifft(v) for v in x]), "inverse NTT")

    from test_stark_prove import _fib_case

    stark, config, trace, pi = _fib_case(10)
    f = config.fri_config
    tc = S._commit_trace(_dev(trace), f.rate_bits, f.cap_height, ctx)
    try:
        alphas = [int(v) for v in synth(0x5001, (config.num_challenges,))]
        want = T.quotient(oracle, stark, oracle.Commit(trace, f.rate_bits, f.cap_height), pi, alphas)
        b, consts, al = S.quotient_program(stark, pi, alphas)
        import torch

        out = torch.empty(want.shape, dtype=torch.int64, device="cuda")
        cbuf = _host_buffer(consts, host)
        _hold(ctx)
        N.check(L.gl_stark_quotient(ctx.h, tc.h, b.program(), len(b.instrs), N.np_ptr(cbuf), len(consts),
                                    N.np_ptr(al), len(al), stark.quotient_degree_factor(), N.vp(out.data_ptr())), ctx.h)
        _overwrite(cbuf)
        ctx.synchronize()
        _same(out.cpu().numpy().view(np.uint64), want, "quotient")
    finally:
        tc.close()

    rows = synth(0x5002, (1 << 12, 11))
    buf = _host_buffer(rows, host)
    out = np.empty((len(rows), 4), dtype=np.uint64)
    _hold(ctx)
    N.check(L.gl_poseidon_hash_many(ctx.h, N.np_ptr(buf), len(rows), 11, N.np_ptr(out), N.MEM_HOST), ctx.h)
    _overwrite(buf)
    _same(out, oracle.hash_many(rows), "digests")
