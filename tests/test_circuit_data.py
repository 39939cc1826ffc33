"""Circuit data from a placed circuit: blind_and_pad, the sigma polynomials (gl_sigma_polys), the constants/sigmas
commitment and the circuit digest (plonk.build_circuit_data, distributed.build_circuit_data).

CPU: a literal restatement of Forest + wire_partition + get_sigma_map (plonk/permutation_argument.rs, union-find with
insertion-ordered sets) against a vectorised one (scipy connected components + stable argsort) on small random
circuits with virtual targets bridging sets, duplicate pairs and self-pairs; the header's index code run on the host
(tests/emu/sigma_emu.cpp) against the restatement; the digest against the oracle's Poseidon; blind_and_pad against
tests/plonk_circuits.zk_circuit; every refusal of gl_sigma_polys raised before the context is used.

GPU (-m gpu): gl_sigma_polys bit-equal to the restatement on every FibonacciCircuit shape, LargeCircuit at 2^18 gates,
no constraints, one set of every routed wire, a 2^22-edge descending chain, random graphs joined by virtual targets,
host and device pairs; the constants/sigmas commitment against PolynomialBatch.from_values; shards concatenating to the
unsharded commitment; build_circuit_data -> prove_with_witness accepted by the restated verifiers (with and without
zero knowledge) only under the built digest; distributed.build_circuit_data + prove_plonk across torchrun ranks
(tests/mgpu_circuit_data_check.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import gl_numpy as gn
import oracle_lib as OL
import plonk_circuits as PC
from conftest import synth
from plonk_circuits import instances_of, pairs_from_sigmas
from plonky2_b200 import _native as N
from ranks import run_ranks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _plonk():
    from plonky2_b200 import plonk

    return plonk


# ------------------------------------------------------------------------------------------------ restatements
def forest_sigma_map(num_wires, num_routed, degree_bits, num_virtual, pairs):
    """Forest (permutation_argument.rs:12-101) and get_sigma_map (:129-157), literally: add every target, merge each
    pair, compress, collect the routed wires into sets in row-major order; each wire maps to the next of its set.
    pairs: Target::index values. Returns the sigma map col' * n + row' at index col * n + row."""
    n = 1 << degree_bits
    parents = list(range(num_wires * n + num_virtual))

    def find(x):
        rep = x
        while parents[rep] != rep:
            rep = parents[rep]
        while parents[x] != x:
            parents[x], x = rep, parents[x]
        return rep

    for a, b in pairs:
        x, y = find(int(a)), find(int(b))
        if x != y:
            parents[y] = x
    for i in range(len(parents)):
        find(i)
    partition = {}
    for row in range(n):
        for col in range(num_routed):
            partition.setdefault(parents[row * num_wires + col], []).append((row, col))
    neighbors = {}
    for subset in partition.values():
        for k, w in enumerate(subset):
            neighbors[w] = subset[(k + 1) % len(subset)]
    out = np.empty(num_routed * n, dtype=np.uint64)
    for col in range(num_routed):
        for row in range(n):
            r, c = neighbors[(row, col)]
            out[col * n + row] = c * n + r
    return out


def component_labels(num_targets, pairs):
    """Connected components of the targets under the pairs (scipy), one label per target."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components

    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    g = coo_matrix((np.ones(len(pairs), dtype=np.int8), (pairs[:, 0], pairs[:, 1])), shape=(num_targets, num_targets))
    return connected_components(g, directed=False)[1]


def vector_sigma_map(num_wires, num_routed, degree_bits, num_virtual, pairs):
    """forest_sigma_map, vectorised: the routed wires sorted stably by component, each mapped to its successor in the
    sorted order (the first of its component for the last)."""
    n = 1 << degree_bits
    labels = component_labels(num_wires * n + num_virtual, pairs)
    i = np.arange(n * num_routed, dtype=np.int64)                       # routed index row * num_routed + col
    keys = labels[(i // num_routed) * num_wires + i % num_routed]
    order = np.argsort(keys, kind="stable")
    sk = keys[order]
    head = np.r_[True, sk[1:] != sk[:-1]]
    first = np.maximum.accumulate(np.where(head, np.arange(len(sk)), 0))
    last = np.r_[sk[1:] != sk[:-1], True]
    succ = np.where(last, order[first], np.r_[order[1:], 0])
    out = np.empty(n * num_routed, dtype=np.uint64)
    out[(order % num_routed) * n + order // num_routed] = (succ % num_routed) * n + succ // num_routed
    return out


def sigma_values(sigma_map, k_is, degree_bits):
    """get_sigma_polys (permutation_argument.rs:113-127): k_is[m / n] * w^(m mod n), as (num_routed, n)."""
    n = 1 << degree_bits
    subgroup = gn.powers(PC.root_of_unity(degree_bits), n)
    m = sigma_map.astype(np.int64)
    return gn.mul(np.array(k_is, dtype=np.uint64)[m // n], subgroup[m % n]).reshape(len(k_is), n)


def random_pairs(rng, num_wires, num_routed, degree_bits, num_virtual, count):
    """Random copy constraints over routed wires and virtual targets, with duplicates and self-pairs."""
    n = 1 << degree_bits
    pool = [r * num_wires + c for r in range(n) for c in range(num_routed)]
    pool += [n * num_wires + v for v in range(num_virtual)]
    pool = np.array(pool, dtype=np.int64)
    pairs = pool[rng.integers(0, len(pool), size=(count, 2))]
    pairs = np.concatenate([pairs, pairs[:3], pairs[:2, :1].repeat(2, 1)])       # duplicates, self-pairs
    # virtual targets that bridge: v joins two wires that no other pair joins
    if num_virtual:
        v = n * num_wires + num_virtual - 1
        pairs = np.concatenate([pairs, [[pool[0], v], [v, pool[len(pool) // 2]]]])
    return pairs


# ----------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("seed", range(6))
def test_restatements_agree_on_random_circuits(seed):
    rng = np.random.default_rng(seed)
    nw, nr, db, nv = 7, 4 + seed % 3, 2 + seed % 3, [0, 3, 9][seed % 3]
    pairs = random_pairs(rng, nw, nr, db, nv, 3 + 5 * seed)
    want = forest_sigma_map(nw, nr, db, nv, pairs)
    assert np.array_equal(vector_sigma_map(nw, nr, db, nv, pairs), want)
    # a non-routed wire bridging two sets joins them too (the reference merges every target)
    n = 1 << db
    bridge = np.array([[0 * nw + nr, 0], [0 * nw + nr, (n - 1) * nw + nr - 1]])
    both = np.concatenate([pairs, bridge])
    got = forest_sigma_map(nw, nr, db, nv, both)
    assert np.array_equal(vector_sigma_map(nw, nr, db, nv, both), got)
    assert got[0] != 0 or n * nr == 1


def test_restatement_is_the_test_circuits_sigmas():
    """On circuits whose cycles the tests wrote in row-major order, the restatement gives their sigmas."""
    plonk = _plonk()
    for c in (PC.FibonacciCircuit(plonk, plonk.CircuitConfig(num_wires=12, num_routed_wires=8,
                                                              max_quotient_degree_factor=4, rate_bits=2), 5),
              PC.FibonacciCircuit(plonk, plonk.CircuitConfig(num_wires=135, num_routed_wires=80), 5, poseidon_rows=3)):
        cfg = c.config
        pairs = pairs_from_sigmas(c)
        m = vector_sigma_map(cfg.num_wires, cfg.num_routed_wires, c.common.degree_bits, 0, pairs)
        assert np.array_equal(sigma_values(m, c.common.k_is, c.common.degree_bits), c.sigmas)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("sigma_emu") / "libsigma_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "emu", "sigma_emu.cpp")])
    L = C.CDLL(out)
    L.emu_sigma_map.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.c_void_p]
    L.emu_sigma_check.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.c_void_p]
    return L


@pytest.mark.parametrize("seed", range(4))
def test_header_index_code_on_host(emu, seed):
    rng = np.random.default_rng(100 + seed)
    nw, nr, db, nv = 9, 5, 3 + seed % 2, 4 * seed
    pairs = random_pairs(rng, nw, nr, db, nv, 10 * (seed + 1))
    T = (nw << db) + nv
    # any representative: scipy's labels, shuffled
    labels = np.random.default_rng(seed).permutation(T).astype(np.uint32)[component_labels(T, pairs)]
    labels = np.ascontiguousarray(labels, dtype=np.uint32)
    got = np.empty(nr << db, dtype=np.uint64)
    emu.emu_sigma_map(labels.ctypes.data, nw, nr, db, T, got.ctypes.data)
    assert np.array_equal(got, forest_sigma_map(nw, nr, db, nv, pairs))
    # wire (0, 0), (0, nr - 1), (0, nr), (0, nw - 1), (1, 0), the last wire, the first and last virtual target (or
    # one past the targets without any), one past the targets, a far index
    t = np.array([0, nr - 1, nr, nw - 1, nw, (nw << db) - 1, nw << db, T - 1, T, 2**40], dtype=np.uint64)
    flags = np.empty(len(t), dtype=np.uint32)
    emu.emu_sigma_check(t.ctypes.data, len(t), nw, nr, db, T, flags.ctypes.data)
    virtual = [0, 0] if nv else [1, 2]
    assert flags.tolist() == [0, 0, 2, 2, 0, 2] + virtual + [1, 1]


@pytest.mark.parametrize("separator", [[], [5, 0, 2**64 - 2**32]])
def test_circuit_digest_restated_with_the_oracle(separator):
    plonk = _plonk()
    cap = synth(0xD16, (16, 4))
    padded = list(separator) + [1]
    while (len(padded) + 1) % 8:
        padded.append(0)
    padded.append(1)
    sep = OL.hash_no_pad(np.array(padded, dtype=np.uint64))
    for db in (3, 20):
        want = OL.hash_no_pad(np.concatenate([cap.reshape(-1), sep, np.array([db], dtype=np.uint64)]))
        assert plonk.circuit_digest(cap, separator, db) == [int(x) for x in want]
    assert plonk.circuit_digest(cap, separator, 3) != plonk.circuit_digest(cap, separator + [0], 3)


def test_blind_and_pad_is_the_zk_test_circuit_layout():
    plonk = _plonk()
    cfg = plonk.standard_recursion_zk_config()
    fri_cfg = PC.quick_fri_config(cfg)
    c, (regular, z_pairs) = PC.zk_circuit(plonk, cfg, fri_cfg)
    rows = instances_of(c)
    num_gates = 2 + 12
    out, regular_rows, pairs = plonk.blind_and_pad(cfg, fri_cfg, rows[:num_gates])
    assert len(out) == c.n
    assert regular_rows == range(num_gates, num_gates + regular)
    assert pairs == [(num_gates + regular + 2 * q, num_gates + regular + 2 * q + 1) for q in range(z_pairs)]
    assert [(g.id(), list(k)) for g, k in out] == [(g.id(), list(k)) for g, k in rows]
    # the same circuit without zero knowledge is only padded
    plain = plonk.CircuitConfig()
    out, regular_rows, pairs = plonk.blind_and_pad(plain, fri_cfg, rows[:num_gates])
    assert len(out) == 16 and len(regular_rows) == 0 and pairs == []
    assert len(plonk.blind_and_pad(plain, fri_cfg, rows[:16])[0]) == 16
    assert len(plonk.blind_and_pad(plain, fri_cfg, [])[0]) == 1


def test_refusals_before_device_work():
    """Every refusal of gl_sigma_polys is a ShapeError before the context is used (the calls pass no context); a valid
    call without a context is refused only then."""
    plonk = _plonk()
    L = N.lib()
    k = np.ones(8, dtype=np.uint64)
    out = np.empty(8 << 2, dtype=np.uint64)

    def call(pairs, nw=12, nr=8, db=2, nv=3):
        p = np.ascontiguousarray(pairs, dtype=np.uint64).reshape(-1)
        rc = L.gl_sigma_polys(None, N.np_ptr(p) if p.size else None, len(p) // 2, N.MEM_HOST, nw, nr, db, nv,
                              N.np_ptr(k), N.np_ptr(out), N.MEM_HOST)
        N.check(rc, None)

    T = (12 << 2) + 3
    with pytest.raises(N.ShapeError, match="num_targets"):
        call([[0, T]])
    with pytest.raises(N.ShapeError, match="not routable"):
        call([[0, 8]])                       # wire (0, 8): column 8 >= num_routed_wires
    with pytest.raises(N.ShapeError, match="not routable"):
        call([[1, 3 * 12 + 11]])
    with pytest.raises(N.ShapeError, match="below 2"):
        call([], nw=2**16, nr=8, db=16, nv=0)
    with pytest.raises(N.ShapeError, match="below 2"):
        call([], nv=2**32)
    with pytest.raises(N.ShapeError, match="num_routed_wires"):
        call([], nw=8, nr=9)
    with pytest.raises(N.NativeError, match="null context"):
        call([[0, T - 1], [3, 12 + 7], [5, 5]])   # a virtual target, routed wires, a self-pair: valid
    # the encoding of build_circuit_data: wire indices past the last row are refused before the device
    with pytest.raises(N.ShapeError, match="past the last"):
        plonk.target_indices([[0, 12 << 2]], 12, 2)
    assert plonk.target_indices([[5, -1], [-3, 0]], 12, 2).tolist() == [[5, 48], [50, 0]]
    # the FRI arity check of build (circuit_builder.rs:1140-1143)
    from plonky2_b200.fri import FriConfig

    cfg = plonk.CircuitConfig(num_wires=12, num_routed_wires=8, max_quotient_degree_factor=4, rate_bits=1,
                              cap_height=2)
    deep = FriConfig(rate_bits=1, cap_height=2, proof_of_work_bits=0, reduction_strategy=("Fixed", [2, 2]),
                     num_query_rounds=2)
    rows = [(plonk.NoopGate(), [])] * 8
    with pytest.raises(N.ShapeError, match="arity is too large"):
        plonk.build_circuit_data(cfg, deep, rows, [])


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


def _device_sigmas(cfg, db, pairs, nv=0, on_device=False):
    import torch

    plonk = _plonk()
    if on_device:
        pairs = torch.from_numpy(np.ascontiguousarray(pairs, dtype=np.int64).reshape(-1, 2)).cuda()
        torch.cuda.synchronize()
    return plonk.sigma_polys(cfg, db, pairs, nv).cpu().numpy().view(np.uint64)


def _want(cfg, db, pairs, nv=0, literal=False):
    from plonky2_b200.plonk import get_unique_coset_shifts

    f = forest_sigma_map if literal else vector_sigma_map
    m = f(cfg.num_wires, cfg.num_routed_wires, db, nv, pairs)
    return sigma_values(m, get_unique_coset_shifts(cfg.num_routed_wires), db)


@pytest.mark.gpu
def test_sigmas_of_every_fibonacci_shape(pb):
    for shape in PC.SHAPES:
        for kw in ({}, dict(break_copy=True)):
            c = PC.shape_circuit(shape, cap_height=1, **kw)
            cfg, db = c.config, c.common.degree_bits
            pairs = pairs_from_sigmas(c)
            want = _want(cfg, db, pairs, literal=True)
            assert np.array_equal(_device_sigmas(cfg, db, pairs), want), (shape, kw)
            # break_copy lists wire (0, 1) last in its set, where the reference has it first: a rotation of the same
            # cycle, so the permutation is the same
            assert np.array_equal(c.sigmas, want), (shape, kw)


@pytest.mark.gpu
def test_sigmas_of_large_circuit_2_18(pb):
    import plonk_large as PL

    plonk = _plonk()
    cfg = plonk.CircuitConfig()
    c = PL.LargeCircuit(plonk, cfg, 18, luts=[(PL.small_table(), 8)])
    nw = cfg.num_wires
    pairs = np.concatenate([np.stack([(R[:-1] * nw + C_[:-1]).reshape(-1), (R[1:] * nw + C_[1:]).reshape(-1)], 1)
                            for R, C_ in c.cycles])
    want = _want(cfg, 18, pairs)
    got = _device_sigmas(cfg, 18, pairs)
    assert np.array_equal(got, want)
    assert np.array_equal(got, c.sigmas)


@pytest.mark.gpu
def test_sigma_edge_cases(pb):
    plonk = _plonk()
    cfg = plonk.CircuitConfig(num_wires=12, num_routed_wires=8)
    from plonky2_b200.plonk import get_unique_coset_shifts

    db, n = 6, 64
    k_is = np.array(get_unique_coset_shifts(8), dtype=np.uint64)
    identity = gn.mul(k_is[:, None], gn.powers(PC.root_of_unity(db), n)[None, :])
    assert np.array_equal(_device_sigmas(cfg, db, np.zeros((0, 2), dtype=np.int64)), identity)
    # one set of every routed wire, given as a star around the last one: each maps to the next in row-major order
    routed = np.array([r * 12 + c for r in range(n) for c in range(8)], dtype=np.int64)
    star = np.stack([np.full(len(routed), routed[-1]), routed], 1)
    got = _device_sigmas(cfg, db, star)
    assert np.array_equal(got, _want(cfg, db, star))
    assert int(got[7, n - 1]) == int(identity[0, 0])          # the last wire wraps to the first
    # random graphs whose sets only virtual targets join, from host and device memory
    for seed in range(3):
        rng = np.random.default_rng(seed)
        pairs = random_pairs(rng, 12, 8, db, 40, 200)
        want = _want(cfg, db, pairs, 40, literal=True)
        assert np.array_equal(_device_sigmas(cfg, db, pairs, 40), want)
        assert np.array_equal(_device_sigmas(cfg, db, pairs, 40, on_device=True), want)
    # device pairs are refused from the device flag
    for bad, what in (([[0, (12 << db) + 40]], "num_targets"), ([[0, 9]], "not routable")):
        with pytest.raises(N.ShapeError, match=what):
            _device_sigmas(cfg, db, np.array(bad), 40, on_device=True)


@pytest.mark.gpu
def test_descending_chain_of_2_22_edges(pb):
    """The worst case for hooking depth: one chain over 2^22 + 1 routed wires given from the last to the first."""
    plonk = _plonk()
    cfg = plonk.CircuitConfig(num_wires=80, num_routed_wires=64)
    db = 16                                           # 2^22 routed wires
    routed = (np.arange(1 << 22, dtype=np.int64) // 64) * 80 + np.arange(1 << 22) % 64
    v = np.int64(80 << db)                            # and one virtual target at the end of the chain
    chain = np.concatenate([routed[::-1], [v]])
    pairs = np.stack([chain[:-1], chain[1:]], 1)
    got = _device_sigmas(cfg, db, pairs, 1)
    # every routed wire is in one set: each maps to the next routed index, the last to the first
    nxt = np.r_[np.arange(1, 1 << 22), 0]
    m = (nxt % 64) * (1 << db) + nxt // 64
    out = np.empty(1 << 22, dtype=np.uint64)
    i = np.arange(1 << 22)
    out[(i % 64) * (1 << db) + i // 64] = m
    from plonky2_b200.plonk import get_unique_coset_shifts

    assert np.array_equal(got, sigma_values(out, get_unique_coset_shifts(64), db))
    assert np.array_equal(got, _want(cfg, db, pairs, 1))


def _fib(plonk, public_inputs=None, **kw):
    cfg = plonk.CircuitConfig(num_wires=135, num_routed_wires=80, cap_height=3)
    return PC.FibonacciCircuit(plonk, cfg, 6, poseidon_rows=4, public_inputs=public_inputs, **kw)


@pytest.mark.gpu
def test_constants_sigmas_commitment_and_shards(pb):
    plonk = _plonk()
    c = _fib(plonk)
    cfg = c.config
    fri_cfg = PC.quick_fri_config(cfg)
    data = plonk.build_circuit_data(cfg, fri_cfg, instances_of(c), pairs_from_sigmas(c))
    cs = data.prover_only.constants_sigmas_commitment
    ref = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height)
    try:
        assert np.array_equal(data.prover_only.sigmas, c.sigmas)
        assert np.array_equal(cs.merkle_tree.cap.hashes, ref.merkle_tree.cap.hashes)
        assert np.array_equal(data.verifier_only.constants_sigmas_cap.hashes, ref.merkle_tree.cap.hashes)
        rows = [0, 1, 77, (c.n << cfg.rate_bits) - 1]
        for r in rows:
            assert np.array_equal(cs.merkle_tree.get(r), ref.merkle_tree.get(r))
        assert np.array_equal(cs.polynomials, ref.polynomials)
        assert data.prover_only.circuit_digest == plonk.circuit_digest(ref.merkle_tree.cap, (), c.common.degree_bits)
        assert data.verifier_only.circuit_digest == data.prover_only.circuit_digest
        # shard by shard in one process: the shards' leaves and caps concatenate to the unsharded commitment
        sig = plonk.sigma_polys(cfg, c.common.degree_bits, plonk.target_indices(pairs_from_sigmas(c), cfg.num_wires,
                                                                                 c.common.degree_bits))
        for G in (1, 2, 4, 8):
            shards = [plonk.commit_constants_sigmas(c.common, c.constant_vecs, sig, shard=(g, G)) for g in range(G)]
            try:
                assert np.array_equal(np.concatenate([s.merkle_tree.cap.hashes for s in shards]),
                                      ref.merkle_tree.cap.hashes), G
                assert np.array_equal(np.concatenate([s.merkle_tree.leaves for s in shards]), ref.merkle_tree.leaves), G
            finally:
                for s in shards:
                    s.close()
    finally:
        cs.close()
        ref.close()


@pytest.mark.gpu
def test_build_then_prove_is_accepted(pb):
    plonk = _plonk()
    c = _fib(plonk, public_inputs=[3, 1, 4, 1, 5], extra=("RandomAccessGate",), lookups=True)
    cfg = c.config
    fri_cfg = PC.quick_fri_config(cfg)
    data = plonk.build_circuit_data(cfg, fri_cfg, instances_of(c), pairs_from_sigmas(c), luts=c.common.luts,
                                    lookup_rows=c.lookup_rows, domain_separator=[7, 8])
    try:
        digest = data.verifier_only.circuit_digest
        proof = plonk.prove_with_witness(data.prover_only, data.common, c.wires, c.public_inputs)
        parts = PC.parts_of(proof, data.verifier_only.constants_sigmas_cap.hashes)
        assert PC.oracle_verify(OL, plonk, c, digest, fri_cfg, parts) is None
        assert PC.oracle_verify(OL, plonk, c, [digest[0] ^ 1] + digest[1:], fri_cfg, parts) is not None
        other = plonk.circuit_digest(data.verifier_only.constants_sigmas_cap, [], c.common.degree_bits)
        assert PC.oracle_verify(OL, plonk, c, other, fri_cfg, parts) is not None
    finally:
        data.prover_only.constants_sigmas_commitment.close()


@pytest.mark.gpu
def test_zero_knowledge_build_then_prove_is_accepted(pb):
    plonk = _plonk()
    cfg = plonk.standard_recursion_zk_config()
    fri_cfg = PC.quick_fri_config(cfg)
    c, (regular, z_pairs) = PC.zk_circuit(plonk, cfg, fri_cfg)
    num_gates = 2 + 12
    instances, _, pairs_rows = plonk.blind_and_pad(cfg, fri_cfg, instances_of(c)[:num_gates])
    skip = [r for pr in pairs_rows for r in pr]
    data = plonk.build_circuit_data(cfg, fri_cfg, instances, pairs_from_sigmas(c, skip))
    try:
        # the pairs carry no copy constraint (the reference's generate_copy): their sigmas are the identity
        k_is = c.common.k_is
        w = PC.root_of_unity(c.common.degree_bits)
        r1 = pairs_rows[0][0]
        assert int(data.prover_only.sigmas[5, r1]) == k_is[5] * pow(w, r1, PC.P) % PC.P
        proof = plonk.prove_with_witness(data.prover_only, data.common, c.wires, c.public_inputs)
        parts = PC.parts_of(proof, data.verifier_only.constants_sigmas_cap.hashes)
        digest = data.verifier_only.circuit_digest
        assert PC.oracle_verify(OL, plonk, c, digest, fri_cfg, parts) is None
        assert PC.oracle_verify(OL, plonk, c, [digest[0] ^ 1] + digest[1:], fri_cfg, parts) is not None
    finally:
        data.prover_only.constants_sigmas_commitment.close()


@pytest.mark.gpu
def test_build_across_ranks(pb):
    """torchrun: distributed.build_circuit_data + prove_plonk give every rank the bytes of the single-device build +
    prove_with_witness (tests/mgpu_circuit_data_check.py)."""
    run_ranks("mgpu_circuit_data_check.py", "MGPU_CIRCUIT_DATA_CHECK OK", timeout=1200)
