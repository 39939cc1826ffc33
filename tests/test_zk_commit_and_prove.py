"""Zero-knowledge commitments and plonky2 proofs.

CPU: blinding_counts against values worked out from circuit_builder.rs:866-909, and the zero-knowledge host logic of
plonk.prove_with_witness with the oracle standing in for the device: its bytes equal the salted CPU twin's (the
oracle's commitments fed the restated salt of each key, hiding = 1 in the transcript, leaf widths + 4), the restated
verifier accepts them, and the proof format reads them back.

GPU (-m gpu): the device salt sampler against the numpy restatement (tests/chacha_ref.py), keyed commitments against
explicit-salt ones and the oracle (from_values, from_coeffs, the incremental path, row-block shards, a shape above 2^24
leaves), fresh keys, the C ABI's errors, and zero-knowledge proofs byte-identical to the salted CPU twin."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import chacha_ref as R
import plonk_circuits as PC
from conftest import synth
from plonk_circuits import KEYS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _plonk():
    from plonky2_b200 import plonk

    return plonk


# name -> (PoseidonGate rows, other gate rows, lookups)
ZK_SHAPES = {"plain": (0, (), False), "poseidon": (9, (), False),
             "lookup": (4, ("ArithmeticExtensionGate", "RandomAccessGate", "CosetInterpolationGate"), True)}


def _zk_circuit(name):
    """A circuit of standard_recursion_zk_config with the blinding rows blinding_counts asks for, padded to a power of
    two like CircuitBuilder::blind_and_pad."""
    plonk = _plonk()
    cfg = plonk.standard_recursion_zk_config()
    poseidon_rows, extra, lookups = ZK_SHAPES[name]
    c, _ = PC.zk_circuit(plonk, cfg, PC.quick_fri_config(cfg), poseidon_rows=poseidon_rows, extra=extra,
                         lookups=lookups)
    return c


# ----------------------------------------------------------------------------------------------------------- CPU
def test_blinding_counts_restate_the_reference():
    from plonky2_b200.fri import standard_recursion_fri_config

    plonk = _plonk()
    cfg, fri = plonk.standard_recursion_zk_config(), standard_recursion_fri_config()
    assert cfg.zero_knowledge and not plonk.CircuitConfig().zero_knowledge
    # 2^12 and 2^13 are too small; at 2^14 the arities are [4, 4, 4] and the final polynomial has 4 coefficients:
    # 28 * (1 + 2 * 45 + 2 * 4) = 2772 FRI openings
    assert plonk.blinding_counts(cfg, fri, 4000) == (2774, 2776)
    # quick_fri_config at 2^10: arities [2, 2, 2, 2], 4 final coefficients: 6 * (1 + 2 * 12 + 2 * 4) = 198
    assert plonk.blinding_counts(cfg, PC.quick_fri_config(cfg), 20) == (200, 202)


def test_zk_fri_instance_and_proof_widths():
    plonk = _plonk()
    c = _zk_circuit("plain")
    inst = plonk.get_fri_instance(c.common, (5, 7))
    assert [o.blinding for o in inst.oracles] == [False, True, True, True]
    c.config.zero_knowledge = False
    assert not any(o.blinding for o in plonk.get_fri_instance(c.common, (5, 7)).oracles)


@pytest.mark.parametrize("name", list(ZK_SHAPES))
def test_zk_prove_host_logic_with_cpu_backends(oracle, name, monkeypatch):
    """prove_with_witness with config.zero_knowledge, its device calls answered by the oracle with the restated salt of
    each key: equal bytes to the salted CPU twin, accepted by the restated verifier, which rejects them when the circuit
    does not say zero knowledge; the bytes read back, and get_challenges replays the prover's transcript."""
    plonk = _plonk()
    c = _zk_circuit(name)
    cfg, cd = c.config, c.common
    digest = [int(x) for x in synth(0x590, (4,))]
    fri_cfg = PC.quick_fri_config(cfg)
    want, parts = PC.oracle_prove(oracle, c, digest, fri_cfg, c.public_inputs, salts=PC.salts(c))
    assert PC.oracle_verify(oracle, plonk, c, digest, fri_cfg, parts) is None
    cfg.zero_knowledge = False       # no hiding in the transcript and unsalted leaf widths: the same proof is rejected
    assert PC.oracle_verify(oracle, plonk, c, digest, fri_cfg, parts) is not None
    cfg.zero_knowledge = True
    ctx, logs, used = PC.cpu_backends(monkeypatch, oracle, c, fri_cfg, salt_keys=KEYS)
    cs = plonk.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height)
    fri_params = fri_cfg.fri_params(cd.degree_bits, True)
    prover_data = plonk.ProverOnlyCircuitData(cs, c.sigmas, digest, fri_params)
    proof = plonk.prove_with_witness(prover_data, cd, c.wires, c.public_inputs, ctx=ctx, salt_keys=KEYS)
    data = proof.to_bytes()
    assert data == want and used == KEYS
    # the proof format: salted initial-tree leaves, round trip, transcript replay, compression
    back = plonk.ProofWithPublicInputs.from_bytes(data, cd, fri_params)
    assert back.to_bytes() == data
    widths = [len(leaf) for leaf, _ in back.proof.opening_proof.query_round_proofs[0].initial_trees_proof.evals_proofs]
    nc = cfg.num_challenges
    assert widths == [cd.num_constants + cfg.num_routed_wires, cfg.num_wires + 4,
                      nc * (1 + cd.num_partial_products + cd.num_lookup_polys) + 4, nc * cd.quotient_degree_factor + 4]
    ch = back.get_challenges(digest, cd, fri_params)
    challenges = [v for kind, v in logs[0] if kind == "challenge"]
    assert ch["plonk_betas"] == challenges[:nc] and ch["plonk_gammas"] == challenges[nc:2 * nc]
    assert back.compress(digest, cd, fri_params).to_bytes() != data
    # a proof whose parameters do not say hiding is refused before any work
    with pytest.raises(plonk.N.ShapeError):
        plonk.prove_with_witness(plonk.ProverOnlyCircuitData(cs, c.sigmas, digest, fri_cfg.fri_params(cd.degree_bits, False)),
                                 cd, c.wires, c.public_inputs, ctx=ctx, salt_keys=KEYS)


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


@pytest.mark.gpu
def test_device_sampler_matches_restatement(pb):
    key = bytes(range(7, 39))
    cases = [(0, 1), (5, 7), (3, 8), (8, 9), (12345, 1000), ((1 << 30) + 3, 65537), ((1 << 35) - 77, 77)]
    for column in range(4):
        for first, count in cases:
            got = pb.random_field_elements_keyed(key, column, first, count)
            assert np.array_equal(got, R.samples(key, column, first, count)), (column, first, count)
            assert (got < np.uint64(R.P)).all()
    big = pb.random_field_elements_keyed(key, 2, 3, 1 << 24)      # counts up to 2^24, unaligned start
    assert np.array_equal(big, R.samples(key, 2, 3, 1 << 24)) and (big < np.uint64(R.P)).all()
    parts = [pb.random_field_elements_keyed(key, 2, 3 + a, b - a)
             for a, b in ((0, 1), (1, 9), (9, 4096 + 5), (4101, 1 << 20), (1 << 20, 1 << 24))]
    assert np.array_equal(np.concatenate(parts), big)             # any (first, count) split is the same stream
    with pytest.raises(pb.ShapeError):
        pb.random_field_elements_keyed(b"short", 0, 0, 1)
    from plonky2_b200 import _native as N

    ctx = pb.default_context()
    out = np.empty(1, dtype=np.uint64)
    assert N.lib().gl_random_field_elements(ctx.h, key, 0, 1 << 35, 1, N.np_ptr(out), N.MEM_HOST) == N.GL_ERR_BAD_ARG


@pytest.mark.gpu
def test_device_sampler_with_a_lowered_bound(pb, tmp_path):
    """tests/cuda/chacha_device.cu built with the acceptance bound at 2^63: about half of the words fall back to later
    attempts, and the device still draws the restated stream."""
    from test_gpu_field_lazy import nvcc_cmd

    exe = str(tmp_path / "chacha_device")
    cmd = nvcc_cmd("GL_CHACHA_BOUND=0x8000000000000000ULL", exe)
    cmd[-1] = os.path.join(ROOT, "tests", "cuda", "chacha_device.cu")
    subprocess.check_call(cmd)
    key = bytes(range(100, 132))
    for column, first, count in ((0, 0, 4096), (3, 13, 50001)):
        out = str(tmp_path / "out.bin")
        subprocess.check_call([exe, key.hex(), str(column), str(first), str(count), out])
        got = np.fromfile(out, dtype="<u8").astype(np.uint64)
        assert np.array_equal(got, R.samples(key, column, first, count, bound=1 << 63))
        assert (got < np.uint64(1 << 63)).all()


def _same_commitment(a, b, o=None):
    assert np.array_equal(a.merkle_tree.cap.hashes, b.merkle_tree.cap.hashes)
    assert np.array_equal(a.merkle_tree.digests, b.merkle_tree.digests)
    assert np.array_equal(a.merkle_tree.leaves, b.merkle_tree.leaves)
    assert np.array_equal(a.get_lde_values(3, 1), b.get_lde_values(3, 1))
    if o is not None:
        assert np.array_equal(a.merkle_tree.cap.hashes, o.cap) and np.array_equal(a.merkle_tree.leaves, o.leaves)


@pytest.mark.gpu
@pytest.mark.parametrize("B,log_n,r,h", [(5, 6, 2, 2), (1, 1, 1, 0), (40, 10, 3, 4), (3, 0, 2, 1)])
def test_keyed_commitment_equals_explicit_salt(pb, oracle, B, log_n, r, h):
    key = bytes(range(32))
    n, N = 1 << log_n, 1 << (log_n + r)
    salt = R.salt_array(key, N)
    vals = synth(0x2A0 + B, (B, n))
    for is_coeffs, mk in ((False, pb.PolynomialBatch.from_values), (True, pb.PolynomialBatch.from_coeffs)):
        keyed = mk(vals, r, True, h, salt_key=key)
        explicit = mk(vals, r, True, h, salt=salt)
        assert keyed.leaf_width == B + 4
        _same_commitment(keyed, explicit, oracle.Commit(vals, r, h, salt=salt, is_coeffs=is_coeffs))
    with pytest.raises(pb.ShapeError):
        pb.PolynomialBatch.from_values(vals, r, True, h, salt=salt, salt_key=key)


@pytest.mark.gpu
def test_keyed_incremental_path(pb):
    """_from_coeff_chunks (the quotient commitment's path) with a key equals from_coeffs with the restated salt."""
    import torch

    key = KEYS[1]
    log_n, r, h, chunks = 7, 3, 3, 4
    polys = synth(0x2B0, (2, chunks << log_n))
    t = torch.from_numpy(polys.view(np.int64)).cuda()
    keyed = pb.PolynomialBatch._from_coeff_chunks(t, chunks, log_n, r, h, blinding=True, salt_key=key)
    explicit = pb.PolynomialBatch.from_coeffs(polys.reshape(2 * chunks, 1 << log_n), r, True, h,
                                              salt=R.salt_array(key, 1 << (log_n + r)))
    _same_commitment(keyed, explicit)
    plain = pb.PolynomialBatch._from_coeff_chunks(t, chunks, log_n, r, h)
    assert plain.leaf_width == 2 * chunks and np.array_equal(plain.get_lde_values(5, 1), keyed.get_lde_values(5, 1))


@pytest.mark.gpu
@pytest.mark.parametrize("G", [2, 4, 8])
def test_keyed_row_block_shards(pb, G):
    key = KEYS[2]
    B, log_n, r, h = 6, 9, 3, 4
    vals = synth(0x2C0, (B, 1 << log_n))
    whole = pb.PolynomialBatch.from_values(vals, r, True, h, salt_key=key)
    shards = [pb.PolynomialBatch.from_values(vals, r, True, h, salt_key=key, shard=(g, G)) for g in range(G)]
    assert np.array_equal(np.concatenate([s.merkle_tree.cap.hashes for s in shards]), whole.merkle_tree.cap.hashes)
    assert np.array_equal(np.concatenate([s.merkle_tree.leaves for s in shards]), whole.merkle_tree.leaves)


@pytest.mark.gpu
def test_keyed_commitment_above_2_pow_24_leaves(pb):
    """2^25 leaves: the keyed salt equals the explicit salt drawn by the device sampler (checked against the
    restatement above) and is correct at rows spot-checked against the restatement."""
    key = KEYS[0]
    B, log_n, r, h = 2, 22, 3, 4
    N = 1 << (log_n + r)
    vals = synth(0x2D0, (B, 1 << log_n))
    salt = np.stack([pb.random_field_elements_keyed(key, s, 0, N) for s in range(4)])
    for j in (0, 1, N // 2 + 12345, N - 1):
        i = int(format(j, "025b")[::-1], 2)
        assert np.array_equal(salt[:, i], [R.samples(key, s, i, 1)[0] for s in range(4)])
    keyed = pb.PolynomialBatch.from_values(vals, r, True, h, salt_key=key)
    explicit = pb.PolynomialBatch.from_values(vals, r, True, h, salt=salt)
    assert np.array_equal(keyed.merkle_tree.cap.hashes, explicit.merkle_tree.cap.hashes)
    rows = [0, 7, N // 3, N - 1]
    assert all(np.array_equal(keyed.merkle_tree.get(j), explicit.merkle_tree.get(j)) for j in rows)


@pytest.mark.gpu
def test_fresh_keys_and_abi_errors(pb):
    from plonky2_b200 import _native as N

    vals = synth(0x2E0, (4, 1 << 8))
    a = pb.PolynomialBatch.from_values(vals, 2, True, 2, salt_key="fresh")
    b = pb.PolynomialBatch.from_values(vals, 2, True, 2, salt_key="fresh")
    assert not np.array_equal(a.merkle_tree.cap.hashes, b.merkle_tree.cap.hashes)
    assert all(np.array_equal(a.get_lde_values(i, 1), b.get_lde_values(i, 1)) for i in (0, 17, 1023))
    ctx, L = pb.default_context(), N.lib()
    for blinding, err in ((0, "without blinding"), (1, "already finished")):
        h = N.vp()
        N.check(L.gl_commit_begin(ctx.h, 4, 8, 2, 2, blinding, 0, 1, None, C.byref(h)), ctx.h)
        N.check(L.gl_commit_add_columns(h, 0, 4, N.np_ptr(vals), 256, N.COLS_VALUES, N.MEM_HOST), ctx.h)
        if blinding:
            N.check(L.gl_commit_finish_keyed(h, KEYS[0]), ctx.h)
        assert L.gl_commit_finish_keyed(h, KEYS[0]) == N.GL_ERR_BAD_ARG
        assert err in L.gl_last_error(ctx.h).decode()
        L.gl_commit_destroy(h)
    with pytest.raises(pb.ShapeError):
        pb.PolynomialBatch.from_values(vals, 2, False, 2, salt_key=KEYS[0])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ZK_SHAPES))
def test_zk_proof_on_device(pb, oracle, name):
    """standard_recursion_zk_config with blinding rows: with fixed salt keys the device proof is byte-identical to the
    salted CPU twin and verifies; a changed salt word or byte of an initial-tree leaf is rejected; two fresh-entropy
    proofs differ and both verify; hiding = false with a zero-knowledge config is refused."""
    plonk = _plonk()
    c = _zk_circuit(name)
    cfg, cd = c.config, c.common
    digest = [int(x) for x in synth(0x591, (4,))]
    fri_cfg = PC.quick_fri_config(cfg)
    fri_params = fri_cfg.fri_params(cd.degree_bits, True)
    want, _ = PC.oracle_prove(oracle, c, digest, fri_cfg, c.public_inputs, salts=PC.salts(c))
    cs = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height)
    cs_cap = cs.merkle_tree.cap.hashes
    prover_data = plonk.ProverOnlyCircuitData(cs, c.sigmas, digest, fri_params)
    data = plonk.prove_with_witness(prover_data, cd, c.wires, c.public_inputs, salt_keys=KEYS).to_bytes()
    assert data == want
    proof = plonk.ProofWithPublicInputs.from_bytes(data, cd, fri_params)
    assert PC.oracle_verify(oracle, plonk, c, digest, fri_cfg, PC.parts_of(proof, cs_cap)) is None
    for oracle_index, word, mask in ((1, -1, 1), (2, -2, 1 << 40), (3, 0, 0xFF)):   # salt words, a polynomial word
        bad = plonk.ProofWithPublicInputs.from_bytes(data, cd, fri_params)
        leaf = bad.proof.opening_proof.query_round_proofs[1].initial_trees_proof.evals_proofs[oracle_index][0]
        leaf[word] ^= np.uint64(mask)
        assert bad.to_bytes() != data
        assert PC.oracle_verify(oracle, plonk, c, digest, fri_cfg, PC.parts_of(bad, cs_cap)) is not None
    fresh = [plonk.prove_with_witness(prover_data, cd, c.wires, c.public_inputs) for _ in range(2)]
    assert fresh[0].to_bytes() != fresh[1].to_bytes()
    for f in fresh:
        assert PC.oracle_verify(oracle, plonk, c, digest, fri_cfg, PC.parts_of(f, cs_cap)) is None
    with pytest.raises(pb.ShapeError):
        plonk.prove_with_witness(plonk.ProverOnlyCircuitData(cs, c.sigmas, digest, fri_cfg.fri_params(cd.degree_bits, False)),
                                 cd, c.wires, c.public_inputs, salt_keys=KEYS)
    cs.close()


@pytest.mark.gpu
def test_cpp_mirror_keyed_commitment(pb, tmp_path):
    """tests/cpp/keyed_commit.cpp builds a keyed commitment through plonky2_b200.hpp's SaltKey overload: the same cap
    as the Python layer's."""
    exe = str(tmp_path / "keyed_commit")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "keyed_commit.cpp"),
                           "-L" + os.path.join(ROOT, "plonky2_b200"), "-lplonky2_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "plonky2_b200")])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    with np.errstate(over="ignore"):
        v = (np.arange(5 * 64, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)).reshape(5, 64)
    c = pb.PolynomialBatch.from_values(v, 2, True, 2, salt_key=bytes(range(32)))
    assert [int(x) for x in r.stdout.split()] == [int(x) for x in c.merkle_tree.cap.hashes.reshape(-1)]
