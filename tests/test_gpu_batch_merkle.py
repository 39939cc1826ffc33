"""SURVEY 8(f) row 4 (first part): BatchMerkleTree, batch Merkle proofs and Merkle path compression on the GPU trees,
restating the reference's own tests (plonky2/src/hash/batch_merkle_tree.rs:167-340, path_compression.rs:116-160) with
expected digests computed by the CPU oracle."""
import os

import numpy as np
import pytest

from conftest import synth

pytestmark = pytest.mark.gpu


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


MAT_1 = np.array([[0, 1], [2, 1], [2, 2], [0, 0]], dtype=np.uint64)
MAT_2 = np.array([[1, 2, 1], [0, 2, 2]], dtype=np.uint64)


def test_commit_single(pb, oracle):
    # batch_merkle_tree.rs:186-228
    fmt = pb.BatchMerkleTree([MAT_1], 0)
    lh = [oracle.hash_or_noop(r) for r in MAT_1]
    d = fmt.digests
    assert np.array_equal(d[0:2], lh[0:2]) and np.array_equal(d[4:6], lh[2:4])
    layer_1 = [oracle.two_to_one(lh[0], lh[1]), oracle.two_to_one(lh[2], lh[3])]
    assert np.array_equal(d[2:4], layer_1)
    root = oracle.two_to_one(layer_1[0], layer_1[1])
    assert np.array_equal(fmt.cap.flatten(), root)
    proof = fmt.open_batch(2)
    assert np.array_equal(proof.siblings, [lh[3], layer_1[0]])
    vals = fmt.values(2)
    assert len(vals) == 1 and np.array_equal(vals[0], [2, 2])
    pb.verify_batch_merkle_proof_to_cap(vals, fmt.leaf_heights, 2, fmt.cap, proof)


def test_commit_mixed(pb, oracle):
    # batch_merkle_tree.rs:231-300
    fmt = pb.BatchMerkleTree([MAT_1, MAT_2], 0)
    lh = [oracle.hash_or_noop(r) for r in MAT_1]
    d = fmt.digests
    assert np.array_equal(d[0:4], lh)
    hidden = [oracle.two_to_one(lh[0], lh[1]), oracle.two_to_one(lh[2], lh[3])]
    layer_1 = [oracle.hash_or_noop(np.concatenate([hidden[k], MAT_2[k]])) for k in range(2)]
    assert np.array_equal(d[4:], layer_1)
    assert np.array_equal(fmt.cap.flatten(), oracle.two_to_one(layer_1[0], layer_1[1]))
    proof = fmt.open_batch(1)
    assert np.array_equal(proof.siblings, [lh[0], layer_1[1]])
    vals = fmt.values(1)
    assert np.array_equal(vals[0], [2, 1]) and np.array_equal(vals[1], [1, 2, 1])
    pb.verify_batch_merkle_proof_to_cap(vals, fmt.leaf_heights, 1, fmt.cap, proof)
    with pytest.raises(ValueError, match="Invalid Merkle proof"):
        bad = [vals[0], vals[1] ^ np.uint64(1)]
        pb.verify_batch_merkle_proof_to_cap(bad, fmt.leaf_heights, 1, fmt.cap, proof)


def test_batch_merkle_trees(pb, oracle):
    # batch_merkle_tree.rs:302-322: three matrices (1024 x 7, 64 x 3, 32 x 100), cap height 3
    mats = [synth(0xF1, (1024, 7)), synth(0xF2, (64, 3)), synth(0xF3, (32, 100))]
    fmt = pb.BatchMerkleTree(mats, 3)
    assert fmt.leaf_heights == [10, 6, 5] and len(fmt.cap) == 8
    # the same tree from the oracle's MerkleTree::new, stage by stage
    _, cap0 = oracle.merkle_build(mats[0], 6)
    _, cap1 = oracle.merkle_build(np.concatenate([cap0, mats[1]], axis=1), 5)
    dig2, cap2 = oracle.merkle_build(np.concatenate([cap1, mats[2]], axis=1), 3)
    assert np.array_equal(fmt.cap.hashes, cap2)
    assert np.array_equal(fmt.digests[-len(dig2):], dig2)
    for index in [0, 1023, 512, 255]:
        proof = fmt.open_batch(index)
        assert len(proof.siblings) == 10 - 3
        pb.verify_batch_merkle_proof_to_cap(fmt.values(index), fmt.leaf_heights, index, fmt.cap, proof)
    fmt.close()


def test_batch_merkle_trees_cap_at_leaves_height(pb):
    # batch_merkle_tree.rs:324-340
    m = synth(0xF4, (16, 7))
    fmt = pb.BatchMerkleTree([m], 4)
    for index in range(16):
        proof = fmt.open_batch(index)
        assert len(proof.siblings) == 0
        pb.verify_batch_merkle_proof_to_cap(fmt.values(index), fmt.leaf_heights, index, fmt.cap, proof)
    with pytest.raises(pb.ShapeError):
        pb.BatchMerkleTree([m], 5)
    with pytest.raises(pb.ShapeError):
        pb.BatchMerkleTree([m, m], 0)   # duplicate heights


def test_path_compression(pb, oracle):
    # path_compression.rs:116-160: h = 10, cap height 3, k random indices; decompress(compress(proofs)) == proofs
    h, cap_height = 10, 3
    vs = synth(0xF5, (1 << h, 1))
    mt = pb.MerkleTree(vs, cap_height)
    k = 1 + int(synth(0xF6, (1,))[0]) % 300
    indices = [int(x) % (1 << h) for x in synth(0xF7, (k,), canonical=False)]
    leaves, paths = mt.open_many(indices)
    proofs = [pb.MerkleProof(p) for p in paths]
    compressed = pb.compress_merkle_proofs(cap_height, indices, proofs)
    assert sum(len(p.siblings) for p in compressed) < sum(len(p.siblings) for p in proofs)
    back = pb.decompress_merkle_proofs([vs[i] for i in indices], indices, compressed, h, cap_height)
    assert len(back) == len(proofs)
    for a, b, i in zip(back, proofs, indices):
        assert np.array_equal(a.siblings, b.siblings)
        assert oracle.merkle_verify(vs[i], i, a.siblings, mt.cap.hashes, cap_height)
    mt.close()


# ----------------------------------------------------------------------------- batch FRI (batch_fri/oracle.rs, batch_fri/prover.rs)
def _batch_case(pb, oracle, lens, counts, rate_bits, cap_height, arity_bits, num_queries, pow_bits, two_points):
    """lens: degree bits per group (decreasing), counts: polynomials per group. Byte-identical proof vs the oracle."""
    polys, degree_of = [], []
    for k, c in zip(lens, counts):
        for j in range(c):
            polys.append(synth(0x100 + 16 * k + j, (1 << k,)))
            degree_of.append(k)
    go = pb.BatchFriOracle.from_values(polys, rate_bits, False, cap_height)
    oo = oracle.BatchCommit(polys, rate_bits, cap_height)
    assert np.array_equal(go.cap.hashes, oo.cap)
    cfg = pb.FriConfig(rate_bits, cap_height, pow_bits, ("Fixed", list(arity_bits)), num_queries)
    params = pb.FriParams(cfg, False, lens[0], list(arity_bits))
    ch, och = pb.Challenger(), oracle.Challenger()
    ch.observe_cap(go.cap)
    och.observe_cap(oo.cap)
    zeta = ch.get_extension_challenge()
    assert och.get_extension_challenge() == zeta
    instances, oinstances = [], []
    for k in lens:
        idx = [i for i, d in enumerate(degree_of) if d == k]
        batches = [pb.FriBatchInfo(zeta, [pb.FriPolynomialInfo(0, i) for i in idx])]
        if two_points:
            gz = pb.field.ext_mul(zeta, (pb.field.primitive_root_of_unity(k), 0))
            batches.append(pb.FriBatchInfo(gz, [pb.FriPolynomialInfo(0, idx[0])]))
        instances.append(pb.FriInstanceInfo([pb.FriOracleInfo(len(polys), False)], batches))
        oinstances.append([(b.point, [(p.oracle_index, p.polynomial_index) for p in b.polynomials]) for b in batches])
    proof = pb.batch_prove_openings(list(lens), instances, [go], ch, params)
    want = oracle.batch_prove_openings([oo], list(lens), oinstances, och, oracle.make_params(rate_bits, cap_height, pow_bits, num_queries, list(arity_bits)))
    assert proof.to_bytes() == want
    go.close()


def test_batch_fri_multiple_polynomials_reference_shape(pb, oracle):
    # batch_fri/prover.rs:341-477: k = 9, 8, 6, rate 1, cap 5, arities [1, 2, 1], 10 queries, no PoW
    _batch_case(pb, oracle, [9, 8, 6], [1, 1, 1], 1, 5, [1, 2, 1], 10, 0, False)


def test_batch_fri_single_polynomial_reference_shape(pb, oracle):
    # batch_fri/prover.rs:275-339
    _batch_case(pb, oracle, [9], [1], 1, 5, [1, 2, 1], 10, 0, False)


def test_batch_fri_groups_two_points_pow(pb, oracle):
    # several polynomials per degree, openings at zeta and g*zeta, grinding, arity 8 then 4
    _batch_case(pb, oracle, [11, 8, 6], [5, 3, 2], 2, 3, [3, 2, 2], 6, 7, True)


def test_fri_proof_compress_roundtrip(pb, oracle):
    """FriProof::compress / decompress (fri/proof.rs:137-360) on a GPU-made proof: smaller, and decompressing with the
    removed evaluations gives back the byte-identical proof (duplicate query indices included)."""
    from plonky2_b200 import fri as F

    log_n, r, h = 9, 2, 2
    cols = synth(0x1F0, (6, 1 << log_n))
    batch = pb.PolynomialBatch.from_values(cols, r, False, h)
    cfg = pb.FriConfig(r, h, 3, ("Fixed", [2, 3]), 40)   # 40 queries over 2^11 points after folding: duplicates at the top
    params = pb.FriParams(cfg, False, log_n, [2, 3])
    ch = pb.Challenger()
    ch.observe_cap(batch.merkle_tree.cap)
    zeta = ch.get_extension_challenge()
    inst = pb.FriInstanceInfo([pb.FriOracleInfo(6, False)], [pb.FriBatchInfo(zeta, [pb.FriPolynomialInfo(0, i) for i in range(6)])])
    taps = {}
    proof = pb.prove_openings(inst, [batch], ch, params, taps=taps)
    indices = taps["query_indices"] if "query_indices" in taps else None
    if indices is None:  # recover the indices from the transcript order: prove_openings' taps may not carry them
        pytest.skip("prove_openings does not expose the query indices")
    comp = proof.compress(indices, params)
    assert len(comp.to_bytes()) < len(proof.to_bytes())
    inferred = []
    for x, qr in zip(indices, proof.query_round_proofs):
        row = []
        for j, st in enumerate(qr.steps):
            row.append(st.evals[x & ((1 << params.reduction_arity_bits[j]) - 1)])
            x >>= params.reduction_arity_bits[j]
        inferred.append(row)
    back = comp.decompress_with(inferred, params, log_n + r)
    assert back.to_bytes() == proof.to_bytes()
    batch.close()
