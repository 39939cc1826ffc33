"""Batch FRI on a Placement: the batch tree's later stages hashed on the device over `previous cap || LDE row`
(gl_commit_finish_prefixed), the row-block sharded BatchFriOracle and distributed.batch_prove_openings_sharded.

CPU: the refusals of the sharded batch prover and of a sharded BatchFriOracle (a world size that is not a power of two or
above 2^cap_height, a blinding oracle), raised before any device work.

GPU (-m gpu): for G = 1, 2, 4, 8 every shard of a BatchFriOracle built in one process, on the reference test's shape
(k = 9, 8, 6, rate 1, cap 5), on several polynomials per degree, with from_coeffs, and on a last group whose stage has
sub-tree height 0: the shards' local caps concatenated equal the single-device cap and the oracle's BatchCommit cap;
each stage's local digests are the rank's block of the oracle's stage tree, built stage by stage as
merkle_build(previous cap || Commit leaves); every owned opening equals the single-device one. The device stage hash at
group widths 1, 4, 8 and 12 (prefixed widths 5, 8, 12 and 16, across the 8-element absorption boundary) against the
oracle. batch_prove_openings_sharded without a process group gives batch_prove_openings' bytes, and on 2 (4 with four
GPUs) torchrun ranks (tests/mgpu_batch_fri_check.py) every rank's bytes equal the single-device proof's and the oracle's,
and the restated batch verifier accepts them."""
import os

import numpy as np
import pytest

from conftest import synth
from plonky2_b200 import _native as N
from plonky2_b200 import distributed as D
from plonky2_b200.fri import FriConfig, FriParams
from ranks import run_ranks

GS = [1, 2, 4, 8]

# (degree bits per group, polynomials per group, rate bits, cap height, from_coeffs)
SHAPES = {
    "reference": ([9, 8, 6], [1, 1, 1], 1, 5, False),
    "several": ([9, 8, 6], [5, 3, 2], 1, 5, False),
    "coeffs": ([9, 8, 6], [2, 1, 3], 1, 5, True),
    "last_subtree_0": ([9, 7, 4], [2, 2, 2], 1, 5, False),   # last stage: 2^5 leaves, cap height 5
}


def _polys(lens, counts, seed=0x300):
    polys = []
    for k, c in zip(lens, counts):
        polys += [synth(seed + 16 * k + j, (1 << k,)) for j in range(c)]
    return polys


# ----------------------------------------------------------------------------------------------------------- CPU
class _Stand:
    """A batch oracle stand-in: only its shard count and blinding."""

    def __init__(self, num_shards, blinding=False):
        self.shard_index, self.num_shards, self.blinding = 0, num_shards, blinding


def _params(cap_height=5, hiding=False):
    return FriParams(FriConfig(1, cap_height, 0, ("Fixed", [1, 2, 1]), 10), hiding, 9, [1, 2, 1])


def test_batch_prove_openings_refusals_before_device_work():
    for world in (1, 2, 4, 8, 16, 32):
        D.check_batch_prove_openings([_Stand(world)], _params(), world)
    for world in (0, 3, 6, 12):
        with pytest.raises(N.ShapeError, match="power-of-two"):
            D.check_batch_prove_openings([_Stand(world)], _params(), world)
    with pytest.raises(N.ShapeError, match="exceed"):
        D.check_batch_prove_openings([_Stand(64)], _params(), 64)
    with pytest.raises(N.ShapeError, match="blinding"):
        D.check_batch_prove_openings([_Stand(2, blinding=True)], _params(), 2)
    with pytest.raises(N.ShapeError, match="blinding"):
        D.check_batch_prove_openings([_Stand(1)], _params(hiding=True), 1)
    with pytest.raises(N.ShapeError, match="row-block shards"):
        D.check_batch_prove_openings([_Stand(2)], _params(), 4)
    # without a process group the world is one rank: the sharded entry point refuses before the prover starts
    with pytest.raises(N.ShapeError, match="blinding"):
        D.batch_prove_openings_sharded([9], [None], [_Stand(1, blinding=True)], None, _params())


def test_sharded_batch_oracle_refusals_before_device_work():
    import plonky2_b200 as p

    polys = _polys([9, 8, 6], [1, 1, 1])
    for shard in ((0, 3), (1, 6)):
        with pytest.raises(N.ShapeError, match="power-of-two"):
            p.BatchFriOracle.from_values(polys, 1, False, 5, shard=shard)
    with pytest.raises(N.ShapeError, match="exceed"):
        p.BatchFriOracle.from_coeffs(polys, 1, False, 5, shard=(0, 64))
    with pytest.raises(NotImplementedError):
        p.BatchFriOracle.from_values(polys, 1, True, 5, shard=(0, 2))


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


def _oracle_stages(oracle, polys, lens, rate_bits, cap_height, is_coeffs):
    """The batch tree stage by stage from the oracle's MerkleTree::new: [(digests, cap)] per stage."""
    stages, cap = [], None
    heights = [d + rate_bits for d in lens]
    for k, d in enumerate(lens):
        cols = np.stack([p for p in polys if len(p) == 1 << d])
        h = heights[k + 1] if k + 1 < len(lens) else cap_height
        c = oracle.Commit(cols, rate_bits, h, is_coeffs=is_coeffs)
        if k == 0:
            dig, cap = c.digests, c.cap
        else:
            dig, cap = oracle.merkle_build(np.concatenate([cap, c.leaves], axis=1), h)
        stages.append((dig, cap))
    return stages


def _build(pb, polys, rate_bits, cap_height, is_coeffs, shard=(0, 1)):
    make = pb.BatchFriOracle.from_coeffs if is_coeffs else pb.BatchFriOracle.from_values
    return make(polys, rate_bits, False, cap_height, shard=shard)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_sharded_batch_oracle_equals_single_device_and_oracle(pb, oracle, shape):
    lens, counts, r, cap_height, is_coeffs = SHAPES[shape]
    polys = _polys(lens, counts)
    whole = _build(pb, polys, r, cap_height, is_coeffs)
    stages = _oracle_stages(oracle, polys, lens, r, cap_height, is_coeffs)
    want_cap = oracle.BatchCommit(polys, r, cap_height, is_coeffs=is_coeffs).cap
    try:
        assert np.array_equal(whole.cap.hashes, want_cap)
        assert np.array_equal(stages[-1][1], want_cap)
        h0 = whole.leaf_heights[0]
        for G in GS:
            caps = []
            for g in range(G):
                mine = _build(pb, polys, r, cap_height, is_coeffs, shard=(g, G))
                try:
                    caps.append(mine.cap.hashes)
                    for k, (grp, (dig, _)) in enumerate(zip(mine.groups, stages)):
                        block = dig.reshape(G, -1, 4)[g] if len(dig) else dig
                        assert np.array_equal(grp.merkle_tree.digests, block), (shape, G, g, "stage", k)
                    rows = (1 << h0) // G
                    local = np.arange(rows, dtype=np.uint64)
                    lv, pt = mine.open_many(local)
                    wlv, wpt = whole.open_many(local + np.uint64(g * rows))
                    assert np.array_equal(lv, wlv) and np.array_equal(pt, wpt), (shape, G, g)
                    for i in (0, rows - 1):
                        for a, b in zip(mine.values(i), whole.values(g * rows + i)):
                            assert np.array_equal(a, b)
                finally:
                    mine.close()
            assert np.array_equal(np.concatenate(caps), want_cap), (shape, G)
    finally:
        whole.close()


@pytest.mark.gpu
@pytest.mark.parametrize("width", [1, 4, 8, 12])
def test_device_stage_hash_widths(pb, oracle, width):
    """Stage 1 hashes `stage 0's cap digest || W-wide row`: W + 4 = 5, 8, 12, 16 words, one or two absorptions."""
    lens, r, cap_height = [7, 5], 2, 3
    polys = _polys(lens, [3, width], seed=0x340 + width)
    go = pb.BatchFriOracle.from_values(polys, r, False, cap_height)
    try:
        c0 = oracle.Commit(np.stack(polys[:3]), r, lens[1] + r)
        c1 = oracle.Commit(np.stack(polys[3:]), r, cap_height)
        leaves = np.concatenate([c0.cap, c1.leaves], axis=1)
        dig, cap = oracle.merkle_build(leaves, cap_height)
        stage = go.groups[1].merkle_tree
        assert np.array_equal(stage.digests, dig) and np.array_equal(stage.cap.hashes, cap)
        assert np.array_equal(go.cap.hashes, oracle.BatchCommit(polys, r, cap_height).cap)
        idx = np.arange(0, 1 << (lens[1] + r), 7, dtype=np.uint64)
        lv, _ = stage.open_many(idx)
        assert np.array_equal(lv, leaves[idx.astype(np.int64)])
        assert np.array_equal(stage.get_rows(0, 4), c1.leaves[:4])
    finally:
        go.close()


def _instances(pb, lens, counts, zeta):
    out, start = [], 0
    for k, c in zip(lens, counts):
        batches = [pb.FriBatchInfo(zeta, [pb.FriPolynomialInfo(0, start + j) for j in range(c)])]
        out.append(pb.FriInstanceInfo([pb.FriOracleInfo(sum(counts), False)], batches))
        start += c
    return out


@pytest.mark.gpu
def test_batch_prove_openings_sharded_on_one_rank_is_batch_prove_openings(pb):
    lens, counts, r, cap_height, arities = [11, 8, 6], [5, 3, 2], 2, 3, [3, 2, 2]
    polys = _polys(lens, counts, seed=0x380)
    params = pb.FriParams(pb.FriConfig(r, cap_height, 7, ("Fixed", arities), 6), False, lens[0], arities)
    go = pb.BatchFriOracle.from_values(polys, r, False, cap_height)
    try:
        proofs = []
        for prove in (pb.batch_prove_openings, D.batch_prove_openings_sharded):
            ch = pb.Challenger()
            ch.observe_cap(go.cap)
            zeta = ch.get_extension_challenge()
            proofs.append(prove(list(lens), _instances(pb, lens, counts, zeta), [go], ch, params).to_bytes())
    finally:
        go.close()
    assert proofs[0] == proofs[1]


@pytest.mark.gpu
def test_batch_prove_openings_across_ranks(pb):
    """torchrun, one rank per GPU (2, or 4 with four GPUs; the ranks share GPU 0 over gloo on a single-GPU machine):
    every rank's bytes equal the single-device proof's and the oracle's, and the restated verifier accepts them."""
    run_ranks("mgpu_batch_fri_check.py", "MGPU_BATCH_FRI_CHECK OK", timeout=900)
