"""BatchMerkleTree (plonky2/src/hash/batch_merkle_tree.rs:16-165), verify_batch_merkle_proof_to_cap
(hash/merkle_proofs.rs:72-107) and Merkle path compression (hash/path_compression.rs:12-113): SURVEY.md section 8(f)
row 4. A batch tree over matrices of decreasing heights is a chain of ordinary Merkle trees -- stage k hashes the rows
`previous stage's cap digest || leaves[k][i]` up to the height of the next matrix -- so every stage is one
gl_merkle_build on the device; only the (small) stage caps pass through the host to be concatenated with the next
matrix."""
import numpy as np

from . import _native as N
from .field import log2_strict
from .hash import MerkleCap, MerkleProof, MerkleTree, PoseidonHash


class BatchMerkleTree:
    """leaves: list of (N_k, W_k) uint64 matrices, heights strictly decreasing powers of two (batch_merkle_tree.rs:34-47)."""

    def __init__(self, leaves, cap_height, ctx=None):
        self.ctx = ctx or N.default_context()
        leaves = [np.ascontiguousarray(m, dtype=np.uint64) for m in leaves]
        if not leaves or any(m.ndim != 2 for m in leaves):
            raise N.ShapeError("leaves must be a non-empty list of (N_k, W_k) matrices")
        heights = [log2_strict(len(m)) for m in leaves]            # "Not a power of two" like the reference's assert
        if any(a <= b for a, b in zip(heights, heights[1:])):
            raise N.ShapeError("matrices must be sorted by height, tallest first, with no duplicate heights")
        if cap_height > heights[-1]:
            raise N.ShapeError("cap_height=%d should be at most last_leaves_cap_height=%d" % (cap_height, heights[-1]))
        self.leaves, self.leaf_heights, self.cap_height = leaves, heights, cap_height
        first = MerkleTree(leaves[0], heights[1] if len(leaves) > 1 else cap_height, self.ctx)
        self.stages, self.cap = _stage_chain(first, leaves[1:], heights, cap_height, self.ctx)

    @property
    def digests(self):
        """The reference's flat `digests`: the stages' digest buffers back to back (batch_merkle_tree.rs:56-110)."""
        parts = [t.digests for t in self.stages]
        return np.concatenate(parts) if parts else np.zeros((0, 4), dtype=np.uint64)

    def open_batch(self, leaf_index):
        """open_batch (batch_merkle_tree.rs:131-152): the stages' sibling paths concatenated."""
        h0 = self.leaf_heights[0]
        sib = [t.open_many([leaf_index >> (h0 - hk)])[1][0] for t, hk in zip(self.stages, self.leaf_heights)]
        return MerkleProof(np.concatenate(sib) if sib else np.zeros((0, 4), dtype=np.uint64))

    def values(self, leaf_index):
        """values (batch_merkle_tree.rs:154-164): the row of every matrix above leaf_index."""
        h0 = self.leaf_heights[0]
        return [m[leaf_index >> (h0 - hk)].copy() for m, hk in zip(self.leaves, self.leaf_heights)]

    def close(self):
        for t in self.stages:
            t.close()


def _stage_chain(first, later, heights, cap_height, ctx):
    """The stages of a batch tree whose matrices have leaf heights `heights`: `first` is stage 0 (any tree with a
    `cap`), stage k >= 1 hashes the rows `previous stage's cap digest || later[k - 1][i]` (cap_hash || cur[i]) up to
    the height of the next matrix, or to cap_height after the last. `later` is read one matrix per stage, so it may be
    a generator. Returns (stages, the batch tree's cap)."""
    stages, cap = [first], first.cap.hashes
    for k, m in enumerate(later, 1):
        t = MerkleTree(np.ascontiguousarray(np.concatenate([cap, m], axis=1)),
                       heights[k + 1] if k + 1 < len(heights) else cap_height, ctx)
        stages.append(t)
        cap = t.cap.hashes
    return stages, MerkleCap(cap)


def verify_batch_merkle_proof_to_cap(leaf_data, leaf_heights, leaf_index, merkle_cap, proof, ctx=None):
    """verify_batch_merkle_proof_to_cap (merkle_proofs.rs:72-107). Raises ValueError("Invalid Merkle proof.")."""
    assert len(leaf_data) == len(leaf_heights)
    cur = PoseidonHash.hash_or_noop(leaf_data[0], ctx)
    height, k = leaf_heights[0], 1
    for sib in proof.siblings:
        bit = leaf_index & 1
        leaf_index >>= 1
        cur = PoseidonHash.two_to_one(sib, cur, ctx) if bit else PoseidonHash.two_to_one(cur, sib, ctx)
        height -= 1
        if k < len(leaf_heights) and height == leaf_heights[k]:
            cur = PoseidonHash.hash_or_noop(np.concatenate([cur, np.asarray(leaf_data[k], dtype=np.uint64)]), ctx)
            k += 1
    assert k == len(leaf_data)
    if not np.array_equal(cur, merkle_cap.hashes[leaf_index]):
        raise ValueError("Invalid Merkle proof.")


def compress_merkle_proofs(cap_height, indices, proofs):
    """compress_merkle_proofs (path_compression.rs:12-50): drop every sibling a verifier can recompute from the other
    opened leaves and proofs."""
    assert len(proofs) > 0
    height = cap_height + len(proofs[0].siblings)
    num_leaves = 1 << height
    known = np.zeros(2 * num_leaves, dtype=bool)
    for i in indices:
        for j in range(height - cap_height):
            known[(i + num_leaves) >> j] = True
    out = []
    for i, p in zip(indices, proofs):
        keep, index = [], i + num_leaves
        for sib in p.siblings:
            s = index ^ 1
            if not known[s]:
                keep.append(sib)
                known[s] = True
            index >>= 1
            known[index] = True
        out.append(MerkleProof(np.array(keep, dtype=np.uint64).reshape(-1, 4)))
    return out


def decompress_merkle_proofs(leaves_data, leaves_indices, compressed_proofs, height, cap_height, ctx=None):
    """decompress_merkle_proofs (path_compression.rs:54-113): rebuild the full sibling paths, hashing layer by layer
    (one batched two_to_one per layer on the device instead of one call per node)."""
    num_leaves = 1 << height
    seen = {}
    digests = PoseidonHash.hash_many(np.asarray(leaves_data, dtype=np.uint64), ctx) if len(leaves_data) else []
    for i, d in zip(leaves_indices, digests):
        seen[i + num_leaves] = d
    its = [iter(p.siblings) for p in compressed_proofs]
    for layer in range(height - cap_height):
        todo, pairs = [], []
        for i, it in zip(leaves_indices, its):
            index = (i + num_leaves) >> layer
            sibling_index = index ^ 1
            if sibling_index not in seen:
                seen[sibling_index] = next(it)
            if (index >> 1) not in seen and (index >> 1) not in todo:
                lo, hi = (index, sibling_index) if index % 2 == 0 else (sibling_index, index)
                todo.append(index >> 1)
                pairs.append(np.concatenate([seen[lo], seen[hi]]))
        if pairs:
            for parent, hsh in zip(todo, PoseidonHash.two_to_one_many(np.array(pairs, dtype=np.uint64), ctx)):
                seen[parent] = hsh
    out = []
    for i in leaves_indices:
        index, sib = i + num_leaves, []
        for _ in range(height - cap_height):
            sib.append(seen[index ^ 1])
            index >>= 1
        out.append(MerkleProof(np.array(sib, dtype=np.uint64).reshape(-1, 4)))
    return out
