"""Batch FRI (plonky2/src/batch_fri/oracle.rs:30-183, batch_fri/prover.rs:30-258): polynomial commitments over
polynomials of several degrees -- one BatchMerkleTree over the degree groups' LDE rows -- and one FRI proof for all of
them, the lower-degree instances being mixed into the folded codeword when it reaches their length. SURVEY 8(f) row 4.

Device path: every degree group is a PolynomialBatch (coefficients and LDE stay on the device) whose own Merkle tree IS
its stage of the batch tree: the tallest group's tree is built to the height of the next group, and every later group's
tree hashes `previous stage's cap digest j || LDE row j` (gl_commit_finish_prefixed), reading the LDE in place and the
previous cap from device memory. Row-block sharded (shard=(g, G)): rank g holds rows [g*N_k/G, (g+1)*N_k/G) of every
group k; the local cap of its stage k-1 has exactly N_k/G entries, the prefixes of its own rows, so every stage is
rank-local and only the last stage's cap entries cross ranks (distributed.Placement.cap). Every instance's composed
polynomial comes from gl_fri_begin on the (replicated) coefficients, and the rounds are fri.fri_committed_trees with the
lower-degree instances mixed in at their LDE sizes."""
import numpy as np

from . import _native as N
from . import fri as F
from .distributed import Placement, _check_world
from .field import log2_strict
from .hash import NUM_HASH_OUT_ELTS, MerkleProof
from .polynomial_batch import PolynomialBatch


class BatchFriOracle:
    """BatchFriOracle<F, C, D> (batch_fri/oracle.rs:30-40); groups[k] is the degree group k and stage k of the batch
    tree. On a shard, leaf indices (values, open_many) are local to this rank's rows of the tallest group."""

    def __init__(self, groups, degree_bits, rate_bits, cap_height, group_of_poly, ctx):
        self.groups, self.degree_bits, self.rate_bits, self.cap_height = groups, degree_bits, rate_bits, cap_height
        self.group_of_poly, self.ctx = group_of_poly, ctx   # polynomial index -> (group, index inside the group)
        self.blinding = False
        self.leaf_heights = [d + rate_bits for d in degree_bits]
        self.shard_index, self.num_shards = groups[0].shard_index, groups[0].num_shards
        self.lde_size = 1 << self.leaf_heights[0]      # leaves of the tallest group (all shards)
        self.leaf_width = sum(g.num_polys for g in groups)

    @property
    def stages(self):
        """The batch tree's stages: stage k is group k's own commitment."""
        return self.groups

    @property
    def cap(self):
        """The batch tree's cap: the last stage's (on a shard, this rank's cap entries)."""
        return self.groups[-1].merkle_tree.cap

    @classmethod
    def from_values(cls, values, rate_bits, blinding, cap_height, ctx=None, shard=(0, 1)):
        """from_values (oracle.rs:45-68): values = list of 1-D arrays, lengths non-increasing powers of two.
        shard=(g, G): this rank's row block of every group, as in PolynomialBatch.from_values."""
        return cls._build(values, rate_bits, blinding, cap_height, False, ctx, shard)

    @classmethod
    def from_coeffs(cls, polynomials, rate_bits, blinding, cap_height, ctx=None, shard=(0, 1)):
        """from_coeffs (oracle.rs:71-131); shard as in from_values."""
        return cls._build(polynomials, rate_bits, blinding, cap_height, True, ctx, shard)

    @classmethod
    def _build(cls, polys, rate_bits, blinding, cap_height, is_coeffs, ctx, shard):
        if blinding:
            raise NotImplementedError("blinding batch oracles are not supported")
        shard = (int(shard[0]), int(shard[1]))
        _check_world("BatchFriOracle", cap_height, shard[1])
        polys = [np.ascontiguousarray(p, dtype=np.uint64).reshape(-1) for p in polys]
        bits = [log2_strict(len(p)) for p in polys]
        if any(a < b for a, b in zip(bits, bits[1:])):
            raise N.ShapeError("polynomials must be sorted by degree, largest first")   # oracle.rs:83
        if cap_height > bits[-1] + rate_bits:
            raise N.ShapeError("cap_height=%d should be at most last_leaves_cap_height=%d" % (cap_height, bits[-1] + rate_bits))
        ctx = ctx or N.default_context()
        degree_bits = sorted(set(bits), reverse=True)
        group_of_poly = [(degree_bits.index(d), bits[:i].count(d)) for i, d in enumerate(bits)]
        groups = []
        try:
            for k, d in enumerate(degree_bits):
                cols = np.stack([p for p, b in zip(polys, bits) if b == d])
                # stage k is built to the next group's height, the last one to cap_height
                h = degree_bits[k + 1] + rate_bits if k + 1 < len(degree_bits) else cap_height
                groups.append(PolynomialBatch._create(cols, rate_bits, False, h, is_coeffs, None, ctx, shard,
                                                      prefix=groups[-1] if groups else None))
        except Exception:
            for g in groups:
                g.close()
            raise
        return cls(groups, degree_bits, rate_bits, cap_height, group_of_poly, ctx)

    @property
    def polynomials(self):
        return [self.groups[g].polynomials[j] for g, j in self.group_of_poly]

    def values(self, leaf_index):
        """BatchMerkleTree::values (batch_merkle_tree.rs:154-164): the row of every group above leaf_index."""
        h0 = self.leaf_heights[0]
        return [g.merkle_tree.get_rows(leaf_index >> (h0 - hk), 1)[0] for g, hk in zip(self.groups, self.leaf_heights)]

    def open_batch(self, leaf_index):
        """BatchMerkleTree::open_batch (batch_merkle_tree.rs:131-152)."""
        return MerkleProof(self.open_many([leaf_index])[1][0])

    @property
    def merkle_tree(self):
        """The initial-tree view fri_prover_query_rounds opens (open_many)."""
        return self

    def open_many(self, indices):
        """For leaf indices of the tallest matrix, one opening per stage: (per index, `values` back to back (q, W);
        per index, `open_batch` siblings (q, L, 4))."""
        idx = np.asarray(indices, dtype=np.uint64)
        h0 = self.leaf_heights[0]
        opened = [g.merkle_tree.open_many(idx >> np.uint64(h0 - hk)) for g, hk in zip(self.groups, self.leaf_heights)]
        # a later stage's leaf is `previous cap digest || the group's row`
        rows = [lv if k == 0 else lv[:, NUM_HASH_OUT_ELTS:] for k, (lv, _) in enumerate(opened)]
        return np.concatenate(rows, axis=1), np.concatenate([pt for _, pt in opened], axis=1)

    def get_lde_values(self, degree_bits_index, index, step, slice_start, slice_len):
        """get_lde_values (oracle.rs:186-199)."""
        return self.groups[degree_bits_index].get_lde_values(index, step)[slice_start:slice_start + slice_len]

    def close(self):
        for g in self.groups:
            g.close()


def batch_prove_openings(degree_bits, instances, oracles, challenger, fri_params, placement=Placement()):
    """BatchFriOracle::prove_openings + batch_fri_proof (oracle.rs:124-183, prover.rs:30-147). instances[i] opens the
    polynomials of degree 2^degree_bits[i]; polynomial indices are indices into each oracle's full polynomial list.
    placement: where the oracles live, as in fri.prove_openings. With row-block shards over several ranks every rank runs
    the composition, the (replicated) round trees, the mixes and the transcript on the replicated coefficients; only the
    initial-tree openings cross ranks (Placement.open_many), and the proof is the same on every rank and byte-identical to
    the single-device proof. The caller must already have observed the full caps (Placement.cap) in `challenger`."""
    assert len(degree_bits) == len(instances)
    ctx = oracles[0].ctx
    alpha = challenger.get_extension_challenge()
    states, params = [], []
    try:
        for db, inst in zip(degree_bits, instances):
            # the polynomials of this instance live in the degree-`db` group of their oracle
            group_batches, handles, index_of = [], [], {}
            for o_idx, o in enumerate(oracles):
                if db in o.degree_bits:
                    index_of[o_idx] = len(handles)
                    handles.append(o.groups[o.degree_bits.index(db)])
            for b in inst.batches:
                polys = []
                for p in b.polynomials:
                    g, j = oracles[p.oracle_index].group_of_poly[p.polynomial_index]
                    assert oracles[p.oracle_index].degree_bits[g] == db, "polynomial of another degree in this instance"
                    polys.append(F.FriPolynomialInfo(index_of[p.oracle_index], j))
                group_batches.append(F.FriBatchInfo(b.point, polys))
            sub = F.FriInstanceInfo([F.FriOracleInfo(h.num_polys, False) for h in handles], group_batches)
            params.append(F.FriParams(fri_params.config, fri_params.hiding, db, fri_params.reduction_arity_bits))
            states.append(F._begin(sub, handles, alpha, params[-1]))
        # batch_fri_committed_trees (prover.rs:88-147) and batch_fri_prover_query_rounds (prover.rs:149-215)
        rate_bits = fri_params.config.rate_bits
        mixes = [(db + rate_bits, st) for db, st in zip(degree_bits[1:], states[1:])]
        caps, final = F.fri_committed_trees(states[0], challenger, params[0], mixes=mixes)
        pow_witness = F.fri_proof_of_work(challenger, fri_params.config, ctx)
        rounds, _ = F.fri_prover_query_rounds(oracles, states[0], challenger, params[0].lde_size(), params[0], placement)
        return F.FriProof(caps, rounds, final, pow_witness)
    finally:
        for st in states:
            st.close()
