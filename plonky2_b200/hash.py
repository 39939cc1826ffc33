"""Poseidon hasher and Merkle tree mirroring plonky2/src/plonk/config.rs:36-77,
plonky2/src/hash/poseidon.rs:804-887, plonky2/src/hash/hashing.rs:97-145 and
plonky2/src/hash/merkle_tree.rs:14-62,193-237. Batched work runs on the GPU; the single
permutation used by the sequential transcript runs on the host from the same source."""
import ctypes as C

import numpy as np

from . import _native as N
from .field import ORDER, log2_strict

SPONGE_RATE = 8
SPONGE_CAPACITY = 4
SPONGE_WIDTH = 12
NUM_HASH_OUT_ELTS = 4


class PoseidonPermutation:
    """PlonkyPermutation for Poseidon-12 on the host (hashing.rs:62-94, poseidon.rs:804-870)."""

    RATE = SPONGE_RATE
    WIDTH = SPONGE_WIDTH

    def __init__(self, elts=()):
        self.state = np.zeros(SPONGE_WIDTH, dtype=np.uint64)
        self.set_from_iter(elts, 0)

    def set_elt(self, elt, idx):
        self.state[idx] = int(elt) % (1 << 64)

    def set_from_slice(self, elts, start_idx):
        elts = [int(e) for e in elts]
        self.state[start_idx:start_idx + len(elts)] = np.array(elts, dtype=np.uint64)

    def set_from_iter(self, elts, start_idx):
        for i, e in zip(range(start_idx, SPONGE_WIDTH), elts):
            self.state[i] = int(e)

    def permute(self):
        N.lib().gl_poseidon_permute_host(N.np_ptr(self.state))

    def squeeze(self):
        return self.state[:SPONGE_RATE]

    def copy(self):
        p = PoseidonPermutation()
        p.state = self.state.copy()
        return p


def _hash_rows(fn, rows, ctx):
    """One digest per row of an (n_items, W) array from the library's batch hash `fn` -> (n_items, 4)."""
    ctx = ctx or N.default_context()
    rows = np.ascontiguousarray(rows, dtype=np.uint64)
    n, w = rows.shape
    out = np.empty((n, 4), dtype=np.uint64)
    if n:
        N.check(fn(ctx.h, N.np_ptr(rows) if w else None, n, w, N.np_ptr(out), N.MEM_HOST), ctx.h)
    return out


class PoseidonHash:
    """Hasher<GoldilocksField> (config.rs:36-77, poseidon.rs:872-887). Hash = 4 canonical u64."""

    HASH_SIZE = 32

    @staticmethod
    def permute_many(states, ctx=None):
        """PoseidonPermutation::permute on every row of an (n_items, 12) array, on the device -> (n_items, 12)."""
        ctx = ctx or N.default_context()
        st = np.array(states, dtype=np.uint64).reshape(-1, SPONGE_WIDTH).copy()
        if len(st):
            N.check(N.lib().gl_poseidon_permute_many(ctx.h, N.np_ptr(st), len(st), N.MEM_HOST), ctx.h)
        return st

    @staticmethod
    def hash_many(rows, ctx=None):
        """hash_or_noop for every row of an (n_items, W) array -> (n_items, 4)."""
        return _hash_rows(N.lib().gl_poseidon_hash_many, rows, ctx)

    @staticmethod
    def hash_or_noop(inputs, ctx=None):
        return PoseidonHash.hash_many(np.asarray(inputs, dtype=np.uint64).reshape(1, -1), ctx)[0]

    @staticmethod
    def hash_no_pad_many(rows, ctx=None):
        """hash_no_pad (always the sponge) for every row of an (n_items, W) array -> (n_items, 4)."""
        return _hash_rows(N.lib().gl_poseidon_hash_no_pad_many, rows, ctx)

    @staticmethod
    def hash_no_pad(inputs, ctx=None):
        return PoseidonHash.hash_no_pad_many(np.asarray(inputs, dtype=np.uint64).reshape(1, -1), ctx)[0]

    @staticmethod
    def hash_no_pad_host(inputs):
        """hash_n_to_hash_no_pad (hash/hashing.rs:96-123) on the HOST permutation: for the verifier-side replays of a
        transcript (a handful of elements), where a device round trip buys nothing."""
        perm = PoseidonPermutation()
        inputs = [int(x) for x in inputs]
        for at in range(0, len(inputs), SPONGE_RATE):
            perm.set_from_slice(inputs[at:at + SPONGE_RATE], 0)
            perm.permute()
        return np.array(perm.squeeze()[:NUM_HASH_OUT_ELTS], dtype=np.uint64)

    @staticmethod
    def _pad(inputs):
        """The pad10*1 rule of hash_pad (config.rs:50-59)."""
        padded = [int(x) for x in inputs] + [1]
        while (len(padded) + 1) % SPONGE_RATE != 0:
            padded.append(0)
        return padded + [1]

    @staticmethod
    def hash_pad(inputs, ctx=None):
        """pad10*1 then hash_no_pad (config.rs:50-59)."""
        return PoseidonHash.hash_no_pad(np.array(PoseidonHash._pad(inputs), dtype=np.uint64), ctx)

    @staticmethod
    def hash_pad_host(inputs):
        """hash_pad on the HOST permutation."""
        return PoseidonHash.hash_no_pad_host(PoseidonHash._pad(inputs))

    @staticmethod
    def two_to_one_many(pairs, ctx=None):
        ctx = ctx or N.default_context()
        pairs = np.ascontiguousarray(pairs, dtype=np.uint64).reshape(-1, 8)
        out = np.empty((len(pairs), 4), dtype=np.uint64)
        if len(pairs):
            N.check(N.lib().gl_poseidon_two_to_one_many(ctx.h, N.np_ptr(pairs), len(pairs), N.np_ptr(out),
                                                        N.MEM_HOST), ctx.h)
        return out

    @staticmethod
    def two_to_one(left, right, ctx=None):
        return PoseidonHash.two_to_one_many(np.concatenate([np.asarray(left, dtype=np.uint64),
                                                            np.asarray(right, dtype=np.uint64)]), ctx)[0]


class MerkleCap:
    """MerkleCap (merkle_tree.rs:14-43): (2^h, 4) array of digests."""

    def __init__(self, hashes):
        self.hashes = np.asarray(hashes, dtype=np.uint64).reshape(-1, 4)

    def __len__(self):
        return len(self.hashes)

    def height(self):
        return log2_strict(len(self.hashes))

    def flatten(self):
        return self.hashes.reshape(-1)

    def __eq__(self, other):
        return isinstance(other, MerkleCap) and np.array_equal(self.hashes, other.hashes)


class MerkleProof:
    def __init__(self, siblings):
        self.siblings = np.asarray(siblings, dtype=np.uint64).reshape(-1, 4)


def _read_digests(fn, h, ctx, count):
    """The (count, 4) digest buffer of a device tree through the library's digest read-back `fn`."""
    out = np.empty((count, 4), dtype=np.uint64)
    if out.size:
        N.check(fn(h, N.np_ptr(out), N.MEM_HOST), ctx.h)
    return out


def _open_leaves(fn, h, ctx, indices, width, layers):
    """(leaves (q, width), sibling paths (q, layers, 4)) of a device tree at `indices` through the library's opening
    `fn`."""
    idx = np.ascontiguousarray(indices, dtype=np.uint64)
    leaves = np.empty((len(idx), width), dtype=np.uint64)
    paths = np.empty((len(idx), layers, 4), dtype=np.uint64)
    if len(idx):
        N.check(fn(h, N.np_ptr(idx), len(idx), N.np_ptr(leaves), N.np_ptr(paths) if paths.size else None), ctx.h)
    return leaves, paths


class MerkleTree(N.Handle):
    """MerkleTree<F, PoseidonHash> built on the GPU (merkle_tree.rs:46-62,193-237). The public fields of
    the reference (`leaves`, `digests`, `cap`) are properties that copy from the device on demand."""
    destroyer = "gl_merkle_destroy"

    def __init__(self, leaves, cap_height, ctx=None):
        self.ctx = ctx or N.default_context()
        # a copy of its own, as the reference's tree owns its Vec: `leaves` and get() stay the leaves the tree was
        # built from when the caller refills its array
        leaves = np.array(leaves, dtype=np.uint64, order="C")
        if leaves.ndim != 2:
            raise N.ShapeError("leaves must be (N, W)")
        self.N, self.W = leaves.shape
        self.cap_height = cap_height
        self._leaves = leaves
        h = N.vp()
        N.check(N.lib().gl_merkle_build(self.ctx.h, N.np_ptr(leaves), self.N, self.W, cap_height, N.MEM_HOST,
                                        C.byref(h)), self.ctx.h)
        self.h = h

    @property
    def leaves(self):
        return self._leaves

    @property
    def cap(self):
        out = np.empty((1 << self.cap_height, 4), dtype=np.uint64)
        N.check(N.lib().gl_merkle_cap(self.h, N.np_ptr(out), N.MEM_HOST), self.ctx.h)
        return MerkleCap(out)

    @property
    def digests(self):
        return _read_digests(N.lib().gl_merkle_digests, self.h, self.ctx, 2 * (self.N - (1 << self.cap_height)))

    def get(self, i):
        return self._leaves[i]

    def open_many(self, indices):
        return _open_leaves(N.lib().gl_merkle_open, self.h, self.ctx, indices, self.W,
                            log2_strict(self.N) - self.cap_height)

    def prove(self, leaf_index):
        return MerkleProof(self.open_many([leaf_index])[1][0])


def verify_merkle_proof_to_cap(leaf_data, leaf_index, merkle_cap, proof, ctx=None):
    """verify_merkle_proof_to_cap (merkle_proofs.rs:55-107), hashing on the GPU one node at a time.
    Raises ValueError("Invalid Merkle proof.") like the reference's ensure!."""
    cur = PoseidonHash.hash_or_noop(leaf_data, ctx)
    for sib in proof.siblings:
        bit = leaf_index & 1
        leaf_index >>= 1
        cur = PoseidonHash.two_to_one(sib, cur, ctx) if bit else PoseidonHash.two_to_one(cur, sib, ctx)
    if not np.array_equal(cur, merkle_cap.hashes[leaf_index]):
        raise ValueError("Invalid Merkle proof.")
