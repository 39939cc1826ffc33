"""PolynomialBatch mirroring plonky2/src/fri/oracle.rs:30-237: a batch of polynomials committed with a
Poseidon Merkle tree over its coset LDE. All bulk data stays on the GPU behind a gl_commit handle; the
reference's public fields (`polynomials`, `merkle_tree.{leaves,digests,cap}`) are read back on demand."""
import ctypes as C

import numpy as np

from . import _native as N
from .field import log2_strict
from .hash import NUM_HASH_OUT_ELTS, MerkleCap, MerkleProof, _open_leaves, _read_digests
from .proof import eval_commitments

SALT_SIZE = 4  # oracle.rs:26


def random_field_elements(count):
    """Uniform canonical field elements from the OS CSPRNG (F::rand, field/src/goldilocks_field.rs:61-64):
    64-bit draws, rejecting values >= p -- vectorised. A 2^23 x 4 salt takes about 0.8 s on a 16-core host
    (not minutes); salt_key= draws it on the device in under a millisecond instead."""
    import os

    from .field import ORDER

    out = np.empty(count, dtype=np.uint64)
    filled = 0
    while filled < count:
        need = count - filled
        cand = np.frombuffer(os.urandom(8 * (need + need // 1024 + 16)), dtype="<u8")
        cand = cand[cand < np.uint64(ORDER)][:need]
        out[filled:filled + len(cand)] = cand
        filled += len(cand)
    return out


def _salt_key(salt_key):
    """A salt_key argument as the C ABI takes it: the 32 key bytes, or None for "fresh" (the library draws a key from
    the OS CSPRNG)."""
    if isinstance(salt_key, str) and salt_key == "fresh":
        return None
    if isinstance(salt_key, (bytes, bytearray)) and len(salt_key) == 32:
        return bytes(salt_key)
    raise N.ShapeError("salt_key must be 32 bytes or 'fresh'")


def random_field_elements_keyed(key, column, first, count, ctx=None):
    """Elements first .. first + count - 1 of stream `column` of the device salt sampler for a 32-byte key
    (gl_random_field_elements; the sampling rule is documented in csrc/gl_chacha.cuh): uniform canonical field elements,
    each a function of (key, column, position) alone. A keyed commitment's salt column s at LDE row i is element i of
    stream s."""
    ctx = ctx or N.default_context()
    key = _salt_key(key)
    if key is None:
        raise N.ShapeError("random_field_elements_keyed needs an explicit 32-byte key")
    out = np.empty(int(count), dtype=np.uint64)
    N.check(N.lib().gl_random_field_elements(ctx.h, key, int(column), int(first), int(count), N.np_ptr(out),
                                             N.MEM_HOST), ctx.h)
    return out


def check_lde_blocks(lde_blocks, cap_height, *, blinding=False, salt=None, salt_key=None, shard=(0, 1), prefix=None):
    """The refusals of lde_blocks=G (a non-resident batch), before any device work: G must be a power of two of at most
    2^cap_height (each block holds whole cap subtrees), and the batch unblinded, unsharded and not a prefixed stage."""
    if lde_blocks is None:
        return
    G = int(lde_blocks)
    if G <= 0 or G & (G - 1):
        raise N.ShapeError("lde_blocks=%d is not a positive power of two" % G)
    if G > 1 << cap_height:
        raise N.ShapeError("lde_blocks=%d exceeds the %d cap entries (cap_height %d): blocks own whole cap subtrees"
                           % (G, 1 << cap_height, cap_height))
    if blinding or salt is not None or salt_key is not None:
        raise N.ShapeError("a non-resident batch (lde_blocks=) cannot be blinded or salted")
    if tuple(shard) != (0, 1):
        raise N.ShapeError("lde_blocks= cannot be combined with shard=")
    if prefix is not None:
        raise N.ShapeError("lde_blocks= cannot be combined with prefix=")


class _DeviceMerkleTree:
    """View of PolynomialBatch.merkle_tree (merkle_tree.rs:46-62) living on the device."""

    def __init__(self, batch):
        self._b = batch

    @property
    def cap(self):
        """The Merkle cap (for a sharded batch: this shard's cap entries; see distributed.gather_cap)."""
        b = self._b
        out = np.empty(((1 << b.cap_height) // b.num_shards, 4), dtype=np.uint64)
        N.check(N.lib().gl_commit_cap(b.h, N.np_ptr(out), N.MEM_HOST), b.ctx.h)
        return MerkleCap(out)

    @property
    def leaves(self):
        return self.get_rows(0, self._b.local_rows)

    def get_rows(self, begin, count):
        b = self._b
        out = np.empty((count, b.leaf_width), dtype=np.uint64)
        if count:
            N.check(N.lib().gl_commit_leaves(b.h, begin, count, N.np_ptr(out), N.MEM_HOST), b.ctx.h)
        return out

    @property
    def digests(self):
        b = self._b
        count = 2 * (b.local_rows - (1 << b.cap_height) // b.num_shards)
        return _read_digests(N.lib().gl_commit_digests, b.h, b.ctx, count)

    def get(self, i):
        return self.get_rows(i, 1)[0]

    def open_many(self, indices):
        """(leaves (q, W), paths (q, L, 4)) for local leaf indices; a prefixed batch's leaves are `prefix || row`, W + 4
        words."""
        b = self._b
        layers = b.degree_log + b.rate_bits - b.cap_height  # local rows and local cap shrink together
        width = b.leaf_width + (NUM_HASH_OUT_ELTS if b.prefixed else 0)
        return _open_leaves(N.lib().gl_commit_open, b.h, b.ctx, indices, width, layers)

    def prove(self, leaf_index):
        return MerkleProof(self.open_many([leaf_index])[1][0])


class PolynomialBatch(N.Handle):
    """PolynomialBatch<F, PoseidonGoldilocksConfig, 2> (oracle.rs:30-37)."""
    destroyer = "gl_commit_destroy"

    def __init__(self, handle, ctx, num_polys, degree_log, rate_bits, cap_height, blinding, shard=(0, 1), lde_blocks=0):
        self.h, self.ctx = handle, ctx
        self.shard_index, self.num_shards = shard
        self.lde_blocks = lde_blocks  # G of a non-resident batch (its LDE is rebuilt block by block where read), else 0
        self.num_polys, self.degree_log, self.rate_bits = num_polys, degree_log, rate_bits
        self.cap_height, self.blinding = cap_height, blinding
        self.leaf_width = num_polys + (SALT_SIZE if blinding else 0)
        self.lde_size = 1 << (degree_log + rate_bits)
        self.local_rows = self.lde_size // self.num_shards  # leaf rows [shard*local_rows, (shard+1)*local_rows)
        self.prefixed = False  # a later stage of a batch Merkle tree: leaf j is `prefix j || LDE row j` (_from_device)
        self.merkle_tree = _DeviceMerkleTree(self)

    @classmethod
    def _create(cls, cols, rate_bits, blinding, cap_height, is_coeffs, salt, ctx, shard=(0, 1), salt_key=None,
                prefix=None, lde_blocks=None):
        check_lde_blocks(lde_blocks, cap_height, blinding=blinding, salt=salt, salt_key=salt_key, shard=shard,
                         prefix=prefix)
        ctx = ctx or N.default_context()
        cols = np.ascontiguousarray(cols, dtype=np.uint64)
        if cols.ndim != 2 or cols.shape[0] == 0:
            raise N.ShapeError("expected a non-empty (num_polys, degree) array")
        B, n = cols.shape
        log_n = log2_strict(n)
        if salt is not None and (salt_key is not None or prefix is not None or lde_blocks is not None):
            raise N.ShapeError("salt= is exclusive with salt_key= and prefix=")
        if blinding and salt_key is None and prefix is None:
            if salt is None:
                # the reference draws the salt from OsRng (oracle.rs:133-137); same source here
                salt = random_field_elements(SALT_SIZE * (n << rate_bits)).reshape(SALT_SIZE, -1)
            salt = np.ascontiguousarray(salt, dtype=np.uint64)
            if salt.shape != (SALT_SIZE, n << rate_bits):
                raise N.ShapeError("salt must be (4, n << rate_bits)")
        else:
            salt = None  # without blinding, a salt argument is ignored
        kind = N.COLS_COEFFS if is_coeffs else N.COLS_VALUES

        def add_columns(h):
            N.check(N.lib().gl_commit_add_columns(h, 0, B, N.np_ptr(cols), n, kind, N.MEM_HOST), ctx.h)

        return cls._from_device(ctx, B, log_n, rate_bits, cap_height, add_columns, blinding=blinding, salt=salt,
                                salt_key=salt_key, shard=shard, prefix=prefix, lde_blocks=lde_blocks, wait=False)

    @classmethod
    def _from_device(cls, ctx, num_polys, degree_log, rate_bits, cap_height, add_columns, *, blinding=False,
                     salt=None, salt_key=None, shard=(0, 1), prefix=None, lde_blocks=None, wait=True):
        """A batch committed incrementally: gl_commit_begin, then add_columns(h) issues the gl_commit_add_columns calls
        on the unfinished handle h, then gl_commit_finish -- with blinding, over the host salt array `salt` (4 x N, by
        LDE row) if given, else through gl_commit_finish_keyed: the salt is drawn on the device from salt_key (32 bytes;
        None or "fresh": a key from the OS CSPRNG). shard=(g, G): only leaf rows [g*N/G, (g+1)*N/G) on this device, as
        in from_values. prefix: a finished PolynomialBatch whose local cap has one entry per local leaf of this one; the
        tree is then a later stage of a batch Merkle tree, over the leaves `its cap entry j || LDE row j`
        (gl_commit_finish_prefixed). lde_blocks=G: a non-resident batch (gl_commit_begin_blocked), as in from_values.
        The columns' device memory only has to live until this returns; wait=False skips that wait on the library's
        stream, for host columns (pageable or pinned) and a host salt, which the library has read when
        gl_commit_add_columns and gl_commit_finish return."""
        check_lde_blocks(lde_blocks, cap_height, blinding=blinding, salt_key=salt_key, shard=shard, prefix=prefix)
        if salt_key is not None and not blinding:
            raise N.ShapeError("salt_key= needs blinding=True")
        if prefix is not None:
            if blinding:
                raise N.ShapeError("a prefixed commitment cannot be blinded")
            entries, rows = (1 << prefix.cap_height) // prefix.num_shards, (1 << (degree_log + rate_bits)) // shard[1]
            if entries != rows:
                raise N.ShapeError("the prefix has %d cap entries for %d leaves" % (entries, rows))
        key = _salt_key(salt_key) if salt_key is not None else None
        h = N.vp()
        if lde_blocks is not None:
            N.check(N.lib().gl_commit_begin_blocked(ctx.h, num_polys, degree_log, rate_bits, cap_height, int(lde_blocks),
                                                    None, C.byref(h)), ctx.h)
        else:
            N.check(N.lib().gl_commit_begin(ctx.h, num_polys, degree_log, rate_bits, cap_height, int(bool(blinding)),
                                            int(shard[0]), int(shard[1]), None, C.byref(h)), ctx.h)
        batch = cls(h, ctx, num_polys, degree_log, rate_bits, cap_height, bool(blinding), (int(shard[0]), int(shard[1])),
                    int(lde_blocks or 0))
        try:
            add_columns(h)
            if prefix is not None:
                N.check(N.lib().gl_commit_finish_prefixed(h, N.lib().gl_commit_dev_cap(prefix.h)), ctx.h)
                batch.prefixed = True
            elif salt is not None:
                N.check(N.lib().gl_commit_finish(h, N.np_ptr(salt), N.MEM_HOST), ctx.h)
            elif blinding:
                N.check(N.lib().gl_commit_finish_keyed(h, key), ctx.h)
            else:
                N.check(N.lib().gl_commit_finish(h, None, N.MEM_DEVICE), ctx.h)
            if wait:
                ctx.synchronize()  # the library's stream-ordered reads of the caller's (torch) columns are done
        except Exception:
            batch.close()
            raise
        return batch

    @classmethod
    def _from_coeff_chunks(cls, polys, chunks, degree_log, rate_bits, cap_height, ctx=None, *, blinding=False,
                           salt_key=None, shard=(0, 1), lde_blocks=None):
        """Every row of the device tensor `polys` cut into `chunks` coefficient polynomials of 2^degree_log, committed
        in row order: the quotient commitment of plonky2 and starky (plonk/prover.rs:319-352, starky/prover.rs:391-421).
        blinding / salt_key / shard / lde_blocks: as in _from_device."""
        check_lde_blocks(lde_blocks, cap_height, blinding=blinding, salt_key=salt_key, shard=shard)
        ctx = ctx or N.default_context()
        n = 1 << degree_log
        ctx.after_caller()

        def add_columns(h):
            for j in range(polys.shape[0]):
                N.check(N.lib().gl_commit_add_columns(h, j * chunks, chunks, N.vp(polys[j].data_ptr()), n,
                                                      N.COLS_COEFFS, N.MEM_DEVICE), ctx.h)

        return cls._from_device(ctx, polys.shape[0] * chunks, degree_log, rate_bits, cap_height, add_columns,
                                blinding=blinding, salt_key=salt_key, shard=shard, lde_blocks=lde_blocks)

    @classmethod
    def from_values(cls, values, rate_bits, blinding, cap_height, timing=None, fft_root_table=None, *,
                    salt=None, ctx=None, shard=(0, 1), salt_key=None, lde_blocks=None):
        """from_values (oracle.rs:57-79). `timing`/`fft_root_table` are accepted for signature parity.
        shard=(g, G): build only leaf rows [g*N/G, (g+1)*N/G) on this device (multi-GPU row-block sharding).
        With blinding, the salt is `salt` (4 x N, by LDE row), else, with salt_key (32 bytes, or "fresh" for a key from
        the OS CSPRNG), drawn on the device: salt column s at LDE row i = random_field_elements_keyed(key, s, i, 1);
        else drawn on the host from the OS CSPRNG.
        lde_blocks=G: a non-resident batch, for LDEs larger than device memory. It keeps its coefficients, digests and cap
        but never its LDE: the LDE is built in G row blocks to be hashed, and the blocks a reader asks for are rebuilt
        (merkle_tree.leaves / get_rows / open_many / prove, get_lde_values). Everything it returns equals the resident
        batch's. check_lde_blocks lists its refusals."""
        return cls._create(values, rate_bits, blinding, cap_height, False, salt, ctx, shard, salt_key,
                           lde_blocks=lde_blocks)

    @classmethod
    def from_coeffs(cls, polynomials, rate_bits, blinding, cap_height, timing=None, fft_root_table=None, *,
                    salt=None, ctx=None, shard=(0, 1), salt_key=None, lde_blocks=None):
        """from_coeffs (oracle.rs:82-112); salt / salt_key / lde_blocks as in from_values."""
        return cls._create(polynomials, rate_bits, blinding, cap_height, True, salt, ctx, shard, salt_key,
                           lde_blocks=lde_blocks)

    @property
    def polynomials(self):
        out = np.empty((self.num_polys, 1 << self.degree_log), dtype=np.uint64)
        N.check(N.lib().gl_commit_coeffs(self.h, N.np_ptr(out), N.MEM_HOST), self.ctx.h)
        return out

    def get_lde_values(self, index, step):
        """get_lde_values (oracle.rs:142-147)."""
        out = np.empty(self.num_polys, dtype=np.uint64)
        N.check(N.lib().gl_commit_get_lde_values(self.h, index, step, N.np_ptr(out)), self.ctx.h)
        return out

    def eval_commitment(self, z):
        """eval_commitment of OpeningSet::new (plonk/proof.rs:313-351): every polynomial at z in F_{p^2};
        returns (num_polys, 2)."""
        return eval_commitments([(self, z)])[0]

    @staticmethod
    def prove_openings(instance, oracles, challenger, fri_params, final_poly_coeff_len=None,
                       max_num_query_steps=None, timing=None):
        """prove_openings (oracle.rs:176-237)."""
        from .fri import prove_openings

        return prove_openings(instance, oracles, challenger, fri_params, final_poly_coeff_len,
                              max_num_query_steps)
