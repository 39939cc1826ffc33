"""Multi-GPU plumbing for the row-block sharded commitment (SURVEY.md section 8e): one process per GPU,
torch.distributed (NCCL on GPUs, gloo in CPU tests) for the exchange the path needs -- an all-gather of the shards'
Merkle-cap entries (2^cap_height x 32 bytes in total) -- and PipelinedCommitter for the optional second axis
(column-sharded iNTT whose stores are the coefficient all-gather over NVLink).

No LDE data ever crosses NVLink: shard g of G evaluates every column on its own coset
(g_shift * w_N^{bitrev(g)}) <w_{N/G}>, hashes its leaves and reduces its own cap subtrees.

prove_stark proves one STARK, prove_with_ctls a multi-STARK system with cross-table lookups, and prove_plonk one
plonky2 circuit, on the ranks of a group with these shards: besides the caps, only the quotient's values on each rank's
shard of the quotient coset (Placement.quotient_from_shards), the partial sums of the openings over each rank's block
of coefficients (Placement.openings_from_shards) and the FRI query openings (Placement.open_many) cross ranks. The
provers take a Placement -- Placement() on one device -- and never ask themselves whether there is more than one rank.
prove_openings_sharded is fri.prove_openings, and batch_prove_openings_sharded batch_fri.batch_prove_openings, on the
oracles' own shards, for a caller that commits the shards itself."""
from dataclasses import dataclass

import numpy as np

from .hash import MerkleCap


def shard_row_range(lde_size, shard_index, num_shards):
    """Leaf rows [begin, end) of the single-device tree that shard `shard_index` owns."""
    assert lde_size % num_shards == 0
    rows = lde_size // num_shards
    return shard_index * rows, (shard_index + 1) * rows


def shard_cap_range(cap_height, shard_index, num_shards):
    """Cap entries [begin, end) owned by the shard (whole cap subtrees: num_shards <= 2^cap_height)."""
    c = 1 << cap_height
    if num_shards > c:
        raise ValueError("num_shards=%d exceeds the cap size %d" % (num_shards, c))
    per = c // num_shards
    return shard_index * per, (shard_index + 1) * per


def owner_of_leaf(leaf_index, lde_size, num_shards):
    """(shard, local leaf index) holding leaf `leaf_index` of the single-device tree."""
    rows = lde_size // num_shards
    return leaf_index // rows, leaf_index % rows


def gather_cap(local_cap, group=None, device=None):
    """All-gather the shards' cap entries into the full MerkleCap (identical on every rank and equal to
    the single-device cap). `local_cap`: (C/G, 4) uint64 array or MerkleCap."""
    import torch
    import torch.distributed as dist

    hashes = local_cap.hashes if isinstance(local_cap, MerkleCap) else np.asarray(local_cap, dtype=np.uint64)
    hashes = np.ascontiguousarray(hashes, dtype=np.uint64).reshape(-1, 4)
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return MerkleCap(hashes.copy())
    world = dist.get_world_size(group)
    t = torch.from_numpy(hashes.view(np.int64).copy())
    if device is not None:
        t = t.to(device)
    out = torch.empty((world * t.shape[0], 4), dtype=torch.int64, device=t.device)
    dist.all_gather_into_tensor(out, t, group=group)
    full = out.cpu().numpy().view(np.uint64).reshape(-1, 4)
    return MerkleCap(full.copy())


@dataclass(frozen=True)
class Placement:
    """Where a prover's commitments live: row block `shard_index` of `num_shards` of every commitment, one block per rank
    of the torch.distributed `group`. Placement() is one device. The provers build every commitment with
    `commit_kwargs`, observe `cap`, and run the quotient, the openings and FRI with `step_kwargs` (fri.prove_openings
    opens its queries with `open_many`); the two compute_quotient_polys and proof.eval_commitments pick their C entry
    point by num_shards and, with several ranks, gather the quotient with `quotient_from_shards` and the openings with
    `openings_from_shards`. Nothing else in the provers tests whether there is more than one rank. On one device both
    keyword sets are empty, so every call a prover makes is the plain single-device call. check_constraints runs with
    `check_kwargs`: each rank checks its own part of H and the ranks merge their reports (`report_from_shards`).
    lde_blocks=G (one device only) makes every commitment non-resident, its LDE built in G row blocks where it is
    hashed or read (PolynomialBatch.from_values); the C entry points take such commitments directly, so step_kwargs
    stays empty, and check_kwargs checks H in G parts one after another."""
    shard_index: int = 0
    num_shards: int = 1
    group: object = None
    lde_blocks: int = 0

    def __post_init__(self):
        from . import _native as N

        if self.lde_blocks and self.num_shards > 1:
            raise N.ShapeError("lde_blocks= proves on one device; it cannot be combined with %d shards" % self.num_shards)

    @property
    def shard(self):
        """(g, G): the shard= of every commitment on this placement; (0, 1) builds the unsharded commitment."""
        return self.shard_index, self.num_shards

    @property
    def commit_kwargs(self):
        """The keyword arguments that build a commitment on this placement: shard=(g, G), lde_blocks=G on one device with
        non-resident commitments, or none on one device, whose default is the unsharded resident commitment."""
        if self.num_shards > 1:
            return dict(shard=self.shard)
        return dict(lde_blocks=self.lde_blocks) if self.lde_blocks else {}

    @property
    def step_kwargs(self):
        """The keyword arguments that run compute_quotient_polys, OpeningSet.new / StarkOpeningSet.new or
        fri.prove_openings on this placement: placement=self, or none on one device, their default."""
        return {} if self.num_shards == 1 else dict(placement=self)

    @property
    def check_kwargs(self):
        """The keyword arguments that run stark.check_constraints / plonk.check_constraints on this placement: parts=G
        for non-resident commitments (H checked in G parts one after another, so that the check's scratch shrinks with
        the LDE's), placement=self with several ranks (each rank checks its own part), or none on one device."""
        if self.num_shards > 1:
            return dict(placement=self)
        return dict(parts=self.lde_blocks) if self.lde_blocks else {}

    def cap(self, commitment):
        """The commitment's full Merkle cap: its own on one device, every rank's cap entries all-gathered otherwise."""
        if self.num_shards == 1:
            return commitment.merkle_tree.cap
        return gather_cap(commitment.merkle_tree.cap, self.group, device=_comm_device(self.group, commitment.ctx))

    def open_many(self, batch, leaf_indices):
        """MerkleTree::get + prove (merkle_tree.rs:226-237) for GLOBAL leaf indices of `batch`, a PolynomialBatch or a
        BatchFriOracle (whose leaves are those of its tallest group). Returns (leaves (q, W), paths (q, L, 4)). On one
        device the tree opens them itself. With several ranks every rank opens the indices it owns on its own GPU (local
        index, local cap subtree -- the sibling path is the same as in the single-device tree; a batch oracle's owner of
        leaf i of the tallest group owns leaf i >> (h0 - hk) of every group, so one rank answers the whole query) and
        the ranks all-gather the results: every rank must call it with the same indices."""
        if self.num_shards == 1:
            return batch.merkle_tree.open_many(leaf_indices)
        import torch.distributed as dist

        idx = [int(i) for i in leaf_indices]
        G = self.num_shards
        mine = [(k, owner_of_leaf(i, batch.lde_size, G)[1]) for k, i in enumerate(idx)
                if owner_of_leaf(i, batch.lde_size, G)[0] == self.shard_index]
        lv, pt = batch.merkle_tree.open_many([loc for _, loc in mine])
        part = [(k, lv[j], pt[j]) for j, (k, _) in enumerate(mine)]
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(self.group) == 1:
            parts = [part]
        else:
            parts = [None] * dist.get_world_size(self.group)
            dist.all_gather_object(parts, part, group=self.group)
        layers = batch.lde_size.bit_length() - 1 - batch.cap_height
        leaves = np.empty((len(idx), batch.leaf_width), dtype=np.uint64)
        paths = np.empty((len(idx), layers, 4), dtype=np.uint64)
        seen = 0
        for p in parts:
            for k, l, q in p:
                leaves[k], paths[k] = l, q
                seen += 1
        if seen != len(idx):
            raise RuntimeError("sharded opening: %d of %d indices were served" % (seen, len(idx)))
        return leaves, paths

    def quotient_from_shards(self, ctx, run_shard, n_alphas, degree_bits, quotient_degree_factor):
        """The quotient's coefficients from the ranks' shards of its values. run_shard(local) writes this rank's values on
        its shard of the quotient coset into `local`, an (n_alphas, size / G) int64 CUDA tensor, through its C entry
        point. Then the ranks all-gather the values and every rank interpolates the whole quotient
        (gl_stark_quotient_from_shards). Collective. Returns the same (n_alphas, size) tensor on every rank. A failure on
        one rank raises on every rank: its own exception there, NativeError elsewhere."""
        import torch

        from . import _native as N

        size = (1 << degree_bits) << (quotient_degree_factor - 1).bit_length()
        dev = "cuda:%d" % ctx.device
        local = torch.empty((n_alphas, size // self.num_shards), dtype=torch.int64, device=dev)
        ctx.after_caller()
        failure = None
        try:
            run_shard(local)
        except Exception as e:  # raised below on every rank, so that no rank waits in the all-gather for this one
            failure = e
        self._agree_on_failure(failure, ctx, N.NativeError, "the quotient failed on rank %d")
        values = all_gather_tensor(local, self.group)
        out = torch.empty((n_alphas, size), dtype=torch.int64, device=dev)
        N.check(N.lib().gl_stark_quotient_from_shards(ctx.h, N.vp(values.data_ptr()), self.num_shards, n_alphas,
                                                      degree_bits, quotient_degree_factor, N.vp(out.data_ptr())), ctx.h)
        ctx.synchronize()
        return out

    def openings_from_shards(self, ctx, run_shard, total):
        """The openings (total, 2) from the ranks' partial sums. run_shard(partial) writes this rank's partial sums of
        the `total` polynomials into `partial`, a (total, 2) uint64 host array, through gl_openings_shard. Then the ranks
        all-gather the partials (16 bytes per polynomial) and every rank adds them up mod p in rank order. Collective.
        Returns the same canonical array on every rank. A failure on one rank raises on every rank: its own exception
        there, NativeError elsewhere."""
        import torch

        from . import _native as N

        partial = np.zeros((total, 2), dtype=np.uint64)
        failure = None
        try:
            run_shard(partial)
        except Exception as e:  # raised below on every rank, so that no rank waits in the all-gather for this one
            failure = e
        self._agree_on_failure(failure, ctx, N.NativeError, "the openings failed on rank %d")
        t = torch.from_numpy(partial.view(np.int64))
        dev = _comm_device(self.group, ctx)
        parts = all_gather_tensor(t.to(dev) if dev else t, self.group).cpu().numpy().view(np.uint64)
        out = parts[0].copy()
        for p in parts[1:]:
            out = _add_mod_p(out, p)
        return out

    def report_from_shards(self, ctx, run_part, max_report):
        """The whole constraint check's (failures, [(row, index)]) from the ranks' parts of H. run_part() checks this
        rank's part through gl_*_check_rows_part and returns its (failures, pairs), at most max_report pairs. Then the
        ranks all-gather one fixed-size record each (failures, the number of pairs, max_report packed pairs) and every
        rank merges them in rank order (_native.merge_reports). Collective. Returns the same report on every rank. A
        failure on one rank raises on every rank: its own exception there, NativeError elsewhere."""
        import torch

        from . import _native as N

        result, failure = (0, []), None
        try:
            result = run_part()
        except Exception as e:  # raised below on every rank, so that no rank waits in the all-gather for this one
            failure = e
        self._agree_on_failure(failure, ctx, N.NativeError, "the constraint check failed on rank %d")
        failures, pairs = result
        record = np.zeros(2 + max_report, dtype=np.uint64)
        record[0], record[1] = failures, len(pairs)
        for k, (row, index) in enumerate(pairs):
            record[2 + k] = (int(row) << 32) | int(index)
        t = torch.from_numpy(record.view(np.int64))
        dev = _comm_device(self.group, ctx)
        records = all_gather_tensor(t.to(dev) if dev else t, self.group).cpu().numpy().view(np.uint64)
        return N.merge_reports([(int(r[0]), [(int(w) >> 32, int(w) & 0xFFFFFFFF) for w in r[2:2 + int(r[1])]])
                                for r in records], max_report)

    def _agree_on_failure(self, failure, ctx, error, message):
        """Every rank learns whether any rank failed. `failure` (an exception, or None) is raised on its own rank, and
        error(message % the first failed rank) on every other rank when one failed. Collective with several ranks: call
        it before any collective that a failed rank would skip, so that no rank waits for one that has raised."""
        if self.num_shards > 1:
            import torch

            flag = torch.tensor([int(failure is not None)], dtype=torch.int64,
                                device=_comm_device(self.group, ctx) or "cpu")
            failed = all_gather_tensor(flag, self.group).view(-1)
        if failure is not None:
            raise failure
        if self.num_shards > 1 and int(failed.sum()):
            raise error(message % int(torch.nonzero(failed)[0]))


def _add_mod_p(a, b):
    """a + b mod p elementwise for canonical uint64 arrays: the wrapped sum minus p (mod 2^64) when the sum is p or
    more, which its wrapping past 2^64 also signals."""
    from .field import ORDER

    s = a + b
    over = (s < a) | (s >= np.uint64(ORDER))
    s[over] -= np.uint64(ORDER)
    return s


def prove_openings_sharded(instance, oracles, challenger, fri_params, group=None, final_poly_coeff_len=None,
                           max_num_query_steps=None):
    """fri.prove_openings when the initial oracles are this rank's row-block shards of `group`: the Placement of the
    oracles' shard, whose open_many routes the query openings between the ranks. Collective; the caller must already
    have observed the full caps (gather_cap) in `challenger`. Returns the same FriProof on every rank, byte-identical to
    the single-device proof."""
    from .fri import prove_openings

    placement = Placement(oracles[0].shard_index, oracles[0].num_shards, group)
    return prove_openings(instance, oracles, challenger, fri_params, final_poly_coeff_len, max_num_query_steps,
                          placement=placement)


def check_batch_prove_openings(oracles, fri_params, world):
    """batch_prove_openings_sharded's refusals, raised identically on every rank before any device work or collective: a
    world size that is not a power of two or exceeds 2^cap_height, oracles that are not row-block sharded over `world`
    ranks, and a blinding (hiding) oracle, which batch FRI does not support."""
    from . import _native as N

    _check_world("batch_prove_openings", fri_params.config.cap_height, world)
    if fri_params.hiding or any(o.blinding for o in oracles):
        raise N.ShapeError("batch FRI does not support blinding oracles")
    if any(o.num_shards != world for o in oracles):
        raise N.ShapeError("the oracles must be row-block shards over the %d ranks" % world)


def batch_prove_openings_sharded(degree_bits, instances, oracles, challenger, fri_params, group=None):
    """batch_fri.batch_prove_openings when the BatchFriOracles are this rank's row-block shards of `group`
    (BatchFriOracle.from_values(..., shard=(rank, world))): the Placement of the oracles' shard, whose open_many routes
    the query openings between the ranks. Collective; the caller must already have observed the full caps
    (Placement.cap) in `challenger`. Returns the same FriProof on every rank, byte-identical to the single-device proof.
    Refusals: check_batch_prove_openings (ShapeError on every rank). Without an initialised process group, or with one
    rank, this is batch_prove_openings."""
    from .batch_fri import batch_prove_openings

    check_batch_prove_openings(oracles, fri_params, _world_size(group))
    placement = Placement(oracles[0].shard_index, oracles[0].num_shards, group)
    return batch_prove_openings(degree_bits, instances, oracles, challenger, fri_params, placement=placement)


def all_gather_tensor(t, group=None):
    """The ranks' tensors `t` (same shape on every rank) stacked in rank order: (world, *t.shape) on t's device, ready
    for the library's stream. Under NCCL the exchange stays on the device; other backends go through the host."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    src = (t.contiguous() if dist.get_backend(group) == "nccl" else t.cpu()).reshape(-1)
    out = torch.empty(world * src.numel(), dtype=t.dtype, device=src.device)
    dist.all_gather_into_tensor(out, src, group=group)
    out = out.to(t.device).view((world,) + tuple(t.shape))
    if out.is_cuda:
        torch.cuda.synchronize(out.device)
    return out


def _comm_device(group, ctx):
    """Where `group`'s collectives take their tensors: the context's GPU under NCCL, the host otherwise."""
    import torch.distributed as dist

    return "cuda:%d" % ctx.device if dist.get_backend(group) == "nccl" else None


def _world_size(group):
    """The number of ranks in `group`: 1 without an initialised process group."""
    import torch.distributed as dist

    return dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1


def _placement(group, ctx):
    """This rank's Placement in `group` (Placement() with one rank or without an initialised process group), and its
    context: `ctx`, or the current CUDA device's when None."""
    import torch
    import torch.distributed as dist

    from . import _native as N

    world = _world_size(group)
    placement = Placement(dist.get_rank(group), world, group) if world > 1 else Placement()
    return placement, ctx if ctx is not None else N.default_context(torch.cuda.current_device())


def _check_world(what, cap_height, world):
    """The world-size refusals of prove_stark and prove_plonk: the same on every rank."""
    from . import _native as N

    if world < 1 or world & (world - 1):
        raise N.ShapeError("%s needs a power-of-two number of ranks, got %d" % (what, world))
    if world > 1 << cap_height:
        raise N.ShapeError("%d ranks exceed the %d cap entries of a commitment (cap_height %d)"
                           % (world, 1 << cap_height, cap_height))


def check_prove_stark(stark, config, world):
    """prove_stark's refusals, raised identically on every rank before any device work or collective."""
    from . import _native as N

    _check_world("prove_stark", config.fri_config.cap_height, world)
    if stark.requires_ctls():
        raise N.ShapeError("prove_stark proves one STARK without cross-table lookups; see "
                           "cross_table_lookup.prove_with_ctls")


def prove_stark(stark, config, trace, public_inputs, group=None, verifier_circuit_fri_params=None, ctx=None,
                check_constraints=False):
    """stark.prove on the ranks of a torch.distributed group (the default group if None): rank g commits row block g
    of the trace, auxiliary and quotient LDEs, evaluates the quotient on its shard of the quotient coset, sums block g
    of the coefficients into the openings and answers the FRI queries that land in its rows; the coefficients and the
    transcript are computed on every rank.
    Collective: every rank passes the same full trace (host columns or a torch CUDA tensor) and returns the same
    StarkProofWithPublicInputs, equal to what stark.prove returns on one device. The world size must be a power of two
    of at most 2^cap_height, and the Stark must not take part in cross-table lookups (ShapeError otherwise, on every
    rank). Without an initialised process group, or with one rank, this is stark.prove. ctx: this rank's context
    (default: the current CUDA device's).
    check_constraints=True (equal on every rank, like every other argument): before the quotient, each rank checks
    every constraint on its own part of H, the rows i = rank (mod world), and the ranks merge their reports; a failure
    raises the same ConstraintError on every rank, with stark.prove's message and report."""
    from . import stark as S

    check_prove_stark(stark, config, _world_size(group))
    placement, ctx = _placement(group, ctx)
    return S._prove(stark, config, trace, public_inputs, verifier_circuit_fri_params, ctx, placement, check_constraints)


def check_prove_with_ctls(starks, config, traces, cross_table_lookups, public_inputs, world):
    """prove_with_ctls's refusals, raised identically on every rank before any device work or collective: everything
    cross_table_lookup.prove_with_ctls refuses; a world size that is not a power of two or exceeds 2^cap_height; a
    table whose quotient coset (n << log2_ceil(quotient_degree_factor) points) has fewer points than there are ranks,
    which a small table has when its quotient degree bits are fewer than rate_bits."""
    from . import _native as N
    from . import cross_table_lookup as X

    params, _ = X.check_prove_shapes(starks, config, traces, cross_table_lookups, public_inputs)
    _check_world("prove_with_ctls", config.fri_config.cap_height, world)
    for i, (s, p) in enumerate(zip(starks, params)):
        qdf = s.quotient_degree_factor()
        size = (1 << p.degree_bits) << max(qdf - 1, 0).bit_length()
        if qdf and size < world:
            raise N.ShapeError("table %d's quotient coset has %d points, fewer than the %d ranks" % (i, size, world))


def prove_with_ctls(starks, config, traces, cross_table_lookups, public_inputs, group=None, ctx=None,
                    check_constraints=False):
    """cross_table_lookup.prove_with_ctls on the ranks of a torch.distributed group (the default group if None): rank g
    commits row block g of every table's trace, auxiliary and quotient LDEs, evaluates each quotient on its shard of
    the quotient coset, sums block g of the coefficients into the openings and answers the FRI queries that land in its
    rows. The CTL and lookup helper and Z columns (from the full traces), the coefficients and the one challenger
    chained through the tables run on every rank. Collective: every rank passes the same full traces (host columns or
    torch CUDA tensors) and returns the same MultiStarkProof, field for field prove_with_ctls's on one device.
    Refusals: check_prove_with_ctls (ShapeError on every rank). Without an initialised process group, or with one rank,
    this is prove_with_ctls. ctx: this rank's context (default: the current CUDA device's).
    check_constraints=True (equal on every rank): every table is checked as prove_stark checks its Stark, each rank on
    its own part of H; a failure raises the same ConstraintError on every rank, with prove_with_ctls's message and
    report."""
    from . import cross_table_lookup as X

    check_prove_with_ctls(starks, config, traces, cross_table_lookups, public_inputs, _world_size(group))
    placement, ctx = _placement(group, ctx)
    return X._prove_with_ctls(starks, config, traces, cross_table_lookups, public_inputs, ctx, placement,
                              check_constraints)


def _check_constants_sigmas_shard(prover_data, rank, world):
    from . import _native as N

    cs = prover_data.constants_sigmas_commitment
    if (cs.shard_index, cs.num_shards) != (rank, world):
        raise N.ShapeError("the constants/sigmas commitment is shard %d of %d; rank %d of %d needs shard %d of %d "
                           "(PolynomialBatch.from_values(..., shard=(rank, world)))"
                           % (cs.shard_index, cs.num_shards, rank, world, rank, world))


def check_prove_plonk(prover_data, common_data, world, rank=0):
    """prove_plonk's refusals on rank `rank` of `world`: a world size that is not a power of two or exceeds
    2^cap_height (the same on every rank), and a constants/sigmas commitment that is not this rank's row-block shard
    (which can differ between ranks; prove_plonk exchanges that outcome so that every rank refuses)."""
    _check_world("prove_plonk", common_data.config.cap_height, world)
    _check_constants_sigmas_shard(prover_data, rank, world)


def prove_plonk(prover_data, common_data, wires, public_inputs, group=None, ctx=None, *, salt_keys=None,
                check_constraints=False):
    """plonk.prove_with_witness on the ranks of a torch.distributed group (the default group if None): rank g commits
    row block g of the wires, Z / partial-product (+ lookup) and quotient LDEs, evaluates the quotient on its shard of
    the quotient coset, sums block g of the replicated coefficients into the openings and answers the FRI queries that
    land in its rows. The Z's, partial products and lookup columns (over all n rows) and the transcript are computed on
    every rank.
    Collective: every rank passes the same full witness and returns the same ProofWithPublicInputs, whose bytes equal
    prove_with_witness's on one device. prover_data.constants_sigmas_commitment must be this rank's row-block shard
    (rank, world), built at circuit build with PolynomialBatch.from_values(..., shard=(rank, world)).

    Refusals (ShapeError, on every rank, before the proof's device work): a world size that is not a power of two or
    above 2^cap_height; a constants/sigmas commitment of another shard index or count on any rank. Without an
    initialised process group, or with one rank, this is prove_with_witness. ctx: this rank's context (default: the
    current CUDA device's).

    Zero knowledge: salt_keys (three 32-byte keys, equal on every rank) give the bytes of
    prove_with_witness(..., salt_keys=salt_keys), since a keyed shard holds the unsharded commitment's salted leaves. With
    None ("fresh" keys) each rank draws its own key for its own rows, without a collective: a leaf's salt is only ever
    read by the rank that owns the leaf (Placement.open_many), so the proof is valid and hiding, but no single-device run
    reproduces it.

    check_constraints=True (equal on every rank): before the quotient, each rank checks every term of the vanishing
    polynomial on its own part of H, the rows i = rank (mod world), and the ranks merge their reports; a failure raises
    the same ConstraintError on every rank, with prove_with_witness's message and report."""
    import torch.distributed as dist

    from . import _native as N
    from . import plonk as P

    world = _world_size(group)
    rank = dist.get_rank(group) if world > 1 else 0
    _check_world("prove_plonk", common_data.config.cap_height, world)
    refusal = None
    try:
        _check_constants_sigmas_shard(prover_data, rank, world)
    except N.ShapeError as e:
        if world == 1:
            raise
        refusal = e
    placement, ctx = _placement(group, ctx)
    # the shard check may fail on some ranks only: every rank learns the outcome before a collective could wait
    placement._agree_on_failure(refusal, ctx, N.ShapeError,
                                "rank %d's constants/sigmas commitment is not its row-block shard")
    return P._prove(prover_data, common_data, wires, public_inputs, ctx, placement, salt_keys, check_constraints)


def build_circuit_data(config, fri_config, instances, copy_constraints, num_virtual_targets=0, luts=(), lookup_rows=(),
                       domain_separator=(), group=None, ctx=None):
    """plonk.build_circuit_data on the ranks of a torch.distributed group (the default group if None): every rank
    computes the sigma polynomials (replicated, they are prove_plonk's input) and commits row block `rank` of the
    constants/sigmas LDE; the ranks all-gather the cap entries for the digest. Collective: every rank passes the same
    circuit and returns the CircuitData prove_plonk needs -- prover_only.constants_sigmas_commitment is this rank's
    shard (rank, world) -- with the digest and verifier_only cap of the single-device build. The world size must be a
    power of two of at most 2^cap_height (ShapeError on every rank). Without an initialised process group, or with one
    rank, this is plonk.build_circuit_data. ctx: this rank's context (default: the current CUDA device's)."""
    from . import plonk as P

    _check_world("build_circuit_data", config.cap_height, _world_size(group))
    placement, ctx = _placement(group, ctx)
    return P._build_circuit_data(config, fri_config, instances, copy_constraints, num_virtual_targets, luts, lookup_rows,
                                 domain_separator, ctx, placement)


def chunk_layout(num_polys, world, chunk_cols=64):
    """Column layout of the pipelined multi-GPU commitment: K chunks of Wc = pc*world consecutive columns; inside
    chunk c rank r transforms columns [c*Wc + r*pc, c*Wc + (r+1)*pc) (clipped to num_polys). Returns (pc, Wc, K)."""
    pc = max(1, chunk_cols // world)
    wc = pc * world
    return pc, wc, (num_polys + wc - 1) // wc


def chunk_columns(num_polys, rank, world, chunk, chunk_cols=64):
    """(first global column, count) of rank `rank`'s sub-block of chunk `chunk` (count may be 0 in the last chunk)."""
    pc, wc, _ = chunk_layout(num_polys, world, chunk_cols)
    b0 = min(chunk * wc + rank * pc, num_polys)
    return b0, min(b0 + pc, num_polys) - b0


class PipelinedCommitter:
    """from_values over G ranks with BOTH axes of SURVEY.md section 8e, in 64-column chunks:

      copy stream : H2D of my 64/G columns of each chunk (host input), issued ahead
      main stream : iNTT(0), iNTT(1), LDE(0), iNTT(2), LDE(1), ... , LDE(K-1), leaf hash, cap subtrees
                    iNTT(c)  = column-sharded inverse transform of MY columns of chunk c into my copy of the matrix
                    LDE(c)   = coset LDE of all 64 columns of chunk c on this rank's row block (gl_commit_add_columns)
      side stream : after iNTT(c): my coefficients -> EVERY rank's matrix over NVLink with 128-byte line stores to the
                    NVSwitch multicast address (gl_bcast; one store per peer mapping without multicast), then a
                    device-side barrier (symmetric-memory signal pads). LDE(c) waits for it; the transfer runs under
                    iNTT(c+1) / LDE(c-1) on a handful of SMs.

    The iNTT (the reference's rayon axis, oracle.rs:65-69) and the H2D are divided by G. Transports:
      "multimem" / "p2p"  as above (torch symmetric memory: CUDA IPC / fabric handles);
      "fused"             the iNTT's last pass stores straight to the multicast address (gl_ntt_bcast): no second
                          kernel, but its transposing stores are 64-byte segments, which NVLink runs well below
                          link speed -- kept for comparison;
      "nccl"              ncclAllGather per chunk on the main stream (fallback when peer mappings are unavailable).
    The commitment is bit-identical to the single-device one.

    Stream contract (checked): `ctx` must have been created on the torch stream that is current when commit() is
    called. The returned handle BORROWS the committer's coefficient matrix: it is valid until the next commit()."""

    def __init__(self, ctx, num_polys, log_n, rate_bits, cap_height, rank, world, device, group=None,
                 transport="auto", chunk_cols=None, copy_ctas=32):
        import torch
        import torch.distributed as dist

        from . import _native as N

        self.ctx, self.B, self.log_n, self.r, self.h = ctx, num_polys, log_n, rate_bits, cap_height
        self.rank, self.world, self.group, self.device = rank, world, group, device
        self.n = 1 << log_n
        if chunk_cols is None:  # 64-column chunks, but at least ~4 chunks so that transfers have an LDE to hide under
            per = -(-num_polys // 4)
            chunk_cols = max(world, min(64, -(-per // world) * world))
        self.chunk_cols, self.copy_ctas = chunk_cols, copy_ctas
        self.pc, self.wc, self.K = chunk_layout(num_polys, world, chunk_cols)
        self.copy = torch.cuda.Stream(device=device)
        self.side = torch.cuda.Stream(device=device)
        self.ctx_side = N.Context(device.index if hasattr(device, "index") else int(device), stream=self.side.cuda_stream)
        self.stage = torch.empty((self.K, self.pc, self.n), dtype=torch.int64, device=device)
        self.h2d_events = [torch.cuda.Event() for _ in range(self.K)]
        self.intt_events = [torch.cuda.Event() for _ in range(self.K)]
        self.bcast_events = [torch.cuda.Event() for _ in range(self.K)]
        self.ready = torch.cuda.Event()
        self.timing = False          # set True to collect the transfer spans per commit()
        self._spans = []
        rows = self.K * self.wc
        self.symm, self.transport, self.transport_note = None, "nccl", ""
        if world > 1 and transport != "nccl":
            try:
                import torch.distributed._symmetric_memory as symm_mem

                g = group if group is not None else dist.group.WORLD
                self.coeffs = symm_mem.empty((rows, self.n), dtype=torch.int64, device=device)
                self.symm = symm_mem.rendezvous(self.coeffs, g)
                mc = int(getattr(self.symm, "multicast_ptr", 0) or 0)
                if transport in ("multimem", "fused") and not mc:
                    raise RuntimeError("no multicast mapping on this system")
                self.transport = transport if transport in ("fused", "p2p") else ("multimem" if mc else "p2p")
                ptrs = [int(p) for p in self.symm.buffer_ptrs]
                self.local = ptrs[rank]
                # multicast: one store reaches every rank (mine included); p2p: one store per peer mapping
                self.dests = [mc] if self.transport in ("multimem", "fused") else [p for i, p in enumerate(ptrs) if i != rank]
                if len(self.dests) > 8:
                    raise RuntimeError("more than 8 peers")
            except Exception as e:  # no peer mappings here: same loop over ncclAllGather
                if transport != "auto":
                    raise
                self.symm, self.transport = None, "nccl"
                self.transport_note = "symmetric memory unavailable: %r" % (e,)
        if self.symm is None:
            self.coeffs = torch.empty((rows, self.n), dtype=torch.int64, device=device)

    def _check_stream(self):
        import torch

        cur = torch.cuda.current_stream(self.device)
        if self.ctx.stream != cur.cuda_stream:
            raise RuntimeError("PipelinedCommitter: the context's stream (0x%x) is not the current torch stream (0x%x); "
                               "create the Context on the torch stream you call commit() under" % (self.ctx.stream, cur.cuda_stream))
        return cur

    def my_columns(self):
        """[(first global column, count)] per chunk: the columns this rank uploads and inverse-transforms."""
        return [chunk_columns(self.B, self.rank, self.world, c, self.chunk_cols) for c in range(self.K)]

    def commit(self, values, from_host):
        """values: torch int64 tensor of ALL columns (B x n) -- pinned host memory if from_host (only this rank's
        sub-blocks are read and uploaded), else on the device. Returns the gl_commit handle (row-block shard)."""
        import ctypes as C

        import torch
        import torch.distributed as dist

        from . import _native as N

        L = N.lib()
        main = self._check_stream()
        n, nbytes = self.n, self.n * 8
        base = self.coeffs.data_ptr()
        mine = self.my_columns()
        if from_host:
            with torch.cuda.stream(self.copy):
                self.copy.wait_stream(main)           # the staging slots' previous readers are queued on `main`
                for c, (b0, cnt) in enumerate(mine):
                    if cnt:
                        self.stage[c, :cnt].copy_(values[b0:b0 + cnt], non_blocking=True)  # H2D of 1/G of the chunk
                    self.h2d_events[c].record(self.copy)
        if self.symm is not None:
            self.symm.barrier(channel=0)              # every rank's LDEs of the previous commitment have read the matrix
            self.ready.record(main)
        h = N.vp()
        N.check(L.gl_commit_begin(self.ctx.h, self.B, self.log_n, self.r, self.h, 0, self.rank, self.world, N.vp(base),
                                  C.byref(h)), self.ctx.h)

        def transform(c):
            b0, cnt = mine[c]
            if from_host:
                main.wait_event(self.h2d_events[c])
            src = self.stage[c].data_ptr() if from_host else (values[b0:b0 + cnt].data_ptr() if cnt else 0)
            off = b0 * nbytes
            if self.transport == "fused":
                if cnt:
                    outs = (N.vp * 1)(N.vp(self.dests[0] + off))
                    N.check(L.gl_ntt_bcast(self.ctx.h, N.vp(src), n, self.log_n, cnt, 1, outs, 1, n), self.ctx.h)
                self.symm.barrier(channel=1)
            elif self.symm is not None:
                if cnt:  # out of place into MY copy of the matrix
                    outs = (N.vp * 1)(N.vp(self.local + off))
                    N.check(L.gl_ntt_bcast(self.ctx.h, N.vp(src), n, self.log_n, cnt, 1, outs, 1, n), self.ctx.h)
                self.intt_events[c].record(main)
                with torch.cuda.stream(self.side):
                    if c == 0:
                        self.side.wait_event(self.ready)
                    self.side.wait_event(self.intt_events[c])
                    if self.timing:
                        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        t0.record(self.side)
                    if cnt:
                        outs = (N.vp * len(self.dests))(*[N.vp(d + off) for d in self.dests])
                        N.check(L.gl_bcast(self.ctx_side.h, N.vp(self.local + off), cnt * n, outs, len(self.dests),
                                           self.copy_ctas), self.ctx_side.h)
                    self.symm.barrier(channel=1)
                    if self.timing:
                        t1.record(self.side)
                        self._spans.append((t0, t1))
                    self.bcast_events[c].record(self.side)
            else:
                if cnt:
                    if not from_host:
                        self.stage[c, :cnt].copy_(values[b0:b0 + cnt], non_blocking=True)
                    N.check(L.gl_ntt(self.ctx.h, N.vp(self.stage[c].data_ptr()), self.log_n, cnt, n, 1, 0, 1, N.MEM_DEVICE),
                            self.ctx.h)
                dist.all_gather_into_tensor(self.coeffs[c * self.wc:(c + 1) * self.wc], self.stage[c], group=self.group)

        def extend(c):
            if self.symm is not None and self.transport != "fused":
                main.wait_event(self.bcast_events[c])
            c0 = c * self.wc
            N.check(L.gl_commit_add_columns(h, c0, min(self.wc, self.B - c0), N.vp(base + c0 * nbytes), n,
                                            N.COLS_COEFFS_CANONICAL, N.MEM_DEVICE), self.ctx.h)

        try:
            for c in range(self.K):
                transform(c)
                if c:
                    extend(c - 1)
            extend(self.K - 1)
            N.check(L.gl_commit_finish(h, None, N.MEM_DEVICE), self.ctx.h)
        except Exception:
            L.gl_commit_destroy(h)
            raise
        return h

    def transfer_ms(self, reset=True):
        """(accumulated ms, commits) of the side-stream [NVLink copy + barrier] spans since the last reset; they run
        under the main stream's transforms except for the last chunk's."""
        import torch

        torch.cuda.synchronize(self.device)
        ms = sum(a.elapsed_time(b) for a, b in self._spans)
        cnt = len(self._spans) // max(1, self.K)
        if reset:
            self._spans = []
        return ms, cnt


ColumnShardedCommitter = PipelinedCommitter  # round-1 name
