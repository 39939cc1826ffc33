"""FRI prover mirroring plonky2/src/fri/{mod,structure,proof,prover,reduction_strategies}.rs and the
pre-FRI part of prove_openings (plonky2/src/fri/oracle.rs:176-237).

The transcript (Challenger) is sequential and stays on the host, exactly as in the reference; every
array-sized step (alpha-batching, division by (X - z), coset LDE, Merkle trees, folding, grinding,
openings) is a CUDA call through the C ABI."""
import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import numpy as np

from . import _native as N
from .distributed import Placement
from .field import ORDER
from .hash import NUM_HASH_OUT_ELTS, MerkleCap


# ------------------------------------------------------------------ parameters (fri/mod.rs:30-143)
@dataclass
class FriConfig:
    rate_bits: int
    cap_height: int
    proof_of_work_bits: int
    reduction_strategy: tuple  # ("ConstantArityBits", arity_bits, final_poly_bits) | ("Fixed", [..])
    num_query_rounds: int

    def rate(self):
        return 1.0 / (1 << self.rate_bits)

    def observe(self, challenger):
        """FriConfig::observe (fri/mod.rs:73-79); the strategy as FriReductionStrategy::serialize
        (reduction_strategies.rs:59-80)."""
        challenger.observe_element(self.rate_bits)
        challenger.observe_element(self.cap_height)
        challenger.observe_element(self.proof_of_work_bits)
        kind = self.reduction_strategy[0]
        if kind == "Fixed":
            challenger.observe_elements([0] + list(self.reduction_strategy[1]))
        elif kind == "ConstantArityBits":
            challenger.observe_elements([1, self.reduction_strategy[1], self.reduction_strategy[2]])
        else:
            raise ValueError("unsupported reduction strategy %r" % (kind,))
        challenger.observe_element(self.num_query_rounds)

    def fri_params(self, degree_bits, hiding):
        arity = reduction_arity_bits(self.reduction_strategy, degree_bits, self.rate_bits, self.cap_height,
                                     self.num_query_rounds)
        return FriParams(self, hiding, degree_bits, arity)


def reduction_arity_bits(strategy, degree_bits, rate_bits, cap_height, num_queries):
    """FriReductionStrategy::reduction_arity_bits (reduction_strategies.rs:30-57)."""
    kind = strategy[0]
    if kind == "Fixed":
        return list(strategy[1])
    if kind == "ConstantArityBits":
        arity_bits, final_poly_bits = strategy[1], strategy[2]
        result = []
        while degree_bits > final_poly_bits and degree_bits + rate_bits - arity_bits >= cap_height:
            result.append(arity_bits)
            assert degree_bits >= arity_bits
            degree_bits -= arity_bits
        return result
    raise ValueError("unsupported reduction strategy %r" % (kind,))


@dataclass
class FriParams:
    config: FriConfig
    hiding: bool
    degree_bits: int
    reduction_arity_bits: List[int]

    def observe(self, challenger):
        """FriParams::observe (fri/mod.rs:145-157)."""
        self.config.observe(challenger)
        challenger.observe_element(int(self.hiding))
        challenger.observe_element(self.degree_bits)
        challenger.observe_elements(self.reduction_arity_bits)

    def total_arities(self):
        return sum(self.reduction_arity_bits)

    def lde_bits(self):
        return self.degree_bits + self.config.rate_bits

    def lde_size(self):
        return 1 << self.lde_bits()

    def final_poly_bits(self):
        return self.degree_bits - self.total_arities()

    def final_poly_len(self):
        return 1 << self.final_poly_bits()


def standard_recursion_fri_config():
    """FriConfig of CircuitConfig::standard_recursion_config (plonk/circuit_data.rs:101-119)."""
    return FriConfig(rate_bits=3, cap_height=4, proof_of_work_bits=16,
                     reduction_strategy=("ConstantArityBits", 4, 5), num_query_rounds=28)


def starky_standard_fast_fri_config():
    """StarkConfig::standard_fast_config (starky/src/config.rs:52-64)."""
    return FriConfig(rate_bits=1, cap_height=4, proof_of_work_bits=16,
                     reduction_strategy=("ConstantArityBits", 4, 5), num_query_rounds=84)


# ------------------------------------------------------------------ instance (fri/structure.rs:14-60)
@dataclass
class FriPolynomialInfo:
    oracle_index: int
    polynomial_index: int

    @staticmethod
    def from_range(oracle_index, polynomial_indices):
        return [FriPolynomialInfo(oracle_index, i) for i in polynomial_indices]


@dataclass
class FriBatchInfo:
    point: Tuple[int, int]
    polynomials: List[FriPolynomialInfo]


@dataclass
class FriOracleInfo:
    num_polys: int
    blinding: bool


@dataclass
class FriInstanceInfo:
    oracles: List[FriOracleInfo]
    batches: List[FriBatchInfo]


# ------------------------------------------------------------------ proof (fri/proof.rs:25-113)
@dataclass
class FriQueryStep:
    evals: np.ndarray          # (arity, 2)
    merkle_proof: np.ndarray   # (len, 4)


@dataclass
class FriInitialTreeProof:
    evals_proofs: List[Tuple[np.ndarray, np.ndarray]]  # per oracle: (leaf (W,), siblings (len, 4))


@dataclass
class FriQueryRound:
    initial_trees_proof: FriInitialTreeProof
    steps: List[FriQueryStep]


@dataclass
class FriProof:
    commit_phase_merkle_caps: List[MerkleCap]
    query_round_proofs: List[FriQueryRound]
    final_poly: np.ndarray  # (len, 2)
    pow_witness: int

    def to_bytes(self):
        """write_fri_proof (util/serialization/mod.rs:1595-1609): canonical little-endian u64s."""
        out = bytearray()

        def put(arr):
            out.extend(np.ascontiguousarray(arr, dtype="<u8").tobytes())

        for cap in self.commit_phase_merkle_caps:
            put(cap.hashes)
        for qr in self.query_round_proofs:
            for leaf, sib in qr.initial_trees_proof.evals_proofs:
                put(leaf)
                out.append(len(sib))
                put(sib)
            for st in qr.steps:
                put(st.evals)
                out.append(len(st.merkle_proof))
                put(st.merkle_proof)
        put(self.final_poly)
        put(np.array([self.pow_witness], dtype=np.uint64))
        return bytes(out)

    @classmethod
    def from_bytes(cls, buf, leaf_widths, params, offset=0):
        """read_fri_proof (util/serialization/mod.rs:564-587): leaf_widths = the oracles' leaf widths (polynomials + salt),
        the rest of the shape comes from the FriParams. Returns (FriProof, next offset)."""
        cap_len = 1 << params.config.cap_height
        pos = offset

        def words(count, shape):
            nonlocal pos
            a = np.frombuffer(buf, dtype="<u8", count=count, offset=pos).astype(np.uint64).reshape(shape)
            pos += 8 * count
            return a

        def merkle_proof():
            nonlocal pos
            length = buf[pos]
            pos += 1
            return words(4 * length, (length, NUM_HASH_OUT_ELTS))

        caps = [MerkleCap(words(4 * cap_len, (cap_len, NUM_HASH_OUT_ELTS))) for _ in params.reduction_arity_bits]
        rounds = []
        for _ in range(params.config.num_query_rounds):
            evals_proofs = []
            for w in leaf_widths:
                leaf = words(w, (w,))
                evals_proofs.append((leaf, merkle_proof()))
            steps = []
            for ab in params.reduction_arity_bits:
                evals = words(2 << ab, (1 << ab, 2))
                steps.append(FriQueryStep(evals, merkle_proof()))
            rounds.append(FriQueryRound(FriInitialTreeProof(evals_proofs), steps))
        final_poly = words(2 * params.final_poly_len(), (params.final_poly_len(), 2))
        pow_witness = int(words(1, (1,))[0])
        return cls(caps, rounds, final_poly, pow_witness), pos

    def compress(self, indices, params):
        """FriProof::compress (fri/proof.rs:137-238): per Merkle tree, drop the siblings the verifier can recompute from
        the other queries (compress_merkle_proofs), drop from every step the evaluation it can infer, and keep one entry
        per distinct index."""
        from .batch_merkle_tree import compress_merkle_proofs
        from .hash import MerkleProof

        cap_height = params.config.cap_height
        arity_bits = params.reduction_arity_bits
        nred = len(arity_bits)
        ntrees = len(self.query_round_proofs[0].initial_trees_proof.evals_proofs)
        it_idx = [[] for _ in range(ntrees)]
        it_leaves = [[] for _ in range(ntrees)]
        it_proofs = [[] for _ in range(ntrees)]
        st_idx = [[] for _ in range(nred)]
        st_evals = [[] for _ in range(nred)]
        st_proofs = [[] for _ in range(nred)]
        for index, qrp in zip(indices, self.query_round_proofs):
            for i, (leaf, sib) in enumerate(qrp.initial_trees_proof.evals_proofs):
                it_idx[i].append(index)
                it_leaves[i].append(leaf)
                it_proofs[i].append(MerkleProof(sib))
            for i, st in enumerate(qrp.steps):
                within = index & ((1 << arity_bits[i]) - 1)
                index >>= arity_bits[i]
                st_idx[i].append(index)
                st_evals[i].append(np.delete(np.asarray(st.evals), within, axis=0))  # remove the inferable element
                st_proofs[i].append(MerkleProof(st.merkle_proof))
        it_proofs = [compress_merkle_proofs(cap_height, i, p) for i, p in zip(it_idx, it_proofs)]
        st_proofs = [compress_merkle_proofs(cap_height, i, p) for i, p in zip(st_idx, st_proofs)]
        initial, steps = {}, [dict() for _ in range(nred)]
        for i, index in enumerate(indices):
            initial.setdefault(index, FriInitialTreeProof([(it_leaves[j][i], it_proofs[j][i].siblings) for j in range(ntrees)]))
            for j in range(nred):
                index >>= arity_bits[j]
                steps[j].setdefault(index, FriQueryStep(st_evals[j][i], st_proofs[j][i].siblings))
        return CompressedFriProof(self.commit_phase_merkle_caps, list(indices), initial, steps, self.final_poly,
                                  self.pow_witness)


@dataclass
class CompressedFriProof:
    """CompressedFriProof / CompressedFriQueryRounds (fri/proof.rs:92-112,124-135)."""
    commit_phase_merkle_caps: List[MerkleCap]
    indices: List[int]
    initial_trees_proofs: dict      # index -> FriInitialTreeProof
    steps: List[dict]               # per reduction: index -> FriQueryStep
    final_poly: np.ndarray
    pow_witness: int

    def to_bytes(self):
        """write_compressed_fri_proof (util/serialization/mod.rs:2034-2076): caps, u32 indices, the initial proofs and
        every reduction's steps in increasing index order, final poly, pow witness."""
        out = bytearray()

        def put(arr):
            out.extend(np.ascontiguousarray(arr, dtype="<u8").tobytes())

        for cap in self.commit_phase_merkle_caps:
            put(cap.hashes)
        out.extend(np.array(self.indices, dtype="<u4").tobytes())
        for _, itp in sorted(self.initial_trees_proofs.items()):
            for leaf, sib in itp.evals_proofs:
                put(leaf)
                out.append(len(sib))
                put(sib)
        for h in self.steps:
            for _, st in sorted(h.items()):
                put(st.evals)
                out.append(len(st.merkle_proof))
                put(st.merkle_proof)
        put(self.final_poly)
        put(np.array([self.pow_witness], dtype=np.uint64))
        return bytes(out)

    def decompress_with(self, inferred_evals, params, lde_bits, ctx=None):
        """CompressedFriProof::decompress (fri/proof.rs:240-360) given the elements the verifier infers
        (`inferred_evals[q][j]` = the evaluation removed from query q's step j; plonk/proof.rs get_inferred_elements
        computes them from the openings): re-insert them, decompress every tree's Merkle proofs and re-expand
        duplicate indices."""
        from .batch_merkle_tree import decompress_merkle_proofs
        from .hash import MerkleProof

        cap_height = params.config.cap_height
        arity_bits = params.reduction_arity_bits
        nred = len(arity_bits)
        ntrees = len(next(iter(self.initial_trees_proofs.values())).evals_proofs)
        # distinct indices in first-seen order, like the reference's `seen` bookkeeping
        it_idx = [[] for _ in range(ntrees)]
        it_leaves = [[] for _ in range(ntrees)]
        it_proofs = [[] for _ in range(ntrees)]
        st_idx = [[] for _ in range(nred)]
        st_evals = [[] for _ in range(nred)]
        st_proofs = [[] for _ in range(nred)]
        seen_init, seen_step = set(), [set() for _ in range(nred)]
        for q, index in enumerate(self.indices):
            if index not in seen_init:
                seen_init.add(index)
                for i, (leaf, sib) in enumerate(self.initial_trees_proofs[index].evals_proofs):
                    it_idx[i].append(index)
                    it_leaves[i].append(leaf)
                    it_proofs[i].append(MerkleProof(sib))
            for j in range(nred):
                within = index & ((1 << arity_bits[j]) - 1)
                index >>= arity_bits[j]
                if index not in seen_step[j]:
                    seen_step[j].add(index)
                    st = self.steps[j][index]
                    ev = np.insert(np.asarray(st.evals), within, np.asarray(inferred_evals[q][j], dtype=np.uint64), axis=0)
                    st_idx[j].append(index)
                    st_evals[j].append(ev)
                    st_proofs[j].append(MerkleProof(st.merkle_proof))
        heights = [lde_bits]
        for a in arity_bits:
            heights.append(heights[-1] - a)
        it_full = [decompress_merkle_proofs(lv, ix, pr, lde_bits, cap_height, ctx) for lv, ix, pr in zip(it_leaves, it_idx, it_proofs)]
        st_full = [decompress_merkle_proofs([e.reshape(-1) for e in ev], ix, pr, heights[j + 1], cap_height, ctx)
                   for j, (ev, ix, pr) in enumerate(zip(st_evals, st_idx, st_proofs))]
        rounds = []
        for index in self.indices:
            init = FriInitialTreeProof([(it_leaves[i][it_idx[i].index(index)], it_full[i][it_idx[i].index(index)].siblings)
                                        for i in range(ntrees)])
            steps = []
            for j in range(nred):
                index >>= arity_bits[j]
                k = st_idx[j].index(index)
                steps.append(FriQueryStep(st_evals[j][k], st_full[j][k].siblings))
            rounds.append(FriQueryRound(init, steps))
        return FriProof(self.commit_phase_merkle_caps, rounds, self.final_poly, self.pow_witness)


def fri_challenges(challenger, commit_phase_merkle_caps, final_poly, pow_witness, degree_bits, config,
                   final_poly_coeff_len=None, max_num_query_steps=None):
    """Challenger::fri_challenges (fri/challenges.rs:28-89): what the verifier (and ProofWithPublicInputs::compress)
    re-derives from a proof. final_poly_coeff_len / max_num_query_steps: the zero caps and zero coefficients a proof
    made for a verifier circuit of other FRI parameters observes (as fri_committed_trees does).
    Returns (fri_alpha, fri_betas, fri_pow_response, fri_query_indices)."""
    lde_size = 1 << (degree_bits + config.rate_bits)
    fri_alpha = challenger.get_extension_challenge()
    fri_betas = []
    for cap in commit_phase_merkle_caps:
        challenger.observe_cap(cap)
        fri_betas.append(challenger.get_extension_challenge())
    if max_num_query_steps is not None:
        zero_cap = [0] * (NUM_HASH_OUT_ELTS << config.cap_height)
        for _ in range(len(commit_phase_merkle_caps), max_num_query_steps):
            challenger.observe_elements(zero_cap)
            challenger.get_extension_challenge()
    final_poly = np.asarray(final_poly, dtype=np.uint64).reshape(-1, 2)
    challenger.observe_elements(final_poly.reshape(-1))
    if final_poly_coeff_len is not None:
        for _ in range(len(final_poly), final_poly_coeff_len):
            challenger.observe_extension_element((0, 0))
    challenger.observe_element(pow_witness)
    fri_pow_response = challenger.get_challenge()
    fri_query_indices = [challenger.get_challenge() % lde_size for _ in range(config.num_query_rounds)]
    return fri_alpha, fri_betas, fri_pow_response, fri_query_indices


# ------------------------------------------------------------------ prover
class _FriState(N.Handle):
    """Owner of a gl_fri handle. value_sharded = (shard, num_shards) when the codeword is row-block sharded
    (_begin_values)."""
    destroyer = "gl_fri_destroy"

    def __init__(self, h, ctx, value_sharded=None):
        self.h, self.ctx, self.value_sharded = h, ctx, value_sharded


def _fri_batches(instance, oracles):
    """The gl_fri_begin* inputs of an instance: the oracles' handle array, the FriBatch array and the index arrays the
    batches point into (keep them alive until the call returns)."""
    handles = (N.vp * len(oracles))(*[o.h for o in oracles])
    barr = (N.FriBatch * len(instance.batches))()
    keep = []
    for i, b in enumerate(instance.batches):
        oi = np.array([p.oracle_index for p in b.polynomials], dtype=np.uint32)
        pi = np.array([p.polynomial_index for p in b.polynomials], dtype=np.uint32)
        keep += [oi, pi]
        barr[i].point[0], barr[i].point[1] = int(b.point[0]) % ORDER, int(b.point[1]) % ORDER
        barr[i].num_polys = len(b.polynomials)
        barr[i].oracle_index = oi.ctypes.data_as(N.u32p)
        barr[i].poly_index = pi.ctypes.data_as(N.u32p)
    return handles, barr, keep


def _begin(instance, oracles, alpha, fri_params):
    ctx = oracles[0].ctx
    handles, barr, keep = _fri_batches(instance, oracles)
    al = np.array([alpha[0], alpha[1]], dtype=np.uint64)
    h = N.vp()
    N.check(N.lib().gl_fri_begin(ctx.h, handles, len(oracles), barr, len(instance.batches), N.np_ptr(al),
                                 fri_params.config.rate_bits, fri_params.config.cap_height, C.byref(h)), ctx.h)
    return _FriState(h, ctx)


def _begin_values(instance, oracles, alpha, opened, fri_params):
    """The pre-FRI part of prove_openings (oracle.rs:186-220) in the value domain (gl_fri_begin_values): `opened` =
    [(num_polys_b, 2) array per batch], the openings f_{b,j}(z_b) the prover already holds (OpeningSet). With row-block
    sharded oracles the state holds this rank's rows only."""
    ctx = oracles[0].ctx
    handles, barr, keep = _fri_batches(instance, oracles)
    op = np.ascontiguousarray(np.concatenate([np.asarray(o, dtype=np.uint64).reshape(-1, 2) for o in opened]), dtype=np.uint64)
    assert len(op) == sum(len(b.polynomials) for b in instance.batches)
    al = np.array([alpha[0], alpha[1]], dtype=np.uint64)
    h = N.vp()
    N.check(N.lib().gl_fri_begin_values(ctx.h, handles, len(oracles), barr, len(instance.batches), N.np_ptr(op.reshape(-1)),
                                        N.np_ptr(al), fri_params.config.cap_height, C.byref(h)), ctx.h)
    return _FriState(h, ctx, (oracles[0].shard_index, oracles[0].num_shards))


def _final_poly_from_values(values, log_len, shift, rate_bits, ctx):
    """Coefficients of the last codeword (prover.rs:134-139) from its values in bit-reversed order: un-reverse,
    coset_ifft on the final coset (both F_{p^2} components), drop the top 1 - 2^-rate_bits (zero) coefficients."""
    from .fft import coset_ifft
    from .field import reverse_bits

    n = 1 << log_len
    nat = np.empty((n, 2), dtype=np.uint64)
    for j in range(n):
        nat[reverse_bits(j, log_len)] = values[j]
    cols = np.ascontiguousarray(nat.T)
    co = coset_ifft(cols, shift, ctx=ctx) if log_len else cols
    return np.ascontiguousarray(co.T[:n >> rate_bits])


def fri_committed_trees(state, challenger, fri_params, final_poly_coeff_len=None, max_num_query_steps=None,
                        shard=None, gather=None, mixes=()):
    """fri_committed_trees (prover.rs:84-150): returns (caps, final_poly coefficients (len, 2)).
    shard=(g, G), gather=fn(local cap words) -> full cap words: every round's tree is row-block sharded over the G
    ranks (this rank hashes only its block of leaves; the values and the fold stay replicated) and the ranks
    all-gather their cap entries -- rounds too small to shard are built whole on every rank.
    mixes=[(log LDE size, state)], sizes decreasing: the lower-degree instances of batch FRI (batch_fri/prover.rs:88-147),
    each mixed into the codeword (gl_fri_mix) after the fold that reaches its size."""
    L, ctx = N.lib(), state.ctx
    cap_words = NUM_HASH_OUT_ELTS << fri_params.config.cap_height
    caps = []
    vs = state.value_sharded
    mixes = list(mixes)
    log_cur = fri_params.lde_bits()
    for arity_bits in fri_params.reduction_arity_bits:
        cap = np.empty(cap_words, dtype=np.uint64)
        if vs is not None and vs[1] > 1:  # the codeword itself is row-block sharded: everything is rank-local
            local = np.empty(cap_words // vs[1], dtype=np.uint64)
            N.check(L.gl_fri_commit_round(state.h, arity_bits, N.np_ptr(local)), ctx.h)
            cap = np.ascontiguousarray(gather(local), dtype=np.uint64).reshape(-1)
            assert cap.size == cap_words
        elif shard is not None and shard[1] > 1 and (shard[1] - 1).bit_length() <= fri_params.config.cap_height:
            local = np.empty(cap_words // shard[1], dtype=np.uint64)
            N.check(L.gl_fri_commit_round_sharded(state.h, arity_bits, shard[0], shard[1], N.np_ptr(local)), ctx.h)
            cap = np.ascontiguousarray(gather(local), dtype=np.uint64).reshape(-1)
            assert cap.size == cap_words
        else:
            N.check(L.gl_fri_commit_round(state.h, arity_bits, N.np_ptr(cap)), ctx.h)
        cap = MerkleCap(cap)
        challenger.observe_cap(cap)
        caps.append(cap)
        beta = challenger.get_extension_challenge()
        b = np.array(beta, dtype=np.uint64)
        N.check(L.gl_fri_fold(state.h, N.np_ptr(b)), ctx.h)
        log_cur -= arity_bits
        if mixes and mixes[0][0] == log_cur:
            N.check(L.gl_fri_mix(state.h, mixes.pop(0)[1].h, N.np_ptr(b)), ctx.h)
    assert not mixes, "reduction_arity_bits must pass through every instance's LDE size (prover.rs:44-57)"
    if max_num_query_steps is not None:
        zero_cap = [0] * cap_words
        for _ in range(len(fri_params.reduction_arity_bits), max_num_query_steps):
            challenger.observe_elements(zero_cap)
            challenger.get_extension_challenge()
    n_final = fri_params.final_poly_len()
    if vs is not None and vs[1] > 1:
        log_last = fri_params.lde_bits() - fri_params.total_arities()
        loc = np.empty(2 * ((1 << log_last) // vs[1]), dtype=np.uint64)
        ln = C.c_size_t()
        N.check(L.gl_fri_values_local(state.h, N.np_ptr(loc), loc.size, C.byref(ln)), ctx.h)
        vals = np.ascontiguousarray(gather(loc), dtype=np.uint64).reshape(-1, 2)
        from .field import coset_shift
        shift = pow(coset_shift(), 1 << fri_params.total_arities(), ORDER)
        coeffs = _final_poly_from_values(vals, log_last, shift, fri_params.config.rate_bits, ctx)
    else:
        buf = np.empty(2 * max(n_final, 1), dtype=np.uint64)
        ln = C.c_size_t()
        N.check(L.gl_fri_final_poly(state.h, N.np_ptr(buf), buf.size, C.byref(ln)), ctx.h)
        coeffs = buf[:2 * ln.value].reshape(-1, 2).copy()
    challenger.observe_extension_elements([(int(c[0]), int(c[1])) for c in coeffs])
    if final_poly_coeff_len is not None:
        for _ in range(len(coeffs), final_poly_coeff_len):
            challenger.observe_extension_element((0, 0))
    return caps, coeffs


def fri_proof_of_work(challenger, config, ctx=None):
    """fri_proof_of_work (prover.rs:153-202); the grind runs on the GPU and returns the smallest nonce."""
    ctx = ctx or N.default_context()
    min_leading_zeros = config.proof_of_work_bits + (64 - ORDER.bit_length())
    inter = challenger.sponge_state.copy()
    pos = len(challenger.input_buffer)
    inter.set_from_iter(challenger.input_buffer, 0)
    nonce = np.zeros(1, dtype=np.uint64)
    st = np.ascontiguousarray(inter.state, dtype=np.uint64)
    N.check(N.lib().gl_fri_pow(ctx.h, N.np_ptr(st), pos, min_leading_zeros, N.np_ptr(nonce)), ctx.h)
    pow_witness = int(nonce[0])
    challenger.observe_element(pow_witness)
    pow_response = challenger.get_challenge()
    leading_zeros = 64 - pow_response.bit_length()
    assert leading_zeros >= min_leading_zeros
    return pow_witness


def fri_prover_query_rounds(oracles, state, challenger, n, fri_params, placement=Placement()):
    """fri_prover_query_rounds / fri_prover_query_round (prover.rs:204-258), batched per tree. The initial trees are
    opened on their placement (Placement.open_many)."""
    L, ctx = N.lib(), state.ctx
    nq = fri_params.config.num_query_rounds
    x_indices = [c % n for c in challenger.get_n_challenges(nq)]
    idx = np.array(x_indices, dtype=np.uint64)
    initial = [placement.open_many(o, idx) for o in oracles]
    steps = []
    cur = idx.copy()
    log_cur = fri_params.lde_bits()
    for r, arity_bits in enumerate(fri_params.reduction_arity_bits):
        cur = cur >> np.uint64(arity_bits)
        w = 2 << arity_bits
        layers = log_cur - arity_bits - fri_params.config.cap_height
        leaves = np.empty((nq, w), dtype=np.uint64)
        paths = np.empty((nq, layers, 4), dtype=np.uint64)
        if nq:
            N.check(L.gl_fri_open(state.h, r, N.np_ptr(np.ascontiguousarray(cur)), nq, N.np_ptr(leaves),
                                  N.np_ptr(paths) if paths.size else None), ctx.h)
        steps.append((leaves, paths))
        log_cur -= arity_bits
    rounds = []
    for q in range(nq):
        init = FriInitialTreeProof([(lv[q], pt[q]) for (lv, pt) in initial])
        st = [FriQueryStep(lv[q].reshape(-1, 2), pt[q]) for (lv, pt) in steps]
        rounds.append(FriQueryRound(init, st))
    return rounds, x_indices


def prove_openings(instance, oracles, challenger, fri_params, final_poly_coeff_len=None,
                   max_num_query_steps=None, taps=None, placement=Placement()):
    """PolynomialBatch::prove_openings -> fri_proof (oracle.rs:176-237, prover.rs:24-70). placement: where the initial
    oracles live. With row-block shards over several ranks, the coefficients are replicated, so every rank runs the
    (small, single-column) FRI commit phase and the transcript redundantly and deterministically; only the initial-tree
    openings cross ranks, and the returned FriProof is the same on every rank and byte-identical to the single-device
    proof. The caller must already have observed the full caps (Placement.cap) in `challenger`."""
    alpha = challenger.get_extension_challenge()
    state = _begin(instance, oracles, alpha, fri_params)
    try:
        if taps is not None:
            n = 1 << oracles[0].degree_log
            fp = np.empty((n, 2), dtype=np.uint64)
            N.check(N.lib().gl_fri_coeffs(state.h, N.np_ptr(fp)), state.ctx.h)
            taps["final_poly"] = fp
        caps, final_coeffs = fri_committed_trees(state, challenger, fri_params, final_poly_coeff_len,
                                                 max_num_query_steps)
        pow_witness = fri_proof_of_work(challenger, fri_params.config, state.ctx)
        n = fri_params.lde_size()
        rounds, x_indices = fri_prover_query_rounds(oracles, state, challenger, n, fri_params, placement)
        if taps is not None:
            taps["pow_witness"] = pow_witness
            taps["query_indices"] = x_indices
        return FriProof(caps, rounds, final_coeffs, pow_witness)
    finally:
        state.close()
