/*
 * gl_oracle.h -- CPU parity ORACLE for the plonky2 prover hot path (TEST INFRASTRUCTURE ONLY).
 *
 * This is a plain, literal C++ restatement of the reference's CPU algorithm
 * (0xPolygonZero/plonky2 @ 5d9da5a) for: Goldilocks field arithmetic, radix-2 NTT/iNTT,
 * coset-LDE, Poseidon-12 sponge, Merkle tree (reference digest layout), Fiat-Shamir
 * challenger and the FRI prover (commit phase, proof-of-work, query openings).
 * Every function cites the reference file:line it follows.
 *
 * USE: only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load this library, and only as the checker / CPU baseline. The product
 * (plonky2_b200/, libplonky2_b200.so) never links, imports or calls it.
 *
 * PINNING STATUS: the reference is Rust (nightly) and cannot be built in this image
 * (no cargo/rustc), so there is no oracle/_ref. The oracle is pinned against every stored
 * vector the reference's own tests hold for this path:
 *   - Poseidon-12 permutation: the 4 known-answer vectors of
 *     plonky2/src/hash/poseidon_goldilocks.rs:466-487 (tests/golden/poseidon_kat.json),
 *     and fast-partial-rounds == naive form (poseidon.rs:944-957);
 *   - bit-reversal: the 256-entry golden table of plonky2/src/util/mod.rs:64-84.
 * For NTT / LDE / Merkle caps / FRI proofs the reference stores NO golden data
 * (SURVEY.md section 4): for those outputs parity is UNPINNED by stored data and rests on
 * the reference tests' own definitions, restated in tests/ (NTT == naive O(n^2) evaluation,
 * field/src/fft.rs:215-282; coset FFT == naive coset evaluation, polynomial/mod.rs:476-516;
 * every Merkle proof verifies against the cap, merkle_tree.rs:269-311; FRI proofs pass the
 * restated verifier, fri/verifier.rs:62-241).
 *
 * All u64 outputs are CANONICAL (< p). Inputs may be any u64 (non-canonical allowed), exactly
 * like the reference's GoldilocksField(pub u64) (field/src/goldilocks_field.rs:23-25).
 */
#ifndef GL_ORACLE_H
#define GL_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- field (field/src/goldilocks_field.rs:198-320,392-449; types.rs:226-272,429-443) ---- */
uint64_t glo_canon(uint64_t a);
uint64_t glo_add(uint64_t a, uint64_t b);
uint64_t glo_sub(uint64_t a, uint64_t b);
uint64_t glo_mul(uint64_t a, uint64_t b);
uint64_t glo_neg(uint64_t a);
uint64_t glo_inv(uint64_t a);                      /* 0 -> 0 (reference returns None) */
uint64_t glo_exp(uint64_t a, uint64_t e);
uint64_t glo_primitive_root_of_unity(uint32_t log_n);
uint64_t glo_inverse_2exp(uint32_t k);
uint64_t glo_coset_shift(void);                    /* MULTIPLICATIVE_GROUP_GENERATOR */
/* quadratic extension F[X]/(X^2-7): (field/src/extension/quadratic.rs:86-100,180-193) */
void glo_ext2_mul(const uint64_t a[2], const uint64_t b[2], uint64_t out[2]);
void glo_ext2_inv(const uint64_t a[2], uint64_t out[2]);

/* ---- bit reversal (util/src/lib.rs:53-101,185-234; plonky2/src/util/mod.rs:33-41) ---- */
uint64_t glo_reverse_bits(uint64_t x, uint32_t bits);
void glo_reverse_index_bits_in_place(uint64_t* arr, size_t n, size_t elem_words);

/* ---- NTT (field/src/fft.rs:14-33,53-91,165-202; polynomial/mod.rs:58-88,199-201,280-293) ---- */
/* in place, natural order in and out. zero_factor = r: top (1 - 2^-r) of the input is zero. */
void glo_fft(uint64_t* buf, uint32_t log_n, uint32_t zero_factor);
void glo_ifft(uint64_t* buf, uint32_t log_n);
void glo_coset_fft(uint64_t* buf, uint32_t log_n, uint64_t shift, uint32_t zero_factor);
void glo_coset_ifft(uint64_t* buf, uint32_t log_n, uint64_t shift);
/* naive O(n^2) evaluation on shift*<omega_n>, the reference tests' definition (fft.rs:251-282) */
void glo_naive_coset_eval(const uint64_t* coeffs, uint32_t log_n, uint64_t shift, uint64_t* out);

/* ---- Poseidon-12 (plonky2/src/hash/poseidon.rs:630-641,689-801; hashing.rs:97-145;
 *      plonk/config.rs:63-74) ---- */
void glo_poseidon(uint64_t st[12]);        /* fast-partial-rounds form, poseidon.rs:766-777 */
void glo_poseidon_naive(uint64_t st[12]);  /* textbook form, poseidon.rs:779-801 */
/* glo_poseidon on n states of 12 words each, in place, split over nthreads */
void glo_poseidon_many(uint64_t* states, size_t n, int nthreads);
/* the smallest nonce < limit such that lane 7 of the permuted state (state with lane pos = nonce) has at least
 * min_leading_zeros leading zeros (fri_proof_of_work, prover.rs:183-194); ~0 if there is none */
uint64_t glo_pow_min_nonce(const uint64_t state[12], uint32_t pos, uint32_t min_leading_zeros, uint64_t limit,
                           int nthreads);
void glo_hash_no_pad(const uint64_t* in, size_t len, uint64_t out[4]);
void glo_hash_or_noop(const uint64_t* in, size_t len, uint64_t out[4]);
void glo_two_to_one(const uint64_t l[4], const uint64_t r[4], uint64_t out[4]);
/* batched convenience for the CPU baseline: n_items inputs of W words, row-major */
void glo_hash_many(const uint64_t* in, size_t n_items, size_t W, uint64_t* out, int nthreads);

/* ---- Merkle tree (plonky2/src/hash/merkle_tree.rs:86-224, merkle_proofs.rs:55-107) ---- */
/* leaves: row-major N x W. digests: 4*2*(N - C) words in the reference layout. cap: 4*C. */
int glo_merkle_build(const uint64_t* leaves, size_t N, size_t W, uint32_t cap_height,
                     uint64_t* digests, uint64_t* cap, int nthreads);
/* siblings: 4*(log N - cap_height) words, bottom-up */
void glo_merkle_prove(size_t leaf_index, size_t N, uint32_t cap_height, const uint64_t* digests,
                      uint64_t* siblings);
int glo_merkle_verify(const uint64_t* leaf, size_t W, size_t leaf_index, const uint64_t* siblings,
                      size_t n_siblings, const uint64_t* cap, uint32_t cap_height);

/* ---- PolynomialBatch (plonky2/src/fri/oracle.rs:57-147) ---- */
typedef struct glo_commit glo_commit;
/* cols: B columns of n words, column b at cols + b*col_stride. salt: NULL or 4 columns of N
 * words (blinding; the reference draws them from OsRng, oracle.rs:133-137). */
glo_commit* glo_commit_new(const uint64_t* cols, size_t col_stride, size_t B, uint32_t log_n,
                           uint32_t rate_bits, uint32_t cap_height, const uint64_t* salt,
                           int is_coeffs, int nthreads);
void glo_commit_free(glo_commit*);
size_t glo_commit_leaf_width(const glo_commit*);
const uint64_t* glo_commit_coeffs(const glo_commit*);   /* B x n, column-major */
const uint64_t* glo_commit_leaves(const glo_commit*);   /* N x W, row-major, leaf j = LDE row bitrev(j) */
const uint64_t* glo_commit_digests(const glo_commit*);  /* 8*(N-C) words */
const uint64_t* glo_commit_cap(const glo_commit*);      /* 4*C words */
/* get_lde_values(index, step) (oracle.rs:142-147): writes B words */
void glo_commit_get_lde_values(const glo_commit*, size_t index, size_t step, uint64_t* out);

/* ---- Challenger (plonky2/src/iop/challenger.rs:30-153) ---- */
typedef struct glo_challenger glo_challenger;
glo_challenger* glo_challenger_new(void);
glo_challenger* glo_challenger_clone(const glo_challenger*);
void glo_challenger_free(glo_challenger*);
void glo_challenger_observe(glo_challenger*, const uint64_t* elems, size_t n);
uint64_t glo_challenger_get_challenge(glo_challenger*);
/* debugging / PoW: copies sponge state (12) and returns input_buffer length */
size_t glo_challenger_state(const glo_challenger*, uint64_t state[12], uint64_t inbuf[8]);

/* ---- FRI prover (plonky2/src/fri/oracle.rs:176-237, prover.rs:24-258) ---- */
typedef struct {
    uint32_t rate_bits;
    uint32_t cap_height;
    uint32_t proof_of_work_bits;
    uint32_t num_query_rounds;
    uint32_t num_reductions;
    uint32_t reduction_arity_bits[32];
} glo_fri_params;

/* One opening batch: a point in F_{p^2} and a list of (oracle_index, polynomial_index). */
typedef struct {
    uint64_t point[2];
    size_t num_polys;
    const uint32_t* oracle_index;
    const uint32_t* poly_index;
} glo_fri_batch;

/* prove_openings: returns the proof serialised exactly like the reference's write_fri_proof
 * (plonky2/src/util/serialization/mod.rs:1595-1609): caps, query rounds (initial leaf + u8 len +
 * siblings per oracle; evals + u8 len + siblings per step), final poly, pow witness; canonical
 * little-endian u64s. *out is malloc'ed (free with glo_free). PoW = SMALLEST qualifying nonce
 * (sequential `find`, maybe_rayon/src/lib.rs:254-259). Returns 0 on success. */
int glo_prove_openings(const glo_commit* const* oracles, size_t n_oracles,
                       const glo_fri_batch* batches, size_t n_batches, glo_challenger* challenger,
                       const glo_fri_params* params, uint8_t** out, size_t* out_len,
                       /* optional taps for stage-by-stage parity (may be NULL): */
                       uint64_t* tap_final_poly /* 2*n words */, uint64_t* tap_betas /* 2*num_reductions */,
                       uint64_t* tap_pow_witness, uint64_t* tap_query_indices);
void glo_free(void*);

/* ---- batch FRI (SURVEY 8f-4): BatchFriOracle::from_values / from_coeffs (plonky2/src/batch_fri/oracle.rs:45-131) over
 *      polynomials of non-increasing lengths 2^log_lens[i] with its BatchMerkleTree (hash/batch_merkle_tree.rs:34-128),
 *      and BatchFriOracle::prove_openings + batch_fri_proof (batch_fri/oracle.rs:124-183, batch_fri/prover.rs:30-215)
 *      serialised like write_fri_proof. Polynomial indices index each oracle's full polynomial list. */
typedef struct glo_batch_commit glo_batch_commit;
glo_batch_commit* glo_batch_commit_new(const uint64_t* const* polys, const uint32_t* log_lens, size_t num_polys,
                                       uint32_t rate_bits, uint32_t cap_height, int is_coeffs);
void glo_batch_commit_free(glo_batch_commit*);
size_t glo_batch_commit_cap(const glo_batch_commit*, uint64_t* out); /* returns the number of cap hashes */
typedef struct {
    const glo_fri_batch* batches;
    size_t n_batches;
} glo_fri_instance;
int glo_batch_prove_openings(const glo_batch_commit* const* oracles, size_t n_oracles, const uint32_t* degree_bits,
                             const glo_fri_instance* instances, size_t n_instances, glo_challenger* challenger,
                             const glo_fri_params* params, uint8_t** out, size_t* out_len);

/* compute_quotient_polys (plonky2/src/plonk/prover.rs:609-815) + eval_vanishing_poly_base_batch
 * (plonk/vanishing_poly.rs:167-340, circuits without lookups) for the gates below. out: num_challenges polynomials of
 * n << log2_ceil(quotient_degree_factor) coefficients. */
#define GLO_GATE_NOOP 0         /* gates/noop.rs */
#define GLO_GATE_CONSTANT 1     /* gates/constant.rs, param = num_consts */
#define GLO_GATE_PUBLIC_INPUT 2 /* gates/public_input.rs */
#define GLO_GATE_ARITHMETIC 3   /* gates/arithmetic_base.rs, param = num_ops */
#define GLO_GATE_POSEIDON 4     /* gates/poseidon.rs */
#define GLO_GATE_ARITHMETIC_EXTENSION 5 /* gates/arithmetic_extension.rs, param = num_ops */
#define GLO_GATE_MUL_EXTENSION 6        /* gates/multiplication_extension.rs, param = num_ops */
#define GLO_GATE_BASE_SUM 7             /* gates/base_sum.rs, param = num_limbs, param2 = B */
#define GLO_GATE_REDUCING 8             /* gates/reducing.rs, param = num_coeffs */
#define GLO_GATE_REDUCING_EXTENSION 9   /* gates/reducing_extension.rs, param = num_coeffs */
#define GLO_GATE_POSEIDON_MDS 10        /* gates/poseidon_mds.rs */
#define GLO_GATE_RANDOM_ACCESS 11       /* gates/random_access.rs, param = bits, param2 = num_copies, param3 = num_extra_constants */
#define GLO_GATE_EXPONENTIATION 12      /* gates/exponentiation.rs, param = num_power_bits */
#define GLO_GATE_COSET_INTERPOLATION 13 /* gates/coset_interpolation.rs, param = subgroup_bits, param2 = degree */
typedef struct {
    uint32_t kind, param;
    uint32_t selector_index;          /* SelectorsInfo.selector_indices[gate] (gates/selectors.rs:17-20) */
    uint32_t group_start, group_end;  /* SelectorsInfo.groups[selector_index] */
    uint32_t param2, param3;
} glo_gate;
typedef struct {
    uint32_t num_wires, num_routed_wires, num_constants /* selectors included */, num_challenges;
    uint32_t quotient_degree_factor, num_selectors, num_partial_products, num_gate_constraints;
    const glo_gate* gates; /* sorted the way CommonCircuitData.gates is */
    size_t n_gates;
    const uint64_t* k_is;
    /* lookups (all 0 / NULL without): the lookup selectors follow the gate selectors in the constants; luts = the tables'
     * (input, output) pairs, concatenated, lut_len[t] pairs each; one LookupWire per table */
    uint32_t num_lookup_selectors, num_lookup_polys;
    size_t n_luts;
    const uint32_t* lut_len;
    const uint64_t *lut_inp, *lut_out;
} glo_circuit;
/* deltas: NUM_COINS_LOOKUP = 4 per challenge (A, B, alpha, delta), NULL without lookups; with lookups zs_partial_products
 * also holds num_lookup_polys polynomials per challenge after the partial products (check_lookup_constraints_batch,
 * vanishing_poly.rs:521-689). */
int glo_plonk_quotient(const glo_circuit* cd, const glo_commit* constants_sigmas, const glo_commit* wires,
                       const glo_commit* zs_partial_products, const uint64_t public_inputs_hash[4], const uint64_t* betas,
                       const uint64_t* gammas, const uint64_t* deltas, const uint64_t* alphas, uint64_t* out);

/* Restated batch-FRI verifier (plonky2/src/batch_fri/verifier.rs:22-251): group_num_polys[o * n_instances + i] =
 * polynomials of oracle o in degree group i; opened_values per instance, per batch, per polynomial (2 words each).
 * challenger in the state batch_prove_openings started from. Returns 0 if the proof verifies. */
int glo_verify_batch_fri_proof(const uint64_t* const* initial_caps, const size_t* group_num_polys, size_t n_oracles,
                               const uint32_t* degree_bits, const glo_fri_instance* instances, size_t n_instances,
                               const uint64_t* opened_values, glo_challenger* challenger, const glo_fri_params* params,
                               const uint8_t* proof, size_t proof_len);

/* Restated FRI verifier (plonky2/src/fri/verifier.rs:62-241, challenges.rs:28-75): checks a
 * serialised proof against the initial caps and the claimed openings. challenger must be in the
 * same state prove_openings started from. opened_values: for each batch, for each polynomial,
 * the F_{p^2} value f(point) (2 words each), concatenated in batch order.
 * Returns 0 if the proof verifies, a positive code naming the failed check otherwise. */
int glo_verify_fri_proof(const uint64_t* const* initial_caps, const size_t* oracle_num_polys,
                         const size_t* oracle_leaf_width, size_t n_oracles,
                         const glo_fri_batch* batches, size_t n_batches,
                         const uint64_t* opened_values, uint32_t degree_bits,
                         glo_challenger* challenger, const glo_fri_params* params,
                         const uint8_t* proof, size_t proof_len);

/* ---- "next" row (SURVEY 8f-3): wires_permutation_partial_products_and_zs
 *      (plonky2/src/plonk/prover.rs:387-449, util/partial_products.rs:13-37) ----
 * wires, sigmas: num_routed columns of n values, column-major (wire_values[col][row]; sigma polynomial values).
 * out: (num_prods + 1) columns of n values, column-major, partial products first and Z LAST (the function's
 * return order; the prover then moves Z to the front, prover.rs:227-232). Returns 0, or 1 on a zero denominator
 * (the reference's batch_multiplicative_inverse panics). */
int glo_partial_products_and_zs(const uint64_t* wires, const uint64_t* sigmas, const uint64_t* k_is,
                                uint32_t log_n, uint32_t num_routed, uint64_t beta, uint64_t gamma,
                                uint32_t degree, uint64_t* out);

/* ---- "next" row (SURVEY 8f-3, second half): compute_lookup_polys (plonky2/src/plonk/prover.rs:458-577) for one
 *      challenge set deltas = (A, B, alpha, delta). wires: witness matrix, wire w of row i at wires[w*n + i].
 *      lookup_rows: triples (last_lu_gate, last_lut_gate, first_lut_gate). out: (num_partial_lookups + 1) columns of n.
 *      Returns 0, or 1 on a zero denominator. */
int glo_lookup_polys(const uint64_t* wires, uint32_t log_n, uint32_t num_routed_wires,
                     uint32_t max_quotient_degree_factor, const uint64_t deltas[4], const uint32_t* lookup_rows,
                     uint32_t n_lookup_wires, uint64_t* out);

/* ---- "next" row (SURVEY 8f-1): compute_quotient_polys of starky for FibonacciStark
 *      (starky/src/prover.rs:488-668, starky/src/fibonacci_stark.rs:73-95). trace: a 2-column commitment; pi = (x0, x1,
 *      result); out = n_alphas polynomials of (n << quotient_degree_bits) coefficients. Returns 0 on success. */
int glo_stark_quotient_fibonacci(const glo_commit* trace, const uint64_t pi[3], const uint64_t* alphas,
                                 size_t n_alphas, uint64_t* out);

/* polynomial evaluation helper for the verifier test: f(z) for base coeffs, z in F_{p^2} */
void glo_eval_poly_base_at_ext(const uint64_t* coeffs, size_t n, const uint64_t z[2], uint64_t out[2]);

#ifdef __cplusplus
}
#endif
#endif
