/*
 * plonky2_b200_check.h -- constraint checks of the H100-native plonky2 / starky prover (sm_90a CUDA), for debug builds:
 * the counterpart of starky's check_constraints (starky/src/prover.rs:241-256,670-820), which the reference runs under
 * #[cfg(debug_assertions)] only. The conventions of plonky2_b200.h hold (status codes, gl_last_error, field elements
 * as uint64_t, non-canonical inputs accepted); the programs and handles are the ones its quotient entry points take.
 * Host inputs (the program and its constants) have been read when a call returns: every call ends in a synchronising
 * read-back of its outputs.
 */
#ifndef PLONKY2_B200_CHECK_H
#define PLONKY2_B200_CHECK_H
#include "plonky2_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* check_constraints (starky/src/prover.rs:670-820) on the device, and its plonky2 counterpart: the program the matching
 * quotient entry point runs, checked on every row i of the trace subgroup H = <w_n> at x = w_n^i (no coset shift), each
 * constraint on its own. The values on H are the NTT of each commitment's coefficients, so every kind of handle is
 * checked alike: resident, non-resident (gl_commit_begin_blocked), a row-block shard (its coefficients are replicated)
 * and salted (GL_VP_LOCAL / GL_VP_NEXT operands are bounded by B, never W: salt columns are not polynomials).
 * A LOCAL operand reads row i, a NEXT operand row (i + 1) mod n. Nothing about the quotient degree is required: a STARK
 * of constraint degree 0 is checked like any other.
 *   gl_stark_check_rows  GL_STARK_EMIT number e (its ordinal among the program's EMITs) of value v fails at row i when
 *                        v is nonzero and its filter is on: GL_STARK_CONSTRAINT always, GL_STARK_TRANSITION at every
 *                        row but n - 1 (z_last = x - w_n^-1), GL_STARK_FIRST_ROW at row 0, GL_STARK_LAST_ROW at row
 *                        n - 1 -- the reference's filter values on H. aux = NULL: the program may not read auxiliary
 *                        columns. consts as for gl_stark_quotient; no alphas.
 *   gl_plonk_check_rows  GL_VP_TERM b fails at row i when its value is nonzero. GL_VP_X is w_n^i, GL_VP_L0 the indicator
 *                        [i = 0]; there is no Z_H and no alpha. On H only the row's own gate has a nonzero selector
 *                        filter, so a failing gate-constraint term at row i is a constraint of the gate at row i.
 * Outputs (HOST memory): *out_failures = the number of failing (row, index) pairs; out_pairs = the first max_report of
 * them in (row, index) order, row then index, 2 x max_report words (may be NULL when max_report is 0);
 * *out_reported = how many were written, min(*out_failures, max_report). GL_OK means the check ran, whether or not
 * anything failed. Refused before any launch: a NULL argument, an unfinished handle, commitments of different degree
 * or of another context, max_report > 65536 (GL_ERR_BAD_ARG / GL_ERR_BAD_SHAPE), and the quotient entry points' program
 * errors with their messages. Scratch: B x n words per commitment read, plus 8 (n + 1) bytes.
 *
 * The _part entry points check one part of H, for checks whose scratch must shrink (a non-resident proof checks its
 * parts one after another) or be split between devices (each rank of a distributed proof checks its own part). Part g
 * of parts = G = 2^s is the rows i = g (mod G), the coset w_n^g <w_M> with M = n / G; its values are a size-M NTT of the
 * coefficients folded mod X^M - w_G^g, and a commitment the program reads with NEXT also gets its values on the next
 * rows, w_n^(g+1) <w_M>. Every row-dependent quantity (the filters, GL_VP_X, GL_VP_L0) is the global row's, and rows
 * are reported as global indices in (row, index) order. (part, parts) = (0, 1) is exactly gl_*_check_rows.
 * Refused before any launch, after the refusals above: parts not a power of two or above n (GL_ERR_BAD_SHAPE), part >=
 * parts (GL_ERR_BAD_ARG). Scratch: B x M words per commitment read, plus B x M more per commitment read with NEXT when
 * G > 1, plus 8 (M + 1) bytes.
 * Merging the G parts' reports gives the whole check's: the failures add up, and the first max_report pairs of the
 * sorted union of the parts' pairs are the whole check's pairs. Each part's pairs are a subsequence of the global (row,
 * index) order, so the global first max_report pairs all lie within their parts' first max_report. */
int gl_stark_check_rows(gl_ctx* ctx, gl_commit* trace, gl_commit* aux, const gl_stark_instr* program, uint32_t n_instr,
                        const uint64_t* consts, uint32_t n_consts, uint32_t max_report, uint64_t* out_failures,
                        uint32_t* out_pairs, uint32_t* out_reported);
int gl_plonk_check_rows(gl_ctx* ctx, gl_commit* const* commits, uint32_t n_commits, const gl_vp_instr* program,
                        uint32_t n_instr, const uint64_t* consts, uint32_t n_consts, uint32_t n_terms,
                        uint32_t max_report, uint64_t* out_failures, uint32_t* out_pairs, uint32_t* out_reported);
int gl_stark_check_rows_part(gl_ctx* ctx, gl_commit* trace, gl_commit* aux, const gl_stark_instr* program,
                             uint32_t n_instr, const uint64_t* consts, uint32_t n_consts, uint32_t part, uint32_t parts,
                             uint32_t max_report, uint64_t* out_failures, uint32_t* out_pairs, uint32_t* out_reported);
int gl_plonk_check_rows_part(gl_ctx* ctx, gl_commit* const* commits, uint32_t n_commits, const gl_vp_instr* program,
                             uint32_t n_instr, const uint64_t* consts, uint32_t n_consts, uint32_t n_terms,
                             uint32_t part, uint32_t parts, uint32_t max_report, uint64_t* out_failures,
                             uint32_t* out_pairs, uint32_t* out_reported);

/* plonky2's two global arguments checked on a witness, before any commitment: what the reference's witness generation
 * stops at (iop/witness.rs:358, "Partition containing {target} was set twice with different values"; gates/lookup.rs:
 * 208-220, "Incorrect input value provided") and what set_lookup_wires (plonk/prover.rs:50-108) writes. They read the
 * witness, the sigma columns and the circuit's shape only: no commitment, no challenge. Witness column c (and sigma
 * column c) is at wires + c * stride, on the host or the device (GL_MEM_HOST / GL_MEM_DEVICE); non-canonical values
 * compare canonically. Outputs (HOST memory) as for gl_plonk_check_rows: *out_failures, the first max_report pairs in
 * (first word, second word) order in out_pairs, *out_reported. Refused before any launch: a NULL argument, max_report >
 * 65536 (GL_ERR_BAD_ARG), a stride below n (GL_ERR_BAD_SHAPE).
 *   gl_plonk_check_copies   routed wire i = row * num_routed_wires + col (row < n = 2^log_n) has the identity value
 *                           k_is[col] * w_n^row and the sigma value sigmas[col][row]; sigma(i) is the routed wire whose
 *                           identity value is i's sigma value. The pair (i, sigma(i)) fails when the two wires' values
 *                           differ. Sigmas that are not a permutation of the identity values are GL_ERR_BAD_ARG (corrupt
 *                           prover data), found on the device; n * num_routed_wires must be below 2^31 - 1
 *                           (GL_ERR_BAD_SHAPE). Both (u64 value, u32 index) lists are radix-sorted: scratch 36 bytes
 *                           per routed wire at the peak (the sorted identity list and both buffers of the sigma list's
 *                           sort), 32 while host sigmas are staged, 20 in the end (sigma, host wires, the report).
 *   gl_plonk_check_lookups  table k of n_luts has the entries luts[2e], luts[2e + 1] (input, output) for e in
 *                           [lut_offsets[k], lut_offsets[k + 1]) and the rows lookup_rows[3k .. 3k + 2] = (last_lu,
 *                           last_lut, first_lut): LookupGate rows [last_lu, last_lut), num_routed_wires / 2 slots of
 *                           (input, output) in wires (2s, 2s + 1); LookupTableGate rows [last_lut, first_lut],
 *                           num_routed_wires / 3 slots of (input, output, multiplicity) in wires (3s, 3s + 1, 3s + 2).
 *                           Entry e is placed at row first_lut - e / (num_routed_wires / 3), slot e % that; slots past
 *                           the LUT hold entry 0 with multiplicity 0. A looking slot counts for the entry the reference's
 *                           input -> index map gives its input (a later entry of one input wins); the run of slots at
 *                           the end of row last_lut - 1 that all hold entry 0 is the reference's padding and counts for
 *                           entry 0. The witness alone cannot tell that padding from real lookups of entry 0 which end
 *                           the row; the two differ only when entry 0's input appears again later in the LUT (the
 *                           reference counts a real lookup for the later entry), and then an honest witness gets two L3
 *                           failures, for entry 0 and that later entry: a known false positive of a witness-only
 *                           check. A failure is the pair (row, 4 * slot + kind): kind 1 (L1) a looking pair that is
 *                           not an entry of the table; 2 (L2) a table slot that does not hold the entry placed there;
 *                           3 (L3) a table slot whose multiplicity is not its entry's count. out_counts (may be NULL):
 *                           every entry's count, laid out as luts. Refused: an empty LUT, rows out of order or past n,
 *                           two tables' rows overlapping (GL_ERR_BAD_ARG), a LUT longer than its table rows hold
 *                           (GL_ERR_BAD_SHAPE). Scratch: the wire columns read (host input), 256 KiB per table, 8 (n + 1)
 *                           bytes. */
int gl_plonk_check_copies(gl_ctx* ctx, const uint64_t* wires, size_t wires_stride, int wires_mem,
                          const uint64_t* sigmas, size_t sigmas_stride, int sigmas_mem, const uint64_t* k_is,
                          uint32_t log_n, uint32_t num_routed_wires, uint32_t max_report, uint64_t* out_failures,
                          uint32_t* out_pairs, uint32_t* out_reported);
int gl_plonk_check_lookups(gl_ctx* ctx, const uint64_t* wires, size_t col_stride, int mem, uint32_t log_n,
                           uint32_t num_routed_wires, const uint16_t* luts, const uint32_t* lut_offsets,
                           const uint32_t* lookup_rows, uint32_t n_luts, uint32_t* out_counts, uint32_t max_report,
                           uint64_t* out_failures, uint32_t* out_pairs, uint32_t* out_reported);

#ifdef __cplusplus
}
#endif
#endif
