/*
 * plonky2_b200_blocked.h -- the plonky2 quotient on non-resident commitments (gl_commit_begin_blocked), for circuits
 * whose commitments' LDEs do not fit on the device. The conventions of plonky2_b200.h hold (status codes,
 * gl_last_error, field elements as uint64_t, non-canonical inputs accepted); the program, constants, alphas and output
 * are those of gl_plonk_quotient. Host inputs (the program, its constants and the alphas) have been read when a call
 * returns: every call ends in a synchronising read-back of its error flags.
 */
#ifndef PLONKY2_B200_BLOCKED_H
#define PLONKY2_B200_BLOCKED_H
#include "plonky2_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* gl_plonk_quotient on commitments that keep no LDE: every handle non-resident with the same num_blocks = G = 2^s. The
 * quotient coset (size = n << log2_ceil(quotient_degree_factor) points) is evaluated in G parts, one after another:
 * part g is the points i = r + G*k (k < M = size / G, r = the s-bit reversal of g), as shard g of
 * gl_plonk_quotient_shard owns them. The part's local values are the LDE of each handle's coefficients onto the part's
 * coset; its next row is read from them when G divides 2^log2_ceil(quotient_degree_factor), else it is the LDE onto
 * the coset times w_n, built only for the commitments the program reads with GL_VP_NEXT. Each part's values go to
 * their points of out_coeffs, and the whole coset then takes gl_plonk_quotient's coset iFFT and trim check: the result
 * and the errors ("Quotient has failed ...", GL_ERR_BAD_ARG) equal gl_plonk_quotient's on resident commitments of the
 * same polynomials, word for word.
 * Refused with GL_ERR_BAD_ARG before any launch: a resident handle, a row-block shard, handles of different G, and G
 * above the quotient coset's points; everything else (program, constants, terms, limits) is checked as in
 * gl_plonk_quotient. The program may not read salt columns (non-resident handles have none).
 * Scratch per part: sum of B x M words over the commitments, twice that for those read with GL_VP_NEXT when the next
 * row leaves the part, plus n_alphas x M words for the part's values (out_coeffs is n_alphas x size words). */
int gl_plonk_quotient_blocked(gl_ctx* ctx, gl_commit* const* commits, uint32_t n_commits, const gl_vp_instr* program,
                              uint32_t n_instr, const uint64_t* consts, uint32_t n_consts, const uint64_t* alphas,
                              uint32_t n_alphas, uint32_t n_terms, uint32_t quotient_degree_factor,
                              uint64_t* out_coeffs);

#ifdef __cplusplus
}
#endif
#endif
