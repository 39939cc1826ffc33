// gl_plonk_blocked_host.cuh -- gl_plonk_quotient_blocked of include/plonky2_b200_blocked.h: the plonky2 quotient on
// non-resident commitments. Included at the end of plonky2_b200.cu, whose plonk_quotient evaluates it: the checks of
// the other plonky2 quotient entry points, then the coset in one part per LDE block (quotient_in_parts, shared with
// the STARK quotient), each part's values from k_plonk_quotient with the shard addressing of gl_plonk_quotient_shard.
#pragma once
#include "../../include/plonky2_b200_blocked.h"

int gl_plonk_quotient_blocked(gl_ctx* ctx, gl_commit* const* commits, uint32_t n_commits, const gl_vp_instr* program,
                              uint32_t n_instr, const uint64_t* consts, uint32_t n_consts, const uint64_t* alphas,
                              uint32_t n_alphas, uint32_t n_terms, uint32_t quotient_degree_factor,
                              uint64_t* out_coeffs) {
    return plonk_quotient(ctx, commits, n_commits, program, n_instr, consts, n_consts, alphas, n_alphas, n_terms,
                          quotient_degree_factor, out_coeffs, PlonkHandles::BLOCKED);
}
