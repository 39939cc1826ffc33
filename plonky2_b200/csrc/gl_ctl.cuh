// gl_ctl.cuh -- one row of starky's cross-table lookup helper columns: partial_sums / get_helper_cols
// (starky/src/cross_table_lookup.rs:383-414, lookup.rs:746-789) for every CtlZData of one table and every challenge,
// before the suffix sum Z.
//
// A table's CtlZData groups come from its entries in one CrossTableLookup: its consecutive looking entries (one group,
// ctl_helper_zs_cols) or its looked entry (a group of one). Each group arrives as a straight-line row program in the
// gl_stark_instr format (GL_STARK_LOCAL = row i, GL_STARK_NEXT = row (i + 1) mod n: Column::eval_table /
// Filter::eval_table), whose GL_STARK_EMIT instructions name, entry by entry, the tuple's values in order
// (GL_CTL_VALUE) and then the entry's filter (GL_CTL_FILTER). For each challenge (beta, gamma) the thread forms
//   combine_j = gamma + sum_k beta^k v_{j,k}             (GrandProductChallenge::combine, lookup.rs:457-464)
// for every entry j, inverts them TOGETHER (Montgomery's trick, one field inversion per (row, group, challenge)), and
// writes, for a group of more than one entry, the helper columns h_k = sum_{j in chunk k} filter_j / combine_j; the
// row's term of Z is sum_k h_k (a single entry: filter / combine, no helper column). Z is the suffix sum of the terms
// (Z[n - 1] = term[n - 1], Z[i] = Z[i + 1] + term[i]), which the caller takes from the multi-CTA additive scan.
//
// The same source runs on the host in tests/emu/ctl_emu.cpp (threads as a loop) against a restatement of the reference.
#pragma once
#include "../../include/plonky2_b200.h"
#include "gl_field.cuh"

namespace gl {

struct CtlParams {
    const uint64_t* trace;        // trace VALUES, column k at trace + k*trace_stride, row order
    size_t trace_stride;
    uint32_t log_n;
    const gl_stark_instr* prog;   // the groups' row programs back to back (validated by the caller)
    uint32_t offsets[GL_CTL_MAX_GROUPS + 1];  // group g: prog[offsets[g] .. offsets[g + 1])
    uint32_t n_groups;
    const uint64_t* consts;
    uint32_t chunk;               // entries per helper column: constraint_degree - 1, or 1 (lookup.rs:757)
    uint64_t betas[GL_STARK_MAX_ALPHAS], gammas[GL_STARK_MAX_ALPHAS];
    uint32_t n_challenges;
    // helper column h_k of (group g, challenge c) at out + (helper_col[g][c] + k) * n (groups of one entry: none)
    uint32_t helper_col[GL_CTL_MAX_GROUPS][GL_STARK_MAX_ALPHAS];
    uint64_t* out;
    uint64_t* term;               // (group g, challenge c)'s term sequence at term + (g * n_challenges + c) * n
};

// Row i. Returns false if a denominator is zero ("Tried to invert zero"); the outputs of that row are then garbage.
// v: GL_CTL_MAX_INSTR words of scratch.
GL_HD bool ctl_row(const CtlParams& p, size_t i, uint64_t* v) {
    const size_t n = (size_t)1 << p.log_n;
    const size_t inext = (i + 1) & (n - 1);
    bool ok = true;
    for (uint32_t g = 0; g < p.n_groups; g++) {
        const gl_stark_instr* prog = p.prog + p.offsets[g];
        const uint32_t n_instr = p.offsets[g + 1] - p.offsets[g];
        // comb[j][c]: entry j's sum_k beta_c^k v_{j,k} so far; pw[c] = beta_c^k of the entry's next value
        uint64_t comb[GL_CTL_MAX_ENTRIES][GL_STARK_MAX_ALPHAS], filt[GL_CTL_MAX_ENTRIES], pw[GL_STARK_MAX_ALPHAS];
        uint32_t ne = 0;
        for (uint32_t c = 0; c < GL_STARK_MAX_ALPHAS; c++) comb[0][c] = 0, pw[c] = 1;
        for (uint32_t k = 0; k < n_instr; k++) {
            const gl_stark_instr in = prog[k];
            uint64_t r = 0;
            switch (in.op) {
                case GL_STARK_LOCAL: r = p.trace[(size_t)in.a * p.trace_stride + i]; break;
                case GL_STARK_NEXT: r = p.trace[(size_t)in.a * p.trace_stride + inext]; break;
                case GL_STARK_CONST: r = p.consts[in.a]; break;
                case GL_STARK_ADD: r = add(v[in.a], v[in.b]); break;
                case GL_STARK_SUB: r = sub(v[in.a], v[in.b]); break;
                case GL_STARK_MUL: r = mul(v[in.a], v[in.b]); break;
                default:  // GL_STARK_EMIT: a value of entry ne's tuple, or its filter (which closes the entry)
                    if (in.b == GL_CTL_VALUE) {
                        for (uint32_t c = 0; c < p.n_challenges; c++) {
                            comb[ne][c] = add(comb[ne][c], mul(pw[c], v[in.a]));
                            pw[c] = mul(pw[c], p.betas[c]);
                        }
                    } else {
                        filt[ne++] = v[in.a];
                        if (ne < GL_CTL_MAX_ENTRIES)
                            for (uint32_t c = 0; c < GL_STARK_MAX_ALPHAS; c++) comb[ne][c] = 0, pw[c] = 1;
                    }
            }
            v[k] = r;
        }
        const uint32_t num_h = ne > 1 ? (ne + p.chunk - 1) / p.chunk : 0;
        for (uint32_t c = 0; c < p.n_challenges; c++) {
            // den[j] = combine_j; pre[j] = den[0] * ... * den[j]
            uint64_t pre[GL_CTL_MAX_ENTRIES], inv_den[GL_CTL_MAX_ENTRIES];
            uint64_t run = 1;
            for (uint32_t j = 0; j < ne; j++) {
                const uint64_t d = add(comb[j][c], p.gammas[c]);
                if (canon(d) == 0) ok = false;
                inv_den[j] = d;
                run = mul(run, d);
                pre[j] = run;
            }
            uint64_t inv_run = inv(run);
            for (uint32_t j = ne; j-- > 0;) {  // 1/den_j = inv_run * pre[j-1], then inv_run *= den_j
                const uint64_t di = j ? mul(inv_run, pre[j - 1]) : inv_run;
                inv_run = mul(inv_run, inv_den[j]);
                inv_den[j] = di;
            }
            uint64_t sum = 0;
            if (num_h == 0) {
                sum = mul(filt[0], inv_den[0]);
            } else {
                for (uint32_t k = 0; k < num_h; k++) {
                    uint64_t h = 0;
                    const uint32_t j1 = (k + 1) * p.chunk < ne ? (k + 1) * p.chunk : ne;
                    for (uint32_t j = k * p.chunk; j < j1; j++) h = add(h, mul(filt[j], inv_den[j]));
                    p.out[((size_t)p.helper_col[g][c] + k) * n + i] = canon(h);
                    sum = add(sum, h);
                }
            }
            p.term[((size_t)g * p.n_challenges + c) * n + i] = canon(sum);
        }
    }
    return ok;
}

}  // namespace gl
