// gl_logup.cuh -- one row of starky's logUp helper columns: lookup_helper_columns / get_helper_cols
// (starky/src/lookup.rs:579-652,746-789) for one Lookup and every challenge, before the running sum Z.
//
// The reference evaluates every looking column, filter, the table and the frequencies column on every row
// (Column::eval_table / Filter::eval_table, lookup.rs:118-129,323-335), inverts each of them column by column
// (F::batch_multiplicative_inverse) and sums. Here one thread owns one row: the Lookup arrives as a small
// straight-line row program in the gl_stark_instr format (GL_STARK_LOCAL = row i, GL_STARK_NEXT = row (i + 1) mod n),
// whose GL_STARK_EMIT instructions name the row's inputs by role (GL_LOGUP_*, include/plonky2_b200.h), and for each
// challenge gamma the row's denominators f_j + gamma and t + gamma are inverted TOGETHER (Montgomery's trick, one
// field inversion per (row, challenge)). The thread writes the helper columns h_k and the row's term of Z,
//   term[i] = sum_k h_k[i] - m[i] / (t[i] + gamma),
// which the multi-CTA additive scan turns into Z (Z[0] = 0, Z[i + 1] = Z[i] + term[i]).
//
// The same source runs on the host in tests/emu/logup_emu.cpp (threads as a loop) against a restatement of the reference.
#pragma once
#include "../../include/plonky2_b200.h"
#include "gl_field.cuh"

namespace gl {

struct LogupParams {
    const uint64_t* trace;        // trace VALUES, column k at trace + k*trace_stride, row order
    size_t trace_stride;
    uint32_t log_n;
    const gl_stark_instr* prog;   // this Lookup's row program (validated by the caller)
    uint32_t n_instr;
    const uint64_t* consts;
    uint32_t chunk;               // looking columns per helper column: constraint_degree - 1, or 1 (lookup.rs:757)
    uint32_t num_h;               // helper columns h_k per challenge: ceil(looking columns / chunk)
    uint64_t gammas[GL_STARK_MAX_ALPHAS];
    uint32_t n_challenges;
    uint64_t* h_out;              // h_k of challenge c at h_out + (c * (num_h + 1) + k) * n  (column num_h is Z)
    uint64_t* term;               // challenge c's term sequence at term + c * n
};

// Row i. Returns false if a denominator is zero ("Tried to invert zero"); the outputs of that row are then garbage.
// v: GL_LOGUP_MAX_INSTR words of scratch.
GL_HD bool logup_row(const LogupParams& p, size_t i, uint64_t* v) {
    const size_t n = (size_t)1 << p.log_n;
    const size_t inext = (i + 1) & (n - 1);
    uint64_t f[GL_LOGUP_MAX_COLUMNS], filt[GL_LOGUP_MAX_COLUMNS];
    uint64_t t = 0, m = 0;
    uint32_t nf = 0, nfl = 0;
    for (uint32_t k = 0; k < p.n_instr; k++) {
        const gl_stark_instr in = p.prog[k];
        uint64_t r = 0;
        switch (in.op) {
            case GL_STARK_LOCAL: r = p.trace[(size_t)in.a * p.trace_stride + i]; break;
            case GL_STARK_NEXT: r = p.trace[(size_t)in.a * p.trace_stride + inext]; break;
            case GL_STARK_CONST: r = p.consts[in.a]; break;
            case GL_STARK_ADD: r = add(v[in.a], v[in.b]); break;
            case GL_STARK_SUB: r = sub(v[in.a], v[in.b]); break;
            case GL_STARK_MUL: r = mul(v[in.a], v[in.b]); break;
            default:  // GL_STARK_EMIT: an input of the row, by role
                if (in.b == GL_LOGUP_LOOKED) f[nf++] = v[in.a];
                else if (in.b == GL_LOGUP_FILTER) filt[nfl++] = v[in.a];
                else if (in.b == GL_LOGUP_TABLE) t = v[in.a];
                else m = v[in.a];
        }
        v[k] = r;
    }
    bool ok = true;
    const size_t nh = (size_t)p.num_h + 1;
    for (uint32_t c = 0; c < p.n_challenges; c++) {
        const uint64_t g = p.gammas[c];
        // den[j] = f_j + gamma (j < nf), den[nf] = t + gamma; pre[j] = den[0] * ... * den[j]
        uint64_t pre[GL_LOGUP_MAX_COLUMNS + 1], inv_den[GL_LOGUP_MAX_COLUMNS + 1];
        uint64_t run = 1;
        for (uint32_t j = 0; j <= nf; j++) {
            const uint64_t d = add(j < nf ? f[j] : t, g);
            if (canon(d) == 0) ok = false;
            inv_den[j] = d;
            run = mul(run, d);
            pre[j] = run;
        }
        uint64_t inv_run = inv(run);
        for (uint32_t j = nf + 1; j-- > 0;) {  // 1/den_j = inv_run * pre[j-1], then inv_run *= den_j
            const uint64_t di = j ? mul(inv_run, pre[j - 1]) : inv_run;
            inv_run = mul(inv_run, inv_den[j]);
            inv_den[j] = di;
        }
        uint64_t sum = 0;
        for (uint32_t k = 0; k < p.num_h; k++) {
            uint64_t h = 0;
            const uint32_t j1 = (k + 1) * p.chunk < nf ? (k + 1) * p.chunk : nf;
            for (uint32_t j = k * p.chunk; j < j1; j++) h = add(h, mul(filt[j], inv_den[j]));
            p.h_out[((size_t)c * nh + k) * n + i] = canon(h);
            sum = add(sum, h);
        }
        p.term[(size_t)c * n + i] = canon(sub(sum, mul(m, inv_den[nf])));
    }
    return ok;
}

}  // namespace gl
