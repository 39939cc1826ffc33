// Host run of the device row arithmetic of starky's logUp helper columns (plonky2_b200/csrc/gl_logup.cuh): the same
// logup_row the kernel k_logup_rows calls per thread, with threads as a loop and host arrays in place of device memory,
// and Z as a sequential running sum. Test infrastructure: built as a shared library and driven by
// tests/test_stark_lookups.py, which compares the result with the restatement of lookup_helper_columns.
#include <vector>
#include "../../plonky2_b200/csrc/gl_logup.cuh"
using namespace gl;

// Arguments as gl_stark_lookup_helpers takes them (include/plonky2_b200.h), with host memory; the parameters are set up
// the way that entry point does. Returns 1 if a denominator was zero.
extern "C" int emu_stark_lookup_helpers(const uint64_t* trace, size_t col_stride, uint32_t log_n,
                                        const gl_stark_instr* program, const uint32_t* lookup_offsets, uint32_t n_lookups,
                                        const uint64_t* consts, const uint64_t* challenges, uint32_t n_challenges,
                                        uint32_t constraint_degree, uint64_t* out) {
    const size_t n = (size_t)1 << log_n;
    const uint32_t chunk = constraint_degree == 0 ? 1 : constraint_degree - 1;
    std::vector<uint64_t> term((size_t)n_challenges * n);
    int bad = 0;
    size_t col = 0;
    for (uint32_t l = 0; l < n_lookups; l++) {
        LogupParams p;
        p.trace = trace;
        p.trace_stride = col_stride;
        p.log_n = log_n;
        p.prog = program + lookup_offsets[l];
        p.n_instr = lookup_offsets[l + 1] - lookup_offsets[l];
        p.consts = consts;
        uint32_t looked = 0;
        for (uint32_t k = 0; k < p.n_instr; k++)
            if (p.prog[k].op == GL_STARK_EMIT && p.prog[k].b == GL_LOGUP_LOOKED) looked++;
        p.chunk = chunk;
        p.num_h = (looked + chunk - 1) / chunk;
        for (uint32_t c = 0; c < GL_STARK_MAX_ALPHAS; c++) p.gammas[c] = c < n_challenges ? canon(challenges[c]) : 0;
        p.n_challenges = n_challenges;
        p.h_out = out + col * n;
        p.term = term.data();
        for (size_t i = 0; i < n; i++) {  // one "thread" per row
            uint64_t v[GL_LOGUP_MAX_INSTR];
            for (int k = 0; k < GL_LOGUP_MAX_INSTR; k++) v[k] = 0xDEADBEEFDEADBEEFull;  // uninitialised on the device
            if (!logup_row(p, i, v)) bad = 1;
        }
        for (uint32_t c = 0; c < n_challenges; c++) {  // Z[0] = 0, Z[i + 1] = Z[i] + term[i]
            uint64_t* z = out + (col + (size_t)c * (p.num_h + 1) + p.num_h) * n;
            uint64_t run = 0;
            for (size_t i = 0; i < n; i++) {
                z[i] = canon(run);
                run = add(run, term[(size_t)c * n + i]);
            }
        }
        col += (size_t)n_challenges * (p.num_h + 1);
    }
    return bad;
}
