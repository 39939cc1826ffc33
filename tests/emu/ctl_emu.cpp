// Host run of the device row arithmetic of starky's cross-table lookup helper columns (plonky2_b200/csrc/gl_ctl.cuh):
// the same ctl_row the kernel k_ctl_rows calls per thread, with threads as a loop and host arrays in place of device
// memory, and Z as a sequential suffix sum. Test infrastructure: built as a shared library and driven by
// tests/test_stark_ctl.py, which compares the result with the restatement of cross_table_lookup_data.
#include <vector>
#include "../../plonky2_b200/csrc/gl_ctl.cuh"
using namespace gl;

// Arguments as gl_stark_ctl_helpers takes them (include/plonky2_b200.h), with host memory and a valid program; the
// parameters are set up the way that entry point does. Returns 1 if a denominator was zero.
extern "C" int emu_stark_ctl_helpers(const uint64_t* trace, size_t col_stride, uint32_t log_n,
                                     const gl_stark_instr* program, const uint32_t* group_offsets, uint32_t n_groups,
                                     const uint64_t* consts, const uint64_t* challenges, uint32_t n_challenges,
                                     uint32_t constraint_degree, const uint32_t* zs_index, uint64_t* out) {
    const size_t n = (size_t)1 << log_n;
    const uint32_t chunk = constraint_degree == 0 ? 1 : constraint_degree - 1;
    std::vector<uint32_t> num_h(n_groups);
    for (uint32_t g = 0; g < n_groups; g++) {
        uint32_t entries = 0;
        for (uint32_t k = group_offsets[g]; k < group_offsets[g + 1]; k++)
            if (program[k].op == GL_STARK_EMIT && program[k].b == GL_CTL_FILTER) entries++;
        num_h[g] = entries > 1 ? (entries + chunk - 1) / chunk : 0;
    }
    const uint32_t n_zs = n_groups * n_challenges;
    std::vector<uint32_t> at(n_zs);
    for (uint32_t k = 0; k < n_zs; k++) at[zs_index[k]] = k;
    CtlParams p;
    uint32_t total_h = 0;
    for (uint32_t z = 0; z < n_zs; z++) {
        const uint32_t g = at[z] / n_challenges, c = at[z] % n_challenges;
        p.helper_col[g][c] = total_h;
        total_h += num_h[g];
    }
    std::vector<uint64_t> term((size_t)n_zs * n);
    p.trace = trace;
    p.trace_stride = col_stride;
    p.log_n = log_n;
    p.prog = program + group_offsets[0];
    for (uint32_t g = 0; g <= n_groups; g++) p.offsets[g] = group_offsets[g] - group_offsets[0];
    p.n_groups = n_groups;
    p.consts = consts;
    p.chunk = chunk;
    for (uint32_t c = 0; c < GL_STARK_MAX_ALPHAS; c++) {
        p.betas[c] = c < n_challenges ? canon(challenges[2 * c]) : 0;
        p.gammas[c] = c < n_challenges ? canon(challenges[2 * c + 1]) : 0;
    }
    p.n_challenges = n_challenges;
    p.out = out;
    p.term = term.data();
    int bad = 0;
    for (size_t i = 0; i < n; i++) {  // one "thread" per row
        uint64_t v[GL_CTL_MAX_INSTR];
        for (int k = 0; k < GL_CTL_MAX_INSTR; k++) v[k] = 0xDEADBEEFDEADBEEFull;  // uninitialised on the device
        if (!ctl_row(p, i, v)) bad = 1;
    }
    for (uint32_t k = 0; k < n_zs; k++) {  // Z[n - 1] = term[n - 1], Z[i] = Z[i + 1] + term[i]
        uint64_t* z = out + ((size_t)total_h + zs_index[k]) * n;
        uint64_t run = 0;
        for (size_t i = n; i-- > 0;) {
            run = add(run, term[(size_t)k * n + i]);
            z[i] = canon(run);
        }
    }
    return bad;
}
