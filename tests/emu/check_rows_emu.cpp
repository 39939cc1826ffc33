// Host run of the row checks of gl_stark_check_rows (plonky2_b200/csrc/gl_stark_rows.cuh) and gl_plonk_check_rows
// (gl_vanishing.cuh): the same stark_check_row / vp_check_row the kernels call per thread, with threads as a loop over
// the rows and host arrays in place of device memory. Test infrastructure: built as a shared library and driven by
// tests/test_check_constraints.py against an exact evaluator of the programs.
//
// Both functions write every row's failure count to counts[i] and, when pairs is not NULL, every failure as a (row,
// index) pair, rows in order (pairs must hold 2 x the total). Both return the total.
#include <vector>
#include "../../plonky2_b200/csrc/gl_stark_rows.cuh"
#include "../../plonky2_b200/csrc/gl_vanishing.cuh"
using namespace gl;

extern "C" uint64_t emu_stark_check_rows(const uint64_t* trace, const uint64_t* aux, uint32_t log_n,
                                         const gl_stark_instr* prog, uint32_t n_instr, const uint64_t* consts,
                                         uint32_t* counts, uint32_t* pairs) {
    StarkRowsParams p{trace, aux, log_n, prog, n_instr, consts};
    std::vector<uint64_t> v(GL_STARK_MAX_INSTR, 0xDEADBEEFDEADBEEFull);  // uninitialised on the device
    uint64_t total = 0;
    for (size_t i = 0; i < ((size_t)1 << log_n); i++) {
        counts[i] = stark_check_row(p, i, v.data(), pairs ? pairs + 2 * total : nullptr);
        total += counts[i];
    }
    return total;
}

extern "C" uint64_t emu_plonk_check_rows(const uint64_t* const* values, uint32_t n_commits, uint32_t log_n,
                                         const gl_vp_instr* prog, uint32_t n_instr, const uint64_t* consts,
                                         uint32_t* counts, uint32_t* pairs) {
    const size_t n = (size_t)1 << log_n;
    const size_t tcnt = 4096 > (n >> 12) + 1 ? 4096 : (n >> 12) + 1;  // x_pow_tables in plonky2_b200.cu
    std::vector<uint64_t> xhi(tcnt), xlo(tcnt);
    const uint64_t w = root_of_unity(log_n), whi = gl::pow(w, 4096);
    uint64_t a = 1, b = 1;
    for (size_t k = 0; k < tcnt; k++, a = mul(a, whi), b = mul(b, w)) {
        xhi[k] = canon(a);
        xlo[k] = canon(b);
    }
    VpRowsParams p{};
    for (uint32_t c = 0; c < n_commits && c < GL_VP_MAX_COMMITS; c++) p.val[c] = values[c];
    p.log_n = log_n;
    p.prog = prog;
    p.n_instr = n_instr;
    p.consts = consts;
    p.xhi = xhi.data();
    p.xlo = xlo.data();
    std::vector<uint64_t> regs(GL_VP_MAX_REGS, 0xDEADBEEFDEADBEEFull);
    uint64_t total = 0;
    for (size_t i = 0; i < n; i++) {
        counts[i] = vp_check_row(p, i, regs.data(), pairs ? pairs + 2 * total : nullptr);
        total += counts[i];
    }
    return total;
}
