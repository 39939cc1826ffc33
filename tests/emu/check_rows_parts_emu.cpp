// Host run of the row checks of gl_stark_check_rows_part (plonky2_b200/csrc/gl_stark_rows.cuh) and
// gl_plonk_check_rows_part (gl_vanishing.cuh) on one part of H: the same stark_check_row / vp_check_row the kernels call
// per thread, with threads as a loop over the part's M = n >> part_log local rows and host arrays in place of device
// memory. Test infrastructure: built as a shared library and driven by tests/test_check_constraints_parts.py against an
// exact evaluator of the programs on the whole of H.
//
// The values are the part's (column k at + k*M, local row j); a *_next array (or entry) holds the values on the next
// rows, and NULL reads them from the local values at (j + 1) mod M. Both functions write every local row's failure
// count to counts[j] and, when pairs is not NULL, every failure as a (global row, index) pair, rows in order (pairs must
// hold 2 x the total). Both return the total.
#include <vector>
#include "../../plonky2_b200/csrc/gl_stark_rows.cuh"
#include "../../plonky2_b200/csrc/gl_vanishing.cuh"
using namespace gl;

extern "C" uint64_t emu_stark_check_rows_part(const uint64_t* trace, const uint64_t* trace_next, const uint64_t* aux,
                                              const uint64_t* aux_next, uint32_t log_n, uint32_t part,
                                              uint32_t part_log, const gl_stark_instr* prog, uint32_t n_instr,
                                              const uint64_t* consts, uint32_t* counts, uint32_t* pairs) {
    StarkRowsParams p{trace, aux, log_n, prog, n_instr, consts};
    p.part_log = part_log;
    p.part = part;
    p.trace_next = trace_next;
    p.aux_next = aux_next;
    std::vector<uint64_t> v(GL_STARK_MAX_INSTR, 0xDEADBEEFDEADBEEFull);  // uninitialised on the device
    uint64_t total = 0;
    for (size_t j = 0; j < ((size_t)1 << (log_n - part_log)); j++) {
        counts[j] = stark_check_row(p, j, v.data(), pairs ? pairs + 2 * total : nullptr);
        total += counts[j];
    }
    return total;
}

extern "C" uint64_t emu_plonk_check_rows_part(const uint64_t* const* values, const uint64_t* const* nexts,
                                              uint32_t n_commits, uint32_t log_n, uint32_t part, uint32_t part_log,
                                              const gl_vp_instr* prog, uint32_t n_instr, const uint64_t* consts,
                                              uint32_t* counts, uint32_t* pairs) {
    const size_t n = (size_t)1 << log_n;
    const size_t tcnt = 4096 > (n >> 12) + 1 ? 4096 : (n >> 12) + 1;  // x_pow_tables in plonky2_b200.cu: n-sized
    std::vector<uint64_t> xhi(tcnt), xlo(tcnt);
    const uint64_t w = root_of_unity(log_n), whi = gl::pow(w, 4096);
    uint64_t a = 1, b = 1;
    for (size_t k = 0; k < tcnt; k++, a = mul(a, whi), b = mul(b, w)) {
        xhi[k] = canon(a);
        xlo[k] = canon(b);
    }
    VpRowsParams p{};
    for (uint32_t c = 0; c < n_commits && c < GL_VP_MAX_COMMITS; c++) {
        p.val[c] = values[c];
        p.val_next[c] = nexts ? nexts[c] : nullptr;
    }
    p.log_n = log_n;
    p.prog = prog;
    p.n_instr = n_instr;
    p.consts = consts;
    p.xhi = xhi.data();
    p.xlo = xlo.data();
    p.part_log = part_log;
    p.part = part;
    std::vector<uint64_t> regs(GL_VP_MAX_REGS, 0xDEADBEEFDEADBEEFull);
    uint64_t total = 0;
    for (size_t j = 0; j < (n >> part_log); j++) {
        counts[j] = vp_check_row(p, j, regs.data(), pairs ? pairs + 2 * total : nullptr);
        total += counts[j];
    }
    return total;
}
