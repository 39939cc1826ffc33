// gl_stark_rows.cuh -- one row of starky's check_constraints (starky/src/prover.rs:670-820): every constraint of a
// STARK's program on one row i of the trace subgroup H = <w_n>, at x = w_n^i, with no coset shift.
//
// The reference evaluates the whole ConstraintConsumer fold on every row and asserts that it is zero (prover.rs:805-818).
// Here each GL_STARK_EMIT is checked on its own, so a failing row names the constraints that fail. The filters are the
// reference's values on H (prover.rs:707-712,731-735): z_last = x - w_n^-1 is zero exactly at row n - 1, lagrange_first
// is [i = 0], lagrange_last [i = n - 1]; a filtered value is nonzero iff the value and the filter are, so the filters are
// these predicates and no product is formed.
//
// Part g of G = 2^part_log of H is the rows i = g + G*j, j < M = n / G: the coset w_n^g <w_M>. A part's values are a
// size-M NTT of the folded coefficients (gl_check_rows_host.cuh), so each part is checked on its own; the whole of H is
// part 0 of 1.
//
// The same source runs on the host in tests/emu/check_rows_emu.cpp and tests/emu/check_rows_parts_emu.cpp (threads as a
// loop).
#pragma once
#include "../../include/plonky2_b200.h"
#include "gl_field.cuh"

namespace gl {

struct StarkRowsParams {
    const uint64_t* trace;   // trace values on the part, column k at trace + k*M, local row j at + j
    const uint64_t* aux;     // auxiliary values on the part, same layout (NULL: the program reads none)
    uint32_t log_n;
    const gl_stark_instr* prog;  // validated by the caller
    uint32_t n_instr;
    const uint64_t* consts;
    // Part addressing; the defaults are the whole of H, part 0 of 1. Local row j is global row i = part + (j << part_log).
    uint32_t part_log = 0;
    size_t part = 0;
    // The next rows i + 1, same layout (NULL: read at local row (j + 1) mod M of trace / aux, the whole of H's case)
    const uint64_t* trace_next = nullptr;
    const uint64_t* aux_next = nullptr;
};

// The number of GL_STARK_EMITs that fail at local row j of the part, global row i. With pairs != NULL, failure m is also
// written as the pair (row i, the EMIT's ordinal in the program) at pairs[2m], pairs[2m + 1], in program order.
// v: GL_STARK_MAX_INSTR words of scratch.
GL_HD uint32_t stark_check_row(const StarkRowsParams& p, size_t j, uint64_t* v, uint32_t* pairs) {
    const size_t n = (size_t)1 << p.log_n;
    const uint32_t log_M = p.log_n - p.part_log;
    const size_t i = p.part + (j << p.part_log);
    const size_t jn = (j + 1) & (((size_t)1 << log_M) - 1);
    const bool first = i == 0, last = i == n - 1;
    uint32_t fails = 0, emit = 0;
    for (uint32_t k = 0; k < p.n_instr; k++) {
        const gl_stark_instr ins = p.prog[k];
        uint64_t r = 0;
        switch (ins.op) {
            case GL_STARK_LOCAL: r = p.trace[((size_t)ins.a << log_M) + j]; break;
            case GL_STARK_NEXT:
                r = p.trace_next ? p.trace_next[((size_t)ins.a << log_M) + j] : p.trace[((size_t)ins.a << log_M) + jn];
                break;
            case GL_STARK_AUX_LOCAL: r = p.aux[((size_t)ins.a << log_M) + j]; break;
            case GL_STARK_AUX_NEXT:
                r = p.aux_next ? p.aux_next[((size_t)ins.a << log_M) + j] : p.aux[((size_t)ins.a << log_M) + jn];
                break;
            case GL_STARK_CONST: r = p.consts[ins.a]; break;
            case GL_STARK_ADD: r = add(v[ins.a], v[ins.b]); break;
            case GL_STARK_SUB: r = sub(v[ins.a], v[ins.b]); break;
            case GL_STARK_MUL: r = mul(v[ins.a], v[ins.b]); break;
            default: {  // GL_STARK_EMIT
                const bool on = ins.b == GL_STARK_CONSTRAINT || (ins.b == GL_STARK_TRANSITION && !last) ||
                                (ins.b == GL_STARK_FIRST_ROW && first) || (ins.b == GL_STARK_LAST_ROW && last);
                if (on && canon(v[ins.a]) != 0) {
                    if (pairs) {
                        pairs[2 * fails] = (uint32_t)i;
                        pairs[2 * fails + 1] = emit;
                    }
                    fails++;
                }
                emit++;
            }
        }
        v[k] = r;
    }
    return fails;
}

}  // namespace gl
