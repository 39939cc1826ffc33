// gl_vanishing.cuh -- one point of plonky2's quotient: eval_vanishing_poly_base_batch
// (plonky2/src/plonk/vanishing_poly.rs:167-340) followed by the division by Z_H (plonk/prover.rs:795-803).
//
// The reference walks the gates' evaluators and the permutation argument point by point on the host, reading every
// commitment's LDE row through get_lde_values. Here the whole vanishing polynomial of a circuit (gate constraints with
// their selector filters, L_0(x)(Z(x) - 1), the partial-product checks) is recorded ONCE on the host as a register
// program and every thread interprets it for its point, reading the LDE columns of up to four commitments in place.
// The instruction stream is uniform across the warp (one broadcast load per instruction); the registers are a
// per-thread array the compiler keeps in local memory, so gates of any size fit without a new kernel.
//
// The same source runs on the host in tests/emu/vanishing_emu.cpp (threads as a loop) against the oracle, and the
// row check below in tests/emu/check_rows_emu.cpp and tests/emu/check_rows_parts_emu.cpp.
#pragma once
#include "../../include/plonky2_b200.h"
#include "gl_field.cuh"

namespace gl {

struct VanishingParams {
    const uint64_t* lde[GL_VP_MAX_COMMITS];  // LDE of commitment c, column k at lde[c] + k*lde_stride[c], leaf order
    size_t lde_stride[GL_VP_MAX_COMMITS];
    uint32_t log_N;                   // log2 of the LDE size (degree_bits + rate_bits)
    uint32_t degree_bits, qd_bits;    // the quotient coset has n << qd_bits points
    const gl_vp_instr* prog;
    uint32_t n_instr;
    const uint64_t* consts;
    const uint64_t* apow;             // apow[k*n_terms + t] = alpha_k^t  (reduce_with_powers_multi, plonk_common.rs:99-116)
    uint32_t n_alphas, n_terms;
    const uint64_t *xhi, *xlo;        // w_size^i = xhi[i >> 12] * xlo[i & 4095]
    uint64_t shift;                   // F::coset_shift()
    uint64_t n_field;                 // n as a field element
    uint64_t zh[GL_VP_MAX_QD], zh_inv[GL_VP_MAX_QD];  // ZeroPolyOnCoset (field/src/zero_poly_coset.rs:20-61)
    uint64_t* out;                    // n_alphas columns of M = size >> shard_log values, local natural order
    unsigned int* flag;               // bit 0: L_0 asked for at x = 1 ("Tried to invert zero")
    // Shard addressing (gl_plonk_quotient_shard); the defaults are the whole coset, shard 0 of 1. Shard g of
    // G = 2^shard_log owns the quotient-coset leaf rows row0 + j (row0 = g*M, j < M), i.e. the points
    // i = bitrev(g) + G*bitrev_M(j); lde[c] then holds those rows at j.
    size_t row0 = 0;
    uint32_t shard_log = 0;
    bool next_in_shard = true;        // the next point's leaf row is in this shard: lde[c] at its row - row0
    const uint64_t* nxt[GL_VP_MAX_COMMITS] = {};  // else the values at x*w_n, leaf order j, column k at + k*nxt_stride
    size_t nxt_stride[GL_VP_MAX_COMMITS] = {};
};

GL_HD size_t vp_bitrev(size_t x, uint32_t bits) {
#if defined(__CUDA_ARCH__)
    return bits ? (size_t)(__brevll((unsigned long long)x) >> (64 - bits)) : 0;
#else
    size_t r = 0;
    for (uint32_t i = 0; i < bits; i++) r |= ((x >> i) & 1u) << (bits - 1 - i);
    return r;
#endif
}

// One point of the coset g*<w_size>, addressed by its LEAF ROW j: the rows get_lde_values(i, step) touches are
// bitrev(i * step) = bitrev_{size_log}(i), i.e. exactly the first `size` leaf rows, so thread j takes point
// i = bitrev_{size_log}(j): every LDE load of a warp is one contiguous 256-byte segment of a column, and only the
// n_alphas result stores (and the few Z(g x) loads) are scattered. Returns false if the program divided by zero.
// regs: GL_VP_MAX_REGS words of scratch. On a shard, j is the local leaf row (p.row0 + j globally); x, Z_H and L_0
// still come from the global point i.
GL_HD bool vp_eval_point(const VanishingParams& p, size_t j, uint64_t* regs) {
    const uint32_t size_log = p.degree_bits + p.qd_bits;
    const size_t size = (size_t)1 << size_log;
    const size_t i = vp_bitrev(p.row0 + j, size_log);
    const size_t inext = (i + ((size_t)1 << p.qd_bits)) & (size - 1);  // next_step = 2^quotient_degree_bits, prover.rs:643
    // get_lde_values(i, step) with step = 2^(rate_bits - quotient_degree_bits) (prover.rs:640, fri/oracle.rs:142-147):
    // leaf row bitrev_{log_N}(i * step) = bitrev_{size_log}(i)
    const size_t jl = j;
    const size_t jn = p.next_in_shard ? vp_bitrev(inext, size_log) - p.row0 : j;
    const uint32_t qmask = (1u << p.qd_bits) - 1;
    const uint64_t x = mul(p.shift, mul(p.xhi[i >> 12], p.xlo[i & 4095]));
    uint64_t acc[GL_VP_MAX_ALPHAS];
#pragma unroll
    for (int a = 0; a < GL_VP_MAX_ALPHAS; a++) acc[a] = 0;
    bool ok = true;
    for (uint32_t k = 0; k < p.n_instr; k++) {
        const gl_vp_instr in = p.prog[k];
        uint64_t r;
        switch (in.op) {
            case GL_VP_LOCAL: r = p.lde[in.a][(size_t)in.b * p.lde_stride[in.a] + jl]; break;
            case GL_VP_NEXT:
                r = p.next_in_shard ? p.lde[in.a][(size_t)in.b * p.lde_stride[in.a] + jn]
                                    : p.nxt[in.a][(size_t)in.b * p.nxt_stride[in.a] + jn];
                break;
            case GL_VP_CONST: r = p.consts[(uint32_t)in.a | ((uint32_t)in.b << 16)]; break;
            case GL_VP_X: r = x; break;
            case GL_VP_L0: {  // eval_l_0: Z_H(x) / (n (x - 1)), zero_poly_coset.rs:58-61
                const uint64_t den = mul(p.n_field, sub(x, 1));
                if (canon(den) == 0) ok = false;
                r = mul(p.zh[i & qmask], inv(den));
                break;
            }
            case GL_VP_ADD: r = add(regs[in.a], regs[in.b]); break;
            case GL_VP_SUB: r = sub(regs[in.a], regs[in.b]); break;
            case GL_VP_MUL: r = mul(regs[in.a], regs[in.b]); break;
            case GL_VP_ADDC: r = add(regs[in.a], p.consts[in.b]); break;
            case GL_VP_MULC: r = mul(regs[in.a], p.consts[in.b]); break;
            default: {  // GL_VP_TERM: vanishing term number b
                const uint64_t t = regs[in.a];
                for (uint32_t a = 0; a < p.n_alphas; a++) acc[a] = add(acc[a], mul(t, p.apow[(size_t)a * p.n_terms + in.b]));
                continue;
            }
        }
        regs[in.dst] = r;
    }
    const uint64_t zi = p.zh_inv[i & qmask];  // eval_inverse(i), prover.rs:796-802
    const uint32_t log_M = size_log - p.shard_log;  // i = bitrev(g) + G*k: local point k = i >> shard_log
    for (uint32_t a = 0; a < p.n_alphas; a++) p.out[((size_t)a << log_M) + (i >> p.shard_log)] = canon(mul(acc[a], zi));
    return ok;
}

// The same program checked on one row i of the trace subgroup H = <w_n>, at x = w_n^i with no coset shift
// (gl_plonk_check_rows): every GL_VP_TERM on its own, without alphas or Z_H. On H, L_0 is the indicator [i = 0] (its
// closed form above divides by zero at x = 1), and only the row's own gate has a nonzero selector filter, so a failing
// gate-constraint term at row i is a constraint of the gate placed at row i.
// Part g of G = 2^part_log of H is the rows i = g + G*j (gl_stark_rows.cuh); the whole of H is part 0 of 1.
struct VpRowsParams {
    const uint64_t* val[GL_VP_MAX_COMMITS];  // commitment c's values on the part, column k at val[c] + k*M, local row j
    uint32_t log_n;
    const gl_vp_instr* prog;          // validated by the caller
    uint32_t n_instr;
    const uint64_t* consts;
    const uint64_t *xhi, *xlo;        // w_n^i = xhi[i >> 12] * xlo[i & 4095]
    // Part addressing; the defaults are the whole of H, part 0 of 1. Local row j is global row i = part + (j << part_log).
    uint32_t part_log = 0;
    size_t part = 0;
    // commitment c's values at the next rows i + 1, same layout (NULL: read at local row (j + 1) mod M of val[c])
    const uint64_t* val_next[GL_VP_MAX_COMMITS] = {};
};

// The number of GL_VP_TERMs whose value is nonzero at local row j of the part, global row i. With pairs != NULL,
// failure m is also written as the pair (row i, the term number b) at pairs[2m], pairs[2m + 1], in program order.
// regs: GL_VP_MAX_REGS words of scratch.
GL_HD uint32_t vp_check_row(const VpRowsParams& p, size_t j, uint64_t* regs, uint32_t* pairs) {
    const uint32_t log_M = p.log_n - p.part_log;
    const size_t i = p.part + (j << p.part_log);
    const size_t jn = (j + 1) & (((size_t)1 << log_M) - 1);
    uint32_t fails = 0;
    for (uint32_t k = 0; k < p.n_instr; k++) {
        const gl_vp_instr ins = p.prog[k];
        uint64_t r;
        switch (ins.op) {
            case GL_VP_LOCAL: r = p.val[ins.a][((size_t)ins.b << log_M) + j]; break;
            case GL_VP_NEXT:
                r = p.val_next[ins.a] ? p.val_next[ins.a][((size_t)ins.b << log_M) + j]
                                      : p.val[ins.a][((size_t)ins.b << log_M) + jn];
                break;
            case GL_VP_CONST: r = p.consts[(uint32_t)ins.a | ((uint32_t)ins.b << 16)]; break;
            case GL_VP_X: r = mul(p.xhi[i >> 12], p.xlo[i & 4095]); break;
            case GL_VP_L0: r = i == 0; break;
            case GL_VP_ADD: r = add(regs[ins.a], regs[ins.b]); break;
            case GL_VP_SUB: r = sub(regs[ins.a], regs[ins.b]); break;
            case GL_VP_MUL: r = mul(regs[ins.a], regs[ins.b]); break;
            case GL_VP_ADDC: r = add(regs[ins.a], p.consts[ins.b]); break;
            case GL_VP_MULC: r = mul(regs[ins.a], p.consts[ins.b]); break;
            default:  // GL_VP_TERM
                if (canon(regs[ins.a]) != 0) {
                    if (pairs) {
                        pairs[2 * fails] = (uint32_t)i;
                        pairs[2 * fails + 1] = ins.b;
                    }
                    fails++;
                }
                continue;
        }
        regs[ins.dst] = r;
    }
    return fails;
}

}  // namespace gl
