// Host run of the device evaluator of plonky2's vanishing polynomial (plonky2_b200/csrc/gl_vanishing.cuh) on ONE SHARD of
// the quotient coset: the same vp_eval_point that k_plonk_quotient calls per thread, with the shard addressing that
// gl_plonk_quotient_shard (plonky2_b200.cu) sets up. Test infrastructure: built as a shared library and driven by
// tests/test_plonk_sharded.py, which hands in each shard's local and next-row buffers and compares the placed shards with
// the whole-coset run of tests/emu/vanishing_emu.cpp.
#include <vector>
#include "../../plonky2_b200/csrc/gl_vanishing.cuh"
using namespace gl;

// Shard g = shard_index of G = 2^shard_log: out = n_alphas columns of M = size >> shard_log values, local natural order.
// loc[c] / loc_stride[c]: commitment c's values at the shard's leaf rows g*M + j (or its whole LDE when the local values
// are read in place on one device); nxt[c] / nxt_stride[c]: its values at x * w_n in leaf order j, used when the next row
// lies in another shard (shard_log > qd_bits; NULL for commitments the program does not read there).
// Returns 1 if the program divided by zero.
extern "C" int emu_plonk_quotient_shard_values(const uint64_t* const* loc, const size_t* loc_stride,
                                               const uint64_t* const* nxt, const size_t* nxt_stride, uint32_t n_commits,
                                               uint32_t rate_bits, uint32_t degree_bits, uint32_t qd_bits,
                                               uint32_t shard_index, uint32_t shard_log, const gl_vp_instr* prog,
                                               uint32_t n_instr, const uint64_t* consts, const uint64_t* alphas,
                                               uint32_t n_alphas, uint32_t n_terms, uint64_t* out) {
    const uint32_t size_log = degree_bits + qd_bits, log_M = size_log - shard_log;
    const size_t size = (size_t)1 << size_log, M = (size_t)1 << log_M;
    std::vector<uint64_t> apow((size_t)n_alphas * n_terms);
    for (uint32_t a = 0; a < n_alphas; a++) {
        uint64_t pw = 1;
        for (uint32_t t = 0; t < n_terms; t++, pw = mul(pw, alphas[a])) apow[(size_t)a * n_terms + t] = canon(pw);
    }
    const uint64_t ws = root_of_unity(size_log);
    const size_t tcnt = 4096 > (size >> 12) + 1 ? 4096 : (size >> 12) + 1;
    std::vector<uint64_t> xhi(tcnt), xlo(tcnt);
    {
        const uint64_t whi = gl::pow(ws, 4096);
        uint64_t a = 1, b = 1;
        for (size_t k = 0; k < tcnt; k++, a = mul(a, whi), b = mul(b, ws)) {
            xhi[k] = canon(a);
            xlo[k] = canon(b);
        }
    }
    VanishingParams p;
    for (uint32_t c = 0; c < GL_VP_MAX_COMMITS; c++) {
        p.lde[c] = c < n_commits ? loc[c] : nullptr;
        p.lde_stride[c] = c < n_commits ? loc_stride[c] : 0;
        p.nxt[c] = c < n_commits ? nxt[c] : nullptr;
        p.nxt_stride[c] = c < n_commits ? nxt_stride[c] : 0;
    }
    p.log_N = degree_bits + rate_bits;
    p.degree_bits = degree_bits;
    p.qd_bits = qd_bits;
    p.prog = prog;
    p.n_instr = n_instr;
    p.consts = consts;
    p.apow = apow.data();
    p.n_alphas = n_alphas;
    p.n_terms = n_terms;
    p.xhi = xhi.data();
    p.xlo = xlo.data();
    p.shift = MULTIPLICATIVE_GROUP_GENERATOR;
    p.n_field = canon((uint64_t)1 << degree_bits);
    uint64_t g_pow_n = MULTIPLICATIVE_GROUP_GENERATOR;
    for (uint32_t k = 0; k < degree_bits; k++) g_pow_n = sqr(g_pow_n);
    const uint64_t wq = root_of_unity(qd_bits);
    uint64_t xq = 1;
    for (uint32_t j = 0; j < GL_VP_MAX_QD; j++) p.zh[j] = p.zh_inv[j] = 0;
    for (uint32_t j = 0; j < (1u << qd_bits); j++, xq = mul(xq, wq)) {
        p.zh[j] = canon(sub(mul(g_pow_n, xq), 1));
        p.zh_inv[j] = canon(gl::inv(p.zh[j]));
    }
    p.out = out;
    p.flag = nullptr;
    p.row0 = (size_t)shard_index << log_M;
    p.shard_log = shard_log;
    p.next_in_shard = shard_log <= qd_bits;
    int bad = 0;
    for (size_t j = 0; j < M; j++) {  // one "thread" per local leaf row
        uint64_t regs[GL_VP_MAX_REGS];
        for (int k = 0; k < GL_VP_MAX_REGS; k++) regs[k] = 0xDEADBEEFDEADBEEFull;  // uninitialised on the device
        if (!vp_eval_point(p, j, regs)) bad = 1;
    }
    return bad;
}
