// gl_check_rows_host.cuh -- kernels and host orchestration of check_constraints (starky/src/prover.rs:670-820) and its
// plonky2 counterpart: gl_stark_check_rows and gl_plonk_check_rows of include/plonky2_b200_check.h. Included at the end
// of plonky2_b200.cu, whose helpers it uses (set_err, DevBuf, upload_program, ntt_natural, x_pow_tables, and the program
// checks stark_program_check / vp_program_check it shares with the quotient entry points). The row arithmetic is
// gl_stark_rows.cuh and vp_check_row in gl_vanishing.cuh.
#pragma once
#include "../../include/plonky2_b200_check.h"

// ---- check_constraints (starky/src/prover.rs:670-820) and its plonky2 counterpart: one thread per row i of H, the row's
// arithmetic is gl_stark_rows.cuh / gl_vanishing.cuh. Two passes of one kernel (check_rows_report): without pairs, the
// row's failure count to off[i]; with pairs, the rows whose exclusive offset off[i] is below max_report write their
// failures at pairs + 2*off[i].
__global__ void __launch_bounds__(128) k_stark_check_rows(StarkRowsParams p, u64* off, uint32_t* pairs, u64 max_report) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ((size_t)1 << p.log_n)) return;
    u64 v[GL_STARK_MAX_INSTR];
    if (!pairs) {
        off[i] = stark_check_row(p, i, v, nullptr);
        return;
    }
    if (off[i] >= max_report || off[i + 1] == off[i]) return;
    stark_check_row(p, i, v, pairs + 2 * off[i]);
}
__global__ void __launch_bounds__(128) k_plonk_check_rows(VpRowsParams p, u64* off, uint32_t* pairs, u64 max_report) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ((size_t)1 << p.log_n)) return;
    u64 regs[GL_VP_MAX_REGS];
    if (!pairs) {
        off[i] = vp_check_row(p, i, regs, nullptr);
        return;
    }
    if (off[i] >= max_report || off[i + 1] == off[i]) return;
    vp_check_row(p, i, regs, pairs + 2 * off[i]);
}

// ---- gl_stark_check_rows / gl_plonk_check_rows: every constraint on every row of H
constexpr uint32_t CHECK_MAX_REPORT = 65536;
// The checks both entry points share for one commitment: on this context, finished, of the first one's degree
static int check_rows_commit(gl_ctx* ctx, const gl_commit* c, const gl_commit* first, const char* what) {
    if (c->ctx != ctx) return set_err(ctx, GL_ERR_BAD_ARG, "the %s commitment belongs to another context", what);
    if (!c->finished) return set_err(ctx, GL_ERR_BAD_ARG, "gl_commit_finish has not been called on the %s commitment", what);
    if (c->degree_log != first->degree_log)
        return set_err(ctx, GL_ERR_BAD_SHAPE, "the %s commitment's degree 2^%u differs from 2^%u", what, c->degree_log,
                       first->degree_log);
    return GL_OK;
}
// c's values on H in natural order, from its coefficients: B columns of n words in `buf`. The coefficients exist on
// every kind of handle (resident, non-resident, a shard's replicated copy, salted), so the check reads them alone.
static int values_on_h(gl_ctx* ctx, const gl_commit* c, DevBuf& buf) {
    const size_t n = (size_t)1 << c->degree_log;
    TRY(buf.alloc((size_t)c->B * n));
    return ntt_natural(ctx, c->coeffs, n, buf.get(), n, (int)c->degree_log, c->B, false, 1);
}
// The two passes of a row kernel over the 2^log_n rows, and the report: the total number of failing (row, index) pairs
// and the first max_report of them in (row, index) order. launch(off, pairs) queues one pass (check_rows kernels).
// Every row whose offset is below max_report writes all of its failures (at most max_per_row, in program order), so
// after sorting the slots the one row that straddles max_report is complete; unwritten slots are all ones and sort last.
static int check_rows_report(gl_ctx* ctx, uint32_t log_n, uint32_t max_per_row, uint32_t max_report,
                             const std::function<int(u64*, uint32_t*)>& launch, uint64_t* out_failures,
                             uint32_t* out_pairs, uint32_t* out_reported) {
    const size_t n = (size_t)1 << log_n;
    DevBuf off(ctx), temp(ctx), dpairs(ctx);
    TRY(off.alloc(n + 1));  // per-row counts, then their exclusive scan; off[n] = the total
    CK(ctx, cudaMemsetAsync(off.get() + n, 0, 8, ctx->stream));
    TRY(launch(off.get(), nullptr));
    size_t temp_bytes = 0;
    CK(ctx, cub::DeviceScan::ExclusiveSum(nullptr, temp_bytes, off.get(), off.get(), (int)(n + 1), ctx->stream));
    TRY(temp.alloc((temp_bytes + 7) / 8));
    CK(ctx, cub::DeviceScan::ExclusiveSum(temp.get(), temp_bytes, off.get(), off.get(), (int)(n + 1), ctx->stream));
    CKL(ctx);
    temp.reset();
    u64 total = 0;
    TRY(d2h(ctx, &total, off.get() + n, 1));
    const uint32_t reported = total < max_report ? (uint32_t)total : max_report;
    if (reported) {
        const size_t slots = (size_t)std::min<u64>(total, (u64)max_report + max_per_row);  // one pair per word
        TRY(dpairs.alloc(slots));
        CK(ctx, cudaMemsetAsync(dpairs.get(), 0xFF, slots * 8, ctx->stream));
        TRY(launch(off.get(), (uint32_t*)dpairs.get()));
        std::vector<u64> h(slots);
        TRY(d2h(ctx, h.data(), dpairs.get(), slots));
        std::vector<std::pair<uint32_t, uint32_t>> pairs(slots);
        for (size_t s = 0; s < slots; s++) pairs[s] = {(uint32_t)h[s], (uint32_t)(h[s] >> 32)};  // (row, index)
        std::sort(pairs.begin(), pairs.end());
        for (uint32_t s = 0; s < reported; s++) {
            out_pairs[2 * s] = pairs[s].first;
            out_pairs[2 * s + 1] = pairs[s].second;
        }
    }
    *out_failures = total;
    *out_reported = reported;
    return GL_OK;
}
int gl_stark_check_rows(gl_ctx* ctx, gl_commit* trace, gl_commit* aux, const gl_stark_instr* program, uint32_t n_instr,
                        const uint64_t* consts, uint32_t n_consts, uint32_t max_report, uint64_t* out_failures,
                        uint32_t* out_pairs, uint32_t* out_reported) {
    if (!ctx || !trace || !program || (n_consts && !consts) || !out_failures || !out_reported || (max_report && !out_pairs))
        return set_err(ctx, GL_ERR_BAD_ARG, "null argument");
    if (n_instr == 0 || n_instr > GL_STARK_MAX_INSTR) return set_err(ctx, GL_ERR_UNSUPPORTED, "program of %u instructions (max %d)", n_instr, GL_STARK_MAX_INSTR);
    if (max_report > CHECK_MAX_REPORT) return set_err(ctx, GL_ERR_BAD_ARG, "max_report %u > %u", max_report, CHECK_MAX_REPORT);
    TRY(check_rows_commit(ctx, trace, trace, "trace"));
    if (aux) TRY(check_rows_commit(ctx, aux, trace, "auxiliary"));
    uint32_t n_emit = 0;
    TRY(stark_program_check(ctx, program, n_instr, trace, aux, n_consts, &n_emit));
    CK(ctx, cudaSetDevice(ctx->device));
    const uint32_t log_n = trace->degree_log;
    DevBuf tv(ctx), av(ctx), dprog(ctx), dconst(ctx);
    TRY(values_on_h(ctx, trace, tv));
    if (aux) TRY(values_on_h(ctx, aux, av));
    TRY(upload_program(ctx, program, (size_t)n_instr * sizeof(gl_stark_instr), consts, n_consts, dprog, dconst));
    const StarkRowsParams p{tv.get(), av.get(), log_n, (const gl_stark_instr*)dprog.get(), n_instr, dconst.get()};
    const size_t n = (size_t)1 << log_n;
    return check_rows_report(ctx, log_n, n_emit, max_report, [&](u64* off, uint32_t* pairs) {
        k_stark_check_rows<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(p, off, pairs, max_report);
        CKL(ctx);
        return GL_OK;
    }, out_failures, out_pairs, out_reported);
}
int gl_plonk_check_rows(gl_ctx* ctx, gl_commit* const* commits, uint32_t n_commits, const gl_vp_instr* program,
                        uint32_t n_instr, const uint64_t* consts, uint32_t n_consts, uint32_t n_terms,
                        uint32_t max_report, uint64_t* out_failures, uint32_t* out_pairs, uint32_t* out_reported) {
    if (!ctx || !commits || !program || (n_consts && !consts) || !out_failures || !out_reported || (max_report && !out_pairs))
        return set_err(ctx, GL_ERR_BAD_ARG, "null argument");
    if (n_commits == 0 || n_commits > GL_VP_MAX_COMMITS) return set_err(ctx, GL_ERR_UNSUPPORTED, "1..%d commitments", GL_VP_MAX_COMMITS);
    if (n_instr == 0) return set_err(ctx, GL_ERR_BAD_ARG, "empty program");
    if (n_terms == 0 || n_terms > 65536) return set_err(ctx, GL_ERR_BAD_ARG, "1..65536 vanishing terms");
    if (max_report > CHECK_MAX_REPORT) return set_err(ctx, GL_ERR_BAD_ARG, "max_report %u > %u", max_report, CHECK_MAX_REPORT);
    for (uint32_t c = 0; c < n_commits; c++) {
        if (!commits[c]) return set_err(ctx, GL_ERR_BAD_ARG, "null commitment");
        char what[32];
        snprintf(what, sizeof(what), "number %u", c);
        TRY(check_rows_commit(ctx, commits[c], commits[0], what));
    }
    uint32_t next_mask = 0, n_term = 0;
    TRY(vp_program_check(ctx, commits, n_commits, program, n_instr, n_consts, n_terms, false, &next_mask, &n_term));
    CK(ctx, cudaSetDevice(ctx->device));
    const uint32_t log_n = commits[0]->degree_log;
    const size_t n = (size_t)1 << log_n;
    std::vector<DevBuf> vals;
    vals.reserve(n_commits);
    VpRowsParams p{};
    for (uint32_t c = 0; c < n_commits; c++) {
        vals.emplace_back(ctx);
        TRY(values_on_h(ctx, commits[c], vals.back()));
        p.val[c] = vals.back().get();
    }
    DevBuf dprog(ctx), dconst(ctx), xtab(ctx);
    TRY(upload_program(ctx, program, (size_t)n_instr * sizeof(gl_vp_instr), consts, n_consts, dprog, dconst));
    TRY(x_pow_tables(ctx, root_of_unity(log_n), n, xtab));
    p.log_n = log_n;
    p.prog = (const gl_vp_instr*)dprog.get();
    p.n_instr = n_instr;
    p.consts = dconst.get();
    p.xhi = xtab.get();
    p.xlo = xtab.get() + x_pow_table_len(n);
    return check_rows_report(ctx, log_n, n_term, max_report, [&](u64* off, uint32_t* pairs) {
        k_plonk_check_rows<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(p, off, pairs, max_report);
        CKL(ctx);
        return GL_OK;
    }, out_failures, out_pairs, out_reported);
}
