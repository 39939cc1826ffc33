// gl_check_rows_host.cuh -- kernels and host orchestration of check_constraints (starky/src/prover.rs:670-820) and its
// plonky2 counterpart: gl_stark_check_rows[_part] and gl_plonk_check_rows[_part] of include/plonky2_b200_check.h.
// Included at the end of plonky2_b200.cu, whose helpers it uses (set_err, DevBuf, upload_program, ntt_natural,
// k_fold_coeffs, x_pow_tables, and the program checks stark_program_check / vp_program_check it shares with the quotient
// entry points). The row arithmetic is gl_stark_rows.cuh and vp_check_row in gl_vanishing.cuh.
#pragma once
#include "../../include/plonky2_b200_check.h"

// ---- check_constraints (starky/src/prover.rs:670-820) and its plonky2 counterpart: one thread per local row j of a
// part of H (all of H: part 0 of 1), the row's arithmetic is gl_stark_rows.cuh / gl_vanishing.cuh. Two passes of one
// kernel (check_rows_report): without pairs, the row's failure count to off[j]; with pairs, the rows whose exclusive
// offset off[j] is below max_report write their failures at pairs + 2*off[j].
__global__ void __launch_bounds__(128) k_stark_check_rows(StarkRowsParams p, u64* off, uint32_t* pairs, u64 max_report) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= ((size_t)1 << (p.log_n - p.part_log))) return;
    u64 v[GL_STARK_MAX_INSTR];
    if (!pairs) {
        off[j] = stark_check_row(p, j, v, nullptr);
        return;
    }
    if (off[j] >= max_report || off[j + 1] == off[j]) return;
    stark_check_row(p, j, v, pairs + 2 * off[j]);
}
__global__ void __launch_bounds__(128) k_plonk_check_rows(VpRowsParams p, u64* off, uint32_t* pairs, u64 max_report) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= ((size_t)1 << (p.log_n - p.part_log))) return;
    u64 regs[GL_VP_MAX_REGS];
    if (!pairs) {
        off[j] = vp_check_row(p, j, regs, nullptr);
        return;
    }
    if (off[j] >= max_report || off[j + 1] == off[j]) return;
    vp_check_row(p, j, regs, pairs + 2 * off[j]);
}

// ---- gl_stark_check_rows[_part] / gl_plonk_check_rows[_part]: every constraint on every row of H, or of one part of it
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
// The part refusals of the _part entry points, on H of 2^log_n rows: parts a power of two of at most n, part below it.
// Sets *part_log.
static int check_rows_parts(gl_ctx* ctx, uint32_t log_n, uint32_t part, uint32_t parts, uint32_t* part_log) {
    if (parts == 0 || (parts & (parts - 1)))
        return set_err(ctx, GL_ERR_BAD_SHAPE, "parts %u is not a power of two", parts);
    if ((uint64_t)parts > ((uint64_t)1 << log_n))
        return set_err(ctx, GL_ERR_BAD_SHAPE, "parts %u > the %llu rows of H", parts, (unsigned long long)1 << log_n);
    if (part >= parts) return set_err(ctx, GL_ERR_BAD_ARG, "part %u >= parts %u", part, parts);
    uint32_t s = 0;
    while ((1u << s) < parts) s++;
    *part_log = s;
    return GL_OK;
}
// c's values on the coset w_n^e <w_M> of H, M = n / 2^s, in natural order: B columns of M words in `buf`, the point
// w_n^e w_M^j at j. Part g of 2^s is e = g; its next rows are e = g + 1 (at g = 2^s - 1, w_M <w_M> = <w_M>: row 0).
// The coefficients are folded mod X^M - w_n^(e M) (k_fold_coeffs), then a size-M NTT with shift w_n^e; at s = 0 (all of
// H, e = 0) it is the NTT of the coefficients alone. The coefficients exist on every kind of handle (resident,
// non-resident, a shard's replicated copy, salted), so the check reads them alone.
static int values_on_part(gl_ctx* ctx, const gl_commit* c, size_t e, uint32_t s, DevBuf& buf) {
    const uint32_t log_M = c->degree_log - s;
    const size_t n = (size_t)1 << c->degree_log, M = (size_t)1 << log_M;
    TRY(buf.alloc((size_t)c->B * M));
    if (s == 0) return ntt_natural(ctx, c->coeffs, n, buf.get(), n, (int)c->degree_log, c->B, false, 1);
    const u64 shift = gl::pow(root_of_unity(c->degree_log), e);
    for (uint32_t b0 = 0; b0 < c->B; b0 += MAX_GRID_Y) {
        const uint32_t bc = (c->B - b0 < MAX_GRID_Y) ? c->B - b0 : MAX_GRID_Y;
        k_fold_coeffs<<<dim3((unsigned)((M + 127) / 128), bc), 128, 0, ctx->stream>>>(
            c->coeffs + (size_t)b0 * n, n, n, M, gl::pow(shift, M), buf.get() + (size_t)b0 * M);
        CKL(ctx);
    }
    return ntt_natural(ctx, buf.get(), M, buf.get(), M, (int)log_M, c->B, false, shift);
}
// c's values on part g of 2^s (*local) and, when the program reads c's next row and s > 0, on the next rows (*next;
// else NULL: the kernel reads the next row from the local values)
static int part_views(gl_ctx* ctx, const gl_commit* c, uint32_t g, uint32_t s, bool reads_next, DevBuf& lbuf,
                      DevBuf& nbuf, const u64** local, const u64** next) {
    TRY(values_on_part(ctx, c, g, s, lbuf));
    *local = lbuf.get();
    *next = nullptr;
    if (!reads_next || s == 0) return GL_OK;
    TRY(values_on_part(ctx, c, (size_t)g + 1, s, nbuf));
    *next = nbuf.get();
    return GL_OK;
}
// The two passes of a row kernel over the `rows` rows of a part (or the routed wires of gl_plonk_check_copies, one per
// row), and the report: the total number of failing (row, index) pairs and the first max_report of them in (row, index)
// order. launch(off, pairs) queues one pass (check_rows kernels). Every row whose offset is below max_report writes
// all of its failures (at most max_per_row, in program order), so after sorting the slots the one row that straddles
// max_report is complete; unwritten slots are all ones and sort last. The rows of a part are in global order, so its
// pairs are too.
static int check_rows_report(gl_ctx* ctx, size_t rows, uint32_t max_per_row, uint32_t max_report,
                             const std::function<int(u64*, uint32_t*)>& launch, uint64_t* out_failures,
                             uint32_t* out_pairs, uint32_t* out_reported) {
    const size_t n = rows;
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
// gl_stark_check_rows (part 0 of 1) and gl_stark_check_rows_part
static int stark_check_rows(gl_ctx* ctx, gl_commit* trace, gl_commit* aux, const gl_stark_instr* program,
                            uint32_t n_instr, const uint64_t* consts, uint32_t n_consts, uint32_t part, uint32_t parts,
                            uint32_t max_report, uint64_t* out_failures, uint32_t* out_pairs, uint32_t* out_reported) {
    if (!ctx || !trace || !program || (n_consts && !consts) || !out_failures || !out_reported || (max_report && !out_pairs))
        return set_err(ctx, GL_ERR_BAD_ARG, "null argument");
    if (n_instr == 0 || n_instr > GL_STARK_MAX_INSTR) return set_err(ctx, GL_ERR_UNSUPPORTED, "program of %u instructions (max %d)", n_instr, GL_STARK_MAX_INSTR);
    if (max_report > CHECK_MAX_REPORT) return set_err(ctx, GL_ERR_BAD_ARG, "max_report %u > %u", max_report, CHECK_MAX_REPORT);
    TRY(check_rows_commit(ctx, trace, trace, "trace"));
    if (aux) TRY(check_rows_commit(ctx, aux, trace, "auxiliary"));
    uint32_t n_emit = 0;
    TRY(stark_program_check(ctx, program, n_instr, trace, aux, n_consts, &n_emit));
    const uint32_t log_n = trace->degree_log;
    uint32_t s = 0;
    TRY(check_rows_parts(ctx, log_n, part, parts, &s));
    bool trace_next = false, aux_next = false;
    for (uint32_t k = 0; k < n_instr; k++) {
        trace_next |= program[k].op == GL_STARK_NEXT;
        aux_next |= program[k].op == GL_STARK_AUX_NEXT;
    }
    CK(ctx, cudaSetDevice(ctx->device));
    DevBuf tv(ctx), tn(ctx), av(ctx), an(ctx), dprog(ctx), dconst(ctx);
    StarkRowsParams p{nullptr, nullptr, log_n, nullptr, n_instr, nullptr};
    TRY(part_views(ctx, trace, part, s, trace_next, tv, tn, &p.trace, &p.trace_next));
    if (aux) TRY(part_views(ctx, aux, part, s, aux_next, av, an, &p.aux, &p.aux_next));
    TRY(upload_program(ctx, program, (size_t)n_instr * sizeof(gl_stark_instr), consts, n_consts, dprog, dconst));
    p.prog = (const gl_stark_instr*)dprog.get();
    p.consts = dconst.get();
    p.part_log = s;
    p.part = part;
    const size_t M = (size_t)1 << (log_n - s);
    return check_rows_report(ctx, M, n_emit, max_report, [&](u64* off, uint32_t* pairs) {
        k_stark_check_rows<<<(unsigned)((M + 127) / 128), 128, 0, ctx->stream>>>(p, off, pairs, max_report);
        CKL(ctx);
        return GL_OK;
    }, out_failures, out_pairs, out_reported);
}
int gl_stark_check_rows(gl_ctx* ctx, gl_commit* trace, gl_commit* aux, const gl_stark_instr* program, uint32_t n_instr,
                        const uint64_t* consts, uint32_t n_consts, uint32_t max_report, uint64_t* out_failures,
                        uint32_t* out_pairs, uint32_t* out_reported) {
    return stark_check_rows(ctx, trace, aux, program, n_instr, consts, n_consts, 0, 1, max_report, out_failures,
                            out_pairs, out_reported);
}
int gl_stark_check_rows_part(gl_ctx* ctx, gl_commit* trace, gl_commit* aux, const gl_stark_instr* program,
                             uint32_t n_instr, const uint64_t* consts, uint32_t n_consts, uint32_t part, uint32_t parts,
                             uint32_t max_report, uint64_t* out_failures, uint32_t* out_pairs, uint32_t* out_reported) {
    return stark_check_rows(ctx, trace, aux, program, n_instr, consts, n_consts, part, parts, max_report,
                            out_failures, out_pairs, out_reported);
}
// gl_plonk_check_rows (part 0 of 1) and gl_plonk_check_rows_part
static int plonk_check_rows(gl_ctx* ctx, gl_commit* const* commits, uint32_t n_commits, const gl_vp_instr* program,
                            uint32_t n_instr, const uint64_t* consts, uint32_t n_consts, uint32_t n_terms, uint32_t part,
                            uint32_t parts, uint32_t max_report, uint64_t* out_failures, uint32_t* out_pairs,
                            uint32_t* out_reported) {
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
    const uint32_t log_n = commits[0]->degree_log;
    uint32_t s = 0;
    TRY(check_rows_parts(ctx, log_n, part, parts, &s));
    CK(ctx, cudaSetDevice(ctx->device));
    const size_t n = (size_t)1 << log_n;
    std::vector<DevBuf> vals, nexts;
    vals.reserve(n_commits);
    nexts.reserve(n_commits);
    VpRowsParams p{};
    for (uint32_t c = 0; c < n_commits; c++) {
        vals.emplace_back(ctx);
        nexts.emplace_back(ctx);
        TRY(part_views(ctx, commits[c], part, s, (next_mask >> c) & 1, vals.back(), nexts.back(), &p.val[c],
                       &p.val_next[c]));
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
    p.part_log = s;
    p.part = part;
    const size_t M = n >> s;
    return check_rows_report(ctx, M, n_term, max_report, [&](u64* off, uint32_t* pairs) {
        k_plonk_check_rows<<<(unsigned)((M + 127) / 128), 128, 0, ctx->stream>>>(p, off, pairs, max_report);
        CKL(ctx);
        return GL_OK;
    }, out_failures, out_pairs, out_reported);
}
int gl_plonk_check_rows(gl_ctx* ctx, gl_commit* const* commits, uint32_t n_commits, const gl_vp_instr* program,
                        uint32_t n_instr, const uint64_t* consts, uint32_t n_consts, uint32_t n_terms,
                        uint32_t max_report, uint64_t* out_failures, uint32_t* out_pairs, uint32_t* out_reported) {
    return plonk_check_rows(ctx, commits, n_commits, program, n_instr, consts, n_consts, n_terms, 0, 1, max_report,
                            out_failures, out_pairs, out_reported);
}
int gl_plonk_check_rows_part(gl_ctx* ctx, gl_commit* const* commits, uint32_t n_commits, const gl_vp_instr* program,
                             uint32_t n_instr, const uint64_t* consts, uint32_t n_consts, uint32_t n_terms,
                             uint32_t part, uint32_t parts, uint32_t max_report, uint64_t* out_failures,
                             uint32_t* out_pairs, uint32_t* out_reported) {
    return plonk_check_rows(ctx, commits, n_commits, program, n_instr, consts, n_consts, n_terms, part, parts,
                            max_report, out_failures, out_pairs, out_reported);
}
