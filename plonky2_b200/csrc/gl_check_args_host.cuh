// gl_check_args_host.cuh -- kernels and host orchestration of plonky2's global-argument checks on a witness:
// gl_plonk_check_copies and gl_plonk_check_lookups of include/plonky2_b200_check.h. Included at the end of
// plonky2_b200.cu after gl_check_rows_host.cuh, whose check_rows_report it reports through; the per-thread code is
// gl_check_args.cuh.
#pragma once
#include "gl_check_args.cuh"

// ---- copy constraints: the identity and sigma values of every routed wire, sorted by value and matched position by
// position (sigma(i_p) = j_p), then one thread per routed wire compares its value with its sigma's
__global__ void __launch_bounds__(256) k_copy_keys(CopyCheck c, size_t count, int sigma, u64* keys, uint32_t* vals) {
    SIGMA_FOR(i, count) {
        keys[i] = sigma ? copy_sigma(c, i) : copy_identity(c, i);
        vals[i] = (uint32_t)i;
    }
}
// Sorted position p: sig[owner of the p-th sigma value] = the wire of the p-th identity value; unequal values mean the
// sigmas are not a permutation of the identities (flag)
__global__ void __launch_bounds__(256) k_copy_match(const u64* id_keys, const uint32_t* id_vals, const u64* sg_keys,
                                                    const uint32_t* sg_vals, size_t count, uint32_t* sig,
                                                    unsigned int* flag) {
    SIGMA_FOR(p, count) {
        if (id_keys[p] != sg_keys[p]) atomicOr(flag, 1u);
        sig[sg_vals[p]] = id_vals[p];
    }
}
// The two passes of check_rows_report with routed wires as rows: wire i's failure (0 or 1) to off[i], then the failing
// wires whose offset is below max_report write (i, sigma(i))
__global__ void __launch_bounds__(256) k_copy_check(CopyCheck c, const uint32_t* sig, size_t count, u64* off,
                                                    uint32_t* pairs, u64 max_report) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    if (!pairs) {
        off[i] = copy_fails(c, i, sig[i]);
        return;
    }
    if (off[i] >= max_report || off[i + 1] == off[i]) return;
    pairs[2 * off[i]] = (uint32_t)i;
    pairs[2 * off[i] + 1] = sig[i];
}

// ---- lookups: every looking slot adds one to the count of the entry it counts for, then one thread per row of H
// checks its slots against the LUT and the counts
__global__ void __launch_bounds__(128) k_lookup_count(LookupCheck p, size_t n, uint32_t* counts) {
    const size_t row = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    bool looking = false;
    const int k = lookup_table_of(p, row, &looking);
    if (k < 0 || !looking) return;
    for (uint32_t s = 0; s < p.num_lu_slots; s++) {
        const uint32_t e = lookup_counted_entry(p, (uint32_t)k, row, s);
        if (e != LOOKUP_NO_ENTRY) atomicAdd(counts + p.lut_off[k] + e, 1u);
    }
}
__global__ void __launch_bounds__(128) k_lookup_check_rows(LookupCheck p, size_t n, u64* off, uint32_t* pairs,
                                                           u64 max_report) {
    const size_t row = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    if (!pairs) {
        off[row] = lookup_check_row(p, row, nullptr);
        return;
    }
    if (off[row] >= max_report || off[row + 1] == off[row]) return;
    lookup_check_row(p, row, pairs + 2 * off[row]);
}

// A device view of `cols` columns of n words, column c at in + c * stride: the caller's memory itself for
// GL_MEM_DEVICE, else a copy in `stage` with stride n (the caller's page-locked memory is read by the time `reads` is
// waited for)
static int columns_in(gl_ctx* ctx, const u64* in, size_t stride, uint32_t cols, size_t n, int mem, DevBuf& stage,
                      HostReads& reads, const u64** view, size_t* view_stride) {
    *view = in;
    *view_stride = stride;
    if (mem != GL_MEM_HOST) return GL_OK;
    TRY(stage.alloc((size_t)cols * n));
    CK(ctx, cudaMemcpy2DAsync(stage.get(), n * 8, in, stride * 8, n * 8, cols, cudaMemcpyHostToDevice, ctx->stream));
    TRY(reads.mark(ctx->stream, mem));
    *view = stage.get();
    *view_stride = n;
    return GL_OK;
}
// The (canonical value, routed index) list of every routed wire sorted by value, identity values (sigma = 0) or sigma
// values (sigma = 1): *keys / *vals, in one of k[0], k[1] and one of v[0], v[1] (the other two are freed). `stage` (the
// sigmas' host copy) is freed once the values are read, before the sort's second buffers exist: 24 bytes per routed
// wire while sorting, 12 after.
static int copy_sorted(gl_ctx* ctx, const CopyCheck& c, size_t count, int sigma, DevBuf* stage, DevBuf* k, DevBuf* v,
                       const u64** keys, const uint32_t** vals) {
    TRY(k[0].alloc(count));
    TRY(v[0].alloc((count + 1) / 2));
    k_copy_keys<<<sigma_blocks(count), 256, 0, ctx->stream>>>(c, count, sigma, k[0].get(), (uint32_t*)v[0].get());
    CKL(ctx);
    if (stage) stage->reset();
    TRY(k[1].alloc(count));
    TRY(v[1].alloc((count + 1) / 2));
    // DoubleBuffer: the sort alternates between the two buffers, and its scratch holds no third copy
    cub::DoubleBuffer<u64> kb(k[0].get(), k[1].get());
    cub::DoubleBuffer<uint32_t> vb((uint32_t*)v[0].get(), (uint32_t*)v[1].get());
    DevBuf temp(ctx);
    size_t temp_bytes = 0;
    CK(ctx, cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, kb, vb, count, 0, 64, ctx->stream));
    TRY(temp.alloc((temp_bytes + 7) / 8));
    CK(ctx, cub::DeviceRadixSort::SortPairs(temp.get(), temp_bytes, kb, vb, count, 0, 64, ctx->stream));
    CKL(ctx);
    k[1 - kb.selector].reset();
    v[1 - vb.selector].reset();
    *keys = kb.Current();
    *vals = vb.Current();
    return GL_OK;
}

int gl_plonk_check_copies(gl_ctx* ctx, const uint64_t* wires, size_t wires_stride, int wires_mem,
                          const uint64_t* sigmas, size_t sigmas_stride, int sigmas_mem, const uint64_t* k_is,
                          uint32_t log_n, uint32_t num_routed_wires, uint32_t max_report, uint64_t* out_failures,
                          uint32_t* out_pairs, uint32_t* out_reported) {
    if (!ctx || !wires || !sigmas || !k_is || !out_failures || !out_reported || (max_report && !out_pairs))
        return set_err(ctx, GL_ERR_BAD_ARG, "null argument");
    if (max_report > CHECK_MAX_REPORT) return set_err(ctx, GL_ERR_BAD_ARG, "max_report %u > %u", max_report, CHECK_MAX_REPORT);
    if (num_routed_wires == 0 || log_n > 30 || ((uint64_t)num_routed_wires << log_n) >= ((uint64_t)1 << 31) - 1)
        return set_err(ctx, GL_ERR_BAD_SHAPE, "need 1 <= num_routed_wires * 2^log_n < 2^31 - 1 routed wires");
    const size_t n = (size_t)1 << log_n, count = (size_t)num_routed_wires << log_n;
    if (num_routed_wires > 1 && (wires_stride < n || sigmas_stride < n))
        return set_err(ctx, GL_ERR_BAD_SHAPE, "a column stride below n = %zu", n);
    CK(ctx, cudaSetDevice(ctx->device));
    HostReads reads(ctx);
    DevBuf dk(ctx), xtab(ctx), ds(ctx), dw(ctx), sig(ctx), dflag(ctx);
    DevBuf ik[2]{DevBuf(ctx), DevBuf(ctx)}, iv[2]{DevBuf(ctx), DevBuf(ctx)}, sk[2]{DevBuf(ctx), DevBuf(ctx)},
        sv[2]{DevBuf(ctx), DevBuf(ctx)};
    const u64 *id_keys, *sg_keys;
    const uint32_t *id_vals, *sg_vals;
    TRY(dk.alloc(num_routed_wires));
    TRY(h2d(ctx, dk.get(), k_is, num_routed_wires));  // a small host array
    TRY(reads.mark(ctx->stream, GL_MEM_HOST));
    TRY(x_pow_tables(ctx, root_of_unity(log_n), n, xtab));
    CopyCheck c{nullptr, 0, nullptr, 0, dk.get(), xtab.get(), xtab.get() + x_pow_table_len(n), num_routed_wires};
    TRY(copy_sorted(ctx, c, count, 0, nullptr, ik, iv, &id_keys, &id_vals));
    TRY(columns_in(ctx, sigmas, sigmas_stride, num_routed_wires, n, sigmas_mem, ds, reads, &c.sigmas, &c.sigmas_stride));
    TRY(copy_sorted(ctx, c, count, 1, &ds, sk, sv, &sg_keys, &sg_vals));
    TRY(sig.alloc((count + 1) / 2));
    TRY(flag_alloc(ctx, dflag));
    k_copy_match<<<sigma_blocks(count), 256, 0, ctx->stream>>>(id_keys, id_vals, sg_keys, sg_vals, count,
                                                               (uint32_t*)sig.get(), (unsigned int*)dflag.get());
    CKL(ctx);
    TRY(flag_status(ctx, dflag, {{1, GL_ERR_BAD_ARG, "the sigmas are not a permutation of the routed wires' identities "
                                                     "k_is[col] * w_n^row"}}));
    for (DevBuf* b : {ik, iv, sk, sv})
        for (int h = 0; h < 2; h++) b[h].reset();
    TRY(columns_in(ctx, wires, wires_stride, num_routed_wires, n, wires_mem, dw, reads, &c.wires, &c.wires_stride));
    const uint32_t* dsig = (const uint32_t*)sig.get();
    TRY(check_rows_report(ctx, count, 1, max_report, [&](u64* off, uint32_t* pairs) {
        k_copy_check<<<(unsigned)((count + 255) / 256), 256, 0, ctx->stream>>>(c, dsig, count, off, pairs, max_report);
        CKL(ctx);
        return GL_OK;
    }, out_failures, out_pairs, out_reported));
    return reads.wait();
}

int gl_plonk_check_lookups(gl_ctx* ctx, const uint64_t* wires, size_t col_stride, int mem, uint32_t log_n,
                           uint32_t num_routed_wires, const uint16_t* luts, const uint32_t* lut_offsets,
                           const uint32_t* lookup_rows, uint32_t n_luts, uint32_t* out_counts, uint32_t max_report,
                           uint64_t* out_failures, uint32_t* out_pairs, uint32_t* out_reported) {
    if (!ctx || !wires || (n_luts && (!luts || !lut_offsets || !lookup_rows)) || !out_failures || !out_reported ||
        (max_report && !out_pairs))
        return set_err(ctx, GL_ERR_BAD_ARG, "null argument");
    if (max_report > CHECK_MAX_REPORT) return set_err(ctx, GL_ERR_BAD_ARG, "max_report %u > %u", max_report, CHECK_MAX_REPORT);
    const uint32_t num_lu_slots = num_routed_wires / 2, num_lut_slots = num_routed_wires / 3;  // lookup.rs, lookup_table.rs
    if (num_lut_slots == 0 || log_n > 30) return set_err(ctx, GL_ERR_BAD_SHAPE, "bad lookup shape");
    const size_t n = (size_t)1 << log_n;
    const uint32_t cols = 3 * num_lut_slots > 2 * num_lu_slots ? 3 * num_lut_slots : 2 * num_lu_slots;
    if (cols > 1 && col_stride < n) return set_err(ctx, GL_ERR_BAD_SHAPE, "a column stride below n = %zu", n);
    if (n_luts && lut_offsets[0] != 0) return set_err(ctx, GL_ERR_BAD_ARG, "lut_offsets[0] must be 0");
    for (uint32_t k = 0; k < n_luts; k++) {
        const uint32_t* r = lookup_rows + 3 * k;
        if (lut_offsets[k + 1] <= lut_offsets[k]) return set_err(ctx, GL_ERR_BAD_ARG, "LUT %u is empty", k);
        if (!(r[0] <= r[1] && r[1] <= r[2] && r[2] < n))
            return set_err(ctx, GL_ERR_BAD_ARG, "lookup rows %u: need last_lu <= last_lut <= first_lut < n", k);
        if ((uint64_t)(r[2] - r[1] + 1) * num_lut_slots < lut_offsets[k + 1] - lut_offsets[k])
            return set_err(ctx, GL_ERR_BAD_SHAPE, "LUT %u: %u entries do not fit its %u LookupTableGate rows", k,
                           lut_offsets[k + 1] - lut_offsets[k], r[2] - r[1] + 1);
        for (uint32_t q = 0; q < k; q++)
            if (r[0] <= lookup_rows[3 * q + 2] && lookup_rows[3 * q] <= r[2])
                return set_err(ctx, GL_ERR_BAD_ARG, "the rows of lookup tables %u and %u overlap", q, k);
    }
    // the tables on the host (a LUT is at most a few 2^16 entries): entry keys, each table's distinct keys sorted, the
    // reference's input -> index map (a later entry of the same input wins)
    const uint32_t total = n_luts ? lut_offsets[n_luts] : 0;
    std::vector<uint32_t> lut(total), keys(total), key_len(n_luts);
    std::vector<uint32_t> index_of((size_t)n_luts << 16, LOOKUP_NO_ENTRY);
    for (uint32_t k = 0; k < n_luts; k++) {
        const uint32_t b = lut_offsets[k], e = lut_offsets[k + 1];
        for (uint32_t t = b; t < e; t++) {
            lut[t] = (uint32_t)luts[2 * t] | (uint32_t)luts[2 * t + 1] << 16;
            index_of[((size_t)k << 16) + luts[2 * t]] = t - b;
        }
        std::copy(lut.begin() + b, lut.begin() + e, keys.begin() + b);
        std::sort(keys.begin() + b, keys.begin() + e);
        key_len[k] = (uint32_t)(std::unique(keys.begin() + b, keys.begin() + e) - (keys.begin() + b));
    }
    CK(ctx, cudaSetDevice(ctx->device));
    HostReads reads(ctx);
    DevBuf dw(ctx), drows(ctx), dlut(ctx), doff(ctx), dkeys(ctx), dlen(ctx), dindex(ctx), dcounts(ctx);
    LookupCheck p{};
    TRY(columns_in(ctx, wires, col_stride, cols, n, mem, dw, reads, &p.wires, &p.stride));
    // u32 arrays in u64-word buffers (pageable sources: staged before cudaMemcpyAsync returns)
    auto up = [&](DevBuf& buf, const uint32_t* src, size_t words) -> int {
        TRY(buf.alloc(words / 2 + 1));
        if (words) CK(ctx, cudaMemcpyAsync(buf.get(), src, words * 4, cudaMemcpyHostToDevice, ctx->stream));
        return GL_OK;
    };
    TRY(up(drows, lookup_rows, (size_t)3 * n_luts));
    TRY(up(dlut, lut.data(), total));
    TRY(up(doff, lut_offsets, n_luts ? n_luts + 1 : 0));
    TRY(up(dkeys, keys.data(), total));
    TRY(up(dlen, key_len.data(), n_luts));
    TRY(up(dindex, index_of.data(), index_of.size()));
    TRY(dcounts.alloc(total / 2 + 1));
    CK(ctx, cudaMemsetAsync(dcounts.get(), 0, (size_t)(total / 2 + 1) * 8, ctx->stream));
    p.num_lu_slots = num_lu_slots;
    p.num_lut_slots = num_lut_slots;
    p.n_luts = n_luts;
    p.rows = (const uint32_t*)drows.get();
    p.lut = (const uint32_t*)dlut.get();
    p.lut_off = (const uint32_t*)doff.get();
    p.keys = (const uint32_t*)dkeys.get();
    p.key_len = (const uint32_t*)dlen.get();
    p.index_of = (const uint32_t*)dindex.get();
    p.counts = (const uint32_t*)dcounts.get();
    const unsigned blocks = (unsigned)((n + 127) / 128);
    if (n_luts) {
        k_lookup_count<<<blocks, 128, 0, ctx->stream>>>(p, n, (uint32_t*)dcounts.get());
        CKL(ctx);
    }
    const uint32_t max_per_row = num_lu_slots > 2 * num_lut_slots ? num_lu_slots : 2 * num_lut_slots;
    TRY(check_rows_report(ctx, n, max_per_row, max_report, [&](u64* off, uint32_t* pairs) {
        k_lookup_check_rows<<<blocks, 128, 0, ctx->stream>>>(p, n, off, pairs, max_report);
        CKL(ctx);
        return GL_OK;
    }, out_failures, out_pairs, out_reported));
    if (out_counts && total) {
        CK(ctx, cudaMemcpyAsync(out_counts, dcounts.get(), (size_t)total * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return reads.wait();
}
