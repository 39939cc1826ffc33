// gl_ntt_host.cuh -- kernels and host orchestration of the multi-pass NTT (included by plonky2_b200.cu).
//   k_ntt_col<LOG>        strided ("column") pass: T adjacent columns-of-the-matrix x 2^LOG strided points per CTA
//   k_ntt_col_cosets<LOG> the LDE's first column pass for up to 8 cosets of a column group in one launch
//   k_ntt_row<LOG, MODE>  contiguous ("row") pass: rows of 2^LOG points, bit-reversed (LDE) or natural-order stores
// The step twiddle table of a pass (<= 8 KiB) is staged into shared memory by a TMA bulk copy (cp.async.bulk +
// mbarrier) that overlaps the global loads of the data; the exchange tile lives next to it.
#pragma once

// ASYNC_TW: fetch the post twiddles with cp.async under step 2 (below). It hides the twiddle loads' long-scoreboard
// stalls and pays off where a pass has the extra coset multiplies to hide them under, but costs more instructions and
// one more barrier, which does not pay on the plain transform: used for coset passes only.
template <int LOG, bool ASYNC_TW>
__global__ void __launch_bounds__(PassCfg<LOG>::COL_THREADS, PassCfg<LOG>::COL_MIN_BLOCKS) k_ntt_col(ColPass cp) {
    using Cf = PassCfg<LOG>;
    extern __shared__ __align__(16) u64 smem[];
    u64* tw_s = smem;                    // 2^LOG words
    u64* S = smem + (1 << LOG);          // exchange tile
    u64* mbar = S + Cf::COL_S_WORDS;
    tma_table_issue(tw_s, cp.tw, (uint32_t)((1 << LOG) * 8), mbar);
    u64 x[Cf::E];
    col_load<LOG>(cp, blockIdx.x, threadIdx.x, x);  // the data loads overlap the table copy
    __syncthreads();                     // mbarrier initialised before anyone polls it
    ColPass c2 = cp;
    c2.tw = tw_s;
    tma_table_wait(mbar);
    col_phase1<LOG>(c2, S, blockIdx.x, threadIdx.x, x);
    if (Cf::R2 == 0) return;
    __syncthreads();
    if (!ASYNC_TW) {
        col_phase2<LOG>(c2, S, blockIdx.x, threadIdx.x);
        return;
    }
    col_phase2_load<LOG>(S, threadIdx.x, x);
    __syncthreads();                     // every thread holds its part of the tile: S is free
    // the E post twiddles of this thread (L2-resident table, 8 KiB row stride) go to thread-private shared-memory
    // slots by cp.async WHILE step 2 runs: as plain loads at their use they were the kernel's main stall
    // (long-scoreboard stalls) because 128 registers leave no room to hoist them
#pragma unroll
    for (int i = 0; i < Cf::E; i++) {
        const u64* src = col_twiddle_src<LOG>(cp, blockIdx.x, threadIdx.x, i);
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(S + col_twiddle_slot<LOG>(threadIdx.x, i))), "l"(src)
                     : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    col_phase2_dft<LOG>(x);
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    col_phase2_store<LOG>(cp, blockIdx.x, threadIdx.x, x, S + col_twiddle_slot<LOG>(threadIdx.x, 0), Cf::COL_THREADS,
                          (size_t)Cf::TPT * Cf::COL_THREADS);
}

// Even LOG (E == TPT): both steps of the pass are "radix-E lazy DFT, normalise, multiply by a twiddle", so ONE copy of
// that body serves both (a rolled 2-trip loop; only the I/O around it differs). The two-copy kernel above is ~90 KiB of
// SASS, large enough for instruction fetch to stall it; this one is about half that.
// The body of one CTA: tile `tile` of the unit at in_off / out_off, step table tw, post table twa, pre-weights uq.
template <int LOG, bool ASYNC_TW>
__device__ __forceinline__ void col_shared_body(const ColPass& cp, const u64* tw, const u64* twa, const u64 (&uq)[32],
                                                size_t in_off, size_t out_off, int tile) {
    using Cf = PassCfg<LOG>;
    static_assert(Cf::E == Cf::TPT, "shared-body column pass needs an even LOG");
    extern __shared__ __align__(16) u64 smem[];
    u64* tw_s = smem;                    // 2^LOG words
    u64* S = smem + (1 << LOG);          // exchange tile
    u64* mbar = S + Cf::COL_S_WORDS;
    tma_table_issue(tw_s, tw, (uint32_t)((1 << LOG) * 8), mbar);
    u64 x[Cf::E];
    col_load_at<LOG>(cp, in_off, tile, threadIdx.x, x);
    __syncthreads();
    tma_table_wait(mbar);
    const int tt = threadIdx.x % Cf::T, t = threadIdx.x / Cf::T;
    const size_t C = (size_t)1 << cp.log_c;
    if (cp.has_uq) {
#pragma unroll
        for (int q = 1; q < Cf::E; q++) x[q] = mul(x[q], uq[q]);
    }
    const u64* twp = tw_s + t;           // step 1: tw[q*TPT + t]
    size_t tws = Cf::TPT;
    bool skip0 = cp.tw_full == 0;        // step 1, q = 0: the twiddle is 1 unless a scale / coset base is folded in
#pragma unroll 1
    for (int s = 0; s < 2; s++) {
        L3 r[Cf::E];
#pragma unroll
        for (int q = 0; q < Cf::E; q++) r[q] = l3_from(x[q]);
        dft_lazy<Cf::R1>(r);
        if (ASYNC_TW && s == 1) asm volatile("cp.async.wait_group 0;" ::: "memory");
#pragma unroll
        for (int q = 0; q < Cf::E; q++) {
            u64 y = l3_norm(r[q]);
            if (!(q == 0 && skip0)) y = mul(y, twp[(size_t)q * tws]);
            x[q] = y;
        }
        if (s == 0) {
#pragma unroll
            for (int q = 0; q < Cf::E; q++) S[q * Cf::COL_QPITCH + t * Cf::T + tt] = x[q];
            __syncthreads();
#pragma unroll
            for (int j = 0; j < Cf::TPT; j++) x[j] = S[t * Cf::COL_QPITCH + j * Cf::T + tt];  // step 2 works on row q = t
            skip0 = false;
            const u64* tw2 = twa + (((size_t)t * Cf::TPT) << cp.log_c) + (size_t)tile * Cf::T + tt;  // output p = t*TPT + j
            if (ASYNC_TW) {
                __syncthreads();         // every thread holds its part of the tile: S is free
#pragma unroll
                for (int j = 0; j < Cf::TPT; j++)
                    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(S + col_twiddle_slot<LOG>(threadIdx.x, j))),
                                 "l"(tw2 + (size_t)j * C)
                                 : "memory");
                asm volatile("cp.async.commit_group;" ::: "memory");
                twp = S + col_twiddle_slot<LOG>(threadIdx.x, 0);
                tws = Cf::COL_THREADS;
            } else {
                twp = tw2;
                tws = C;
            }
        }
    }
    u64* dst = cp.out + out_off + (size_t)tile * Cf::T + tt;
#pragma unroll
    for (int j = 0; j < Cf::TPT; j++) dst[((size_t)t * Cf::TPT + j) * C] = x[j];
}
template <int LOG, bool ASYNC_TW>
__global__ void __launch_bounds__(PassCfg<LOG>::COL_THREADS, PassCfg<LOG>::COL_MIN_BLOCKS) k_ntt_col_shared(ColPass cp) {
    size_t in_off, out_off;
    int tile;
    col_unit<LOG>(cp, blockIdx.x, in_off, out_off, tile);
    col_shared_body<LOG, ASYNC_TW>(cp, cp.tw, cp.twa, cp.uq, in_off, out_off, tile);
}
// The first column pass of up to 8 cosets of an LDE in one launch (ColCosets, gl_ntt.cuh): the same body per CTA, with
// the tables and pre-weights of the CTA's coset.
template <int LOG>
__global__ void __launch_bounds__(PassCfg<LOG>::COL_THREADS, PassCfg<LOG>::COL_MIN_BLOCKS) k_ntt_col_cosets(ColCosets cc) {
    size_t in_off, out_off;
    int c, tile;
    col_cosets_unit<LOG>(cc, blockIdx.x, c, in_off, out_off, tile);
    col_shared_body<LOG, true>(cc.cp, cc.tw[c], cc.twa[c], cc.uq[c], in_off, out_off, tile);
}

template <int LOG, int MODE>
__global__ void __launch_bounds__(PassCfg<LOG>::ROW_THREADS, PassCfg<LOG>::ROW_MIN_BLOCKS) k_ntt_row(RowPass rp) {
    using Cf = PassCfg<LOG>;
    extern __shared__ __align__(16) u64 smem[];
    u64* tw_s = smem;
    u64* S = smem + (1 << LOG);
    u64* mbar = S + ntt_row_smem_bytes(LOG, MODE == RM_NATURAL) / 8;
    RowPass r2 = rp;
    u64 x[Cf::E];
    if (Cf::R2 > 0 && LOG >= 4) {        // tables of >= 128 bytes: TMA bulk copy (16-byte granularity)
        tma_table_issue(tw_s, rp.tw, (uint32_t)((1 << LOG) * 8), mbar);
        row_load<LOG, MODE>(rp, blockIdx.x, threadIdx.x, x);
        __syncthreads();
        r2.tw = tw_s;
        tma_table_wait(mbar);
    } else {
        row_load<LOG, MODE>(rp, blockIdx.x, threadIdx.x, x);
    }
    row_phase1<LOG, MODE>(r2, S, blockIdx.x, threadIdx.x, x);
    if (Cf::R2 == 0) {
        if (MODE == RM_BITREV) {
            row_store_bitrev<LOG>(r2, blockIdx.x, threadIdx.x, 0, x);
        } else {
            row_gather_write<LOG>(S, threadIdx.x, 0, x);
            __syncthreads();
            row_store_natural<LOG>(r2, S, blockIdx.x, threadIdx.x, blockDim.x);
        }
        return;
    }
    __syncwarp();  // a line's TPT <= 32 threads sit in one warp
    if (MODE == RM_BITREV) {
#pragma unroll
        for (int m = 0; m < Cf::NSUB; m++) {
            u64 z[Cf::TPT];
            row_phase2_load<LOG>(S, threadIdx.x, m, z);
            pass_step2<LOG>(z);
            row_store_bitrev<LOG>(r2, blockIdx.x, threadIdx.x, m, z);
        }
    } else {
        u64 z[Cf::NSUB][Cf::TPT];
#pragma unroll
        for (int m = 0; m < Cf::NSUB; m++) {
            row_phase2_load<LOG>(S, threadIdx.x, m, z[m]);
            pass_step2<LOG>(z[m]);
        }
        __syncthreads();  // the gather tile aliases the exchange buffers
#pragma unroll
        for (int m = 0; m < Cf::NSUB; m++) row_gather_write<LOG>(S, threadIdx.x, m, z[m]);
        __syncthreads();
        row_store_natural<LOG>(r2, S, blockIdx.x, threadIdx.x, blockDim.x);
    }
}

// Row pass with ONE copy of the radix-E lazy DFT for both steps (even LOG, E == TPT); see k_ntt_col_shared.
template <int LOG, int MODE>
__global__ void __launch_bounds__(PassCfg<LOG>::ROW_THREADS, PassCfg<LOG>::ROW_MIN_BLOCKS) k_ntt_row_shared(RowPass rp) {
    using Cf = PassCfg<LOG>;
    static_assert(Cf::E == Cf::TPT && Cf::R2 > 0 && LOG >= 4, "shared-body row pass needs an even LOG >= 4");
    extern __shared__ __align__(16) u64 smem[];
    u64* tw_s = smem;
    u64* S = smem + (1 << LOG);
    u64* mbar = S + ntt_row_smem_bytes(LOG, MODE == RM_NATURAL) / 8;
    u64 x[Cf::E];
    tma_table_issue(tw_s, rp.tw, (uint32_t)((1 << LOG) * 8), mbar);
    row_load<LOG, MODE>(rp, blockIdx.x, threadIdx.x, x);
    __syncthreads();
    tma_table_wait(mbar);
    const int l = threadIdx.x / Cf::TPT, t = threadIdx.x % Cf::TPT;
    u64* Sl = S + (size_t)l * Cf::ROW_S_WORDS;
    if (rp.has_uq) {
#pragma unroll
        for (int q = 1; q < Cf::E; q++) x[q] = mul(x[q], rp.uq[q]);
    }
    const bool skip0 = rp.tw_full == 0;
    // step 2 has no twiddle: `do_mul` (a uniform, loop-carried flag) skips the multiplies there, so that the DFT AND the
    // normalise/multiply code exist once and only the exchange differs between the trips
    bool do_mul = true;
#pragma unroll 1
    for (int s = 0; s < 2; s++) {
        L3 r[Cf::E];
#pragma unroll
        for (int q = 0; q < Cf::E; q++) r[q] = l3_from(x[q]);
        dft_lazy<Cf::R1>(r);
#pragma unroll
        for (int q = 0; q < Cf::E; q++) {
            u64 y = l3_norm(r[q]);
            if (do_mul && !(q == 0 && skip0)) y = mul(y, tw_s[q * Cf::TPT + t]);
            x[q] = y;
        }
        if (s == 0) {
#pragma unroll
            for (int q = 0; q < Cf::E; q++) Sl[q * Cf::ROW_PITCH + t] = x[q];
            __syncwarp();  // a line's TPT <= 32 threads sit in one warp
#pragma unroll
            for (int j = 0; j < Cf::TPT; j++) x[j] = Sl[t * Cf::ROW_PITCH + j];
            do_mul = false;
        }
    }
    if (MODE == RM_BITREV) {
        __syncwarp();  // the line's step-2 loads from the exchange buffer are done
        row_stage_bitrev<LOG>(S, threadIdx.x, x);
        __syncwarp();
        row_store_bitrev_staged<LOG>(rp, S, blockIdx.x, threadIdx.x);
    } else {
        __syncthreads();  // the gather tile aliases the exchange buffers
        row_gather_write<LOG>(S, threadIdx.x, 0, x);
        __syncthreads();
        row_store_natural<LOG>(rp, S, blockIdx.x, threadIdx.x, blockDim.x);
    }
}

__global__ void k_fill_step(int log, u64 scale, u64 base, u64* out) {
    uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < (1u << log)) out[j] = table_step_entry(log, j, scale, base);
}
__global__ void k_fill_post(int a, int b, u64 base, u64* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < ((size_t)1 << (a + b))) out[i] = table_post_entry(a, b, i, base);
}
// out[t*count + i] = bases[t]^i  for t < ntab
__global__ void k_fill_pows(const u64* bases, int ntab, size_t count, u64* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count * ntab) return;
    size_t t = i / count, e = i % count;
    out[i] = gl::pow(bases[t], e);
}
// data[b*stride + k] *= hi[k >> lowbits] * lo[k & mask]
__global__ void k_mul_pows(u64* data, size_t stride, size_t n, const u64* hi, const u64* lo, int lowbits) {
    size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    u64* col = data + (size_t)blockIdx.y * stride;
    u64 f = mul(hi[k >> lowbits], lo[k & (((size_t)1 << lowbits) - 1)]);
    col[k] = canon(mul(col[k], f));
}

template <int LOG>
static int launch_col(gl_ctx* ctx, const ColPass& cp, size_t ncols) {
    const int nblocks = col_blocks<LOG>(cp, ncols);
    const size_t smem = ((size_t)(1 << LOG) + PassCfg<LOG>::COL_S_WORDS) * 8 + 16;
    auto go = [&](auto kern) -> int {
        const void* fn = (const void*)kern;
        if (!ctx->smem_attr_done.count(fn)) {  // function attributes are per device: track them per context
            CK(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            CK(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
            ctx->smem_attr_done.insert(fn);
        }
        kern<<<nblocks, PassCfg<LOG>::COL_THREADS, smem, ctx->stream>>>(cp);
        CKL(ctx);
        return GL_OK;
    };
    if constexpr (PassCfg<LOG>::E == PassCfg<LOG>::TPT) {
        if (ctx->ntt_variant == 0) return cp.has_uq ? go(k_ntt_col_shared<LOG, true>) : go(k_ntt_col_shared<LOG, false>);
    }
    return cp.has_uq ? go(k_ntt_col<LOG, true>) : go(k_ntt_col<LOG, false>);
}
template <int LOG, int MODE>
static int launch_row(gl_ctx* ctx, const RowPass& rp) {
    const size_t smem = (size_t)(1 << LOG) * 8 + ntt_row_smem_bytes(LOG, MODE == RM_NATURAL) + 16;
    auto go = [&](auto kern) -> int {
        const void* fn = (const void*)kern;
        if (!ctx->smem_attr_done.count(fn)) {
            CK(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            CK(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
            ctx->smem_attr_done.insert(fn);
        }
        kern<<<row_blocks<LOG>(rp), PassCfg<LOG>::ROW_THREADS, smem, ctx->stream>>>(rp);
        CKL(ctx);
        return GL_OK;
    };
    if constexpr (PassCfg<LOG>::E == PassCfg<LOG>::TPT && LOG >= 4) {
        if (ctx->ntt_variant == 0) return go(k_ntt_row_shared<LOG, MODE>);
    }
    return go(k_ntt_row<LOG, MODE>);
}
static int dispatch_col(gl_ctx* ctx, int a, const ColPass& cp, size_t ncols) {
    switch (a) {
        case 5: return launch_col<5>(ctx, cp, ncols);
        case 6: return launch_col<6>(ctx, cp, ncols);
        case 7: return launch_col<7>(ctx, cp, ncols);
        case 8: return launch_col<8>(ctx, cp, ncols);
        case 9: return launch_col<9>(ctx, cp, ncols);
        case 10: return launch_col<10>(ctx, cp, ncols);
    }
    return set_err(ctx, GL_ERR_UNSUPPORTED, "column pass log %d", a);
}
template <int LOG>
static int launch_col_cosets(gl_ctx* ctx, const ColCosets& cc) {
    const size_t smem = ((size_t)(1 << LOG) + PassCfg<LOG>::COL_S_WORDS) * 8 + 16;
    auto kern = k_ntt_col_cosets<LOG>;
    const void* fn = (const void*)kern;
    if (!ctx->smem_attr_done.count(fn)) {
        CK(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CK(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
        ctx->smem_attr_done.insert(fn);
    }
    kern<<<col_cosets_blocks<LOG>(cc), PassCfg<LOG>::COL_THREADS, smem, ctx->stream>>>(cc);
    CKL(ctx);
    return GL_OK;
}
// the coset-batched first column pass exists for the shared-body (even) pass sizes only
static bool col_cosets_supported(int a) { return a == 6 || a == 8 || a == 10; }
static int dispatch_col_cosets(gl_ctx* ctx, int a, const ColCosets& cc) {
    switch (a) {
        case 6: return launch_col_cosets<6>(ctx, cc);
        case 8: return launch_col_cosets<8>(ctx, cc);
        case 10: return launch_col_cosets<10>(ctx, cc);
    }
    return set_err(ctx, GL_ERR_UNSUPPORTED, "coset column pass log %d", a);
}
static int dispatch_row(gl_ctx* ctx, int b, int mode, const RowPass& rp) {
#define ROW_CASE(L)                                                     \
    case L:                                                             \
        return mode == RM_BITREV ? launch_row<L, RM_BITREV>(ctx, rp) : launch_row<L, RM_NATURAL>(ctx, rp);
    switch (b) {
        ROW_CASE(1) ROW_CASE(2) ROW_CASE(3) ROW_CASE(4) ROW_CASE(5) ROW_CASE(6) ROW_CASE(7) ROW_CASE(8) ROW_CASE(9) ROW_CASE(10)
    }
#undef ROW_CASE
    return set_err(ctx, GL_ERR_UNSUPPORTED, "row pass log %d", b);
}

// ---- cached tables (per context = per device)
static void table_cache_trim(gl_ctx* ctx, size_t incoming_bytes) {
    const size_t cap = (size_t)3 << 30;  // bound the cache: drop everything when it would exceed 3 GiB
    if (ctx->table_bytes + incoming_bytes <= cap) return;
    for (auto& kv : ctx->step_tabs) cudaFreeAsync(kv.second, ctx->stream);
    for (auto& kv : ctx->post_tabs) cudaFreeAsync(kv.second, ctx->stream);
    ctx->step_tabs.clear();
    ctx->post_tabs.clear();
    ctx->table_bytes = 0;
}
static int get_step(gl_ctx* ctx, int log, u64 scale, u64 base, const u64** out) {
    auto key = std::make_tuple(log, canon(scale), canon(base));
    auto it = ctx->step_tabs.find(key);
    if (it == ctx->step_tabs.end()) {
        const size_t words = ((size_t)1 << log) < 2 ? 2 : ((size_t)1 << log);
        DevBuf p(ctx);
        TRY(p.alloc(words));
        k_fill_step<<<((1 << log) + 255) / 256, 256, 0, ctx->stream>>>(log, canon(scale), canon(base), p.get());
        CKL(ctx);
        ctx->table_bytes += words * 8;
        it = ctx->step_tabs.emplace(key, p.release()).first;
    }
    *out = it->second;
    return GL_OK;
}
static int get_post(gl_ctx* ctx, int a, int b, u64 base, const u64** out) {
    auto key = std::make_tuple(a, b, canon(base));
    auto it = ctx->post_tabs.find(key);
    if (it == ctx->post_tabs.end()) {
        const size_t words = (size_t)1 << (a + b);
        DevBuf p(ctx);
        TRY(p.alloc(words));
        k_fill_post<<<(unsigned)((words + 255) / 256), 256, 0, ctx->stream>>>(a, b, canon(base), p.get());
        CKL(ctx);
        ctx->table_bytes += words * 8;
        it = ctx->post_tabs.emplace(key, p.release()).first;
    }
    *out = it->second;
    return GL_OK;
}
// Columns per multi-pass group (scratch = group * n * 8 bytes). The passes are instruction-bound, so large launches
// (full waves) beat keeping the intermediate L2-resident (tools/ntt_sweep.py, round 1): as many columns as fit 1 GiB.
// A group of the coset-batched LDE holds `cosets` transforms per column: it is 1/cosets as many columns, so that the
// scratch and the size of a launch stay the same.
static uint32_t group_cols(const gl_ctx* ctx, int log_n, uint32_t ncols, uint32_t cosets = 1) {
    uint32_t g = ctx->ntt_group;
    if (g == 0) {
        size_t col_bytes = (size_t)8 << log_n;
        size_t target = (size_t)1 << 30;
        g = (uint32_t)(target / col_bytes);
        if (g < 8) g = 8;
    }
    g = (g + 7) & ~7u;
    if (cosets > 1) {
        g = g / cosets ? g / cosets : 1;
        return g < ncols ? g : ncols;
    }
    if (g > ((ncols + 7) & ~7u)) g = (ncols + 7) & ~7u;
    return g;
}

// Upload `bases` (host) and build ntab tables of `count` powers each on the device.
static int build_pow_tables(gl_ctx* ctx, const std::vector<u64>& bases, size_t count, DevBuf& out) {
    const int ntab = (int)bases.size();
    DevBuf dbases(ctx);
    TRY(dbases.alloc(ntab));
    TRY(h2d(ctx, dbases.get(), bases.data(), ntab));  // pageable source: staged by the runtime before the call returns
    TRY(out.alloc(count * ntab));
    size_t total = count * ntab;
    k_fill_pows<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>(dbases.get(), ntab, count, out.get());
    CKL(ctx);
    return GL_OK;
}

// One forward transform of `ncols` device columns: in (natural order) -> out, either natural order (mode RM_NATURAL,
// optional index reversal + scale for the inverse) or bit-reversed order at out + col*out_stride + row0 (RM_BITREV).
// shift != 1: evaluate on the coset shift*<w_n> (input scaled by shift^j). `in` is never written unless in == out.
struct PeerOuts {  // extra destinations of a natural-order transform (same addressing as `out`)
    int n = 0;
    u64* p[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
};
static int ntt_forward(gl_ctx* ctx, const u64* in, size_t in_stride, u64* out, size_t out_stride, size_t row0, int log_n,
                       uint32_t ncols, int mode, bool reverse, u64 scale, u64 shift, const PeerOuts* peers = nullptr) {
    if (ncols == 0) return GL_OK;
    if (log_n < 1 || log_n > 3 * NTT_MAX_LOG_PASS) return set_err(ctx, GL_ERR_UNSUPPORTED, "log_n %d not in 1..30", log_n);
    const NttPlan pl = ntt_plan(log_n);
    const size_t n = (size_t)1 << log_n;
    table_cache_trim(ctx, 2 * n * 8 + (1 << 16));  // only here, before any table of this call is fetched
    NttJob job;
    ntt_make_job(log_n, pl, scale, shift, job);
    RowPass& rp = job.rp;
    rp.out_stride = out_stride;
    rp.reverse = reverse ? 1 : 0;
    rp.row0 = row0;
    rp.n_peer = peers ? peers->n : 0;
    for (int i = 0; i < rp.n_peer; i++) rp.out_peer[i] = peers->p[i];
    TRY(get_step(ctx, job.row_step.a, job.row_step.scale, job.row_step.base, &rp.tw));
    if (pl.a1 == 0) {  // single pass
        rp.in = in;
        rp.in_stride = in_stride;
        rp.out = out;
        rp.ncols = (int)ncols;
        return dispatch_row(ctx, pl.b, mode, rp);
    }
    // multi-pass: column pass(es) into the group scratch, then the row pass
    const uint32_t G = group_cols(ctx, log_n, ncols);
    TRY(ensure_scratch(ctx, (size_t)G * n));
    ColPass &c1 = job.c1, &c2 = job.c2;
    c1.out = ctx->scratch;
    c1.in_stride = in_stride;
    c1.out_stride = n;
    TRY(get_step(ctx, job.c1_step.a, job.c1_step.scale, job.c1_step.base, &c1.tw));
    TRY(get_post(ctx, job.c1_post.a, job.c1_post.b, job.c1_post.base, &c1.twa));
    if (pl.a2) {
        c2.in = c2.out = ctx->scratch;  // in place: a CTA rewrites exactly the tile it read
        c2.in_stride = c2.out_stride = n;
        TRY(get_step(ctx, job.c2_step.a, job.c2_step.scale, job.c2_step.base, &c2.tw));
        TRY(get_post(ctx, job.c2_post.a, job.c2_post.b, job.c2_post.base, &c2.twa));
    }
    rp.in = ctx->scratch;
    rp.in_stride = n;
    for (uint32_t g0 = 0; g0 < ncols; g0 += G) {
        const uint32_t gc = (ncols - g0 < G) ? ncols - g0 : G;
        c1.in = in + (size_t)g0 * in_stride;
        TRY(dispatch_col(ctx, pl.a1, c1, gc));
        if (pl.a2) TRY(dispatch_col(ctx, pl.a2, c2, gc));
        rp.out = out + (size_t)g0 * out_stride;
        for (int i = 0; i < rp.n_peer; i++) rp.out_peer[i] = peers->p[i] + (size_t)g0 * out_stride;
        rp.ncols = (int)gc;
        TRY(dispatch_row(ctx, pl.b, mode, rp));
    }
    return GL_OK;
}

// data[b*stride] = canon(data[b*stride] * f) for the degenerate n = 1 transform
__global__ void k_scale1(u64* data, size_t stride, uint32_t ncols, u64 f) {
    uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < ncols) data[(size_t)b * stride] = canon(mul(data[(size_t)b * stride], f));
}

// Natural-order NTT / iNTT of `ncols` device columns (in -> out, may alias), optional coset shift
// (forward: evaluate on shift*<w_n>; inverse: interpolate from values on shift*<w_n>).
static int ntt_natural(gl_ctx* ctx, const u64* in, size_t in_stride, u64* out, size_t out_stride, int log_n,
                       uint32_t ncols, bool inverse, u64 shift, const PeerOuts* peers = nullptr) {
    if (ncols == 0) return GL_OK;
    const size_t n = (size_t)1 << log_n;
    if (peers && peers->n && (log_n == 0 || canon(shift) != 1))
        return set_err(ctx, GL_ERR_UNSUPPORTED, "multi-destination transforms need log_n >= 1 and no coset shift");
    if (log_n == 0) {
        if (in != out)
            CK(ctx, cudaMemcpy2DAsync(out, out_stride * 8, in, in_stride * 8, 8, ncols, cudaMemcpyDeviceToDevice,
                                      ctx->stream));
        k_scale1<<<(ncols + 127) / 128, 128, 0, ctx->stream>>>(out, out_stride, ncols, 1);  // canonicalise
        CKL(ctx);
        return GL_OK;
    }
    if (!inverse) return ntt_forward(ctx, in, in_stride, out, out_stride, 0, log_n, ncols, RM_NATURAL, false, 1, shift, peers);
    // inverse = forward + index reversal + 1/n (fft.rs:68-91), then coefficients *= shift^-k (polynomial/mod.rs:63-73)
    TRY(ntt_forward(ctx, in, in_stride, out, out_stride, 0, log_n, ncols, RM_NATURAL, true, inverse_2exp((uint32_t)log_n), 1,
                    peers));
    if (canon(shift) != 1) {
        const int lowbits = log_n > 12 ? 12 : log_n;
        const size_t lo_cnt = (size_t)1 << lowbits, hi_cnt = (size_t)1 << (log_n - lowbits);
        const u64 sinv = gl::inv(shift);
        const size_t tcnt = lo_cnt > hi_cnt ? lo_cnt : hi_cnt;
        DevBuf tabs(ctx);
        TRY(build_pow_tables(ctx, std::vector<u64>{gl::pow(sinv, lo_cnt), sinv}, tcnt, tabs));
        for (uint32_t b0 = 0; b0 < ncols; b0 += MAX_GRID_Y) {  // one column per blockIdx.y, which is capped
            const uint32_t bc = (ncols - b0 < MAX_GRID_Y) ? ncols - b0 : MAX_GRID_Y;
            k_mul_pows<<<dim3((unsigned)((n + 255) / 256), bc), 256, 0, ctx->stream>>>(
                out + (size_t)b0 * out_stride, out_stride, n, tabs.get(), tabs.get() + tcnt, lowbits);
            CKL(ctx);
        }
    }
    return GL_OK;
}

// degenerate n = 1 LDE: lde[col][c] = coeff[col]
__global__ void k_lde_const(const u64* coeffs, size_t stride, uint32_t ncols, int ncos, u64* lde, size_t lde_stride) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ncols * (uint32_t)ncos) return;
    uint32_t col = i / ncos, c = i % ncos;
    lde[(size_t)col * lde_stride + c] = canon(coeffs[(size_t)col * stride]);
}

// Coset LDE of device coefficient columns into COLUMN-MAJOR evaluations in the reference's leaf order:
//   lde[col*lde_stride + c*n + j] = P_col( g * w_N^{bitrev_r(c)} * w_n^{bitrev(j)} ),  g = base_shift,
// i.e. leaf row (c*n + j) of the reference's transposed + bit-reversed matrix (oracle.rs:97-98) is the vector of
// these entries over all columns: block c is the size-n NTT (bit-reversed stores) on the coset g*w_N^{bitrev(c)}<w_n>.
//
// Multi-pass plans with an even first column pass run every pass once per column group for up to 8 cosets at a time
// (lde_make_cosets_job): a group is G/8 columns x 8 cosets, the same G transforms per launch and the same scratch as
// one coset of G columns, but the coefficients are read from HBM once per group instead of once per coset. Single-pass
// sizes, odd first passes and ctx->lde_per_coset run one transform per coset and group.
static int lde_columns(gl_ctx* ctx, const u64* coeffs, size_t coeff_stride, uint32_t ncols, int log_n, int rate_bits,
                       u64 base_shift, u64* lde, size_t lde_stride) {
    if (ncols == 0) return GL_OK;
    const size_t n = (size_t)1 << log_n;
    const int ncos = 1 << rate_bits;
    if (log_n == 0) {
        k_lde_const<<<(ncols * ncos + 127) / 128, 128, 0, ctx->stream>>>(coeffs, coeff_stride, ncols, ncos, lde, lde_stride);
        CKL(ctx);
        return GL_OK;
    }
    const NttPlan pl = ntt_plan(log_n);
    if (ncos > 1 && pl.a1 && col_cosets_supported(pl.a1) && ctx->ntt_variant == 0 && !ctx->lde_per_coset) {
        const int log_kc = rate_bits < COL_LOG_MAX_COSETS ? rate_bits : COL_LOG_MAX_COSETS, kc = 1 << log_kc;
        const uint32_t G = group_cols(ctx, log_n, ncols, kc);
        TRY(ensure_scratch(ctx, (size_t)G * kc * n));
        for (uint32_t g0 = 0; g0 < ncols; g0 += G) {
            const uint32_t gc = (ncols - g0 < G) ? ncols - g0 : G;
            for (int c0 = 0; c0 < ncos; c0 += kc) {
                table_cache_trim(ctx, (size_t)(kc + 1) * (n * 8 + (1 << 16)));  // before any table of this job is fetched
                NttJob job;
                ColCosets cc;
                TableReq steps[1 << COL_LOG_MAX_COSETS], posts[1 << COL_LOG_MAX_COSETS];
                lde_make_cosets_job(log_n, pl, rate_bits, base_shift, c0, log_kc, job, cc, steps, posts);
                for (int c = 0; c < kc; c++) {
                    TRY(get_step(ctx, steps[c].a, steps[c].scale, steps[c].base, &cc.tw[c]));
                    TRY(get_post(ctx, posts[c].a, posts[c].b, posts[c].base, &cc.twa[c]));
                }
                cc.cp.in = coeffs + (size_t)g0 * coeff_stride;
                cc.cp.in_stride = coeff_stride;
                cc.cp.out = ctx->scratch;
                cc.cp.out_stride = n;
                cc.ncols = (int)gc;
                TRY(dispatch_col_cosets(ctx, pl.a1, cc));
                if (pl.a2) {
                    ColPass& c2 = job.c2;
                    c2.in = c2.out = ctx->scratch;
                    c2.in_stride = c2.out_stride = n;
                    TRY(get_step(ctx, job.c2_step.a, job.c2_step.scale, job.c2_step.base, &c2.tw));
                    TRY(get_post(ctx, job.c2_post.a, job.c2_post.b, job.c2_post.base, &c2.twa));
                    TRY(dispatch_col(ctx, pl.a2, c2, (size_t)gc * kc));
                }
                RowPass& rp = job.rp;
                TRY(get_step(ctx, job.row_step.a, job.row_step.scale, job.row_step.base, &rp.tw));
                rp.in = ctx->scratch;
                rp.in_stride = n;
                rp.out = lde + (size_t)g0 * lde_stride;
                rp.out_stride = lde_stride;
                rp.row0 = (size_t)c0 * n;
                rp.cos_step = n;
                rp.ncols = (int)(gc * kc);
                TRY(dispatch_row(ctx, pl.b, RM_BITREV, rp));
            }
        }
        return GL_OK;
    }
    const u64 wN = root_of_unity((uint32_t)(log_n + rate_bits));
    // group-outer / coset-inner
    const uint32_t G = log_n > NTT_MAX_LOG_PASS ? group_cols(ctx, log_n, ncols) : ncols;
    for (uint32_t g0 = 0; g0 < ncols; g0 += G) {
        const uint32_t gc = (ncols - g0 < G) ? ncols - g0 : G;
        for (int c = 0; c < ncos; c++) {
            const u64 s = mul(base_shift, gl::pow(wN, bitrev32((uint32_t)c, (uint32_t)rate_bits)));
            TRY(ntt_forward(ctx, coeffs + (size_t)g0 * coeff_stride, coeff_stride, lde + (size_t)g0 * lde_stride, lde_stride,
                            (size_t)c * n, log_n, gc, RM_BITREV, false, 1, s));
        }
    }
    return GL_OK;
}
