// gl_ntt.cuh -- batched Goldilocks NTT, multi-pass (n = 2^(a1 [+ a2] + b)), every pass a two-step radix-(<=32)
// in-register transform with ONE shared-memory exchange.
//
// Replaces (reference, CPU): fft_classic / ifft_with_options      field/src/fft.rs:68-202
//                            coset_fft_with_options, lde          field/src/polynomial/mod.rs:199-201,280-293
//                            lde_values + transpose + bit-reverse plonky2/src/fri/oracle.rs:97-98,114-139
//
// Decomposition (four-/six-step without explicit transposes), for two passes n = R * C:
//   X[k1 + R*k2] = sum_{j2<C} w_n^{j2*k1} w_C^{j2*k2} ( sum_{j1<R} x[j1*C + j2] w_R^{j1*k1} )
// * column pass ("A", strided): a CTA owns T adjacent j2 (T*8-byte global segments) and all R = 2^LOG values of
//   j1; writes Y[p][j2] * w_n^{k1*j2} with p = bitrev(k1) (the in-place DIF order).
// * row pass ("B", contiguous): TPT threads own one row of C = 2^LOG contiguous elements and store either
//     - bit-reversed   out[row_base + bitrev(k2)]  -- the LDE: with column-major leaves this IS the reference's
//                       leaf order (transpose + reverse_index_bits, oracle.rs:97-98), for even LOG transposed per line through
//                       shared memory so that each store instruction writes adjacent words, or
//     - natural order  out[k1 + R*k2] (NTT / iNTT API), gathered through shared memory so that a CTA writes
//                       segments of adjacent k1 (optional index reversal for the inverse, fft.rs:80-90).
//   Three passes (n > 2^20) run the column pass twice (the second time inside every row of the first).
// Inside a pass, 2^LOG = E * TPT with E = 2^ceil(LOG/2) <= 32 values per thread:
//   step 1: radix-E DIF over the high index bits in registers (lazy 3-word butterflies with shift twiddles,
//           gl_lazy.cuh; w_32 = 2^6), one general multiply by  scale * base^t * w_{2^LOG}^{t * k}  per element,
//   exchange through shared memory (padded pitch: conflict-free 64-bit accesses; a warp-local __syncwarp for rows),
//   step 2: radix-TPT DIF over the low bits; element (q, j) is the output of bit-reversed position q*TPT + j.
// Coset scaling s^j of the forward coset NTT (j = (t + TPT*q)*C + j2) costs ONE extra multiply per element:
// (s^(C*TPT))^q are per-register constants, (s^C)^t is folded into the step table and s^j2 into the post table.
//
// Every per-thread phase below is a plain function so that tests/emu can run the same code on the CPU
// (threads as a loop, barriers between phases) to check indexing and the table formulas.
#pragma once
#include "gl_lazy.cuh"

namespace gl {

constexpr int NTT_MAX_LOG_PASS = 10;  // largest single pass: 32 x 32
constexpr int NTT_COL_MIN_LOG = 5;    // smallest strided pass the planner uses

GL_HD constexpr int ntt_r2(int log) { return log / 2; }
GL_HD constexpr int ntt_r1(int log) { return log - log / 2; }

template <int LOG>
struct PassCfg {
    static constexpr int R1 = ntt_r1(LOG), R2 = ntt_r2(LOG);
    static constexpr int E = 1 << R1, TPT = 1 << R2, NSUB = E / TPT;  // NSUB = 1 or 2 sub-transforms per thread in step 2
    // ---- row pass: TPT threads per row, rows packed into warps; LPC rows ("lines") per CTA
    static constexpr int ROW_THREADS = (TPT * 8 < 32) ? 32 : TPT * 8;
    static constexpr int LPC = ROW_THREADS / TPT;
    // resident CTAs per SM the kernels are compiled for: 512 threads/SM (128 registers) when a thread holds 32 lazy
    // values, 768 threads/SM (80 registers) below
    static constexpr int ROW_MIN_BLOCKS = (E >= 32 ? 512 : 768) / ROW_THREADS;
    static constexpr int ROW_PITCH = TPT + 1;                 // u64 words: odd => conflict-free exchange
    static constexpr int ROW_S_WORDS = E * ROW_PITCH;         // exchange buffer per line
    static constexpr int GATHER_PITCH = (1 << LOG) + 2;       // natural-order gather tile: line pitch = 2 (mod 16)
    // ---- column pass: T adjacent columns-of-the-matrix per CTA
    static constexpr int T = (256 / TPT) < 8 ? 8 : (256 / TPT);
    static constexpr int COL_THREADS = T * TPT;
    static constexpr int COL_MIN_BLOCKS = (E >= 32 ? 512 : 768) / COL_THREADS;
    static constexpr int COL_QPITCH = TPT * T + 8;            // words per q-row: 8 (mod 16) => conflict-free when T = 8
    static constexpr int COL_S_WORDS = E * COL_QPITCH;
};
GL_HD constexpr size_t ntt_row_smem_bytes(int log, bool natural) {
    const int r1 = ntt_r1(log), r2 = ntt_r2(log), E = 1 << r1, TPT = 1 << r2;
    const int threads = (TPT * 8 < 32) ? 32 : TPT * 8, lpc = threads / TPT;
    const size_t s = (size_t)lpc * E * (TPT + 1), g = natural ? (size_t)lpc * ((1 << log) + 2) : 0;
    return (s > g ? s : g) * 8;
}
GL_HD constexpr size_t ntt_col_smem_bytes(int log) {
    const int r1 = ntt_r1(log), r2 = ntt_r2(log), E = 1 << r1, TPT = 1 << r2;
    const int T = (256 / TPT) < 8 ? 8 : (256 / TPT);
    return (size_t)E * (TPT * T + 8) * 8;
}

// ---------------------------------------------------------------- table entries
// step table of a 2^LOG pass: tw[q*TPT + t] = scale * base^t * w_{2^LOG}^(t * bitrev_R1(q))
GL_HD uint64_t table_step_entry(int log, uint32_t idx, uint64_t scale, uint64_t base) {
    const int r1 = ntt_r1(log), r2 = ntt_r2(log);
    const uint32_t t = idx & ((1u << r2) - 1), q = idx >> r2;
    const uint64_t k = bitrev32(q, (uint32_t)r1);
    uint64_t v = pow(root_of_unity((uint32_t)log), k * t);
    if (base != 1) v = mul(v, pow(base, t));
    if (scale != 1) v = mul(v, scale);
    return v;
}
// post table of a column pass with R = 2^a rows over C = 2^b columns: twa[p*C + j2] = w_{R*C}^(bitrev_a(p) * j2) * base^j2
GL_HD uint64_t table_post_entry(int a, int b, size_t idx, uint64_t base) {
    const size_t p = idx >> b, j2 = idx & (((size_t)1 << b) - 1);
    const uint64_t k1 = bitrev32((uint32_t)p, (uint32_t)a);
    uint64_t v = pow(root_of_unity((uint32_t)(a + b)), k1 * j2);
    if (base != 1) v = mul(v, pow(base, j2));
    return v;
}

// ---------------------------------------------------------------- shared step code
// step 1 of a pass on one thread: x[q] (q < E) natural -> y[q] = DFT_E(x)[bitrev(q)] * tw[q*TPT + t], normalised u64.
// uq: optional per-register pre-scale (coset), uq[0] unused. tw_full: multiply slot 0 too (scale/base non-trivial).
template <int LOG>
GL_HD void pass_step1(uint64_t* x, const uint64_t* tw, const uint64_t* uq, bool tw_full, int t) {
    using Cf = PassCfg<LOG>;
    L3 r[Cf::E];
#pragma unroll
    for (int q = 0; q < Cf::E; q++) {
        uint64_t v = x[q];
        if (uq && q) v = mul(v, uq[q]);
        r[q] = l3_from(v);
    }
    dft_lazy<Cf::R1>(r);
#pragma unroll
    for (int q = 0; q < Cf::E; q++) {
        uint64_t y = l3_norm(r[q]);
        if (Cf::R2 > 0 && (q || tw_full)) y = mul(y, tw[q * Cf::TPT + t]);
        if (Cf::R2 == 0 && tw_full) y = mul(y, tw[0]);  // 2-point pass: only the scale (t = 0)
        x[q] = y;
    }
}
// step 2 on one thread: z[j] (j < TPT) natural -> z[j] = DFT_TPT(z)[bitrev(j)], normalised u64 (not canonical)
template <int LOG>
GL_HD void pass_step2(uint64_t* z) {
    using Cf = PassCfg<LOG>;
    L3 r[Cf::TPT];
#pragma unroll
    for (int j = 0; j < Cf::TPT; j++) r[j] = l3_from(z[j]);
    dft_lazy<Cf::R2>(r);
#pragma unroll
    for (int j = 0; j < Cf::TPT; j++) z[j] = l3_norm(r[j]);
}

// ---------------------------------------------------------------- column pass
struct ColPass {
    const uint64_t* in;    // unit (col, rb): in + col*in_stride + rb*(R*C); element (j1, j2) at [j1*C + j2]
    uint64_t* out;         // same addressing with out_stride; element (p, j2) at [p*C + j2]  (may alias `in`)
    size_t in_stride, out_stride;
    const uint64_t* tw;    // step table, R entries
    const uint64_t* twa;   // post table, R*C entries
    int log_c;             // log2 C
    int log_rb;            // log2 (row blocks per column): 0 except for the middle pass of a three-pass plan
    int tw_full;
    int has_uq;
    uint64_t uq[32];
};
template <int LOG>
GL_HD void col_unit(const ColPass& cp, int blk, size_t& in_off, size_t& out_off, int& tile) {
    using Cf = PassCfg<LOG>;
    const int tiles = (1 << cp.log_c) / Cf::T;
    tile = blk % tiles;
    const int unit = blk / tiles;
    const size_t rb = (size_t)unit & (((size_t)1 << cp.log_rb) - 1), col = (size_t)unit >> cp.log_rb;
    const size_t blk_words = (size_t)1 << (LOG + cp.log_c);
    in_off = col * cp.in_stride + rb * blk_words;
    out_off = col * cp.out_stride + rb * blk_words;
}
// phase 1a: global loads (tid < COL_THREADS); phase 1b: step 1 + write the exchange tile
template <int LOG>
GL_HD void col_load_at(const ColPass& cp, size_t in_off, int tile, int tid, uint64_t* x) {
    using Cf = PassCfg<LOG>;
    const int tt = tid % Cf::T, t = tid / Cf::T;
    const size_t C = (size_t)1 << cp.log_c;
    const uint64_t* src = cp.in + in_off + (size_t)tile * Cf::T + tt;
#pragma unroll
    for (int q = 0; q < Cf::E; q++) x[q] = src[(size_t)(t + Cf::TPT * q) * C];
}
template <int LOG>
GL_HD void col_load(const ColPass& cp, int blk, int tid, uint64_t* x) {
    size_t in_off, out_off;
    int tile;
    col_unit<LOG>(cp, blk, in_off, out_off, tile);
    col_load_at<LOG>(cp, in_off, tile, tid, x);
}

// ---------------------------------------------------------------- column pass over several cosets at once
// The first column pass of a coset LDE for 2^log_cos cosets of the same coefficient columns in one launch. Only the
// coset's pre-weights and its two tables differ between cosets; `cp` holds everything else (cp.tw, cp.twa and cp.uq
// unused). Coset c of matrix column col goes to out + (col * 2^log_cos + c) * out_stride.
constexpr int COL_LOG_MAX_COSETS = 3;  // 8 cosets: the parameter block stays under 4 KiB
struct ColCosets {
    ColPass cp;
    int log_cos;
    int ncols;
    const uint64_t* tw[1 << COL_LOG_MAX_COSETS];
    const uint64_t* twa[1 << COL_LOG_MAX_COSETS];
    uint64_t uq[1 << COL_LOG_MAX_COSETS][32];
};
// CTA blk -> (coset c, matrix column col, tile), cosets fastest, then columns: the CTAs that read one coefficient tile
// run side by side, so that tile can come from HBM once and from L2 for the other cosets, and the CTAs that read one
// tile's rows of a coset's post table run within a few waves of each other.
template <int LOG>
GL_HD void col_cosets_unit(const ColCosets& cc, int blk, int& c, size_t& in_off, size_t& out_off, int& tile) {
    c = blk & ((1 << cc.log_cos) - 1);
    const int rest = blk >> cc.log_cos;
    const size_t col = (size_t)(rest % cc.ncols);
    tile = rest / cc.ncols;
    in_off = col * cc.cp.in_stride;
    out_off = ((col << cc.log_cos) + c) * cc.cp.out_stride;
}
template <int LOG>
GL_HD int col_cosets_blocks(const ColCosets& cc) {
    return (cc.ncols << cc.log_cos) * (int)(((size_t)1 << cc.cp.log_c) / PassCfg<LOG>::T);
}
template <int LOG>
GL_HD void col_phase1(const ColPass& cp, uint64_t* S, int blk, int tid, uint64_t* x) {
    using Cf = PassCfg<LOG>;
    const int tt = tid % Cf::T, t = tid / Cf::T;
    size_t in_off, out_off;
    int tile;
    col_unit<LOG>(cp, blk, in_off, out_off, tile);
    const size_t C = (size_t)1 << cp.log_c;
    pass_step1<LOG>(x, cp.tw, cp.has_uq ? cp.uq : nullptr, cp.tw_full != 0, t);
    if (Cf::R2 == 0) {  // single step: x[q] is the output of position q
        uint64_t* dst = cp.out + out_off + (size_t)tile * Cf::T + tt;
        const uint64_t* twa = cp.twa + (size_t)tile * Cf::T + tt;
#pragma unroll
        for (int q = 0; q < Cf::E; q++) dst[(size_t)q * C] = mul(x[q], twa[(size_t)q * C]);
        return;
    }
#pragma unroll
    for (int q = 0; q < Cf::E; q++) S[q * Cf::COL_QPITCH + t * Cf::T + tt] = x[q];
}
// phase 2 (after a CTA barrier), in three parts so that the kernel can fetch the post twiddles asynchronously while
// step 2 computes:  (a) exchange tile -> registers,  (b) step 2,  (c) post twiddle + store.
// Twiddle of output (m, j) of thread tid: twa[p*C] with p = (t + TPT*m)*TPT + j; col_twiddle_slot() is where the
// kernel parks it in shared memory (thread-private slots, consecutive threads -> consecutive words).
template <int LOG>
GL_HD void col_phase2_load(const uint64_t* S, int tid, uint64_t* z /* [NSUB * TPT] */) {
    using Cf = PassCfg<LOG>;
    const int tt = tid % Cf::T, t = tid / Cf::T;
#pragma unroll
    for (int m = 0; m < Cf::NSUB; m++) {
        const int q = t + Cf::TPT * m;
#pragma unroll
        for (int j = 0; j < Cf::TPT; j++) z[m * Cf::TPT + j] = S[q * Cf::COL_QPITCH + j * Cf::T + tt];
    }
}
template <int LOG>
GL_HD void col_phase2_dft(uint64_t* z) {
    using Cf = PassCfg<LOG>;
#pragma unroll
    for (int m = 0; m < Cf::NSUB; m++) pass_step2<LOG>(z + m * Cf::TPT);
}
template <int LOG>
GL_HD int col_twiddle_slot(int tid, int i) { return i * PassCfg<LOG>::COL_THREADS + tid; }
template <int LOG>
GL_HD const uint64_t* col_twiddle_src(const ColPass& cp, int blk, int tid, int i) {
    using Cf = PassCfg<LOG>;
    const int tt = tid % Cf::T, t = tid / Cf::T;
    size_t in_off, out_off;
    int tile;
    col_unit<LOG>(cp, blk, in_off, out_off, tile);
    const int m = i / Cf::TPT, j = i % Cf::TPT;
    const size_t p = (size_t)(t + Cf::TPT * m) * Cf::TPT + j;
    return cp.twa + (p << cp.log_c) + (size_t)tile * Cf::T + tt;
}
// tws: the E twiddles of this thread, that of output (m, j) at tws[m * stride_m + j * stride_j]
template <int LOG>
GL_HD void col_phase2_store(const ColPass& cp, int blk, int tid, const uint64_t* z, const uint64_t* tws, size_t stride_j,
                            size_t stride_m) {
    using Cf = PassCfg<LOG>;
    const int tt = tid % Cf::T, t = tid / Cf::T;
    size_t in_off, out_off;
    int tile;
    col_unit<LOG>(cp, blk, in_off, out_off, tile);
    const size_t C = (size_t)1 << cp.log_c;
    uint64_t* dst = cp.out + out_off + (size_t)tile * Cf::T + tt;
#pragma unroll
    for (int m = 0; m < Cf::NSUB; m++) {
#pragma unroll
        for (int j = 0; j < Cf::TPT; j++) {
            const int i = m * Cf::TPT + j;
            const size_t p = (size_t)(t + Cf::TPT * m) * Cf::TPT + j;
            dst[p * C] = mul(z[i], tws[m * stride_m + j * stride_j]);
        }
    }
}
// the whole phase on one thread, twiddles straight from the table (tests/emu; the kernel interleaves the parts)
template <int LOG>
GL_HD void col_phase2(const ColPass& cp, const uint64_t* S, int blk, int tid) {
    using Cf = PassCfg<LOG>;
    if (Cf::R2 == 0) return;
    uint64_t z[Cf::E];
    col_phase2_load<LOG>(S, tid, z);
    col_phase2_dft<LOG>(z);
    // consecutive outputs of a thread are rows p, p+1, ...: their twiddles are 2^log_c words apart in the table
    const size_t C = (size_t)1 << cp.log_c;
    col_phase2_store<LOG>(cp, blk, tid, z, col_twiddle_src<LOG>(cp, blk, tid, 0), C, (size_t)Cf::TPT * Cf::TPT * C);
}

// ---------------------------------------------------------------- row pass
enum RowMode { RM_BITREV = 0, RM_NATURAL = 1 };
struct RowPass {
    const uint64_t* in;    // line (col, prow): in + col*in_stride + (prow << LOG)
    uint64_t* out;
    size_t in_stride, out_stride;
    const uint64_t* tw;    // step table, 2^LOG entries
    int log_r;             // log2 (rows per column) = log2(n) - LOG
    int ncols;
    int tw_full;
    int has_uq;
    int reverse;           // RM_NATURAL: write to (n - k) mod n   (ifft index reversal, fft.rs:80-90)
    size_t row0;           // RM_BITREV: offset added to the output position (first row of this coset block)
    int log_cos;           // RM_BITREV: input column v is coset (v mod 2^log_cos) of output column v >> log_cos,
    size_t cos_step;       //   which starts cos_step words after the previous coset's
    int n_peer;           // RM_NATURAL: additional destinations with the same addressing as `out` (peer GPUs'
    uint64_t* out_peer[7]; // coefficient buffers mapped over NVLink: the store IS the all-gather)
    uint64_t uq[32];
};
// line l of CTA blk -> (col, prow, kbase). RM_BITREV enumerates rows in storage order; RM_NATURAL enumerates them by
// the natural low index kbase (adjacent lines of a CTA = adjacent output addresses), prow = bitrev(kbase).
template <int LOG, int MODE>
GL_HD bool row_line(const RowPass& rp, int blk, int l, size_t& col, size_t& prow, size_t& kbase) {
    using Cf = PassCfg<LOG>;
    const size_t L = (size_t)blk * Cf::LPC + l;
    const size_t R = (size_t)1 << rp.log_r;
    col = L >> rp.log_r;
    const size_t low = L & (R - 1);
    if (MODE == RM_BITREV) {
        prow = low;
        kbase = 0;
    } else {
        kbase = low;
        prow = rp.log_r ? (size_t)bitrev32((uint32_t)low, (uint32_t)rp.log_r) : 0;
    }
    return col < (size_t)rp.ncols;
}
template <int LOG>
GL_HD int row_blocks(const RowPass& rp) {
    using Cf = PassCfg<LOG>;
    const size_t lines = (size_t)rp.ncols << rp.log_r;
    return (int)((lines + Cf::LPC - 1) / Cf::LPC);
}
// phase 1a: global loads; phase 1b: step 1, write this line's exchange buffer (lines of a warp are independent:
// warp-level barrier). For LOG with R2 == 0 the outputs stay in x[] (returned) and phase 2 is skipped.
template <int LOG, int MODE>
GL_HD void row_load(const RowPass& rp, int blk, int tid, uint64_t* x) {
    using Cf = PassCfg<LOG>;
    const int l = tid / Cf::TPT, t = tid % Cf::TPT;
    size_t col, prow, kbase;
    const bool live = row_line<LOG, MODE>(rp, blk, l, col, prow, kbase);
    const uint64_t* src = rp.in + col * rp.in_stride + (prow << LOG) + t;
#pragma unroll
    for (int q = 0; q < Cf::E; q++) x[q] = live ? src[Cf::TPT * q] : 0;
}
template <int LOG, int MODE>
GL_HD void row_phase1(const RowPass& rp, uint64_t* S, int blk, int tid, uint64_t* x) {
    using Cf = PassCfg<LOG>;
    const int l = tid / Cf::TPT, t = tid % Cf::TPT;
    pass_step1<LOG>(x, rp.tw, rp.has_uq ? rp.uq : nullptr, rp.tw_full != 0, t);
    if (Cf::R2 == 0) return;
    uint64_t* Sl = S + (size_t)l * Cf::ROW_S_WORDS;
#pragma unroll
    for (int q = 0; q < Cf::E; q++) Sl[q * Cf::ROW_PITCH + t] = x[q];
}
// natural index of the element at bit-reversed position pos = q*TPT + j
template <int LOG>
GL_HD uint32_t row_natural_index(int q, int j) {
    using Cf = PassCfg<LOG>;
    return bitrev32((uint32_t)q, Cf::R1) + (uint32_t)Cf::E * (Cf::R2 ? bitrev32((uint32_t)j, Cf::R2) : 0u);
}
// phase 2: step 2 and the output of RM_BITREV (canonical u64, pairs of adjacent positions), or the gather tile of
// RM_NATURAL (G may alias S: the caller puts a CTA barrier between the reads of S and the writes of G).
template <int LOG>
GL_HD void row_phase2_load(const uint64_t* S, int tid, int m, uint64_t* z) {
    using Cf = PassCfg<LOG>;
    const int l = tid / Cf::TPT, t = tid % Cf::TPT;
    const uint64_t* Sl = S + (size_t)l * Cf::ROW_S_WORDS;
    const int q = t + Cf::TPT * m;
#pragma unroll
    for (int j = 0; j < Cf::TPT; j++) z[j] = Sl[q * Cf::ROW_PITCH + j];
}
// first output word of row prow of input column col (RM_BITREV)
template <int LOG>
GL_HD uint64_t* row_bitrev_dst(const RowPass& rp, size_t col, size_t prow) {
    const size_t cos = col & (((size_t)1 << rp.log_cos) - 1);
    return rp.out + (col >> rp.log_cos) * rp.out_stride + rp.row0 + cos * rp.cos_step + (prow << LOG);
}
template <int LOG>
GL_HD void row_store_bitrev(const RowPass& rp, int blk, int tid, int m, const uint64_t* z) {
    using Cf = PassCfg<LOG>;
    const int l = tid / Cf::TPT, t = tid % Cf::TPT;
    size_t col, prow, kbase;
    if (!row_line<LOG, RM_BITREV>(rp, blk, l, col, prow, kbase)) return;
    uint64_t* dst = row_bitrev_dst<LOG>(rp, col, prow);
    if constexpr (Cf::R2 == 0) {  // z = x[q]: position q, this thread holds the whole line
#pragma unroll
        for (int q = 0; q < Cf::E; q++) dst[q] = canon(z[q]);
    } else {
        const int q = t + Cf::TPT * m;
        uint64_t* d = dst + (size_t)q * Cf::TPT;
#if defined(__CUDA_ARCH__)
#pragma unroll
        for (int j = 0; j < Cf::TPT; j += 2) {
            ulonglong2 v;
            v.x = canon(z[j]);
            v.y = canon(z[j + 1]);
            *reinterpret_cast<ulonglong2*>(d + j) = v;  // 16-byte aligned: q*TPT + j even, rows 8*2^LOG bytes
        }
#else
        for (int j = 0; j < Cf::TPT; j++) d[j] = canon(z[j]);
#endif
    }
}
// RM_BITREV of a single-step-2 line (E == TPT) through the line's exchange buffer, in two parts with a warp barrier
// between them: thread t holds positions t*TPT + j (row_stage_bitrev writes them to row t of the buffer), then stores
// positions k*TPT + t (column t), so that every store instruction of a line writes TPT adjacent words. Stored from the
// registers, each 128-bit store instruction of a warp writes 16 bytes at 32 places 256 bytes apart.
template <int LOG>
GL_HD void row_stage_bitrev(uint64_t* S, int tid, const uint64_t* z) {
    using Cf = PassCfg<LOG>;
    static_assert(Cf::E == Cf::TPT, "one step-2 transform per thread");
    const int l = tid / Cf::TPT, t = tid % Cf::TPT;
    uint64_t* Sl = S + (size_t)l * Cf::ROW_S_WORDS;
#pragma unroll
    for (int j = 0; j < Cf::TPT; j++) Sl[t * Cf::ROW_PITCH + j] = canon(z[j]);
}
template <int LOG>
GL_HD void row_store_bitrev_staged(const RowPass& rp, const uint64_t* S, int blk, int tid) {
    using Cf = PassCfg<LOG>;
    const int l = tid / Cf::TPT, t = tid % Cf::TPT;
    size_t col, prow, kbase;
    if (!row_line<LOG, RM_BITREV>(rp, blk, l, col, prow, kbase)) return;
    uint64_t* dst = row_bitrev_dst<LOG>(rp, col, prow) + t;
    const uint64_t* Sl = S + (size_t)l * Cf::ROW_S_WORDS + t;
#pragma unroll
    for (int k = 0; k < Cf::E; k++) dst[(size_t)k * Cf::TPT] = Sl[k * Cf::ROW_PITCH];
}
template <int LOG>
GL_HD void row_gather_write(uint64_t* G, int tid, int m, const uint64_t* z) {
    using Cf = PassCfg<LOG>;
    const int l = tid / Cf::TPT, t = tid % Cf::TPT;
    uint64_t* Gl = G + (size_t)l * Cf::GATHER_PITCH;
    if (Cf::R2 == 0) {
#pragma unroll
        for (int q = 0; q < Cf::E; q++) Gl[row_natural_index<LOG>(q, 0)] = canon(z[q]);
        return;
    }
    const int q = t + Cf::TPT * m;
#pragma unroll
    for (int j = 0; j < Cf::TPT; j++) Gl[row_natural_index<LOG>(q, j)] = canon(z[j]);
}
// phase 3 (RM_NATURAL, after a CTA barrier): G[line][k2] -> out[col][kbase + R*k2] (or the reversed index)
template <int LOG>
GL_HD void row_store_natural(const RowPass& rp, const uint64_t* G, int blk, int tid, int nthreads) {
    using Cf = PassCfg<LOG>;
    const size_t R = (size_t)1 << rp.log_r, n = R << LOG;
    for (int e = tid; e < Cf::LPC * (1 << LOG); e += nthreads) {
        int l, k2;
        if (rp.log_r) {  // adjacent lines = adjacent addresses: lines fastest
            l = e % Cf::LPC;
            k2 = e / Cf::LPC;
        } else {         // single pass: a line is contiguous in k2
            k2 = e & ((1 << LOG) - 1);
            l = e >> LOG;
        }
        size_t col, prow, kbase;
        if (!row_line<LOG, RM_NATURAL>(rp, blk, l, col, prow, kbase)) continue;
        size_t k = kbase + ((size_t)k2 << rp.log_r);
        if (rp.reverse) k = (n - k) & (n - 1);
        const uint64_t v = G[(size_t)l * Cf::GATHER_PITCH + k2];
        const size_t at = col * rp.out_stride + k;
        rp.out[at] = v;
        for (int p = 0; p < rp.n_peer; p++) rp.out_peer[p][at] = v;
    }
}

// ---------------------------------------------------------------- plan
// n = 2^log_n as up to three passes: a1 (strided), a2 (strided inside the rows of the first), b (contiguous).
struct NttPlan {
    int a1, a2, b;
};
GL_HD NttPlan ntt_plan(int log_n) {
    NttPlan p{0, 0, log_n};
    if (log_n <= NTT_MAX_LOG_PASS) return p;
    if (log_n <= 2 * NTT_MAX_LOG_PASS) {
        p.b = (log_n + 1) / 2;
        p.a1 = log_n - p.b;
        return p;
    }
    p.b = (log_n + 2) / 3;
    p.a2 = (log_n - p.b + 1) / 2;
    p.a1 = log_n - p.b - p.a2;
    return p;
}


// ---------------------------------------------------------------- job = the passes of one forward transform
// Everything except device pointers: which tables each pass needs (TableReq) and the scalar parameters of the
// pass descriptors. Shared by the CUDA host code (tables from the per-context cache) and tests/emu (tables computed
// on the CPU), so the orchestration arithmetic -- coset bases, uq constants, scale placement -- is tested without a GPU.
struct TableReq {
    int a, b;              // step table: log = a (b unused); post table: (a, b)
    uint64_t scale, base;
};
struct NttJob {
    NttPlan pl;
    ColPass c1, c2;        // c1 used iff pl.a1, c2 iff pl.a2
    RowPass rp;
    TableReq c1_step, c1_post, c2_step, c2_post, row_step;
};
// Forward transform of size 2^log_n on the coset shift*<w_n> (shift = 1: none), outputs multiplied by `scale`.
inline void ntt_make_job(int log_n, NttPlan pl, uint64_t scale, uint64_t shift, NttJob& job) {
    job = NttJob{};
    job.pl = pl;
    const bool coset = canon(shift) != 1;
    const uint64_t one = 1;
    RowPass& rp = job.rp;
    rp.log_r = log_n - pl.b;
    auto fill_uq = [](uint64_t* uq, int log_pass, uint64_t sq) {
        const int E = 1 << ntt_r1(log_pass);
        uint64_t acc = 1;
        for (int q = 0; q < E; q++, acc = mul(acc, sq)) uq[q] = canon(acc);
    };
    if (pl.a1 == 0) {  // single pass: j = t + TPT*q
        job.row_step = TableReq{pl.b, 0, scale, coset ? shift : one};
        rp.tw_full = (canon(scale) != 1 || coset) ? 1 : 0;
        rp.has_uq = coset ? 1 : 0;
        if (coset) fill_uq(rp.uq, pl.b, pow(shift, (uint64_t)1 << ntt_r2(pl.b)));
        return;
    }
    const int c1_log = log_n - pl.a1;  // j = j1*C1 + j', j1 = t + TPT*q
    ColPass& c1 = job.c1;
    c1.log_c = c1_log;
    c1.log_rb = 0;
    job.c1_step = TableReq{pl.a1, 0, one, coset ? pow(shift, (uint64_t)1 << c1_log) : one};
    job.c1_post = TableReq{pl.a1, c1_log, one, coset ? shift : one};
    c1.tw_full = coset ? 1 : 0;
    c1.has_uq = coset ? 1 : 0;
    if (coset) fill_uq(c1.uq, pl.a1, pow(shift, ((uint64_t)1 << ntt_r2(pl.a1)) << c1_log));
    if (pl.a2) {
        ColPass& c2 = job.c2;
        c2.log_c = pl.b;
        c2.log_rb = pl.a1;
        job.c2_step = TableReq{pl.a2, 0, one, one};
        job.c2_post = TableReq{pl.a2, pl.b, one, one};
    }
    job.row_step = TableReq{pl.b, 0, scale, one};
    rp.tw_full = canon(scale) != 1 ? 1 : 0;
}
// Cosets c0 .. c0 + 2^log_kc - 1 of the coset LDE of size-2^log_n columns on base_shift * <w_N>, N = 2^(log_n +
// rate_bits), coset c on base_shift * w_N^bitrev(c) <w_n> (lde_columns in gl_ntt_host.cuh), as ONE job of a multi-pass
// plan: cc is the first column pass over all of them, steps[c] / posts[c] its tables; the a2 pass and the row pass do
// not depend on the coset and run over all 2^log_kc cosets of every column as job.c2 and job.rp.
inline void lde_make_cosets_job(int log_n, NttPlan pl, int rate_bits, uint64_t base_shift, int c0, int log_kc,
                                NttJob& job, ColCosets& cc, TableReq* steps, TableReq* posts) {
    const uint64_t wN = root_of_unity((uint32_t)(log_n + rate_bits));
    cc = ColCosets{};
    for (int c = 0; c < (1 << log_kc); c++) {
        const uint64_t s = mul(base_shift, pow(wN, bitrev32((uint32_t)(c0 + c), (uint32_t)rate_bits)));
        NttJob jc;
        ntt_make_job(log_n, pl, 1, s, jc);
        if (c == 0) job = jc;
        steps[c] = jc.c1_step;
        posts[c] = jc.c1_post;
        for (int q = 0; q < 32; q++) cc.uq[c][q] = jc.c1.has_uq ? jc.c1.uq[q] : 1;  // s = 1: no coset, weights 1
    }
    cc.cp = job.c1;
    cc.cp.has_uq = cc.cp.tw_full = 1;  // one pair of flags for every coset: s = 1 multiplies by ones
    cc.log_cos = log_kc;
    job.rp.log_cos = log_kc;
}
template <int LOG>
GL_HD int col_blocks(const ColPass& cp, size_t ncols) {
    return (int)((ncols << cp.log_rb) * (((size_t)1 << cp.log_c) / PassCfg<LOG>::T));
}

}  // namespace gl
