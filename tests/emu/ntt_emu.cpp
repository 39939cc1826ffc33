// CPU emulation of the CUDA NTT pass code (threads as loops, phases as barriers) checked against the oracle.
// The SAME source that the sm_90a kernels compile (gl_ntt.cuh phase functions, ntt_make_job) runs here with the
// host formulation of the lazy field type. Test infrastructure: built and run by tests/test_emu.py.
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../../plonky2_b200/csrc/gl_ntt.cuh"
#include "../../oracle/gl_oracle.h"
using namespace gl;

template <int LOG>
void emu_col(const ColPass& cp, size_t ncols) {
    using Cf = PassCfg<LOG>;
    std::vector<uint64_t> S(Cf::COL_S_WORDS);
    std::vector<std::vector<uint64_t>> x(Cf::COL_THREADS, std::vector<uint64_t>(Cf::E));
    const int nblocks = col_blocks<LOG>(cp, ncols);
    for (int blk = 0; blk < nblocks; blk++) {
        for (int tid = 0; tid < Cf::COL_THREADS; tid++) col_load<LOG>(cp, blk, tid, x[tid].data());
        for (int tid = 0; tid < Cf::COL_THREADS; tid++) col_phase1<LOG>(cp, S.data(), blk, tid, x[tid].data());
        for (int tid = 0; tid < Cf::COL_THREADS; tid++) col_phase2<LOG>(cp, S.data(), blk, tid);
    }
}
template <int LOG, int MODE>
void emu_row(const RowPass& rp) {
    using Cf = PassCfg<LOG>;
    const int NT = Cf::ROW_THREADS;
    std::vector<uint64_t> S(ntt_row_smem_bytes(LOG, MODE == RM_NATURAL) / 8 + 8);
    std::vector<std::vector<uint64_t>> x(NT, std::vector<uint64_t>(Cf::E));
    std::vector<std::vector<uint64_t>> z(NT, std::vector<uint64_t>(Cf::E));
    const int nblocks = row_blocks<LOG>(rp);
    for (int blk = 0; blk < nblocks; blk++) {
        for (int tid = 0; tid < NT; tid++) row_load<LOG, MODE>(rp, blk, tid, x[tid].data());
        for (int tid = 0; tid < NT; tid++) row_phase1<LOG, MODE>(rp, S.data(), blk, tid, x[tid].data());
        if (Cf::R2 == 0) {
            if (MODE == RM_BITREV) {
                for (int tid = 0; tid < NT; tid++) row_store_bitrev<LOG>(rp, blk, tid, 0, x[tid].data());
            } else {
                for (int tid = 0; tid < NT; tid++) row_gather_write<LOG>(S.data(), tid, 0, x[tid].data());
                for (int tid = 0; tid < NT; tid++) row_store_natural<LOG>(rp, S.data(), blk, tid, NT);
            }
            continue;
        }
        for (int tid = 0; tid < NT; tid++)
            for (int m = 0; m < Cf::NSUB; m++) {
                row_phase2_load<LOG>(S.data(), tid, m, z[tid].data() + m * Cf::TPT);
                pass_step2<LOG>(z[tid].data() + m * Cf::TPT);
            }
        if (MODE == RM_BITREV) {
            for (int tid = 0; tid < NT; tid++)
                for (int m = 0; m < Cf::NSUB; m++) row_store_bitrev<LOG>(rp, blk, tid, m, z[tid].data() + m * Cf::TPT);
        } else {
            for (int tid = 0; tid < NT; tid++)
                for (int m = 0; m < Cf::NSUB; m++) row_gather_write<LOG>(S.data(), tid, m, z[tid].data() + m * Cf::TPT);
            for (int tid = 0; tid < NT; tid++) row_store_natural<LOG>(rp, S.data(), blk, tid, NT);
        }
    }
}
#define DISPATCH(LOGV, CALL)                                                   \
    switch (LOGV) {                                                            \
        case 1: { constexpr int L = 1; CALL; } break;                          \
        case 2: { constexpr int L = 2; CALL; } break;                          \
        case 3: { constexpr int L = 3; CALL; } break;                          \
        case 4: { constexpr int L = 4; CALL; } break;                          \
        case 5: { constexpr int L = 5; CALL; } break;                          \
        case 6: { constexpr int L = 6; CALL; } break;                          \
        case 7: { constexpr int L = 7; CALL; } break;                          \
        case 8: { constexpr int L = 8; CALL; } break;                          \
        case 9: { constexpr int L = 9; CALL; } break;                          \
        case 10: { constexpr int L = 10; CALL; } break;                        \
        default: abort();                                                      \
    }

static std::vector<uint64_t> step_table(const TableReq& r) {
    std::vector<uint64_t> t(((size_t)1 << r.a) < 2 ? 2 : ((size_t)1 << r.a));
    for (size_t j = 0; j < ((size_t)1 << r.a); j++) t[j] = table_step_entry(r.a, (uint32_t)j, r.scale, r.base);
    return t;
}
static std::vector<uint64_t> post_table(const TableReq& r) {
    std::vector<uint64_t> t((size_t)1 << (r.a + r.b));
    for (size_t j = 0; j < t.size(); j++) t[j] = table_post_entry(r.a, r.b, j, r.base);
    return t;
}
static uint64_t rnd(uint64_t& st) {
    st += 0x9E3779B97F4A7C15ULL;
    uint64_t z = st;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}

// one forward transform through the emulated passes (mirrors ntt_forward in gl_ntt_host.cuh)
static void emu_forward(const uint64_t* in, size_t in_stride, uint64_t* out, size_t out_stride, size_t row0, int log_n,
                        NttPlan pl, size_t ncols, int mode, bool reverse, uint64_t scale, uint64_t shift) {
    const size_t n = (size_t)1 << log_n;
    NttJob job;
    ntt_make_job(log_n, pl, scale, shift, job);
    std::vector<uint64_t> rt = step_table(job.row_step), c1s, c1p, c2s, c2p, scratch;
    RowPass& rp = job.rp;
    rp.tw = rt.data();
    rp.out = out;
    rp.out_stride = out_stride;
    rp.reverse = reverse;
    rp.row0 = row0;
    rp.ncols = (int)ncols;
    if (pl.a1 == 0) {
        rp.in = in;
        rp.in_stride = in_stride;
    } else {
        scratch.resize(ncols * n);
        c1s = step_table(job.c1_step);
        c1p = post_table(job.c1_post);
        job.c1.in = in;
        job.c1.in_stride = in_stride;
        job.c1.out = scratch.data();
        job.c1.out_stride = n;
        job.c1.tw = c1s.data();
        job.c1.twa = c1p.data();
        DISPATCH(pl.a1, emu_col<L>(job.c1, ncols));
        if (pl.a2) {
            c2s = step_table(job.c2_step);
            c2p = post_table(job.c2_post);
            job.c2.in = job.c2.out = scratch.data();
            job.c2.in_stride = job.c2.out_stride = n;
            job.c2.tw = c2s.data();
            job.c2.twa = c2p.data();
            DISPATCH(pl.a2, emu_col<L>(job.c2, ncols));
        }
        rp.in = scratch.data();
        rp.in_stride = n;
    }
    if (mode == RM_BITREV) { DISPATCH(pl.b, (emu_row<L, RM_BITREV>(rp))); }
    else { DISPATCH(pl.b, (emu_row<L, RM_NATURAL>(rp))); }
}

// mode: 0 forward natural, 1 inverse natural (reverse + 1/n), 2 coset forward natural, 3 column-major coset LDE
static int check(int log_n, NttPlan pl, int ncols, int mode, int rate_bits) {
    const size_t n = (size_t)1 << log_n;
    uint64_t st = 1234 + log_n * 77 + mode + pl.a2 * 13;
    std::vector<uint64_t> in((size_t)ncols * n);
    for (auto& x : in) x = rnd(st);
    int bad = 0;
    if (mode <= 2) {
        std::vector<uint64_t> out((size_t)ncols * n, 0xDEAD);
        const uint64_t shift = mode == 2 ? (rnd(st) | 1) : 1;
        emu_forward(in.data(), n, out.data(), n, 0, log_n, pl, ncols, RM_NATURAL, mode == 1,
                    mode == 1 ? inverse_2exp((uint32_t)log_n) : 1, shift);
        for (int c = 0; c < ncols && !bad; c++) {
            std::vector<uint64_t> ref(in.begin() + c * n, in.begin() + (c + 1) * n);
            if (mode == 0) glo_fft(ref.data(), log_n, 0);
            else if (mode == 1) glo_ifft(ref.data(), log_n);
            else glo_coset_fft(ref.data(), log_n, shift, 0);
            for (size_t i = 0; i < n; i++)
                if (out[c * n + i] != ref[i]) {
                    printf("MISMATCH log_n=%d plan=(%d,%d,%d) mode=%d col=%d i=%zu got=%llx want=%llx\n", log_n, pl.a1, pl.a2,
                           pl.b, mode, c, i, (unsigned long long)out[c * n + i], (unsigned long long)ref[i]);
                    bad = 1;
                    break;
                }
        }
    } else {
        const int ncos = 1 << rate_bits;
        const size_t N = n << rate_bits;
        std::vector<uint64_t> lde((size_t)ncols * N, 0xDEAD);
        const uint64_t g = MULTIPLICATIVE_GROUP_GENERATOR, wN = root_of_unity(log_n + rate_bits);
        for (int c = 0; c < ncos; c++) {
            const uint64_t s = mul(g, pow(wN, bitrev32(c, rate_bits)));
            emu_forward(in.data(), n, lde.data(), N, (size_t)c * n, log_n, pl, ncols, RM_BITREV, false, 1, s);
        }
        // reference: zero-padded coset FFT of size N on g, natural order; lde[col][j] = ref[bitrev_N(j)]
        for (int c = 0; c < ncols && !bad; c++) {
            std::vector<uint64_t> ref(N, 0);
            for (size_t i = 0; i < n; i++) ref[i] = canon(in[c * n + i]);
            glo_coset_fft(ref.data(), log_n + rate_bits, g, 0);
            for (size_t j = 0; j < N; j++) {
                const size_t i = bitrev32((uint32_t)j, log_n + rate_bits);
                if (lde[c * N + j] != ref[i]) {
                    printf("LDE MISMATCH log_n=%d plan=(%d,%d,%d) col=%d j=%zu\n", log_n, pl.a1, pl.a2, pl.b, c, j);
                    bad = 1;
                    break;
                }
            }
        }
    }
    return bad;
}

int main(int argc, char** argv) {
    const int max_log = argc > 1 ? atoi(argv[1]) : 13;
    int bad = 0, cases = 0;
    for (int log_n = 1; log_n <= max_log; log_n++) {
        const NttPlan pl = ntt_plan(log_n);
        for (int mode = 0; mode < 4; mode++) {
            bad |= check(log_n, pl, log_n > 11 ? 2 : 3, mode, mode == 3 ? (log_n > 10 ? 1 : 2) : 0);
            cases++;
        }
    }
    // forced multi-pass plans at small sizes: every column-pass size, both NSUB cases, and the three-pass structure
    const NttPlan forced[] = {{5, 0, 6}, {6, 0, 7}, {7, 0, 7}, {8, 0, 6}, {9, 0, 5}, {5, 5, 6}, {6, 5, 6}, {5, 7, 6}, {7, 7, 7}};
    for (const NttPlan& pl : forced) {
        const int log_n = pl.a1 + pl.a2 + pl.b;
        for (int mode = 0; mode < 4; mode++) {
            bad |= check(log_n, pl, 2, mode, 1);
            cases++;
        }
    }
    if (max_log >= 20) {  // the 10 + 10 plan of the headline config (slow: only when asked for)
        bad |= check(20, ntt_plan(20), 1, 0, 0);
        bad |= check(20, ntt_plan(20), 1, 3, 0);
        cases += 2;
    }
    printf("%s (%d cases)\n", bad ? "EMU FAILED" : "EMU OK", cases);
    return bad;
}
