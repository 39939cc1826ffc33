// CPU emulation of the coset-batched LDE (k_ntt_col_cosets + the row pass over all cosets of a group, lde_columns in
// gl_ntt_host.cuh) checked against the oracle and against the per-coset path. The job arithmetic is the SAME source the
// device uses (lde_make_cosets_job, col_cosets_unit, the RowPass coset addressing); the passes run through the
// emulation of ntt_emu.cpp, included here without its main. Test infrastructure: built and run by
// tests/test_emu_lde_cosets.py.
#include <algorithm>
#define main ntt_emu_main
#include "ntt_emu.cpp"
#undef main

// blocks [blk0, blk1) of a plain column pass (emu_col runs all of them)
template <int LOG>
void emu_col_tiles(const ColPass& cp, int blk0, int blk1) {
    using Cf = PassCfg<LOG>;
    std::vector<uint64_t> S(Cf::COL_S_WORDS);
    std::vector<std::vector<uint64_t>> x(Cf::COL_THREADS, std::vector<uint64_t>(Cf::E));
    for (int blk = blk0; blk < blk1; blk++) {
        for (int tid = 0; tid < Cf::COL_THREADS; tid++) col_load<LOG>(cp, blk, tid, x[tid].data());
        for (int tid = 0; tid < Cf::COL_THREADS; tid++) col_phase1<LOG>(cp, S.data(), blk, tid, x[tid].data());
        for (int tid = 0; tid < Cf::COL_THREADS; tid++) col_phase2<LOG>(cp, S.data(), blk, tid);
    }
}
// the coset-batched first column pass: every CTA runs the phases of the plain pass on the unit, tables and pre-weights
// that col_cosets_unit gives it (as k_ntt_col_cosets does)
template <int LOG>
void emu_col_cosets(const ColCosets& cc) {
    const int nblocks = col_cosets_blocks<LOG>(cc);
    for (int blk = 0; blk < nblocks; blk++) {
        int c, tile;
        size_t in_off, out_off;
        col_cosets_unit<LOG>(cc, blk, c, in_off, out_off, tile);
        ColPass cp = cc.cp;
        cp.in += in_off;
        cp.out += out_off;
        cp.tw = cc.tw[c];
        cp.twa = cc.twa[c];
        for (int q = 0; q < 32; q++) cp.uq[q] = cc.uq[c][q];
        emu_col_tiles<LOG>(cp, tile, tile + 1);
    }
}
// the row pass of the LDE as k_ntt_row_shared runs it for even LOG >= 4 (bit-reversed stores staged through the
// exchange buffer), else as k_ntt_row does
template <int LOG>
void emu_row_lde(const RowPass& rp) {
    using Cf = PassCfg<LOG>;
    if constexpr (Cf::E == Cf::TPT && LOG >= 4) {
        const int NT = Cf::ROW_THREADS;
        std::vector<uint64_t> S(ntt_row_smem_bytes(LOG, false) / 8);
        std::vector<std::vector<uint64_t>> x(NT, std::vector<uint64_t>(Cf::E));
        for (int blk = 0; blk < row_blocks<LOG>(rp); blk++) {
            for (int tid = 0; tid < NT; tid++) row_load<LOG, RM_BITREV>(rp, blk, tid, x[tid].data());
            for (int tid = 0; tid < NT; tid++) row_phase1<LOG, RM_BITREV>(rp, S.data(), blk, tid, x[tid].data());
            for (int tid = 0; tid < NT; tid++) {
                row_phase2_load<LOG>(S.data(), tid, 0, x[tid].data());
                pass_step2<LOG>(x[tid].data());
            }
            for (int tid = 0; tid < NT; tid++) row_stage_bitrev<LOG>(S.data(), tid, x[tid].data());
            for (int tid = 0; tid < NT; tid++) row_store_bitrev_staged<LOG>(rp, S.data(), blk, tid);
        }
    } else {
        emu_row<LOG, RM_BITREV>(rp);
    }
}
// the coset-batched LDE of lde_columns (gl_ntt_host.cuh): columns in groups of G, cosets 2^log_kc at a time
static void emu_lde_cosets(const uint64_t* in, size_t ncols, uint64_t* lde, size_t lde_stride, int log_n, NttPlan pl,
                           int rate_bits, uint64_t base_shift, int log_kc, size_t G) {
    const size_t n = (size_t)1 << log_n;
    const int ncos = 1 << rate_bits, kc = 1 << log_kc;
    std::vector<uint64_t> scratch(G * kc * n);
    for (size_t g0 = 0; g0 < ncols; g0 += G) {
        const size_t gc = ncols - g0 < G ? ncols - g0 : G;
        for (int c0 = 0; c0 < ncos; c0 += kc) {
            NttJob job;
            ColCosets cc;
            TableReq steps[1 << COL_LOG_MAX_COSETS], posts[1 << COL_LOG_MAX_COSETS];
            lde_make_cosets_job(log_n, pl, rate_bits, base_shift, c0, log_kc, job, cc, steps, posts);
            std::vector<std::vector<uint64_t>> st(kc), pt(kc);
            for (int c = 0; c < kc; c++) {
                st[c] = step_table(steps[c]);
                pt[c] = post_table(posts[c]);
                cc.tw[c] = st[c].data();
                cc.twa[c] = pt[c].data();
            }
            std::fill(scratch.begin(), scratch.end(), 0xBAD);
            cc.cp.in = in + g0 * n;
            cc.cp.in_stride = n;
            cc.cp.out = scratch.data();
            cc.cp.out_stride = n;
            cc.ncols = (int)gc;
            DISPATCH(pl.a1, emu_col_cosets<L>(cc));
            std::vector<uint64_t> c2s, c2p, rt = step_table(job.row_step);
            if (pl.a2) {
                c2s = step_table(job.c2_step);
                c2p = post_table(job.c2_post);
                job.c2.in = job.c2.out = scratch.data();
                job.c2.in_stride = job.c2.out_stride = n;
                job.c2.tw = c2s.data();
                job.c2.twa = c2p.data();
                DISPATCH(pl.a2, emu_col<L>(job.c2, gc * kc));
            }
            RowPass& rp = job.rp;
            rp.tw = rt.data();
            rp.in = scratch.data();
            rp.in_stride = n;
            rp.out = lde + g0 * lde_stride;
            rp.out_stride = lde_stride;
            rp.row0 = (size_t)c0 * n;
            rp.cos_step = n;
            rp.ncols = (int)(gc * kc);
            DISPATCH(pl.b, emu_row_lde<L>(rp));
        }
    }
}
// coset-batched LDE of ncols random columns (groups of G columns, 2^log_kc cosets per job) against the oracle and
// against the per-coset path, on the coset base `shift` (1: the cosets of <w_N> itself, coset 0 trivial)
static int check_cosets(int log_n, NttPlan pl, int ncols, int rate_bits, int log_kc, size_t G, uint64_t shift) {
    const size_t n = (size_t)1 << log_n, N = n << rate_bits;
    uint64_t st = 4321 + log_n * 31 + rate_bits * 7 + log_kc;
    std::vector<uint64_t> in((size_t)ncols * n);
    for (auto& x : in) x = rnd(st);
    std::vector<uint64_t> lde((size_t)ncols * N, 0xDEAD), per((size_t)ncols * N, 0xDEAD);
    emu_lde_cosets(in.data(), ncols, lde.data(), N, log_n, pl, rate_bits, shift, log_kc, G);
    const uint64_t wN = root_of_unity(log_n + rate_bits);
    for (int c = 0; c < (1 << rate_bits); c++) {
        const uint64_t s = mul(shift, pow(wN, bitrev32(c, rate_bits)));
        emu_forward(in.data(), n, per.data(), N, (size_t)c * n, log_n, pl, ncols, RM_BITREV, false, 1, s);
    }
    for (int c = 0; c < ncols; c++) {
        std::vector<uint64_t> ref(N, 0);
        for (size_t i = 0; i < n; i++) ref[i] = canon(in[c * n + i]);
        glo_coset_fft(ref.data(), log_n + rate_bits, shift, 0);
        for (size_t j = 0; j < N; j++) {
            const size_t i = bitrev32((uint32_t)j, log_n + rate_bits);
            if (lde[c * N + j] != ref[i] || per[c * N + j] != ref[i]) {
                printf("COSET LDE MISMATCH log_n=%d plan=(%d,%d,%d) rate_bits=%d kc=%d G=%zu col=%d j=%zu got=%llx per=%llx "
                       "want=%llx\n", log_n, pl.a1, pl.a2, pl.b, rate_bits, 1 << log_kc, G, c, j,
                       (unsigned long long)lde[c * N + j], (unsigned long long)per[c * N + j], (unsigned long long)ref[i]);
                return 1;
            }
        }
    }
    return 0;
}

int main() {
    int bad = 0, cases = 0;
    // coset-batched LDE: every even first pass (6, 8, 10), a three-pass plan, rates 1..4 (rate 4: two jobs of 8
    // cosets), groups that do not divide the column count, the trivial coset (shift 1) next to the LDE's own, and row
    // passes of 6, 8 and 10 (staged stores) next to odd ones
    struct CosetCase {
        NttPlan pl;
        int ncols, rate_bits;
        size_t G;
        uint64_t shift;
    };
    const uint64_t g = MULTIPLICATIVE_GROUP_GENERATOR;
    const CosetCase cosets[] = {{{6, 0, 5}, 3, 1, 2, g}, {{6, 0, 6}, 5, 2, 2, g},  {{8, 0, 5}, 3, 3, 1, g},
                                {{6, 0, 5}, 2, 4, 2, g}, {{6, 0, 7}, 3, 3, 2, 1},  {{6, 5, 6}, 3, 2, 2, g},
                                {{8, 6, 5}, 2, 1, 1, 7}, {{10, 0, 5}, 1, 2, 1, g}, {{6, 0, 8}, 3, 1, 2, g},
                                {{6, 0, 10}, 1, 1, 1, g}};
    for (const CosetCase& k : cosets) {
        const int log_n = k.pl.a1 + k.pl.a2 + k.pl.b;
        const int log_kc = k.rate_bits < COL_LOG_MAX_COSETS ? k.rate_bits : COL_LOG_MAX_COSETS;
        bad |= check_cosets(log_n, k.pl, k.ncols, k.rate_bits, log_kc, k.G, k.shift);
        cases++;
    }
    printf("%s (%d cases)\n", bad ? "COSET EMU FAILED" : "COSET EMU OK", cases);
    return bad;
}
