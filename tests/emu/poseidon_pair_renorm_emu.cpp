// Host run of the partial-round pair's limb renormalisation (partial_pair_renorm in gl_poseidon.cuh, built with
// -DGL_FP64_ON_HOST, optionally -DGL_PAIR_RENORM_F64) on the edges of its input range: every pair of limbs
// |L|, |H| < 2^49 must come back as limbs with the same value mod p and inside the bounds the next pair's exactness
// argument uses. The whole permutation is checked by poseidon_f64_emu.cpp; random states rarely reach these edges.
// Test infrastructure: built and run by tests/test_emu_pair_renorm.py.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include "../../plonky2_b200/csrc/gl_poseidon.cuh"
#if !defined(GL_PARTIAL_F64)
#error "build with -DGL_FP64_ON_HOST"
#endif
using namespace gl;
static uint64_t rnd(uint64_t& st) {
    st += 0x9E3779B97F4A7C15ULL;
    uint64_t z = st;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}
static uint64_t modp(__int128 v) {
    const __int128 p = (__int128)P;
    v %= p;
    return (uint64_t)(v < 0 ? v + p : v);
}
int main(int argc, char** argv) {
    const int iters = argc > 1 ? atoi(argv[1]) : 1000000;
    const int64_t E = (1LL << 49) - 1, T = 1LL << 32;
#if defined(GL_PAIR_RENORM_F64)
    const double lo = -(double)(1LL << 31) - (double)(1 << 18), hi = (double)(1LL << 31) + (double)(1 << 18);
#else
    const double lo = -(double)(1 << 18), hi = (double)T + (double)(1 << 18);
#endif
    const int64_t edge[] = {0, 1, -1, E, -E, E - 1, -E + 1, T, -T, T - 1, -T + 1, T + 1, -T - 1, E - T + 1, -E + T - 1,
                            (1LL << 48), -(1LL << 48), 0x7FFFFFFFLL, -0x80000000LL, 3 * T, -3 * T, E & ~(T - 1),
                            -(E & ~(T - 1))};
    const int ne = sizeof(edge) / sizeof(edge[0]);
    int bad = 0;
    double lmin = 0, lmax = 0;
    uint64_t st = 11;
    for (int i = 0; i < ne * ne + iters; i++) {
        int64_t L, H;
        if (i < ne * ne) {
            L = edge[i % ne];
            H = edge[i / ne];
        } else {
            L = (int64_t)(rnd(st) % (2 * (uint64_t)E + 1)) - E;
            H = (int64_t)(rnd(st) % (2 * (uint64_t)E + 1)) - E;
            if (i % 3 == 1) L = edge[rnd(st) % ne];
            if (i % 3 == 2) H = edge[rnd(st) % ne];
        }
        double l = (double)L, h = (double)H;
        partial_pair_renorm(l, h);
        const bool integral = l == std::floor(l) && h == std::floor(h);
        const bool in_range = l > lo && l < hi && h > lo && h < hi;
        const bool same = integral && modp((__int128)L + ((__int128)H << 32)) ==
                                          modp((__int128)(int64_t)l + ((__int128)(int64_t)h << 32));
        if (!(in_range && same)) {
            if (bad < 8) printf("L=%lld H=%lld -> L'=%.0f H'=%.0f%s\n", (long long)L, (long long)H, l, h,
                                same ? " (out of range)" : " (wrong value)");
            bad++;
        }
        lmin = std::fmin(lmin, std::fmin(l, h));
        lmax = std::fmax(lmax, std::fmax(l, h));
    }
    printf("renormalised limbs in [%.0f, %.0f], bounds (%.0f, %.0f)\n", lmin, lmax, lo, hi);
    printf(bad ? "PAIR RENORM EMU FAILED (%d)\n" : "PAIR RENORM EMU OK\n", bad);
    return bad != 0;
}
