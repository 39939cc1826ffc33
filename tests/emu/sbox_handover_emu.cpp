// Host run of the full round's two hand-overs between the integer and FP64 pipes (gl_poseidon.cuh built with
// -DGL_FP64_ON_HOST -DGL_FORCE_32BIT_PATH, so the device formulations run in plain C++), against unsigned __int128:
//  * sbox7_f64: the limb pair (L, H) of x^7 must be integers with L + 2^32*H = x^7 (mod p), -2^33 < L < 2^32 and
//    0 <= H < 2^33 (the bounds circ12_f64 and the seed biases rely on);
//  * f64_pair_to_u64: for integers 0 <= al, ah < 2^52 the u64 result must be congruent to al + 2^32*ah.
// Inputs: edge words (0, 1, p - 1, p, 2^64 - 1, around 2^32 boundaries) and random words.
// Test infrastructure: built and run by tests/test_emu_full_round_handover.py.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include "../../plonky2_b200/csrc/gl_poseidon.cuh"
#if !defined(GL_FP64_PATH)
#error "build with -DGL_FP64_ON_HOST"
#endif
using namespace gl;
typedef unsigned __int128 u128;
static const u128 PP = (u128)P;
static uint64_t rnd(uint64_t& st) {
    st += 0x9E3779B97F4A7C15ULL;
    uint64_t z = st;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}
static uint64_t mulmod(uint64_t a, uint64_t b) { return (uint64_t)(((u128)a * b) % PP); }
static uint64_t pow7(uint64_t x) {
    const uint64_t x2 = mulmod(x, x), x4 = mulmod(x2, x2);
    return mulmod(mulmod(x2, x), x4);
}
static int bad = 0;
static void check_sbox(uint64_t x) {
    double L, H;
    sbox7_f64(x, L, H);
    const bool ints = L == std::floor(L) && H == std::floor(H);
    const bool bounds = L > -8589934592.0 && L < 4294967296.0 && H >= 0 && H < 8589934592.0;
    bool eq = false;
    if (ints && bounds) {
        const int64_t l = (int64_t)L;
        const u128 v = ((u128)(uint64_t)H << 32) + 2 * PP + (u128)(__int128)l;  // + 2p keeps it non-negative
        eq = (uint64_t)(v % PP) == pow7(x);
    }
    if (!(ints && bounds && eq) && bad++ < 10)
        printf("sbox7_f64(%#llx): L = %.17g H = %.17g (%s)\n", (unsigned long long)x, L, H,
               !ints ? "not integers" : !bounds ? "out of bounds" : "wrong value");
}
static void check_ret(uint64_t al, uint64_t ah) {
    const uint64_t r = f64_pair_to_u64((double)al, (double)ah);
    const uint64_t want = (uint64_t)((((u128)ah << 32) + al) % PP);
    if ((uint64_t)((u128)r % PP) != want && bad++ < 10)
        printf("f64_pair_to_u64(%#llx, %#llx) = %#llx, want %#llx (mod p)\n", (unsigned long long)al,
               (unsigned long long)ah, (unsigned long long)r, (unsigned long long)want);
}
int main(int argc, char** argv) {
    const long iters = argc > 1 ? atol(argv[1]) : (1L << 24);
    const uint64_t M52 = (1ULL << 52) - 1;
    const uint64_t edge[] = {0, 1, 2, P - 1, P - 2, P, P + 1, 0xFFFFFFFEULL, 0xFFFFFFFFULL, 0x100000000ULL,
                             0x100000001ULL, 1ULL << 63, P - (1ULL << 32), ~0ULL, ~0ULL - 1, 0xFFFFFFFF00000000ULL,
                             0xFFFFFFFEFFFFFFFFULL, 0x00000001FFFFFFFFULL, 0x7FFFFFFF80000000ULL};
    const int ne = sizeof(edge) / sizeof(edge[0]);
    for (int i = 0; i < ne; i++) {
        check_sbox(edge[i]);
        for (int j = 0; j < ne; j++) check_ret(edge[i] & M52, edge[j] & M52);
    }
    const uint64_t ret_edge[] = {0, 1, 0xFFFFFFFFULL, 0x100000000ULL, 0xFFFFFFFFFFFFFULL, M52, M52 - 1,
                                 (1ULL << 51) + 0xFFFFFFFFULL, 0xFFFFF00000000ULL, 0xFFFFEFFFFFFFFULL};
    for (uint64_t a : ret_edge)
        for (uint64_t b : ret_edge) check_ret(a, b);
    uint64_t st = 11;
    for (long i = 0; i < iters; i++) {
        const uint64_t v = rnd(st), w = rnd(st);
        check_sbox(i % 4 == 1 ? (v | 0xFFFFFFF0FFFFFFF0ULL) : i % 4 == 2 ? edge[v % ne] ^ (w & 7) : v);
        check_ret(v & M52, w & M52);
        check_ret((v & 0xFFFFFFFFULL) | (M52 & ~0xFFFFFFFFULL), w & M52);  // high limb words near 2^32 carries
    }
    printf(bad ? "HANDOVER EMU FAILED (%d)\n" : "HANDOVER EMU OK\n", bad);
    return bad != 0;
}
