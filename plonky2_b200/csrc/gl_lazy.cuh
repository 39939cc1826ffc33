// gl_lazy.cuh -- lazily reduced Goldilocks values for the NTT butterflies.
//
// The reference's butterflies (field/src/fft.rs:165-202) reduce after every add/sub (goldilocks_field.rs:245-290);
// on the integer pipes a fully reduced modular add costs about a dozen instructions and a sub 8. Here a value
// travels through the add/sub levels of an in-register radix-2^M transform as THREE 32-bit words
//        v = w0 + w1*2^32 + e*2^64        (e a small SIGNED word: the carries and borrows accumulated so far)
// so that add and sub are 3 carry-chain instructions with no fix-up, and is only brought back to one u64 where a
// 64x64 multiplication needs it (l3_norm). Power-of-two twiddles (w_32 = 2^6 ... w_4 = 2^48, SURVEY appendix A.2)
// act directly on the lazy form: the 128-bit signed product v*2^r is folded with 2^64 = 2^32 - 1, 2^96 = -1
// (X^2 = X - 1, X^3 = -1 for X = 2^32) back into three words (l3_shift) -- no separate reduction before or after.
// Range discipline (checked on the device by tests/test_gpu_field_lazy.py, which runs tests/cuda/field_lazy_device.cu,
// and by the parity suite): inputs of a radix-2^M transform have e = 0; every level at most doubles |v|; l3_shift
// accepts |v| < 2^94 and returns |v| < 2^67, so e stays far below the 2^20 that l3_norm allows.
#pragma once
#include "gl_field.cuh"

namespace gl {

struct L3 {
    uint32_t w0, w1;
    int32_t e;
};

GL_HD L3 l3_from(uint64_t x) { return L3{(uint32_t)x, (uint32_t)(x >> 32), 0}; }

#if defined(__CUDA_ARCH__)
__device__ __forceinline__ L3 l3_add(L3 a, L3 b) {
    L3 r;
    asm("add.cc.u32 %0, %3, %6;\n\taddc.cc.u32 %1, %4, %7;\n\taddc.u32 %2, %5, %8;"
        : "=r"(r.w0), "=r"(r.w1), "=r"(r.e)
        : "r"(a.w0), "r"(a.w1), "r"(a.e), "r"(b.w0), "r"(b.w1), "r"(b.e));
    return r;
}
__device__ __forceinline__ L3 l3_sub(L3 a, L3 b) {
    L3 r;
    asm("sub.cc.u32 %0, %3, %6;\n\tsubc.cc.u32 %1, %4, %7;\n\tsubc.u32 %2, %5, %8;"
        : "=r"(r.w0), "=r"(r.w1), "=r"(r.e)
        : "r"(a.w0), "r"(a.w1), "r"(a.e), "r"(b.w0), "r"(b.w1), "r"(b.e));
    return r;
}
// v * 2^S (mod p), 0 <= S < 96 a compile-time constant, S = 32q + r.
// With (c0, c1, c2, c3) the four words of the signed 128-bit value v * 2^r (c3 signed):
//   q = 0:  (c0 - c2 - c3) + (c1 + c2) X
//   q = 1:  (-c1 - c2)     + (c0 + c1 - c3) X
//   q = 2:  (c3 - c0 - c1) + (c0 - c2 - c3) X           (X = 2^32, X^2 = X - 1, X^3 = -1)
// each evaluated as   (unsigned base words) - (a small signed 64/96-bit quantity T)   in one 3-word subtraction.
template <int S>
__device__ __forceinline__ L3 l3_shift(L3 a) {
    static_assert(S >= 0 && S < 96, "shift out of range");
    if constexpr (S == 0) return a;
    constexpr int q = S / 32, r = S % 32;
    uint32_t c0, c1, c2;
    int32_t c3;
    if constexpr (r == 0) {
        c0 = a.w0;
        c1 = a.w1;
        c2 = (uint32_t)a.e;
        c3 = a.e >> 31;
    } else {
        c0 = a.w0 << r;
        c1 = __funnelshift_l(a.w0, a.w1, r);
        c2 = __funnelshift_l(a.w1, (uint32_t)a.e, r);
        c3 = a.e >> (32 - r);
    }
    const int32_t s3 = c3 >> 31;  // sign extension of c3
    L3 o;
    if (q == 0) {
        uint32_t t0, t1, b1, be;  // T = c2 + c3 ; base = c0 + (c1 + c2) X
        asm("add.cc.u32 %0, %2, %3;\n\taddc.u32 %1, %4, 0;" : "=r"(t0), "=r"(t1) : "r"(c2), "r"((uint32_t)c3), "r"((uint32_t)s3));
        asm("add.cc.u32 %0, %2, %3;\n\taddc.u32 %1, 0, 0;" : "=r"(b1), "=r"(be) : "r"(c1), "r"(c2));
        asm("sub.cc.u32 %0, %3, %5;\n\tsubc.cc.u32 %1, %4, %6;\n\tsubc.u32 %2, %7, %8;"
            : "=r"(o.w0), "=r"(o.w1), "=r"(o.e)
            : "r"(c0), "r"(b1), "r"(t0), "r"(t1), "r"(be), "r"((int32_t)t1 >> 31));
    } else if (q == 1) {
        uint32_t b1, be, t0, t1;  // base = (c0 + c1) X ; T = (c1 + c2) + c3 X
        int32_t t2;
        asm("add.cc.u32 %0, %2, %3;\n\taddc.u32 %1, 0, 0;" : "=r"(b1), "=r"(be) : "r"(c0), "r"(c1));
        asm("add.cc.u32 %0, %3, %4;\n\taddc.cc.u32 %1, %5, 0;\n\taddc.u32 %2, %6, 0;"
            : "=r"(t0), "=r"(t1), "=r"(t2)
            : "r"(c1), "r"(c2), "r"((uint32_t)c3), "r"(s3));
        asm("sub.cc.u32 %0, 0, %3;\n\tsubc.cc.u32 %1, %4, %5;\n\tsubc.u32 %2, %6, %7;"
            : "=r"(o.w0), "=r"(o.w1), "=r"(o.e)
            : "r"(t0), "r"(b1), "r"(t1), "r"(be), "r"(t2));
    } else {
        uint32_t u0, u1, v0, v1, t1;  // base = c0 X ; T = (c0 + c1 - c3) + (c2 + c3) X
        int32_t t2;
        asm("add.cc.u32 %0, %2, %3;\n\taddc.u32 %1, 0, 0;" : "=r"(u0), "=r"(u1) : "r"(c0), "r"(c1));
        asm("sub.cc.u32 %0, %0, %2;\n\tsubc.u32 %1, %1, %3;" : "+r"(u0), "+r"(u1) : "r"((uint32_t)c3), "r"((uint32_t)s3));
        asm("add.cc.u32 %0, %2, %3;\n\taddc.u32 %1, %4, 0;" : "=r"(v0), "=r"(v1) : "r"(c2), "r"((uint32_t)c3), "r"((uint32_t)s3));
        asm("add.cc.u32 %0, %2, %3;\n\taddc.u32 %1, %4, %5;" : "=r"(t1), "=r"(t2) : "r"(u1), "r"(v0), "r"((int32_t)u1 >> 31), "r"(v1));
        asm("sub.cc.u32 %0, 0, %3;\n\tsubc.cc.u32 %1, %4, %5;\n\tsubc.u32 %2, 0, %6;"
            : "=r"(o.w0), "=r"(o.w1), "=r"(o.e)
            : "r"(u0), "r"(c0), "r"(t1), "r"(t2));
    }
    return o;
}
// lazy -> one u64 congruent to v (any representative in [0, 2^64)); needs |e| < 2^20.
// Adds K = 2^20 * p = 2^20 + (2^32 - 2^20) * 2^32 + (2^20 - 1) * 2^64 so the top word is non-negative, then reduce96.
__device__ __forceinline__ uint64_t l3_norm(L3 a) {
    uint32_t w0, w1, e;
    asm("add.cc.u32 %0, %3, 0x00100000;\n\taddc.cc.u32 %1, %4, 0xfff00000;\n\taddc.u32 %2, %5, 0x000fffff;"
        : "=r"(w0), "=r"(w1), "=r"(e)
        : "r"(a.w0), "r"(a.w1), "r"(a.e));
    return reduce96(pack64(w0, w1), e);
}
#else
// ---- host formulation (tests/emu): same values mod p, not the same word patterns
inline __int128 l3_val(L3 a) { return (__int128)a.w0 + ((__int128)a.w1 << 32) + (__int128)a.e * ((__int128)1 << 64); }
inline L3 l3_of(__int128 v) {
    L3 r;
    r.w0 = (uint32_t)(unsigned __int128)v;
    r.w1 = (uint32_t)((unsigned __int128)v >> 32);
    r.e = (int32_t)(v >> 64);
    return r;
}
inline L3 l3_add(L3 a, L3 b) { return l3_of(l3_val(a) + l3_val(b)); }
inline L3 l3_sub(L3 a, L3 b) { return l3_of(l3_val(a) - l3_val(b)); }
inline uint64_t l3_norm(L3 a) {
    __int128 v = l3_val(a) % (__int128)P;
    if (v < 0) v += P;
    return (uint64_t)v;
}
template <int S>
inline L3 l3_shift(L3 a) { return l3_from(mul_pow2(l3_norm(a), (uint32_t)S)); }
#endif

// 2^M-point DIF DFT on lazy values, natural in, bit-reversed out, w_{2^M} = 2^(192 / 2^M). Fully unrolled: every
// shift amount is a compile-time constant.
template <int S>
GL_HD L3 l3_shift_c(L3 a) { return l3_shift<S>(a); }
template <int M, int L, int B>
struct DftLazyBfly {
    static GL_HD void run(L3* r) {
        constexpr int half = 1 << (M - 1 - L);
        constexpr int j = B % half, blk = (B / half) * 2 * half;
        constexpr int sh = (96 / half) * j;
        const L3 u = r[blk + j], v = r[blk + j + half];
        r[blk + j] = l3_add(u, v);
        r[blk + j + half] = l3_shift_c<sh>(l3_sub(u, v));
        if constexpr (B + 1 < (1 << (M - 1))) DftLazyBfly<M, L, B + 1>::run(r);
        else if constexpr (L + 1 < M) DftLazyBfly<M, L + 1, 0>::run(r);
    }
};
template <int M>
GL_HD void dft_lazy(L3* r) {
    if constexpr (M > 0) DftLazyBfly<M, 0, 0>::run(r);
}

}  // namespace gl
