// gl_field.cuh -- Goldilocks field arithmetic, p = 2^64 - 2^32 + 1, for sm_90a device code
// (and the host, for the transcript's single permutations).
//
// Semantics follow the reference's GoldilocksField (field/src/goldilocks_field.rs:23-25,198-320,
// 392-449): an element is ANY u64 (non-canonical values in [p, 2^64) are allowed and represent
// themselves mod p); add/sub/mul return a u64 congruent to the exact result; canonicalisation
// (to_canonical_u64, :216-224) happens only where values are stored for hashing/comparison/output.
//
// This is not a translation of the x86 code: on the device the 64x64->128 product is four IMAD.WIDE.U32
// (ptxas' carry-in/carry-out forms) and the reduction uses 2^64 = 2^32 - 1, 2^96 = -1 (mod p) with 32-bit
// carry chains written in PTX (Montgomery-free, as BASELINE.json asks): reduce128 is 11 instructions, a
// general add 10, a modmul 4 IMAD.WIDE + 14 (tools/microbench.cu; tools/variants ranks the formulations).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define GL_HD __host__ __device__ __forceinline__
#define GL_D __device__ __forceinline__
#else
#define GL_HD inline
#define GL_D inline
#endif

namespace gl {

constexpr uint64_t P = 0xFFFFFFFF00000001ULL;
constexpr uint64_t EPS = 0xFFFFFFFFULL;  // 2^32 - 1 = 2^64 mod p
// field/src/goldilocks_field.rs:80,87
constexpr uint64_t MULTIPLICATIVE_GROUP_GENERATOR = 14293326489335486720ULL;
constexpr uint64_t POWER_OF_TWO_GENERATOR = 7277203076849721926ULL;
constexpr uint32_t TWO_ADICITY = 32;

GL_HD uint64_t canon(uint64_t x) { return x >= P ? x - P : x; }

#if defined(__CUDA_ARCH__)
// ---- device formulations: 32-bit carry chains in PTX (ptxas spreads them over IADD3.X / IMAD.X) ----
__device__ __forceinline__ uint32_t lo32(uint64_t v) { return (uint32_t)v; }
__device__ __forceinline__ uint32_t hi32(uint64_t v) { return (uint32_t)(v >> 32); }
__device__ __forceinline__ uint64_t pack64(uint32_t lo, uint32_t hi) {
    uint64_t r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "r"(lo), "r"(hi));
    return r;
}
#endif

// a + b (mod p), any u64 inputs, result in [0, 2^64).
GL_HD uint64_t add(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
    uint32_t r0, r1;
    asm("{\n\t.reg .u32 c, m;\n\t"
        "add.cc.u32 %0, %2, %4;\n\t"
        "addc.cc.u32 %1, %3, %5;\n\t"
        "addc.u32 c, 0, 0;\n\t"
        "neg.s32 m, c;\n\t"          // carry: += 2^64 mod p = 2^32 - 1
        "add.cc.u32 %0, %0, m;\n\t"
        "addc.cc.u32 %1, %1, 0;\n\t"
        "addc.u32 c, 0, 0;\n\t"      // second carry: only if both inputs are non-canonical
        "neg.s32 m, c;\n\t"
        "add.cc.u32 %0, %0, m;\n\t"
        "addc.u32 %1, %1, 0;\n\t}"
        : "=&r"(r0), "=&r"(r1)
        : "r"(lo32(a)), "r"(hi32(a)), "r"(lo32(b)), "r"(hi32(b)));
    return pack64(r0, r1);
#else
    uint64_t s = a + b;
    // carry out of 2^64: add 2^64 mod p = EPS. A second carry is possible only when both inputs
    // are non-canonical (goldilocks_field.rs:245-267); handle it so any u64 pair is safe.
    uint64_t c = (s < a) ? EPS : 0;
    uint64_t t = s + c;
    return (t < c) ? t + EPS : t;
#endif
}
// a + b (mod p) when b is CANONICAL (b < p): a single carry fix-up suffices
// (Field64::add_canonical_u64, goldilocks_field.rs:200-205).
GL_HD uint64_t add_canonical(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
    uint32_t r0, r1;
    asm("{\n\t.reg .u32 c, m;\n\t"
        "add.cc.u32 %0, %2, %4;\n\t"
        "addc.cc.u32 %1, %3, %5;\n\t"
        "addc.u32 c, 0, 0;\n\t"
        "neg.s32 m, c;\n\t"
        "add.cc.u32 %0, %0, m;\n\t"
        "addc.u32 %1, %1, 0;\n\t}"
        : "=&r"(r0), "=&r"(r1)
        : "r"(lo32(a)), "r"(hi32(a)), "r"(lo32(b)), "r"(hi32(b)));
    return pack64(r0, r1);
#else
    uint64_t s = a + b;
    return (s < a) ? s + EPS : s;
#endif
}
// a - b (mod p)
GL_HD uint64_t sub(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
    uint32_t r0, r1;
    asm("{\n\t.reg .u32 m;\n\t"
        "sub.cc.u32 %0, %2, %4;\n\t"
        "subc.cc.u32 %1, %3, %5;\n\t"
        "subc.u32 m, 0, 0;\n\t"      // 0xFFFFFFFF on borrow: -= 2^64 mod p
        "sub.cc.u32 %0, %0, m;\n\t"
        "subc.cc.u32 %1, %1, 0;\n\t"
        "subc.u32 m, 0, 0;\n\t"      // second borrow: only if b is non-canonical and a tiny
        "sub.cc.u32 %0, %0, m;\n\t"
        "subc.u32 %1, %1, 0;\n\t}"
        : "=&r"(r0), "=&r"(r1)
        : "r"(lo32(a)), "r"(hi32(a)), "r"(lo32(b)), "r"(hi32(b)));
    return pack64(r0, r1);
#else
    uint64_t d = a - b;
    uint64_t c = (a < b) ? EPS : 0;
    uint64_t t = d - c;
    return (d < c) ? t - EPS : t;
#endif
}
GL_HD uint64_t neg(uint64_t a) {
    uint64_t c = canon(a);
    return c ? P - c : 0;
}

// Reduce hi*2^64 + lo (mod p) to [0, 2^64): lo - (hi >> 32) + (hi & EPS) * EPS
// (the reference's reduce128, goldilocks_field.rs:401-415, re-expressed on 32-bit halves).
GL_HD uint64_t reduce128(uint64_t lo, uint64_t hi) {
#if defined(__CUDA_ARCH__) && defined(GL_REDUCE_V1)
    // x = lo - hh (borrow b), r = x + hl*EPS (carry c); true value = r_wrapped + (c - b)*2^64, and
    // 2^64 = EPS (mod p): apply the signed fix-up (c - b)*EPS in one 64-bit add (it cannot wrap).
    uint32_t r0, r1;
    asm("{\n\t.reg .u32 t0, t1, nb, d, f0, f1;\n\t"
        "sub.cc.u32 t0, 0, %4;\n\t"        // t = hl * (2^32 - 1) = (hl << 32) - hl
        "subc.u32 t1, %4, 0;\n\t"
        "sub.cc.u32 %0, %2, %5;\n\t"       // x = lo - hh
        "subc.cc.u32 %1, %3, 0;\n\t"
        "subc.u32 nb, 0, 0;\n\t"           // -b
        "add.cc.u32 %0, %0, t0;\n\t"       // r = x + t
        "addc.cc.u32 %1, %1, t1;\n\t"
        "addc.u32 d, nb, 0;\n\t"           // d = c - b in {-1, 0, 1}
        "neg.s32 f0, d;\n\t"               // d*EPS = (d >> 31 : -d)
        "shr.s32 f1, d, 31;\n\t"
        "add.cc.u32 %0, %0, f0;\n\t"
        "addc.u32 %1, %1, f1;\n\t}"
        : "=&r"(r0), "=&r"(r1)
        : "r"(lo32(lo)), "r"(hi32(lo)), "r"(lo32(hi)), "r"(hi32(hi)));
    return pack64(r0, r1);
#elif defined(__CUDA_ARCH__)
    // value = lo + hl*2^32 - (hl + hh)   (2^64 = 2^32 - 1, 2^96 = -1):  A = lo + (hl << 32) only touches the high
    // word (carry ca), s = hl + hh is 33 bits, r = A - s (borrow b); true value = r_wrapped + (ca - b)*2^64 and
    // 2^64 = EPS (mod p): apply the signed fix-up d*EPS, d = ca - b in {-1, 0, 1}, in one 64-bit add. It cannot
    // wrap: d = 1 means A >= 2^64 so r_wrapped < 2^64 - 2^32 + ... (r = A - 2^64 - s + [0] <= 2^64 - 2^32 - 1);
    // d = -1 means A < s < 2^33 so r_wrapped = 2^64 + A - s >= 2^64 - 2^33 > EPS.
    uint32_t r0, r1;
    asm("{\n\t.reg .u32 s0, s1, a1, ca, d, f0, f1;\n\t"
        "add.cc.u32 s0, %4, %5;\n\t"       // s = hl + hh
        "addc.u32 s1, 0, 0;\n\t"
        "add.cc.u32 a1, %3, %4;\n\t"       // A = lo + (hl << 32)
        "addc.u32 ca, 0, 0;\n\t"
        "sub.cc.u32 %0, %2, s0;\n\t"       // r = A - s
        "subc.cc.u32 %1, a1, s1;\n\t"
        "subc.u32 d, ca, 0;\n\t"           // d = ca - b
        "neg.s32 f0, d;\n\t"               // d*EPS = (d >> 31 : -d)
        "shr.s32 f1, d, 31;\n\t"
        "add.cc.u32 %0, %0, f0;\n\t"
        "addc.u32 %1, %1, f1;\n\t}"
        : "=&r"(r0), "=&r"(r1)
        : "r"(lo32(lo)), "r"(hi32(lo)), "r"(lo32(hi)), "r"(hi32(hi)));
    return pack64(r0, r1);
#else
    uint64_t hh = hi >> 32;
    uint64_t hl = hi & EPS;
    uint64_t t0 = lo - hh;
    if (lo < hh) t0 -= EPS;           // borrow: subtract 2^64 mod p
    uint64_t t1 = (hl << 32) - hl;    // hl * (2^32 - 1)
    uint64_t r = t0 + t1;
    return (r < t1) ? r + EPS : r;    // carry: add 2^64 mod p (cannot carry again)
#endif
}
// Reduce hi*2^64 + lo with hi < 2^32 (a "u96").
GL_HD uint64_t reduce96(uint64_t lo, uint32_t hi) {
#if defined(__CUDA_ARCH__)
    uint32_t r0, r1;
    asm("{\n\t.reg .u32 t0, t1, c, m;\n\t"
        "sub.cc.u32 t0, 0, %4;\n\t"
        "subc.u32 t1, %4, 0;\n\t"
        "add.cc.u32 %0, %2, t0;\n\t"
        "addc.cc.u32 %1, %3, t1;\n\t"
        "addc.u32 c, 0, 0;\n\t"
        "neg.s32 m, c;\n\t"
        "add.cc.u32 %0, %0, m;\n\t"
        "addc.u32 %1, %1, 0;\n\t}"
        : "=&r"(r0), "=&r"(r1)
        : "r"(lo32(lo)), "r"(hi32(lo)), "r"(hi));
    return pack64(r0, r1);
#else
    uint64_t t1 = ((uint64_t)hi << 32) - hi;
    uint64_t r = lo + t1;
    return (r < t1) ? r + EPS : r;
#endif
}

// GL_FORCE_32BIT_PATH lets tests/emu run the device formulation on the host.
GL_HD void mul_wide(uint64_t a, uint64_t b, uint64_t& lo, uint64_t& hi) {
#if defined(__CUDA_ARCH__)
    // One 128-bit product: 4 IMAD.WIDE.U32 (one with carry-out, one with carry-in) + 3 adds/moves. Written as
    // `lo = a * b; hi = __umul64hi(a, b)` the two halves are lowered separately and ptxas does NOT merge them:
    // 5 IMAD.WIDE + 2 IMAD + 4 adds (cuobjdump), i.e. +50 % on the FMA-heavy pipe that bounds these kernels.
#if defined(GL_MUL_EXPLICIT)
    // Variant: four independent IMAD.WIDE.U32 and the column sums on the ALU pipe (3-input IADD3 chains), instead
    // of ptxas' carry-in/carry-out IMAD.WIDE forms + IMAD.X + IMAD.MOV (all on the FMA-heavy pipe).
    uint32_t r0, r1, r2, r3;
    asm("{\n\t.reg .u64 z, x, y, w;\n\t.reg .u32 z1, x0, x1, y0, y1, w0, w1;\n\t"
        "mul.wide.u32 z, %4, %6;\n\t"
        "mul.wide.u32 x, %5, %6;\n\t"
        "mul.wide.u32 y, %4, %7;\n\t"
        "mul.wide.u32 w, %5, %7;\n\t"
        "mov.b64 {%0, z1}, z;\n\t"
        "mov.b64 {x0, x1}, x;\n\t"
        "mov.b64 {y0, y1}, y;\n\t"
        "mov.b64 {w0, w1}, w;\n\t"
        "add.cc.u32 %1, z1, x0;\n\t"
        "addc.cc.u32 %2, w0, x1;\n\t"
        "addc.u32 %3, w1, 0;\n\t"
        "add.cc.u32 %1, %1, y0;\n\t"
        "addc.cc.u32 %2, %2, y1;\n\t"
        "addc.u32 %3, %3, 0;\n\t}"
        : "=&r"(r0), "=&r"(r1), "=&r"(r2), "=&r"(r3)
        : "r"(lo32(a)), "r"(hi32(a)), "r"(lo32(b)), "r"(hi32(b)));
    lo = pack64(r0, r1);
    hi = pack64(r2, r3);
#else
    const unsigned __int128 p = (unsigned __int128)a * b;
    lo = (uint64_t)p;
    hi = (uint64_t)(p >> 64);
#endif
#elif defined(GL_FORCE_32BIT_PATH)
    uint32_t a0 = (uint32_t)a, a1 = (uint32_t)(a >> 32);
    uint32_t b0 = (uint32_t)b, b1 = (uint32_t)(b >> 32);
    uint64_t p00 = (uint64_t)a0 * b0;
    uint64_t mid = (uint64_t)a0 * b1 + (p00 >> 32);          // < 2^64, cannot overflow
    uint64_t mid2 = (uint64_t)a1 * b0 + (uint32_t)mid;       // < 2^64
    hi = (uint64_t)a1 * b1 + (mid >> 32) + (mid2 >> 32);     // exact high half
    lo = (mid2 << 32) | (uint32_t)p00;
#else
    unsigned __int128 p = (unsigned __int128)a * b;
    lo = (uint64_t)p;
    hi = (uint64_t)(p >> 64);
#endif
}
// a^2 = a0^2 + 2*a0*a1*2^32 + a1^2*2^64 with THREE IMAD.WIDE.U32, the cross term added twice on the ALU pipe.
// Poseidon's S-box squares with it (sqr_3w): with 4 CTAs/SM of 128 threads (no spills) it ranks above the
// four-product form in tools/variants (DESIGN.md §4). The generic sqr keeps mul_wide unless GL_SQR_3WIDE.
GL_HD void sqr_wide_3w(uint64_t a, uint64_t& lo, uint64_t& hi) {
#if defined(__CUDA_ARCH__)
    uint32_t r0, r1, r2, r3;
    asm("{\n\t.reg .u64 z, c, w;\n\t.reg .u32 z1, c0, c1, w0, w1;\n\t"
        "mul.wide.u32 z, %4, %4;\n\t"
        "mul.wide.u32 c, %4, %5;\n\t"
        "mul.wide.u32 w, %5, %5;\n\t"
        "mov.b64 {%0, z1}, z;\n\t"
        "mov.b64 {c0, c1}, c;\n\t"
        "mov.b64 {w0, w1}, w;\n\t"
        "add.cc.u32 %1, z1, c0;\n\t"
        "addc.cc.u32 %2, w0, c1;\n\t"
        "addc.u32 %3, w1, 0;\n\t"
        "add.cc.u32 %1, %1, c0;\n\t"
        "addc.cc.u32 %2, %2, c1;\n\t"
        "addc.u32 %3, %3, 0;\n\t}"
        : "=&r"(r0), "=&r"(r1), "=&r"(r2), "=&r"(r3)
        : "r"(lo32(a)), "r"(hi32(a)));
    lo = pack64(r0, r1);
    hi = pack64(r2, r3);
#elif defined(GL_FORCE_32BIT_PATH)
    uint32_t a0 = (uint32_t)a, a1 = (uint32_t)(a >> 32);
    uint64_t p00 = (uint64_t)a0 * a0;
    uint64_t p01 = (uint64_t)a0 * a1;
    uint64_t p11 = (uint64_t)a1 * a1;
    // a^2 = p00 + 2*p01*2^32 + p11*2^64
    uint64_t m = p01 + (p00 >> 32);                           // < 2^64
    uint64_t m2 = p01 + (uint32_t)m;                          // < 2^64
    hi = p11 + (m >> 32) + (m2 >> 32);
    lo = (m2 << 32) | (uint32_t)p00;
#else
    unsigned __int128 p = (unsigned __int128)a * a;
    lo = (uint64_t)p;
    hi = (uint64_t)(p >> 64);
#endif
}
GL_HD void sqr_wide(uint64_t a, uint64_t& lo, uint64_t& hi) {
#if defined(GL_SQR_3WIDE) || (defined(GL_FORCE_32BIT_PATH) && !defined(__CUDA_ARCH__))
    sqr_wide_3w(a, lo, hi);
#else
    mul_wide(a, a, lo, hi);
#endif
}

GL_HD uint64_t mul(uint64_t a, uint64_t b) {
    uint64_t lo, hi;
    mul_wide(a, b, lo, hi);
    return reduce128(lo, hi);
}
GL_HD uint64_t sqr(uint64_t a) {
    uint64_t lo, hi;
    sqr_wide(a, lo, hi);
    return reduce128(lo, hi);
}
GL_HD uint64_t sqr_3w(uint64_t a) {
    uint64_t lo, hi;
    sqr_wide_3w(a, lo, hi);
    return reduce128(lo, hi);
}
// a * b + c (mod p) with one reduction (multiply_accumulate, goldilocks_field.rs:184-188)
GL_HD uint64_t mul_add(uint64_t a, uint64_t b, uint64_t c) {
    uint64_t lo, hi;
    mul_wide(a, b, lo, hi);
#if defined(__CUDA_ARCH__)
    uint32_t l0, l1, h0, h1;  // a*b + c < 2^128
    asm("add.cc.u32 %0, %4, %6;\n\taddc.cc.u32 %1, %5, %7;\n\taddc.cc.u32 %2, %8, 0;\n\taddc.u32 %3, %9, 0;"
        : "=&r"(l0), "=&r"(l1), "=&r"(h0), "=&r"(h1)
        : "r"(lo32(lo)), "r"(hi32(lo)), "r"(lo32(c)), "r"(hi32(c)), "r"(lo32(hi)), "r"(hi32(hi)));
    return reduce128(pack64(l0, l1), pack64(h0, h1));
#else
    uint64_t l2 = lo + c;
    hi += (l2 < lo);  // a*b + c < 2^128
    return reduce128(l2, hi);
#endif
}

// a * 2^k (mod p), 0 <= k < 96, using 2^64 = EPS, 2^96 = -1.
GL_HD uint64_t mul_pow2(uint64_t a, uint32_t k) {
    if (k == 0) return a;
    if (k < 32) {
        uint64_t lo = a << k;
        uint32_t hi = (uint32_t)(a >> (64 - k));
        return reduce96(lo, hi);
    } else if (k == 32) {
        return reduce96(a << 32, (uint32_t)(a >> 32));
    } else if (k < 64) {
        uint64_t lo = a << k;
        uint64_t hi = a >> (64 - k);  // < 2^k, k < 64
        return reduce128(lo, hi);
    } else {
        // 64 <= k < 96, k = 64 + j: with (v2:v1:v0) = a << j (96 bits, v2 < 2^31),
        // a*2^k = v0*2^64 + v1*2^96 + v2*2^128 = v0*(2^32 - 1) - v1 - v2*2^32   (2^96 = -1, 2^128 = -2^32)
        //       = (v0 << 32) - ((v2 << 32) + v0 + v1):  one modular subtraction; the subtrahend is < 2^63 < p,
        // so a single borrow fix-up is exact.
        uint32_t j = k - 64;
        uint64_t sh = j ? (a << j) : a;
        uint32_t v0 = (uint32_t)sh, v1 = (uint32_t)(sh >> 32);
        uint32_t v2 = j ? (uint32_t)(a >> (64 - j)) : 0u;
        uint64_t A = (uint64_t)v0 << 32;
        uint64_t B = ((uint64_t)v2 << 32) + v0 + v1;
        uint64_t d = A - B;
        return (A < B) ? d - EPS : d;
    }
}

GL_HD uint64_t pow(uint64_t base, uint64_t e) {
    uint64_t cur = base, acc = 1;
    while (e) {
        if (e & 1) acc = mul(acc, cur);
        cur = sqr(cur);
        e >>= 1;
    }
    return acc;
}
GL_HD uint64_t inv(uint64_t a) { return pow(a, P - 2); }  // try_inverse, goldilocks_field.rs:108-147
// primitive_root_of_unity, field/src/types.rs:268-272
GL_HD uint64_t root_of_unity(uint32_t log_n) {
    uint64_t b = POWER_OF_TWO_GENERATOR;
    for (uint32_t i = log_n; i < TWO_ADICITY; i++) b = sqr(b);
    return b;
}
// inverse_2exp, field/src/types.rs:226-266
GL_HD uint64_t inverse_2exp(uint32_t k) { return P - ((P - 1) >> k); }

// ---- quadratic extension F[X]/(X^2 - 7) (goldilocks_extensions.rs:14-27, quadratic.rs:180-193)
struct E2 {
    uint64_t a, b;
};
GL_HD E2 e2_add(E2 x, E2 y) { return E2{add(x.a, y.a), add(x.b, y.b)}; }
GL_HD E2 e2_sub(E2 x, E2 y) { return E2{sub(x.a, y.a), sub(x.b, y.b)}; }
GL_HD E2 e2_mul(E2 x, E2 y) {
    // c0 = a0*b0 + 7*a1*b1 ; c1 = a0*b1 + a1*b0
    uint64_t t = mul(x.b, y.b);
    uint64_t t7 = sub(mul_pow2(t, 3), t);
    return E2{mul_add(x.a, y.a, t7), mul_add(x.a, y.b, mul(x.b, y.a))};
}
GL_HD E2 e2_scale(E2 x, uint64_t s) { return E2{mul(x.a, s), mul(x.b, s)}; }
GL_HD E2 e2_inv(E2 x) {
    uint64_t t = sqr(x.b);
    uint64_t norm = sub(sqr(x.a), sub(mul_pow2(t, 3), t));
    uint64_t ni = inv(norm);
    return E2{mul(x.a, ni), mul(neg(x.b), ni)};
}
GL_HD E2 e2_pow(E2 base, uint64_t e) {
    E2 cur = base, acc = E2{1, 0};
    while (e) {
        if (e & 1) acc = e2_mul(acc, cur);
        cur = e2_mul(cur, cur);
        e >>= 1;
    }
    return acc;
}

GL_HD uint32_t bitrev32(uint32_t x, uint32_t bits) {
#if defined(__CUDA_ARCH__)
    return bits ? (__brev(x) >> (32 - bits)) : 0;
#else
    uint32_t r = 0;
    for (uint32_t i = 0; i < bits; i++) r |= ((x >> i) & 1u) << (bits - 1 - i);
    return r;
#endif
}

}  // namespace gl
