// gl_poseidon.cuh -- Poseidon-12 (x^7, 4 + 22 + 4 rounds) over Goldilocks and the sponge built on it.
//
// Replaces (reference, CPU): Poseidon::poseidon and layers  plonky2/src/hash/poseidon.rs:630-641,689-777
//                            hash_n_to_m_no_pad / compress    plonky2/src/hash/hashing.rs:97-145
//                            Hasher::hash_or_noop             plonky2/src/plonk/config.rs:63-74
//
// One thread owns one 12-lane state. The kernels built on this are bound by instruction issue on the integer
// pipes (IMAD.WIDE alone costs ~5 issue cycles, tools/pipe_mix.cu), so everything that is linear with small
// constants runs on the FP64 pipe instead, exactly (integers < 2^53 in doubles):
//  * full rounds: x^7 = two squarings + two multiplies per lane on the integer pipes; the last 128-bit product is
//    handed to the FP64 pipe unreduced (sbox7_f64: 2^64 = 2^32 - 1, 2^96 = -1 turn its four words into a signed
//    limb pair, built as 2^52-offset bit patterns by integer adds, one FP64 add each), the circulant MDS runs on two
//    32-bit-limb vectors through x^12 - 1 = (x^6 - 1)(x^6 + 1) (circ12_f64: 96 FP64 operations per vector) with the
//    NEXT round's constants as seeds, and a short 2^64 = 2^32 - 1 fold per lane brings the state back
//    (f64_pair_to_u64);
//  * partial rounds: lanes 1..11 never leave the FP64 pipe for all 22 rounds and two rounds are one linear step
//    (poseidon_partial_rounds_f64) -- the reference's "fast" w_hat / v factorisation (23 64x64 products per
//    round) is only used on the host and under -DGL_PARTIAL_FAST;
//  * f64 -> u64 conversions are F2I on the XU pipe; the squarings are three 32x32 products each (sqr_3w).
// The rounds are rolled loops (one copy of each round body) so the permutation fits the instruction cache.
// Each of these steps (single 128-bit product, FP64-resident partial rounds, two rounds per step, split circulant
// MDS) was kept because it raised the leaf-hash permutation rate over the integer fast form; tools/variants/
// re-ranks the alternatives on the GPU at hand.
#pragma once
#include "gl_field.cuh"
#include "gl_poseidon_constants.h"

// Evaluate the MDS layer's 6-bit-constant products on the FP64 pipe: DFMA issues at the same 64 lanes/clk/SM as
// IMAD on its own pipe (tools/pipe_mix.cu: a DFMA + IMAD stream runs at the speed of either alone), and every
// sum is < 2^53, so doubles are exact. Define GL_MDS_INT to force the integer (IMAD.WIDE) formulation.
// Other measured alternatives kept as switches: GL_PARTIAL_FAST (integer rounds everywhere),
// GL_CVT_MAGIC (2^52 magic-number conversions on the FP64 pipe everywhere), GL_SBOX_I2F (I2F in the S-box),
// GL_SBOX_SQR4 (four-product squarings in the S-box), GL_PAIR_RENORM_F64 (the partial-round pair's former form:
// two separate rank-one updates, renormalisation on the FP64 pipe), GL_SBOX_MOVE_HANDOVER (the S-box's FP64 limbs
// from four register-built 2^52 + w doubles and five DADDs), GL_RET_REDUCE96 (f64_pair_to_u64 through a full 96-bit
// reduction); gl_field.cuh: GL_SQR_3WIDE, GL_MUL_EXPLICIT, GL_REDUCE_V1. tools/variants/ ranks them with one GPU call.
#if !defined(GL_MDS_INT) && !defined(GL_MDS_FP64)
#define GL_MDS_FP64 1
#endif
// The FP64 formulation is device code; tests/emu compiles it for the host too (-DGL_FP64_ON_HOST) to check its
// exactness argument against the integer formulation without a GPU (IEEE doubles and fma behave identically).
#if defined(GL_MDS_FP64) && (defined(__CUDA_ARCH__) || defined(GL_FP64_ON_HOST))
#define GL_FP64_PATH 1
#endif
// Partial rounds: FP64-resident by default where the FP64 path exists (see poseidon_partial_rounds_f64);
// -DGL_PARTIAL_FAST selects the integer "fast" factorisation (w_hat / v vectors) everywhere.
#if defined(GL_FP64_PATH) && !defined(GL_PARTIAL_FAST)
#define GL_PARTIAL_F64 1
#endif

namespace gl {

struct PoseidonTables {
    uint64_t rc[360];
    uint64_t fast_first[12];
    uint64_t fast_rc[22];
    uint64_t vs[22 * 11];
    uint64_t w_hats[22 * 11];
    uint64_t init[11 * 11];
    uint64_t zeros[12];  // "no constants" block for the last round's folded constant layer
    // MDS first row (poseidon_goldilocks.rs:24) read from the constant bank ON PURPOSE: as literals the
    // compiler strength-reduces x2 / x16 / x18 ... into shift+add sequences on the (bottleneck) ALU pipe;
    // as constant-bank operands every term is one IMAD.WIDE.U32 on the FMA pipe.
    uint32_t mds_circ[12];
    uint32_t mds_00;  // circ[0] + diag[0]
    uint32_t pad_;
    double mds_f64[13];  // the same constants as doubles ([12] = circ[0] + diag[0]) for the FP64-pipe variant
    // constants that follow full round r's MDS (r = 0..7: rounds 1-3, partial first layer, rounds 27-29, none),
    // pre-split into 32-bit halves AS DOUBLES ([2i] = low half of lane i, [2i+1] = high half): the FP64 MDS
    // starts its accumulators from them straight out of the constant bank.
    // row 8: the ORIGINAL first partial-round constants (ALL_ROUND_CONSTANTS[48..59]) for the FP64-resident
    // partial rounds, which run in the original (non-"fast") basis.
    double nrc_f64[9][24];
    // the same rows + the bias (bl2, bh2) = (2^42 + 2^10, 2^42 - 2^11) = 0 (mod p) on every lane (the MDS inputs
    // that come from sbox7_f64 have signed low limbs, |L| < 2^33), in the SEED form of circ12_f64:
    // [0..5] = (kL[r] + kL[r+6])/2, [6..11] = (kL[r] - kL[r+6])/2 for the low limbs kL, [12..23] for the high limbs.
    double nrcs_f64[9][24];
    // FP64-resident partial rounds, two rounds per linear step (poseidon_partial_rounds_f64): with cA / cB the
    // constant layers that follow rounds A = 2*pair and B = 2*pair + 1 (ALL_ROUND_CONSTANTS[12*(5+r) + i]),
    // x' = C*C*x~ + 8*x~0*C[:,0] + (a^7 - a)*M[:,0] + 8*a*e0 + k2 with a = (M x~)_0 + cA_0 and
    // k2 = M*cA + cB - 8*cA_0*e0 (mod p). pks_f64[pair] = k2 split in 32-bit halves PLUS a bias (bl, bh) =
    // (2^50 + 2^18, 2^50 - 2^19), bl + 2^32*bh = 2^18 * p = 0 (mod p), on every lane that is converted back to an
    // integer afterwards (lane 0 always; all lanes after the last pair), in the seed form of circ12_f64;
    // pan_f64[pair] = cA_0 split WITHOUT bias (the bias is added at the conversion).
    double pks_f64[11][24];
    double pan_f64[11][2];
    // The default pair (poseidon_partial_rounds_f64) holds lanes 1..11 SHIFTED: y = x - d[pair] (mod p) with d[0] = 0,
    // d[pair + 1] = C*C*d[pair] + k2[pair] on lanes 1..11 (d_0 = 0 always), so that a pair adds no constant to them
    // and only these few constants are read inside the loop:
    // pk0_f64[pair] = lane 0's constant e0 = (C*C*d + k2)_0 + bias, halved: the seed of both row-0 accumulators of
    // circ12_f64 (the halves cancel in out[6]); pad_f64[pair] = cA_0 + (M*d)_0 in 32-bit halves, no bias;
    // pdf_f64 = d[11] + bias on lanes 1..11 ([2(i-1)] low half, [2(i-1)+1] high half), added once after the last pair.
    double pk0_f64[11][2];
    double pad_f64[11][2];
    double pdf_f64[22];
};

#if defined(__CUDACC__)
__constant__ PoseidonTables c_pos;
#endif

inline const PoseidonTables& host_poseidon_tables() {
    static PoseidonTables t = [] {
        PoseidonTables x;
        for (int i = 0; i < 360; i++) x.rc[i] = GL_POSEIDON_RC[i];
        for (int i = 0; i < 12; i++) x.fast_first[i] = GL_POSEIDON_FAST_FIRST_RC[i];
        for (int i = 0; i < 22; i++) x.fast_rc[i] = GL_POSEIDON_FAST_RC[i];
        for (int i = 0; i < 242; i++) x.vs[i] = GL_POSEIDON_FAST_VS[i];
        for (int i = 0; i < 242; i++) x.w_hats[i] = GL_POSEIDON_FAST_W_HATS[i];
        for (int i = 0; i < 121; i++) x.init[i] = GL_POSEIDON_FAST_INIT_MATRIX[i];
        for (int i = 0; i < 12; i++) x.zeros[i] = 0;
        for (int i = 0; i < 12; i++) x.mds_circ[i] = (uint32_t)GL_POSEIDON_MDS_CIRC[i];
        x.mds_00 = (uint32_t)(GL_POSEIDON_MDS_CIRC[0] + GL_POSEIDON_MDS_DIAG[0]);
        x.pad_ = 0;
        for (int i = 0; i < 12; i++) x.mds_f64[i] = (double)GL_POSEIDON_MDS_CIRC[i];
        x.mds_f64[12] = (double)(GL_POSEIDON_MDS_CIRC[0] + GL_POSEIDON_MDS_DIAG[0]);
        for (int r = 0; r < 9; r++) {
            const uint64_t* src = (r < 3) ? &x.rc[12 * (r + 1)] : (r == 3) ? x.fast_first
                                : (r < 7) ? &x.rc[12 * (r + 23)] : (r == 7) ? x.zeros : &x.rc[48];
            for (int i = 0; i < 12; i++) {
                x.nrc_f64[r][2 * i] = (double)(uint32_t)src[i];
                x.nrc_f64[r][2 * i + 1] = (double)(uint32_t)(src[i] >> 32);
            }
            // bl2 + 2^32*bh2 = 2^10 + 2^42 + 2^74 - 2^43 = 2^74 - 2^42 + 2^10 = 2^10 * p
            const double b2[2] = {4398046511104.0 + 1024.0, 4398046511104.0 - 2048.0};
            for (int q = 0; q < 6; q++)
                for (int l = 0; l < 2; l++) {  // limb: 0 = low, 1 = high
                    const double k0 = x.nrc_f64[r][2 * q + l] + b2[l], k6 = x.nrc_f64[r][2 * (q + 6) + l] + b2[l];
                    x.nrcs_f64[r][12 * l + q] = (k0 + k6) * 0.5;
                    x.nrcs_f64[r][12 * l + 6 + q] = (k0 - k6) * 0.5;
                }
        }
        // bias: bl = 2^50 + 2^18, bh = 2^50 - 2^19;  bl + 2^32*bh = 2^82 - 2^50 + 2^18 = 2^18 * p
        const double bl = 1125899906842624.0 + 262144.0, bh = 1125899906842624.0 - 524288.0;
        // pair tables
        uint64_t M[12][12];
        for (int i = 0; i < 12; i++)
            for (int j = 0; j < 12; j++)
                M[i][j] = GL_POSEIDON_MDS_CIRC[(j - i + 12) % 12] + ((i == 0 && j == 0) ? GL_POSEIDON_MDS_DIAG[0] : 0);
        const unsigned __int128 PP = (unsigned __int128)0xFFFFFFFF00000001ULL;
        uint64_t CC[12][12];  // C*C, C = M without its diagonal
        for (int i = 0; i < 12; i++)
            for (int j = 0; j < 12; j++) {
                CC[i][j] = 0;
                for (int t = 0; t < 12; t++) CC[i][j] += GL_POSEIDON_MDS_CIRC[(t - i + 12) % 12] * GL_POSEIDON_MDS_CIRC[(j - t + 12) % 12];
            }
        uint64_t d[12] = {0};  // the shift of lanes 1..11 going into pair pr
        for (int pr = 0; pr < 11; pr++) {
            const uint64_t* cA = &x.rc[12 * (5 + 2 * pr)];      // constants after round A = 2*pr
            const uint64_t* cB = &x.rc[12 * (5 + 2 * pr + 1)];  // constants after round B = 2*pr + 1
            x.pan_f64[pr][0] = (double)(uint32_t)cA[0];
            x.pan_f64[pr][1] = (double)(uint32_t)(cA[0] >> 32);
            double k2[12][2];
            uint64_t k2r[12];
            for (int i = 0; i < 12; i++) {
                unsigned __int128 k = cB[i];
                for (int t = 0; t < 12; t++) k += (unsigned __int128)M[i][t] * cA[t];
                if (i == 0) k += 8 * (PP - cA[0] % PP);  // - 8*cA_0 on lane 0
                const uint64_t kr = (uint64_t)(k % PP);
                k2r[i] = kr;
                const bool biased = (i == 0) || (pr == 10);
                k2[i][0] = (double)(uint32_t)kr + (biased ? bl : 0.0);
                k2[i][1] = (double)(uint32_t)(kr >> 32) + (biased ? bh : 0.0);
            }
            {
                unsigned __int128 a = cA[0];
                for (int t = 0; t < 12; t++) a += (unsigned __int128)M[0][t] * d[t];
                const uint64_t ar = (uint64_t)(a % PP);
                x.pad_f64[pr][0] = (double)(uint32_t)ar;
                x.pad_f64[pr][1] = (double)(uint32_t)(ar >> 32);
                uint64_t e[12];
                for (int i = 0; i < 12; i++) {
                    unsigned __int128 v = k2r[i];
                    for (int t = 0; t < 12; t++) v += (unsigned __int128)CC[i][t] * d[t];
                    e[i] = (uint64_t)(v % PP);
                }
                x.pk0_f64[pr][0] = ((double)(uint32_t)e[0] + bl) * 0.5;
                x.pk0_f64[pr][1] = ((double)(uint32_t)(e[0] >> 32) + bh) * 0.5;
                d[0] = 0;
                for (int i = 1; i < 12; i++) d[i] = e[i];
            }
            for (int q = 0; q < 6; q++)
                for (int l = 0; l < 2; l++) {
                    x.pks_f64[pr][12 * l + q] = (k2[q][l] + k2[q + 6][l]) * 0.5;
                    x.pks_f64[pr][12 * l + 6 + q] = (k2[q][l] - k2[q + 6][l]) * 0.5;
                }
        }
        for (int i = 1; i < 12; i++) {
            x.pdf_f64[2 * (i - 1)] = (double)(uint32_t)d[i] + bl;
            x.pdf_f64[2 * (i - 1) + 1] = (double)(uint32_t)(d[i] >> 32) + bh;
        }
        return x;
    }();
    return t;
}

#if defined(__CUDA_ARCH__)
#define GL_POS (c_pos)
#else
#define GL_POS (host_poseidon_tables())
#endif

// 160-bit accumulator for sums of 64x64 products.
struct Acc160 {
    uint64_t lo, hi;
    uint32_t top;
};
GL_HD void acc_mul(Acc160& a, uint64_t x, uint64_t y) {
    uint64_t pl, ph;
    mul_wide(x, y, pl, ph);
#if defined(__CUDA_ARCH__)
    asm("add.cc.u64 %0, %0, %3;\n\taddc.cc.u64 %1, %1, %4;\n\taddc.u32 %2, %2, 0;"
        : "+l"(a.lo), "+l"(a.hi), "+r"(a.top)
        : "l"(pl), "l"(ph));
#else
    unsigned __int128 s = (unsigned __int128)a.lo + pl;
    a.lo = (uint64_t)s;
    unsigned __int128 h = (unsigned __int128)a.hi + ph + (uint64_t)(s >> 64);
    a.hi = (uint64_t)h;
    a.top += (uint32_t)(h >> 64);
#endif
}
GL_HD uint64_t acc_reduce(const Acc160& a) {
    // top*2^128 + hi*2^64 + lo ; 2^128 = 2^96 * 2^32 = -2^32 (mod p)
    uint64_t r = reduce128(a.lo, a.hi);
    return sub(r, (uint64_t)a.top << 32);
}

// Compile-time copy of the MDS matrix M[i][j] = circ[(j - i) mod 12] (+ diag on [0][0]), so that fully unrolled
// FP64 code gets its entries as literal operands (DFMA immediates).
GL_HD constexpr uint32_t mds_entry(int i, int j) {
    constexpr uint32_t circ[12] = {17, 15, 41, 16, 2, 28, 13, 13, 39, 18, 34, 20};  // poseidon_goldilocks.rs:24
    return circ[(j - i + 12) % 12] + ((i == 0 && j == 0) ? 8u : 0u);                  // diag = [8, 0, ...]: :25
}

// The circulant part C (first row circ) through x^12 - 1 = (x^6 - 1)(x^6 + 1): with v+- = v[0..5] +- v[6..11] and
// c+- = (circ[0..5] +- circ[6..11]) / 2, out[r] +- out[r+6] are a cyclic / negacyclic length-6 correlation:
//   S+[r] = sum_j v+[j] * c+[(j - r) mod 6],   S-[r] = sum_{j>=r} v-[j] * c-[j - r] - sum_{j<r} v-[j] * c-[j - r + 6],
//   out[r] = S+[r] + S-[r],  out[r+6] = S+[r] - S-[r]
// = 12 + 72 + 12 FP64 operations instead of 144 (the halves make some values multiples of 1/2: still exact).
// MdsCirc is C itself, MdsCirc2 is C*C (two partial rounds in one step), entries < 2^14.4.
struct MdsCirc {
    static GL_HD constexpr double c(int d) {
        constexpr double circ[12] = {17, 15, 41, 16, 2, 28, 13, 13, 39, 18, 34, 20};
        return circ[((d % 12) + 12) % 12];
    }
};
struct MdsCirc2 {
    static GL_HD constexpr double c(int d) {  // (C*C x)[r] = sum_l x[l] * c2[(l - r) mod 12],  c2 = circ (*) circ
        double a = 0;
        for (int t = 0; t < 12; t++) a += MdsCirc::c(t) * MdsCirc::c(d - t);
        return a;
    }
};
template <class K>
GL_HD constexpr double circ_half_p(int k) { return (K::c(k) + K::c(k + 6)) * 0.5; }
template <class K>
GL_HD constexpr double circ_half_m(int k) { return (K::c(k) - K::c(k + 6)) * 0.5; }

#if !defined(GL_F64_TRACK)
#define GL_F64_TRACK(x)  // tests/emu hooks the largest limb magnitude here
#endif
#if defined(GL_FP64_PATH)
// ---- exact integer arithmetic on the FP64 pipe: every double below holds an integer of magnitude < 2^53 ----
GL_HD double f64_fma(double a, double b, double c) {
#if defined(__CUDA_ARCH__)
    return fma(a, b, c);
#else
    return __builtin_fma(a, b, c);
#endif
}
GL_HD double u32_to_f64(uint32_t x) {
#if defined(__CUDA_ARCH__) && defined(GL_CVT_MAGIC)
    return __hiloint2double(0x43300000, (int)x) - 4503599627370496.0;  // bits(2^52 + x) = 0x43300000:x (MOV + DADD)
#else
    return (double)x;  // I2F.F64.U32 on the (idle) XU pipe: one instruction, exact
#endif
}
// The double 2^52 + x (bit pattern 0x43300000:x), exact for any 32-bit x.
GL_HD double u32_magic_f64(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __hiloint2double(0x43300000, (int)x);
#else
    const uint64_t b = 0x4330000000000000ULL | x;
    double d;
    __builtin_memcpy(&d, &b, 8);
    return d;
#endif
}
// The words of a double's bit pattern, and a double from a bit pattern (register moves on the device).
GL_HD uint32_t f64_lo_word(double x) {
#if defined(__CUDA_ARCH__)
    return (uint32_t)__double2loint(x);
#else
    uint64_t b;
    __builtin_memcpy(&b, &x, 8);
    return (uint32_t)b;
#endif
}
GL_HD uint32_t f64_hi_word(double x) {
#if defined(__CUDA_ARCH__)
    return (uint32_t)__double2hiint(x);
#else
    uint64_t b;
    __builtin_memcpy(&b, &x, 8);
    return (uint32_t)(b >> 32);
#endif
}
GL_HD double f64_from_bits(uint64_t b) {
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)b);
#else
    double d;
    __builtin_memcpy(&d, &b, 8);
    return d;
#endif
}
// al + 2^32 * ah (mod p) for NON-NEGATIVE integers al, ah < 2^52 held in doubles.
GL_HD uint64_t f64_pair_to_u64(double al, double ah) {
#if (defined(__CUDA_ARCH__) || defined(GL_FORCE_32BIT_PATH)) && !defined(GL_CVT_MAGIC) && !defined(GL_RET_REDUCE96)
    // ul = al, uh = ah < 2^52 as integers (F2I.U64.F64 on the XU pipe). With uh = uh0 + 2^32*uh1 and 2^64 = 2^32 - 1:
    //   ul + 2^32*uh = ul + uh1*(2^32 - 1) + 2^32*uh0  (mod p).
    // b = ul + uh1*(2^32 - 1) < 2^52 + 2^52 cannot wrap (one IADD3 + IADD3.X); adding uh0 to its high word wraps at
    // most once (carry c), and then that word is below 2^21, so the fix-up c*(2^32 - 1) cannot wrap: 8 instructions
    // in one PTX carry chain instead of the 96-bit reduction's 10 plus the assembly of its input (written in C, ptxas
    // turns b into an extra IMAD.WIDE and the carry test into compares and selects). The result is some u64
    // congruent to the value, not necessarily the one reduce96 gives; the host build computes the same u64.
#if defined(__CUDA_ARCH__)
    const uint64_t ul = __double2ull_rz(al), uh = __double2ull_rz(ah);
    uint32_t r0, r1;
    asm("{\n\t.reg .u32 t, m;\n\t"
        "add.u32 t, %3, %5;\n\t"         // ul1 + uh1 < 2^21
        "sub.cc.u32 %0, %2, %5;\n\t"     // b = ul + uh1*(2^32 - 1): a borrow implies uh1 > 0, so t > 0
        "subc.u32 %1, t, 0;\n\t"
        "add.cc.u32 %1, %1, %4;\n\t"     // + 2^32*uh0, carry c
        "addc.u32 m, 0, 0;\n\t"
        "neg.s32 m, m;\n\t"              // m = -c: c*(2^32 - 1) = c*2^32 - c, the 2^32 part is the carry itself
        "add.cc.u32 %0, %0, m;\n\t"
        "addc.u32 %1, %1, 0;\n\t}"
        : "=&r"(r0), "=&r"(r1)
        : "r"(lo32(ul)), "r"(hi32(ul)), "r"(lo32(uh)), "r"(hi32(uh)));
    return pack64(r0, r1);
#else
    const uint64_t ul = (uint64_t)al, uh = (uint64_t)ah;
    const uint32_t uh1 = (uint32_t)(uh >> 32);
    const uint64_t b = ul + (((uint64_t)uh1 << 32) - uh1);
    const uint64_t s = b + (uh << 32);
    return s < b ? s + EPS : s;
#endif
#elif defined(__CUDA_ARCH__) && !defined(GL_CVT_MAGIC)
    // F2I.U64.F64 (XU pipe, exact on integers) instead of the 2^52 magic add (FP64 pipe) + mask: fewer instructions
    const uint64_t ul = __double2ull_rz(al), uh = __double2ull_rz(ah);
    uint32_t r1, r2;
    asm("add.cc.u32 %0, %2, %3;\n\taddc.u32 %1, %4, 0;" : "=r"(r1), "=r"(r2) : "r"(hi32(ul)), "r"(lo32(uh)), "r"(hi32(uh)));
    return reduce96(pack64(lo32(ul), r1), r2);
#elif defined(__CUDA_ARCH__)
    // bits(2^52 + v) = 0x43300000 | (v >> 32) : (v & 0xffffffff) for v < 2^52
    const double bl = al + 4503599627370496.0, bh = ah + 4503599627370496.0;
    const uint32_t al0 = (uint32_t)__double2loint(bl), al1 = (uint32_t)__double2hiint(bl) & 0xFFFFFu;
    const uint32_t ah0 = (uint32_t)__double2loint(bh), ah1 = (uint32_t)__double2hiint(bh) & 0xFFFFFu;
    uint32_t r1, r2;
    asm("add.cc.u32 %0, %2, %3;\n\taddc.u32 %1, %4, 0;" : "=r"(r1), "=r"(r2) : "r"(al1), "r"(ah0), "r"(ah1));
    return reduce96(pack64(al0, r1), r2);
#else
    const unsigned __int128 v = (unsigned __int128)(uint64_t)al + ((unsigned __int128)(uint64_t)ah << 32);
    return reduce96((uint64_t)v, (uint32_t)(v >> 64));
#endif
}
// out = Circ(K) * v + k for one limb vector, the constants k given as SEEDS: seed[r] = (k[r] + k[r+6]) / 2,
// seed[6 + r] = (k[r] - k[r+6]) / 2 (r < 6). See MdsCirc above.
template <class K>
GL_HD void circ12_f64(const double v[12], const double* seed, double out[12]) {
    double vp[6], vm[6];
#pragma unroll
    for (int j = 0; j < 6; j++) {
        vp[j] = v[j] + v[j + 6];
        vm[j] = v[j] - v[j + 6];
    }
#pragma unroll
    for (int r = 0; r < 6; r++) {
        double sp = seed[r], sm = seed[6 + r];
#pragma unroll
        for (int j = 0; j < 6; j++) {
            sp = f64_fma(vp[j], circ_half_p<K>((j - r + 6) % 6), sp);
            sm = f64_fma(vm[j], j >= r ? circ_half_m<K>(j - r) : -circ_half_m<K>(j - r + 6), sm);
        }
        GL_F64_TRACK(sp);
        GL_F64_TRACK(sm);
        out[r] = sp + sm;
        out[r + 6] = sp - sm;
    }
}
#endif  // GL_FP64_PATH

GL_HD uint64_t sbox7(uint64_t x) {  // sbox_monomial, poseidon.rs:689-696
    uint64_t x2 = sqr(x);
    uint64_t x4 = sqr(x2);
    uint64_t x3 = mul(x, x2);
    return mul(x3, x4);
}

#if defined(GL_FP64_PATH)
// x^7 handed to the FP64 MDS WITHOUT the last modular reduction: with x^3 * x^4 = (p3 p2 p1 p0) in 32-bit
// words, 2^64 = 2^32 - 1 and 2^96 = -1 give  x^7 = (p0 - p2 - p3) + 2^32 * (p1 + p2)  (mod p), i.e. exactly a
// (signed) limb pair (L, H), |L| < 2^33.6, 0 <= H < 2^33: three FP64 adds replace the 11-instruction integer
// reduce128, and the MDS constants carry a bias = 0 (mod p) that makes its outputs positive again.
// The squarings are the three-product form (sqr_3w; -DGL_SBOX_SQR4 restores mul_wide's four). The limbs enter the
// FP64 pipe as bit patterns built on the integer pipes (2 IADD3-class instructions and one DADD per limb), not through
// I2F.F64, which costs about 6 issue clocks when mixed with IMAD.WIDE (tools/pipe_mix2.cu; -DGL_SBOX_I2F), nor as four
// 2^52 + w doubles (bits 0x43300000:w, a register move each) combined by five DADDs (-DGL_SBOX_MOVE_HANDOVER):
// H = (m1 - 2^53) + m2, L = (m0 - m2) - (m3 - 2^52). All three forms give the same integers L and H.
GL_HD void sbox7_f64(uint64_t x, double& L, double& H) {
#if defined(GL_SBOX_SQR4)
    const uint64_t x2 = sqr(x);
    const uint64_t x4 = sqr(x2);
#else
    const uint64_t x2 = sqr_3w(x);
    const uint64_t x4 = sqr_3w(x2);
#endif
    const uint64_t x3 = mul(x, x2);
    uint64_t lo, hi;
    mul_wide(x3, x4, lo, hi);
#if !defined(GL_SBOX_I2F) && !defined(GL_SBOX_MOVE_HANDOVER)
    // The limbs built as bit patterns on the integer pipes: 2^52 + H and 1.5 * 2^52 + L, each a 64-bit add of
    // 32-bit words to the pattern's constant (IADD3 + IADD3.X), then one DADD removes the offset. H = w1 + w2 < 2^33
    // and -2^33 < L = w0 - w2 - w3 < 2^32 are the same integers as below, so the patterns hold them exactly
    // (2^52 <= 2^52 + H < 2^53 and 2^52 <= 1.5 * 2^52 + L < 2^53: one unit in the last place is 1).
    const uint64_t hb = 0x4330000000000000ULL + (lo >> 32) + (uint32_t)hi;
    const uint64_t lb = 0x4338000000000000ULL + (uint32_t)lo - (uint64_t)(uint32_t)hi - (hi >> 32);
    H = f64_from_bits(hb) - 4503599627370496.0;  // 2^52
    L = f64_from_bits(lb) - 6755399441055744.0;  // 1.5 * 2^52
#elif !defined(GL_SBOX_I2F)
    const double m0 = u32_magic_f64((uint32_t)lo), m1 = u32_magic_f64((uint32_t)(lo >> 32));
    const double m2 = u32_magic_f64((uint32_t)hi), m3 = u32_magic_f64((uint32_t)(hi >> 32));
    H = (m1 - 9007199254740992.0) + m2;
    L = (m0 - m2) - (m3 - 4503599627370496.0);
#else
    const double d0 = u32_to_f64((uint32_t)lo), d1 = u32_to_f64((uint32_t)(lo >> 32));
    const double d2 = u32_to_f64((uint32_t)hi), d3 = u32_to_f64((uint32_t)(hi >> 32));
    L = (d0 - d2) - d3;
    H = d1 + d2;
#endif
}
#endif

// mds_layer (poseidon.rs:269-290; out[r] = sum_i s[(i+r)%12]*circ[i] + s[r]*diag[r]) on 32-bit halves,
// FUSED with the constant layer that follows it (poseidon.rs:630-641): the accumulators start from the
// next round's constants `nrc` (canonical u64s), so the constant addition costs nothing.
// `nrcd` (device, optional): the same constants pre-split as doubles (PoseidonTables::nrc_f64[r]).
GL_HD void mds_layer_add(uint64_t s[12], const uint64_t* nrc, const double* nrcd = nullptr) {
    (void)nrcd;
    const PoseidonTables& T = GL_POS;
#if defined(GL_FP64_PATH)
    // Evaluate the 12x12 small-constant products on the FP64 pipe (idle otherwise). Every term is
    // (32-bit half) x (6-bit constant) and a 13-term sum stays < 2^42, so double arithmetic is EXACT.
    {
        double dl[12], dh[12];
#pragma unroll
        for (int i = 0; i < 12; i++) {
            dl[i] = u32_to_f64((uint32_t)s[i]);
            dh[i] = u32_to_f64((uint32_t)(s[i] >> 32));
        }
#pragma unroll
        for (int r = 0; r < 12; r++) {
            double al, ah;
            if (nrcd) {
                al = nrcd[2 * r];
                ah = nrcd[2 * r + 1];
            } else {
                const uint64_t c = nrc[r];
                al = u32_to_f64((uint32_t)c);
                ah = u32_to_f64((uint32_t)(c >> 32));
            }
#pragma unroll
            for (int i = 0; i < 12; i++) {
                const double m = (r == 0 && i == 0) ? T.mds_f64[12] : T.mds_f64[i];
                al = f64_fma(dl[(i + r) % 12], m, al);
                ah = f64_fma(dh[(i + r) % 12], m, ah);
            }
            s[r] = f64_pair_to_u64(al, ah);
        }
    }
#else
    uint32_t lo[12], hi[12];
#pragma unroll
    for (int i = 0; i < 12; i++) {
        lo[i] = (uint32_t)s[i];
        hi[i] = (uint32_t)(s[i] >> 32);
    }
#pragma unroll
    for (int r = 0; r < 12; r++) {
        const uint64_t c = nrc[r];
        uint64_t al = (uint32_t)c, ah = c >> 32;
#pragma unroll
        for (int i = 0; i < 12; i++) {
            const uint32_t m = (r == 0 && i == 0) ? T.mds_00 : T.mds_circ[i];  // diag = [8,0,...,0]
#if defined(__CUDA_ARCH__)
            // explicit mad.wide: the C form makes nvcc emit an extra (zero) high-word add per term
            asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(al) : "r"(lo[(i + r) % 12]), "r"(m));
            asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(ah) : "r"(hi[(i + r) % 12]), "r"(m));
#else
            al += (uint64_t)lo[(i + r) % 12] * m;
            ah += (uint64_t)hi[(i + r) % 12] * m;
#endif
        }
        // value = al + ah * 2^32, al,ah < 2^42  ->  96-bit (l64, h32)
#if defined(__CUDA_ARCH__)
        uint32_t r1, r2;
        asm("add.cc.u32 %0, %2, %3;\n\taddc.u32 %1, %4, 0;"
            : "=r"(r1), "=r"(r2)
            : "r"(hi32(al)), "r"(lo32(ah)), "r"(hi32(ah)));
        s[r] = reduce96(pack64(lo32(al), r1), r2);
#else
        uint64_t l64 = al + (ah << 32);
        uint32_t h32 = (uint32_t)(ah >> 32) + (l64 < al ? 1u : 0u);
        s[r] = reduce96(l64, h32);
#endif
    }
#endif
}
GL_HD void mds_layer(uint64_t s[12]) { mds_layer_add(s, GL_POS.zeros); }

// One full round WITHOUT its own constant layer (already folded into the previous MDS / added by the
// caller) but WITH the next round's: sbox_layer, then mds_layer + next constants.
GL_HD void full_round_fused(uint64_t s[12], const uint64_t* next_rc, const double* next_rcd = nullptr) {
#pragma unroll
    for (int i = 0; i < 12; i++) s[i] = sbox7(s[i]);
    mds_layer_add(s, next_rc, next_rcd);
}
#if defined(GL_FP64_PATH)
// The same round with the S-box outputs going straight to the FP64 pipe (sbox7_f64) and the split-circulant MDS;
// `rcs` = a row of PoseidonTables::nrcs_f64 (next constants + bias, seed form).
GL_HD void full_round_f64(uint64_t s[12], const double* rcs) {
    double dl[12], dh[12];
#pragma unroll
    for (int i = 0; i < 12; i++) sbox7_f64(s[i], dl[i], dh[i]);
    double ol[12], oh[12];
    circ12_f64<MdsCirc>(dl, rcs, ol);
    ol[0] = f64_fma(dl[0], 8.0, ol[0]);  // + diag[0] * v[0]
    circ12_f64<MdsCirc>(dh, rcs + 12, oh);
    oh[0] = f64_fma(dh[0], 8.0, oh[0]);
#pragma unroll
    for (int r = 0; r < 12; r++) {
        GL_F64_TRACK(ol[r]);
        GL_F64_TRACK(oh[r]);
        s[r] = f64_pair_to_u64(ol[r], oh[r]);
    }
}
#endif
// Plain full round (constant_layer, sbox_layer, mds_layer; poseidon.rs:741-749) -- used by tools/microbench.
GL_HD void full_round(uint64_t s[12], const uint64_t* rc) {
#pragma unroll
    for (int i = 0; i < 12; i++) s[i] = add_canonical(s[i], rc[i]);
    full_round_fused(s, GL_POS.zeros);
}

// partial_rounds, poseidon.rs:751-764 (fast form), minus partial_first_constant_layer which the caller
// folds into the preceding MDS. Kept compact on purpose: the init matrix runs as a rolled loop over output
// lanes (results staged in a small local array) and the 22 rounds as a rolled loop, so that the whole
// permutation stays close to the instruction-cache size (the fully unrolled form is ~9k instructions and
// stalls on instruction fetch).
GL_HD void poseidon_partial_rounds_noconst(uint64_t s[12]) {
    const PoseidonTables& T = GL_POS;
    // mds_partial_layer_init (poseidon.rs:413-441)
    {
        uint64_t res[11];
#pragma unroll 1
        for (int c = 0; c < 11; c++) {
            Acc160 a = {0, 0, 0};
#pragma unroll
            for (int r = 1; r < 12; r++) acc_mul(a, s[r], T.init[(r - 1) * 11 + c]);
            res[c] = acc_reduce(a);
        }
#pragma unroll
        for (int i = 1; i < 12; i++) s[i] = res[i - 1];
    }
#pragma unroll 1
    for (int r = 0; r < 22; r++) {
        uint64_t s0 = add_canonical(sbox7(s[0]), T.fast_rc[r]);
        // mds_partial_layer_fast (poseidon.rs:514-542)
        Acc160 a = {0, 0, 0};
        acc_mul(a, s0, T.mds_00);
#pragma unroll
        for (int i = 1; i < 12; i++) acc_mul(a, s[i], T.w_hats[r * 11 + i - 1]);
#pragma unroll
        for (int i = 1; i < 12; i++) s[i] = mul_add(s0, T.vs[r * 11 + i - 1], s[i]);
        s[0] = acc_reduce(a);
    }
}
#if defined(GL_FP64_PATH)
// partial_rounds (poseidon.rs:751-764) in the ORIGINAL basis (constant_layer, x^7 on lane 0, mds_layer -- the
// reference's poseidon_naive form, poseidon.rs:779-801), with lanes 1..11 kept RESIDENT ON THE FP64 PIPE: they
// pass through no non-linearity for 22 rounds, only through the small-constant circulant MDS, so each lane is
// held as two doubles (L, H), value = L + 2^32*H (mod p). Only lane 0 crosses to the integer pipes (x^7).
// Two rounds are ONE linear step: lane 0's second S-box input needs just row 0 of the first MDS, so with
// x~ = (x0^7, x1..x11), M = C + 8*e0*e0^T (C circulant) a PAIR of rounds is
//     a  = (M x~)_0 + cA_0                                                        (12 DFMAs per limb)
//     x' = Q x~ + a^7 * M[:,0] + k,   Q = M diag(0,1..1) M,  k = M diag(0,1..1) cA + cB
//        = C*C*x~ + 8*x~0*C[:,0] + (a^7 - a)*M[:,0] + 8*a*e0 + k2,   k2 = M*cA + cB - 8*cA_0*e0
// so that the split-circulant form (circ12_f64) applies to C*C, and with M[:,0] = C[:,0] + 8*e0 the three rank-one
// terms are one: 8*x~0*C[:,0] + (a^7 - a)*M[:,0] + 8*a*e0 = (8*x~0 + a^7 - a)*C[:,0] + 8*a^7*e0
// (partial_pair_limbs): 96 + 15 FP64 operations per limb (-DGL_PAIR_RENORM_F64: 96 + 26, the terms one by one).
// All matrix entries are compile-time literals (DFMA immediates). The constants k2 would cost 24 constant loads
// indexed by the pair counter per pair, so lanes 1..11 are held shifted, y = x - d[pair] (mod p), with
// d[pair + 1] = C*C*d[pair] + k2 chosen on the host so that a pair adds nothing to them: only lane 0's constant and
// a's (PoseidonTables::pk0_f64 / pad_f64) are read per pair, and d[11] once after the last pair (pdf_f64).
// Under GL_PAIR_RENORM_F64 the pair reads k2 and cA_0 from pks_f64 / pan_f64.
// Exactness: limbs are integers. After a renormalisation -2^18 < L, H < 2^32 + 2^18 (partial_pair_renorm;
// |L|, |H| <= 2^31 + 2^18 under GL_PAIR_RENORM_F64); the row sums of Q are <= 264^2 (those of C*C are 256^2),
// lane 0 enters with |L| < 2^33.6, 0 <= H < 2^33 (sbox7_f64), so an unbiased lane of a pair stays < 2^49 < 2^53 and
// the sums of halves inside circ12_f64 below 2^52; then lanes 1..11 are renormalised: X + 1.5*2^52 exposes
// X = r + 2^32*q in its bit pattern, and 2^64 = 2^32 - 1 folds the high limb's q back (5 ALU + 4 FP64
// instructions per lane; under GL_PAIR_RENORM_F64 9 FP64 operations that round to multiples of 2^32 with
// 1.5*2^84). Limbs that are converted to integers (lane 0 twice per pair, all lanes after the last pair) can be
// negative, so their constants carry a bias (bl, bh) = 0 (mod p) of 2^50 and f64_pair_to_u64 sees non-negative
// integers < 2^51 (tests/emu/poseidon_f64_emu.cpp tracks the bound).
// Versus the "fast" integer form (23 64x64 products + 12 reductions per round, all on the integer pipes that
// bound this kernel): no init matrix, ~90 integer instructions per round instead of ~520.
// In: s after full round 4's MDS + first partial constant layer (original constants). Out: s after the last
// partial round's MDS + the 5th full round's constant layer.
// One limb vector of a pair: v <- C*C*v + k + (rank-one terms), with x0 = v[0] = x~0's limb, z = a^7's, a = a's.
// k: the constants in seed form (GL_PAIR_RENORM_F64, a row of pks_f64), else lane 0's halved constant only
// (pk0_f64: the shifted lanes 1..11 get none).
GL_HD void partial_pair_limbs(double v[12], const double* k, double z, double a) {
    const double x0 = v[0];
    double n[12];
#if defined(GL_PAIR_RENORM_F64)
    circ12_f64<MdsCirc2>(v, k, n);
#else
    const double seed[12] = {k[0], 0, 0, 0, 0, 0, k[0], 0, 0, 0, 0, 0};  // out[0] = 2*k[0], out[6] = 0
    circ12_f64<MdsCirc2>(v, seed, n);
#endif
#if defined(GL_PAIR_RENORM_F64)
    const double za = z - a;
#pragma unroll
    for (int i = 0; i < 12; i++) {
        n[i] = f64_fma(x0, 8.0 * MdsCirc::c(12 - i), n[i]);  // 8 * x~0 * C[:,0]
        n[i] = f64_fma(za, (double)mds_entry(i, 0), n[i]);   // (a^7 - a) * M[:,0]
    }
    n[0] = f64_fma(a, 8.0, n[0]);
#else
    // 8*x~0*C[:,0] + (a^7 - a)*M[:,0] + 8*a*e0 = (8*x~0 + a^7 - a)*C[:,0] + 8*a^7*e0   (M[:,0] = C[:,0] + 8*e0)
    const double w = f64_fma(x0, 8.0, z - a);
#pragma unroll
    for (int i = 0; i < 12; i++) n[i] = f64_fma(w, MdsCirc::c(12 - i), n[i]);
    n[0] = f64_fma(z, 8.0, n[0]);
#endif
#pragma unroll
    for (int i = 0; i < 12; i++) {
        v[i] = n[i];
        GL_F64_TRACK(n[i]);
    }
}
// Renormalise a lane between pairs: integers |L|, |H| < 2^49 -> L', H' with L' + 2^32*H' = L + 2^32*H (mod p).
GL_HD void partial_pair_renorm(double& L, double& H) {
#if defined(GL_PAIR_RENORM_F64)
    // on the FP64 pipe: round H to a multiple of 2^32 (x + 1.5*2^84 - 1.5*2^84), move that carry into L with
    // 2^64 = 2^32 - 1, round L the same way and move its carry into H: |L'|, |H'| <= 2^31 + 2^18, 9 FP64 operations
    const double C84 = 29014219670751100192948224.0;  // 1.5 * 2^84: x + C84 is rounded to a multiple of 2^32
    const double I32 = 2.3283064365386962890625e-10;  // 2^-32
    const double th = (H + C84) - C84;
    const double hlo = H - th;
    const double l2 = f64_fma(th, -I32, L);
    const double tl = (l2 + C84) - C84;
    L = l2 - tl;
    H = f64_fma(tl, I32, f64_fma(th, I32, hlo));
#else
    // through the integer pipes: X + 1.5*2^52 (exact, |X| < 2^51) has the bit pattern hX : rX = 0x43380000 + qX : rX
    // with X = rX + 2^32*qX, 0 <= rX < 2^32, |qX| <= 2^17. With 2^64 = 2^32 - 1 the value is
    // (rL - qH) + 2^32*(rH + qL + qH). Both limbs are assembled as 2^52-offset bit patterns by a three-input add
    // and its carry (IADD3, IADD3.X and for H' a LOP3 that ORs in the exponent, on the ALU pipe, nearly idle here),
    // and one DADD each removes the offset: 4 FP64 and 5 ALU instructions instead of 9 FP64 ones,
    // -2^18 < L', H' < 2^32 + 2^18.
    const double tL = L + 6755399441055744.0, tH = H + 6755399441055744.0;  // + 1.5 * 2^52
    const uint32_t rL = f64_lo_word(tL), hL = f64_hi_word(tL), rH = f64_lo_word(tH), hH = f64_hi_word(tH);
    // 2^52 + 2^32 + rL - (qH + 2^19)  and  2^52 + rH + (qL + qH + 0x86700000)
    const uint64_t yl = (0x4330000143300000ULL + rL) - hH;
    const uint64_t yh = 0x4330000000000000ULL + rH + hL + hH;
    L = f64_from_bits(yl) - 4503603921813504.0;  // 2^52 + 2^32 - 2^19
    H = f64_from_bits(yh) - 4503601882857472.0;  // 2^52 + 0x86700000
#endif
}
GL_HD void poseidon_partial_rounds_f64(uint64_t s[12]) {
    const PoseidonTables& T = GL_POS;
    double L[12], H[12];
#pragma unroll
    for (int i = 1; i < 12; i++) {
        L[i] = u32_to_f64((uint32_t)s[i]);
        H[i] = u32_to_f64((uint32_t)(s[i] >> 32));
    }
    uint64_t s0 = s[0];
#pragma unroll 1
    for (int rp = 0; rp < 11; rp++) {
        sbox7_f64(s0, L[0], H[0]);  // x~0 = x0^7: signed low limb, |L[0]| < 2^33
        // a = (M x~)_0 + cA_0 (no bias in the limbs; the bias (bl, bh) = 0 (mod p) is added for the conversion only)
#if defined(GL_PAIR_RENORM_F64)
        double aL = T.pan_f64[rp][0], aH = T.pan_f64[rp][1];
#else
        double aL = T.pad_f64[rp][0], aH = T.pad_f64[rp][1];  // + (M d)_0: lanes 1..11 hold x - d
#endif
#pragma unroll
        for (int j = 0; j < 12; j++) {
            aL = f64_fma(L[j], (double)mds_entry(0, j), aL);
            aH = f64_fma(H[j], (double)mds_entry(0, j), aH);
        }
        double zL, zH;
        sbox7_f64(f64_pair_to_u64(aL + (1125899906842624.0 + 262144.0), aH + (1125899906842624.0 - 524288.0)), zL, zH);
#if defined(GL_PAIR_RENORM_F64)
        const double* k = T.pks_f64[rp];
        partial_pair_limbs(L, k, zL, aL);
        partial_pair_limbs(H, k + 12, zH, aH);
#else
        partial_pair_limbs(L, &T.pk0_f64[rp][0], zL, aL);
        partial_pair_limbs(H, &T.pk0_f64[rp][1], zH, aH);
#endif
        s0 = f64_pair_to_u64(L[0], H[0]);
        if (rp != 10) {
#pragma unroll
            for (int i = 1; i < 12; i++) partial_pair_renorm(L[i], H[i]);
        }
    }
    s[0] = s0;
#if !defined(GL_PAIR_RENORM_F64)
#pragma unroll
    for (int i = 1; i < 12; i++) {  // x = y + d[11], plus the conversion bias
        L[i] += T.pdf_f64[2 * (i - 1)];
        H[i] += T.pdf_f64[2 * (i - 1) + 1];
        GL_F64_TRACK(L[i]);
        GL_F64_TRACK(H[i]);
    }
#endif
#pragma unroll
    for (int i = 1; i < 12; i++) s[i] = f64_pair_to_u64(L[i], H[i]);
}
#endif  // GL_FP64_PATH

GL_HD void poseidon_partial_rounds(uint64_t s[12]) {
#pragma unroll
    for (int i = 0; i < 12; i++) s[i] = add_canonical(s[i], GL_POS.fast_first[i]);
    poseidon_partial_rounds_noconst(s);
}

// Poseidon::poseidon, poseidon.rs:766-777. One rolled loop over the 8 full rounds (a single copy of the
// round body in the instruction stream); every constant layer except the first of each half is folded into
// the preceding MDS. SYNC (device only): a CTA barrier per full round keeps all warps of the CTA in the same
// round body, which improves instruction-cache locality (+10 % in tools/microbench); all threads of the CTA
// must then call this the same number of times.
template <bool SYNC = false>
GL_HD void poseidon_permute_t(uint64_t s[12]) {
    const PoseidonTables& T = GL_POS;
#pragma unroll
    for (int i = 0; i < 12; i++) s[i] = add_canonical(s[i], T.rc[i]);
#pragma unroll 1
    for (int r = 0; r < 8; r++) {
        // constants that follow this round's MDS: next full round's, or the partial rounds' first layer,
        // or nothing (after the partial rounds the 5th full round's constants are added explicitly)
#if defined(GL_PARTIAL_F64)
        const uint64_t* nrc = (r < 3) ? &T.rc[12 * (r + 1)] : (r == 3) ? &T.rc[48]
                            : (r < 7) ? &T.rc[12 * (r + 23)] : T.zeros;
        (void)nrc;
        full_round_f64(s, T.nrcs_f64[r == 3 ? 8 : r]);
#else
        const uint64_t* nrc = (r < 3) ? &T.rc[12 * (r + 1)] : (r == 3) ? T.fast_first
                            : (r < 7) ? &T.rc[12 * (r + 23)] : T.zeros;
        full_round_fused(s, nrc, T.nrc_f64[r]);
#endif
#if defined(__CUDA_ARCH__)
        if (SYNC) __syncthreads();
#endif
        if (r == 3) {
#if defined(GL_PARTIAL_F64)
            poseidon_partial_rounds_f64(s);  // ends with the 5th full round's constant layer folded in
#else
            poseidon_partial_rounds_noconst(s);
#pragma unroll
            for (int i = 0; i < 12; i++) s[i] = add_canonical(s[i], T.rc[12 * 26 + i]);
#endif
        }
    }
}
GL_HD void poseidon_permute(uint64_t s[12]) { poseidon_permute_t<false>(s); }

// compress / two_to_one (hashing.rs:97-114): state = [l, r, 0,0,0,0]; one permutation; lanes 0..3.
template <bool SYNC = false>
GL_HD void two_to_one(const uint64_t l[4], const uint64_t r[4], uint64_t out[4]) {
    uint64_t s[12] = {l[0], l[1], l[2], l[3], r[0], r[1], r[2], r[3], 0, 0, 0, 0};
    poseidon_permute_t<SYNC>(s);
#pragma unroll
    for (int i = 0; i < 4; i++) out[i] = canon(s[i]);
}

// hash_or_noop over a strided leaf (config.rs:63-74 + hashing.rs:118-141, overwrite-mode sponge):
// element k of the leaf is in[k * stride].
template <bool NOOP_SHORT = true, bool SYNC = false>
GL_HD void hash_or_noop_strided(const uint64_t* in, size_t stride, uint32_t W, uint64_t out[4]) {
    if (NOOP_SHORT && W <= 4) {
#pragma unroll
        for (uint32_t i = 0; i < 4; i++) out[i] = (i < W) ? canon(in[i * stride]) : 0;
        return;
    }
    uint64_t s[12];
#pragma unroll
    for (int i = 0; i < 12; i++) s[i] = 0;
    for (uint32_t off = 0; off < W; off += 8) {
#pragma unroll
        for (uint32_t i = 0; i < 8; i++)
            if (off + i < W) s[i] = in[(size_t)(off + i) * stride];
        poseidon_permute_t<SYNC>(s);
    }
#pragma unroll
    for (int i = 0; i < 4; i++) out[i] = canon(s[i]);
}

// hash_or_noop of the leaf `prefix[0..4) || in[k * stride], k < W` (a later stage of a batch Merkle tree,
// batch_merkle_tree.rs:84-96: the previous stage's cap digest, then the row). W + 4 > 4 words: always hashed.
template <bool SYNC = false>
GL_HD void hash_prefixed_strided(const uint64_t* prefix, const uint64_t* in, size_t stride, uint32_t W,
                                 uint64_t out[4]) {
    uint64_t s[12];
#pragma unroll
    for (int i = 0; i < 4; i++) s[i] = prefix[i];
#pragma unroll
    for (uint32_t i = 0; i < 8; i++) s[4 + i] = (i < 4 && i < W) ? in[(size_t)i * stride] : 0;
    poseidon_permute_t<SYNC>(s);
    for (uint32_t off = 4; off < W; off += 8) {
#pragma unroll
        for (uint32_t i = 0; i < 8; i++)
            if (off + i < W) s[i] = in[(size_t)(off + i) * stride];
        poseidon_permute_t<SYNC>(s);
    }
#pragma unroll
    for (int i = 0; i < 4; i++) out[i] = canon(s[i]);
}

}  // namespace gl
