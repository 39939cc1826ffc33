// SASS-count lab: in-register radix-32 DIF variants. Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -cubin -o /tmp/dft_lab.cubin dft_lab.cu
#include "../../plonky2_b200/csrc/gl_field.cuh"
using namespace gl;
typedef uint64_t u64;

// ---- variant A: current primitives
template <int M>
__device__ __forceinline__ void dftA(u64* r) {
#pragma unroll
    for (int l = 0; l < M; l++) {
        const int half = 1 << (M - 1 - l);
#pragma unroll
        for (int b = 0; b < (1 << (M - 1)); b++) {
            const int j = b % half, blk = (b / half) * 2 * half;
            u64 u = r[blk + j], v = r[blk + j + half];
            r[blk + j] = add(u, v);
            r[blk + j + half] = mul_pow2(sub(u, v), (uint32_t)((96 / half) * j));
        }
    }
}
// ---- variant B: canonical in / canonical out
__device__ __forceinline__ u64 csub(u64 a, u64 b) {
    uint32_t r0, r1;
    asm("{\n\t.reg .u32 m;\n\t"
        "sub.cc.u32 %0, %2, %4;\n\tsubc.cc.u32 %1, %3, %5;\n\tsubc.u32 m, 0, 0;\n\t"
        "sub.cc.u32 %0, %0, m;\n\tsubc.u32 %1, %1, 0;\n\t}"
        : "=&r"(r0), "=&r"(r1) : "r"(lo32(a)), "r"(hi32(a)), "r"(lo32(b)), "r"(hi32(b)));
    return pack64(r0, r1);
}
__device__ __forceinline__ u64 cneg_p(u64 b) {  // p - b in (0, p]
    uint32_t r0, r1;
    asm("sub.cc.u32 %0, 1, %2;\n\tsubc.u32 %1, 0xffffffff, %3;" : "=r"(r0), "=r"(r1) : "r"(lo32(b)), "r"(hi32(b)));
    return pack64(r0, r1);
}
__device__ __forceinline__ u64 ccanon(u64 x) {
    uint32_t t0, t1, c;
    asm("add.cc.u32 %0, %3, 0xffffffff;\n\taddc.cc.u32 %1, %4, 0;\n\taddc.u32 %2, 0, 0;" : "=r"(t0), "=r"(t1), "=r"(c) : "r"(lo32(x)), "r"(hi32(x)));
    return c ? pack64(t0, t1) : x;
}
template <int M>
__device__ __forceinline__ void dftB(u64* r) {
#pragma unroll
    for (int l = 0; l < M; l++) {
        const int half = 1 << (M - 1 - l);
#pragma unroll
        for (int b = 0; b < (1 << (M - 1)); b++) {
            const int j = b % half, blk = (b / half) * 2 * half;
            u64 u = r[blk + j], v = r[blk + j + half];
            r[blk + j] = csub(u, cneg_p(v));
            u64 d = csub(u, v);
            const uint32_t k = (uint32_t)((96 / half) * j);
            r[blk + j + half] = k ? ccanon(mul_pow2(d, k)) : d;
        }
    }
}
template <int V>
__global__ void k_dft32(const u64* in, u64* out) {
    u64 r[32];
    const size_t t = blockIdx.x * blockDim.x + threadIdx.x;
#pragma unroll
    for (int i = 0; i < 32; i++) r[i] = in[t + (size_t)i * 4096];
    if (V == 0) dftA<5>(r);
    if (V == 1) dftB<5>(r);
#pragma unroll
    for (int i = 0; i < 32; i++) out[t + (size_t)i * 4096] = r[i];
}
template __global__ void k_dft32<0>(const u64*, u64*);
template __global__ void k_dft32<1>(const u64*, u64*);
// single ops for reference
__global__ void k_add(const u64* in, u64* out) { out[threadIdx.x] = add(in[threadIdx.x], in[threadIdx.x + 32]); }
__global__ void k_sub(const u64* in, u64* out) { out[threadIdx.x] = sub(in[threadIdx.x], in[threadIdx.x + 32]); }
__global__ void k_mul(const u64* in, u64* out) { out[threadIdx.x] = mul(in[threadIdx.x], in[threadIdx.x + 32]); }
__global__ void k_csub(const u64* in, u64* out) { out[threadIdx.x] = csub(in[threadIdx.x], in[threadIdx.x + 32]); }
__global__ void k_cadd(const u64* in, u64* out) { out[threadIdx.x] = csub(in[threadIdx.x], cneg_p(in[threadIdx.x + 32])); }
__global__ void k_canon(const u64* in, u64* out) { out[threadIdx.x] = ccanon(in[threadIdx.x]); }
template <int K> __global__ void k_shift(const u64* in, u64* out) { out[threadIdx.x] = mul_pow2(in[threadIdx.x], K); }
template __global__ void k_shift<12>(const u64*, u64*);
template __global__ void k_shift<36>(const u64*, u64*);
template __global__ void k_shift<48>(const u64*, u64*);
template __global__ void k_shift<72>(const u64*, u64*);
