// Round-2 follow-up to pipe_mix.cu: issue cost of the instruction classes the NTT / Poseidon rewrites lean on
// (IMAD.HI, IMAD.WIDE without addend, funnel shifts, carry chains, PRMT, SHFL, LDS) alone and mixed.
// Also: the 64x64->128 product as ptxas builds it from unsigned __int128 (IMAD.WIDE.U32 + IMAD.WIDE.U32.X, with the
// moves and carry materialisation it brings), mixed at the full-round body's ratios with IADD3, DFMA and I2F;
// mul.lo.u32 + mul.hi.u32 of the same operands (ptxas may fuse them back into one IMAD.WIDE: check the SASS); and
// LDC.64 from a __constant__ table at a loop-variant index, the form the rolled round loops load constants in.
// Each stream has ILP independent chains per thread; 16 warps per SMSP hide latency, so the numbers are
// issue/pipe throughput: cycles per warp-instruction per SMSP.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/pipe_mix2 tools/pipe_mix2.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
constexpr int ILP = 8, ITERS = 2048;

enum { S_HI = 1, S_MULHI = 2, S_WIDE_ACC = 4, S_WIDE_NOACC = 8, S_SHF = 16, S_CARRY = 32, S_PRMT = 64, S_SHFL = 128,
       S_LO = 256, S_LOP = 512, S_DFMA = 1024, S_LDS = 2048, S_IADD3 = 4096, S_SEL = 8192, S_MUL128 = 16384,
       S_LOHI = 32768, S_LDC = 65536, S_I2F = 131072 };
__constant__ double c_tab[64];

template <int M>
__global__ void k_mix(uint64_t* out, uint32_t ix, double dx) {
    __shared__ uint64_t sh[256 * 2];
    uint32_t a[ILP], b[ILP], c[ILP], h[ILP];
    uint64_t w[ILP];
    double d[ILP];
    for (int i = 0; i < ILP; i++) {
        a[i] = threadIdx.x * 3 + i; b[i] = threadIdx.x + 7 * i; c[i] = 0x9E3779B9u * (threadIdx.x + i + 1);
        h[i] = c[i] ^ 0x1234567u; w[i] = threadIdx.x + i; d[i] = threadIdx.x + i;
    }
    sh[threadIdx.x] = threadIdx.x; sh[threadIdx.x + 256] = 1;
    __syncthreads();
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) {
            if (M & S_HI) asm volatile("mad.hi.u32 %0, %0, %1, %2;" : "+r"(h[i]) : "r"(ix * 0x85EBCA6Bu), "r"(i + 7));
            if (M & S_MULHI) asm volatile("mul.hi.u32 %0, %0, %1;" : "+r"(h[i]) : "r"(ix * 0x85EBCA6Bu + 0xF0000000u));
            if (M & S_WIDE_ACC) asm volatile("{\n\t.reg .u32 t;\n\tcvt.u32.u64 t, %0;\n\tmad.wide.u32 %0, t, %1, %0;\n\t}" : "+l"(w[i]) : "r"(ix));
            if (M & S_WIDE_NOACC) asm volatile("{\n\t.reg .u32 t, u;\n\tmov.b64 {t, u}, %0;\n\txor.b32 t, t, u;\n\tmul.wide.u32 %0, t, %1;\n\t}" : "+l"(w[i]) : "r"(ix * 0x85EBCA6Bu + 0xF0000001u));
            if (M & S_SHF) asm volatile("shf.l.wrap.b32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b[i]), "r"(ix + 5));
            if (M & S_CARRY) asm volatile("add.cc.u32 %0, %0, %2;\n\taddc.u32 %1, %1, %3;" : "+r"(a[i]), "+r"(b[i]) : "r"(ix), "r"(ix + 1));
            if (M & S_PRMT) asm volatile("prmt.b32 %0, %0, %1, 0x2103;" : "+r"(c[i]) : "r"(ix));
            if (M & S_SHFL) asm volatile("shfl.sync.bfly.b32 %0, %0, 1, 0x1f, 0xffffffff;" : "+r"(c[i]));
            if (M & S_LO) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(b[i]) : "r"(ix), "r"(i + 1));
            if (M & S_LOP) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(ix), "r"(i + 5));
            if (M & S_DFMA) asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[i]) : "d"(dx), "d"(1.0));
            if (M & S_LDS) { uint32_t idx = (c[i] & 255u); uint64_t v; asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"((uint32_t)__cvta_generic_to_shared(&sh[idx]))); c[i] = (uint32_t)v + (uint32_t)(v >> 32); }
            if (M & S_IADD3) asm volatile("{\n\t.reg .u32 t;\n\tadd.u32 t, %0, %1;\n\tadd.u32 %0, t, %2;\n\t}" : "+r"(a[i]) : "r"(ix), "r"(b[i]));
            if (M & S_MUL128) {
                const unsigned __int128 q = (unsigned __int128)w[i] * (w[i] ^ ((uint64_t)ix << 32 | 0x9E3779B9u));
                w[i] = (uint64_t)q ^ (uint64_t)(q >> 64);
            }
            if (M & S_LOHI) asm volatile("{\n\t.reg .u32 t, u;\n\tmul.lo.u32 t, %0, %1;\n\tmul.hi.u32 u, %0, %1;\n\txor.b32 %0, t, u;\n\t}" : "+r"(h[i]) : "r"(ix * 0x85EBCA6Bu + 0xF0000001u));
            if (M & S_LDC) d[i] += c_tab[(it + i) & 63];
            if (M & S_I2F) d[i] += (double)(b[i] += ix);
            if (M & S_SEL) asm volatile("{\n\t.reg .pred p;\n\tsetp.lt.u32 p, %0, %1;\n\tselp.u32 %0, %2, %0, p;\n\t}" : "+r"(a[i]) : "r"(ix + 77), "r"(b[i]));
        }
    }
    uint64_t s = 0;
    for (int i = 0; i < ILP; i++) s += (uint64_t)d[i] + a[i] + b[i] + c[i] + h[i] + w[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <typename F>
static float timeit(F f) {
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    f(); cudaDeviceSynchronize();
    float best = 1e30f;
    for (int r = 0; r < 3; r++) { cudaEventRecord(e0); f(); cudaEventRecord(e1); cudaEventSynchronize(e1); float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms; }
    return best;
}
int main() {
    cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
    int clk_khz = 0; cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
    const int sms = prop.multiProcessorCount, blocks = sms * 8, threads = 256;
    uint64_t* out; cudaMalloc(&out, (size_t)blocks * threads * 8);
    const double per_class = (double)blocks * threads * ITERS * ILP;
    printf("%s, %d SMs, %d MHz. cycles per group per SMSP (a group = one PTX statement of each class in the stream)\n", prop.name, sms, clk_khz / 1000);
    auto rep = [&](const char* name, float ms) {
        double groups_per_smsp = per_class / 32.0 / (sms * 4.0);
        printf("%-36s %8.3f ms  %6.2f cycles/group/SMSP\n", name, ms, ms * 1e-3 * clk_khz * 1e3 / groups_per_smsp);
    };
#define RUN(M, name) rep(name, timeit([&] { k_mix<(M)><<<blocks, threads>>>(out, 3, 1.0000001); }))
    RUN(S_HI, "IMAD.HI (mad.hi.u32)");
    RUN(S_MULHI, "mul.hi.u32");
    RUN(S_LO, "IMAD (mad.lo.u32)");
    RUN(S_WIDE_ACC, "IMAD.WIDE acc");
    RUN(S_WIDE_NOACC, "xor + IMAD.WIDE no acc");
    RUN(S_LOP, "LOP3");
    RUN(S_SHF, "SHF");
    RUN(S_CARRY, "add.cc + addc (2 instr)");
    RUN(S_IADD3, "add + add (IADD3?)");
    RUN(S_SEL, "setp + selp (2 instr)");
    RUN(S_PRMT, "PRMT");
    RUN(S_SHFL, "SHFL.BFLY");
    RUN(S_LDS, "LDS.64 + 2 int");
    RUN(S_HI | S_LO, "IMAD.HI + IMAD");
    RUN(S_HI | S_LOP, "IMAD.HI + LOP3");
    RUN(S_HI | S_DFMA, "IMAD.HI + DFMA");
    RUN(S_HI | S_LO | S_LOP, "IMAD.HI + IMAD + LOP3");
    RUN(S_HI | S_WIDE_ACC, "IMAD.HI + IMAD.WIDE");
    RUN(S_SHF | S_LOP, "SHF + LOP3");
    RUN(S_SHF | S_LO, "SHF + IMAD");
    RUN(S_CARRY | S_LO, "carry pair + IMAD");
    RUN(S_CARRY | S_DFMA, "carry pair + DFMA");
    RUN(S_SHFL | S_LOP, "SHFL + LOP3");
    RUN(S_SHFL | S_LO | S_LOP, "SHFL + IMAD + LOP3");
    RUN(S_LDS | S_LO, "LDS.64 + 2 int + IMAD");
    RUN(S_LOP | S_LO | S_DFMA | S_SHF, "LOP3 + IMAD + DFMA + SHF");
    // one group of these = one 128-bit product (4 IMAD.WIDE) plus its companions; the full-round body has per
    // product about 2.4 IADD3, 0.6 IMAD.MOV, 1.2 DFMA, 0.4 I2F, 0.13 LDC.64
    RUN(S_MUL128, "128-bit product (u128)");
    RUN(S_LOHI, "mul.lo + mul.hi same operands");
    RUN(S_LDC, "LDC.64 (loop-variant index) + DADD");
    RUN(S_I2F, "IADD + I2F.F64.U32 + DADD");
    RUN(S_MUL128 | S_IADD3, "128-bit product + 2 IADD3");
    RUN(S_MUL128 | S_IADD3 | S_DFMA, "128-bit product + 2 IADD3 + DFMA");
    RUN(S_MUL128 | S_IADD3 | S_DFMA | S_I2F, "128-bit + 2 IADD3 + DFMA + I2F");
    RUN(S_MUL128 | S_LDC, "128-bit product + LDC.64");
    RUN(S_WIDE_ACC | S_IADD3 | S_DFMA, "IMAD.WIDE acc + 2 IADD3 + DFMA");
    return 0;
}
