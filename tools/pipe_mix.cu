// Which H100 pipes share an issue port? Times pure and interleaved streams of DFMA (FP64), IMAD / IMAD.WIDE
// (FMA-heavy), LOP3 (ALU), IMAD.HI and I2F.F64 (XU), each with 8 independent chains per thread. If two classes share a port the
// mixed stream takes the SUM of the pure times, otherwise about the MAX. Output feeds the cost model in DESIGN.md.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/pipe_mix tools/pipe_mix.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
constexpr int ILP = 8, ITERS = 2048;
template <int D, int I, int W, int A, int X, int HI = 0>
__global__ void k_mix(uint64_t* out, double dx, uint32_t ix) {
    double d[ILP];
    uint32_t a[ILP], m[ILP], xs[ILP], hs[ILP];
    uint64_t w[ILP];
    for (int i = 0; i < ILP; i++) {
        d[i] = threadIdx.x + i; a[i] = threadIdx.x * 3 + i; m[i] = threadIdx.x + 7 * i; w[i] = threadIdx.x + i; xs[i] = threadIdx.x + i; hs[i] = 0x9E3779B9u * (threadIdx.x + i + 1);
    }
    double acc = 0;
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) {
            if (D) asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[i]) : "d"(dx), "d"(1.0));
            if (I) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(m[i]) : "r"(ix), "r"(i + 1));
            if (HI) asm volatile("mad.hi.u32 %0, %0, %1, %2;" : "+r"(hs[i]) : "r"(ix * 0x85EBCA6Bu), "r"(i + 7));
            if (W) asm volatile("{\n\t.reg .u32 t;\n\tcvt.u32.u64 t, %0;\n\tmad.wide.u32 %0, t, %1, %0;\n\t}" : "+l"(w[i]) : "r"(ix));
            if (A) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(ix), "r"(i + 5));
            if (X) asm volatile("{\n\t.reg .f64 t;\n\t.reg .u32 h;\n\tcvt.rn.f64.u32 t, %0;\n\tmov.b64 {%0, h}, t;\n\t}" : "+r"(xs[i]));
        }
    }
    uint64_t s = 0;
    for (int i = 0; i < ILP; i++) s += (uint64_t)d[i] + a[i] + m[i] + w[i] + xs[i] + hs[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s + (uint64_t)acc;
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
    printf("%s, %d SMs, %d MHz. Columns: stream, ms, cycles per warp-instruction-group per SMSP (one instr of each class in the stream)\n", prop.name, sms, clk_khz / 1000);
    auto rep = [&](const char* name, float ms) {
        // cycles per (one instruction of each class) per SMSP: ms*clk / (warp-instr groups per SMSP)
        double groups_per_smsp = per_class / 32.0 / (sms * 4.0);
        printf("%-28s %8.3f ms  %6.2f cycles/group/SMSP\n", name, ms, ms * 1e-3 * clk_khz * 1e3 / groups_per_smsp);
    };
#define RUN(D, I, W, A, X, name) rep(name, timeit([&] { k_mix<D, I, W, A, X><<<blocks, threads>>>(out, 1.0000001, 3); }))
    RUN(1, 0, 0, 0, 0, "DFMA");
    RUN(0, 1, 0, 0, 0, "IMAD");
    RUN(0, 0, 1, 0, 0, "IMAD.WIDE");
    RUN(0, 0, 0, 1, 0, "LOP3");
    RUN(0, 0, 0, 0, 1, "I2F.F64");
    RUN(1, 1, 0, 0, 0, "DFMA+IMAD");
    RUN(1, 0, 1, 0, 0, "DFMA+IMAD.WIDE");
    RUN(1, 0, 0, 1, 0, "DFMA+LOP3");
    RUN(0, 1, 0, 1, 0, "IMAD+LOP3");
    RUN(0, 0, 1, 1, 0, "IMAD.WIDE+LOP3");
    RUN(1, 1, 0, 1, 0, "DFMA+IMAD+LOP3");
    RUN(1, 0, 0, 0, 1, "DFMA+I2F");
    RUN(0, 1, 0, 0, 1, "IMAD+I2F");
    RUN(1, 1, 1, 1, 1, "all five");
#define RUNH(D, I, W, A, X, name) rep(name, timeit([&] { k_mix<D, I, W, A, X, 1><<<blocks, threads>>>(out, 1.0000001, 3); }))
    RUNH(0, 0, 0, 0, 0, "IMAD.HI");
    RUNH(0, 1, 0, 0, 0, "IMAD.HI+IMAD");
    RUNH(0, 0, 0, 1, 0, "IMAD.HI+LOP3");
    RUNH(1, 0, 0, 0, 0, "IMAD.HI+DFMA");
    return 0;
}
