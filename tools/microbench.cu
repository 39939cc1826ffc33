// Integer-pipe microbenchmarks for H100 (what bounds Goldilocks arithmetic): issue rates of
// IMAD.WIDE.U32, 32-bit IMAD, IADD3 / carry chains, and the library's own modmul / modadd / Poseidon.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o /tmp/microbench tools/microbench.cu
#include <cstdio>
#include <cuda_runtime.h>
#include "../plonky2_b200/csrc/gl_poseidon.cuh"
using namespace gl;

constexpr int ILP = 8, ITERS = 4096;

__global__ void k_imad_wide(uint64_t* out, uint32_t a, uint32_t b) {
    uint64_t acc[ILP];
    for (int i = 0; i < ILP; i++) acc[i] = threadIdx.x + i;
    uint32_t x = a + threadIdx.x, y = b;
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) acc[i] = (uint64_t)x * (uint32_t)(y + i) + acc[i];
        x ^= (uint32_t)acc[0];
    }
    uint64_t s = 0;
    for (int i = 0; i < ILP; i++) s += acc[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void k_imad32(uint64_t* out, uint32_t a, uint32_t b) {
    uint32_t acc[ILP];
    for (int i = 0; i < ILP; i++) acc[i] = threadIdx.x + i;
    uint32_t x = a + threadIdx.x;
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) acc[i] = acc[i] * x + (b + i);
        x += acc[0];
    }
    uint32_t s = 0;
    for (int i = 0; i < ILP; i++) s += acc[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void k_add64(uint64_t* out, uint64_t a) {
    uint64_t acc[ILP];
    for (int i = 0; i < ILP; i++) acc[i] = threadIdx.x + i;
    uint64_t x = a + threadIdx.x;
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) acc[i] = acc[i] + (x ^ acc[(i + 1) % ILP]);
    }
    uint64_t s = 0;
    for (int i = 0; i < ILP; i++) s += acc[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void k_dfma(uint64_t* out, double a) {
    double acc[ILP];
    for (int i = 0; i < ILP; i++) acc[i] = threadIdx.x + i;
    double x = a + threadIdx.x;
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) acc[i] = fma(acc[i], x, 1.0 + i);
    }
    double s = 0;
    for (int i = 0; i < ILP; i++) s += acc[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = (uint64_t)s;
}
__global__ void k_modmul(uint64_t* out, uint64_t a) {
    uint64_t acc[ILP];
    for (int i = 0; i < ILP; i++) acc[i] = a * (threadIdx.x + i + 1);
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) acc[i] = mul(acc[i], acc[(i + 1) % ILP]);
    }
    uint64_t s = 0;
    for (int i = 0; i < ILP; i++) s += acc[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void k_modsqr(uint64_t* out, uint64_t a) {
    uint64_t acc[ILP];
    for (int i = 0; i < ILP; i++) acc[i] = a * (threadIdx.x + i + 1);
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) acc[i] = sqr(acc[i]);
    }
    uint64_t s = 0;
    for (int i = 0; i < ILP; i++) s += acc[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void k_modadd(uint64_t* out, uint64_t a) {
    uint64_t acc[ILP];
    for (int i = 0; i < ILP; i++) acc[i] = a * (threadIdx.x + i + 1);
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) acc[i] = add(acc[i], acc[(i + 1) % ILP]);
    }
    uint64_t s = 0;
    for (int i = 0; i < ILP; i++) s += acc[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void k_mulpow2(uint64_t* out, uint64_t a) {
    uint64_t acc[ILP];
    for (int i = 0; i < ILP; i++) acc[i] = a * (threadIdx.x + i + 1);
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) acc[i] = mul_pow2(acc[i], 12 * (i % 7) + 12);
    }
    uint64_t s = 0;
    for (int i = 0; i < ILP; i++) s += acc[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void __launch_bounds__(128) k_poseidon(uint64_t* out, uint64_t a, int reps) {
    uint64_t s[12];
    for (int i = 0; i < 12; i++) s[i] = a * (threadIdx.x + blockIdx.x * 131 + i + 1);
    for (int r = 0; r < reps; r++) poseidon_permute(s);
    out[blockIdx.x * blockDim.x + threadIdx.x] = s[0];
}
// variant: big CTA, all warps kept in the same round by a barrier (instruction-cache locality)
template <int THREADS>
__global__ void __launch_bounds__(THREADS) k_poseidon_sync(uint64_t* out, uint64_t a, int reps) {
    uint64_t s[12];
    for (int i = 0; i < 12; i++) s[i] = a * (threadIdx.x + blockIdx.x * 131 + i + 1);
    for (int r = 0; r < reps; r++) poseidon_permute_t<true>(s);
    out[blockIdx.x * blockDim.x + threadIdx.x] = s[0];
}
template <int THREADS, int MINB>
__global__ void __launch_bounds__(THREADS, MINB) k_poseidon_sync_occ(uint64_t* out, uint64_t a, int reps) {
    uint64_t s[12];
    for (int i = 0; i < 12; i++) s[i] = a * (threadIdx.x + blockIdx.x * 131 + i + 1);
    for (int r = 0; r < reps; r++) poseidon_permute_t<true>(s);
    out[blockIdx.x * blockDim.x + threadIdx.x] = s[0];
}
// two independent permutations per thread, interleaved round by round (more ILP, pipe diversity inside a warp)
GL_D void poseidon_permute_x2(uint64_t a[12], uint64_t b[12]) {
    const PoseidonTables& T = c_pos;
#pragma unroll
    for (int i = 0; i < 12; i++) { a[i] = add_canonical(a[i], T.rc[i]); b[i] = add_canonical(b[i], T.rc[i]); }
#pragma unroll 1
    for (int r = 0; r < 8; r++) {
        const uint64_t* nrc = (r < 3) ? &T.rc[12 * (r + 1)] : (r == 3) ? T.fast_first : (r < 7) ? &T.rc[12 * (r + 23)] : T.zeros;
#pragma unroll
        for (int i = 0; i < 12; i++) { a[i] = sbox7(a[i]); b[i] = sbox7(b[i]); }
        mds_layer_add(a, nrc);
        mds_layer_add(b, nrc);
        __syncthreads();
        if (r == 3) {
            poseidon_partial_rounds_noconst(a);
            poseidon_partial_rounds_noconst(b);
#pragma unroll
            for (int i = 0; i < 12; i++) { a[i] = add_canonical(a[i], T.rc[12 * 26 + i]); b[i] = add_canonical(b[i], T.rc[12 * 26 + i]); }
        }
    }
}
template <int THREADS, int MINB>
__global__ void __launch_bounds__(THREADS, MINB) k_poseidon_x2(uint64_t* out, uint64_t a0, int reps) {
    uint64_t a[12], b[12];
    for (int i = 0; i < 12; i++) { a[i] = a0 * (threadIdx.x + blockIdx.x * 131 + i + 1); b[i] = a[i] ^ 0x5555; }
    for (int r = 0; r < reps; r++) poseidon_permute_x2(a, b);
    out[blockIdx.x * blockDim.x + threadIdx.x] = a[0] ^ b[0];
}
template <int THREADS>
__global__ void __launch_bounds__(THREADS) k_poseidon_plain(uint64_t* out, uint64_t a, int reps) {
    uint64_t s[12];
    for (int i = 0; i < 12; i++) s[i] = a * (threadIdx.x + blockIdx.x * 131 + i + 1);
    for (int r = 0; r < reps; r++) poseidon_permute(s);
    out[blockIdx.x * blockDim.x + threadIdx.x] = s[0];
}
__global__ void __launch_bounds__(128) k_partial(uint64_t* out, uint64_t a, int reps) {
    uint64_t s[12];
    for (int i = 0; i < 12; i++) s[i] = a * (threadIdx.x + blockIdx.x * 131 + i + 1);
    for (int r = 0; r < reps; r++) poseidon_partial_rounds(s);
    out[blockIdx.x * blockDim.x + threadIdx.x] = s[0];
}
__global__ void __launch_bounds__(128) k_fullround(uint64_t* out, uint64_t a, int reps) {
    uint64_t s[12];
    for (int i = 0; i < 12; i++) s[i] = a * (threadIdx.x + blockIdx.x * 131 + i + 1);
    for (int r = 0; r < reps; r++) full_round(s, &c_pos.rc[12 * (r & 3)]);
    out[blockIdx.x * blockDim.x + threadIdx.x] = s[0];
}
__global__ void __launch_bounds__(128) k_mds(uint64_t* out, uint64_t a, int reps) {
    uint64_t s[12];
    for (int i = 0; i < 12; i++) s[i] = a * (threadIdx.x + blockIdx.x * 131 + i + 1);
    for (int r = 0; r < reps; r++) mds_layer(s);
    out[blockIdx.x * blockDim.x + threadIdx.x] = s[0];
}

template <class F>
static double timeit(F f) {
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    f();
    cudaDeviceSynchronize();
    cudaEventRecord(a);
    f();
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    return ms;
}
int main() {
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    int sms = prop.multiProcessorCount;
    int clk_khz = 0;
    cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
    const PoseidonTables& t = host_poseidon_tables();
    cudaMemcpyToSymbol(c_pos, &t, sizeof(PoseidonTables));
    uint64_t* out;
    const int blocks = sms * 16, threads = 256;
    cudaMalloc(&out, (size_t)blocks * threads * 8);
    printf("device %s, %d SMs, max clock %d MHz\n", prop.name, sms, clk_khz / 1000);
    const double nops = (double)blocks * threads * ITERS * ILP;
    auto rep = [&](const char* name, double ms, double ops) {
        printf("%-26s %8.3f ms  %8.2f Gop/s  %6.2f op/clk/SM @max-clock\n", name, ms, ops / ms / 1e6,
               ops / (ms * 1e-3) / sms / (clk_khz * 1e3));
    };
    rep("IMAD.WIDE.U32 (64b acc)", timeit([&] { k_imad_wide<<<blocks, threads>>>(out, 3, 5); }), nops);
    rep("IMAD 32-bit", timeit([&] { k_imad32<<<blocks, threads>>>(out, 3, 5); }), nops);
    rep("add64 (+xor)", timeit([&] { k_add64<<<blocks, threads>>>(out, 3); }), nops);
    rep("DFMA (fp64 pipe)", timeit([&] { k_dfma<<<blocks, threads>>>(out, 1.0000001); }), nops);
    rep("gl::mul", timeit([&] { k_modmul<<<blocks, threads>>>(out, 3); }), nops);
    rep("gl::sqr", timeit([&] { k_modsqr<<<blocks, threads>>>(out, 3); }), nops);
    rep("gl::add", timeit([&] { k_modadd<<<blocks, threads>>>(out, 3); }), nops);
    rep("gl::mul_pow2 (const k)", timeit([&] { k_mulpow2<<<blocks, threads>>>(out, 3); }), nops);
    const int reps = 64, pb = sms * 32, pt = 128;
    double perms = (double)pb * pt * reps;
    double ms = timeit([&] { k_poseidon<<<pb, pt>>>(out, 3, reps); });
    printf("%-26s %8.3f ms  %8.2f Mperm/s\n", "poseidon_permute", ms, perms / ms / 1e3);
    ms = timeit([&] { k_partial<<<pb, pt>>>(out, 3, reps); });
    printf("%-26s %8.3f ms  %8.2f M partial-blocks/s\n", "partial rounds (22+init)", ms, perms / ms / 1e3);
    ms = timeit([&] { k_poseidon_plain<256><<<pb / 2, 256>>>(out, 3, reps); });
    printf("%-26s %8.3f ms  %8.2f Mperm/s\n", "poseidon plain CTA=256", ms, perms / ms / 1e3);
    ms = timeit([&] { k_poseidon_plain<512><<<pb / 4, 512>>>(out, 3, reps); });
    printf("%-26s %8.3f ms  %8.2f Mperm/s\n", "poseidon plain CTA=512", ms, perms / ms / 1e3);
    ms = timeit([&] { k_poseidon_sync<256><<<pb / 2, 256>>>(out, 3, reps); });
    printf("%-26s %8.3f ms  %8.2f Mperm/s\n", "poseidon sync CTA=256", ms, perms / ms / 1e3);
    ms = timeit([&] { k_poseidon_sync<512><<<pb / 4, 512>>>(out, 3, reps); });
    printf("%-26s %8.3f ms  %8.2f Mperm/s\n", "poseidon sync CTA=512", ms, perms / ms / 1e3);
    ms = timeit([&] { k_poseidon_sync<768><<<pb / 6, 768>>>(out, 3, reps); });
    printf("%-26s %8.3f ms  %8.2f Mperm/s\n", "poseidon sync CTA=768", ms, perms * (pb / 6 * 6) / pb / ms / 1e3);
    ms = timeit([&] { k_poseidon_sync_occ<256, 4><<<pb / 2, 256>>>(out, 3, reps); });
    printf("%-26s %8.3f ms  %8.2f Mperm/s\n", "sync CTA=256 minb=4 (64r)", ms, perms / ms / 1e3);
    ms = timeit([&] { k_poseidon_sync_occ<512, 2><<<pb / 4, 512>>>(out, 3, reps); });
    printf("%-26s %8.3f ms  %8.2f Mperm/s\n", "sync CTA=512 minb=2 (64r)", ms, perms / ms / 1e3);
    ms = timeit([&] { k_poseidon_sync_occ<256, 3><<<pb / 2, 256>>>(out, 3, reps); });
    printf("%-26s %8.3f ms  %8.2f Mperm/s\n", "sync CTA=256 minb=3 (80r)", ms, perms / ms / 1e3);
    ms = timeit([&] { k_poseidon_sync_occ<128, 5><<<pb, 128>>>(out, 3, reps); });
    printf("%-26s %8.3f ms  %8.2f Mperm/s\n", "sync CTA=128 minb=5 (96r)", ms, perms / ms / 1e3);
    ms = timeit([&] { k_poseidon_x2<128, 3><<<pb / 2, 128>>>(out, 3, reps); });
    printf("%-26s %8.3f ms  %8.2f Mperm/s\n", "x2 CTA=128 minb=3", ms, perms / ms / 1e3);
    ms = timeit([&] { k_poseidon_x2<128, 2><<<pb / 2, 128>>>(out, 3, reps); });
    printf("%-26s %8.3f ms  %8.2f Mperm/s\n", "x2 CTA=128 minb=2", ms, perms / ms / 1e3);
    ms = timeit([&] { k_poseidon_x2<64, 4><<<pb, 64>>>(out, 3, reps); });
    printf("%-26s %8.3f ms  %8.2f Mperm/s\n", "x2 CTA=64 minb=4", ms, perms / ms / 1e3);
    ms = timeit([&] { k_fullround<<<pb, pt>>>(out, 3, reps * 8); });
    printf("%-26s %8.3f ms  %8.2f M full-rounds/s (x8 per perm => %.2f Mperm/s if only full rounds)\n", "full_round", ms,
           perms * 8 / ms / 1e3, perms / ms / 1e3);
    ms = timeit([&] { k_mds<<<pb, pt>>>(out, 3, reps * 8); });
    printf("%-26s %8.3f ms  %8.2f M mds/s\n", "mds_layer", ms, perms * 8 / ms / 1e3);
    return 0;
}
