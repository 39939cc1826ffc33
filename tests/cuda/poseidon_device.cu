// poseidon_device.cu -- runs the DEVICE Poseidon of gl_poseidon.cuh, built once per compile-time switch, on states and
// leaf matrices from a file and writes every output back, for tests/test_gpu_poseidon.py to check against the CPU
// oracle. The host only uploads the constant tables (host_poseidon_tables) and moves data.
//
//   poseidon_device IN OUT
// IN  (u64 words): NS NM, then
//     NS x 12                  states
//     per matrix: W N, then N x W words, leaf j = row j
// OUT (u64 words):
//     NS x 12                  poseidon_permute_t<false>(state), canonical (the k_permute_many / k_fri_pow / two_to_one body)
//     per matrix: N x 4        hash_or_noop_strided<true, true> on the column-major copy (element stride N) under
//                              __launch_bounds__(128, 4), the leaf hash's budget; the last CTA is partly dead when
//                              N % 128 != 0 and its dead threads hash leaf N - 1, as in k_leaf_hash
//                 N x 4        the same under __launch_bounds__(128, 5) (the GL_HASH_MINB=5 budget)
//                 N x 4        hash_or_noop_strided<false> on the rows (hash_no_pad)
//   built with -DPOSEIDON_TRACK, then per launch above, in the same order: one slot per launched thread holding the
//   largest |x| that thread passed to GL_F64_TRACK (an FP64 limb), as the bits of a double
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#if defined(POSEIDON_TRACK)
// per-thread running maximum of the FP64 limbs, one global slot per thread of the current launch (no atomics: a slot
// belongs to one thread)
__device__ double* g_track;
__host__ __device__ inline void track_limb(double x) {
#if defined(__CUDA_ARCH__)
    double* slot = g_track + ((size_t)blockIdx.x * blockDim.x + threadIdx.x);
    const double a = fabs(x);
    if (a > *slot) *slot = a;
#else
    (void)x;
#endif
}
#define GL_F64_TRACK(x) track_limb(x)
#endif

#include "gl_poseidon.cuh"

using namespace gl;
typedef unsigned long long u64;

#define CHECK(call)                                                                               \
    do {                                                                                          \
        cudaError_t e_ = (call);                                                                  \
        if (e_ != cudaSuccess) {                                                                  \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
            exit(2);                                                                              \
        }                                                                                         \
    } while (0)

constexpr int CTA = 128;

extern "C" __global__ void __launch_bounds__(CTA) k_permute(u64* st, size_t n) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    uint64_t s[12];
#pragma unroll
    for (int k = 0; k < 12; k++) s[k] = st[12 * j + k];
    poseidon_permute_t<false>(s);
#pragma unroll
    for (int k = 0; k < 12; k++) st[12 * j + k] = canon(s[k]);
}

// k_leaf_hash's body: every thread of the CTA runs the barrier-synchronised permutation
__device__ __forceinline__ void leaf_body(const u64* cols, size_t N, uint32_t W, u64* out) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = j < N;
    if (!live) j = N - 1;
    uint64_t h[4];
    hash_or_noop_strided<true, true>((const uint64_t*)cols + j, N, W, h);
    if (!live) return;
    for (int k = 0; k < 4; k++) out[4 * j + k] = h[k];
}
extern "C" __global__ void __launch_bounds__(CTA, 4) k_leaf_minb4(const u64* cols, size_t N, uint32_t W, u64* out) {
    leaf_body(cols, N, W, out);
}
extern "C" __global__ void __launch_bounds__(CTA, 5) k_leaf_minb5(const u64* cols, size_t N, uint32_t W, u64* out) {
    leaf_body(cols, N, W, out);
}

extern "C" __global__ void __launch_bounds__(CTA) k_no_pad(const u64* rows, size_t N, uint32_t W, u64* out) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= N) return;
    uint64_t h[4];
    hash_or_noop_strided<false>((const uint64_t*)rows + j * W, 1, W, h);
    for (int k = 0; k < 4; k++) out[4 * j + k] = h[k];
}

static u64* to_dev(const u64* h, size_t words) {
    u64* d;
    CHECK(cudaMalloc(&d, (words ? words : 1) * 8));
    if (h && words) CHECK(cudaMemcpy(d, h, words * 8, cudaMemcpyHostToDevice));
    return d;
}
static void append(std::vector<u64>& out, const u64* d, size_t words) {
    const size_t at = out.size();
    out.resize(at + words);
    if (words) CHECK(cudaMemcpy(out.data() + at, d, words * 8, cudaMemcpyDeviceToHost));
}
static unsigned grid(size_t n) { return (unsigned)((n + CTA - 1) / CTA); }

// the limb slots of one launch of `blocks` CTAs: zeroed before it, appended to `slots` after it
struct Track {
    std::vector<u64> slots;
    double* d = nullptr;
    size_t cap = 0, used = 0;
    void begin(unsigned blocks) {
#if defined(POSEIDON_TRACK)
        used = (size_t)blocks * CTA;
        if (used > cap) {
            if (d) CHECK(cudaFree(d));
            CHECK(cudaMalloc(&d, used * 8));
            cap = used;
            CHECK(cudaMemcpyToSymbol(g_track, &d, sizeof(d)));
        }
        CHECK(cudaMemset(d, 0, used * 8));
#else
        (void)blocks;
#endif
    }
    void end() {
#if defined(POSEIDON_TRACK)
        CHECK(cudaDeviceSynchronize());
        append(slots, (const u64*)d, used);
#endif
    }
};

int main(int argc, char** argv) {
    if (argc != 3) {
        fprintf(stderr, "usage: %s IN OUT\n", argv[0]);
        return 1;
    }
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 1;
    std::vector<u64> in;
    {
        u64 buf[4096];
        size_t got;
        while ((got = fread(buf, 8, 4096, f)) > 0) in.insert(in.end(), buf, buf + got);
    }
    fclose(f);
    if (in.size() < 2) return 1;
    const size_t ns = in[0], nm = in[1];
    size_t at = 2 + 12 * ns;
    if (in.size() < at) return 1;
    CHECK(cudaMemcpyToSymbol(c_pos, &host_poseidon_tables(), sizeof(PoseidonTables)));

    std::vector<u64> out;
    Track tr;
    {
        u64* d = to_dev(in.data() + 2, 12 * ns);
        tr.begin(grid(ns));
        if (ns) k_permute<<<grid(ns), CTA>>>(d, ns);
        CHECK(cudaGetLastError());
        tr.end();
        append(out, d, 12 * ns);
        CHECK(cudaFree(d));
    }
    for (size_t m = 0; m < nm; m++) {
        if (in.size() < at + 2) return 1;
        const uint32_t W = (uint32_t)in[at];
        const size_t N = in[at + 1];
        at += 2;
        if (N == 0 || W == 0 || in.size() < at + N * W) {
            fprintf(stderr, "matrix %zu: bad shape W=%u N=%zu\n", m, W, N);
            return 1;
        }
        const u64* rows = in.data() + at;
        at += N * W;
        std::vector<u64> cm(N * W);
        for (size_t j = 0; j < N; j++)
            for (uint32_t k = 0; k < W; k++) cm[(size_t)k * N + j] = rows[j * W + k];
        u64* d_cols = to_dev(cm.data(), N * W);
        u64* d_rows = to_dev(rows, N * W);
        u64* d_out = to_dev(nullptr, 4 * N);
        tr.begin(grid(N));
        k_leaf_minb4<<<grid(N), CTA>>>(d_cols, N, W, d_out);
        CHECK(cudaGetLastError());
        tr.end();
        append(out, d_out, 4 * N);
        CHECK(cudaMemset(d_out, 0, 4 * N * 8));
        tr.begin(grid(N));
        k_leaf_minb5<<<grid(N), CTA>>>(d_cols, N, W, d_out);
        CHECK(cudaGetLastError());
        tr.end();
        append(out, d_out, 4 * N);
        CHECK(cudaMemset(d_out, 0, 4 * N * 8));
        tr.begin(grid(N));
        k_no_pad<<<grid(N), CTA>>>(d_rows, N, W, d_out);
        CHECK(cudaGetLastError());
        tr.end();
        append(out, d_out, 4 * N);
        for (u64* d : {d_cols, d_rows, d_out}) CHECK(cudaFree(d));
    }
    if (at != in.size()) {
        fprintf(stderr, "input has %zu words, the header and shapes describe %zu\n", in.size(), at);
        return 1;
    }
    CHECK(cudaDeviceSynchronize());
    out.insert(out.end(), tr.slots.begin(), tr.slots.end());
    if (tr.d) CHECK(cudaFree(tr.d));

    FILE* g = fopen(argv[2], "wb");
    if (!g || fwrite(out.data(), 8, out.size(), g) != out.size()) return 1;
    fclose(g);
    printf("poseidon_device: %zu words written\n", out.size());
    return 0;
}
