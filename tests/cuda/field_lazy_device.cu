// field_lazy_device.cu -- runs the DEVICE formulations of gl_field.cuh and gl_lazy.cuh (PTX carry chains, lazy
// 3-word values) on operands from a file and writes every result back, for tests/test_gpu_field_lazy.py to check
// against plain integer arithmetic. The host never computes a field operation here: the reference is in Python.
//
//   field_lazy_device IN OUT
// IN  (u64 words): NP NPOW NL NN ND, then
//     NP x (a, b, c, d)        field operands
//     NPOW words               operands of mul_pow2 for every k in 0..95
//     NL x (w0, w1, e)         lazy values for l3_add / l3_sub (with the next entry) and l3_shift<S>, S in 0..95
//     NN x (w0, w1, e)         lazy values for l3_norm
//     ND x 32 words            DFT inputs: dft_lazy<M> runs on the first 2^M words, M = 1..5
// OUT (u64 words, e sign-extended):
//     NP x 11                  add sub neg mul sqr mul_add reduce96(a, lo32(b)) reduce128(a, b) canon(a) e2_mul(ab, cd)
//     NPOW x 96                mul_pow2(x, k)
//     NL x 6                   l3_add(v_i, v_i+1), l3_sub(v_i, v_i+1)
//     NL x 96 x 3              l3_shift<S>(v_i)
//     NN                       l3_norm(v_i)
//     per M = 1..5: ND x 2^M   l3_norm(dft_lazy<M>(x))[j]  (bit-reversed order), then ND x 1: max |e| before l3_norm
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#include "gl_lazy.cuh"

using namespace gl;
typedef unsigned long long u64;

#define CHECK(call)                                                                                 \
    do {                                                                                            \
        cudaError_t e_ = (call);                                                                    \
        if (e_ != cudaSuccess) {                                                                    \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #call, cudaGetErrorString(e_));   \
            exit(2);                                                                                \
        }                                                                                           \
    } while (0)

__device__ L3 load_l3(const u64* p) { return L3{(uint32_t)p[0], (uint32_t)p[1], (int32_t)(int64_t)p[2]}; }
__device__ void store_l3(u64* p, L3 v) {
    p[0] = v.w0;
    p[1] = v.w1;
    p[2] = (u64)(int64_t)v.e;
}

__global__ void k_field(const u64* in, size_t np, u64* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= np) return;
    const u64 a = in[4 * i], b = in[4 * i + 1], c = in[4 * i + 2], d = in[4 * i + 3];
    u64* o = out + 11 * i;
    o[0] = add(a, b);
    o[1] = sub(a, b);
    o[2] = neg(a);
    o[3] = mul(a, b);
    o[4] = sqr(a);
    o[5] = mul_add(a, b, c);
    o[6] = reduce96(a, (uint32_t)b);
    o[7] = reduce128(a, b);
    o[8] = canon(a);
    const E2 r = e2_mul(E2{a, b}, E2{c, d});
    o[9] = r.a;
    o[10] = r.b;
}

__global__ void k_pow2(const u64* in, size_t n, u64* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (uint32_t k = 0; k < 96; k++) out[96 * i + k] = mul_pow2(in[i], k);
}

template <int S>
__device__ void shift_all(L3 v, u64* o) {
    store_l3(o + 3 * S, l3_shift<S>(v));
    if constexpr (S + 1 < 96) shift_all<S + 1>(v, o);
}
__global__ void k_lazy(const u64* in, size_t nl, u64* out_addsub, u64* out_shift) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nl) return;
    const L3 a = load_l3(in + 3 * i), b = load_l3(in + 3 * ((i + 1) % nl));
    store_l3(out_addsub + 6 * i, l3_add(a, b));
    store_l3(out_addsub + 6 * i + 3, l3_sub(a, b));
    shift_all<0>(a, out_shift + 96 * 3 * i);
}

__global__ void k_norm(const u64* in, size_t nn, u64* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nn) out[i] = l3_norm(load_l3(in + 3 * i));
}

template <int M>
__global__ void k_dft(const u64* in, size_t nd, u64* out, u64* max_e) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nd) return;
    L3 r[1 << M];
    for (int j = 0; j < (1 << M); j++) r[j] = l3_from(in[32 * i + j]);
    dft_lazy<M>(r);
    u64 m = 0;
    for (int j = 0; j < (1 << M); j++) {
        const u64 e = (u64)(r[j].e < 0 ? -(int64_t)r[j].e : (int64_t)r[j].e);
        m = e > m ? e : m;
        out[(size_t)i * (1 << M) + j] = l3_norm(r[j]);
    }
    max_e[i] = m;
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
static unsigned grid(size_t n) { return (unsigned)((n + 127) / 128); }

template <int M>
static void run_dft(const u64* d_in, size_t nd, std::vector<u64>& out) {
    u64* d_out = to_dev(nullptr, nd << M);
    u64* d_e = to_dev(nullptr, nd);
    if (nd) k_dft<M><<<grid(nd), 128>>>(d_in, nd, d_out, d_e);
    CHECK(cudaGetLastError());
    append(out, d_out, nd << M);
    append(out, d_e, nd);
    CHECK(cudaFree(d_out));
    CHECK(cudaFree(d_e));
}

int main(int argc, char** argv) {
    if (argc != 3) {
        fprintf(stderr, "usage: %s IN OUT\n", argv[0]);
        return 1;
    }
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 1;
    std::vector<u64> in;
    u64 buf[4096];
    size_t got;
    while ((got = fread(buf, 8, 4096, f)) > 0) in.insert(in.end(), buf, buf + got);
    fclose(f);
    if (in.size() < 5) return 1;
    const size_t np = in[0], npow = in[1], nl = in[2], nn = in[3], nd = in[4];
    const size_t want = 5 + 4 * np + npow + 3 * nl + 3 * nn + 32 * nd;
    if (in.size() != want) {
        fprintf(stderr, "input has %zu words, header says %zu\n", in.size(), want);
        return 1;
    }
    const u64* p = in.data() + 5;
    u64* d_pairs = to_dev(p, 4 * np);
    p += 4 * np;
    u64* d_pow = to_dev(p, npow);
    p += npow;
    u64* d_lazy = to_dev(p, 3 * nl);
    p += 3 * nl;
    u64* d_norm = to_dev(p, 3 * nn);
    p += 3 * nn;
    u64* d_dft = to_dev(p, 32 * nd);

    std::vector<u64> out;
    u64* o_field = to_dev(nullptr, 11 * np);
    u64* o_pow = to_dev(nullptr, 96 * npow);
    u64* o_addsub = to_dev(nullptr, 6 * nl);
    u64* o_shift = to_dev(nullptr, 96 * 3 * nl);
    u64* o_norm = to_dev(nullptr, nn);
    if (np) k_field<<<grid(np), 128>>>(d_pairs, np, o_field);
    CHECK(cudaGetLastError());
    if (npow) k_pow2<<<grid(npow), 128>>>(d_pow, npow, o_pow);
    CHECK(cudaGetLastError());
    if (nl) k_lazy<<<grid(nl), 128>>>(d_lazy, nl, o_addsub, o_shift);
    CHECK(cudaGetLastError());
    if (nn) k_norm<<<grid(nn), 128>>>(d_norm, nn, o_norm);
    CHECK(cudaGetLastError());
    append(out, o_field, 11 * np);
    append(out, o_pow, 96 * npow);
    append(out, o_addsub, 6 * nl);
    append(out, o_shift, 96 * 3 * nl);
    append(out, o_norm, nn);
    run_dft<1>(d_dft, nd, out);
    run_dft<2>(d_dft, nd, out);
    run_dft<3>(d_dft, nd, out);
    run_dft<4>(d_dft, nd, out);
    run_dft<5>(d_dft, nd, out);
    CHECK(cudaDeviceSynchronize());
    for (u64* d : {d_pairs, d_pow, d_lazy, d_norm, d_dft, o_field, o_pow, o_addsub, o_shift, o_norm}) CHECK(cudaFree(d));

    FILE* g = fopen(argv[2], "wb");
    if (!g || fwrite(out.data(), 8, out.size(), g) != out.size()) return 1;
    fclose(g);
    printf("field_lazy_device: %zu words written\n", out.size());
    return 0;
}
