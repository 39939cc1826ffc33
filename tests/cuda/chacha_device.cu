// chacha_device.cu -- runs the device salt sampler of gl_chacha.cuh (k_chacha_elements) as built with this binary's
// GL_CHACHA_BOUND, so that tests/test_zk_commit_and_prove.py can check a build with a lowered acceptance bound on the device.
//
//   chacha_device KEYHEX COLUMN FIRST COUNT OUT      writes COUNT u64 words (elements (COLUMN, FIRST ..)) to OUT
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#include "gl_chacha.cuh"

using namespace gl;

#define CHECK(call)                                                                                 \
    do {                                                                                            \
        cudaError_t e_ = (call);                                                                    \
        if (e_ != cudaSuccess) {                                                                    \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #call, cudaGetErrorString(e_));   \
            exit(2);                                                                                \
        }                                                                                           \
    } while (0)

int main(int argc, char** argv) {
    if (argc != 6) {
        fprintf(stderr, "usage: %s KEYHEX COLUMN FIRST COUNT OUT\n", argv[0]);
        return 1;
    }
    uint8_t key[32];
    for (int j = 0; j < 32; j++) {
        unsigned v;
        if (sscanf(argv[1] + 2 * j, "%2x", &v) != 1) return 1;
        key[j] = (uint8_t)v;
    }
    const uint32_t column = (uint32_t)strtoul(argv[2], nullptr, 0);
    const uint64_t first = strtoull(argv[3], nullptr, 0), count = strtoull(argv[4], nullptr, 0);
    uint64_t* d;
    CHECK(cudaMalloc(&d, count * 8));
    const uint64_t blocks = ((first + count - 1) >> 3) - (first >> 3) + 1;
    k_chacha_elements<<<(unsigned)((blocks + 255) / 256), 256>>>(chacha_key_from_bytes(key), column, first, count, d);
    CHECK(cudaGetLastError());
    std::vector<uint64_t> h(count);
    CHECK(cudaMemcpy(h.data(), d, count * 8, cudaMemcpyDeviceToHost));
    CHECK(cudaFree(d));
    FILE* f = fopen(argv[5], "wb");
    if (!f || fwrite(h.data(), 8, count, f) != count) return 1;
    fclose(f);
    return 0;
}
