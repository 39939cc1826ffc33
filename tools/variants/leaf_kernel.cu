// One copy of the production leaf-hash kernel (k_leaf_hash in plonky2_b200.cu), compiled to a cubin per
// compile-time variant (-DGL_... switches, launch bounds) by build.sh and timed by variant_bench.cu through the
// driver API. This is how kernel variants are ranked in one GPU run.
#include "../../plonky2_b200/csrc/gl_poseidon.cuh"
#ifndef VB_THREADS
#define VB_THREADS 128
#endif
#ifndef VB_MINB
#define VB_MINB 4  // HASH_MINB of plonky2_b200.cu
#endif
#ifndef VB_SYNC
#define VB_SYNC 1
#endif
extern "C" __global__ void __launch_bounds__(VB_THREADS, VB_MINB)
k_leaf(const uint64_t* leaves, size_t N, uint32_t W, uint64_t* out) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = j < N;
    if (!live) j = N - 1;
    uint64_t h[4];
    gl::hash_or_noop_strided<true, VB_SYNC != 0>(leaves + j, N, W, h);  // column-major, like the production LDE
    if (!live) return;
    out[4 * j] = h[0];
    out[4 * j + 1] = h[1];
    out[4 * j + 2] = h[2];
    out[4 * j + 3] = h[3];
}
extern "C" __global__ void k_threads(int* t) { *t = VB_THREADS; }
