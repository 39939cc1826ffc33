// gl_chacha.cuh -- salt for zero-knowledge commitments, drawn on the device from a ChaCha20 keystream.
//
// A blinded PolynomialBatch appends GL_SALT_SIZE = 4 uniformly random columns to every leaf (plonky2/src/fri/oracle.rs:
// 26,133-137; the reference draws them from OsRng with F::rand, field/src/goldilocks_field.rs:61-67). Drawing 4 x N
// words on the host and copying them over costs as much as the commitment itself at N = 2^23, so the salt is a keyed
// function evaluated where it is stored. The code here is __host__ __device__ so that tests/emu runs the same source.
//
// The keystream is the ChaCha20 block function of RFC 8439 section 2.3: a 256-bit key (8 little-endian words), a 32-bit
// block counter and a 96-bit nonce (3 little-endian words); a block is 64 bytes = 8 little-endian u64 words.
//
// Sampling rule. Salt element (s, i) -- stream column s (salt column s of a commitment, s < 4) and position i (the LDE
// row) -- is the first of the words
//     word (i mod 8) of block (i / 8) of the stream with nonce (s, a, 0),   a = 0, 1, 2, ...
// that is below CHACHA_BOUND (= p unless a test build lowers it). Accepted words are uniform on [0, CHACHA_BOUND):
// exactly uniform canonical field elements, like F::rand. At p a word is rejected with probability 2^-32. Every element
// is a pure function of (key, s, i), so any split of the rows -- row-block shards, (first, count) ranges -- draws the
// same values, and a host restatement reproduces them. Positions are below 2^35 (the 32-bit block counter).
#pragma once
#include <stdint.h>

#include "gl_field.cuh"

#ifndef GL_CHACHA_BOUND
#define GL_CHACHA_BOUND 0xFFFFFFFF00000001ULL
#endif

namespace gl {

constexpr uint64_t CHACHA_BOUND = GL_CHACHA_BOUND;
static_assert(CHACHA_BOUND > 0 && CHACHA_BOUND <= P, "the acceptance bound must lie in (0, p]");
constexpr uint64_t CHACHA_MAX_POSITION = (uint64_t)1 << 35;  // 2^32 blocks of 8 words

struct ChaChaKey {
    uint32_t w[8];
};

GL_HD ChaChaKey chacha_key_from_bytes(const uint8_t k[32]) {
    ChaChaKey key;
    for (int j = 0; j < 8; j++)
        key.w[j] = (uint32_t)k[4 * j] | (uint32_t)k[4 * j + 1] << 8 | (uint32_t)k[4 * j + 2] << 16 |
                   (uint32_t)k[4 * j + 3] << 24;
    return key;
}

GL_HD uint32_t chacha_rotl(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
#define GL_CHACHA_QR(a, b, c, d)                 \
    a += b, d ^= a, d = chacha_rotl(d, 16);     \
    c += d, b ^= c, b = chacha_rotl(b, 12);     \
    a += b, d ^= a, d = chacha_rotl(d, 8);      \
    c += d, b ^= c, b = chacha_rotl(b, 7)

// The ChaCha20 block function (RFC 8439 section 2.3): out = the 16 serialised state words
GL_HD void chacha20_block(const ChaChaKey& key, uint32_t counter, uint32_t n0, uint32_t n1, uint32_t n2, uint32_t out[16]) {
    uint32_t x[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, key.w[0], key.w[1], key.w[2], key.w[3],
                      key.w[4],    key.w[5],    key.w[6],    key.w[7],    counter,  n0,       n1,       n2};
    uint32_t s[16];
#pragma unroll
    for (int j = 0; j < 16; j++) s[j] = x[j];
#pragma unroll 1
    for (int r = 0; r < 10; r++) {
        GL_CHACHA_QR(x[0], x[4], x[8], x[12]);
        GL_CHACHA_QR(x[1], x[5], x[9], x[13]);
        GL_CHACHA_QR(x[2], x[6], x[10], x[14]);
        GL_CHACHA_QR(x[3], x[7], x[11], x[15]);
        GL_CHACHA_QR(x[0], x[5], x[10], x[15]);
        GL_CHACHA_QR(x[1], x[6], x[11], x[12]);
        GL_CHACHA_QR(x[2], x[7], x[8], x[13]);
        GL_CHACHA_QR(x[3], x[4], x[9], x[14]);
    }
#pragma unroll
    for (int j = 0; j < 16; j++) out[j] = x[j] + s[j];
}
#undef GL_CHACHA_QR

// word (pos mod 8) of block (pos / 8) of the stream with nonce (column, attempt, 0)
GL_HD uint64_t chacha_word(const ChaChaKey& key, uint32_t column, uint32_t attempt, uint64_t pos) {
    uint32_t b[16];
    chacha20_block(key, (uint32_t)(pos >> 3), column, attempt, 0, b);
    const int k = (int)(pos & 7);
    return (uint64_t)b[2 * k] | (uint64_t)b[2 * k + 1] << 32;
}
// the sampling rule from attempt 1 on, for a position whose attempt-0 word was rejected
GL_HD uint64_t chacha_sample_retry(const ChaChaKey& key, uint32_t column, uint64_t pos) {
    for (uint32_t a = 1;; a++) {
        const uint64_t w = chacha_word(key, column, a, pos);
        if (w < CHACHA_BOUND) return w;
    }
}
// salt element (column, pos)
GL_HD uint64_t chacha_sample(const ChaChaKey& key, uint32_t column, uint64_t pos) {
    const uint64_t w = chacha_word(key, column, 0, pos);
    return w < CHACHA_BOUND ? w : chacha_sample_retry(key, column, pos);
}

// The 8 elements of positions [8 * blk, 8 * blk + 8): one attempt-0 block, later attempts only for rejected words
GL_HD void chacha_sample_block(const ChaChaKey& key, uint32_t column, uint64_t blk, uint64_t out[8]) {
    uint32_t b[16];
    chacha20_block(key, (uint32_t)blk, column, 0, 0, b);
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint64_t w = (uint64_t)b[2 * k] | (uint64_t)b[2 * k + 1] << 32;
        out[k] = w < CHACHA_BOUND ? w : chacha_sample_retry(key, column, 8 * blk + k);
    }
}

GL_HD uint64_t chacha_bitrev(uint64_t x, uint32_t bits) {
    uint64_t r = 0;
    for (uint32_t k = 0; k < bits; k++) r |= ((x >> k) & 1) << (bits - 1 - k);
    return r;
}

// One thread of the salt fill. The salt columns of a commitment with N = 2^log_N leaves are stored column-major in leaf
// order: salt column s at leaf j holds element (s, bitrev(j)) -- the LDE row of leaf j (oracle.rs:142-147), the same
// convention as an explicit salt array laid out by LDE row. This handle owns leaves [leaf0, leaf0 + nloc), written to
// out[s * stride + (j - leaf0)].
// For log_N >= 3, item t (of salt_fill_items) owns block bitrev_{log_N - 3}(t0 + t), t0 = leaf0 mod N/8: its rows
// 8 * bitrev(t0 + t) + k sit at leaves t0 + t + bitrev_3(k) * N/8, so consecutive items write consecutive leaves.
// For log_N < 3 a single item draws block 0.
GL_HD size_t salt_fill_items(uint32_t log_N, uint64_t nloc) {
    if (log_N < 3) return 1;
    const uint64_t q = (uint64_t)1 << (log_N - 3);
    return (size_t)(nloc < q ? nloc : q);
}
GL_HD void salt_fill_item(const ChaChaKey& key, uint32_t s, uint64_t t, uint32_t log_N, uint64_t leaf0, uint64_t nloc,
                          uint64_t* out, uint64_t stride) {
    uint64_t w[8];
    if (log_N < 3) {
        chacha_sample_block(key, s, 0, w);
        for (uint64_t row = 0; row < ((uint64_t)1 << log_N); row++) {
            const uint64_t j = chacha_bitrev(row, log_N);
            if (j >= leaf0 && j - leaf0 < nloc) out[s * stride + (j - leaf0)] = w[row];
        }
        return;
    }
    const uint32_t lq = log_N - 3;
    const uint64_t q = (uint64_t)1 << lq;
    const uint64_t tt = (leaf0 & (q - 1)) + t;
    chacha_sample_block(key, s, chacha_bitrev(tt, lq), w);
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint64_t j = tt + (chacha_bitrev((uint64_t)k, 3) << lq);
        if (j >= leaf0 && j - leaf0 < nloc) out[s * stride + (j - leaf0)] = w[k];
    }
}

#if defined(__CUDACC__)
// salt columns s = blockIdx.y of a commitment's (shard of the) column-major LDE: out = the first salt column
__global__ void k_chacha_salt(ChaChaKey key, uint32_t log_N, uint64_t leaf0, uint64_t nloc, uint64_t* out,
                              uint64_t stride) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= salt_fill_items(log_N, nloc)) return;
    salt_fill_item(key, blockIdx.y, t, log_N, leaf0, nloc, out, stride);
}
// out[j] = element (column, first + j), j < count: one block per thread
__global__ void k_chacha_elements(ChaChaKey key, uint32_t column, uint64_t first, uint64_t count, uint64_t* out) {
    const uint64_t blk = (first >> 3) + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (8 * blk >= first + count) return;
    uint64_t w[8];
    chacha_sample_block(key, column, blk, w);
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint64_t pos = 8 * blk + k;
        if (pos >= first && pos < first + count) out[pos - first] = w[k];
    }
}
#endif

}  // namespace gl
