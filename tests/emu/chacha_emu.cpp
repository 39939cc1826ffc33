// Host run of the device salt sampler (plonky2_b200/csrc/gl_chacha.cuh): the block function, the per-thread bodies of
// k_chacha_elements and k_chacha_salt with threads as loops. Test infrastructure: built as a shared library (once with
// the default acceptance bound, once with a lowered one) and driven by tests/test_chacha_salt.py, which compares it with
// a Python restatement of RFC 8439 and of the sampling rule.
#include <vector>
#include "../../plonky2_b200/csrc/gl_chacha.cuh"
using namespace gl;

extern "C" uint64_t emu_chacha_bound() { return CHACHA_BOUND; }

extern "C" void emu_chacha_block(const uint8_t key[32], uint32_t counter, uint32_t n0, uint32_t n1, uint32_t n2,
                                 uint32_t out[16]) {
    chacha20_block(chacha_key_from_bytes(key), counter, n0, n1, n2, out);
}

// out[j] = element (column, first + j): k_chacha_elements' body (one block per "thread"), and chacha_sample per position
extern "C" int emu_chacha_elements(const uint8_t key[32], uint32_t column, uint64_t first, uint64_t count, uint64_t* out) {
    const ChaChaKey k = chacha_key_from_bytes(key);
    for (uint64_t blk = first >> 3; 8 * blk < first + count; blk++) {
        uint64_t w[8];
        chacha_sample_block(k, column, blk, w);
        for (int j = 0; j < 8; j++) {
            const uint64_t pos = 8 * blk + j;
            if (pos >= first && pos < first + count) out[pos - first] = w[j];
        }
    }
    int bad = 0;
    for (uint64_t j = 0; j < count; j++) bad |= chacha_sample(k, column, first + j) != out[j];
    return bad;
}

// the 4 salt columns of leaves [leaf0, leaf0 + nloc) of an LDE of 2^log_N rows: out = 4 x nloc words (k_chacha_salt)
extern "C" void emu_salt_fill(const uint8_t key[32], uint32_t log_N, uint64_t leaf0, uint64_t nloc, uint64_t* out) {
    const ChaChaKey k = chacha_key_from_bytes(key);
    for (uint32_t s = 0; s < 4; s++)
        for (uint64_t t = 0; t < salt_fill_items(log_N, nloc); t++) salt_fill_item(k, s, t, log_N, leaf0, nloc, out, nloc);
}
