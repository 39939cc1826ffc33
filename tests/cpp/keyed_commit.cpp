// A zero-knowledge commitment through the C++ mirror (include/plonky2_b200.hpp): PolynomialBatch::from_values with a
// SaltKey, the salt drawn on the device. Prints the cap words (one per line, decimal) of
// 5 polynomials of 64 values v[b][i] = (b * 64 + i) * 0x9E3779B97F4A7C15 mod 2^64, rate_bits 2, cap_height 2,
// key bytes 0..31; tests/test_zk_commit_and_prove.py compares them with the Python layer's keyed commitment.
#include <cstdio>

#include "plonky2_b200.hpp"

int main() {
    using namespace plonky2_b200;
    Context ctx(0);
    std::vector<std::vector<F>> v(5, std::vector<F>(64));
    for (size_t b = 0; b < 5; b++)
        for (size_t i = 0; i < 64; i++) v[b][i] = (uint64_t)(b * 64 + i) * 0x9E3779B97F4A7C15ull;
    std::array<uint8_t, 32> key;
    for (int j = 0; j < 32; j++) key[j] = (uint8_t)j;
    PolynomialBatch pb = PolynomialBatch::from_values(ctx, v, 2, true, 2, SaltKey::of(key));
    if (pb.leaf_width() != 9) return 1;
    for (const F& w : pb.cap().flatten()) printf("%llu\n", (unsigned long long)w);
    return 0;
}
