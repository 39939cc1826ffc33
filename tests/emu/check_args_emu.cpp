// Host run of the per-thread code of gl_plonk_check_copies and gl_plonk_check_lookups (plonky2_b200/csrc/
// gl_check_args.cuh): the same copy_identity / copy_sigma / copy_fails and lookup_counted_entry / lookup_check_row the
// kernels call, with threads as loops, std::sort in place of the device radix sort, and the tables prepared as
// gl_check_args_host.cuh prepares them. Test infrastructure: built as a shared library and driven by
// tests/test_check_arguments.py against a restatement of the reference's partition and lookup rules.
#include <algorithm>
#include <utility>
#include <vector>

#include "../../plonky2_b200/csrc/gl_check_args.cuh"
using namespace gl;

// Every failing (i, sigma(i)) pair in ascending i at pairs (2 words each); returns their number, or ~0 when the sigmas
// are not a permutation of the identity values. Columns are n words apart.
extern "C" uint64_t emu_check_copies(const uint64_t* wires, const uint64_t* sigmas, const uint64_t* k_is,
                                     uint32_t log_n, uint32_t num_routed, uint32_t* pairs) {
    const size_t n = (size_t)1 << log_n, count = n * num_routed;
    const size_t tlen = 4096 > (n >> 12) + 1 ? 4096 : (n >> 12) + 1;  // x_pow_tables in plonky2_b200.cu
    const uint64_t w = root_of_unity(log_n), w4096 = pow(w, 4096);
    std::vector<uint64_t> xhi(tlen), xlo(tlen);
    for (size_t t = 0; t < tlen; t++) {
        xhi[t] = t ? mul(xhi[t - 1], w4096) : 1;
        xlo[t] = t ? mul(xlo[t - 1], w) : 1;
    }
    const CopyCheck c{wires, n, sigmas, n, k_is, xhi.data(), xlo.data(), num_routed};
    std::vector<std::pair<uint64_t, uint32_t>> id(count), sg(count);
    for (size_t i = 0; i < count; i++) {
        id[i] = {copy_identity(c, i), (uint32_t)i};
        sg[i] = {copy_sigma(c, i), (uint32_t)i};
    }
    std::sort(id.begin(), id.end());
    std::sort(sg.begin(), sg.end());
    std::vector<uint32_t> sig(count);
    for (size_t p = 0; p < count; p++) {
        if (id[p].first != sg[p].first) return ~0ull;
        sig[sg[p].second] = id[p].second;
    }
    uint64_t total = 0;
    for (size_t i = 0; i < count; i++)
        if (copy_fails(c, i, sig[i])) {
            pairs[2 * total] = (uint32_t)i;
            pairs[2 * total + 1] = sig[i];
            total++;
        }
    return total;
}

// Every failure as (row, 4 * slot + kind), rows in order, at pairs (2 words each; room for every slot of every row);
// counts: every entry's count, laid out as luts. Returns the number of failures. luts: (input, output) u16 pairs,
// table k at lut_offsets[k]; rows: (last_lu, last_lut, first_lut) per table. Columns are n words apart.
extern "C" uint64_t emu_check_lookups(const uint64_t* wires, uint32_t log_n, uint32_t num_routed, const uint16_t* luts,
                                      const uint32_t* lut_offsets, const uint32_t* rows, uint32_t n_luts,
                                      uint32_t* counts, uint32_t* pairs) {
    const size_t n = (size_t)1 << log_n;
    const uint32_t total = lut_offsets[n_luts];
    std::vector<uint32_t> lut(total), keys(total), key_len(n_luts);
    std::vector<uint32_t> index_of((size_t)n_luts << 16, LOOKUP_NO_ENTRY);
    for (uint32_t k = 0; k < n_luts; k++) {
        const uint32_t b = lut_offsets[k], e = lut_offsets[k + 1];
        for (uint32_t t = b; t < e; t++) {
            lut[t] = (uint32_t)luts[2 * t] | (uint32_t)luts[2 * t + 1] << 16;
            index_of[((size_t)k << 16) + luts[2 * t]] = t - b;
        }
        std::copy(lut.begin() + b, lut.begin() + e, keys.begin() + b);
        std::sort(keys.begin() + b, keys.begin() + e);
        key_len[k] = (uint32_t)(std::unique(keys.begin() + b, keys.begin() + e) - (keys.begin() + b));
    }
    std::fill(counts, counts + total, 0u);
    LookupCheck p{wires, n, num_routed / 2, num_routed / 3, n_luts, rows, lut.data(), lut_offsets, keys.data(),
                  key_len.data(), index_of.data(), counts};
    for (size_t row = 0; row < n; row++) {
        bool looking = false;
        const int k = lookup_table_of(p, row, &looking);
        if (k < 0 || !looking) continue;
        for (uint32_t s = 0; s < p.num_lu_slots; s++) {
            const uint32_t e = lookup_counted_entry(p, (uint32_t)k, row, s);
            if (e != LOOKUP_NO_ENTRY) counts[lut_offsets[k] + e]++;
        }
    }
    uint64_t fails = 0;
    for (size_t row = 0; row < n; row++) fails += lookup_check_row(p, row, pairs + 2 * fails);
    return fails;
}
