// Host run of the index code of the device sigma polynomials (plonky2_b200/csrc/gl_sigma.cuh): the routed wires' keys
// and values as k_sigma_keys builds them from the component labels, a stable sort in place of the device radix sort, and
// the same sigma_is_head / sigma_successor / sigma_out_index that k_sigma_heads and k_sigma_fill call per thread, with
// threads as loops. Test infrastructure: built as a shared library and driven by tests/test_circuit_data.py, which
// compares the result with the restatement of Forest::wire_partition + get_sigma_map.
#include <algorithm>
#include <numeric>
#include <vector>

#include "../../plonky2_b200/csrc/gl_sigma.cuh"
using namespace gl;

// labels: the component label of every target (num_targets words, any representative). out: get_sigma_map's value
// col' * n + row' of the successor, at the wire's own index col * n + row (num_routed x n words).
extern "C" void emu_sigma_map(const uint32_t* labels, uint32_t num_wires, uint32_t num_routed, uint32_t log_n,
                              uint64_t num_targets, uint64_t* out) {
    const SigmaShape s{num_wires, num_routed, log_n, num_targets};
    const size_t count = ((size_t)1 << log_n) * num_routed;
    std::vector<uint32_t> keys(count), vals(count), order(count), skeys(count), svals(count), heads(num_targets);
    for (size_t i = 0; i < count; i++) {
        keys[i] = labels[sigma_target(i, s)];
        vals[i] = (uint32_t)i;
    }
    std::iota(order.begin(), order.end(), 0u);
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return keys[a] < keys[b]; });
    for (size_t p = 0; p < count; p++) {
        skeys[p] = keys[order[p]];
        svals[p] = vals[order[p]];
    }
    for (size_t p = 0; p < count; p++)
        if (sigma_is_head(skeys.data(), p)) heads[skeys[p]] = (uint32_t)p;
    for (size_t p = 0; p < count; p++) {
        const uint32_t j = sigma_successor(skeys.data(), svals.data(), heads.data(), count, p);
        out[sigma_out_index(svals[p], s)] = ((uint64_t)(j % num_routed) << log_n) + j / num_routed;
    }
}

// sigma_check_target of every index: 0, SIGMA_OUT_OF_RANGE or SIGMA_NOT_ROUTED
extern "C" void emu_sigma_check(const uint64_t* targets, size_t count, uint32_t num_wires, uint32_t num_routed,
                                uint32_t log_n, uint64_t num_targets, uint32_t* out) {
    const SigmaShape s{num_wires, num_routed, log_n, num_targets};
    for (size_t i = 0; i < count; i++) out[i] = sigma_check_target(targets[i], s);
}
