// gl_sigma.cuh -- the index part of plonky2's sigma polynomials: CircuitBuilder::sigma_vecs
// (plonk/circuit_builder.rs:993-1028) with Forest::wire_partition and WirePartition::get_sigma_map / get_sigma_polys
// (plonk/permutation_argument.rs:90-157).
//
// Targets are numbered as Target::index (iop/target.rs:55-60): wire (row, col) is row * num_wires + col, virtual
// target i is n * num_wires + i. Routed wire (row, col), col < num_routed, has the row-major routed index
// row * num_routed + col, the order in which wire_partition pushes wires into their sets. Once every target carries the
// label of its connected component, the routed wires sorted stably by label (values = routed indices, ascending) form
// one segment per partition set in row-major order; wire i's sigma is the next wire of its segment, or the segment's
// first wire for the last one: sigma(row, col) = k_is[col'] * w_n^row' for that successor (row', col').
//
// The kernels in plonky2_b200.cu call these functions per thread; tests/emu/sigma_emu.cpp runs them on the host.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "gl_field.cuh"

namespace gl {

struct SigmaShape {
    uint32_t num_wires, num_routed, log_n;
    uint64_t num_targets;  // n * num_wires + num_virtual_targets (< 2^32: the labels are u32)
};

// The target of routed index i
GL_HD uint64_t sigma_target(uint64_t i, const SigmaShape& s) {
    return (i / s.num_routed) * s.num_wires + i % s.num_routed;
}

constexpr uint32_t SIGMA_OUT_OF_RANGE = 1;  // a target index >= num_targets
constexpr uint32_t SIGMA_NOT_ROUTED = 2;    // a wire of column >= num_routed (CircuitBuilder::connect asserts routability)
// 0, or the reason the copy-constraint endpoint t is refused
GL_HD uint32_t sigma_check_target(uint64_t t, const SigmaShape& s) {
    if (t >= s.num_targets) return SIGMA_OUT_OF_RANGE;
    if (t < ((uint64_t)s.num_wires << s.log_n) && t % s.num_wires >= s.num_routed) return SIGMA_NOT_ROUTED;
    return 0;
}

// Sorted position p starts a segment (a partition set)
GL_HD bool sigma_is_head(const uint32_t* keys, size_t p) { return p == 0 || keys[p] != keys[p - 1]; }

// The routed index that sorted position p maps to: the next one of its segment, else the segment's head
// (heads[label] = the head's position)
GL_HD uint32_t sigma_successor(const uint32_t* keys, const uint32_t* vals, const uint32_t* heads, size_t count,
                               size_t p) {
    return (p + 1 < count && keys[p + 1] == keys[p]) ? vals[p + 1] : vals[heads[keys[p]]];
}

// Where routed index i's sigma value goes in the column-major output (column col at out + col * n)
GL_HD size_t sigma_out_index(uint32_t i, const SigmaShape& s) {
    return ((size_t)(i % s.num_routed) << s.log_n) + i / s.num_routed;
}

}  // namespace gl
