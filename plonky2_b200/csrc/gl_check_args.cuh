// gl_check_args.cuh -- the per-thread code of plonky2's two global-argument checks on a witness,
// gl_plonk_check_copies and gl_plonk_check_lookups of include/plonky2_b200_check.h. They find what the reference's
// witness generation stops at (iop/witness.rs:358, "Partition containing {target} was set twice with different values";
// gates/lookup.rs:208-220, "Incorrect input value provided") and what set_lookup_wires (plonk/prover.rs:50-108) writes.
//
// Copies. Routed wire i = row * num_routed + col has the identity value k_is[col] * w_n^row and the sigma value
// sigmas[col][row]; sigma(i) is the routed wire whose identity value is i's sigma value. Sorting both lists by value
// pairs them up position by position: position p holds the owner i_p of a sigma value and the wire j_p whose identity
// it is, so sigma(i_p) = j_p. Wire i fails when canon(wire(i)) != canon(wire(sigma(i))).
//
// Lookups. Table k of lookup_rows (last_lu, last_lut, first_lut) has LookupGate rows [last_lu, last_lut), whose slot s
// holds (input, output) in wires (2s, 2s + 1), and LookupTableGate rows [last_lut, first_lut], whose slot s holds
// (input, output, multiplicity) in wires (3s, 3s + 1, 3s + 2). LUT entry e sits in row first_lut - e / num_lut_slots,
// slot e % num_lut_slots; the slots past the LUT's length hold entry 0 with multiplicity 0. A looking slot counts for
// the entry the reference's input -> index map gives its input (a later entry wins over an earlier one of the same
// input), except the padding: the run of slots at the end of row last_lut - 1 that all hold exactly entry 0 counts for
// entry 0. (The reference knows how many lookups it placed; a witness does not. Real lookups of entry 0 that end the
// row are taken for padding, which matters only when entry 0's input appears again later in the LUT: then an honest
// witness gets two L3 failures, a known false positive.) The failures of a row, slot by slot, as
// (row, 4 * slot + kind):
//   LOOKUP_L1  a looking slot whose (input, output) is not an entry of the LUT;
//   LOOKUP_L2  a table slot whose (input, output) is not the entry placed there;
//   LOOKUP_L3  a table slot whose multiplicity is not the count of its entry (0 past the LUT's length).
//
// The kernels in gl_check_args_host.cuh call these functions per thread; tests/emu/check_args_emu.cpp runs them on the
// host.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "gl_field.cuh"

namespace gl {

// ---- copies
struct CopyCheck {
    const uint64_t* wires;  // routed column c at wires + c * wires_stride
    size_t wires_stride;
    const uint64_t* sigmas;  // sigma column c at sigmas + c * sigmas_stride
    size_t sigmas_stride;
    const uint64_t* k_is;  // num_routed coset shifts
    const uint64_t *xhi, *xlo;  // w_n^r = xhi[r >> 12] * xlo[r & 4095]
    uint32_t num_routed;
};

GL_HD uint64_t copy_wire(const CopyCheck& c, uint64_t i) {
    return canon(c.wires[(i % c.num_routed) * c.wires_stride + i / c.num_routed]);
}
// The identity value k_is[col] * w_n^row of routed wire i, canonical
GL_HD uint64_t copy_identity(const CopyCheck& c, uint64_t i) {
    const uint64_t row = i / c.num_routed;
    return canon(mul(c.k_is[i % c.num_routed], mul(c.xhi[row >> 12], c.xlo[row & 4095])));
}
// The sigma value of routed wire i, canonical
GL_HD uint64_t copy_sigma(const CopyCheck& c, uint64_t i) {
    return canon(c.sigmas[(i % c.num_routed) * c.sigmas_stride + i / c.num_routed]);
}
// Wire i breaks its copy constraint: sig = sigma(i)
GL_HD bool copy_fails(const CopyCheck& c, uint64_t i, uint32_t sig) { return copy_wire(c, i) != copy_wire(c, sig); }

// ---- lookups
constexpr uint32_t LOOKUP_L1 = 1, LOOKUP_L2 = 2, LOOKUP_L3 = 3;
constexpr uint32_t LOOKUP_NO_ENTRY = 0xFFFFFFFFu;

struct LookupCheck {
    const uint64_t* wires;  // column c at wires + c * stride
    size_t stride;
    uint32_t num_lu_slots, num_lut_slots, n_luts;
    const uint32_t* rows;     // (last_lu, last_lut, first_lut) per table
    const uint32_t* lut;      // every table's entries as keys input | output << 16, table k at lut_off[k]
    const uint32_t* lut_off;  // n_luts + 1 offsets
    const uint32_t* keys;     // table k's distinct keys in ascending order at lut_off[k], key_len[k] of them
    const uint32_t* key_len;
    const uint32_t* index_of;  // 65536 words per table: input -> the reference's entry, LOOKUP_NO_ENTRY if none
    const uint32_t* counts;    // the count of every entry, laid out as lut (read by lookup_check_row)
};

// The key input | output << 16 of a pair whose values are canonically below 2^16; false otherwise
GL_HD bool lookup_key(uint64_t in, uint64_t out, uint32_t* key) {
    in = canon(in);
    out = canon(out);
    if (in >> 16 || out >> 16) return false;
    *key = (uint32_t)(in | out << 16);
    return true;
}
GL_HD bool lookup_has_key(const LookupCheck& p, uint32_t k, uint32_t key) {
    const uint32_t* keys = p.keys + p.lut_off[k];
    uint32_t lo = 0, hi = p.key_len[k];
    while (lo < hi) {
        const uint32_t mid = (lo + hi) / 2;
        if (keys[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    return lo < p.key_len[k] && keys[lo] == key;
}
// The table whose LookupGate rows (*looking) or LookupTableGate rows hold `row`, or -1
GL_HD int lookup_table_of(const LookupCheck& p, size_t row, bool* looking) {
    for (uint32_t k = 0; k < p.n_luts; k++) {
        const uint32_t* r = p.rows + 3 * k;
        if (row >= r[0] && row <= r[2]) {
            *looking = row < r[1];
            return (int)k;
        }
    }
    return -1;
}
// The wire pair of looking slot s
GL_HD uint64_t lookup_in(const LookupCheck& p, size_t row, uint32_t s) { return p.wires[2 * s * p.stride + row]; }
GL_HD uint64_t lookup_out(const LookupCheck& p, size_t row, uint32_t s) { return p.wires[(2 * s + 1) * p.stride + row]; }
// The entry of table k that looking slot (row, s) counts for, or LOOKUP_NO_ENTRY
GL_HD uint32_t lookup_counted_entry(const LookupCheck& p, uint32_t k, size_t row, uint32_t s) {
    const uint32_t first = p.lut[p.lut_off[k]];
    if (row + 1 == p.rows[3 * k + 1]) {  // the last LookupGate row: is s in the padding run?
        bool pad = true;
        for (uint32_t t = s; t < p.num_lu_slots && pad; t++) {
            uint32_t key;
            pad = lookup_key(lookup_in(p, row, t), lookup_out(p, row, t), &key) && key == first;
        }
        if (pad) return 0;
    }
    const uint64_t in = canon(lookup_in(p, row, s));
    return in >> 16 ? LOOKUP_NO_ENTRY : p.index_of[((size_t)k << 16) + in];
}
// The failures of `row` (every kind, slot by slot); with pairs, failure m is written as (row, 4 * slot + kind) at
// pairs[2m], pairs[2m + 1]. Reads p.counts.
GL_HD uint32_t lookup_check_row(const LookupCheck& p, size_t row, uint32_t* pairs) {
    bool looking = false;
    const int kk = lookup_table_of(p, row, &looking);
    if (kk < 0) return 0;
    const uint32_t k = (uint32_t)kk, off = p.lut_off[k], len = p.lut_off[k + 1] - off;
    uint32_t fails = 0;
    auto fail = [&](uint32_t s, uint32_t kind) {
        if (pairs) {
            pairs[2 * fails] = (uint32_t)row;
            pairs[2 * fails + 1] = 4 * s + kind;
        }
        fails++;
    };
    if (looking) {
        for (uint32_t s = 0; s < p.num_lu_slots; s++) {
            uint32_t key;
            if (!lookup_key(lookup_in(p, row, s), lookup_out(p, row, s), &key) || !lookup_has_key(p, k, key))
                fail(s, LOOKUP_L1);
        }
        return fails;
    }
    const size_t first_lut = p.rows[3 * k + 2];
    for (uint32_t s = 0; s < p.num_lut_slots; s++) {
        const size_t e = (first_lut - row) * p.num_lut_slots + s;
        const uint64_t* w = p.wires + (size_t)3 * s * p.stride + row;
        uint32_t key;
        if (!lookup_key(w[0], w[p.stride], &key) || key != p.lut[off + (e < len ? e : 0)]) fail(s, LOOKUP_L2);
        if (canon(w[2 * p.stride]) != (e < len ? p.counts[off + e] : 0)) fail(s, LOOKUP_L3);
    }
    return fails;
}

}  // namespace gl
