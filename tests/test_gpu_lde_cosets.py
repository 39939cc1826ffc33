"""The coset-batched LDE against the per-coset path and the CPU oracle, bit for bit (run with `-m gpu` on an H100).

Multi-pass plans with an even first column pass (gl_ntt_host.cuh, lde_columns) run the first column pass of up to 8
cosets of a column group in one launch (k_ntt_col_cosets) and the row pass over all of them in another; everything else
(single-pass sizes, odd first passes) keeps one transform per coset. Bit 30 of gl_ctx_set_ntt_group selects the
per-coset loop everywhere, so every commitment here is built twice, once per path, and the caps and leaves must be
identical and equal the oracle's. The shapes cover rate_bits 1..4 (rate 4: two jobs of 8 cosets), single-, two- and
three-pass sizes, column counts that are not a multiple of 8 or of the group, short last groups, sharded commitments
(each shard is the LDE on its own coset base), non-resident commitments (blocks as large as n and smaller than n) and
salted commitments.
"""
import numpy as np
import pytest

from conftest import P, synth

pytestmark = pytest.mark.gpu

PER_COSET_BIT = 1 << 30


@pytest.fixture(scope="module")
def pb():
    import os

    import torch

    if not torch.cuda.is_available():
        if os.environ.get("GL_REQUIRE_GPU") == "1":
            raise AssertionError("GPU tests need a CUDA device")
        pytest.skip("no CUDA device (gpu-marked tests run on an H100)")
    import plonky2_b200 as p

    p.default_context()
    return p


@pytest.fixture(scope="module", params=["default groups", "24-column groups"])
def paths(request, pb):
    """(batched, per-coset) contexts; with 24-column groups a rate-1/8 LDE takes 3 columns x 8 cosets at a time."""
    group = 0 if request.param == "default groups" else 24
    ctxs = [pb.Context(0), pb.Context(0)]
    if group:
        ctxs[0].set_ntt_group(group)
    ctxs[1].set_ntt_group(group | PER_COSET_BIT)
    yield ctxs
    for c in ctxs:
        c.close()


def _coeffs(seed, B, log_n):
    return synth(seed, (B, 1 << log_n), canonical=False)


def _both(pb, paths, coeffs, rate_bits, cap_height, **kw):
    """cap and all leaf rows of from_coeffs on the batched and the per-coset path; asserts they are identical"""
    out = []
    for ctx in paths:
        c = pb.PolynomialBatch.from_coeffs(coeffs, rate_bits, kw.get("salt") is not None, cap_height, ctx=ctx, **kw)
        try:
            out.append((c.merkle_tree.cap.hashes.copy(), c.merkle_tree.get_rows(0, c.local_rows)))
        finally:
            c.close()  # before the context it was built on
    (cap_b, leaves_b), (cap_p, leaves_p) = out
    tag = "B=%d log_n=%d rate_bits=%d %s" % (coeffs.shape[0], int(np.log2(coeffs.shape[1])), rate_bits, kw)
    bad = np.argwhere(leaves_b != leaves_p)
    assert not len(bad), tag + ": batched != per-coset at leaf row %d column %d" % tuple(bad[0])
    assert np.array_equal(cap_b, cap_p), tag + ": caps differ"
    return cap_b, leaves_b


# (log_n, rate_bits, B): plans (a1, a2, b) of gl_ntt.cuh ntt_plan
SHAPES = [
    (9, 3, 13),    # single pass: per coset
    (12, 1, 13),   # (6, -, 6): batched, 2 cosets
    (12, 4, 11),   # (6, -, 6): batched, 16 cosets as two jobs of 8
    (13, 2, 21),   # (6, -, 7)
    (15, 3, 9),    # (7, -, 8): odd first pass, per coset
    (16, 3, 21),   # (8, -, 8)
    (20, 3, 3),    # (10, -, 10): the benchmark's plan
    (21, 1, 3),    # (7, 7, 7): three passes, odd first pass
    (24, 1, 2),    # (8, 8, 8): three passes, batched
]


@pytest.mark.parametrize("log_n,rate_bits,B", SHAPES)
def test_lde_batched_matches_per_coset_and_oracle(pb, oracle, paths, log_n, rate_bits, B):
    coeffs = _coeffs(0xC05E + 97 * log_n + rate_bits, B, log_n)
    cap, leaves = _both(pb, paths, coeffs, rate_bits, 4)
    if log_n + rate_bits > 23:
        return  # the oracle's tree is minutes here: the per-coset path is the reference at this size
    o = oracle.Commit(coeffs % np.uint64(P), rate_bits, 4, is_coeffs=True)
    assert np.array_equal(cap, o.cap), "log_n=%d rate_bits=%d B=%d: cap != oracle" % (log_n, rate_bits, B)
    assert np.array_equal(leaves, o.leaves), "log_n=%d rate_bits=%d B=%d: leaves != oracle" % (log_n, rate_bits, B)


@pytest.mark.parametrize("log_n,rate_bits,shards", [(12, 3, 2), (16, 2, 4), (20, 3, 8)])
def test_sharded_lde(pb, oracle, paths, log_n, rate_bits, shards):
    """shard g of G holds leaf rows [g*N/G, (g+1)*N/G): the LDE on the coset base of the shard"""
    B = 5
    coeffs = _coeffs(0x5AAD + log_n, B, log_n)
    o = oracle.Commit(coeffs % np.uint64(P), rate_bits, 4, is_coeffs=True)
    rows = (1 << (log_n + rate_bits)) // shards
    for g in range(shards):
        cap, leaves = _both(pb, paths, coeffs, rate_bits, 4, shard=(g, shards))
        assert np.array_equal(leaves, o.leaves[g * rows:(g + 1) * rows]), "shard %d/%d leaves != oracle" % (g, shards)
        per = (1 << 4) // shards
        assert np.array_equal(cap, o.cap[g * per:(g + 1) * per]), "shard %d/%d cap != oracle" % (g, shards)


@pytest.mark.parametrize("log_n,rate_bits,blocks", [(12, 3, 8), (16, 1, 4), (16, 3, 16)])
def test_non_resident_lde(pb, oracle, paths, log_n, rate_bits, blocks):
    """lde_blocks=G rebuilds blocks of N/G rows: as large as n (8 of 2^15), and smaller than n (the fold path)"""
    B = 11
    coeffs = _coeffs(0xB10C + log_n + blocks, B, log_n)
    cap, leaves = _both(pb, paths, coeffs, rate_bits, 4, lde_blocks=blocks)
    o = oracle.Commit(coeffs % np.uint64(P), rate_bits, 4, is_coeffs=True)
    assert np.array_equal(cap, o.cap) and np.array_equal(leaves, o.leaves), \
        "lde_blocks=%d log_n=%d rate_bits=%d != oracle" % (blocks, log_n, rate_bits)


@pytest.mark.parametrize("log_n,rate_bits", [(12, 3), (16, 2)])
def test_salted_lde(pb, oracle, paths, log_n, rate_bits):
    B = 7
    coeffs = _coeffs(0x5A17 + log_n, B, log_n)
    salt = synth(0x5A18 + log_n, (4, 1 << (log_n + rate_bits)))
    cap, leaves = _both(pb, paths, coeffs, rate_bits, 4, salt=salt)
    o = oracle.Commit(coeffs % np.uint64(P), rate_bits, 4, salt=salt, is_coeffs=True)
    assert np.array_equal(cap, o.cap) and np.array_equal(leaves, o.leaves), \
        "salted log_n=%d rate_bits=%d != oracle" % (log_n, rate_bits)
