"""Full-scale parity of the configurations bench.py times (BASELINE.json configs[1] and configs[4]) against golden
fixtures made by the CPU oracle (tools/make_fullscale_fixtures.py, committed under tests/golden/): the cap, 64 sampled
leaf rows (by digest, 4 of them word for word) with their Merkle paths, and a checksum of the coefficient matrix.
The input is the SURVEY 8(d) splitmix64 generator, regenerated here; nothing on this path needs the 100-s oracle run
or anything outside the repository. Run with `-m gpu` on an H100."""
import json
import os

import numpy as np
import pytest

from conftest import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load_fixture(name):
    path = os.path.join(ROOT, "tests", "golden", "fullscale_%s.json" % name)
    if not os.path.exists(path):
        pytest.skip("fixture %s not generated" % path)
    return json.load(open(path))


@pytest.fixture(scope="module")
def pb():
    import torch

    if not torch.cuda.is_available():
        if os.environ.get("GL_REQUIRE_GPU") == "1":
            raise AssertionError("GPU tests need a CUDA device")
        pytest.skip("no CUDA device (gpu-marked tests run on an H100)")
    import plonky2_b200 as p

    p.default_context()
    return p


def coeff_checksum(coeffs):
    with np.errstate(over="ignore"):
        w = np.arange(1, coeffs.shape[1] + 1, dtype=np.uint64)
        return int(np.bitwise_xor.reduce((coeffs * w).sum(axis=1, dtype=np.uint64) * np.arange(1, coeffs.shape[0] + 1, dtype=np.uint64)))


def check_against_fixture(pb, oracle, fx, batch, row_offset=0, local_cap=None):
    """batch holds leaf rows [row_offset, row_offset + batch.local_rows) of the commitment the fixture describes."""
    cfg = fx["config"]
    cap = np.array(fx["cap"], dtype=np.uint64)
    h_local = cfg["cap_height"] - (batch.num_shards.bit_length() - 1)
    got_cap = batch.merkle_tree.cap.hashes
    per = len(cap) // batch.num_shards
    assert np.array_equal(got_cap, cap[batch.shard_index * per:(batch.shard_index + 1) * per]), "cap differs from the oracle's"
    idx = [i for i in fx["leaf_indices"] if row_offset <= i < row_offset + batch.local_rows]
    assert idx or batch.num_shards > 1
    if not idx:
        return 0
    rows, paths = batch.merkle_tree.open_many([i - row_offset for i in idx])
    for k, i in enumerate(idx):
        j = fx["leaf_indices"].index(i)
        assert [int(x) for x in rows[k][:8]] == fx["leaf_head"][j], ("leaf head", i)
        assert [int(x) for x in oracle.hash_or_noop(rows[k])] == fx["leaf_digests"][j], ("leaf digest", i)
        if j < 4:
            assert [int(x) for x in rows[k]] == fx["full_rows"][j], ("leaf row", i)
            want = np.array(fx["siblings"][j], dtype=np.uint64)
            assert np.array_equal(paths[k], want[:paths.shape[1]]), ("siblings", i)
        # every opening verifies against (this shard's part of) the oracle's cap (merkle_proofs.rs:55-107)
        assert oracle.merkle_verify(rows[k], i - row_offset, paths[k], got_cap, h_local), ("merkle path", i)
    return len(idx)


@pytest.mark.parametrize("name", ["small", "cfg2", "cfg5"])
def test_fullscale_commit_matches_oracle_fixture(pb, oracle, name):
    fx = load_fixture(name)
    cfg = fx["config"]
    vals = synth(cfg["seed"], (cfg["columns"], 1 << cfg["log_n"]))
    c = pb.PolynomialBatch.from_values(vals, cfg["rate_bits"], False, cfg["cap_height"])  # HOST buffers in
    try:
        assert check_against_fixture(pb, oracle, fx, c) == len(fx["leaf_indices"])
        assert coeff_checksum(c.polynomials) == fx["coeff_checksum"], "coefficients differ from the oracle's"
    finally:
        c.close()


@pytest.mark.parametrize("name,shards", [("small", 2), ("small", 8), ("cfg2", 4)])
def test_fullscale_row_block_shards_one_gpu(pb, oracle, name, shards):
    """The row-block sharding bench.py --gpus N times, every shard built on THIS GPU in turn: each shard's cap
    entries and openings must be the oracle's (SURVEY 8e)."""
    fx = load_fixture(name)
    cfg = fx["config"]
    vals = synth(cfg["seed"], (cfg["columns"], 1 << cfg["log_n"]))
    seen = 0
    for g in range(shards):
        c = pb.PolynomialBatch.from_values(vals, cfg["rate_bits"], False, cfg["cap_height"], shard=(g, shards))
        try:
            seen += check_against_fixture(pb, oracle, fx, c, row_offset=g * c.local_rows)
        finally:
            c.close()
    assert seen == len(fx["leaf_indices"])
