"""world_size-2 gloo test of the multi-GPU host logic (plonky2_b200/distributed.py) on CPU: each rank
owns one row block of the commitment (its leaves/cap come from the oracle here, since there is no GPU),
the ranks all-gather their cap entries, and every rank must end with the single-device cap."""
import numpy as np
import pytest

from ranks import spawn_ranks


def _worker(rank, world):
    import oracle_lib
    from conftest import synth
    from plonky2_b200 import distributed as D

    B, log_n, r, h = 5, 6, 2, 3
    N = 1 << (log_n + r)
    vals = synth(0x55, (B, 1 << log_n))
    full = oracle_lib.Commit(vals, r, h, nthreads=1)
    lo, hi = D.shard_row_range(N, rank, world)
    clo, chi = D.shard_cap_range(h, rank, world)
    # this rank's shard: its own leaves reduced to its own cap entries
    _, local_cap = oracle_lib.merkle_build(full.leaves[lo:hi], h - int(np.log2(world)), nthreads=1)
    assert np.array_equal(local_cap, full.cap[clo:chi])
    cap = D.gather_cap(local_cap)
    ok = np.array_equal(cap.hashes, full.cap)
    owner = D.owner_of_leaf(N - 1, N, world)
    return rank, bool(ok), owner


def test_cap_all_gather_two_ranks():
    res = spawn_ranks(_worker, 2, timeout=180)
    assert [r[0] for r in res] == [0, 1]
    assert all(r[1] for r in res)
    assert all(r[2] == (1, 127) for r in res)


def test_shard_ranges():
    from plonky2_b200 import distributed as D

    assert D.shard_row_range(1 << 10, 3, 8) == (384, 512)
    assert D.shard_cap_range(4, 3, 8) == (6, 8)
    with pytest.raises(ValueError):
        D.shard_cap_range(2, 0, 8)
    assert D.owner_of_leaf(700, 1024, 4) == (2, 188)
    # single process: gather_cap is the identity
    cap = np.arange(16, dtype=np.uint64).reshape(4, 4)
    assert np.array_equal(D.gather_cap(cap).hashes, cap)


def test_placement_open_many_routing_single_process():
    """Routing logic of Placement.open_many with a fake local batch (no GPU, no process group): owned indices are
    opened locally with the local index; an index owned by another shard makes the single-process call fail loudly.
    On one device (Placement()) the tree opens the indices itself and the cap is the commitment's own."""
    from plonky2_b200 import distributed as D

    class FakeTree:
        cap = np.arange(8, dtype=np.uint64).reshape(2, 4)

        def open_many(self, idx):
            idx = list(idx)
            return (np.array([[100 + i, 7] for i in idx], dtype=np.uint64).reshape(len(idx), 2),
                    np.zeros((len(idx), 3, 4), dtype=np.uint64))

    class FakeBatch:
        num_shards, shard_index, lde_size, leaf_width = 2, 1, 64, 2
        degree_log, rate_bits, cap_height = 5, 1, 3
        merkle_tree = FakeTree()

    shard = D.Placement(1, 2)
    lv, pt = shard.open_many(FakeBatch(), [32, 63])   # both owned by shard 1 -> local 0 and 31
    assert lv[:, 0].tolist() == [100, 131] and pt.shape == (2, 3, 4)
    with pytest.raises(RuntimeError):
        shard.open_many(FakeBatch(), [5])             # owned by shard 0, nobody serves it here
    one = D.Placement()
    assert one.shard == (0, 1)
    lv, pt = one.open_many(FakeBatch(), [5, 32])      # the tree's own indices
    assert lv[:, 0].tolist() == [105, 132] and pt.shape == (2, 3, 4)
    assert one.cap(FakeBatch()) is FakeBatch.merkle_tree.cap


def _failure_worker(rank, world):
    from plonky2_b200 import distributed as D

    placement = D.Placement(rank, world, None)
    try:
        placement._agree_on_failure(ValueError("rank 1's own failure") if rank == 1 else None, None, RuntimeError,
                                    "rank %d failed")
        return rank, None
    except Exception as e:
        return rank, "%s: %s" % (type(e).__name__, e)


def test_failure_on_one_rank_raises_on_every_rank():
    """Placement._agree_on_failure over two gloo ranks, rank 1 failing: rank 1 raises its own exception, rank 0 the
    agreed error naming rank 1, and neither waits for the other."""
    res = spawn_ranks(_failure_worker, 2, timeout=180)
    assert res == [(0, "RuntimeError: rank 1 failed"), (1, "ValueError: rank 1's own failure")]


@pytest.mark.parametrize("num_polys,world", [(234, 8), (234, 4), (234, 2), (64, 8), (5, 4), (3, 8), (16, 1), (300, 2)])
def test_chunk_layout_tiles_the_coefficient_matrix(num_polys, world):
    """PipelinedCommitter's layout contract (SURVEY 8e, column axis): chunk c = Wc consecutive global columns, rank r's
    sub-block = pc consecutive columns at c*Wc + r*pc, so that (a) the fused iNTT stores / the per-chunk all-gather of
    the ranks' (pc, n) blocks in rank order IS rows [c*Wc, (c+1)*Wc) of the coefficient matrix, (b) every column is
    transformed by exactly one rank, (c) gathered chunks are contiguous column ranges for gl_commit_add_columns."""
    from plonky2_b200 import distributed as D

    pc, wc, K = D.chunk_layout(num_polys, world)
    assert wc == pc * world and K * wc >= num_polys > (K - 1) * wc
    covered = []
    for c in range(K):
        for rank in range(world):
            b0, cnt = D.chunk_columns(num_polys, rank, world, c)
            assert 0 <= cnt <= pc and b0 == min(c * wc + rank * pc, num_polys) and b0 + cnt <= num_polys
            covered += list(range(b0, b0 + cnt))
    assert covered == list(range(num_polys))


def _pipeline_worker(rank, world, num_polys, n):
    """The committer's data movement with gloo standing in for NCCL: per chunk every rank contributes its (pc, n)
    block and the all-gather lands in rows [c*Wc, (c+1)*Wc) of the matrix."""
    import torch
    import torch.distributed as dist

    from plonky2_b200 import distributed as D

    pc, wc, K = D.chunk_layout(num_polys, world)
    full = torch.arange(num_polys * n, dtype=torch.int64).reshape(num_polys, n) * 3 + 1  # "coefficients" of column b
    coeffs = torch.zeros((K * wc, n), dtype=torch.int64)
    for c in range(K):
        b0, cnt = D.chunk_columns(num_polys, rank, world, c)
        stage = torch.full((pc, n), -1, dtype=torch.int64)
        stage[:cnt] = full[b0:b0 + cnt]
        dist.all_gather_into_tensor(coeffs[c * wc:(c + 1) * wc], stage)
    return rank, bool(torch.equal(coeffs[:num_polys], full))


@pytest.mark.parametrize("num_polys", [11, 70])
def test_pipelined_gather_layout_two_ranks_gloo(num_polys):
    res = spawn_ranks(_pipeline_worker, 2, (num_polys, 8), timeout=120)
    assert res == [(0, True), (1, True)]
