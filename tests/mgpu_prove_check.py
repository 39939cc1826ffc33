"""Multi-rank end-to-end check (run under torchrun, one rank per GPU):
sharded commitments -> all-gather of caps -> prove_openings with routed initial-tree openings, and the pipelined
column-sharded commitment over every coefficient transport. Rank 0 compares caps and the proof bytes with the CPU
oracle. With fewer GPUs than ranks (a single-GPU machine) all ranks share GPU 0 and exchange through gloo, since NCCL
refuses two ranks on one device; the NVLink transports need a GPU per rank and are then left out.
Launched by tests/test_gpu_parity.py, or by hand:  python -m torch.distributed.run --nproc-per-node 2 ... this file
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np
import torch

import plonky2_b200 as pb
from conftest import synth
from plonky2_b200 import distributed as D
from ranks import finish_rank, init_rank


def main():
    rank, world, dev, ctx = init_rank()
    shared = torch.cuda.device_count() < world
    log_n, r, h = 10, 3, 4
    Bs = [7, 5, 3]
    vals = [synth(0x60 + i, (B, 1 << log_n)) for i, B in enumerate(Bs)]
    commits = [pb.PolynomialBatch.from_values(v, r, False, h, ctx=ctx, shard=(rank, world)) for v in vals]
    caps = [D.gather_cap(c.merkle_tree.cap, device=dev) for c in commits]
    ch = pb.Challenger()
    for cap in caps:
        ch.observe_cap(cap)
    zeta = (1234567, 7654321)
    gz = pb.field.ext_mul(zeta, (pb.field.primitive_root_of_unity(log_n), 0))
    allp = [pb.FriPolynomialInfo(o, i) for o, B in enumerate(Bs) for i in range(B)]
    inst = pb.FriInstanceInfo([pb.FriOracleInfo(B, False) for B in Bs],
                              [pb.FriBatchInfo(zeta, allp), pb.FriBatchInfo(gz, [pb.FriPolynomialInfo(2, 0)])])
    params = pb.FriParams(pb.FriConfig(r, h, 8, ("Fixed", [4, 2]), 12), False, log_n, [4, 2])
    proof = D.prove_openings_sharded(inst, commits, ch, params)
    failures = []
    # column-sharded iNTT whose stores are the coefficient all-gather + row-block sharded LDE/Merkle (PipelinedCommitter)
    import ctypes as C
    from plonky2_b200 import _native as N_
    Bc, lg = 70, 12  # two chunks of 64 columns, the second one partial
    vals_c = synth(0x77, (Bc, 1 << lg))
    # torch copies / NCCL and the library must share ONE stream: make the context on a torch stream
    tstream = torch.cuda.Stream(device=dev)
    ctx2 = pb.Context(dev.index, stream=tstream.cuda_stream)
    with torch.cuda.stream(tstream):
        host = torch.from_numpy(vals_c.view(np.int64).copy()).pin_memory()
        caps_c, transports = [], []
        for transport in (("nccl",) if shared else ("auto", "fused", "p2p", "nccl")):
            try:
                cm = D.PipelinedCommitter(ctx2, Bc, lg, 2, 3, rank, world, dev, transport=transport)
            except Exception as e:  # a transport this system lacks (no multicast / no peer mappings) is reported, not fatal
                transports.append("%s unavailable: %r" % (transport, e))
                continue
            transports.append(cm.transport + (" (%s)" % cm.transport_note if cm.transport_note else ""))
            for from_host in (True, False, True):  # back-to-back commitments reuse the matrix: exercises the hand-over barriers
                src = host if from_host else host.to(dev)
                hnd = cm.commit(src, from_host=from_host)
                lcap = np.empty(((1 << 3) // world, 4), dtype=np.uint64)
                N_.check(N_.lib().gl_commit_cap(hnd, N_.np_ptr(lcap), N_.MEM_HOST), ctx2.h)
                N_.lib().gl_commit_destroy(hnd)
                caps_c.append(lcap)
    torch.cuda.synchronize(dev)
    full_caps_c = [D.gather_cap(lc, device=dev) for lc in caps_c]
    if rank == 0:
        import oracle_lib

        ocommits = [oracle_lib.Commit(v, r, h) for v in vals]
        for k, (cap, o) in enumerate(zip(caps, ocommits)):
            if not np.array_equal(cap.hashes, o.cap):
                failures.append("commitment %d: the gathered cap differs from the oracle's" % k)
        och = oracle_lib.Challenger()
        for o in ocommits:
            och.observe_cap(o.cap)
        obatches = [(b.point, [(p.oracle_index, p.polynomial_index) for p in b.polynomials]) for b in inst.batches]
        oproof = oracle_lib.prove_openings(ocommits, obatches, och, oracle_lib.make_params(r, h, 8, 12, [4, 2]))
        if proof.to_bytes() != oproof:
            failures.append("prove_openings_sharded: the proof bytes differ from the oracle's")
        want = oracle_lib.Commit(vals_c, 2, 3).cap
        if not full_caps_c:
            failures.append("PipelinedCommitter: no coefficient transport ran")
        for k, fc in enumerate(full_caps_c):
            if not np.array_equal(fc.hashes, want):
                failures.append("PipelinedCommitter commitment %d: the gathered cap differs from the oracle's" % k)
    finish_rank("MGPU_PROVE_CHECK", failures, transports=transports)


if __name__ == "__main__":
    main()
