"""distributed.prove_with_ctls across ranks (run under torchrun, one rank per GPU): for the three-table CTL system of
tests/test_stark_ctl.py (its CPU table also has a logUp lookup) from host columns and from torch device traces, and for
a variant whose memory table has a logUp lookup of its own, every rank's MultiStarkProof equals
cross_table_lookup.prove_with_ctls's on its own device, table count and every table field for field (proof_diff), and
rank 0 has the restated verifier (tests/stark_twin.py) accept it. Too many ranks for the cap and a wrong trace count
are refused on every rank. With fewer GPUs than ranks all ranks share GPU 0 and exchange through gloo, since NCCL
refuses two ranks on one device. Launched by tests/test_stark_ctl_sharded.py, or by hand:
  python -m torch.distributed.run --standalone --nproc-per-node 2 tests/mgpu_ctl_check.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np


def lookup_system():
    """test_stark_ctl's system with a logUp lookup in the memory table too: three extra columns (looking value, table,
    frequencies) after the six the CTLs read, and the matching traces."""
    from plonky2_b200.lookup import Column, Filter, Lookup
    from test_stark_ctl import CpuTable, LookedTable, MemTable, system_ctls, system_traces
    from plonky2_b200 import stark as S

    class MemWithLookup(MemTable):
        COLUMNS = 9

        def lookups(self):
            return [Lookup([Column.single(6)], Column.single(7), Column.single(8), [Filter.default()])]

    traces, pis = system_traces(log_cpu=9, log_mem=8, log_looked=10, seed=11)
    mem = traces[1]
    nm = mem.shape[1]
    rng = np.random.default_rng(0xC71)
    rv = rng.integers(0, nm, nm).astype(np.uint64)
    extra = np.stack([rv, np.arange(nm, dtype=np.uint64),
                      np.bincount(rv.astype(np.int64), minlength=nm).astype(np.uint64)])
    traces[1] = np.ascontiguousarray(np.concatenate([mem, extra]))
    return ([CpuTable(), MemWithLookup(), LookedTable()], S.StarkConfig.standard_fast_config(), system_ctls(), traces,
            pis)


def main():
    import torch

    import plonky2_b200 as pb
    import stark_twin as T
    from plonky2_b200 import _native as N
    from plonky2_b200 import cross_table_lookup as X
    from plonky2_b200 import distributed as D
    from ranks import finish_rank, init_rank
    from test_stark_ctl import system, system_traces

    rank, _, dev, ctx = init_rank()
    failures = []

    starks, config, ctls = system()
    traces, pis = system_traces(log_cpu=10, log_mem=9, log_looked=11, seed=7)
    device = [torch.from_numpy(np.ascontiguousarray(t).view(np.int64)).to(dev) for t in traces]
    torch.cuda.synchronize(dev)
    cases = [("system_host", starks, config, ctls, traces, pis),
             ("system_device", starks, config, ctls, device, pis),
             ("mem_lookup_host", *lookup_system())]
    proofs = []
    for name, st, cfg, cl, arg, pi in cases:
        got = D.prove_with_ctls(st, cfg, arg, cl, pi, ctx=ctx)
        want = X.prove_with_ctls(st, cfg, arg, cl, pi, ctx=ctx)
        bad = T.proof_diff(got, want)
        if bad:
            failures.append("%s: %s differ" % (name, bad))
        proofs.append((name, st, cfg, cl, got))
    # refusals, on every rank, before any collective
    tiny = type(config)(100, 2, pb.FriConfig(1, 0, 16, ("ConstantArityBits", 4, 5), 84))
    for what, args in (("cap_height 0", (starks, tiny, traces, ctls, pis)),
                       ("trace count", (starks, config, traces[:2], ctls, pis))):
        try:
            D.prove_with_ctls(*args, ctx=ctx)
            failures.append("%s: not refused" % what)
        except N.ShapeError:
            pass
    if rank == 0:
        import oracle_lib

        for name, st, cfg, cl, proof in proofs:
            verdict = T.verify_with_ctls(oracle_lib, st, cfg, cl, proof)
            if verdict is not None:
                failures.append("%s: the restated verifier rejects the proof: %s" % (name, verdict))
    finish_rank("MGPU_CTL_CHECK", failures)


if __name__ == "__main__":
    main()
