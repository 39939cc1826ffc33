"""distributed.prove_stark across ranks (run under torchrun, one rank per GPU): for FibonacciStark and the lookup
RangeCheckStark of tests/test_stark_lookups.py at 2^12 - 2^14 rows in standard_fast_config, from host columns and from
a torch device trace, every rank's proof equals stark.prove's on its own device field for field (proof_diff) and
rank 0 has the restated verifier (tests/stark_twin.py) accept it; a verifier circuit's FRI shape passes through; too
many ranks for the cap and a Stark with CTLs are refused on every rank. With fewer GPUs than ranks all ranks share
GPU 0 and exchange through gloo, since NCCL refuses two ranks on one device. Launched by
tests/test_gpu_stark_sharded.py, or by hand:
  python -m torch.distributed.run --standalone --nproc-per-node 2 tests/mgpu_stark_check.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np
import torch

import plonky2_b200 as pb
import stark_twin as T
from plonky2_b200 import _native as N
from plonky2_b200 import distributed as D
from plonky2_b200 import stark as S
from ranks import finish_rank, init_rank


class _CtlStark(S.FibonacciStark):
    def requires_ctls(self):
        return True


def main():
    from test_stark_lookups import RangeCheckStark

    rank, _, dev, ctx = init_rank()
    config = S.StarkConfig.standard_fast_config()
    failures = []

    def fib(log_n):
        stark = S.FibonacciStark(1 << log_n)
        trace = stark.generate_trace(0, 1)
        return stark, trace, [0, 1, int(trace[1, -1])]

    cases = [("fibonacci_12", *fib(12), "host"), ("fibonacci_14", *fib(14), "device"),
             ("range_check_12", RangeCheckStark(), RangeCheckStark.generate_trace(12), [0], "host"),
             ("range_check_13", RangeCheckStark(), RangeCheckStark.generate_trace(13), [0], "device"),
             ("range_check_14", RangeCheckStark(), RangeCheckStark.generate_trace(14), [0], "host")]
    proofs = []
    for name, stark, trace, pi, source in cases:
        arg = trace
        if source == "device":
            arg = torch.from_numpy(np.ascontiguousarray(trace).view(np.int64)).to(dev)
            torch.cuda.synchronize(dev)
        got = D.prove_stark(stark, config, arg, pi, ctx=ctx)
        want = S.prove(stark, config, arg, pi, ctx=ctx)
        bad = T.proof_diff(got, want)
        if bad:
            failures.append("%s: %s differ" % (name, bad))
        proofs.append((name, stark, got))
    # a verifier circuit's FRI shape (zero caps and coefficients observed): the same transcript on every path
    stark, trace, pi = fib(12)
    vp = config.fri_params(14)
    bad = T.proof_diff(D.prove_stark(stark, config, trace, pi, verifier_circuit_fri_params=vp, ctx=ctx),
                       S.prove(stark, config, trace, pi, verifier_circuit_fri_params=vp, ctx=ctx))
    if bad:
        failures.append("verifier_circuit_fri_params: %s differ" % bad)
    # refusals, on every rank, before any collective
    tiny = S.StarkConfig(100, 2, pb.FriConfig(1, 0, 16, ("ConstantArityBits", 4, 5), 84))
    for what, st, cfg in (("cap_height 0", stark, tiny), ("CTLs", _CtlStark(1 << 12), config)):
        try:
            D.prove_stark(st, cfg, trace, pi, ctx=ctx)
            failures.append("%s: not refused" % what)
        except N.ShapeError:
            pass
    if rank == 0:
        import oracle_lib

        for name, stark, proof in proofs:
            verdict = T.verify(oracle_lib, stark, config, proof)
            if verdict is not None:
                failures.append("%s: the restated verifier rejects the proof: %s" % (name, verdict))
    finish_rank("MGPU_STARK_CHECK", failures)


if __name__ == "__main__":
    main()
