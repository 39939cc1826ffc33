"""check_constraints=True on the distributed provers (run under torchrun, one rank per GPU): distributed.prove_stark,
prove_with_ctls and prove_plonk, each rank checking its own part of H (the rows i = rank mod world) and the ranks
merging their reports.
- Holding inputs (FibonacciStark, the lookup RangeCheckStark, the CTL system of tests/test_stark_ctl.py, LargeCircuit
  at 2^13 gates with lookups) give every rank the proof it gives without the flag.
- A broken trace cell, a broken CTL Z value and a broken witness each raise ConstraintError on every rank, with the
  message and report of the single-device prover on the same inputs.
- A NativeError raised by one rank's check raises on every rank, and no rank waits in a collective.
With fewer GPUs than ranks all ranks share GPU 0 and exchange through gloo, since NCCL refuses two ranks on one device.
Launched by tests/test_check_constraints_parts.py, or by hand:
  python -m torch.distributed.run --standalone --nproc-per-node 2 tests/mgpu_check_constraints_check.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np

import plonky2_b200 as pb
from plonky2_b200 import _native as N
from plonky2_b200 import distributed as D
from plonky2_b200 import stark as S
from ranks import finish_rank, init_rank

P = 0xFFFFFFFF00000001
DIGEST = [11, 22, 33, 44]


def error_of(fn):
    """(message, failures, entries) of the ConstraintError fn raises, or the name of what it did instead."""
    try:
        fn()
    except N.ConstraintError as e:
        return str(e), e.report.failures, e.report.entries
    except Exception as e:  # noqa: BLE001 -- reported as a failure of this check
        return "raised %r" % (e,)
    return "did not raise"


def main():
    import stark_twin as T
    from plonky2_b200 import cross_table_lookup as X
    from plonky2_b200 import plonk
    from plonky2_b200.fri import standard_recursion_fri_config
    import plonk_large as PL
    from test_stark_ctl import system, system_traces
    from test_stark_lookups import RangeCheckStark

    rank, world, _, ctx = init_rank()
    config = S.StarkConfig.standard_fast_config()
    failures = []

    # ---- prove_stark
    fib = S.FibonacciStark(1 << 10)
    fib_trace = fib.generate_trace(0, 1)
    fib_pis = [0, 1, int(fib_trace[1, -1])]
    for name, stark, trace, pis in (("fibonacci", fib, fib_trace, fib_pis),
                                    ("range_check", RangeCheckStark(), RangeCheckStark.generate_trace(10), [0])):
        bad = T.proof_diff(D.prove_stark(stark, config, trace, pis, ctx=ctx, check_constraints=True),
                           D.prove_stark(stark, config, trace, pis, ctx=ctx))
        if bad:
            failures.append("prove_stark %s: %s differ with the flag" % (name, bad))
    broken = fib_trace.copy()
    for r in (0, 1, 517, -1):
        broken[1, r] = (int(broken[1, r]) + 1) % P
    want = error_of(lambda: S.prove(fib, config, broken, fib_pis, ctx=ctx, check_constraints=True))
    got = error_of(lambda: D.prove_stark(fib, config, broken, fib_pis, ctx=ctx, check_constraints=True))
    if not isinstance(want, tuple) or got != want:
        failures.append("prove_stark broken trace on rank %d: %r, single device %r" % (rank, got, want))

    # a NativeError from rank 1's check raises on every rank
    real = N.check_rows

    def fails_on_rank_1(*a, **k):
        if rank == 1:
            raise N.NativeError("injected on rank 1")
        return real(*a, **k)
    N.check_rows = fails_on_rank_1
    try:
        D.prove_stark(fib, config, fib_trace, fib_pis, ctx=ctx, check_constraints=True)
        failures.append("a failed check on rank 1 did not raise on rank %d" % rank)
    except N.NativeError as e:
        want_msg = "injected on rank 1" if rank == 1 else "the constraint check failed on rank 1"
        if want_msg not in str(e):
            failures.append("rank %d raised %r" % (rank, e))
    finally:
        N.check_rows = real

    # ---- prove_with_ctls
    starks, ctl_config, ctls = system()
    traces, pis = system_traces()
    got = D.prove_with_ctls(starks, ctl_config, traces, ctls, pis, ctx=ctx, check_constraints=True)
    plain = D.prove_with_ctls(starks, ctl_config, traces, ctls, pis, ctx=ctx)
    bad = T.proof_diff(got, plain)
    if bad:
        failures.append("prove_with_ctls: %s differ with the flag" % bad)
    real_ctl = X.cross_table_lookup_data

    def broken_ctl(*a, **k):                          # the looked table's last CTL Z, one value changed at row 5
        data = real_ctl(*a, **k)
        data[2].auxiliary[-1, 5] = 12345
        return data
    X.cross_table_lookup_data = broken_ctl
    try:
        want = error_of(lambda: X.prove_with_ctls(starks, ctl_config, traces, ctls, pis, ctx=ctx,
                                                  check_constraints=True))
        got = error_of(lambda: D.prove_with_ctls(starks, ctl_config, traces, ctls, pis, ctx=ctx,
                                                 check_constraints=True))
    finally:
        X.cross_table_lookup_data = real_ctl
    if not isinstance(want, tuple) or not want[0].startswith("Constraint failed in LookedTable") or got != want:
        failures.append("prove_with_ctls broken CTL value on rank %d: %r, single device %r" % (rank, got, want))

    # ---- prove_plonk
    c = PL.large_circuit(13, public_inputs=[3, 1, 4])
    cfg, cd = c.config, c.common
    fri_params = standard_recursion_fri_config().fri_params(cd.degree_bits, False)
    whole = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height, ctx=ctx)
    mine = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height, ctx=ctx,
                                          shard=(rank, world))
    try:
        sharded = plonk.ProverOnlyCircuitData(mine, c.sigmas, DIGEST, fri_params)
        single = plonk.ProverOnlyCircuitData(whole, c.sigmas, DIGEST, fri_params)
        got = D.prove_plonk(sharded, cd, c.wires, c.public_inputs, ctx=ctx, check_constraints=True).to_bytes()
        if got != D.prove_plonk(sharded, cd, c.wires, c.public_inputs, ctx=ctx).to_bytes():
            failures.append("prove_plonk: rank %d's bytes differ with the flag" % rank)
        wires = c.wires.copy()
        (row, col) = c.partition()[1][2]
        wires[col, row] = (int(wires[col, row]) + 1) % P          # a copy constraint
        wires[3, 4321] = (int(wires[3, 4321]) + 7) % P              # and whatever gate sits at row 4321
        want = error_of(lambda: plonk.prove_with_witness(single, cd, wires, c.public_inputs, ctx=ctx,
                                                         check_constraints=True))
        got = error_of(lambda: D.prove_plonk(sharded, cd, wires, c.public_inputs, ctx=ctx, check_constraints=True))
        if not isinstance(want, tuple) or got != want:
            failures.append("prove_plonk broken witness on rank %d: %r, single device %r" % (rank, got, want))
    finally:
        whole.close()
        mine.close()

    finish_rank("MGPU_CHECK_CONSTRAINTS", failures)


if __name__ == "__main__":
    main()
