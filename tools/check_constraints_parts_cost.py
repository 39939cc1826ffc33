"""What check_constraints costs when H is checked in G parts (stark.check_constraints / plonk.check_constraints with
parts=G, gl_*_check_rows_part), for G = 1, 2, 4, 8, 16, on the two workloads of tools/check_constraints_cost.py:

  stark  the 64-column x 2^24 FibonacciPairsStark of tools/stark_prove_cost.py (standard_fast_config), trace
         commitment resident (the check reads the coefficients alone, whatever the handle);
  plonk  tests/plonk_large.LargeCircuit at 2^18 gates, its constants / sigmas, wires and Z / partial-product / lookup
         commitments made as prove_with_witness makes them.

For each G: the median of --reps checks after --warmup (host clock; every part ends in a synchronising read-back), and
the library's device high-water mark during one check above what was in use before it (Context.device_bytes, so above
the handles). G = 1 is the whole check (gl_*_check_rows). The reports of every G must equal G = 1's.

Then, unless --over-log-n is 0, LargeCircuit at 2^22 gates proved with lde_blocks=16 (a shape whose resident
commitments exceed the card) without and with check_constraints=True, which checks it in 16 parts: proof time, the
library's high-water mark, and whether the two proofs' bytes are equal.

Prints one JSON line with the GPU's name, power limit and maximum SM clock.

Usage: python tools/check_constraints_parts_cost.py [--stark-log-n 24] [--plonk-log-n 18] [--over-log-n 22] [--reps 3]
       [--warmup 1] [--parts 1,2,4,8,16]"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
MIB, GIB = 1 << 20, 1 << 30


def _sweep(ctx, check, parts, reps, warmup):
    """{"G=g": {check_ms, high_water_mib, same_report}} for check(parts=g) -> ConstraintReport."""
    out, first = {}, None
    for G in parts:
        for _ in range(warmup):
            check(G)
        times = []
        for _ in range(reps):
            t0 = time.perf_counter()
            check(G)
            times.append((time.perf_counter() - t0) * 1e3)
        in_use, _ = ctx.device_bytes(reset_high=True)
        report = check(G)
        high = ctx.device_bytes()[1] - in_use
        key = (report.failures, report.entries)
        first = key if first is None else first
        out["G=%d" % G] = {"check_ms": round(statistics.median(times), 2), "check_ms_all": [round(t, 2) for t in times],
                           "high_water_mib": round(high / MIB, 1), "same_report": key == first}
    return out


def stark_case(log_n, parts, reps, warmup):
    import torch

    import plonky2_b200 as pb
    from plonky2_b200 import stark as S
    from stark_prove_cost import FibonacciPairsStark, fibonacci_pairs_trace

    ctx = pb.default_context()
    stark, config = FibonacciPairsStark(), S.StarkConfig.standard_fast_config()
    trace = fibonacci_pairs_trace(log_n)
    torch.cuda.synchronize()
    tc = S._commit_trace(trace, config.fri_config.rate_bits, config.fri_config.cap_height, ctx)
    del trace
    try:
        return {"rows": 1 << log_n, "columns": stark.COLUMNS,
                "runs": _sweep(ctx, lambda G: S.check_constraints(stark, tc, [], parts=G), parts, reps, warmup)}
    finally:
        tc.close()


def plonk_case(log_n, parts, reps, warmup):
    import plonk_circuits as PC
    import plonk_large as PL
    import plonky2_b200 as pb
    from plonky2_b200 import plonk
    from test_gpu_plonk_large import _device_commitments

    ctx = pb.default_context()
    c = PL.large_circuit(log_n)
    betas, gammas, alphas, deltas = PC.challenges(0x6a00, c)
    cs, w, z, _ = _device_commitments(pb, c, (betas, gammas, alphas, deltas))
    try:
        def check(G):
            return plonk.check_constraints(c.common, cs, c.public_inputs_hash, w, z, betas, gammas, deltas, parts=G)

        return {"gates": c.n, "polynomials": sum(b.num_polys for b in (cs, w, z)),
                "runs": _sweep(ctx, check, parts, reps, warmup)}
    finally:
        for b in (cs, w, z):
            b.close()


def over_memory_case(log_n):
    import plonk_large as PL
    import plonky2_b200 as pb
    from plonk_blocked_cost import footprint, prover_data
    from plonky2_b200 import plonk

    ctx = pb.default_context()
    t0 = time.perf_counter()
    c = PL.large_circuit(log_n, luts="range16", public_inputs=[3, 1, 4])
    out = {"shape": "LargeCircuit 2^%d gates, standard_recursion_config, range16 tables, lde_blocks=16" % log_n,
           "host_build_s": round(time.perf_counter() - t0, 1),
           "resident_commitments_gib": round(footprint(c) / GIB, 2)}
    pd = prover_data(pb, c, 16)
    try:
        proofs = {}
        for check in (False, True):
            ctx.device_bytes(reset_high=True)
            t0 = time.perf_counter()
            proofs[check] = plonk.prove_with_witness(pd, c.common, c.wires, c.public_inputs, lde_blocks=16,
                                                     check_constraints=check).to_bytes()
            ctx.synchronize()
            out["with_check" if check else "without_check"] = {
                "prove_ms": round((time.perf_counter() - t0) * 1e3, 2),
                "library_high_water_gib": round(ctx.device_bytes()[1] / GIB, 3)}
        out["same_proof_bytes"] = proofs[False] == proofs[True]
    finally:
        pd.constants_sigmas_commitment.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stark-log-n", type=int, default=24)
    ap.add_argument("--plonk-log-n", type=int, default=18)
    ap.add_argument("--over-log-n", type=int, default=22, help="gates (log2) of the lde_blocks=16 proof; 0 skips it")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--parts", default="1,2,4,8,16")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("check_constraints_parts_cost.py measures on a CUDA device; none is present")
    from stark_prove_cost import gpu_info

    parts = [int(g) for g in args.parts.split(",")]
    out = {"gpu": gpu_info(), "reps": args.reps, "warmup": args.warmup}
    if args.over_log_n:        # first, while the memory pool is empty
        out["over_memory"] = over_memory_case(args.over_log_n)
    out["stark"] = stark_case(args.stark_log_n, parts, args.reps, args.warmup)
    out["plonk"] = plonk_case(args.plonk_log_n, parts, args.reps, args.warmup)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
