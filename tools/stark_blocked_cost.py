"""What non-resident commitments (stark.prove(..., lde_blocks=G)) cost, at tools/stark_prove_cost.py's shape: 64
Fibonacci-pair columns x 2^24 rows, StarkConfig.standard_fast_config (rate 1/2).

The resident proof, then G = 1, 2, 4, 8, 16 blocks: the median of --reps proofs after --warmup (each ends in a
device synchronise), one proof's phases with a synchronise after each (commitments: trace and quotient; quotient;
openings; FRI, which rebuilds the blocks its queries open), the library's device high-water mark during one proof
(gl_ctx_device_bytes; torch's caching allocator, which holds the trace, is not in it), and whether the proof equals the
resident proof field for field.

Also, and first (while the memory pool is empty), one proof with G = 16 of a shape whose resident footprint, computed from shapes, exceeds the card's total memory:
224 columns x 2^24 rows (the 64 constrained Fibonacci-pair columns and 160 unconstrained copies of them). The resident
proof is never attempted at that size. If the free memory does not cover the blocked footprint, it is skipped with the
reason.

Prints one JSON line with the GPU's name and power limit.

Usage: python tools/stark_blocked_cost.py [--log-n 24] [--reps 3] [--warmup 1]"""
import argparse
import importlib.util
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
GIB = 1 << 30


def _cost_module():
    spec = importlib.util.spec_from_file_location("stark_prove_cost", os.path.join(ROOT, "tools", "stark_prove_cost.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


M = _cost_module()


class WidePairsStark(M.FibonacciPairsStark):
    """FibonacciPairsStark's 64 constrained columns followed by `extra` unconstrained ones (committed and opened)."""

    def __init__(self, extra):
        self.COLUMNS = 2 * M.PAIRS + extra


def phase_times(stark, config, trace, ctx, lde_blocks):
    """One proof with a device synchronise after each phase, timed by wrapping the functions `prove` calls."""
    import plonky2_b200.fri as fri_mod
    import plonky2_b200.proof as proof_mod
    import plonky2_b200.stark as stark_mod

    times = {}
    patches = [(stark_mod, "_commit_trace", "commitments"), (stark_mod, "commit_quotient_polys", "commitments"),
               (stark_mod, "compute_quotient_polys", "quotient"), (proof_mod, "eval_commitments", "openings"),
               (fri_mod, "prove_openings", "fri")]
    saved = []
    for mod, name, label in patches:
        fn = getattr(mod, name)

        def wrapper(*a, _fn=fn, _label=label, **k):
            ctx.synchronize()
            t0 = time.perf_counter()
            r = _fn(*a, **k)
            ctx.synchronize()
            times[_label] = times.get(_label, 0.0) + (time.perf_counter() - t0) * 1e3
            return r

        saved.append((mod, name, fn))
        setattr(mod, name, wrapper)
    try:
        stark_mod.prove(stark, config, trace, [], ctx=ctx, lde_blocks=lde_blocks)
    finally:
        for mod, name, fn in saved:
            setattr(mod, name, fn)
    return {k: round(v, 2) for k, v in times.items()}


def same_proof(a, b):
    pa, pb = a.proof, b.proof
    if not (np.array_equal(pa.trace_cap.hashes, pb.trace_cap.hashes)
            and np.array_equal(pa.quotient_polys_cap.hashes, pb.quotient_polys_cap.hashes)):
        return False
    fa, fb = pa.openings.to_fri_openings(), pb.openings.to_fri_openings()
    return (len(fa) == len(fb) and all(np.array_equal(u, v) for u, v in zip(fa, fb))
            and pa.opening_proof.to_bytes() == pb.opening_proof.to_bytes())


def footprint(columns, quotient_polys, log_n, rate_bits, cap_height, lde_blocks):
    """Device bytes of the proof's commitments, from shapes: coefficients, digests and cap of the trace and quotient
    commitments, plus the whole LDE (resident) or one block of the widest (lde_blocks = G), twice when a block has fewer
    rows than the trace (the folded coefficients beside it). The trace itself, the NTT group scratch and FRI's own trees
    come on top."""
    N = 1 << (log_n + rate_bits)
    words = (columns + quotient_polys) << log_n
    words += 2 * (8 * (N - (1 << cap_height)) + (4 << cap_height))
    if lde_blocks is None:
        words += (columns + quotient_polys) * N
    else:
        words += columns * N // lde_blocks * (2 if N // lde_blocks < 1 << log_n else 1)
    return words * 8


def measure(stark, config, trace, ctx, lde_blocks, reps, warmup):
    from plonky2_b200 import stark as S

    for _ in range(warmup):
        S.prove(stark, config, trace, [], ctx=ctx, lde_blocks=lde_blocks)
    ms = []
    proof = None
    for _ in range(reps):
        ctx.device_bytes(reset_high=True)
        t0 = time.perf_counter()
        proof = S.prove(stark, config, trace, [], ctx=ctx, lde_blocks=lde_blocks)
        ctx.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    _, high = ctx.device_bytes()
    return proof, {"prove_ms_median": round(float(np.median(ms)), 2), "prove_ms": [round(m, 2) for m in ms],
                   "library_high_water_gib": round(high / GIB, 3),
                   "phases_ms_one_proof": phase_times(stark, config, trace, ctx, lde_blocks)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=24)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--blocks", default="1,2,4,8,16")
    ap.add_argument("--wide-extra", type=int, default=160, help="unconstrained columns of the over-memory shape")
    args = ap.parse_args()

    import torch

    import plonky2_b200 as pb
    from plonky2_b200 import stark as S

    ctx = pb.default_context()
    config = S.StarkConfig.standard_fast_config()
    rate_bits, cap_height = config.fri_config.rate_bits, config.fri_config.cap_height
    wide = WidePairsStark(args.wide_extra)
    nq = wide.num_quotient_polys(config)
    resident_bytes = footprint(wide.COLUMNS, nq, args.log_n, rate_bits, cap_height, None)
    blocked_bytes = footprint(wide.COLUMNS, nq, args.log_n, rate_bits, cap_height, 16)
    trace_bytes = wide.COLUMNS << (args.log_n + 3)
    free, total = torch.cuda.mem_get_info()
    over = {"shape": "%d columns x 2^%d rows, G = 16" % (wide.COLUMNS, args.log_n),
            "resident_commitments_gib": round(resident_bytes / GIB, 2), "card_total_gib": round(total / GIB, 2),
            "blocked_commitments_gib": round(blocked_bytes / GIB, 2), "trace_gib": round(trace_bytes / GIB, 2),
            "free_gib": round(free / GIB, 2)}
    need = blocked_bytes + trace_bytes + 4 * GIB  # and the NTT group scratch, FRI's trees and staging
    if resident_bytes <= total:
        over["skipped"] = "the resident footprint fits the card; raise --wide-extra"
    elif need > free:
        over["skipped"] = "free memory %.1f GiB does not cover the blocked footprint %.1f GiB" % (free / GIB, need / GIB)
    else:
        base = M.fibonacci_pairs_trace(args.log_n)
        wtrace = torch.empty((wide.COLUMNS, base.shape[1]), dtype=base.dtype, device=base.device)
        for c in range(0, wide.COLUMNS, base.shape[0]):
            wtrace[c:c + base.shape[0]] = base[:wide.COLUMNS - c]
        del base
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        ctx.device_bytes(reset_high=True)
        t0 = time.perf_counter()
        S.prove(wide, config, wtrace, [], ctx=ctx, lde_blocks=16)
        ctx.synchronize()
        over["prove_ms"] = round((time.perf_counter() - t0) * 1e3, 2)
        over["library_high_water_gib"] = round(ctx.device_bytes()[1] / GIB, 3)
        del wtrace
        torch.cuda.empty_cache()

    stark = M.FibonacciPairsStark()
    trace = M.fibonacci_pairs_trace(args.log_n)
    torch.cuda.synchronize()
    resident, row = measure(stark, config, trace, ctx, None, args.reps, args.warmup)
    runs = {"resident": row}
    for G in [int(g) for g in args.blocks.split(",")]:
        proof, row = measure(stark, config, trace, ctx, G, args.reps, args.warmup)
        row["equals_resident_proof"] = same_proof(proof, resident)
        runs["G=%d" % G] = row

    print(json.dumps({"gpu": M.gpu_info(), "workload": "starky prove, lde_blocks: FibonacciPairsStark, 64 columns x 2^%d "
                                                      "rows, standard_fast_config" % args.log_n,
                      "reps": args.reps, "warmup": args.warmup, "runs": runs, "over_memory": over}))


if __name__ == "__main__":
    main()
