"""distributed.prove_stark at BASELINE config 5's shape: FibonacciPairsStark (tools/stark_prove_cost.py; 64 columns of
32 Fibonacci pairs) at 2^24 rows, StarkConfig.standard_fast_config (rate 1/2, cap height 4).

Under torchrun with one GPU per rank (NCCL):
    python -m torch.distributed.run --standalone --nproc-per-node G tools/stark_prove_sharded_cost.py [--log-n 24]
prints one JSON line from rank 0: the card's name, power limit and maximum SM clock, the world size, the median over
--reps of the slowest rank's prove_stark time (each rep starts behind a barrier and ends in a device synchronise), one
proof's per-phase times on rank 0 (measured in a separate proof, with a synchronise after each phase; "cap_gathers" is
the cap all-gathers, "quotient" includes the value all-gather), and stark.prove's median on rank 0's GPU alone. With
fewer GPUs than ranks it refuses: ranks sharing a GPU measure contention, not scaling.

Without torchrun, --per-shard G times one shard's device work for every g < G on one GPU, one after another -- the trace
shard commitment, the shard quotient (gl_stark_quotient_shard), then, after interpolating the gathered values once
(gl_stark_quotient_from_shards), the quotient shard commitment -- and labels the result "per-shard device time, no
communication". --per-shard 1 is the same steps on one device. Neither mode is part of bench.py."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from stark_prove_cost import FibonacciPairsStark, fibonacci_pairs_trace, gpu_info  # noqa: E402

WORKLOAD = "starky prove: FibonacciPairsStark, 64 columns x 2^%d rows, standard_fast_config"


def _timed_phases(ctx):
    """Wrap the functions prove_stark calls so that each records its time after a device synchronise. Returns (times,
    restore)."""
    import plonky2_b200.distributed as dist_mod
    import plonky2_b200.fri as fri_mod
    import plonky2_b200.proof as proof_mod
    import plonky2_b200.stark as stark_mod

    times = {}
    patches = [(stark_mod, "_commit_trace", "trace_commitment"), (dist_mod.Placement, "cap", "cap_gathers"),
               (stark_mod, "_bind_constraints", "binding_step"), (stark_mod, "compute_quotient_polys", "quotient"),
               (stark_mod, "commit_quotient_polys", "quotient_commitment"), (proof_mod, "eval_commitments", "openings"),
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

    def restore():
        for mod, name, fn in saved:
            setattr(mod, name, fn)
    return times, restore


def distributed_run(args):
    import torch
    import torch.distributed as dist

    import plonky2_b200 as pb
    from plonky2_b200 import distributed as D
    from plonky2_b200 import stark as S

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    if torch.cuda.device_count() < world:
        if rank == 0:
            print("refusing to report a scaling number: %d ranks on %d GPU(s); ranks sharing a GPU measure contention. "
                  "Run with one GPU per rank, or without torchrun as --per-shard %d (per-shard device time, no "
                  "communication)." % (world, torch.cuda.device_count(), world), file=sys.stderr)
        sys.exit(2)
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    ctx = pb.default_context(local)
    stark, config = FibonacciPairsStark(), S.StarkConfig.standard_fast_config()
    trace = fibonacci_pairs_trace(args.log_n, device=dev)
    torch.cuda.synchronize(dev)

    def one():
        dist.barrier()
        t0 = time.perf_counter()
        D.prove_stark(stark, config, trace, [], ctx=ctx)
        ctx.synchronize()
        t = torch.tensor([(time.perf_counter() - t0) * 1e3], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    for _ in range(args.warmup):
        one()
    ms = [one() for _ in range(args.reps)]
    times, restore = _timed_phases(ctx)
    try:
        one()
    finally:
        restore()
    single = None
    if rank == 0:
        for _ in range(args.warmup):
            S.prove(stark, config, trace, [], ctx=ctx)
        single = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            S.prove(stark, config, trace, [], ctx=ctx)
            ctx.synchronize()
            single.append((time.perf_counter() - t0) * 1e3)
        print(json.dumps({"gpu": gpu_info(), "workload": WORKLOAD % args.log_n, "world": world, "backend": "nccl",
                          "prove_stark_ms_median": round(float(np.median(ms)), 2), "prove_stark_ms": [round(m, 2) for m in ms],
                          "phases_ms_rank0_one_proof": {k: round(v, 2) for k, v in times.items()},
                          "one_device_prove_ms_median": round(float(np.median(single)), 2),
                          "reps": args.reps, "warmup": args.warmup}))
    dist.barrier()
    dist.destroy_process_group()


def per_shard_run(args):
    import torch

    import plonky2_b200 as pb
    from plonky2_b200 import _native as N
    from plonky2_b200 import stark as S
    from conftest import synth

    G = args.per_shard
    ctx = pb.default_context()
    stark, config = FibonacciPairsStark(), S.StarkConfig.standard_fast_config()
    rate_bits, cap_height = config.fri_config.rate_bits, config.fri_config.cap_height
    trace = fibonacci_pairs_trace(args.log_n)
    alphas = [int(v) for v in synth(0x5D0, (config.num_challenges,))]
    b, consts, al = S.quotient_program(stark, [], alphas)
    qdf = stark.quotient_degree_factor()
    size = (1 << args.log_n) << (qdf - 1).bit_length()
    values = torch.empty((G, len(al), size // G), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()     # the trace generator's kernels run on torch's stream, not the context's

    def timed(fn):
        ctx.synchronize()
        t0 = time.perf_counter()
        r = fn()
        ctx.synchronize()
        return r, (time.perf_counter() - t0) * 1e3

    def trace_and_quotient(g):
        tc, t_commit = timed(lambda: S._commit_trace(trace, rate_bits, cap_height, ctx, shard=(g, G)))
        try:
            _, t_q = timed(lambda: N.check(N.lib().gl_stark_quotient_shard(
                ctx.h, tc.h, None, b.program(), len(b.instrs), N.np_ptr(consts) if len(consts) else None, len(consts),
                N.np_ptr(al), len(al), qdf, N.vp(values[g].data_ptr())), ctx.h))
        finally:
            tc.close()
        return t_commit, t_q

    for _ in range(args.warmup):
        trace_and_quotient(0)
    shards = [dict(g=g) for g in range(G)]
    for s in shards:
        s["trace_commitment_ms"], s["shard_quotient_ms"] = (round(v, 2) for v in trace_and_quotient(s["g"]))
    quotient = torch.empty((len(al), size), dtype=torch.int64, device="cuda")
    _, t_from = timed(lambda: N.check(N.lib().gl_stark_quotient_from_shards(
        ctx.h, N.vp(values.data_ptr()), G, len(al), args.log_n, qdf, N.vp(quotient.data_ptr())), ctx.h))
    for s in shards:
        qc, t = timed(lambda: S.commit_quotient_polys(stark, quotient, args.log_n, rate_bits, cap_height, ctx,
                                                      shard=(s["g"], G)))
        qc.close()
        s["quotient_commitment_ms"] = round(t, 2)
    steps = ("trace_commitment_ms", "shard_quotient_ms", "quotient_commitment_ms")
    print(json.dumps({"gpu": gpu_info(), "workload": WORKLOAD % args.log_n,
                      "label": "per-shard device time, no communication", "shards": G,
                      "per_shard": shards, "slowest_shard_ms": {k: max(s[k] for s in shards) for k in steps},
                      "from_shards_ms (every rank)": round(t_from, 2), "warmup": args.warmup}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=24)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--per-shard", type=int, default=None, metavar="G",
                    help="time one shard's device work for each g < G on one GPU (no torchrun)")
    args = ap.parse_args()
    if args.per_shard is not None:
        if "WORLD_SIZE" in os.environ:
            ap.error("--per-shard runs in one process, without torchrun")
        per_shard_run(args)
    elif "WORLD_SIZE" in os.environ:
        distributed_run(args)
    else:
        ap.error("run under torchrun with one GPU per rank, or with --per-shard G")


if __name__ == "__main__":
    main()
