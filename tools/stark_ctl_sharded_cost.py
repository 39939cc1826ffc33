"""distributed.prove_with_ctls at tools/stark_ctl_cost.py's system: three tables of 2^22 x 6, 2^21 x 3 and 2^20 x 3
columns (--log-n sets the largest) tied by one CTL, StarkConfig.standard_fast_config (rate 1/2, cap height 4).

Under torchrun with one GPU per rank (NCCL):
    python -m torch.distributed.run --standalone --nproc-per-node G tools/stark_ctl_sharded_cost.py [--log-n 22]
prints one JSON line from rank 0: the card's name, power limit and maximum SM clock, the world size, the median over
--reps of the slowest rank's prove_with_ctls time (each rep starts behind a barrier and ends in a device synchronise) and
cross_table_lookup.prove_with_ctls's median on rank 0's GPU alone. With fewer GPUs than ranks it refuses: ranks sharing
a GPU measure contention, not scaling.

Without torchrun, --per-shard G times one shard's device work for every g < G on one GPU, one shard after another,
summed over the three tables: the trace shard commitment, the auxiliary shard commitment (CTL helper and Z columns
computed once beforehand, as every rank computes them), the shard quotient (gl_stark_quotient_shard), then -- after
interpolating each table's gathered values once (gl_stark_quotient_from_shards) -- the quotient shard commitment and
the shard's openings (gl_openings_shard: every request of StarkOpeningSet.new). The result is labelled "per-shard device
time, no communication". --per-shard 1 is the same steps on one device; its openings are gl_openings' launches. Neither
mode is part of bench.py."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from stark_ctl_cost import system  # noqa: E402
from stark_prove_cost import gpu_info  # noqa: E402

WORKLOAD = ("prove_with_ctls: 3 tables of 2^%d x 6, 2^%d x 3, 2^%d x 3 columns, one CTL (2 + 1 looking entries of "
            "pairs), standard_fast_config")


def _device_traces(host, dev):
    import torch

    traces = [torch.from_numpy(t.view(np.int64)).to(dev) for t in host]
    torch.cuda.synchronize(dev)
    return traces


def distributed_run(args):
    import torch
    import torch.distributed as dist

    import plonky2_b200 as pb
    from plonky2_b200 import distributed as D
    from plonky2_b200 import stark as S
    from plonky2_b200.cross_table_lookup import prove_with_ctls

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
    config = S.StarkConfig.standard_fast_config()
    starks, ctls, host = system(args.log_n)
    traces = _device_traces(host, dev)
    pis = [[]] * len(starks)

    def one():
        dist.barrier()
        t0 = time.perf_counter()
        D.prove_with_ctls(starks, config, traces, ctls, pis, ctx=ctx)
        ctx.synchronize()
        t = torch.tensor([(time.perf_counter() - t0) * 1e3], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    for _ in range(args.warmup):
        one()
    ms = [one() for _ in range(args.reps)]
    if rank == 0:
        for _ in range(args.warmup):
            prove_with_ctls(starks, config, traces, ctls, pis, ctx=ctx)
        single = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            prove_with_ctls(starks, config, traces, ctls, pis, ctx=ctx)
            ctx.synchronize()
            single.append((time.perf_counter() - t0) * 1e3)
        print(json.dumps({"gpu": gpu_info(), "workload": WORKLOAD % (args.log_n, args.log_n - 1, args.log_n - 2),
                          "world": world, "backend": "nccl",
                          "prove_with_ctls_ms_median": round(float(np.median(ms)), 2),
                          "prove_with_ctls_ms": [round(m, 2) for m in ms],
                          "one_device_prove_ms_median": round(float(np.median(single)), 2),
                          "reps": args.reps, "warmup": args.warmup}))
    dist.barrier()
    dist.destroy_process_group()


def per_shard_run(args):
    import torch

    import plonky2_b200 as pb
    from plonky2_b200 import _native as N
    from plonky2_b200 import cross_table_lookup as X
    from plonky2_b200 import field as F
    from plonky2_b200 import stark as S
    from plonky2_b200.lookup import GrandProductChallenge
    from conftest import synth

    G = args.per_shard
    ctx = pb.default_context()
    dev = torch.device("cuda", ctx.device)
    config = S.StarkConfig.standard_fast_config()
    rate_bits, cap_height = config.fri_config.rate_bits, config.fri_config.cap_height
    starks, ctls, host = system(args.log_n)
    traces = _device_traces(host, dev)
    r = [int(v) for v in synth(0x5C8, (2 * config.num_challenges + config.num_challenges + 2,))]
    challenges = [GrandProductChallenge(r[2 * k], r[2 * k + 1]) for k in range(config.num_challenges)]
    alphas = r[2 * config.num_challenges:2 * config.num_challenges + config.num_challenges]
    zeta = (r[-2], r[-1])
    max_degree = X.check_ctl_shapes(starks, ctls, config.num_challenges)
    ctl_data = X.cross_table_lookup_data(traces, ctls, challenges, max_degree, ctx)
    tables = []
    for i, (stark, d) in enumerate(zip(starks, ctl_data)):
        log_n = F.log2_strict(traces[i].shape[1])
        qdf = stark.quotient_degree_factor()
        size = (1 << log_n) << (qdf - 1).bit_length()
        tables.append(dict(stark=stark, log_n=log_n, qdf=qdf, aux=d.auxiliary, ctl_vars=X.ctl_shape_vars(d),
                           values=torch.empty((G, len(alphas), size // G), dtype=torch.int64, device=dev),
                           g_zeta=F.ext_mul((F.primitive_root_of_unity(log_n), 0), zeta),
                           num_ctl_zs=len(d.zs_columns)))
    ctx.synchronize()

    def timed(fn):
        ctx.synchronize()
        t0 = time.perf_counter()
        out = fn()
        ctx.synchronize()
        return out, (time.perf_counter() - t0) * 1e3

    def first_steps(g, t):
        """Trace and auxiliary shard commitments and the shard quotient of table t: (commitments, times)."""
        tc, t_trace = timed(lambda: S._commit_trace(traces[t["i"]], rate_bits, cap_height, ctx, shard=(g, G)))
        ac, t_aux = timed(lambda: S.commit_auxiliary_polys(t["aux"], rate_bits, cap_height, ctx, shard=(g, G)))
        b, consts, al = S.quotient_program(t["stark"], [], alphas, ac, None, t["ctl_vars"])
        _, t_q = timed(lambda: N.check(N.lib().gl_stark_quotient_shard(
            ctx.h, tc.h, ac.h, b.program(), len(b.instrs), N.np_ptr(consts) if len(consts) else None, len(consts),
            N.np_ptr(al), len(al), t["qdf"], N.vp(t["values"][g].data_ptr())), ctx.h))
        return (tc, ac), (t_trace, t_aux, t_q)

    def openings(t, tc, ac, qc, g):
        """Every request of StarkOpeningSet.new for a table with CTLs, shard g of G."""
        reqs = [(tc, 0), (tc, 1), (ac, 0), (ac, 1), (qc, 0), (ac, 2)]
        points = np.array([zeta, t["g_zeta"], (1, 0)], dtype=np.uint64).reshape(-1)
        handles = (N.vp * len(reqs))(*[c.h for c, _ in reqs])
        pidx = np.array([p for _, p in reqs], dtype=np.uint32)
        out = np.empty((sum(c.num_polys for c, _ in reqs), 2), dtype=np.uint64)
        N.check(N.lib().gl_openings_shard(ctx.h, handles, pidx.ctypes.data_as(N.u32p), len(reqs), N.np_ptr(points), 3,
                                          g, G, N.np_ptr(out), N.MEM_HOST), ctx.h)
        return out

    for i, t in enumerate(tables):
        t["i"] = i
    for _ in range(args.warmup):
        for t in tables:
            cs, _ = first_steps(0, t)
            for c in cs:
                c.close()
    steps = ("trace_commitment_ms", "auxiliary_commitment_ms", "shard_quotient_ms", "quotient_commitment_ms",
             "openings_ms")
    shards = [dict(g=g, **{k: 0.0 for k in steps}) for g in range(G)]
    held = {}
    for s in shards:
        for t in tables:
            held[(s["g"], t["i"])], times = first_steps(s["g"], t)
            for k, v in zip(steps[:3], times):
                s[k] += v
    t_from = 0.0
    for t in tables:
        t["quotient"] = torch.empty((len(alphas), t["values"].shape[2] * G), dtype=torch.int64, device=dev)
        _, ms = timed(lambda: N.check(N.lib().gl_stark_quotient_from_shards(
            ctx.h, N.vp(t["values"].data_ptr()), G, len(alphas), t["log_n"], t["qdf"], N.vp(t["quotient"].data_ptr())),
            ctx.h))
        t_from += ms
    if args.warmup:  # the openings' first launches
        tc, ac = held[(0, 0)]
        qc = S.commit_quotient_polys(tables[0]["stark"], tables[0]["quotient"], tables[0]["log_n"], rate_bits,
                                     cap_height, ctx, shard=(0, G))
        openings(tables[0], tc, ac, qc, 0)
        qc.close()
    for s in shards:
        for t in tables:
            tc, ac = held.pop((s["g"], t["i"]))
            qc, ms = timed(lambda: S.commit_quotient_polys(t["stark"], t["quotient"], t["log_n"], rate_bits, cap_height,
                                                           ctx, shard=(s["g"], G)))
            s["quotient_commitment_ms"] += ms
            _, ms = timed(lambda: openings(t, tc, ac, qc, s["g"]))
            s["openings_ms"] += ms
            for c in (tc, ac, qc):
                c.close()
    for s in shards:
        for k in steps:
            s[k] = round(s[k], 2)
    print(json.dumps({"gpu": gpu_info(), "workload": WORKLOAD % (args.log_n, args.log_n - 1, args.log_n - 2),
                      "label": "per-shard device time, no communication", "shards": G, "per_shard": shards,
                      "slowest_shard_ms": {k: max(s[k] for s in shards) for k in steps},
                      "from_shards_ms (every rank)": round(t_from, 2), "warmup": args.warmup}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=22)
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
