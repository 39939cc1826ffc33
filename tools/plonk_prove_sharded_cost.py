"""distributed.prove_plonk on a circuit of the standard recursion config (135 wires, 80 routed, rate 3, quotient degree
factor 8, cap height 4): tests/plonk_large.LargeCircuit at 2^--log-n gates (default 18) with the 2^16-entry range table
and a small table.

Under torchrun with one GPU per rank (NCCL):
    python -m torch.distributed.run --standalone --nproc-per-node G tools/plonk_prove_sharded_cost.py [--log-n 18]
prints one JSON line from rank 0: the card's name, power limit and maximum SM clock, the world size, the median over
--reps of the slowest rank's prove_plonk time (each rep starts behind a barrier and ends in a device synchronise), and
prove_with_witness's median on rank 0's GPU alone. With fewer GPUs than ranks it refuses: ranks sharing a GPU measure
contention, not scaling.

Without torchrun, --per-shard G times one shard's device work for every g < G on one GPU, one after another -- the
wires and Z / partial-product (+ lookup) shard commitments, the shard quotient (gl_plonk_quotient_shard), then, after
interpolating the gathered values once (gl_stark_quotient_from_shards), the quotient shard commitment -- and labels the
result "per-shard device time, no communication". The Z columns themselves are computed once, over all rows, as every
rank computes them. --per-shard 1 is the same steps on one device. Neither mode is part of bench.py."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from stark_prove_cost import gpu_info  # noqa: E402

WORKLOAD = "plonky2 prove: LargeCircuit, 2^%d gates, standard_recursion_config, 2^16-entry lookup table"
DIGEST = [11, 22, 33, 44]


def _circuit(log_n):
    import plonk_large as PL

    from plonky2_b200 import plonk

    return PL.LargeCircuit(plonk, plonk.CircuitConfig(), log_n, seed=log_n,
                           luts=[(PL.range_table(), 64), (PL.small_table(), 2)], public_inputs=[3, 1, 4, 1, 5])


def _fri_params(c):
    from plonky2_b200.fri import standard_recursion_fri_config

    return standard_recursion_fri_config().fri_params(c.common.degree_bits, False)


def distributed_run(args):
    import torch
    import torch.distributed as dist

    import plonky2_b200 as pb
    from plonky2_b200 import distributed as D
    from plonky2_b200 import plonk

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
    c = _circuit(args.log_n)
    cfg, cd = c.config, c.common
    fri_params = _fri_params(c)
    cs = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height, ctx=ctx,
                                        shard=(rank, world))
    prover_data = plonk.ProverOnlyCircuitData(cs, c.sigmas, DIGEST, fri_params)

    def one():
        dist.barrier()
        t0 = time.perf_counter()
        D.prove_plonk(prover_data, cd, c.wires, c.public_inputs, ctx=ctx)
        ctx.synchronize()
        t = torch.tensor([(time.perf_counter() - t0) * 1e3], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    for _ in range(args.warmup):
        one()
    ms = [one() for _ in range(args.reps)]
    cs.close()
    if rank == 0:
        whole = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height, ctx=ctx)
        one_device = plonk.ProverOnlyCircuitData(whole, c.sigmas, DIGEST, fri_params)
        for _ in range(args.warmup):
            plonk.prove_with_witness(one_device, cd, c.wires, c.public_inputs, ctx=ctx)
        single = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            plonk.prove_with_witness(one_device, cd, c.wires, c.public_inputs, ctx=ctx)
            ctx.synchronize()
            single.append((time.perf_counter() - t0) * 1e3)
        whole.close()
        print(json.dumps({"gpu": gpu_info(), "workload": WORKLOAD % args.log_n, "world": world, "backend": "nccl",
                          "prove_plonk_ms_median": round(float(np.median(ms)), 2), "prove_plonk_ms": [round(m, 2) for m in ms],
                          "one_device_prove_ms_median": round(float(np.median(single)), 2),
                          "reps": args.reps, "warmup": args.warmup}))
    dist.barrier()
    dist.destroy_process_group()


def per_shard_run(args):
    import ctypes as C

    import torch

    import plonky2_b200 as pb
    from conftest import synth
    from plonky2_b200 import _native as N
    from plonky2_b200 import plonk
    from plonky2_b200.prover import compute_all_lookup_polys, wires_permutation_partial_products_and_zs

    G = args.per_shard
    ctx = pb.default_context()
    c = _circuit(args.log_n)
    cfg, cd = c.config, c.common
    nc, nr, rate_bits, cap_height = cfg.num_challenges, cfg.num_routed_wires, cfg.rate_bits, cfg.cap_height
    v = [int(x) for x in synth(0x7F8, (7 * nc,))]
    betas, gammas, alphas, deltas = v[:nc], v[nc:2 * nc], v[2 * nc:3 * nc], v[3 * nc:]
    zs, pps = [], []
    for beta, gamma in zip(betas, gammas):
        out = wires_permutation_partial_products_and_zs(c.wires[:nr], c.sigmas, cd.k_is, beta, gamma,
                                                        cd.quotient_degree_factor, ctx)
        zs.append(out[-1])
        pps += list(out[:-1])
    zv = np.concatenate([np.stack(zs + pps),
                         compute_all_lookup_polys(c.wires, nr, cfg.max_quotient_degree_factor, deltas, c.lookup_rows, nc,
                                                  ctx)])
    qdf = cd.quotient_degree_factor
    size = c.n << (qdf - 1).bit_length()
    values = torch.empty((G, nc, size // G), dtype=torch.int64, device="cuda")
    ctx.synchronize()

    def timed(fn):
        ctx.synchronize()
        t0 = time.perf_counter()
        r = fn()
        ctx.synchronize()
        return r, (time.perf_counter() - t0) * 1e3

    def shard_work(g):
        cs = pb.PolynomialBatch.from_values(c.constants_sigmas, rate_bits, False, cap_height, ctx=ctx, shard=(g, G))
        commits = [cs]
        try:
            w, t_w = timed(lambda: pb.PolynomialBatch.from_values(c.wires, rate_bits, False, cap_height, ctx=ctx,
                                                                  shard=(g, G)))
            commits.append(w)
            z, t_z = timed(lambda: pb.PolynomialBatch.from_values(zv, rate_bits, False, cap_height, ctx=ctx,
                                                                  shard=(g, G)))
            commits.append(z)
            prog, consts, al = plonk.quotient_program(cd, commits, c.public_inputs_hash, betas, gammas, alphas, deltas)
            handles = (C.c_void_p * 3)(*[x.h for x in commits])
            _, t_q = timed(lambda: N.check(N.lib().gl_plonk_quotient_shard(
                ctx.h, handles, 3, prog, len(prog), N.np_ptr(consts), len(consts), N.np_ptr(al), len(al),
                cd.num_vanishing_terms(), qdf, N.vp(values[g].data_ptr())), ctx.h))
        finally:
            for x in commits:
                x.close()
        return t_w, t_z, t_q

    for _ in range(args.warmup):
        shard_work(0)
    shards = [dict(g=g) for g in range(G)]
    for s in shards:
        s["wires_commitment_ms"], s["zs_commitment_ms"], s["shard_quotient_ms"] = (round(t, 2) for t in shard_work(s["g"]))
    quotient = torch.empty((nc, size), dtype=torch.int64, device="cuda")
    _, t_from = timed(lambda: N.check(N.lib().gl_stark_quotient_from_shards(
        ctx.h, N.vp(values.data_ptr()), G, nc, cd.degree_bits, qdf, N.vp(quotient.data_ptr())), ctx.h))
    for s in shards:
        qc, t = timed(lambda: plonk.commit_quotient_polys(cd, quotient, ctx, shard=(s["g"], G)))
        qc.close()
        s["quotient_commitment_ms"] = round(t, 2)
    steps = ("wires_commitment_ms", "zs_commitment_ms", "shard_quotient_ms", "quotient_commitment_ms")
    print(json.dumps({"gpu": gpu_info(), "workload": WORKLOAD % args.log_n,
                      "label": "per-shard device time, no communication", "shards": G,
                      "per_shard": shards, "slowest_shard_ms": {k: max(s[k] for s in shards) for k in steps},
                      "from_shards_ms (every rank)": round(t_from, 2), "warmup": args.warmup}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=18)
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
