"""Batch FRI at a user-sized shape: BatchFriOracle.from_values over degree groups (default 2^22 x 8, 2^20 x 32 and
2^18 x 64 polynomials at rate 1/2, cap height 4) and batch_prove_openings with every polynomial opened at one point,
28 queries and 16 bits of proof of work. The reduction arities are 4, 4 (down to the last group's LDE size, which
the folded codeword must pass through) and then 16.

    python tools/batch_fri_cost.py [--reps 5]
prints one JSON line: the card's name, power limit and maximum SM clock; the median over --reps of whole proofs
(commitment + batch_prove_openings, each ending in a device synchronise), of the commitment alone and of the prover
alone; one proof's phases, each closed by a device synchronise (group commitments and stages, FRI begin per degree,
commit rounds, mixes, proof of work, queries); and the stage chain of the groups after the tallest measured both ways
-- on the device (each group's commitment hashing `previous cap || LDE row` in place), and through the host round trip
this project used before: a cap-height-0 commitment of the group, its LDE rows read back (get_rows), concatenated with
the previous cap on the host and hashed again by MerkleTree -- with the two caps checked equal.

    python tools/batch_fri_cost.py --per-shard G
builds the row-block shard g of every group for every g < G on one GPU, one after another, and reports each shard's
commitment time and the median over --reps of the prover's replicated work (every rank runs it whole), labelled "per-shard device
time, no communication": nothing here measures the cap all-gather or the query exchange between GPUs. Neither mode is
part of bench.py."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from stark_prove_cost import gpu_info  # noqa: E402

P = 0xFFFFFFFF00000001


def _polys(groups, seed=7):
    rng = np.random.default_rng(seed)
    out = []
    for log_n, count in groups:
        m = rng.integers(0, 2**63, size=(count, 1 << log_n), dtype=np.uint64) % np.uint64(P)
        out += list(m)
    return out


def _instances(pb, groups, zeta):
    out, start = [], 0
    total = sum(c for _, c in groups)
    for _, c in groups:
        batch = pb.FriBatchInfo(zeta, [pb.FriPolynomialInfo(0, start + j) for j in range(c)])
        out.append(pb.FriInstanceInfo([pb.FriOracleInfo(total, False)], [batch]))
        start += c
    return out


def _prove(pb, oracle, groups, params):
    ch = pb.Challenger()
    ch.observe_cap(oracle.cap)
    zeta = ch.get_extension_challenge()
    return pb.batch_prove_openings([g for g, _ in groups], _instances(pb, groups, zeta), [oracle], ch, params)


class _Phases:
    """Wraps module functions and library entry points so that each call is closed by a device synchronise and its
    wall time is added to a label."""

    def __init__(self, ctx):
        self.ctx, self.ms, self.undo = ctx, {}, []

    def wrap(self, owner, name, label):
        fn = getattr(owner, name)

        def timed(*a, **k):
            self.ctx.synchronize()
            t0 = time.perf_counter()
            r = fn(*a, **k)
            self.ctx.synchronize()
            key = label(*a, **k) if callable(label) else label
            self.ms[key] = self.ms.get(key, 0.0) + (time.perf_counter() - t0) * 1e3
            return r

        setattr(owner, name, timed)
        self.undo.append((owner, name, fn))

    def restore(self):
        for owner, name, fn in reversed(self.undo):
            setattr(owner, name, fn)


def one_proof_phases(pb, polys, groups, args, params, ctx):
    from plonky2_b200 import _native as N
    from plonky2_b200 import fri as F
    from plonky2_b200.polynomial_batch import PolynomialBatch

    ph = _Phases(ctx)
    ph.wrap(PolynomialBatch, "_create",
            lambda cols, *a, **k: "commit group 2^%d x %d%s" % (int(np.log2(cols.shape[1])), cols.shape[0],
                                                               " (stage over previous cap)" if k.get("prefix") else ""))
    ph.wrap(F, "_begin", lambda inst, oracles, alpha, params: "fri begin, degree 2^%d" % params.degree_bits)
    ph.wrap(N.lib(), "gl_fri_commit_round", "fri commit rounds")
    ph.wrap(N.lib(), "gl_fri_fold", "fri folds")
    ph.wrap(N.lib(), "gl_fri_mix", "fri mixes")
    ph.wrap(F, "fri_proof_of_work", "proof of work")
    ph.wrap(F, "fri_prover_query_rounds", "queries")
    try:
        o = pb.BatchFriOracle.from_values(polys, args.rate_bits, False, args.cap_height)
        _prove(pb, o, groups, params)
        o.close()
    finally:
        ph.restore()
    return {k: round(v, 2) for k, v in ph.ms.items()}


def stage_chain_both_ways(pb, polys, groups, args, ctx):
    """(device ms, host round trip ms) for the stages of every group after the tallest, with the caps checked equal."""
    from plonky2_b200.polynomial_batch import PolynomialBatch

    r, heights = args.rate_bits, [g + args.rate_bits for g, _ in groups]
    cols, start = [], 0
    for _, c in groups:
        cols.append(np.stack(polys[start:start + c]))
        start += c
    first = PolynomialBatch.from_values(cols[0], r, False, heights[1])
    dev_ms = host_ms = 0.0
    caps = []
    for path in ("device", "host"):
        prev, made = first, []
        cap = first.merkle_tree.cap.hashes
        for k in range(1, len(groups)):
            h = heights[k + 1] if k + 1 < len(groups) else args.cap_height
            ctx.synchronize()
            t0 = time.perf_counter()
            if path == "device":
                t = PolynomialBatch._create(cols[k], r, False, h, False, None, ctx, prefix=prev)
                prev = t
            else:  # the former chain: a full cap-height-0 tree, the rows to the host and back, hashed again
                g = PolynomialBatch.from_values(cols[k], r, False, 0)
                rows = g.merkle_tree.get_rows(0, 1 << heights[k])
                t = pb.MerkleTree(np.ascontiguousarray(np.concatenate([cap, rows], axis=1)), h, ctx)
                made.append(g)
            cap = (t.merkle_tree if path == "device" else t).cap.hashes
            ctx.synchronize()
            ms = (time.perf_counter() - t0) * 1e3
            made.append(t)
            if path == "device":
                dev_ms += ms
            else:
                host_ms += ms
        caps.append(cap)
        for t in made:
            t.close()
    first.close()
    assert np.array_equal(caps[0], caps[1]), "device and host stage chains disagree"
    return round(dev_ms, 2), round(host_ms, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", default="22:8,20:32,18:64", help="log_n:count per degree group, tallest first")
    ap.add_argument("--rate-bits", type=int, default=1)
    ap.add_argument("--cap-height", type=int, default=4)
    ap.add_argument("--arity-bits", default="2,2,4,4,4")
    ap.add_argument("--queries", type=int, default=28)
    ap.add_argument("--pow-bits", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--per-shard", type=int, default=0, metavar="G")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("batch_fri_cost.py measures on a GPU; none is visible")
    import plonky2_b200 as pb

    ctx = pb.default_context(0)
    groups = [tuple(int(x) for x in g.split(":")) for g in args.groups.split(",")]
    arities = [int(a) for a in args.arity_bits.split(",")]
    cfg = pb.FriConfig(args.rate_bits, args.cap_height, args.pow_bits, ("Fixed", arities), args.queries)
    params = pb.FriParams(cfg, False, groups[0][0], arities)
    polys = _polys(groups)
    res = {"gpu": gpu_info(), "workload": "batch FRI, groups " + ", ".join("2^%d x %d" % g for g in groups),
           "rate_bits": args.rate_bits, "cap_height": args.cap_height, "arity_bits": arities,
           "queries": args.queries, "pow_bits": args.pow_bits}

    # warm-up: every shape once (module load, NTT tables, allocator)
    o = pb.BatchFriOracle.from_values(polys, args.rate_bits, False, args.cap_height)
    want = _prove(pb, o, groups, params).to_bytes()
    o.close()

    if args.per_shard:
        G = args.per_shard
        per = []
        for g in range(G):
            ctx.synchronize()
            t0 = time.perf_counter()
            s = pb.BatchFriOracle.from_values(polys, args.rate_bits, False, args.cap_height, shard=(g, G))
            ctx.synchronize()
            per.append(round((time.perf_counter() - t0) * 1e3, 2))
            s.close()
        o = pb.BatchFriOracle.from_values(polys, args.rate_bits, False, args.cap_height)
        runs = []
        for _ in range(args.reps):
            ctx.synchronize()
            t0 = time.perf_counter()
            _prove(pb, o, groups, params)
            ctx.synchronize()
            runs.append((time.perf_counter() - t0) * 1e3)
        replicated = round(statistics.median(runs), 2)
        o.close()
        res.update({"label": "per-shard device time, no communication", "num_shards": G,
                    "shard_commit_ms": per, "replicated_prover_ms (every rank, whole)": replicated,
                    "slowest_shard_commit_plus_prover_ms": round(max(per) + replicated, 2)})
        print(json.dumps(res), flush=True)
        return

    total, commit, prove = [], [], []
    for _ in range(args.reps):
        ctx.synchronize()
        t0 = time.perf_counter()
        o = pb.BatchFriOracle.from_values(polys, args.rate_bits, False, args.cap_height)
        ctx.synchronize()
        t1 = time.perf_counter()
        got = _prove(pb, o, groups, params).to_bytes()
        ctx.synchronize()
        t2 = time.perf_counter()
        o.close()
        assert got == want, "proofs differ between repetitions"
        total.append((t2 - t0) * 1e3)
        commit.append((t1 - t0) * 1e3)
        prove.append((t2 - t1) * 1e3)
    res.update({"reps": args.reps, "proof_ms_median": round(statistics.median(total), 2),
                "proof_ms_all": [round(t, 2) for t in total],
                "commit_ms_median": round(statistics.median(commit), 2),
                "prover_ms_median": round(statistics.median(prove), 2),
                "phases_ms (one proof, synchronised per phase)": one_proof_phases(pb, polys, groups, args, params, ctx)})
    stage_chain_both_ways(pb, polys, groups, args, ctx)   # warm-up of the host path's shapes
    dev, host = stage_chain_both_ways(pb, polys, groups, args, ctx)
    res.update({"later_stages_device_ms": dev, "later_stages_host_round_trip_ms": host})
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
