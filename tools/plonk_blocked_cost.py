"""What non-resident commitments (plonk.prove_with_witness(..., lde_blocks=G)) cost: tests/plonk_large.LargeCircuit in
standard_recursion_config (135 wires, 80 routed, rate 1/8, quotient degree factor 8, 2 challenges) with the 2^16-entry
range table and a small table, at 2^20 gates by default.

The resident proof, then G = 1, 2, 4, 8, 16 blocks (the constants/sigmas commitment built with the same G): the median
of --reps proofs after --warmup (each ends in a device synchronise), one proof's phases with a synchronise after each
(commitments: wires, Z / partial products / lookups, quotient; quotient; openings; FRI, which rebuilds the blocks its
queries open), the library's device high-water mark during one proof (gl_ctx_device_bytes), and whether the proof's
bytes equal the resident proof's.

Also, and first (while the memory pool is empty), one proof with G = 16 at --over-log-n gates (2^22 by default), a
shape whose resident commitment footprint, computed from the widths, exceeds the card's total memory. The resident
proof is never attempted at that size; if the footprint fits the card, the run is skipped with the reason.

Prints one JSON line with the GPU's name, power limit and maximum SM clock.

Usage: python tools/plonk_blocked_cost.py [--log-n 20] [--over-log-n 22] [--reps 3] [--warmup 1]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
GIB = 1 << 30
DIGEST = [1, 2, 3, 4]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def widths(c):
    """The polynomials of the four commitments: constants/sigmas, wires, Z / partial products / lookups, quotient."""
    cfg, cd = c.config, c.common
    return [c.constants_sigmas.shape[0], cfg.num_wires,
            cd.num_zs_partial_products_polys() + cfg.num_challenges * cd.num_lookup_polys,
            cfg.num_challenges * cd.quotient_degree_factor]


def footprint(c):
    """Device bytes of the four commitments held resident, from the widths: 8·(B·n + B·N + 8·(N − C) + 4·C) each
    (coefficients, LDE, digests, cap; DESIGN §3)."""
    cfg = c.config
    n, C_ = 1 << c.common.degree_bits, 1 << cfg.cap_height
    N_ = n << cfg.rate_bits
    return sum(8 * (B * n + B * N_ + 8 * (N_ - C_) + 4 * C_) for B in widths(c))


def prover_data(pb, c, G):
    from plonky2_b200 import plonk
    from plonky2_b200.fri import standard_recursion_fri_config

    cfg = c.config
    fri_params = standard_recursion_fri_config().fri_params(c.common.degree_bits, False)
    cs = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height, lde_blocks=G)
    return plonk.ProverOnlyCircuitData(cs, c.sigmas, DIGEST, fri_params)


def prove(c, pd, G):
    from plonky2_b200 import plonk

    return plonk.prove_with_witness(pd, c.common, c.wires, c.public_inputs, lde_blocks=G).to_bytes()


def phase_times(c, pd, ctx, G):
    """One proof with a device synchronise after each phase, timed by wrapping the functions prove_with_witness calls."""
    import plonky2_b200.fri as fri_mod
    import plonky2_b200.plonk as plonk_mod
    import plonky2_b200.polynomial_batch as pb_mod
    import plonky2_b200.proof as proof_mod
    import plonky2_b200.prover as prover_mod

    times = {}
    patches = [(pb_mod.PolynomialBatch, "from_values", "commitments"), (prover_mod, "commit_zs_partial_products",
               "commitments"), (plonk_mod, "commit_quotient_polys", "commitments"),
               (plonk_mod, "compute_quotient_polys", "quotient"), (proof_mod.OpeningSet, "new", "openings"),
               (fri_mod, "prove_openings", "fri")]
    saved = []
    for owner, name, label in patches:
        fn = owner.__dict__[name]
        call = fn.__func__ if isinstance(fn, classmethod) else fn

        def wrapper(*a, _fn=call, _label=label, **k):
            ctx.synchronize()
            t0 = time.perf_counter()
            r = _fn(*a, **k)
            ctx.synchronize()
            times[_label] = times.get(_label, 0.0) + (time.perf_counter() - t0) * 1e3
            return r

        saved.append((owner, name, fn))
        setattr(owner, name, classmethod(wrapper) if isinstance(fn, classmethod) else wrapper)
    try:
        prove(c, pd, G)
    finally:
        for owner, name, fn in saved:
            setattr(owner, name, fn)
    return {k: round(v, 2) for k, v in times.items()}


def measure(pb, c, ctx, G, reps, warmup):
    pd = prover_data(pb, c, G)
    try:
        for _ in range(warmup):
            prove(c, pd, G)
        ms = []
        for _ in range(reps):
            ctx.device_bytes(reset_high=True)
            t0 = time.perf_counter()
            data = prove(c, pd, G)
            ctx.synchronize()
            ms.append((time.perf_counter() - t0) * 1e3)
        _, high = ctx.device_bytes()
        return data, {"prove_ms_median": round(float(np.median(ms)), 2), "prove_ms": [round(m, 2) for m in ms],
                      "library_high_water_gib": round(high / GIB, 3),
                      "phases_ms_one_proof": phase_times(c, pd, ctx, G)}
    finally:
        pd.constants_sigmas_commitment.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--over-log-n", type=int, default=22, help="gates (log2) of the over-memory proof; 0 skips it")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--blocks", default="1,2,4,8,16")
    args = ap.parse_args()

    import torch

    import plonk_large as PL
    import plonky2_b200 as pb

    ctx = pb.default_context()
    free, total = torch.cuda.mem_get_info()
    over = {"card_total_gib": round(total / GIB, 2), "free_gib": round(free / GIB, 2)}
    if args.over_log_n:
        t0 = time.perf_counter()
        big = PL.large_circuit(args.over_log_n, luts="range16", public_inputs=[3, 1, 4])
        over["shape"] = "LargeCircuit 2^%d gates, standard_recursion_config, range16 tables, G = 16" % args.over_log_n
        over["host_build_s"] = round(time.perf_counter() - t0, 1)
        over["polys"] = widths(big)
        over["resident_commitments_gib"] = round(footprint(big) / GIB, 2)
        if footprint(big) <= total:
            over["skipped"] = "the resident footprint fits the card; raise --over-log-n"
        else:
            pd = prover_data(pb, big, 16)
            try:
                ctx.device_bytes(reset_high=True)
                t0 = time.perf_counter()
                prove(big, pd, 16)
                ctx.synchronize()
                over["prove_ms"] = round((time.perf_counter() - t0) * 1e3, 2)
                over["library_high_water_gib"] = round(ctx.device_bytes()[1] / GIB, 3)
            finally:
                pd.constants_sigmas_commitment.close()
        del big

    c = PL.large_circuit(args.log_n, luts="range16", public_inputs=[3, 1, 4])
    resident, row = measure(pb, c, ctx, None, args.reps, args.warmup)
    row["resident_commitments_gib"] = round(footprint(c) / GIB, 2)
    runs = {"resident": row}
    for G in [int(g) for g in args.blocks.split(",")]:
        data, row = measure(pb, c, ctx, G, args.reps, args.warmup)
        row["equals_resident_proof"] = data == resident
        runs["G=%d" % G] = row

    print(json.dumps({"gpu": gpu_info(), "workload": "plonky2 prove_with_witness, lde_blocks: LargeCircuit 2^%d gates, "
                      "standard_recursion_config, range16 tables, polys %s" % (args.log_n, widths(c)),
                      "reps": args.reps, "warmup": args.warmup, "runs": runs, "over_memory": over}))


if __name__ == "__main__":
    main()
