"""A starky proof WITH a logUp lookup at a size a user would run: RangeCheckStark below, 2^22 rows by default, eight
16-bit limb columns looked up in one 2^16-entry table column, half of them behind a selector filter,
StarkConfig.standard_fast_config (rate 1/2, so constraint degree 3: chunks of two looking columns per helper column).

Prints one JSON line: the GPU's name and power limit, the median of --reps full proofs after --warmup (each ends in a
device synchronise), one proof's per-phase times (trace commitment, lookup helper columns, auxiliary commitment,
constraint-binding step, quotient, quotient commitment, openings, FRI; measured in a separate run with a synchronise
after each phase), and whether the restated verifier of tests/stark_twin.py accepts the proof.

Usage: python tools/stark_lookup_cost.py [--log-n 22] [--reps 3] [--warmup 1]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from stark_prove_cost import gpu_info  # noqa: E402

LIMBS, TABLE_BITS = 8, 16
SEL, TABLE, FREQ = LIMBS, LIMBS + 1, LIMBS + 2


def _stark_base():
    from plonky2_b200.stark import Stark

    return Stark


class RangeCheckStark(_stark_base()):
    """Columns: LIMBS limbs, a boolean selector, the table 0 .. 2^16 - 1 (repeated), its frequencies. One lookup of every
    limb into the table; odd limbs are filtered by the selector. Constraints: the selector is boolean, the table starts
    at 0."""
    COLUMNS, PUBLIC_INPUTS = LIMBS + 3, 0

    def eval(self, v, y):
        s = v.local(SEL)
        y.constraint(s * s - s)
        y.constraint_first_row(v.local(TABLE))

    def constraint_degree(self):
        return 3

    def lookups(self):
        from plonky2_b200.lookup import Column, Filter, Lookup

        filters = [Filter.new_simple(Column.single(SEL)) if k % 2 else Filter.default() for k in range(LIMBS)]
        return [Lookup(Column.singles(range(LIMBS)), Column.single(TABLE), Column.single(FREQ), filters)]


def range_check_trace(log_n, seed=0x22):
    """(COLUMNS, 2^log_n) uint64 host columns: random limbs (out of range where the selector filters them out)."""
    n = 1 << log_n
    t = min(n, 1 << TABLE_BITS)
    rng = np.random.default_rng(seed)
    tr = np.zeros((LIMBS + 3, n), dtype=np.uint64)
    sel = rng.integers(0, 2, n).astype(np.uint64)
    tr[SEL] = sel
    counted = []
    for k in range(LIMBS):
        limb = rng.integers(0, t, n).astype(np.uint64)
        if k % 2:
            tr[k] = np.where(sel == 1, limb, limb + np.uint64(1 << 40))
            counted.append(limb[sel == 1])
        else:
            tr[k] = limb
            counted.append(limb)
    tr[TABLE] = np.arange(n, dtype=np.uint64) % np.uint64(t)
    tr[FREQ, :t] = np.bincount(np.concatenate(counted).astype(np.int64), minlength=t)
    return tr


def phase_times(stark, config, trace, ctx):
    """One proof with a device synchronise after each phase, timed by wrapping the functions `prove` calls."""
    import plonky2_b200.fri as fri_mod
    import plonky2_b200.proof as proof_mod
    import plonky2_b200.stark as stark_mod

    times = {}

    def timed(mod, name, label):
        fn = getattr(mod, name)

        def wrapper(*a, **k):
            ctx.synchronize()
            t0 = time.perf_counter()
            r = fn(*a, **k)
            ctx.synchronize()
            times[label] = times.get(label, 0.0) + (time.perf_counter() - t0) * 1e3
            return r
        return fn, wrapper

    patches = [(stark_mod, "_device_trace", "trace_to_device"), (stark_mod, "_commit_trace", "trace_commitment"),
               (stark_mod, "compute_lookup_helper_columns", "lookup helper columns"),
               (stark_mod, "commit_auxiliary_polys", "auxiliary commitment"),
               (stark_mod, "_bind_constraints", "binding_step"), (stark_mod, "compute_quotient_polys", "quotient"),
               (stark_mod, "commit_quotient_polys", "quotient_commitment"), (proof_mod, "eval_commitments", "openings"),
               (fri_mod, "prove_openings", "fri")]
    saved = []
    for mod, name, label in patches:
        fn, w = timed(mod, name, label)
        saved.append((mod, name, fn))
        setattr(mod, name, w)
    try:
        t0 = time.perf_counter()
        stark_mod.prove(stark, config, trace, [], ctx=ctx)
        ctx.synchronize()
        times["total"] = (time.perf_counter() - t0) * 1e3
    finally:
        for mod, name, fn in saved:
            setattr(mod, name, fn)
    return {k: round(v, 2) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=22)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()

    import oracle_lib
    import stark_twin as T
    import torch

    import plonky2_b200 as pb
    from plonky2_b200 import stark as S

    ctx = pb.default_context()
    stark, config = RangeCheckStark(), S.StarkConfig.standard_fast_config()
    host = range_check_trace(args.log_n)
    trace = torch.from_numpy(host.view(np.int64)).cuda()    # a device trace: the proofs below time no H2D copy
    torch.cuda.synchronize()
    for _ in range(args.warmup):
        S.prove(stark, config, trace, [], ctx=ctx)
    ms = []
    proof = None
    for _ in range(args.reps):
        t0 = time.perf_counter()
        proof = S.prove(stark, config, trace, [], ctx=ctx)
        ctx.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    accepted = T.verify(oracle_lib, stark, config, proof) is None
    phases = phase_times(stark, config, trace, ctx)
    out = {"gpu": gpu_info(),
           "workload": "starky prove with logUp: RangeCheckStark, %d limb columns (%d filtered) in a 2^%d table, "
                       "%d columns x 2^%d rows, %d auxiliary columns, standard_fast_config"
                       % (LIMBS, LIMBS // 2, TABLE_BITS, stark.COLUMNS, args.log_n,
                          stark.num_lookup_helper_columns(config)),
           "prove_ms_median": round(float(np.median(ms)), 2), "prove_ms": [round(m, 2) for m in ms], "reps": args.reps,
           "warmup": args.warmup, "phases_ms_one_proof": phases, "restated_verifier_accepts": accepted,
           "fri_proof_bytes": len(proof.proof.opening_proof.to_bytes())}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
