"""A multi-STARK proof WITH cross-table lookups at sizes a user would run: three tables of 2^22, 2^21 and 2^20 rows
(--log-n sets the largest), StarkConfig.standard_fast_config. The 2^22-row table looks twice into the 2^20-row table
(two consecutive entries: one CTL helper column per challenge), the 2^21-row table once; the tuples are pairs of
columns behind sparse boolean selectors.

Prints one JSON line: the GPU's name and power limit, the median of --reps full proofs after --warmup (each ends in a
device synchronise), one proof's per-phase times (trace commitments, CTL helper columns, auxiliary commitments,
constraint-binding steps, quotients, quotient commitments, openings, FRI; measured in a separate run with a synchronise
after each phase, summed over the tables), and whether the restated verifier of tests/stark_twin.py accepts.

Usage: python tools/stark_ctl_cost.py [--log-n 22] [--reps 3] [--warmup 1]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from stark_prove_cost import gpu_info  # noqa: E402
from plonky2_b200.stark import Stark  # noqa: E402


class _Table(Stark):
    """Pairs of tuple columns, each pair followed by its boolean selector; the selectors are constrained boolean."""
    PUBLIC_INPUTS = 0

    def __init__(self, pairs):
        self.pairs = pairs
        self.COLUMNS = 3 * pairs

    def eval(self, v, y):
        for k in range(self.pairs):
            s = v.local(3 * k + 2)
            y.constraint(s * s - s)

    def constraint_degree(self):
        return 3

    def requires_ctls(self):
        return True


def system(log_n):
    """Tables (2 pairs at 2^log_n, 1 pair at 2^(log_n - 1), the looked pair at 2^(log_n - 2)), the CTL, host traces."""
    from plonky2_b200.cross_table_lookup import CrossTableLookup, TableWithColumns
    from plonky2_b200.lookup import Column, Filter

    rng = np.random.default_rng(0x5C7)
    sizes = [1 << log_n, 1 << (log_n - 1), 1 << (log_n - 2)]
    traces = [np.zeros((3 * p, n), dtype=np.uint64) for p, n in zip((2, 1, 1), sizes)]
    rows = []
    for t, every in ((0, 16), (1, 8)):
        tr = traces[t]
        for k in range(tr.shape[0] // 3):
            tr[3 * k:3 * k + 2] = rng.integers(0, 1 << 62, (2, tr.shape[1]), dtype=np.uint64)
            sel = (rng.integers(0, every, tr.shape[1]) == 0).astype(np.uint64)
            tr[3 * k + 2] = sel
            rows.append(tr[3 * k:3 * k + 2, sel == 1])
    looked = traces[2]
    picked = np.concatenate(rows, axis=1)
    assert picked.shape[1] <= sizes[2]
    where = rng.permutation(sizes[2])[:picked.shape[1]]
    looked[0:2] = rng.integers(0, 1 << 62, (2, sizes[2]), dtype=np.uint64)
    looked[0:2, where] = picked
    looked[2, where] = 1
    entry = lambda t, k: TableWithColumns(t, Column.singles([3 * k, 3 * k + 1]),  # noqa: E731
                                          Filter.new_simple(Column.single(3 * k + 2)))
    ctl = CrossTableLookup([entry(0, 0), entry(0, 1), entry(1, 0)], entry(2, 0))
    return [_Table(2), _Table(1), _Table(1)], [ctl], traces


def phase_times(starks, config, traces, ctls, ctx):
    """One proof with a device synchronise after each phase, timed by wrapping the functions prove_with_ctls calls."""
    import plonky2_b200.cross_table_lookup as ctl_mod
    import plonky2_b200.fri as fri_mod
    import plonky2_b200.proof as proof_mod
    import plonky2_b200.stark as stark_mod

    times = {}

    def timed(fn, label):
        def wrapper(*a, **k):
            ctx.synchronize()
            t0 = time.perf_counter()
            r = fn(*a, **k)
            ctx.synchronize()
            times[label] = times.get(label, 0.0) + (time.perf_counter() - t0) * 1e3
            return r
        return wrapper

    patches = [(stark_mod, "_commit_trace", "trace_commitments"),
               (ctl_mod, "compute_ctl_helper_columns", "ctl_helper_columns"),
               (stark_mod, "commit_auxiliary_polys", "auxiliary_commitments"),
               (stark_mod, "_bind_constraints", "binding_steps"), (stark_mod, "compute_quotient_polys", "quotients"),
               (stark_mod, "commit_quotient_polys", "quotient_commitments"),
               (proof_mod, "eval_commitments", "openings"), (fri_mod, "prove_openings", "fri")]
    saved = []
    for mod, name, label in patches:
        fn = getattr(mod, name)
        saved.append((mod, name, fn))
        setattr(mod, name, timed(fn, label))
    try:
        t0 = time.perf_counter()
        ctl_mod.prove_with_ctls(starks, config, traces, ctls, [[]] * len(starks), ctx=ctx)
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
    from plonky2_b200.cross_table_lookup import prove_with_ctls

    ctx = pb.default_context()
    config = S.StarkConfig.standard_fast_config()
    starks, ctls, host = system(args.log_n)
    traces = [torch.from_numpy(t.view(np.int64)).cuda() for t in host]    # device traces: no H2D copy is timed
    torch.cuda.synchronize()
    pis = [[]] * len(starks)
    for _ in range(args.warmup):
        prove_with_ctls(starks, config, traces, ctls, pis, ctx=ctx)
    ms = []
    proof = None
    for _ in range(args.reps):
        t0 = time.perf_counter()
        proof = prove_with_ctls(starks, config, traces, ctls, pis, ctx=ctx)
        ctx.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    accepted = T.verify_with_ctls(oracle_lib, starks, config, ctls, proof) is None
    phases = phase_times(starks, config, traces, ctls, ctx)
    out = {"gpu": gpu_info(),
           "workload": "prove_with_ctls: 3 tables of 2^%d x 6, 2^%d x 3, 2^%d x 3 columns, one CTL (2 + 1 looking "
                       "entries of pairs), standard_fast_config" % (args.log_n, args.log_n - 1, args.log_n - 2),
           "prove_ms_median": round(float(np.median(ms)), 2), "prove_ms": [round(m, 2) for m in ms], "reps": args.reps,
           "warmup": args.warmup, "phases_ms_one_proof": phases, "restated_verifier_accepts": accepted}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
