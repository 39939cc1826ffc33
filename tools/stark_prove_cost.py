"""A full starky proof at BASELINE config 5's shape: 64 columns x 2^24 rows, StarkConfig.standard_fast_config (rate
1/2, cap height 4, five arity-16 FRI rounds, 84 queries, 16 bits of grinding).

The STARK is FibonacciPairsStark below: 32 independent Fibonacci pairs (x, y) -> (y, x + y), two transition
constraints per pair, so any trace the generator writes satisfies it. The first row is the SURVEY 8(d) splitmix64
counter generator's (seed 0x05, tests/conftest.py synth); the rows below it are written on the device (segment starts
from the pair's matrix power on the host, then one modular addition per row and segment).

Prints one JSON line: the GPU's name and power limit, the median of --reps full proofs after --warmup (each ends in a
device synchronise), one proof's per-phase times (trace commitment, constraint-binding step, quotient, quotient
commitment, openings, FRI; measured in a separate run with a synchronise after each phase), whether the restated
verifier of tests/stark_twin.py accepts the proof, and the CPU twin's time at the largest size it proves in a few seconds.

Usage: python tools/stark_prove_cost.py [--log-n 24] [--reps 3] [--warmup 1]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

P = 0xFFFFFFFF00000001
PAIRS = 32


def _stark_base():
    from plonky2_b200.stark import Stark

    return Stark


class FibonacciPairsStark(_stark_base()):
    """64 columns: pair k is (column 2k, column 2k + 1) with x' = y, y' = x + y. No public inputs; constraint degree 2
    (the transition filter), so one quotient chunk per challenge."""
    COLUMNS, PUBLIC_INPUTS = 2 * PAIRS, 0

    def eval(self, v, y):
        for k in range(PAIRS):
            x0, x1 = v.local(2 * k), v.local(2 * k + 1)
            y.constraint_transition(v.next(2 * k) - x1)
            y.constraint_transition(v.next(2 * k + 1) - x0 - x1)

    def constraint_degree(self):
        return 2


def _fib_matrix_pow(e):
    """[[F(e-1), F(e)], [F(e), F(e+1)]] mod p: the pair map applied e times."""
    def mul(a, b):
        return [[(a[0][0] * b[0][0] + a[0][1] * b[1][0]) % P, (a[0][0] * b[0][1] + a[0][1] * b[1][1]) % P],
                [(a[1][0] * b[0][0] + a[1][1] * b[1][0]) % P, (a[1][0] * b[0][1] + a[1][1] * b[1][1]) % P]]
    r, m = [[1, 0], [0, 1]], [[0, 1], [1, 1]]
    while e:
        if e & 1:
            r = mul(r, m)
        m = mul(m, m)
        e >>= 1
    return r


def _i64(v):
    return v - (1 << 64) if v >= (1 << 63) else v


def _add_mod(a, b):
    """a + b mod p on int64 tensors holding canonical u64 words (wrapping adds, unsigned compares by flipping the sign
    bit): 2^64 = 2^32 - 1 (mod p)."""
    import torch

    lo = -(1 << 63)
    s = a + b
    s = s + ((s ^ lo) < (a ^ lo)).to(torch.int64) * 0xFFFFFFFF
    return torch.where((s ^ lo) >= (_i64(P) ^ lo), s + 0xFFFFFFFF, s)


def fibonacci_pairs_trace(log_n, seed=0x05, device="cuda"):
    """(64, 2^log_n) int64 tensor on `device`: row 0 = synth(seed, (64,)), row r + 1 = the pair map of row r."""
    import torch
    from conftest import synth

    n = 1 << log_n
    seg = 1 << (log_n // 2)
    nseg = n // seg
    first = [int(v) for v in synth(seed, (2 * PAIRS,))]
    m = _fib_matrix_pow(seg)
    starts = np.empty((2 * PAIRS, nseg), dtype=np.uint64)
    for k in range(PAIRS):
        x, y = first[2 * k], first[2 * k + 1]
        for s in range(nseg):
            starts[2 * k, s], starts[2 * k + 1, s] = x, y
            x, y = (m[0][0] * x + m[0][1] * y) % P, (m[1][0] * x + m[1][1] * y) % P
    cur = torch.from_numpy(starts.view(np.int64)).to(device)
    out = torch.empty((2 * PAIRS, nseg, seg), dtype=torch.int64, device=device)
    for j in range(seg):
        out[:, :, j] = cur
        x, y = cur[0::2], cur[1::2]
        cur = torch.stack([y, _add_mod(x, y)], dim=1).reshape(2 * PAIRS, nseg)
    return out.reshape(2 * PAIRS, n)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


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

    patches = [(stark_mod, "_commit_trace", "trace_commitment"), (stark_mod, "_bind_constraints", "binding_step"),
               (stark_mod, "compute_quotient_polys", "quotient"), (stark_mod, "commit_quotient_polys",
                                                                    "quotient_commitment"),
               (proof_mod, "eval_commitments", "openings"), (fri_mod, "prove_openings", "fri")]
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


def cpu_twin(stark, config, budget_s):
    """The CPU twin (tests/stark_twin.py: the oracle's commitments, openings and FRI, the quotient on the host) at growing
    row counts; the largest that finishes within budget_s."""
    import oracle_lib
    import stark_twin as T

    best = None
    for log_n in range(6, 25, 2):
        trace = fibonacci_pairs_trace(log_n, device="cpu").numpy().view(np.uint64)
        t0 = time.perf_counter()
        T.twin_prove(oracle_lib, stark, config, trace, [])
        dt = time.perf_counter() - t0
        if dt > budget_s:
            break
        best = {"log_n": log_n, "seconds": round(dt, 3)}
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=24)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--cpu-budget", type=float, default=4.0, help="seconds the CPU twin may take per proof")
    args = ap.parse_args()

    import oracle_lib
    import stark_twin as T
    import torch

    import plonky2_b200 as pb
    from plonky2_b200 import stark as S

    ctx = pb.default_context()
    stark, config = FibonacciPairsStark(), S.StarkConfig.standard_fast_config()
    t0 = time.perf_counter()
    trace = fibonacci_pairs_trace(args.log_n)
    torch.cuda.synchronize()     # the generator's kernels run on torch's stream, not the context's
    gen_ms = (time.perf_counter() - t0) * 1e3
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
    out = {"gpu": gpu_info(), "workload": "starky prove: FibonacciPairsStark, %d columns x 2^%d rows, standard_fast_config"
                                         % (stark.COLUMNS, args.log_n),
           "trace_generation_ms": round(gen_ms, 1), "prove_ms_median": round(float(np.median(ms)), 2),
           "prove_ms": [round(m, 2) for m in ms], "reps": args.reps, "warmup": args.warmup,
           "phases_ms_one_proof": phases, "restated_verifier_accepts": accepted,
           "fri_proof_bytes": len(proof.proof.opening_proof.to_bytes()),
           "cpu_twin_largest_within_budget": cpu_twin(stark, config, args.cpu_budget)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
