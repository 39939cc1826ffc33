"""Cost of building plonky2 circuit data at 2^20 rows x 135 wires (standard_recursion_config): the device sigma
polynomials (gl_sigma_polys) and the constants/sigmas commitment, each timed over repeated runs after a warm-up with a
host clock around work that ends in a device synchronise, and the vectorised CPU restatement of the sigma step
(scipy connected components + stable argsort, tests/test_circuit_data.vector_sigma_map) at the same shape -- a
restatement in Python, not the Rust reference.

The copy constraints: `density` pairs per row between random routed wires (one pair joins two random routed wires of
the whole trace; with the default of 8 per row there are 8 M pairs over 84 M routed wires), plus 2^16 virtual targets
each joined to two random routed wires. Prints one JSON line with the card's name, power limit and SM clock.

  python tools/circuit_build_cost.py [--log-n 20] [--density 8] [--reps 5] [--out PATH]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [v.strip() for v in r.stdout.splitlines()[0].split(",")])) if r.returncode == 0 else {}


def stats(ts):
    ts = sorted(ts)
    return dict(median_ms=1e3 * ts[len(ts) // 2], min_ms=1e3 * ts[0], max_ms=1e3 * ts[-1], runs=len(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--density", type=int, default=8, help="copy-constraint pairs per row")
    ap.add_argument("--virtual", type=int, default=1 << 16)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch

    import plonky2_b200 as pb
    from plonky2_b200 import plonk
    from test_circuit_data import vector_sigma_map

    cfg = plonk.CircuitConfig()                   # standard_recursion_config: 135 wires, 80 routed
    db, n = a.log_n, 1 << a.log_n
    nw, nr = cfg.num_wires, cfg.num_routed_wires
    rng = np.random.default_rng(1)
    routed = lambda k: (rng.integers(0, n, k) * nw + rng.integers(0, nr, k)).astype(np.int64)  # noqa: E731
    e = a.density * n
    v = (n * nw + np.arange(a.virtual, dtype=np.int64)).repeat(2)
    pairs = np.concatenate([np.stack([routed(e), routed(e)], 1), np.stack([v, routed(len(v))], 1)]).astype(np.uint64)
    ctx = pb.default_context()
    rows = [(plonk.ArithmeticGate.new_from_config(cfg), [3, 5])] * n
    common, constant_vecs = plonk.CommonCircuitData.from_gate_instances(cfg, rows)

    def sigma():
        s = plonk.sigma_polys(cfg, db, pairs, a.virtual, ctx)
        ctx.synchronize()
        return s

    sig = sigma()                                 # warm-up
    ts = []
    for _ in range(a.reps):
        del sig
        t0 = time.perf_counter()
        sig = sigma()
        ts.append(time.perf_counter() - t0)
    sigma_t = stats(ts)
    ts = []
    for k in range(a.reps + 1):
        t0 = time.perf_counter()
        c = plonk.commit_constants_sigmas(common, constant_vecs, sig, ctx)   # synchronises before it returns
        dt = time.perf_counter() - t0
        c.close()
        if k:
            ts.append(dt)
    commit_t = stats(ts)
    got = sig[:, :4096].cpu().numpy().view(np.uint64).copy()
    del sig
    torch.cuda.empty_cache()
    ts, want = [], None
    for _ in range(a.cpu_reps):
        t0 = time.perf_counter()
        want = vector_sigma_map(nw, nr, db, a.virtual, pairs.astype(np.int64))
        ts.append(time.perf_counter() - t0)
    cpu_t = stats(ts)
    import test_circuit_data as T
    from plonky2_b200.plonk import get_unique_coset_shifts

    check = T.sigma_values(want, get_unique_coset_shifts(nr), db)[:, :4096]
    res = dict(shape=dict(rows=n, num_wires=nw, num_routed_wires=nr, pairs=len(pairs), virtual_targets=a.virtual,
                          pairs_per_row=a.density),
               device_sigma=sigma_t, constants_sigmas_commit=commit_t, cpu_vectorised_restatement_sigma=cpu_t,
               device_matches_restatement_first_4096_rows=bool(np.array_equal(got, check)),
               host_cpus=os.cpu_count(), gpu=gpu_info())
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
