"""What plonk.check_copy_constraints (gl_plonk_check_copies) and plonk.check_lookups (gl_plonk_check_lookups) cost on
tests/plonk_large.LargeCircuit in standard_recursion_config (80 routed wires; the 2^16-entry range table and a small
table), for each --log-n (default 20 and 22 gates).

For each size and check: the median of --reps calls after --warmup (host clock; both calls end in a synchronising
read-back), with the witness already on the device as a CUDA tensor and the sigmas on the host, as
prover_data.sigmas is; the kernel times of one call from torch.profiler (CUDA time per kernel name); the library's
device high-water mark during one call above what was in use before it (Context.device_bytes). A size whose circuit
cannot be built or checked is reported as not measured, with the reason.

Prints one JSON line with the card's name and power limit; with --out, writes it there too.

Usage: python tools/check_arguments_cost.py [--log-n 20,22] [--reps 5] [--warmup 1] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
MIB = 1 << 20


def gpu_info():
    q = "name,power.limit"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [v.strip() for v in r.stdout.splitlines()[0].split(",")])) if r.returncode == 0 else {}


def measure(ctx, call, reps, warmup):
    import torch
    from torch.profiler import ProfilerActivity, profile

    for _ in range(warmup):
        call()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        report = call()
        times.append((time.perf_counter() - t0) * 1e3)
    in_use, _ = ctx.device_bytes(reset_high=True)
    call()
    high = ctx.device_bytes()[1] - in_use
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        if t:
            kernels[ev.key[:90]] = round(t / 1e3, 3)
    return {"median_ms": round(statistics.median(times), 2), "all_ms": [round(t, 2) for t in times],
            "high_water_mib": round(high / MIB, 1), "failures": report.failures,
            "kernels_ms": dict(sorted(kernels.items(), key=lambda kv: -kv[1])[:12])}


def case(log_n, reps, warmup):
    import numpy as np
    import torch

    import plonk_large as PL
    import plonky2_b200 as pb
    from plonky2_b200 import plonk

    t0 = time.perf_counter()
    c = PL.large_circuit(log_n, luts="range16")
    build_s = time.perf_counter() - t0
    ctx = pb.default_context()
    wires = torch.from_numpy(c.wires.view(np.int64)).cuda()
    torch.cuda.synchronize()

    class Data:
        sigmas = c.sigmas
    out = {"routed_wires": c.config.num_routed_wires << log_n, "circuit_build_s": round(build_s, 1)}
    out["copies"] = measure(ctx, lambda: plonk.check_copy_constraints(Data, c.common, wires), reps, warmup)
    out["lookups"] = measure(ctx, lambda: plonk.check_lookups(c.common, wires), reps, warmup)
    del wires
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", default="20,22")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"gpu": gpu_info()}
    for log_n in [int(x) for x in a.log_n.split(",")]:
        try:
            res["2^%d" % log_n] = case(log_n, a.reps, a.warmup)
        except Exception as e:  # a size that does not fit is reported, not fatal
            res["2^%d" % log_n] = {"not_measured": "%s: %s" % (type(e).__name__, e)}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
