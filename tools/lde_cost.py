"""Where the coset LDE's time goes, pass by pass (run on the H100). Prints one JSON line.

One commitment of B coefficient columns of 2^log_n values at rate 2^-rate_bits (default: bench.py's cfg2 shape,
234 x 2^20, rate 1/8) is timed launch by launch with torch.profiler (CUDA kernel activity) after a warm-up, and so is
the bare forward NTT of one column group at the same size. The line gives each NTT pass kernel's launches and device
time, per coset and per column group, the HBM bytes each pass moves by the shapes, and the card's name, power limit and
max SM clock read in the same run.

    python tools/lde_cost.py [--config cfg5] [--per-coset] [--reps 10]

--per-coset selects the library's one-transform-per-coset LDE loop (the A/B switch of gl_ctx_set_ntt_group)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"cfg2": (234, 20, 3), "cfg5": (64, 24, 1)}
PER_COSET_BIT = 1 << 30


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return (q.stdout.strip().splitlines() or [q.stderr.strip()])[0]


def kernel_times(prof):
    """device time (ms) and launch count per NTT pass kernel"""
    out = {}
    for ev in prof.events():
        if ev.device_type.name != "CUDA" or "k_ntt" not in ev.name:
            continue
        t, k = out.get(ev.name, (0.0, 0))
        out[ev.name] = (t + ev.time_range.elapsed_us() / 1e3, k + 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2", choices=sorted(SHAPES))
    ap.add_argument("--per-coset", action="store_true")
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    from plonky2_b200 import _native as N

    L = N.lib()
    B, log_n, r = SHAPES[args.config]
    n, ncos = 1 << log_n, 1 << r
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    ctx = N.Context(0, stream=stream.cuda_stream)
    if args.per_coset:
        ctx.set_ntt_group(PER_COSET_BIT)
    group = max(8, (1 << 30) // (8 * n))  # the library's default transforms per launch (gl_ntt_host.cuh group_cols)
    with torch.cuda.stream(stream):
        coeffs = torch.randint(0, 2**63 - 1, (B, n), dtype=torch.int64, device=dev)
        ntt_buf = torch.randint(0, 2**63 - 1, (min(group, B), n), dtype=torch.int64, device=dev)

        def lde():
            h = N.vp()
            N.check(L.gl_commit_create(ctx.h, C.c_void_p(coeffs.data_ptr()), n, B, log_n, r, 4, None, 1, N.MEM_DEVICE,
                                       C.byref(h)), ctx.h)
            return h

        def ntt():
            N.check(L.gl_ntt(ctx.h, C.c_void_p(ntt_buf.data_ptr()), log_n, ntt_buf.shape[0], n, 0, 0, 1, N.MEM_DEVICE),
                    ctx.h)

        for _ in range(3):  # warm-up: modules, tables, scratch, clocks
            L.gl_commit_destroy(lde())
            ntt()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                L.gl_commit_destroy(lde())
            torch.cuda.synchronize()
        lde_k = kernel_times(prof)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                ntt()
            torch.cuda.synchronize()
        ntt_k = kernel_times(prof)

    def passes(ks, reps):
        return {name: {"launches": k // reps, "ms": round(t / reps, 4), "ms_per_launch": round(t / k, 4)}
                for name, (t, k) in sorted(ks.items())}

    elems = B * n * ncos  # coset elements of the LDE
    lde_p = passes(lde_k, args.reps)
    lde_ms = sum(p["ms"] for p in lde_p.values())
    batched = any("cosets" in name for name in lde_p)
    word = 8
    # HBM bytes by the shapes: the first column pass reads the coefficients once per coset (per-coset loop) or once
    # per group (batched) and writes one scratch column per coset; the middle pass (three-pass plans) and the row pass
    # read and write one column per coset.
    col_read = B * n * word * (1 if batched else ncos)
    col_write = elems * word
    line = {
        "config": args.config, "shape": {"B": B, "log_n": log_n, "rate_bits": r},
        "path": "batched cosets" if batched else "per coset",
        "gpu": gpu_info(),
        "lde_ms": round(lde_ms, 3), "lde_ps_per_coset_element": round(lde_ms * 1e9 / elems, 2),
        "lde_passes": lde_p,
        "lde_bytes": {"first_col_pass_read": col_read, "first_col_pass_write": col_write,
                      "middle_col_pass_read_write": 2 * elems * word if log_n > 20 else 0,
                      "row_pass_read_write": 2 * elems * word},
        "ntt_columns": ntt_buf.shape[0], "ntt_passes": passes(ntt_k, args.reps),
        "ntt_ps_per_element": round(sum(t for t, _ in ntt_k.values()) / args.reps * 1e9 / (ntt_buf.shape[0] * n), 2),
        "ntt_bytes_per_pass": 2 * ntt_buf.shape[0] * n * word,
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
