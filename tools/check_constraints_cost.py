"""What check_constraints costs on the device, next to the quotient it guards, for two workloads:

  stark  the 64-column x 2^24 FibonacciPairsStark of tools/stark_prove_cost.py (StarkConfig.standard_fast_config: rate
         1/2, one quotient chunk per challenge), trace commitment resident;
  plonk  tests/plonk_large.LargeCircuit at 2^18 gates (the standard recursion config's wires, quotient degree factor 8,
         rate 3, two small lookup tables), its constants / sigmas, wires and Z / partial-product / lookup commitments
         made as prove_with_witness makes them.

For each: the median of --reps checks (stark.check_constraints / plonk.check_constraints, host clock; each call ends in
a synchronising read-back) after --warmup, the median of the same number of quotient evaluations
(compute_quotient_polys, synchronised), the library's device high-water mark during one check above what was in use
before it (Context.device_bytes; the scratch is the values on H, sum of B x n words, plus 8 (n + 1) bytes of row
offsets), and, from one check under torch.profiler in a run of its own, the kernel time of the NTTs onto H and of the
row-check kernel. Prints one JSON line with the GPU's name, power limit and maximum SM clock.

Usage: python tools/check_constraints_cost.py [--stark-log-n 24] [--plonk-log-n 18] [--reps 5] [--warmup 1]"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]


def _median_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return round(statistics.median(times), 2)


def _high_water_mib(ctx, fn):
    in_use, _ = ctx.device_bytes(reset_high=True)
    fn()
    _, high = ctx.device_bytes()
    return round((high - in_use) / 2**20, 1)


def _kernel_ms(fn, check_kernel):
    """One call under torch.profiler: {ntt_onto_h, row_check, other} kernel milliseconds. The NTT onto H is the
    k_ntt_* passes and their k_fill_* twiddle tables; other = the scan, the x tables and the rest."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {"ntt_onto_h": 0.0, "row_check": 0.0, "other": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        name = e.key
        if check_kernel in name:
            out["row_check"] += t / 1e3
        elif "k_ntt" in name or "k_fill" in name:
            out["ntt_onto_h"] += t / 1e3
        elif t > 0 and not name.startswith(("cuda", "Memcpy", "Memset")):
            out["other"] += t / 1e3
    return {k: round(v, 2) for k, v in out.items()}


def stark_case(log_n, reps, warmup):
    import torch

    import plonky2_b200 as pb
    from plonky2_b200 import stark as S
    from stark_prove_cost import FibonacciPairsStark, fibonacci_pairs_trace

    ctx = pb.default_context()
    stark, config = FibonacciPairsStark(), S.StarkConfig.standard_fast_config()
    trace = fibonacci_pairs_trace(log_n)
    torch.cuda.synchronize()
    tc = S._commit_trace(trace, config.fri_config.rate_bits, config.fri_config.cap_height, ctx)
    del trace
    try:
        report = S.check_constraints(stark, tc, [])
        assert report.failures == 0, report
        alphas = [3, 5]

        def quotient():
            q = S.compute_quotient_polys(stark, tc, [], alphas)
            del q

        return {"rows": 1 << log_n, "columns": stark.COLUMNS,
                "check_ms": _median_ms(lambda: S.check_constraints(stark, tc, []), reps, warmup),
                "quotient_ms": _median_ms(quotient, reps, warmup),
                "check_high_water_mib": _high_water_mib(ctx, lambda: S.check_constraints(stark, tc, [])),
                "values_on_h_mib": round(stark.COLUMNS * (8 << log_n) / 2**20, 1),
                "check_kernels_ms": _kernel_ms(lambda: S.check_constraints(stark, tc, []), "k_stark_check_rows")}
    finally:
        tc.close()


def plonk_case(log_n, reps, warmup):
    import plonk_circuits as PC
    import plonk_large as PL
    import plonky2_b200 as pb
    from plonky2_b200 import plonk
    from test_gpu_plonk_large import _device_commitments

    ctx = pb.default_context()
    c = PL.large_circuit(log_n)
    betas, gammas, alphas, deltas = PC.challenges(0x6a00, c)
    cs, w, z, _ = _device_commitments(pb, c, (betas, gammas, alphas, deltas))
    try:
        def check():
            return plonk.check_constraints(c.common, cs, c.public_inputs_hash, w, z, betas, gammas, deltas)

        report = check()
        assert report.failures == 0, report

        def quotient():
            q = plonk.compute_quotient_polys(c.common, cs, c.public_inputs_hash, w, z, betas, gammas, alphas, deltas)
            del q

        widths = sum(b.num_polys for b in (cs, w, z))
        return {"gates": c.n, "polynomials": widths,
                "check_ms": _median_ms(check, reps, warmup),
                "quotient_ms": _median_ms(quotient, reps, warmup),
                "check_high_water_mib": _high_water_mib(ctx, check),
                "values_on_h_mib": round(widths * (8 << log_n) / 2**20, 1),
                "check_kernels_ms": _kernel_ms(check, "k_plonk_check_rows")}
    finally:
        for b in (cs, w, z):
            b.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stark-log-n", type=int, default=24)
    ap.add_argument("--plonk-log-n", type=int, default=18)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("check_constraints_cost.py measures on a CUDA device; none is present")
    from stark_prove_cost import gpu_info

    out = {"gpu": gpu_info(), "stark": stark_case(args.stark_log_n, args.reps, args.warmup),
           "plonk": plonk_case(args.plonk_log_n, args.reps, args.warmup)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
