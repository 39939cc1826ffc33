"""What zero knowledge costs on the device.

1. Salt for one blinded commitment of N = 2^23 LDE rows (4 x 2^23 elements, 268 MB): the device sampler
   (gl_random_field_elements into device memory, the kernel gl_commit_finish_keyed runs) against the host path
   (random_field_elements from os.urandom, then the H2D copy a host-salted commitment makes).
2. plonk.prove_with_witness with and without zero knowledge on bench.py's 2^12-row circuit (standard_recursion_config,
   standard FRI parameters), alternating. The witness is the same in both: the timing does not depend on what the
   blinding rows hold.

Prints one JSON line with the GPU's name and power limit. Usage: python tools/zk_prove_cost.py [--reps R]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def salt_fill(reps):
    import torch

    import plonky2_b200 as pb
    from plonky2_b200 import _native as N
    from plonky2_b200.polynomial_batch import random_field_elements

    ctx = pb.default_context()
    N_rows = 1 << 23
    buf = torch.empty((4, N_rows), dtype=torch.int64, device="cuda")
    key = bytes(range(32))
    stream = torch.cuda.ExternalStream(ctx.stream)

    def device_once():
        for s in range(4):
            N.check(N.lib().gl_random_field_elements(ctx.h, key, s, 0, N_rows, N.vp(buf[s].data_ptr()), N.MEM_DEVICE),
                    ctx.h)

    device_once()
    ctx.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev_ms = []
    for _ in range(reps):
        a.record(stream)
        device_once()
        b.record(stream)
        b.synchronize()
        dev_ms.append(a.elapsed_time(b))
    host_ms, draw_ms = [], []
    for _ in range(max(1, reps // 4)):
        t0 = time.perf_counter()
        salt = random_field_elements(4 * N_rows)
        t1 = time.perf_counter()
        buf.copy_(torch.from_numpy(salt.view(np.int64)).view(4, N_rows))
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        draw_ms.append((t1 - t0) * 1e3)
        host_ms.append((t2 - t0) * 1e3)
    return {"elements": 4 * N_rows, "bytes": 32 * N_rows, "device_sampler_ms_median": float(np.median(dev_ms)),
            "device_sampler_GBps": 32 * N_rows / (np.median(dev_ms) * 1e6),
            "host_draw_ms_median": float(np.median(draw_ms)), "host_draw_plus_h2d_ms_median": float(np.median(host_ms))}


def prove_cost(reps):
    import plonk_circuits as PC

    import plonky2_b200 as pb
    from plonky2_b200 import plonk

    degree_bits = 12
    extra = ("ArithmeticExtensionGate", "MulExtensionGate", "BaseSumGate", "ReducingGate", "ReducingExtensionGate",
             "PoseidonMdsGate", "RandomAccessGate", "ExponentiationGate", "CosetInterpolationGate")
    cfg = plonk.CircuitConfig()
    c = PC.FibonacciCircuit(plonk, cfg, degree_bits, seed=7, poseidon_rows=256, extra=extra, public_inputs=[1, 2, 3])
    fri = pb.standard_recursion_fri_config()
    ctx = pb.default_context()
    cs = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height, ctx=ctx)
    digest = [0x11, 0x22, 0x33, 0x44]
    data = {zk: plonk.ProverOnlyCircuitData(cs, c.sigmas, digest, fri.fri_params(degree_bits, zk)) for zk in (False, True)}
    sizes, times = {}, {False: [], True: []}

    def once(zk):
        cfg.zero_knowledge = zk
        t0 = time.perf_counter()
        b = plonk.prove_with_witness(data[zk], c.common, c.wires, c.public_inputs, ctx=ctx).to_bytes()
        return time.perf_counter() - t0, len(b)

    for zk in (False, True):
        once(zk)
    for _ in range(reps):
        for zk in (False, True):
            t, sizes[zk] = once(zk)
            times[zk].append(t * 1e3)
    cs.close()
    off, on = float(np.median(times[False])), float(np.median(times[True]))
    return {"plain_ms_median": off, "zk_ms_median": on, "zk_over_plain": on / off, "plain_proof_bytes": sizes[False],
            "zk_proof_bytes": sizes[True], "reps": reps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=8)
    args = ap.parse_args()
    out = {"gpu": gpu_info(), "salt_fill_4x2^23": salt_fill(args.reps), "prove_2^12_rows": prove_cost(args.reps)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
