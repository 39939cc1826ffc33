"""Rank whole-library build variants (NTT / LDE / Merkle kernels) in one GPU run.

    python tools/lib_variants.py build            # here (no GPU): nvcc one libplonky2_b200 per variant into tools/variants/out/
    python tools/lib_variants.py run [cols]       # on the H100: time every variant, check they agree bit for bit

Each variant is the production source compiled with extra -D switches (VARIANTS below); `run` loads one library per
subprocess (plonky2_b200._native.LIB_PATH override), times the bare 2^20 NTT, one cfg2-shaped commitment (per-phase
CUDA-event times from the library's profiling scopes) and prints a checksum of the NTT output and of the cap -- all
variants must print the same checksums. The Poseidon-only harness is tools/variants/build.sh + variant_bench.cu."""
import hashlib
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tools", "variants", "out")
CSRC = os.path.join(ROOT, "plonky2_b200", "csrc")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
              "-shared"]
# name -> extra flags. Field-level switches live in gl_field.cuh, Poseidon ones in gl_poseidon.cuh.
VARIANTS = {
    "base": [],
    "redv1": ["-DGL_REDUCE_V1"],
    "sqr3": ["-DGL_SQR_3WIDE"],
    "mulx": ["-DGL_MUL_EXPLICIT"],
    "pfast": ["-DGL_PARTIAL_FAST"],
    "minb5": ["-DGL_HASH_MINB=5"],
    "sboxsqr4": ["-DGL_SBOX_SQR4"],
    "sboxi2f": ["-DGL_SBOX_I2F"],
    "pairf64": ["-DGL_PAIR_RENORM_F64"],
    "parent": ["-DGL_HASH_MINB=5", "-DGL_SBOX_SQR4", "-DGL_SBOX_I2F"],
}


def build():
    os.makedirs(OUT, exist_ok=True)
    procs = []
    for name, flags in VARIANTS.items():
        lib = os.path.join(OUT, "lib_%s.so" % name)
        cmd = ["nvcc"] + NVCC_FLAGS + flags + ["-o", lib, "plonky2_b200.cu"]
        procs.append((name, subprocess.Popen(cmd, cwd=CSRC, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)))
    for name, p in procs:
        _, err = p.communicate()
        if p.returncode:
            sys.stderr.write(err.decode()[-2000:])
            raise SystemExit("build of variant %s failed" % name)
        print("built", name)


def time_one(lib_path, cols):
    import ctypes as C

    sys.path.insert(0, ROOT)
    import torch

    from plonky2_b200 import _native as N

    N.LIB_PATH = lib_path
    L = N.lib()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    ctx = N.Context(0, stream=stream.cuda_stream)
    ctx.set_profiling(True)
    log_n, ntt_cols, r, h = 20, 64, 3, 4
    n = 1 << log_n
    with torch.cuda.stream(stream):
        g = torch.Generator(device=dev)
        g.manual_seed(7)
        vals = torch.randint(0, 2**63 - 1, (max(cols, ntt_cols), n), dtype=torch.int64, device=dev, generator=g)
        buf = vals[:ntt_cols].clone()
        N.check(L.gl_ntt(ctx.h, C.c_void_p(buf.data_ptr()), log_n, ntt_cols, n, 0, 0, 1, N.MEM_DEVICE), ctx.h)
        torch.cuda.synchronize()
        ntt_sum = hashlib.sha256(buf.cpu().numpy().tobytes()).hexdigest()[:16]
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        best = 1e9
        for _ in range(3):
            a.record(stream)
            for _ in range(5):
                N.check(L.gl_ntt(ctx.h, C.c_void_p(buf.data_ptr()), log_n, ntt_cols, n, 0, 0, 1, N.MEM_DEVICE), ctx.h)
            e.record(stream)
            torch.cuda.synchronize()
            best = min(best, a.elapsed_time(e) / 5)
        cap = torch.empty(4 << h, dtype=torch.int64, device=dev)

        def commit():
            hnd = N.vp()
            N.check(L.gl_commit_create_sharded(ctx.h, C.c_void_p(vals.data_ptr()), n, cols, log_n, r, h, None, 0,
                                               N.MEM_DEVICE, 0, 1, C.byref(hnd)), ctx.h)
            N.check(L.gl_commit_cap(hnd, C.c_void_p(cap.data_ptr()), N.MEM_DEVICE), ctx.h)
            L.gl_commit_destroy(hnd)

        commit()
        torch.cuda.synchronize()
        ctx.reset_phases()
        steps = 3
        a.record(stream)
        for _ in range(steps):
            commit()
        e.record(stream)
        torch.cuda.synchronize()
        ms = a.elapsed_time(e) / steps
        ph = {k: v[0] / steps for k, v in ctx.phase_ms().items()}
        cap_sum = hashlib.sha256(cap.cpu().numpy().tobytes()).hexdigest()[:16]
    print("%-10s ntt64x2^20 %.3f ms | commit %d x 2^20 %.1f ms (intt %.1f lde %.1f leaf %.1f levels %.1f) | ntt %s cap %s"
          % (os.path.basename(lib_path)[4:-3], best, cols, ms, ph.get("intt", 0), ph.get("lde", 0), ph.get("leaf_hash", 0),
             ph.get("merkle_levels", 0), ntt_sum, cap_sum), flush=True)


def run(cols):
    libs = sorted(f for f in os.listdir(OUT) if f.startswith("lib_") and f.endswith(".so"))
    for f in libs:
        subprocess.call([sys.executable, os.path.abspath(__file__), "time", os.path.join(OUT, f), str(cols)])


if __name__ == "__main__":
    cmd = sys.argv[1] if len(sys.argv) > 1 else "build"
    if cmd == "build":
        build()
    elif cmd == "run":
        run(int(sys.argv[2]) if len(sys.argv) > 2 else 64)
    elif cmd == "time":
        time_one(sys.argv[2], int(sys.argv[3]))
