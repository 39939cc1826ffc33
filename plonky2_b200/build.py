"""Build the in-tree CUDA library (sm_90a, H100) with nvcc. No torch dependency: the product is a plain
C-ABI shared object (include/plonky2_b200.h)."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libplonky2_b200.so")
SOURCES = ["plonky2_b200.cu"]
DEPS = ["plonky2_b200.cu", "gl_chacha.cuh", "gl_ctl.cuh", "gl_field.cuh", "gl_lazy.cuh", "gl_logup.cuh", "gl_ntt.cuh", "gl_ntt_host.cuh", "gl_poseidon.cuh", "gl_poseidon_constants.h",
        "gl_sigma.cuh", "gl_stark_rows.cuh", "gl_vanishing.cuh", "gl_check_rows_host.cuh", "gl_check_args.cuh", "gl_check_args_host.cuh", "gl_plonk_blocked_host.cuh",
        os.path.join("..", "..", "include", "plonky2_b200.h"), os.path.join("..", "..", "include", "plonky2_b200_check.h"),
        os.path.join("..", "..", "include", "plonky2_b200_blocked.h"),
        os.path.abspath(__file__)]  # this file holds NVCC_FLAGS (the target architecture among them)
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]


def nvcc_path():
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found; cannot build libplonky2_b200.so")
    return p


def is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, d)) > t for d in DEPS)


def build(force=False, verbose=False):
    """Compile plonky2_b200/csrc/*.cu -> plonky2_b200/libplonky2_b200.so (cross-compiles without a GPU)."""
    if not force and not is_stale():
        return LIB
    cmd = [nvcc_path()] + NVCC_FLAGS + ["-o", LIB] + SOURCES
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
    subprocess.check_call(cmd, cwd=CSRC)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
