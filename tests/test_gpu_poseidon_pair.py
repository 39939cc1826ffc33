"""The device Poseidon built with the partial-round pair's former form (-DGL_PAIR_RENORM_F64), plain and with
GL_F64_TRACK, through the harness of test_gpu_poseidon.py (tests/cuda/poseidon_device.cu): every lane of about 2^20
permuted states and every digest of the leaf matrices against the CPU oracle, and in the tracked build no FP64 limb
at or above 2^51. The default build, whose pair renormalises its limbs through the integer pipes, is covered there."""
import subprocess

import numpy as np
import pytest

import test_gpu_poseidon as tp
from test_gpu_poseidon import cuda_device, state_set  # noqa: F401  (fixtures)

PAIR_VARIANTS = ["GL_PAIR_RENORM_F64", "tracked:GL_PAIR_RENORM_F64"]


def _compile(tmp_path, variants, compile_only):
    outs, logs = {}, {}
    for v in variants:
        out = str(tmp_path / (tp._exe_name(v) + (".o" if compile_only else "")))
        r = subprocess.run(tp.nvcc_cmd(v, out, compile_only), capture_output=True, text=True)
        assert r.returncode == 0, "variant %s: %s" % (v, r.stdout + r.stderr)
        outs[v], logs[v] = out, r.stdout + r.stderr
    return outs, logs


def test_former_pair_compiles_without_leaf_hash_spills(tmp_path):
    try:
        from plonky2_b200.build import nvcc_path

        nvcc_path()
    except RuntimeError:
        pytest.skip("nvcc not available")
    _, logs = _compile(tmp_path, ["default", "GL_PAIR_RENORM_F64"], compile_only=True)
    for v, log in logs.items():
        s = tp.spills(log)
        assert s.get("k_leaf_minb4") == 0, "variant %s: k_leaf_minb4 spills %s B" % (v, s.get("k_leaf_minb4"))


@pytest.mark.gpu
def test_device_poseidon_former_pair(cuda_device, state_set, oracle, tmp_path):  # noqa: F811
    exes, _ = _compile(tmp_path, PAIR_VARIANTS, compile_only=False)
    mats = [tp.leaf_rows(n, W, 0x700 + W) for W, n in tp.HARNESS_MATRICES]
    words = [np.array([len(state_set["states"]), len(mats)], dtype=np.uint64), state_set["states"].reshape(-1)]
    for m in mats:
        words += [np.array([m.shape[1], m.shape[0]], dtype=np.uint64), m.reshape(-1)]
    inp = str(tmp_path / "in.bin")
    np.concatenate(words).tofile(inp)
    expected = [(oracle.hash_many(m), tp.expected_no_pad(oracle, m)) for m in mats]
    ns = len(state_set["states"])
    sizes = [12 * ns] + [4 * n for _, n in tp.HARNESS_MATRICES for _ in range(3)]
    launches = [ns] + [n for _, n in tp.HARNESS_MATRICES for _ in range(3)]
    for v, exe in exes.items():
        out_path = str(tmp_path / ("out_%s.bin" % tp._exe_name(v)))
        r = subprocess.run([exe, inp, out_path], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, "variant %s: %s" % (v, r.stdout + r.stderr)
        out = np.fromfile(out_path, dtype=np.uint64)
        tracked = v.startswith("tracked:")
        slots = [-(-n // 128) * 128 for n in launches] if tracked else []
        assert len(out) == sum(sizes) + sum(slots), "variant %s: %d output words" % (v, len(out))
        parts = np.split(out, np.cumsum(sizes + slots)[:-1])
        tp.check_states("variant %s, poseidon_permute_t" % v, parts[0].reshape(ns, 12), state_set)
        k = 1
        for (W, n), (want_noop, want_no_pad) in zip(tp.HARNESS_MATRICES, expected):
            for kernel, want in (("leaf hash MINB=4", want_noop), ("leaf hash MINB=5", want_noop),
                                 ("hash_no_pad", want_no_pad)):
                tp.check_digests("variant %s, %s, W=%d N=%d" % (v, kernel, W, n), parts[k].reshape(n, 4), want)
                k += 1
        if tracked:
            top = max(float(parts[k + i].view(np.float64).max()) for i in range(len(slots)))
            print("variant %s: largest FP64 limb 2^%.2f (bound 2^51)" % (v, np.log2(top)))
            assert 2.0**40 < top < tp.F64_LIMB_BOUND, "variant %s: largest FP64 limb 2^%.2f" % (v, np.log2(top))
