"""The device Poseidon with the full round's former hand-overs restored (-DGL_SBOX_MOVE_HANDOVER, -DGL_RET_REDUCE96,
both), built from tests/cuda/poseidon_device.cu like test_gpu_poseidon.py's switches: every lane of about 2^20
permuted states and every digest of the leaf-hash harness (launch budgets 4 and 5, hash_no_pad) against the oracle.
The default build, with the new forms, is test_gpu_poseidon.py's "default" and "tracked:default"."""
import subprocess

import numpy as np
import pytest

import test_gpu_poseidon as tgp
from test_gpu_poseidon import cuda_device, state_set  # noqa: F401  (fixtures)

SWITCHES = ["GL_SBOX_MOVE_HANDOVER", "GL_RET_REDUCE96", "GL_SBOX_MOVE_HANDOVER+GL_RET_REDUCE96"]


@pytest.fixture(scope="module")
def runs(cuda_device, tmp_path_factory, state_set, oracle):  # noqa: F811
    tmp = tmp_path_factory.mktemp("poseidon_handover")
    mats = [tgp.leaf_rows(n, W, 0x700 + W) for W, n in tgp.HARNESS_MATRICES]
    words = [np.array([len(state_set["states"]), len(mats)], dtype=np.uint64), state_set["states"].reshape(-1)]
    for m in mats:
        words += [np.array([m.shape[1], m.shape[0]], dtype=np.uint64), m.reshape(-1)]
    inp = str(tmp / "in.bin")
    np.concatenate(words).tofile(inp)
    outs = {}
    for v in SWITCHES:
        exe = str(tmp / tgp._exe_name(v))
        r = subprocess.run(tgp.nvcc_cmd(v, exe), capture_output=True, text=True)
        assert r.returncode == 0, "switch %s: %s" % (v, r.stdout + r.stderr)
        out = str(tmp / ("out_%s.bin" % tgp._exe_name(v)))
        r = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, "switch %s: %s" % (v, r.stdout + r.stderr)
        outs[v] = out
    expected = [(oracle.hash_many(m), tgp.expected_no_pad(oracle, m)) for m in mats]
    return dict(outs=outs, expected=expected)


@pytest.mark.gpu
@pytest.mark.parametrize("switch", SWITCHES)
def test_device_poseidon_handover_switch(cuda_device, state_set, runs, switch):  # noqa: F811
    out = np.fromfile(runs["outs"][switch], dtype=np.uint64)
    ns = len(state_set["states"])
    sizes = [12 * ns] + [4 * n for _, n in tgp.HARNESS_MATRICES for _ in range(3)]
    assert len(out) == sum(sizes), "switch %s: %d output words" % (switch, len(out))
    parts = np.split(out, np.cumsum(sizes)[:-1])
    tgp.check_states("switch %s, poseidon_permute_t" % switch, parts[0].reshape(ns, 12), state_set)
    k = 1
    for (W, n), (want_noop, want_no_pad) in zip(tgp.HARNESS_MATRICES, runs["expected"]):
        for kernel, want in (("leaf hash MINB=4", want_noop), ("leaf hash MINB=5", want_noop),
                             ("hash_no_pad", want_no_pad)):
            tgp.check_digests("switch %s, %s, W=%d N=%d" % (switch, kernel, W, n), parts[k].reshape(n, 4), want)
            k += 1
