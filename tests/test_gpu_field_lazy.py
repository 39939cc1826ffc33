"""Device unit test of the Goldilocks primitives (gl_field.cuh) and the lazy butterfly arithmetic (gl_lazy.cuh).

tests/emu runs the host formulations of these functions; the device ones are PTX carry chains, and the lazy ones
exist on the host only as an __int128 restatement, so a carry or sign bug in the PTX is invisible there.
tests/cuda/field_lazy_device.cu runs the device code on edge operands and about 10^6 random ones, once per
arithmetic variant of gl_field.cuh, and the results are checked here with Python integers.

  - add sub neg mul sqr mul_add reduce96 reduce128 canon e2_mul, and mul_pow2 for every k in 0..95: congruent to the
    exact result mod p (neg and canon: the canonical value);
  - l3_add / l3_sub: the exact signed sum / difference;
  - l3_shift<S> for every S in 0..95 on values up to the documented input bound |v| < 2^94: congruent to v * 2^S and,
    for S > 0, inside the documented output bound |v| < 2^67 (S = 0 is the identity);
  - l3_norm at |e| up to 2^20 - 1;
  - dft_lazy<M>, M = 1..5, on square waves of 0 / 2^64 - 1 and all 2^64 - 1 against a naive DFT mod p, with the largest
    |e| before l3_norm under the 2^20 that l3_norm allows.
"""
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from conftest import EDGE, P, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cuda", "field_lazy_device.cu")
CSRC = os.path.join(ROOT, "plonky2_b200", "csrc")
VARIANTS = ["", "GL_MUL_EXPLICIT", "GL_SQR_3WIDE", "GL_REDUCE_V1"]
M64 = 2**64 - 1
NRANDOM = 1 << 20
# p + 2^32 does not fit in 64 bits
EDGE_SET = sorted(set(EDGE + [2**32 + 1, 2**63 - 1, 2**63 + 1, P - 2**32, 0xFFFFFFFF12345678, 0x12345678FFFFFFFF,
                              0x00000000FFFFFFFF, 0xFFFFFFFF00000000]))
L3_BOUND, NORM_E_BOUND, SHIFT_OUT_BOUND = 2**94, 2**20, 2**67


def nvcc_cmd(define, out, compile_only=False):
    """The library's NVCC_FLAGS without the shared-object flags (-shared, -Xcompiler -fPIC)."""
    from plonky2_b200.build import NVCC_FLAGS, nvcc_path

    flags, skip = [], False
    for i, f in enumerate(NVCC_FLAGS):
        if skip:
            skip = False
            continue
        if f == "-Xcompiler" and NVCC_FLAGS[i + 1] == "-fPIC":
            skip = True
            continue
        if f != "-shared":
            flags.append(f)
    cmd = [nvcc_path()] + flags + ["-I", CSRC] + (["-D" + define] if define else [])
    return cmd + (["-c"] if compile_only else []) + ["-o", out, SRC]


def _compile_all(tmp_path, compile_only):
    outs = [str(tmp_path / ("field_lazy_%s%s" % (v or "default", ".o" if compile_only else ""))) for v in VARIANTS]
    with ThreadPoolExecutor(max_workers=len(VARIANTS)) as ex:
        res = list(ex.map(lambda vo: subprocess.run(nvcc_cmd(vo[0], vo[1], compile_only), capture_output=True, text=True),
                          zip(VARIANTS, outs)))
    for v, r in zip(VARIANTS, res):
        assert r.returncode == 0, "variant %r: %s" % (v, r.stdout + r.stderr)
    return dict(zip(VARIANTS, outs))


def test_field_lazy_device_compiles_for_every_variant(tmp_path):
    """sm_90a compile of the device unit test with the default arithmetic and each -D variant (no device needed)."""
    try:
        from plonky2_b200.build import nvcc_path

        nvcc_path()
    except RuntimeError:
        pytest.skip("nvcc not available")
    _compile_all(tmp_path, compile_only=True)


# ----------------------------------------------------------------------------- operands and exact references
def _signed(u):
    u = int(u)
    return u - 2**64 if u >= 2**63 else u


def l3_words(v):
    """(w0, w1, e) of the signed value v (|v| < 2^95), e sign-extended to a u64 word."""
    return v & 0xFFFFFFFF, (v >> 32) & 0xFFFFFFFF, (v >> 64) & M64


def l3_value(w0, w1, e):
    return int(w0) + (int(w1) << 32) + _signed(e) * 2**64


def bitrev(x, bits):
    return int(format(x, "0%db" % bits)[::-1], 2) if bits else 0


def make_inputs():
    rng = np.random.default_rng(0xF1E1D)
    E = len(EDGE_SET)
    pairs = [(a, b, EDGE_SET[(i + 3 * j) % E], EDGE_SET[(5 * i + j) % E])
             for i, a in enumerate(EDGE_SET) for j, b in enumerate(EDGE_SET)]
    rnd = synth(0xF1, (NRANDOM, 4), canonical=False)
    # a quarter near 2^64 - 1, a quarter near p, the rest uniform
    q = NRANDOM // 4
    small = rnd[:q] & np.uint64(0xFFFF)
    rnd[:q, :2] = np.uint64(M64) - small[:, :2]
    rnd[q:2 * q, :2] = np.uint64(P) + (rnd[q:2 * q, :2] & np.uint64(0xFFFF)) - np.uint64(0x8000)
    pairs = np.concatenate([np.array(pairs, dtype=np.uint64), rnd])
    pow_words = np.concatenate([np.array(EDGE_SET, dtype=np.uint64), synth(0xF2, (4096,), canonical=False)])
    # lazy values for add / sub / shift: the bound 2^94 and just inside it, both signs, e = 0 and +-1 with extreme words
    lazy = []
    for s in (1, -1):
        lazy += [s * (L3_BOUND - 1), s * (L3_BOUND - 2**64), s * (L3_BOUND - 2**63 - 1), s * 2**93, s * (2**93 + 1)]
        for w in (0, 1, 2**32 - 1, 2**32, 2**63, P - 1, P, M64):
            lazy += [w, w + s * 2**64]
    lazy += [int(v) for v in rng.integers(-(2**62), 2**62, 8000)]
    lazy += [int(a) * 2**32 + int(b) for a, b in zip(rng.integers(-(2**61), 2**61, 16000), rng.integers(0, 2**32, 16000))]
    lazy = [v for v in lazy if abs(v) < L3_BOUND]
    norm = []
    for e in (0, 1, -1, NORM_E_BOUND - 1, -(NORM_E_BOUND - 1), NORM_E_BOUND // 2, -(NORM_E_BOUND // 2)):
        for w in (0, 1, 2**32 - 1, 2**32, P - 1, P, M64, 0xFFFFFFFF12345678):
            norm.append(e * 2**64 + w)
    norm += [int(e) * 2**64 + int(w) for e, w in zip(rng.integers(-(NORM_E_BOUND - 1), NORM_E_BOUND, 4000),
                                                      synth(0xF3, (4000,), canonical=False))]
    j = np.arange(32, dtype=np.uint64)
    dft = [np.full(32, M64, dtype=np.uint64), np.full(32, P - 1, dtype=np.uint64),
           np.resize(np.array(EDGE, dtype=np.uint64), 32)]
    for k in range(1, 6):
        sq = np.where((j >> np.uint64(k - 1)) & np.uint64(1), np.uint64(M64), np.uint64(0))
        dft += [sq, np.uint64(M64) - sq]
    dft += list(synth(0xF4, (2000, 32), canonical=False))
    dft = np.stack(dft)
    return pairs, pow_words, lazy, norm, dft


def write_inputs(path, pairs, pow_words, lazy, norm, dft):
    hdr = np.array([len(pairs), len(pow_words), len(lazy), len(norm), len(dft)], dtype=np.uint64)
    lz = np.array([l3_words(v) for v in lazy], dtype=np.uint64).reshape(-1)
    nm = np.array([l3_words(v) for v in norm], dtype=np.uint64).reshape(-1)
    np.concatenate([hdr, pairs.reshape(-1), pow_words, lz, nm, dft.reshape(-1)]).tofile(path)


@pytest.fixture(scope="module")
def reference():
    """Inputs and canonical expected values, computed once for every variant."""
    pairs, pow_words, lazy, norm, dft = make_inputs()
    A, B, Cc, D = (pairs[:, i].tolist() for i in range(4))
    exp = np.array([[(a + b) % P, (a - b) % P, (-a) % P, a * b % P, a * a % P, (a * b + c) % P,
                     (a + ((b & 0xFFFFFFFF) << 64)) % P, (a + (b << 64)) % P, a % P, (a * c + 7 * b * d) % P,
                     (a * d + b * c) % P] for a, b, c, d in zip(A, B, Cc, D)], dtype=np.uint64)
    pw = np.array([[x * (1 << k) % P for k in range(96)] for x in pow_words.tolist()], dtype=np.uint64)
    dft_exp = {}
    for m in range(1, 6):
        n = 1 << m
        w = pow(2, 192 >> m, P)  # dft_lazy's root: w_{2^M} = 2^(192 / 2^M)
        tw = [pow(w, t, P) for t in range(n)]
        X = [[sum(int(x[i]) * tw[i * k % n] for i in range(n)) % P for k in range(n)] for x in dft.tolist()]
        dft_exp[m] = np.array([[r[bitrev(j, m)] for j in range(n)] for r in X], dtype=np.uint64)
    return dict(pairs=pairs, pow_words=pow_words, lazy=lazy, norm=norm, dft=dft, exp=exp, pw=pw, dft_exp=dft_exp)


@pytest.fixture(scope="module")
def cuda_device():
    import torch

    if not torch.cuda.is_available():
        if os.environ.get("GL_REQUIRE_GPU") == "1":
            raise AssertionError("GPU tests need a CUDA device")
        pytest.skip("no CUDA device (gpu-marked tests run on an H100)")


@pytest.fixture(scope="module")
def device_runs(cuda_device, tmp_path_factory, reference):
    tmp = tmp_path_factory.mktemp("field_lazy")
    exes = _compile_all(tmp, compile_only=False)
    inp = str(tmp / "in.bin")
    r = reference
    write_inputs(inp, r["pairs"], r["pow_words"], r["lazy"], r["norm"], r["dft"])
    outs = {}
    for v, exe in exes.items():
        out = str(tmp / ("out_%s.bin" % (v or "default")))
        res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, "variant %r: %s" % (v, res.stdout + res.stderr)
        outs[v] = np.fromfile(out, dtype=np.uint64)
    return outs


def _first_bad(mask):
    bad = np.nonzero(~mask)[0]
    return None if not bad.size else int(bad[0])


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_field_and_lazy_primitives_on_device(cuda_device, reference, device_runs, variant):
    r = reference
    out = device_runs[variant]
    tag = "variant %s" % (variant or "default")
    np_, npow, nl, nn, nd = len(r["pairs"]), len(r["pow_words"]), len(r["lazy"]), len(r["norm"]), len(r["dft"])
    sizes = [11 * np_, 96 * npow, 6 * nl, 288 * nl, nn] + [s for m in range(1, 6) for s in (nd << m, nd)]
    assert len(out) == sum(sizes), tag
    parts = np.split(out, np.cumsum(sizes)[:-1])

    # field primitives: congruent mod p; neg and canon exactly canonical
    field = parts[0].reshape(np_, 11)
    names = ["add", "sub", "neg", "mul", "sqr", "mul_add", "reduce96", "reduce128", "canon", "e2_mul.c0", "e2_mul.c1"]
    for k, name in enumerate(names):
        got = field[:, k] if name in ("neg", "canon") else field[:, k] % np.uint64(P)
        i = _first_bad(got == r["exp"][:, k])
        assert i is None, "%s: %s(%s) = %#x, want %#x (mod p)" % (tag, name, ", ".join(hex(int(x)) for x in r["pairs"][i]),
                                                                  int(field[i, k]), int(r["exp"][i, k]))
    pw = parts[1].reshape(npow, 96) % np.uint64(P)
    bad = np.argwhere(pw != r["pw"])
    assert not bad.size, "%s: mul_pow2(%#x, %d)" % (tag, int(r["pow_words"][bad[0][0]]), bad[0][1])

    # lazy add / sub: exact
    lazy = r["lazy"]
    addsub = parts[2].reshape(nl, 2, 3).tolist()
    for i in range(nl):
        a, b = lazy[i], lazy[(i + 1) % nl]
        assert l3_value(*addsub[i][0]) == a + b, "%s: l3_add(%d, %d)" % (tag, a, b)
        assert l3_value(*addsub[i][1]) == a - b, "%s: l3_sub(%d, %d)" % (tag, a, b)
    # l3_shift<S>: congruent to v * 2^S; for S > 0 (S = 0 is the identity) |result| < 2^67
    sh = parts[3].reshape(nl, 96, 3).tolist()
    for i, v in enumerate(lazy):
        assert l3_value(*sh[i][0]) == v, "%s: l3_shift<0>(%d)" % (tag, v)
        for s in range(1, 96):
            o = l3_value(*sh[i][s])
            assert (o - v * (1 << s)) % P == 0 and abs(o) < SHIFT_OUT_BOUND, "%s: l3_shift<%d>(%d) = %d" % (tag, s, v, o)
    # l3_norm at |e| < 2^20
    for v, o in zip(r["norm"], parts[4].tolist()):
        assert (o - v) % P == 0, "%s: l3_norm(%d) = %#x" % (tag, v, o)

    # dft_lazy<M> vs a naive DFT mod p, and the largest |e| it produces
    k = 5
    for m in range(1, 6):
        got = parts[k].reshape(nd, 1 << m) % np.uint64(P)
        max_e = parts[k + 1]
        k += 2
        bad = np.argwhere(got != r["dft_exp"][m])
        assert not bad.size, "%s: dft_lazy<%d> input %d output %d" % (tag, m, bad[0][0], bad[0][1])
        assert int(max_e.max()) < NORM_E_BOUND, "%s: dft_lazy<%d> reached |e| = %d" % (tag, m, int(max_e.max()))
