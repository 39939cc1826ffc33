"""The device Poseidon under every build switch and launch budget, the library's Poseidon entry points at scale, Merkle
trees across the cooperative-level split, and proof-of-work grinding past one batch. Expected values come from the CPU
oracle (oracle/gl_oracle.cpp), which shares no code with the device.

1. tests/cuda/poseidon_device.cu includes gl_poseidon.cuh only and is built once per compile-time switch (VARIANTS),
   three of them also with GL_F64_TRACK recording the largest FP64 limb (TRACKED). Each build runs
   poseidon_permute_t<false> on about 2^20 states of the input classes of `poseidon_states`, and
   hash_or_noop_strided<true, true> on column-major leaf matrices under __launch_bounds__(128, 4) and (128, 5) with a
   partly dead last CTA, and hash_or_noop_strided<false> on the same rows. Every lane of every output is compared. The
   tracked builds also assert that no FP64 limb reaches 2^51, the bound of gl_poseidon.cuh's exactness argument.
2. PoseidonHash.permute_many / hash_many / hash_no_pad_many / two_to_one_many through the ABI (default build) on the
   same state set and on 2^18 rows per width.
3. Merkle trees through MerkleTree (row-major leaves) and PolynomialBatch.from_values (column-major LDE), every digest
   and the cap. tree_build hands a level whose node count fits the resident cooperative grid (4 CTAs x SMs x 128
   threads) to k_merkle_upper, which then finishes the tree, unless it is the level that writes the cap; otherwise the
   level runs k_merkle_level. On a 132-SM H100 (grid 67 584 threads):
     N = 2^16, 2^17        cap < log N - 1: straight to k_merkle_upper;  cap = log N - 1: k_merkle_level writes the cap
     N = 2^18              cap 0, 4: k_merkle_level for level 1, then k_merkle_upper;
                           cap log N - 2, log N - 1: k_merkle_level for every level, the last one writing the cap
     N = 2^20              cap 0, 4: k_merkle_level for levels 1-3, then k_merkle_upper;  cap log N - 2, log N - 1: as 2^18
   `merkle_split` computes this for the SM count at hand, and the tests check it against the library's launch count.
4. gl_fri_pow at 12 to 20 bits with seeds chosen on the CPU (oracle.pow_min_nonce) so that the smallest nonce lies in
   the first batch, in a later batch, or in the second grid-stride pass of its batch.
"""
import functools
import os
import re
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import gl_numpy as gn
from conftest import EDGE, P, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cuda", "poseidon_device.cu")
CSRC = os.path.join(ROOT, "plonky2_b200", "csrc")
M64 = 2**64 - 1
# compile-time switches of gl_poseidon.cuh / gl_field.cuh; "a+b" builds both
VARIANTS = ["default", "GL_SBOX_I2F", "GL_SBOX_SQR4", "GL_CVT_MAGIC", "GL_PARTIAL_FAST", "GL_MDS_INT", "GL_MUL_EXPLICIT",
            "GL_SQR_3WIDE", "GL_REDUCE_V1", "GL_SBOX_SQR4+GL_SBOX_I2F"]
TRACKED = ["tracked:default", "tracked:GL_SBOX_I2F", "tracked:GL_CVT_MAGIC"]
F64_LIMB_BOUND = 2.0**51
# leaf matrices of the harness: (W, N); N % 128 != 0 leaves the last CTA partly dead
HARNESS_MATRICES = [(3, 3005), (8, 20077), (9, 20033), (12, 8193), (17, 8291), (135, 2093)]
MDS_CIRC = [17, 15, 41, 16, 2, 28, 13, 13, 39, 18, 34, 20]
MDS_DIAG0 = 8


def defines(variant):
    tracked = variant.startswith("tracked:")
    v = variant.split(":", 1)[1] if tracked else variant
    d = [] if v == "default" else v.split("+")
    return (["POSEIDON_TRACK"] if tracked else []) + d


def nvcc_cmd(variant, out, compile_only=False):
    """The library's NVCC_FLAGS without the shared-object flags (-shared, -Xcompiler -fPIC), ptxas verbose."""
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
    cmd = [nvcc_path()] + flags + ["-Xptxas", "-v", "-I", CSRC] + ["-D" + d for d in defines(variant)]
    return cmd + (["-c"] if compile_only else []) + ["-o", out, SRC]


def _exe_name(variant):
    return "poseidon_" + re.sub(r"[^A-Za-z0-9]+", "_", variant)


def _compile_all(tmp_path, compile_only):
    variants = VARIANTS + TRACKED
    outs = [str(tmp_path / (_exe_name(v) + (".o" if compile_only else ""))) for v in variants]
    workers = max(1, min(len(variants), os.cpu_count() or 1))
    with ThreadPoolExecutor(max_workers=workers) as ex:
        res = list(ex.map(lambda vo: subprocess.run(nvcc_cmd(vo[0], vo[1], compile_only), capture_output=True, text=True),
                          zip(variants, outs)))
    for v, r in zip(variants, res):
        assert r.returncode == 0, "variant %s: %s" % (v, r.stdout + r.stderr)
    return dict(zip(variants, outs)), {v: r.stdout + r.stderr for v, r in zip(variants, res)}


def spills(ptxas_log):
    """{kernel: spill store bytes} from nvcc -Xptxas -v output."""
    out, fn = {}, None
    for line in ptxas_log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            fn = m.group(1)
        m = re.search(r"(\d+) bytes spill stores", line)
        if m and fn:
            out[fn] = int(m.group(1))
            fn = None
    return out


def test_poseidon_device_compiles_for_every_variant(tmp_path):
    """sm_90a compile of the device harness for every switch and the tracked builds (no device needed). Prints the
    spill stores of each leaf-hash budget: the MINB=5 instance spilled when this was written, so its spill path is part
    of what the device test runs."""
    try:
        from plonky2_b200.build import nvcc_path

        nvcc_path()
    except RuntimeError:
        pytest.skip("nvcc not available")
    _, logs = _compile_all(tmp_path, compile_only=True)
    for v in VARIANTS + TRACKED:
        s = spills(logs[v])
        assert "k_leaf_minb4" in s and "k_leaf_minb5" in s, "variant %s: no ptxas report for the leaf kernels" % v
        print("variant %-26s spill stores: k_leaf_minb4 %d B, k_leaf_minb5 %d B, k_permute %d B"
              % (v, s["k_leaf_minb4"], s["k_leaf_minb5"], s.get("k_permute", -1)))


# ----------------------------------------------------------------------------- inputs
@functools.lru_cache(maxsize=None)
def round_constants():
    """ALL_ROUND_CONSTANTS (poseidon.rs:59-157) as the device reads them, from gl_poseidon_constants.h."""
    text = open(os.path.join(CSRC, "gl_poseidon_constants.h")).read()
    body = re.search(r"GL_POSEIDON_RC\[360\]\s*=\s*\{(.*?)\};", text, re.S).group(1)
    rc = [int(x, 16) for x in re.findall(r"0x([0-9a-fA-F]+)ULL", body)]
    assert len(rc) == 360
    return rc


def _product_words(a, b):
    """The four 32-bit words of the exact 128-bit product a * b of u64 arrays, as int64 arrays (low word first)."""
    m, s = np.uint64(0xFFFFFFFF), np.uint64(32)
    with np.errstate(over="ignore"):
        a0, a1, b0, b1 = a & m, a >> s, b & m, b >> s
        p00, p01, p10, p11 = a0 * b0, a0 * b1, a1 * b0, a1 * b1
        t = (p00 >> s) + (p01 & m) + (p10 & m)
        t2 = (t >> s) + (p01 >> s) + (p10 >> s) + (p11 & m)
        return [w.astype(np.int64) for w in (p00 & m, t & m, t2 & m, (t2 >> s) + (p11 >> s))]


def sbox_limbs(x):
    """sbox7_f64's signed limb pair (L, H) of canonical S-box inputs x: with x^3 * x^4 = (p3 p2 p1 p0) in 32-bit words
    of canonical x^3, x^4, L = p0 - p2 - p3 and H = p1 + p2."""
    x2 = gn.mul(x, x)
    w0, w1, w2, w3 = _product_words(gn.mul(x, x2), gn.mul(x2, x2))
    return w0 - w2 - w3, w1 + w2


def sbox_limbs_exact(x):
    x2 = x * x % P
    prod = (x * x2 % P) * (x2 * x2 % P)
    w = [(prod >> (32 * k)) & 0xFFFFFFFF for k in range(4)]
    return w[0] - w[2] - w[3], w[1] + w[2]


ADV_POOL = 1024
ADV_L_BOUND = 2**33 - 2**31  # every lane of an adversarial L state has L below -ADV_L_BOUND
ADV_H_BOUND = 2**33 - 2**28  # every lane of an adversarial H state has H above ADV_H_BOUND


@functools.lru_cache(maxsize=None)
def adversarial_targets():
    """First-round S-box inputs x with extreme sbox7_f64 limbs, from a vectorised search over 2^22 random x: the
    ADV_POOL most negative L (p0 near 0, p2 and p3 near 2^32) and the ADV_POOL largest H (p1 and p2 near 2^32)."""
    rng = np.random.default_rng(0xAD5B0C)
    xl, ll, xh, hh = [], [], [], []
    for _ in range(4):
        x = rng.integers(0, P, size=1 << 20, dtype=np.uint64)
        L, H = sbox_limbs(x)
        il, ih = np.argsort(L)[:ADV_POOL], np.argsort(H)[-ADV_POOL:]
        xl.append(x[il]), ll.append(L[il]), xh.append(x[ih]), hh.append(H[ih])
    xl, ll, xh, hh = (np.concatenate(a) for a in (xl, ll, xh, hh))
    return xl[np.argsort(ll)[:ADV_POOL]], xh[np.argsort(hh)[-ADV_POOL:]]


def adversarial_states(n, kind, seed, lanes=12):
    """n states whose first-round S-box inputs x_i = s_i + rc_i are all extreme of one kind ("L" or "H") in lanes
    0..lanes-1 (the other lanes are 0): s_i = x_i - rc_i (mod p)."""
    xl, xh = adversarial_targets()
    pool = xl if kind == "L" else xh
    rng = np.random.default_rng(seed)
    x = pool[rng.integers(0, len(pool), size=(n, lanes))]
    rc = np.array(round_constants()[:lanes], dtype=np.uint64)
    st = np.zeros((n, 12), dtype=np.uint64)
    st[:, :lanes] = gn.sub(x, rc)
    return st


def _classes(parts):
    states, classes, at = [], [], 0
    for name, a in parts:
        a = np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 12)
        states.append(a)
        classes.append((name, at, at + len(a)))
        at += len(a)
    return np.concatenate(states), classes


@functools.lru_cache(maxsize=None)
def poseidon_states():
    """About 2^20 12-lane states in named classes -> (states, [(class, first, end)])."""
    rng = np.random.default_rng(0x905E1D)
    edge = np.array(EDGE, dtype=np.uint64)
    small = lambda shape: rng.integers(0, 1 << 16, size=shape, dtype=np.uint64)  # noqa: E731
    one_lane = np.zeros((12 * 24, 12), dtype=np.uint64)
    vals = list(EDGE) + [int(v) for v in synth(0x9E2, (12,), canonical=False)]
    for lane in range(12):
        for k, v in enumerate(vals):
            one_lane[24 * lane + k, lane] = v
    capacity = np.zeros((1 << 14, 12), dtype=np.uint64)
    capacity[:, 8:] = synth(0x9E3, (1 << 14, 4), canonical=False)
    capacity[::2, 8:] = edge[rng.integers(0, len(edge), size=((1 << 13), 4))]
    chains = []
    for c in range(16):
        s = synth(0x9E4 + c, (1, 12), canonical=False)
        for _ in range(64):
            chains.append(s[0])
            s = _oracle().poseidon_many(s)
    parts = [
        ("edge words in every lane", edge[rng.integers(0, len(edge), size=(1 << 14, 12))]),
        ("edge words, cyclic", np.array([[EDGE[(i + 5 * l) % len(EDGE)] for l in range(12)] for i in range(len(EDGE))],
                                        dtype=np.uint64)),
        ("both halves near 2^32", synth(0x9E5, (1 << 16, 12), canonical=False) | np.uint64(0xFFFFFFF0FFFFFFF0)),
        ("2^64 - 1 - small", np.uint64(M64) - small((1 << 15, 12))),
        ("p + small", np.uint64(P) + (small((1 << 15, 12)) & np.uint64(0xFFF))),
        ("p - small", np.uint64(P) - np.uint64(1) - small((1 << 15, 12))),
        ("all zero", np.zeros((1, 12), dtype=np.uint64)),
        ("all p - 1", np.full((1, 12), P - 1, dtype=np.uint64)),
        ("one nonzero lane", one_lane),
        ("capacity lanes 8-11 nonzero", capacity),
        ("chains of 64 permutations", np.array(chains)),
        ("adversarial first-round L", adversarial_states(1 << 15, "L", 0xA1)),
        ("adversarial first-round H", adversarial_states(1 << 15, "H", 0xA2)),
    ]
    used = sum(len(np.asarray(a).reshape(-1, 12)) for _, a in parts)
    parts.insert(0, ("random non-canonical", synth(0x9E1, ((1 << 20) - used, 12), canonical=False)))
    return _classes(parts)


def leaf_rows(n, W, seed):
    """n leaves of width W: random non-canonical words, with edge words, near-2^32 halves, all 2^64 - 1 and (first 8
    elements = the first permutation's lanes 0-7) adversarial first-round inputs mixed in at spread-out rows."""
    rows = synth(seed, (n, W), canonical=False)
    rng = np.random.default_rng(seed)
    edge = np.array(EDGE, dtype=np.uint64)
    rows[1::16] = edge[rng.integers(0, len(edge), size=rows[1::16].shape)]
    rows[3::16] |= np.uint64(0xFFFFFFF0FFFFFFF0)
    rows[5::16] = np.uint64(M64)
    lanes = min(W, 8)
    for off, kind in ((7, "L"), (9, "H")):
        rows[off::16, :lanes] = adversarial_states(len(rows[off::16]), kind, seed + off, lanes=8)[:, :lanes]
    return rows


def expected_no_pad(oracle, rows):
    """hash_no_pad of every row: the sponge for W > 4 is hash_or_noop; for W <= 4 one permutation of [row, 0, ...]."""
    n, W = rows.shape
    if W > 4:
        return oracle.hash_many(rows)
    st = np.zeros((n, 12), dtype=np.uint64)
    st[:, :W] = rows
    return oracle.poseidon_many(st)[:, :4]


def _oracle():
    import oracle_lib

    oracle_lib.lib()
    return oracle_lib


def test_adversarial_states_reach_the_intended_first_round_limbs():
    """The adversarial classes, checked with exact Python integers: round 1's S-box input x_i = s_i + rc_i gives
    |L| > 2^33 - 2^31 (or H > 2^33 - 2^28) in every lane, with one sign, so that the circulant row sums reach
    264 * |L|; the vectorised limbs agree with the exact ones."""
    rc = round_constants()[:12]
    row_sum = MDS_CIRC[0] + MDS_DIAG0 + sum(MDS_CIRC[1:])
    assert row_sum == 264
    for kind in ("L", "H"):
        st = adversarial_states(256, kind, 0xC0 + ord(kind))
        worst = []
        for i, s in enumerate(st.tolist()):
            limbs = [sbox_limbs_exact((s[l] + rc[l]) % P) for l in range(12)]
            for l, (L, H) in enumerate(limbs):
                if kind == "L":
                    assert L < -ADV_L_BOUND, "adversarial L state %d lane %d: L = %d" % (i, l, L)
                else:
                    assert H > ADV_H_BOUND, "adversarial H state %d lane %d: H = %d" % (i, l, H)
            v = [L if kind == "L" else H for L, H in limbs]
            rows = [abs(sum((MDS_CIRC[(j - r) % 12] + (MDS_DIAG0 if r == j == 0 else 0)) * v[j] for j in range(12)))
                    for r in range(12)]
            worst.append(max(rows))
            assert min(rows) > 256 * (ADV_L_BOUND if kind == "L" else ADV_H_BOUND), (kind, i)
        print("adversarial %s: largest first-round MDS row sum 2^%.3f (264 * 2^33 = 2^%.3f)"
              % (kind, np.log2(max(worst)), np.log2(264 * 2.0**33)))
    # the vectorised search arithmetic against exact integers
    x = np.concatenate(adversarial_targets() + (synth(0xC3, (4096,)),))
    L, H = sbox_limbs(x)
    for i in range(0, len(x), 7):
        assert (int(L[i]), int(H[i])) == sbox_limbs_exact(int(x[i])), int(x[i])


# ----------------------------------------------------------------------------- device harness, every switch
@pytest.fixture(scope="module")
def cuda_device():
    import torch

    if not torch.cuda.is_available():
        if os.environ.get("GL_REQUIRE_GPU") == "1":
            raise AssertionError("GPU tests need a CUDA device")
        pytest.skip("no CUDA device (gpu-marked tests run on an H100)")
    return torch.cuda.get_device_properties(0)


@pytest.fixture(scope="module")
def state_set(oracle):
    states, classes = poseidon_states()
    return dict(states=states, classes=classes, expected=oracle.poseidon_many(states))


@pytest.fixture(scope="module")
def harness_runs(cuda_device, tmp_path_factory, state_set, oracle):
    tmp = tmp_path_factory.mktemp("poseidon_device")
    exes, _ = _compile_all(tmp, compile_only=False)
    mats = [leaf_rows(n, W, 0x700 + W) for W, n in HARNESS_MATRICES]
    words = [np.array([len(state_set["states"]), len(mats)], dtype=np.uint64), state_set["states"].reshape(-1)]
    for m in mats:
        words += [np.array([m.shape[1], m.shape[0]], dtype=np.uint64), m.reshape(-1)]
    inp = str(tmp / "in.bin")
    np.concatenate(words).tofile(inp)
    expected = [(oracle.hash_many(m), expected_no_pad(oracle, m)) for m in mats]
    outs = {}
    for v, exe in exes.items():
        out = str(tmp / ("out_%s.bin" % _exe_name(v)))
        r = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, "variant %s: %s" % (v, r.stdout + r.stderr)
        outs[v] = out
    return dict(outs=outs, mats=mats, expected=expected)


def _first_bad(got, want):
    bad = np.argwhere(got != want)
    return None if not bad.size else tuple(int(b) for b in bad[0])


def check_states(tag, got, state_set):
    """Every lane of every permuted state; the message names the class, the state and the lane."""
    want = state_set["expected"]
    assert got.shape == want.shape, tag
    for name, lo, hi in state_set["classes"]:
        b = _first_bad(got[lo:hi], want[lo:hi])
        if b is not None:
            i, lane = lo + b[0], b[1]
            raise AssertionError("%s, class %r: state %d lane %d = %#x, want %#x (input %s)"
                                 % (tag, name, i, lane, int(got[i, lane]), int(want[i, lane]),
                                    [hex(int(w)) for w in state_set["states"][i]]))


def check_digests(tag, got, want):
    b = _first_bad(got, want)
    assert b is None, "%s: leaf %d lane %d = %#x, want %#x" % (tag, b[0], b[1], int(got[b]), int(want[b]))


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS + TRACKED)
def test_device_poseidon_variant(cuda_device, state_set, harness_runs, variant):
    out = np.fromfile(harness_runs["outs"][variant], dtype=np.uint64)
    ns = len(state_set["states"])
    sizes = [12 * ns] + [4 * n for _, n in HARNESS_MATRICES for _ in range(3)]
    launches = [ns] + [n for _, n in HARNESS_MATRICES for _ in range(3)]
    slots = [-(-n // 128) * 128 for n in launches] if variant in TRACKED else []
    assert len(out) == sum(sizes) + sum(slots), "variant %s: %d output words" % (variant, len(out))
    parts = np.split(out, np.cumsum(sizes + slots)[:-1])
    check_states("variant %s, poseidon_permute_t" % variant, parts[0].reshape(ns, 12), state_set)
    k = 1
    for (W, n), (want_noop, want_no_pad) in zip(HARNESS_MATRICES, harness_runs["expected"]):
        for kernel, want in (("leaf hash MINB=4", want_noop), ("leaf hash MINB=5", want_noop), ("hash_no_pad", want_no_pad)):
            check_digests("variant %s, %s, W=%d N=%d" % (variant, kernel, W, n), parts[k].reshape(n, 4), want)
            k += 1
    if variant in TRACKED:
        names = ["poseidon_permute_t"] + ["%s W=%d" % (kn, W) for W, _ in HARNESS_MATRICES
                                          for kn in ("leaf hash MINB=4", "leaf hash MINB=5", "hash_no_pad")]
        maxima = [float(parts[k + i].view(np.float64).max()) for i in range(len(slots))]
        top = max(maxima)
        print("variant %s: largest FP64 limb 2^%.2f (bound 2^51)" % (variant, np.log2(top)))
        for name, m in zip(names, maxima):
            assert m < F64_LIMB_BOUND, "variant %s, %s: an FP64 limb reached 2^%.2f" % (variant, name, np.log2(m))
        # GL_FP64_PATH builds only: the FP64 partial rounds hold limbs far above 2^32
        assert top > 2.0**40, "variant %s: the FP64 limbs were not tracked" % variant


# ----------------------------------------------------------------------------- the library's entry points at scale
@pytest.fixture(scope="module")
def pb(cuda_device):
    import plonky2_b200 as p

    p.default_context()  # fails loudly if the CUDA extension is missing
    return p


@pytest.mark.gpu
def test_permute_many_every_lane(pb, state_set):
    got = pb.PoseidonHash.permute_many(state_set["states"])
    check_states("PoseidonHash.permute_many", got, state_set)


HASH_ROWS = 1 << 18


@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 4, 5, 8, 9, 12, 16, 17, 135])
def test_hash_entry_points_2pow18_rows(pb, oracle, W):
    rows = leaf_rows(HASH_ROWS, W, 0x800 + W)
    check_digests("hash_many W=%d" % W, pb.PoseidonHash.hash_many(rows), oracle.hash_many(rows))
    check_digests("hash_no_pad_many W=%d" % W, pb.PoseidonHash.hash_no_pad_many(rows), expected_no_pad(oracle, rows))


@pytest.mark.gpu
def test_two_to_one_many_2pow18_pairs(pb, oracle):
    pairs = leaf_rows(HASH_ROWS, 8, 0x900)
    st = np.zeros((HASH_ROWS, 12), dtype=np.uint64)
    st[:, :8] = pairs
    check_digests("two_to_one_many", pb.PoseidonHash.two_to_one_many(pairs), oracle.poseidon_many(st)[:, :4])


# ----------------------------------------------------------------------------- Merkle trees across the kernel split
def merkle_split(N, cap_height, sm_count, ctas_per_sm=4):
    """tree_build's kernels for N leaves: (number of k_merkle_level launches, whether k_merkle_upper finishes)."""
    log_n = N.bit_length() - 1
    sub_log = log_n - cap_height
    coop = ctas_per_sm * sm_count * 128
    levels = 0
    for i in range(1, sub_log + 1):
        if (N >> i) <= coop and i < sub_log:
            return levels, True
        levels += 1
    return levels, False


def split_name(levels, upper):
    if not levels:
        return "k_merkle_upper only" if upper else "leaf hash only"
    return "k_merkle_level x%d%s" % (levels, " + k_merkle_upper" if upper else ", the last one writing the cap")


def digest_where(idx, N, cap_height):
    """(cap subtree, layer, node) of digest row idx in the reference layout (merkle_tree.rs:176-187)."""
    L = N >> cap_height
    c, pos = divmod(idx, 2 * (L - 1))
    t = pos // 2 + 1
    layer = (t & -t).bit_length() - 1
    return c, layer, 2 * (t >> (layer + 1)) + (pos & 1)


def check_tree(tag, N, cap_height, digests, cap, want_digests, want_cap):
    b = _first_bad(digests, want_digests)
    if b is not None:
        c, layer, q = digest_where(b[0], N, cap_height)
        raise AssertionError("%s: digest %d (cap subtree %d, layer %d, node %d) lane %d = %#x, want %#x"
                             % (tag, b[0], c, layer, q, b[1], int(digests[b]), int(want_digests[b])))
    b = _first_bad(cap, want_cap)
    assert b is None, "%s: cap entry %d lane %d = %#x, want %#x" % (tag, b[0], b[1], int(cap[b]), int(want_cap[b]))


# (log N, W, cap height): every N with cap heights 0, 4, log N - 2 and log N - 1, the widths spread over them
MERKLE_ROW_MAJOR = [(16, 135, 0), (16, 1, 4), (16, 5, 14), (16, 9, 15),
                    (17, 8, 0), (17, 9, 4), (17, 1, 15), (17, 5, 16),
                    (18, 5, 0), (18, 8, 4), (18, 9, 16), (18, 1, 17),
                    (20, 9, 0), (20, 5, 4), (20, 8, 18), (20, 1, 19)]
# (log N, B, rate bits, cap height) of PolynomialBatch.from_values, N = n << rate bits leaves
MERKLE_COLUMN_MAJOR = [(16, 135, 3, 4), (16, 9, 2, 15), (17, 5, 2, 16), (17, 8, 1, 0), (18, 9, 3, 4), (18, 1, 1, 17),
                       (20, 8, 1, 0), (20, 9, 2, 18), (20, 5, 1, 19)]


@pytest.mark.gpu
@pytest.mark.parametrize("log_n,W,h", MERKLE_ROW_MAJOR)
def test_merkle_tree_every_digest(pb, oracle, cuda_device, log_n, W, h):
    N = 1 << log_n
    levels, upper = merkle_split(N, h, cuda_device.multi_processor_count)
    tag = "MerkleTree N=2^%d W=%d cap %d (%s)" % (log_n, W, h, split_name(levels, upper))
    leaves = leaf_rows(N, W, 0xA00 + log_n * 7 + h)
    ctx = pb.default_context()
    before = ctx.launch_count
    t = pb.MerkleTree(leaves, h)
    # one leaf-hash launch, then the level launches and the cooperative launch the split predicts
    assert ctx.launch_count - before == 1 + levels + int(upper), tag
    d, cap = oracle.merkle_build(leaves, h)
    check_tree(tag, N, h, t.digests, t.cap.hashes, d, cap)
    t.close()


@pytest.mark.gpu
@pytest.mark.parametrize("log_N,B,r,h", MERKLE_COLUMN_MAJOR)
def test_from_values_tree_every_digest(pb, oracle, cuda_device, log_N, B, r, h):
    N = 1 << log_N
    tag = "from_values N=2^%d B=%d rate %d cap %d (%s)" % (log_N, B, r, h,
                                                         split_name(*merkle_split(N, h, cuda_device.multi_processor_count)))
    vals = synth(0xB00 + log_N * 7 + h, (B, N >> r), canonical=False)
    c = pb.PolynomialBatch.from_values(vals, r, False, h)
    o = oracle.Commit(vals, r, h)
    check_tree(tag, N, h, c.merkle_tree.digests, c.merkle_tree.cap.hashes, o.digests, o.cap)
    c.close()


@pytest.mark.gpu
def test_merkle_openings_every_leaf_2pow16_canonical(pb, oracle):
    N, W, h = 1 << 16, 9, 4
    leaves = leaf_rows(N, W, 0xC00)
    t = pb.MerkleTree(leaves, h)
    d, cap = oracle.merkle_build(leaves, h)
    lv, paths = t.open_many(np.arange(N))
    # opened leaves are outputs: the canonical forms of the (non-canonical) leaf words
    check_digests("opened leaves", lv, np.where(leaves >= np.uint64(P), leaves - np.uint64(P), leaves))
    # every opening verifies against the oracle's cap; a sample of sibling paths equals the oracle's
    for i in range(N):
        assert oracle.merkle_verify(lv[i], i, paths[i], cap, h), "leaf %d: the opening does not verify" % i
    for i in range(0, N, 4099):
        assert np.array_equal(paths[i], oracle.merkle_prove(i, N, h, d)), "leaf %d" % i
    t.close()


@pytest.mark.gpu
def test_merkle_openings_random_2pow20_canonical(pb, oracle):
    N, W, h = 1 << 20, 8, 4
    leaves = leaf_rows(N, W, 0xC01)
    t = pb.MerkleTree(leaves, h)
    d, cap = oracle.merkle_build(leaves, h)
    idx = np.random.default_rng(0xC02).integers(0, N, size=4096)
    lv, paths = t.open_many(idx)
    canon = np.where(leaves >= np.uint64(P), leaves - np.uint64(P), leaves)
    for k, i in enumerate(idx.tolist()):
        assert np.array_equal(lv[k], canon[i]), "leaf %d" % i
        want = oracle.merkle_prove(i, N, h, d)
        b = _first_bad(paths[k], want)
        assert b is None, "leaf %d: sibling at layer %d lane %d" % (i, b[0], b[1])
    t.close()


# ----------------------------------------------------------------------------- proof-of-work past one batch
def pow_batches(bits):
    """gl_fri_pow's batches (start, count): 2 << min(bits, 24) candidates, at least 4096, growing 4x up to 2^24."""
    batch, start = max(4096, 2 << min(bits, 24)), 0
    while True:
        yield start, batch
        start += batch
        batch = batch * 4 if batch < (1 << 24) else batch


def locate(nonce, bits):
    """(batch index, offset in the batch, batch size) of a nonce."""
    for k, (start, count) in enumerate(pow_batches(bits)):
        if nonce < start + count:
            return k, nonce - start, count


def pow_state(seed, pos):
    """A transcript state with words that are not canonical (gl_fri_pow canonicalises them)."""
    st = synth(0xD00 + seed, (12,), canonical=False)
    st[(pos + 1) % 12] = np.uint64(P + seed)
    st[(pos + 5) % 12] = np.uint64(M64 - seed)
    return st


POW_BITS = [12, 16, 17, 18, 20]
POW_POS_BASE = {12: 0, 16: 2, 17: 4, 18: 7, 20: 10}  # lane pos = base + case index (mod 8): every pos 0..7 is used


def device_pow(pb, st, pos, bits):
    ctx = pb.default_context()
    nonce = np.zeros(1, dtype=np.uint64)
    pb._native.check(pb._native.lib().gl_fri_pow(ctx.h, pb._native.np_ptr(st), pos, bits, pb._native.np_ptr(nonce)),
                     ctx.h)
    return int(nonce[0])


@pytest.mark.gpu
@pytest.mark.parametrize("bits", POW_BITS)
def test_fri_pow_smallest_nonce_past_one_batch(pb, oracle, cuda_device, bits):
    grid_pass = cuda_device.multi_processor_count * 8 * 128  # k_fri_pow's grid: 8 CTAs of 128 per SM
    batches = pow_batches(bits)
    b0, b1 = next(batches), next(batches)
    limit = b1[0] + b1[1]  # the first two batches
    cases = [("first batch", lambda k, off, cnt: k == 0),
             ("a later batch", lambda k, off, cnt: k >= 1)]
    if bits >= 17:
        # only the grid-stride loop visits these candidates
        cases.append(("the second grid pass of its batch", lambda k, off, cnt: grid_pass <= off < min(2 * grid_pass, cnt)))
    for ci, (name, want_case) in enumerate(cases):
        pos = (POW_POS_BASE[bits] + ci) % 8
        for seed in range(400):
            st = pow_state(seed * 16 + ci, pos)
            want = oracle.pow_min_nonce(st, pos, bits, limit)
            if want != oracle.NO_NONCE and want_case(*locate(want, bits)):
                break
        else:
            raise AssertionError("%d bits: no seed puts the smallest nonce in %s" % (bits, name))
        got = device_pow(pb, st, pos, bits)
        k, off, cnt = locate(want, bits)
        assert got == want, ("%d bits, pos %d, smallest nonce in %s (batch %d, offset %d of %d, grid pass %d): "
                             "device %d, oracle %d" % (bits, pos, name, k, off, cnt, grid_pass, got, want))
        s = st.copy()
        s[pos] = got
        resp = int(oracle.poseidon(s)[7])
        assert 64 - resp.bit_length() >= bits, "%d bits: response %#x" % (bits, resp)


@pytest.mark.gpu
def test_fri_pow_zero_bits_is_nonce_zero(pb):
    for seed in range(3):
        assert device_pow(pb, pow_state(seed, seed), seed, 0) == 0
