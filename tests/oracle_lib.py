"""ctypes binding of the CPU parity oracle (oracle/libgl_oracle.so).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's CPU-baseline
legs. The product package (plonky2_b200/) never imports this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
LIB_PATH = os.path.join(ORACLE_DIR, "libgl_oracle.so")
P = 0xFFFFFFFF00000001

u64 = C.c_uint64
u64p = C.POINTER(C.c_uint64)
u32p = C.POINTER(C.c_uint32)


def build_oracle():
    """Compile the oracle if the shared object is missing or stale."""
    deps = [os.path.join(ORACLE_DIR, f) for f in ("gl_oracle.cpp", "gl_oracle.h", "gl_poseidon_constants.h", "Makefile")]
    if os.path.exists(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(p) for p in deps):
        return LIB_PATH
    subprocess.check_call(["make", "-C", ORACLE_DIR, "libgl_oracle.so"], stdout=subprocess.DEVNULL)
    return LIB_PATH


class FriParams(C.Structure):
    _fields_ = [
        ("rate_bits", C.c_uint32),
        ("cap_height", C.c_uint32),
        ("proof_of_work_bits", C.c_uint32),
        ("num_query_rounds", C.c_uint32),
        ("num_reductions", C.c_uint32),
        ("reduction_arity_bits", C.c_uint32 * 32),
    ]


class FriInstance(C.Structure):
    pass


class FriBatch(C.Structure):
    _fields_ = [
        ("point", C.c_uint64 * 2),
        ("num_polys", C.c_size_t),
        ("oracle_index", u32p),
        ("poly_index", u32p),
    ]


FriInstance._fields_ = [("batches", C.POINTER(FriBatch)), ("n_batches", C.c_size_t)]

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    build_oracle()
    L = C.CDLL(LIB_PATH)
    for name in ("glo_canon", "glo_neg", "glo_inv"):
        getattr(L, name).restype = u64
        getattr(L, name).argtypes = [u64]
    for name in ("glo_add", "glo_sub", "glo_mul", "glo_exp"):
        getattr(L, name).restype = u64
        getattr(L, name).argtypes = [u64, u64]
    L.glo_primitive_root_of_unity.restype = u64
    L.glo_primitive_root_of_unity.argtypes = [C.c_uint32]
    L.glo_inverse_2exp.restype = u64
    L.glo_inverse_2exp.argtypes = [C.c_uint32]
    L.glo_coset_shift.restype = u64
    L.glo_ext2_mul.argtypes = [u64p, u64p, u64p]
    L.glo_ext2_inv.argtypes = [u64p, u64p]
    L.glo_reverse_bits.restype = u64
    L.glo_reverse_bits.argtypes = [u64, C.c_uint32]
    L.glo_reverse_index_bits_in_place.argtypes = [u64p, C.c_size_t, C.c_size_t]
    L.glo_fft.argtypes = [u64p, C.c_uint32, C.c_uint32]
    L.glo_ifft.argtypes = [u64p, C.c_uint32]
    L.glo_coset_fft.argtypes = [u64p, C.c_uint32, u64, C.c_uint32]
    L.glo_coset_ifft.argtypes = [u64p, C.c_uint32, u64]
    L.glo_naive_coset_eval.argtypes = [u64p, C.c_uint32, u64, u64p]
    L.glo_poseidon.argtypes = [u64p]
    L.glo_poseidon_naive.argtypes = [u64p]
    L.glo_poseidon_many.argtypes = [u64p, C.c_size_t, C.c_int]
    L.glo_pow_min_nonce.restype = u64
    L.glo_pow_min_nonce.argtypes = [u64p, C.c_uint32, C.c_uint32, u64, C.c_int]
    L.glo_hash_no_pad.argtypes = [u64p, C.c_size_t, u64p]
    L.glo_hash_or_noop.argtypes = [u64p, C.c_size_t, u64p]
    L.glo_two_to_one.argtypes = [u64p, u64p, u64p]
    L.glo_hash_many.argtypes = [u64p, C.c_size_t, C.c_size_t, u64p, C.c_int]
    L.glo_merkle_build.restype = C.c_int
    L.glo_merkle_build.argtypes = [u64p, C.c_size_t, C.c_size_t, C.c_uint32, u64p, u64p, C.c_int]
    L.glo_merkle_prove.argtypes = [C.c_size_t, C.c_size_t, C.c_uint32, u64p, u64p]
    L.glo_merkle_verify.restype = C.c_int
    L.glo_merkle_verify.argtypes = [u64p, C.c_size_t, C.c_size_t, u64p, C.c_size_t, u64p, C.c_uint32]
    L.glo_commit_new.restype = C.c_void_p
    L.glo_commit_new.argtypes = [u64p, C.c_size_t, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, u64p,
                                 C.c_int, C.c_int]
    L.glo_commit_free.argtypes = [C.c_void_p]
    L.glo_commit_leaf_width.restype = C.c_size_t
    L.glo_commit_leaf_width.argtypes = [C.c_void_p]
    for name in ("glo_commit_coeffs", "glo_commit_leaves", "glo_commit_digests", "glo_commit_cap"):
        getattr(L, name).restype = u64p
        getattr(L, name).argtypes = [C.c_void_p]
    L.glo_commit_get_lde_values.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, u64p]
    L.glo_challenger_new.restype = C.c_void_p
    L.glo_challenger_clone.restype = C.c_void_p
    L.glo_challenger_clone.argtypes = [C.c_void_p]
    L.glo_challenger_free.argtypes = [C.c_void_p]
    L.glo_challenger_observe.argtypes = [C.c_void_p, u64p, C.c_size_t]
    L.glo_challenger_get_challenge.restype = u64
    L.glo_challenger_get_challenge.argtypes = [C.c_void_p]
    L.glo_challenger_state.restype = C.c_size_t
    L.glo_challenger_state.argtypes = [C.c_void_p, u64p, u64p]
    L.glo_prove_openings.restype = C.c_int
    L.glo_prove_openings.argtypes = [C.POINTER(C.c_void_p), C.c_size_t, C.POINTER(FriBatch), C.c_size_t,
                                     C.c_void_p, C.POINTER(FriParams), C.POINTER(C.POINTER(C.c_uint8)),
                                     C.POINTER(C.c_size_t), u64p, u64p, u64p, u64p]
    L.glo_free.argtypes = [C.c_void_p]
    L.glo_verify_fri_proof.restype = C.c_int
    L.glo_verify_fri_proof.argtypes = [C.POINTER(u64p), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t),
                                       C.c_size_t, C.POINTER(FriBatch), C.c_size_t, u64p, C.c_uint32,
                                       C.c_void_p, C.POINTER(FriParams), C.POINTER(C.c_uint8), C.c_size_t]
    L.glo_eval_poly_base_at_ext.argtypes = [u64p, C.c_size_t, u64p, u64p]
    L.glo_batch_commit_new.restype = C.c_void_p
    L.glo_batch_commit_new.argtypes = [C.POINTER(u64p), u32p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_int]
    L.glo_batch_commit_free.argtypes = [C.c_void_p]
    L.glo_batch_commit_cap.restype = C.c_size_t
    L.glo_batch_commit_cap.argtypes = [C.c_void_p, u64p]
    L.glo_batch_prove_openings.restype = C.c_int
    L.glo_batch_prove_openings.argtypes = [C.POINTER(C.c_void_p), C.c_size_t, u32p, C.POINTER(FriInstance), C.c_size_t,
                                           C.c_void_p, C.POINTER(FriParams), C.POINTER(C.POINTER(C.c_uint8)),
                                           C.POINTER(C.c_size_t)]
    L.glo_verify_batch_fri_proof.restype = C.c_int
    L.glo_verify_batch_fri_proof.argtypes = [C.POINTER(u64p), C.POINTER(C.c_size_t), C.c_size_t, u32p, C.POINTER(FriInstance),
                                             C.c_size_t, u64p, C.c_void_p, C.POINTER(FriParams), C.POINTER(C.c_uint8), C.c_size_t]
    L.glo_lookup_polys.restype = C.c_int
    L.glo_lookup_polys.argtypes = [u64p, C.c_uint32, C.c_uint32, C.c_uint32, u64p, u32p, C.c_uint32, u64p]
    L.glo_stark_quotient_fibonacci.restype = C.c_int
    L.glo_stark_quotient_fibonacci.argtypes = [C.c_void_p, u64p, u64p, C.c_size_t, u64p]
    L.glo_partial_products_and_zs.restype = C.c_int
    L.glo_partial_products_and_zs.argtypes = [u64p, u64p, u64p, C.c_uint32, C.c_uint32, u64, u64, C.c_uint32, u64p]
    _lib = L
    return L


def ptr(a):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(u64p)


def nproc():
    try:
        return len(os.sched_getaffinity(0))
    except AttributeError:
        return os.cpu_count() or 1


# ---------------------------------------------------------------- convenience wrappers
def fft(a, zero_factor=0):
    a = np.ascontiguousarray(a, dtype=np.uint64).copy()
    lib().glo_fft(ptr(a), int(np.log2(len(a))), zero_factor)
    return a


def ifft(a):
    a = np.ascontiguousarray(a, dtype=np.uint64).copy()
    lib().glo_ifft(ptr(a), int(np.log2(len(a))))
    return a


def coset_fft(a, shift, zero_factor=0):
    a = np.ascontiguousarray(a, dtype=np.uint64).copy()
    lib().glo_coset_fft(ptr(a), int(np.log2(len(a))), shift, zero_factor)
    return a


def coset_ifft(a, shift):
    a = np.ascontiguousarray(a, dtype=np.uint64).copy()
    lib().glo_coset_ifft(ptr(a), int(np.log2(len(a))), shift)
    return a


def naive_coset_eval(coeffs, shift=1):
    coeffs = np.ascontiguousarray(coeffs, dtype=np.uint64)
    out = np.empty_like(coeffs)
    lib().glo_naive_coset_eval(ptr(coeffs), int(np.log2(len(coeffs))), shift, ptr(out))
    return out


def poseidon(state, naive=False):
    s = np.array(state, dtype=np.uint64)
    (lib().glo_poseidon_naive if naive else lib().glo_poseidon)(ptr(s))
    return s


def poseidon_many(states, nthreads=None):
    """The permutation of every row of an (n, 12) array -> (n, 12), canonical."""
    s = np.array(states, dtype=np.uint64).reshape(-1, 12).copy()
    if len(s):
        lib().glo_poseidon_many(ptr(s), len(s), nthreads or nproc())
    return s


NO_NONCE = 2**64 - 1


def pow_min_nonce(state, pos, min_leading_zeros, limit, nthreads=None):
    """The smallest nonce < limit whose permuted state (lane pos = nonce) has lane 7 with at least min_leading_zeros
    leading zeros, or NO_NONCE."""
    s = np.array(state, dtype=np.uint64).reshape(12)
    return int(lib().glo_pow_min_nonce(ptr(s), pos, min_leading_zeros, limit, nthreads or nproc()))


def hash_no_pad(x):
    x = np.ascontiguousarray(x, dtype=np.uint64)
    out = np.empty(4, dtype=np.uint64)
    lib().glo_hash_no_pad(ptr(x) if len(x) else None, len(x), ptr(out))
    return out


def hash_or_noop(x):
    x = np.ascontiguousarray(x, dtype=np.uint64)
    out = np.empty(4, dtype=np.uint64)
    lib().glo_hash_or_noop(ptr(x) if len(x) else None, len(x), ptr(out))
    return out


def two_to_one(l, r):
    l = np.ascontiguousarray(l, dtype=np.uint64)
    r = np.ascontiguousarray(r, dtype=np.uint64)
    out = np.empty(4, dtype=np.uint64)
    lib().glo_two_to_one(ptr(l), ptr(r), ptr(out))
    return out


def hash_many(rows, nthreads=None):
    rows = np.ascontiguousarray(rows, dtype=np.uint64)
    n, w = rows.shape
    out = np.empty((n, 4), dtype=np.uint64)
    lib().glo_hash_many(ptr(rows), n, w, ptr(out), nthreads or nproc())
    return out


def merkle_build(leaves, cap_height, nthreads=None):
    """leaves: (N, W) uint64. Returns (digests (2(N-C),4), cap (C,4))."""
    leaves = np.ascontiguousarray(leaves, dtype=np.uint64)
    N, W = leaves.shape
    Cn = 1 << cap_height
    digests = np.zeros((max(2 * (N - Cn), 0), 4), dtype=np.uint64)
    cap = np.zeros((Cn, 4), dtype=np.uint64)
    dp = ptr(digests) if digests.size else None
    rc = lib().glo_merkle_build(ptr(leaves), N, W, cap_height, dp, ptr(cap), nthreads or nproc())
    if rc != 0:
        raise ValueError("cap_height=%d should be at most log2(leaves.len())" % cap_height)
    return digests, cap


def merkle_prove(leaf_index, N, cap_height, digests):
    nl = int(np.log2(N)) - cap_height
    sib = np.zeros((nl, 4), dtype=np.uint64)
    if nl:
        lib().glo_merkle_prove(leaf_index, N, cap_height, ptr(digests), ptr(sib))
    return sib


def merkle_verify(leaf, leaf_index, siblings, cap, cap_height):
    leaf = np.ascontiguousarray(leaf, dtype=np.uint64)
    siblings = np.ascontiguousarray(siblings, dtype=np.uint64).reshape(-1, 4)
    cap = np.ascontiguousarray(cap, dtype=np.uint64)
    sp = ptr(siblings) if siblings.size else None
    return bool(lib().glo_merkle_verify(ptr(leaf), len(leaf), leaf_index, sp, len(siblings), ptr(cap),
                                        cap_height))


class Commit:
    """Oracle PolynomialBatch (plonky2/src/fri/oracle.rs:30-112)."""

    def __init__(self, cols, rate_bits, cap_height, salt=None, is_coeffs=False, nthreads=None):
        cols = np.ascontiguousarray(cols, dtype=np.uint64)
        self.B, self.n = cols.shape
        self.log_n = int(np.log2(self.n))
        assert 1 << self.log_n == self.n
        self.rate_bits, self.cap_height = rate_bits, cap_height
        self.N = self.n << rate_bits
        sp = None
        if salt is not None:
            salt = np.ascontiguousarray(salt, dtype=np.uint64)
            assert salt.shape == (4, self.N)
            sp = ptr(salt)
        self.h = lib().glo_commit_new(ptr(cols), self.n, self.B, self.log_n, rate_bits, cap_height, sp,
                                      int(is_coeffs), nthreads or nproc())
        if not self.h:
            raise ValueError("cap_height too large")
        self.W = lib().glo_commit_leaf_width(self.h)

    def _arr(self, p, shape):
        n = int(np.prod(shape))
        if n == 0:
            return np.zeros(shape, dtype=np.uint64)
        return np.ctypeslib.as_array(p, shape=(n,)).reshape(shape).copy()

    @property
    def coeffs(self):
        return self._arr(lib().glo_commit_coeffs(self.h), (self.B, self.n))

    @property
    def leaves(self):
        return self._arr(lib().glo_commit_leaves(self.h), (self.N, self.W))

    @property
    def digests(self):
        return self._arr(lib().glo_commit_digests(self.h), (2 * (self.N - (1 << self.cap_height)), 4))

    @property
    def cap(self):
        return self._arr(lib().glo_commit_cap(self.h), (1 << self.cap_height, 4))

    def leaf_rows(self, indices):
        """Rows of the leaf matrix without copying all of it (full-scale fixtures)."""
        view = np.ctypeslib.as_array(lib().glo_commit_leaves(self.h), shape=(self.N * self.W,)).reshape(self.N, self.W)
        return np.stack([view[int(i)].copy() for i in indices])

    def prove(self, leaf_index):
        """Merkle siblings of one leaf, bottom-up (merkle_tree.rs:151-190), without copying the digests."""
        nl = self.log_n + self.rate_bits - self.cap_height
        sib = np.zeros((nl, 4), dtype=np.uint64)
        if nl:
            lib().glo_merkle_prove(int(leaf_index), self.N, self.cap_height, lib().glo_commit_digests(self.h), ptr(sib))
        return sib

    def get_lde_values(self, index, step):
        out = np.empty(self.B, dtype=np.uint64)
        lib().glo_commit_get_lde_values(self.h, index, step, ptr(out))
        return out

    def __del__(self):
        if getattr(self, "h", None):
            lib().glo_commit_free(self.h)
            self.h = None


class Challenger:
    """Oracle Challenger (plonky2/src/iop/challenger.rs:16-153)."""

    def __init__(self, h=None):
        self.h = h or lib().glo_challenger_new()

    def clone(self):
        return Challenger(lib().glo_challenger_clone(self.h))

    def observe_elements(self, xs):
        xs = np.ascontiguousarray(xs, dtype=np.uint64).ravel()
        if len(xs):
            lib().glo_challenger_observe(self.h, ptr(xs), len(xs))

    def observe_element(self, x):
        self.observe_elements(np.array([x], dtype=np.uint64))

    def observe_cap(self, cap):
        self.observe_elements(np.asarray(cap, dtype=np.uint64).ravel())

    def get_challenge(self):
        return int(lib().glo_challenger_get_challenge(self.h))

    def get_n_challenges(self, n):
        return [self.get_challenge() for _ in range(n)]

    def get_extension_challenge(self):
        return (self.get_challenge(), self.get_challenge())

    def state(self):
        st = np.zeros(12, dtype=np.uint64)
        ib = np.zeros(8, dtype=np.uint64)
        n = lib().glo_challenger_state(self.h, ptr(st), ptr(ib))
        return st, ib[:n]

    def __del__(self):
        if getattr(self, "h", None):
            lib().glo_challenger_free(self.h)
            self.h = None


def log_transcripts(monkeypatch):
    """Make every Challenger the product creates log what it observes and draws, for replay(). Returns the list that
    gets one log per Challenger made."""
    import plonky2_b200.challenger as challenger_mod

    logs = []

    class LoggingChallenger(challenger_mod.Challenger):
        def __init__(self):
            super().__init__()
            self.log = []
            logs.append(self.log)

        def observe_element(self, element):
            self.log.append(("observe", int(element)))
            super().observe_element(element)

        def get_challenge(self):
            v = super().get_challenge()
            self.log.append(("challenge", v))
            return v

    monkeypatch.setattr(challenger_mod, "Challenger", LoggingChallenger)
    return logs


def replay(log):
    """An oracle Challenger that continues the product's transcript: it observes what the product observed and draws
    each challenge the product drew, asserting that the two are equal."""
    ch = Challenger()
    for kind, v in log:
        if kind == "observe":
            ch.observe_element(v)
        else:
            assert ch.get_challenge() == v
    return ch


def make_params(rate_bits, cap_height, pow_bits, num_queries, arity_bits):
    p = FriParams()
    p.rate_bits, p.cap_height = rate_bits, cap_height
    p.proof_of_work_bits, p.num_query_rounds = pow_bits, num_queries
    p.num_reductions = len(arity_bits)
    for i, a in enumerate(arity_bits):
        p.reduction_arity_bits[i] = a
    return p


def _make_batches(batches):
    """batches: list of (point(2-tuple), [(oracle_index, poly_index), ...])."""
    arr = (FriBatch * len(batches))()
    keep = []
    for i, (point, polys) in enumerate(batches):
        oi = np.array([p[0] for p in polys], dtype=np.uint32)
        pi = np.array([p[1] for p in polys], dtype=np.uint32)
        keep += [oi, pi]
        arr[i].point[0], arr[i].point[1] = int(point[0]), int(point[1])
        arr[i].num_polys = len(polys)
        arr[i].oracle_index = oi.ctypes.data_as(u32p)
        arr[i].poly_index = pi.ctypes.data_as(u32p)
    return arr, keep


def prove_openings(commits, batches, challenger, params, taps=False):
    L = lib()
    handles = (C.c_void_p * len(commits))(*[c.h for c in commits])
    barr, keep = _make_batches(batches)
    out = C.POINTER(C.c_uint8)()
    out_len = C.c_size_t()
    n = commits[0].n
    t_final = np.zeros(2 * n, dtype=np.uint64)
    t_betas = np.zeros(2 * max(1, params.num_reductions), dtype=np.uint64)
    t_pow = np.zeros(1, dtype=np.uint64)
    t_idx = np.zeros(max(1, params.num_query_rounds), dtype=np.uint64)
    rc = L.glo_prove_openings(handles, len(commits), barr, len(batches), challenger.h, C.byref(params),
                              C.byref(out), C.byref(out_len), ptr(t_final), ptr(t_betas), ptr(t_pow),
                              ptr(t_idx))
    if rc != 0:
        raise RuntimeError("oracle prove_openings failed rc=%d" % rc)
    proof = bytes(C.string_at(out, out_len.value))
    L.glo_free(out)
    if taps:
        return proof, dict(final_poly=t_final.reshape(n, 2), betas=t_betas.reshape(-1, 2)[:params.num_reductions],
                           pow_witness=int(t_pow[0]), query_indices=t_idx[:params.num_query_rounds].copy())
    return proof


def verify_fri_proof(caps, num_polys, leaf_widths, batches, opened_values, degree_bits, challenger, params,
                     proof):
    L = lib()
    caps = [np.ascontiguousarray(c, dtype=np.uint64) for c in caps]
    cap_ptrs = (u64p * len(caps))(*[ptr(c) for c in caps])
    npolys = (C.c_size_t * len(caps))(*num_polys)
    widths = (C.c_size_t * len(caps))(*leaf_widths)
    barr, keep = _make_batches(batches)
    ov = np.ascontiguousarray(opened_values, dtype=np.uint64).ravel()
    buf = (C.c_uint8 * len(proof)).from_buffer_copy(proof)
    return L.glo_verify_fri_proof(cap_ptrs, npolys, widths, len(caps), barr, len(batches), ptr(ov),
                                  degree_bits, challenger.h, C.byref(params), buf, len(proof))


def eval_poly_base_at_ext(coeffs, z):
    coeffs = np.ascontiguousarray(coeffs, dtype=np.uint64)
    zz = np.array(z, dtype=np.uint64)
    out = np.zeros(2, dtype=np.uint64)
    lib().glo_eval_poly_base_at_ext(ptr(coeffs), len(coeffs), ptr(zz), ptr(out))
    return (int(out[0]), int(out[1]))


def partial_products_and_zs(wires, sigmas, k_is, beta, gamma, degree):
    """wires, sigmas: (num_routed, n). Returns (num_prods + 1, n): partial products then Z."""
    wires = np.ascontiguousarray(wires, dtype=np.uint64)
    sigmas = np.ascontiguousarray(sigmas, dtype=np.uint64)
    k_is = np.ascontiguousarray(k_is, dtype=np.uint64)
    R, n = wires.shape
    chunks = (R + degree - 1) // degree
    out = np.zeros((chunks, n), dtype=np.uint64)
    rc = lib().glo_partial_products_and_zs(ptr(wires), ptr(sigmas), ptr(k_is), int(np.log2(n)), R, int(beta),
                                           int(gamma), degree, ptr(out))
    if rc != 0:
        raise ZeroDivisionError("Tried to invert zero")
    return out


def stark_quotient_fibonacci(trace_commit, public_inputs, alphas):
    """compute_quotient_polys for FibonacciStark on an oracle Commit of the 2-column trace: (num_alphas, size) coeffs."""
    pi = np.array([int(x) for x in public_inputs], dtype=np.uint64)
    al = np.array([int(x) for x in alphas], dtype=np.uint64)
    size = trace_commit.n  # quotient_degree_factor = 1
    out = np.zeros((len(al), size), dtype=np.uint64)
    rc = lib().glo_stark_quotient_fibonacci(trace_commit.h, ptr(pi), ptr(al), len(al), ptr(out))
    if rc != 0:
        raise RuntimeError("oracle stark quotient rc=%d" % rc)
    return out


def lookup_polys(wires, num_routed_wires, max_quotient_degree_factor, deltas, lookup_rows):
    """compute_lookup_polys: wires (num_wires, n); lookup_rows [(last_lu, last_lut, first_lut)]. -> (P + 1, n)."""
    wires = np.ascontiguousarray(wires, dtype=np.uint64)
    n = wires.shape[1]
    P_ = -(-(num_routed_wires // 2) // (max_quotient_degree_factor - 1))
    out = np.zeros((P_ + 1, n), dtype=np.uint64)
    d = np.array([int(x) for x in deltas], dtype=np.uint64)
    lr = np.array(lookup_rows, dtype=np.uint32).reshape(-1)
    rc = lib().glo_lookup_polys(ptr(wires), int(np.log2(n)), num_routed_wires, max_quotient_degree_factor, ptr(d),
                                lr.ctypes.data_as(u32p), len(lr) // 3, ptr(out))
    if rc != 0:
        raise ZeroDivisionError("Tried to invert zero")
    return out


class BatchCommit:
    """Oracle BatchFriOracle (plonky2/src/batch_fri/oracle.rs:30-131): polys = list of 1-D arrays, lengths non-increasing."""

    def __init__(self, polys, rate_bits, cap_height, is_coeffs=False):
        self.polys = [np.ascontiguousarray(p, dtype=np.uint64) for p in polys]
        ptrs = (u64p * len(self.polys))(*[ptr(p) for p in self.polys])
        logs = np.array([int(np.log2(len(p))) for p in self.polys], dtype=np.uint32)
        self.h = lib().glo_batch_commit_new(ptrs, logs.ctypes.data_as(u32p), len(self.polys), rate_bits, cap_height,
                                            int(is_coeffs))
        if not self.h:
            raise ValueError("bad batch commitment shape")

    @property
    def cap(self):
        n = lib().glo_batch_commit_cap(self.h, None)
        out = np.zeros((n, 4), dtype=np.uint64)
        lib().glo_batch_commit_cap(self.h, ptr(out))
        return out

    def __del__(self):
        if getattr(self, "h", None):
            lib().glo_batch_commit_free(self.h)
            self.h = None


def batch_prove_openings(commits, degree_bits, instances, challenger, params):
    """instances: per degree, a list of (point, [(oracle_index, poly_index), ...]) batches. Returns the proof bytes."""
    L = lib()
    handles = (C.c_void_p * len(commits))(*[c.h for c in commits])
    insts = (FriInstance * len(instances))()
    keep = []
    for i, batches in enumerate(instances):
        barr, k = _make_batches(batches)
        keep += [barr, k]
        insts[i].batches = C.cast(barr, C.POINTER(FriBatch))
        insts[i].n_batches = len(batches)
    db = np.array(degree_bits, dtype=np.uint32)
    out = C.POINTER(C.c_uint8)()
    out_len = C.c_size_t()
    rc = L.glo_batch_prove_openings(handles, len(commits), db.ctypes.data_as(u32p), insts, len(instances), challenger.h,
                                    C.byref(params), C.byref(out), C.byref(out_len))
    if rc != 0:
        raise RuntimeError("oracle batch prove_openings failed rc=%d" % rc)
    proof = bytes(C.string_at(out, out_len.value))
    L.glo_free(out)
    return proof


def verify_batch_fri_proof(caps, group_num_polys, degree_bits, instances, opened_values, challenger, params, proof):
    """caps: per oracle (C, 4); group_num_polys: per oracle, per degree group; instances as in batch_prove_openings;
    opened_values: flat sequence of F_{p^2} values (per instance, per batch, per polynomial)."""
    L = lib()
    caps = [np.ascontiguousarray(c, dtype=np.uint64) for c in caps]
    cap_ptrs = (u64p * len(caps))(*[ptr(c) for c in caps])
    flat = [int(x) for row in group_num_polys for x in row]
    gnp = (C.c_size_t * len(flat))(*flat)
    insts = (FriInstance * len(instances))()
    keep = []
    for i, batches in enumerate(instances):
        barr, k = _make_batches(batches)
        keep += [barr, k]
        insts[i].batches = C.cast(barr, C.POINTER(FriBatch))
        insts[i].n_batches = len(batches)
    db = np.array(degree_bits, dtype=np.uint32)
    ov = np.ascontiguousarray(opened_values, dtype=np.uint64).ravel()
    buf = (C.c_uint8 * len(proof)).from_buffer_copy(proof)
    return L.glo_verify_batch_fri_proof(cap_ptrs, gnp, len(caps), db.ctypes.data_as(u32p), insts, len(instances), ptr(ov),
                                        challenger.h, C.byref(params), buf, len(proof))


class GloGate(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("param", C.c_uint32), ("selector_index", C.c_uint32),
                ("group_start", C.c_uint32), ("group_end", C.c_uint32), ("param2", C.c_uint32),
                ("param3", C.c_uint32)]


class GloCircuit(C.Structure):
    _fields_ = [("num_wires", C.c_uint32), ("num_routed_wires", C.c_uint32), ("num_constants", C.c_uint32),
                ("num_challenges", C.c_uint32), ("quotient_degree_factor", C.c_uint32), ("num_selectors", C.c_uint32),
                ("num_partial_products", C.c_uint32), ("num_gate_constraints", C.c_uint32),
                ("gates", C.POINTER(GloGate)), ("n_gates", C.c_size_t), ("k_is", u64p),
                ("num_lookup_selectors", C.c_uint32), ("num_lookup_polys", C.c_uint32), ("n_luts", C.c_size_t),
                ("lut_len", u32p), ("lut_inp", u64p), ("lut_out", u64p)]


(GATE_NOOP, GATE_CONSTANT, GATE_PUBLIC_INPUT, GATE_ARITHMETIC, GATE_POSEIDON, GATE_ARITHMETIC_EXTENSION, GATE_MUL_EXTENSION,
 GATE_BASE_SUM, GATE_REDUCING, GATE_REDUCING_EXTENSION, GATE_POSEIDON_MDS, GATE_RANDOM_ACCESS, GATE_EXPONENTIATION,
 GATE_COSET_INTERPOLATION) = range(14)


def plonk_quotient(circuit, constants_sigmas, wires, zs_partial_products, public_inputs_hash, betas, gammas, alphas,
                   deltas=()):
    """compute_quotient_polys of a plonky2 circuit. circuit: dict(num_wires, num_routed_wires, num_constants,
    num_challenges, quotient_degree_factor, num_selectors, num_partial_products, num_gate_constraints, k_is,
    gates=[(kind, param, selector_index, group_start, group_end)] in CommonCircuitData.gates order); the commitments
    are oracle Commits. -> (num_challenges, n << log2_ceil(quotient_degree_factor)) coefficients."""
    gates = (GloGate * len(circuit["gates"]))()
    for i, g in enumerate(circuit["gates"]):
        gates[i].kind, gates[i].param, gates[i].selector_index, gates[i].group_start, gates[i].group_end = g[:5]
        gates[i].param2 = g[5] if len(g) > 5 else 0
        gates[i].param3 = g[6] if len(g) > 6 else 0
    k_is = np.array([int(k) for k in circuit["k_is"]], dtype=np.uint64)
    cd = GloCircuit()
    for f in ("num_wires", "num_routed_wires", "num_constants", "num_challenges", "quotient_degree_factor", "num_selectors",
              "num_partial_products", "num_gate_constraints"):
        setattr(cd, f, int(circuit[f]))
    cd.gates, cd.n_gates, cd.k_is = gates, len(circuit["gates"]), ptr(k_is)
    luts = circuit.get("luts", [])
    lut_len = np.array([len(t) for t in luts] + [0], dtype=np.uint32)
    lut_inp = np.array([p[0] for t in luts for p in t] + [0], dtype=np.uint64)
    lut_out = np.array([p[1] for t in luts for p in t] + [0], dtype=np.uint64)
    cd.num_lookup_selectors, cd.num_lookup_polys = circuit.get("num_lookup_selectors", 0), circuit.get("num_lookup_polys", 0)
    cd.n_luts, cd.lut_len, cd.lut_inp, cd.lut_out = len(luts), lut_len.ctypes.data_as(u32p), ptr(lut_inp), ptr(lut_out)
    de = np.array([int(x) for x in deltas] + [0], dtype=np.uint64)
    pih = np.array([int(x) for x in public_inputs_hash], dtype=np.uint64)
    be, ga, al = (np.array([int(x) for x in v], dtype=np.uint64) for v in (betas, gammas, alphas))
    qd_bits = (int(circuit["quotient_degree_factor"]) - 1).bit_length()
    out = np.zeros((len(al), wires.n << qd_bits), dtype=np.uint64)
    L = lib()
    L.glo_plonk_quotient.restype = C.c_int
    L.glo_plonk_quotient.argtypes = [C.POINTER(GloCircuit), C.c_void_p, C.c_void_p, C.c_void_p, u64p, u64p, u64p, u64p, u64p,
                                     u64p]
    rc = L.glo_plonk_quotient(C.byref(cd), constants_sigmas.h, wires.h, zs_partial_products.h, ptr(pih), ptr(be), ptr(ga),
                              ptr(de), ptr(al), ptr(out))
    if rc != 0:
        raise RuntimeError("oracle plonk quotient rc=%d" % rc)
    return out
