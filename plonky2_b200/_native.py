"""ctypes binding of libplonky2_b200.so (the C ABI in include/plonky2_b200.h).

The CUDA library is the ONLY compute backend: if it is missing, or no CUDA device is present, the
calls below raise -- there is no CPU fallback."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libplonky2_b200.so")

GL_OK = 0
GL_ERR_BAD_SHAPE, GL_ERR_OOM, GL_ERR_CUDA, GL_ERR_UNSUPPORTED, GL_ERR_BAD_ARG, GL_ERR_POW_FAILED, GL_ERR_DIV_ZERO = 1, 2, 3, 4, 5, 6, 7
MEM_HOST, MEM_DEVICE = 0, 1
COLS_VALUES, COLS_COEFFS, COLS_COEFFS_CANONICAL = 0, 1, 2

u64p = C.POINTER(C.c_uint64)
u32p = C.POINTER(C.c_uint32)
vp = C.c_void_p

EXPORTS = [
    "gl_ctx_create", "gl_ctx_destroy", "gl_last_error", "gl_ctx_synchronize", "gl_ctx_launch_count",
    "gl_ctx_set_ntt_group", "gl_ctx_set_profiling", "gl_ctx_phase_ms", "gl_ctx_reset_phases", "gl_ctx_stream", "gl_ntt",
    "gl_ntt_bcast", "gl_bcast", "gl_commit_create", "gl_commit_create_sharded", "gl_commit_begin", "gl_commit_add_columns",
    "gl_commit_finish", "gl_commit_shard", "gl_commit_destroy", "gl_commit_num_polys",
    "gl_commit_leaf_width", "gl_commit_degree_log", "gl_commit_rate_bits", "gl_commit_cap_height",
    "gl_commit_cap", "gl_commit_coeffs", "gl_commit_leaves", "gl_commit_digests", "gl_commit_get_lde_values",
    "gl_commit_open", "gl_commit_eval_ext", "gl_openings", "gl_openings_shard", "gl_stark_quotient", "gl_stark_quotient_aux", "gl_stark_quotient_shard", "gl_stark_quotient_from_shards", "gl_stark_lookup_helpers", "gl_stark_ctl_helpers", "gl_plonk_quotient", "gl_plonk_quotient_shard", "gl_lookup_polys", "gl_sigma_polys", "gl_commit_dev_lde", "gl_commit_dev_coeffs", "gl_partial_products_and_zs", "gl_poseidon_permute_host",
    "gl_poseidon_permute_many", "gl_poseidon_hash_many", "gl_poseidon_hash_no_pad_many", "gl_poseidon_two_to_one_many", "gl_merkle_build", "gl_merkle_destroy",
    "gl_merkle_cap", "gl_merkle_digests", "gl_merkle_open", "gl_fri_begin", "gl_fri_begin_values", "gl_fri_values_local", "gl_fri_begin_from_coeffs",
    "gl_fri_destroy", "gl_fri_coeffs", "gl_fri_commit_round", "gl_fri_commit_round_sharded", "gl_fri_mix", "gl_fri_fold", "gl_fri_final_poly",
    "gl_fri_open", "gl_fri_num_rounds", "gl_fri_pow", "gl_commit_finish_keyed", "gl_random_field_elements",
    "gl_commit_finish_prefixed", "gl_commit_dev_cap", "gl_commit_begin_blocked", "gl_commit_lde_blocks",
    "gl_ctx_device_bytes",
]
# the constraint checks of include/plonky2_b200_check.h
CHECK_EXPORTS = ["gl_stark_check_rows", "gl_plonk_check_rows", "gl_stark_check_rows_part", "gl_plonk_check_rows_part",
                 "gl_plonk_check_copies", "gl_plonk_check_lookups"]
# the plonky2 quotient on non-resident commitments of include/plonky2_b200_blocked.h
BLOCKED_EXPORTS = ["gl_plonk_quotient_blocked"]


class FriBatch(C.Structure):
    _fields_ = [("point", C.c_uint64 * 2), ("num_polys", C.c_size_t), ("oracle_index", u32p),
                ("poly_index", u32p)]


class ShapeError(ValueError):
    """Mirrors the reference's shape panics (fft.rs:171-177, merkle_tree.rs:195-200, oracle.rs:128)."""


class NativeError(RuntimeError):
    pass


class ConstraintError(ValueError):
    """A trace or witness that breaks a constraint, found by a prover's check_constraints=True (the reference's
    "Constraint failed in {Stark} at row {row}", starky/src/prover.rs:812). `report` is the ConstraintReport."""

    def __init__(self, message, report):
        super().__init__(message)
        self.report = report


class ConstraintReport:
    """What gl_stark_check_rows / gl_plonk_check_rows found: `failures`, the number of failing (row, index) pairs, and
    `entries`, the first of them in (row, index) order as (row, index, label)."""

    def __init__(self, failures, entries):
        self.failures, self.entries = int(failures), list(entries)

    def __bool__(self):
        """True when nothing failed."""
        return self.failures == 0

    def __repr__(self):
        return "ConstraintReport(failures=%d, entries=%r)" % (self.failures, self.entries)


MAX_REPORT = 65536


def check_rows(fn, ctx, args, max_report):
    """Run the check entry point `fn` (gl_stark_check_rows, gl_plonk_check_rows or their _part counterparts) with `args`
    between the context and max_report. Returns (failures, [(row, index)])."""
    max_report = int(max_report)
    if not 0 <= max_report <= MAX_REPORT:
        raise ValueError("max_report must be in 0..%d" % MAX_REPORT)
    failures, reported = C.c_uint64(), C.c_uint32()
    pairs = np.zeros(2 * max(max_report, 1), dtype=np.uint32)
    check(fn(ctx.h, *args, max_report, C.byref(failures), pairs.ctypes.data_as(u32p), C.byref(reported)), ctx.h)
    return failures.value, [(int(r), int(i)) for r, i in pairs[:2 * reported.value].reshape(-1, 2)]


def check_parts(parts):
    """parts=G of check_constraints: a positive power of two (ShapeError otherwise, before any device work)."""
    if not isinstance(parts, (int, np.integer)) or parts < 1 or parts & (parts - 1):
        raise ShapeError("parts=%r is not a positive power of two" % (parts,))
    return int(parts)


def check_rows_in_parts(fn, fn_part, ctx, args, max_report, log_n, parts=1, placement=None):
    """The whole check of H by the entry point `fn` (gl_stark_check_rows / gl_plonk_check_rows), or by its _part
    counterpart `fn_part` in parts of H, with `args` between the context and (part, parts) or max_report. Returns
    (failures, [(row, index)]), the same in every case:
    - placement of G > 1 ranks (distributed.Placement): this rank checks part shard_index of min(G, n) (a rank >= n has
      no rows) and the ranks merge their reports (Placement.report_from_shards). Collective.
    - parts=G on one device: the min(G, n) parts one after another, merged (merge_reports); each part's scratch is 1/G
      of the whole check's.
    - otherwise the whole check, one call of `fn`."""
    parts = check_parts(parts)
    n = 1 << int(log_n)
    if placement is not None and placement.num_shards > 1:
        g, G = placement.shard_index, min(placement.num_shards, n)

        def run_part():
            return check_rows(fn_part, ctx, args + (g, G), max_report) if g < G else (0, [])
        return placement.report_from_shards(ctx, run_part, max_report)
    if parts == 1:
        return check_rows(fn, ctx, args, max_report)
    G = min(parts, n)
    return merge_reports([check_rows(fn_part, ctx, args + (g, G), max_report) for g in range(G)], max_report)


def merge_reports(parts, max_report):
    """The whole check's (failures, [(row, index)]) from its parts' reports, each (failures, pairs) as check_rows returns
    it for one part of H with the same max_report: the failures add up, and the pairs are the first max_report of the
    sorted union of the parts' pairs. This is exact: a part's pairs are a subsequence of the global (row, index) order,
    so the global first max_report pairs all lie within their parts' first max_report."""
    parts = list(parts)
    return sum(int(f) for f, _ in parts), sorted(p for _, pairs in parts for p in pairs)[:int(max_report)]


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeError(
            "libplonky2_b200.so is not built (run `python -c 'import __graft_entry__ as g; g.build()'`); "
            "plonky2_b200 has no CPU fallback")
    L = C.CDLL(LIB_PATH)
    L.gl_ctx_create.argtypes = [C.c_int, vp, C.POINTER(vp)]
    L.gl_ctx_destroy.argtypes = [vp]
    L.gl_ctx_destroy.restype = None
    L.gl_last_error.argtypes = [vp]
    L.gl_last_error.restype = C.c_char_p
    L.gl_ctx_synchronize.argtypes = [vp]
    L.gl_ctx_device_bytes.argtypes = [vp, u64p, u64p, C.c_int]
    L.gl_ctx_launch_count.argtypes = [vp]
    L.gl_ctx_launch_count.restype = C.c_uint64
    L.gl_ctx_set_ntt_group.argtypes = [vp, C.c_uint32]
    L.gl_ntt.argtypes = [vp, vp, C.c_uint32, C.c_uint32, C.c_size_t, C.c_int, C.c_uint32, C.c_uint64, C.c_int]
    L.gl_ctx_stream.argtypes = [vp]
    L.gl_ctx_stream.restype = vp
    L.gl_ntt_bcast.argtypes = [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_int, C.POINTER(vp), C.c_uint32, C.c_size_t]
    L.gl_bcast.argtypes = [vp, vp, C.c_size_t, C.POINTER(vp), C.c_uint32, C.c_uint32]
    L.gl_commit_begin.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_uint32,
                                  vp, C.POINTER(vp)]
    L.gl_commit_begin_blocked.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp,
                                          C.POINTER(vp)]
    L.gl_commit_add_columns.argtypes = [vp, C.c_uint32, C.c_uint32, vp, C.c_size_t, C.c_int, C.c_int]
    L.gl_commit_finish.argtypes = [vp, vp, C.c_int]
    L.gl_commit_finish_keyed.argtypes = [vp, C.c_char_p]
    L.gl_commit_finish_prefixed.argtypes = [vp, vp]
    L.gl_random_field_elements.argtypes = [vp, C.c_char_p, C.c_uint32, C.c_uint64, C.c_size_t, vp, C.c_int]
    L.gl_commit_create.argtypes = [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp,
                                   C.c_int, C.c_int, C.POINTER(vp)]
    L.gl_commit_create_sharded.argtypes = [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp,
                                           C.c_int, C.c_int, C.c_uint32, C.c_uint32, C.POINTER(vp)]
    L.gl_commit_shard.argtypes = [vp, u32p, u32p]
    L.gl_ctx_set_profiling.argtypes = [vp, C.c_int]
    L.gl_ctx_phase_ms.argtypes = [vp, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]
    L.gl_ctx_reset_phases.argtypes = [vp]
    L.gl_commit_destroy.argtypes = [vp]
    L.gl_commit_destroy.restype = None
    for n in ("gl_commit_num_polys", "gl_commit_leaf_width", "gl_commit_degree_log", "gl_commit_rate_bits",
              "gl_commit_cap_height", "gl_commit_lde_blocks"):
        getattr(L, n).argtypes = [vp]
        getattr(L, n).restype = C.c_uint32
    L.gl_commit_cap.argtypes = [vp, vp, C.c_int]
    L.gl_commit_coeffs.argtypes = [vp, vp, C.c_int]
    L.gl_commit_leaves.argtypes = [vp, C.c_size_t, C.c_size_t, vp, C.c_int]
    L.gl_commit_digests.argtypes = [vp, vp, C.c_int]
    L.gl_commit_get_lde_values.argtypes = [vp, C.c_size_t, C.c_size_t, vp]
    L.gl_commit_open.argtypes = [vp, vp, C.c_size_t, vp, vp]
    L.gl_commit_eval_ext.argtypes = [vp, vp, vp]
    L.gl_openings.argtypes = [vp, C.POINTER(vp), u32p, C.c_size_t, vp, C.c_size_t, vp, C.c_int]
    L.gl_openings_shard.argtypes = [vp, C.POINTER(vp), u32p, C.c_size_t, vp, C.c_size_t, C.c_uint32, C.c_uint32, vp,
                                    C.c_int]
    L.gl_stark_quotient.argtypes = [vp, vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, C.c_uint32, vp]
    L.gl_stark_quotient_aux.argtypes = [vp, vp, vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, C.c_uint32, vp]
    L.gl_stark_quotient_shard.argtypes = [vp, vp, vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, C.c_uint32, vp]
    L.gl_stark_quotient_from_shards.argtypes = [vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp]
    L.gl_stark_lookup_helpers.argtypes = [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, vp, u32p, C.c_uint32, vp,
                                          C.c_uint32, vp, C.c_uint32, C.c_uint32, vp]
    L.gl_stark_ctl_helpers.argtypes = [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, vp, u32p, C.c_uint32, vp, C.c_uint32,
                                       vp, C.c_uint32, C.c_uint32, u32p, vp]
    L.gl_plonk_quotient.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, C.c_uint32,
                                    C.c_uint32, vp]
    L.gl_plonk_quotient_shard.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32,
                                          C.c_uint32, C.c_uint32, vp]
    L.gl_plonk_quotient_blocked.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32,
                                            C.c_uint32, C.c_uint32, vp]
    L.gl_stark_check_rows.argtypes = [vp, vp, vp, vp, C.c_uint32, vp, C.c_uint32, C.c_uint32, u64p, u32p, u32p]
    L.gl_plonk_check_rows.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, C.c_uint32, C.c_uint32, u64p,
                                      u32p, u32p]
    L.gl_stark_check_rows_part.argtypes = [vp, vp, vp, vp, C.c_uint32, vp, C.c_uint32, C.c_uint32, C.c_uint32,
                                           C.c_uint32, u64p, u32p, u32p]
    L.gl_plonk_check_rows_part.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, C.c_uint32, C.c_uint32,
                                           C.c_uint32, C.c_uint32, u64p, u32p, u32p]
    L.gl_plonk_check_copies.argtypes = [vp, vp, C.c_size_t, C.c_int, vp, C.c_size_t, C.c_int, vp, C.c_uint32,
                                        C.c_uint32, C.c_uint32, u64p, u32p, u32p]
    L.gl_plonk_check_lookups.argtypes = [vp, vp, C.c_size_t, C.c_int, C.c_uint32, C.c_uint32, vp, u32p, u32p,
                                         C.c_uint32, u32p, C.c_uint32, u64p, u32p, u32p]
    L.gl_lookup_polys.argtypes = [vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, vp, u32p, C.c_uint32, vp, C.c_int]
    L.gl_sigma_polys.argtypes = [vp, vp, C.c_size_t, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, vp, vp,
                                 C.c_int]
    L.gl_commit_dev_lde.argtypes = [vp, C.POINTER(C.c_size_t)]
    L.gl_commit_dev_lde.restype = vp
    L.gl_commit_dev_coeffs.argtypes = [vp]
    L.gl_commit_dev_coeffs.restype = vp
    L.gl_commit_dev_cap.argtypes = [vp]
    L.gl_commit_dev_cap.restype = vp
    L.gl_partial_products_and_zs.argtypes = [vp, vp, vp, vp, C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint64,
                                             C.c_uint32, vp, C.c_int]
    L.gl_poseidon_permute_host.argtypes = [vp]
    L.gl_poseidon_permute_host.restype = None
    L.gl_poseidon_permute_many.argtypes = [vp, vp, C.c_size_t, C.c_int]
    L.gl_poseidon_hash_many.argtypes = [vp, vp, C.c_size_t, C.c_uint32, vp, C.c_int]
    L.gl_poseidon_hash_no_pad_many.argtypes = [vp, vp, C.c_size_t, C.c_uint32, vp, C.c_int]
    L.gl_poseidon_two_to_one_many.argtypes = [vp, vp, C.c_size_t, vp, C.c_int]
    L.gl_merkle_build.argtypes = [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_int, C.POINTER(vp)]
    L.gl_merkle_destroy.argtypes = [vp]
    L.gl_merkle_destroy.restype = None
    L.gl_merkle_cap.argtypes = [vp, vp, C.c_int]
    L.gl_merkle_digests.argtypes = [vp, vp, C.c_int]
    L.gl_merkle_open.argtypes = [vp, vp, C.c_size_t, vp, vp]
    L.gl_fri_begin.argtypes = [vp, C.POINTER(vp), C.c_size_t, C.POINTER(FriBatch), C.c_size_t, vp, C.c_uint32,
                               C.c_uint32, C.POINTER(vp)]
    L.gl_fri_begin_values.argtypes = [vp, C.POINTER(vp), C.c_size_t, C.POINTER(FriBatch), C.c_size_t, vp, vp, C.c_uint32,
                                      C.POINTER(vp)]
    L.gl_fri_values_local.argtypes = [vp, vp, C.c_size_t, C.POINTER(C.c_size_t)]
    L.gl_fri_begin_from_coeffs.argtypes = [vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(vp)]
    L.gl_fri_destroy.argtypes = [vp]
    L.gl_fri_destroy.restype = None
    L.gl_fri_coeffs.argtypes = [vp, vp]
    L.gl_fri_commit_round.argtypes = [vp, C.c_uint32, vp]
    L.gl_fri_commit_round_sharded.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, vp]
    L.gl_fri_mix.argtypes = [vp, vp, vp]
    L.gl_fri_fold.argtypes = [vp, vp]
    L.gl_fri_final_poly.argtypes = [vp, vp, C.c_size_t, C.POINTER(C.c_size_t)]
    L.gl_fri_open.argtypes = [vp, C.c_uint32, vp, C.c_size_t, vp, vp]
    L.gl_fri_num_rounds.argtypes = [vp]
    L.gl_fri_num_rounds.restype = C.c_uint32
    L.gl_fri_pow.argtypes = [vp, vp, C.c_uint32, C.c_uint32, vp]
    _lib = L
    return L


def check(rc, ctx=None):
    if rc == GL_OK:
        return
    msg = lib().gl_last_error(ctx)
    msg = msg.decode() if msg else "error %d" % rc
    if rc == GL_ERR_BAD_SHAPE:
        raise ShapeError(msg)
    if rc == GL_ERR_OOM:
        raise MemoryError(msg)
    if rc == GL_ERR_DIV_ZERO:
        raise ZeroDivisionError(msg)
    raise NativeError("plonky2_b200 native error %d: %s" % (rc, msg))


def np_ptr(a):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"], "need contiguous uint64"
    return a.ctypes.data_as(vp)


class Handle:
    """Owner of one library handle `h`, destroyed by the library function named `destroyer`. close() is idempotent;
    collecting the object closes it too."""
    destroyer = None
    h = None

    def close(self):
        if self.h:
            getattr(lib(), self.destroyer)(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Context(Handle):
    """One gl_ctx per (device, stream) (SURVEY.md section 8b, threading row)."""
    destroyer = "gl_ctx_destroy"
    _torch_stream = None

    def __init__(self, device=0, stream=None):
        h = vp()
        check(lib().gl_ctx_create(int(device), vp(stream) if stream else None, C.byref(h)))
        self.h = h
        self.device = device

    def synchronize(self):
        check(lib().gl_ctx_synchronize(self.h), self.h)

    def after_caller(self):
        """Order this context's stream after everything queued so far on torch's current stream of its device: the
        library's later reads of a caller's tensor see the values that stream is still producing, and its writes into
        a tensor torch allocated land after the reads torch queued on the block's previous tenant. An event wait on the
        device: the host does not block. Every function that hands a torch tensor to the library calls it before its
        first library call."""
        import torch

        if self._torch_stream is None:
            self._torch_stream = torch.cuda.ExternalStream(self.stream, device=torch.device("cuda", self.device))
        self._torch_stream.wait_stream(torch.cuda.current_stream(self._torch_stream.device))

    @property
    def stream(self):
        """The cudaStream_t (as an int) every call on this context is ordered on."""
        return int(lib().gl_ctx_stream(self.h) or 0)

    def device_bytes(self, reset_high=False):
        """(in_use, high): bytes of the device's default memory pool in use now and at most since the last reset, after
        this context's queued work has run; reset_high then resets the high-water mark to the current use. Every device
        buffer of the library, on any context of this device, comes from that pool; torch's caching allocator does not
        (gl_ctx_device_bytes)."""
        in_use, high = C.c_uint64(), C.c_uint64()
        check(lib().gl_ctx_device_bytes(self.h, C.byref(in_use), C.byref(high), int(bool(reset_high))), self.h)
        return in_use.value, high.value

    @property
    def launch_count(self):
        return int(lib().gl_ctx_launch_count(self.h))

    def set_ntt_group(self, columns):
        check(lib().gl_ctx_set_ntt_group(self.h, int(columns)), self.h)

    PHASES = {"intt": 0, "lde": 1, "leaf_hash": 2, "merkle_levels": 3}

    def set_profiling(self, on):
        check(lib().gl_ctx_set_profiling(self.h, int(bool(on))), self.h)

    def reset_phases(self):
        check(lib().gl_ctx_reset_phases(self.h), self.h)

    def phase_ms(self):
        """{phase: (accumulated ms, scopes)} from CUDA events on this context's stream."""
        out = {}
        for name, pid in self.PHASES.items():
            ms, cnt = C.c_double(), C.c_uint64()
            check(lib().gl_ctx_phase_ms(self.h, pid, C.byref(ms), C.byref(cnt)), self.h)
            out[name] = (ms.value, cnt.value)
        return out


_default_ctx = {}


def default_context(device=0):
    """Process-wide default context per device (created on first use; fails loudly without a GPU)."""
    if device not in _default_ctx:
        _default_ctx[device] = Context(device)
    return _default_ctx[device]
