"""Pieces of plonky2/src/plonk/prover.rs adjacent to the hot path ("next" rows of SURVEY.md section 8f) that
run on the GPU: the Z / partial-product columns of the permutation argument."""
import numpy as np

from . import _native as N
from .field import log2_strict


def wires_permutation_partial_products_and_zs(wires, sigmas, k_is, beta, gamma, degree, ctx=None):
    """wires_permutation_partial_products_and_zs (prover.rs:387-449): wires, sigmas are (num_routed, n) arrays of
    column values; returns (num_partial_products + 1, n): the partial-product columns, then Z (the reference's
    return order; the prover moves Z to the front before committing, prover.rs:227-232)."""
    ctx = ctx or N.default_context()
    wires = np.ascontiguousarray(wires, dtype=np.uint64)
    sigmas = np.ascontiguousarray(sigmas, dtype=np.uint64)
    k_is = np.ascontiguousarray(k_is, dtype=np.uint64)
    if wires.shape != sigmas.shape or wires.ndim != 2 or len(k_is) != wires.shape[0]:
        raise N.ShapeError("wires, sigmas must be (num_routed, n) and k_is (num_routed,)")
    R, n = wires.shape
    log_n = log2_strict(n)
    out = np.empty(((R + degree - 1) // degree, n), dtype=np.uint64)
    rc = N.lib().gl_partial_products_and_zs(ctx.h, N.np_ptr(wires), N.np_ptr(sigmas), N.np_ptr(k_is), log_n, R,
                                            int(beta), int(gamma), int(degree), N.np_ptr(out), N.MEM_HOST)
    N.check(rc, ctx.h)   # GL_ERR_DIV_ZERO -> ZeroDivisionError ("Tried to invert zero"), others keep their own type
    return out


def commit_zs_partial_products(wires_dev, sigmas_dev, k_is, betas, gammas, degree, rate_bits, cap_height, ctx=None, *,
                               blinding=False, salt_key=None, shard=(0, 1), lde_blocks=None):
    """The second commitment of prove() without leaving the device (prover.rs:220-254):
    all_wires_permutation_partial_products for every challenge pair (beta_i, gamma_i) -> Z's moved to the front
    (`[plonk_z_vecs, partial_products.concat()].concat()`) -> PolynomialBatch::from_values.

    wires_dev, sigmas_dev: torch int64 CUDA tensors of shape (num_routed, n) -- the routed wire columns (the same
    device matrix the wires commitment was built from) and the sigma value columns (resident since circuit build).
    Each gl_partial_products_and_zs call writes its columns straight into a device staging matrix; each column group is
    then handed to the incremental commitment (gl_commit_add_columns, GL_MEM_DEVICE): no H2D, no D2H.
    The caller's tensors may still be in production on its current torch stream: the library's work is ordered after it.
    With blinding the salt is drawn on the device from salt_key (PolynomialBatch._from_device). shard=(g, G): only row
    block g of G of the LDE and tree on this device (the columns are computed over all n rows either way).
    lde_blocks=G: a non-resident batch, its LDE built in G row blocks where it is hashed or read.
    Returns the PolynomialBatch (num_challenges * (num_partial_products + 1) polynomials)."""
    import torch

    from .polynomial_batch import PolynomialBatch

    ctx = ctx or N.default_context()
    R, n = wires_dev.shape
    if sigmas_dev.shape != (R, n) or len(k_is) != R or len(betas) != len(gammas):
        raise N.ShapeError("wires, sigmas must be (num_routed, n), k_is (num_routed,), betas/gammas equally long")
    log_n = log2_strict(n)
    k_is = np.ascontiguousarray(k_is, dtype=np.uint64)
    nch = len(betas)
    M = (R + degree - 1) // degree          # columns per challenge: M - 1 partial products, then Z
    stage = torch.empty((M, n), dtype=torch.int64, device=wires_dev.device)  # must outlive _from_device's synchronise
    ctx.after_caller()
    L = N.lib()

    def add_columns(h):
        for i in range(nch):
            N.check(L.gl_partial_products_and_zs(ctx.h, N.vp(wires_dev.data_ptr()), N.vp(sigmas_dev.data_ptr()),
                                                 N.np_ptr(k_is), log_n, R, int(betas[i]), int(gammas[i]), int(degree),
                                                 N.vp(stage.data_ptr()), N.MEM_DEVICE), ctx.h)
            # Z (last column of the call) is polynomial i; the partial products follow all Z's
            N.check(L.gl_commit_add_columns(h, i, 1, N.vp(stage[M - 1].data_ptr()), n, N.COLS_VALUES, N.MEM_DEVICE), ctx.h)
            if M > 1:
                N.check(L.gl_commit_add_columns(h, nch + i * (M - 1), M - 1, N.vp(stage.data_ptr()), n, N.COLS_VALUES,
                                                N.MEM_DEVICE), ctx.h)

    return PolynomialBatch._from_device(ctx, nch * M, log_n, rate_bits, cap_height, add_columns, blinding=blinding,
                                        salt_key=salt_key, shard=shard, lde_blocks=lde_blocks)


def compute_lookup_polys(wires, num_routed_wires, max_quotient_degree_factor, deltas, lookup_rows, ctx=None):
    """compute_lookup_polys (prover.rs:458-577) for one challenge set deltas = (A, B, alpha, delta): the RE polynomial
    and the partial Sum/LDC polynomials as value columns, (num_partial_lookups + 1, n). wires: (num_wires, n) witness
    matrix (host array); lookup_rows: [(last_lu_gate, last_lut_gate, first_lut_gate)] (LookupWire)."""
    ctx = ctx or N.default_context()
    wires = np.ascontiguousarray(wires, dtype=np.uint64)
    if wires.ndim != 2:
        raise N.ShapeError("wires must be (num_wires, n)")
    n = wires.shape[1]
    log_n = log2_strict(n)
    need = max(3 * (num_routed_wires // 3), 2 * (num_routed_wires // 2))
    if wires.shape[0] < need:
        raise N.ShapeError("the witness must hold at least %d wires" % need)
    P_ = -(-(num_routed_wires // 2) // (max_quotient_degree_factor - 1))
    out = np.empty((P_ + 1, n), dtype=np.uint64)
    d = np.array([int(x) for x in deltas], dtype=np.uint64)
    lr = np.array(lookup_rows, dtype=np.uint32).reshape(-1)
    N.check(N.lib().gl_lookup_polys(ctx.h, N.np_ptr(np.ascontiguousarray(wires[:need])), log_n, num_routed_wires,
                                    max_quotient_degree_factor, N.np_ptr(d), lr.ctypes.data_as(N.u32p), len(lr) // 3,
                                    N.np_ptr(out), N.MEM_HOST), ctx.h)
    return out


def compute_all_lookup_polys(wires, num_routed_wires, max_quotient_degree_factor, deltas, lookup_rows, num_challenges,
                             ctx=None):
    """compute_all_lookup_polys (prover.rs:579-607): one compute_lookup_polys per challenge (4 deltas each), concatenated."""
    parts = [compute_lookup_polys(wires, num_routed_wires, max_quotient_degree_factor, deltas[4 * c:4 * c + 4], lookup_rows,
                                  ctx) for c in range(num_challenges)]
    return np.concatenate(parts) if parts else np.zeros((0, wires.shape[1]), dtype=np.uint64)
