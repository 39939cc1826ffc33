"""One plonky2 circuit proved across ranks: the sharded quotient (gl_plonk_quotient_shard + gl_stark_quotient_from_shards)
and distributed.prove_plonk.

CPU: prove_plonk's refusals (a world size that is not a power of two or above 2^cap_height, a constants/sigmas
commitment of another shard), raised before any device work. The kernel's per-point source with shard addressing
(tests/emu/vanishing_shard_emu.cpp, gl_vanishing.cuh compiled for the host): for every shard g < G its local and next-row
buffers are built from the oracle's LDE (read in place) or from the polynomials' coset values (computed), and the
shards' values placed at r + G*k equal the whole-coset run of tests/emu/vanishing_emu.cpp bit for bit -- G = 1 ... 16 at
(quotient degree factor 8, rate 3), which takes both next-row branches, at (8, 5) and (3, 3), where the local values are
computed, and on a circuit with a lookup table.

GPU (-m gpu): every shard of the three commitments built in one process, each shard's values from
gl_plonk_quotient_shard, concatenated and interpolated by gl_stark_quotient_from_shards: torch.equal to
gl_plonk_quotient's coefficients for G = 1 ... 16 on a small circuit with every gate type and a lookup, on LargeCircuit at
2^13 gates with the 2^16-entry table at (8, 3), (8, 5) and (3, 3), and at 2^16 gates with G = 8 (the high half of the x
power table). The entry point's errors; a broken witness failing the trim check after the gather. prove_plonk on one
rank gives prove_with_witness's bytes, with and without zero knowledge; on 2 (4 with four GPUs) torchrun ranks
(tests/mgpu_plonk_check.py) every rank's bytes equal prove_with_witness's and the restated verifiers accept them."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import plonk_circuits as PC
import plonk_large as PL
from conftest import synth
from plonk_circuits import LOOKUP_64, RECURSION_5
from plonky2_b200 import _native as N
from plonky2_b200 import distributed as D
from ranks import run_ranks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSET_SHIFT = 14293326489335486720   # F::coset_shift()
GS = [1, 2, 4, 8, 16]


def _plonk():
    from plonky2_b200 import plonk

    return plonk


def _small_circuit(shape, cap_height=4, **kw):
    """A FibonacciCircuit with a cap of 2^cap_height entries, enough for 16 shards."""
    return PC.shape_circuit(shape, cap_height, **kw)


# ----------------------------------------------------------------------------------------------------------- CPU
class _Stand:
    """A constants/sigmas commitment stand-in: only its shard."""

    def __init__(self, shard_index, num_shards):
        self.shard_index, self.num_shards = shard_index, num_shards


class _ProverData:
    def __init__(self, cs):
        self.constants_sigmas_commitment = cs


def test_prove_plonk_refusals_before_device_work():
    cd = _small_circuit((12, 8, 4, 2, 4)).common
    assert cd.config.cap_height == 4
    for world in (1, 2, 4, 8, 16):
        D.check_prove_plonk(_ProverData(_Stand(world - 1, world)), cd, world, world - 1)
    for world in (0, 3, 6, 12):
        with pytest.raises(N.ShapeError, match="power-of-two"):
            D.check_prove_plonk(_ProverData(_Stand(0, world)), cd, world)
    with pytest.raises(N.ShapeError, match="exceed the 16 cap entries"):
        D.check_prove_plonk(_ProverData(_Stand(0, 32)), cd, 32)
    for stand, rank, world in (((0, 1), 1, 2), ((1, 4), 1, 2), ((0, 2), 0, 1), ((0, 1), 0, 2)):
        with pytest.raises(N.ShapeError, match="constants/sigmas commitment is shard %d of %d" % stand):
            D.check_prove_plonk(_ProverData(_Stand(*stand)), cd, world, rank)
    # without a process group prove_plonk is one rank; it refuses a sharded constants/sigmas commitment before it looks
    # for a device
    wires = np.zeros((cd.config.num_wires, 1 << cd.degree_bits), dtype=np.uint64)
    with pytest.raises(N.ShapeError, match="constants/sigmas commitment is shard 1 of 2"):
        D.prove_plonk(_ProverData(_Stand(1, 2)), cd, wires, [])


@pytest.fixture(scope="module")
def emu_libs(tmp_path_factory):
    """(the whole-coset run, the shard run) of the kernel's per-point source, compiled for the host."""
    libs = []
    for name in ("vanishing_emu", "vanishing_shard_emu"):
        out = str(tmp_path_factory.mktemp("gl_emu") / ("lib%s.so" % name))
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-DGL_FORCE_32BIT_PATH", "-shared", "-fPIC", "-o", out,
                               os.path.join(ROOT, "tests", "emu", name + ".cpp")])
        libs.append(C.CDLL(out))
    whole, shard = libs
    whole.emu_plonk_quotient_values.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                                C.c_void_p]
    shard.emu_plonk_quotient_shard_values.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                                      C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                      C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                                      C.c_uint32, C.c_void_p]
    return whole, shard


def _bitrev(x, bits):
    r = np.zeros_like(x)
    for b in range(bits):
        r |= ((x >> b) & 1) << (bits - 1 - b)
    return r


def _ptrs(arrays):
    """(uint64_t* const* , size_t*) of column-major 2-D arrays (None: NULL)."""
    ptrs = (C.POINTER(C.c_uint64) * len(arrays))(*[a.ctypes.data_as(C.POINTER(C.c_uint64)) if a is not None
                                                    else C.POINTER(C.c_uint64)() for a in arrays])
    strides = (C.c_size_t * len(arrays))(*[a.shape[1] if a is not None else 0 for a in arrays])
    return ptrs, strides


@pytest.mark.parametrize("shape", [RECURSION_5, (135, 80, 8, 5, 5), (13, 8, 3, 3, 4), LOOKUP_64])
def test_shard_addressing_through_the_kernel_source_on_host(oracle, emu_libs, shape):
    whole_lib, shard_lib = emu_libs
    plonk = _plonk()
    c = _small_circuit(shape)
    cfg, cd = c.config, c.common
    nc, rate_bits, db = cfg.num_challenges, cfg.rate_bits, cd.degree_bits
    betas, gammas, alphas, deltas = PC.challenges(0x7A0 + shape[3] + shape[4], c)
    commits = [oracle.Commit(v, rate_bits, 1) for v in
               (c.constants_sigmas, c.wires, c.oracle_zs_partial_products(oracle, betas, gammas, deltas))]
    b = cd.vanishing_program()
    prog, _ = b.compile()
    consts = plonk.program_constants(cd, b, c.public_inputs_hash, betas, gammas, deltas)
    al = np.array(alphas, dtype=np.uint64)
    qd = (cd.quotient_degree_factor - 1).bit_length()
    size_log = db + qd
    size = 1 << size_log
    # the whole-coset run
    ldes = [np.ascontiguousarray(o.leaves.T) for o in commits]
    want = np.zeros((nc, size), dtype=np.uint64)
    ptrs, strides = _ptrs(ldes)
    assert whole_lib.emu_plonk_quotient_values(ptrs, strides, 3, rate_bits, db, qd, prog, len(prog), consts.ctypes.data,
                                               al.ctypes.data, nc, cd.num_vanishing_terms(), want.ctypes.data) == 0
    # every polynomial on the quotient coset g<w_size>, natural order: what a computed buffer holds, re-addressed
    coset = [np.stack([oracle.coset_fft(np.concatenate([p, np.zeros(size - c.n, dtype=np.uint64)]), COSET_SHIFT)
                       for p in o.coeffs]) for o in commits]
    for G in GS:
        s = G.bit_length() - 1
        M = size // G
        in_place = s == 0 or qd == rate_bits
        got = np.zeros((nc, size), dtype=np.uint64)
        for g in range(G):
            points = _bitrev(np.arange(g * M, (g + 1) * M, dtype=np.int64), size_log)   # global point of local leaf j
            if s == 0:
                loc = ldes
            elif in_place:
                rows = (c.n << rate_bits) // G
                loc = [np.ascontiguousarray(o.leaves[g * rows:(g + 1) * rows].T) for o in commits]
            else:
                loc = [np.ascontiguousarray(v[:, points]) for v in coset]
            nxt = [None] * 3
            if s > qd:
                nxt = [np.ascontiguousarray(v[:, (points + (1 << qd)) % size]) for v in coset]
            out = np.zeros((nc, M), dtype=np.uint64)
            lp, ls = _ptrs(loc)
            np_, ns = _ptrs(nxt)
            rc = shard_lib.emu_plonk_quotient_shard_values(lp, ls, np_, ns, 3, rate_bits, db, qd, g, s, prog, len(prog),
                                                           consts.ctypes.data, al.ctypes.data, nc,
                                                           cd.num_vanishing_terms(), out.ctypes.data)
            assert rc == 0
            r = int(_bitrev(np.array([g]), s)[0]) if s else 0
            got[:, r::G] = out
        bad = np.argwhere(got != want)
        assert not bad.size, "G = %d: first wrong (challenge, point) %s of %d" % (G, bad[0], len(bad))


# ----------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def pb():
    import torch

    if not torch.cuda.is_available():
        if os.environ.get("GL_REQUIRE_GPU") == "1":
            raise AssertionError("GPU tests need a CUDA device")
        pytest.skip("no CUDA device (gpu-marked tests run on an H100)")
    import plonky2_b200 as p

    p.default_context()
    return p


def _z_columns(c, ch):
    """The Z's, partial products and lookup columns of the circuit's second commitment (prove_with_witness's order)."""
    from plonky2_b200.prover import compute_all_lookup_polys, wires_permutation_partial_products_and_zs

    cfg, cd = c.config, c.common
    nr, nc = cfg.num_routed_wires, cfg.num_challenges
    betas, gammas, _, deltas = ch
    zs, pps = [], []
    for beta, gamma in zip(betas, gammas):
        out = wires_permutation_partial_products_and_zs(c.wires[:nr], c.sigmas, cd.k_is, beta, gamma, cd.quotient_degree_factor)
        zs.append(out[-1])
        pps += list(out[:-1])
    cols = [np.stack(zs + pps)]
    if cd.luts:
        cols.append(compute_all_lookup_polys(c.wires, nr, cfg.max_quotient_degree_factor, deltas, c.lookup_rows, nc))
    return np.concatenate(cols)


def _commitments(pb, c, zv, shard=(0, 1)):
    """The constants / sigmas, wires and Z commitments, row block shard[0] of shard[1] (cap height 4)."""
    rate_bits = c.config.rate_bits
    return [pb.PolynomialBatch.from_values(v, rate_bits, False, 4, shard=shard) for v in (c.constants_sigmas, c.wires, zv)]


def _shard_call(ctx, commits, program, qdf, n_terms, out, n_alphas=None):
    prog, consts, al = program
    handles = (C.c_void_p * len(commits))(*[x.h for x in commits])
    return N.lib().gl_plonk_quotient_shard(ctx.h, handles, len(commits), prog, len(prog), N.np_ptr(consts), len(consts),
                                           N.np_ptr(al), len(al) if n_alphas is None else n_alphas, n_terms, qdf,
                                           N.vp(out.data_ptr()))


def _from_shards(ctx, values, G, n_alphas, degree_bits, qdf, out):
    return N.lib().gl_stark_quotient_from_shards(ctx.h, N.vp(values.data_ptr()), G, n_alphas, degree_bits, qdf,
                                                 N.vp(out.data_ptr()))


def _check_sharded_against_whole(pb, c, seed, shard_counts):
    """For each G: every shard's gl_plonk_quotient_shard, then gl_stark_quotient_from_shards, torch.equal to
    gl_plonk_quotient on the whole commitments."""
    import torch

    plonk = _plonk()
    ctx = pb.default_context()
    cd = c.common
    ch = PC.challenges(seed, c)
    betas, gammas, alphas, deltas = ch
    zv = _z_columns(c, ch)
    whole = _commitments(pb, c, zv)
    try:
        want = plonk.compute_quotient_polys(cd, whole[0], c.public_inputs_hash, whole[1], whole[2], betas, gammas, alphas,
                                            deltas)
        program = plonk.quotient_program(cd, whole, c.public_inputs_hash, betas, gammas, alphas, deltas)
    finally:
        for x in whole:
            x.close()
    qdf, nc = cd.quotient_degree_factor, c.config.num_challenges
    size = c.n << (qdf - 1).bit_length()
    for G in shard_counts:
        values = torch.empty((G, nc, size // G), dtype=torch.int64, device="cuda")
        for g in range(G):
            commits = _commitments(pb, c, zv, (g, G))
            try:
                rc = _shard_call(ctx, commits, program, qdf, cd.num_vanishing_terms(), values[g])
                assert rc == N.GL_OK, N.lib().gl_last_error(ctx.h)
            finally:
                for x in commits:
                    x.close()
        got = torch.empty((nc, size), dtype=torch.int64, device="cuda")
        assert _from_shards(ctx, values, G, nc, cd.degree_bits, qdf, got) == N.GL_OK, N.lib().gl_last_error(ctx.h)
        ctx.synchronize()
        assert torch.equal(got, want), "G = %d" % G


def _large(degree_bits, qdf=8, rate_bits=3, **kw):
    return PL.large_circuit(degree_bits, qdf=qdf, rate_bits=rate_bits, luts="range16", **kw)


@pytest.mark.gpu
def test_sharded_quotient_equals_whole_small_circuit(pb):
    """Every gate type and a lookup table on 64 gates, standard recursion config: local values in place, the next row in
    the same shard up to G = 8 and computed at G = 16."""
    _check_sharded_against_whole(pb, _small_circuit(LOOKUP_64), 0x7B0, GS)


@pytest.mark.gpu
@pytest.mark.parametrize("qdf,rate_bits", [(8, 3), (8, 5), (3, 3)])
def test_sharded_quotient_equals_whole_2_13(pb, qdf, rate_bits):
    """LargeCircuit at 2^13 gates with the 2^16-entry table: (8, 3) reads the local values in place; (8, 5) and (3, 3)
    compute them on every shard; the next row is computed once G exceeds 2^log2_ceil(qdf)."""
    _check_sharded_against_whole(pb, _large(13, qdf, rate_bits), 0x7C0 + qdf + rate_bits, GS)


@pytest.mark.gpu
def test_sharded_quotient_equals_whole_2_16(pb):
    """2^16 gates, a coset of 2^19 points: every entry of the x power table's high half, G = 8."""
    _check_sharded_against_whole(pb, _large(16), 0x7D0, [8])


@pytest.mark.gpu
def test_entry_point_errors(pb):
    """Commitments of different shard index or count, or a whole handle among shards: GL_ERR_BAD_ARG naming both; an
    unfinished handle: GL_ERR_BAD_ARG; 5 challenges: GL_ERR_UNSUPPORTED. A broken witness at (qdf 3, rate 3) passes
    gl_plonk_quotient_shard on every shard and fails the trim check in gl_stark_quotient_from_shards."""
    import torch

    plonk = _plonk()
    ctx = pb.default_context()
    L = N.lib()
    c = _small_circuit(LOOKUP_64)
    cd = c.common
    ch = PC.challenges(0x7E0, c)
    betas, gammas, alphas, deltas = ch
    zv = _z_columns(c, ch)
    base = _commitments(pb, c, zv, (0, 2))
    made = list(base)
    program = plonk.quotient_program(cd, base, c.public_inputs_hash, betas, gammas, alphas, deltas)
    qdf, nt = cd.quotient_degree_factor, cd.num_vanishing_terms()
    out = torch.empty((2, (c.n << 3) // 2), dtype=torch.int64, device="cuda")
    assert _shard_call(ctx, base, program, qdf, nt, out) == N.GL_OK, L.gl_last_error(ctx.h)
    for k, shard in ((1, (1, 2)), (2, (0, 4)), (2, (0, 1))):
        other = pb.PolynomialBatch.from_values((c.constants_sigmas, c.wires, zv)[k], c.config.rate_bits, False, 4,
                                               shard=shard)
        made.append(other)
        mixed = list(base)
        mixed[k] = other
        assert _shard_call(ctx, mixed, program, qdf, nt, out) == N.GL_ERR_BAD_ARG, shard
        want = b"commitment %d is shard %d of %d, commitment 0 shard 0 of 2" % (k, shard[0], shard[1])
        assert want in L.gl_last_error(ctx.h)
    h = N.vp()
    N.check(L.gl_commit_begin(ctx.h, zv.shape[0], cd.degree_bits, c.config.rate_bits, 4, 0, 0, 2, None, C.byref(h)), ctx.h)

    class _H:
        def __init__(self, h):
            self.h = h

    assert _shard_call(ctx, [base[0], base[1], _H(h)], program, qdf, nt, out) == N.GL_ERR_BAD_ARG
    assert b"gl_commit_finish has not been called" in L.gl_last_error(ctx.h)
    L.gl_commit_destroy(h)
    five = (program[0], program[1], np.arange(1, 6, dtype=np.uint64))
    assert _shard_call(ctx, base, five, qdf, nt, out) == N.GL_ERR_UNSUPPORTED
    # one past each register-program limit, refused before any launch: 5 commitments, 65 537 terms, register 256, a
    # CONST index (a | b << 16) equal to n_consts through its high half
    consts = np.arange(65537, dtype=np.uint64)
    cases = [(base + base[:2], program, nt, b"1..4 commitments", N.GL_ERR_UNSUPPORTED),
             (base, program, 65537, b"1..65536 vanishing terms", N.GL_ERR_BAD_ARG)]
    for instrs in ([(plonk.OP_X, 256, 0, 0)], [(plonk.OP_X, 0, 0, 0), (plonk.OP_CONST, 1, 1, 1)]):
        prog = (plonk.VpInstr * len(instrs))(*[plonk.VpInstr(*i) for i in instrs])
        cases.append((base, (prog, consts, program[2]), nt, b"bad instruction %d" % (len(instrs) - 1), N.GL_ERR_BAD_ARG))
    for commits, prog, terms, msg, status in cases:
        before = ctx.launch_count
        assert _shard_call(ctx, commits, prog, qdf, terms, out) == status, msg
        assert msg in L.gl_last_error(ctx.h) and ctx.launch_count == before
    for x in made:
        x.close()

    # quotient degree factor 3 on a coset of 4n points: the top n coefficients must vanish
    c3 = _large(13, 3, 3, break_arith=5000)
    cd3 = c3.common
    ch3 = PC.challenges(0x7E1, c3)
    zv3 = _z_columns(c3, ch3)
    G, size = 4, c3.n << 2
    values = torch.empty((G, 2, size // G), dtype=torch.int64, device="cuda")
    program3 = None
    for g in range(G):
        commits = _commitments(pb, c3, zv3, (g, G))
        try:
            if program3 is None:
                program3 = plonk.quotient_program(cd3, commits, c3.public_inputs_hash, *ch3)
            rc = _shard_call(ctx, commits, program3, 3, cd3.num_vanishing_terms(), values[g])
            assert rc == N.GL_OK, L.gl_last_error(ctx.h)
        finally:
            for x in commits:
                x.close()
    whole = torch.empty((2, size), dtype=torch.int64, device="cuda")
    assert _from_shards(ctx, values, G, 2, cd3.degree_bits, 3, whole) == N.GL_ERR_BAD_ARG
    assert b"Quotient has failed" in L.gl_last_error(ctx.h)


@pytest.mark.gpu
@pytest.mark.parametrize("zk", [False, True])
def test_prove_plonk_on_one_rank_is_prove_with_witness(pb, zk):
    """Without a process group prove_plonk is prove_with_witness: the same bytes (zero knowledge with explicit keys)."""
    plonk = _plonk()
    digest = [int(x) for x in synth(0x7F0, (4,))]
    if zk:
        cfg = plonk.standard_recursion_zk_config()
        c, _ = PC.zk_circuit(plonk, cfg, PC.quick_fri_config(cfg))
        kw = dict(salt_keys=PC.KEYS)
    else:
        c, kw = _small_circuit(LOOKUP_64, public_inputs=[3, 1, 4, 1, 5]), {}
    cd = c.common
    cs = pb.PolynomialBatch.from_values(c.constants_sigmas, c.config.rate_bits, False, c.config.cap_height)
    try:
        fri_params = PC.quick_fri_config(c.config).fri_params(cd.degree_bits, zk)
        prover_data = plonk.ProverOnlyCircuitData(cs, c.sigmas, digest, fri_params)
        want = plonk.prove_with_witness(prover_data, cd, c.wires, c.public_inputs, **kw).to_bytes()
        got = D.prove_plonk(prover_data, cd, c.wires, c.public_inputs, **kw).to_bytes()
    finally:
        cs.close()
    assert got == want


@pytest.mark.gpu
def test_prove_plonk_across_ranks(pb):
    """torchrun, one rank per GPU (2, or 4 with four GPUs; the ranks share GPU 0 over gloo on a single-GPU machine):
    every rank's bytes equal prove_with_witness's and the restated verifiers accept them; refusals on every rank."""
    run_ranks("mgpu_plonk_check.py", "MGPU_PLONK_CHECK OK", timeout=1200)
