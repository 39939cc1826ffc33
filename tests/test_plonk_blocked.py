"""plonky2 on non-resident commitments (lde_blocks=G): gl_plonk_quotient_blocked of include/plonky2_b200_blocked.h,
compute_quotient_polys on such handles, build_circuit_data(..., lde_blocks=G) and prove_with_witness(..., lde_blocks=G).

CPU: the header's entry point is exported and bound with its parameter count; every refusal of prove_with_witness's
lde_blocks (check_lde_blocks', G above the quotient coset's points, a resident or other-G constants/sigmas commitment, a
zero-knowledge config), build_circuit_data's and compute_quotient_polys' (resident and non-resident handles together) is
a ShapeError raised before any device work.

GPU (-m gpu): gl_plonk_quotient_blocked equals gl_plonk_quotient on resident handles word for word for G = 1 ... 16 --
the quotient coset equal to the LDE coset (qdf 8 at rate 3: the next row inside the part up to G = 8, outside it at 16)
and smaller (qdf 8 at rate 5), with and without lookups, and a random program at the GL_VP_MAX_* limits; a broken
witness fails with the resident call's message at every G; the entry point's refusals; non-canonical constants and
alphas and page-locked inputs overwritten on return leave the result as it was. Proofs with lde_blocks are byte for
byte the resident proofs (LargeCircuit at 2^13 gates with lookups, and without: the device Z path), with and without
check_constraints, and the restated verifier accepts them; a broken witness raises the resident run's ConstraintError.
build_circuit_data's non-resident commitment has the resident digest and cap. At 2^16 gates the library's high-water
mark with G = 8 is lower than resident by at least half the LDE bytes, and no proof leaks device memory."""
import ctypes as C
import os
import re
from types import SimpleNamespace as NS

import numpy as np
import pytest

import plonk_circuits as PC
import plonk_large as PL
from conftest import P, synth
from plonk_circuits import LOOKUP_64, RECURSION_5
from plonky2_b200 import _native as N
from test_gpu_programs import VP_CONSTS, VP_MAX_TERMS, vp_program
from test_plonk_sharded import _large, _small_circuit, _z_columns

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GS = [1, 2, 4, 8, 16]
VP_LOCAL, VP_TERM = 0, 8


def _plonk():
    from plonky2_b200 import plonk

    return plonk


# ----------------------------------------------------------------------------------------------------------- CPU
def test_binding_matches_the_header():
    with open(os.path.join(ROOT, "include", "plonky2_b200_blocked.h")) as f:
        header = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    assert sorted(re.findall(r"\b(gl_[a-z0-9_]+)\s*\(", header)) == sorted(N.BLOCKED_EXPORTS)
    for name, nargs in (("gl_plonk_quotient_blocked", 12),):
        decl = re.search(r"int %s\(([^;]*)\);" % name, header).group(1)
        assert decl.count(",") + 1 == nargs
        assert len(getattr(N.lib(), name).argtypes) == nargs


def _common(degree_bits=6, qdf=8, cap_height=4, zk=False):
    """What prove_with_witness's lde_blocks checks read of CommonCircuitData."""
    return NS(config=NS(cap_height=cap_height, zero_knowledge=zk), degree_bits=degree_bits, quotient_degree_factor=qdf)


def _prover_data(cs_blocks):
    return NS(constants_sigmas_commitment=NS(lde_blocks=cs_blocks))


def test_refusals_before_device_work():
    """On a machine without a device each of these raises ShapeError, not the NativeError of context creation."""
    plonk = _plonk()

    def prove(G, cd=None, cs_blocks=None):
        return plonk.prove_with_witness(_prover_data(G if cs_blocks is None else cs_blocks), cd or _common(), None, [],
                                        lde_blocks=G)

    for G in (0, -2, 3, 6):
        with pytest.raises(N.ShapeError, match="positive power of two"):
            prove(G)
    with pytest.raises(N.ShapeError, match="exceeds the 16 cap entries"):
        prove(32)
    with pytest.raises(N.ShapeError, match="zero knowledge"):
        prove(4, _common(zk=True))
    # 16 blocks <= 2^cap_height, but more than the 8 points of a 4-gate circuit's coset at quotient degree 2
    with pytest.raises(N.ShapeError, match="exceeds the 8 points of the quotient coset"):
        prove(16, _common(degree_bits=2, qdf=2))
    with pytest.raises(N.ShapeError, match="constants/sigmas commitment is resident"):
        prove(4, cs_blocks=0)
    with pytest.raises(N.ShapeError, match="constants/sigmas commitment is non-resident in 2 blocks"):
        prove(4, cs_blocks=2)
    for G in (3, 32):
        with pytest.raises(N.ShapeError, match="lde_blocks"):
            plonk.build_circuit_data(plonk.CircuitConfig(cap_height=4), None, [], [], lde_blocks=G)
    for blocks in ((0, 4, 4), (4, 0, 0), (2, 4, 4)):
        commits = [NS(lde_blocks=b) for b in blocks]
        with pytest.raises(N.ShapeError, match="all resident or all non-resident"):
            plonk.compute_quotient_polys(None, commits[0], None, commits[1], commits[2], [], [], [])


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


def _commitments(pb, c, zv, lde_blocks=None):
    """The constants / sigmas, wires and Z commitments, resident (None) or non-resident in lde_blocks blocks."""
    cfg = c.config
    return [pb.PolynomialBatch.from_values(v, cfg.rate_bits, False, cfg.cap_height, lde_blocks=lde_blocks)
            for v in (c.constants_sigmas, c.wires, zv)]


def _quotients(pb, c, seed, blocks):
    """compute_quotient_polys on resident commitments, then on non-resident ones of each G in blocks: tensors, or the
    NativeError's message."""
    plonk = _plonk()
    ch = PC.challenges(seed, c)
    zv = _z_columns(c, ch)
    out = []
    for G in [None] + list(blocks):
        commits = _commitments(pb, c, zv, G)
        try:
            assert [x.lde_blocks for x in commits] == [G or 0] * 3
            out.append(plonk.compute_quotient_polys(c.common, commits[0], c.public_inputs_hash, commits[1], commits[2],
                                                    *ch))
        except N.NativeError as e:
            out.append(str(e))
        finally:
            for x in commits:
                x.close()
    return out


CIRCUITS = {
    # every gate type and a lookup table on 64 gates: coset = LDE coset; the next row leaves the part at G = 16
    "lookup64": lambda: _small_circuit(LOOKUP_64),
    # standard recursion config without lookups, 32 gates
    "recursion32": lambda: _small_circuit(RECURSION_5),
    # 2^13 gates with the 2^16-entry table at rate 5: a quotient coset of a quarter of the LDE coset
    "large_8_5": lambda: _large(13, 8, 5),
    # 2^13 gates without lookups
    "large_nolut": lambda: PL.large_circuit(13, luts=None),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CIRCUITS))
def test_blocked_quotient_equals_resident(pb, name):
    import torch

    want, *got = _quotients(pb, CIRCUITS[name](), 0xB70 + len(name), GS)
    assert isinstance(want, torch.Tensor)
    for G, g in zip(GS, got):
        assert isinstance(g, torch.Tensor), (G, g)
        assert torch.equal(g, want), G


@pytest.mark.gpu
def test_broken_witness_fails_like_the_resident_call(pb):
    """Quotient degree factor 3 (a coset of 4n points): the top n coefficients of a broken witness's quotient do not
    vanish, at every G as on resident handles."""
    want, *got = _quotients(pb, _large(13, 3, 3, break_arith=5000), 0xB80, [1, 4, 16])
    assert isinstance(want, str) and "Quotient has failed" in want
    assert got == [want] * 3


# ---- random programs at the interpreter's limits, straight through the C entry points
WIDTHS = [3, 9, 1, 5]


def _random_case(pb, qdf, seed):
    """Four unsalted commitments at rate 3 on 2^5 rows, a 256-register program with 70 000 constants and 65 536 terms,
    4 alphas: (prog, consts, alphas, {G: commitments}) with the resident ones at G = None."""
    prog = np.ascontiguousarray(vp_program(seed, 1500, WIDTHS, VP_CONSTS, VP_MAX_TERMS, salted=-1))
    consts = synth(seed + 1, (VP_CONSTS,))
    alphas = synth(seed + 2, (4,))
    vals = [synth(seed + 3 + c, (w, 1 << 5)) for c, w in enumerate(WIDTHS)]
    commits = {G: [pb.PolynomialBatch.from_values(v, 3, False, 4, lde_blocks=G) for v in vals] for G in [None] + GS}
    return prog, consts, alphas, commits


def _call(ctx, fn, commits, prog, consts, alphas, qdf, out):
    handles = (C.c_void_p * len(commits))(*[x.h for x in commits])
    return fn(ctx.h, handles, len(commits), prog.ctypes.data_as(N.vp), len(prog), N.np_ptr(consts), len(consts),
              N.np_ptr(alphas), len(alphas), VP_MAX_TERMS, qdf, N.vp(out.data_ptr()))


@pytest.mark.gpu
@pytest.mark.parametrize("qdf", [2, 8])
def test_random_program_at_the_limits(pb, qdf):
    """qdf 8 at rate 3: the resident call reads the LDE in place; qdf 2: a quotient coset of 2n points, computed from
    the coefficients on both sides, the next row outside the part from G = 4 on."""
    import torch

    ctx = pb.default_context()
    L = N.lib()
    prog, consts, alphas, commits = _random_case(pb, qdf, 0xB90 + qdf)
    size = 32 << (qdf - 1).bit_length()
    try:
        want = torch.empty((4, size), dtype=torch.int64, device="cuda")
        N.check(_call(ctx, L.gl_plonk_quotient, commits[None], prog, consts, alphas, qdf, want), ctx.h)
        for G in GS:
            got = torch.full((4, size), -1, dtype=torch.int64, device="cuda")
            N.check(_call(ctx, L.gl_plonk_quotient_blocked, commits[G], prog, consts, alphas, qdf, got), ctx.h)
            assert torch.equal(got, want), G
    finally:
        for cs in commits.values():
            for x in cs:
                x.close()


def _twin(a):
    """Every word below 2^32 - 1 replaced by its non-canonical twin x + p."""
    return np.where(a < np.uint64(2**32 - 1), a + np.uint64(P), a)


def _pinned(a):
    """A page-locked host copy of the array `a` (any dtype), as a numpy view of a pinned torch tensor."""
    import torch

    t = torch.empty(a.nbytes, dtype=torch.uint8, pin_memory=True)
    assert t.is_pinned()
    v = t.numpy().view(a.dtype).reshape(a.shape)
    v[...] = a
    return v


@pytest.mark.gpu
def test_host_input_contracts(pb):
    """The conventions plonky2_b200_blocked.h takes from plonky2_b200.h: non-canonical constants and alphas give the
    same words, and the program, constants and alphas have been read when the call returns -- page-locked copies
    overwritten as soon as it returns leave the result as it was."""
    import torch

    ctx = pb.default_context()
    fn = N.lib().gl_plonk_quotient_blocked
    qdf = 8
    prog, consts, alphas, commits = _random_case(pb, qdf, 0xBA0)
    consts[::5] = np.arange(0, len(consts), 5, dtype=np.uint64)   # words below 2^32 - 1 have a non-canonical twin
    alphas[:2] = [5, 2**32 - 2]
    try:
        want = torch.empty((4, 256), dtype=torch.int64, device="cuda")
        N.check(_call(ctx, fn, commits[4], prog, consts, alphas, qdf, want), ctx.h)
        got = torch.empty_like(want)
        assert (_twin(consts) != consts).any() and (_twin(alphas) != alphas).any()
        N.check(_call(ctx, fn, commits[4], prog, _twin(consts), _twin(alphas), qdf, got), ctx.h)
        assert torch.equal(got, want)
        pp, pc, pa = _pinned(prog), _pinned(consts), _pinned(alphas)
        got = torch.empty_like(want)
        N.check(_call(ctx, fn, commits[4], pp, pc, pa, qdf, got), ctx.h)
        pp[...], pc[...], pa[...] = 0xFFFF, 0, 0   # a program of invalid opcodes, zero constants and alphas
        ctx.synchronize()
        assert torch.equal(got, want)
    finally:
        for cs in commits.values():
            for x in cs:
                x.close()


@pytest.mark.gpu
def test_entry_point_refusals(pb):
    """A resident handle, a row-block shard, handles of different G and G above the quotient coset: GL_ERR_BAD_ARG
    before any launch. gl_plonk_quotient's own refusal of a non-resident handle is unchanged."""
    import torch

    ctx = pb.default_context()
    L = N.lib()
    vals = synth(0xBB0, (2, 4))
    prog = np.array([(VP_LOCAL, 0, 0, 0), (VP_TERM, 0, 0, 0)], dtype=np.uint16)
    consts, alphas = np.zeros(1, dtype=np.uint64), np.array([5], dtype=np.uint64)
    out = torch.empty((1, 64), dtype=torch.int64, device="cuda")
    made = []

    def batch(**kw):
        made.append(pb.PolynomialBatch.from_values(vals, 3, False, 4, **kw))
        return made[-1]

    def call(commits, qdf=8):
        before = ctx.launch_count
        handles = (C.c_void_p * len(commits))(*[x.h for x in commits])
        rc = L.gl_plonk_quotient_blocked(ctx.h, handles, len(commits), prog.ctypes.data_as(N.vp), len(prog),
                                         N.np_ptr(consts), 1, N.np_ptr(alphas), 1, 1, qdf, N.vp(out.data_ptr()))
        assert rc == N.GL_OK or ctx.launch_count == before
        return rc, L.gl_last_error(ctx.h).decode()

    try:
        b2, b4, res, shard = batch(lde_blocks=2), batch(lde_blocks=4), batch(), batch(shard=(1, 2))
        assert call([b2, res]) == (N.GL_ERR_BAD_ARG, "commitment 1 is resident: the blocked quotient takes "
                                   "non-resident handles (gl_plonk_quotient reads a resident LDE)")
        assert call([res])[0] == N.GL_ERR_BAD_ARG
        assert call([b2, shard]) == (N.GL_ERR_BAD_ARG, "commitment 1 is row-block shard 1 of 2: the blocked quotient "
                                     "takes non-resident handles")
        assert call([b2, b4]) == (N.GL_ERR_BAD_ARG, "commitment 1 is in 4 LDE blocks, commitment 0 in 2")
        # 4 rows at qdf 2: a quotient coset of 8 points, fewer than 16 blocks (the LDE has 32 rows, the cap 16 entries)
        assert call([batch(lde_blocks=16)], qdf=2) == (N.GL_ERR_BAD_ARG, "16 LDE blocks of a quotient coset of 2^3 points")
        assert call([batch(lde_blocks=4)], qdf=2)[0] == N.GL_OK
        rc = L.gl_plonk_quotient(ctx.h, (C.c_void_p * 1)(b2.h), 1, prog.ctypes.data_as(N.vp), len(prog),
                                 N.np_ptr(consts), 1, N.np_ptr(alphas), 1, 1, 8, N.vp(out.data_ptr()))
        assert rc == N.GL_ERR_BAD_ARG and b"not resident" in L.gl_last_error(ctx.h)
    finally:
        for x in made:
            x.close()


# ---- whole proofs
DIGEST = [int(x) for x in synth(0xBC0, (4,))]


def _prove(pb, c, G=None, wires=None, check=False):
    """prove_with_witness with the constants/sigmas commitment and every other one resident (G = None) or in G blocks:
    (proof bytes, the parts the restated verifier reads)."""
    from plonky2_b200.fri import standard_recursion_fri_config

    plonk = _plonk()
    cfg, cd = c.config, c.common
    fri_params = standard_recursion_fri_config().fri_params(cd.degree_bits, False)
    cs = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height, lde_blocks=G)
    try:
        prover_data = plonk.ProverOnlyCircuitData(cs, c.sigmas, DIGEST, fri_params)
        data = plonk.prove_with_witness(prover_data, cd, c.wires if wires is None else wires, c.public_inputs,
                                        check_constraints=check, lde_blocks=G).to_bytes()
        cs_cap = cs.merkle_tree.cap.hashes
    finally:
        cs.close()
    return data, PC.parts_of(plonk.ProofWithPublicInputs.from_bytes(data, cd, fri_params), cs_cap)


@pytest.mark.gpu
@pytest.mark.parametrize("luts", ["small", None])
def test_prove_blocked_equals_resident(pb, oracle, luts):
    """LargeCircuit at 2^13 gates, standard recursion config, with two lookup tables and without (the device Z path):
    the bytes of G = 1, 4, 16 (and of G = 4 with check_constraints) are the resident proof's, and the verifier accepts
    each."""
    from plonky2_b200.fri import standard_recursion_fri_config

    c = PL.large_circuit(13, luts=luts, public_inputs=[3, 1, 4, 1, 5])
    want, _ = _prove(pb, c)
    for G, check in ((1, False), (4, False), (16, False), (4, True)):
        got, parts = _prove(pb, c, G, check=check)
        assert got == want, (G, check)
        assert PC.oracle_verify(oracle, _plonk(), c, DIGEST, standard_recursion_fri_config(), parts) is None, G


@pytest.mark.gpu
def test_broken_witness_raises_the_resident_constraint_error(pb):
    c = PL.large_circuit(13, qdf=8, break_arith=5000, public_inputs=[3, 1, 4])
    errors = []
    for G in (None, 4):
        with pytest.raises(N.ConstraintError) as e:
            _prove(pb, c, G, check=True)
        errors.append((str(e.value), e.value.report.failures, e.value.report.entries))
    assert "at row %d" % c.broken_row in errors[0][0]
    assert errors[1] == errors[0]


@pytest.mark.gpu
def test_build_circuit_data_blocked(pb):
    """The constants/sigmas commitment of build_circuit_data(..., lde_blocks=G) is non-resident, with the resident
    commitment's cap, polynomials and circuit digest."""
    from plonk_circuits import instances_of, pairs_from_sigmas

    plonk = _plonk()
    cfg = plonk.CircuitConfig(num_wires=135, num_routed_wires=80, cap_height=3)
    c = PC.FibonacciCircuit(plonk, cfg, 6, poseidon_rows=4)
    fri_cfg = PC.quick_fri_config(cfg)
    args = (cfg, fri_cfg, instances_of(c), pairs_from_sigmas(c))
    want = plonk.build_circuit_data(*args)
    wcs = want.prover_only.constants_sigmas_commitment
    try:
        for G in (1, 2, 8):
            got = plonk.build_circuit_data(*args, lde_blocks=G)
            cs = got.prover_only.constants_sigmas_commitment
            try:
                assert cs.lde_blocks == G and N.lib().gl_commit_lde_blocks(cs.h) == G
                assert np.array_equal(got.verifier_only.constants_sigmas_cap.hashes,
                                      want.verifier_only.constants_sigmas_cap.hashes)
                assert np.array_equal(cs.merkle_tree.cap.hashes, wcs.merkle_tree.cap.hashes)
                assert np.array_equal(cs.polynomials, wcs.polynomials)
                assert got.prover_only.circuit_digest == want.prover_only.circuit_digest
                assert got.verifier_only.circuit_digest == want.verifier_only.circuit_digest
            finally:
                cs.close()
    finally:
        wcs.close()


@pytest.mark.gpu
def test_blocked_proof_lowers_the_high_water_mark(pb):
    """LargeCircuit at 2^16 gates, standard recursion config with lookups: the four commitments' LDEs hold about 1.1 GB
    at rate 1/8. Each proof runs once unmeasured first, so that the context's cached tables and scratch exist."""
    from plonky2_b200.fri import standard_recursion_fri_config

    plonk = _plonk()
    c = PL.large_circuit(16, public_inputs=[2, 7])
    cfg, cd = c.config, c.common
    fri_params = standard_recursion_fri_config().fri_params(cd.degree_bits, False)
    ctx = pb.default_context()
    widths = [c.constants_sigmas.shape[0], cfg.num_wires, cd.num_zs_partial_products_polys()
              + cfg.num_challenges * cd.num_lookup_polys, cfg.num_challenges * cd.quotient_degree_factor]
    lde_bytes = 8 * sum(widths) << (cd.degree_bits + cfg.rate_bits)
    proofs, highs = {}, {}
    for G in (None, 8):
        cs = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height, lde_blocks=G)
        try:
            prover_data = plonk.ProverOnlyCircuitData(cs, c.sigmas, DIGEST, fri_params)
            plonk.prove_with_witness(prover_data, cd, c.wires, c.public_inputs, lde_blocks=G)
            before, _ = ctx.device_bytes(reset_high=True)
            proofs[G] = plonk.prove_with_witness(prover_data, cd, c.wires, c.public_inputs, lde_blocks=G).to_bytes()
            after, highs[G] = ctx.device_bytes()
            assert after == before, (G, before, after)
        finally:
            cs.close()
    assert proofs[8] == proofs[None]
    assert highs[None] - highs[8] >= lde_bytes // 2, (highs, lde_bytes)
