"""plonky2's quotient, lookup columns and whole proofs at the size of real circuits (run with `-m gpu` on an H100).

The other plonky2 tests stop at 64..128 gates. Several paths of the device prover only run on larger circuits or other
rates:
  - vp_eval_point reads x = shift * xhi[i >> 12] * xlo[i & 4095]; the hi half of the power table is only read on cosets
    of more than 4096 points, and every entry of it only on cosets of 2^16 points and more;
  - with rate_bits > log2_ceil(quotient_degree_factor) the coset is smaller than the LDE (step > 1), and the next-row
    leaf is bitrev over the coset's size, not the LDE's;
  - the RE lookup column's scan (k_affine_scan) gives a thread more than one item only past 1024 LookupTableGate rows,
    and RE is the only column whose multiplier delta^L is not 1;
  - a 2^16-entry table, two tables, 1..4 challenges, and whole proofs at 2^13..2^20 gates.
Circuits come from tests/plonk_large.py. Up to 2^13 gates the oracle's quotient is the bit-exact reference; above, the
device quotient is checked with the verifier's own identity (plonk/verifier.rs:85-107) at random points of F_p and
F_{p^2}, from the device commitments' coefficients evaluated on the CPU (oracle_lib.eval_poly_base_at_ext).
The 2^20-gate case runs only with GL_LARGE_PLONK_20=1."""
import os
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import plonk_circuits as PC
import plonk_large as PL
from conftest import synth

G = 14293326489335486720   # F::coset_shift()


def _plonk():
    from plonky2_b200 import plonk

    return plonk


def _points(seed):
    """Two points of F_p and two of F_{p^2}."""
    r = [int(x) for x in synth(seed, (6,))]
    return [(r[0], 0), (r[1], 0), (r[2], r[3]), (r[4], r[5])]


def _chunks(q, c):
    """quotient_poly.chunks(n) of every challenge after trim_to_len(qdf * n) (prover.rs:319-331)."""
    qdf, n = c.common.quotient_degree_factor, c.n
    return np.concatenate([q[i, :qdf * n].reshape(qdf, n) for i in range(q.shape[0])])


def _identity_failures(oracle, c, cs_coeffs, w_coeffs, z_coeffs, chunks, ch, points):
    betas, gammas, alphas, deltas = ch
    with ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 1)) as pool:
        return PL.quotient_identity_failures(_plonk(), c.common, c.public_inputs_hash, cs_coeffs, w_coeffs, z_coeffs, chunks,
                                             betas, gammas, alphas, deltas, points, oracle.eval_poly_base_at_ext, pool)


# ----------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("nc", [1, 4])
@pytest.mark.parametrize("luts", [None, "small"])
@pytest.mark.parametrize("degree_bits", [6, 7, 8])
def test_builder_passes_the_verifier_identity(oracle, degree_bits, luts, nc):
    """The builder's circuits are satisfied: the oracle's quotient has no coefficients past qdf * n and meets the
    verifier's identity at two points of F_p and two of F_{p^2}."""
    c = PL.large_circuit(degree_bits, nc=nc, cap_height=1, luts=luts)
    ch = PC.challenges(0x6100 + degree_bits, c)
    cfg = c.config
    cs, w = oracle.Commit(c.constants_sigmas, cfg.rate_bits, 1), oracle.Commit(c.wires, cfg.rate_bits, 1)
    z = oracle.Commit(c.oracle_zs_partial_products(oracle, *ch[:2], ch[3]), cfg.rate_bits, 1)
    q = oracle.plonk_quotient(c.oracle_circuit(), cs, w, z, c.public_inputs_hash, ch[0], ch[1], ch[2], ch[3])
    assert q.shape == (nc, c.n << 3) and not q[:, 8 * c.n:].any()
    assert not _identity_failures(oracle, c, cs.coeffs, w.coeffs, z.coeffs, _chunks(q, c), ch, _points(0x6110))


def test_builder_at_quotient_degree_factor_3(oracle):
    """qdf 3 with lookups: the coset has 4n points and the top n quotient coefficients vanish."""
    c = PL.large_circuit(8, qdf=3, cap_height=1)
    ch = PC.challenges(0x6120, c)
    cfg = c.config
    cs, w = oracle.Commit(c.constants_sigmas, cfg.rate_bits, 1), oracle.Commit(c.wires, cfg.rate_bits, 1)
    z = oracle.Commit(c.oracle_zs_partial_products(oracle, *ch[:2], ch[3]), cfg.rate_bits, 1)
    q = oracle.plonk_quotient(c.oracle_circuit(), cs, w, z, c.public_inputs_hash, ch[0], ch[1], ch[2], ch[3])
    assert q.shape == (2, 4 * c.n) and not q[:, 3 * c.n:].any()
    assert not _identity_failures(oracle, c, cs.coeffs, w.coeffs, z.coeffs, _chunks(q, c), ch, _points(0x6121))


def test_vectorised_sigmas_equal_the_loop_form():
    """sigma_values equals get_sigma_map written out wire by wire (as tests/plonk_circuits.FibonacciCircuit does) on the
    same partition; every cycle is a true cycle of distinct routed wires."""
    c = PL.large_circuit(8, cap_height=1)
    nr, n = c.config.num_routed_wires, c.n
    neighbor = {}
    for members in c.partition():
        assert len(set(members)) == len(members) and all(col < nr for _, col in members)
        for i, wire in enumerate(members):
            assert wire not in neighbor, "a wire in two copy cycles"
            neighbor[wire] = members[(i + 1) % len(members)]
    assert len(neighbor) > 20 * (n // 4)          # the addend copies, the long cycles and the Poseidon chain
    omega = PC.root_of_unity(c.common.degree_bits)
    subgroup = [pow(omega, r, PC.P) for r in range(n)]
    want = np.empty((nr, n), dtype=np.uint64)
    for col in range(nr):
        for row in range(n):
            nrow, ncol = neighbor.get((row, col), (row, col))
            want[col, row] = c.common.k_is[ncol] * subgroup[nrow] % PC.P
    assert np.array_equal(c.sigmas, want)
    # the copied wires carry equal values
    for members in c.partition():
        assert len({int(c.wires[col, row]) for row, col in members}) == 1


@pytest.mark.parametrize("change", ["coset_value", "partial_product", "re"])
def test_identity_rejects_a_wrong_column(oracle, change):
    """The identity accepts the oracle's quotient at 2^8 gates and rejects it after one change: one coset value of the
    quotient before the coset iNTT, one partial-product value, or one RE (lookup) value."""
    c = PL.large_circuit(8, cap_height=1)
    ch = PC.challenges(0x6130, c)
    cfg, cd = c.config, c.common
    cs, w = oracle.Commit(c.constants_sigmas, cfg.rate_bits, 1), oracle.Commit(c.wires, cfg.rate_bits, 1)
    zv = c.oracle_zs_partial_products(oracle, *ch[:2], ch[3])
    z = oracle.Commit(zv, cfg.rate_bits, 1)
    q = oracle.plonk_quotient(c.oracle_circuit(), cs, w, z, c.public_inputs_hash, ch[0], ch[1], ch[2], ch[3])
    points = _points(0x6131)
    assert not _identity_failures(oracle, c, cs.coeffs, w.coeffs, z.coeffs, _chunks(q, c), ch, points)
    z_coeffs = z.coeffs
    if change == "coset_value":
        vals = oracle.coset_fft(q[1], G)
        vals[3 * c.n + 5] = (int(vals[3 * c.n + 5]) + 1) % PC.P
        q = q.copy()
        q[1] = oracle.coset_ifft(vals, G)
    else:
        col = cd.config.num_challenges + 3 if change == "partial_product" else cd.num_zs_partial_products_polys()
        row = c.n // 2 if change == "partial_product" else c.lookup_rows[0][1] + 1
        zv = zv.copy()
        zv[col, row] = (int(zv[col, row]) + 1) % PC.P
        z_coeffs = np.stack([oracle.ifft(v) for v in zv])
    bad = _identity_failures(oracle, c, cs.coeffs, w.coeffs, z_coeffs, _chunks(q, c), ch, points)
    assert {x for x, _ in bad} == set(points)     # every point sees it
    # each challenge's vanishing polynomial combines every challenge's terms: a wrong column breaks all of them
    assert {k for _, k in bad} == ({1} if change == "coset_value" else {0, 1})


# ----------------------------------------------------------------------------- GPU
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


def _device_commitments(pb, c, ch):
    """The prover's first three commitments on the device (prove_with_witness's route with lookups): constants /
    sigmas, wires, then Z's, partial products and lookup columns from gl_partial_products_and_zs and gl_lookup_polys.
    Returns (cs, w, z, the Z / partial-product / lookup value columns)."""
    from plonky2_b200.prover import compute_all_lookup_polys, wires_permutation_partial_products_and_zs

    cfg, cd = c.config, c.common
    nr, nc = cfg.num_routed_wires, cfg.num_challenges
    betas, gammas, _, deltas = ch
    cs = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height)
    w = pb.PolynomialBatch.from_values(c.wires, cfg.rate_bits, False, cfg.cap_height)
    zs, pps = [], []
    for beta, gamma in zip(betas, gammas):
        out = wires_permutation_partial_products_and_zs(c.wires[:nr], c.sigmas, cd.k_is, beta, gamma, cd.quotient_degree_factor)
        zs.append(out[-1])
        pps += list(out[:-1])
    cols = [np.stack(zs + pps)]
    if cd.luts:
        cols.append(compute_all_lookup_polys(c.wires, nr, cfg.max_quotient_degree_factor, deltas, c.lookup_rows, nc))
    zv = np.concatenate(cols)
    z = pb.PolynomialBatch.from_values(zv, cfg.rate_bits, False, cfg.cap_height)
    return cs, w, z, zv


def _device_quotient(c, cs, w, z, ch):
    from plonky2_b200 import plonk

    betas, gammas, alphas, deltas = ch
    return plonk.compute_quotient_polys(c.common, cs, c.public_inputs_hash, w, z, betas, gammas, alphas, deltas)


def _check_quotient_against_oracle(pb, oracle, c, seed):
    """gl_plonk_quotient bit for bit against the oracle's quotient, and the quotient commitment's cap."""
    from plonky2_b200 import plonk

    cfg = c.config
    ch = PC.challenges(seed, c)
    ocs, ow = oracle.Commit(c.constants_sigmas, cfg.rate_bits, cfg.cap_height), oracle.Commit(c.wires, cfg.rate_bits, cfg.cap_height)
    oz = oracle.Commit(c.oracle_zs_partial_products(oracle, *ch[:2], ch[3]), cfg.rate_bits, cfg.cap_height)
    want = oracle.plonk_quotient(c.oracle_circuit(), ocs, ow, oz, c.public_inputs_hash, *ch)
    cs, w, z, _ = _device_commitments(pb, c, ch)
    try:
        for mine, theirs in ((cs, ocs), (w, ow), (z, oz)):
            assert np.array_equal(mine.merkle_tree.cap.hashes, theirs.cap)
        q = _device_quotient(c, cs, w, z, ch)
        got = q.cpu().numpy().view(np.uint64)
        bad = np.argwhere(got != want)
        assert not bad.size, "first wrong (challenge, coefficient) %s of %d" % (bad[0], len(bad))
        qc = plonk.commit_quotient_polys(c.common, q)
        oq = oracle.Commit(_chunks(want, c), cfg.rate_bits, cfg.cap_height, is_coeffs=True)
        assert np.array_equal(qc.merkle_tree.cap.hashes, oq.cap)
        qc.close()
    finally:
        for b in (cs, w, z):
            b.close()


def _fri_cfg(c):
    """standard_recursion_config's FRI: rate 3, cap height 4, 28 queries, 16 grinding bits, arity 2^4."""
    from plonky2_b200.fri import standard_recursion_fri_config

    assert (c.config.rate_bits, c.config.cap_height) == (3, 4)

    return standard_recursion_fri_config()


def _prove(pb, c, digest, wires=None):
    """plonk.prove_with_witness on the device -> (proof bytes, the parts oracle_verify reads, as read back with
    ProofWithPublicInputs.from_bytes)."""
    from plonky2_b200 import plonk

    cfg, cd = c.config, c.common
    fri_params = _fri_cfg(c).fri_params(cd.degree_bits, False)
    cs = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height)
    try:
        prover_data = plonk.ProverOnlyCircuitData(cs, c.sigmas, digest, fri_params)
        data = plonk.prove_with_witness(prover_data, cd, c.wires if wires is None else wires, c.public_inputs).to_bytes()
        cs_cap = cs.merkle_tree.cap.hashes
    finally:
        cs.close()
    proof = plonk.ProofWithPublicInputs.from_bytes(data, cd, fri_params)
    return data, PC.parts_of(proof, cs_cap)


def _verify(oracle, c, digest, parts):
    return PC.oracle_verify(oracle, _plonk(), c, digest, _fri_cfg(c), parts)


DIGEST = [int(x) for x in synth(0x6190, (4,))]
PUBLIC_INPUTS = [3, 1, 4, 1, 5, 9, 2, 6]


@pytest.mark.gpu
def test_a_recursion_circuit_2_13_is_bit_exact(pb, oracle):
    """Case a: the standard recursion config (135 wires, 80 routed, qdf 8, rate 3) at 2^13 gates with every gate type,
    Poseidon rows, the 2^16-entry range table and a small table. The quotient over its 2^16-point coset equals the
    oracle's bit for bit, and prove_with_witness gives the CPU prover's bytes, which the restated verifier accepts."""
    c = PL.large_circuit(13, luts="range16", public_inputs=PUBLIC_INPUTS)
    _check_quotient_against_oracle(pb, oracle, c, 0x6200)
    want, _ = PC.oracle_prove(oracle, c, DIGEST, _fri_cfg(c), c.public_inputs)
    got, parts = _prove(pb, c, DIGEST)
    assert got == want
    assert _verify(oracle, c, DIGEST, parts) is None


@pytest.mark.gpu
@pytest.mark.parametrize("qdf,rate_bits", [(8, 5), (3, 3)])
def test_quotient_with_a_coset_smaller_than_the_lde(pb, oracle, qdf, rate_bits):
    """Case b: step = 2^(rate_bits - qd_bits) = 4 (qdf 8 at rate 5) and 2 (qdf 3 at rate 3, with the trim check): the
    local and next-row leaves are bitrev over the coset's size. Bit-exact against the oracle, and the quotient cap."""
    _check_quotient_against_oracle(pb, oracle, PL.large_circuit(13, qdf=qdf, rate_bits=rate_bits), 0x6210 + qdf)


class _PeakDeviceMemory:
    """The device's peak memory in use (total - free, sampled every 2 ms) while the block runs: the library allocates
    with cudaMalloc, outside torch's allocator statistics."""

    def __enter__(self):
        import torch

        self.total = torch.cuda.mem_get_info()[1]
        self.base = self.peak = self.total - torch.cuda.mem_get_info()[0]
        self.stop = threading.Event()

        def sample():
            while not self.stop.is_set():
                self.peak = max(self.peak, self.total - torch.cuda.mem_get_info()[0])
                time.sleep(0.002)

        self.thread = threading.Thread(target=sample, daemon=True)
        self.thread.start()
        return self

    def __exit__(self, *exc):
        self.stop.set()
        self.thread.join()


def _check_identity_on_device(pb, oracle, c, seed):
    """Case c / f: the device's Z and partial products bit-exact against the oracle's; the device's lookup columns
    against the oracle's; the device quotient's chunks meet the verifier's identity at four points."""
    from plonky2_b200 import plonk

    cfg, cd = c.config, c.common
    nr, nc = cfg.num_routed_wires, cfg.num_challenges
    ch = PC.challenges(seed, c)
    cs, w, z, zv = _device_commitments(pb, c, ch)
    try:
        nprod = cd.num_partial_products
        for i in range(nc):
            want = oracle.partial_products_and_zs(c.wires[:nr], c.sigmas, cd.k_is, ch[0][i], ch[1][i], cd.quotient_degree_factor)
            assert np.array_equal(zv[i], want[-1]), "Z of challenge %d" % i
            assert np.array_equal(zv[nc + i * nprod:nc + (i + 1) * nprod], want[:-1]), "partial products of challenge %d" % i
        qc = plonk.commit_quotient_polys(cd, _device_quotient(c, cs, w, z, ch))
        try:
            bad = _identity_failures(oracle, c, cs.polynomials, w.polynomials, z.polynomials, qc.polynomials, ch,
                                     _points(seed + 1))
        finally:
            qc.close()
        assert not bad, "the verifier identity fails at (point, challenge) %s" % bad
    finally:
        for b in (cs, w, z):
            b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("degree_bits,nc", [(16, 4), (18, 2)])
def test_quotient_identity_at_2_16_and_2_18(pb, oracle, degree_bits, nc):
    """Case c: the standard config at 2^16 and 2^18 gates (cosets of 2^19 and 2^21 points), both lookup tables."""
    c = PL.large_circuit(degree_bits, nc=nc, luts="range16")
    with _PeakDeviceMemory() as mem:
        _check_identity_on_device(pb, oracle, c, 0x6220 + degree_bits)
    print("\n2^%d gates, %d challenges: peak device memory %.2f GiB (%.2f GiB in use before)"
          % (degree_bits, nc, mem.peak / 2**30, mem.base / 2**30))


@pytest.mark.gpu
def test_lookups_and_proof_2_16(pb, oracle):
    """Case d: 2^16 gates with the 2^16-entry table (2521 LookupTableGate rows, so the RE scan gives a thread several
    rows) and a small table. The lookup columns equal the oracle's bit for bit; RE at last_lut is the table's
    lut_re_poly_evals. The device proof, read back with from_bytes, is accepted by the restated verifier and rejected
    after tampering with an opening, the public inputs, one wire of a looking pair, or one table multiplicity."""
    from plonky2_b200.prover import compute_all_lookup_polys

    c = PL.large_circuit(16, luts="range16", public_inputs=PUBLIC_INPUTS)
    cfg, cd = c.config, c.common
    nr, nc = cfg.num_routed_wires, cfg.num_challenges
    assert c.lookup_rows[0][2] - c.lookup_rows[0][1] + 1 == 2521
    deltas = PC.challenges(0x6230, c)[3]
    got = compute_all_lookup_polys(c.wires, nr, cfg.max_quotient_degree_factor, deltas, c.lookup_rows, nc)
    npoly = cd.num_lookup_polys
    for k in range(nc):
        d = deltas[4 * k:4 * k + 4]
        want = oracle.lookup_polys(c.wires, nr, cfg.max_quotient_degree_factor, d, c.lookup_rows)
        bad = np.argwhere(got[k * npoly:(k + 1) * npoly] != want)
        assert not bad.size, "challenge %d: first wrong (column, row) %s of %d" % (k, bad[0], len(bad))
        re_evals = cd.lut_re_poly_evals(d)
        for (_, last_lut, _), re in zip(c.lookup_rows, re_evals):
            assert int(got[k * npoly, last_lut]) == re
    data, parts = _prove(pb, c, DIGEST)
    assert _verify(oracle, c, DIGEST, parts) is None
    bad = dict(parts, openings=dict(parts["openings"]))
    wv = bad["openings"]["wires"].copy()
    wv[5, 1] ^= np.uint64(1)
    bad["openings"]["wires"] = wv
    assert _verify(oracle, c, DIGEST, bad) is not None
    assert _verify(oracle, c, DIGEST, dict(parts, public_inputs=PUBLIC_INPUTS[:-1] + [7])) is not None
    last_lu, _, first_lut = c.lookup_rows[0]
    for col, row in ((1, last_lu + 3), (2, first_lut)):    # a looking output, the multiplicity of table entry 0
        wires = c.wires.copy()
        wires[col, row] = (int(wires[col, row]) + 1) % PC.P
        assert _verify(oracle, c, DIGEST, _prove(pb, c, DIGEST, wires)[1]) is not None


@pytest.mark.gpu
@pytest.mark.parametrize("qdf", [3, 8])
def test_a_bad_witness_past_row_4096_is_rejected(pb, oracle, qdf):
    """Case e: one arithmetic output off by one at a row past 4096. qdf 3: the quotient has a non-zero tail and
    compute_quotient_polys raises "Quotient has failed". qdf 8 (no tail to check): the proof is made and the verifier
    rejects it."""
    from plonky2_b200 import NativeError

    c = PL.large_circuit(13, qdf=qdf, break_arith=5000, public_inputs=PUBLIC_INPUTS)
    assert c.broken_row > 4096
    if qdf == 3:
        ch = PC.challenges(0x6240, c)
        cs, w, z, _ = _device_commitments(pb, c, ch)
        try:
            with pytest.raises((NativeError, ValueError), match="Quotient has failed"):
                _device_quotient(c, cs, w, z, ch)
        finally:
            for b in (cs, w, z):
                b.close()
    else:
        assert _verify(oracle, c, DIGEST, _prove(pb, c, DIGEST)[1]) == "vanishing polynomial identity fails for challenge 0"


@pytest.mark.gpu
@pytest.mark.skipif(os.environ.get("GL_LARGE_PLONK_20") != "1",
                    reason="2^20 gates: set GL_LARGE_PLONK_20=1 (the witness alone is 1.1 GB on the host)")
def test_recursion_circuit_2_20(pb, oracle):
    """Case f: the standard config at 2^20 gates: the verifier identity of the device quotient, and the device proof
    accepted by the restated verifier."""
    c = PL.large_circuit(20, luts="range16", public_inputs=PUBLIC_INPUTS)
    _check_identity_on_device(pb, oracle, c, 0x6250)
    assert _verify(oracle, c, DIGEST, _prove(pb, c, DIGEST)[1]) is None
