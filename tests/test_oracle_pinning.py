"""Pin the CPU oracle against every stored vector / definitional check the reference's own tests hold
for the hot path (SURVEY.md section 8c). CPU only.

Reference tests mirrored here:
  * Poseidon KATs + fast==naive      plonky2/src/hash/poseidon_goldilocks.rs:455-495, poseidon.rs:926-957
    (and the batched permutation and the proof-of-work search the device tests take expected values from)
  * bit-reversal golden table         plonky2/src/util/mod.rs:60-126
  * prime-field edge arithmetic       field/src/prime_field_testing.rs:7-17,69-183
  * fft_and_ifft vs naive evaluation  field/src/fft.rs:215-282
  * coset fft/ifft vs naive           field/src/polynomial/mod.rs:476-516
  * Merkle proofs for every leaf      plonky2/src/hash/merkle_tree.rs:253-311
  * digest layout == commit_single    plonky2/src/hash/batch_merkle_tree.rs:185-228
"""
import json
import os

import numpy as np
import pytest

from conftest import EDGE, P, synth

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def test_poseidon_known_answer_vectors(oracle):
    kat = json.load(open(os.path.join(GOLD, "poseidon_kat.json")))
    assert len(kat["vectors"]) == 4
    for v in kat["vectors"]:
        inp = [int(x) for x in v["input"]]
        exp = [int(x) for x in v["output"]]
        assert oracle.poseidon(inp).tolist() == exp
        assert oracle.poseidon(inp, naive=True).tolist() == exp


def test_poseidon_fast_equals_naive(oracle):
    xs = synth(0x77, (200, 12), canonical=False)
    for row in xs:
        assert oracle.poseidon(row).tolist() == oracle.poseidon(row, naive=True).tolist()


def test_poseidon_many_equals_one_state_at_a_time(oracle):
    # the batched permutation the device tests take their expected values from, against the pinned single-state forms
    kat = json.load(open(os.path.join(GOLD, "poseidon_kat.json")))
    st = synth(0x78, (4096, 12), canonical=False)
    st[:4] = np.array([[int(x) for x in v["input"]] for v in kat["vectors"]], dtype=np.uint64)
    st[4:4 + len(EDGE)] = np.array([EDGE[i:] + EDGE[:i] for i in range(len(EDGE))], dtype=np.uint64)
    st[100:600] |= np.uint64(0xFFFFFFF0FFFFFFF0)
    st[600:1100] = np.uint64(2**64 - 1) - (st[600:1100] & np.uint64(0xFF))
    st[1100:1600, :8] = 0
    got = oracle.poseidon_many(st, nthreads=3)
    assert got[:4].tolist() == [[int(x) for x in v["output"]] for v in kat["vectors"]]
    for i, row in enumerate(st):
        want = oracle.poseidon(row).tolist()
        assert got[i].tolist() == want, i
        assert oracle.poseidon(row, naive=True).tolist() == want, i
    assert np.array_equal(oracle.poseidon_many(st, nthreads=1), got)


def test_pow_min_nonce_is_the_first_qualifying_nonce(oracle):
    # fri_proof_of_work's rule (prover.rs:183-194), restated as a plain loop over the oracle permutation
    for bits in range(11):
        pos = bits % 8
        st = synth(0x79 + bits, (12,), canonical=False)
        st[(pos + 3) % 12] = np.uint64(P + bits)  # a word that is not canonical
        want = 0
        while True:
            s = st.copy()
            s[pos] = want
            if 64 - int(oracle.poseidon(s)[7]).bit_length() >= bits:
                break
            want += 1
        assert oracle.pow_min_nonce(st, pos, bits, 1 << 20) == want, bits
        assert oracle.pow_min_nonce(st, pos, bits, want + 1, nthreads=1) == want, bits
        assert oracle.pow_min_nonce(st, pos, bits, want) == oracle.NO_NONCE, bits


def test_bit_reversal_golden_table(oracle):
    table = json.load(open(os.path.join(GOLD, "bitrev256.json")))["table"]
    arr = np.arange(256, dtype=np.uint64)
    oracle.lib().glo_reverse_index_bits_in_place(oracle.ptr(arr), 256, 1)
    assert arr.tolist() == table
    assert oracle.lib().glo_reverse_bits(0b1000000000, 10) == 1
    assert oracle.lib().glo_reverse_bits(0b01011, 5) == 0b11010
    arr4 = np.array([10, 20, 30, 40], dtype=np.uint64)
    oracle.lib().glo_reverse_index_bits_in_place(oracle.ptr(arr4), 4, 1)
    assert arr4.tolist() == [10, 30, 20, 40]


def test_prime_field_edge_arithmetic(oracle):
    L = oracle.lib()
    ins = [int(x) for x in json.load(open(os.path.join(GOLD, "field_edge_inputs.json")))["inputs"]]
    ins = ins[::3] + EDGE
    for a in ins:
        assert L.glo_neg(a) == (-a) % P
        assert L.glo_canon(a) == a % P
        for b in ins:
            assert L.glo_add(a, b) == (a + b) % P
            assert L.glo_sub(a, b) == (a - b) % P
            assert L.glo_mul(a, b) == (a * b) % P
    for a in ins:
        if a % P:
            assert L.glo_mul(L.glo_inv(a), a) == 1


def test_field_constants(oracle):
    L = oracle.lib()
    # SURVEY appendix A items 2-4
    assert L.glo_primitive_root_of_unity(6) == 8
    assert L.glo_primitive_root_of_unity(1) == P - 1
    assert L.glo_primitive_root_of_unity(20) == 1971462654193939361
    assert L.glo_primitive_root_of_unity(23) == 5936499541590631774
    assert L.glo_coset_shift() == 14293326489335486720
    for k in range(0, 33):
        assert L.glo_mul(L.glo_inverse_2exp(k), pow(2, k, P)) == 1
    w32 = L.glo_primitive_root_of_unity(32)
    assert pow(w32, 1 << 32, P) == 1 and pow(w32, 1 << 31, P) == P - 1


def test_ext2(oracle):
    xs = synth(0x99, (20, 4), canonical=False)
    for a0, a1, b0, b1 in xs.tolist():
        out = np.zeros(2, dtype=np.uint64)
        oracle.lib().glo_ext2_mul(oracle.ptr(np.array([a0, a1], dtype=np.uint64)),
                                  oracle.ptr(np.array([b0, b1], dtype=np.uint64)), oracle.ptr(out))
        assert out.tolist() == [(a0 * b0 + 7 * a1 * b1) % P, (a0 * b1 + a1 * b0) % P]
        inv = np.zeros(2, dtype=np.uint64)
        oracle.lib().glo_ext2_inv(oracle.ptr(np.array([a0, a1], dtype=np.uint64)), oracle.ptr(inv))
        i0, i1 = inv.tolist()
        assert [(a0 * i0 + 7 * a1 * i1) % P, (a0 * i1 + a1 * i0) % P] == [1, 0]


def test_fft_and_ifft_match_naive(oracle):
    # field/src/fft.rs:215-249: degree 200 padded to 256, deterministic coefficients i*1337 % 100
    degree, padded = 200, 256
    coeffs = np.array([(i * 1337) % 100 for i in range(degree)] + [0] * (padded - degree), dtype=np.uint64)
    naive = oracle.naive_coset_eval(coeffs, 1)
    points = oracle.fft(coeffs)
    assert points.tolist() == naive.tolist()
    assert oracle.ifft(points).tolist() == coeffs.tolist()
    for r in range(4):
        # zero_factor only valid when the top (1 - 2^-r) is zero: extend by zeros like the reference
        ext = np.concatenate([coeffs, np.zeros(padded * ((1 << r) - 1), dtype=np.uint64)])
        assert oracle.fft(ext, zero_factor=r).tolist() == oracle.fft(ext).tolist()


@pytest.mark.parametrize("log_n", [0, 1, 2, 3, 5, 8])
def test_coset_fft_matches_naive(oracle, log_n):
    n = 1 << log_n
    coeffs = synth(0x31 + log_n, (n,))
    shift = int(synth(0x41, (1,))[0]) or 3
    got = oracle.coset_fft(coeffs, shift)
    assert got.tolist() == oracle.naive_coset_eval(coeffs, shift).tolist()
    assert oracle.coset_ifft(got, shift).tolist() == coeffs.tolist()
    # pure-python definition as a third opinion
    w = oracle.lib().glo_primitive_root_of_unity(log_n)
    exp = [sum(int(c) * pow(shift * pow(w, i, P) % P, k, P) for k, c in enumerate(coeffs)) % P for i in range(n)]
    assert got.tolist() == exp


def test_sponge_semantics(oracle):
    # hash_or_noop no-op threshold (config.rs:63-74) and overwrite-mode partial chunk (hashing.rs:118-141)
    for w in range(0, 5):
        x = synth(0x51, (w,), canonical=False)
        exp = [int(v) % P for v in x] + [0] * (4 - w)
        assert oracle.hash_or_noop(x).tolist() == exp
    x = synth(0x52, (12,))
    st = np.zeros(12, dtype=np.uint64)
    st[:8] = x[:8]
    st = oracle.poseidon(st)
    st[:4] = x[8:]  # partial chunk overwrites only its own length; lanes 4.. keep previous output
    st = oracle.poseidon(st)
    assert oracle.hash_no_pad(x).tolist() == st[:4].tolist()
    assert oracle.hash_or_noop(x).tolist() == st[:4].tolist()
    l, r = synth(0x53, (4,)), synth(0x54, (4,))
    st = oracle.poseidon(np.concatenate([l, r, np.zeros(4, dtype=np.uint64)]))
    assert oracle.two_to_one(l, r).tolist() == st[:4].tolist()


@pytest.mark.parametrize("cap_height", [0, 1, 3, 8])
def test_merkle_every_proof_verifies(oracle, cap_height):
    # merkle_tree.rs:269-311: 256 leaves x 7
    leaves = synth(0x61, (256, 7))
    digests, cap = oracle.merkle_build(leaves, cap_height)
    for i in range(256):
        sib = oracle.merkle_prove(i, 256, cap_height, digests)
        assert len(sib) == 8 - cap_height
        assert oracle.merkle_verify(leaves[i], i, sib, cap, cap_height)
    bad = leaves[3].copy()
    bad[0] ^= np.uint64(1)
    assert not oracle.merkle_verify(bad, 3, oracle.merkle_prove(3, 256, cap_height, digests), cap, cap_height)


def test_merkle_cap_too_big(oracle):
    with pytest.raises(ValueError):
        oracle.merkle_build(synth(1, (8, 5)), 4)


def test_merkle_digest_layout(oracle):
    # batch_merkle_tree.rs:185-228 (commit_single): explicit layout for 4 leaves, cap_height 0
    leaves = synth(0x62, (4, 9))
    digests, cap = oracle.merkle_build(leaves, 0)
    h = [oracle.hash_or_noop(l) for l in leaves]
    h01, h23 = oracle.two_to_one(h[0], h[1]), oracle.two_to_one(h[2], h[3])
    root = oracle.two_to_one(h01, h23)
    assert digests.tolist() == [x.tolist() for x in (h[0], h[1], h01, h23, h[2], h[3])]
    assert cap.tolist() == [root.tolist()]
    # closed form of SURVEY row a12 vs the recursive fill, 64 leaves, cap_height 2
    leaves = synth(0x63, (64, 5))
    digests, cap = oracle.merkle_build(leaves, 2)
    sub = 2 * (16 - 1)
    for c in range(4):
        layer = [oracle.hash_or_noop(l) for l in leaves[16 * c:16 * (c + 1)]]
        i = 0
        while len(layer) > 1:
            for q, node in enumerate(layer):
                pos = 2 * (((q >> 1) << (i + 1)) + (1 << i) - 1) + (q & 1)
                assert digests[c * sub + pos].tolist() == node.tolist()
            layer = [oracle.two_to_one(layer[2 * k], layer[2 * k + 1]) for k in range(len(layer) // 2)]
            i += 1
        assert cap[c].tolist() == layer[0].tolist()


def test_commit_matches_definition(oracle):
    # from_values == ifft -> lde -> coset_fft -> transpose -> bit-reverse rows -> MerkleTree (oracle.rs:57-112)
    B, log_n, r, hc = 5, 4, 2, 1
    n, N = 1 << log_n, 1 << (log_n + r)
    vals = synth(0x71, (B, n))
    c = oracle.Commit(vals, r, hc)
    coeffs = np.stack([oracle.ifft(v) for v in vals])
    assert c.coeffs.tolist() == coeffs.tolist()
    g = oracle.lib().glo_coset_shift()
    lde = np.stack([oracle.naive_coset_eval(np.concatenate([co, np.zeros(N - n, dtype=np.uint64)]), g)
                    for co in coeffs])
    leaves = c.leaves
    for j in range(N):
        i = oracle.lib().glo_reverse_bits(j, log_n + r)
        assert leaves[j].tolist() == lde[:, i].tolist()
    d, cap = oracle.merkle_build(leaves, hc)
    assert c.cap.tolist() == cap.tolist() and c.digests.tolist() == d.tolist()
    assert c.get_lde_values(3, 2).tolist() == lde[:, 6].tolist()
    # original values are the LDE's restriction? (values = P on <w_n>, LDE on g<w_N>: check via coeffs instead)
    c2 = oracle.Commit(coeffs, r, hc, is_coeffs=True)
    assert c2.cap.tolist() == c.cap.tolist()


def test_challenger_semantics(oracle):
    # challenger.rs:82-92,129-144: pop from the back; partial input flush overwrites only its length
    ch = oracle.Challenger()
    xs = synth(0x81, (11,))
    ch.observe_elements(xs)
    st = np.zeros(12, dtype=np.uint64)
    st[:8] = xs[:8]
    st = oracle.poseidon(st)
    st[:3] = xs[8:]
    st = oracle.poseidon(st)
    got = ch.get_n_challenges(8)
    assert got == st[:8][::-1].tolist()
    nxt = oracle.poseidon(st)
    assert ch.get_challenge() == int(nxt[7])


def test_stark_quotient_fibonacci_satisfies_the_verifier_identity(oracle):
    """The oracle's compute_quotient_polys restatement (starky/src/prover.rs:488-668) is pinned by the verifier's own
    check (starky/src/verifier.rs:150-190): at a random point z, sum_k alpha^.. C_k(z) == Z_H(z) * q(z)."""
    import plonky2_b200 as pb

    P_ = int(P)
    log_n, r, h = 7, 1, 0
    n = 1 << log_n
    stark = pb.FibonacciStark(n)
    trace = stark.generate_trace(3, 5)
    pi = [3, 5, int(trace[1, n - 1])]
    alphas = [int(x) for x in synth(0xD1, (2,))]
    tc = oracle.Commit(trace, r, h)
    q = oracle.stark_quotient_fibonacci(tc, pi, alphas)
    assert q.shape == (2, n)
    coeffs = tc.coeffs
    z = int(synth(0xD2, (1,))[0])
    w = pb.field.primitive_root_of_unity(log_n)
    last = pow(w, P_ - 2, P_)

    def ev(c, x):
        acc = 0
        for v in c[::-1]:
            acc = (acc * x + int(v)) % P_
        return acc

    l = [ev(coeffs[k], z) for k in range(2)]
    nx = [ev(coeffs[k], z * w % P_) for k in range(2)]
    zh = (pow(z, n, P_) - 1) % P_
    l_first = zh * pow(n * (z - 1) % P_, P_ - 2, P_) % P_
    l_last = zh * last % P_ * pow(n * (z - last) % P_, P_ - 2, P_) % P_
    z_last = (z - last) % P_
    cons = [(l[0] - pi[0]) * l_first, (l[1] - pi[1]) * l_first, (l[1] - pi[2]) * l_last, (nx[0] - l[1]) * z_last,
            (nx[1] - l[0] - l[1]) * z_last]
    for j, a in enumerate(alphas):
        acc = 0
        for c in cons:
            acc = (acc * a + c) % P_
        assert acc == zh * ev(q[j], z) % P_
    # a wrong public input makes the vanishing polynomial indivisible by Z_H: the "quotient" picks up high coefficients
    bad = oracle.stark_quotient_fibonacci(tc, [3, 5, (pi[2] + 1) % P_], alphas)
    acc = 0
    for c in [(l[0] - 3) * l_first, (l[1] - 5) * l_first, (l[1] - pi[2] - 1) * l_last, cons[3], cons[4]]:
        acc = (acc * alphas[0] + c) % P_
    assert acc != zh * ev(bad[0], z) % P_


def test_batch_fri_with_one_degree_equals_plain_fri(oracle):
    """Pin of the batch-FRI restatement (batch_fri/oracle.rs, batch_fri/prover.rs): with a single degree group the
    BatchMerkleTree is the MerkleTree and batch_fri_proof is fri_proof, so the proof bytes must equal the plain
    prove_openings bytes (which the restated verifier accepts, see above)."""
    log_n, r, h = 8, 2, 3
    cols = synth(0xD8, (3, 1 << log_n))
    bc = oracle.BatchCommit([c for c in cols], r, h)
    pc = oracle.Commit(cols, r, h)
    assert np.array_equal(bc.cap, pc.cap)
    params = oracle.make_params(r, h, 5, 6, [2, 3])
    ch1, ch2 = oracle.Challenger(), oracle.Challenger()
    for ch in (ch1, ch2):
        ch.observe_cap(pc.cap)
    z = (12345, 67890)
    batches = [(z, [(0, 0), (0, 1), (0, 2)]), ((777, 1), [(0, 1)])]
    a = oracle.batch_prove_openings([bc], [log_n], [batches], ch1, params)
    b = oracle.prove_openings([pc], batches, ch2, params)
    assert a == b


def test_lookup_polys_restatement_satisfies_the_lookup_argument(oracle):
    """Pin of the compute_lookup_polys restatement (plonk/prover.rs:458-577) by the argument's own invariant: with
    multiplicities that count the looked-up pairs, the running Sum - LDC ends at 0 in the last partial polynomial at the
    last lookup row ("If the lookup argument is valid, then it must be equal to 0", prover.rs:456-457), and does not when
    one looking pair is not in the table. RE is checked against its definition (Horner in delta over the table rows)."""
    P_ = int(P)
    routed, qdf, log_n = 6, 3, 5          # 3 looking slots, 2 table slots per row; P = 2 partial polynomials
    n = 1 << log_n
    last_lu, last_lut, first_lut = 4, 8, 10   # LU rows 4..7, LUT rows 8..10
    wires = np.zeros((routed, n), dtype=np.uint64)
    table = [(int(a), int(b)) for a, b in synth(0xD9, (6, 2))]
    rng = [int(x) for x in synth(0xDA, (12,), canonical=False)]
    counts = [0] * 6
    k = 0
    for row in range(last_lu, last_lut):
        for s in range(3):
            e = rng[k] % 6
            k += 1
            counts[e] += 1
            wires[2 * s, row], wires[2 * s + 1, row] = table[e]
    for i, (a, b) in enumerate(table):
        row, s = last_lut + i // 2, i % 2
        wires[3 * s, row], wires[3 * s + 1, row], wires[3 * s + 2, row] = a, b, counts[i]
    deltas = [int(x) for x in synth(0xDB, (4,))]
    out = oracle.lookup_polys(wires, routed, qdf, deltas, [(last_lu, last_lut, first_lut)])
    assert out.shape == (3, n)
    assert int(out[2, last_lu]) == 0                      # Sum(end) - LDC(end)
    assert not out[:, :last_lu].any() and not out[:, first_lut + 1:].any()
    # RE by its definition
    re = 0
    for row in range(first_lut, last_lut - 1, -1):
        for s in range(2):
            re = (re * deltas[3] + int(wires[3 * s, row]) + deltas[1] * int(wires[3 * s + 1, row])) % P_
        assert int(out[0, row]) == re
    bad = wires.copy()
    bad[0, last_lu] = (int(bad[0, last_lu]) + 1) % P_     # a looking pair that is not in the table
    out2 = oracle.lookup_polys(bad, routed, qdf, deltas, [(last_lu, last_lut, first_lut)])
    assert int(out2[2, last_lu]) != 0


def test_partial_products_restatement_satisfies_the_permutation_argument(oracle):
    """Pin of the wires_permutation_partial_products_and_zs restatement (plonk/prover.rs:387-449) by the permutation
    argument itself: for wire values that respect the copy constraints encoded in sigma, the grand product telescopes,
    Z(g^n) = Z(1) = 1 -- and every partial product obeys pp_m(x) = pp_{m-1}(x) * q_m(x) (util/partial_products.rs:13-37)."""
    P_ = int(P)
    import plonky2_b200.field as F

    R, log_n, deg = 4, 3, 2
    n = 1 << log_n
    w = F.primitive_root_of_unity(log_n)
    k_is = [1, 7, 49, 343]
    wires = synth(0xDC, (R, n)).copy()
    ids = np.array([[k_is[j] * pow(w, i, P_) % P_ for i in range(n)] for j in range(R)], dtype=np.uint64)
    sigmas = ids.copy()
    # copy constraints: (row 1, wire 0) == (row 5, wire 2) and (row 2, wire 1) == (row 2, wire 3): swap their ids in sigma
    sigmas[0, 1], sigmas[2, 5] = ids[2, 5], ids[0, 1]
    sigmas[1, 2], sigmas[3, 2] = ids[3, 2], ids[1, 2]
    wires[2, 5] = wires[0, 1]
    wires[3, 2] = wires[1, 2]
    beta, gamma = [int(x) for x in synth(0xDD, (2,))]
    out = oracle.partial_products_and_zs(wires, sigmas, np.array(k_is, dtype=np.uint64), beta, gamma, deg)
    assert out.shape == (2, n)          # one partial product column, then Z
    pp, Z = out[0], out[1]

    def q(i, m):
        num = den = 1
        for j in range(m * deg, min((m + 1) * deg, R)):
            num = num * (int(wires[j, i]) + beta * int(ids[j, i]) + gamma) % P_
            den = den * (int(wires[j, i]) + beta * int(sigmas[j, i]) + gamma) % P_
        return num * pow(den, P_ - 2, P_) % P_

    assert int(Z[0]) == 1
    for i in range(n):
        assert int(pp[i]) == int(Z[i]) * q(i, 0) % P_
        nxt = int(pp[i]) * q(i, 1) % P_
        assert nxt == (int(Z[i + 1]) if i + 1 < n else 1)     # the product wraps around to Z(1) = 1
    wires[2, 5] = (int(wires[2, 5]) + 1) % P_                   # break one copy constraint: the product no longer closes
    out2 = oracle.partial_products_and_zs(wires, sigmas, np.array(k_is, dtype=np.uint64), beta, gamma, deg)
    last = int(out2[0][n - 1]) * (lambda i: q(i, 1))(n - 1) % P_
    assert last != 1


def test_batch_fri_proof_passes_the_restated_batch_verifier(oracle):
    """Pin of the multi-degree batch-FRI restatement: its proof (the reference test's shape, batch_fri/prover.rs:341-477,
    plus a richer one) is accepted by the restated verify_batch_fri_proof (batch_fri/verifier.rs:22-251) with the
    polynomials' true openings, and rejected with a wrong opening or a flipped byte."""
    for lens, counts, r, h, arities, nq, pow_bits in ([9, 8, 6], [1, 1, 1], 1, 5, [1, 2, 1], 10, 0), ([10, 8, 6], [3, 2, 2], 2, 3, [2, 2, 2], 5, 4):
        polys, degree_of = [], []
        for k, c in zip(lens, counts):
            for j in range(c):
                polys.append(synth(0x200 + 16 * k + j, (1 << k,)))
                degree_of.append(k)
        oo = oracle.BatchCommit(polys, r, h)
        coeffs = [oracle.ifft(p) for p in polys]
        och = oracle.Challenger()
        och.observe_cap(oo.cap)
        zeta = och.get_extension_challenge()
        instances, opened = [], []
        for k in lens:
            idx = [i for i, d in enumerate(degree_of) if d == k]
            instances.append([(zeta, [(0, i) for i in idx])])
            opened += [oracle.eval_poly_base_at_ext(coeffs[i], zeta) for i in idx]
        vch = och.clone()
        params = oracle.make_params(r, h, pow_bits, nq, arities)
        proof = oracle.batch_prove_openings([oo], lens, instances, och, params)
        ov = np.array(opened, dtype=np.uint64)
        assert oracle.verify_batch_fri_proof([oo.cap], [counts], lens, instances, ov, vch.clone(), params, proof) == 0
        bad = ov.copy()
        bad[0, 0] ^= np.uint64(1)
        assert oracle.verify_batch_fri_proof([oo.cap], [counts], lens, instances, bad, vch.clone(), params, proof) != 0
        flipped = bytearray(proof)
        flipped[len(flipped) // 2] ^= 8
        assert oracle.verify_batch_fri_proof([oo.cap], [counts], lens, instances, ov, vch.clone(), params, bytes(flipped)) != 0


def test_partial_products_reference_golden_numbers(oracle):
    """The reference's own numbers (util/partial_products.rs:118-145): v = [1..6], denominators 1, z_x = 1: chunk products
    [2, 12, 30] -> partial products [2, 24] and z_gx = 720 at degree 2; [6, 120] -> [6] and 720 at degree 3. Realised
    through the restated wires_permutation_partial_products_and_zs with w = 0, beta = 1, gamma = 0, k_i = v on row 0
    (x = 1) and sigma = 1 there: numerators v, denominators 1."""
    from plonky2_b200.plonk import num_partial_products

    v = [1, 2, 3, 4, 5, 6]
    wires = np.zeros((6, 2), dtype=np.uint64)
    sigmas = np.ones((6, 2), dtype=np.uint64)
    sigmas[:, 1] = synth(0xDE, (6,))      # row 1 is arbitrary
    for degree, pps in ((2, [2, 24]), (3, [6])):
        out = oracle.partial_products_and_zs(wires, sigmas, np.array(v, dtype=np.uint64), 1, 0, degree)
        assert num_partial_products(len(v), degree) == len(pps) == out.shape[0] - 1
        assert [int(x) for x in out[:-1, 0]] == pps          # the partial products of row 0
        assert int(out[-1, 0]) == 1 and int(out[-1, 1]) == 720   # Z(1) = 1, Z(g) = z_gx
