"""Test infrastructure: plonky2 circuits at the size of a real recursion circuit (2^13 .. 2^20 gates), built with numpy.

LargeCircuit produces what tests/plonk_circuits.FibonacciCircuit produces (common, wires, sigmas, constants_sigmas,
lookup_rows, public_inputs_hash, oracle_circuit(), oracle_zs_partial_products()), so oracle_prove, oracle_verify,
fri_batches and ProofWithPublicInputs.from_bytes work on it. Its rows:
  - row 0 PublicInputGate, row 1 ConstantGate(2);
  - ArithmeticGate rows fill the circuit; every operation out = m0 * m1 * c0 + addend * c1 is independent, with random
    operands and random per-row constants (c0, c1). The addend of the operation k at arithmetic row t is copied from the
    out of operation k + 7 (mod num_ops) at arithmetic row t - D, D > 4096 rows once there are enough of them;
  - three long copy cycles span the whole trace (one of them through the ConstantGate's wire);
  - PoseidonGate rows (a hash chain: outputs 0..3 copied into the next row's inputs 0..3) and one row of every other
    gate type, spread over four places: the start, the middle, past row 4096 (the middle third on small circuits), and
    the last rows before the lookup section;
  - optionally lookup tables, laid out as CircuitBuilder::add_all_lookups (gadgets/lookup.rs:80-155) lays them out: per
    table its LookupGate rows, its LookupTableGate rows "upside down", then one NoopGate row;
  - NoopGate rows pad to 2^degree_bits.
The sigmas come from one vectorised get_sigma_map (permutation_argument.rs:113-157) over the copy cycles."""
import numpy as np

import gl_numpy as gn
import oracle_lib as OL
import plonk_circuits as PC

P = PC.P
QDF3_EXTRA = ("ArithmeticExtensionGate", "MulExtensionGate", "BaseSumGate", "ReducingGate", "ReducingExtensionGate",
              "PoseidonMdsGate")   # the gate types of degree < 4, which fit quotient_degree_factor 3


def range_table(bits=16):
    """A 2^bits-entry table over u16 inputs: input e, output an affine map of e (mod 2^16)."""
    e = np.arange(1 << bits, dtype=np.int64)
    return list(zip(e.tolist(), ((e * 40503 + 11) & 0xFFFF).tolist()))


def small_table():
    return [(3 * e + 1, (e * e + 7) & 0xFFFF) for e in range(30)]


class LargeCircuit:
    """luts: a list of (table, number of LookupGate rows). break_arith: an arithmetic row at which one operation's out
    is off by one (the vanishing polynomial is then not divisible by Z_H)."""

    def __init__(self, plonk, config, degree_bits, seed=1, poseidon_rows=8, extra=PC.OTHER_GATES, luts=(),
                 public_inputs=None, break_arith=None):
        rng = np.random.default_rng(seed)
        n = 1 << degree_bits
        self.config, self.n = config, n
        nw, nr = config.num_wires, config.num_routed_wires
        arith = plonk.ArithmeticGate.new_from_config(config)
        K = arith.num_ops
        lu_slots, lut_slots = nr // 2, nr // 3
        # ---- rows: lookup section at the end of the circuit, two NoopGate rows of padding after it at least
        lookup_rows = []
        body_end = n - 2 - sum(lu_rows + -(-len(lut) // lut_slots) + 1 for lut, lu_rows in luts)
        extra_rows = [PC.extra_gate_row(plonk, config, name, rng)[:3] for name in extra]
        specials = ["poseidon"] * poseidon_rows + list(range(len(extra_rows)))
        groups = [specials[g::4] for g in range(4)]
        anchors = [2, n // 2, 4096 + 37 if n > 8192 else n // 3 + 5, body_end - len(groups[3])]
        kind = {}                                 # row -> "poseidon" or an index into extra_rows
        for g, a in zip(groups, anchors):
            for k, s in enumerate(g):
                assert a + k not in kind and 2 <= a + k < body_end, "circuit too small for its special rows"
                kind[a + k] = s
        arows = np.array([r for r in range(2, body_end) if r not in kind], dtype=np.int64)
        A = len(arows)
        self.arith_rows = arows
        instances = [(plonk.PublicInputGate(), [])] * n
        c0c1 = [int(v) for v in PC.rnd(rng, 2)]
        instances[1] = (plonk.ConstantGate(2), c0c1)
        consts = PC.rnd(rng, (2, A))
        for t, r in enumerate(arows.tolist()):
            instances[r] = (arith, consts[:, t])
        for r, s in kind.items():
            instances[r] = (plonk.PoseidonGate(), []) if s == "poseidon" else extra_rows[s][:2]
        row = body_end
        for t, (lut, lu_rows) in enumerate(luts):
            last_lu, last_lut = row, row + lu_rows
            first_lut = last_lut + -(-len(lut) // lut_slots) - 1
            instances[last_lu:last_lut] = [(plonk.LookupGate.new_from_config(config, t), [])] * lu_rows
            instances[last_lut:first_lut + 1] = [(plonk.LookupTableGate.new_from_config(config, t), [])] * (first_lut + 1 - last_lut)
            lookup_rows.append((last_lu, last_lut, first_lut))
            row = first_lut + 2
        for r in [fl + 1 for _, _, fl in lookup_rows] + list(range(row, n)):
            instances[r] = (plonk.NoopGate(), [])
        self.common, self.constant_vecs = plonk.CommonCircuitData.from_gate_instances(config, instances, [l for l, _ in luts],
                                                                                      lookup_rows)
        self.lookup_rows = lookup_rows
        self.public_inputs = public_inputs
        if public_inputs is None:
            self.public_inputs_hash = [int(v) for v in PC.rnd(rng, 4)]
        else:   # C::InnerHasher::hash_no_pad(&public_inputs), prover.rs:155
            self.public_inputs_hash = [int(v) for v in OL.hash_no_pad(np.array(public_inputs, dtype=np.uint64))]
        # ---- witness
        wires = PC.rnd(rng, (nw, n))
        wires[0:4, 0] = self.public_inputs_hash
        wires[0, 1], wires[1, 1] = c0c1
        cycles = []                               # (rows, cols), each of shape (L, m): m cycles of length L
        m0, m1, addend = PC.rnd(rng, (K, A)), PC.rnd(rng, (K, A)), PC.rnd(rng, (K, A))
        stride = max(1, A // 16)
        idx_a = np.arange(0, A, stride)           # cycle through the ConstantGate's c0 and m0 of operation 3
        m0[3 % K, idx_a] = c0c1[0]
        cycles.append((np.concatenate([[1], arows[idx_a]])[:, None], np.concatenate([[0], np.full(len(idx_a), 4 * (3 % K))])[:, None]))
        idx_b = np.arange(stride // 2, A, stride)   # two cycles of random values through m1 of operations 5 and 11
        for k in (5 % K, 11 % K):
            m1[k, idx_b] = int(PC.rnd(rng))
            cycles.append((arows[idx_b][:, None], np.full((len(idx_b), 1), 4 * k + 1)))
        D = 4097 if A > 4097 + 256 else max(1, A // 3)
        src = (np.arange(K) + 7) % K              # addend of operation k <- out of operation src[k]
        out = np.empty((K, A), dtype=np.uint64)
        for s in range(0, A, D):
            e = min(s + D, A)
            if s >= D:
                addend[:, s:e] = out[src, s - D:e - D]
            out[:, s:e] = gn.add(gn.mul(gn.mul(m0[:, s:e], m1[:, s:e]), consts[0, s:e]), gn.mul(addend[:, s:e], consts[1, s:e]))
        for k in range(K):
            wires[4 * k, arows], wires[4 * k + 1, arows], wires[4 * k + 2, arows], wires[4 * k + 3, arows] = (
                m0[k], m1[k], addend[k], out[k])
        if A > D:                                 # the addend copies: pairs (out at t - D, addend at t)
            t = np.arange(D, A)
            rows = np.stack([np.repeat(arows[t - D][None], K, 0).reshape(-1), np.repeat(arows[t][None], K, 0).reshape(-1)])
            cols = np.stack([np.repeat(4 * src[:, None] + 3, len(t), 1).reshape(-1),
                             np.repeat(4 * np.arange(K)[:, None] + 2, len(t), 1).reshape(-1)])
            cycles.append((rows, cols))
        prev = None
        PG = plonk.PoseidonGate
        for r in sorted(r for r, s in kind.items() if s == "poseidon"):
            inputs = [int(v) for v in PC.rnd(rng, 12)]
            if prev is not None:
                inputs[:4] = [int(wires[PG.wire_output(i), prev]) for i in range(4)]
                cycles.append((np.array([[prev] * 4, [r] * 4]), np.array([[PG.wire_output(i) for i in range(4)],
                                                                           [PG.wire_input(i) for i in range(4)]])))
            for k, v in PC.poseidon_gate_witness(plonk, inputs, r & 1).items():
                wires[k, r] = v
            prev = r
        for r, s in kind.items():
            if s != "poseidon":
                for k, v in extra_rows[s][2].items():
                    wires[k, r] = v
        for (lut, lu_rows), (last_lu, last_lut, first_lut) in zip(luts, lookup_rows):
            tab = np.array(lut, dtype=np.uint64)
            padded = np.concatenate([tab, np.repeat(tab[:1], (-len(tab)) % lut_slots, 0)])
            pick = rng.integers(0, len(tab), size=(lu_rows, lu_slots))
            for s_ in range(lu_slots):
                wires[2 * s_, last_lu:last_lut] = tab[pick[:, s_], 0]
                wires[2 * s_ + 1, last_lu:last_lut] = tab[pick[:, s_], 1]
            counts = np.bincount(pick.reshape(-1), minlength=len(padded)).astype(np.uint64)
            e = np.arange(len(padded))
            r_, s_ = first_lut - e // lut_slots, e % lut_slots
            wires[3 * s_, r_], wires[3 * s_ + 1, r_], wires[3 * s_ + 2, r_] = padded[:, 0], padded[:, 1], counts
        if break_arith is not None:
            r = int(arows[np.searchsorted(arows, break_arith)])
            wires[3, r] = (int(wires[3, r]) + 1) % P
            self.broken_row = r
        self.wires = wires
        self.cycles = cycles
        self.sigmas = sigma_values(self.common.k_is, nr, n, degree_bits, cycles)
        self.constants_sigmas = np.concatenate([np.stack(self.constant_vecs), self.sigmas])

    def partition(self):
        """The copy cycles as lists of (row, column) wires, in cycle order."""
        return [list(zip(R[:, j].tolist(), C_[:, j].tolist())) for R, C_ in self.cycles for j in range(R.shape[1])]

    oracle_circuit = PC.FibonacciCircuit.oracle_circuit
    oracle_zs_partial_products = PC.FibonacciCircuit.oracle_zs_partial_products


def large_circuit(degree_bits, qdf=8, rate_bits=3, nc=2, cap_height=4, luts="small", **kw):
    """A LargeCircuit of the standard recursion config's wires with the given quotient degree factor, rate, number of
    challenges and cap height. luts: None, "small" (two small tables) or "range16" (the 2^16-entry range table and a
    small table)."""
    from plonky2_b200 import plonk

    tables = {None: [], "small": [(small_table(), 2), ([(7 * e + 2, e) for e in range(41)], 1)],
              "range16": [(range_table(), 64), (small_table(), 2)]}[luts]
    if qdf == 3:
        kw.setdefault("extra", QDF3_EXTRA)
        kw.setdefault("poseidon_rows", 0)
    config = plonk.CircuitConfig(max_quotient_degree_factor=qdf, rate_bits=rate_bits, num_challenges=nc,
                                 cap_height=cap_height)
    return LargeCircuit(plonk, config, degree_bits, seed=degree_bits + 10 * nc + qdf, luts=tables, **kw)


def sigma_values(k_is, num_routed_wires, n, degree_bits, cycles):
    """get_sigma_map + get_sigma_polys, vectorised: sigma[col][row] = k_is[col'] * w^row' with (row', col') the next wire
    of (row, col)'s cycle (itself when it is in none)."""
    nxt_row = np.repeat(np.arange(n, dtype=np.int64)[None], num_routed_wires, 0)
    nxt_col = np.repeat(np.arange(num_routed_wires, dtype=np.int64)[:, None], n, 1)
    for R, C_ in cycles:
        nxt_row[C_, R] = np.roll(R, -1, axis=0)
        nxt_col[C_, R] = np.roll(C_, -1, axis=0)
    subgroup = gn.powers(PC.root_of_unity(degree_bits), n)
    return gn.mul(np.array(k_is, dtype=np.uint64)[nxt_col], subgroup[nxt_row])


def quotient_identity_failures(plonk, cd, public_inputs_hash, cs_coeffs, wires_coeffs, zs_coeffs, quotient_chunks, betas,
                               gammas, alphas, deltas, points, ev, pool=None):
    """The verifier's check of the quotient (plonk/verifier.rs:85-107) at each point x of `points` (pairs (a, b) of
    F_{p^2}; b = 0 for a base-field point), from the committed polynomials' coefficients:
        vanishing(x)[k] == Z_H(x) * sum_j x^(j n) q_{k,j}(x)      for every challenge k,
    q_{k,j} = quotient_chunks[k * qdf + j]. ev(coeffs, point) evaluates one polynomial. Any wrong quotient coefficient,
    or any wrong Z, partial-product or lookup column, breaks it except with probability about degree / p per point.
    Returns the (point, challenge) pairs where it fails."""
    import plonky2_b200.field as F

    nc, qdf = cd.config.num_challenges, cd.quotient_degree_factor
    g = PC.root_of_unity(cd.degree_bits)
    bad = []
    for x in points:
        o = PC.openings_at(cd, cs_coeffs, wires_coeffs, zs_coeffs, x, F.ext_mul((g, 0), x), ev, pool)
        vanishing, z_h, xn = PC.vanishing_at(plonk, cd, PC.Fp2(*x), o, public_inputs_hash, betas, gammas, alphas, deltas)
        q = [PC.Fp2(*v) for v in (pool.map(lambda p: ev(p, x), quotient_chunks) if pool else
                                  [ev(p, x) for p in quotient_chunks])]
        for k in range(nc):
            acc = PC.Fp2(0)
            for t in reversed(q[k * qdf:(k + 1) * qdf]):                       # reduce_with_powers(chunks, x^n)
                acc = acc * xn + t
            if not vanishing[k] == z_h * acc:
                bad.append((x, k))
    return bad
