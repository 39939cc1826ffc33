"""Test infrastructure: a Fibonacci-style plonky2 circuit built by hand (the CircuitBuilder is out of scope): gate
instances, a witness that satisfies every gate, copy constraints and the sigma polynomials they induce
(WirePartition::get_sigma_polys, plonky2/src/plonk/permutation_argument.rs:113-157); its zero-knowledge layout
(zk_circuit); the CPU twin of plonky2's prover and a restated verifier, with and without zero knowledge (oracle_prove,
oracle_verify, parts_of); and the oracle standing in for prove_with_witness's device calls (cpu_backends). Used by the
CPU pins and the GPU parity tests of the plonky2 quotient and proofs."""
import numpy as np

import gl_numpy as gn
import oracle_lib as OL

P = 0xFFFFFFFF00000001
G = 14293326489335486720   # MULTIPLICATIVE_GROUP_GENERATOR
KEYS = [bytes([k]) * 32 for k in (0x11, 0x22, 0x33)]   # salt keys of the wires, Z and quotient commitments
# every gate type FibonacciCircuit can add a row of (extra=), besides its arithmetic and Poseidon rows
OTHER_GATES = ("ArithmeticExtensionGate", "MulExtensionGate", "BaseSumGate", "BaseSumGate4", "ReducingGate",
               "ReducingExtensionGate", "PoseidonMdsGate", "RandomAccessGate", "ExponentiationGate",
               "CosetInterpolationGate")
# shape_circuit's shapes: (num_wires, num_routed_wires, max_quotient_degree_factor, rate_bits, degree_bits[,
# poseidon_rows[, other gates[, lookups]]])
SHAPES = [
    (12, 8, 4, 2, 4),     # two selector groups, partial-product chunks of 4
    (13, 8, 3, 2, 4),     # quotient_degree_factor 3: coset of 4n points, the top n coefficients must vanish
    (24, 16, 8, 3, 3),    # one selector for all gates, chunks of 8
    (135, 80, 8, 3, 5),   # CircuitConfig::standard_recursion_config
    (135, 80, 8, 3, 5, 9),  # ... with nine PoseidonGate rows (a hash chain): two selector groups, 123 gate constraints
    (135, 80, 8, 3, 5, 4, OTHER_GATES),   # ... and a row of every other gate type built so far: three selector groups
    # ... plus a lookup table of 30 entries on two LookupTableGate rows and 80 lookups on two LookupGate rows
    (135, 80, 8, 3, 5, 4, OTHER_GATES, True),
]
RECURSION_5 = SHAPES[3]                              # standard_recursion_config, 32 gates
LOOKUP_64 = (135, 80, 8, 3, 6, 4, OTHER_GATES, True)  # every gate type and a lookup table on 64 gates


def shape_circuit(shape, cap_height, num_challenges=2, **kw):
    """The FibonacciCircuit of a shape tuple, with a cap of 2^cap_height entries."""
    from plonky2_b200 import plonk

    nw, nr, qdf, rate_bits, degree_bits = shape[:5]
    for k, name in ((5, "poseidon_rows"), (6, "extra"), (7, "lookups")):
        if len(shape) > k:
            kw.setdefault(name, shape[k])
    cfg = plonk.CircuitConfig(num_wires=nw, num_routed_wires=nr, max_quotient_degree_factor=qdf, rate_bits=rate_bits,
                              cap_height=cap_height, num_challenges=num_challenges)
    return FibonacciCircuit(plonk, cfg, degree_bits, seed=nw + qdf + len(shape), **kw)


def quick_fri_config(config):
    """standard_recursion_config's FRI shape with fewer queries and grinding bits, so that the CPU twin stays quick."""
    from plonky2_b200.fri import FriConfig

    return FriConfig(rate_bits=config.rate_bits, cap_height=config.cap_height, proof_of_work_bits=6,
                     reduction_strategy=("ConstantArityBits", 2, 2), num_query_rounds=6)


def challenges(seed, c):
    """(betas, gammas, alphas, deltas) of a circuit: deltas only with lookups."""
    from conftest import synth

    nc = c.config.num_challenges
    v = [int(x) for x in synth(seed, (7 * nc,))]
    return v[:nc], v[nc:2 * nc], v[2 * nc:3 * nc], (v[3 * nc:] if c.common.luts else [])


def salts(c):
    """The salt arrays (4 x N, chacha_ref's restatement) of KEYS at the circuit's LDE size."""
    import chacha_ref as R

    return [R.salt_array(k, c.n << c.config.rate_bits) for k in KEYS]


def root_of_unity(bits):
    import plonky2_b200.field as F   # host-side field helpers (pure Python)

    return F.primitive_root_of_unity(bits)


def rnd(rng, shape=None):
    return rng.integers(0, P, size=shape, dtype=np.uint64)


class Fp:
    """A Goldilocks element as a plain Python int: lets the product's gate code (written over expression handles) run on
    numbers, for witness generation and for evaluating the vanishing polynomial at one point."""
    __slots__ = ("v",)

    def __init__(self, v):
        self.v = int(v) % P

    @staticmethod
    def _c(o):
        return o.v if isinstance(o, Fp) else int(o) % P

    def __add__(self, o):
        return Fp(self.v + Fp._c(o))

    def __sub__(self, o):
        return Fp(self.v - Fp._c(o))

    def __rsub__(self, o):
        return Fp(Fp._c(o) - self.v)

    def __mul__(self, o):
        return Fp(self.v * Fp._c(o))

    __radd__, __rmul__ = __add__, __mul__

    def __int__(self):
        return self.v


class PointVars:
    """EvaluationVarsBase over numbers: the values of the constants, wires and public-input hash at one point."""

    def __init__(self, constants, wires, public_inputs_hash, prefix=0):
        self.c, self.w, self.pih, self.prefix = constants, wires, public_inputs_hash, prefix

    def local_constant(self, i):
        return Fp(self.c[self.prefix + i])

    def local_wire(self, i):
        return Fp(self.w[i])

    def public_inputs_hash(self, i):
        return Fp(self.pih[i])

    def remove_prefix(self, n):
        return PointVars(self.c, self.w, self.pih, self.prefix + n)


def poseidon_gate_witness(plonk, inputs, swap):
    """PoseidonGenerator::run_once (gates/poseidon.rs:440-540): wire index -> value for one PoseidonGate row."""
    G_ = plonk.PoseidonGate
    t = plonk.poseidon_tables()
    wires = {G_.wire_input(i): int(inputs[i]) for i in range(12)}
    wires[G_.WIRE_SWAP] = int(swap)
    for i in range(4):
        wires[G_.wire_delta(i)] = int(swap) * (int(inputs[i + 4]) - int(inputs[i])) % P
    state = [Fp(v) for v in inputs]
    if swap:
        for i in range(4):
            state[i], state[i + 4] = state[i + 4], state[i]
    round_ctr = 0
    for r in range(4):
        state = G_._constant_layer(state, round_ctr)
        if r != 0:
            for i in range(12):
                wires[G_.wire_full_sbox_0(r, i)] = int(state[i])
        state = G_._mds_layer([G_._sbox_monomial(x) for x in state])
        round_ctr += 1
    state = [state[i] + t["FAST_FIRST_RC"][i] for i in range(12)]
    state = G_._mds_partial_layer_init(state)
    for r in range(22):
        wires[G_.wire_partial_sbox(r)] = int(state[0])
        state[0] = G_._sbox_monomial(state[0])
        if r < 21:
            state[0] = state[0] + t["FAST_RC"][r]
        state = G_._mds_partial_layer_fast(state, r)
    round_ctr += 22
    for r in range(4):
        state = G_._constant_layer(state, round_ctr)
        for i in range(12):
            wires[G_.wire_full_sbox_1(r, i)] = int(state[i])
        state = G_._mds_layer([G_._sbox_monomial(x) for x in state])
        round_ctr += 1
    for i in range(12):
        wires[G_.wire_output(i)] = int(state[i])
    return wires


def _ext(rng):
    return [int(v) for v in rnd(rng, 2)]


def _emul(plonk, x, y):
    r = plonk.Ext2(Fp(x[0]), Fp(x[1])) * plonk.Ext2(Fp(y[0]), Fp(y[1]))
    return [int(r.a), int(r.b)]


def extra_gate_row(plonk, config, name, rng):
    """(gate, constants, {wire: value}) of one row holding a satisfied instance of the named gate, the way the gate's
    generator fills it (gates/<gate>.rs: *Generator::run_once)."""
    wires = {}
    if name in ("ArithmeticExtensionGate", "MulExtensionGate"):
        arith = name == "ArithmeticExtensionGate"
        gate = getattr(plonk, name).new_from_config(config)
        consts = [int(v) for v in rnd(rng, 2 if arith else 1)]
        stride = 8 if arith else 6
        for i in range(gate.num_ops):
            m0, m1, addend = _ext(rng), _ext(rng), _ext(rng)
            prod = _emul(plonk, m0, m1)
            out = [(prod[k] * consts[0] + (addend[k] * consts[1] if arith else 0)) % P for k in range(2)]
            vals = m0 + m1 + (addend if arith else []) + out
            for k, v in enumerate(vals):
                wires[stride * i + k] = v
        return gate, consts, wires
    if name == "BaseSumGate":
        gate = plonk.BaseSumGate.new_from_config(config, 2)
        limbs = [int(v) & 1 for v in rnd(rng, gate.num_limbs)]
        wires[0] = sum(b << i for i, b in enumerate(limbs)) % P
        for i, b in enumerate(limbs):
            wires[1 + i] = b
        return gate, [], wires
    if name == "BaseSumGate4":
        gate = plonk.BaseSumGate(31, 4)
        limbs = [int(v) & 3 for v in rnd(rng, gate.num_limbs)]
        wires[0] = sum(b * 4 ** i for i, b in enumerate(limbs)) % P
        for i, b in enumerate(limbs):
            wires[1 + i] = b
        return gate, [], wires
    if name in ("ReducingGate", "ReducingExtensionGate"):
        cls = getattr(plonk, name)
        gate = cls(cls.max_coeffs_len(config.num_wires, config.num_routed_wires))
        ext = name == "ReducingExtensionGate"
        alpha, acc = _ext(rng), _ext(rng)
        wires[2], wires[3], wires[4], wires[5] = alpha + acc
        for i in range(gate.num_coeffs):
            coeff = _ext(rng) if ext else [int(rnd(rng)), 0]
            if ext:
                wires[6 + 2 * i], wires[7 + 2 * i] = coeff
            else:
                wires[6 + i] = coeff[0]
            prod = _emul(plonk, acc, alpha)
            acc = [(prod[0] + coeff[0]) % P, (prod[1] + coeff[1]) % P]
            at = gate.wires_accs(i)
            wires[at], wires[at + 1] = acc
        return gate, [], wires
    if name == "PoseidonMdsGate":
        gate = plonk.PoseidonMdsGate()
        ins = [_ext(rng) for _ in range(12)]
        outs = plonk.PoseidonGate._mds_layer([plonk.Ext2(Fp(a), Fp(b)) for a, b in ins])
        for i in range(12):
            wires[2 * i], wires[2 * i + 1] = ins[i]
            wires[2 * (12 + i)], wires[2 * (12 + i) + 1] = int(outs[i].a), int(outs[i].b)
        return gate, [], wires
    if name == "RandomAccessGate":
        gate = plonk.RandomAccessGate.new_from_config(config, 4)
        consts = [int(v) for v in rnd(rng, gate.num_extra_constants)]
        for copy in range(gate.num_copies):
            index = int(rnd(rng)) % gate.vec_size()
            items = [int(v) for v in rnd(rng, gate.vec_size())]
            wires[gate.wire_access_index(copy)] = index
            wires[gate.wire_claimed_element(copy)] = items[index]
            for i, v in enumerate(items):
                wires[gate.wire_list_item(i, copy)] = v
            for i in range(gate.bits):
                wires[gate.wire_bit(i, copy)] = (index >> i) & 1
        for i, v in enumerate(consts):
            wires[gate.wire_extra_constant(i)] = v
        return gate, consts, wires
    if name == "ExponentiationGate":
        gate = plonk.ExponentiationGate.new_from_config(config)
        n = gate.num_power_bits
        base = int(rnd(rng))
        bits = [int(v) & 1 for v in rnd(rng, n)]
        wires[0] = base
        cur = 1
        for i in range(n):
            wires[gate.wire_power_bit(i)] = bits[i]
        for i in range(n):                       # ExponentiationGenerator::run_once (exponentiation.rs:272-300)
            cur = cur * cur % P if i else 1
            cur = cur * (base if bits[n - 1 - i] else 1) % P
            wires[gate.wire_intermediate_value(i)] = cur
        wires[gate.wire_output()] = cur
        assert cur == pow(base, sum(b << i for i, b in enumerate(bits)), P)
        return gate, [], wires
    if name == "CosetInterpolationGate":
        gate = plonk.CosetInterpolationGate(4, config.max_quotient_degree_factor)
        E = lambda v: plonk.Ext2(Fp(v[0]), Fp(v[1]))
        shift = int(rnd(rng)) | 1
        values = [_ext(rng) for _ in range(gate.num_points())]
        point = _ext(rng)
        shift_inv = pow(shift, P - 2, P)
        shifted = [point[0] * shift_inv % P, point[1] * shift_inv % P]
        wires[0] = shift
        for i, v in enumerate(values):
            wires[gate.wires_value(i)], wires[gate.wires_value(i) + 1] = v
        at = gate.start_evaluation_point()
        wires[at], wires[at + 1] = point
        at = gate.wires_shifted_evaluation_point()
        wires[at], wires[at + 1] = shifted
        d = gate.degree()
        vals = [E(v) for v in values]
        acc = gate.partial_interpolate(0, d, vals, E(shifted), None)      # InterpolationGenerator::run_once
        for i in range(gate.num_intermediates()):
            for at, e in ((gate.wires_intermediate_eval(i), acc[0]), (gate.wires_intermediate_prod(i), acc[1])):
                wires[at], wires[at + 1] = int(e.a), int(e.b)
            start = 1 + (d - 1) * (i + 1)
            acc = gate.partial_interpolate(start, min(start + d - 1, gate.num_points()), vals, E(shifted), acc)
        at = gate.start_evaluation_value()
        wires[at], wires[at + 1] = int(acc[0].a), int(acc[0].b)
        return gate, [], wires, dict(shift=shift, values=values, point=point, value=[int(acc[0].a), int(acc[0].b)])
    raise KeyError(name)


def oracle_gate_kind(g):
    """(kind, param, param2) of tests/oracle_lib.plonk_quotient for a product gate object."""
    name = type(g).__name__
    return {"NoopGate": (OL.GATE_NOOP, 0, 0), "ConstantGate": (OL.GATE_CONSTANT, getattr(g, "num_consts", 0), 0),
            "PublicInputGate": (OL.GATE_PUBLIC_INPUT, 0, 0), "ArithmeticGate": (OL.GATE_ARITHMETIC, getattr(g, "num_ops", 0), 0),
            "PoseidonGate": (OL.GATE_POSEIDON, 0, 0),
            "ArithmeticExtensionGate": (OL.GATE_ARITHMETIC_EXTENSION, getattr(g, "num_ops", 0), 0),
            "MulExtensionGate": (OL.GATE_MUL_EXTENSION, getattr(g, "num_ops", 0), 0),
            "BaseSumGate": (OL.GATE_BASE_SUM, getattr(g, "num_limbs", 0), getattr(g, "base", 0)),
            "ReducingGate": (OL.GATE_REDUCING, getattr(g, "num_coeffs", 0), 0),
            "ReducingExtensionGate": (OL.GATE_REDUCING_EXTENSION, getattr(g, "num_coeffs", 0), 0),
            "PoseidonMdsGate": (OL.GATE_POSEIDON_MDS, 0, 0),
            "RandomAccessGate": (OL.GATE_RANDOM_ACCESS, getattr(g, "bits", 0), getattr(g, "num_copies", 0),
                                 getattr(g, "num_extra_constants", 0)),
            "ExponentiationGate": (OL.GATE_EXPONENTIATION, getattr(g, "num_power_bits", 0), 0),
            "CosetInterpolationGate": (OL.GATE_COSET_INTERPOLATION, getattr(g, "subgroup_bits", 0), getattr(g, "_degree", 0)),
            "LookupGate": (OL.GATE_NOOP, 0, 0), "LookupTableGate": (OL.GATE_NOOP, 0, 0),   # no constraints of their own
            }[name]


class FibonacciCircuit:
    """Row 0: PublicInputGate; row 1: ConstantGate(2) holding (F_0, 1); then ArithmeticGate rows whose operations compute
    out = m0 * m1 + addend with m0 = previous out, m1 = the constant 1, addend = the out before that (copy
    constraints); NoopGate rows pad to 2^degree_bits. Unconstrained wires carry random values."""

    def __init__(self, plonk, config, degree_bits, seed=1, arithmetic_rows=None, break_gate=False, break_copy=False,
                 poseidon_rows=0, break_poseidon=False, extra=(), break_extra=None, lookups=False, break_lookup=None,
                 public_inputs=None):
        rng = np.random.default_rng(seed)
        n = 1 << degree_bits
        self.config, self.n = config, n
        arith = plonk.ArithmeticGate.new_from_config(config)
        num_ops = arith.num_ops
        n_lookup_rows = 4 if lookups else 0      # two LookupGate rows, then two LookupTableGate rows
        arithmetic_rows = (arithmetic_rows if arithmetic_rows is not None
                           else n - 5 - poseidon_rows - len(extra) - n_lookup_rows)
        assert 2 + arithmetic_rows + poseidon_rows + len(extra) + n_lookup_rows < n
        extra_rows = [extra_gate_row(plonk, config, name, rng) for name in extra]
        self.extra_info = [r[3] if len(r) > 3 else None for r in extra_rows]
        extra_rows = [r[:3] for r in extra_rows]
        f0 = int(rnd(rng))
        instances = [(plonk.PublicInputGate(), []), (plonk.ConstantGate(2), [f0, 1])]
        instances += [(arith, [1, 1])] * arithmetic_rows
        instances += [(plonk.PoseidonGate(), [])] * poseidon_rows
        instances += [(g, consts) for g, consts, _ in extra_rows]
        luts, lookup_rows = [], []
        if lookups:
            # rows are "upside down" (circuit_builder.rs:75-87): LookupGate rows [last_lu, last_lut), table rows
            # [last_lut, first_lut], table entry e at row first_lut - e / slots, slot e % slots, padded with entry 0
            last_lu = len(instances)
            last_lut, first_lut = last_lu + 2, last_lu + 3
            instances += [(plonk.LookupGate.new_from_config(config), [])] * 2
            instances += [(plonk.LookupTableGate.new_from_config(config), [])] * 2
            luts = [[(3 * e + 1, (e * e + 7) & 0xFFFF) for e in range(30)]]
            lookup_rows = [(last_lu, last_lut, first_lut)]
        instances += [(plonk.NoopGate(), [])] * (n - len(instances))
        self.common, self.constant_vecs = plonk.CommonCircuitData.from_gate_instances(config, instances, luts, lookup_rows)
        self.lookup_rows = lookup_rows
        self.public_inputs = public_inputs
        if public_inputs is None:
            self.public_inputs_hash = [int(v) for v in rnd(rng, 4)]
        else:   # C::InnerHasher::hash_no_pad(&public_inputs), prover.rs:155
            self.public_inputs_hash = [int(v) for v in OL.hash_no_pad(np.array(public_inputs, dtype=np.uint64))]
        wires = rnd(rng, (config.num_wires, n))
        wires[0:4, 0] = self.public_inputs_hash
        wires[0, 1], wires[1, 1] = f0, 1
        # partition of the routed wires: sets of (row, column) that must carry one value
        sets = {"one": [(1, 1)], "f0": [(1, 0)]}
        prev, prevprev = ("f0", f0), ("one", 1)
        t = 0
        for r in range(2, 2 + arithmetic_rows):
            for k in range(num_ops):
                m0, m1, addend = prev[1], 1, prevprev[1]
                out = (m0 * m1 + addend) % P
                wires[4 * k, r], wires[4 * k + 1, r], wires[4 * k + 2, r], wires[4 * k + 3, r] = m0, m1, addend, out
                sets[prev[0]].append((r, 4 * k))
                sets["one"].append((r, 4 * k + 1))
                sets[prevprev[0]].append((r, 4 * k + 2))
                name = "out%d" % t
                sets[name] = [(r, 4 * k + 3)]
                prevprev, prev = prev, (name, out)
                t += 1
        # PoseidonGate rows: a hash chain -- the first four outputs of a row are copied into the first four inputs of the
        # next one (copy constraints on PoseidonGate wires), alternating the swap flag
        self.poseidon_io = []
        prev_out = None
        for q in range(poseidon_rows):
            r = 2 + arithmetic_rows + q
            inputs = [int(v) for v in rnd(rng, 12)]
            if prev_out is not None:
                inputs[:4] = prev_out[:4]
            pw = poseidon_gate_witness(plonk, inputs, q & 1)
            for k, v in pw.items():
                wires[k, r] = v
            if prev_out is not None:
                for i in range(4):
                    sets["p%d_%d" % (q, i)] = [(r - 1, plonk.PoseidonGate.wire_output(i)), (r, plonk.PoseidonGate.wire_input(i))]
            prev_out = [pw[plonk.PoseidonGate.wire_output(i)] for i in range(12)]
            self.poseidon_io.append((inputs, q & 1, prev_out))
        for q, (_, _, ew) in enumerate(extra_rows):      # rows of the other gate types, each with a satisfying witness
            r = 2 + arithmetic_rows + poseidon_rows + q
            for k, v in ew.items():
                wires[k, r] = v
            if break_extra == q:
                k = max(ew)
                wires[k, r] = (int(wires[k, r]) + 1) % P
        if lookups:
            lut = luts[0]
            lu_slots, lut_slots = config.num_routed_wires // 2, config.num_routed_wires // 3
            padded = lut + [lut[0]] * ((lut_slots - len(lut) % lut_slots) % lut_slots)
            counts = [0] * len(padded)
            for r in range(last_lu, last_lut):
                for s_ in range(lu_slots):
                    e = int(rnd(rng)) % len(lut) if (r + s_) % 5 else 0       # unused slots look up entry 0
                    counts[e] += 1
                    wires[2 * s_, r], wires[2 * s_ + 1, r] = lut[e]
            for e, (a, b_) in enumerate(padded):
                r, s_ = first_lut - e // lut_slots, e % lut_slots
                wires[3 * s_, r], wires[3 * s_ + 1, r], wires[3 * s_ + 2, r] = a, b_, counts[e]
            if break_lookup == "pair":       # a looking pair that is not in the table
                wires[1, last_lu] = (int(wires[1, last_lu]) + 1) % P
            if break_lookup == "table":      # a table row that differs from the committed table
                wires[4, last_lut] = (int(wires[4, last_lut]) + 1) % P
        if break_poseidon:  # one partial-round S-box input off by one
            r = 2 + arithmetic_rows
            k = plonk.PoseidonGate.wire_partial_sbox(7)
            wires[k, r] = (int(wires[k, r]) + 1) % P
        if break_gate:     # one arithmetic output off by one: the vanishing polynomial is no longer divisible by Z_H
            wires[3, 2] = (int(wires[3, 2]) + 1) % P
        if break_copy:     # a copy constraint violated while every gate still holds
            wires[1, 0] = (int(wires[1, 0]) + 1) % P
            sets["one"].append((0, 1))
        self.wires = wires
        # get_sigma_map: the next wire of the same set, wrapping around; a wire alone in its set maps to itself
        neighbor = {}
        for members in sets.values():
            for i, w in enumerate(members):
                neighbor[w] = members[(i + 1) % len(members)]
        k_is = self.common.k_is
        omega = root_of_unity(degree_bits)
        subgroup = [1]
        for _ in range(n - 1):
            subgroup.append(subgroup[-1] * omega % P)
        sig = np.empty((config.num_routed_wires, n), dtype=np.uint64)
        for col in range(config.num_routed_wires):
            for row in range(n):
                nr, ncol = neighbor.get((row, col), (row, col))
                sig[col, row] = k_is[ncol] * subgroup[nr] % P
        self.sigmas = sig
        self.constants_sigmas = np.concatenate([np.stack(self.constant_vecs), sig])

    def oracle_circuit(self):
        """The dict tests/oracle_lib.plonk_quotient takes, from the product's CommonCircuitData."""
        cd = self.common
        gates = []
        for i, g in enumerate(cd.gates):
            sel = cd.selectors_info.selector_indices[i]
            grp = cd.selectors_info.groups[sel]
            kind, param, param2, *rest = oracle_gate_kind(g)
            gates.append((kind, param, sel, grp.start, grp.stop, param2, rest[0] if rest else 0))
        cfg = cd.config
        return dict(num_wires=cfg.num_wires, num_routed_wires=cfg.num_routed_wires, num_constants=cd.num_constants,
                    num_challenges=cfg.num_challenges, quotient_degree_factor=cd.quotient_degree_factor,
                    num_selectors=cd.selectors_info.num_selectors(), num_partial_products=cd.num_partial_products,
                    num_gate_constraints=cd.num_gate_constraints, k_is=cd.k_is, gates=gates, luts=cd.luts,
                    num_lookup_selectors=cd.num_lookup_selectors, num_lookup_polys=cd.num_lookup_polys)

    def oracle_zs_partial_products(self, oracle, betas, gammas, deltas=()):
        """[plonk_z_vecs, partial_products.concat(), lookup polys] (plonk/prover.rs:227-245) from the oracle's restatements."""
        cfg = self.config
        zs, pps = [], []
        for beta, gamma in zip(betas, gammas):
            out = oracle.partial_products_and_zs(self.wires[:cfg.num_routed_wires], self.sigmas, self.common.k_is, beta, gamma,
                                                 self.common.quotient_degree_factor)
            zs.append(out[-1])
            pps += list(out[:-1])
        lk = []
        for c in range(len(betas) if self.common.luts else 0):   # compute_all_lookup_polys (prover.rs:579-607)
            lk += list(oracle.lookup_polys(self.wires, cfg.num_routed_wires, cfg.max_quotient_degree_factor,
                                           deltas[4 * c:4 * c + 4], self.lookup_rows))
        return np.stack(zs + pps + lk)


def zk_circuit(plonk, config, fri_config, seed=7, arithmetic_rows=12, poseidon_rows=0, extra=(), lookups=False,
               public_inputs=(3, 1, 4, 1, 5)):
    """A FibonacciCircuit with the blinding rows of CircuitBuilder::blind (plonk/circuit_builder.rs:911-970) that
    blinding_counts asks for -- regular_rows NoopGate rows with random values on every wire, then z_pairs pairs of
    NoopGate rows with one random value per routed wire in both rows of the pair and a copy constraint between them --
    padded with NoopGate rows to a power of two (CircuitBuilder::blind_and_pad). Returns (circuit, (regular_rows,
    z_pairs))."""
    num_gates = 2 + arithmetic_rows + poseidon_rows + len(extra) + (4 if lookups else 0)
    regular, z_pairs = plonk.blinding_counts(config, fri_config, num_gates)
    degree_bits = (num_gates + regular + 2 * z_pairs).bit_length()   # at least one padding row after the blinding
    c = FibonacciCircuit(plonk, config, degree_bits, seed=seed, arithmetic_rows=arithmetic_rows,
                         poseidon_rows=poseidon_rows, extra=extra, lookups=lookups, public_inputs=list(public_inputs))
    # FibonacciCircuit fills the NoopGate rows after the gates with random wires, each wire alone in its copy set: the
    # regular blinding rows as they are. Each Z pair gets one value per routed wire and the 2-cycle sigma of its set.
    omega = root_of_unity(degree_bits)
    k_is = c.common.k_is
    for q in range(z_pairs):
        r1 = num_gates + regular + 2 * q
        r2 = r1 + 1
        for w in range(config.num_routed_wires):
            assert int(c.sigmas[w, r1]) == k_is[w] * pow(omega, r1, P) % P   # not copied anywhere yet
            c.wires[w, r2] = c.wires[w, r1]
            c.sigmas[w, r1] = k_is[w] * pow(omega, r2, P) % P
            c.sigmas[w, r2] = k_is[w] * pow(omega, r1, P) % P
    c.constants_sigmas = np.concatenate([np.stack(c.constant_vecs), c.sigmas])
    return c, (regular, z_pairs)


def instances_of(c):
    """The gate instances [(gate, constants)] of a test circuit, read back from its selector and constant columns."""
    from plonky2_b200 import plonk

    cd = c.common
    info = cd.selectors_info
    nsel = info.num_selectors()
    consts = c.constant_vecs[nsel + cd.num_lookup_selectors:]
    out = []
    for row in range(c.n):
        vals = [int(c.constant_vecs[s][row]) for s in range(nsel)]
        i = vals[0] if nsel == 1 else next(v for v in vals if v != plonk.UNUSED_SELECTOR)
        g = cd.gates[i]
        out.append((g, [int(k[row]) for k in consts[:g.num_constants()]]))
    return out


def pairs_from_sigmas(c, skip_rows=()):
    """Copy constraints (Target::index) reproducing a test circuit's cycles: each wire paired with its sigma successor.
    Rows in skip_rows are left out."""
    cfg = c.config
    nw, nr, n = cfg.num_wires, cfg.num_routed_wires, c.n
    k_is = c.common.k_is
    subgroup = gn.powers(root_of_unity(c.common.degree_bits), n)
    where = {}
    for col in range(nr):
        for row, v in enumerate(gn.mul(np.full(n, k_is[col], dtype=np.uint64), subgroup).tolist()):
            where[v] = (row, col)
    skip = set(skip_rows)
    pairs = []
    for col in range(nr):
        for row in range(n):
            r, cc = where[int(c.sigmas[col, row])]
            if (r, cc) != (row, col) and row not in skip:
                pairs.append((row * nw + col, r * nw + cc))
    return np.array(pairs, dtype=np.int64).reshape(-1, 2)


# ---------------------------------------------------------------------------------------------------------------------
# The whole prover and verifier of plonky2 for these circuits, on the CPU, from the oracle's restatements:
# prove_with_partition_witness (plonk/prover.rs:132-360) and verify_with_challenges (plonk/verifier.rs:40-120).
class Fp2:
    """F_{p^2} = F_p[X]/(X^2 - 7) as numbers, with base-field scalars accepted on either side (ints)."""
    __slots__ = ("a", "b")

    def __init__(self, a, b=0):
        self.a, self.b = int(a) % P, int(b) % P

    @staticmethod
    def of(o):
        return o if isinstance(o, Fp2) else Fp2(int(o))

    def __add__(self, o):
        o = Fp2.of(o)
        return Fp2(self.a + o.a, self.b + o.b)

    def __sub__(self, o):
        o = Fp2.of(o)
        return Fp2(self.a - o.a, self.b - o.b)

    def __rsub__(self, o):
        return Fp2.of(o) - self

    def __mul__(self, o):
        o = Fp2.of(o)
        return Fp2(self.a * o.a + 7 * self.b * o.b, self.a * o.b + self.b * o.a)

    __radd__, __rmul__ = __add__, __mul__

    def inverse(self):
        d = pow((self.a * self.a - 7 * self.b * self.b) % P, P - 2, P)
        return Fp2(self.a * d, -self.b * d)

    def __eq__(self, o):
        o = Fp2.of(o)
        return self.a == o.a and self.b == o.b

    def __int__(self):
        assert self.b == 0
        return self.a

    def tup(self):
        return (self.a, self.b)


class ExtPointVars:
    """EvaluationVars over F_{p^2} numbers (plonk/vars.rs:14-20)."""

    def __init__(self, constants, wires, public_inputs_hash, prefix=0):
        self.c, self.w, self.pih, self.prefix = constants, wires, public_inputs_hash, prefix

    def local_constant(self, i):
        return self.c[self.prefix + i]

    def local_wire(self, i):
        return self.w[i]

    def public_inputs_hash(self, i):
        return Fp2(self.pih[i])

    def remove_prefix(self, n):
        return ExtPointVars(self.c, self.w, self.pih, self.prefix + n)


def openings_at(cd, cs_coeffs, wires_coeffs, zs_coeffs, zeta, zeta_next, ev, pool=None):
    """The openings vanishing_at reads (OpeningSet::new, plonk/proof.rs:313-351) from the coefficients of the
    constants / sigmas, wires and Z / partial-products (+ lookup) polynomials: ev(coeffs, point) -> (a, b) evaluates one
    polynomial at a point of F_{p^2}; `pool` (an Executor) runs the evaluations side by side."""
    nc, n_zs_pp = cd.config.num_challenges, cd.num_zs_partial_products_polys()
    jobs = [(p, zeta) for p in list(cs_coeffs) + list(wires_coeffs) + list(zs_coeffs)]
    jobs += [(p, zeta_next) for p in list(zs_coeffs[:nc]) + list(zs_coeffs[n_zs_pp:])]
    vals = [Fp2(*v) for v in (pool.map(lambda a: ev(*a), jobs) if pool else [ev(*a) for a in jobs])]
    ncs, nw, nz = len(cs_coeffs), len(wires_coeffs), len(zs_coeffs)
    cs, w, z, nxt = vals[:ncs], vals[ncs:ncs + nw], vals[ncs + nw:ncs + nw + nz], vals[ncs + nw + nz:]
    return dict(constants=cs[:cd.num_constants], plonk_sigmas=cs[cd.num_constants:], wires=w, plonk_zs=z[:nc],
                partial_products=z[nc:n_zs_pp], lookup_zs=z[n_zs_pp:], plonk_zs_next=nxt[:nc], lookup_zs_next=nxt[nc:])


def vanishing_at(plonk, cd, x, o, public_inputs_hash, betas, gammas, alphas, deltas=()):
    """eval_vanishing_poly (vanishing_poly.rs:57-164) at one point x, an Fp2 (a base-field point has b = 0), from the
    polynomials' values there: `o` maps constants, plonk_sigmas, wires, plonk_zs, partial_products, lookup_zs (at x) and
    plonk_zs_next, lookup_zs_next (at g x) to lists of Fp2. Gates: ConstantGate, PublicInputGate and ArithmeticGate are
    restated here; the others run the product's value-generic gate code over F_{p^2} numbers (the oracle restates every
    gate independently in C++). The cost does not depend on n. Returns ([vanishing(x) per challenge], Z_H(x), x^n)."""
    cfg = cd.config
    nc, n = cfg.num_challenges, 1 << cd.degree_bits
    constants, sigmas, wires = o["constants"], o["plonk_sigmas"], o["wires"]
    zs, zs_next, pps = o["plonk_zs"], o["plonk_zs_next"], o["partial_products"]
    lk, lk_next = o["lookup_zs"], o["lookup_zs_next"]
    nsel = cd.selectors_info.num_selectors()
    local = constants[nsel + cd.num_lookup_selectors:]
    vars_ = ExtPointVars(constants, wires, public_inputs_hash)
    constraint_terms = [Fp2(0)] * cd.num_gate_constraints                     # evaluate_gate_constraints
    for i, gate in enumerate(cd.gates):
        sel = cd.selectors_info.selector_indices[i]
        s = constants[sel]
        filt = Fp2(1)
        for j in list(cd.selectors_info.groups[sel]) + ([plonk.UNUSED_SELECTOR] if nsel > 1 else []):
            if j != i:
                filt = filt * (j - s)
        kind, param = oracle_gate_kind(gate)[:2]
        if kind == OL.GATE_CONSTANT:
            res = [local[t] - wires[t] for t in range(param)]
        elif kind == OL.GATE_PUBLIC_INPUT:
            res = [wires[t] - public_inputs_hash[t] for t in range(4)]
        elif kind == OL.GATE_ARITHMETIC:
            res = [wires[4 * t + 3] - (wires[4 * t] * wires[4 * t + 1] * local[0] + wires[4 * t + 2] * local[1])
                   for t in range(param)]
        else:
            res = gate.eval_unfiltered(vars_.remove_prefix(nsel + cd.num_lookup_selectors))
        for t, r in enumerate(res):
            constraint_terms[t] = constraint_terms[t] + Fp2.of(r) * filt
    xn = x
    for _ in range(cd.degree_bits):
        xn = xn * xn
    z_h = xn - 1
    l_0_x = z_h * ((x - 1) * n).inverse()                                      # eval_l_0, plonk_common.rs:69-79
    nr, qdf, nprod = cfg.num_routed_wires, cd.quotient_degree_factor, cd.num_partial_products
    z1, pp_terms, lookup_terms = [], [], []

    def product(vs):
        acc = Fp2(1)
        for v in vs:
            acc = acc * v
        return acc

    for i in range(nc):
        z1.append(l_0_x * (zs[i] - 1))
        if cd.luts:
            npoly = cd.num_lookup_polys
            d = deltas[4 * i:4 * i + 4]
            lookup_terms += [Fp2.of(v) for v in plonk.check_lookup_constraints(
                cd, vars_, lk[npoly * i:npoly * (i + 1)], lk_next[npoly * i:npoly * (i + 1)],
                constants[nsel:nsel + cd.num_lookup_selectors], d, cd.lut_re_poly_evals(d), product)]
        num = [wires[j] + x * (betas[i] * cd.k_is[j] % P) + gammas[i] for j in range(nr)]
        den = [wires[j] + sigmas[j] * betas[i] + gammas[i] for j in range(nr)]
        accs = [zs[i]] + pps[i * nprod:(i + 1) * nprod] + [zs_next[i]]
        for k in range(nprod + 1):
            pp_terms.append(accs[k] * product(num[k * qdf:(k + 1) * qdf]) - accs[k + 1] * product(den[k * qdf:(k + 1) * qdf]))
    terms = z1 + pp_terms + lookup_terms + constraint_terms
    vanishing = []
    for i in range(nc):
        acc = Fp2(0)
        for t in reversed(terms):                                              # reduce_with_powers_multi
            acc = acc * alphas[i] + t
        vanishing.append(acc)
    return vanishing, z_h, xn


def fri_batches(cd, zeta):
    """get_fri_instance (plonk/circuit_data.rs:530-660) as the oracle's (point, [(oracle, polynomial)]) lists."""
    import plonky2_b200.field as F

    cfg = cd.config
    nc = cfg.num_challenges
    n_pre, n_zs_pp = cd.num_constants + cfg.num_routed_wires, cd.num_zs_partial_products_polys()
    n_lookup, n_quot = nc * cd.num_lookup_polys, nc * cd.quotient_degree_factor
    lookup = [(2, i) for i in range(n_zs_pp, n_zs_pp + n_lookup)]
    all_polys = ([(0, i) for i in range(n_pre)] + [(1, i) for i in range(cfg.num_wires)] + [(2, i) for i in range(n_zs_pp)]
                 + [(3, i) for i in range(n_quot)] + lookup)
    g = F.primitive_root_of_unity(cd.degree_bits)
    zeta_next = F.ext_mul((g, 0), zeta)
    return [(zeta, all_polys), (zeta_next, [(2, i) for i in range(nc)] + lookup)], [n_pre, cfg.num_wires, n_zs_pp + n_lookup, n_quot]


def observe_fri_params(ch, fri_cfg, degree_bits, arity_bits, hiding):
    """FriParams::observe (fri/mod.rs:73-79,145-157) for a ConstantArityBits strategy."""
    ch.observe_elements([fri_cfg.rate_bits, fri_cfg.cap_height, fri_cfg.proof_of_work_bits])
    ch.observe_elements([1, fri_cfg.reduction_strategy[1], fri_cfg.reduction_strategy[2]])
    ch.observe_element(fri_cfg.num_query_rounds)
    ch.observe_elements([int(hiding), degree_bits] + list(arity_bits))


def salt_widths(widths):
    """Leaf widths of the four plonky2 oracles with hiding: constants / sigmas unsalted, the others + SALT_SIZE."""
    return [w + (4 if k else 0) for k, w in enumerate(widths)]


def oracle_prove(oracle, c, circuit_digest, fri_cfg, public_inputs, taps=False, *, salts=None):
    """prove_with_partition_witness with the oracle's pieces. Returns (proof bytes = write_proof_with_public_inputs,
    parts) where parts carries what the verifier reads from the proof. With c.config.zero_knowledge (FriParams.hiding)
    salts are the (4 x N) salt arrays of the wires, Z and quotient commitments; the constants / sigmas commitment is
    never salted. Without zero knowledge there are no salts."""
    cd, cfg = c.common, c.config
    nc, nr, n = cfg.num_challenges, cfg.num_routed_wires, c.n
    hiding = cfg.zero_knowledge
    if (salts is not None) != hiding:
        raise ValueError("salts are required with zero knowledge and refused without")
    salt_wires, salt_zs, salt_quotient = salts if hiding else (None, None, None)
    arity_bits = fri_cfg.fri_params(cd.degree_bits, hiding).reduction_arity_bits
    public_inputs_hash = [int(x) for x in oracle.hash_no_pad(np.array(public_inputs, dtype=np.uint64))]
    assert public_inputs_hash == c.public_inputs_hash
    cs = oracle.Commit(c.constants_sigmas, cfg.rate_bits, cfg.cap_height)
    wc = oracle.Commit(c.wires, cfg.rate_bits, cfg.cap_height, salt=salt_wires)
    ch = oracle.Challenger()
    observe_fri_params(ch, fri_cfg, cd.degree_bits, arity_bits, hiding)
    ch.observe_elements(circuit_digest)
    ch.observe_elements(public_inputs_hash)
    ch.observe_cap(wc.cap)
    betas, gammas = ch.get_n_challenges(nc), ch.get_n_challenges(nc)
    deltas = (betas + gammas + ch.get_n_challenges(2 * nc)) if cd.luts else []
    zc = oracle.Commit(c.oracle_zs_partial_products(oracle, betas, gammas, deltas), cfg.rate_bits, cfg.cap_height,
                       salt=salt_zs)
    ch.observe_cap(zc.cap)
    alphas = ch.get_n_challenges(nc)
    q = oracle.plonk_quotient(c.oracle_circuit(), cs, wc, zc, public_inputs_hash, betas, gammas, alphas, deltas)
    qdf = cd.quotient_degree_factor
    assert not q[:, qdf * n:].any(), "Quotient has failed, the vanishing polynomial is not divisible by Z_H"
    chunks = np.concatenate([q[i, :qdf * n].reshape(qdf, n) for i in range(nc)])
    qc = oracle.Commit(chunks, cfg.rate_bits, cfg.cap_height, salt=salt_quotient, is_coeffs=True)
    ch.observe_cap(qc.cap)
    zeta = ch.get_extension_challenge()
    batches, num_polys = fri_batches(cd, zeta)
    commits = [cs, wc, zc, qc]

    def ev(commit, z):
        return np.array([oracle.eval_poly_base_at_ext(p, z) for p in commit.coeffs], dtype=np.uint64).reshape(-1, 2)

    zeta_next = batches[1][0]
    cs_e, w_e, z_e, z_next, q_e = ev(cs, zeta), ev(wc, zeta), ev(zc, zeta), ev(zc, zeta_next), ev(qc, zeta)
    n_zs_pp = cd.num_zs_partial_products_polys()
    o = dict(constants=cs_e[:cd.num_constants], plonk_sigmas=cs_e[cd.num_constants:], wires=w_e, plonk_zs=z_e[:nc],
             plonk_zs_next=z_next[:nc], partial_products=z_e[nc:n_zs_pp], quotient_polys=q_e, lookup_zs=z_e[n_zs_pp:],
             lookup_zs_next=z_next[n_zs_pp:])
    zeta_batch = np.concatenate([o["constants"], o["plonk_sigmas"], o["wires"], o["plonk_zs"], o["partial_products"],
                                 o["quotient_polys"], o["lookup_zs"]])
    next_batch = np.concatenate([o["plonk_zs_next"], o["lookup_zs_next"]])
    ch.observe_elements(zeta_batch.reshape(-1))
    ch.observe_elements(next_batch.reshape(-1))
    params = oracle.make_params(cfg.rate_bits, cfg.cap_height, fri_cfg.proof_of_work_bits, fri_cfg.num_query_rounds, arity_bits)
    fri_taps = None
    if taps:
        fri_bytes, fri_taps = oracle.prove_openings(commits, batches, ch, params, taps=True)
    else:
        fri_bytes = oracle.prove_openings(commits, batches, ch, params)

    def le(a):
        return np.ascontiguousarray(a, dtype="<u8").tobytes()

    out = le(wc.cap) + le(zc.cap) + le(qc.cap)
    for k in ("constants", "plonk_sigmas", "wires", "plonk_zs", "plonk_zs_next", "lookup_zs", "lookup_zs_next",
              "partial_products", "quotient_polys"):
        out += le(o[k])
    out += fri_bytes + le(np.array([len(public_inputs)], dtype=np.uint64)) + le(np.array(public_inputs, dtype=np.uint64))
    parts = dict(constants_sigmas_cap=cs.cap, wires_cap=wc.cap, zs_cap=zc.cap, quotient_cap=qc.cap, openings=o,
                 fri_bytes=fri_bytes, public_inputs=list(public_inputs), taps=fri_taps)
    return out, parts


def oracle_verify(oracle, plonk, c, circuit_digest, fri_cfg, parts):
    """verify (plonk/verifier.rs:20-120): get_challenges (plonk/get_challenges.rs:26-90) replayed on a fresh transcript,
    eval_vanishing_poly at zeta in F_{p^2} (vanishing_at), the quotient identity, then verify_fri_proof (the oracle's).
    With c.config.zero_knowledge (FriParams.hiding) the salted oracles' leaves are SALT_SIZE wider, and the FRI check
    strips the salt (fri/verifier.rs fri_combine_initial). Returns None or the reason of the rejection."""
    cd, cfg = c.common, c.config
    nc = cfg.num_challenges
    o = parts["openings"]
    hiding = cfg.zero_knowledge
    arity_bits = fri_cfg.fri_params(cd.degree_bits, hiding).reduction_arity_bits
    public_inputs_hash = [int(x) for x in oracle.hash_no_pad(np.array(parts["public_inputs"], dtype=np.uint64))]
    ch = oracle.Challenger()
    observe_fri_params(ch, fri_cfg, cd.degree_bits, arity_bits, hiding)
    ch.observe_elements(circuit_digest)
    ch.observe_elements(public_inputs_hash)
    ch.observe_cap(parts["wires_cap"])
    betas, gammas = ch.get_n_challenges(nc), ch.get_n_challenges(nc)
    deltas = (betas + gammas + ch.get_n_challenges(2 * nc)) if cd.luts else []
    ch.observe_cap(parts["zs_cap"])
    alphas = ch.get_n_challenges(nc)
    ch.observe_cap(parts["quotient_cap"])
    zeta = ch.get_extension_challenge()
    zeta_batch = np.concatenate([o["constants"], o["plonk_sigmas"], o["wires"], o["plonk_zs"], o["partial_products"],
                                 o["quotient_polys"], o["lookup_zs"]])
    next_batch = np.concatenate([o["plonk_zs_next"], o["lookup_zs_next"]])
    ch.observe_elements(zeta_batch.reshape(-1))
    ch.observe_elements(next_batch.reshape(-1))

    def E(arr):
        return [Fp2(int(v[0]), int(v[1])) for v in arr]

    qdf = cd.quotient_degree_factor
    ev = {k: E(v) for k, v in o.items()}
    vanishing, z_h_zeta, xn = vanishing_at(plonk, cd, Fp2(*zeta), ev, public_inputs_hash, betas, gammas, alphas, deltas)
    quot = ev["quotient_polys"]
    for i in range(nc):
        chunk = Fp2(0)
        for t in reversed(quot[i * qdf:(i + 1) * qdf]):                        # reduce_with_powers(chunk, zeta^n)
            chunk = chunk * xn + t
        if not vanishing[i] == z_h_zeta * chunk:
            return "vanishing polynomial identity fails for challenge %d" % i
    batches, num_polys = fri_batches(cd, zeta)
    params = oracle.make_params(cfg.rate_bits, cfg.cap_height, fri_cfg.proof_of_work_bits, fri_cfg.num_query_rounds, arity_bits)
    rc = oracle.verify_fri_proof([parts["constants_sigmas_cap"], parts["wires_cap"], parts["zs_cap"], parts["quotient_cap"]],
                                 num_polys, salt_widths(num_polys) if hiding else num_polys, batches,
                                 np.concatenate([zeta_batch.reshape(-1), next_batch.reshape(-1)]),
                                 cd.degree_bits, ch, params, parts["fri_bytes"])
    return None if rc == 0 else "FRI proof rejected (rc=%d)" % rc


OPENING_KEYS = ("constants", "plonk_sigmas", "wires", "plonk_zs", "plonk_zs_next", "partial_products", "quotient_polys",
                "lookup_zs", "lookup_zs_next")


def parts_of(proof, constants_sigmas_cap):
    """What oracle_verify reads, from a ProofWithPublicInputs and the circuit's constants / sigmas cap."""
    p, o = proof.proof, proof.proof.openings
    return dict(constants_sigmas_cap=constants_sigmas_cap, wires_cap=p.wires_cap.hashes,
                zs_cap=p.plonk_zs_partial_products_cap.hashes, quotient_cap=p.quotient_polys_cap.hashes,
                openings={k: getattr(o, k) for k in OPENING_KEYS}, fri_bytes=p.opening_proof.to_bytes(),
                public_inputs=list(proof.public_inputs))


def cpu_backends(monkeypatch, oracle, c, fri_cfg, salt_keys=None):
    """Stand the oracle's pieces in for plonk.prove_with_witness's device calls on circuit c: commitments, Z / partial
    products, lookup columns, quotient, evaluations, the public-input hash and prove_openings, which replays the
    product's transcript into the oracle's Challenger. With salt_keys every salted commitment takes
    chacha_ref.salt_array(key, N) of its key. Returns (the context stand-in, the transcript logs, the salt keys used in
    order). The patched plonk.PolynomialBatch.from_values makes the constants / sigmas commitment."""
    import chacha_ref as R

    import plonky2_b200.fri as fri_mod
    import plonky2_b200.hash as hash_mod
    import plonky2_b200.proof as proof_mod
    import plonky2_b200.prover as prover_mod
    from plonky2_b200 import plonk

    cfg, cd = c.config, c.common
    N = c.n << cfg.rate_bits
    used = []

    def salt(blinding, salt_key):
        if not blinding:
            assert salt_key is None
            return None
        assert salt_keys is not None and salt_key in salt_keys
        used.append(salt_key)
        return R.salt_array(salt_key, N)

    class Cap:
        def __init__(self, hashes):
            self.hashes = hashes

    class Tree:
        def __init__(self, commit):
            self.cap = Cap(commit.cap)

    class Batch:   # a PolynomialBatch whose device work is done by the oracle
        def __init__(self, commit):
            self.o, self.merkle_tree, self.num_polys, self.degree_log = commit, Tree(commit), commit.B, commit.log_n
            self.ctx = ctx

        @classmethod
        def from_values(cls, values, rate_bits, blinding, cap_height, ctx=None, salt_key=None):
            return cls(oracle.Commit(values, rate_bits, cap_height, salt=salt(blinding, salt_key)))

        def close(self):
            pass

    class Ctx:
        device, h = 0, None

    ctx = Ctx()

    def commit_zs(wires_dev, sigmas_dev, k_is, betas, gammas, degree, rate_bits, cap_height, ctx=None, blinding=False,
                  salt_key=None):
        assert np.array_equal(wires_dev, c.wires[:cfg.num_routed_wires]) and np.array_equal(sigmas_dev, c.sigmas)
        return Batch(oracle.Commit(c.oracle_zs_partial_products(oracle, betas, gammas), rate_bits, cap_height,
                                   salt=salt(blinding, salt_key)))

    def quotient(cd_, cs, pih, w, z, betas, gammas, alphas, deltas=()):
        return oracle.plonk_quotient(c.oracle_circuit(), cs.o, w.o, z.o, pih, betas, gammas, alphas, deltas)

    def commit_quotient(cd_, q, ctx=None, blinding=False, salt_key=None):
        qdf, n = cd.quotient_degree_factor, c.n
        chunks = np.concatenate([q[i, :qdf * n].reshape(qdf, n) for i in range(q.shape[0])])
        return Batch(oracle.Commit(chunks, cfg.rate_bits, cfg.cap_height, salt=salt(blinding, salt_key),
                                   is_coeffs=True))

    def evals(requests):
        return [np.array([oracle.eval_poly_base_at_ext(p, z) for p in b.o.coeffs], dtype=np.uint64).reshape(-1, 2)
                for b, z in requests]

    class FriBytes:
        def __init__(self, b):
            self.b = b

        def to_bytes(self):
            return self.b

    def prove_openings(instance, oracles, challenger, fri_params):
        assert [o.blinding for o in instance.oracles] == [False] + [salt_keys is not None] * 3
        assert [o.num_polys for o in instance.oracles] == [b.num_polys for b in oracles]
        batches = [(b.point, [(p.oracle_index, p.polynomial_index) for p in b.polynomials]) for b in instance.batches]
        params = oracle.make_params(cfg.rate_bits, cfg.cap_height, fri_cfg.proof_of_work_bits, fri_cfg.num_query_rounds,
                                    fri_params.reduction_arity_bits)
        return FriBytes(oracle.prove_openings([b.o for b in oracles], batches, oracle.replay(challenger.log), params))

    logs = oracle.log_transcripts(monkeypatch)
    monkeypatch.setattr(plonk, "PolynomialBatch", Batch)
    monkeypatch.setattr(plonk, "_to_device", lambda columns, ctx: np.ascontiguousarray(columns, dtype=np.uint64))
    monkeypatch.setattr(plonk, "compute_quotient_polys", quotient)
    monkeypatch.setattr(plonk, "commit_quotient_polys", commit_quotient)
    monkeypatch.setattr(prover_mod, "commit_zs_partial_products", commit_zs)
    monkeypatch.setattr(prover_mod, "wires_permutation_partial_products_and_zs",
                        lambda w, s, k, beta, gamma, degree, ctx=None: oracle.partial_products_and_zs(w, s, k, beta, gamma, degree))
    monkeypatch.setattr(prover_mod, "compute_all_lookup_polys",
                        lambda w, nr, qdf, deltas, rows, nc, ctx=None: np.concatenate(
                            [oracle.lookup_polys(w, nr, qdf, deltas[4 * k:4 * k + 4], rows) for k in range(nc)]))
    monkeypatch.setattr(proof_mod, "eval_commitments", evals)
    monkeypatch.setattr(fri_mod, "prove_openings", prove_openings)
    monkeypatch.setattr(hash_mod.PoseidonHash, "hash_no_pad", staticmethod(lambda x, ctx=None: oracle.hash_no_pad(x)))
    return ctx, logs, used
