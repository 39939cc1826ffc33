"""plonky2's quotient polynomials on the device (SURVEY.md section 8f row 1): compute_quotient_polys
(plonky2/src/plonk/prover.rs:609-815) over eval_vanishing_poly_base_batch (plonky2/src/plonk/vanishing_poly.rs:167-340),
the gates' constraint evaluators (plonky2/src/gates/*.rs), and the prover that strings the device pieces together
(prove_with_witness = prove_with_partition_witness, plonk/prover.rs:132-360; Proof / CompressedProof and their byte formats).

The reference evaluates, for every point of the quotient coset, each gate's constraints times its selector filter, the
terms L_0(x)(Z(x) - 1) and the partial-product checks of the permutation argument, and combines them with powers of
alpha. Here that walk is done ONCE per circuit, symbolically: gates implement eval_unfiltered over expression handles,
`vanishing_program` records the whole vanishing polynomial as a register program, and gl_plonk_quotient interprets it
for all points on the GPU, reading the three commitments' LDEs in place. Placing a circuit (CircuitBuilder's gates,
targets and generators, witness generation) stays with the caller; from the placed circuit, `blind_and_pad` and
`build_circuit_data` restate the rest of `CircuitBuilder::build` (gate order, selector polynomials, constant columns,
k_is, counts, the sigma polynomials on the device, the constants/sigmas commitment, the circuit digest).
Lookup circuits carry the extra terms of `check_lookup_constraints` (the RE / Sum / LDC checks over the lookup selectors)."""
import ctypes as C
import heapq
import os
import re

import numpy as np

from . import _native as N
from . import distributed
from . import field as F
from .polynomial_batch import SALT_SIZE, PolynomialBatch

OP_LOCAL, OP_NEXT, OP_CONST, OP_X, OP_L0, OP_ADD, OP_SUB, OP_MUL, OP_TERM, OP_ADDC, OP_MULC = range(11)
_BINARY, _UNARY_CONST = (OP_ADD, OP_SUB, OP_MUL), (OP_ADDC, OP_MULC)
MAX_REGS = 256
UNUSED_SELECTOR = 0xFFFFFFFF   # gates/selectors.rs:14
# LookupSelectors (gates/selectors.rs:33-40), LookupChallenges and NUM_COINS_LOOKUP (plonk/circuit_builder.rs:60-73)
LOOKUP_TRANS_SRE, LOOKUP_TRANS_LDC, LOOKUP_INIT_SRE, LOOKUP_LAST_LDC, LOOKUP_START_END = range(5)
LOOKUP_CHALLENGE_A, LOOKUP_CHALLENGE_B, LOOKUP_CHALLENGE_ALPHA, LOOKUP_CHALLENGE_DELTA = range(4)
NUM_COINS_LOOKUP = 4
# commitment indices of the program's loads
CONSTANTS_SIGMAS, WIRES, ZS_PARTIAL_PRODUCTS = 0, 1, 2


class VpInstr(C.Structure):
    _fields_ = [("op", C.c_uint16), ("dst", C.c_uint16), ("a", C.c_uint16), ("b", C.c_uint16)]


class CircuitConfig:
    """CircuitConfig (plonk/circuit_data.rs:60-131); defaults = standard_recursion_config."""

    def __init__(self, num_wires=135, num_routed_wires=80, num_constants=2, num_challenges=2,
                 max_quotient_degree_factor=8, rate_bits=3, cap_height=4, *, zero_knowledge=False):
        self.num_wires, self.num_routed_wires, self.num_constants = num_wires, num_routed_wires, num_constants
        self.num_challenges, self.max_quotient_degree_factor = num_challenges, max_quotient_degree_factor
        self.rate_bits, self.cap_height = rate_bits, cap_height
        self.zero_knowledge = bool(zero_knowledge)


def standard_recursion_zk_config():
    """CircuitConfig::standard_recursion_zk_config (plonk/circuit_data.rs:135-140)."""
    return CircuitConfig(zero_knowledge=True)


def blinding_counts(config, fri_config, num_gates):
    """CircuitBuilder::blinding_counts with num_blinding_gates (plonk/circuit_builder.rs:866-909): (regular_poly_openings,
    z_openings), the number of values a proof reveals per "regular" polynomial (opened at zeta and in the FRI queries) and
    per Z polynomial (also at g zeta), for a circuit of num_gates gates before blinding, under the FRI config fri_config.
    A zero-knowledge circuit (CircuitBuilder::blind, :911-970) then gets regular_poly_openings NoopGate rows with random
    values on every wire, and z_openings pairs of NoopGate rows with the same random value on each routed wire of the
    pair and a copy constraint between them; filling them is witness generation (RandomValueGenerator)."""
    degree_estimate = 1 << max(0, int(num_gates) - 1).bit_length()
    while True:
        arities = [1 << b for b in fri_config.fri_params(F.log2_strict(degree_estimate),
                                                         config.zero_knowledge).reduction_arity_bits]
        product = 1
        for a in arities:
            product *= a
        fri_openings = fri_config.num_query_rounds * (1 + F.D * sum(a - 1 for a in arities)
                                                      + F.D * (degree_estimate // product))
        regular_poly_openings, z_openings = F.D + fri_openings, 2 * F.D + fri_openings
        if num_gates + regular_poly_openings + 2 * z_openings <= degree_estimate:
            return regular_poly_openings, z_openings
        degree_estimate *= 2


# ------------------------------------------------------------------ expressions
class Expr:
    """A base-field value of the vanishing program (the F / P of eval_unfiltered_base_*)."""
    __slots__ = ("b", "idx")

    def __init__(self, b, idx):
        self.b, self.idx = b, idx

    def _bin(self, op, other, swap=False):
        if isinstance(other, ConstRef):      # a bound or program constant: the immediate forms r + c, r * c
            if op in (OP_MUL, OP_ADD):
                return self.b._push(OP_MULC if op == OP_MUL else OP_ADDC, self.idx, other.k)
            other = other.value()
        elif not isinstance(other, Expr):    # a known field constant
            c = int(other) % F.ORDER
            if op == OP_MUL:
                return self.b._push(OP_MULC, self.idx, self.b.const_index(c))
            if op == OP_ADD:
                return self.b._push(OP_ADDC, self.idx, self.b.const_index(c))
            if not swap:                     # r - c
                return self.b._push(OP_ADDC, self.idx, self.b.const_index(-c))
            neg = self.b._push(OP_MULC, self.idx, self.b.const_index(-1))     # c - r
            return self.b._push(OP_ADDC, neg.idx, self.b.const_index(c))
        x, y = (other, self) if swap else (self, other)
        return self.b._push(op, x.idx, y.idx)

    def __add__(self, o):
        return self._bin(OP_ADD, o)

    def __sub__(self, o):
        return self._bin(OP_SUB, o)

    def __rsub__(self, o):
        return self._bin(OP_SUB, o, swap=True)

    def __mul__(self, o):
        return self._bin(OP_MUL, o)

    __radd__, __rmul__ = __add__, __mul__


class ConstRef:
    """Entry k of the program's constant table (a challenge, a public-input word, a literal): an operand of the
    immediate forms; becomes a register value only when it has to."""
    __slots__ = ("b", "k")

    def __init__(self, b, k):
        self.b, self.k = b, k

    def value(self):
        return self.b._push(OP_CONST, self.k)

    def __add__(self, o):
        return o + self if isinstance(o, Expr) else self.value() + o

    def __mul__(self, o):
        return o * self if isinstance(o, Expr) else self.value() * o

    def __sub__(self, o):
        return self.value() - o

    def __rsub__(self, o):
        return o - self.value()

    __radd__, __rmul__ = __add__, __mul__


class VanishingBuilder:
    """Records values in SSA form (common subexpressions shared), then compiles them to the register program of
    include/plonky2_b200.h (dead values dropped, registers reused after a value's last use)."""

    def __init__(self, num_bound):
        self.instrs = []
        self.consts = [None] * num_bound     # consts[0:num_bound] are bound at evaluation time
        self.num_bound = num_bound
        self._const_index = {}
        self._cache = {}
        self.terms = {}                      # term number -> value index
        self.term_order = None               # evaluation order of the terms (default: by number)
        self.scope = None

    def _push(self, op, a=0, b=0):
        if op in (OP_ADD, OP_MUL) and a > b:
            a, b = b, a                      # commutative: one cache entry
        # arithmetic is shared within one scope (a gate, the permutation argument) only: an accidental match between
        # two gates would keep a value alive from one gate's use to the other's
        key = (op, a, b, self.scope if (op in _BINARY or op in _UNARY_CONST) else None)
        e = self._cache.get(key)
        if e is None:
            self.instrs.append((op, a, b))
            e = self._cache[key] = Expr(self, len(self.instrs) - 1)
        return e

    def local(self, commitment, column):
        return self._push(OP_LOCAL, commitment, column)

    def next(self, commitment, column):
        return self._push(OP_NEXT, commitment, column)

    def bound(self, k):
        assert 0 <= k < self.num_bound
        return ConstRef(self, k)

    def const_index(self, v):
        v = int(v) % F.ORDER
        k = self._const_index.get(v)
        if k is None:
            k = self._const_index[v] = len(self.consts)
            self.consts.append(v)
            assert k < 65536
        return k

    def constant(self, v):
        return ConstRef(self, self.const_index(v))

    def x(self):
        return self._push(OP_X)

    def l0(self):
        return self._push(OP_L0)

    def term(self, number, e):
        assert number not in self.terms
        self.terms[number] = (e.value() if isinstance(e, ConstRef) else e).idx

    def product(self, es):
        """Iterator::product over field values (empty product = ONE)."""
        acc = None
        for e in es:
            acc = e if acc is None else acc * e
        return acc if acc is not None else self.constant(1).value()

    def compile(self):
        """-> (VpInstr array, n_regs). Scheduling: the terms are taken in `term_order` and every value is emitted when a
        term first needs it (depth first), so a product chain never has more than its running product and one factor
        alive. Loads and constants are re-issued per term instead of being kept across terms (a register lives in
        thread-local memory: keeping one costs what a coalesced load costs, and a small register set stays in L1);
        arithmetic values, x and L_0(x) are shared. Registers are then assigned by a linear scan."""
        ins = self.instrs
        order = self.term_order if self.term_order is not None else sorted(self.terms)
        assert sorted(order) == sorted(self.terms)
        REMAT = (OP_LOCAL, OP_NEXT, OP_CONST)
        seq = []                 # (op, a, b): operands are positions in seq for ADD/SUB/MUL/TERM
        shared = {}              # SSA value -> position in seq
        height = [0] * len(ins)  # the deeper operand of an instruction is evaluated first (Sethi-Ullman): a leaf
        for k, (op, a, b) in enumerate(ins):     # loaded before descending into a long chain would wait in a register
            if op in _BINARY:
                height[k] = 1 + max(height[a], height[b])
            elif op in _UNARY_CONST:
                height[k] = 1 + height[a]

        def emit(root, local):
            def pos(v):
                return local[v] if ins[v][0] in REMAT else shared[v]
            stack = [(root, 0)]
            while stack:
                v, state = stack.pop()
                op, a, b = ins[v]
                if op in REMAT:
                    if v not in local:
                        local[v] = len(seq)
                        seq.append((op, a, b))
                elif v in shared:
                    continue
                elif op in (OP_X, OP_L0):
                    shared[v] = len(seq)
                    seq.append((op, 0, 0))
                elif state == 0:
                    if op in _BINARY:
                        first, second = (a, b) if height[a] >= height[b] else (b, a)
                        stack += [(v, 1), (second, 0), (first, 0)]
                    else:
                        stack += [(v, 1), (a, 0)]
                else:
                    shared[v] = len(seq)
                    seq.append((op, pos(a), pos(b) if op in _BINARY else b))
            return pos(root)

        for number in order:
            r = emit(self.terms[number], {})
            seq.append((OP_TERM, r, number))
        last_use = {}
        for k, (op, a, b) in enumerate(seq):
            if op in _BINARY:
                last_use[a] = last_use[b] = k
            elif op == OP_TERM or op in _UNARY_CONST:
                last_use[a] = k
        out, reg_of, free, n_regs = [], {}, [], 0
        for k, (op, a, b) in enumerate(seq):
            if op == OP_TERM:
                out.append((OP_TERM, 0, reg_of[a], b))
                if last_use[a] == k:
                    heapq.heappush(free, reg_of[a])
                continue
            ra = rb = 0
            if op in _BINARY or op in _UNARY_CONST:
                ra, rb = reg_of[a], (reg_of[b] if op in _BINARY else b)
                for v in ({a, b} if op in _BINARY else {a}):
                    if last_use[v] == k:
                        heapq.heappush(free, reg_of[v])   # dst may reuse it: an instruction reads before it writes
            if free:
                dst = heapq.heappop(free)
            else:
                dst, n_regs = n_regs, n_regs + 1
            reg_of[k] = dst
            if op in _BINARY or op in _UNARY_CONST:
                out.append((op, dst, ra, rb))
            elif op == OP_CONST:
                out.append((op, dst, a & 0xFFFF, a >> 16))
            else:
                out.append((op, dst, a, b))
            assert k in last_use
        if n_regs > MAX_REGS:
            raise N.NativeError("vanishing program needs %d registers (max %d)" % (n_regs, MAX_REGS))
        arr = (VpInstr * len(out))()
        for i, (op, dst, a, b) in enumerate(out):
            arr[i].op, arr[i].dst, arr[i].a, arr[i].b = op, dst, a, b
        return arr, n_regs


# ------------------------------------------------------------------ gates
class EvaluationVarsBase:
    """EvaluationVarsBase (plonk/vars.rs:22-27,94-100): local_constants / local_wires / public_inputs_hash as lazily
    recorded loads."""

    def __init__(self, b, num_wires, num_constants, prefix=0):
        self.b, self.num_wires, self.num_constants, self.prefix = b, num_wires, num_constants, prefix

    def local_constant(self, i):
        assert 0 <= self.prefix + i < self.num_constants
        return self.b.local(CONSTANTS_SIGMAS, self.prefix + i)

    def local_wire(self, i):
        assert 0 <= i < self.num_wires
        return self.b.local(WIRES, i)

    def public_inputs_hash(self, i):
        assert 0 <= i < 4
        return self.b.bound(i)

    def remove_prefix(self, n):
        return EvaluationVarsBase(self.b, self.num_wires, self.num_constants, self.prefix + n)


class Gate:
    """Gate<F, D> (gates/gate.rs:30-300): id, num_wires, num_constants, degree, num_constraints, eval_unfiltered."""

    def id(self):
        raise NotImplementedError

    def num_wires(self):
        raise NotImplementedError

    def num_constants(self):
        raise NotImplementedError

    def degree(self):
        raise NotImplementedError

    def num_constraints(self):
        raise NotImplementedError

    def eval_unfiltered(self, vars):
        """-> list of num_constraints() Exprs (eval_unfiltered_base_one / _packed)."""
        raise NotImplementedError


class NoopGate(Gate):
    """gates/noop.rs"""

    def id(self):
        return "NoopGate"

    def num_wires(self):
        return 0

    def num_constants(self):
        return 0

    def degree(self):
        return 0

    def num_constraints(self):
        return 0

    def eval_unfiltered(self, vars):
        return []


class ConstantGate(Gate):
    """gates/constant.rs:20-130: wire i must equal constant i."""

    def __init__(self, num_consts):
        self.num_consts = num_consts

    def id(self):
        return "ConstantGate { num_consts: %d }" % self.num_consts

    def num_wires(self):
        return self.num_consts

    def num_constants(self):
        return self.num_consts

    def degree(self):
        return 1

    def num_constraints(self):
        return self.num_consts

    def eval_unfiltered(self, vars):
        return [vars.local_constant(i) - vars.local_wire(i) for i in range(self.num_consts)]


class PublicInputGate(Gate):
    """gates/public_input.rs:22-114: wires 0..4 carry the hash of the public inputs."""

    def id(self):
        return "PublicInputGate"

    def num_wires(self):
        return 4

    def num_constants(self):
        return 0

    def degree(self):
        return 1

    def num_constraints(self):
        return 4

    def eval_unfiltered(self, vars):
        return [vars.local_wire(i) - vars.public_inputs_hash(i) for i in range(4)]


class ArithmeticGate(Gate):
    """gates/arithmetic_base.rs:28-186: num_ops operations output = const_0 * m0 * m1 + const_1 * addend on wires
    (4i, 4i+1, 4i+2, 4i+3)."""

    def __init__(self, num_ops):
        self.num_ops = num_ops

    @classmethod
    def new_from_config(cls, config):
        return cls(config.num_routed_wires // 4)

    def id(self):
        return "ArithmeticGate { num_ops: %d }" % self.num_ops

    def num_wires(self):
        return 4 * self.num_ops

    def num_constants(self):
        return 2

    def degree(self):
        return 3

    def num_constraints(self):
        return self.num_ops

    def eval_unfiltered(self, vars):
        const_0, const_1 = vars.local_constant(0), vars.local_constant(1)
        out = []
        for i in range(self.num_ops):
            m0, m1 = vars.local_wire(4 * i), vars.local_wire(4 * i + 1)
            addend, output = vars.local_wire(4 * i + 2), vars.local_wire(4 * i + 3)
            computed_output = m0 * m1 * const_0 + addend * const_1
            out.append(output - computed_output)
        return out


class Ext2:
    """F_{p^2} = F_p[X]/(X^2 - 7) (field/src/extension/quadratic.rs:14-120) over any value type with + - * (expression
    handles on the host program path, plain numbers in the tests): what vars.get_local_ext returns."""
    __slots__ = ("a", "b")
    W = 7

    def __init__(self, a, b):
        self.a, self.b = a, b

    def __add__(self, o):
        return Ext2(self.a + o.a, self.b + o.b) if isinstance(o, Ext2) else Ext2(self.a + o, self.b)

    def __sub__(self, o):
        return Ext2(self.a - o.a, self.b - o.b) if isinstance(o, Ext2) else Ext2(self.a - o, self.b)

    def __mul__(self, o):
        if isinstance(o, Ext2):
            return Ext2(self.a * o.a + self.b * o.b * self.W, self.a * o.b + self.b * o.a)
        return Ext2(self.a * o, self.b * o)          # scalar_mul

    scalar_mul = __mul__

    def to_basefield_array(self):
        return [self.a, self.b]


def get_local_ext(vars, start):
    """EvaluationVarsBase::get_local_ext (plonk/vars.rs:101-110) for D = 2."""
    return Ext2(vars.local_wire(start), vars.local_wire(start + 1))


D = 2


class ArithmeticExtensionGate(Gate):
    """gates/arithmetic_extension.rs:24-170: num_ops operations output = const_0 * m0 * m1 + const_1 * addend in F_{p^2}."""

    def __init__(self, num_ops):
        self.num_ops = num_ops

    @classmethod
    def new_from_config(cls, config):
        return cls(config.num_routed_wires // (4 * D))

    def id(self):
        return "ArithmeticExtensionGate { num_ops: %d }" % self.num_ops

    def num_wires(self):
        return self.num_ops * 4 * D

    def num_constants(self):
        return 2

    def degree(self):
        return 3

    def num_constraints(self):
        return self.num_ops * D

    def eval_unfiltered(self, vars):
        const_0, const_1 = vars.local_constant(0), vars.local_constant(1)
        out = []
        for i in range(self.num_ops):
            m0, m1 = get_local_ext(vars, 4 * D * i), get_local_ext(vars, 4 * D * i + D)
            addend, output = get_local_ext(vars, 4 * D * i + 2 * D), get_local_ext(vars, 4 * D * i + 3 * D)
            computed_output = (m0 * m1).scalar_mul(const_0) + addend.scalar_mul(const_1)
            out += (output - computed_output).to_basefield_array()
        return out


class MulExtensionGate(Gate):
    """gates/multiplication_extension.rs:24-157: num_ops operations output = const_0 * m0 * m1 in F_{p^2}."""

    def __init__(self, num_ops):
        self.num_ops = num_ops

    @classmethod
    def new_from_config(cls, config):
        return cls(config.num_routed_wires // (3 * D))

    def id(self):
        return "MulExtensionGate { num_ops: %d }" % self.num_ops

    def num_wires(self):
        return self.num_ops * 3 * D

    def num_constants(self):
        return 1

    def degree(self):
        return 3

    def num_constraints(self):
        return self.num_ops * D

    def eval_unfiltered(self, vars):
        const_0 = vars.local_constant(0)
        out = []
        for i in range(self.num_ops):
            m0, m1 = get_local_ext(vars, 3 * D * i), get_local_ext(vars, 3 * D * i + D)
            output = get_local_ext(vars, 3 * D * i + 2 * D)
            out += (output - (m0 * m1).scalar_mul(const_0)).to_basefield_array()
        return out


class BaseSumGate(Gate):
    """gates/base_sum.rs:27-171 (BaseSumGate<B>): wire 0 = sum of the limbs (wires 1..) in base B, little endian; every
    limb range-checked by prod_{i<B} (limb - i)."""
    WIRE_SUM, START_LIMBS = 0, 1

    def __init__(self, num_limbs, base=2):
        self.num_limbs, self.base = num_limbs, base

    @classmethod
    def new_from_config(cls, config, base=2):
        log_floor, x = 0, F.ORDER - 1                       # log_floor(F::ORDER - 1, B)
        while x >= base:
            x //= base
            log_floor += 1
        return cls(min(log_floor, config.num_routed_wires - cls.START_LIMBS), base)

    def id(self):
        return "BaseSumGate { num_limbs: %d } + Base: %d" % (self.num_limbs, self.base)

    def num_wires(self):
        return 1 + self.num_limbs

    def num_constants(self):
        return 0

    def degree(self):
        return self.base

    def num_constraints(self):
        return 1 + self.num_limbs

    def eval_unfiltered(self, vars):
        total = vars.local_wire(self.WIRE_SUM)
        limbs = [vars.local_wire(self.START_LIMBS + i) for i in range(self.num_limbs)]
        computed = None                                     # reduce_with_powers(limbs, B): Horner from the top limb
        for limb in reversed(limbs):
            computed = limb if computed is None else computed * self.base + limb
        out = [computed - total]
        for limb in limbs:
            acc = limb                                      # (limb - 0)
            for i in range(1, self.base):
                acc = acc * (limb - i)
            out.append(acc)
        return out


class ReducingGate(Gate):
    """gates/reducing.rs:25-185: acc_{i} = acc_{i-1} * alpha + coeff_i over F_{p^2} with base-field coefficients; the last
    accumulator is the output (wires 0..D)."""

    def __init__(self, num_coeffs):
        self.num_coeffs = num_coeffs

    @staticmethod
    def max_coeffs_len(num_wires, num_routed_wires):
        return min(num_routed_wires - 3 * D, (num_wires - 2 * D) // (D + 1))

    START_COEFFS = 3 * D

    def start_accs(self):
        return self.START_COEFFS + self.num_coeffs

    def wires_accs(self, i):
        return 0 if i == self.num_coeffs - 1 else self.start_accs() + D * i

    def id(self):
        return "ReducingGate { num_coeffs: %d }" % self.num_coeffs

    def num_wires(self):
        return 2 * D + self.num_coeffs * (D + 1)

    def num_constants(self):
        return 0

    def degree(self):
        return 2

    def num_constraints(self):
        return D * self.num_coeffs

    def coeff(self, vars, i):
        return vars.local_wire(self.START_COEFFS + i)

    def eval_unfiltered(self, vars):
        alpha, acc = get_local_ext(vars, D), get_local_ext(vars, 2 * D)
        out = []
        for i in range(self.num_coeffs):
            acc_i = get_local_ext(vars, self.wires_accs(i))
            out += (acc * alpha + self.coeff(vars, i) - acc_i).to_basefield_array()
            acc = acc_i
        return out


class ReducingExtensionGate(ReducingGate):
    """gates/reducing_extension.rs:24-185: the same with coefficients in F_{p^2}."""

    @staticmethod
    def max_coeffs_len(num_wires, num_routed_wires):
        return min((num_routed_wires - 3 * D) // D, (num_wires - 2 * D) // (D * 2))

    def start_accs(self):
        return self.START_COEFFS + self.num_coeffs * D

    def id(self):
        return "ReducingExtensionGate { num_coeffs: %d }" % self.num_coeffs

    def num_wires(self):
        return 2 * D + 2 * D * self.num_coeffs

    def coeff(self, vars, i):
        return get_local_ext(vars, self.START_COEFFS + i * D)


_POSEIDON = None


def poseidon_tables():
    """The Poseidon-12 parameter tables (plonky2/src/hash/poseidon.rs:59-157, poseidon_goldilocks.rs:24-215), read from
    the same generated header the kernels compile (csrc/gl_poseidon_constants.h)."""
    global _POSEIDON
    if _POSEIDON is None:
        text = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "gl_poseidon_constants.h")).read()
        tabs = {}
        for name, count, body in re.findall(r"GL_POSEIDON_(\w+)\[(\d+)\]\s*=\s*\{([^}]*)\}", text):
            vals = [int(v, 16) for v in re.findall(r"0x([0-9a-fA-F]+)", body)]
            assert len(vals) == int(count), name
            tabs[name] = vals
        assert len(tabs["RC"]) == 360 and len(tabs["FAST_VS"]) == 242 and len(tabs["FAST_INIT_MATRIX"]) == 121
        _POSEIDON = tabs
    return _POSEIDON


SPONGE_WIDTH, HALF_N_FULL_ROUNDS, N_PARTIAL_ROUNDS = 12, 4, 22


class PoseidonGate(Gate):
    """gates/poseidon.rs:28-420: one Poseidon permutation of 12 wires with the swap flag for Merkle proofs; the S-box
    inputs of every round but the first are wires, so that each constraint has degree 7."""
    WIRE_SWAP = 2 * SPONGE_WIDTH
    START_DELTA = 2 * SPONGE_WIDTH + 1
    START_FULL_0 = START_DELTA + 4
    START_PARTIAL = START_FULL_0 + SPONGE_WIDTH * (HALF_N_FULL_ROUNDS - 1)
    START_FULL_1 = START_PARTIAL + N_PARTIAL_ROUNDS
    END = START_FULL_1 + SPONGE_WIDTH * HALF_N_FULL_ROUNDS

    @staticmethod
    def wire_input(i):
        return i

    @staticmethod
    def wire_output(i):
        return SPONGE_WIDTH + i

    @classmethod
    def wire_delta(cls, i):
        return cls.START_DELTA + i

    @classmethod
    def wire_full_sbox_0(cls, round, i):
        assert 0 < round < HALF_N_FULL_ROUNDS
        return cls.START_FULL_0 + SPONGE_WIDTH * (round - 1) + i

    @classmethod
    def wire_partial_sbox(cls, round):
        return cls.START_PARTIAL + round

    @classmethod
    def wire_full_sbox_1(cls, round, i):
        return cls.START_FULL_1 + SPONGE_WIDTH * round + i

    def id(self):
        return "PoseidonGate(PhantomData<plonky2_field::goldilocks_field::GoldilocksField>)<WIDTH=12>"

    def num_wires(self):
        return self.END

    def num_constants(self):
        return 0

    def degree(self):
        return 7

    def num_constraints(self):
        return SPONGE_WIDTH * (2 * HALF_N_FULL_ROUNDS - 1) + N_PARTIAL_ROUNDS + SPONGE_WIDTH + 1 + 4

    # the layers of hash/poseidon.rs over expression handles
    @staticmethod
    def _constant_layer(state, round_ctr):
        rc = poseidon_tables()["RC"]
        return [state[i] + rc[i + SPONGE_WIDTH * round_ctr] for i in range(SPONGE_WIDTH)]

    @staticmethod
    def _sbox_monomial(x):
        x2 = x * x
        x4 = x2 * x2
        return x * x2 * x4

    @staticmethod
    def _mds_layer(state):
        """mds_row_shf (poseidon.rs:180-200): result[r] = sum_i state[(i + r) % 12] * CIRC[i] + state[r] * DIAG[r]."""
        t = poseidon_tables()
        circ, diag = t["MDS_CIRC"], t["MDS_DIAG"]
        out = []
        for r in range(SPONGE_WIDTH):
            acc = None
            for i in range(SPONGE_WIDTH):
                term = state[(i + r) % SPONGE_WIDTH] * (circ[i] + (diag[r] if i == 0 else 0))
                acc = term if acc is None else acc + term
            out.append(acc)
        return out

    @staticmethod
    def _mds_partial_layer_init(state):
        m = poseidon_tables()["FAST_INIT_MATRIX"]
        out = [state[0]]
        for c in range(1, SPONGE_WIDTH):
            acc = None
            for r in range(1, SPONGE_WIDTH):
                term = state[r] * m[(r - 1) * 11 + (c - 1)]
                acc = term if acc is None else acc + term
            out.append(acc)
        return out

    @staticmethod
    def _mds_partial_layer_fast(state, r):
        t = poseidon_tables()
        d = state[0] * (t["MDS_CIRC"][0] + t["MDS_DIAG"][0])
        for i in range(1, SPONGE_WIDTH):
            d = d + state[i] * t["FAST_W_HATS"][r * 11 + i - 1]
        return [d] + [state[0] * t["FAST_VS"][r * 11 + i - 1] + state[i] for i in range(1, SPONGE_WIDTH)]

    def eval_unfiltered(self, vars):
        """eval_unfiltered_base_one (poseidon.rs:204-283)."""
        t = poseidon_tables()
        w = vars.local_wire
        out = []
        swap = w(self.WIRE_SWAP)
        out.append(swap * (swap - 1))
        for i in range(4):
            out.append(swap * (w(self.wire_input(i + 4)) - w(self.wire_input(i))) - w(self.wire_delta(i)))
        state = [None] * SPONGE_WIDTH
        for i in range(4):
            state[i] = w(self.wire_input(i)) + w(self.wire_delta(i))
            state[i + 4] = w(self.wire_input(i + 4)) - w(self.wire_delta(i))
        for i in range(8, SPONGE_WIDTH):
            state[i] = w(self.wire_input(i))
        round_ctr = 0
        for r in range(HALF_N_FULL_ROUNDS):
            state = self._constant_layer(state, round_ctr)
            if r != 0:
                for i in range(SPONGE_WIDTH):
                    sbox_in = w(self.wire_full_sbox_0(r, i))
                    out.append(state[i] - sbox_in)
                    state[i] = sbox_in
            state = self._mds_layer([self._sbox_monomial(x) for x in state])
            round_ctr += 1
        state = [state[i] + t["FAST_FIRST_RC"][i] for i in range(SPONGE_WIDTH)]
        state = self._mds_partial_layer_init(state)
        for r in range(N_PARTIAL_ROUNDS):
            sbox_in = w(self.wire_partial_sbox(r))
            out.append(state[0] - sbox_in)
            state[0] = self._sbox_monomial(sbox_in)
            if r < N_PARTIAL_ROUNDS - 1:
                state[0] = state[0] + t["FAST_RC"][r]
            state = self._mds_partial_layer_fast(state, r)
        round_ctr += N_PARTIAL_ROUNDS
        for r in range(HALF_N_FULL_ROUNDS):
            state = self._constant_layer(state, round_ctr)
            for i in range(SPONGE_WIDTH):
                sbox_in = w(self.wire_full_sbox_1(r, i))
                out.append(state[i] - sbox_in)
                state[i] = sbox_in
            state = self._mds_layer([self._sbox_monomial(x) for x in state])
            round_ctr += 1
        for i in range(SPONGE_WIDTH):
            out.append(state[i] - w(self.wire_output(i)))
        return out


class PoseidonMdsGate(Gate):
    """gates/poseidon_mds.rs:28-221: outputs = MDS * inputs for 12 elements of F_{p^2} (the MDS layer acts on both
    components)."""

    def id(self):
        return "PoseidonMdsGate(PhantomData<plonky2_field::goldilocks_field::GoldilocksField>)<WIDTH=12>"

    def num_wires(self):
        return 2 * D * SPONGE_WIDTH

    def num_constants(self):
        return 0

    def degree(self):
        return 1

    def num_constraints(self):
        return SPONGE_WIDTH * D

    def eval_unfiltered(self, vars):
        inputs = [get_local_ext(vars, i * D) for i in range(SPONGE_WIDTH)]
        computed = PoseidonGate._mds_layer(inputs)                 # mds_layer_field
        out = []
        for i in range(SPONGE_WIDTH):
            out += (get_local_ext(vars, (SPONGE_WIDTH + i) * D) - computed[i]).to_basefield_array()
        return out


class RandomAccessGate(Gate):
    """gates/random_access.rs:33-343: num_copies lookups claimed_element = list[access_index] in lists of 2^bits wires,
    through the bit decomposition of the index; leftover routed wires pinned to constants."""

    def __init__(self, num_copies, bits, num_extra_constants):
        self.num_copies, self.bits, self.num_extra_constants = num_copies, bits, num_extra_constants

    @classmethod
    def new_from_config(cls, config, bits):
        vec_size = 1 << bits
        max_copies = min(config.num_routed_wires // (2 + vec_size), config.num_wires // (2 + vec_size + bits))
        max_extra_constants = config.num_routed_wires - (2 + vec_size) * max_copies
        return cls(max_copies, bits, min(max_extra_constants, config.num_constants))

    def vec_size(self):
        return 1 << self.bits

    def wire_access_index(self, copy):
        return (2 + self.vec_size()) * copy

    def wire_claimed_element(self, copy):
        return (2 + self.vec_size()) * copy + 1

    def wire_list_item(self, i, copy):
        return (2 + self.vec_size()) * copy + 2 + i

    def wire_extra_constant(self, i):
        return (2 + self.vec_size()) * self.num_copies + i

    def num_routed_wires(self):
        return (2 + self.vec_size()) * self.num_copies + self.num_extra_constants

    def wire_bit(self, i, copy):
        return self.num_routed_wires() + copy * self.bits + i

    def id(self):
        return ("RandomAccessGate { bits: %d, num_copies: %d, num_extra_constants: %d, _phantom: PhantomData<plonky2_field::"
                "goldilocks_field::GoldilocksField> }<D=2>" % (self.bits, self.num_copies, self.num_extra_constants))

    def num_wires(self):
        return self.wire_bit(self.bits - 1, self.num_copies - 1) + 1

    def num_constants(self):
        return self.num_extra_constants

    def degree(self):
        return self.bits + 1

    def num_constraints(self):
        return self.num_copies * (self.bits + 2) + self.num_extra_constants

    def eval_unfiltered(self, vars):
        w = vars.local_wire
        out = []
        for copy in range(self.num_copies):
            bits = [w(self.wire_bit(i, copy)) for i in range(self.bits)]
            for b in bits:
                out.append(b * (b - 1))
            acc = None                                  # bits.rev().fold(0, |acc, b| acc + acc + b)
            for b in reversed(bits):
                acc = b if acc is None else acc + acc + b
            out.append(acc - w(self.wire_access_index(copy)))
            items = [w(self.wire_list_item(i, copy)) for i in range(self.vec_size())]
            for b in bits:
                items = [x + b * (y - x) for x, y in zip(items[0::2], items[1::2])]
            out.append(items[0] - w(self.wire_claimed_element(copy)))
        for i in range(self.num_extra_constants):
            out.append(vars.local_constant(i) - w(self.wire_extra_constant(i)))
        return out


class ExponentiationGate(Gate):
    """gates/exponentiation.rs:33-243: output = base^power from the power's bits (wires 1.., little endian) by square and
    multiply with one intermediate wire per bit."""

    def __init__(self, num_power_bits):
        self.num_power_bits = num_power_bits

    @classmethod
    def new_from_config(cls, config):
        return cls(min(config.num_routed_wires - 2, (config.num_wires - 2) // 2))

    def wire_power_bit(self, i):
        return 1 + i

    def wire_output(self):
        return 1 + self.num_power_bits

    def wire_intermediate_value(self, i):
        return 2 + self.num_power_bits + i

    def id(self):
        return ("ExponentiationGate { num_power_bits: %d, _phantom: PhantomData<plonky2_field::goldilocks_field::"
                "GoldilocksField> }<D=2>" % self.num_power_bits)

    def num_wires(self):
        return self.wire_intermediate_value(self.num_power_bits - 1) + 1

    def num_constants(self):
        return 0

    def degree(self):
        return 4

    def num_constraints(self):
        return self.num_power_bits + 1

    def eval_unfiltered(self, vars):
        w = vars.local_wire
        base = w(0)
        n = self.num_power_bits
        inter = [w(self.wire_intermediate_value(i)) for i in range(n)]
        out = []
        for i in range(n):
            cur_bit = w(self.wire_power_bit(n - i - 1))          # little-endian bits, accumulated big-endian
            factor = cur_bit * base + (1 - cur_bit)
            computed = factor if i == 0 else inter[i - 1] * inter[i - 1] * factor
            out.append(computed - inter[i])
        out.append(w(self.wire_output()) - inter[n - 1])
        return out


def two_adic_subgroup(bits):
    """Field::two_adic_subgroup (field/src/types.rs:283-287)."""
    g, out, x = F.primitive_root_of_unity(bits), [], 1
    for _ in range(1 << bits):
        out.append(x)
        x = x * g % F.ORDER
    return out


def barycentric_weights(points):
    """barycentric_weights (field/src/interpolation.rs:53-65) for base-field abscissae."""
    out = []
    for i, xi in enumerate(points):
        d = 1
        for j, xj in enumerate(points):
            if j != i:
                d = d * (xi - xj) % F.ORDER
        out.append(pow(d, F.ORDER - 2, F.ORDER))
    return out


class CosetInterpolationGate(Gate):
    """gates/coset_interpolation.rs:30-397: evaluates at an F_{p^2} point the interpolant of 2^subgroup_bits F_{p^2}
    values given on a coset shift*H, as barycentric partial sums with every (degree-1)-th intermediate on a wire."""

    def __init__(self, subgroup_bits, max_degree=None):
        n_points = 1 << subgroup_bits
        max_degree = n_points if max_degree is None else max_degree
        assert max_degree > 1, "need at least quadratic constraints"
        n_intermediates = (n_points - 2) // (max_degree - 1)
        self.subgroup_bits = subgroup_bits
        self._degree = (n_points - 2) // (n_intermediates + 1) + 2
        self.domain = two_adic_subgroup(subgroup_bits)
        self.barycentric_weights = barycentric_weights(self.domain)

    def num_points(self):
        return 1 << self.subgroup_bits

    def wires_value(self, i):
        return 1 + i * D

    def start_evaluation_point(self):
        return 1 + self.num_points() * D

    def start_evaluation_value(self):
        return self.start_evaluation_point() + D

    def start_intermediates(self):
        return self.start_evaluation_value() + D

    def num_intermediates(self):
        return (self.num_points() - 2) // (self._degree - 1)

    def wires_intermediate_eval(self, i):
        return self.start_intermediates() + D * i

    def wires_intermediate_prod(self, i):
        return self.start_intermediates() + D * (self.num_intermediates() + i)

    def wires_shifted_evaluation_point(self):
        return self.start_intermediates() + D * 2 * self.num_intermediates()

    def id(self):
        return "CosetInterpolationGate { subgroup_bits: %d, degree: %d, barycentric_weights: %r }<D=2>" % (
            self.subgroup_bits, self._degree, self.barycentric_weights)

    def num_wires(self):
        return self.start_intermediates() + D * (2 * self.num_intermediates() + 1)

    def num_constants(self):
        return 0

    def degree(self):
        return self._degree

    def num_constraints(self):
        return D + D + 2 * D * self.num_intermediates()

    def partial_interpolate(self, lo, hi, values, x, acc):
        """partial_interpolate (coset_interpolation.rs:553-580) over domain[lo:hi]; acc = (eval, partial product) or None
        for the initial (0, 1)."""
        for i in range(lo, hi):
            val = values[i].scalar_mul(self.barycentric_weights[i])
            term = x - self.domain[i]
            acc = (val, term) if acc is None else (acc[0] * term + val * acc[1], acc[1] * term)
        return acc

    def eval_unfiltered(self, vars):
        shift = vars.local_wire(0)
        point = get_local_ext(vars, self.start_evaluation_point())
        shifted = get_local_ext(vars, self.wires_shifted_evaluation_point())
        out = (point - shifted.scalar_mul(shift)).to_basefield_array()
        values = [get_local_ext(vars, self.wires_value(i)) for i in range(self.num_points())]
        d = self._degree
        acc = self.partial_interpolate(0, d, values, shifted, None)
        for i in range(self.num_intermediates()):
            ie = get_local_ext(vars, self.wires_intermediate_eval(i))
            ip = get_local_ext(vars, self.wires_intermediate_prod(i))
            out += (ie - acc[0]).to_basefield_array()
            out += (ip - acc[1]).to_basefield_array()
            start = 1 + (d - 1) * (i + 1)
            acc = self.partial_interpolate(start, min(start + d - 1, self.num_points()), values, shifted, (ie, ip))
        out += (get_local_ext(vars, self.start_evaluation_value()) - acc[0]).to_basefield_array()
        return out


class LookupGate(Gate):
    """gates/lookup.rs:34-170: stores num_slots (input, output) pairs looked up in a table; no constraints of its own
    (the lookup argument's terms are in `check_lookup_constraints`)."""

    def __init__(self, num_slots, lut_index=0):
        self.num_slots, self.lut_index = num_slots, lut_index

    @classmethod
    def new_from_config(cls, config, lut_index=0):
        return cls(config.num_routed_wires // 2, lut_index)

    def id(self):
        return "LookupGate {num_slots: %d, lut_hash: %d}" % (self.num_slots, self.lut_index)

    def num_wires(self):
        return self.num_slots * 2

    def num_constants(self):
        return 0

    def degree(self):
        return 0

    def num_constraints(self):
        return 0

    def eval_unfiltered(self, vars):
        return []


class LookupTableGate(LookupGate):
    """gates/lookup_table.rs:36-188: num_slots table entries (input, output, multiplicity); no constraints of its own."""

    @classmethod
    def new_from_config(cls, config, lut_index=0):
        return cls(config.num_routed_wires // 3, lut_index)

    def id(self):
        return "LookupTableGate {num_slots: %d, lut_hash: %d}" % (self.num_slots, self.lut_index)

    def num_wires(self):
        return self.num_slots * 3


# ------------------------------------------------------------------ circuit data
class SelectorsInfo:
    """gates/selectors.rs:16-26"""

    def __init__(self, selector_indices, groups):
        self.selector_indices, self.groups = selector_indices, groups

    def num_selectors(self):
        return len(self.groups)


def selector_polynomials(gates, instance_gate_indices, max_degree):
    """selector_polynomials (gates/selectors.rs:114-194). gates: sorted gate list; instance_gate_indices[row] = index of
    the row's gate in `gates`. -> (list of selector value columns, SelectorsInfo)."""
    n, num_gates = len(instance_gate_indices), len(gates)
    max_gate_degree = gates[-1].degree()
    idx = np.asarray(instance_gate_indices, dtype=np.uint64)
    if max_gate_degree + num_gates - 1 <= max_degree:
        return [idx.copy()], SelectorsInfo([0] * num_gates, [range(0, num_gates)])
    if max_gate_degree >= max_degree:
        raise ValueError("%s has too high degree. Consider increasing `quotient_degree_factor`." % gates[-1].id())
    groups, start = [], 0
    while start < num_gates:
        size = 0
        while start + size < num_gates and size + gates[start + size].degree() < max_degree:
            size += 1
        groups.append(range(start, start + size))
        start += size
    group_of = [next(j for j, r in enumerate(groups) if i in r) for i in range(num_gates)]
    polys = []
    for g in range(len(groups)):
        col = np.full(n, UNUSED_SELECTOR, dtype=np.uint64)
        for row, i in enumerate(instance_gate_indices):
            if group_of[i] == g:
                col[row] = i
        polys.append(col)
    return polys, SelectorsInfo(group_of, groups)


def num_partial_products(n, max_degree):
    """util/partial_products.rs:40-46"""
    return -(-n // max_degree) - 1


class CommonCircuitData:
    """The fields of CommonCircuitData (plonk/circuit_data.rs:420-560) the quotient needs."""

    def __init__(self, config, degree_bits, gates, selectors_info, num_constants, k_is, luts=(), lookup_rows=()):
        self.config, self.degree_bits, self.gates, self.selectors_info = config, degree_bits, gates, selectors_info
        self.luts = [list(t) for t in luts]                                   # LookupTable = [(input, output)] of u16
        self.lookup_rows = [tuple(r) for r in lookup_rows]                    # LookupWire triples, one per table
        self.num_lookup_selectors = (LOOKUP_START_END + len(self.lookup_rows)) if self.luts else 0
        # 1 RE polynomial and ceil(num_lu_slots / (max_quotient_degree_factor - 1)) partial Sum/LDC polynomials
        self.num_lookup_polys = (-(-(config.num_routed_wires // 2) // (config.max_quotient_degree_factor - 1)) + 1
                                 if self.luts else 0)                        # circuit_builder.rs:1245-1251
        self.quotient_degree_factor = config.max_quotient_degree_factor       # circuit_builder.rs:1146
        self.num_gate_constraints = max([g.num_constraints() for g in gates] + [0])   # circuit_builder.rs:1236-1240
        self.num_constants = num_constants
        self.k_is = [int(k) for k in k_is]
        self.num_partial_products = num_partial_products(config.num_routed_wires, self.quotient_degree_factor)
        self._program = None

    @classmethod
    def from_gate_instances(cls, config, instances, luts=(), lookup_rows=()):
        """The part of CircuitBuilder::build (plonk/circuit_builder.rs:1146-1171) that fixes the constants commitment:
        instances = [(gate, constants)] per row (already padded to a power of two). Gates are sorted by (degree, id);
        returns (common_data, constant_vecs) with constant_vecs = selector columns, the lookup selectors
        (selectors_lookup + selector_ends_lookups, gates/selectors.rs:50-108; lookup_rows = one LookupWire triple
        (last_lu_gate, last_lut_gate, first_lut_gate) per table of `luts`), then the constant columns."""
        n = len(instances)
        degree_bits = F.log2_strict(n)
        by_id = {}
        for g, _ in instances:
            by_id.setdefault(g.id(), g)
        gates = sorted(by_id.values(), key=lambda g: (g.degree(), g.id()))
        index = {g.id(): i for i, g in enumerate(gates)}
        rows = [index[g.id()] for g, _ in instances]
        constant_vecs, info = selector_polynomials(gates, rows, config.max_quotient_degree_factor + 1)
        if luts:
            assert len(luts) == len(lookup_rows)
            sel = [np.zeros(n, dtype=np.uint64) for _ in range(LOOKUP_START_END)]
            for last_lu_row, last_lut_row, first_lut_row in lookup_rows:
                sel[LOOKUP_TRANS_SRE][last_lut_row:first_lut_row + 1] = 1
                sel[LOOKUP_TRANS_LDC][last_lu_row:last_lut_row] = 1
                sel[LOOKUP_INIT_SRE][first_lut_row + 1] = 1
                sel[LOOKUP_LAST_LDC][last_lu_row] = 1
            for _, last_lut_row, _ in lookup_rows:
                ends = np.zeros(n, dtype=np.uint64)
                ends[last_lut_row] = 1
                sel.append(ends)
            constant_vecs += sel
        max_constants = max(g.num_constants() for g in gates)          # constant_polys, circuit_builder.rs:970-991
        for k in range(max_constants):
            constant_vecs.append(np.array([int(c[k]) % F.ORDER if k < len(c) else 0 for _, c in instances], dtype=np.uint64))
        k_is = get_unique_coset_shifts(config.num_routed_wires)
        return cls(config, degree_bits, gates, info, len(constant_vecs), k_is, luts, lookup_rows), constant_vecs

    def quotient_degree(self):
        return self.quotient_degree_factor << self.degree_bits

    def constants_range(self):
        return range(0, self.num_constants)

    def sigmas_range(self):
        return range(self.num_constants, self.num_constants + self.config.num_routed_wires)

    def zs_range(self):
        return range(0, self.config.num_challenges)

    def partial_products_range(self):
        return range(self.config.num_challenges, (self.num_partial_products + 1) * self.config.num_challenges)

    def num_zs_partial_products_polys(self):
        return self.config.num_challenges * (1 + self.num_partial_products)

    def lookup_range(self, i):
        """The lookup polynomials of challenge i in the zs_partial_products_lookup commitment."""
        start = self.num_zs_partial_products_polys() + i * self.num_lookup_polys
        return range(start, start + self.num_lookup_polys)

    def num_lookup_terms(self):
        """Constraints check_lookup_constraints yields per challenge (vanishing_poly.rs:231-236)."""
        return (4 + len(self.luts) + 2 * (self.num_lookup_polys - 1)) if self.luts else 0

    def num_vanishing_terms(self):
        nc = self.config.num_challenges
        return nc + nc * (self.num_partial_products + 1) + nc * self.num_lookup_terms() + self.num_gate_constraints

    def lut_re_poly_evals(self, deltas):
        """get_lut_poly(..).eval(delta) per table (vanishing_poly.rs:30-52, prover.rs:653-681) for ONE challenge's
        deltas = (A, B, alpha, delta): sum_k (input_k + B output_k) delta^(len - 1 - k) over the table padded with its
        first entry to whole LookupTableGate rows."""
        b, delta = int(deltas[LOOKUP_CHALLENGE_B]), int(deltas[LOOKUP_CHALLENGE_DELTA])
        nb_slots = self.config.num_routed_wires // 3
        out = []
        for lut in self.luts:
            padded = list(lut) + [lut[0]] * ((nb_slots - len(lut) % nb_slots) % nb_slots)
            acc = 0
            for inp, outp in padded:
                acc = (acc * delta + inp + b * outp) % F.ORDER
            out.append(acc)
        return out

    def vanishing_program(self):
        if self._program is None:
            self._program = vanishing_program(self)
        return self._program


def get_unique_coset_shifts(num_shifts):
    """get_unique_coset_shifts (field/src/cosets.rs:9-24): g^0 .. g^(num_shifts-1)."""
    out, x = [], 1
    for _ in range(num_shifts):
        out.append(x)
        x = x * F.MULTIPLICATIVE_GROUP_GENERATOR % F.ORDER
    return out


def compute_filter(b, row, group_range, s, many_selector):
    """compute_filter (gates/gate.rs:326-333)."""
    idx = [i for i in group_range if i != row] + ([UNUSED_SELECTOR] if many_selector else [])
    return b.product([i - s for i in idx]) if idx else None


def check_lookup_constraints(cd, vars, local_lookup_zs, next_lookup_zs, lookup_selectors, deltas, lut_re_poly_evals,
                             product):
    """check_lookup_constraints_batch (plonk/vanishing_poly.rs:521-689) for one challenge, over any value type.
    deltas = (A, B, alpha, delta); product = the value type's product-of-a-list (ONE for an empty list)."""
    cfg = cd.config
    num_lu_slots, num_lut_slots = cfg.num_routed_wires // 2, cfg.num_routed_wires // 3
    lu_degree = cd.quotient_degree_factor - 1
    num_sldc_polys = len(local_lookup_zs) - 1
    lut_degree = -(-num_lut_slots // num_sldc_polys)
    w = vars.local_wire
    z_re, next_z_re = local_lookup_zs[0], next_lookup_zs[0]
    z_x, z_gx = local_lookup_zs[1:], next_lookup_zs[1:]
    d_a, d_b, d_alpha, d_delta = deltas
    looked = [w(3 * s) + w(3 * s + 1) * d_a for s in range(num_lut_slots)]        # Sum / LDC combos
    looking = [w(2 * s) + w(2 * s + 1) * d_a for s in range(num_lu_slots)]
    lookup = [w(3 * s) + w(3 * s + 1) * d_b for s in range(num_lut_slots)]        # RE combos
    out = [lookup_selectors[LOOKUP_LAST_LDC] * z_x[num_sldc_polys - 1],           # last LDC
           lookup_selectors[LOOKUP_INIT_SRE] * z_x[0],                            # initial Sum
           lookup_selectors[LOOKUP_INIT_SRE] * z_re]                              # initial RE
    for r in range(LOOKUP_START_END, cd.num_lookup_selectors):                    # final RE, one per table
        out.append(lookup_selectors[r] * (z_re - lut_re_poly_evals[r - LOOKUP_START_END]))
    cur_sum = next_z_re                                                           # RE row transition
    for elt in lookup:
        cur_sum = cur_sum * d_delta + elt
    out.append(lookup_selectors[LOOKUP_TRANS_SRE] * (z_re - cur_sum))
    for poly in range(num_sldc_polys):
        lut_rng = range(poly * lut_degree, min((poly + 1) * lut_degree, num_lut_slots))
        lu_rng = range(poly * lu_degree, min((poly + 1) * lu_degree, num_lu_slots))
        lut_f = {i: d_alpha - looked[i] for i in lut_rng}
        lu_f = {i: d_alpha - looking[i] for i in lu_rng}
        lut_prod = product([lut_f[i] for i in lut_rng])
        lu_prod = product([lu_f[i] for i in lu_rng])
        lu_sum_prods = None                                                        # sum_i prod_{j != i} (alpha - combo_j)
        for i in lu_rng:
            t = product([lu_f[j] for j in lu_rng if j != i])
            lu_sum_prods = t if lu_sum_prods is None else lu_sum_prods + t
        lut_sum_prods_with_mul = None                                              # sum_i mult_i prod_{j != i} (...)
        for i in lut_rng:
            t = w(3 * i + 2) * product([lut_f[j] for j in lut_rng if j != i])
            lut_sum_prods_with_mul = t if lut_sum_prods_with_mul is None else lut_sum_prods_with_mul + t
        prev = z_gx[num_sldc_polys - 1] if poly == 0 else z_x[poly - 1]
        diff = z_x[poly] - prev
        sum_transition = lut_prod * diff
        if lut_sum_prods_with_mul is not None:
            sum_transition = sum_transition - lut_sum_prods_with_mul
        ldc_transition = lu_prod * diff
        if lu_sum_prods is not None:
            ldc_transition = ldc_transition + lu_sum_prods
        out.append(lookup_selectors[LOOKUP_TRANS_SRE] * sum_transition)
        out.append(lookup_selectors[LOOKUP_TRANS_LDC] * ldc_transition)
    return out


def vanishing_program(cd):
    """eval_vanishing_poly_base_batch (plonk/vanishing_poly.rs:167-340) recorded for one point. Bound constants:
    public_inputs_hash (4), betas (num_challenges), gammas (num_challenges), then with lookups the deltas
    (NUM_COINS_LOOKUP per challenge) and the tables' RE evaluations (per challenge, per table). Term numbers follow the
    reference's order: vanishing_z_1_terms, vanishing_partial_products_terms, vanishing_all_lookup_terms, gate constraints."""
    cfg = cd.config
    nc, nr = cfg.num_challenges, cfg.num_routed_wires
    n_luts = len(cd.luts)
    b = VanishingBuilder(4 + 2 * nc + (nc * (NUM_COINS_LOOKUP + n_luts) if n_luts else 0))
    vars = EvaluationVarsBase(b, cfg.num_wires, cd.num_constants)
    num_selectors = cd.selectors_info.num_selectors()
    # evaluate_gate_constraints_base_batch (vanishing_poly.rs:702-728) with Gate::eval_filtered_base_batch (gate.rs:159-185)
    constraint_terms = [None] * cd.num_gate_constraints
    for i, gate in enumerate(cd.gates):
        b.scope = ("gate", i)
        sel = cd.selectors_info.selector_indices[i]
        filt = compute_filter(b, i, cd.selectors_info.groups[sel], vars.local_constant(sel), num_selectors > 1)
        res = gate.eval_unfiltered(vars.remove_prefix(num_selectors + cd.num_lookup_selectors))
        assert len(res) <= cd.num_gate_constraints, "num_constraints() gave too low of a number"
        for j, r in enumerate(res):
            r = r if filt is None else r * filt
            constraint_terms[j] = r if constraint_terms[j] is None else constraint_terms[j] + r
    b.scope = "permutation"
    x, l_0_x = b.x(), b.l0()
    num_prods, max_degree = cd.num_partial_products, cd.quotient_degree_factor
    for i in range(nc):
        beta, gamma = b.bound(4 + i), b.bound(4 + nc + i)
        z_x, z_gx = b.local(ZS_PARTIAL_PRODUCTS, i), b.next(ZS_PARTIAL_PRODUCTS, i)
        b.term(i, l_0_x * (z_x - 1))                                      # L_0(x) (Z(x) - 1)
        numerators, denominators = [], []
        for j in range(nr):
            wire_value = vars.local_wire(j)
            s_id = x * cd.k_is[j]
            s_sigma = b.local(CONSTANTS_SIGMAS, cd.num_constants + j)
            numerators.append(wire_value + beta * s_id + gamma)
            denominators.append(wire_value + beta * s_sigma + gamma)
        # check_partial_products (util/partial_products.rs:52-76)
        accs = [z_x] + [b.local(ZS_PARTIAL_PRODUCTS, nc + i * num_prods + k) for k in range(num_prods)] + [z_gx]
        for k in range(num_prods + 1):
            num = b.product(numerators[k * max_degree:(k + 1) * max_degree])
            den = b.product(denominators[k * max_degree:(k + 1) * max_degree])
            b.term(nc + i * (num_prods + 1) + k, accs[k] * num - accs[k + 1] * den)
    lookup_base = nc + nc * (num_prods + 1)
    n_lookup = cd.num_lookup_terms()
    for i in range(nc if n_luts else 0):                                  # vanishing_poly.rs:266-285
        b.scope = ("lookup", i)
        at = 4 + 2 * nc + i * NUM_COINS_LOOKUP
        deltas = [b.bound(at + k) for k in range(NUM_COINS_LOOKUP)]
        re_evals = [b.bound(4 + 2 * nc + nc * NUM_COINS_LOOKUP + i * n_luts + t) for t in range(n_luts)]
        rng = cd.lookup_range(i)
        terms = check_lookup_constraints(cd, vars, [b.local(ZS_PARTIAL_PRODUCTS, c) for c in rng],
                                         [b.next(ZS_PARTIAL_PRODUCTS, c) for c in rng],
                                         [vars.local_constant(num_selectors + r) for r in range(cd.num_lookup_selectors)],
                                         deltas, re_evals, b.product)
        assert len(terms) == n_lookup
        for k, t in enumerate(terms):
            b.term(lookup_base + i * n_lookup + k, t)
    base = lookup_base + nc * n_lookup
    for j, t in enumerate(constraint_terms):
        if t is not None:
            b.term(base + j, t)
    # evaluation order: the challenges' checks of one wire chunk next to each other (they share the chunk's k_i x)
    b.term_order = (list(range(nc)) + [nc + i * (num_prods + 1) + k for k in range(num_prods + 1) for i in range(nc)]
                    + list(range(lookup_base, base)) + [base + j for j, t in enumerate(constraint_terms) if t is not None])
    return b


def program_constants(common_data, b, public_inputs_hash, betas, gammas, deltas=()):
    """The constant table of one evaluation of the vanishing program `b`: the values bound per proof
    (public_inputs_hash, betas, gammas, deltas, lut_re_poly_evals) followed by the program's literals."""
    nc = common_data.config.num_challenges
    bound = [int(v) % F.ORDER for v in list(public_inputs_hash) + list(betas) + list(gammas) + list(deltas)]
    for i in range(nc if common_data.luts else 0):   # lut_re_poly_evals (prover.rs:653-681): per challenge and table
        bound += common_data.lut_re_poly_evals(deltas[NUM_COINS_LOOKUP * i:NUM_COINS_LOOKUP * (i + 1)])
    assert len(bound) == b.num_bound
    return np.array(bound + b.consts[b.num_bound:], dtype=np.uint64)


def compute_quotient_polys(common_data, constants_sigmas_commitment, public_inputs_hash, wires_commitment,
                           zs_partial_products_commitment, betas, gammas, alphas, deltas=(),
                           placement=distributed.Placement()):
    """compute_quotient_polys (plonk/prover.rs:609-815) on the device: a torch int64 CUDA tensor (num_challenges, size) of
    quotient-polynomial coefficients, size = n << log2_ceil(quotient_degree_factor). The three PolynomialBatch handles
    stay where they are; nothing but the program and the challenges crosses PCIe. On a placement of several ranks the
    commitments are this rank's row-block shards: each rank evaluates the vanishing polynomial over Z_H on its shard of
    the quotient coset (gl_plonk_quotient_shard), and every rank gets the same quotient
    (Placement.quotient_from_shards; collective, a failure on any rank raises on every rank). On non-resident
    commitments (lde_blocks=G, all of one G) the quotient coset is evaluated in G parts, one per LDE block
    (gl_plonk_quotient_blocked), to the same result; resident and non-resident commitments together are a ShapeError."""
    import torch

    commits = [constants_sigmas_commitment, wires_commitment, zs_partial_products_commitment]
    blocks = sorted({c.lde_blocks for c in commits})
    if len(blocks) > 1:
        raise N.ShapeError("the quotient's commitments must be all resident or all non-resident with one lde_blocks, "
                           "got lde_blocks %s (0: resident)" % [c.lde_blocks for c in commits])
    prog, consts, al = quotient_program(common_data, commits, public_inputs_hash, betas, gammas, alphas, deltas)
    nc = common_data.config.num_challenges
    qdf = common_data.quotient_degree_factor
    ctx = wires_commitment.ctx
    handles = (C.c_void_p * 3)(*[c.h for c in commits])
    ctx.after_caller()
    if placement.num_shards > 1:
        def run_shard(local):
            N.check(N.lib().gl_plonk_quotient_shard(ctx.h, handles, 3, prog, len(prog), N.np_ptr(consts), len(consts),
                                                    N.np_ptr(al), nc, common_data.num_vanishing_terms(), qdf,
                                                    N.vp(local.data_ptr())), ctx.h)

        return placement.quotient_from_shards(ctx, run_shard, nc, common_data.degree_bits, qdf)
    size = (1 << common_data.degree_bits) << (qdf - 1).bit_length()
    out = torch.empty((nc, size), dtype=torch.int64, device="cuda:%d" % ctx.device)
    quotient = N.lib().gl_plonk_quotient_blocked if blocks[0] else N.lib().gl_plonk_quotient
    N.check(quotient(ctx.h, handles, 3, prog, len(prog), N.np_ptr(consts), len(consts), N.np_ptr(al), nc,
                     common_data.num_vanishing_terms(), qdf, N.vp(out.data_ptr())), ctx.h)
    ctx.synchronize()
    return out


def quotient_program(common_data, commits, public_inputs_hash, betas, gammas, alphas, deltas=()):
    """What gl_plonk_quotient and gl_plonk_quotient_shard take besides the three commitments (constants / sigmas, wires,
    Z / partial products [+ lookups]): the compiled vanishing program, its constants and the alphas, as arrays. Raises
    ShapeError for wrong challenge counts or commitments of the wrong width or degree."""
    cfg = common_data.config
    nc = cfg.num_challenges
    if not (len(betas) == len(gammas) == len(alphas) == nc) or len(public_inputs_hash) != 4:
        raise N.ShapeError("expected %d betas, gammas, alphas and a 4-element public_inputs_hash" % nc)
    n_luts = len(common_data.luts)
    if len(deltas) != (NUM_COINS_LOOKUP * nc if n_luts else 0):
        raise N.ShapeError("expected %d lookup challenges (deltas)" % (NUM_COINS_LOOKUP * nc if n_luts else 0))
    expect = [common_data.num_constants + cfg.num_routed_wires, cfg.num_wires,
              nc * (1 + common_data.num_partial_products + common_data.num_lookup_polys)]
    for c, w in zip(commits, expect):
        if c.num_polys != w or c.degree_log != common_data.degree_bits:
            raise N.ShapeError("commitment with %d polynomials of degree 2^%d, expected %d of 2^%d"
                               % (c.num_polys, c.degree_log, w, common_data.degree_bits))
    b = common_data.vanishing_program()
    prog, _ = b.compile()
    consts = program_constants(common_data, b, public_inputs_hash, betas, gammas, deltas)
    return prog, consts, np.array([int(a) % F.ORDER for a in alphas], dtype=np.uint64)


def check_constraints(common_data, constants_sigmas_commitment, public_inputs_hash, wires_commitment,
                      zs_partial_products_commitment, betas, gammas, deltas=(), max_report=64, parts=1, placement=None):
    """The vanishing polynomial's terms checked on every row of the trace subgroup H, each on its own
    (gl_plonk_check_rows): the program compute_quotient_polys runs, at x = w_n^i without alphas or Z_H. Takes what
    compute_quotient_polys takes but the alphas. Returns a ConstraintReport whose entries are (row, term number, label)
    for the first max_report (0..65536) failing (row, term) pairs in (row, term) order; the labels follow
    vanishing_program's term layout, and a gate constraint's label names the gate placed at that row.
    parts=G (a power of two): H is checked in min(G, n) parts one after another (gl_plonk_check_rows_part), each with
    1/G of the whole check's scratch; the report is the same. placement: a distributed.Placement of several ranks, whose
    commitments these are: each rank checks its own part and the ranks merge their reports (collective; every rank
    returns the same report). The labels are attached after the merge, from local evaluations of the constants/sigmas
    commitment, so every rank labels the same pairs alike."""
    parts = N.check_parts(parts)
    commits = [constants_sigmas_commitment, wires_commitment, zs_partial_products_commitment]
    # no alphas: the betas stand in for quotient_program's count check, and its alpha array is not used
    prog, consts, _ = quotient_program(common_data, commits, public_inputs_hash, betas, gammas, betas, deltas)
    ctx = wires_commitment.ctx
    handles = (C.c_void_p * 3)(*[c.h for c in commits])
    L = N.lib()
    failures, pairs = N.check_rows_in_parts(L.gl_plonk_check_rows, L.gl_plonk_check_rows_part, ctx,
                                            (handles, 3, prog, len(prog), N.np_ptr(consts), len(consts),
                                             common_data.num_vanishing_terms()), max_report, common_data.degree_bits,
                                            parts, placement)
    return N.ConstraintReport(failures, _term_labels(common_data, constants_sigmas_commitment, pairs))


def _raise_on_failure(common_data, *commitments_and_challenges, **check_kwargs):
    """prove_with_witness's check_constraints=True: ConstraintError with the first failure's row and label and the
    total. check_kwargs: the placement's (Placement.check_kwargs)."""
    report = check_constraints(common_data, *commitments_and_challenges, **check_kwargs)
    if report.failures:
        row, _, label = report.entries[0]
        raise N.ConstraintError("Constraint failed in the circuit at row %d: %s; %d failing (row, term) pairs in all"
                                % (row, label, report.failures), report)


def _term_labels(cd, constants_sigmas_commitment, pairs):
    """(row, term, label) for check_constraints' (row, term) pairs, by vanishing_program's term layout. The gate at a
    gate constraint's row is read from the selector polynomials evaluated at w_n^row."""
    nc, num_prods = cd.config.num_challenges, cd.num_partial_products
    n_lookup = cd.num_lookup_terms()
    lookup_base = nc + nc * (num_prods + 1)
    base = lookup_base + nc * n_lookup
    gate_rows = sorted({row for row, t in pairs if t >= base})
    gates = {}
    if gate_rows:
        from .proof import eval_commitments

        w = F.primitive_root_of_unity(cd.degree_bits)
        num_selectors = cd.selectors_info.num_selectors()
        evals = eval_commitments([(constants_sigmas_commitment, (pow(w, row, F.ORDER), 0)) for row in gate_rows])
        for row, ev in zip(gate_rows, evals):
            sel = [int(v) for v in ev[:num_selectors, 0]]
            used = [v for v in sel if v != UNUSED_SELECTOR]
            gates[row] = cd.gates[used[0]].id() if used and used[0] < len(cd.gates) else "no gate"
    out = []
    for row, t in pairs:
        if t < nc:
            label = "Z(1) = 1 of challenge %d" % t
        elif t < lookup_base:
            i, k = (t - nc) // (num_prods + 1), (t - nc) % (num_prods + 1)
            label = "partial-product check %d of challenge %d" % (k, i)
            if k == num_prods and row == (1 << cd.degree_bits) - 1:
                label += " (the permutation does not close: a copy constraint is violated)"
        elif t < base:
            i, k = (t - lookup_base) // n_lookup, (t - lookup_base) % n_lookup
            label = "lookup term %d of challenge %d" % (k, i)
        else:
            label = "gate constraint %d of %s" % (t - base, gates[row])
        out.append((row, t, label))
    return out


def _witness_columns(a, rows, n, what):
    """(the array read, its column stride, memory kind, CUDA device or None) of a (rows, n) array whose column c is row c: a
    host array (read in place when it is already C-contiguous uint64, page-locked or not) or a CUDA tensor of 8-byte
    words with unit stride along n. ShapeError for any other shape."""
    try:
        import torch
    except ImportError:  # pragma: no cover
        torch = None
    if torch is not None and isinstance(a, torch.Tensor) and a.is_cuda:
        if tuple(a.shape) != (rows, n) or a.element_size() != 8 or (n > 1 and a.stride(1) != 1):
            raise N.ShapeError("%s must be a (%d, %d) tensor of 8-byte words, unit stride along the rows"
                               % (what, rows, n))
        return a, a.stride(0), N.MEM_DEVICE, a.device.index or 0
    h = np.ascontiguousarray(a, dtype=np.uint64)
    if h.shape != (rows, n):
        raise N.ShapeError("%s must be (%d, %d), got %s" % (what, rows, n, h.shape))
    return h, n, N.MEM_HOST, None


def _witness_values(w, rows, cols):
    """Canonical values of the witness entries (rows[i], cols[i]) of a host array or CUDA tensor, as ints."""
    rows, cols = np.asarray(rows, dtype=np.int64), np.asarray(cols, dtype=np.int64)
    if isinstance(w, np.ndarray):
        v = w[rows, cols] if len(rows) else np.zeros(0, dtype=np.uint64)
    else:
        import torch

        idx = torch.from_numpy(rows).to(w.device), torch.from_numpy(cols).to(w.device)
        v = w[idx].cpu().numpy().view(np.uint64) if len(rows) else np.zeros(0, dtype=np.uint64)
    return [int(x) % F.ORDER for x in v.tolist()]


def _check_max_report(max_report):
    if not isinstance(max_report, (int, np.integer)) or not 0 <= max_report <= N.MAX_REPORT:
        raise N.ShapeError("max_report=%r must be in 0..%d" % (max_report, N.MAX_REPORT))
    return int(max_report)


def check_copy_constraints(prover_data, common_data, wires, max_report=64, ctx=None):
    """The copy constraints checked on a witness (gl_plonk_check_copies), before any commitment: routed wire (row, col)
    must carry the value of wire sigma(row, col), the routed wire whose identity value k_is[col'] * w_n^row' is its
    sigma value prover_data.sigmas[col][row]; the cycles of sigma include the joins through virtual targets. This is
    what the reference's witness generation stops at ("Partition containing {target} was set twice with different
    values"). wires: the (num_wires, n) witness, a host array or a CUDA tensor (the library's stream is ordered after
    torch's current stream first). Returns a ConstraintReport of every failing wire and the first max_report of them in
    (row, col) order, as (row, col, "wire (row, col) = v is copied to wire (row', col') = v'"). ShapeError before any
    device work for a witness or sigmas of the wrong shape or max_report outside 0..65536; NativeError for sigmas that
    are not a permutation of the identity values."""
    cd, cfg = common_data, common_data.config
    n, nr = 1 << cd.degree_bits, cfg.num_routed_wires
    max_report = _check_max_report(max_report)
    w, ws, wmem, wdev = _witness_columns(wires, cfg.num_wires, n, "the witness")
    sg, ss, smem, sdev = _witness_columns(prover_data.sigmas, nr, n, "prover_data.sigmas")
    k_is = np.array(cd.k_is, dtype=np.uint64)
    if len(k_is) != nr:
        raise N.ShapeError("common_data.k_is has %d shifts for %d routed wires" % (len(k_is), nr))
    ctx = ctx or N.default_context(wdev if wdev is not None else sdev or 0)
    if N.MEM_DEVICE in (wmem, smem):
        ctx.after_caller()
    wp, sp = [N.vp(a.data_ptr()) if m == N.MEM_DEVICE else N.np_ptr(a) for a, m in ((w, wmem), (sg, smem))]
    failures, reported = C.c_uint64(), C.c_uint32()
    pairs = np.zeros(2 * max(max_report, 1), dtype=np.uint32)
    N.check(N.lib().gl_plonk_check_copies(ctx.h, wp, ws, wmem, sp, ss, smem, N.np_ptr(k_is), cd.degree_bits, nr,
                                          max_report, C.byref(failures), pairs.ctypes.data_as(N.u32p),
                                          C.byref(reported)), ctx.h)
    pairs = pairs[:2 * reported.value].reshape(-1, 2).astype(np.int64)
    i, j = pairs[:, 0], pairs[:, 1]
    vi = _witness_values(w, i % nr, i // nr)
    vj = _witness_values(w, j % nr, j // nr)
    entries = [(int(a // nr), int(a % nr), "wire (%d, %d) = %d is copied to wire (%d, %d) = %d"
                % (a // nr, a % nr, va, b // nr, b % nr, vb)) for a, b, va, vb in zip(i, j, vi, vj)]
    return N.ConstraintReport(failures.value, entries)


LOOKUP_KINDS = {1: "L1", 2: "L2", 3: "L3"}


def check_lookups(common_data, wires, max_report=64, ctx=None):
    """The lookup argument checked on a witness (gl_plonk_check_lookups), before any commitment, table by table of
    common_data.luts, laid out by common_data.lookup_rows as set_lookup_wires (plonk/prover.rs:50-108) lays them out.
    Three kinds of failure, each named by (row, slot):
    - L1: a looking slot of a LookupGate row whose (input, output) is not an entry of its table (the reference's
      witness generation stops at it: "Incorrect input value provided");
    - L2: a slot of a LookupTableGate row whose (input, output) is not the table entry placed there;
    - L3: a slot of a LookupTableGate row whose multiplicity is not the number of looking slots that count for its
      entry, as the reference counts them (by input, a later entry of one input winning; the padding of the last
      LookupGate row for entry 0). The padding is the run of entry-0 pairs that ends that row: when entry 0's input
      appears again later in a LUT and real lookups of entry 0 end the row, an honest witness gets two L3 entries
      (a known false positive of a check that sees the witness only).
    wires: the (num_wires, n) witness, a host array or a CUDA tensor. Returns a ConstraintReport of every failure and
    the first max_report of them in (row, slot, kind) order, as (row, slot, label); the label names the table, the kind
    and the values. ShapeError before any device work for a witness of the wrong shape or max_report outside
    0..65536."""
    cd, cfg = common_data, common_data.config
    n, nr = 1 << cd.degree_bits, cfg.num_routed_wires
    max_report = _check_max_report(max_report)
    w, ws, wmem, wdev = _witness_columns(wires, cfg.num_wires, n, "the witness")
    luts = [np.asarray(t, dtype=np.int64).reshape(-1, 2) for t in cd.luts]
    if len(cd.lookup_rows) != len(luts):
        raise N.ShapeError("%d lookup tables but %d lookup_rows triples" % (len(luts), len(cd.lookup_rows)))
    if any(len(t) == 0 or (t < 0).any() or (t >> 16).any() for t in luts):
        raise N.ShapeError("lookup tables must be non-empty lists of u16 (input, output) pairs")
    flat = np.ascontiguousarray(np.concatenate(luts) if luts else np.zeros((1, 2)), dtype=np.uint16)
    offsets = np.concatenate([[0], np.cumsum([len(t) for t in luts])]).astype(np.uint32)
    rows = np.ascontiguousarray(np.array(cd.lookup_rows, dtype=np.uint32).reshape(-1))
    counts = np.zeros(max(int(offsets[-1]), 1), dtype=np.uint32)
    ctx = ctx or N.default_context(wdev or 0)
    if wmem == N.MEM_DEVICE:
        ctx.after_caller()
    wp = N.vp(w.data_ptr()) if wmem == N.MEM_DEVICE else N.np_ptr(w)
    failures, reported = C.c_uint64(), C.c_uint32()
    pairs = np.zeros(2 * max(max_report, 1), dtype=np.uint32)
    N.check(N.lib().gl_plonk_check_lookups(ctx.h, wp, ws, wmem, cd.degree_bits, nr, flat.ctypes.data_as(N.vp),
                                           offsets.ctypes.data_as(N.u32p), rows.ctypes.data_as(N.u32p), len(luts),
                                           counts.ctypes.data_as(N.u32p), max_report, C.byref(failures),
                                           pairs.ctypes.data_as(N.u32p), C.byref(reported)), ctx.h)
    pairs = pairs[:2 * reported.value].reshape(-1, 2).astype(np.int64)
    row, slot, kind = pairs[:, 0], pairs[:, 1] >> 2, pairs[:, 1] & 3
    # the values each label names: a looking slot's pair, or a table slot's pair and multiplicity
    looking = kind == 1
    c0 = np.where(looking, 2 * slot, 3 * slot)
    v_in, v_out = _witness_values(w, c0, row), _witness_values(w, c0 + 1, row)
    # a multiplicity exists in table slots only: a looking slot's 3 * slot + 2 can lie past the witness's columns
    table = ~looking
    v_mul = [None] * len(row)
    for t, m in zip(np.flatnonzero(table).tolist(), _witness_values(w, 3 * slot[table] + 2, row[table])):
        v_mul[t] = m
    nts = nr // 3
    entries = []
    for r, s, k, a, b, m in zip(row.tolist(), slot.tolist(), kind.tolist(), v_in, v_out, v_mul):
        t = next(q for q, (lu, _, fl) in enumerate(cd.lookup_rows) if lu <= r <= fl)
        head = "lookup table %d, %s: " % (t, LOOKUP_KINDS[k])
        if k == 1:
            label = head + "looking slot (%d, %d) holds (%d, %d), which is not an entry of the table" % (r, s, a, b)
        else:
            e = (cd.lookup_rows[t][2] - r) * nts + s
            exp = tuple(int(x) for x in luts[t][e if e < len(luts[t]) else 0])
            if k == 2:
                label = head + "table slot (%d, %d) holds (%d, %d), but entry %d%s is (%d, %d)" % (
                    r, s, a, b, e, "" if e < len(luts[t]) else " (padding, entry 0)", *exp)
            else:
                cnt = int(counts[offsets[t] + e]) if e < len(luts[t]) else 0
                label = head + "table slot (%d, %d) of entry %d records multiplicity %d, but it is looked up %d times" % (
                    r, s, e, m, cnt)
        entries.append((r, s, label))
    return N.ConstraintReport(failures.value, entries)


def commit_quotient_polys(common_data, quotient_polys, ctx=None, *, blinding=False, salt_key=None, shard=(0, 1),
                          lde_blocks=None):
    """'split up quotient polys' + 'commit to quotient polys' (plonk/prover.rs:319-352): every polynomial is cut into
    quotient_degree_factor chunks of n coefficients (trim_to_len(quotient_degree) was checked by the kernel call), all
    chunks committed with from_coeffs -- straight from the device tensor compute_quotient_polys returned. With blinding
    the salt is drawn on the device from salt_key (PolynomialBatch._from_device). shard=(g, G): row block g of G only.
    lde_blocks=G: a non-resident batch."""
    cfg = common_data.config
    return PolynomialBatch._from_coeff_chunks(quotient_polys, common_data.quotient_degree_factor,
                                              common_data.degree_bits, cfg.rate_bits, cfg.cap_height, ctx,
                                              blinding=blinding, salt_key=salt_key, shard=shard, lde_blocks=lde_blocks)


# ------------------------------------------------------------------ prove (plonk/prover.rs:113-360)
class ProverOnlyCircuitData:
    """The fields of ProverOnlyCircuitData (plonk/circuit_data.rs:330-370) prove() reads: the constants/sigmas commitment
    (resident on the device since circuit build), the sigma value columns, the circuit digest, the FRI parameters."""

    def __init__(self, constants_sigmas_commitment, sigmas, circuit_digest, fri_params):
        self.constants_sigmas_commitment, self.sigmas = constants_sigmas_commitment, sigmas
        self.circuit_digest, self.fri_params = [int(x) for x in circuit_digest], fri_params


class VerifierOnlyCircuitData:
    """VerifierOnlyCircuitData (plonk/circuit_data.rs:372-380): the constants/sigmas Merkle cap and the circuit digest."""

    def __init__(self, constants_sigmas_cap, circuit_digest):
        self.constants_sigmas_cap, self.circuit_digest = constants_sigmas_cap, [int(x) for x in circuit_digest]


class CircuitData:
    """CircuitData (plonk/circuit_data.rs:150-160) as build_circuit_data returns it."""

    def __init__(self, common, prover_only, verifier_only):
        self.common, self.prover_only, self.verifier_only = common, prover_only, verifier_only


# ------------------------------------------------------------------ circuit build (plonk/circuit_builder.rs:911-1321)
def blind_and_pad(config, fri_config, instances):
    """CircuitBuilder::blind_and_pad (plonk/circuit_builder.rs:911-968) on the gate instances [(gate, constants)] the
    builder holds once every gate is placed. With config.zero_knowledge it appends the rows blinding_counts asks for:
    regular_poly_openings NoopGate rows, whose every wire the witness fills with a random value, then z_openings pairs
    of NoopGate rows, whose two rows carry one random value per routed wire. Then NoopGate rows pad to a power of two.
    Returns (instances, regular_rows, z_pairs): regular_rows a range of rows, z_pairs a list of (row_1, row_2).

    The reference ties a pair's two rows with generate_copy (a CopyGenerator of witness generation,
    circuit_builder.rs:507-510), not with connect, so the pairs add no copy constraint and their sigmas stay the
    identity; the copy constraints are unchanged."""
    out = list(instances)
    regular_rows, z_pairs = range(len(out), len(out)), []
    if config.zero_knowledge:
        regular, z_openings = blinding_counts(config, fri_config, len(out))
        regular_rows = range(len(out), len(out) + regular)
        out += [(NoopGate(), [])] * regular
        for _ in range(z_openings):
            z_pairs.append((len(out), len(out) + 1))
            out += [(NoopGate(), [])] * 2
    out += [(NoopGate(), [])] * ((1 << max(0, len(out) - 1).bit_length()) - len(out))
    return out, regular_rows, z_pairs


def target_indices(copy_constraints, num_wires, degree_bits):
    """Copy constraints in the degree-independent encoding -- wire (row, col) -> row * num_wires + col, virtual target
    i -> -(i + 1) -- as an (E, 2) uint64 array of Target::index values (iop/target.rs:55-60): virtual target i becomes
    n * num_wires + i. A wire index past the last row is refused (it would alias a virtual target)."""
    pairs = np.asarray(copy_constraints, dtype=np.int64).reshape(-1, 2)
    wires = num_wires << degree_bits
    if (pairs >= wires).any():
        raise N.ShapeError("copy constraint wire index %d is past the last of the %d rows"
                           % (int(pairs.max()), 1 << degree_bits))
    return np.ascontiguousarray(np.where(pairs >= 0, pairs, wires - 1 - pairs), dtype=np.uint64)


def sigma_polys(config, degree_bits, pairs, num_virtual_targets=0, ctx=None):
    """The sigma polynomials' values (CircuitBuilder::sigma_vecs, plonk/circuit_builder.rs:993-1028) on the device:
    gl_sigma_polys. pairs: the copy constraints' Target::index values, an (E, 2) host array or a CUDA int64 tensor on
    the context's device. Returns a (num_routed_wires, n) int64 CUDA tensor: row c is sigma column c."""
    import torch

    ctx = ctx or N.default_context()
    nr, n = config.num_routed_wires, 1 << degree_bits
    k_is = np.array(get_unique_coset_shifts(nr), dtype=np.uint64)
    if isinstance(pairs, torch.Tensor):
        host, n_pairs, ptr, mem = None, pairs.numel() // 2, N.vp(pairs.data_ptr()), N.MEM_DEVICE
    else:
        host = np.ascontiguousarray(pairs, dtype=np.uint64).reshape(-1, 2)
        n_pairs, mem = len(host), N.MEM_HOST
        ptr = N.np_ptr(host) if n_pairs else None
    out = torch.empty((nr, n), dtype=torch.int64, device="cuda:%d" % ctx.device)
    ctx.after_caller()
    N.check(N.lib().gl_sigma_polys(ctx.h, ptr, n_pairs, mem, config.num_wires, nr, degree_bits, int(num_virtual_targets),
                                   N.np_ptr(k_is), N.vp(out.data_ptr()), N.MEM_DEVICE), ctx.h)
    ctx.synchronize()  # the tensor goes to torch, whose stream is not the context's
    return out


def commit_constants_sigmas(common_data, constant_vecs, sigmas, ctx=None, shard=(0, 1), lde_blocks=None):
    """The constants/sigmas commitment (circuit_builder.rs:1177-1188, never blinded): the constant columns (host), then
    the sigma columns read in place from the device tensor sigma_polys returned. shard=(g, G): row block g of G.
    lde_blocks=G: a non-resident batch."""
    cfg = common_data.config
    ctx = ctx or N.default_context()
    consts = np.ascontiguousarray(np.stack(constant_vecs), dtype=np.uint64)
    n = 1 << common_data.degree_bits
    ctx.after_caller()

    def add_columns(h):
        N.check(N.lib().gl_commit_add_columns(h, 0, len(consts), N.np_ptr(consts), n, N.COLS_VALUES, N.MEM_HOST), ctx.h)
        N.check(N.lib().gl_commit_add_columns(h, len(consts), cfg.num_routed_wires, N.vp(sigmas.data_ptr()), n,
                                              N.COLS_VALUES, N.MEM_DEVICE), ctx.h)

    return PolynomialBatch._from_device(ctx, len(consts) + cfg.num_routed_wires, common_data.degree_bits, cfg.rate_bits,
                                        cfg.cap_height, add_columns, shard=shard, lde_blocks=lde_blocks)


def circuit_digest(constants_sigmas_cap, domain_separator, degree_bits):
    """The circuit digest (circuit_builder.rs:1252-1264): hash_no_pad(cap.flatten() || hash_pad(domain_separator) ||
    [degree_bits]), on the host permutation."""
    from .hash import PoseidonHash

    cap = getattr(constants_sigmas_cap, "hashes", constants_sigmas_cap)
    separator = PoseidonHash.hash_pad_host([int(x) % F.ORDER for x in domain_separator])
    parts = [int(x) for x in np.asarray(cap, dtype=np.uint64).reshape(-1)] + [int(x) for x in separator] + [degree_bits]
    return [int(x) for x in PoseidonHash.hash_no_pad_host(parts)]


def build_circuit_data(config, fri_config, instances, copy_constraints, num_virtual_targets=0, luts=(), lookup_rows=(),
                       domain_separator=(), ctx=None, lde_blocks=None):
    """CircuitBuilder::build_with_options(true) (plonk/circuit_builder.rs:1061-1321) from the placed circuit on one
    device: `instances` already through blind_and_pad, the copy constraints as an (E, 2) array in target_indices'
    encoding, num_virtual_targets virtual targets. Returns CircuitData(common, prover_only, verifier_only), equal to the
    reference's: the sigma polynomials and the constants/sigmas commitment are computed on the device, the digest
    from the cap. prover_only.sigmas is the host (num_routed_wires, n) array prove_with_witness reads.
    distributed.build_circuit_data builds the same data with the commitment sharded over ranks. lde_blocks=G: the
    constants/sigmas commitment is non-resident (PolynomialBatch.from_values), as prove_with_witness(lde_blocks=G)
    needs it; its digest and cap are the resident commitment's."""
    from .stark import lde_placement

    return _build_circuit_data(config, fri_config, instances, copy_constraints, num_virtual_targets, luts, lookup_rows,
                               domain_separator, ctx, lde_placement(config.cap_height, lde_blocks))


def _build_circuit_data(config, fri_config, instances, copy_constraints, num_virtual_targets, luts, lookup_rows,
                        domain_separator, ctx, placement):
    """build_circuit_data on a distributed.Placement: the constants/sigmas commitment is this rank's row block, its cap
    the gathered full cap. The sigmas are computed on every rank."""
    degree_bits = F.log2_strict(len(instances))
    pairs = target_indices(copy_constraints, config.num_wires, degree_bits)
    fri_params = fri_config.fri_params(degree_bits, config.zero_knowledge)
    if fri_params.total_arities() > degree_bits + fri_config.rate_bits - fri_config.cap_height:
        raise N.ShapeError("FRI total reduction arity is too large.")
    common, constant_vecs = CommonCircuitData.from_gate_instances(config, instances, luts, lookup_rows)
    ctx = ctx or N.default_context()
    sigmas = sigma_polys(config, degree_bits, pairs, num_virtual_targets, ctx)
    commitment = commit_constants_sigmas(common, constant_vecs, sigmas, ctx, **placement.commit_kwargs)
    try:
        host_sigmas = sigmas.cpu().numpy().view(np.uint64)
        del sigmas
        cap = placement.cap(commitment)
        digest = circuit_digest(cap, domain_separator, degree_bits)
    except Exception:
        commitment.close()
        raise
    return CircuitData(common, ProverOnlyCircuitData(commitment, host_sigmas, digest, fri_params),
                       VerifierOnlyCircuitData(cap, digest))


def _le_words(arr):
    return np.ascontiguousarray(arr, dtype="<u8").tobytes()


class Proof:
    """Proof<F, C, D> (plonk/proof.rs:26-40)."""

    def __init__(self, wires_cap, plonk_zs_partial_products_cap, quotient_polys_cap, openings, opening_proof):
        self.wires_cap, self.plonk_zs_partial_products_cap = wires_cap, plonk_zs_partial_products_cap
        self.quotient_polys_cap, self.openings, self.opening_proof = quotient_polys_cap, openings, opening_proof

    def to_bytes(self):
        """write_proof (util/serialization/mod.rs:1977-1987) with write_opening_set (:1436-1449)."""
        o = self.openings
        out = _le_words(self.wires_cap.hashes) + _le_words(self.plonk_zs_partial_products_cap.hashes)
        out += _le_words(self.quotient_polys_cap.hashes)
        for part in (o.constants, o.plonk_sigmas, o.wires, o.plonk_zs, o.plonk_zs_next, o.lookup_zs, o.lookup_zs_next,
                     o.partial_products, o.quotient_polys):
            out += _le_words(part)
        return out + self.opening_proof.to_bytes()


    def compress(self, indices, params):
        """Proof::compress (plonk/proof.rs:56-76)."""
        return CompressedProof(self.wires_cap, self.plonk_zs_partial_products_cap, self.quotient_polys_cap, self.openings,
                               self.opening_proof.compress(indices, params))

    @classmethod
    def from_bytes(cls, buf, common_data, fri_params, offset=0):
        """read_proof (util/serialization/mod.rs: read_merkle_cap x3, read_opening_set, read_fri_proof). Returns
        (Proof, next offset)."""
        from .fri import FriProof
        from .hash import MerkleCap
        from .proof import OpeningSet

        cd, cfg = common_data, common_data.config
        nc = cfg.num_challenges
        pos = offset

        def words(count, shape):
            nonlocal pos
            a = np.frombuffer(buf, dtype="<u8", count=count, offset=pos).astype(np.uint64).reshape(shape)
            pos += 8 * count
            return a

        cap_len = 1 << cfg.cap_height
        caps = [MerkleCap(words(4 * cap_len, (cap_len, 4))) for _ in range(3)]

        def ext_vec(k):
            return words(2 * k, (k, 2))

        n_lookup = nc * cd.num_lookup_polys
        constants, sigmas, wires = ext_vec(cd.num_constants), ext_vec(cfg.num_routed_wires), ext_vec(cfg.num_wires)
        zs, zs_next, lk, lk_next = ext_vec(nc), ext_vec(nc), ext_vec(n_lookup), ext_vec(n_lookup)
        pps, quot = ext_vec(nc * cd.num_partial_products), ext_vec(nc * cd.quotient_degree_factor)
        openings = OpeningSet(constants=constants, plonk_sigmas=sigmas, wires=wires, plonk_zs=zs, plonk_zs_next=zs_next,
                              partial_products=pps, quotient_polys=quot, lookup_zs=lk, lookup_zs_next=lk_next)
        salt = SALT_SIZE if fri_params.hiding else 0          # salt_size(hiding): the salted oracles' leaves
        widths = [cd.num_constants + cfg.num_routed_wires, cfg.num_wires + salt,
                  nc * (1 + cd.num_partial_products + cd.num_lookup_polys) + salt, nc * cd.quotient_degree_factor + salt]
        fri, pos = FriProof.from_bytes(buf, widths, fri_params, pos)
        return cls(caps[0], caps[1], caps[2], openings, fri), pos


class CompressedProof(Proof):
    """CompressedProof (plonk/proof.rs:128-141): a Proof whose opening_proof is a CompressedFriProof; to_bytes =
    write_compressed_proof (util/serialization/mod.rs:2080-2093)."""


class ProofWithPublicInputs:
    """ProofWithPublicInputs (plonk/proof.rs:82-88)."""

    def __init__(self, proof, public_inputs):
        self.proof, self.public_inputs = proof, [int(x) % F.ORDER for x in public_inputs]

    def to_bytes(self):
        """write_proof_with_public_inputs (util/serialization/mod.rs:2001-2015)."""
        pis = np.array(self.public_inputs, dtype=np.uint64)
        return self.proof.to_bytes() + _le_words(np.array([len(pis)], dtype=np.uint64)) + _le_words(pis)

    @classmethod
    def from_bytes(cls, buf, common_data, fri_params):
        """read_proof_with_public_inputs (util/serialization/mod.rs)."""
        proof, pos = Proof.from_bytes(buf, common_data, fri_params)
        n = int(np.frombuffer(buf, dtype="<u8", count=1, offset=pos)[0])
        pis = np.frombuffer(buf, dtype="<u8", count=n, offset=pos + 8)
        if pos + 8 + 8 * n != len(buf):
            raise N.ShapeError("trailing bytes after the proof")
        return cls(proof, [int(x) for x in pis])

    def get_public_inputs_hash(self):
        from .hash import PoseidonHash

        return [int(x) for x in PoseidonHash.hash_no_pad_host(self.public_inputs)]

    def get_challenges(self, circuit_digest, common_data, fri_params):
        """get_challenges (plonk/get_challenges.rs:26-90): the transcript replayed on the host from the proof alone."""
        from .challenger import Challenger
        from .fri import fri_challenges

        cd, p = common_data, self.proof
        nc = cd.config.num_challenges
        ch = Challenger()
        fri_params.observe(ch)
        ch.observe_hash(circuit_digest)
        ch.observe_hash(self.get_public_inputs_hash())
        ch.observe_cap(p.wires_cap)
        betas, gammas = ch.get_n_challenges(nc), ch.get_n_challenges(nc)
        deltas = (betas + gammas + ch.get_n_challenges(NUM_COINS_LOOKUP * nc - 2 * nc)) if cd.num_lookup_polys else []
        ch.observe_cap(p.plonk_zs_partial_products_cap)
        alphas = ch.get_n_challenges(nc)
        ch.observe_cap(p.quotient_polys_cap)
        zeta = ch.get_extension_challenge()
        for batch in p.openings.to_fri_openings():
            ch.observe_elements(batch.reshape(-1))
        fp = p.opening_proof
        fri_alpha, fri_betas, fri_pow_response, indices = fri_challenges(ch, fp.commit_phase_merkle_caps, fp.final_poly,
                                                                         fp.pow_witness, cd.degree_bits, fri_params.config)
        return dict(plonk_betas=betas, plonk_gammas=gammas, plonk_deltas=deltas, plonk_alphas=alphas, plonk_zeta=zeta,
                    fri_alpha=fri_alpha, fri_betas=fri_betas, fri_pow_response=fri_pow_response, fri_query_indices=indices)

    def fri_query_indices(self, circuit_digest, common_data, fri_params):
        return self.get_challenges(circuit_digest, common_data, fri_params)["fri_query_indices"]

    def compress(self, circuit_digest, common_data, fri_params):
        """ProofWithPublicInputs::compress (plonk/proof.rs:93-104)."""
        indices = self.fri_query_indices(circuit_digest, common_data, fri_params)
        return CompressedProofWithPublicInputs(self.proof.compress(indices, fri_params), self.public_inputs)


class CompressedProofWithPublicInputs(ProofWithPublicInputs):
    """CompressedProofWithPublicInputs (plonk/proof.rs:163-170)."""

    def to_bytes(self):
        """write_compressed_proof_with_public_inputs (util/serialization/mod.rs:2097-2111): the public inputs follow
        without a length."""
        return self.proof.to_bytes() + _le_words(np.array(self.public_inputs, dtype=np.uint64))


def get_fri_instance(cd, zeta):
    """CommonCircuitData::get_fri_instance (plonk/circuit_data.rs:530-660): every polynomial at zeta, the Z's and the
    lookup polynomials also at g * zeta. The wires, Z / partial-product and quotient oracles are blinded in a
    zero-knowledge circuit (fri_oracles, :575-600); the constants / sigmas never are."""
    from .fri import FriBatchInfo, FriInstanceInfo, FriOracleInfo, FriPolynomialInfo

    cfg = cd.config
    nc = cfg.num_challenges
    n_pre = cd.num_constants + cfg.num_routed_wires                                   # num_preprocessed_polys
    n_zs_pp, n_lookup = cd.num_zs_partial_products_polys(), nc * cd.num_lookup_polys
    n_quot = nc * cd.quotient_degree_factor
    lookup = FriPolynomialInfo.from_range(2, range(n_zs_pp, n_zs_pp + n_lookup))
    all_polys = (FriPolynomialInfo.from_range(0, range(n_pre)) + FriPolynomialInfo.from_range(1, range(cfg.num_wires))
                 + FriPolynomialInfo.from_range(2, range(n_zs_pp)) + FriPolynomialInfo.from_range(3, range(n_quot)) + lookup)
    g = F.primitive_root_of_unity(cd.degree_bits)
    zeta_next = F.ext_mul((g, 0), zeta)
    zk = cfg.zero_knowledge
    oracles = [FriOracleInfo(n_pre, False), FriOracleInfo(cfg.num_wires, zk), FriOracleInfo(n_zs_pp + n_lookup, zk),
               FriOracleInfo(n_quot, zk)]
    return FriInstanceInfo(oracles, [FriBatchInfo(zeta, all_polys),
                                     FriBatchInfo(zeta_next, FriPolynomialInfo.from_range(2, range(nc)) + lookup)])


def _to_device(columns, ctx):
    """Host value columns -> torch int64 tensor on the context's GPU (the layout gl_partial_products_and_zs reads)."""
    import torch

    dev = "cuda:%d" % ctx.device
    t = torch.from_numpy(np.ascontiguousarray(columns, dtype=np.uint64).view(np.int64)).to(dev)
    torch.cuda.synchronize(dev)
    return t


def prove_with_witness(prover_data, common_data, wires, public_inputs, ctx=None, *, salt_keys=None,
                       check_constraints=False, lde_blocks=None):
    """prove_with_partition_witness (plonk/prover.rs:132-360) from the full witness matrix `wires` (num_wires, n) -- the
    generators' output -- to ProofWithPublicInputs, every array-sized step on the device: wires commitment, Z / partial
    products (+ lookup) commitment, quotient polynomials from the LDEs in place and their commitment, the openings at
    zeta and g zeta, the FRI opening proof. The transcript runs on the host exactly as in the reference.

    With config.zero_knowledge the wires, Z / partial-product (+ lookup) and quotient commitments are salted, as
    prover.rs:179,249,297 do (the constants / sigmas commitment never is), and prover_data.fri_params.hiding must be set.
    The salt is drawn on the device: salt_keys = three 32-byte keys (wires, Z's, quotient) give a reproducible proof;
    None draws a fresh key from the OS CSPRNG per commitment. The blinding rows of the circuit (blinding_counts) are part
    of the witness, which the caller generates.

    check_constraints=True: after the Z / partial-product commitment, before the quotient, every term of the vanishing
    polynomial is checked on every row of H with the proof's own challenges (check_constraints), and a failure raises
    ConstraintError naming the row and the term; the proof is unchanged. With lde_blocks=G the check runs in G parts
    of H, one after another, with the same message and report.

    lde_blocks=G: the wires, Z / partial-product (+ lookup) and quotient commitments are non-resident
    (PolynomialBatch.from_values), for circuits whose LDEs exceed device memory; prover_data must come from
    build_circuit_data(..., lde_blocks=G). The quotient is evaluated in G parts of its coset and every LDE block is
    rebuilt from the coefficients where it is hashed or read; the proof is the same. Refused with ShapeError before any
    device work: check_lde_blocks' refusals, G above the quotient coset's points, a constants/sigmas commitment that is
    resident or of another G, and a zero-knowledge config (a non-resident batch cannot be blinded)."""
    from .stark import lde_placement

    placement = lde_placement(common_data.config.cap_height, lde_blocks)
    if lde_blocks is not None:
        _check_lde_blocks(prover_data, common_data, placement.lde_blocks)
    return _prove(prover_data, common_data, wires, public_inputs, ctx, placement, salt_keys, check_constraints)


def _check_lde_blocks(prover_data, common_data, G):
    """prove_with_witness's refusals of lde_blocks=G beyond check_lde_blocks'."""
    if common_data.config.zero_knowledge:
        raise N.ShapeError("lde_blocks= cannot prove with zero knowledge: a non-resident batch cannot be blinded")
    size = (1 << common_data.degree_bits) << (common_data.quotient_degree_factor - 1).bit_length()
    if G > size:
        raise N.ShapeError("lde_blocks=%d exceeds the %d points of the quotient coset" % (G, size))
    cs_blocks = prover_data.constants_sigmas_commitment.lde_blocks
    if cs_blocks != G:
        raise N.ShapeError("lde_blocks=%d, but the constants/sigmas commitment is %s: build it with "
                           "build_circuit_data(..., lde_blocks=%d)"
                           % (G, "non-resident in %d blocks" % cs_blocks if cs_blocks else "resident", G))


def _prove(prover_data, common_data, wires, public_inputs, ctx, placement, salt_keys=None, check_constraints=False):
    """prove_with_witness on a distributed.Placement. With G > 1 ranks this one holds row block g of the wires,
    Z / partial-product (+ lookup) and quotient commitments, and prover_data.constants_sigmas_commitment is that shard
    too: the caps are all-gathered before they are observed, the quotient is evaluated shard by shard and all-gathered,
    each rank sums its block of the coefficients into the openings and the ranks add up the partial sums, and FRI routes
    the query openings between the ranks. The Z's, partial products and lookup columns and the transcript run on every
    rank, so every rank returns the same proof. check_constraints runs with placement.check_kwargs: each rank checks its
    own part of H and every rank raises the same ConstraintError."""
    from .challenger import Challenger
    from .fri import prove_openings
    from .hash import PoseidonHash
    from .proof import OpeningSet
    from .prover import commit_zs_partial_products, compute_all_lookup_polys, wires_permutation_partial_products_and_zs

    ctx = ctx or N.default_context()
    cd, cfg = common_data, common_data.config
    nc, nr = cfg.num_challenges, cfg.num_routed_wires
    has_lookup = bool(cd.luts)
    wires = np.ascontiguousarray(wires, dtype=np.uint64)
    if wires.shape != (cfg.num_wires, 1 << cd.degree_bits):
        raise N.ShapeError("the witness must be (num_wires, n)")
    zk = cfg.zero_knowledge
    if bool(prover_data.fri_params.hiding) != zk:
        raise N.ShapeError("fri_params.hiding (%s) must equal config.zero_knowledge (%s)"
                           % (bool(prover_data.fri_params.hiding), zk))
    if salt_keys is not None and (not zk or len(salt_keys) != 3):
        raise N.ShapeError("salt_keys: three 32-byte keys (wires, Z's, quotient), for a zero-knowledge config only")
    # keyword arguments of the three salted commitments (none without zero knowledge)
    salted = [dict(salt_key=salt_keys[i] if salt_keys is not None else "fresh") if zk else {} for i in range(3)]
    public_inputs_hash = [int(x) for x in PoseidonHash.hash_no_pad(np.array(public_inputs, dtype=np.uint64), ctx)]
    on = placement.commit_kwargs
    wires_commitment = PolynomialBatch.from_values(wires, cfg.rate_bits, zk, cfg.cap_height, ctx=ctx, **salted[0], **on)
    commitments = [wires_commitment]
    try:
        challenger = Challenger()
        prover_data.fri_params.observe(challenger)                     # observe the FRI config
        challenger.observe_hash(prover_data.circuit_digest)            # observe the instance
        challenger.observe_hash(public_inputs_hash)
        wires_cap = placement.cap(wires_commitment)
        challenger.observe_cap(wires_cap)
        betas = challenger.get_n_challenges(nc)
        gammas = challenger.get_n_challenges(nc)
        deltas = (betas + gammas + challenger.get_n_challenges(NUM_COINS_LOOKUP * nc - 2 * nc)) if has_lookup else []
        if cd.quotient_degree_factor >= nr:
            raise N.ShapeError("When the number of routed wires is smaller that the degree, we should change the logic to "
                               "avoid computing partial products.")
        if has_lookup:
            # Z's, partial products and the RE / Sum / LDC columns are committed together (prover.rs:227-262)
            zs, pps = [], []
            for beta, gamma in zip(betas, gammas):
                out = wires_permutation_partial_products_and_zs(wires[:nr], prover_data.sigmas, cd.k_is, beta, gamma,
                                                                cd.quotient_degree_factor, ctx)
                zs.append(out[-1])
                pps += list(out[:-1])
            lookup_polys = compute_all_lookup_polys(wires, nr, cfg.max_quotient_degree_factor, deltas, cd.lookup_rows, nc, ctx)
            zs_commitment = PolynomialBatch.from_values(np.concatenate([np.stack(zs + pps), lookup_polys]), cfg.rate_bits,
                                                        zk, cfg.cap_height, ctx=ctx, **salted[1], **on)
        else:
            wires_dev, sigmas_dev = _to_device(wires[:nr], ctx), _to_device(prover_data.sigmas, ctx)
            zs_commitment = commit_zs_partial_products(wires_dev, sigmas_dev, cd.k_is, betas, gammas,
                                                       cd.quotient_degree_factor, cfg.rate_bits, cfg.cap_height, ctx,
                                                       **(dict(blinding=True, **salted[1]) if zk else {}), **on)
        commitments.append(zs_commitment)
        zs_cap = placement.cap(zs_commitment)
        challenger.observe_cap(zs_cap)
        alphas = challenger.get_n_challenges(nc)
        cs = prover_data.constants_sigmas_commitment
        if check_constraints:
            _raise_on_failure(cd, cs, public_inputs_hash, wires_commitment, zs_commitment, betas, gammas, deltas,
                              **placement.check_kwargs)
        quotient_polys = compute_quotient_polys(cd, cs, public_inputs_hash, wires_commitment, zs_commitment, betas,
                                                gammas, alphas, deltas, **placement.step_kwargs)
        quotient_commitment = commit_quotient_polys(cd, quotient_polys, ctx,
                                                    **(dict(blinding=True, **salted[2]) if zk else {}), **on)
        commitments.append(quotient_commitment)
        del quotient_polys
        quotient_cap = placement.cap(quotient_commitment)
        challenger.observe_cap(quotient_cap)
        zeta = challenger.get_extension_challenge()
        g = F.primitive_root_of_unity(cd.degree_bits)
        if F.ext_pow(zeta, 1 << cd.degree_bits) == (1, 0):
            raise N.NativeError("Opening point is in the subgroup.")
        n_zs_pp = cd.num_zs_partial_products_polys()
        openings = OpeningSet.new(zeta, g, cs, wires_commitment, zs_commitment, quotient_commitment,
                                  constants_range=cd.constants_range(), sigmas_range=cd.sigmas_range(), zs_range=cd.zs_range(),
                                  partial_products_range=cd.partial_products_range(),
                                  lookup_range=range(n_zs_pp, n_zs_pp + nc * cd.num_lookup_polys),
                                  **placement.step_kwargs)
        for batch in openings.to_fri_openings():                       # Challenger::observe_openings
            challenger.observe_elements(batch.reshape(-1))
        oracles = [cs, wires_commitment, zs_commitment, quotient_commitment]
        opening_proof = prove_openings(get_fri_instance(cd, zeta), oracles, challenger, prover_data.fri_params,
                                       **placement.step_kwargs)
        proof = Proof(wires_cap, zs_cap, quotient_cap, openings, opening_proof)
        return ProofWithPublicInputs(proof, public_inputs)
    finally:
        for c in commitments:
            c.close()
