"""starky's prover path adjacent to the commitment kernels (SURVEY.md section 8f row 1): Stark constraints, the quotient
polynomials and their commitment, mirroring starky/src/{stark.rs, constraint_consumer.rs, prover.rs:391-421,488-668,
fibonacci_stark.rs}. The constraints of a Stark are recorded ONCE as a straight-line program (ConstraintBuilder) and
evaluated by gl_stark_quotient on every point of the quotient coset, reading the trace LDE in place on the device."""
import ctypes as C

import numpy as np

from . import _native as N
from . import field as F
from .polynomial_batch import PolynomialBatch

OP_LOCAL, OP_NEXT, OP_CONST, OP_ADD, OP_SUB, OP_MUL, OP_EMIT = range(7)
KIND_CONSTRAINT, KIND_TRANSITION, KIND_FIRST_ROW, KIND_LAST_ROW = range(4)


class StarkInstr(C.Structure):
    _fields_ = [("op", C.c_uint16), ("a", C.c_uint16), ("b", C.c_uint16), ("pad_", C.c_uint16)]


class Expr:
    """A value of the constraint program (the P: PackedField of eval_packed_generic)."""

    def __init__(self, b, idx):
        self.b, self.idx = b, idx

    def _bin(self, op, other):
        other = other if isinstance(other, Expr) else self.b.constant(other)
        return self.b._push(op, self.idx, other.idx)

    def __add__(self, o):
        return self._bin(OP_ADD, o)

    def __sub__(self, o):
        return self._bin(OP_SUB, o)

    def __mul__(self, o):
        return self._bin(OP_MUL, o)

    __radd__, __rmul__ = __add__, __mul__


class ConstraintBuilder:
    """Records eval_packed_generic as instructions; doubles as the ConstraintConsumer (constraint_consumer.rs:46-84)."""

    def __init__(self, num_columns, num_public_inputs):
        self.instrs, self.consts = [], [None] * num_public_inputs  # consts[0:num_pi] are bound at evaluation time
        self.num_columns, self.num_pi = num_columns, num_public_inputs
        self._cache = {}

    def _push(self, op, a=0, b=0):
        key = (op, a, b)
        if op != OP_EMIT and key in self._cache:
            return self._cache[key]
        self.instrs.append((op, a, b))
        e = Expr(self, len(self.instrs) - 1)
        if op != OP_EMIT:
            self._cache[key] = e
        return e

    # StarkEvaluationFrame (evaluation_frame.rs:12-40)
    def local(self, col):
        assert 0 <= col < self.num_columns
        return self._push(OP_LOCAL, col)

    def next(self, col):
        assert 0 <= col < self.num_columns
        return self._push(OP_NEXT, col)

    def public_input(self, k):
        assert 0 <= k < self.num_pi
        return self._push(OP_CONST, k)

    def constant(self, v):
        v = int(v) % F.ORDER
        if v not in self.consts[self.num_pi:]:
            self.consts.append(v)
        return self._push(OP_CONST, self.num_pi + self.consts[self.num_pi:].index(v))

    # ConstraintConsumer
    def constraint(self, e):
        self._push(OP_EMIT, e.idx, KIND_CONSTRAINT)

    def constraint_transition(self, e):
        self._push(OP_EMIT, e.idx, KIND_TRANSITION)

    def constraint_first_row(self, e):
        self._push(OP_EMIT, e.idx, KIND_FIRST_ROW)

    def constraint_last_row(self, e):
        self._push(OP_EMIT, e.idx, KIND_LAST_ROW)

    def program(self):
        arr = (StarkInstr * len(self.instrs))()
        for i, (op, a, b) in enumerate(self.instrs):
            arr[i].op, arr[i].a, arr[i].b = op, a, b
        return arr


class Stark:
    """Stark<F, D> (starky/src/stark.rs:24-120): COLUMNS, PUBLIC_INPUTS, eval (eval_packed_generic), constraint_degree."""
    COLUMNS = 0
    PUBLIC_INPUTS = 0

    def eval(self, vars, yield_constr):
        raise NotImplementedError

    def constraint_degree(self):
        raise NotImplementedError

    def quotient_degree_factor(self):
        """stark.rs:87-92"""
        d = self.constraint_degree()
        return 0 if d == 0 else max(1, d - 1)

    def constraint_program(self):
        b = ConstraintBuilder(self.COLUMNS, self.PUBLIC_INPUTS)
        self.eval(b, b)
        return b


class FibonacciStark(Stark):
    """FibonacciStark (starky/src/fibonacci_stark.rs:19-120): columns (x0, x1), x0' = x1, x1' = x0 + x1; public inputs
    x0, x1 of the first row and x1 of the last row."""
    COLUMNS = 2
    PUBLIC_INPUTS = 3
    PI_INDEX_X0, PI_INDEX_X1, PI_INDEX_RES = 0, 1, 2

    def __init__(self, num_rows):
        self.num_rows = num_rows

    def generate_trace(self, x0, x1):
        """generate_trace (fibonacci_stark.rs:42-53): two columns of num_rows values."""
        cols = np.empty((2, self.num_rows), dtype=np.uint64)
        a, b = int(x0) % F.ORDER, int(x1) % F.ORDER
        for i in range(self.num_rows):
            cols[0, i], cols[1, i] = a, b
            a, b = b, (a + b) % F.ORDER
        return cols

    def eval(self, vars, yield_constr):
        """eval_packed_generic (fibonacci_stark.rs:73-95)."""
        l0, l1, n0, n1 = vars.local(0), vars.local(1), vars.next(0), vars.next(1)
        yield_constr.constraint_first_row(l0 - vars.public_input(self.PI_INDEX_X0))
        yield_constr.constraint_first_row(l1 - vars.public_input(self.PI_INDEX_X1))
        yield_constr.constraint_last_row(l1 - vars.public_input(self.PI_INDEX_RES))
        yield_constr.constraint_transition(n0 - l1)           # x0' <- x1
        yield_constr.constraint_transition(n1 - l0 - l1)      # x1' <- x0 + x1

    def constraint_degree(self):
        return 2


def compute_quotient_polys(stark, trace_commitment, public_inputs, alphas):
    """compute_quotient_polys (prover.rs:488-668) on the device. Returns a torch int64 CUDA tensor (num_challenges, size)
    of quotient-polynomial coefficients, size = n << log2_ceil(quotient_degree_factor), or None if the Stark has no
    quotient. Raises if the vanishing polynomial is not divisible by Z_H."""
    import torch

    qdf = stark.quotient_degree_factor()
    if qdf == 0:
        return None
    b = stark.constraint_program()
    consts = np.array([int(x) % F.ORDER for x in public_inputs] + b.consts[b.num_pi:], dtype=np.uint64)
    if len(public_inputs) != stark.PUBLIC_INPUTS:
        raise N.ShapeError("expected %d public inputs" % stark.PUBLIC_INPUTS)
    al = np.array([int(a) % F.ORDER for a in alphas], dtype=np.uint64)
    qd_bits = (qdf - 1).bit_length()
    size = (1 << trace_commitment.degree_log) << qd_bits
    ctx = trace_commitment.ctx
    out = torch.empty((len(al), size), dtype=torch.int64, device="cuda:%d" % ctx.device)
    prog = b.program()
    N.check(N.lib().gl_stark_quotient(ctx.h, trace_commitment.h, prog, len(b.instrs), N.np_ptr(consts), len(consts),
                                      N.np_ptr(al), len(al), qdf, N.vp(out.data_ptr())), ctx.h)
    ctx.synchronize()
    return out


def commit_quotient_polys(stark, quotient_polys, degree_bits, rate_bits, cap_height, ctx=None):
    """'split quotient polys' + 'compute quotient commitment' (prover.rs:391-421): every polynomial is cut into
    quotient_degree_factor chunks of n coefficients, all chunks are committed with from_coeffs -- straight from the
    device tensor compute_quotient_polys returned."""
    return PolynomialBatch._from_coeff_chunks(quotient_polys, stark.quotient_degree_factor(), degree_bits, rate_bits,
                                              cap_height, ctx)
