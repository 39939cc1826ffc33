"""starky's prover (SURVEY.md section 8f rows 1 and 1'), mirroring starky/src/{config.rs, stark.rs,
constraint_consumer.rs, vanishing_poly.rs, prover.rs, proof.rs, get_challenges.rs, fibonacci_stark.rs} for STARKs
with or without logUp lookups (lookup.py) and cross-table lookups (cross_table_lookup.py). The constraints of a Stark --
its own, then those of its lookups, then those of its CTLs -- are recorded ONCE as a straight-line program
(ConstraintBuilder): gl_stark_quotient[_aux] evaluates it on every point of the quotient coset, reading the trace and
auxiliary LDEs in place on the device, and eval_vanishing_poly evaluates the same instructions at one point of F_{p^2}
on the host (the constraint-binding step of the prover, and any verifier). `prove` (one STARK) and
cross_table_lookup.prove_with_ctls (several) both run prove_with_commitment, which strings the device steps together in
the reference's order with the transcript on the host; the lookup helper columns are written on the device by
gl_stark_lookup_helpers, the CTL helper and Z columns by gl_stark_ctl_helpers. distributed.prove_stark runs the same
prove_with_commitment on row-block shards over several GPUs (its distributed.Placement)."""
import ctypes as C

import numpy as np

from . import _native as N
from . import distributed as D
from . import field as F
from .fri import starky_standard_fast_fri_config
from .polynomial_batch import PolynomialBatch, check_lde_blocks
from .proof import StarkOpeningSet

OP_LOCAL, OP_NEXT, OP_CONST, OP_ADD, OP_SUB, OP_MUL, OP_EMIT, OP_AUX_LOCAL, OP_AUX_NEXT = range(9)
KIND_CONSTRAINT, KIND_TRANSITION, KIND_FIRST_ROW, KIND_LAST_ROW = range(4)
KIND_NAMES = ("every row", "transition", "first row", "last row")


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

    def __init__(self, num_columns, num_public_inputs, num_aux=0, num_lookup_challenges=0, num_ctl_vars=0):
        # consts[0:num_bound] -- the public inputs, the lookup challenges, then each CTL Z's (beta, gamma) -- are bound
        # at evaluation time
        self.num_lookup_challenges = num_lookup_challenges
        self.num_bound = num_public_inputs + num_lookup_challenges + 2 * num_ctl_vars
        self.instrs, self.consts = [], [None] * self.num_bound
        self.num_columns, self.num_pi, self.num_aux = num_columns, num_public_inputs, num_aux
        self._cache = {}
        # what check_constraints names each EMIT by: the Stark's own constraints are numbered in emission order, the
        # lookup and CTL recorders open a scope of their own (begin_scope) whose checks are numbered from 0
        self.labels, self._scope, self._scope_count = [], "constraint", 0

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

    # the auxiliary polynomials (LookupCheckVars, lookup.rs:791-801)
    def aux_local(self, col):
        assert 0 <= col < self.num_aux
        return self._push(OP_AUX_LOCAL, col)

    def aux_next(self, col):
        assert 0 <= col < self.num_aux
        return self._push(OP_AUX_NEXT, col)

    def lookup_challenge(self, c):
        assert 0 <= c < self.num_lookup_challenges
        return self._push(OP_CONST, self.num_pi + c)

    def ctl_challenge(self, k):
        """(beta, gamma) of the program's k-th CTL Z polynomial."""
        base = self.num_pi + self.num_lookup_challenges + 2 * k
        assert base + 2 <= self.num_bound
        return self._push(OP_CONST, base), self._push(OP_CONST, base + 1)

    def constant(self, v):
        v = int(v) % F.ORDER
        if v not in self.consts[self.num_bound:]:
            self.consts.append(v)
        return self._push(OP_CONST, self.num_bound + self.consts[self.num_bound:].index(v))

    def begin_scope(self, name):
        """Label the EMITs that follow as checks 0, 1, ... of `name` (a lookup's challenge, a CTL Z)."""
        self._scope, self._scope_count = name + ", check", 0

    # ConstraintConsumer
    def _emit(self, e, kind):
        self._push(OP_EMIT, e.idx, kind)
        self.labels.append("%s %d (%s)" % (self._scope, self._scope_count, KIND_NAMES[kind]))
        self._scope_count += 1

    def constraint(self, e):
        self._emit(e, KIND_CONSTRAINT)

    def constraint_transition(self, e):
        self._emit(e, KIND_TRANSITION)

    def constraint_first_row(self, e):
        self._emit(e, KIND_FIRST_ROW)

    def constraint_last_row(self, e):
        self._emit(e, KIND_LAST_ROW)

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

    def lookups(self):
        """stark.rs:251-254: the Stark's logUp lookups (lookup.Lookup), none by default."""
        return []

    def uses_lookups(self):
        """stark.rs:266-270"""
        return len(self.lookups()) > 0

    def num_lookup_helper_columns(self, config):
        """stark.rs:256-264: the auxiliary polynomials of all lookups and challenges."""
        return self._helper_columns_per_challenge() * config.num_challenges

    def _helper_columns_per_challenge(self):
        return sum(lookup.num_helper_columns(self.constraint_degree()) for lookup in self.lookups())

    def requires_ctls(self):
        """stark.rs:272-278: whether the Stark takes part in cross-table lookups; False by default."""
        return False

    def constraint_program(self, num_lookup_challenges=0, ctl_vars=None):
        """The Stark's constraints (eval_packed_generic), then -- with lookups -- those of the logUp argument for
        num_lookup_challenges challenges, then -- with ctl_vars (CtlCheckVars; only their shape is read) -- those of
        its cross-table lookups (eval_vanishing_poly, vanishing_poly.rs:41-61): the order of the alpha-fold. The
        auxiliary columns are [lookup helpers | CTL helpers | CTL Zs]."""
        if not self.uses_lookups() and ctl_vars is None:
            b = ConstraintBuilder(self.COLUMNS, self.PUBLIC_INPUTS)
            self.eval(b, b)
            return b
        from .lookup import eval_packed_lookups_generic

        nl = self._helper_columns_per_challenge() * num_lookup_challenges if self.uses_lookups() else 0
        ctl_vars = ctl_vars or []
        num_ctl = sum(len(v.helper_columns) for v in ctl_vars) + len(ctl_vars)
        b = ConstraintBuilder(self.COLUMNS, self.PUBLIC_INPUTS, nl + num_ctl,
                              num_lookup_challenges if self.uses_lookups() else 0, len(ctl_vars))
        self.eval(b, b)
        if self.uses_lookups():
            eval_packed_lookups_generic(self, self.lookups(), b, num_lookup_challenges, b)
        if ctl_vars:
            from .cross_table_lookup import eval_cross_table_lookup_checks

            eval_cross_table_lookup_checks(b, ctl_vars, b, self.constraint_degree(), nl)
        return b

    def num_quotient_polys(self, config):
        """stark.rs:95-98"""
        return self.quotient_degree_factor() * config.num_challenges

    def fri_instance(self, zeta, g, config, num_ctl_helpers=0, num_ctl_zs=0):
        """fri_instance (stark.rs:101-170): the trace oracle and -- with lookups or CTLs -- the auxiliary oracle opened
        at zeta and g * zeta, the quotient oracle -- present only when the Stark has constraints -- at zeta, and -- with
        CTLs -- the auxiliary oracle's CTL Z columns at 1."""
        from .fri import FriBatchInfo, FriInstanceInfo, FriOracleInfo, FriPolynomialInfo

        trace_info = FriPolynomialInfo.from_range(0, range(self.COLUMNS))
        oracles = [FriOracleInfo(self.COLUMNS, False)]
        nl = self.num_lookup_helper_columns(config) if self.uses_lookups() else 0
        if self.uses_lookups() or self.requires_ctls():
            num_aux = nl + num_ctl_helpers + num_ctl_zs
            trace_info = trace_info + FriPolynomialInfo.from_range(len(oracles), range(num_aux))
            oracles.append(FriOracleInfo(num_aux, False))
        quotient_info = []
        nq = self.num_quotient_polys(config)
        if nq > 0:
            quotient_info = FriPolynomialInfo.from_range(len(oracles), range(nq))
            oracles.append(FriOracleInfo(nq, False))
        zeta_next = F.ext_mul((int(g) % F.ORDER, 0), zeta)
        batches = [FriBatchInfo(zeta, trace_info + quotient_info), FriBatchInfo(zeta_next, trace_info)]
        if self.requires_ctls():
            batches.append(FriBatchInfo((1, 0), FriPolynomialInfo.from_range(
                1, range(nl + num_ctl_helpers, nl + num_ctl_helpers + num_ctl_zs))))
        return FriInstanceInfo(oracles, batches)


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


def compute_quotient_polys(stark, trace_commitment, public_inputs, alphas, auxiliary_polys_commitment=None,
                           lookup_challenges=None, ctl_vars=None, placement=D.Placement()):
    """compute_quotient_polys (prover.rs:488-668) on the device. Returns a torch int64 CUDA tensor (num_challenges, size)
    of quotient-polynomial coefficients, size = n << log2_ceil(quotient_degree_factor), or None if the Stark has no
    quotient. Raises if the vanishing polynomial is not divisible by Z_H. A Stark with lookups also needs the auxiliary
    commitment (its LDE is read in place, like the trace's) and the lookup challenges; one with CTLs the auxiliary
    commitment and ctl_vars (CtlCheckVars of its CTL data's shape; their challenges are bound like the public
    inputs). On a placement of several ranks the commitments are this rank's row-block shards: each rank evaluates
    C(x)/Z_H(x) on its shard of the quotient coset (gl_stark_quotient_shard), and every rank gets the same quotient
    (Placement.quotient_from_shards; collective, a failure on any rank raises on every rank)."""
    import torch

    qdf = stark.quotient_degree_factor()
    if qdf == 0:
        return None
    b, consts, al = quotient_program(stark, public_inputs, alphas, auxiliary_polys_commitment, lookup_challenges,
                                     ctl_vars)
    ctx = trace_commitment.ctx
    prog = b.program()
    ctx.after_caller()
    if placement.num_shards > 1:
        aux_h = auxiliary_polys_commitment.h if auxiliary_polys_commitment is not None else None

        def run_shard(local):
            N.check(N.lib().gl_stark_quotient_shard(ctx.h, trace_commitment.h, aux_h, prog, len(b.instrs),
                                                    N.np_ptr(consts), len(consts), N.np_ptr(al), len(al), qdf,
                                                    N.vp(local.data_ptr())), ctx.h)

        return placement.quotient_from_shards(ctx, run_shard, len(al), trace_commitment.degree_log, qdf)
    size = (1 << trace_commitment.degree_log) << (qdf - 1).bit_length()
    out = torch.empty((len(al), size), dtype=torch.int64, device="cuda:%d" % ctx.device)
    if stark.uses_lookups() or ctl_vars is not None:
        N.check(N.lib().gl_stark_quotient_aux(ctx.h, trace_commitment.h, auxiliary_polys_commitment.h, prog,
                                              len(b.instrs), N.np_ptr(consts), len(consts), N.np_ptr(al), len(al), qdf,
                                              N.vp(out.data_ptr())), ctx.h)
    else:
        N.check(N.lib().gl_stark_quotient(ctx.h, trace_commitment.h, prog, len(b.instrs), N.np_ptr(consts), len(consts),
                                          N.np_ptr(al), len(al), qdf, N.vp(out.data_ptr())), ctx.h)
    ctx.synchronize()
    return out


def quotient_program(stark, public_inputs, alphas, auxiliary_polys_commitment=None, lookup_challenges=None,
                     ctl_vars=None):
    """What gl_stark_quotient[_aux] and gl_stark_quotient_shard take besides the commitments: the constraint program
    (ConstraintBuilder), its constants (public inputs, lookup challenges, CTL challenges, then the program's own) and
    the alphas, as uint64 arrays. Raises ShapeError for missing auxiliary inputs or a wrong number of public inputs."""
    if stark.uses_lookups() and (auxiliary_polys_commitment is None or lookup_challenges is None):
        raise N.ShapeError("a Stark with lookups needs the auxiliary commitment and the lookup challenges")
    if ctl_vars is not None and auxiliary_polys_commitment is None:
        raise N.ShapeError("a Stark with CTLs needs the auxiliary commitment")
    challenges = [int(c) % F.ORDER for c in lookup_challenges] if stark.uses_lookups() else []
    b = stark.constraint_program(len(challenges), ctl_vars)
    consts = np.array([int(x) % F.ORDER for x in public_inputs] + challenges + _ctl_bound(ctl_vars) + b.consts[b.num_bound:],
                      dtype=np.uint64)
    if len(public_inputs) != stark.PUBLIC_INPUTS:
        raise N.ShapeError("expected %d public inputs" % stark.PUBLIC_INPUTS)
    return b, consts, np.array([int(a) % F.ORDER for a in alphas], dtype=np.uint64)


def check_constraints(stark, trace_commitment, public_inputs, auxiliary_polys_commitment=None, lookup_challenges=None,
                      ctl_vars=None, max_report=64, parts=1, placement=None):
    """check_constraints (starky/src/prover.rs:670-820) on the device: every constraint of the Stark -- its own, then its
    lookups', then its CTLs' -- on every row of the trace subgroup H, each constraint on its own (gl_stark_check_rows).
    Takes what compute_quotient_polys takes but the alphas, on any kind of commitment (resident, non-resident, a
    row-block shard: its coefficients are replicated); a Stark of constraint degree 0 is checked too. Returns a
    ConstraintReport: the number of failing (row, constraint) pairs and the first max_report (0..65536) of them in
    (row, constraint) order as (row, EMIT ordinal, label), the label naming the Stark's own constraint by its number in
    eval_packed_generic's order, a lookup's check by lookup and challenge, or a CTL check by its Z.
    parts=G (a power of two): H is checked in min(G, n) parts one after another (gl_stark_check_rows_part), each with
    1/G of the whole check's scratch; the report is the same. placement: a distributed.Placement of several ranks, whose
    commitments these are: each rank checks its own part and the ranks merge their reports (collective; every rank
    returns the same report)."""
    parts = N.check_parts(parts)
    b, consts, _ = quotient_program(stark, public_inputs, [], auxiliary_polys_commitment, lookup_challenges, ctl_vars)
    ctx = trace_commitment.ctx
    aux_h = auxiliary_polys_commitment.h if auxiliary_polys_commitment is not None else None
    L = N.lib()
    failures, pairs = N.check_rows_in_parts(L.gl_stark_check_rows, L.gl_stark_check_rows_part, ctx,
                                            (trace_commitment.h, aux_h, b.program(), len(b.instrs), N.np_ptr(consts),
                                             len(consts)), max_report, trace_commitment.degree_log, parts, placement)
    return N.ConstraintReport(failures, [(row, e, b.labels[e]) for row, e in pairs])


def _raise_on_failure(stark, trace_commitment, public_inputs, **quotient_args):
    """check_constraints=True of the provers: ConstraintError with the reference's wording, the first failure's label
    and the total."""
    report = check_constraints(stark, trace_commitment, public_inputs, **quotient_args)
    if report.failures:
        row, _, label = report.entries[0]
        raise N.ConstraintError("Constraint failed in %s at row %d: %s; %d failing (row, constraint) pairs in all"
                                % (type(stark).__name__, row, label, report.failures), report)


def _ctl_bound(ctl_vars):
    """The CTL challenges a constraint program binds after the public inputs and lookup challenges."""
    return [int(v) % F.ORDER for c in (ctl_vars or []) for v in (c.challenges.beta, c.challenges.gamma)]


def check_lookup_shapes(stark):
    """The reference's panics for a Stark's lookups, raised before any device work: constraint degree 1 (division by
    zero in num_helper_columns) and chunks of more than two looking columns (todo! in eval_helper_columns)."""
    for lookup in stark.lookups():
        lookup.check_chunks(stark.constraint_degree())


def compute_lookup_helper_columns(stark, trace, lookup_challenges, ctx, out=None):
    """The lookup helper columns (prover.rs:177-195, lookup_helper_columns) on the device: for every lookup, for every
    challenge, the h_k columns and Z, from the trace values `trace` -- a (COLUMNS, n) int64 CUDA tensor, read in place.
    Returns a (num_lookup_helper_columns, n) int64 CUDA tensor of values: `out` if given (a contiguous view, e.g. the
    first rows of a table's auxiliary buffer), else a new one. `trace` may still be in production, and `out` still be
    read, on the caller's current torch stream: the library's work is ordered after it."""
    import torch

    from .lookup import row_programs

    check_lookup_shapes(stark)
    cols, n = trace.shape
    prog, offsets, consts = row_programs(stark.lookups(), stark.COLUMNS)
    ch = np.array([int(c) % F.ORDER for c in lookup_challenges], dtype=np.uint64)
    shape = (stark._helper_columns_per_challenge() * len(ch), n)
    if out is None:
        out = torch.empty(shape, dtype=torch.int64, device=trace.device)
    elif tuple(out.shape) != shape or not out.is_contiguous():
        raise N.ShapeError("the lookup helper output must be a contiguous %r tensor" % (shape,))
    ctx.after_caller()
    N.check(N.lib().gl_stark_lookup_helpers(ctx.h, N.vp(trace.data_ptr()), n, cols, F.log2_strict(n), prog,
                                            offsets.ctypes.data_as(N.u32p), len(offsets) - 1,
                                            N.np_ptr(consts) if len(consts) else None, len(consts), N.np_ptr(ch), len(ch),
                                            stark.constraint_degree(), N.vp(out.data_ptr())), ctx.h)
    ctx.synchronize()
    return out


def commit_auxiliary_polys(helper_columns, rate_bits, cap_height, ctx, **on):
    """The auxiliary commitment (prover.rs:216-230): PolynomialBatch::from_values of the helper columns, never blinded,
    committed straight from the device tensor compute_lookup_helper_columns returned. on: shard=(g, G) commits row
    block g of G only."""
    B, n = helper_columns.shape
    ctx.after_caller()

    def add_columns(h):
        N.check(N.lib().gl_commit_add_columns(h, 0, B, N.vp(helper_columns.data_ptr()), n, N.COLS_VALUES, N.MEM_DEVICE),
                ctx.h)

    return PolynomialBatch._from_device(ctx, B, F.log2_strict(n), rate_bits, cap_height, add_columns, **on)


def commit_quotient_polys(stark, quotient_polys, degree_bits, rate_bits, cap_height, ctx=None, **on):
    """'split quotient polys' + 'compute quotient commitment' (prover.rs:391-421): every polynomial is cut into
    quotient_degree_factor chunks of n coefficients, all chunks are committed with from_coeffs -- straight from the
    device tensor compute_quotient_polys returned. on: shard=(g, G) commits row block g of G only."""
    return PolynomialBatch._from_coeff_chunks(quotient_polys, stark.quotient_degree_factor(), degree_bits, rate_bits,
                                              cap_height, ctx, **on)


class StarkConfig:
    """StarkConfig (starky/src/config.rs:21-117): target security, number of challenges, FRI configuration."""

    def __init__(self, security_bits, num_challenges, fri_config):
        self.security_bits, self.num_challenges, self.fri_config = security_bits, num_challenges, fri_config

    @classmethod
    def standard_fast_config(cls):
        """config.rs:52-64: rate 1/2, ~100 bits of conjectured security."""
        return cls(100, 2, starky_standard_fast_fri_config())

    def fri_params(self, degree_bits):
        """config.rs:67-69: starky never hides."""
        return self.fri_config.fri_params(degree_bits, False)

    def observe(self, challenger):
        """config.rs:102-107"""
        challenger.observe_element(self.security_bits)
        challenger.observe_element(self.num_challenges)
        self.fri_config.observe(challenger)


def eval_l_0_and_l_last(log_n, x):
    """eval_l_0_and_l_last (vanishing_poly.rs:96-106) at x in F_{p^2}: L_0(x) = (x^n - 1) / (n (x - 1)),
    L_{n-1}(x) = (x^n - 1) / (n (g x - 1))."""
    n = ((1 << log_n) % F.ORDER, 0)
    g = (F.primitive_root_of_unity(log_n), 0)
    z_x = F.ext_sub(F.ext_pow(x, 1 << log_n), (1, 0))
    l_0 = F.ext_mul(z_x, F.ext_inverse(F.ext_mul(n, F.ext_sub(x, (1, 0)))))
    l_last = F.ext_mul(z_x, F.ext_inverse(F.ext_mul(n, F.ext_sub(F.ext_mul(g, x), (1, 0)))))
    return l_0, l_last


def eval_vanishing_poly(stark, local_values, next_values, public_inputs, alphas, x, degree_bits, auxiliary_polys=None,
                        auxiliary_polys_next=None, lookup_challenges=None, ctl_vars=None):
    """compute_eval_vanishing_poly (vanishing_poly.rs:108-173): the Stark's constraint program -- the instructions
    gl_stark_quotient runs -- evaluated at one point x of F_{p^2}, with the local and next rows (with lookups, the
    auxiliary polynomials' local and next values, of which the lookup helper columns are read; with CTLs, the
    CtlCheckVars' helper and Z values) as F_{p^2} values and the public inputs, lookup challenges, CTL challenges and
    program constants as base-field values; the constraints are filtered by z_last = x - g^{-1}, L_0(x), L_{n-1}(x) and
    folded with every alpha as ConstraintConsumer does (constraint_consumer.rs:46-84). Returns num_challenges F_{p^2}
    values (c0, c1)."""
    challenges = []
    if stark.uses_lookups():
        if auxiliary_polys is None or auxiliary_polys_next is None or lookup_challenges is None:
            raise N.ShapeError("a Stark with lookups needs the auxiliary values and the lookup challenges")
        challenges = [int(c) % F.ORDER for c in lookup_challenges]
    b = stark.constraint_program(len(challenges), ctl_vars)
    if len(public_inputs) != stark.PUBLIC_INPUTS:
        raise N.ShapeError("expected %d public inputs, got %d" % (stark.PUBLIC_INPUTS, len(public_inputs)))
    if ctl_vars is not None:     # [lookup helpers | CTL helpers | CTL Zs], as the program reads them
        nl = stark._helper_columns_per_challenge() * len(challenges)
        if challenges and (len(auxiliary_polys) < nl or len(auxiliary_polys_next) < nl):
            raise N.ShapeError("expected %d lookup auxiliary values" % nl)
        helpers = [h for v in ctl_vars for h in v.helper_columns]
        auxiliary_polys = list(auxiliary_polys[:nl] if challenges else []) + helpers + [v.local_z for v in ctl_vars]
        auxiliary_polys_next = (list(auxiliary_polys_next[:nl] if challenges else []) + [(0, 0)] * len(helpers)
                                + [v.next_z for v in ctl_vars])
    elif challenges and (len(auxiliary_polys) != b.num_aux or len(auxiliary_polys_next) != b.num_aux):
        raise N.ShapeError("expected %d auxiliary values" % b.num_aux)
    consts = [int(v) % F.ORDER for v in public_inputs] + challenges + _ctl_bound(ctl_vars) + b.consts[b.num_bound:]
    x = (int(x[0]) % F.ORDER, int(x[1]) % F.ORDER)
    l_0, l_last = eval_l_0_and_l_last(degree_bits, x)
    z_last = F.ext_sub(x, (F.inverse(F.primitive_root_of_unity(degree_bits)), 0))
    filters = {KIND_CONSTRAINT: None, KIND_TRANSITION: z_last, KIND_FIRST_ROW: l_0, KIND_LAST_ROW: l_last}

    def ext(v):
        return (int(v[0]) % F.ORDER, int(v[1]) % F.ORDER)

    acc = [(0, 0)] * len(alphas)
    vals = []
    for op, a, c in b.instrs:
        r = (0, 0)
        if op == OP_LOCAL:
            r = ext(local_values[a])
        elif op == OP_NEXT:
            r = ext(next_values[a])
        elif op == OP_AUX_LOCAL:
            r = ext(auxiliary_polys[a])
        elif op == OP_AUX_NEXT:
            r = ext(auxiliary_polys_next[a])
        elif op == OP_CONST:
            r = (consts[a], 0)
        elif op == OP_ADD:
            r = F.ext_add(vals[a], vals[c])
        elif op == OP_SUB:
            r = F.ext_sub(vals[a], vals[c])
        elif op == OP_MUL:
            r = F.ext_mul(vals[a], vals[c])
        else:  # OP_EMIT
            e = vals[a] if filters[c] is None else F.ext_mul(vals[a], filters[c])
            acc = [F.ext_add(F.ext_mul(s, (int(al) % F.ORDER, 0)), e) for s, al in zip(acc, alphas)]
        vals.append(r)
    return acc


def _dummy_openings(challenger, num_trace_polys, pow_degree, num_aux_polys=0):
    """get_dummy_polys (get_challenges.rs:201-256, prover.rs:272-319): simulated local, next, auxiliary and next
    auxiliary values c_i, c_i^d, c_i^{d^2}, ... from fresh extension challenges c_i, d = pow_degree. Returns (local,
    next) without auxiliary polynomials, else (local, next, aux, aux_next)."""
    log_pow_degree = (pow_degree - 1).bit_length()
    num_extension_powers = max(1, 50 // log_pow_degree - 1)
    total = 2 * num_trace_polys + 2 * num_aux_polys
    zetas = challenger.get_n_extension_challenges(-(-total // num_extension_powers))
    per_zeta = min(num_extension_powers + 1, total)
    evals = []
    for z in zetas:
        for _ in range(per_zeta):
            evals.append(z)
            z = F.ext_pow(z, pow_degree)
    t, a = num_trace_polys, num_aux_polys
    if a == 0:
        return evals[:t], evals[t:2 * t]
    return evals[:t], evals[t:2 * t], evals[2 * t:2 * t + a], evals[2 * t + a:total]


def _bind_constraints(stark, challenger, public_inputs, num_challenges, degree_bits, lookup_challenges=None,
                      ctl_vars=None, num_aux=None):
    """The constraint-binding step (prover.rs:239-370, get_challenges.rs:94-163): alphas', simulated openings, zeta',
    the vanishing polynomial there observed; returns the alphas the quotient uses. A Stark with lookups also simulates
    its auxiliary polynomials and evaluates the lookup constraints with the lookup challenges; with ctl_vars (the shape
    of its CTL data) the CTL helper and Z values are read from the simulated auxiliary polynomials too
    (prover.rs:321-350), of which there are num_aux."""
    from .cross_table_lookup import CtlCheckVars

    alphas_prime = challenger.get_n_challenges(num_challenges)
    pow_degree = max(2, stark.constraint_degree() + 1)
    if num_aux is None:
        num_aux = 0 if lookup_challenges is None else stark._helper_columns_per_challenge() * len(lookup_challenges)
    if num_aux == 0:
        local, nxt = _dummy_openings(challenger, stark.COLUMNS, pow_degree)
        aux = {}
    else:
        local, nxt, a, a_next = _dummy_openings(challenger, stark.COLUMNS, pow_degree, num_aux)
        aux = dict(auxiliary_polys=a, auxiliary_polys_next=a_next, lookup_challenges=lookup_challenges)
        if ctl_vars is not None:
            nl = stark._helper_columns_per_challenge() * len(lookup_challenges) if lookup_challenges is not None else 0
            total = sum(len(v.helper_columns) for v in ctl_vars)
            dummy, start = [], nl
            for i, v in enumerate(ctl_vars):
                k = len(v.helper_columns)
                dummy.append(CtlCheckVars(a[start:start + k], a[nl + total + i], a_next[nl + total + i], v.challenges,
                                          v.columns, v.filter))
                start += k
            aux["ctl_vars"] = dummy
    zeta_prime = challenger.get_extension_challenge()
    challenger.observe_extension_elements(eval_vanishing_poly(stark, local, nxt, public_inputs, alphas_prime, zeta_prime,
                                                              degree_bits, **aux))
    return challenger.get_n_challenges(num_challenges)


class StarkProof:
    """StarkProof (starky/src/proof.rs:30-53): trace cap, quotient cap (None for a Stark without
    constraints), StarkOpeningSet, FriProof, and the auxiliary polynomials' cap (None for a Stark without lookups or CTLs). The
    reference has no byte format for it (serde only); opening_proof.to_bytes() is write_fri_proof."""

    def __init__(self, trace_cap, quotient_polys_cap, openings, opening_proof, auxiliary_polys_cap=None):
        self.trace_cap, self.quotient_polys_cap = trace_cap, quotient_polys_cap
        self.openings, self.opening_proof = openings, opening_proof
        self.auxiliary_polys_cap = auxiliary_polys_cap

    def recover_degree_bits(self, config):
        """proof.rs:45-52: from the length of the first initial-tree Merkle proof."""
        siblings = self.opening_proof.query_round_proofs[0].initial_trees_proof.evals_proofs[0][1]
        return config.fri_config.cap_height + len(siblings) - config.fri_config.rate_bits


class StarkProofWithPublicInputs:
    """StarkProofWithPublicInputs (proof.rs:133-145)."""

    def __init__(self, proof, public_inputs):
        self.proof, self.public_inputs = proof, [int(v) % F.ORDER for v in public_inputs]

    def get_challenges(self, stark, config, verifier_circuit_fri_params=None, challenger=None, ctl_challenges=None,
                       ctl_vars=None, ignore_trace_cap=False):
        """get_challenges (get_challenges.rs:37-199,323-357) replayed from the proof alone: the public inputs, the
        config, the trace cap (unless ignore_trace_cap), the lookup challenges -- ctl_challenges when given, else drawn
        if there is an auxiliary cap -- and the auxiliary cap (get_challenges.rs:67-92), the constraint-binding step
        (with ctl_vars, the table's CtlCheckVars), the quotient cap, zeta, the openings, then FRI's challenges. A
        multi-STARK replay passes its challenger. Returns a dict: lookup_challenge_set (None without an auxiliary cap
        or CTL challenges), stark_alphas, stark_zeta, fri_alpha, fri_betas, fri_pow_response, fri_query_indices."""
        from .challenger import Challenger
        from .fri import fri_challenges
        from .lookup import get_grand_product_challenge_set

        p = self.proof
        degree_bits = p.recover_degree_bits(config)
        ch = challenger if challenger is not None else Challenger()
        ch.observe_elements(self.public_inputs)
        config.observe(ch)
        if not ignore_trace_cap:
            ch.observe_cap(p.trace_cap)
        lookup_challenge_set = lookup_challenges = None
        if ctl_challenges is not None:
            lookup_challenge_set = list(ctl_challenges)
        elif p.auxiliary_polys_cap is not None:
            lookup_challenge_set = get_grand_product_challenge_set(ch, config.num_challenges)
        if p.auxiliary_polys_cap is not None:
            ch.observe_cap(p.auxiliary_polys_cap)
        if stark.uses_lookups():
            if lookup_challenge_set is None:
                raise N.ShapeError("Missing auxiliary_polys_cap")
            lookup_challenges = [c.beta for c in lookup_challenge_set]
        num_aux = None
        if ctl_vars is not None:
            num_aux = len(p.openings.auxiliary_polys) if p.openings.auxiliary_polys is not None else 0
        alphas = _bind_constraints(stark, ch, self.public_inputs, config.num_challenges, degree_bits, lookup_challenges,
                                   ctl_vars, num_aux)
        if p.quotient_polys_cap is not None:
            ch.observe_cap(p.quotient_polys_cap)
        zeta = ch.get_extension_challenge()
        for batch in p.openings.to_fri_openings():                      # Challenger::observe_openings
            ch.observe_elements(batch.reshape(-1))
        final_len = steps = None
        if verifier_circuit_fri_params is not None:
            vp = verifier_circuit_fri_params
            final_len, steps = 1 << (vp.degree_bits - vp.total_arities()), len(vp.reduction_arity_bits)
        fp = p.opening_proof
        fri_alpha, fri_betas, pow_response, indices = fri_challenges(ch, fp.commit_phase_merkle_caps, fp.final_poly,
                                                                     fp.pow_witness, degree_bits, config.fri_config,
                                                                     final_len, steps)
        return dict(lookup_challenge_set=lookup_challenge_set, stark_alphas=alphas, stark_zeta=zeta, fri_alpha=fri_alpha,
                    fri_betas=fri_betas, fri_pow_response=pow_response, fri_query_indices=indices)


def _commit_trace(trace, rate_bits, cap_height, ctx, **on):
    """The trace commitment (prover.rs:83-94) from host columns or from a (COLUMNS, n) torch CUDA tensor on the context's
    device (read in place, never copied to the host). on: shard=(g, G) commits row block g of G only."""
    if hasattr(trace, "data_ptr"):
        import torch

        if not trace.is_cuda or trace.dim() != 2 or trace.element_size() != 8:
            raise N.ShapeError("a torch trace must be a (COLUMNS, n) CUDA tensor of 64-bit words")
        cols = trace.contiguous().view(torch.int64)
        B, n = cols.shape
        log_n = F.log2_strict(n)
        ctx.after_caller()

        def add_columns(h):
            N.check(N.lib().gl_commit_add_columns(h, 0, B, N.vp(cols.data_ptr()), n, N.COLS_VALUES, N.MEM_DEVICE), ctx.h)

        return PolynomialBatch._from_device(ctx, B, log_n, rate_bits, cap_height, add_columns, **on)
    return PolynomialBatch.from_values(trace, rate_bits, False, cap_height, ctx=ctx, **on)


def _device_trace(trace, ctx):
    """The trace as ONE (COLUMNS, n) int64 CUDA tensor that the trace commitment and the lookup helper columns both read:
    a torch CUDA trace as it is (made contiguous), host columns copied to the context's device once."""
    import torch

    if hasattr(trace, "data_ptr"):
        if not trace.is_cuda or trace.dim() != 2 or trace.element_size() != 8:
            raise N.ShapeError("a torch trace must be a (COLUMNS, n) CUDA tensor of 64-bit words")
        dev = trace.contiguous().view(torch.int64)
    else:
        host = np.ascontiguousarray(trace, dtype=np.uint64).view(np.int64)
        dev = torch.from_numpy(host).to("cuda:%d" % ctx.device)
    ctx.after_caller()  # a copy above is on torch's stream; the library reads the tensor on the context's
    return dev


def _check_prove_shapes(stark, config, trace, public_inputs, verifier_circuit_fri_params=None, lde_blocks=0):
    """prove's checks (prover.rs:53-81,153-162), before any device work. Returns the ProveParams of the trace.
    lde_blocks=G (non-resident commitments, lde_placement): G at most the quotient coset's size, since the quotient is
    evaluated in one part of it per block."""
    shape = tuple(trace.shape)
    if len(shape) != 2 or shape[0] != stark.COLUMNS:
        raise N.ShapeError("the trace must be (COLUMNS = %d, n), got %r" % (stark.COLUMNS, shape))
    if len(public_inputs) != stark.PUBLIC_INPUTS:
        raise N.ShapeError("expected %d public inputs, got %d" % (stark.PUBLIC_INPUTS, len(public_inputs)))
    degree_bits = F.log2_strict(shape[1])
    fri_params = config.fri_params(degree_bits)
    rate_bits, cap_height = config.fri_config.rate_bits, config.fri_config.cap_height
    if fri_params.total_arities() > degree_bits + rate_bits - cap_height:
        raise N.ShapeError("FRI total reduction arity is too large.")
    if stark.constraint_degree() > (1 << rate_bits) + 1:
        raise N.ShapeError("The degree of the Stark constraints must be <= blowup_factor + 1")
    final_poly_coeff_len = max_num_query_steps = None
    if verifier_circuit_fri_params is not None:
        vp = verifier_circuit_fri_params
        if vp.config != fri_params.config:
            raise N.ShapeError("verifier_circuit_fri_params.config differs from the proof's FRI config")
        strategy = config.fri_config.reduction_strategy
        if strategy[0] != "ConstantArityBits":
            raise N.ShapeError("Fri Reduction Strategy is not ConstantArityBits")
        final_poly_coeff_len = 1 << (vp.degree_bits - vp.total_arities())       # final_poly_coeff_len (fri/prover.rs:77)
        if final_poly_coeff_len != 1 << (1 + strategy[2]):
            raise N.ShapeError("the verifier circuit's final polynomial has %d coefficients, expected %d"
                               % (final_poly_coeff_len, 1 << (1 + strategy[2])))
        max_num_query_steps = len(vp.reduction_arity_bits)
    qdf = stark.quotient_degree_factor()
    if lde_blocks and qdf:
        size = (1 << degree_bits) << (qdf - 1).bit_length()
        if lde_blocks > size:
            raise N.ShapeError("lde_blocks=%d exceeds the %d points of the quotient coset" % (lde_blocks, size))
    return ProveParams(degree_bits, fri_params, final_poly_coeff_len, max_num_query_steps)


class ProveParams:
    """What prove_with_commitment needs of the checks: degree_bits, the FRI parameters and the verifier-circuit FRI
    shape (final_poly_coeff_len, max_num_query_steps; None without a verifier circuit)."""

    def __init__(self, degree_bits, fri_params, final_poly_coeff_len, max_num_query_steps):
        self.degree_bits, self.fri_params = degree_bits, fri_params
        self.final_poly_coeff_len, self.max_num_query_steps = final_poly_coeff_len, max_num_query_steps


def lde_placement(cap_height, lde_blocks):
    """The one-device Placement of a prover's lde_blocks argument: Placement() for None (resident commitments), else
    non-resident commitments of lde_blocks row blocks under a cap of 2^cap_height entries (refused as
    PolynomialBatch.check_lde_blocks refuses it, before any device work). The starky and plonky2 provers share it."""
    if lde_blocks is None:
        return D.Placement()
    check_lde_blocks(lde_blocks, cap_height)
    return D.Placement(lde_blocks=int(lde_blocks))


def prove(stark, config, trace, public_inputs, verifier_circuit_fri_params=None, ctx=None, lde_blocks=None,
          check_constraints=False):
    """prove (starky/src/prover.rs:40-114) for one Stark: trace = (COLUMNS, n) host columns or torch CUDA tensor ->
    StarkProofWithPublicInputs. The trace commitment, then a fresh challenger observing the public inputs, the config
    and the trace cap, then prove_with_commitment without CTLs. verifier_circuit_fri_params: the FRI parameters of a
    verifier circuit made for another degree (ConstantArityBits only); the transcript then observes the zero caps and
    coefficients that verifier expects. A torch trace may still be in production on the caller's current torch stream:
    the library's work is ordered after it. Raises ShapeError / NativeError with the reference's messages; every
    commitment is released on every exit path. lde_blocks=G: every commitment is non-resident
    (PolynomialBatch.from_values), for traces whose LDEs exceed device memory; the proof is the same. G must be a power
    of two of at most 2^cap_height and of at most the quotient coset's size (ShapeError before any device work).
    check_constraints=True: every constraint is checked on every row of H before the quotient, where the reference's
    debug builds check them (prover.rs:241-256), and a failure raises ConstraintError naming the row and the constraint;
    the proof is unchanged. With lde_blocks=G the check runs in G parts of H, one after another, with the same message
    and report."""
    return _prove(stark, config, trace, public_inputs, verifier_circuit_fri_params, ctx,
                  lde_placement(config.fri_config.cap_height, lde_blocks), check_constraints)


def _prove(stark, config, trace, public_inputs, verifier_circuit_fri_params, ctx, placement, check_constraints=False):
    """prove on a distributed.Placement (see prove_with_commitment)."""
    from .challenger import Challenger

    params = _check_prove_shapes(stark, config, trace, public_inputs, verifier_circuit_fri_params, placement.lde_blocks)
    ctx = ctx or N.default_context()
    public_inputs = [int(v) % F.ORDER for v in public_inputs]
    rate_bits, cap_height = config.fri_config.rate_bits, config.fri_config.cap_height
    if stark.uses_lookups():
        check_lookup_shapes(stark)
        trace = _device_trace(trace, ctx)
    trace_commitment = _commit_trace(trace, rate_bits, cap_height, ctx, **placement.commit_kwargs)
    try:
        challenger = Challenger()
        challenger.observe_elements(public_inputs)
        config.observe(challenger)
        trace_cap = placement.cap(trace_commitment)
        challenger.observe_cap(trace_cap)
        return prove_with_commitment(stark, config, trace, trace_commitment, trace_cap, None, None, challenger,
                                     public_inputs, params, ctx=ctx, placement=placement,
                                     check_constraints=check_constraints)
    finally:
        trace_commitment.close()


def prove_with_commitment(stark, config, trace, trace_commitment, trace_cap, ctl_data, ctl_challenges, challenger,
                          public_inputs, params, ctx=None, placement=D.Placement(), check_constraints=False):
    """prove_with_commitment (starky/src/prover.rs:125-484): one table's proof from its committed trace, on a challenger
    that has already observed what precedes it (the config and trace_cap, the trace's full cap, among them). Every
    array-sized step runs on the device (lookup helper columns and the auxiliary commitment, quotient from the LDEs in
    place, quotient commitment, openings, FRI); the transcript and the constraint-binding step run on the host. With ctl_challenges the lookups use their
    betas (prover.rs:165-168). With ctl_data (cross_table_lookup.CtlData, its CTL columns already in its auxiliary
    buffer) the auxiliary oracle is [lookup helpers | CTL helpers | CTL Zs], the CTL constraints join the quotient and
    the openings carry ctl_zs_first. trace: the values the lookup helper columns read (a CUDA tensor when the Stark has
    lookups). params: _check_prove_shapes's. placement: a distributed.Placement of G ranks proves on them, this one
    holding row block g of every commitment (trace_commitment too): the caps are all-gathered before they are observed,
    the quotient is evaluated shard by shard and all-gathered, the openings are summed over each rank's block of the
    coefficients and added up, and FRI routes the query openings between the ranks.
    Everything else runs redundantly on every rank, so every rank returns the same proof. Every commitment made here is
    released on every exit path; the trace commitment stays the caller's. check_constraints=True: after the auxiliary
    commitment, check_constraints with the proof's own challenges, on the placement (placement.check_kwargs: part by
    part for non-resident commitments, each rank its own part with several ranks); ConstraintError if anything fails,
    with the same message and report on every rank."""
    from .fri import prove_openings
    from .lookup import get_grand_product_challenge_set

    ctx = ctx or N.default_context()
    degree_bits = params.degree_bits
    rate_bits, cap_height = config.fri_config.rate_bits, config.fri_config.cap_height
    uses_lookups = stark.uses_lookups()
    commitments = []
    try:
        aux_commitment = lookup_challenges = ctl_vars = None
        nl = 0
        quotient_args = {}
        if uses_lookups:                                                # prover.rs:164-195
            if ctl_challenges is not None:
                lookup_challenges = [c.beta for c in ctl_challenges]
            else:
                lookup_challenges = [c.beta for c in get_grand_product_challenge_set(challenger, config.num_challenges)]
            nl = stark._helper_columns_per_challenge() * len(lookup_challenges)
            quotient_args = dict(lookup_challenges=lookup_challenges)
        if ctl_data is not None:                                        # prover.rs:196-230
            from .cross_table_lookup import ctl_shape_vars

            auxiliary = ctl_data.auxiliary
            if uses_lookups:
                compute_lookup_helper_columns(stark, trace, lookup_challenges, ctx, out=auxiliary[:nl])
            ctl_vars = ctl_shape_vars(ctl_data)
            quotient_args["ctl_vars"] = ctl_vars
        elif uses_lookups:
            auxiliary = compute_lookup_helper_columns(stark, trace, lookup_challenges, ctx)
        if uses_lookups or ctl_data is not None:
            aux_commitment = commit_auxiliary_polys(auxiliary, rate_bits, cap_height, ctx, **placement.commit_kwargs)
            commitments.append(aux_commitment)
            del auxiliary
            if ctl_data is not None:
                ctl_data.auxiliary = None
            aux_cap = placement.cap(aux_commitment)
            challenger.observe_cap(aux_cap)
            quotient_args["auxiliary_polys_commitment"] = aux_commitment
        if check_constraints:                                            # prover.rs:241-256
            _raise_on_failure(stark, trace_commitment, public_inputs, **quotient_args, **placement.check_kwargs)
        num_ctl_polys = ctl_data.num_ctl_helper_polys() if ctl_data is not None else []
        num_ctl_helpers, num_ctl_zs = sum(num_ctl_polys), len(num_ctl_polys)
        alphas = _bind_constraints(stark, challenger, public_inputs, config.num_challenges, degree_bits,
                                   lookup_challenges, ctl_vars, nl + num_ctl_helpers + num_ctl_zs if ctl_vars else None)
        quotient_polys = compute_quotient_polys(stark, trace_commitment, public_inputs, alphas, **quotient_args,
                                                **placement.step_kwargs)
        quotient_commitment = None
        if quotient_polys is not None:
            quotient_commitment = commit_quotient_polys(stark, quotient_polys, degree_bits, rate_bits, cap_height, ctx,
                                                        **placement.commit_kwargs)
            commitments.append(quotient_commitment)
            del quotient_polys
            quotient_cap = placement.cap(quotient_commitment)
            challenger.observe_cap(quotient_cap)
        zeta = challenger.get_extension_challenge()
        if F.ext_pow(zeta, 1 << degree_bits) == (1, 0):
            raise N.NativeError("Opening point is in the subgroup.")
        g = F.primitive_root_of_unity(degree_bits)
        ctl_first = dict(num_ctl_zs_first=(nl + num_ctl_helpers, num_ctl_zs)) if stark.requires_ctls() else {}
        openings = StarkOpeningSet.new(zeta, g, trace_commitment, aux_commitment, quotient_commitment, **ctl_first,
                                       **placement.step_kwargs)
        for batch in openings.to_fri_openings():                        # Challenger::observe_openings
            challenger.observe_elements(batch.reshape(-1))
        instance = stark.fri_instance(zeta, g, config, num_ctl_helpers, num_ctl_zs)
        opening_proof = prove_openings(instance, [trace_commitment] + commitments, challenger, params.fri_params,
                                       params.final_poly_coeff_len, params.max_num_query_steps, **placement.step_kwargs)
        proof = StarkProof(trace_cap,
                           quotient_cap if quotient_commitment is not None else None,
                           openings, opening_proof,
                           aux_cap if aux_commitment is not None else None)
        return StarkProofWithPublicInputs(proof, public_inputs)
    finally:
        for c in commitments:
            c.close()
