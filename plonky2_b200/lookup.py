"""starky's logUp lookup argument (starky/src/lookup.rs:33-863, https://eprint.iacr.org/2022/1530) within one STARK (the
cross-table lookups, which reuse Column / Filter and eval_helper_columns, are cross_table_lookup.py): Column / Filter /
Lookup, the grand-product challenges, the lookup constraints recorded into a STARK's constraint program
(eval_packed_lookups_generic) and the row programs gl_stark_lookup_helpers runs to write the helper columns on the
device (lookup_helper_columns)."""
import numpy as np

from . import _native as N
from . import field as F


class Column:
    """Column<F> (lookup.rs:132-399): a linear combination of the current row's columns, of the next row's columns, and
    a constant. Coefficients and the constant are field elements (Python ints)."""

    def __init__(self, linear_combination=(), next_row_linear_combination=(), constant=0):
        self.linear_combination = [(int(c), int(f) % F.ORDER) for c, f in linear_combination]
        self.next_row_linear_combination = [(int(c), int(f) % F.ORDER) for c, f in next_row_linear_combination]
        self.constant = int(constant) % F.ORDER

    @classmethod
    def single(cls, c):
        return cls([(c, 1)])

    @classmethod
    def singles(cls, cs):
        return [cls.single(c) for c in cs]

    @classmethod
    def single_next_row(cls, c):
        return cls((), [(c, 1)])

    @classmethod
    def singles_next_row(cls, cs):
        return [cls.single_next_row(c) for c in cs]

    @classmethod
    def constant(cls, constant):  # on an instance, `constant` is the combination's constant term
        return cls((), (), constant)

    @classmethod
    def zero(cls):
        return cls.constant(0)

    @classmethod
    def one(cls):
        return cls.constant(1)

    @classmethod
    def linear_combination_with_constant(cls, iterable, constant):
        v = list(iterable)
        if not v:
            raise N.ShapeError("a linear combination needs at least one column")
        if len({c for c, _ in v}) != len(v):
            raise N.ShapeError("Duplicate columns.")
        return cls(v, (), constant)

    @classmethod
    def linear_combination(cls, iterable):
        return cls.linear_combination_with_constant(iterable, 0)

    @classmethod
    def linear_combination_and_next_row_with_constant(cls, iterable, next_row_iterable, constant):
        v, nv = list(iterable), list(next_row_iterable)
        if not v and not nv:
            raise N.ShapeError("a linear combination needs at least one column")
        if len({c for c, _ in v}) != len(v) or len({c for c, _ in nv}) != len(nv):
            raise N.ShapeError("Duplicate columns.")
        return cls(v, nv, constant)

    @classmethod
    def le_bits(cls, cs):
        return cls.linear_combination((c, 1 << k) for k, c in enumerate(cs))

    @classmethod
    def le_bits_with_constant(cls, cs, constant):
        return cls.linear_combination_with_constant(((c, 1 << k) for k, c in enumerate(cs)), constant)

    @classmethod
    def le_bytes(cls, cs):
        return cls.linear_combination((c, pow(256, k, F.ORDER)) for k, c in enumerate(cs))

    @classmethod
    def sum(cls, cs):
        return cls.linear_combination((c, 1) for c in cs)

    def _expr(self, vars, with_next):
        terms = [vars.local(c) if f == 1 else vars.local(c) * f for c, f in self.linear_combination]
        if with_next:
            terms += [vars.next(c) if f == 1 else vars.next(c) * f for c, f in self.next_row_linear_combination]
        if self.constant or not terms:
            terms.append(vars.constant(self.constant))
        acc = terms[0]
        for t in terms[1:]:
            acc = acc + t
        return acc

    def eval(self, vars):
        """Column::eval (lookup.rs:292-303): the current row only."""
        return self._expr(vars, False)

    def eval_with_next(self, vars):
        """Column::eval_with_next (lookup.rs:305-321); on a row program, also eval_table (lookup.rs:323-335)."""
        return self._expr(vars, True)


class Filter:
    """Filter<F> (lookup.rs:33-130): sum of products of column pairs plus a sum of columns. The default is the constant
    1."""

    def __init__(self, products=(), constants=()):
        self.products = [(a, b) for a, b in products]
        self.constants = list(constants)

    @classmethod
    def new(cls, products, constants):
        return cls(products, constants)

    @classmethod
    def new_simple(cls, col):
        return cls((), [col])

    @classmethod
    def default(cls):
        return cls((), [Column.one()])

    def eval_filter(self, vars):
        """Filter::eval_filter (lookup.rs:69-84); on a row program, also eval_table (lookup.rs:118-129)."""
        terms = [a.eval_with_next(vars) * b.eval_with_next(vars) for a, b in self.products]
        terms += [c.eval_with_next(vars) for c in self.constants]
        if not terms:
            return vars.constant(0)
        acc = terms[0]
        for t in terms[1:]:
            acc = acc + t
        return acc


def helper_chunk_size(constraint_degree):
    """constraint_degree.checked_sub(1).unwrap_or(1) (lookup.rs:439,670,757); 0 is the reference's division by zero."""
    return 1 if constraint_degree == 0 else constraint_degree - 1


class Lookup:
    """Lookup<F> (lookup.rs:403-442): looking columns (f_i), the table column (t), the frequencies column (m) and one
    filter per looking column."""

    def __init__(self, columns, table_column, frequencies_column, filter_columns):
        self.columns, self.table_column = list(columns), table_column
        self.frequencies_column, self.filter_columns = frequencies_column, list(filter_columns)
        if len(self.columns) != len(self.filter_columns):
            raise N.ShapeError("a Lookup needs one filter per looking column (%d columns, %d filters)"
                               % (len(self.columns), len(self.filter_columns)))

    def num_helper_columns(self, constraint_degree):
        """lookup.rs:433-441: one h column per chunk of constraint_degree - 1 looking columns, plus Z."""
        chunk = helper_chunk_size(constraint_degree)
        if chunk == 0:
            raise N.ShapeError("attempt to divide by zero: a STARK of constraint degree 1 cannot have lookups")
        return -(-len(self.columns) // chunk) + 1

    def check_chunks(self, constraint_degree):
        """eval_helper_columns (lookup.rs:669-693) handles chunks of 1 or 2 looking columns; longer ones are the
        reference's todo!("Allow other constraint degrees")."""
        self.num_helper_columns(constraint_degree)
        if helper_chunk_size(constraint_degree) > 2 and len(self.columns) > 2:
            raise N.ShapeError("Allow other constraint degrees: a chunk of %d looking columns"
                               % min(len(self.columns), helper_chunk_size(constraint_degree)))


class GrandProductChallenge:
    """GrandProductChallenge<F> (lookup.rs:444-465)."""

    def __init__(self, beta, gamma):
        self.beta, self.gamma = int(beta), int(gamma)

    def __eq__(self, other):
        return (self.beta, self.gamma) == (other.beta, other.gamma)

    def __repr__(self):
        return "GrandProductChallenge(beta=%d, gamma=%d)" % (self.beta, self.gamma)


def get_grand_product_challenge_set(challenger, num_challenges):
    """get_grand_product_challenge_set (lookup.rs:525-543): num_challenges (beta, gamma) pairs, beta drawn first."""
    out = []
    for _ in range(num_challenges):
        beta = challenger.get_challenge()
        gamma = challenger.get_challenge()
        out.append(GrandProductChallenge(beta, gamma))
    return out


def eval_helper_columns(filters, columns, helper_columns, constraint_degree, challenge, consumer, vars, combine=None):
    """eval_helper_columns (lookup.rs:655-695). A lookup's columns are single values combined with its challenge
    (beta = 1, gamma = challenge): combine(x) = x + gamma; a cross-table lookup passes its own combine (a tuple's
    GrandProductChallenge::combine)."""
    if not helper_columns:
        return
    if combine is None:
        combine = lambda x: x + challenge  # noqa: E731
    chunk_size = helper_chunk_size(constraint_degree)
    for k, h in enumerate(helper_columns):
        chunk, fs = columns[k * chunk_size:(k + 1) * chunk_size], filters[k * chunk_size:(k + 1) * chunk_size]
        if len(chunk) == 2:
            combin0, combin1 = combine(chunk[0]), combine(chunk[1])
            f0, f1 = fs[0].eval_filter(vars), fs[1].eval_filter(vars)
            consumer.constraint(combin1 * combin0 * h - f0 * combin1 - f1 * combin0)
        elif len(chunk) == 1:
            combin = combine(chunk[0])
            consumer.constraint(combin * h - fs[0].eval_filter(vars))
        else:
            raise N.ShapeError("Allow other constraint degrees: a chunk of %d looking columns" % len(chunk))


def eval_packed_lookups_generic(stark, lookups, vars, num_lookup_challenges, yield_constr):
    """eval_packed_lookups_generic (lookup.rs:804-863) recorded into a ConstraintBuilder: for every lookup, for every
    challenge, the helper-column constraints, Z = 0 on the first row and the unfiltered step
    (Z' - Z)(t + gamma) - (sum_k h_k (t + gamma) - m). The auxiliary columns are read with aux_local / aux_next, the
    challenges with lookup_challenge (bound at evaluation time like the public inputs)."""
    degree = stark.constraint_degree()
    start = 0
    for li, lookup in enumerate(lookups):
        nh = lookup.num_helper_columns(degree)
        for c in range(num_lookup_challenges):
            yield_constr.begin_scope("lookup %d, challenge %d" % (li, c))
            challenge = vars.lookup_challenge(c)
            lookup_columns = [col.eval_with_next(vars) for col in lookup.columns]
            helpers = [vars.aux_local(start + k) for k in range(nh - 1)]
            eval_helper_columns(lookup.filter_columns, lookup_columns, helpers, degree, challenge, yield_constr, vars)
            z, next_z = vars.aux_local(start + nh - 1), vars.aux_next(start + nh - 1)
            table_with_challenge = lookup.table_column.eval(vars) + challenge
            hsum = vars.constant(0)
            for h in helpers:
                hsum = hsum + h
            y = hsum * table_with_challenge - lookup.frequencies_column.eval(vars)
            yield_constr.constraint_first_row(z)
            yield_constr.constraint((next_z - z) * table_with_challenge - y)
            start += nh


def row_programs(lookups, num_columns):
    """The row programs of gl_stark_lookup_helpers (include/plonky2_b200.h): one ConstraintBuilder per lookup with the
    looking columns and filters (eval_table: current and next row), then the table and frequencies columns, emitted by
    role. Returns (instructions (StarkInstr array), offsets (uint32, n_lookups + 1), constants (uint64))."""
    from .stark import OP_CONST, OP_EMIT, ConstraintBuilder, StarkInstr

    LOOKED, FILTER, TABLE, FREQUENCIES = range(4)
    consts, instrs, offsets = [], [], [0]
    for lookup in lookups:
        b = ConstraintBuilder(num_columns, 0)
        for col, filt in zip(lookup.columns, lookup.filter_columns):
            b._push(OP_EMIT, col.eval_with_next(b).idx, LOOKED)
            b._push(OP_EMIT, filt.eval_filter(b).idx, FILTER)
        b._push(OP_EMIT, lookup.table_column.eval_with_next(b).idx, TABLE)
        b._push(OP_EMIT, lookup.frequencies_column.eval_with_next(b).idx, FREQUENCIES)
        for op, a, c in b.instrs:                     # the lookups share one constant table
            if op == OP_CONST:
                v = b.consts[a]
                if v not in consts:
                    consts.append(v)
                a = consts.index(v)
            instrs.append((op, a, c))
        offsets.append(len(instrs))
    arr = (StarkInstr * len(instrs))()
    for i, (op, a, c) in enumerate(instrs):
        arr[i].op, arr[i].a, arr[i].b = op, a, c
    return arr, np.array(offsets, dtype=np.uint32), np.array(consts, dtype=np.uint64)
