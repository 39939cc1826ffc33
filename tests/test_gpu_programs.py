"""The four constraint-program interpreters on seeded random programs that reach every declared limit, compared word for
word with exact evaluators: k_stark_quotient (gl_stark_quotient[_aux], gl_stark_quotient_shard), k_logup_rows
(gl_logup.cuh, gl_stark_lookup_helpers), k_ctl_rows (gl_ctl.cuh, gl_stark_ctl_helpers) and k_plonk_quotient
(gl_vanishing.cuh, gl_plonk_quotient[_shard]).

The builders (ConstraintBuilder, lookup.py, cross_table_lookup.py, plonk.py) emit a few program shapes and none at a
limit. The generators here draw only programs the host checks accept, and pin one dimension at a time at its limit, read
from include/plonky2_b200.h: 512 STARK instructions, 16 looking columns, 16 CTL groups, 8 entries, 32 values, 256
row-program instructions, 256 registers, 4 commitments, 4 challenges, quotient degree factor 8, 65 536 vanishing terms.
They draw every opcode and EMIT role, operands a == b, values read hundreds of instructions after they were written,
registers overwritten while others still hold older values, constants past 65 535 (GL_VP_CONST's high half), ADDC / MULC
at constant 65 535, TERM 65 535 and repeated terms, LOCAL of a salt column, NEXT on every commitment.

The evaluators restate what each kernel writes: the STARK quotient through check_quotient_values
(test_gpu_stark_large.py), the logUp and CTL columns through stark_twin's helper_columns and partial_sums fed the rows a
small row-program evaluator computes, the plonky2 quotient through a register-file evaluator (x, Z_H, L_0 and the alpha
powers as gl_vanishing.cuh's contract states them). The LDE values come from the handles' own leaves: point i of the
quotient coset g<w_size> is leaf row bitrev(i) of the first `size` rows (get_lde_values with step 2^(rate - qd_bits)).

CPU: the same programs through the host builds of the logUp, CTL and vanishing interpreters (tests/emu) against the
evaluators.
GPU (-m gpu): every entry point at its limits; one random STARK program also on non-resident handles and on row-block
shards, equal to the whole result."""
import ctypes as C
import os
import re
import subprocess
from types import SimpleNamespace as NS

import numpy as np
import pytest

import gl_numpy as G
import stark_twin as T
from conftest import P, synth
from plonky2_b200 import _native as N
from plonky2_b200 import field as E
from plonky2_b200 import stark as S
from test_gpu_stark_large import check_quotient_values

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_limits():
    with open(os.path.join(ROOT, "include", "plonky2_b200.h")) as f:
        return {m.group(1): int(m.group(2)) for m in re.finditer(r"#define (GL_\w+_MAX_\w+) (\d+)", f.read())}


LIM = _header_limits()
STARK_MAX_INSTR, MAX_ALPHAS, MAX_QD = LIM["GL_STARK_MAX_INSTR"], LIM["GL_STARK_MAX_ALPHAS"], LIM["GL_STARK_MAX_QD"]
LOGUP_MAX_COLUMNS, LOGUP_MAX_INSTR = LIM["GL_LOGUP_MAX_COLUMNS"], LIM["GL_LOGUP_MAX_INSTR"]
CTL_MAX_GROUPS, CTL_MAX_ENTRIES = LIM["GL_CTL_MAX_GROUPS"], LIM["GL_CTL_MAX_ENTRIES"]
CTL_MAX_VALUES, CTL_MAX_INSTR = LIM["GL_CTL_MAX_VALUES"], LIM["GL_CTL_MAX_INSTR"]
VP_MAX_REGS, VP_MAX_COMMITS = LIM["GL_VP_MAX_REGS"], LIM["GL_VP_MAX_COMMITS"]
VP_MAX_TERMS = 65536                    # TERM's b is 16 bits; gl_plonk_quotient takes 1..65536 terms
VP_CONSTS = 70000                       # past 65 536: GL_VP_CONST's index needs its high half
LOGUP_LOOKED, LOGUP_FILTER, LOGUP_TABLE, LOGUP_FREQUENCIES = range(4)
CTL_VALUE, CTL_FILTER = 0, 1
VP_LOCAL, VP_NEXT, VP_CONST, VP_X, VP_L0, VP_ADD, VP_SUB, VP_MUL, VP_TERM, VP_ADDC, VP_MULC = range(11)
SALT = 4


def _brev(n_bits):
    return G.brev(np.arange(1 << n_bits), n_bits).astype(np.int64)


# ------------------------------------------------------------------------------------------------------ generators
class _Values:
    """The indices of a row program's values a later instruction may read (every non-EMIT instruction), drawn so that
    some reads go back to value 0 and some hundreds of instructions back."""

    def __init__(self, rng):
        self.rng, self.idx = rng, []

    def pick(self, k):
        r, idx = self.rng.random(), self.idx
        if r < 0.08:
            return idx[0]
        far = [j for j in idx[:64] if k - j >= 200]
        if r < 0.2 and far:
            return int(self.rng.choice(far))
        return int(self.rng.choice(idx[-12:]))


def _leaf(rng, op, n_cols, n_consts, n_aux):
    """(op, a) of an instruction that reads no earlier value; operands favour the first and last column or constant."""
    def edge(n):
        r = rng.random()
        return 0 if r < 0.2 else n - 1 if r < 0.4 else int(rng.integers(n))
    if op in (S.OP_LOCAL, S.OP_NEXT):
        return op, edge(n_cols)
    if op in (S.OP_AUX_LOCAL, S.OP_AUX_NEXT):
        return op, edge(n_aux)
    return op, edge(n_consts)


def _arith(rng, vals, k):
    op = int(rng.choice([S.OP_ADD, S.OP_SUB, S.OP_MUL]))
    a = vals.pick(k)
    return op, a, a if rng.random() < 0.15 else vals.pick(k)


def stark_program(seed, n_instr, n_cols, n_consts, n_aux=0, emit_every=8):
    """A gl_stark_instr program ((n_instr, 4) uint16) of every opcode (the auxiliary ones with n_aux) and every EMIT
    kind. No instruction reads an EMIT's slot. The last three instructions read v[0]."""
    rng = np.random.default_rng(seed)
    leaves = [S.OP_LOCAL, S.OP_NEXT, S.OP_CONST] + ([S.OP_AUX_LOCAL, S.OP_AUX_NEXT] if n_aux else [])
    prog = np.zeros((n_instr, 4), dtype=np.uint16)
    vals = _Values(rng)
    for k in range(n_instr):
        tail = n_instr - k
        if k < len(leaves):
            op, a = _leaf(rng, leaves[k], n_cols, n_consts, n_aux)
            b = 0
        elif tail == 3:
            op, a, b = S.OP_MUL, 0, 0
        elif tail == 2:
            op, a, b = S.OP_SUB, k - 1, 0
        elif tail == 1 or rng.random() < 1 / emit_every:
            op, a, b = S.OP_EMIT, (k - 1 if tail == 1 else vals.pick(k)), int(rng.integers(4))
        elif rng.random() < 0.3:
            op, a = _leaf(rng, int(rng.choice(leaves)), n_cols, n_consts, n_aux)
            b = 0
        else:
            op, a, b = _arith(rng, vals, k)
        prog[k, :3] = op, a, b
        if op != S.OP_EMIT:
            vals.idx.append(k)
    return prog


def row_program(rng, n_instr, n_cols, n_consts, emits):
    """A row program of n_instr instructions whose EMITs are `emits` (roles, in order) on values drawn from the
    program, spread over it; every other instruction reads the trace (both rows), a constant or earlier values."""
    assert n_instr >= len(emits) + 2
    prog = np.zeros((n_instr, 4), dtype=np.uint16)
    at = set((np.sort(rng.choice(np.arange(2, n_instr - 1), len(emits) - 1, replace=False))).tolist()) | {n_instr - 1}
    vals = _Values(rng)
    roles = iter(emits)
    for k in range(n_instr):
        if k in at:
            op, a, b = S.OP_EMIT, vals.pick(k), next(roles)
        elif k < 2 or rng.random() < 0.35:
            op, a = _leaf(rng, [S.OP_LOCAL, S.OP_NEXT, S.OP_CONST][k] if k < 2 else
                          int(rng.choice([S.OP_LOCAL, S.OP_NEXT, S.OP_CONST])), n_cols, n_consts, 0)
            b = 0
        else:
            op, a, b = _arith(rng, vals, k)
        prog[k, :3] = op, a, b
        if op != S.OP_EMIT:
            vals.idx.append(k)
    return prog


def logup_lookup(rng, n_instr, n_looking, n_cols, n_consts):
    """One Lookup's row program: each looking column's value then its filter, the table, the frequencies (the roles in
    the order the kernel takes them: looking values and filters each in column order)."""
    emits = [LOGUP_LOOKED, LOGUP_FILTER] * n_looking + [LOGUP_TABLE, LOGUP_FREQUENCIES]
    return row_program(rng, n_instr, n_cols, n_consts, emits)


def ctl_group(rng, n_instr, values_per_entry, n_cols, n_consts):
    """One CTL group's row program: for each entry its values, then its filter."""
    emits = [r for nv in values_per_entry for r in [CTL_VALUE] * nv + [CTL_FILTER]]
    return row_program(rng, n_instr, n_cols, n_consts, emits)


def vp_program(seed, n_extra, widths, n_consts, n_terms, salted):
    """A gl_vp_instr program: first every register written once, in a random order, by every opcode; then n_extra
    instructions that overwrite registers (dst == a among them) while others keep older values, with CONST past 65 535,
    ADDC / MULC at 65 535, TERM n_terms - 1 and repeated terms, LOCAL of a salt column of commitment `salted`, NEXT of
    every commitment."""
    rng = np.random.default_rng(seed)
    prog = []
    written = []

    def src():
        r = rng.random()
        if r < 0.1:
            return written[0]
        if r < 0.2 and len(written) > 200:
            return written[int(rng.integers(0, len(written) - 180))]
        return written[-1 - int(rng.integers(min(len(written), 12)))]

    def leaf(op):
        if op in (VP_LOCAL, VP_NEXT):
            c = int(rng.integers(len(widths)))
            return op, c, int(rng.integers(widths[c]))
        if op == VP_CONST:
            i = int(rng.choice([0, 65535, 65536, n_consts - 1, int(rng.integers(n_consts))]))
            return op, i & 0xFFFF, i >> 16
        return op, 0, 0

    def arith(dst):
        op = int(rng.choice([VP_ADD, VP_SUB, VP_MUL, VP_ADDC, VP_MULC, VP_ADD, VP_MUL]))
        a = dst if (dst in written and rng.random() < 0.25) else src()
        if op in (VP_ADDC, VP_MULC):
            return op, a, int(rng.choice([65535, int(rng.integers(65536))]))
        return op, a, a if rng.random() < 0.15 else src()

    def emit(op, dst, a, b):
        prog.append((op, dst, a, b))
        if op != VP_TERM:
            if dst in written:
                written.remove(dst)
            written.append(dst)

    forced = [(VP_LOCAL, c, widths[c] - 1) for c in range(len(widths))]     # the salted one: its last salt column
    forced += [(VP_NEXT, c, 0) for c in range(len(widths))] + [(VP_X, 0, 0), (VP_L0, 0, 0)]
    forced += [(VP_CONST, 65535, 0), (VP_CONST, 0, 1), (VP_CONST, (n_consts - 1) & 0xFFFF, (n_consts - 1) >> 16)]
    order = rng.permutation(VP_MAX_REGS)
    for k, dst in enumerate(order):
        dst = int(dst)
        if k < len(forced):
            op, a, b = forced[k]
        elif rng.random() < 0.4:
            op, a, b = leaf(int(rng.choice([VP_LOCAL, VP_NEXT, VP_CONST, VP_X, VP_L0])))
        else:
            op, a, b = arith(dst)
        emit(op, dst, a, b)
    for k in range(n_extra):
        r = rng.random()
        if r < 0.2:
            t = int(rng.choice([0, 1, n_terms - 1, n_terms - 1, int(rng.integers(n_terms))]))
            emit(VP_TERM, int(rng.integers(VP_MAX_REGS)), src(), t)
        elif r < 0.35:
            op, a, b = leaf(int(rng.choice([VP_LOCAL, VP_NEXT, VP_CONST, VP_X, VP_L0])))
            emit(op, int(rng.integers(VP_MAX_REGS)), a, b)
        else:
            dst = int(rng.integers(VP_MAX_REGS))
            op, a, b = arith(dst)
            emit(op, dst, a, b)
    emit(VP_TERM, 0, src(), n_terms - 1)
    return np.array(prog, dtype=np.uint16)


# ------------------------------------------------------------------------------------------------------ evaluators
def row_emits(prog, trace, consts):
    """The row program on every row (NEXT: row (i + 1) mod n): the EMITs' (role, value row) in program order."""
    n = trace.shape[1]
    v, emits = {}, []
    for k, (op, a, b, _) in enumerate(prog):
        if op == S.OP_LOCAL:
            v[k] = trace[a]
        elif op == S.OP_NEXT:
            v[k] = np.roll(trace[a], -1)
        elif op == S.OP_CONST:
            v[k] = np.full(n, consts[a], dtype=np.uint64)
        elif op == S.OP_ADD:
            v[k] = G.add(v[a], v[b])
        elif op == S.OP_SUB:
            v[k] = G.sub(v[a], v[b])
        elif op == S.OP_MUL:
            v[k] = G.mul(v[a], v[b])
        else:
            emits.append((int(b), v[a]))
    return emits


def _single(k):
    """Column::single(k) and Filter::new_simple over it, for stark_twin's restatements."""
    col = NS(constant=0, linear_combination=[(k, 1)], next_row_linear_combination=[])
    return col, NS(products=[], constants=[col])


def logup_expected(prog, offsets, trace, consts, challenges, degree):
    """gl_stark_lookup_helpers' output: every lookup, every challenge, h_k then Z (stark_twin.helper_columns)."""
    out = []
    for l in range(len(offsets) - 1):
        emits = row_emits(prog[offsets[l]:offsets[l + 1]], trace, consts)
        by = {r: [v for role, v in emits if role == r] for r in range(4)}
        rows = np.stack(by[LOGUP_LOOKED] + by[LOGUP_FILTER] + by[LOGUP_TABLE] + by[LOGUP_FREQUENCIES])
        L = len(by[LOGUP_LOOKED])
        lookup = NS(columns=[_single(j)[0] for j in range(L)], filter_columns=[_single(L + j)[1] for j in range(L)],
                    table_column=_single(2 * L)[0], frequencies_column=_single(2 * L + 1)[0])
        for g in challenges:
            out += T.helper_columns(lookup, rows, int(g) % P, degree)[0]
    return np.stack(out)


def ctl_expected(prog, offsets, trace, consts, pairs, degree, zs_index):
    """gl_stark_ctl_helpers' output: the helper columns of every zs position in order, then one Z per position
    (stark_twin.partial_sums, ctl_aux)."""
    nch = len(pairs)
    per = {}
    for g in range(len(offsets) - 1):
        emits = row_emits(prog[offsets[g]:offsets[g + 1]], trace, consts)
        rows = np.stack([v for _, v in emits])
        entries, cols = [], []
        for k, (role, _) in enumerate(emits):
            if role == CTL_VALUE:
                cols.append(_single(k)[0])
            else:
                entries.append((cols, _single(k)[1]))
                cols = []
        for c, (beta, gamma) in enumerate(pairs):
            z = T.partial_sums(rows, entries, (int(beta) % P, int(gamma) % P), degree)
            per[g * nch + c] = dict(helpers=z[:-1], z=z[-1])
    at = {int(z): k for k, z in enumerate(zs_index)}
    return T.ctl_aux([per[at[z]] for z in range(len(zs_index))], trace.shape[1])


def _inv(a):
    return G.pow_scalar(a, P - 2)


def vp_expected(prog, local, consts, alphas, log_n, qd_bits):
    """gl_plonk_quotient_shard's values on the whole coset (n_alphas x size, natural order): the register program at
    every point x_i = shift * w_size^i, local[c] the commitment's (W, size) values there, the next row 2^qd_bits points
    on; X = x, L0 = Z_H(x) / (n (x - 1)), TERM t adds r * alpha^t; then / Z_H(x)."""
    n, size = 1 << log_n, 1 << (log_n + qd_bits)
    shift, w = E.coset_shift(), E.primitive_root_of_unity(log_n + qd_bits)
    x = G.mul(G.powers(w, size), np.uint64(shift))
    zh_c = [(pow(shift * pow(w, j, P), n, P) - 1) % P for j in range(1 << qd_bits)]
    zh = np.array(zh_c, dtype=np.uint64)[np.arange(size) & ((1 << qd_bits) - 1)]
    l0 = G.mul(zh, _inv(G.mul(G.sub(x, np.uint64(1)), np.uint64(n))))
    acc = [np.zeros(size, dtype=np.uint64) for _ in alphas]
    r = {}
    for op, dst, a, b in prog.tolist():
        if op == VP_LOCAL:
            v = local[a][b]
        elif op == VP_NEXT:
            v = np.roll(local[a][b], -(1 << qd_bits))
        elif op == VP_CONST:
            v = np.full(size, consts[a | b << 16], dtype=np.uint64)
        elif op == VP_X:
            v = x
        elif op == VP_L0:
            v = l0
        elif op == VP_ADD:
            v = G.add(r[a], r[b])
        elif op == VP_SUB:
            v = G.sub(r[a], r[b])
        elif op == VP_MUL:
            v = G.mul(r[a], r[b])
        elif op == VP_ADDC:
            v = G.add(r[a], np.uint64(consts[b]))
        elif op == VP_MULC:
            v = G.mul(r[a], np.uint64(consts[b]))
        else:
            acc = [G.add(s, G.mul(r[a], np.uint64(pow(int(al), b, P)))) for s, al in zip(acc, alphas)]
            continue
        r[dst] = v
    zi = np.array([pow(z, P - 2, P) for z in zh_c], dtype=np.uint64)[np.arange(size) & ((1 << qd_bits) - 1)]
    return np.stack([G.mul(s, zi) for s in acc])


# ------------------------------------------------------------------------------------------------------ cases
def logup_case(degree):
    """Three lookups back to back from offset 5 (the five instructions before are invalid and must not be read): 16
    looking columns in 256 instructions, 5 in 100, 1 in 40; 4 challenges."""
    rng = np.random.default_rng(0x106 + degree)
    n_cols, n_consts = 6, 9
    progs = [logup_lookup(rng, LOGUP_MAX_INSTR, LOGUP_MAX_COLUMNS, n_cols, n_consts),
             logup_lookup(rng, 100, 5, n_cols, n_consts), logup_lookup(rng, 40, 1, n_cols, n_consts)]
    junk = np.full((5, 4), 0xFFFF, dtype=np.uint16)
    prog = np.ascontiguousarray(np.concatenate([junk] + progs))
    offsets = np.cumsum([5] + [len(p) for p in progs]).astype(np.uint32)
    consts = synth(0x107, (n_consts,))
    challenges = [int(v) for v in synth(0x108 + degree, (MAX_ALPHAS,))]
    return prog, offsets, consts, challenges, n_cols


def _logup_num_columns(offsets, prog, nch, degree):
    chunk = degree - 1 if degree > 1 else 1
    total = 0
    for l in range(len(offsets) - 1):
        p = prog[offsets[l]:offsets[l + 1]]
        looked = int(((p[:, 0] == S.OP_EMIT) & (p[:, 2] == LOGUP_LOOKED)).sum())
        total += nch * (-(-looked // chunk) + 1)
    return total


def ctl_case(degree):
    """16 groups from offset 7: one of 8 entries, one entry of 32 values, one of 256 instructions, single-entry groups
    among the others; 4 challenges; a random zs_index permutation."""
    rng = np.random.default_rng(0xC71 + degree)
    n_cols, n_consts = 7, 5
    shapes = [([1, 3, 2, 1, 4, 1, 2, 2], 80), ([CTL_MAX_VALUES], 60), ([3, 2, 2], CTL_MAX_INSTR)]
    for g in range(CTL_MAX_GROUPS - 3):
        k = [1, 2, 1, 3, 1][g % 5]
        shapes.append(([int(v) for v in rng.integers(1, 5, k)], int(rng.integers(12, 40)) + 4 * k))
    assert max(len(s) for s, _ in shapes) == CTL_MAX_ENTRIES
    progs = [ctl_group(rng, n, s, n_cols, n_consts) for s, n in shapes]
    junk = np.full((7, 4), 0xFFFF, dtype=np.uint16)
    prog = np.ascontiguousarray(np.concatenate([junk] + progs))
    offsets = np.cumsum([7] + [len(p) for p in progs]).astype(np.uint32)
    consts = synth(0xC72, (n_consts,))
    pairs = [tuple(int(v) for v in synth(0xC73 + c, (2,))) for c in range(MAX_ALPHAS)]
    zs_index = rng.permutation(CTL_MAX_GROUPS * MAX_ALPHAS).astype(np.uint32)
    return prog, offsets, consts, pairs, zs_index, n_cols, [len(s) for s, _ in shapes]


def _ctl_num_columns(entries, nch, degree):
    chunk = degree - 1 if degree > 1 else 1
    return sum(-(-e // chunk) if e > 1 else 0 for e in entries) * nch + len(entries) * nch


VP_WIDTHS, VP_SALTED = [3, 9, 1, 5], 1


def vp_case(seed):
    prog = vp_program(seed, 1500, [w + (SALT if c == VP_SALTED else 0) for c, w in enumerate(VP_WIDTHS)], VP_CONSTS,
                      VP_MAX_TERMS, VP_SALTED)
    consts = synth(seed + 1, (VP_CONSTS,))
    alphas = [int(v) for v in synth(seed + 2, (MAX_ALPHAS,))]
    return np.ascontiguousarray(prog), consts, alphas


def test_generators_reach_every_limit_and_opcode():
    """The programs the device and host tests run hold what the file's docstring promises."""
    p = stark_program(0x5A, STARK_MAX_INSTR, 5, 4, n_aux=2)
    assert len(p) == STARK_MAX_INSTR and set(p[:, 0]) == set(range(9))
    assert set(p[p[:, 0] == S.OP_EMIT, 2]) == set(range(4))
    assert (p[-3:-1, 2] == 0).all() and (p[-3, 1] == 0) and ((p[:, 0] >= 3) & (p[:, 0] <= 5) & (p[:, 1] == p[:, 2])).any()
    ar = (p[:, 0] >= S.OP_ADD) & (p[:, 0] <= S.OP_EMIT)
    assert (np.arange(len(p))[ar] - p[ar, 1] >= 200).any()
    prog, offsets, *_ = logup_case(3)
    assert offsets[0] == 5 and offsets[1] - offsets[0] == LOGUP_MAX_INSTR
    assert ((prog[5:5 + LOGUP_MAX_INSTR, 0] == S.OP_EMIT) & (prog[5:5 + LOGUP_MAX_INSTR, 2] == 0)).sum() == 16
    prog, offsets, _, _, zs, _, entries = ctl_case(9)
    assert len(entries) == CTL_MAX_GROUPS and max(entries) == CTL_MAX_ENTRIES and 1 in entries
    assert (np.diff(offsets) == CTL_MAX_INSTR).any() and offsets[0] == 7 and not (zs == np.arange(len(zs))).all()
    vp, consts, _ = vp_case(0x7A0)
    assert set(vp[:, 0]) == set(range(11))
    dst = vp[vp[:, 0] != VP_TERM, 1]
    assert set(dst) == set(range(VP_MAX_REGS)) and len(dst) > VP_MAX_REGS
    nd = vp[:, 0] != VP_TERM
    assert (nd & (vp[:, 1] == vp[:, 2]) & np.isin(vp[:, 0], [VP_ADD, VP_SUB, VP_MUL, VP_ADDC, VP_MULC])).any()
    ci = vp[vp[:, 0] == VP_CONST, 2].astype(np.int64) | (vp[vp[:, 0] == VP_CONST, 3].astype(np.int64) << 16)
    assert ci.max() == VP_CONSTS - 1 and (ci < 65536).any() and 65535 in ci and 65536 in ci
    assert 65535 in vp[np.isin(vp[:, 0], [VP_ADDC, VP_MULC]), 3]
    terms = vp[vp[:, 0] == VP_TERM, 3]
    assert VP_MAX_TERMS - 1 in terms and len(terms) > len(set(terms))
    loc = vp[vp[:, 0] == VP_LOCAL]
    assert ((loc[:, 2] == VP_SALTED) & (loc[:, 3] >= VP_WIDTHS[VP_SALTED])).any()
    assert set(vp[vp[:, 0] == VP_NEXT, 2]) == set(range(VP_MAX_COMMITS))


# ------------------------------------------------------------------------------------------------------ host runs
vp, u32, sz = C.c_void_p, C.c_uint32, C.c_size_t
EMU_ARGS = {
    "logup_emu": ("emu_stark_lookup_helpers", [vp, sz, u32, vp, vp, u32, vp, vp, u32, u32, vp]),
    "ctl_emu": ("emu_stark_ctl_helpers", [vp, sz, u32, vp, vp, u32, vp, vp, u32, u32, vp, vp]),
    "vanishing_emu": ("emu_plonk_quotient_values", [vp, vp, u32, u32, u32, u32, vp, u32, vp, vp, u32, u32, vp]),
}


@pytest.fixture(scope="module")
def emus(tmp_path_factory):
    out = {}
    for name, (fn, argtypes) in EMU_ARGS.items():
        so = str(tmp_path_factory.mktemp(name) / ("lib%s.so" % name))
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-DGL_FORCE_32BIT_PATH", "-shared", "-fPIC", "-o", so,
                               os.path.join(ROOT, "tests", "emu", name + ".cpp")])
        f = getattr(C.CDLL(so), fn)
        f.argtypes = argtypes
        out[name] = f
    return out


@pytest.mark.parametrize("degree", [0, 2, 3, 17])
def test_logup_programs_on_host(emus, degree):
    prog, offsets, consts, challenges, n_cols = logup_case(degree)
    log_n = 6
    trace = synth(0x109, (n_cols, 1 << log_n))
    want = logup_expected(prog, offsets, trace, consts, challenges, degree)
    assert want.shape[0] == _logup_num_columns(offsets, prog, len(challenges), degree)
    got = np.zeros_like(want)
    ch = np.array(challenges, dtype=np.uint64)
    rc = emus["logup_emu"](trace.ctypes.data, 1 << log_n, log_n, prog.ctypes.data,
                                    offsets.ctypes.data, len(offsets) - 1, consts.ctypes.data, ch.ctypes.data,
                                    len(ch), degree, got.ctypes.data)
    assert rc == 0
    bad = np.argwhere(got != want)
    assert len(bad) == 0, "first differing (column, row): %s of %s" % (bad[0], want.shape)


@pytest.mark.parametrize("degree", [0, 3, 9])
def test_ctl_programs_on_host(emus, degree):
    prog, offsets, consts, pairs, zs_index, n_cols, entries = ctl_case(degree)
    log_n = 5
    trace = synth(0xC74, (n_cols, 1 << log_n))
    want = ctl_expected(prog, offsets, trace, consts, pairs, degree, zs_index)
    assert want.shape[0] == _ctl_num_columns(entries, len(pairs), degree)
    got = np.zeros_like(want)
    ch = np.array([v % P for pr in pairs for v in pr], dtype=np.uint64)
    rc = emus["ctl_emu"](trace.ctypes.data, 1 << log_n, log_n, prog.ctypes.data,
                                 offsets.ctypes.data, len(offsets) - 1, consts.ctypes.data, ch.ctypes.data, len(pairs),
                                 degree, zs_index.ctypes.data, got.ctypes.data)
    assert rc == 0
    bad = np.argwhere(got != want)
    assert len(bad) == 0, "first differing (column, row): %s of %s" % (bad[0], want.shape)


@pytest.mark.parametrize("qdf", [2, 3, 5, 8])
def test_vanishing_programs_on_host(emus, qdf):
    """The register program on random leaves (the interpreter reads leaf rows, whatever they hold): leaf row j of the
    first `size` holds point bitrev(j)."""
    log_n, rate_bits = 4, 3
    qd_bits = (qdf - 1).bit_length()
    size_log = log_n + qd_bits
    prog, consts, alphas = vp_case(0x7A0 + qdf)
    widths = [w + (SALT if c == VP_SALTED else 0) for c, w in enumerate(VP_WIDTHS)]
    leaves = [np.ascontiguousarray(synth(0x7B0 + c, (w, 1 << size_log))) for c, w in enumerate(widths)]
    local = [lv[:, _brev(size_log)] for lv in leaves]
    want = vp_expected(prog, local, consts, alphas, log_n, qd_bits)
    got = np.zeros_like(want)
    ptrs = (C.c_void_p * VP_MAX_COMMITS)(*[lv.ctypes.data for lv in leaves])
    strides = (C.c_size_t * VP_MAX_COMMITS)(*[1 << size_log] * VP_MAX_COMMITS)
    al = np.array(alphas, dtype=np.uint64)
    rc = emus["vanishing_emu"](ptrs, strides, VP_MAX_COMMITS, rate_bits, log_n, qd_bits, prog.ctypes.data,
                                     len(prog), consts.ctypes.data, al.ctypes.data, len(al), VP_MAX_TERMS,
                                     got.ctypes.data)
    assert rc == 0
    bad = np.argwhere(got != want)
    assert len(bad) == 0, "first differing (alpha, point): %s of %s" % (bad[0], want.shape)


# ------------------------------------------------------------------------------------------------------ GPU
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


def _to_device(a):
    import torch

    dev = torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return dev


def _host(t):
    return t.cpu().numpy().view(np.uint64)


def coset_values(batch, size_log):
    """The batch's values on the quotient coset of 2^size_log points, natural order, from its own leaves ((W, size))."""
    rows = batch.merkle_tree.get_rows(0, 1 << size_log)
    return np.ascontiguousarray(rows[_brev(size_log)].T)


def _assert_same(got, want, what):
    bad = np.argwhere(got != want)
    assert len(bad) == 0, "%s: first differing %s of %s" % (what, bad[0], want.shape)


# (log_n, rate_bits, quotient degree factor, instructions, alphas, auxiliary columns): 512 instructions at every factor
# 1..8 on a coset of up to 256 points; log_n 3, where one partial CTA covers the coset; 2^17 points at log_n 16
STARK_CASES = [(5, 3, q, STARK_MAX_INSTR, (1, MAX_ALPHAS)[q % 2], 2 * (q % 3 == 0)) for q in range(1, MAX_QD + 1)]
STARK_CASES += [(3, 3, 8, STARK_MAX_INSTR, MAX_ALPHAS, 2), (3, 2, 3, 300, 1, 0), (16, 1, 2, 160, 2, 1)]


def _stark_call(ctx, fn, trace, aux, prog, consts, alphas, qdf, out):
    L = N.lib()
    al = np.array(alphas, dtype=np.uint64)
    args = (prog.ctypes.data, len(prog), N.np_ptr(consts), len(consts), N.np_ptr(al), len(al), qdf,
            N.vp(out.data_ptr()))
    if fn == "whole":
        if aux is None:
            return L.gl_stark_quotient(ctx.h, trace.h, *args)
        return L.gl_stark_quotient_aux(ctx.h, trace.h, aux.h, *args)
    return L.gl_stark_quotient_shard(ctx.h, trace.h, aux.h if aux is not None else None, *args)


def _coset_fft(oracle, coeffs):
    return np.stack([oracle.coset_fft(np.ascontiguousarray(c), E.coset_shift()) for c in coeffs])


@pytest.mark.gpu
@pytest.mark.parametrize("log_n,rate_bits,qdf,n_instr,n_alphas,n_aux", STARK_CASES)
def test_stark_quotient_random_programs(pb, oracle, log_n, rate_bits, qdf, n_instr, n_alphas, n_aux):
    """Power-of-two factors: gl_stark_quotient[_aux]'s coefficients, back on the coset, against the evaluator. Other
    factors: gl_stark_quotient_shard's values on the whole handle (shard 0 of 1); gl_stark_quotient refuses the random
    program ("Quotient has failed") and accepts a degree-correct one (b = a^(qdf + 1) row by row)."""
    import torch

    ctx = pb.default_context()
    qd_bits = (qdf - 1).bit_length()
    n, size_log = 1 << log_n, log_n + qd_bits
    n_cols, n_consts = 5, 6
    prog = stark_program(0x57A + 31 * log_n + qdf, n_instr, n_cols, n_consts, n_aux)
    consts = synth(0x57B, (n_consts,))
    alphas = [int(v) for v in synth(0x57C + qdf, (n_alphas,))]
    tc = pb.PolynomialBatch.from_values(synth(0x57D, (n_cols, n)), rate_bits, False, 2)
    ac = pb.PolynomialBatch.from_values(synth(0x57E, (n_aux, n)), rate_bits, False, 2) if n_aux else None
    b = NS(instrs=[tuple(int(x) for x in r[:3]) for r in prog])
    tv, av = coset_values(tc, size_log), coset_values(ac, size_log) if n_aux else None
    out = torch.empty((n_alphas, 1 << size_log), dtype=torch.int64, device="cuda")
    pow2 = qdf & (qdf - 1) == 0
    N.check(_stark_call(ctx, "whole" if pow2 else "shard", tc, ac, prog, consts, alphas, qdf, out), ctx.h)
    q = _host(out)
    if pow2:
        q = _coset_fft(oracle, q)
    check_quotient_values(b, consts, alphas, q, tv, av, log_n, qd_bits)
    if not pow2:
        assert _stark_call(ctx, "whole", tc, ac, prog, consts, alphas, qdf, out) == N.GL_ERR_BAD_ARG
        assert b"Quotient has failed" in N.lib().gl_last_error(ctx.h)
        # C = a^d - b, d = qdf + 1, has degree d (n - 1): its quotient has degree below qdf n. Value k >= 2 is a^k.
        d = qdf + 1
        a = synth(0x57F, (n,))
        good = pb.PolynomialBatch.from_values(np.stack([a, G.pow_scalar(a, d)]), rate_bits, False, 2)
        gp = [(S.OP_LOCAL, 0, 0), (S.OP_LOCAL, 1, 0), (S.OP_MUL, 0, 0)] + [(S.OP_MUL, k - 1, 0) for k in range(3, d + 1)]
        gp += [(S.OP_SUB, d, 1), (S.OP_EMIT, d + 1, S.KIND_CONSTRAINT)]
        gp = np.array([g + (0,) for g in gp], dtype=np.uint16)
        N.check(_stark_call(ctx, "whole", good, None, gp, consts, alphas, qdf, out), ctx.h)
        gq = _host(out)
        assert not gq[:, qdf * n:].any()
        check_quotient_values(NS(instrs=[tuple(int(x) for x in r[:3]) for r in gp]), consts, alphas,
                              _coset_fft(oracle, gq), coset_values(good, size_log), None, log_n, qd_bits)
        good.close()
    for c in (tc, ac):
        if c is not None:
            c.close()


@pytest.mark.gpu
def test_stark_quotient_non_resident_and_sharded_equal_whole(pb):
    """One random 512-instruction program with auxiliary reads, quotient degree factor 2 at rate 2 (the quotient coset
    is not the LDE coset): non-resident handles of 2 and 4 LDE blocks, and 2 and 4 row-block shards on one GPU through
    gl_stark_quotient_from_shards, equal the resident whole result word for word."""
    import torch

    ctx = pb.default_context()
    L = N.lib()
    log_n, rate_bits, qdf, n_cols, n_aux, n_consts = 7, 2, 2, 5, 2, 6
    size = 2 << log_n
    prog = stark_program(0x5B5, STARK_MAX_INSTR, n_cols, n_consts, n_aux)
    consts = synth(0x5B6, (n_consts,))
    alphas = [int(v) for v in synth(0x5B7, (3,))]
    tv, avals = synth(0x5B8, (n_cols, 1 << log_n)), synth(0x5B9, (n_aux, 1 << log_n))

    def commit(**kw):
        return (pb.PolynomialBatch.from_values(tv, rate_bits, False, 2, **kw),
                pb.PolynomialBatch.from_values(avals, rate_bits, False, 2, **kw))

    def whole(tc, ac):
        out = torch.empty((len(alphas), size), dtype=torch.int64, device="cuda")
        N.check(_stark_call(ctx, "whole", tc, ac, prog, consts, alphas, qdf, out), ctx.h)
        return _host(out)

    tc, ac = commit()
    want = whole(tc, ac)
    tc.close(), ac.close()
    for blocks in (2, 4):
        tc, ac = commit(lde_blocks=blocks)
        _assert_same(whole(tc, ac), want, "%d LDE blocks" % blocks)
        tc.close(), ac.close()
    for G_ in (2, 4):
        values = torch.empty((G_, len(alphas), size // G_), dtype=torch.int64, device="cuda")
        for g in range(G_):
            tc, ac = commit(shard=(g, G_))
            N.check(_stark_call(ctx, "shard", tc, ac, prog, consts, alphas, qdf, values[g]), ctx.h)
            tc.close(), ac.close()
        out = torch.empty((len(alphas), size), dtype=torch.int64, device="cuda")
        N.check(L.gl_stark_quotient_from_shards(ctx.h, N.vp(values.data_ptr()), G_, len(alphas), log_n, qdf,
                                                N.vp(out.data_ptr())), ctx.h)
        _assert_same(_host(out), want, "%d shards" % G_)


@pytest.mark.gpu
@pytest.mark.parametrize("degree", [0, 2, 3, 17])
def test_logup_helpers_random_programs(pb, degree):
    """16 looking columns in 256 instructions, 4 challenges, three lookups from offset 5, NEXT reads on row n - 1."""
    import torch

    ctx = pb.default_context()
    prog, offsets, consts, challenges, n_cols = logup_case(degree)
    log_n = 8
    trace = synth(0x10A, (n_cols, 1 << log_n))
    want = logup_expected(prog, offsets, trace, consts, challenges, degree)
    dev = _to_device(trace)
    out = torch.empty(want.shape, dtype=torch.int64, device="cuda")
    ch = np.array(challenges, dtype=np.uint64)
    N.check(N.lib().gl_stark_lookup_helpers(ctx.h, N.vp(dev.data_ptr()), 1 << log_n, n_cols, log_n, prog.ctypes.data,
                                            offsets.ctypes.data_as(N.u32p), len(offsets) - 1, N.np_ptr(consts),
                                            len(consts), N.np_ptr(ch), len(ch), degree, N.vp(out.data_ptr())), ctx.h)
    _assert_same(_host(out), want, "logUp columns")


@pytest.mark.gpu
@pytest.mark.parametrize("degree", [0, 3, 9])
def test_ctl_helpers_random_programs(pb, degree):
    """16 groups (8 entries, a 32-value entry, 256 instructions, single entries) from offset 7, 4 challenges, a random
    zs_index."""
    import torch

    ctx = pb.default_context()
    prog, offsets, consts, pairs, zs_index, n_cols, _ = ctl_case(degree)
    log_n = 8
    trace = synth(0xC75, (n_cols, 1 << log_n))
    want = ctl_expected(prog, offsets, trace, consts, pairs, degree, zs_index)
    dev = _to_device(trace)
    out = torch.empty(want.shape, dtype=torch.int64, device="cuda")
    ch = np.array([v % P for pr in pairs for v in pr], dtype=np.uint64)
    N.check(N.lib().gl_stark_ctl_helpers(ctx.h, N.vp(dev.data_ptr()), 1 << log_n, n_cols, log_n, prog.ctypes.data,
                                         offsets.ctypes.data_as(N.u32p), len(offsets) - 1, N.np_ptr(consts),
                                         len(consts), N.np_ptr(ch), len(pairs), degree,
                                         zs_index.ctypes.data_as(N.u32p), N.vp(out.data_ptr())), ctx.h)
    _assert_same(_host(out), want, "CTL columns")


@pytest.mark.gpu
@pytest.mark.parametrize("qdf", [2, 3, 5, 8])
def test_plonk_quotient_random_programs(pb, oracle, qdf):
    """Four commitments of widths 3, 9 (salted), 1 and 5 at rate_bits 3; all 256 registers, 70 000 constants, 65 536
    terms, 4 alphas: gl_plonk_quotient_shard's values on whole handles against the evaluator, and for power-of-two
    factors gl_plonk_quotient's coefficients against their coset iFFT."""
    import torch

    ctx = pb.default_context()
    L = N.lib()
    log_n, rate_bits = 5, 3
    qd_bits = (qdf - 1).bit_length()
    size_log = log_n + qd_bits
    prog, consts, alphas = vp_case(0x7C0 + qdf)
    commits = [pb.PolynomialBatch.from_values(synth(0x7D0 + c, (w, 1 << log_n)), rate_bits, c == VP_SALTED, 2)
               for c, w in enumerate(VP_WIDTHS)]
    want = vp_expected(prog, [coset_values(c, size_log) for c in commits], consts, alphas, log_n, qd_bits)
    handles = (C.c_void_p * len(commits))(*[c.h for c in commits])
    al = np.array(alphas, dtype=np.uint64)
    out = torch.empty(want.shape, dtype=torch.int64, device="cuda")

    def call(fn):
        return fn(ctx.h, handles, len(commits), prog.ctypes.data, len(prog), N.np_ptr(consts), len(consts), N.np_ptr(al),
                  len(al), VP_MAX_TERMS, qdf, N.vp(out.data_ptr()))

    N.check(call(L.gl_plonk_quotient_shard), ctx.h)
    _assert_same(_host(out), want, "values")
    if qdf & (qdf - 1) == 0:
        N.check(call(L.gl_plonk_quotient), ctx.h)
        coeffs = np.stack([oracle.coset_ifft(np.ascontiguousarray(v), E.coset_shift()) for v in want])
        _assert_same(_host(out), coeffs, "coefficients")
    for c in commits:
        c.close()
