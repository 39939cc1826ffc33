"""starky's cross-table lookups (starky/src/cross_table_lookup.rs): several STARK tables proved together, tied by CTLs
whose looking tables' filtered, combined rows must be the looked table's. TableWithColumns / CrossTableLookup, the
per-table CTL data (CtlZData / CtlData) whose helper and Z columns gl_stark_ctl_helpers writes on the device, the
CtlCheckVars a proof's openings give the constraints, the multi-STARK prover prove_with_ctls with its transcript and
MultiStarkProof.get_challenges replaying it, and check_ctls (debug_utils), the multiset check on host traces. The CTL
constraints themselves (eval_cross_table_lookup_checks) are recorded into a Stark's constraint program by stark.py;
verify_cross_table_lookups is a verifier step and, like the other verifiers, is restated by the tests."""
from collections import Counter

import numpy as np

from . import _native as N
from . import field as F
from .lookup import Column, Filter, GrandProductChallenge, helper_chunk_size  # noqa: F401 (re-exported for users)

CTL_VALUE, CTL_FILTER = 0, 1


class TableWithColumns:
    """TableWithColumns<F> (cross_table_lookup.rs:63-82): a table index, the tuple's columns (lookup.Column) and a
    filter (lookup.Filter) selecting the rows."""

    def __init__(self, table, columns, filter):
        self.table, self.columns, self.filter = int(table), list(columns), filter


class CrossTableLookup:
    """CrossTableLookup<F> (cross_table_lookup.rs:84-142): the looking tables' selected tuples, all together, are the
    looked table's as a multiset."""

    def __init__(self, looking_tables, looked_table):
        self.looking_tables, self.looked_table = list(looking_tables), looked_table
        if not all(len(t.columns) == len(looked_table.columns) for t in self.looking_tables):
            raise N.ShapeError("assertion failed: every looking table has the looked table's width (%d columns)"
                               % len(looked_table.columns))

    @staticmethod
    def num_ctl_helpers_zs_all(ctls, table, num_challenges, constraint_degree):
        """cross_table_lookup.rs:110-141: (helper columns of `table` over all CTLs and challenges, its Z columns, its
        helper columns per CTL for one challenge)."""
        num_helpers = num_ctls = 0
        by_ctl = [0] * len(ctls)
        for i, ctl in enumerate(ctls):
            appearances = sum(t.table == table for t in [ctl.looked_table] + ctl.looking_tables)
            if appearances > 1:
                if constraint_degree < 2:
                    raise N.ShapeError("attempt to divide by zero: table %d has CTL helper columns at constraint "
                                       "degree %d" % (table, constraint_degree))
                by_ctl[i] = -(-appearances // (constraint_degree - 1))
                num_helpers += by_ctl[i]
            if appearances > 0:
                num_ctls += 1
        return num_helpers * num_challenges, num_ctls * num_challenges, by_ctl


class CtlZData:
    """CtlZData<F> (cross_table_lookup.rs:151-186): one Z polynomial of a table -- one CTL, one challenge, the table's
    entries in it -- with its helper columns. helper_columns / z are rows of the table's auxiliary values (device
    tensor views when made by the prover)."""

    def __init__(self, helper_columns, z, challenge, columns, filter):
        self.helper_columns, self.z, self.challenge = helper_columns, z, challenge
        self.columns, self.filter = columns, filter


class CtlData:
    """CtlData<F> (cross_table_lookup.rs:144-222): a table's CtlZData in the reference's order. `auxiliary`, when set,
    is the table's whole auxiliary-values buffer, [lookup helpers | CTL helpers | CTL Zs], that the CTL columns were
    written into and that the auxiliary commitment reads."""

    def __init__(self, zs_columns, auxiliary=None, num_lookup_columns=0):
        self.zs_columns, self.auxiliary, self.num_lookup_columns = list(zs_columns), auxiliary, num_lookup_columns

    def ctl_helper_polys(self):
        return [h for z in self.zs_columns for h in z.helper_columns]

    def ctl_z_polys(self):
        return [z.z for z in self.zs_columns]

    def num_ctl_helper_polys(self):
        return [len(z.helper_columns) for z in self.zs_columns]


class CtlCheckVars:
    """CtlCheckVars (cross_table_lookup.rs:416-548): one Z polynomial's openings (helper columns at zeta, Z at zeta and
    g * zeta, as F_{p^2} pairs), its challenge, and the entries' columns and filters."""

    def __init__(self, helper_columns, local_z, next_z, challenges, columns, filter):
        self.helper_columns, self.local_z, self.next_z = list(helper_columns), local_z, next_z
        self.challenges, self.columns, self.filter = challenges, list(columns), list(filter)

    @classmethod
    def from_proof(cls, table_idx, proof, cross_table_lookups, ctl_challenges, num_lookup_columns,
                   total_num_helper_columns, num_helper_ctl_columns):
        """cross_table_lookup.rs:443-547: the table's CTL openings, skipping its lookup helper columns."""
        o = proof.openings
        if o.auxiliary_polys is None or o.auxiliary_polys_next is None:
            raise N.ShapeError("We cannot have CTLs without auxiliary polynomials.")
        zs = list(zip(o.auxiliary_polys[num_lookup_columns:], o.auxiliary_polys_next[num_lookup_columns:]))
        z_index = start = 0
        out = []
        for i, ctl in enumerate(cross_table_lookups):
            for challenge in ctl_challenges:
                mine = [t for t in ctl.looking_tables if t.table == table_idx]
                if mine:
                    local_z, next_z = zs[total_num_helper_columns + z_index]
                    helpers = [h for h, _ in zs[start:start + num_helper_ctl_columns[i]]]
                    start += num_helper_ctl_columns[i]
                    z_index += 1
                    out.append(cls(helpers, local_z, next_z, challenge, [t.columns for t in mine],
                                   [t.filter for t in mine]))
                if ctl.looked_table.table == table_idx:
                    local_z, next_z = zs[total_num_helper_columns + z_index]
                    z_index += 1
                    out.append(cls([], local_z, next_z, challenge, [ctl.looked_table.columns],
                                   [ctl.looked_table.filter]))
        return out


def combine(vars, values, beta, gamma):
    """GrandProductChallenge::combine (lookup.rs:457-464) recorded: reduce_with_powers(values, beta) + gamma."""
    if not values:
        return gamma
    acc = values[-1]
    for v in reversed(values[:-1]):
        acc = acc * beta + v
    return acc + gamma


def eval_cross_table_lookup_checks(vars, ctl_vars, consumer, constraint_degree, num_lookup_columns):
    """eval_cross_table_lookup_checks (cross_table_lookup.rs:558-629) recorded into a ConstraintBuilder: for every CTL
    Z, its helper-column constraints (lookup.eval_helper_columns with the tuple's combine), then Z's last-row value and
    transition -- Z - sum h and Z - Z' - sum h with helper columns, else the one- or two-entry forms with combine. The
    columns and filters are read with eval_with_next; the auxiliary columns after the lookup helpers are the CTL helper
    columns of every Z, then the Zs; each Z's (beta, gamma) is bound at evaluation time (ctl_challenge)."""
    from .lookup import eval_helper_columns

    total = sum(len(v.helper_columns) for v in ctl_vars)
    start = num_lookup_columns
    for i, v in enumerate(ctl_vars):
        consumer.begin_scope("CTL Z %d" % i)
        beta, gamma = vars.ctl_challenge(i)
        comb = lambda values: combine(vars, values, beta, gamma)  # noqa: E731
        evals = [[c.eval_with_next(vars) for c in cols] for cols in v.columns]
        helpers = [vars.aux_local(start + k) for k in range(len(v.helper_columns))]
        start += len(helpers)
        local_z = vars.aux_local(num_lookup_columns + total + i)
        next_z = vars.aux_next(num_lookup_columns + total + i)
        eval_helper_columns(v.filter, evals, helpers, constraint_degree, None, consumer, vars, combine=comb)
        if helpers:
            h_sum = helpers[0]
            for h in helpers[1:]:
                h_sum = h_sum + h
            consumer.constraint_last_row(local_z - h_sum)
            consumer.constraint_transition(local_z - next_z - h_sum)
        elif len(v.columns) > 1:
            combin0, combin1 = comb(evals[0]), comb(evals[1])
            f0, f1 = v.filter[0].eval_filter(vars), v.filter[1].eval_filter(vars)
            consumer.constraint_last_row(combin0 * combin1 * local_z - f0 * combin1 - f1 * combin0)
            consumer.constraint_transition(combin0 * combin1 * (local_z - next_z) - f0 * combin1 - f1 * combin0)
        else:
            combin0 = comb(evals[0])
            f0 = v.filter[0].eval_filter(vars)
            consumer.constraint_last_row(combin0 * local_z - f0)
            consumer.constraint_transition(combin0 * (local_z - next_z) - f0)


def table_groups(cross_table_lookups, table):
    """The table's CtlZData groups for one challenge, in the reference's zs_columns order (cross_table_lookup_data,
    cross_table_lookup.rs:270-339): per CTL, its looking entries (one group: check_ctl_shapes keeps them consecutive),
    then its looked entry. Returns [(ctl index, [TableWithColumns])]."""
    out = []
    for i, ctl in enumerate(cross_table_lookups):
        mine = [t for t in ctl.looking_tables if t.table == table]
        if mine:
            out.append((i, mine))
        if ctl.looked_table.table == table:
            out.append((i, [ctl.looked_table]))
    return out


def ctl_row_programs(groups, num_columns):
    """The row programs of gl_stark_ctl_helpers (include/plonky2_b200.h): per group, per entry, the tuple's columns
    then the filter (eval_table: current and next row), emitted by role. Returns (instructions (StarkInstr array),
    offsets (uint32, len(groups) + 1), constants (uint64))."""
    from .stark import OP_CONST, OP_EMIT, ConstraintBuilder, StarkInstr

    consts, instrs, offsets = [], [], [0]
    for _, entries in groups:
        b = ConstraintBuilder(num_columns, 0)
        for t in entries:
            for col in t.columns:
                b._push(OP_EMIT, col.eval_with_next(b).idx, CTL_VALUE)
            b._push(OP_EMIT, t.filter.eval_filter(b).idx, CTL_FILTER)
        for op, a, c in b.instrs:                     # the groups share one constant table
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


def zs_layout(groups, num_challenges, constraint_degree):
    """Where each (group, challenge) lands in the table's CTL columns: (zs_index (uint32, g * num_challenges + c ->
    zs position), helper columns per group, total helper columns)."""
    chunk = helper_chunk_size(constraint_degree)
    num_h = [-(-len(entries) // chunk) if len(entries) > 1 else 0 for _, entries in groups]
    zs_index = np.zeros(len(groups) * num_challenges, dtype=np.uint32)
    pos = 0
    for i in sorted({ctl for ctl, _ in groups}):
        for c in range(num_challenges):
            for g, (ctl, _) in enumerate(groups):
                if ctl == i:
                    zs_index[g * num_challenges + c] = pos
                    pos += 1
    return zs_index, num_h, sum(num_h) * num_challenges


def compute_ctl_helper_columns(trace, groups, ctl_challenges, constraint_degree, ctx, out):
    """cross_table_lookup_data for one table (cross_table_lookup.rs:270-414) on the device: every CTL helper and Z
    column of the table, for every group and challenge, written into `out` -- a (helpers + Zs, n) int64 CUDA tensor
    view, ctl_helper_polys() then ctl_z_polys() -- from the trace values `trace`, a (COLUMNS, n) int64 CUDA tensor read
    in place."""
    cols, n = trace.shape
    prog, offsets, consts = ctl_row_programs(groups, cols)
    zs_index, _, num_helpers = zs_layout(groups, len(ctl_challenges), constraint_degree)
    if tuple(out.shape) != (num_helpers + len(zs_index), n) or not out.is_contiguous():
        raise N.ShapeError("the CTL output must be a contiguous (%d, %d) tensor" % (num_helpers + len(zs_index), n))
    ch = np.array([int(v) % F.ORDER for c in ctl_challenges for v in (c.beta, c.gamma)], dtype=np.uint64)
    ctx.after_caller()
    N.check(N.lib().gl_stark_ctl_helpers(ctx.h, N.vp(trace.data_ptr()), n, cols, F.log2_strict(n), prog,
                                         offsets.ctypes.data_as(N.u32p), len(offsets) - 1,
                                         N.np_ptr(consts) if len(consts) else None, len(consts), N.np_ptr(ch),
                                         len(ctl_challenges), constraint_degree, zs_index.ctypes.data_as(N.u32p),
                                         N.vp(out.data_ptr())), ctx.h)
    ctx.synchronize()


def _alloc_auxiliary(num_rows, n, device_trace):
    """The table's auxiliary-values buffer on the trace's device."""
    import torch

    return torch.empty((num_rows, n), dtype=torch.int64, device=device_trace.device)


def cross_table_lookup_data(traces, cross_table_lookups, ctl_challenges, max_constraint_degree, ctx,
                            num_lookup_columns=None):
    """cross_table_lookup_data (cross_table_lookup.rs:270-339) on the device, one gl_stark_ctl_helpers call per table
    taking part in a CTL. traces: (COLUMNS, n) int64 CUDA tensors. Each table's CTL columns go into a fresh auxiliary
    buffer after num_lookup_columns[i] rows left for its lookup helper columns. Returns one CtlData per table (None for
    a table without CTLs)."""
    out = []
    for i, trace in enumerate(traces):
        groups = table_groups(cross_table_lookups, i)
        if not groups:
            out.append(None)
            continue
        nl = num_lookup_columns[i] if num_lookup_columns else 0
        zs_index, num_h, num_helpers = zs_layout(groups, len(ctl_challenges), max_constraint_degree)
        n = trace.shape[1]
        aux = _alloc_auxiliary(nl + num_helpers + len(zs_index), n, trace)
        compute_ctl_helper_columns(trace, groups, ctl_challenges, max_constraint_degree, ctx, aux[nl:])
        out.append(_ctl_data(groups, ctl_challenges, zs_index, num_h, aux, nl))
    return out


def _ctl_data(groups, ctl_challenges, zs_index, num_h, aux, nl):
    """The CtlZData of a table's auxiliary buffer laid out by zs_layout."""
    nc = len(ctl_challenges)
    total_h = sum(num_h) * nc
    at = {int(z): k for k, z in enumerate(zs_index)}
    zs, h = [], nl
    for z in range(len(zs_index)):
        g, c = divmod(at[z], nc)
        entries = groups[g][1]
        zs.append(CtlZData([aux[h + k] for k in range(num_h[g])], aux[nl + total_h + z], ctl_challenges[c],
                           [t.columns for t in entries], [t.filter for t in entries]))
        h += num_h[g]
    return CtlData(zs, aux, nl)


def ctl_shape_vars(ctl_data):
    """CtlCheckVars carrying the shape of a table's CTL data (helper counts, challenges, columns, filters) without
    values: what a constraint program needs."""
    return [CtlCheckVars([None] * len(z.helper_columns), None, None, z.challenge, z.columns, z.filter)
            for z in ctl_data.zs_columns]


def check_ctl_shapes(starks, cross_table_lookups, num_challenges):
    """The shapes the multi-STARK prover refuses, before any device work: a table index out of range; a table in a CTL
    whose requires_ctls() is False, or the reverse; CTL helper columns at constraint degree < 2 (the reference's
    chunks(0)) or in chunks of more than two entries (its todo!); a table's looking entries of one CTL that are not
    consecutive, or a table both looked and looking in one CTL (the reference's prover and verifier then count its
    columns differently); a table with CTL helper columns whose constraint degree differs from the system's largest
    (get_helper_cols and eval_helper_columns then chunk differently). Returns max_constraint_degree."""
    num_tables = len(starks)
    max_degree = max(s.constraint_degree() for s in starks)
    involved = set()
    for i, ctl in enumerate(cross_table_lookups):
        tables = [t.table for t in ctl.looking_tables] + [ctl.looked_table.table]
        for t in tables:
            if not 0 <= t < num_tables:
                raise N.ShapeError("CTL %d names table %d of %d" % (i, t, num_tables))
        involved.update(tables)
        looking = [t.table for t in ctl.looking_tables]
        for t in set(looking):
            idx = [k for k, v in enumerate(looking) if v == t]
            if idx != list(range(idx[0], idx[0] + len(idx))):
                raise N.ShapeError("CTL %d: table %d's looking entries are not consecutive" % (i, t))
            if t == ctl.looked_table.table:
                raise N.ShapeError("CTL %d: table %d is both looked and looking" % (i, t))
            if len(idx) > 1:
                d = starks[t].constraint_degree()
                if max_degree < 2:
                    raise N.ShapeError("attempt to divide by zero: CTL %d gives table %d helper columns at constraint "
                                       "degree %d" % (i, t, max_degree))
                if d != max_degree:
                    raise N.ShapeError("CTL %d: table %d has CTL helper columns at constraint degree %d, not the "
                                       "system's %d" % (i, t, d, max_degree))
                if helper_chunk_size(max_degree) > 2 and len(idx) > 2:
                    raise N.ShapeError("Allow other constraint degrees: a chunk of %d CTL entries"
                                       % min(len(idx), helper_chunk_size(max_degree)))
    for t, s in enumerate(starks):
        if (t in involved) != bool(s.requires_ctls()):
            raise N.ShapeError("table %d %s a CTL but requires_ctls() is %s"
                               % (t, "takes part in" if t in involved else "takes no part in", s.requires_ctls()))
    return max_degree


class MultiStarkProof:
    """The proofs of a multi-STARK system, one StarkProofWithPublicInputs per table, made by prove_with_ctls."""

    def __init__(self, stark_proofs):
        self.stark_proofs = list(stark_proofs)

    def ctl_vars(self, starks, config, cross_table_lookups, ctl_challenges):
        """Every table's CtlCheckVars::from_proof (None for a table without CTLs)."""
        out = []
        for i, (stark, p) in enumerate(zip(starks, self.stark_proofs)):
            if not stark.requires_ctls():
                out.append(None)
                continue
            total, _, by_ctl = CrossTableLookup.num_ctl_helpers_zs_all(cross_table_lookups, i, config.num_challenges,
                                                                        stark.constraint_degree())
            nl = stark.num_lookup_helper_columns(config) if stark.uses_lookups() else 0
            out.append(CtlCheckVars.from_proof(i, p.proof, cross_table_lookups, ctl_challenges, nl, total, by_ctl))
        return out

    def get_challenges(self, starks, config, cross_table_lookups):
        """The prover's transcript replayed from the proofs alone (get_challenges.rs:37-73,323-357 with the CTL
        challenges and ignore_trace_cap): every trace cap, the CTL challenge set, then table by table its public inputs,
        the config and its challenges. Returns dict(ctl_challenges, stark_challenges: one get_challenges dict per
        table)."""
        from .challenger import Challenger
        from .lookup import get_grand_product_challenge_set

        if len(starks) != len(self.stark_proofs):
            raise N.ShapeError("expected %d proofs, got %d" % (len(starks), len(self.stark_proofs)))
        ch = Challenger()
        for p in self.stark_proofs:
            ch.observe_cap(p.proof.trace_cap)
        ctl_challenges = get_grand_product_challenge_set(ch, config.num_challenges)
        ctl_vars = self.ctl_vars(starks, config, cross_table_lookups, ctl_challenges)
        out = [p.get_challenges(s, config, challenger=ch, ctl_challenges=ctl_challenges, ctl_vars=v,
                                ignore_trace_cap=True)
               for s, p, v in zip(starks, self.stark_proofs, ctl_vars)]
        return dict(ctl_challenges=ctl_challenges, stark_challenges=out)


def check_prove_shapes(starks, config, traces, cross_table_lookups, public_inputs, lde_blocks=0):
    """prove_with_ctls's refusals, before any device work: trace and public-input counts, every table's
    stark.prove checks (with lde_blocks), check_ctl_shapes and check_lookup_shapes. Returns (each table's ProveParams,
    max_constraint_degree)."""
    from . import stark as S

    if len(traces) != len(starks):
        raise N.ShapeError("expected %d traces, got %d" % (len(starks), len(traces)))
    if len(public_inputs) != len(starks):
        raise N.ShapeError("expected %d public-input lists, got %d" % (len(starks), len(public_inputs)))
    params = [S._check_prove_shapes(s, config, t, p, lde_blocks=lde_blocks)
              for s, t, p in zip(starks, traces, public_inputs)]
    max_degree = check_ctl_shapes(starks, cross_table_lookups, config.num_challenges)
    for s in starks:
        S.check_lookup_shapes(s)
    return params, max_degree


def prove_with_ctls(starks, config, traces, cross_table_lookups, public_inputs, ctx=None, lde_blocks=None,
                    check_constraints=False):
    """A multi-STARK proof with cross-table lookups: every table's trace commitment, every trace cap observed in table
    order, the CTL challenge set (get_ctl_data), every table's CTL helper and Z columns on the device
    (cross_table_lookup_data at the system's largest constraint degree), then table by table on the same challenger its
    public inputs, the config and prove_with_commitment with its CTL data -- the order the reference's verifier-side
    replay accepts. traces: per table (COLUMNS, n) host columns or a torch CUDA tensor, read on the device once; a torch
    trace may still be in production on the caller's current torch stream, the library's work is ordered after it. Raises
    ShapeError before any device work for every shape the reference cannot prove or verify (check_prove_shapes).
    Returns a MultiStarkProof. distributed.prove_with_ctls proves the same system across several GPUs. lde_blocks=G:
    every commitment is non-resident, as in stark.prove; G must also be at most every table's quotient coset size.
    check_constraints=True checks every table's constraints (its own, lookups and CTLs) as stark.prove does."""
    from . import stark as S

    return _prove_with_ctls(starks, config, traces, cross_table_lookups, public_inputs, ctx,
                            S.lde_placement(config.fri_config.cap_height, lde_blocks), check_constraints)


def _prove_with_ctls(starks, config, traces, cross_table_lookups, public_inputs, ctx, placement,
                     check_constraints=False):
    """prove_with_ctls on a distributed.Placement: every trace is committed with placement.commit_kwargs and observed
    as placement.cap, and each table runs prove_with_commitment on the placement. The CTL helper and Z columns are
    computed from the full traces on every rank."""
    from .challenger import Challenger
    from .lookup import get_grand_product_challenge_set
    from . import stark as S

    params, max_degree = check_prove_shapes(starks, config, traces, cross_table_lookups, public_inputs,
                                            placement.lde_blocks)
    ctx = ctx or N.default_context()
    public_inputs = [[int(v) % F.ORDER for v in p] for p in public_inputs]
    rate_bits, cap_height = config.fri_config.rate_bits, config.fri_config.cap_height
    dev_traces, commitments = [], []
    try:
        for s, t in zip(starks, traces):
            dt = S._device_trace(t, ctx) if (s.requires_ctls() or s.uses_lookups()) else t
            dev_traces.append(dt)
            commitments.append(S._commit_trace(dt, rate_bits, cap_height, ctx, **placement.commit_kwargs))
        challenger = Challenger()
        caps = [placement.cap(c) for c in commitments]
        for cap in caps:
            challenger.observe_cap(cap)
        ctl_challenges = get_grand_product_challenge_set(challenger, config.num_challenges)
        nls = [s.num_lookup_helper_columns(config) if s.uses_lookups() else 0 for s in starks]
        ctl_data = cross_table_lookup_data([t if s.requires_ctls() else None for s, t in zip(starks, dev_traces)],
                                           cross_table_lookups, ctl_challenges, max_degree, ctx, nls)
        proofs = []
        for i, s in enumerate(starks):
            challenger.observe_elements(public_inputs[i])
            config.observe(challenger)
            proofs.append(S.prove_with_commitment(s, config, dev_traces[i], commitments[i], caps[i], ctl_data[i],
                                                  ctl_challenges, challenger, public_inputs[i], params[i], ctx=ctx,
                                                  placement=placement, check_constraints=check_constraints))
            ctl_data[i] = None
        return MultiStarkProof(proofs)
    finally:
        for c in commitments:
            c.close()


def check_ctls(traces, cross_table_lookups, extra_looking_values=None):
    """debug_utils::check_ctls (cross_table_lookup.rs:955-1063) on host traces: for every CTL the looking tables'
    selected tuples, with extra_looking_values[ctl index] (a list of tuples) added, must equal the looked table's as a
    multiset; a filter must be 0 or 1. Raises ValueError otherwise."""
    extra_looking_values = extra_looking_values or {}
    for i, ctl in enumerate(cross_table_lookups):
        looking, looked = Counter(), Counter()
        for t in ctl.looking_tables:
            looking.update(_selected_rows(traces, t))
        looked.update(_selected_rows(traces, ctl.looked_table))
        for row in extra_looking_values.get(i, []):
            looking[tuple(int(v) % F.ORDER for v in row)] += 1
        if looking != looked:
            diff = (looking - looked) + (looked - looking)
            row = next(iter(diff))
            raise ValueError("Cross-table lookup %d: row %r appears %d times in the looking tables and %d times in the "
                             "looked table" % (i, row, looking[row], looked[row]))


def _column_rows(column, trace):
    """Column::eval_table on every row: the current row's combination, the next row's (row n - 1 reads row 0), the
    constant."""
    acc = np.full(trace.shape[1], column.constant, dtype=object)
    for c, f in column.linear_combination:
        acc = (acc + trace[c].astype(object) * f) % F.ORDER
    for c, f in column.next_row_linear_combination:
        acc = (acc + np.roll(trace[c], -1).astype(object) * f) % F.ORDER
    return acc


def _filter_rows(filt, trace):
    """Filter::eval_table on every row."""
    acc = np.zeros(trace.shape[1], dtype=object)
    for a, b in filt.products:
        acc = (acc + _column_rows(a, trace) * _column_rows(b, trace)) % F.ORDER
    for c in filt.constants:
        acc = (acc + _column_rows(c, trace)) % F.ORDER
    return acc


def _selected_rows(traces, t):
    trace = np.asarray(traces[t.table], dtype=np.uint64)
    filt = _filter_rows(t.filter, trace)
    if any(int(f) not in (0, 1) for f in filt):
        raise ValueError("Non-binary filter?")
    cols = [_column_rows(c, trace) for c in t.columns]
    return [tuple(int(c[r]) for c in cols) for r in range(trace.shape[1]) if int(filt[r]) == 1]
