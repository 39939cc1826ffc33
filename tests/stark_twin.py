"""starky proofs on the CPU: a twin of the product's provers built from the oracle's pieces, and a restated verifier.
Test infrastructure only.

The twin keeps the reference's layering. prove_table restates prove_with_commitment (starky/src/prover.rs:125-484) on a
challenger that has already observed what precedes the table, and verify_table restates
verify_stark_proof_with_challenges (verifier.rs:30-332) with the transcript of get_challenges.rs. Lookups and
cross-table lookups (CTLs) are optional parts of that one path: the auxiliary oracle [lookup helpers | CTL helpers |
CTL Zs] is present only when it is non-empty. twin_prove and verify are the one-STARK prove / verify_stark_proof;
twin_prove_with_ctls and verify_with_ctls are the multi-STARK prove_with_ctls and its verifier
(CtlCheckVars::from_proof, verify_cross_table_lookups).

The commitments, the Challenger, the openings (eval_poly_base_at_ext), prove_openings and verify_fri_proof are the
oracle's. The quotient is the oracle's for a FibonacciStark without an auxiliary oracle and otherwise host_quotient: the
product's constraint program evaluated over numpy object arrays on the quotient coset, divided by Z_H, coset_ifft'd by
the oracle. The constraint-binding step and the verifier evaluate the constraints with the product's
eval_vanishing_poly, which the tests check against hand-written formulas.

The lookup and CTL columns are restated literally over Python integers, with one inversion per element (not the batch
form the device uses). helper_columns restates lookup_helper_columns / get_helper_cols (lookup.rs:579-652,746-789) with
Column::eval_table / Filter::eval_table row by row (lookup.rs:118-129,323-343), then the running sum Z.
cross_table_lookup_data restates cross_table_lookup.rs:270-414: the looking tables grouped by itertools' group_by,
GrandProductChallenge::combine, the helper columns per chunk of constraint_degree - 1 entries and Z as the suffix sum of
their row sums."""
import numpy as np

P = 0xFFFFFFFF00000001
SHIFT = 7  # F::coset_shift() = MULTIPLICATIVE_GROUP_GENERATOR


def _ext_pow(a, e):
    from plonky2_b200 import field as F

    return F.ext_pow(a, e)


def root_of_unity(bits):
    from plonky2_b200 import field as F

    return F.primitive_root_of_unity(bits)


def observe_config(ch, config):
    """StarkConfig::observe (config.rs:102-107) with FriConfig::observe (fri/mod.rs:73-79), ConstantArityBits."""
    f = config.fri_config
    ch.observe_elements([config.security_bits, config.num_challenges, f.rate_bits, f.cap_height, f.proof_of_work_bits])
    ch.observe_elements([1, f.reduction_strategy[1], f.reduction_strategy[2], f.num_query_rounds])


def _draw_lookup_challenges(ch, num_challenges):
    """get_grand_product_challenge_set (lookup.rs:525-543) on the oracle's Challenger: (beta, gamma) pairs."""
    out = []
    for _ in range(num_challenges):
        beta = ch.get_challenge()
        out.append((beta, ch.get_challenge()))
    return out


# ------------------------------------------------------------------------------------------------ lookup columns
def _inv_each(values):
    """Per-element inversion; a zero is the reference's batch_multiplicative_inverse panic."""
    out = np.empty(len(values), dtype=object)
    for i, v in enumerate(values):
        v = int(v) % P
        if v == 0:
            raise ZeroDivisionError("Tried to invert zero")
        out[i] = pow(v, P - 2, P)
    return out


def eval_table(column, trace):
    """Column::eval_table on every row (eval_all_rows, lookup.rs:337-343): trace[c][row] * f over the current row,
    trace[c][(row + 1) % n] * f over the next row, plus the constant."""
    n = trace.shape[1]
    acc = np.full(n, column.constant, dtype=object)
    for c, f in column.linear_combination:
        acc = (acc + trace[c].astype(object) * f) % P
    for c, f in column.next_row_linear_combination:
        acc = (acc + np.roll(trace[c], -1).astype(object) * f) % P
    return acc


def filter_eval_table(filt, trace):
    """Filter::eval_table (lookup.rs:118-129)."""
    acc = np.zeros(trace.shape[1], dtype=object)
    for a, b in filt.products:
        acc = (acc + eval_table(a, trace) * eval_table(b, trace)) % P
    for c in filt.constants:
        acc = (acc + eval_table(c, trace)) % P
    return acc


def helper_columns(lookup, trace, challenge, constraint_degree):
    """lookup_helper_columns (lookup.rs:579-652) for one challenge: the h_k columns, then Z."""
    trace = np.asarray(trace, dtype=np.uint64)
    chunk = constraint_degree - 1 if constraint_degree >= 1 else 1
    assert chunk > 0, "attempt to divide by zero"
    n = trace.shape[1]
    cols = []
    for k in range(0, len(lookup.columns), chunk):      # get_helper_cols: per chunk, sum of filter / (f + challenge)
        acc = None
        for col, filt in zip(lookup.columns[k:k + chunk], lookup.filter_columns[k:k + chunk]):
            combined = _inv_each((eval_table(col, trace) + challenge) % P) * filter_eval_table(filt, trace) % P
            acc = combined if acc is None else (acc + combined) % P
        cols.append(acc)
    table_inverse = _inv_each((eval_table(lookup.table_column, trace) + challenge) % P)
    frequencies = eval_table(lookup.frequencies_column, trace)
    x = (sum(cols, np.zeros(n, dtype=object)) - frequencies * table_inverse) % P
    z = np.zeros(n, dtype=object)
    for i in range(n - 1):
        z[i + 1] = (z[i] + x[i]) % P
    return [np.array([int(v) for v in c], dtype=np.uint64) for c in cols + [z]], int((z[n - 1] + x[n - 1]) % P)


def aux_columns(stark, trace, challenges):
    """prover.rs:177-195: every lookup, every challenge, in that order. Returns ((num_aux, n) uint64, [Z at the wrap])."""
    out, wraps = [], []
    for lookup in stark.lookups():
        for c in challenges:
            cols, wrap = helper_columns(lookup, trace, c, stark.constraint_degree())
            out += cols
            wraps.append(wrap)
    return np.stack(out), wraps


# --------------------------------------------------------------------------------------------------- CTL columns
def combine_rows(columns, trace, beta, gamma):
    """GrandProductChallenge::combine of a tuple on every row: sum_k beta^k Column_k::eval_table + gamma."""
    acc = np.zeros(trace.shape[1], dtype=object)
    for k, col in enumerate(columns):
        acc = (acc + eval_table(col, trace) * pow(beta, k, P)) % P
    return (acc + gamma) % P


def partial_sums(trace, entries, challenge, constraint_degree):
    """partial_sums / get_helper_cols (cross_table_lookup.rs:383-414, lookup.rs:746-789): entries = [(columns,
    filter)]. Returns the helper columns then Z when there is more than one entry, else [Z]."""
    trace = np.asarray(trace, dtype=np.uint64)
    beta, gamma = challenge
    chunk = constraint_degree - 1 if constraint_degree >= 1 else 1
    assert chunk > 0, "chunks(0)"
    n = trace.shape[1]
    helpers = []
    for k in range(0, len(entries), chunk):
        acc = np.zeros(n, dtype=object)
        for cols, filt in entries[k:k + chunk]:
            acc = (acc + _inv_each(combine_rows(cols, trace, beta, gamma)) * filter_eval_table(filt, trace)) % P
        helpers.append(acc)
    z = np.zeros(n, dtype=object)
    z[n - 1] = sum(int(h[n - 1]) for h in helpers) % P
    for i in range(n - 2, -1, -1):
        z[i] = (z[i + 1] + sum(int(h[i]) for h in helpers)) % P
    out = helpers + [z] if len(entries) > 1 else [z]
    return [np.array([int(v) for v in c], dtype=np.uint64) for c in out]


def cross_table_lookup_data(traces, ctls, challenges, constraint_degree):
    """cross_table_lookup_data (cross_table_lookup.rs:270-339): per table, its CtlZData as dicts (helpers, z,
    challenge, columns, filter) in the reference's order."""
    data = [[] for _ in traces]
    for ctl in ctls:
        for ch in challenges:
            groups = []                                       # itertools::group_by(|t| t.table)
            for t in ctl.looking_tables:
                if groups and groups[-1][0] == t.table:
                    groups[-1][1].append(t)
                else:
                    groups.append((t.table, [t]))
            for table, grp in groups:
                cols = partial_sums(traces[table], [(t.columns, t.filter) for t in grp], ch, constraint_degree)
                mine = [t for t in ctl.looking_tables if t.table == table]
                data[table].append(dict(helpers=cols[:-1], z=cols[-1], challenge=ch, columns=[t.columns for t in mine],
                                        filter=[t.filter for t in mine]))
            lt = ctl.looked_table
            z = partial_sums(traces[lt.table], [(lt.columns, lt.filter)], ch, constraint_degree)[0]
            data[lt.table].append(dict(helpers=[], z=z, challenge=ch, columns=[lt.columns], filter=[lt.filter]))
    return data


def ctl_aux(zs_columns, n):
    """get_ctl_auxiliary_polys: every helper column, then every Z."""
    cols = [h for z in zs_columns for h in z["helpers"]] + [z["z"] for z in zs_columns]
    return np.stack(cols) if cols else np.zeros((0, n), dtype=np.uint64)


class _Vars:
    """A CtlCheckVars-like record over plain values."""

    def __init__(self, helper_columns, local_z, next_z, challenges, columns, filter):
        self.helper_columns, self.local_z, self.next_z = helper_columns, local_z, next_z
        self.challenges, self.columns, self.filter = challenges, columns, filter


def _gpc(pair):
    from plonky2_b200.lookup import GrandProductChallenge

    return GrandProductChallenge(*pair)


def _shape_vars(zs_columns):
    return [_Vars([None] * len(z["helpers"]), None, None, _gpc(z["challenge"]), z["columns"], z["filter"])
            for z in zs_columns]


def num_ctl_helpers_zs_all(ctls, table, num_challenges, constraint_degree):
    """cross_table_lookup.rs:114-141."""
    num_helpers = num_ctls = 0
    by_ctl = [0] * len(ctls)
    for i, ctl in enumerate(ctls):
        k = sum(t.table == table for t in [ctl.looked_table] + ctl.looking_tables)
        if k > 1:
            by_ctl[i] = -(-k // (constraint_degree - 1))
            num_helpers += by_ctl[i]
        if k > 0:
            num_ctls += 1
    return num_helpers * num_challenges, num_ctls * num_challenges, by_ctl


def ctl_vars_from_proof(table, proof, ctls, challenges, num_lookup_columns, total_helpers, by_ctl):
    """CtlCheckVars::from_proof (cross_table_lookup.rs:443-547)."""
    o = proof.openings
    zs = list(zip(o.auxiliary_polys[num_lookup_columns:], o.auxiliary_polys_next[num_lookup_columns:]))
    z_index = start = 0
    out = []
    for i, ctl in enumerate(ctls):
        for c in challenges:
            mine = [t for t in ctl.looking_tables if t.table == table]
            if mine:
                lz, nz = zs[total_helpers + z_index]
                out.append(_Vars([h for h, _ in zs[start:start + by_ctl[i]]], lz, nz, _gpc(c), [t.columns for t in mine],
                                 [t.filter for t in mine]))
                start += by_ctl[i]
                z_index += 1
            if ctl.looked_table.table == table:
                lz, nz = zs[total_helpers + z_index]
                z_index += 1
                out.append(_Vars([], lz, nz, _gpc(c), [ctl.looked_table.columns], [ctl.looked_table.filter]))
    return out


# ---------------------------------------------------------------------------------------------------- the prover
def bind_constraints(ch, stark, public_inputs, num_challenges, degree_bits, lookup_challenges=None, num_aux=0,
                     ctl_vars=None):
    """prover.rs:239-370 / get_challenges.rs:94-163 on the oracle's Challenger: alphas', the dummy openings of the trace
    and of the num_aux auxiliary polynomials, zeta', the vanishing polynomial observed; returns the alphas. With
    ctl_vars (only their shape is read) the CTL helper and Z values are the dummy auxiliary values at their places in
    [lookup helpers | CTL helpers | CTL Zs] (prover.rs:321-350)."""
    from plonky2_b200 import stark as S

    alphas_prime = ch.get_n_challenges(num_challenges)
    pow_degree = max(2, stark.constraint_degree() + 1)
    k = max(1, 50 // (pow_degree - 1).bit_length() - 1)
    C = stark.COLUMNS
    total = 2 * C + 2 * num_aux
    zetas = [ch.get_extension_challenge() for _ in range((total + k - 1) // k)]
    dummy = []
    for z in zetas:
        for _ in range(min(k + 1, total)):
            dummy.append(z)
            z = _ext_pow(z, pow_degree)
    zeta_prime = ch.get_extension_challenge()
    aux, aux_next = dummy[2 * C:2 * C + num_aux], dummy[2 * C + num_aux:total]
    dummy_vars = None
    if ctl_vars is not None:
        first_z = num_aux - len(ctl_vars)
        start = first_z - sum(len(v.helper_columns) for v in ctl_vars)
        dummy_vars = []
        for i, v in enumerate(ctl_vars):
            m = len(v.helper_columns)
            dummy_vars.append(_Vars(aux[start:start + m], aux[first_z + i], aux_next[first_z + i], v.challenges,
                                    v.columns, v.filter))
            start += m
    evals = S.eval_vanishing_poly(stark, dummy[:C], dummy[C:2 * C], public_inputs, alphas_prime, zeta_prime,
                                  degree_bits, aux, aux_next, lookup_challenges, dummy_vars)
    ch.observe_elements([w for e in evals for w in e])
    return ch.get_n_challenges(num_challenges)


def host_quotient(oracle, stark, trace_coeffs, public_inputs, alphas, aux_coeffs=None, lookup_challenges=None,
                  ctl_vars=None):
    """compute_quotient_polys (prover.rs:488-668) on the host: the product's constraint program (with its lookup and
    CTL terms, over the auxiliary LDE) over numpy object arrays on the quotient coset, divided by Z_H, coset_ifft'd.
    Returns (num_challenges, n << log2_ceil(qdf)) coefficients, or None without constraints; raises like
    prover.rs:396-401 when the vanishing polynomial is not divisible by Z_H."""
    from plonky2_b200 import stark as S

    qdf = stark.quotient_degree_factor()
    if qdf == 0:
        return None
    n = trace_coeffs.shape[1]
    log_n = n.bit_length() - 1
    qd_bits = (qdf - 1).bit_length()
    size = n << qd_bits

    def lde(coeffs):
        vals = []
        for c in coeffs:
            pad = np.zeros(size, dtype=np.uint64)
            pad[:n] = c
            vals.append(oracle.coset_fft(pad, SHIFT).astype(object))
        return vals

    tv, av = lde(trace_coeffs), lde(aux_coeffs) if aux_coeffs is not None else []
    w = root_of_unity(log_n + qd_bits)
    xs, x = [], SHIFT
    for _ in range(size):
        xs.append(x)
        x = x * w % P
    xs = np.array(xs, dtype=object)
    g = root_of_unity(log_n)
    zh = np.array([(pow(int(v), n, P) - 1) % P for v in xs], dtype=object)
    inv = np.vectorize(lambda v: pow(int(v), P - 2, P), otypes=[object])
    filters = [None, (xs - pow(g, P - 2, P)) % P, zh * inv(n * (xs - 1) % P) % P, zh * inv(n * (xs * g - 1) % P) % P]
    challenges = [int(c) % P for c in lookup_challenges] if stark.uses_lookups() else []
    b = stark.constraint_program(len(challenges), ctl_vars)
    bound = [int(v) % P for c in ctl_vars or [] for v in (c.challenges.beta, c.challenges.gamma)]
    consts = [int(v) % P for v in public_inputs] + challenges + bound + b.consts[b.num_bound:]
    step = 1 << qd_bits
    acc = [np.zeros(size, dtype=object) for _ in alphas]
    v = []
    for op, a, c in b.instrs:
        r = None
        if op == S.OP_LOCAL:
            r = tv[a]
        elif op == S.OP_NEXT:
            r = np.roll(tv[a], -step)
        elif op == S.OP_AUX_LOCAL:
            r = av[a]
        elif op == S.OP_AUX_NEXT:
            r = np.roll(av[a], -step)
        elif op == S.OP_CONST:
            r = consts[a]
        elif op == S.OP_ADD:
            r = (v[a] + v[c]) % P
        elif op == S.OP_SUB:
            r = (v[a] - v[c]) % P
        elif op == S.OP_MUL:
            r = v[a] * v[c] % P
        else:
            e = v[a] if filters[c] is None else v[a] * filters[c] % P
            acc = [(s * (int(al) % P) + e) % P for s, al in zip(acc, alphas)]
        v.append(r)
    zh_inv = inv(zh)
    out = np.stack([oracle.coset_ifft(np.array([int(t) for t in s * zh_inv % P], dtype=np.uint64), SHIFT) for s in acc])
    if out[:, qdf * n:].any():
        raise ValueError("Quotient has failed, the vanishing polynomial is not divisible by Z_H")
    return out


def quotient(oracle, stark, trace_commit, public_inputs, alphas, aux_coeffs=None, lookup_challenges=None,
             ctl_vars=None):
    """The oracle's own quotient for a FibonacciStark without an auxiliary oracle, host_quotient otherwise."""
    from plonky2_b200.stark import FibonacciStark

    if isinstance(stark, FibonacciStark) and aux_coeffs is None:
        return oracle.stark_quotient_fibonacci(trace_commit, public_inputs, alphas)
    return host_quotient(oracle, stark, trace_commit.coeffs, public_inputs, alphas, aux_coeffs, lookup_challenges,
                         ctl_vars)


def quotient_chunks(stark, q, n):
    qdf = stark.quotient_degree_factor()
    return np.concatenate([q[i, :qdf * n].reshape(qdf, n) for i in range(q.shape[0])])


def _ev(oracle, commit, z):
    return np.array([oracle.eval_poly_base_at_ext(p, z) for p in commit.coeffs], dtype=np.uint64).reshape(-1, 2)


def fri_batches(stark, config, zeta, g, num_aux=0, ctl_first=None):
    """fri_instance (stark.rs:101-170): the trace, auxiliary (num_aux polynomials; none without) and quotient oracles
    at zeta, the trace and auxiliary oracles at g * zeta, and with CTLs the auxiliary oracle's CTL Zs (ctl_first)
    at 1."""
    from plonky2_b200 import field as F

    nq = stark.num_quotient_polys(config)
    opened_next = [(0, i) for i in range(stark.COLUMNS)] + [(1, j) for j in range(num_aux)]
    qi = 2 if num_aux else 1
    out = [(zeta, opened_next + [(qi, j) for j in range(nq)]), (F.ext_mul((g, 0), zeta), opened_next)]
    if ctl_first is not None:
        out.append(((1, 0), [(1, j) for j in ctl_first]))
    return out


def prove_table(oracle, stark, config, trace, trace_commit, ch, public_inputs, lookup_challenge_set=None, ctl_zs=()):
    """prove_with_commitment (prover.rs:125-484) with the oracle's pieces, on a challenger that has observed what
    precedes the table. lookup_challenge_set: the (beta, gamma) pairs whose betas the lookups use (None without lookups
    or CTLs); ctl_zs: the table's CtlZData from cross_table_lookup_data (empty without CTLs). Returns a dict:
    public_inputs, trace_cap, aux_cap, quotient_cap, local_values, next_values, auxiliary_polys, auxiliary_polys_next,
    ctl_zs_first, quotient_polys, fri_bytes, alphas, zeta; what the table does not have is None."""
    f = config.fri_config
    n = trace.shape[1]
    degree_bits = n.bit_length() - 1
    betas = [b for b, _ in lookup_challenge_set] if lookup_challenge_set is not None else None
    lookup_aux = aux_columns(stark, trace, betas)[0] if stark.uses_lookups() else np.zeros((0, n), dtype=np.uint64)
    aux = np.concatenate([lookup_aux, ctl_aux(ctl_zs, n)])          # [lookup helpers | CTL helpers | CTL Zs]
    ctl_vars = _shape_vars(ctl_zs) if stark.requires_ctls() else None
    commits, ac, qc = [trace_commit], None, None
    if len(aux):
        ac = oracle.Commit(aux, f.rate_bits, f.cap_height)
        commits.append(ac)
        ch.observe_cap(ac.cap)
    alphas = bind_constraints(ch, stark, public_inputs, config.num_challenges, degree_bits, betas, len(aux), ctl_vars)
    q = quotient(oracle, stark, trace_commit, public_inputs, alphas, ac.coeffs if ac is not None else None, betas,
                 ctl_vars)
    if q is not None:
        qc = oracle.Commit(quotient_chunks(stark, q, n), f.rate_bits, f.cap_height, is_coeffs=True)
        commits.append(qc)
        ch.observe_cap(qc.cap)
    zeta = ch.get_extension_challenge()
    ctl_first = range(len(aux) - len(ctl_zs), len(aux)) if stark.requires_ctls() else None
    batches = fri_batches(stark, config, zeta, root_of_unity(degree_bits), len(aux), ctl_first)
    zn = batches[1][0]
    local, nxt = _ev(oracle, trace_commit, zeta), _ev(oracle, trace_commit, zn)
    al, an = (_ev(oracle, ac, zeta), _ev(oracle, ac, zn)) if ac is not None else (None, None)
    quot = _ev(oracle, qc, zeta) if qc is not None else None
    first = aux[list(ctl_first), 0] if ctl_first is not None else None
    ch.observe_elements(np.concatenate([v for v in (local, al, quot) if v is not None]).reshape(-1))
    ch.observe_elements(np.concatenate([v for v in (nxt, an) if v is not None]).reshape(-1))
    if first is not None:
        ch.observe_elements(np.stack([first, np.zeros_like(first)], axis=1).reshape(-1))
    arity_bits = f.fri_params(degree_bits, False).reduction_arity_bits
    params = oracle.make_params(f.rate_bits, f.cap_height, f.proof_of_work_bits, f.num_query_rounds, arity_bits)
    fri_bytes = oracle.prove_openings(commits, batches, ch, params)
    return dict(public_inputs=list(public_inputs), trace_cap=trace_commit.cap,
                aux_cap=ac.cap if ac is not None else None, quotient_cap=qc.cap if qc is not None else None,
                local_values=local, next_values=nxt, auxiliary_polys=al, auxiliary_polys_next=an, ctl_zs_first=first,
                quotient_polys=quot, fri_bytes=fri_bytes, alphas=alphas, zeta=zeta)


def twin_prove(oracle, stark, config, trace, public_inputs):
    """prove (prover.rs:40-114): the public inputs, the config and the trace cap observed, the lookup challenges drawn
    if the Stark uses lookups, then prove_table. Returns prove_table's dict with lookup_challenge_set (None without
    lookups)."""
    f = config.fri_config
    trace = np.ascontiguousarray(trace, dtype=np.uint64)
    tc = oracle.Commit(trace, f.rate_bits, f.cap_height)
    pis = [int(v) % P for v in public_inputs]
    ch = oracle.Challenger()
    ch.observe_elements(pis)
    observe_config(ch, config)
    ch.observe_cap(tc.cap)
    pairs = _draw_lookup_challenges(ch, config.num_challenges) if stark.uses_lookups() else None
    return dict(prove_table(oracle, stark, config, trace, tc, ch, pis, pairs), lookup_challenge_set=pairs)


def twin_prove_with_ctls(oracle, starks, config, traces, ctls, public_inputs):
    """prove_with_ctls: every trace cap observed, the CTL challenges drawn, then per table its public inputs, the
    config and prove_table. Returns dict(ctl_challenges, ctl_data, tables: prove_table's dict per table)."""
    f = config.fri_config
    traces = [np.ascontiguousarray(t, dtype=np.uint64) for t in traces]
    tcs = [oracle.Commit(t, f.rate_bits, f.cap_height) for t in traces]
    ch = oracle.Challenger()
    for tc in tcs:
        ch.observe_cap(tc.cap)
    pairs = _draw_lookup_challenges(ch, config.num_challenges)
    data = cross_table_lookup_data(traces, ctls, pairs, max(s.constraint_degree() for s in starks))
    tables = []
    for stark, trace, tc, pis, zs in zip(starks, traces, tcs, public_inputs, data):
        pis = [int(v) % P for v in pis]
        ch.observe_elements(pis)
        observe_config(ch, config)
        tables.append(prove_table(oracle, stark, config, trace, tc, ch, pis, pairs, zs))
    return dict(ctl_challenges=pairs, ctl_data=data, tables=tables)


# -------------------------------------------------------------------------------------------------- the verifier
def check_lookup_options(stark, config, proof, num_ctl_helpers=0, num_ctl_zs=0):
    """check_lookup_options (verifier.rs:287-332), with ctl_zs_first present exactly when the Stark requires CTLs.
    Returns None or the reason."""
    o = proof.openings
    if stark.uses_lookups() or stark.requires_ctls():
        num_aux = stark.num_lookup_helper_columns(config) + num_ctl_helpers + num_ctl_zs
        if proof.auxiliary_polys_cap is None:
            return "Missing auxiliary_polys_cap"
        if o.auxiliary_polys is None:
            return "Missing auxiliary_polys"
        if o.auxiliary_polys_next is None:
            return "Missing auxiliary_polys_next"
        if len(proof.auxiliary_polys_cap.hashes) != 1 << config.fri_config.cap_height:
            return "auxiliary cap height"
        if len(o.auxiliary_polys) != num_aux or len(o.auxiliary_polys_next) != num_aux:
            return "opened auxiliary values"
    elif proof.auxiliary_polys_cap is not None or o.auxiliary_polys is not None or o.auxiliary_polys_next is not None:
        return "auxiliary data for a Stark without lookups or CTLs"
    if (o.ctl_zs_first is not None) != stark.requires_ctls() or (
            o.ctl_zs_first is not None and len(o.ctl_zs_first) != num_ctl_zs):
        return "ctl_zs_first length"
    return None


def verify_table(oracle, stark, config, proof_with_pis, ch, ctl_challenges=None, ctl_vars=None):
    """verify_stark_proof_with_challenges (verifier.rs:68-285) with the transcript of get_challenges.rs:37-199 replayed
    on the oracle's Challenger ch. For one STARK ch is fresh: it observes the trace cap after the config and draws the
    lookup challenges if there is an auxiliary cap. For a table of a multi-STARK proof ch has observed every trace cap
    and drawn ctl_challenges, whose betas the lookups use, and ctl_vars are the table's CtlCheckVars. ch continues past
    FRI's challenges, for the next table. Returns None if accepted, else the reason."""
    from plonky2_b200 import field as F
    from plonky2_b200 import stark as S
    from plonky2_b200.fri import fri_challenges

    p, pis = proof_with_pis.proof, list(proof_with_pis.public_inputs)
    o, f = p.openings, config.fri_config
    nq = stark.num_quotient_polys(config)
    num_ctl_zs = len(ctl_vars or [])
    if len(pis) != stark.PUBLIC_INPUTS:                                 # validate_proof_shape (verifier.rs:220-285)
        return "public inputs"
    if len(p.trace_cap.hashes) != 1 << f.cap_height:
        return "trace cap height"
    if (p.quotient_polys_cap is None) != (nq == 0) or (nq and len(p.quotient_polys_cap.hashes) != 1 << f.cap_height):
        return "quotient cap"
    if len(o.local_values) != stark.COLUMNS or len(o.next_values) != stark.COLUMNS:
        return "opened trace values"
    if (o.quotient_polys is None) != (nq == 0) or (nq and len(o.quotient_polys) != nq):
        return "opened quotient values"
    reason = check_lookup_options(stark, config, p, sum(len(v.helper_columns) for v in ctl_vars or []), num_ctl_zs)
    if reason is not None:
        return reason
    degree_bits = p.recover_degree_bits(config)
    ch.observe_elements(pis)
    observe_config(ch, config)
    challenges = ctl_challenges
    if ctl_challenges is None:
        ch.observe_cap(p.trace_cap.hashes)
        if p.auxiliary_polys_cap is not None:
            challenges = _draw_lookup_challenges(ch, config.num_challenges)
    if p.auxiliary_polys_cap is not None:
        ch.observe_cap(p.auxiliary_polys_cap.hashes)
    betas = [b for b, _ in challenges] if challenges is not None else None
    num_aux = len(o.auxiliary_polys) if o.auxiliary_polys is not None else 0
    alphas = bind_constraints(ch, stark, pis, config.num_challenges, degree_bits, betas, num_aux, ctl_vars)
    if p.quotient_polys_cap is not None:
        ch.observe_cap(p.quotient_polys_cap.hashes)
    zeta = ch.get_extension_challenge()
    opened = [np.concatenate([np.asarray(v) for v in (o.local_values, o.auxiliary_polys, o.quotient_polys)
                              if v is not None]),
              np.concatenate([np.asarray(v) for v in (o.next_values, o.auxiliary_polys_next) if v is not None])]
    if stark.requires_ctls():
        first = np.asarray(o.ctl_zs_first, dtype=np.uint64)
        opened.append(np.stack([first, np.zeros_like(first)], axis=1))
    for batch in opened:
        ch.observe_elements(batch.reshape(-1))
    vanishing = S.eval_vanishing_poly(stark, o.local_values, o.next_values, pis, alphas, zeta, degree_bits,
                                      o.auxiliary_polys, o.auxiliary_polys_next, betas, ctl_vars)
    zeta_pow_deg = _ext_pow(zeta, 1 << degree_bits)
    z_h = F.ext_sub(zeta_pow_deg, (1, 0))
    qdf = stark.quotient_degree_factor()
    for i in range(nq // max(qdf, 1)):
        t = (0, 0)
        for v in reversed(o.quotient_polys[i * qdf:(i + 1) * qdf]):        # reduce_with_powers(chunk, zeta^n)
            t = F.ext_add(F.ext_mul(t, zeta_pow_deg), (int(v[0]), int(v[1])))
        if vanishing[i] != F.ext_mul(z_h, t):
            return "Mismatch between evaluation and opening of quotient polynomial"
    ctl_first = range(num_aux - num_ctl_zs, num_aux) if stark.requires_ctls() else None
    batches = fri_batches(stark, config, zeta, root_of_unity(degree_bits), num_aux, ctl_first)
    arity_bits = config.fri_params(degree_bits).reduction_arity_bits
    params = oracle.make_params(f.rate_bits, f.cap_height, f.proof_of_work_bits, f.num_query_rounds, arity_bits)
    oracles = [(c, w) for c, w in ((p.trace_cap, stark.COLUMNS), (p.auxiliary_polys_cap, num_aux),
                                   (p.quotient_polys_cap, nq)) if c is not None]
    widths = [w for _, w in oracles]
    rc = oracle.verify_fri_proof([c.hashes for c, _ in oracles], widths, widths, batches,
                                 np.concatenate([b.reshape(-1) for b in opened]), degree_bits, ch.clone(), params,
                                 p.opening_proof.to_bytes())
    if rc != 0:
        return "verify_fri_proof rc=%d" % rc
    fp = p.opening_proof                  # the next table's transcript continues after FRI's
    fri_challenges(ch, [c.hashes for c in fp.commit_phase_merkle_caps], fp.final_poly, fp.pow_witness, degree_bits, f)
    return None


def verify(oracle, stark, config, proof_with_pis):
    """verify_stark_proof (verifier.rs:30-62) of a stark.StarkProofWithPublicInputs. Returns None if accepted, else
    the reason."""
    return verify_table(oracle, stark, config, proof_with_pis, oracle.Challenger())


def verify_cross_table_lookups(ctls, ctl_zs_first, num_challenges, extra_looking_sums=None):
    """verify_cross_table_lookups (cross_table_lookup.rs:852-898). Returns None or the reason."""
    extra_looking_sums = extra_looking_sums or {}
    its = [iter(int(v) for v in z) if z is not None else iter(()) for z in ctl_zs_first]
    for index, ctl in enumerate(ctls):
        seen = []
        for t in ctl.looking_tables:
            if t.table not in seen:
                seen.append(t.table)
        for c in range(num_challenges):
            s = sum(next(its[t]) for t in seen) + (extra_looking_sums[index][c] if index in extra_looking_sums else 0)
            if s % P != next(its[ctl.looked_table.table]):
                return "Cross-table lookup %d verification failed." % index
    return None


def verify_with_ctls(oracle, starks, config, ctls, multi_proof, extra_looking_sums=None):
    """The multi-STARK verifier: the transcript of prove_with_ctls, every table's verify_table with its CtlCheckVars,
    then verify_cross_table_lookups. Returns None if accepted, else the reason (with the table)."""
    proofs = multi_proof.stark_proofs
    if len(proofs) != len(starks):
        return "number of proofs"
    ch = oracle.Challenger()
    for p in proofs:
        ch.observe_cap(p.proof.trace_cap.hashes)
    challenges = _draw_lookup_challenges(ch, config.num_challenges)
    for i, (stark, p) in enumerate(zip(starks, proofs)):
        ctl_vars = None
        if stark.requires_ctls():
            o = p.proof.openings
            if o.auxiliary_polys is None:
                return "table %d: We cannot have CTLs without auxiliary polynomials." % i
            total, num_zs, by_ctl = num_ctl_helpers_zs_all(ctls, i, config.num_challenges, stark.constraint_degree())
            nl = stark.num_lookup_helper_columns(config)
            if len(o.auxiliary_polys) != nl + total + num_zs or len(o.auxiliary_polys_next) != nl + total + num_zs:
                return "table %d: opened auxiliary values" % i
            ctl_vars = ctl_vars_from_proof(i, p.proof, ctls, challenges, nl, total, by_ctl)
        reason = verify_table(oracle, stark, config, p, ch, challenges, ctl_vars)
        if reason is not None:
            return "table %d: %s" % (i, reason)
    return verify_cross_table_lookups(ctls, [p.proof.openings.ctl_zs_first for p in proofs], config.num_challenges,
                                      extra_looking_sums)


# ------------------------------------------------------------------------------------------- comparing proofs
def proof_diff(a, b, path=""):
    """Where two proof objects differ, [] when they are equal. The walk compares arrays (shape and words), integers,
    lists, dicts and the attributes of every object, and also to_bytes() where an object has one; a list of another
    length is reported by its two lengths and not walked."""
    if isinstance(a, (list, tuple)) and isinstance(b, (list, tuple)):
        if len(a) != len(b):
            return ["%s: %d entries against %d" % (path, len(a), len(b))]
        return [d for k, (x, y) in enumerate(zip(a, b)) for d in proof_diff(x, y, "%s[%d]" % (path, k))]
    if isinstance(a, dict) and isinstance(b, dict):
        if sorted(a) != sorted(b):
            return ["%s: keys %s against %s" % (path, sorted(a), sorted(b))]
        return [d for k in sorted(a) for d in proof_diff(a[k], b[k], "%s.%s" % (path, k))]
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        same = isinstance(a, np.ndarray) and isinstance(b, np.ndarray) and a.shape == b.shape and np.array_equal(a, b)
        return [] if same else [path]
    if isinstance(a, (int, np.integer)) and isinstance(b, (int, np.integer)):
        return [] if int(a) == int(b) else [path]
    if hasattr(a, "__dict__") and type(a) is type(b):
        diff = proof_diff(vars(a), vars(b), path)
        if hasattr(a, "to_bytes") and a.to_bytes() != b.to_bytes():
            diff.append(path + ".to_bytes()")
        return diff
    return [] if type(a) is type(b) and a == b else [path]


def assert_matches_twin(proof, twin):
    """The product's proof equals the twin's: a StarkProofWithPublicInputs against twin_prove's dict, a MultiStarkProof
    against twin_prove_with_ctls' (the table count first, then table by table). Public inputs, the trace, auxiliary and
    quotient caps, every opening including ctl_zs_first, and the FRI bytes (which end with the proof-of-work witness);
    what the twin does not have (None) the proof must not have either."""
    if "tables" in twin:
        assert len(proof.stark_proofs) == len(twin["tables"]), "number of tables"
        for p, t in zip(proof.stark_proofs, twin["tables"]):
            assert_matches_twin(p, t)
        return
    p, o = proof.proof, proof.proof.openings
    assert proof.public_inputs == twin["public_inputs"], "public_inputs"
    for key, got in (("trace_cap", p.trace_cap), ("aux_cap", p.auxiliary_polys_cap),
                     ("quotient_cap", p.quotient_polys_cap)):
        want = twin[key]
        assert (got is None) == (want is None) and (want is None or np.array_equal(got.hashes, want)), key
    for key in ("local_values", "next_values", "auxiliary_polys", "auxiliary_polys_next", "quotient_polys",
                "ctl_zs_first"):
        got, want = getattr(o, key), twin[key]
        assert (got is None) == (want is None) and (want is None or np.array_equal(got, want)), key
    assert p.opening_proof.to_bytes() == twin["fri_bytes"], "fri_bytes"
