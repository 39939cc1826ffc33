"""Multi-STARK proofs WITH cross-table lookups on the CPU: a restatement of cross_table_lookup_data, a twin of
prove_with_ctls, and a restated verifier (CtlCheckVars::from_proof, verify_stark_proof_with_challenges with ctl_vars,
verify_cross_table_lookups). Test infrastructure only.

cross_table_lookup_data restates cross_table_lookup.rs:270-414 literally over Python integers: the looking tables
grouped by itertools' group_by, Column::eval_table / Filter::eval_table row by row, GrandProductChallenge::combine, one
inversion per element (not the batch form the device uses), the helper columns per chunk of constraint_degree - 1
entries and Z as the suffix sum of their row sums. twin_prove follows the multi-STARK order (every trace cap, the CTL
challenges, then per table its public inputs, the config and prover.rs:125-484) with the oracle's Commit, Challenger,
openings and prove_openings; the quotient is evaluated on the host over the trace and auxiliary LDEs with the product's
constraint program, as tests/stark_lookup_twin.py does for lookups."""
import numpy as np

import stark_lookup_twin as LT
import stark_twin as T

P = 0xFFFFFFFF00000001
SHIFT = T.SHIFT


def combine_rows(columns, trace, beta, gamma):
    """GrandProductChallenge::combine of a tuple on every row: sum_k beta^k Column_k::eval_table + gamma."""
    acc = np.zeros(trace.shape[1], dtype=object)
    for k, col in enumerate(columns):
        acc = (acc + LT.eval_table(col, trace) * pow(beta, k, P)) % P
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
            acc = (acc + LT._inv_each(combine_rows(cols, trace, beta, gamma)) * LT.filter_eval_table(filt, trace)) % P
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


def bind_constraints(ch, stark, public_inputs, num_challenges, degree_bits, lookup_challenges, num_aux, nl, ctl_shape):
    """prover.rs:239-370 on the oracle's Challenger with the auxiliary polynomials and the CTL vars simulated."""
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
            z = T._ext_pow(z, pow_degree)
    zeta_prime = ch.get_extension_challenge()
    aux, aux_next = dummy[2 * C:2 * C + num_aux], dummy[2 * C + num_aux:total]
    nh = sum(len(v.helper_columns) for v in ctl_shape)
    ctl_vars, start = [], nl
    for i, v in enumerate(ctl_shape):
        m = len(v.helper_columns)
        ctl_vars.append(_Vars(aux[start:start + m], aux[nl + nh + i], aux_next[nl + nh + i], v.challenges, v.columns,
                              v.filter))
        start += m
    extra = dict(auxiliary_polys=aux, auxiliary_polys_next=aux_next, ctl_vars=ctl_vars)
    if stark.uses_lookups():
        extra["lookup_challenges"] = lookup_challenges
    evals = S.eval_vanishing_poly(stark, dummy[:C], dummy[C:2 * C], public_inputs, alphas_prime, zeta_prime,
                                  degree_bits, **extra)
    ch.observe_elements([w for e in evals for w in e])
    return ch.get_n_challenges(num_challenges)


def host_quotient(oracle, stark, trace_coeffs, aux_coeffs, public_inputs, alphas, lookup_challenges, ctl_shape):
    """compute_quotient_polys (prover.rs:488-668) on the host with the auxiliary LDE and the CTL constraints: the
    product's constraint program over numpy object arrays on the quotient coset, divided by Z_H, coset_ifft'd."""
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

    tv, av = lde(trace_coeffs), lde(aux_coeffs)
    w = T.root_of_unity(log_n + qd_bits)
    xs = np.array([SHIFT * pow(w, i, P) % P for i in range(size)], dtype=object)
    g = T.root_of_unity(log_n)
    last = pow(g, P - 2, P)
    zh = np.array([(pow(int(v), n, P) - 1) % P for v in xs], dtype=object)
    inv = np.vectorize(lambda v: pow(int(v), P - 2, P), otypes=[object])
    filters = [None, (xs - last) % P, zh * inv(n * (xs - 1) % P) % P, zh * inv(n * (xs * g - 1) % P) % P]
    challenges = [int(c) % P for c in lookup_challenges] if stark.uses_lookups() else []
    b = stark.constraint_program(len(challenges), ctl_shape)
    bound = [int(v) % P for c in ctl_shape for v in (c.challenges.beta, c.challenges.gamma)]
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


def fri_batches(stark, config, zeta, g, num_aux, ctl_first):
    """fri_instance (stark.rs:101-170) with CTLs: trace, auxiliary and quotient oracles at zeta, trace and auxiliary at
    g * zeta, the auxiliary oracle's CTL Zs (range ctl_first) at 1."""
    from plonky2_b200 import field as F

    nq = stark.num_quotient_polys(config)
    opened_next = [(0, i) for i in range(stark.COLUMNS)] + [(1, j) for j in range(num_aux)]
    qi = 2 if num_aux else 1
    out = [(zeta, opened_next + [(qi, j) for j in range(nq)]), (F.ext_mul((g, 0), zeta), opened_next)]
    if ctl_first is not None:
        out.append(((1, 0), [(1, j) for j in ctl_first]))
    return out


def _shape_vars(zs_columns):
    return [_Vars([None] * len(z["helpers"]), None, None, _gpc(z["challenge"]), z["columns"], z["filter"])
            for z in zs_columns]


def twin_prove(oracle, starks, config, traces, ctls, public_inputs):
    """prove_with_ctls with the oracle's pieces. Returns dict(ctl_challenges, ctl_data, tables: per table a dict
    trace_cap, aux_cap, quotient_cap, local_values, next_values, auxiliary_polys, auxiliary_polys_next, ctl_zs_first,
    quotient_polys, fri_bytes, alphas, zeta)."""
    f = config.fri_config
    traces = [np.ascontiguousarray(t, dtype=np.uint64) for t in traces]
    tcs = [oracle.Commit(t, f.rate_bits, f.cap_height) for t in traces]
    ch = oracle.Challenger()
    for tc in tcs:
        ch.observe_cap(tc.cap)
    pairs = LT._draw_lookup_challenges(ch, config.num_challenges)
    max_degree = max(s.constraint_degree() for s in starks)
    data = cross_table_lookup_data(traces, ctls, pairs, max_degree)
    betas = [b for b, _ in pairs]
    tables = []
    for i, (stark, trace, tc) in enumerate(zip(starks, traces, tcs)):
        n = trace.shape[1]
        degree_bits = n.bit_length() - 1
        pis = [int(v) % P for v in public_inputs[i]]
        ch.observe_elements(pis)
        T.observe_config(ch, config)
        lookup_aux = LT.aux_columns(stark, trace, betas)[0] if stark.uses_lookups() else np.zeros((0, n), np.uint64)
        nl = lookup_aux.shape[0]
        aux = np.concatenate([lookup_aux, ctl_aux(data[i], n)])
        shape = _shape_vars(data[i]) if stark.requires_ctls() else []
        ac = None
        if aux.shape[0]:
            ac = oracle.Commit(aux, f.rate_bits, f.cap_height)
            ch.observe_cap(ac.cap)
        alphas = bind_constraints(ch, stark, pis, config.num_challenges, degree_bits, betas, aux.shape[0], nl, shape)
        q = host_quotient(oracle, stark, tc.coeffs, ac.coeffs if ac is not None else np.zeros((0, n), np.uint64), pis,
                          alphas, betas, shape)
        commits, qc = [tc] + ([ac] if ac is not None else []), None
        if q is not None:
            qc = oracle.Commit(T.quotient_chunks(stark, q, n), f.rate_bits, f.cap_height, is_coeffs=True)
            commits.append(qc)
            ch.observe_cap(qc.cap)
        zeta = ch.get_extension_challenge()
        g = T.root_of_unity(degree_bits)
        nh = sum(len(z["helpers"]) for z in data[i])
        ctl_first = range(nl + nh, aux.shape[0]) if stark.requires_ctls() else None
        batches = fri_batches(stark, config, zeta, g, aux.shape[0], ctl_first)
        zn = batches[1][0]
        local, nxt = T._ev(oracle, tc, zeta), T._ev(oracle, tc, zn)
        al = T._ev(oracle, ac, zeta) if ac is not None else None
        an = T._ev(oracle, ac, zn) if ac is not None else None
        quot = T._ev(oracle, qc, zeta) if qc is not None else None
        first = np.array([int(aux[j, 0]) for j in ctl_first], dtype=np.uint64) if ctl_first is not None else None
        ch.observe_elements(np.concatenate([local] + ([al] if al is not None else []) +
                                           ([quot] if quot is not None else [])).reshape(-1))
        ch.observe_elements(np.concatenate([nxt] + ([an] if an is not None else [])).reshape(-1))
        if first is not None:
            ch.observe_elements(np.stack([first, np.zeros_like(first)], axis=1).reshape(-1))
        arity_bits = f.fri_params(degree_bits, False).reduction_arity_bits
        params = oracle.make_params(f.rate_bits, f.cap_height, f.proof_of_work_bits, f.num_query_rounds, arity_bits)
        fri_bytes = oracle.prove_openings(commits, batches, ch, params)
        tables.append(dict(trace_cap=tc.cap, aux_cap=ac.cap if ac is not None else None,
                           quotient_cap=qc.cap if qc is not None else None, local_values=local, next_values=nxt,
                           auxiliary_polys=al, auxiliary_polys_next=an, ctl_zs_first=first, quotient_polys=quot,
                           fri_bytes=fri_bytes, alphas=alphas, zeta=zeta, aux_values=aux))
    return dict(ctl_challenges=pairs, ctl_data=data, tables=tables)


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


def verify_table(oracle, stark, config, proof_with_pis, ch, challenges, ctl_vars):
    """verify_stark_proof_with_challenges (verifier.rs:30-285) for one table of a multi-STARK proof: the challenger
    has observed every trace cap and drawn the CTL challenges; validate_proof_shape includes the ctl_zs_first length.
    Returns None if accepted, else the reason."""
    from plonky2_b200 import field as F
    from plonky2_b200 import stark as S
    from plonky2_b200.fri import fri_challenges

    p, pis = proof_with_pis.proof, list(proof_with_pis.public_inputs)
    o, f = p.openings, config.fri_config
    nq = stark.num_quotient_polys(config)
    nl = stark.num_lookup_helper_columns(config) if stark.uses_lookups() else 0
    ctl_vars = ctl_vars or []
    nh, nz = sum(len(v.helper_columns) for v in ctl_vars), len(ctl_vars)
    num_aux = nl + nh + nz
    if len(pis) != stark.PUBLIC_INPUTS:
        return "public inputs"
    if len(o.local_values) != stark.COLUMNS or len(o.next_values) != stark.COLUMNS:
        return "opened trace values"
    if (o.quotient_polys is None) != (nq == 0) or (nq and len(o.quotient_polys) != nq):
        return "opened quotient values"
    if stark.uses_lookups() or stark.requires_ctls():
        if p.auxiliary_polys_cap is None or o.auxiliary_polys is None or o.auxiliary_polys_next is None:
            return "Missing auxiliary data"
        if len(o.auxiliary_polys) != num_aux or len(o.auxiliary_polys_next) != num_aux:
            return "opened auxiliary values"
        if stark.requires_ctls() and (o.ctl_zs_first is None or len(o.ctl_zs_first) != nz):
            return "ctl_zs_first length"
    elif p.auxiliary_polys_cap is not None or o.ctl_zs_first is not None:
        return "auxiliary data for a Stark without lookups or CTLs"
    degree_bits = p.recover_degree_bits(config)
    ch.observe_elements(pis)
    T.observe_config(ch, config)
    betas = [b for b, _ in challenges]
    if p.auxiliary_polys_cap is not None:
        ch.observe_cap(p.auxiliary_polys_cap.hashes)
    alphas = bind_constraints(ch, stark, pis, config.num_challenges, degree_bits, betas, num_aux, nl, ctl_vars)
    if p.quotient_polys_cap is not None:
        ch.observe_cap(p.quotient_polys_cap.hashes)
    zeta = ch.get_extension_challenge()
    aux, aux_next = ([o.auxiliary_polys], [o.auxiliary_polys_next]) if num_aux else ([], [])
    zeta_batch = np.concatenate([o.local_values] + aux + ([o.quotient_polys] if nq else []))
    next_batch = np.concatenate([np.asarray(o.next_values)] + aux_next)
    ch.observe_elements(zeta_batch.reshape(-1))
    ch.observe_elements(next_batch.reshape(-1))
    first_batch = None
    if stark.requires_ctls():
        first = np.asarray(o.ctl_zs_first, dtype=np.uint64)
        first_batch = np.stack([first, np.zeros_like(first)], axis=1)
        ch.observe_elements(first_batch.reshape(-1))
    extra = dict(ctl_vars=ctl_vars) if stark.requires_ctls() else {}
    if num_aux:
        extra.update(auxiliary_polys=o.auxiliary_polys, auxiliary_polys_next=o.auxiliary_polys_next)
    if stark.uses_lookups():
        extra["lookup_challenges"] = betas
    vanishing = S.eval_vanishing_poly(stark, o.local_values, o.next_values, pis, alphas, zeta, degree_bits, **extra)
    zeta_pow_deg = T._ext_pow(zeta, 1 << degree_bits)
    z_h = F.ext_sub(zeta_pow_deg, (1, 0))
    qdf = stark.quotient_degree_factor()
    for i in range(nq // max(qdf, 1)):
        t = (0, 0)
        for v in reversed(o.quotient_polys[i * qdf:(i + 1) * qdf]):
            t = F.ext_add(F.ext_mul(t, zeta_pow_deg), (int(v[0]), int(v[1])))
        if vanishing[i] != F.ext_mul(z_h, t):
            return "Mismatch between evaluation and opening of quotient polynomial"
    g = T.root_of_unity(degree_bits)
    ctl_first = range(nl + nh, num_aux) if stark.requires_ctls() else None
    batches = fri_batches(stark, config, zeta, g, num_aux, ctl_first)
    arity_bits = config.fri_params(degree_bits).reduction_arity_bits
    params = oracle.make_params(f.rate_bits, f.cap_height, f.proof_of_work_bits, f.num_query_rounds, arity_bits)
    caps = [p.trace_cap.hashes] + ([p.auxiliary_polys_cap.hashes] if num_aux else []) + (
        [p.quotient_polys_cap.hashes] if nq else [])
    widths = [stark.COLUMNS] + ([num_aux] if num_aux else []) + ([nq] if nq else [])
    opened = [zeta_batch.reshape(-1), next_batch.reshape(-1)] + ([first_batch.reshape(-1)] if first_batch is not None
                                                                 else [])
    rc = oracle.verify_fri_proof(caps, widths, widths, batches, np.concatenate(opened), degree_bits, ch.clone(), params,
                                 p.opening_proof.to_bytes())
    fp = p.opening_proof                  # the next table's transcript continues after FRI's
    fri_challenges(ch, [c.hashes for c in fp.commit_phase_merkle_caps], fp.final_poly, fp.pow_witness, degree_bits, f)
    return None if rc == 0 else "verify_fri_proof rc=%d" % rc


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


def verify(oracle, starks, config, ctls, multi_proof, extra_looking_sums=None):
    """The multi-STARK verifier: the transcript of prove_with_ctls, every table's STARK check with its CtlCheckVars,
    then verify_cross_table_lookups. Returns None if accepted, else the reason (with the table)."""
    proofs = multi_proof.stark_proofs
    if len(proofs) != len(starks):
        return "number of proofs"
    ch = oracle.Challenger()
    for p in proofs:
        ch.observe_cap(p.proof.trace_cap.hashes)
    challenges = LT._draw_lookup_challenges(ch, config.num_challenges)
    for i, (stark, p) in enumerate(zip(starks, proofs)):
        ctl_vars = None
        if stark.requires_ctls():
            if p.proof.openings.auxiliary_polys is None:
                return "table %d: We cannot have CTLs without auxiliary polynomials." % i
            total, num_zs, by_ctl = num_ctl_helpers_zs_all(ctls, i, config.num_challenges, stark.constraint_degree())
            nl = stark.num_lookup_helper_columns(config) if stark.uses_lookups() else 0
            o = p.proof.openings
            if len(o.auxiliary_polys) != nl + total + num_zs or len(o.auxiliary_polys_next) != nl + total + num_zs:
                return "table %d: opened auxiliary values" % i
            ctl_vars = ctl_vars_from_proof(i, p.proof, ctls, challenges, nl, total, by_ctl)
        reason = verify_table(oracle, stark, config, p, ch, challenges, ctl_vars)
        if reason is not None:
            return "table %d: %s" % (i, reason)
    return verify_cross_table_lookups(ctls, [p.proof.openings.ctl_zs_first for p in proofs], config.num_challenges,
                                      extra_looking_sums)
