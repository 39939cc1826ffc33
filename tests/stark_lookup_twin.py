"""starky proofs WITH logUp lookups on the CPU: a restatement of lookup_helper_columns, a twin of stark.prove with the
auxiliary oracle, and a restated verify_stark_proof with check_lookup_options. Test infrastructure only.

helper_columns restates lookup_helper_columns / get_helper_cols (starky/src/lookup.rs:579-652,746-789) literally over
Python integers: Column::eval_table / Filter::eval_table row by row (lookup.rs:118-129,323-335), one inversion per element
(not the batch form the device uses), then the running sum Z. twin_prove follows prover.rs:40-484 with the oracle's
Commit, Challenger, openings and prove_openings; the quotient is evaluated on the host over the trace and auxiliary LDEs
(the product's constraint program, whose lookup terms the tests check against hand-written formulas), divided by Z_H and
coset_ifft'd by the oracle. verify restates verifier.rs:30-330. The lookup-free path of tests/stark_twin.py is reused
unchanged (observe_config, quotient_chunks, _ev)."""
import numpy as np

import stark_twin as T

P = 0xFFFFFFFF00000001
SHIFT = T.SHIFT


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


def bind_constraints(ch, stark, public_inputs, num_challenges, degree_bits, lookup_challenges, num_aux):
    """prover.rs:239-370 on the oracle's Challenger with the auxiliary polynomials simulated too (prover.rs:272-319)."""
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
    extra = {}
    if lookup_challenges is not None:
        extra = dict(auxiliary_polys=dummy[2 * C:2 * C + num_aux], auxiliary_polys_next=dummy[2 * C + num_aux:total],
                     lookup_challenges=lookup_challenges)
    evals = S.eval_vanishing_poly(stark, dummy[:C], dummy[C:2 * C], public_inputs, alphas_prime, zeta_prime, degree_bits,
                                  **extra)
    ch.observe_elements([w for e in evals for w in e])
    return ch.get_n_challenges(num_challenges)


def host_quotient(oracle, stark, trace_coeffs, aux_coeffs, public_inputs, alphas, lookup_challenges):
    """compute_quotient_polys (prover.rs:488-668) on the host with the auxiliary LDE: the product's constraint program
    (lookup terms included) over numpy object arrays on the quotient coset, divided by Z_H, coset_ifft'd."""
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
    challenges = [int(c) % P for c in lookup_challenges]
    b = stark.constraint_program(len(challenges))
    consts = [int(v) % P for v in public_inputs] + challenges + b.consts[b.num_bound:]
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


def fri_batches(stark, config, zeta, g):
    """fri_instance (stark.rs:101-170): trace, auxiliary and quotient oracles."""
    from plonky2_b200 import field as F

    nq = stark.num_quotient_polys(config)
    na = stark.num_lookup_helper_columns(config)
    opened_next = [(0, i) for i in range(stark.COLUMNS)] + [(1, j) for j in range(na)]
    return [(zeta, opened_next + [(2, j) for j in range(nq)]), (F.ext_mul((g, 0), zeta), opened_next)]


def _draw_lookup_challenges(ch, num_challenges):
    """get_grand_product_challenge_set (lookup.rs:525-543) on the oracle's Challenger: (beta, gamma) pairs."""
    out = []
    for _ in range(num_challenges):
        beta = ch.get_challenge()
        out.append((beta, ch.get_challenge()))
    return out


def twin_prove(oracle, stark, config, trace, public_inputs):
    """prove (prover.rs:40-484) for a Stark with lookups with the oracle's pieces. Returns a dict: trace_cap, aux_cap,
    quotient_cap (or None), local_values, next_values, auxiliary_polys, auxiliary_polys_next, quotient_polys (or None),
    fri_bytes, lookup_challenge_set, alphas, zeta."""
    f = config.fri_config
    trace = np.ascontiguousarray(trace, dtype=np.uint64)
    n = trace.shape[1]
    degree_bits = n.bit_length() - 1
    arity_bits = f.fri_params(degree_bits, False).reduction_arity_bits
    tc = oracle.Commit(trace, f.rate_bits, f.cap_height)
    ch = oracle.Challenger()
    ch.observe_elements([int(v) % P for v in public_inputs])
    T.observe_config(ch, config)
    ch.observe_cap(tc.cap)
    pairs = _draw_lookup_challenges(ch, config.num_challenges)
    betas = [b for b, _ in pairs]
    aux, _ = aux_columns(stark, trace, betas)
    ac = oracle.Commit(aux, f.rate_bits, f.cap_height)
    ch.observe_cap(ac.cap)
    alphas = bind_constraints(ch, stark, public_inputs, config.num_challenges, degree_bits, betas, aux.shape[0])
    q = host_quotient(oracle, stark, tc.coeffs, ac.coeffs, public_inputs, alphas, betas)
    commits, qc = [tc, ac], None
    if q is not None:
        qc = oracle.Commit(T.quotient_chunks(stark, q, n), f.rate_bits, f.cap_height, is_coeffs=True)
        commits.append(qc)
        ch.observe_cap(qc.cap)
    zeta = ch.get_extension_challenge()
    g = T.root_of_unity(degree_bits)
    batches = fri_batches(stark, config, zeta, g)
    zn = batches[1][0]
    local, nxt, al, an = T._ev(oracle, tc, zeta), T._ev(oracle, tc, zn), T._ev(oracle, ac, zeta), T._ev(oracle, ac, zn)
    quot = T._ev(oracle, qc, zeta) if qc is not None else None
    ch.observe_elements(np.concatenate([local, al] + ([quot] if quot is not None else [])).reshape(-1))
    ch.observe_elements(np.concatenate([nxt, an]).reshape(-1))
    params = oracle.make_params(f.rate_bits, f.cap_height, f.proof_of_work_bits, f.num_query_rounds, arity_bits)
    fri_bytes = oracle.prove_openings(commits, batches, ch, params)
    return dict(trace_cap=tc.cap, aux_cap=ac.cap, quotient_cap=qc.cap if qc is not None else None, local_values=local,
                next_values=nxt, auxiliary_polys=al, auxiliary_polys_next=an, quotient_polys=quot, fri_bytes=fri_bytes,
                lookup_challenge_set=pairs, alphas=alphas, zeta=zeta)


def check_lookup_options(stark, config, proof):
    """check_lookup_options (verifier.rs:287-332) without CTLs. Returns None or the reason."""
    o = proof.openings
    if stark.uses_lookups():
        num_aux = stark.num_lookup_helper_columns(config)
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
        return "auxiliary data for a Stark without lookups"
    return None


def verify(oracle, stark, config, proof_with_pis):
    """verify_stark_proof (verifier.rs:30-285) with lookups and check_lookup_options. Returns None if accepted, else
    the reason."""
    from plonky2_b200 import field as F
    from plonky2_b200 import stark as S

    p, pis = proof_with_pis.proof, list(proof_with_pis.public_inputs)
    o, f = p.openings, config.fri_config
    nq = stark.num_quotient_polys(config)
    if len(pis) != stark.PUBLIC_INPUTS:
        return "public inputs"
    if len(p.trace_cap.hashes) != 1 << f.cap_height:
        return "trace cap height"
    if (p.quotient_polys_cap is None) != (nq == 0) or (nq and len(p.quotient_polys_cap.hashes) != 1 << f.cap_height):
        return "quotient cap"
    if len(o.local_values) != stark.COLUMNS or len(o.next_values) != stark.COLUMNS:
        return "opened trace values"
    if (o.quotient_polys is None) != (nq == 0) or (nq and len(o.quotient_polys) != nq):
        return "opened quotient values"
    reason = check_lookup_options(stark, config, p)
    if reason is not None:
        return reason
    degree_bits = p.recover_degree_bits(config)
    ch = oracle.Challenger()
    ch.observe_elements(pis)
    T.observe_config(ch, config)
    ch.observe_cap(p.trace_cap.hashes)
    betas = None
    if p.auxiliary_polys_cap is not None:
        betas = [b for b, _ in _draw_lookup_challenges(ch, config.num_challenges)]
        ch.observe_cap(p.auxiliary_polys_cap.hashes)
    num_aux = len(o.auxiliary_polys) if o.auxiliary_polys is not None else 0
    alphas = bind_constraints(ch, stark, pis, config.num_challenges, degree_bits, betas, num_aux)
    if p.quotient_polys_cap is not None:
        ch.observe_cap(p.quotient_polys_cap.hashes)
    zeta = ch.get_extension_challenge()
    aux, aux_next = [o.auxiliary_polys] if num_aux else [], [o.auxiliary_polys_next] if num_aux else []
    zeta_batch = np.concatenate([o.local_values] + aux + ([o.quotient_polys] if nq else []))
    next_batch = np.concatenate([np.asarray(o.next_values)] + aux_next)
    ch.observe_elements(zeta_batch.reshape(-1))
    ch.observe_elements(next_batch.reshape(-1))
    extra = {}
    if stark.uses_lookups():
        extra = dict(auxiliary_polys=o.auxiliary_polys, auxiliary_polys_next=o.auxiliary_polys_next,
                     lookup_challenges=betas)
    vanishing = S.eval_vanishing_poly(stark, o.local_values, o.next_values, pis, alphas, zeta, degree_bits, **extra)
    zeta_pow_deg = T._ext_pow(zeta, 1 << degree_bits)
    z_h = F.ext_sub(zeta_pow_deg, (1, 0))
    qdf = stark.quotient_degree_factor()
    for i in range(nq // max(qdf, 1)):
        t = (0, 0)
        for v in reversed(o.quotient_polys[i * qdf:(i + 1) * qdf]):        # reduce_with_powers(chunk, zeta^n)
            t = F.ext_add(F.ext_mul(t, zeta_pow_deg), (int(v[0]), int(v[1])))
        if vanishing[i] != F.ext_mul(z_h, t):
            return "Mismatch between evaluation and opening of quotient polynomial"
    g = T.root_of_unity(degree_bits)
    batches = fri_batches(stark, config, zeta, g)
    arity_bits = config.fri_params(degree_bits).reduction_arity_bits
    params = oracle.make_params(f.rate_bits, f.cap_height, f.proof_of_work_bits, f.num_query_rounds, arity_bits)
    caps = [p.trace_cap.hashes] + ([p.auxiliary_polys_cap.hashes] if num_aux else []) + (
        [p.quotient_polys_cap.hashes] if nq else [])
    widths = [stark.COLUMNS] + ([num_aux] if num_aux else []) + ([nq] if nq else [])
    opened = np.concatenate([zeta_batch.reshape(-1), next_batch.reshape(-1)])
    rc = oracle.verify_fri_proof(caps, widths, widths, batches, opened, degree_bits, ch, params,
                                 p.opening_proof.to_bytes())
    return None if rc == 0 else "verify_fri_proof rc=%d" % rc
