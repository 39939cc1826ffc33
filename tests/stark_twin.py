"""starky proofs on the CPU: a twin of stark.prove assembled from the oracle's pieces, and a restated verify_stark_proof.

twin_prove follows starky/src/prover.rs:40-484 (no lookups, no CTLs) with the oracle's Commit, Challenger, openings
(eval_poly_base_at_ext) and prove_openings; the quotient is the oracle's for FibonacciStark and, for any other Stark,
host_quotient: the constraint program evaluated over numpy object arrays on the quotient coset, divided by Z_H,
coset_ifft'd by the oracle. The constraint-binding step restates get_dummy_polys (get_challenges.rs:201-256) here and
evaluates the constraints with the product's eval_vanishing_poly, which the tests check against hand-written formulas.

verify restates verify_stark_proof (verifier.rs:30-285): shape validation, the transcript replayed on the oracle's
Challenger, the quotient identity at zeta, and the oracle's verify_fri_proof. Returns None or the reason."""
import numpy as np

P = 0xFFFFFFFF00000001
SHIFT = 7  # F::coset_shift() = MULTIPLICATIVE_GROUP_GENERATOR


def _stark_mod():
    from plonky2_b200 import stark

    return stark


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


def bind_constraints(ch, stark, public_inputs, num_challenges, degree_bits):
    """prover.rs:239-370 / get_challenges.rs:94-163 on the oracle's Challenger: alphas', dummy openings, zeta', the
    vanishing polynomial observed; returns the alphas."""
    alphas_prime = ch.get_n_challenges(num_challenges)
    pow_degree = max(2, stark.constraint_degree() + 1)
    log_pow_degree = (pow_degree - 1).bit_length()
    k = max(1, 50 // log_pow_degree - 1)
    total = 2 * stark.COLUMNS
    zetas = [ch.get_extension_challenge() for _ in range((total + k - 1) // k)]
    dummy = []
    for z in zetas:
        for _ in range(min(k + 1, total)):
            dummy.append(z)
            z = _ext_pow(z, pow_degree)
    zeta_prime = ch.get_extension_challenge()
    evals = _stark_mod().eval_vanishing_poly(stark, dummy[:stark.COLUMNS], dummy[stark.COLUMNS:total], public_inputs,
                                             alphas_prime, zeta_prime, degree_bits)
    ch.observe_elements([w for e in evals for w in e])
    return ch.get_n_challenges(num_challenges)


def host_quotient(oracle, stark, coeffs, public_inputs, alphas):
    """compute_quotient_polys (prover.rs:488-668) on the host: (num_challenges, n << log2_ceil(qdf)) coefficients, or
    None without constraints; raises like prover.rs:396-401 when the vanishing polynomial is not divisible by Z_H."""
    qdf = stark.quotient_degree_factor()
    if qdf == 0:
        return None
    B, n = coeffs.shape
    log_n = n.bit_length() - 1
    qd_bits = (qdf - 1).bit_length()
    size = n << qd_bits
    vals = []
    for c in coeffs:
        pad = np.zeros(size, dtype=np.uint64)
        pad[:n] = c
        vals.append(oracle.coset_fft(pad, SHIFT).astype(object))
    w = root_of_unity(log_n + qd_bits)
    xs, x = [], SHIFT
    for _ in range(size):
        xs.append(x)
        x = x * w % P
    xs = np.array(xs, dtype=object)
    last = pow(root_of_unity(log_n), P - 2, P)
    zh = np.array([(pow(int(v), n, P) - 1) % P for v in xs], dtype=object)
    inv = np.vectorize(lambda v: pow(int(v), P - 2, P), otypes=[object])
    z_last = (xs - last) % P
    l_0 = zh * inv(n * (xs - 1) % P) % P
    l_last = zh * inv(n * (xs * root_of_unity(log_n) - 1) % P) % P
    filters = [None, z_last, l_0, l_last]
    b = stark.constraint_program()
    consts = [int(v) % P for v in public_inputs] + b.consts[b.num_pi:]
    step = 1 << qd_bits
    acc = [np.zeros(size, dtype=object) for _ in alphas]
    v = []
    for op, a, c in b.instrs:
        r = None
        if op == 0:
            r = vals[a]
        elif op == 1:
            r = np.roll(vals[a], -step)
        elif op == 2:
            r = consts[a]
        elif op == 3:
            r = (v[a] + v[c]) % P
        elif op == 4:
            r = (v[a] - v[c]) % P
        elif op == 5:
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


def quotient(oracle, stark, trace_commit, public_inputs, alphas):
    from plonky2_b200.stark import FibonacciStark

    if isinstance(stark, FibonacciStark):
        return oracle.stark_quotient_fibonacci(trace_commit, public_inputs, alphas)
    return host_quotient(oracle, stark, trace_commit.coeffs, public_inputs, alphas)


def quotient_chunks(stark, q, n):
    qdf = stark.quotient_degree_factor()
    return np.concatenate([q[i, :qdf * n].reshape(qdf, n) for i in range(q.shape[0])])


def _ev(oracle, commit, z):
    return np.array([oracle.eval_poly_base_at_ext(p, z) for p in commit.coeffs], dtype=np.uint64).reshape(-1, 2)


def fri_batches(stark, config, zeta, g):
    from plonky2_b200 import field as F

    nq = stark.num_quotient_polys(config)
    trace = [(0, i) for i in range(stark.COLUMNS)]
    return [(zeta, trace + [(1, j) for j in range(nq)]), (F.ext_mul((g, 0), zeta), trace)]


def twin_prove(oracle, stark, config, trace, public_inputs):
    """prove (prover.rs:40-484) with the oracle's pieces. Returns a dict: trace_cap, quotient_cap (or None),
    local_values, next_values, quotient_polys (or None), fri_bytes, alphas, zeta."""
    f = config.fri_config
    trace = np.ascontiguousarray(trace, dtype=np.uint64)
    n = trace.shape[1]
    degree_bits = n.bit_length() - 1
    arity_bits = f.fri_params(degree_bits, False).reduction_arity_bits
    tc = oracle.Commit(trace, f.rate_bits, f.cap_height)
    ch = oracle.Challenger()
    ch.observe_elements([int(v) % P for v in public_inputs])
    observe_config(ch, config)
    ch.observe_cap(tc.cap)
    alphas = bind_constraints(ch, stark, public_inputs, config.num_challenges, degree_bits)
    q = quotient(oracle, stark, tc, public_inputs, alphas)
    commits, qc = [tc], None
    if q is not None:
        qc = oracle.Commit(quotient_chunks(stark, q, n), f.rate_bits, f.cap_height, is_coeffs=True)
        commits.append(qc)
        ch.observe_cap(qc.cap)
    zeta = ch.get_extension_challenge()
    g = root_of_unity(degree_bits)
    batches = fri_batches(stark, config, zeta, g)
    local, nxt = _ev(oracle, tc, zeta), _ev(oracle, tc, batches[1][0])
    quot = _ev(oracle, qc, zeta) if qc is not None else None
    ch.observe_elements(np.concatenate([local] + ([quot] if quot is not None else [])).reshape(-1))
    ch.observe_elements(nxt.reshape(-1))
    params = oracle.make_params(f.rate_bits, f.cap_height, f.proof_of_work_bits, f.num_query_rounds, arity_bits)
    fri_bytes = oracle.prove_openings(commits, batches, ch, params)
    return dict(trace_cap=tc.cap, quotient_cap=qc.cap if qc is not None else None, local_values=local,
                next_values=nxt, quotient_polys=quot, fri_bytes=fri_bytes, alphas=alphas, zeta=zeta)


def verify(oracle, stark, config, proof_with_pis):
    """verify_stark_proof (verifier.rs:30-285) of a stark.StarkProofWithPublicInputs. Returns None if accepted, else
    the reason."""
    from plonky2_b200 import field as F

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
    degree_bits = p.recover_degree_bits(config)
    ch = oracle.Challenger()
    ch.observe_elements(pis)
    observe_config(ch, config)
    ch.observe_cap(p.trace_cap.hashes)
    alphas = bind_constraints(ch, stark, pis, config.num_challenges, degree_bits)
    if p.quotient_polys_cap is not None:
        ch.observe_cap(p.quotient_polys_cap.hashes)
    zeta = ch.get_extension_challenge()
    zeta_batch = np.concatenate([o.local_values] + ([o.quotient_polys] if nq else []))
    ch.observe_elements(zeta_batch.reshape(-1))
    ch.observe_elements(np.asarray(o.next_values).reshape(-1))
    vanishing = _stark_mod().eval_vanishing_poly(stark, o.local_values, o.next_values, pis, alphas, zeta, degree_bits)
    zeta_pow_deg = _ext_pow(zeta, 1 << degree_bits)
    z_h = F.ext_sub(zeta_pow_deg, (1, 0))
    qdf = stark.quotient_degree_factor()
    for i in range(nq // max(qdf, 1)):
        t = (0, 0)
        for v in reversed(o.quotient_polys[i * qdf:(i + 1) * qdf]):        # reduce_with_powers(chunk, zeta^n)
            t = F.ext_add(F.ext_mul(t, zeta_pow_deg), (int(v[0]), int(v[1])))
        if vanishing[i] != F.ext_mul(z_h, t):
            return "Mismatch between evaluation and opening of quotient polynomial"
    g = root_of_unity(degree_bits)
    batches = fri_batches(stark, config, zeta, g)
    arity_bits = config.fri_params(degree_bits).reduction_arity_bits
    params = oracle.make_params(f.rate_bits, f.cap_height, f.proof_of_work_bits, f.num_query_rounds, arity_bits)
    caps = [p.trace_cap.hashes] + ([p.quotient_polys_cap.hashes] if nq else [])
    widths = [stark.COLUMNS] + ([nq] if nq else [])
    opened = np.concatenate([zeta_batch.reshape(-1), np.asarray(o.next_values).reshape(-1)])
    rc = oracle.verify_fri_proof(caps, widths, widths, batches, opened, degree_bits, ch, params,
                                 p.opening_proof.to_bytes())
    return None if rc == 0 else "verify_fri_proof rc=%d" % rc
