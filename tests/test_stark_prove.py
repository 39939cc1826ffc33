"""starky proofs end to end (stark.prove, StarkProofWithPublicInputs.get_challenges, eval_vanishing_poly).

CPU: the F_{p^2} constraint evaluator against hand-written formulas; prove's host logic with the oracle standing in for
the device calls -- accepted by the restated verifier (tests/stark_twin.py), field-for-field equal to the CPU twin, its
transcript replayed by get_challenges, tampered proofs rejected; a STARK without constraints (no quotient oracle); the
ConstantArityBits path of verifier_circuit_fri_params; every shape error.

GPU (-m gpu): stark.prove on the device equal to the CPU twin field by field and accepted by the restated verifier for
FibonacciStark at 2^5 / 2^10 / 2^16 rows, a cubic toy STARK, the unconstrained STARK and a 64-column STARK at 2^16 rows
(a device trace); a wrong cell raises "Quotient has failed"; the verifier_circuit_fri_params path on the device."""
import importlib.util
import os

import numpy as np
import pytest

import stark_twin as T
from conftest import P, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _S():
    from plonky2_b200 import stark

    return stark


def _cubic_stark():
    S = _S()

    class CubicStark(S.Stark):
        """The toy of test_stark_quotient_generic_program_higher_degree: a' = a^2 b + 1, b' = b + 3a."""
        COLUMNS, PUBLIC_INPUTS = 2, 1

        def eval(self, v, y):
            a, b = v.local(0), v.local(1)
            y.constraint_first_row(a - v.public_input(0))
            y.constraint_transition(v.next(0) - (a * a * b + 1))
            y.constraint_transition(v.next(1) - (b + a * 3))
            y.constraint(a * 0)

        def constraint_degree(self):
            return 4

        @staticmethod
        def trace(n, a=5, b=9):
            tr = np.empty((2, n), dtype=np.uint64)
            for i in range(n):
                tr[0, i], tr[1, i] = a, b
                a, b = (a * a * b + 1) % P, (b + 3 * a) % P
            return tr

    return CubicStark()


def _unconstrained_stark():
    S = _S()

    class UnconstrainedStark(S.Stark):
        """unconstrained_stark.rs: two columns, no constraints, constraint degree 0."""
        COLUMNS, PUBLIC_INPUTS = 2, 0

        def eval(self, v, y):
            pass

        def constraint_degree(self):
            return 0

    return UnconstrainedStark()


def _pairs_module():
    spec = importlib.util.spec_from_file_location("stark_prove_cost", os.path.join(ROOT, "tools", "stark_prove_cost.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _cubic_config():
    """rate 1/4 (constraint degree 4 needs blowup >= 3), fewer queries and grinding bits than standard_fast_config."""
    from plonky2_b200.fri import FriConfig

    return _S().StarkConfig(100, 2, FriConfig(rate_bits=2, cap_height=2, proof_of_work_bits=8,
                                              reduction_strategy=("ConstantArityBits", 2, 3), num_query_rounds=20))


def _fib_case(log_n):
    S = _S()
    n = 1 << log_n
    stark = S.FibonacciStark(n)
    trace = stark.generate_trace(0, 1)
    return stark, S.StarkConfig.standard_fast_config(), trace, [0, 1, int(trace[1, n - 1])]


# ----------------------------------------------------------------------------------------------------------- CPU
def test_eval_vanishing_poly_matches_hand_written_formulas():
    from plonky2_b200 import field as E

    S = _S()
    log_n = 6
    n = 1 << log_n
    g = E.primitive_root_of_unity(log_n)
    last = E.inverse(g)
    x = tuple(int(v) for v in synth(0x7A0, (2,)))
    vals = [tuple(int(w) for w in synth(0x7A1 + k, (2,))) for k in range(4)]
    alphas = [int(a) for a in synth(0x7A5, (2,))]
    zh = E.ext_sub(E.ext_pow(x, n), (1, 0))
    l_0 = E.ext_mul(zh, E.ext_inverse(E.ext_mul((n, 0), E.ext_sub(x, (1, 0)))))
    l_last = E.ext_mul(E.ext_mul(zh, (last, 0)), E.ext_inverse(E.ext_mul((n, 0), E.ext_sub(x, (last, 0)))))
    assert S.eval_l_0_and_l_last(log_n, x) == (l_0, l_last)
    z_last = E.ext_sub(x, (last, 0))

    def fold(cons):
        out = []
        for al in alphas:
            acc = (0, 0)
            for c in cons:
                acc = E.ext_add(E.ext_mul(acc, (al, 0)), c)
            out.append(acc)
        return out

    # FibonacciStark
    l0, l1, n0, n1 = vals
    pi = [3, 5, 8]
    cons = [E.ext_mul(E.ext_sub(l0, (pi[0], 0)), l_0), E.ext_mul(E.ext_sub(l1, (pi[1], 0)), l_0),
            E.ext_mul(E.ext_sub(l1, (pi[2], 0)), l_last), E.ext_mul(E.ext_sub(n0, l1), z_last),
            E.ext_mul(E.ext_sub(E.ext_sub(n1, l0), l1), z_last)]
    assert S.eval_vanishing_poly(S.FibonacciStark(n), [l0, l1], [n0, n1], pi, alphas, x, log_n) == fold(cons)
    # the cubic toy: a' = a^2 b + 1, b' = b + 3a, plus an unfiltered 0
    a, b, na, nb = vals
    cons = [E.ext_mul(E.ext_sub(a, (pi[0], 0)), l_0),
            E.ext_mul(E.ext_sub(na, E.ext_add(E.ext_mul(E.ext_mul(a, a), b), (1, 0))), z_last),
            E.ext_mul(E.ext_sub(nb, E.ext_add(b, E.ext_mul(a, (3, 0)))), z_last), (0, 0)]
    assert S.eval_vanishing_poly(_cubic_stark(), [a, b], [na, nb], pi[:1], alphas, x, log_n) == fold(cons)
    assert S.eval_vanishing_poly(_unconstrained_stark(), [a, b], [na, nb], [], alphas, x, log_n) == [(0, 0), (0, 0)]
    with pytest.raises(S.N.ShapeError):
        S.eval_vanishing_poly(S.FibonacciStark(n), [l0, l1], [n0, n1], pi[:2], alphas, x, log_n)


def test_host_quotient_matches_oracle(oracle):
    """The twin's generic quotient (used for every Stark but FibonacciStark) equals the oracle's Fibonacci one."""
    stark, _, trace, pi = _fib_case(6)
    tc = oracle.Commit(trace, 1, 2)
    alphas = [int(a) for a in synth(0x7B0, (2,))]
    assert np.array_equal(T.host_quotient(oracle, stark, tc.coeffs, pi, alphas),
                          oracle.stark_quotient_fibonacci(tc, pi, alphas))
    cubic = _cubic_stark()        # quotient_degree_factor 3: coefficients past 3n must vanish
    tr = cubic.trace(1 << 6)
    assert not T.host_quotient(oracle, cubic, oracle.Commit(tr, 2, 2).coeffs, [5], alphas)[:, 3 << 6:].any()
    tr[1, 7] ^= np.uint64(1)
    with pytest.raises(ValueError, match="Quotient has failed"):
        T.host_quotient(oracle, cubic, oracle.Commit(tr, 2, 2).coeffs, [5], alphas)


def _cpu_backends(monkeypatch, oracle, stark, calls):
    """Replace prove's device calls by the oracle: commitments, quotient, openings, FRI. Returns the list of transcript
    logs (one per Challenger made)."""
    import plonky2_b200.fri as fri_mod
    import plonky2_b200.proof as proof_mod
    from plonky2_b200.fri import FriProof
    from plonky2_b200.hash import MerkleCap

    S = _S()

    class Tree:
        def __init__(self, commit):
            self.cap = MerkleCap(commit.cap)

    class Batch:
        def __init__(self, commit):
            self.o, self.merkle_tree, self.num_polys = commit, Tree(commit), commit.B

        @classmethod
        def from_values(cls, values, rate_bits, blinding, cap_height, ctx=None):
            assert not blinding
            return cls(oracle.Commit(values, rate_bits, cap_height))

        def close(self):
            calls.append("close")

    def commit_quotient(stark_, q, degree_bits, rate_bits, cap_height, ctx=None):
        return Batch(oracle.Commit(T.quotient_chunks(stark_, q, 1 << degree_bits), rate_bits, cap_height, is_coeffs=True))

    def prove_openings(instance, oracles, challenger, fri_params, final_poly_coeff_len=None, max_num_query_steps=None):
        calls.append(("prove_openings", final_poly_coeff_len, max_num_query_steps))
        och = oracle.replay(challenger.log)
        batches = [(b.point, [(p.oracle_index, p.polynomial_index) for p in b.polynomials]) for b in instance.batches]
        f = fri_params.config
        params = oracle.make_params(f.rate_bits, f.cap_height, f.proof_of_work_bits, f.num_query_rounds,
                                    fri_params.reduction_arity_bits)
        data, taps = oracle.prove_openings([b.o for b in oracles], batches, och, params, taps=True)
        calls.append(("fri_taps", taps))
        return FriProof.from_bytes(data, [o.num_polys for o in instance.oracles], fri_params)[0]

    class Ctx:
        device, h = 0, None

    logs = oracle.log_transcripts(monkeypatch)
    monkeypatch.setattr(S, "PolynomialBatch", Batch)
    monkeypatch.setattr(S, "compute_quotient_polys", lambda stark_, tc, pis, alphas: T.quotient(oracle, stark_, tc.o, pis, alphas))
    monkeypatch.setattr(S, "commit_quotient_polys", commit_quotient)
    monkeypatch.setattr(proof_mod, "eval_commitments", lambda requests: [T._ev(oracle, b.o, z) for b, z in requests])
    monkeypatch.setattr(fri_mod, "prove_openings", prove_openings)
    return logs, Ctx()


def _tampered(proof, what):
    import copy

    from plonky2_b200.fri import FriProof

    bad = copy.deepcopy(proof)
    if what == "public_input":
        bad.public_inputs[-1] = (bad.public_inputs[-1] + 1) % P
    elif what == "opening":
        bad.proof.openings.next_values[0, 1] ^= np.uint64(1)
    else:   # one byte of the first initial-tree leaf of the FRI proof
        fp = bad.proof.opening_proof
        data = bytearray(fp.to_bytes())
        data[32 * len(fp.commit_phase_merkle_caps) * len(proof.proof.trace_cap.hashes) + 2] ^= 0x10
        widths = [len(leaf) for leaf, _ in fp.query_round_proofs[0].initial_trees_proof.evals_proofs]
        degree_bits = proof.proof.recover_degree_bits(_S().StarkConfig.standard_fast_config())
        params = _S().StarkConfig.standard_fast_config().fri_params(degree_bits)
        bad.proof.opening_proof = FriProof.from_bytes(bytes(data), widths, params)[0]
    return bad


@pytest.mark.parametrize("case", ["fibonacci", "unconstrained"])
def test_prove_host_logic_with_cpu_backends(oracle, monkeypatch, case):
    """FibonacciStark at the reference's test shape (fibonacci_stark.rs: 2^5 rows, public inputs [0, 1, fib],
    standard_fast_config) and the unconstrained STARK: prove's host logic with the oracle's pieces gives the twin's
    proof, the restated verifier accepts it, get_challenges replays the prover's transcript, tampering is rejected."""
    S = _S()
    if case == "fibonacci":
        stark, config, trace, pi = _fib_case(5)
    else:
        stark, config = _unconstrained_stark(), S.StarkConfig.standard_fast_config()
        trace, pi = synth(0x7C0, (2, 32)), []
    twin = T.twin_prove(oracle, stark, config, trace, pi)
    calls = []
    logs, ctx = _cpu_backends(monkeypatch, oracle, stark, calls)
    proof = S.prove(stark, config, trace, pi, ctx=ctx)
    assert calls.count("close") == (2 if case == "fibonacci" else 1)
    assert [c for c in calls if isinstance(c, tuple) and c[0] == "prove_openings"] == [("prove_openings", None, None)]
    T.assert_matches_twin(proof, twin)
    assert T.verify(oracle, stark, config, proof) is None
    assert len(proof.proof.opening_proof.query_round_proofs[0].initial_trees_proof.evals_proofs) == (
        2 if case == "fibonacci" else 1)
    assert proof.proof.recover_degree_bits(config) == 5
    # get_challenges: the prover's host draws are a prefix of the replay's, and the FRI indices are the oracle's
    ch = proof.get_challenges(stark, config)
    prover_draws = [v for kind, v in logs[0] if kind == "challenge"]
    replay_draws = [v for kind, v in logs[1] if kind == "challenge"]
    assert replay_draws[:len(prover_draws)] == prover_draws
    assert ch["stark_alphas"] == twin["alphas"] and ch["stark_zeta"] == twin["zeta"]
    taps = [c[1] for c in calls if isinstance(c, tuple) and c[0] == "fri_taps"][0]
    assert ch["fri_query_indices"] == [int(i) for i in taps["query_indices"]]
    for what in (["public_input"] if pi else []) + ["opening", "fri_byte"]:
        assert T.verify(oracle, stark, config, _tampered(proof, what)) is not None, what


def test_verifier_circuit_fri_params_and_shape_errors(oracle, monkeypatch):
    """The ConstantArityBits branch (prover.rs:62-81) hands the verifier circuit's final polynomial length and step
    count to prove_openings; every shape error is raised before any commitment, with the reference's wording."""
    from plonky2_b200.fri import FriConfig

    S = _S()
    stark, config, trace, pi = _fib_case(5)
    calls = []
    logs, ctx = _cpu_backends(monkeypatch, oracle, stark, calls)
    S.prove(stark, config, trace, pi, verifier_circuit_fri_params=config.fri_params(10), ctx=ctx)
    assert ("prove_openings", 64, 1) in calls                      # 2^10 -> arities [4], final 2^6 = 1 << (1 + 5)
    calls.clear()
    with pytest.raises(S.N.ShapeError, match="final polynomial"):
        S.prove(stark, config, trace, pi, verifier_circuit_fri_params=config.fri_params(9), ctx=ctx)
    fixed = S.StarkConfig(100, 2, FriConfig(1, 4, 16, ("Fixed", [1]), 84))
    with pytest.raises(S.N.ShapeError, match="not ConstantArityBits"):
        S.prove(stark, fixed, trace, pi, verifier_circuit_fri_params=fixed.fri_params(5), ctx=ctx)
    with pytest.raises(S.N.ShapeError, match="config differs"):
        S.prove(stark, config, trace, pi, verifier_circuit_fri_params=fixed.fri_params(5), ctx=ctx)
    big = S.StarkConfig(100, 2, FriConfig(1, 4, 16, ("Fixed", [2, 2]), 84))
    with pytest.raises(S.N.ShapeError, match="FRI total reduction arity is too large."):
        S.prove(stark, big, trace, pi, ctx=ctx)
    with pytest.raises(S.N.ShapeError, match="expected 3 public inputs, got 2"):
        S.prove(stark, config, trace, pi[:2], ctx=ctx)
    with pytest.raises(S.N.ShapeError, match="COLUMNS"):
        S.prove(stark, config, trace[:1], pi, ctx=ctx)
    with pytest.raises(S.N.ShapeError, match="blowup_factor"):
        S.prove(_cubic_stark(), config, _cubic_stark().trace(32), [5], ctx=ctx)
    assert "close" not in calls

    # an opening point in the subgroup: zeta is drawn right after the quotient cap is observed
    import plonky2_b200.challenger as challenger_mod

    base = challenger_mod.Challenger
    w = S.F.primitive_root_of_unity(5)

    class SubgroupZeta(base):
        caps = 0

        def observe_cap(self, cap):
            self.caps += 1
            super().observe_cap(cap)

        def get_extension_challenge(self):
            v = super().get_extension_challenge()
            return (w, 0) if self.caps == 2 else v

    monkeypatch.setattr(challenger_mod, "Challenger", SubgroupZeta)
    with pytest.raises(S.N.NativeError, match="Opening point is in the subgroup."):
        S.prove(stark, config, trace, pi, ctx=ctx)
    assert calls.count("close") == 2                               # both commitments released on the error path


def test_fibonacci_pairs_trace_generator():
    """tools/stark_prove_cost.py's device trace generator (run here on torch's CPU backend) satisfies the pair map."""
    m = _pairs_module()
    tr = m.fibonacci_pairs_trace(7, device="cpu").numpy().view(np.uint64)
    assert tr.shape == (64, 128) and np.array_equal(tr[:, 0], synth(0x05, (64,)))
    for k in range(32):
        x, y = int(tr[2 * k, 0]), int(tr[2 * k + 1, 0])
        for r in range(128):
            assert (int(tr[2 * k, r]), int(tr[2 * k + 1, r])) == (x, y)
            x, y = y, (x + y) % P
    stark = m.FibonacciPairsStark()
    assert len(stark.constraint_program().instrs) == 288


# ----------------------------------------------------------------------------------------------------------- GPU
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


def _gpu_case(name):
    S = _S()
    if name.startswith("fibonacci"):
        return _fib_case(int(name.split("_")[1]))
    if name == "cubic":
        stark = _cubic_stark()
        return stark, _cubic_config(), stark.trace(1 << 8), [5]
    if name == "unconstrained":
        return _unconstrained_stark(), S.StarkConfig.standard_fast_config(), synth(0x7C1, (2, 32)), []
    m = _pairs_module()
    return m.FibonacciPairsStark(), S.StarkConfig.standard_fast_config(), m.fibonacci_pairs_trace(16), []


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fibonacci_5", "fibonacci_10", "fibonacci_16", "cubic", "unconstrained", "pairs64_16"])
def test_prove_on_device_equals_cpu_twin(pb, oracle, name):
    """stark.prove on the device: caps, openings, final polynomial, PoW witness and write_fri_proof bytes equal the CPU
    twin's; the restated verifier accepts the proof and get_challenges replays the twin's alphas and zeta."""
    from plonky2_b200.fri import FriProof

    S = _S()
    stark, config, trace, pi = _gpu_case(name)
    host_trace = trace.cpu().numpy().view(np.uint64) if hasattr(trace, "data_ptr") else trace
    proof = S.prove(stark, config, trace, pi)
    twin = T.twin_prove(oracle, stark, config, host_trace, pi)
    T.assert_matches_twin(proof, twin)
    fp = proof.proof.opening_proof
    degree_bits = host_trace.shape[1].bit_length() - 1
    widths = [stark.COLUMNS] + ([stark.num_quotient_polys(config)] if stark.constraint_degree() else [])
    tw = FriProof.from_bytes(twin["fri_bytes"], widths, config.fri_params(degree_bits))[0]
    assert np.array_equal(fp.final_poly, tw.final_poly) and fp.pow_witness == tw.pow_witness
    assert all(np.array_equal(a.hashes, b.hashes) for a, b in zip(fp.commit_phase_merkle_caps, tw.commit_phase_merkle_caps))
    assert T.verify(oracle, stark, config, proof) is None
    ch = proof.get_challenges(stark, config)
    assert ch["stark_alphas"] == twin["alphas"] and ch["stark_zeta"] == twin["zeta"]


@pytest.mark.gpu
def test_prove_on_device_with_a_wrong_cell(pb, oracle):
    """One wrong cell: with quotient_degree_factor > 1 the quotient's top chunk does not vanish and prove raises
    "Quotient has failed" (prover.rs:396-401). FibonacciStark's quotient has one chunk, so the reference's trim cannot
    fail there; its proof is made, and the verifier rejects it at zeta."""
    S = _S()
    stark, config, trace, pi = _fib_case(10)
    trace = trace.copy()
    trace[0, 300] ^= np.uint64(1)
    assert T.verify(oracle, stark, config, S.prove(stark, config, trace, pi)) == (
        "Mismatch between evaluation and opening of quotient polynomial")
    cubic = _cubic_stark()
    tr = cubic.trace(1 << 8)
    tr[1, 100] ^= np.uint64(1)
    with pytest.raises(pb.NativeError, match="Quotient has failed"):
        S.prove(cubic, _cubic_config(), tr, [5])


@pytest.mark.gpu
def test_prove_on_device_for_a_verifier_circuit_of_another_degree(pb, oracle):
    """verifier_circuit_fri_params = the parameters of a 2^10-row verifier for a 2^5-row proof: get_challenges with the
    same parameters replays a transcript under which the proof of work holds and every query's initial-tree leaves open
    against the trace and quotient caps at the replayed indices; without them the replay differs."""
    S = _S()
    stark, config, trace, pi = _fib_case(5)
    vp = config.fri_params(10)
    proof = S.prove(stark, config, trace, pi, verifier_circuit_fri_params=vp)
    ch = proof.get_challenges(stark, config, vp)
    pow_bits = config.fri_config.proof_of_work_bits
    assert 64 - ch["fri_pow_response"].bit_length() >= pow_bits + 64 - P.bit_length()
    caps = [proof.proof.trace_cap.hashes, proof.proof.quotient_polys_cap.hashes]
    for index, qr in zip(ch["fri_query_indices"], proof.proof.opening_proof.query_round_proofs):
        for (leaf, sib), cap in zip(qr.initial_trees_proof.evals_proofs, caps):
            assert oracle.merkle_verify(leaf, index, sib, cap, config.fri_config.cap_height)
    plain = proof.get_challenges(stark, config)
    assert plain["stark_zeta"] == ch["stark_zeta"] and plain["fri_query_indices"] != ch["fri_query_indices"]
