"""Test infrastructure for zero-knowledge proofs, on top of tests/plonk_circuits.py:

- `zk_circuit`: a FibonacciCircuit with the blinding rows of CircuitBuilder::blind (plonk/circuit_builder.rs:911-970) --
  regular_rows NoopGate rows with random values on every wire, then z_pairs pairs of NoopGate rows with one random
  value per routed wire in both rows of the pair and a copy constraint between them -- counted by plonk.blinding_counts.
- `oracle_prove_zk` / `oracle_verify_zk`: the CPU twin and the restated verifier of plonk_circuits with hiding = true:
  the wires, Z / partial-product and quotient commitments salted with explicit salt arrays, hiding observed in the
  transcript, and the salted oracles' leaves 4 words wider in the FRI check (which strips the salt,
  fri/verifier.rs fri_combine_initial)."""
import contextlib

import numpy as np

import oracle_lib as OL
import plonk_circuits as PC

P = PC.P


def zk_circuit(plonk, config, fri_config, seed=7, arithmetic_rows=12, poseidon_rows=0, extra=(), lookups=False,
               public_inputs=(3, 1, 4, 1, 5)):
    """The circuit's gates, then the blinding rows blinding_counts asks for, padded with NoopGate rows to a power of
    two (CircuitBuilder::blind_and_pad). Returns (circuit, (regular_rows, z_pairs))."""
    num_gates = 2 + arithmetic_rows + poseidon_rows + len(extra) + (4 if lookups else 0)
    regular, z_pairs = plonk.blinding_counts(config, fri_config, num_gates)
    degree_bits = (num_gates + regular + 2 * z_pairs).bit_length()   # at least one padding row after the blinding
    c = PC.FibonacciCircuit(plonk, config, degree_bits, seed=seed, arithmetic_rows=arithmetic_rows,
                            poseidon_rows=poseidon_rows, extra=extra, lookups=lookups, public_inputs=list(public_inputs))
    # FibonacciCircuit fills the NoopGate rows after the gates with random wires, each wire alone in its copy set: the
    # regular blinding rows as they are. Each Z pair gets one value per routed wire and the 2-cycle sigma of its set.
    omega = PC.root_of_unity(degree_bits)
    k_is = c.common.k_is
    for q in range(z_pairs):
        r1 = num_gates + regular + 2 * q
        r2 = r1 + 1
        for w in range(config.num_routed_wires):
            assert int(c.sigmas[w, r1]) == k_is[w] * pow(omega, r1, P) % P   # not copied anywhere yet
            c.wires[w, r2] = c.wires[w, r1]
            c.sigmas[w, r1] = k_is[w] * pow(omega, r2, P) % P
            c.sigmas[w, r2] = k_is[w] * pow(omega, r1, P) % P
    c.constants_sigmas = np.concatenate([np.stack(c.constant_vecs), c.sigmas])
    return c, (regular, z_pairs)


def salt_widths(widths):
    """Leaf widths of the four plonky2 oracles with hiding: constants / sigmas unsalted, the others + SALT_SIZE."""
    return [w + (4 if k else 0) for k, w in enumerate(widths)]


class _SaltedOracle:
    """oracle_lib as the zero-knowledge twin uses it: the first commitment (constants / sigmas) is unsalted, the next
    ones take the given salt arrays in order (wires, Z's, quotient); verify_fri_proof reads salted leaves."""

    def __init__(self, salts):
        self._salts, self._commits = list(salts), 0

    def __getattr__(self, name):
        return getattr(OL, name)

    def Commit(self, cols, rate_bits, cap_height, salt=None, is_coeffs=False):
        k = self._commits
        self._commits += 1
        return OL.Commit(cols, rate_bits, cap_height, salt=self._salts[k - 1] if k else None, is_coeffs=is_coeffs)

    def verify_fri_proof(self, caps, num_polys, leaf_widths, *args, **kw):
        return OL.verify_fri_proof(caps, num_polys, salt_widths(leaf_widths), *args, **kw)


@contextlib.contextmanager
def _hiding():
    """plonk_circuits' transcript with FriParams.hiding = true (fri/mod.rs:145-157)."""
    plain = PC.observe_fri_params

    def observe(ch, fri_cfg, degree_bits, arity_bits):
        ch.observe_elements([fri_cfg.rate_bits, fri_cfg.cap_height, fri_cfg.proof_of_work_bits])
        ch.observe_elements([1, fri_cfg.reduction_strategy[1], fri_cfg.reduction_strategy[2]])
        ch.observe_element(fri_cfg.num_query_rounds)
        ch.observe_elements([1, degree_bits] + list(arity_bits))

    PC.observe_fri_params = observe
    try:
        yield
    finally:
        PC.observe_fri_params = plain


def oracle_prove_zk(c, circuit_digest, fri_cfg, salts):
    """plonk_circuits.oracle_prove with hiding and salts = the (4 x N) salt arrays of the wires, Z and quotient
    commitments. Returns (proof bytes, parts)."""
    with _hiding():
        return PC.oracle_prove(_SaltedOracle(salts), c, circuit_digest, fri_cfg, c.public_inputs)


def oracle_verify_zk(plonk, c, circuit_digest, fri_cfg, parts):
    """plonk_circuits.oracle_verify for a zero-knowledge proof: None or the reason of the rejection."""
    with _hiding():
        return PC.oracle_verify(_SaltedOracle(()), plonk, c, circuit_digest, fri_cfg, parts)
