"""The suite's own helpers, on the CPU: the multi-rank launchers of tests/ranks.py leave no rank running when a test
fails or hangs, and the proof comparisons of tests/stark_twin.py (proof_diff, assert_matches_twin) catch every change
they must."""
import copy
import os
import time

import numpy as np
import pytest

from conftest import synth
from ranks import run_ranks, spawn_ranks

SLEEPER = """import os, sys, time
open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "pids", str(os.getpid())), "w").close()
time.sleep(60)
"""


def _sleeper(rank, world, directory):
    open(os.path.join(directory, str(os.getpid())), "w").close()
    time.sleep(60)


def _alive(pid):
    try:
        os.kill(pid, 0)
    except ProcessLookupError:
        return False
    return True


def test_hung_ranks_are_reaped(tmp_path):
    """run_ranks and spawn_ranks on ranks that record their pid and sleep for 60 s, past a 20 s timeout: each helper
    fails, and afterwards none of the ranks exists. The sleep is bounded so that the ranks end on their own even if a
    helper does not reap them."""
    (tmp_path / "torchrun" / "pids").mkdir(parents=True)
    (tmp_path / "spawned").mkdir()
    script = tmp_path / "torchrun" / "sleeper.py"
    script.write_text(SLEEPER)
    with pytest.raises(pytest.fail.Exception, match="timed out"):
        run_ranks(str(script), "never printed", timeout=20)
    with pytest.raises(AssertionError, match="did not return within"):
        spawn_ranks(_sleeper, 2, (str(tmp_path / "spawned"),), timeout=20)
    for name in ("torchrun/pids", "spawned"):
        pids = [int(p) for p in os.listdir(tmp_path / name)]
        assert len(pids) >= 2, name
        assert not [pid for pid in pids if _alive(pid)], name


def _stark_proof(seed):
    """A StarkProofWithPublicInputs with CTLs, from plain arrays: no device."""
    from plonky2_b200.fri import FriInitialTreeProof, FriProof, FriQueryRound, FriQueryStep
    from plonky2_b200.hash import MerkleCap
    from plonky2_b200.proof import StarkOpeningSet
    from plonky2_b200.stark import StarkProof, StarkProofWithPublicInputs

    def w(k, shape):
        return synth(16 * seed + k, shape)

    openings = StarkOpeningSet(w(0, (3, 2)), w(1, (3, 2)), w(2, (2, 2)), w(3, (2, 2)), w(4, (2, 2)), w(5, (2,)))
    query = FriQueryRound(FriInitialTreeProof([(w(6, (3,)), w(7, (2, 4))), (w(8, (2,)), w(9, (2, 4)))]),
                          [FriQueryStep(w(10, (2, 2)), w(11, (1, 4)))])
    fri = FriProof([MerkleCap(w(12, (2, 4)))], [query], w(13, (1, 2)), 1000 + seed)
    proof = StarkProof(MerkleCap(w(14, (2, 4))), MerkleCap(w(15, (2, 4))), openings, fri, MerkleCap(w(16, (2, 4))))
    return StarkProofWithPublicInputs(proof, [seed, 2, 3])


def _twin_of(proof):
    """The dict twin_prove would return for `proof`."""
    p, o = proof.proof, proof.proof.openings
    return dict(public_inputs=list(proof.public_inputs), trace_cap=p.trace_cap.hashes.copy(),
                aux_cap=p.auxiliary_polys_cap.hashes.copy(), quotient_cap=p.quotient_polys_cap.hashes.copy(),
                **{k: getattr(o, k).copy() for k in ("local_values", "next_values", "auxiliary_polys",
                                                     "auxiliary_polys_next", "quotient_polys", "ctl_zs_first")},
                fri_bytes=p.opening_proof.to_bytes())


FRI = ".proof.opening_proof"
CHANGES = {   # what is changed, and where proof_diff must report it
    "public input": [".public_inputs[1]"],
    "cap": [".proof.auxiliary_polys_cap.hashes"],
    "opening": [".proof.openings.next_values"],
    "ctl_zs_first": [".proof.openings.ctl_zs_first"],
    "FRI query": [FRI + ".query_round_proofs[0].initial_trees_proof.evals_proofs[1][0]", FRI + ".to_bytes()"],
    "pow witness": [FRI + ".pow_witness", FRI + ".to_bytes()"],
    "opening batch dropped": [".proof.openings.ctl_zs_first"],
}


def _changed(proof, what):
    bad = copy.deepcopy(proof)
    p = bad.proof
    if what == "public input":
        bad.public_inputs[1] += 1
    elif what == "cap":
        p.auxiliary_polys_cap.hashes[1, 3] ^= np.uint64(1)
    elif what == "opening":
        p.openings.next_values[2, 1] ^= np.uint64(1)
    elif what == "ctl_zs_first":
        p.openings.ctl_zs_first[1] ^= np.uint64(1)
    elif what == "FRI query":
        p.opening_proof.query_round_proofs[0].initial_trees_proof.evals_proofs[1][0][0] ^= np.uint64(1)
    elif what == "pow witness":
        p.opening_proof.pow_witness ^= 1
    else:   # the CTL batch of to_fri_openings
        p.openings.ctl_zs_first = None
    return bad


def test_proof_comparisons_catch_every_change():
    """proof_diff names one flipped word in a public input, a cap, an opening, ctl_zs_first, a FRI query and the pow
    witness, a dropped opening batch and a dropped table, in a StarkProofWithPublicInputs and in table 1 of a two-table
    MultiStarkProof; assert_matches_twin fails for each against the twin dicts of the unchanged proofs, which pass."""
    import stark_twin as T
    from plonky2_b200.cross_table_lookup import MultiStarkProof

    one, two = _stark_proof(1), _stark_proof(2)
    multi = MultiStarkProof([one, two])
    twin = {"tables": [_twin_of(one), _twin_of(two)]}
    assert T.proof_diff(multi, copy.deepcopy(multi)) == []
    T.assert_matches_twin(two, twin["tables"][1])
    T.assert_matches_twin(multi, twin)
    for what, paths in CHANGES.items():
        bad = _changed(two, what)
        assert T.proof_diff(two, bad) == paths, what
        assert T.proof_diff(multi, MultiStarkProof([one, bad])) == [".stark_proofs[1]" + p for p in paths], what
        with pytest.raises(AssertionError):
            T.assert_matches_twin(bad, twin["tables"][1])
        with pytest.raises(AssertionError):
            T.assert_matches_twin(MultiStarkProof([one, bad]), twin)
    dropped = MultiStarkProof([one])
    assert T.proof_diff(multi, dropped) == [".stark_proofs: 2 entries against 1"]
    with pytest.raises(AssertionError, match="number of tables"):
        T.assert_matches_twin(dropped, twin)
