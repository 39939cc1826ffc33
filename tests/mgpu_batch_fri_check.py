"""distributed.batch_prove_openings_sharded across ranks (run under torchrun, one rank per GPU): each rank commits its
row-block shard of a BatchFriOracle, the ranks all-gather the cap (Placement.cap), and for the reference test's shape
(k = 9, 8, 6, rate 1, cap 5) and one with several polynomials per degree, two opening points and grinding, every rank's
proof bytes equal batch_prove_openings' on its own device and the oracle's; rank 0 has the restated batch verifier
(oracle.verify_batch_fri_proof) accept the proof, and reject it with one opened value flipped and with one word of an
initial-tree leaf flipped. A world size above 2^cap_height is refused on every rank. With fewer GPUs than ranks all ranks
share GPU 0 and exchange through gloo, since NCCL refuses two ranks on one device. Launched by
tests/test_batch_fri_sharded.py, or by hand:
  python -m torch.distributed.run --standalone --nproc-per-node 2 tests/mgpu_batch_fri_check.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import plonky2_b200 as pb  # noqa: E402
from plonky2_b200 import _native as N  # noqa: E402
from plonky2_b200 import distributed as D  # noqa: E402
from plonky2_b200.fri import FriProof  # noqa: E402
from ranks import finish_rank, init_rank  # noqa: E402

# (degree bits per group, polynomials per group, rate bits, cap height, arities, queries, PoW bits, two points)
CASES = {
    "reference": ([9, 8, 6], [1, 1, 1], 1, 5, [1, 2, 1], 10, 0, False),
    "groups_two_points_pow": ([11, 8, 6], [5, 3, 2], 2, 3, [3, 2, 2], 6, 7, True),
}


def _polys(lens, counts):
    from conftest import synth

    return [synth(0x3C0 + 16 * k + j, (1 << k,)) for k, c in zip(lens, counts) for j in range(c)]


def _instances(lens, counts, zeta, two_points):
    """The device instances, the oracle's, and the opened values in the verifier's order."""
    insts, oinsts, points = [], [], []
    start = 0
    for k, c in zip(lens, counts):
        batches = [pb.FriBatchInfo(zeta, [pb.FriPolynomialInfo(0, start + j) for j in range(c)])]
        if two_points:
            gz = pb.field.ext_mul(zeta, (pb.field.primitive_root_of_unity(k), 0))
            batches.append(pb.FriBatchInfo(gz, [pb.FriPolynomialInfo(0, start)]))
        insts.append(pb.FriInstanceInfo([pb.FriOracleInfo(sum(counts), False)], batches))
        oinsts.append([(b.point, [(p.oracle_index, p.polynomial_index) for p in b.polynomials]) for b in batches])
        points += [(b.point, [p.polynomial_index for p in b.polynomials]) for b in batches]
        start += c
    return insts, oinsts, points


def main():
    import oracle_lib

    rank, world, _, ctx = init_rank()
    placement = D.Placement(rank, world, None)
    failures, verified = [], []

    for name, (lens, counts, r, cap_height, arities, nq, pow_bits, two_points) in CASES.items():
        polys = _polys(lens, counts)
        params = pb.FriParams(pb.FriConfig(r, cap_height, pow_bits, ("Fixed", arities), nq), False, lens[0], arities)
        whole = pb.BatchFriOracle.from_values(polys, r, False, cap_height, ctx=ctx)
        mine = pb.BatchFriOracle.from_values(polys, r, False, cap_height, ctx=ctx, shard=(rank, world))
        try:
            cap = placement.cap(mine)
            if not np.array_equal(cap.hashes, whole.cap.hashes):
                failures.append("%s: rank %d's gathered cap differs from the single-device cap" % (name, rank))
            proofs = []
            for oracle_, prove in ((whole, pb.batch_prove_openings), (mine, D.batch_prove_openings_sharded)):
                ch = pb.Challenger()
                ch.observe_cap(cap)
                zeta = ch.get_extension_challenge()
                insts, oinsts, points = _instances(lens, counts, zeta, two_points)
                proofs.append(prove(list(lens), insts, [oracle_], ch, params))
            got, want = proofs[1].to_bytes(), proofs[0].to_bytes()
            if got != want:
                failures.append("%s: rank %d's bytes differ from the single-device proof's" % (name, rank))
            oo = oracle_lib.BatchCommit(polys, r, cap_height)
            och = oracle_lib.Challenger()
            och.observe_cap(oo.cap)
            och.get_extension_challenge()
            vch = och.clone()
            oparams = oracle_lib.make_params(r, cap_height, pow_bits, nq, arities)
            if oracle_lib.batch_prove_openings([oo], list(lens), oinsts, och, oparams) != got:
                failures.append("%s: rank %d's bytes differ from the oracle's" % (name, rank))
            coeffs = [oracle_lib.ifft(p) for p in polys]
            opened = np.array([oracle_lib.eval_poly_base_at_ext(coeffs[i], pt) for pt, idx in points for i in idx],
                              dtype=np.uint64)
            verified.append((name, oo, counts, lens, oinsts, opened, vch, oparams, proofs[1]))
        finally:
            whole.close()
            mine.close()

    # refusal on every rank: more ranks than cap entries
    try:
        pb.BatchFriOracle.from_values(_polys([9, 8, 6], [1, 1, 1]), 1, False, 0, ctx=ctx, shard=(rank, world))
        failures.append("cap_height 0: not refused on rank %d" % rank)
    except N.ShapeError:
        pass

    if rank == 0:
        for name, oo, counts, lens, oinsts, opened, vch, oparams, proof in verified:
            data = proof.to_bytes()
            if oracle_lib.verify_batch_fri_proof([oo.cap], [counts], lens, oinsts, opened, vch.clone(), oparams, data):
                failures.append("%s: the restated verifier rejects the proof" % name)
            bad = opened.copy()
            bad[0, 0] ^= np.uint64(1)
            if not oracle_lib.verify_batch_fri_proof([oo.cap], [counts], lens, oinsts, bad, vch.clone(), oparams, data):
                failures.append("%s: the verifier accepts a flipped opened value" % name)
            leaf, sib = proof.query_round_proofs[0].initial_trees_proof.evals_proofs[0]
            flipped = leaf.copy()
            flipped[0] ^= np.uint64(1)
            proof.query_round_proofs[0].initial_trees_proof.evals_proofs[0] = (flipped, sib)
            tampered = FriProof.to_bytes(proof)
            if not oracle_lib.verify_batch_fri_proof([oo.cap], [counts], lens, oinsts, opened, vch.clone(), oparams,
                                                     tampered):
                failures.append("%s: the verifier accepts a flipped initial-tree leaf" % name)
    finish_rank("MGPU_BATCH_FRI_CHECK", failures)


if __name__ == "__main__":
    main()
