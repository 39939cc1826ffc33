"""distributed.prove_plonk across ranks (run under torchrun, one rank per GPU): for a circuit without lookups (the device
Z path), one with every gate type and a lookup table (the host Z path), LargeCircuit at 2^13 gates in the standard
recursion config, and a zero-knowledge circuit with explicit salt keys, every rank's proof bytes equal
prove_with_witness's on its own device, and rank 0 has the restated verifier (tests/plonk_circuits.oracle_verify, with
and without zero knowledge) accept them; a zero-knowledge proof with fresh keys is accepted too. Too many ranks for the
cap and a constants/sigmas commitment of the wrong shard -- on one rank only -- are refused on every rank. With fewer GPUs
than ranks all ranks share GPU 0 and exchange through gloo, since NCCL refuses two ranks on one device. Launched by
tests/test_plonk_sharded.py, or by hand:
  python -m torch.distributed.run --standalone --nproc-per-node 2 tests/mgpu_plonk_check.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


import plonky2_b200 as pb  # noqa: E402
from plonky2_b200 import _native as N  # noqa: E402
from plonky2_b200 import distributed as D  # noqa: E402
from plonky2_b200 import plonk  # noqa: E402
from ranks import finish_rank, init_rank  # noqa: E402

DIGEST = [11, 22, 33, 44]


def main():
    import oracle_lib
    import plonk_circuits as PC
    import plonk_large as PL
    from plonk_circuits import KEYS, LOOKUP_64, RECURSION_5, quick_fri_config, shape_circuit

    from plonky2_b200.fri import standard_recursion_fri_config

    rank, world, _, ctx = init_rank()
    failures = []

    zk_cfg = plonk.standard_recursion_zk_config()
    zk_c, _ = PC.zk_circuit(plonk, zk_cfg, quick_fri_config(zk_cfg))
    cases = [("no_lookups", shape_circuit(RECURSION_5, 4, public_inputs=[3, 1, 4, 1, 5]), None, {}),
             ("lookups", shape_circuit(LOOKUP_64, 4, public_inputs=[2, 7, 1, 8]), None, {}),
             ("large_2_13", PL.large_circuit(13, luts="range16", public_inputs=[3, 1, 4, 1, 5, 9, 2, 6]),
              standard_recursion_fri_config(), {}),
             ("zk_keys", zk_c, None, dict(salt_keys=KEYS))]
    verified = []
    for name, c, fri_cfg, kw in cases:
        cfg, cd = c.config, c.common
        fri_cfg = fri_cfg or quick_fri_config(cfg)
        zk = cfg.zero_knowledge
        fri_params = fri_cfg.fri_params(cd.degree_bits, zk)
        whole = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height, ctx=ctx)
        mine = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height, ctx=ctx,
                                              shard=(rank, world))
        try:
            want = plonk.prove_with_witness(plonk.ProverOnlyCircuitData(whole, c.sigmas, DIGEST, fri_params), cd,
                                            c.wires, c.public_inputs, ctx=ctx, **kw).to_bytes()
            sharded = plonk.ProverOnlyCircuitData(mine, c.sigmas, DIGEST, fri_params)
            got = D.prove_plonk(sharded, cd, c.wires, c.public_inputs, ctx=ctx, **kw).to_bytes()
            if got != want:
                failures.append("%s: rank %d's bytes differ from prove_with_witness's" % (name, rank))
            verified.append((name, c, fri_cfg, fri_params, got, whole.merkle_tree.cap.hashes))
            if zk:
                fresh = D.prove_plonk(sharded, cd, c.wires, c.public_inputs, ctx=ctx).to_bytes()
                verified.append(("zk_fresh", c, fri_cfg, fri_params, fresh, whole.merkle_tree.cap.hashes))
        finally:
            whole.close()
            mine.close()

    # refusals on every rank: too many ranks for the cap; a constants/sigmas commitment of the wrong shard on rank 0 only
    c = cases[0][1]
    cfg, cd = c.config, c.common
    fri_params = quick_fri_config(cfg).fri_params(cd.degree_bits, False)
    tiny = shape_circuit((12, 8, 4, 2, 4), 0)
    cs_tiny = pb.PolynomialBatch.from_values(tiny.constants_sigmas, 2, False, 0, ctx=ctx)
    wrong = pb.PolynomialBatch.from_values(c.constants_sigmas, cfg.rate_bits, False, cfg.cap_height, ctx=ctx,
                                           shard=((rank + 1) % world if rank == 0 else rank, world))
    try:
        for what, pd, c_ in (("cap_height 0", plonk.ProverOnlyCircuitData(cs_tiny, tiny.sigmas, DIGEST, fri_params),
                              tiny),
                             ("wrong shard on rank 0", plonk.ProverOnlyCircuitData(wrong, c.sigmas, DIGEST, fri_params),
                              c)):
            try:
                D.prove_plonk(pd, c_.common, c_.wires, c_.public_inputs, ctx=ctx)
                failures.append("%s: not refused on rank %d" % (what, rank))
            except N.ShapeError:
                pass
    finally:
        cs_tiny.close()
        wrong.close()

    if rank == 0:
        for name, c, fri_cfg, fri_params, data, cs_cap in verified:
            parts = PC.parts_of(plonk.ProofWithPublicInputs.from_bytes(data, c.common, fri_params), cs_cap)
            verdict = PC.oracle_verify(oracle_lib, plonk, c, DIGEST, fri_cfg, parts)
            if verdict is not None:
                failures.append("%s: the restated verifier rejects the proof: %s" % (name, verdict))
    finish_rank("MGPU_PLONK_CHECK", failures)


if __name__ == "__main__":
    main()
