"""distributed.build_circuit_data across ranks (run under torchrun, one rank per GPU): on every rank the digest and the
verifier's cap equal the single-device plonk.build_circuit_data's, the constants/sigmas commitment is the rank's row
block, and prove_plonk on that data gives the bytes of prove_with_witness on the single-device data -- for a circuit
with a lookup table and every gate type, and for a zero-knowledge circuit with explicit salt keys. With fewer GPUs than
ranks all ranks share GPU 0 and exchange through gloo. Launched by tests/test_circuit_data.py, or by hand:
  python -m torch.distributed.run --standalone --nproc-per-node 2 tests/mgpu_circuit_data_check.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


from plonky2_b200 import distributed as D  # noqa: E402
from plonky2_b200 import plonk  # noqa: E402
from ranks import finish_rank, init_rank  # noqa: E402


def main():
    import numpy as np

    from plonk_circuits import (KEYS, LOOKUP_64, instances_of, pairs_from_sigmas, quick_fri_config, shape_circuit,
                                zk_circuit)

    rank, world, _, ctx = init_rank()
    failures = []

    zk_cfg = plonk.standard_recursion_zk_config()
    zk_c, _ = zk_circuit(plonk, zk_cfg, quick_fri_config(zk_cfg))
    zk_rows, _, zk_pairs = plonk.blind_and_pad(zk_cfg, quick_fri_config(zk_cfg), instances_of(zk_c)[:14])
    lookup = shape_circuit(LOOKUP_64, 4, public_inputs=[2, 7, 1, 8])
    cases = [("lookups", lookup, instances_of(lookup), pairs_from_sigmas(lookup), {}),
             ("zk_keys", zk_c, zk_rows, pairs_from_sigmas(zk_c, [r for p in zk_pairs for r in p]),
              dict(salt_keys=KEYS))]
    for name, c, rows, pairs, kw in cases:
        cd = c.common
        args = (c.config, quick_fri_config(c.config), rows, pairs, 0, cd.luts, c.lookup_rows, [9])
        whole = plonk.build_circuit_data(*args, ctx=ctx)
        mine = D.build_circuit_data(*args, ctx=ctx)
        try:
            cs = mine.prover_only.constants_sigmas_commitment
            if (cs.shard_index, cs.num_shards) != (rank, world):
                failures.append("%s: rank %d holds shard %d of %d" % (name, rank, cs.shard_index, cs.num_shards))
            if mine.verifier_only.circuit_digest != whole.verifier_only.circuit_digest:
                failures.append("%s: rank %d's digest differs" % (name, rank))
            if not np.array_equal(mine.verifier_only.constants_sigmas_cap.hashes,
                                  whole.verifier_only.constants_sigmas_cap.hashes):
                failures.append("%s: rank %d's cap differs" % (name, rank))
            want = plonk.prove_with_witness(whole.prover_only, whole.common, c.wires, c.public_inputs, ctx=ctx,
                                            **kw).to_bytes()
            got = D.prove_plonk(mine.prover_only, mine.common, c.wires, c.public_inputs, ctx=ctx, **kw).to_bytes()
            if got != want:
                failures.append("%s: rank %d's proof bytes differ from the single-device build's" % (name, rank))
        finally:
            whole.prover_only.constants_sigmas_commitment.close()
            mine.prover_only.constants_sigmas_commitment.close()

    finish_rank("MGPU_CIRCUIT_DATA_CHECK", failures)


if __name__ == "__main__":
    main()
