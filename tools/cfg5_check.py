"""BASELINE.json configs[4] at full scale on ONE GPU: starky-shaped trace commitment (n = 2^24 rows, rate_bits 1,
64 columns, cap 4) + FRI commit phase / PoW / 84 query openings (arity 16 x5), accepted by the restated native
verifier (oracle) with openings computed by the GPU eval_commitment and spot-checked on the CPU.
Run on the H100:  python tools/cfg5_check.py [log_n] [cols]
"""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import oracle_lib
import plonky2_b200 as pb
from conftest import synth

log_n = int(sys.argv[1]) if len(sys.argv) > 1 else 24
B = int(sys.argv[2]) if len(sys.argv) > 2 else 64
r, h = 1, 4
ctx = pb.default_context(0)
vals = synth(0x05, (B, 1 << log_n))
t0 = time.perf_counter()
c = pb.PolynomialBatch.from_values(vals, r, False, h)
cap = c.merkle_tree.cap
t_commit = time.perf_counter() - t0
cfg = pb.starky_standard_fast_fri_config()
params = cfg.fri_params(log_n, False)
zeta = (0x1122334455667788 % pb.field.ORDER, 0x99AABBCCDDEEFF00 % pb.field.ORDER)
gz = pb.field.ext_mul(zeta, (pb.field.primitive_root_of_unity(log_n), 0))
inst = pb.FriInstanceInfo([pb.FriOracleInfo(B, False)],
                          [pb.FriBatchInfo(zeta, [pb.FriPolynomialInfo(0, i) for i in range(B)]),
                           pb.FriBatchInfo(gz, [pb.FriPolynomialInfo(0, 0), pb.FriPolynomialInfo(0, 1)])])
ch = pb.Challenger(); ch.observe_cap(cap)
och = oracle_lib.Challenger(); och.observe_cap(cap.hashes)
t0 = time.perf_counter()
ev_z = c.eval_commitment(zeta); ev_gz = c.eval_commitment(gz)
t_open = time.perf_counter() - t0
t0 = time.perf_counter()
proof = pb.prove_openings(inst, [c], ch, params)
t_fri = time.perf_counter() - t0
pbytes = proof.to_bytes()
# spot-check two openings on the CPU (Horner over 2^log_n coefficients)
co = c.polynomials
assert tuple(int(x) for x in ev_z[3]) == oracle_lib.eval_poly_base_at_ext(co[3], zeta)
assert tuple(int(x) for x in ev_gz[1]) == oracle_lib.eval_poly_base_at_ext(co[1], gz)
opened = np.concatenate([ev_z.reshape(-1), ev_gz[:2].reshape(-1)])
obatches = [(b.point, [(p.oracle_index, p.polynomial_index) for p in b.polynomials]) for b in inst.batches]
oparams = oracle_lib.make_params(r, h, 16, 84, params.reduction_arity_bits)
rc = oracle_lib.verify_fri_proof([cap.hashes], [B], [B], obatches, opened, log_n, och, oparams, pbytes)
bad = bytearray(pbytes); bad[len(bad) // 2] ^= 4
rc_bad = oracle_lib.verify_fri_proof([cap.hashes], [B], [B], obatches, opened, log_n, oracle_lib.Challenger(), oparams, bytes(bad))
print("cfg5 n=2^%d cols=%d: commit %.1f ms (host in), openings %.1f ms, prove_openings %.1f ms, proof %d bytes, arities %s"
      % (log_n, B, t_commit * 1e3, t_open * 1e3, t_fri * 1e3, len(pbytes), params.reduction_arity_bits))
print("verifier rc=%d (0 = accepted), corrupted proof rc=%d (non-zero = rejected)" % (rc, rc_bad))
assert rc == 0 and rc_bad != 0
print("CFG5 CHECK OK")
