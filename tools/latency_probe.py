"""Where does a recursion-sized proof spend its wall time? (run on the H100)"""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import plonky2_b200 as pb
from plonky2_b200 import fri as F, _native as N
from conftest import synth

log_n, r, h = 14, 3, 4
n = 1 << log_n
Bs = [84, 135, 20, 16]
data = [synth(0x40 + i, (B, n)) for i, B in enumerate(Bs)]
ctx = pb.default_context(0)
cfg = pb.standard_recursion_fri_config(); params = cfg.fri_params(log_n, False)
zeta = (123456789, 987654321); gz = pb.field.ext_mul(zeta, (pb.field.primitive_root_of_unity(log_n), 0))
allp = [pb.FriPolynomialInfo(o, i) for o, B in enumerate(Bs) for i in range(B)]
inst = pb.FriInstanceInfo([pb.FriOracleInfo(B, False) for B in Bs], [pb.FriBatchInfo(zeta, allp), pb.FriBatchInfo(gz, [pb.FriPolynomialInfo(2, 0), pb.FriPolynomialInfo(2, 1)])])
const = pb.PolynomialBatch.from_values(data[0], r, False, h)
T = {}
def tick(name, t0):
    ctx.synchronize(); T[name] = T.get(name, 0) + time.perf_counter() - t0
for it in range(6):
    if it == 1: T.clear()
    ch = pb.Challenger(); ch.observe_cap(const.merkle_tree.cap)
    t0 = time.perf_counter(); w = pb.PolynomialBatch.from_values(data[1], r, False, h); tick("commit135", t0)
    t0 = time.perf_counter(); cap = w.merkle_tree.cap; tick("cap_d2h", t0)
    t0 = time.perf_counter(); ch.observe_cap(cap); ch.get_n_challenges(4); tick("challenger", t0)
    t0 = time.perf_counter(); z = pb.PolynomialBatch.from_values(data[2], r, False, h); tick("commit20", t0)
    ch.observe_cap(z.merkle_tree.cap)
    t0 = time.perf_counter(); q = pb.PolynomialBatch.from_coeffs(data[3], r, False, h); tick("commit16c", t0)
    ch.observe_cap(q.merkle_tree.cap)
    oracles = [const, w, z, q]
    t0 = time.perf_counter(); alpha = ch.get_extension_challenge(); st = F._begin(inst, oracles, alpha, params); tick("fri_begin", t0)
    t0 = time.perf_counter(); caps, fc = F.fri_committed_trees(st, ch, params); tick("fri_commit_phase", t0)
    t0 = time.perf_counter(); pw = F.fri_proof_of_work(ch, params.config, ctx); tick("fri_pow", t0)
    t0 = time.perf_counter(); rounds, xi = F.fri_prover_query_rounds(oracles, st, ch, params.lde_size(), params); tick("fri_queries", t0)
    t0 = time.perf_counter(); b = F.FriProof(caps, rounds, fc, pw).to_bytes(); tick("serialize", t0)
    st.close(); w.close(); z.close(); q.close()
tot = sum(T.values())
for k, v in T.items(): print("%-18s %8.3f ms" % (k, v / 5 * 1e3))
print("total %.3f ms; launches/proof ~%d" % (tot / 5 * 1e3, ctx.launch_count // 6))
