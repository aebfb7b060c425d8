"""Kernel micro-benchmarks (BASELINE.json configs[2]/[3] shaped): dense sumcheck rounds on 2^LOGN tables (per-round GB/s vs the HBM roofline),
row commitments (MSM terms/s), and the full SNARK::prove.  CUDA-event times from the library's profiler.  Usage: bench_kernels.py [logn] [--snark]"""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import spartan_b200 as sb
from spartan_b200 import api

logn = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 22
try:
    peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    peak = 3350.0   # H100 SXM data sheet (bench.py's fallback)
ctx = sb.default_context()
n = 1 << logn
rng = np.random.default_rng(0)


def rand_table(n):
    t = rng.integers(0, 2**63, size=(n, 4), dtype=np.uint64)
    t[:, 3] &= np.uint64(0x0FFFFFFFFFFFFFFF)  # < q: valid Montgomery residues
    return t


res = {"logn": logn}
for kind, nt, name in [(2, 4, "cubic4"), (0, 2, "quad"), (1, 3, "cubic3")]:
    polys = [sb.DensePolynomial(rand_table(n)) for _ in range(nt)]
    r = sb.prg_scalars("r", 1)[0]
    api.sumcheck_eval(kind, polys)
    api.prof_enable(True)
    e = api.sumcheck_eval(kind, polys)
    rep = api.prof_report(); api.prof_enable(False)
    ev = rep["sc_eval"]
    rounds = []
    for j in range(6):
        api.prof_enable(True)
        api.sumcheck_fold_eval(kind, polys, r)
        rep = api.prof_report(); api.prof_enable(False)
        v = rep["sc_fold_eval"]
        rounds.append((v["bytes"] / 1e9 / (v["ms"] / 1e3), v["ms"] * 1e3))
    res[name] = {"eval_GBs": ev["bytes"] / 1e9 / (ev["ms"] / 1e3), "fold_eval_GBs_by_round": [round(a) for a, _ in rounds], "fold_eval_us_by_round": [round(b, 1) for _, b in rounds],
                 "frac_of_hbm_round0": rounds[0][0] / peak}
    del polys
for (L, R) in [(1024, 1024), (2048, 4096)]:
    g = sb.MultiCommitGens(R, b"bench-msm")
    p = sb.DensePolynomial(rand_table(L * R))
    p.commit(g, L, R)
    api.prof_enable(True)
    p.commit(g, L, R)
    rep = api.prof_report(); api.prof_enable(False)
    ms = rep["msm_rows"]["ms"]
    res["commit_%dx%d" % (L, R)] = {"ms": round(ms, 3), "Mterms_per_s": round(L * R / ms / 1e3, 1), "M_table_adds_per_s": round(L * R * 32 / ms / 1e3, 1)}
    del p, g
if "--snark" in sys.argv:
    m = 1 << 20
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(m, m, 10, seed=0)
    gens = sb.SNARKGens(m, m, 10, m)
    comm = sb.SNARK.encode(inst, gens)
    dv = sb.DensePolynomial(vars_.limbs)
    for _ in range(2):
        sb.SNARK.prove(inst, comm, dv, inputs, gens, b"example", sb.tape_seed(0))
    ts = []
    for _ in range(3):
        api.timer_start(); sb.SNARK.prove(inst, comm, dv, inputs, gens, b"example", sb.tape_seed(0)); ts.append(api.timer_stop_ms())
    res["snark_2p20_ms"] = round(min(ts), 2)
    api.prof_enable(True); sb.SNARK.prove(inst, comm, dv, inputs, gens, b"example", sb.tape_seed(0)); rep = api.prof_report(); api.prof_enable(False)
    res["snark_kernel_ms"] = {k: round(v["ms"], 2) for k, v in sorted(rep.items(), key=lambda kv: -kv[1]["ms"])[:6]}
print(json.dumps(res), flush=True)
