"""Row-commitment MSM micro-benchmark (the 2048 x 4096 shape of commit_nondet_witness and the 1024 x 1024 witness commitment)."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import spartan_b200 as sb
from spartan_b200 import api
rng = np.random.default_rng(0)


def rand_table(n):
    t = rng.integers(0, 2**63, size=(n, 4), dtype=np.uint64)
    t[:, 3] &= np.uint64(0x0FFFFFFFFFFFFFFF)
    return t


res = {}
for (L, R) in [(1024, 1024), (2048, 4096)]:
    g = sb.MultiCommitGens(R, b"bench-msm")
    p = sb.DensePolynomial(rand_table(L * R))
    p.commit(g, L, R)
    ms = []
    for _ in range(3):
        api.prof_enable(True); p.commit(g, L, R); rep = api.prof_report(); api.prof_enable(False)
        ms.append(rep["msm_rows"]["ms"])
    res["commit_%dx%d_ms" % (L, R)] = round(min(ms), 3)
    del p, g
print(json.dumps(res), flush=True)
