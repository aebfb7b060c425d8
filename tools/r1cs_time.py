"""Wall time of the caller's R1CSProof (sp_r1cs_prove_t / sp_r1cs_verify_t) from both sources of the matrices, on two shapes of 2^k constraints
and 2^k variables, one entry per row in each of A, B and C:
  uniform   A = B = the identity, C = diag(vars): (A z)_i (B z)_i = z_i^2 = (C z)_i
  col       A holds every entry in column 0 (the heavy constant column of real circuits), B = the identity, C = z_0 times the identity
  instance  the matrices as an Instance: its products are k_spmv, one thread per row (phase one) or column (phase two), as in NIZK::prove
  spmat     the matrices as a SparseMatProducts: the tiled products of sp_spmat_multiply_vec / sp_spmat_eval_table
Both are satisfied by any vars (pseudo-random below 2^62).  The instance source is skipped on the heavy column above
--instance-col-max (k_spmv gives one thread the whole column in phase two: seconds at 2^20).  Prove and verify are timed around one call each
(the verify with the evals Instance.evaluate gives), median of --reps, after one warm-up call per shape and source.

    python tools/r1cs_time.py [--log2 16 18 20] [--reps 3] [--instance-col-max 18] [--out file.json]

Prints the GPU's name, power limit and maximum SM clock first: the numbers belong to that card."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:
        return "unknown (%s)" % e


def instance(sb, k, shape, small):
    """small: the n vars as integers < 2^62"""
    import torch
    n = 1 << k
    dev = torch.device("cuda", sb.default_context().device)
    i = torch.arange(n, dtype=torch.int64, device=dev)
    one = torch.zeros((n, 32), dtype=torch.uint8, device=dev)
    one[:, 0] = 1
    canon = np.zeros((n, 32), dtype=np.uint8)
    canon[:, :8] = small.astype("<u8").view(np.uint8).reshape(n, 8)
    c_vals = torch.from_numpy(canon).to(dev)
    if shape == "col":
        a_col, c_vals = torch.zeros_like(i), c_vals[:1].expand(n, 32).contiguous()
    else:
        a_col = i
    mats = ((i, a_col, one), (i, i.clone(), one), (i, i.clone(), c_vals))
    return sb.Instance.from_tensors(n, n, 0, *mats)


def spmat(sb, inst):
    from oracle.spartan_ref import core as oc
    x, y = inst.num_cons.bit_length() - 1, (2 * inst.num_vars).bit_length() - 1
    polys = []
    for m in range(3):
        row, col, val = inst.export(m)
        polys.append(sb.SparseMatPolynomial(x, y, row, col, oc.to_ints(val)))
    return sb.SparseMatPolynomial.multi_products(polys)


def timed(f):
    t0 = time.perf_counter()
    out = f()
    return out, 1e3 * (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2", type=int, nargs="+", default=[16, 18, 20])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--instance-col-max", type=int, default=18)
    ap.add_argument("--out")
    a = ap.parse_args()
    import spartan_b200 as sb
    from oracle.spartan_ref import core as oc
    print("gpu:", gpu_info())
    rows = []
    for k in a.log2:
        n = 1 << k
        gens = sb.R1CSGens(b"r1cs-time", n, n)
        small = np.random.default_rng(k).integers(0, 1 << 62, size=n, dtype=np.uint64)
        v = sb.DensePolynomial(oc.to_arr([int(x) for x in small]))
        inputs = oc.zeros(0)
        for shape in ("uniform", "col"):
            inst = instance(sb, k, shape, small)
            sources = [("spmat", spmat(sb, inst))]
            if shape == "uniform" or k <= a.instance_col_max:
                sources.append(("instance", inst))
            for name, mats in sources:
                prove_ms, verify_ms = [], []
                for rep in range(a.reps + 1):
                    (proof, rx, ry), tp = timed(lambda: sb.R1CSProof.prove(mats, v, inputs, gens, sb.Transcript(b"t"), sb.RandomTape(sb.tape_seed(rep))))
                    evals = inst.evaluate(rx, ry)
                    _, tv = timed(lambda: proof.verify(n, n, inputs, evals, sb.Transcript(b"t"), gens))
                    if rep:
                        prove_ms.append(tp)
                        verify_ms.append(tv)
                row = {"log2": k, "shape": shape, "source": name, "prove_ms": statistics.median(prove_ms), "verify_ms": statistics.median(verify_ms),
                       "proof_bytes": len(proof.data)}
                print(json.dumps(row), flush=True)
                rows.append(row)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"gpu": gpu_info(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
