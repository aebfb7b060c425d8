"""Device time of SPARK on the caller's matrices (sp_spark_*): for b matrices of nz random entries each, 2^x rows and 2^y columns,
  commit_ms     SparseMatPolynomial.multi_commit: host entries to the device, ingestion, timestamps and the comb_ops / comb_mem commitments
  prove_ms      SparseMatPolyEvalProof.prove at a random (rx, ry) on a fresh transcript, the evaluations computed on the device
Times are CUDA events on the context's stream around each call (sp_timer_start / sp_timer_stop_ms); each call ends with its results on the
host.  Median of --reps runs after one warm-up run of each shape.  The generators are built once per shape, outside the timed calls.

    python tools/spark_time.py [--shapes 20:20:20:3 20:20:20:4] [--reps 3] [--out file.json]      (shape = log2 nz : x : y : b)

Prints the GPU's name and power limit first: the numbers belong to that card."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:   # the numbers are still printed; say that the card could not be named
        return "unknown (%s)" % e


def matrices(sb, rng, lgnz, x, y, b):
    n = 1 << lgnz
    out = []
    for _ in range(b):
        vals = np.zeros((n, 32), dtype=np.uint8)
        vals[:, :31] = rng.integers(0, 256, (n, 31), dtype=np.uint8)   # below 2^248 < q
        out.append(sb.SparseMatPolynomial(x, y, rng.integers(0, 1 << x, n, dtype=np.uint64), rng.integers(0, 1 << y, n, dtype=np.uint64), vals))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=["20:20:20:3", "20:20:20:4"], help="log2 nz:x:y:b")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import spartan_b200 as sb
    from spartan_b200 import api
    info = gpu_info()
    print("GPU:", info, flush=True)
    rows = []
    for shape in a.shapes:
        lgnz, x, y, b = (int(v) for v in shape.split(":"))
        rng = np.random.default_rng(lgnz * 1000 + b)
        polys = matrices(sb, rng, lgnz, x, y, b)
        gens = sb.SparseMatPolyCommitmentGens(b"spark-time", x, y, 1 << lgnz, b)
        rx, ry = sb.prg_scalars("spark-time-rx", x), sb.prg_scalars("spark-time-ry", y)
        commit_ms, prove_ms = [], []
        for rep in range(a.reps + 1):
            api.timer_start()
            comm, dense = sb.SparseMatPolynomial.multi_commit(polys, gens)
            t_commit = api.timer_stop_ms()
            api.timer_start()
            proof, ev = sb.SparseMatPolyEvalProof.prove(dense, rx, ry, None, gens, b"spark-time", sb.RandomTape(sb.tape_seed(rep)))
            t_prove = api.timer_stop_ms()
            if rep:   # rep 0 warms the shape up
                commit_ms.append(t_commit); prove_ms.append(t_prove)
            del dense
        proof.verify(comm, rx, ry, ev, gens, b"spark-time")
        row = {"log2_nz": lgnz, "x": x, "y": y, "b": b, "commit_ms": round(statistics.median(commit_ms), 2),
               "prove_ms": round(statistics.median(prove_ms), 2), "proof_bytes": len(proof.data)}
        print(json.dumps(row), flush=True)
        rows.append(row)
        del gens
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"gpu": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
