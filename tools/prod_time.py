"""Device time of the caller's product circuits (sp_prod_*): for k circuits of 2^m fingerprinted leaves (the memory check's
ts*r^2 + val*r + addr - gamma over three tables),
  build_ms      ProductCircuits: the leaves and the first product layer (k_prod_leaves), the other layers (hadamard_many) and the k products
  prove_ms      ProductCircuitEvalProofBatched.prove of the circuits on a fresh transcript
  leaves_ms     the k_prod_leaves kernel alone, from the per-kernel CUDA-event profile of a separate build
With --dotp KD > 0, each build also writes KD dot products (val, the read fingerprint, weight 1) beside the circuits and each proof proves them
(prove_dotp), and the profiled build reports
  dotp_ms       the k_dotp_operands kernel alone, and dotp_gbs its bytes over that time: 32 B per entry of each distinct source table read and
                96 B per entry of each dot product's operands written
Times are CUDA events on the context's stream around each call (sp_timer_start / sp_timer_stop_ms); each call ends with its results on the
host.  Median of --reps runs after one warm-up run of each shape.

    python tools/prod_time.py [--shapes 20:1 20:8 20:24 22:8] [--dotp KD] [--reps 5] [--out file.json]

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


def random_table(rng, n):
    """n field elements as Montgomery limbs (below 2^251 < q)"""
    a = rng.integers(0, 2 ** 63, size=(n, 4), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=(n, 4), dtype=np.uint64)
    a[:, 3] &= np.uint64((1 << 59) - 1)
    return a


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=["20:1", "20:8", "20:24", "22:8"], help="m:k")
    ap.add_argument("--dotp", type=int, default=0, help="dot products beside the circuits (0: circuits alone)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import spartan_b200 as sb
    info = gpu_info()
    print("GPU:", info, flush=True)
    rows = []
    for shape in a.shapes:
        m, k = (int(x) for x in shape.split(":"))
        rng = np.random.default_rng(m * 100 + k)
        polys = [sb.DensePolynomial(random_table(rng, 1 << m)) for _ in range(3)]   # addr, val, ts
        r, r2, g = random_table(rng, 3)   # r, r^2 and -gamma stand-ins: the times do not depend on the values
        kinds = [([(1, r)], 1), ([(2, r2), (1, r), (0, 1)], 0), ([(2, r2), (1, r), (0, 1)], 0), ([(2, r2), (1, r)], 1)]
        leaves = [sb.ProductLeaves(kinds[c % 4][0], index_coeff=kinds[c % 4][1], const=g) for c in range(k)]
        dotps = [(sb.ProductLeaves([(1, 1)]), sb.ProductLeaves(kinds[1][0], const=g), sb.ProductLeaves([], const=1))] * a.dotp or None

        def build():
            sb.api.timer_start()
            pc = sb.ProductCircuits(polys, leaves, dotps)
            return pc, sb.api.timer_stop_ms()

        def prove(pc):
            t = sb.Transcript(b"prod_time")
            sb.api.timer_start()
            (sb.ProductCircuitEvalProofBatched.prove_dotp if a.dotp else sb.ProductCircuitEvalProofBatched.prove)(pc, t)
            return sb.api.timer_stop_ms()

        prove(build()[0])   # warm-up
        bt, pt = [], []
        for _ in range(a.reps):
            pc, ms = build()
            bt.append(ms)
            pt.append(prove(pc))
            del pc
        sb.api.prof_enable(True)
        pc, _ = build()
        rep = sb.api.prof_report()
        sb.api.prof_enable(False)
        del pc
        row = {"m": m, "k": k, "leaves": k << m, "build_ms": statistics.median(bt), "prove_ms": statistics.median(pt),
               "leaves_ms": rep.get("prod_leaves", {}).get("ms"), "hadamard_ms": rep.get("hadamard", {}).get("ms"), "gpu": info}
        if a.dotp:
            d = rep["dotp_operands"]
            row.update(kd=a.dotp, dotp_ms=d["ms"], dotp_gbs=d["bytes"] / (d["ms"] * 1e6))
        rows.append(row)
        print(json.dumps(row), flush=True)
        del polys
        sb.release_cached_memory()
    if a.out:
        json.dump({"gpu": info, "rows": rows}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
