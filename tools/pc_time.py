"""Wall time of the polynomial-commitment entries on the caller's tables (sp_pc_*): for tables of 2^m entries and k tables,
  commit       poly_commit of the k tables' merge, with a random tape (blinds)
  prove        PolyEvalProof.prove (k = 1) or prove_joint (k > 1) at a random point, on the commitment's blinds
  verify       PolyEvalProof.verify_plain (k = 1) or verify_joint
  host_merge   k > 1 only: what a caller without prove_joint does instead: evaluate the k tables (DensePolynomial.evaluate), download them,
               concatenate and zero-pad on the host, upload the merge and run PolyEvalProof.prove on it (Zr computed on the device)
Every call returns its result to the host, so a host clock around it measures the whole call.  Median of --reps runs after one warm-up run
of each.  The gens are built once per m, for the largest k, and the smaller merges use views of them (same bytes, same tables).

    python tools/pc_time.py [--m 16 20 24] [--k 1 4 8] [--reps 5] [--out file.json]

Prints the GPU's name and power limit first: the numbers belong to that card."""
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
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:   # the numbers are still printed; say that the card could not be named
        return "unknown (%s)" % e


def random_table(rng, n):
    """n field elements as Montgomery limbs (below 2^251 < q)"""
    a = rng.integers(0, 2 ** 63, size=(n, 4), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=(n, 4), dtype=np.uint64)
    a[:, 3] &= np.uint64((1 << 59) - 1)
    return a


def median_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(1e3 * (time.perf_counter() - t0))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, nargs="+", default=[16, 20, 24])
    ap.add_argument("--k", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import spartan_b200 as sb
    print("GPU:", gpu_info(), flush=True)
    rows = []
    for m in a.m:
        rng = np.random.default_rng(m)
        kmax = max(a.k)
        tabs = [random_table(rng, 1 << m) for _ in range(kmax)]
        polys = [sb.DensePolynomial(t) for t in tabs]
        r = random_table(rng, m)
        big = sb.PolyCommitmentGens(m + (kmax - 1).bit_length(), b"pc_time")
        for k in a.k:
            c = (k - 1).bit_length()
            g = big.view(m + c)
            ps = polys[:k]
            tape = sb.RandomTape()
            comm, blinds = sb.poly_commit(ps if k > 1 else ps[0], g, tape)
            row = {"m": m, "k": k, "entries": (1 << m) * k}
            row["commit_ms"] = median_ms(lambda: sb.poly_commit(ps if k > 1 else ps[0], g, sb.RandomTape()), a.reps)
            if k == 1:
                proof, _, Zr = sb.PolyEvalProof.prove(ps[0], blinds, r, None, None, g, sb.Transcript(b"t"), tape)
                row["prove_ms"] = median_ms(lambda: sb.PolyEvalProof.prove(ps[0], blinds, r, None, None, g, sb.Transcript(b"t"), sb.RandomTape()), a.reps)
                row["verify_ms"] = median_ms(lambda: proof.verify_plain(g, sb.Transcript(b"t"), r, Zr, comm), a.reps)
            else:
                proof, evals = sb.PolyEvalProof.prove_joint(ps, blinds, r, g, sb.Transcript(b"t"), tape)
                row["prove_ms"] = median_ms(lambda: sb.PolyEvalProof.prove_joint(ps, blinds, r, g, sb.Transcript(b"t"), sb.RandomTape()), a.reps)
                row["verify_ms"] = median_ms(lambda: proof.verify_joint(g, sb.Transcript(b"t"), r, evals, comm), a.reps)
                r_joint = np.vstack([random_table(rng, c), r])

                def host_merge():
                    for p in ps:
                        p.evaluate(r)
                    z = np.concatenate([p.to_numpy() for p in ps] + [np.zeros(((2 ** c - k) << m, 4), dtype=np.uint64)])
                    sb.PolyEvalProof.prove(sb.DensePolynomial(z), blinds, r_joint, None, None, g, sb.Transcript(b"t"), sb.RandomTape())
                row["host_merge_ms"] = median_ms(host_merge, a.reps)
            rows.append(row)
            print(json.dumps(row), flush=True)
        del polys, big, g
        sb.release_cached_memory()
    if a.out:
        json.dump({"gpu": gpu_info(), "rows": rows}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
