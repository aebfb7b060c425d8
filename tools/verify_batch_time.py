"""Per-proof verification time: k single SNARK.verify / NIZK.verify calls against one verify_batch of the same k proofs, in alternating runs in one
process, at 2^16 and 2^20 (synthetic instances) for k = 1, 8 and 32; then where the time goes (SP_FINE_TIMERS=1, csrc/verifier.cpp FineTimers):
for the batch, decompression, replay with the deferred checker, the device final pass and the re-runs of rejected proofs; for a single verify,
the group checks, the inner-product MSM, the C_LZ MSM and instance_evaluate.

    python tools/verify_batch_time.py [--sizes 16,20] [--ks 1,8,32] [--reps 5] [--out file.json]

Prints the GPU's name and power limit first: the numbers belong to that card."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

os.environ["SP_FINE_TIMERS"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:   # the numbers are still printed; say that the card could not be named
        return "unknown (%s)" % e


def fine(ctx):
    return {k[5:]: round(v, 3) for k, v in ctx.timings().items() if k.startswith("fine:")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,20")
    ap.add_argument("--ks", default="1,8,32")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import spartan_b200 as sb
    ctx = sb.default_context()
    print("GPU: %s" % gpu_info(), flush=True)
    rows = []
    for lg in [int(x) for x in a.sizes.split(",")]:
        n = 1 << lg
        inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=0)
        kmax = max(int(x) for x in a.ks.split(","))
        sg = sb.SNARKGens(n, n, 10, n)
        comm = sb.SNARK.encode(inst, sg)
        ng = sb.NIZKGens(n, n, 10)
        kinds = {
            "snark": (sb.SNARK, comm, sg, [sb.SNARK.prove(inst, comm, vars_, inputs, sg, b"t", sb.tape_seed(j)) for j in range(kmax)]),
            "nizk": (sb.NIZK, inst, ng, [sb.NIZK.prove(inst, vars_, inputs, ng, b"t", sb.tape_seed(j)) for j in range(kmax)]),
        }
        for kind, (P, stmt, gens, proofs) in kinds.items():
            proofs[0].verify(stmt, inputs, b"t", gens)          # warm-up of both paths
            assert all(r is None for r in P.verify_batch(proofs[:2], stmt, [inputs] * len(proofs[:2]), b"t", gens))
            for k in [int(x) for x in a.ks.split(",")]:
                ps = proofs[:k]
                single, batch, split_b, split_s = [], [], [], []
                for _ in range(a.reps):
                    t0 = time.perf_counter()
                    for p in ps:
                        p.verify(stmt, inputs, b"t", gens)
                    single.append((time.perf_counter() - t0) * 1e3 / k)
                    split_s.append(fine(ctx))                   # the last single call's phases
                    t0 = time.perf_counter()
                    res = P.verify_batch(ps, stmt, [inputs] * k, b"t", gens)
                    batch.append((time.perf_counter() - t0) * 1e3 / k)
                    split_b.append(fine(ctx))
                    assert all(r is None for r in res)
                row = dict(gpu=gpu_info(), kind=kind, log2_n=lg, k=k, reps=a.reps,
                           single_ms_per_proof=round(statistics.median(single), 3), batch_ms_per_proof=round(statistics.median(batch), 3),
                           single_runs=[round(x, 3) for x in single], batch_runs=[round(x, 3) for x in batch],
                           batch_split_ms=split_b[len(split_b) // 2], single_split_ms=split_s[len(split_s) // 2])
                rows.append(row)
                print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
