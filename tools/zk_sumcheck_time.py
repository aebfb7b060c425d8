"""Device time of the zero-knowledge sumcheck of a caller-defined polynomial (ZKSumcheckInstanceProof.prove) against the plain sumcheck
(sumcheck_prove) of the same tables and composition, on these shapes:
  quad     A*B at 2^20 and 2^22 (prove_quad's composition);
  cubic    A*B*C - A*D at 2^20 and 2^22 (prove_cubic_with_additive_term's);
  degree6  a degree-6 polynomial of 6 tables and 6 terms at 2^20.
Each call is timed with CUDA events on the context's stream around the whole call (host round trips and the ZK rounds' host sigma work
included), median of --reps runs, the two provers alternating on fresh uploads of the same tables.

    python tools/zk_sumcheck_time.py [--reps 5] [--out file.json]

Prints the GPU's name and power limit first: the numbers belong to that card.  Fails without a GPU."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

Q = 2**252 + 27742317777372353535851937790883648493


def gpu_info():
    return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip().splitlines()[0]


def to_limbs(x):
    return np.frombuffer((x * 2**256 % Q).to_bytes(32, "little"), dtype=np.uint64).copy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import spartan_b200 as sb
    ctx = sb.default_context()
    print("GPU: %s" % gpu_info(), flush=True)
    rng = np.random.default_rng(0)

    def coeff():
        return to_limbs(int.from_bytes(rng.bytes(32), "little") % Q)
    one, minus_one = to_limbs(1), to_limbs(Q - 1)
    deg6 = [(coeff(), (0, 1, 2, 3, 4, 5)), (coeff(), (5, 5, 0, 1, 2)), (coeff(), (1, 2)), (one, (3,)), (coeff(), (4, 4, 4, 0)), (minus_one, (2, 3, 5))]
    cases = [("quad", lg, 2, [(one, (0, 1))]) for lg in (20, 22)]
    cases += [("cubic", lg, 4, [(one, (0, 1, 2)), (minus_one, (0, 3))]) for lg in (20, 22)]
    cases.append(("degree6", 20, 6, deg6))
    gens = {}
    rows = []
    for name, lg, k, terms in cases:
        N = 1 << lg
        host = [sb.prg_scalars("zk-time-%s-%d" % (name, j), N) for j in range(k)]
        comp = sb.Composition(terms)
        d = comp.degree
        if d not in gens:
            gens[d] = (sb.MultiCommitGens(1, b"zk-time-gens-1"), sb.MultiCommitGens(d + 1, b"zk-time-gens-n"))
        g1, gn = gens[d]
        claim, blind = to_limbs(12345), to_limbs(678)

        def timed(fn):
            polys = [sb.DensePolynomial(h) for h in host]
            sb.api.timer_start(ctx)
            fn(polys)
            return sb.api.timer_stop_ms(ctx)

        drivers = {
            "zk": lambda polys: sb.ZKSumcheckInstanceProof.prove(polys, comp, claim, blind, lg, g1, gn, sb.Transcript(b"time"),
                                                                 sb.RandomTape(sb.tape_seed(1))),
            "plain": lambda polys: sb.sumcheck_prove(polys, comp, claim, lg, sb.Transcript(b"time")),
        }
        for f in drivers.values():   # warm-up: module loads, allocator, host tables
            timed(f)
        times = {dname: [] for dname in drivers}
        for _ in range(a.reps):
            for dname, f in drivers.items():
                times[dname].append(timed(f))
        row = {"case": name, "log2_len": lg, "tables": k, "terms": len(terms), "degree": d}
        for dname, ts in times.items():
            row["%s_ms" % dname] = round(statistics.median(ts), 3)
            row["%s_ms_min" % dname] = round(min(ts), 3)
        row["zk_over_plain"] = round(row["zk_ms"] / row["plain_ms"], 3)
        print(json.dumps(row), flush=True)
        rows.append(row)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"gpu": gpu_info(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
