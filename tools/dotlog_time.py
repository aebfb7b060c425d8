"""Time DotProductProofLog.prove / verify of the caller's vectors (sp_dotlog_*) at n = 2^8 (table path), 2^9 (folding path), 2^12, 2^16, 2^20 and
2^24, x and a resident on the device.  Each call is timed with CUDA events on the context's stream around the whole call (it ends in a device
synchronise), median of --reps runs after one warm-up call of each.  The prove is split into its own lines, from the host sub-phase timers
(SP_FINE_TIMERS) of the timed runs and the per-kernel CUDA events (sp_prof) of one more run:
  Cx          the commitment <x, G> + blind_x h (folding path: one bucket MSM of n terms)
  absorb a    the transcript absorbing the n scalars of a (host, serial, linear in n; the verifier does the same work)
  rounds      the log2 n rounds, absorb a excluded (host wall clock: launches, waits and the host's group work)
  fold        the generator-fold kernel (dotlog_fold), summed over the rounds
  msm         the round MSMs and Cx's (msm_var and msm_var_segmented)
The table path has no fold kernel and runs its MSMs in the inner-product kernel (ipa_msm): its fold and msm lines stay 0.

    python tools/dotlog_time.py [--logn 8 9 12 16 20 24] [--reps 5] [--out file.json]

Prints the GPU's name and power limit first: the numbers belong to that card.  Fails without a GPU."""
import argparse
import json
import os
import statistics
import subprocess
import sys

os.environ.setdefault("SP_FINE_TIMERS", "1")
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip().splitlines()[0]


def limbs(rng, n):
    """n residues < 2^252 as Montgomery limbs (every such value is an element)"""
    t = rng.integers(0, 2 ** 63, size=(n, 4), dtype=np.uint64)
    t[:, 3] &= np.uint64(0x0FFFFFFFFFFFFFFF)
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logn", type=int, nargs="+", default=[8, 9, 12, 16, 20, 24])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import spartan_b200 as sb
    ctx = sb.default_context()
    print("GPU: %s" % gpu_info(), flush=True)
    rng = np.random.default_rng(0)
    one, two = limbs(rng, 2)
    rows = []
    for logn in args.logn:
        n = 1 << logn
        reps = args.reps if logn <= 20 else 1
        gens = sb.DotProductProofGens(n, b"dotlog-time")
        X, A = sb.DensePolynomial(limbs(rng, n)), sb.DensePolynomial(limbs(rng, n))

        def prove():
            T = sb.Transcript(b"dotlog-time")
            sb.api.timer_start(ctx)
            p, Cx, Cy = sb.DotProductProofLog.prove(gens, T, sb.RandomTape(sb.tape_seed(0)), X, one, A, None, two)
            return sb.api.timer_stop_ms(ctx), ctx.timings(), (p, Cx, Cy)

        def verify(p, Cx, Cy):
            T = sb.Transcript(b"dotlog-time")
            sb.api.timer_start(ctx)
            p.verify(n, gens, T, A, Cx, Cy)
            return sb.api.timer_stop_ms(ctx), ctx.timings()

        _, _, out = prove()
        verify(*out)
        pt, vt, fine = [], [], []
        for _ in range(reps):
            ms, tm, out = prove()
            pt.append(ms)
            fine.append(tm)
            vt.append(verify(*out)[0])
        sb.api.prof_enable(True)
        prove()
        prof = sb.api.prof_report()
        sb.api.prof_enable(False)
        med = lambda key: statistics.median(f.get(key, 0.0) for f in fine)
        row = {"logn": logn, "path": "table" if n <= 256 else "folding", "prove_ms": statistics.median(pt), "verify_ms": statistics.median(vt),
               "reps": reps, "Cx_ms": med("fine:dotlog Cx"), "absorb_a_ms": med("fine:dotlog absorb a"),
               "rounds_ms": med("fine:dotlog rounds") - med("fine:dotlog absorb a"),
               "fold_kernel_ms": prof.get("dotlog_fold", {}).get("ms", 0.0),
               "msm_kernel_ms": sum(prof.get(k, {}).get("ms", 0.0) for k in ("msm_var", "msm_var_segmented")),
               "proof_bytes": len(out[0].data)}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del gens, X, A
        sb.release_cached_memory()
    if args.out:
        json.dump({"gpu": gpu_info(), "rows": rows}, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
