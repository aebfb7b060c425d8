"""Device time of whole sumchecks of caller-defined polynomials (sumcheck_prove: one fused launch per round, challenges drawn on the host as
soon as a round's evaluations land) on these shapes:
  cubic       A*B*C at 2^20 and 2^22, against the same proof driven round by round through the kind-1 operator entries
              (sp_sumcheck_eval / sp_sumcheck_fold_eval: evaluations copied out, transcript on the host, one C call per round);
  product     the product-layer shape sum_i c_i A_i B_i C with one shared C at 2^20, with as many instances as SP_SC_MAX_TABLES allows
              (3: 7 tables; the 12 instances of a SNARK's product layers would need 25 tables);
  degree5     a degree-5 polynomial of 6 tables and 8 terms at 2^22.
Each sumcheck is timed with CUDA events on the context's stream around the whole call (host round trips included), median of --reps runs,
the two cubic drivers alternating.  A separate profiled run gives the fused streaming rounds' rate (k_scp_fold_eval) against the algorithmic
48 bytes per table entry per round.

    python tools/sumcheck_poly_time.py [--reps 5] [--out file.json]

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

Q = 2**252 + 27742317777372353535851937790883648493
R_INV = pow(2**256, -1, Q)


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:   # the numbers are still printed; say that the card could not be named
        return "unknown (%s)" % e


def to_int(limbs):
    return int.from_bytes(np.ascontiguousarray(limbs, dtype=np.uint64).tobytes(), "little") * R_INV % Q


def to_limbs(x):
    return np.frombuffer((x * 2**256 % Q).to_bytes(32, "little"), dtype=np.uint64).copy()


def cubic_from_evals(e0, e1, e2, e3):
    """UniPoly::from_evals (unipoly.rs:23-54) for four points"""
    six_inv, two_inv = pow(6, -1, Q), pow(2, -1, Q)
    a = six_inv * (e3 - 3 * e2 + 3 * e1 - e0) % Q
    b = two_inv * (2 * e0 - 5 * e1 + 4 * e2 - e3) % Q
    c = (e1 - e0 - a - b) % Q
    return [e0 % Q, c, b, a]


def round_by_round(sb, polys, claim, n, T):
    """the A*B*C proof through sp_sumcheck_eval / sp_sumcheck_fold_eval, the host keeping the transcript (prove_cubic, sumcheck.rs:183-252)"""
    import ctypes as C
    e, r = claim, None
    ev = sb.api.sumcheck_eval(1, polys)
    for j in range(n):
        e0, e2, e3 = (to_int(x) for x in ev)
        coeffs = cubic_from_evals(e0, (e - e0) % Q, e2, e3)
        T.append_message(b"poly", b"UniPoly_begin")
        for c in coeffs:
            T.append_message(b"coeff", c.to_bytes(32, "little"))
        T.append_message(b"poly", b"UniPoly_end")
        out = np.zeros(4, dtype=np.uint64)
        sb.lib.sp_scalar_from_bytes_wide(C.c_char_p(T.challenge_bytes(b"challenge_nextround", 64)), out.ctypes.data_as(C.c_void_p))
        r = to_int(out)
        if j + 1 < n:
            ev = sb.api.sumcheck_fold_eval(1, polys, out)
        else:
            sb.api.fold_top(polys, out)
        e = sum(c * pow(r, i, Q) for i, c in enumerate(coeffs)) % Q
    return e


def timed(sb, ctx, fn):
    sb.api.timer_start(ctx)
    out = fn()
    return sb.api.timer_stop_ms(ctx), out


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
    one = to_limbs(1)
    cases = []
    for lg in (20, 22):
        cases.append(("cubic", lg, 3, [(one, (0, 1, 2))]))
    cases.append(("product", 20, 7, [(coeff(), (i, 3 + i, 6)) for i in range(3)]))
    deg5 = [(coeff(), (0, 1, 2, 3, 4)), (coeff(), (5, 5, 0, 1, 2)), (coeff(), (1, 2)), (coeff(), (3,)), (coeff(), (4, 5, 0)),
            (coeff(), (2, 2, 2, 2)), (coeff(), (0, 5)), (one, (1, 3, 5, 1, 3))]
    cases.append(("degree5", 22, 6, deg5))
    rows = []
    for name, lg, k, terms in cases:
        N = 1 << lg
        host = [sb.prg_scalars("scpoly-time-%s-%d" % (name, j), N) for j in range(k)]
        comp = sb.Composition(terms)
        claim = to_limbs(12345)

        def generic():
            polys = [sb.DensePolynomial(h) for h in host]
            t = sb.Transcript(b"time")
            return timed(sb, ctx, lambda: sb.sumcheck_prove(polys, comp, claim, lg, t))

        def operator():
            polys = [sb.DensePolynomial(h) for h in host]
            t = sb.Transcript(b"time")
            return timed(sb, ctx, lambda: round_by_round(sb, polys, 12345, lg, t))
        drivers = {"generic": generic}
        if name == "cubic":
            drivers["operator_kind1"] = operator
        for f in drivers.values():   # warm-up: module loads, allocator, attributes
            f()
        if name == "cubic":   # the two drivers prove the same bytes: same final claim
            assert to_int(generic()[1][3]) == operator()[1]
        times = {d: [] for d in drivers}
        for _ in range(a.reps):
            for d, f in drivers.items():
                times[d].append(f()[0])
        # profiled run of the generic driver: time and algorithmic bytes per kernel family
        polys = [sb.DensePolynomial(h) for h in host]
        ctx_t = sb.Transcript(b"time")
        sb.api.prof_enable(True)
        sb.sumcheck_prove(polys, comp, claim, lg, ctx_t)
        prof = sb.api.prof_report()
        sb.api.prof_enable(False)
        row = {"case": name, "log2_len": lg, "tables": k, "terms": len(terms), "degree": comp.degree}
        for d, ts in times.items():
            row["%s_ms" % d] = round(statistics.median(ts), 3)
            row["%s_ms_min" % d] = round(min(ts), 3)
        st = prof.get("scp_fold_eval")
        if st:
            row["streaming_rounds"] = st["launches"]
            row["streaming_ms"] = round(st["ms"], 3)
            row["streaming_GBps"] = round(st["bytes"] / st["ms"] / 1e6, 1)
            row["largest_round_GBps"] = round(st["largest_bytes"] / st["largest_ms"] / 1e6, 1)
        for fam in ("scp_eval", "scp_fold_eval_small", "fold_top", "heads"):
            if fam in prof:
                row["%s_ms" % fam] = round(prof[fam]["ms"], 3)
        print(json.dumps(row), flush=True)
        rows.append(row)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"gpu": gpu_info(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
