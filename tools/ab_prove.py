"""Timing of SNARK::prove at 2^logn under the current environment (the library reads SP_MSM_WINDOW and SP_FINE_TIMERS from it, so every
variant is its own process): median and best of `reps` device-timed proofs, the phase timers of the last one and the sha256 of the proof bytes
(which no window width may change).  usage: ab_prove.py LABEL [logn=20] [reps=7]"""
import hashlib, json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import spartan_b200 as sb
from spartan_b200 import api
label = sys.argv[1] if len(sys.argv) > 1 else "default"
logn = int(sys.argv[2]) if len(sys.argv) > 2 else 20
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 7
n = 1 << logn
inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=0)
gens = sb.SNARKGens(n, n, 10, n)
comm = sb.SNARK.encode(inst, gens)
dv = sb.DensePolynomial(vars_.limbs)
for _ in range(3):
    p = sb.SNARK.prove(inst, comm, dv, inputs, gens, b"example", sb.tape_seed(0))
ms = []
for _ in range(reps):
    api.timer_start()
    p = sb.SNARK.prove(inst, comm, dv, inputs, gens, b"example", sb.tape_seed(0))
    ms.append(api.timer_stop_ms())
ms.sort()
out = {"label": label, "logn": logn, "median_ms": round(ms[len(ms) // 2], 3), "best_ms": round(ms[0], 3), "sha256": hashlib.sha256(p.bytes).hexdigest()[:16],
       "bytes": len(p.bytes), "phases": {k: round(v, 2) for k, v in inst.ctx.timings().items()},
       "env": {k: v for k, v in os.environ.items() if k.startswith("SP_")}}
print(json.dumps(out), flush=True)
