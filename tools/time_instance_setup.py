"""Time the setup of a caller's R1CS instance at the synthetic shape (2^n constraints, 2^n variables, 10 inputs, 2^n entries per matrix):

  new        Instance.new from prepared (row, col, 32-byte value) triples: Python packing plus sp_instance_create
  create     sp_instance_create alone, from prepared numpy arrays (the C++ part of Instance.new)
  tensors    Instance.from_tensors from prepared CUDA tensors ("not measured" by a build without it)
  encode     SNARK::encode of the instance (SNARKGens excluded)

Each figure is wall-clock time around the call followed by a device synchronise, the median (and minimum) of --reps runs.  The GPU's name and
power limit are read in the same run and printed with the numbers.  Usage: python tools/time_instance_setup.py [--logn 20 22] [--reps 5]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import spartan_b200 as sb  # noqa: E402
from spartan_b200 import api  # noqa: E402

Q = 2**252 + 27742317777372353535851937790883648493
R_INV = pow((1 << 256) % Q, -1, Q)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(sb.default_context().device)],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as e:   # the numbers are still printed; the line says what could not be read
        return "unknown (%s)" % e, "unknown"


def canonical(val):
    """(n, 4) Montgomery limbs -> (n, 32) uint8 canonical little-endian"""
    b = np.ascontiguousarray(val).tobytes()
    out = b"".join((int.from_bytes(b[i:i + 32], "little") * R_INV % Q).to_bytes(32, "little") for i in range(0, len(b), 32))
    return np.frombuffer(out, dtype=np.uint8).reshape(-1, 32).copy()


def prepare(logn):
    n = 1 << logn
    inst, _, _ = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=0)
    mats = []
    for m in range(3):
        row, col, val = inst.export(m)
        mats.append((row, col, canonical(val)))
    return n, mats


def timed(f, reps):
    import torch
    ts, out = [], None
    for _ in range(reps):
        out = None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = f()
        torch.cuda.synchronize()
        ts.append(1e3 * (time.perf_counter() - t0))
    return out, {"median_ms": round(float(np.median(ts)), 2), "min_ms": round(min(ts), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logn", type=int, nargs="+", default=[20, 22])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--label", default="")
    a = ap.parse_args()
    import torch
    ctx = sb.default_context()
    dev = "cuda:%d" % ctx.device
    name, power = gpu_info()
    for logn in a.logn:
        n, mats = prepare(logn)
        res = {"label": a.label, "logn": logn, "gpu": name, "power_limit": power}
        triples = []
        for row, col, val in mats:
            vb = val.tobytes()
            triples.append(list(zip(row.tolist(), col.tolist(), [vb[i:i + 32] for i in range(0, len(vb), 32)])))
        _, res["new"] = timed(lambda: sb.Instance.new(n, n, 10, *triples, ctx=ctx), a.reps)
        del triples

        def create():
            h = C.c_void_p()
            args = []
            for row, col, val in mats:
                args += [api._p(row), api._p(col), api._p(val), C.c_size_t(len(row))]
            ctx.check(api.lib.sp_instance_create(ctx.h, C.c_size_t(n), C.c_size_t(n), C.c_size_t(10), *args, C.byref(h)))
            return api.Instance(ctx, h)
        inst, res["create"] = timed(create, a.reps)
        if hasattr(sb.Instance, "from_tensors"):
            tens = [tuple(torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (row.view(np.int64), col.view(np.int64), val)) for row, col, val in mats]
            inst, res["tensors"] = timed(lambda: sb.Instance.from_tensors(n, n, 10, *tens, ctx=ctx), a.reps)
            del tens
        else:
            res["tensors"] = "not measured (no Instance.from_tensors in this build)"
        gens = sb.SNARKGens(n, n, 10, n, ctx=ctx)
        _, res["encode"] = timed(lambda: sb.SNARK.encode(inst, gens), a.reps)
        print(json.dumps(res), flush=True)
        del inst, gens
        sb.release_cached_memory()


if __name__ == "__main__":
    main()
