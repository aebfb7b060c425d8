"""Device time of the products of the caller's matrices (sp_spmat_multiply_vec / sp_spmat_eval_table) on three shapes of 2^k entries in a
2^k x 2^k matrix, b = 3 matrices of the shape per call (the R1CS prover's A, B, C):
  uniform   one entry per row and per column
  row       every entry on one row
  col       every entry in one column (the R1CS constant column)
  mv_ms     SparseMatProducts.multiply_vec: the three M z
  et_ms     SparseMatProducts.compute_eval_table_sparse with weights: the three M^T e into scratch and their weighted sum
Times are CUDA events on the context's stream around --iters calls (sp_timer_start / sp_timer_stop_ms), per call, median of --reps.  GB/s are
algorithmic bytes over that time: per entry a 4-byte key, a 4-byte source index, a 32-byte value and a 32-byte gather of z or e; 32 bytes per
output; the weighted sum reads the b tables and writes one more.  For comparison, the thread-per-row kernel of the R1CS prover (k_spmv, through
the spd_spmv hook of libsp_devtest.so and the library's per-kernel event profiler) on the CSR (for M z) and the CSC (for M^T e) of one matrix
of the same shape; the thread-per-row numbers are per matrix, multiply by three to compare.

    python tools/spmat_time.py [--log2 20 22] [--reps 5] [--iters 10] [--out file.json]

Prints the GPU's name, power limit and maximum SM clock first: the numbers belong to that card."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_GBS = 3350.0   # H100 SXM data sheet


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:
        return "unknown (%s)" % e


def entries(rng, k, shape):
    n = 1 << k
    if shape == "uniform":
        rows, cols = np.arange(n, dtype=np.uint64), rng.permutation(n).astype(np.uint64)
    elif shape == "row":
        rows, cols = np.zeros(n, dtype=np.uint64), rng.integers(0, n, n, dtype=np.uint64)
    else:
        rows, cols = rng.integers(0, n, n, dtype=np.uint64), np.zeros(n, dtype=np.uint64)
    vals = np.zeros((n, 32), dtype=np.uint8)
    vals[:, :31] = rng.integers(0, 256, (n, 31), dtype=np.uint8)   # below 2^248 < q
    return rows, cols, vals


def limbs(rng, n):
    v = rng.integers(0, 2 ** 63, (n, 4), dtype=np.uint64)
    v[:, 3] >>= 8                                                    # below 2^247 < q: reduced Montgomery limbs
    return v


def timed(api, fn, reps, iters):
    fn()
    out = []
    for _ in range(reps):
        api.timer_start()
        for _ in range(iters):
            fn()
        out.append(api.timer_stop_ms() / iters)
    return statistics.median(out)


class Spmv:
    """k_spmv on host CSR arrays through libsp_devtest.so; kernel time from the library's event profiler"""

    def __init__(self):
        self.lib = C.CDLL(os.path.join(ROOT, "spartan_b200", "libsp_devtest.so"))
        vp, sz = C.c_void_p, C.c_size_t
        self.lib.spd_spmv.argtypes = [sz, sz, vp, vp, vp, sz, vp, vp]
        self.lib.spd_prof_enable.argtypes = [C.c_int]
        self.lib.spd_prof_report.argtypes = [C.c_char_p, sz]
        self.lib.spd_prof_report.restype = sz

    def ms(self, major, minor, vals_limbs, nmajor, x, reps):
        order = np.argsort(major, kind="stable")
        idx = np.ascontiguousarray(minor[order].astype(np.uint32))
        val = np.ascontiguousarray(vals_limbs[order])
        ptr = np.zeros(nmajor + 1, dtype=np.uint32)
        ptr[1:] = np.cumsum(np.bincount(major.astype(np.int64), minlength=nmajor))
        out = np.zeros((nmajor, 4), dtype=np.uint64)
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        times = []
        for _ in range(reps):
            self.lib.spd_prof_enable(1)
            rc = self.lib.spd_spmv(nmajor, len(idx), p(ptr), p(idx), p(val), len(x), p(x), p(out))
            assert rc == 0, rc
            buf = C.create_string_buffer(1 << 16)
            self.lib.spd_prof_report(buf, len(buf))
            self.lib.spd_prof_enable(0)
            rec = [r.split(":") for r in buf.value.decode().split(";") if r.startswith("spmv:")]
            times.append(float(rec[0][2]))
        return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2", nargs="+", type=int, default=[20, 22])
    ap.add_argument("--shapes", nargs="+", default=["uniform", "row", "col"])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--spmv-reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import spartan_b200 as sb
    from spartan_b200 import api
    info = gpu_info()
    print("GPU:", info, flush=True)
    spmv = Spmv()
    rows_out = []
    b = 3
    for k in a.log2:
        n = 1 << k
        for shape in a.shapes:
            rng = np.random.default_rng(k * 10 + len(shape))
            ents = [entries(rng, k, shape) for _ in range(b)]
            P = sb.SparseMatPolynomial.multi_products([sb.SparseMatPolynomial(k, k, r, c, v) for r, c, v in ents])
            z, e = sb.DensePolynomial(limbs(rng, n)), sb.DensePolynomial(limbs(rng, n))
            w = limbs(rng, b)
            mv = timed(api, lambda: P.multiply_vec(n, n, z), a.reps, a.iters)
            et = timed(api, lambda: P.compute_eval_table_sparse(e, n, n, weights=w), a.reps, a.iters)
            bytes_mv = b * (72.0 * n + 32.0 * n)
            bytes_et = b * (72.0 * n + 32.0 * n) + 32.0 * n * (b + 1)
            row = {"log2_nnz": k, "shape": shape, "b": b, "mv_ms": round(mv, 4), "et_ms": round(et, 4),
                   "mv_GBs": round(bytes_mv / mv / 1e6, 1), "et_GBs": round(bytes_et / et / 1e6, 1),
                   "mv_roofline_share": round(bytes_mv / mv / 1e6 / HBM_GBS, 3), "et_roofline_share": round(bytes_et / et / 1e6 / HBM_GBS, 3)}
            # the thread-per-row kernel on one matrix of the shape: CSR for M z, CSC for M^T e
            r, c, v = ents[0]
            vl = limbs(rng, n)
            row["spmv_csr_ms_per_matrix"] = round(spmv.ms(r, c, vl, n, limbs(rng, n), a.spmv_reps), 4)
            row["spmv_csc_ms_per_matrix"] = round(spmv.ms(c, r, vl, n, limbs(rng, n), a.spmv_reps), 4)
            print(json.dumps(row), flush=True)
            rows_out.append(row)
            del P
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"gpu": info, "rows": rows_out}, f, indent=1)


if __name__ == "__main__":
    main()
