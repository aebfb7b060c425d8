"""Private SNARKGens against views into one GeneratorTables(2^20, 2^20, 10, 2^20): creation time and the library's live device bytes at 2^16, 2^18
and 2^20, then device-timed SNARK.prove at 2^16 and 2^18 on each kind.

Private gens for 2^18 built while 2^20 tables are alive get narrower windows (GenSet::finish sizes each table against the HBM free at the time), so
the proof timing runs the two kinds in alternating blocks, each on an otherwise empty device: build the gens (private, or the tables and their views),
prove `--proofs` times per size after one warm-up proof, free.  Every proof is checked against the first one of its size.

    python tools/gen_tables_time.py [--blocks 2] [--proofs 5] [--out file.json]

Prints the GPU's name and power limit first: the numbers belong to that card."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SIZES, PROVE_SIZES = (16, 18, 20), (16, 18)


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:   # the numbers are still printed; say that the card could not be named
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=2, help="blocks of each kind in the proof timing (private, views, private, views, ...)")
    ap.add_argument("--proofs", type=int, default=5, help="timed proofs per size per block")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import spartan_b200 as sb
    from spartan_b200 import api
    ctx = sb.default_context()
    card = gpu_info()
    print("GPU: %s" % card, flush=True)
    n20 = 1 << 20
    rows = []

    def emit(row):
        row["gpu"] = card
        rows.append(row)
        print(json.dumps(row), flush=True)

    def timed(fn):
        t0 = time.perf_counter()
        out = fn()
        return out, (time.perf_counter() - t0) * 1e3   # the constructors return once their tables are built (they synchronise)

    # ---- creation time and live device bytes
    for lg in SIZES:
        n = 1 << lg
        sb.release_cached_memory()   # cached blocks count as used memory to the window-width choice
        live0 = sb.device_bytes_live()
        g, ms = timed(lambda: sb.SNARKGens(n, n, 10, n))
        emit(dict(what="private SNARKGens", log2_n=lg, create_ms=round(ms, 1), device_bytes=sb.device_bytes_live() - live0))
        del g
    sb.release_cached_memory()
    live0 = sb.device_bytes_live()
    tables, ms = timed(lambda: sb.GeneratorTables(n20, n20, 10, n20))
    emit(dict(what="GeneratorTables", log2_n=20, create_ms=round(ms, 1), device_bytes=sb.device_bytes_live() - live0, sets=tables.info()))
    views = []
    for lg in SIZES:
        n = 1 << lg
        live1 = sb.device_bytes_live()
        v, ms = timed(lambda: sb.SNARKGens(n, n, 10, n, tables=tables))
        views.append(v)
        emit(dict(what="SNARKGens view", log2_n=lg, create_ms=round(ms, 1), device_bytes=sb.device_bytes_live() - live1))
    emit(dict(what="tables + views for 2^16, 2^18, 2^20", device_bytes=sb.device_bytes_live() - live0))
    del views, tables

    # ---- proof time, alternating blocks
    stmts = {lg: sb.Instance.produce_synthetic_r1cs(1 << lg, 1 << lg, 10, seed=0) for lg in PROVE_SIZES}
    want, times = {}, {(k, lg): [] for k in ("private", "view") for lg in PROVE_SIZES}
    for block in range(2 * a.blocks):
        kind = "private" if block % 2 == 0 else "view"
        sb.release_cached_memory()
        tables = sb.GeneratorTables(n20, n20, 10, n20) if kind == "view" else None
        for lg in PROVE_SIZES:
            n = 1 << lg
            inst, vars_, inputs = stmts[lg]
            if tables is None:
                sb.release_cached_memory()
            gens = sb.SNARKGens(n, n, 10, n, tables=tables)
            comm = sb.SNARK.encode(inst, gens)
            dvars = sb.DensePolynomial(vars_.limbs)
            for j in range(a.proofs + 1):
                api.timer_start(ctx)
                proof = sb.SNARK.prove(inst, comm, dvars, inputs, gens, b"example", sb.tape_seed(0))
                ms = api.timer_stop_ms(ctx)
                assert want.setdefault(lg, proof.bytes) == proof.bytes, "proof bytes differ between blocks"
                if j:
                    times[(kind, lg)].append(ms)
            del gens, comm, dvars
        del tables
    for lg in PROVE_SIZES:
        p, v = times[("private", lg)], times[("view", lg)]
        emit(dict(what="SNARK.prove device ms", log2_n=lg, private_median=round(statistics.median(p), 3), view_median=round(statistics.median(v), 3),
                  private_runs=[round(x, 3) for x in p], view_runs=[round(x, 3) for x in v]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
