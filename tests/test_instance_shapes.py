"""Seeded satisfiable R1CS instances of the shapes real circuits have, and a mirror of the prover's shape-dependent decisions.

produce_synthetic_r1cs makes one entry per row in each of A, B and C, so every proof built from it has nnz = num_cons in all three matrices and,
above 1024 constraints, num_vars = num_cons: the SPARK ops size N is num_cons, the memory size is 2N, no matrix is padded and rx is one entry
shorter than ry.  shape_instance(spec, seed) makes instances with several entries per row, empty rows, one heavy row, a heavy column, duplicate
(row, col) entries, explicit 0 / 1 / q-1 values, entries on input columns and nnz chosen per matrix, so that N, the memory size and the two
sumcheck phases vary independently.  The instance comes in two forms: COO triples for spartan_b200.Instance.new and the oracle's r1cs.Instance.

Satisfiable by construction: every non-empty row of C holds one pivot entry on the constant column (z = 1) whose value is
(Az)_i (Bz)_i - (rest of C z)_i; rows without a pivot hold no entry in any matrix.  Az, Bz and the rest of Cz come from the oracle's C multiply_vec.

plan() restates the size rules of snark.cpp (snark_encode, plan_jG for layer 0 of the ops and memory product-layer batches, the early / split
commitment of the dereferenced values), prover.cpp (the witness commitment, the two R1CS sumcheck phases) and kernels.cu / kernels_sc.cu
(msm_rows_use_row_table, SC_SMALL_MAX).  CASES lists the instances tests/test_gpu_instance_shapes.py proves on the GPU together with the branches
each must reach; test_mirror_places_every_case fails when a threshold changes and a case drops off its branch.  Those tests run without a GPU."""
import zlib
from dataclasses import dataclass

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import r1cs, spark

Q = oc.Q
G_MIN = 16384          # snark.cpp batched_prove: 2 * Ctx::SHARD_MIN_LOCAL entries per table for an eq-factored round
SC_SMALL_MAX = 1024    # kernels_sc.cu: a round on len entries uses the small-table kernel when len / 4 <= SC_SMALL_MAX


@dataclass(frozen=True)
class Spec:
    name: str
    num_cons: int
    num_vars: int
    num_inputs: int
    nnz: tuple                 # entries of A, B, C; C's count includes one pivot per active row
    active_rows: int = 0       # rows holding entries (0: all); the others are empty in all three matrices
    heavy: tuple = None        # (matrix, entries): that many of the matrix's entries on one row
    heavy_col: float = 0.0     # fraction of every matrix's entries on one variable column
    col_pool: int = 0          # entries draw their columns from this many columns (0: all), plus the constant and some input columns
    dup: float = 0.0           # fraction of every matrix's entries that repeat another entry's (row, col)
    via_new: bool = False      # oracle instance through r1cs.Instance.new (padding of num_cons / num_vars, remap of the input columns)


@dataclass
class ShapeInstance:
    spec: Spec
    triples: list              # [A, B, C]: lists of (row, col, 32 canonical bytes) in the caller's column space
    oracle: r1cs.Instance
    vars: np.ndarray           # num_vars Montgomery scalars
    inputs: list               # canonical ints

    def input_bytes(self):
        return [v.to_bytes(32, "little") for v in self.inputs]


def shape_instance(spec, seed=0):
    rng = np.random.default_rng([seed, zlib.crc32(spec.name.encode())])
    nc, nv, ni = spec.num_cons, spec.num_vars, spec.num_inputs
    ncols = nv + 1 + ni
    const = nv
    active = np.sort(rng.choice(nc, size=spec.active_rows or nc, replace=False)).astype(np.uint64)
    inputs_cols = nv + 1 + np.arange(min(ni, 8))
    pool = np.arange(ncols) if not spec.col_pool else np.unique(np.concatenate([rng.choice(ncols, spec.col_pool, replace=False), [const], inputs_cols]))
    hcol = int(pool[0]) if pool[0] < nv else 0
    vars_ = oc.prg_scalars("shape-vars-" + spec.name, nv, seed)
    vars_[: min(nv, 3)] = oc.to_arr([0, 1, Q - 1])[: min(nv, 3)]
    inputs = oc.prg_scalars("shape-inputs-" + spec.name, ni, seed)
    z = np.concatenate([vars_, oc.to_arr([1]), inputs])
    special = oc.to_arr([0, 1, Q - 1])
    mats = []
    for m in range(3):
        n = spec.nnz[m] - (len(active) if m == 2 else 0)
        assert n >= 0, "C needs one pivot per active row"
        rows = rng.choice(active, size=n)
        cols = pool[rng.integers(0, len(pool), size=n)].astype(np.uint64)
        nd = int(spec.dup * n)
        if nd:
            src, dst = rng.integers(0, n, nd), rng.integers(0, n, nd)
            rows[dst], cols[dst] = rows[src], cols[src]
        if spec.heavy and spec.heavy[0] == m:
            rows[: spec.heavy[1]] = active[0]
        nh = int(spec.heavy_col * n)
        if nh:
            cols[rng.choice(n, nh, replace=False)] = hcol
        k = min(len(inputs_cols), n)
        cols[:k] = inputs_cols[:k]
        vals = oc.prg_scalars("shape-%s-%d" % (spec.name, m), n, seed)
        idx = rng.choice(n, min(n, 3 * max(1, n // 64)), replace=False)
        vals[idx] = special[np.arange(len(idx)) % 3]
        mats.append([rows, cols, vals])
    Az, Bz, Crest = (r1cs.SparseMat(0, 0, r, c, v).multiply_vec(nc, ncols, z) for r, c, v in mats)
    piv = oc.lincomb3(oc.hadamard(Az, Bz), Crest, oc.zeros(nc), 1, Q - 1, 0)[active.astype(np.int64)]
    r, c, v = mats[2]
    perm = rng.permutation(len(r) + len(active))
    mats[2] = [np.concatenate([r, active])[perm], np.concatenate([c, np.full(len(active), const, dtype=np.uint64)])[perm], np.concatenate([v, piv])[perm]]
    triples = []
    for r, c, v in mats:
        triples.append([(int(a), int(b), x.to_bytes(32, "little")) for a, b, x in zip(r, c, oc.to_ints(v))])
    if spec.via_new:
        oi = r1cs.Instance.new(nc, nv, ni, *triples)
    else:
        assert oc.next_pow2(nc) == nc >= 2 and oc.next_pow2(nv) == nv and ni < nv, "a direct oracle instance needs the padded dimensions"
        nx, ny = oc.log_2(nc), oc.log_2(2 * nv)
        oi = r1cs.Instance(r1cs.R1CSShape(nc, nv, ni, *(r1cs.SparseMat(nx, ny, r, c, v) for r, c, v in mats)))
    return ShapeInstance(spec, triples, oi, vars_, oc.to_ints(inputs))


# ---------------------------------------------------------------------------------------------------------------- mirror of the size rules
def log2c(x):
    return max(0, (x - 1).bit_length())


def uses_row_table(L, R):                      # kernels.cu msm_rows_use_row_table
    return L >= 64 and R >= 512


def commit_shape(n):                           # DensePolynomial::commit: L x R with L = 2^(ell/2), R = 2^(ell - ell/2)
    ell = log2c(n)
    return 1 << (ell // 2), 1 << (ell - ell // 2)


def plan_jG(n):
    """eq-factored rounds of layer 0 of a batch of product circuits over n entries on one GPU (snark.cpp plan_jG, no zero challenge)"""
    half = n // 2
    rounds, jG = log2c(half), 0
    if rounds >= 2:
        while jG + 1 < rounds and (half >> jG) >= G_MIN:
            jG += 1
    return jG


def gens_widths(num_cons, num_vars, num_inputs, nz):
    """row widths (n_ops, n_mem, n_derefs) of SNARKGens' SPARK commitment generators (snark.cpp SnarkGens, sparse_mlpoly.rs:292-317)"""
    nvp = oc.next_pow2(max(num_vars, num_inputs + 1))
    lgnz = log2c(oc.next_pow2(nz))
    v_ops, v_mem, v_der = lgnz + 4, max(log2c(num_cons), log2c(2 * nvp)) + 1, lgnz + 3
    return tuple(1 << (v - v // 2) for v in (v_ops, v_mem, v_der))


def plan(num_cons, num_vars, num_inputs, nnz, overlap=True):
    """what the prover does for an instance made by Instance::new(num_cons, num_vars, num_inputs, ...) with nnz entries per matrix"""
    ncp = 2 if num_cons in (0, 1) else oc.next_pow2(num_cons)
    nvp = oc.next_pow2(max(num_vars, num_inputs + 1))
    nnzp = [n + max(0, ncp - n) if num_cons in (0, 1) else n for n in nnz]
    N = max(oc.next_pow2(n) for n in nnzp)
    x, y = log2c(ncp), log2c(2 * nvp)
    cells = 1 << max(x, y)
    Ld, Rd = commit_shape(8 * N)
    early = overlap and N % Rd == 0
    derefs = (3 * N // Rd, Rd) if early else (Ld, Rd)
    return dict(num_cons=ncp, num_vars=nvp, N=N, cells=cells, ops_layers=log2c(N), pad=tuple(N - n for n in nnzp),
                ops_jG=plan_jG(N), mem_jG=plan_jG(cells),
                witness=commit_shape(nvp), comb_ops=commit_shape(16 * N), comb_mem=commit_shape(2 * cells), early=early, derefs=derefs,
                witness_rt=uses_row_table(*commit_shape(nvp)), comb_ops_rt=uses_row_table(*commit_shape(16 * N)), derefs_rt=uses_row_table(*derefs),
                phase1_streams=ncp // 4 > SC_SMALL_MAX, phase2_streams=2 * nvp // 4 > SC_SMALL_MAX,
                rx=x, ry=y, pad_rx=max(0, y - x), pad_ry=max(0, x - y))


def spec_plan(spec, overlap=True):
    return plan(spec.num_cons, spec.num_vars, spec.num_inputs, spec.nnz, overlap)


# ---------------------------------------------------------------------------------------------------------------- the cases
# Each GPU case with the branches it must reach.  The scaled-down families (same construction, oracle-sized) are proved by the oracle here.
CASES = {
    "dense_rows": (Spec("dense_rows", 1 << 10, 1 << 10, 10, ((1 << 16) + 5, 1 << 10, 3 << 10), heavy=(0, 4096), heavy_col=0.05, dup=0.02),
                   dict(N=1 << 17, cells=1 << 11, ops_jG=3, mem_jG=0, comb_ops=(1024, 2048), comb_ops_rt=True, early=True, derefs=(384, 1024),
                        derefs_rt=True, pad=(2 ** 17 - 2 ** 16 - 5, 2 ** 17 - 2 ** 10, 2 ** 17 - 3 * 2 ** 10), phase1_streams=False,
                        phase2_streams=False)),
    "tall_sparse": (Spec("tall_sparse", 1 << 18, 1 << 8, 5, ((1 << 12) - 3,) * 3, active_rows=2048),
                    dict(N=1 << 12, cells=1 << 18, ops_jG=0, mem_jG=4, phase1_streams=True, phase2_streams=False, pad_ry=9, pad_rx=0, early=True)),
    "wide": (Spec("wide", 1 << 9, 1 << 17, 100, (1 << 17, 1 << 9, 1 << 9), col_pool=4096),
             dict(N=1 << 17, cells=1 << 18, ops_jG=3, mem_jG=4, witness=(256, 512), witness_rt=True, phase1_streams=False, phase2_streams=True,
                  pad_rx=9, pad_ry=0)),
    "dups": (Spec("dups", 1 << 14, 1 << 14, 10, (1 << 15, (1 << 14) + 7, 1 << 14), active_rows=12288, dup=1 / 8),
             dict(N=1 << 15, cells=1 << 15, ops_jG=1, mem_jG=1, derefs=(192, 512), derefs_rt=True, phase1_streams=True, phase2_streams=True)),
    "padding": (Spec("padding", 3000, 5000, 37, (7001, 3000, 4500), active_rows=2600, via_new=True),
                dict(num_cons=4096, num_vars=8192, N=8192, cells=16384, phase1_streams=False, phase2_streams=True)),
    "many_inputs": (Spec("many_inputs", 16, 3, 40, (40, 24, 30), via_new=True),
                    dict(num_vars=64, N=64, cells=128)),
}

SCALED = [
    Spec("dense_rows_s", 64, 64, 5, ((1 << 10) + 5, 64, 192), heavy=(0, 256), heavy_col=0.05, dup=0.02),
    Spec("tall_sparse_s", 1 << 10, 16, 3, (61, 61, 61), active_rows=40),
    Spec("wide_s", 32, 1 << 10, 20, (1 << 10, 32, 32), col_pool=256),
    Spec("dups_s", 256, 256, 10, (512, 263, 256), active_rows=192, dup=1 / 8),
    Spec("padding_s", 300, 500, 37, (701, 300, 450), active_rows=260, via_new=True),
    CASES["many_inputs"][0],
]

_cache = {}


def cached_instance(spec, seed=0):
    if (spec, seed) not in _cache:
        _cache[(spec, seed)] = shape_instance(spec, seed)
    return _cache[(spec, seed)]


@pytest.mark.parametrize("name", list(CASES))
def test_mirror_places_every_case(name):
    spec, want = CASES[name]
    got = spec_plan(spec)
    assert {k: got[k] for k in want} == want
    if name == "tall_sparse":   # with the background commitment off, the non-early path left-pads ry (snark.cpp snark_prove)
        off = spec_plan(spec, overlap=False)
        assert not off["early"] and off["pad_ry"] == 9


def test_mirror_reaches_the_uncovered_branches():
    """together the cases reach what produce_synthetic_r1cs never does: ops jG = 1 and 3, a memory batch smaller than the ops batch and one far
    larger, each R1CS phase streaming while the other is small, ry shorter than rx, and the witness rows on the row tables below 2^20"""
    plans = {n: spec_plan(s) for n, (s, _) in CASES.items()}
    assert {1, 3} <= {p["ops_jG"] for p in plans.values()}
    assert any(p["cells"] < p["N"] for p in plans.values()) and any(p["cells"] >= 32 * p["N"] for p in plans.values())
    assert any(p["phase1_streams"] and not p["phase2_streams"] for p in plans.values())
    assert any(p["phase2_streams"] and not p["phase1_streams"] for p in plans.values())
    assert any(p["pad_ry"] > 1 for p in plans.values()) and any(p["pad_rx"] > 1 for p in plans.values())
    assert any(p["witness_rt"] and p["num_vars"] < 1 << 20 for p in plans.values())


def test_mirror_single_op_instance():
    """num_cons = 2 with one entry per matrix: N = 1 and product circuits of zero layers, which snark_encode must refuse"""
    p = plan(2, 2, 1, (1, 1, 1))
    assert p["N"] == 1 and p["ops_layers"] == 0


def test_generator_buckets_change_exactly_one_spark_width():
    """one power-of-two bucket up or down changes exactly one of the comb_ops / derefs generator widths (their log-sizes differ by one), so a
    mismatched bucket is caught either by SNARK::encode (comb_ops) or by SNARK::prove (derefs)"""
    for lg in range(4, 22):
        base = gens_widths(512, 512, 10, 1 << lg)
        assert gens_widths(512, 512, 10, (1 << (lg - 1)) + 1) == base
        for other in (1 << (lg - 1), 1 << (lg + 1)):
            w = gens_widths(512, 512, 10, other)
            assert w[1] == base[1] and (w[0] != base[0]) != (w[2] != base[2])


@pytest.mark.parametrize("name", list(CASES))
def test_case_is_satisfiable_and_shaped(name):
    spec, _ = CASES[name]
    si = cached_instance(spec)
    assert si.oracle.is_sat(si.vars, si.inputs)
    assert [len(t) for t in si.triples] == list(spec.nnz)
    p = spec_plan(spec)
    M = (si.oracle.inst.A, si.oracle.inst.B, si.oracle.inst.C)
    assert (si.oracle.inst.num_cons, si.oracle.inst.num_vars) == (p["num_cons"], p["num_vars"])
    assert max(Mx.get_num_nz_entries() for Mx in M) == p["N"]
    rows = set(int(r) for Mx in M for r in Mx.row)
    assert len(rows) == (spec.active_rows or spec.num_cons)
    if spec.heavy:
        assert np.bincount(M[spec.heavy[0]].row.astype(np.int64)).max() >= spec.heavy[1]
    if spec.dup:
        for Mx in M:
            keys = Mx.row * np.uint64(1 << 32) + Mx.col
            assert len(np.unique(keys)) < len(keys)
    if spec.col_pool:
        assert len(np.unique(M[0].col)) < spec.num_vars // 8
    # entries on input columns (after Instance::new's remap), and explicit 0 / 1 / q-1 values, in every matrix that holds more than pivots
    nvp = si.oracle.inst.num_vars
    for m, Mx in enumerate(M):
        if m == 2 and spec.nnz[2] == (spec.active_rows or spec.num_cons):
            continue
        assert (Mx.col > np.uint64(nvp)).any()
        assert {0, 1, Q - 1} <= set(oc.to_ints(Mx.val[:4096]))
    # a wrong value of the most used variable breaks satisfiability
    cols = np.concatenate([Mx.col for Mx in M]).astype(np.int64)
    bad = si.vars.copy()
    bad[int(np.bincount(cols[cols < spec.num_vars]).argmax())] = oc.to_arr([12345])[0]
    assert not si.oracle.is_sat(bad, si.inputs)


@pytest.mark.parametrize("spec", SCALED, ids=[s.name for s in SCALED])
def test_oracle_proves_scaled_down_family(spec):
    """each shape family at oracle size: SNARK encode / prove / verify and NIZK prove / verify by the oracle"""
    si = cached_instance(spec, 1)
    oi = si.oracle
    assert oi.is_sat(si.vars, si.inputs)
    nz = max(spec.nnz)
    gens = spark.SNARKGens(spec.num_cons, spec.num_vars, spec.num_inputs, nz)
    comm, decomm = spark.SNARK.encode(oi, gens)
    proof = spark.SNARK.prove(oi, comm, decomm, si.vars, si.inputs, gens, oc.Transcript(b"shapes"), r1cs.tape_seed(1))
    parsed, pos = pr.deser(spark.SNARK, proof.ser())
    assert pos == len(proof.ser())
    parsed.verify(comm, si.inputs, oc.Transcript(b"shapes"), gens)
    bad = list(si.inputs)
    bad[0] = (bad[0] + 1) % Q
    with pytest.raises((pr.ProofVerifyError, AssertionError)):
        parsed.verify(comm, bad, oc.Transcript(b"shapes"), gens)
    ngens = r1cs.NIZKGens(spec.num_cons, spec.num_vars, spec.num_inputs)
    nizk = r1cs.NIZK.prove(oi, si.vars, si.inputs, ngens, oc.Transcript(b"shapes"), r1cs.tape_seed(1))
    nizk.verify(oi, si.inputs, oc.Transcript(b"shapes"), ngens)


def test_oracle_rejects_single_op_instance():
    """the reference panics when every matrix has at most one entry (ProductCircuit over one entry); so does the oracle"""
    one = (1).to_bytes(32, "little")
    oi = r1cs.Instance.new(2, 2, 1, [(0, 0, one)], [(0, 0, one)], [(0, 0, one)])
    gens = spark.SNARKGens(2, 2, 1, 1)
    comm, decomm = spark.SNARK.encode(oi, gens)
    assert comm.comm.num_ops == 1
    with pytest.raises(AssertionError):
        spark.SNARK.prove(oi, comm, decomm, oc.to_arr([1, 0]), [0], gens, oc.Transcript(b"shapes"), r1cs.tape_seed(0))
