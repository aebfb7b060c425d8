"""The SPARK evaluation proof for any batch size b, on the oracle alone (no GPU): a test-local generalisation of the reference's
ProductLayerProof::prove, which asserts b = 3 (sparse_mlpoly.rs:1121-1122), with the ops batch ordered row.read[b], row.write[b], col.read[b],
col.write[b] and the dot-product circuits left_0, right_0, left_1, right_1, ..  At b = 3 it gives the oracle's own proof bytes; at b = 1, 2, 4
the oracle's general verify accepts it.  Also: the library's SparkDims against SparseMatPolyCommitmentGens's formulas over a grid of shapes."""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import r1cs as r1
from oracle.spartan_ref import spark as sk

Q = oc.Q
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ----------------------------------------------------------------------------- the generalised prover (the oracle's, with b for 3)
def product_layer_prove(row_layer, col_layer, dense, derefs, evals, T):
    """sk.ProductLayerProof.prove for any number of matrices"""
    T.append_protocol_name(b"Sparse polynomial product layer proof")

    def side(layer, name):
        init, audit = layer.init.evaluate(), layer.audit.evaluate()
        read = [c.evaluate() for c in layer.read_vec]
        write = [c.evaluate() for c in layer.write_vec]
        ws, rs = 1, 1
        for w in write:
            ws = ws * w % Q
        for r_ in read:
            rs = rs * r_ % Q
        assert init * ws % Q == rs * audit % Q
        T.append_scalar(b"claim_%s_eval_init" % name, init)
        T.append_scalars(b"claim_%s_eval_read" % name, read)
        T.append_scalars(b"claim_%s_eval_write" % name, write)
        T.append_scalar(b"claim_%s_eval_audit" % name, audit)
        return init, read, write, audit
    er = side(row_layer, b"row")
    ec = side(col_layer, b"col")
    b = len(evals)
    assert b == len(derefs.row_ops_val) == len(derefs.col_ops_val) == len(dense.val)
    dotps, el, erv = [], [], []
    for i in range(b):
        circ = sk.DotProductCircuit(derefs.row_ops_val[i].copy(), derefs.col_ops_val[i].copy(), dense.val[i].copy())
        left, right = circ.split()
        e_l, e_r = left.evaluate(), right.evaluate()
        T.append_scalar(b"claim_eval_dotp_left", e_l)
        T.append_scalar(b"claim_eval_dotp_right", e_r)
        assert (e_l + e_r) % Q == evals[i] % Q
        el.append(e_l); erv.append(e_r); dotps += [left, right]
    prods = row_layer.read_vec + row_layer.write_vec + col_layer.read_vec + col_layer.write_vec
    proof_ops, rand_ops = sk.ProductCircuitEvalProofBatched.prove(prods, dotps, T)
    proof_mem, rand_mem = sk.ProductCircuitEvalProofBatched.prove([row_layer.init, row_layer.audit, col_layer.init, col_layer.audit], [], T)
    return sk.ProductLayerProof(er, ec, (el, erv), proof_mem, proof_ops), rand_mem, rand_ops


def spark_prove(dense, rx, ry, evals, gens, T, tape):
    """sk.SparseMatPolyEvalProof.prove with product_layer_prove"""
    T.append_protocol_name(b"Sparse polynomial evaluation proof")
    assert len(evals) == dense.batch_size
    rx_ext, ry_ext = sk.equalize(rx, ry)
    mem_rx, mem_ry = oc.eq_evals(rx_ext), oc.eq_evals(ry_ext)
    derefs = dense.deref(mem_rx, mem_ry)
    comm_derefs, _ = pr.poly_commit(derefs.comb, gens.gens_derefs, None)
    sk.SparseMatPolyEvalProof._append_derefs_comm(comm_derefs, T)
    r_mem_check = T.challenge_vector(b"challenge_r_hash", 2)
    row_layer = sk.build_layers(mem_rx, dense.row, derefs.row_ops_val, (r_mem_check[0], r_mem_check[1]))
    col_layer = sk.build_layers(mem_ry, dense.col, derefs.col_ops_val, (r_mem_check[0], r_mem_check[1]))
    T.append_protocol_name(b"Sparse polynomial evaluation proof")
    ppl, rand_mem, rand_ops = product_layer_prove(row_layer, col_layer, dense, derefs, evals, T)
    phl = sk.HashLayerProof.prove((rand_mem, rand_ops), dense, derefs, gens, T, tape)
    return sk.SparseMatPolyEvalProof(comm_derefs, sk.PolyEvalNetworkProof(ppl, phl))


# ----------------------------------------------------------------------------- cases
def matrices(tag, b, x, y, nnzs):
    rng = np.random.default_rng(zlib.crc32(repr((tag, b, x, y, nnzs)).encode()))
    out = []
    for i, n in enumerate(nnzs):
        rows = rng.integers(0, 1 << x, n, dtype=np.uint64)
        cols = rng.integers(0, 1 << y, n, dtype=np.uint64)
        out.append(r1.SparseMat(x, y, rows, cols, oc.prg_scalars("spark-model-%s-%d" % (tag, i), n)))
    return out


def evaluate(polys, rx, ry):
    trx, try_ = oc.eq_evals(rx), oc.eq_evals(ry)
    return [p.evaluate_with_tables(trx, try_) for p in polys]


def run(b, x, y, nnzs, tag):
    polys = matrices(tag, b, x, y, nnzs)
    gens = sk.SparseMatPolyCommitmentGens(b"spark-model", x, y, max(nnzs), b)
    comm, dense = sk.multi_commit(polys, gens)
    rx = oc.to_ints(oc.prg_scalars("spark-model-rx-" + tag, x)) if x else []
    ry = oc.to_ints(oc.prg_scalars("spark-model-ry-" + tag, y)) if y else []
    evals = evaluate(polys, rx, ry)
    return polys, gens, comm, dense, rx, ry, evals


@pytest.mark.parametrize("x,y,nnzs", [(4, 4, [16, 9, 3]), (2, 5, [7, 32, 1]), (6, 3, [40, 40, 40])])
def test_b3_equals_the_oracle_prover(x, y, nnzs):
    _, gens, comm, dense, rx, ry, evals = run(3, x, y, nnzs, "b3-%d-%d" % (x, y))
    seed = oc.to_ints(oc.prg_scalars("spark-model-seed", 1))[0]
    T1, T2 = oc.Transcript(b"m"), oc.Transcript(b"m")
    t1, t2 = oc.RandomTape(b"proof", seed), oc.RandomTape(b"proof", seed)
    mine = spark_prove(dense, rx, ry, evals, gens, T1, t1)
    theirs = sk.SparseMatPolyEvalProof.prove(dense, rx, ry, evals, gens, T2, t2)
    assert pr.ser(mine) == pr.ser(theirs)
    assert T1.challenge_bytes(b"after", 32) == T2.challenge_bytes(b"after", 32)
    assert t1.tape.challenge_bytes(b"after", 32) == t2.tape.challenge_bytes(b"after", 32)


@pytest.mark.parametrize("b,x,y,nnzs", [(1, 4, 4, [13]), (1, 0, 3, [8]), (2, 5, 2, [20, 3]), (4, 3, 3, [8, 2, 5, 7]), (4, 1, 6, [30, 1, 64, 0])])
def test_general_b_is_accepted_by_the_oracle_verifier(b, x, y, nnzs):
    _, gens, comm, dense, rx, ry, evals = run(b, x, y, nnzs, "gen-%d-%d-%d" % (b, x, y))
    seed = oc.to_ints(oc.prg_scalars("spark-model-seed", 1))[0]
    proof = spark_prove(dense, rx, ry, evals, gens, oc.Transcript(b"m"), oc.RandomTape(b"proof", seed))
    proof.verify(comm, rx, ry, evals, gens, oc.Transcript(b"m"))
    bad = list(evals)
    bad[-1] = (bad[-1] + 1) % Q
    with pytest.raises(pr.ProofVerifyError):
        proof.verify(comm, rx, ry, bad, gens, oc.Transcript(b"m"))


def test_spark_dims_match_the_commitment_gens_formulas():
    path = os.path.join(ROOT, "spartan_b200", "libsp_hosttest_portable.so")
    if not os.path.exists(path):
        import __graft_entry__ as ge
        ge.build_hosttest()
    lib = C.CDLL(path)
    out = (C.c_size_t * 6)()
    for x in (0, 1, 5, 10, 20, 30):
        for y in (0, 1, 7, 20, 30):
            for nz in (0, 1, 2, 3, 1000, 1 << 10, (1 << 20) + 1, 1 << 24):
                for b in (1, 2, 3, 4):
                    lib.sph_spark_dims(C.c_size_t(x), C.c_size_t(y), C.c_size_t(nz), C.c_size_t(b), out)
                    v_ops = oc.log_2(oc.next_pow2(nz)) + oc.log_2(oc.next_pow2(b * 5))
                    v_mem = max(x, y) + 1
                    v_der = oc.log_2(oc.next_pow2(nz)) + oc.log_2(oc.next_pow2(b * 2))
                    want = [v_ops, v_mem, v_der] + [1 << (v - v // 2) for v in (v_ops, v_mem, v_der)]
                    assert list(out) == want, (x, y, nz, b)
