"""Per-kernel launch counts of the prover's inner-product proofs and sumchecks: DotProductProofLog on both generator layouts (the table layout
up to SP_DOTLOG_TABLE_MAX_N, the folding layout above it, across the segmented / bucket thresholds of its rounds), PolyEvalProof and its joint
opening, the ZK and plain sumchecks of caller-defined polynomials, and whole NIZK and SNARK proofs.  The counts are pinned: a change to how these
paths drive the device shows up here, kernel family by kernel family.

Each call runs once unprofiled (lazily built host tables and scratch), then again with the library's profiler on.  Run this file as a script
to print the counts of every case as JSON (the numbers to pin after a deliberate change):

    python tests/test_gpu_prover_launches.py [out.json]"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
Q = 2**252 + 27742317777372353535851937790883648493
LABEL = b"launch-gpu"


def L(x):
    """x as Montgomery limbs"""
    return np.frombuffer((x % Q * 2**256 % Q).to_bytes(32, "little"), dtype=np.uint64).copy()


def S(sb, tag, n):
    return sb.prg_scalars("launches-" + tag, n)


def dotlog(sb, logn):
    n = 1 << logn
    g = sb.DotProductProofGens(n, LABEL)
    x, a = S(sb, "dotlog-x-%d" % n, n), S(sb, "dotlog-a-%d" % n, n)

    def run():
        proof, Cx, Cy = sb.DotProductProofLog.prove(g, sb.Transcript(LABEL), sb.RandomTape(sb.tape_seed(1)), x, L(3), a, None, L(4))
        return proof.data + Cx + Cy
    return run


def polyeval(sb, ell):
    g = sb.PolyCommitmentGens(ell, LABEL)
    Z = S(sb, "polyeval-%d" % ell, 1 << ell)
    blinds = S(sb, "polyeval-blinds-%d" % ell, 1 << (ell // 2))
    r = S(sb, "polyeval-r-%d" % ell, ell)

    def run():
        proof, C_Zr, Zr = sb.PolyEvalProof.prove(sb.DensePolynomial(Z), blinds, r, None, L(9), g, sb.Transcript(LABEL), sb.RandomTape(sb.tape_seed(2)))
        return proof.data + C_Zr + Zr.tobytes()
    return run


def polyeval_joint(sb, m, k):
    ell = m + (k - 1).bit_length()
    g = sb.PolyCommitmentGens(ell, LABEL)
    Z = [S(sb, "joint-%d-%d-%d" % (m, k, j), 1 << m) for j in range(k)]
    r = S(sb, "joint-r-%d-%d" % (m, k), m)

    def run():
        proof, evals = sb.PolyEvalProof.prove_joint([sb.DensePolynomial(z) for z in Z], None, r, g, sb.Transcript(LABEL), sb.RandomTape(sb.tape_seed(3)))
        return proof.data + evals.tobytes()
    return run


COMPOSITIONS = {   # degree -> (tables, terms)
    1: (2, [(1, (0,)), (5, (1,))]),
    3: (4, [(1, (0, 1, 2)), (Q - 1, (0, 3))]),
    6: (6, [(7, (0, 1, 2, 3, 4, 5)), (11, (5, 5, 0, 1, 2)), (1, (3,)), (Q - 1, (2, 3, 5))]),
}
ROUNDS = 10


def composition(sb, d):
    k, terms = COMPOSITIONS[d]
    return k, sb.Composition([(L(c), fs) for c, fs in terms])


def zk_sumcheck(sb, d):
    k, comp = composition(sb, d)
    g1, gn = sb.MultiCommitGens(1, LABEL + b"-1"), sb.MultiCommitGens(d + 1, LABEL + b"-n")
    tabs = [S(sb, "zk-%d-%d" % (d, j), 1 << ROUNDS) for j in range(k)]

    def run():
        polys = [sb.DensePolynomial(t) for t in tabs]
        proof, r, finals, bp = sb.ZKSumcheckInstanceProof.prove(polys, comp, L(0), L(0), ROUNDS, g1, gn, sb.Transcript(LABEL), sb.RandomTape(sb.tape_seed(4)))
        return proof.data + r.tobytes() + finals.tobytes() + bp.tobytes()
    return run


def sumcheck(sb):
    k, comp = composition(sb, 3)
    tabs = [S(sb, "sc-%d" % j, 1 << ROUNDS) for j in range(k)]

    def run():
        proof, r, finals, e = sb.sumcheck_prove([sb.DensePolynomial(t) for t in tabs], comp, L(0), ROUNDS, sb.Transcript(LABEL))
        return proof + r.tobytes() + finals.tobytes() + e.tobytes()
    return run


R1CS_SHAPE = (1 << 12, 1 << 12, 10)


def nizk(sb):
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(*R1CS_SHAPE, seed=5)
    gens = sb.NIZKGens(*R1CS_SHAPE)
    return lambda: sb.NIZK.prove(inst, vars_, inputs, gens, b"launches", sb.tape_seed(5)).bytes


def snark(sb):
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(*R1CS_SHAPE, seed=6)
    gens = sb.SNARKGens(*R1CS_SHAPE, R1CS_SHAPE[0])
    comm = sb.SNARK.encode(inst, gens)
    return lambda: sb.SNARK.prove(inst, comm, vars_, inputs, gens, b"launches", sb.tape_seed(6)).bytes


CASES = {}
for _lg in (0, 8, 9, 11, 12, 16):
    CASES["dotlog-2^%d" % _lg] = lambda sb, lg=_lg: dotlog(sb, lg)
for _ell in (0, 5, 12):
    CASES["polyeval-ell%d" % _ell] = lambda sb, ell=_ell: polyeval(sb, ell)
CASES["polyeval-joint-m10-k3"] = lambda sb: polyeval_joint(sb, 10, 3)
for _d in (1, 3, 6):
    CASES["zk-sumcheck-d%d" % _d] = lambda sb, d=_d: zk_sumcheck(sb, d)
CASES["sumcheck-d3"] = sumcheck
CASES["nizk-2^12"] = nizk
CASES["snark-2^12"] = snark


def measure(sb, case):
    """(kernel family -> launches, total launches, digest of the call's outputs) of the second of two identical calls"""
    run = CASES[case](sb)
    run()
    sb.api.prof_enable(True)
    try:
        before = sb.kernel_launches()
        out = run()
        total = sb.kernel_launches() - before
        rep = sb.api.prof_report()
    finally:
        sb.api.prof_enable(False)
    return {k: v["launches"] for k, v in sorted(rep.items())}, total, hashlib.sha256(out).hexdigest()


EXPECTED = {   # case: (kernel family -> launches, total launches)
    'dotlog-2^0': ({'compress_batch': 1, 'dot': 1, 'msm_rows': 2}, 8),
    'dotlog-2^11': ({'dot': 23, 'dotlog_fold': 11, 'dotlog_scalars': 11, 'ipa_fold_ab': 11, 'msm_var': 1, 'msm_var_segmented': 11, 'pip_accumulate': 1, 'pip_reduce': 1, 'pip_sort': 1}, 88),
    'dotlog-2^12': ({'dot': 25, 'dotlog_fold': 12, 'dotlog_scalars': 12, 'ipa_fold_ab': 12, 'msm_var': 3, 'msm_var_segmented': 11, 'pip_accumulate': 3, 'pip_reduce': 3, 'pip_sort': 3}, 108),
    'dotlog-2^16': ({'dot': 33, 'dotlog_fold': 16, 'dotlog_scalars': 16, 'ipa_fold_ab': 16, 'msm_var': 11, 'msm_var_segmented': 11, 'pip_accumulate': 11, 'pip_reduce': 11, 'pip_sort': 11}, 192),
    'dotlog-2^8': ({'dot': 1, 'ipa_fold_ab': 8, 'ipa_msm': 10, 'msm_rows': 1}, 23),
    'dotlog-2^9': ({'dot': 19, 'dotlog_fold': 9, 'dotlog_scalars': 9, 'ipa_fold_ab': 9, 'msm_var': 1, 'msm_var_segmented': 9, 'pip_accumulate': 1, 'pip_reduce': 1, 'pip_sort': 1}, 74),
    'nizk-2^12': ({'bound_rows': 1, 'compress_batch': 3, 'dot': 1, 'eq_evals': 5, 'fold_top': 2, 'ipa_fold_ab': 6, 'ipa_msm': 8, 'lincomb3': 1, 'msm_rows': 11, 'sc_eval': 2, 'sc_fold_eval': 1, 'sc_fold_eval_small': 22, 'spmv': 6}, 90),
    'polyeval-ell0': ({'bound_rows': 1, 'compress_batch': 1, 'dot': 1, 'eq_evals': 2, 'msm_rows': 2}, 12),
    'polyeval-ell12': ({'bound_rows': 1, 'dot': 1, 'eq_evals': 2, 'ipa_fold_ab': 6, 'ipa_msm': 8, 'msm_rows': 1}, 23),
    'polyeval-ell5': ({'bound_rows': 1, 'dot': 1, 'eq_evals': 2, 'ipa_fold_ab': 3, 'ipa_msm': 5, 'msm_rows': 1}, 17),
    'polyeval-joint-m10-k3': ({'bound_rows': 1, 'bound_rows_many': 1, 'dot_many': 1, 'eq_evals': 2, 'ipa_fold_ab': 6, 'ipa_msm': 8, 'msm_rows': 1}, 25),
    'snark-2^12': ({'bound_rows': 4, 'compress_batch': 5, 'dot': 7, 'dot_many': 2, 'eq_evals': 63, 'fold_top': 4, 'gather': 6, 'hadamard': 23, 'ipa_fold_ab': 29, 'ipa_msm': 37, 'lincomb3': 1, 'msm_rows': 16, 'sc_eval': 25, 'sc_fold_eval': 1, 'sc_fold_eval_small': 143, 'spark_hash': 16, 'spmv': 6}, 445),
    'sumcheck-d3': ({'fold_top': 1, 'scp_eval': 1, 'scp_fold_eval_small': 9}, 12),
    'zk-sumcheck-d1': ({'compress_batch': 1, 'fold_top': 1, 'msm_rows': 4, 'scp_eval': 1, 'scp_fold_eval_small': 9}, 21),
    'zk-sumcheck-d3': ({'compress_batch': 1, 'fold_top': 1, 'msm_rows': 4, 'scp_eval': 1, 'scp_fold_eval_small': 9}, 21),
    'zk-sumcheck-d6': ({'compress_batch': 1, 'fold_top': 1, 'msm_rows': 4, 'scp_eval': 1, 'scp_fold_eval_small': 9}, 21),
}


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    sb.default_context()
    return sb


@pytest.mark.parametrize("case", sorted(CASES))
def test_launch_counts(sb, case):
    families, total, _ = measure(sb, case)
    want_families, want_total = EXPECTED[case]
    assert total == want_total, (case, total, families)
    assert families == want_families, case


if __name__ == "__main__":
    import spartan_b200 as sb_mod
    sb_mod.default_context()
    res = {}
    for c in sorted(CASES):
        fam, tot, dig = measure(sb_mod, c)
        res[c] = {"families": fam, "total": tot, "digest": dig}
        print(c, tot, fam, flush=True)
    text = json.dumps(res, indent=1, sort_keys=True)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(text)
    else:
        print(text)
