"""Dot products beside the caller's product circuits on the GPU (sp_prod_build_dotp / sp_prod_prove_dotp_t / sp_prod_verify_dotp_t,
ProductCircuits(dotps=...) / ProductCircuitEvalProofBatched.prove_dotp / verify_dotp): products, half sums, proof bytes, rand, leaf and operand
evaluations and transcript states against the oracle's ProductCircuitEvalProofBatched.prove with the split DotProductCircuits, for operands of
every kind, on both sides of batched_prove's eq-factored threshold (2^17 entries: the dot-product instances take the second standard launch of
layer 0's eq-factored rounds) and of one 64-table heads gather (k = 2, kd = 11 at m <= 2); both verifiers accepting, and rejecting a flipped
dotp claim; a sparse evaluation proved from dereferenced values on one transcript with the oracle replaying the verifier; the refusals; the
launch counts; and the heads cases again under the memory-check mode."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import spark as sk
from test_gpu_product import build_launches, leaf_eval, leaf_vector, prove_launches

pytestmark = pytest.mark.gpu
Q = oc.Q
LABEL = b"prod-dotp-gpu"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NT = 4
KKD = [(1, 1), (3, 2), (22, 1), (2, 11)]
CASES = [(m, k, kd) for m in (1, 2, 3, 6, 12) for k, kd in KKD] + [(17, 3, 2)]


def case_id(c):
    return "m%d-k%d-kd%d" % c


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    sb.default_context()
    return sb


def ints(a):
    return oc.to_ints(np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4))


def transcripts(sb, products, halves, label=LABEL):
    """the oracle's and the library's transcript after the same caller prefix, the products and the half sums absorbed"""
    ot, st = oc.Transcript(label), sb.Transcript(label)
    for t in (ot, st):
        t.append_message(b"app", b"prefix")
    for p in list(products) + list(halves):
        ot.append_scalar(b"claim", p)
        st.append_message(b"claim", oc.scalar_to_bytes(p))
    return ot, st


def same_transcript(ot, st):
    return ot.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64)


def descs(m, k, kd):
    """circuit leaves (a plain table, or a fingerprint of three tables) and the operands of each dot product, cycling over the kinds: a plain
    table, a three-source form, an index term, a constant weight of one, and one table read by several operands"""
    r, g, s = oc.to_ints(oc.prg_scalars("prod-dotp-gpu-rg-%d-%d-%d" % (m, k, kd), 3))
    leaves = [([(c % NT, 1)], 0, 0) if c % 2 == 0 else ([(1, r * r % Q), (2, r), (3, 1)], 0, -g % Q) for c in range(k)]
    kinds = [(([(0, 1)], 0, 0), ([(1, r), (2, s), (3, 1)], 0, g), ([], 0, 1)),
             (([], 1, 0), ([(2, 1)], 0, 0), ([(1, 1)], 0, 0)),
             (([(3, r)], s, 0), ([(3, 1)], 0, g), ([(3, 1), (0, s)], 0, 0)),
             (([(1, 1)], 0, 0), ([(0, 1)], 0, 0), ([], Q - 1, r))]
    return leaves, [kinds[d % len(kinds)] for d in range(kd)]


def lib_forms(sb, ds):
    return [sb.ProductLeaves(s, index_coeff=i, const=c) for s, i, c in ds]


def tables(m, tag):
    T = [oc.prg_scalars("prod-dotp-gpu-%s-%d-%d" % (tag, m, j), 1 << m) for j in range(NT)]
    T[0][0] = oc.to_arr([0])[0]
    T[3][-1] = oc.to_arr([Q - 1])[0]
    return T


def oracle_side(T, ld, dd, n):
    cs = [sk.ProductCircuit(leaf_vector(d, T, n)) for d in ld]
    ops = [[leaf_vector(o, T, n) for o in ds] for ds in dd]
    dps = []
    for o in ops:
        dps.extend(sk.DotProductCircuit(*o).split())
    return cs, ops, dps


# ---------------------------------------------------------------------------------------------------- parity with the oracle, both verifiers
@pytest.mark.parametrize("m,k,kd", CASES, ids=[case_id(c) for c in CASES])
def test_parity(sb, m, k, kd):
    n = 1 << m
    T = tables(m, "par")
    ld, dd = descs(m, k, kd)
    polys = [sb.DensePolynomial(t) for t in T]
    pc = sb.ProductCircuits(polys, lib_forms(sb, ld), [lib_forms(sb, ds) for ds in dd])
    cs, ops, dps = oracle_side(T, ld, dd, n)
    products, halves = [c.evaluate() for c in cs], [d.evaluate() for d in dps]
    assert ints(pc.products) == products and pc.dotp_claims.shape == (kd, 2, 4) and ints(pc.dotp_claims) == halves
    ot, st = transcripts(sb, products, halves)
    proof, rand, evals, dotp = sb.ProductCircuitEvalProofBatched.prove_dotp(pc, st)
    want, orand = sk.ProductCircuitEvalProofBatched.prove(cs, dps, ot)
    assert proof == pr.ser(want)
    assert ints(rand) == orand
    assert ints(evals) == [oc.evaluate(v, orand) for v in [leaf_vector(d, T, n) for d in ld]]
    assert dotp.shape == (kd, 3, 4) and ints(dotp) == [oc.evaluate(v, orand) for o in ops for v in o]
    assert same_transcript(ot, st)
    for p, t in zip(polys, T):   # read, never modified
        assert np.array_equal(p.to_numpy(), t)
    # both verifiers accept, with the prover's claims; sp_prod_leaf_eval of the operand forms gives the dotp claims
    ot, vt = transcripts(sb, products, halves)
    vrand, vclaims, vdotp = sb.ProductCircuitEvalProofBatched.verify_dotp(proof, pc.products, pc.dotp_claims, m, vt)
    assert np.array_equal(vrand, rand) and np.array_equal(vclaims, evals) and np.array_equal(vdotp, dotp)
    oclaims, odotp, orand2 = pr.deser(sk.ProductCircuitEvalProofBatched, proof)[0].verify(products, halves, n, ot)
    assert orand2 == orand and oclaims == ints(evals) and odotp == ints(dotp)
    assert same_transcript(ot, vt)
    tev = oc.to_arr([oc.evaluate(t, orand) for t in T])
    for d, ds in enumerate(dd):
        assert ints(sb.product_leaf_eval(lib_forms(sb, ds), tev, rand)) == ints(dotp[d]) == [leaf_eval(o, ints(tev), orand) for o in ds]
    # a flipped dotp claim: both reject
    bad = pr.deser(sk.ProductCircuitEvalProofBatched, proof)[0]
    bad.claims_dotp[2][-1] = (bad.claims_dotp[2][-1] + 1) % Q
    ot, vt = transcripts(sb, products, halves)
    with pytest.raises(sb.ProofVerifyError):
        sb.ProductCircuitEvalProofBatched.verify_dotp(pr.ser(bad), pc.products, pc.dotp_claims, m, vt)
    with pytest.raises(pr.ProofVerifyError):
        bad.verify(products, halves, n, ot)
    assert same_transcript(ot, vt)


# ---------------------------------------------------------------------------------------------------- launch counts
def eq_factored_rounds(m):
    """batched_prove's eq-factored rounds of layer 0 (tables of 2^(m-1) entries, m - 1 rounds): those whose tables hold >= 2^14 entries, all
    but the last round at most; the dot-product instances take a second launch in each"""
    rounds, half, jG = m - 1, 1 << (m - 1), 0
    if rounds >= 2:
        while jG + 1 < rounds and (half >> jG) >= 16384:
            jG += 1
    return jG


def test_launch_counts(sb):
    """build: build_launches(m, k) and one k_dotp_operands launch.  Prove: prove_launches(m), one more per eq-factored round of layer 0, and,
    when the last layer's 2k + 6kd tables exceed the 64 of one k_fold_top or k_heads launch, one more heads gather at m <= 2 and one more launch
    of each bind that layer 0 makes with fold_top: its one round at m = 2, the switch out of its eq-factored rounds at m >= 15"""
    for m in (1, 2, 3, 12, 15, 16, 17):
        for k, kd in KKD:
            T = tables(m, "launch")
            ld, dd = descs(m, k, kd)
            polys = [sb.DensePolynomial(t) for t in T]
            l0 = sb.kernel_launches()
            pc = sb.ProductCircuits(polys, lib_forms(sb, ld), [lib_forms(sb, ds) for ds in dd])
            l1 = sb.kernel_launches()
            _, st = transcripts(sb, ints(pc.products), ints(pc.dotp_claims))
            sb.ProductCircuitEvalProofBatched.prove_dotp(pc, st)
            l2 = sb.kernel_launches()
            over = 2 * k + 6 * kd > 64
            jG = eq_factored_rounds(m)
            extra = jG + (1 if over and m <= 2 else 0) + (1 if over and (m == 2 or jG > 0) else 0)
            assert (l1 - l0, l2 - l1) == (build_launches(m, k) + 1, prove_launches(m) + extra), (m, k, kd)


# ---------------------------------------------------------------------------------------------------- a sparse evaluation from dereferenced values
def test_sparse_evaluation_one_transcript(sb):
    """v = sum_j E[addr_j] val_j for committed (addr, val) and the public eq table E = eq(r_x, .), as SPARK proves it from the dereferenced values
    d_j = E[addr_j]: a read-only memory check of d against E (init, read, write, audit) and the dot product (d, val, 1), on one transcript"""
    m = 10
    n = 1 << m
    rng = np.random.default_rng(5)
    r_x = oc.to_ints(oc.prg_scalars("prod-dotp-gpu-rx", m))
    E = oc.eq_evals(r_x)
    addr = rng.integers(0, n, size=n, dtype=np.uint64)
    read_ts, audit = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint64)
    for i, a in enumerate(addr):
        read_ts[i] = audit[a]
        audit[a] += 1
    d = np.ascontiguousarray(E[addr.astype(np.int64)])
    val = oc.prg_scalars("prod-dotp-gpu-val", n)
    T = [oc.from_u64(addr), d, oc.from_u64(read_ts), val, E, oc.from_u64(audit)]   # ops: addr, d, read_ts, val; memory: E, audit_ts
    v = sum(a * b for a, b in zip(oc.to_ints(d), oc.to_ints(val))) % Q
    big = sb.PolyCommitmentGens(m + 2, LABEL)
    g_ops, g_mem = big, big.view(m + 1)
    og = pr.PolyCommitmentGens(m + 2, LABEL)
    polys = [sb.DensePolynomial(t) for t in T]
    seed = ints(sb.tape_seed(23))[0]
    stape, otape = sb.RandomTape(sb.tape_seed(23)), oc.RandomTape(b"proof", seed)

    def head(t, comms, chal):
        t.append_message(b"app", b"sparse evaluation")
        for label, c in zip((b"comm_ops", b"comm_mem"), comms):
            c.append_to_transcript(label, t)
        return [oc.scalar_from_bytes_wide(chal(t)) for _ in range(2)]

    def memory_descs(r, g):
        r2 = r * r % Q
        return [([(4, r)], 1, -g % Q), ([(2, r2), (1, r), (0, 1)], 0, -g % Q), ([(2, r2), (1, r), (0, 1)], 0, (r2 - g) % Q), ([(5, r2), (4, r)], 1, -g % Q)]

    dot = [(([(1, 1)], 0, 0), ([(3, 1)], 0, 0), ([], 0, 1))]   # (d, val, 1)

    # the library, as a caller drives it
    st = sb.Transcript(LABEL)
    c_ops, _ = sb.poly_commit(polys[:4], g_ops)
    c_mem, _ = sb.poly_commit(polys[4:], g_mem)
    r, g = head(st, (c_ops, c_mem), lambda t: t.challenge_bytes(b"challenge_r_hash", 64))
    ld = memory_descs(r, g)
    pc = sb.ProductCircuits(polys, lib_forms(sb, ld), [lib_forms(sb, ds) for ds in dot])
    prods, halves = ints(pc.products), ints(pc.dotp_claims)
    assert prods[0] * prods[2] % Q == prods[1] * prods[3] % Q and sum(halves) % Q == v
    for p in prods + halves:
        st.append_message(b"claim", oc.scalar_to_bytes(p))
    proof, rand, _, dotp = sb.ProductCircuitEvalProofBatched.prove_dotp(pc, st)
    st.append_message(b"protocol-name", b"Derefs evaluation proof")
    p_ops, ev_ops = sb.PolyEvalProof.prove_joint(polys[:4], None, rand, g_ops, st, stape)
    st.append_message(b"protocol-name", b"Derefs evaluation proof")
    p_mem, ev_mem = sb.PolyEvalProof.prove_joint(polys[4:], None, rand, g_mem, st, stape)

    # the oracle replays the verifier on the library's bytes
    ot = oc.Transcript(LABEL)
    oc_ops, _ = pr.poly_commit(sk.merge(T[:4]), og)
    oc_mem, _ = pr.poly_commit(sk.merge(T[4:]), og)
    assert (oc_ops.C, oc_mem.C) == (c_ops.C, c_mem.C)
    assert head(ot, (oc_ops, oc_mem), lambda t: t.challenge_bytes(b"challenge_r_hash", 64)) == [r, g]
    assert prods[0] * prods[2] % Q == prods[1] * prods[3] % Q                      # the multiset equation: init * write == read * audit
    assert sum(halves) % Q == v                                                     # the half sums add up to the claimed value
    for p in prods + halves:
        ot.append_scalar(b"claim", p)
    oclaims, odotp, orand = pr.deser(sk.ProductCircuitEvalProofBatched, proof)[0].verify(prods, halves, n, ot)
    assert orand == ints(rand) and odotp == ints(dotp)
    evals = ints(ev_ops) + ints(ev_mem)
    sk.DerefsEvalProof(pr.deser(pr.PolyEvalProof, p_ops.data)[0]).verify(orand, evals[:4], [], og, oc_ops, ot)
    sk.DerefsEvalProof(pr.deser(pr.PolyEvalProof, p_mem.data)[0]).verify(orand, evals[4:], [], og, oc_mem, ot)
    eq = 1
    for a, b in zip(r_x, orand):
        eq = eq * (a * b + (1 - a) * (1 - b)) % Q
    assert evals[4] == eq                                                           # E is public: the verifier evaluates it itself
    assert oclaims == [leaf_eval(ds, evals, orand) for ds in ld]                   # leaf forms at rand
    assert odotp == [leaf_eval(o, evals, orand) for o in dot[0]]                   # operand forms at rand
    assert same_transcript(ot, st)


# ---------------------------------------------------------------------------------------------------- refusals leave everything as it was
def test_refusals_leave_inputs_alone(sb):
    m = 5
    T = tables(m, "refuse")
    polys = [sb.DensePolynomial(t) for t in T]
    bad = np.full(4, 2 ** 64 - 1, dtype=np.uint64)   # limbs >= q
    st = sb.Transcript(LABEL)
    st0 = st.state.raw
    plain = sb.ProductLeaves([(0, 1)])
    one = sb.ProductLeaves([], const=1)
    triple = [plain, sb.ProductLeaves([(1, 1)]), one]

    def refused(fn, exc, what):
        live = sb.device_bytes_live()
        l0 = sb.kernel_launches()
        with pytest.raises(exc) as e:
            fn()
        assert what in str(e.value), str(e.value)
        assert st.state.raw == st0
        assert sb.device_bytes_live() == live and sb.kernel_launches() == l0
        for p, t in zip(polys, T):
            assert np.array_equal(p.to_numpy(), t)

    E, S = sb.SpartanB200Error, sb.R1CSError
    refused(lambda: sb.ProductCircuits(polys, [plain] * 3, [triple] * 11), E, "11 dot products next to 3 circuits")   # k + 2 kd = 25
    refused(lambda: sb.ProductCircuits(polys, [plain], []), E, "0 dot products next to 1 circuits")
    refused(lambda: sb.ProductCircuits(polys, [plain], [[plain, sb.ProductLeaves([(1, bad)]), one]]), S, "dot product 0 right: coefficient")
    refused(lambda: sb.ProductCircuits(polys, [plain], [[plain, plain, sb.ProductLeaves([(4, 1)])]]), E, "dot product 0 weight: source 0 is table 4")
    # sp_prod_prove_t on a handle with dot products: refused, the handle kept for prove_dotp
    pc = sb.ProductCircuits(polys, [plain], [triple])
    refused(lambda: sb.ProductCircuitEvalProofBatched.prove(pc, st), E, "sp_prod_prove_dotp_t")
    sb.ProductCircuitEvalProofBatched.prove_dotp(pc, sb.Transcript(LABEL))
    # a second proof on a spent handle
    refused(lambda: sb.ProductCircuitEvalProofBatched.prove_dotp(pc, st), E, "consumed")
    # prove_dotp of a handle without dot products: the plain proof's bytes
    a, b = sb.ProductCircuits(polys, [plain]), sb.ProductCircuits(polys, [plain])
    p1 = sb.ProductCircuitEvalProofBatched.prove(a, sb.Transcript(LABEL))
    p2 = sb.ProductCircuitEvalProofBatched.prove_dotp(b, sb.Transcript(LABEL))
    assert p1[0] == p2[0] and np.array_equal(p1[1], p2[1]) and p2[3].shape == (0, 3, 4)


# ---------------------------------------------------------------------------------------------------- the heads cases under the memory-check mode
def test_heads_cases_under_memcheck(tmp_path):
    """m = 1 and 2 at k = 2, kd = 11: the last layer's 70 final claims go through two heads gathers"""
    if os.environ.get("SP_MEMCHECK_OUT"):
        pytest.skip("already running under the memory-check mode")
    out = tmp_path / "memcheck.json"
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "tests"), ROOT] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    env["SP_MEMCHECK_OUT"] = str(out)
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "memcheck_plugin", "-p", "no:cacheprovider", "-k", "m1-k2-kd11 or m2-k2-kd11",
           os.path.join(ROOT, "tests", "test_gpu_product_dotp.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-20000:]
    assert "2 passed" in p.stdout, p.stdout[-2000:]
    tot = json.load(open(out))
    assert tot["violations"] == 0, tot
    assert tot["blocks_filled"] > 0 and tot["context_refills"] > 0, tot
