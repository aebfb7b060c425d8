"""Polynomial commitments and evaluation proofs of the caller's tables on the GPU (sp_pc_*, PolyCommitmentGens / poly_commit / PolyEvalProof):
byte parity with the oracle's poly_commit, PolyEvalProof and DerefsEvalProof for single and merged tables (the table-list row MSM and the
gathered merge), the verifiers against the oracle's proofs and their mutants, a sumcheck and its openings on one transcript, gens views, the
refusals, the launch counts, and the parity cases again under the memory-check mode."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import spark as sk

pytestmark = pytest.mark.gpu
Q = oc.Q
LABEL = b"pc-gpu"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL_VARS = 18   # the module's gens: views of one set for every num_vars up to this


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    sb.default_context()
    return sb


@pytest.fixture(scope="module")
def big(sb):
    return sb.PolyCommitmentGens(SMALL_VARS, LABEL)


_ogens = {}


def ogens(ell):
    """the oracle's PolyCommitmentGens (they depend on n only)"""
    n = 1 << (ell - ell // 2)
    if n not in _ogens:
        _ogens[n] = pr.PolyCommitmentGens(ell, LABEL)
    return _ogens[n]


def shape(m, k):
    c = oc.log_2(oc.next_pow2(k))
    return c, m + c


def rows_in_tables(m, c):
    return (m + c + 1) // 2 <= m


def table(tag, n):
    return oc.prg_scalars("pc-gpu-" + tag, n)


def ints(a):
    return oc.to_ints(np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4))


def seed_int(sb, i):
    return ints(sb.tape_seed(i))[0]


def tapes(sb, i):
    return sb.RandomTape(sb.tape_seed(i)), oc.RandomTape(b"proof", seed_int(sb, i))


def transcripts(sb, prefix=b"prefix"):
    ot, st = oc.Transcript(LABEL), sb.Transcript(LABEL)
    ot.append_message(b"app", prefix)
    st.append_message(b"app", prefix)
    return ot, st


def same_transcript(ot, st):
    return ot.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64)


def same_tape(otape, stape):
    return otape.tape.challenge_bytes(b"after", 64) == stape.challenge_bytes(b"after", 64)


def launches(sb):
    rep = sb.api.prof_report()
    return {k: rep[k]["launches"] if k in rep else 0 for k in ("msm_rows", "msm_rows_tables", "bound_rows_many")}


# ---------------------------------------------------------------------------------------------------- commitments
@pytest.mark.parametrize("ell", range(0, SMALL_VARS + 1))
@pytest.mark.parametrize("with_tape", [False, True])
def test_commit_parity(sb, big, ell, with_tape):
    Z = table("commit-%d" % ell, 1 << ell)
    poly = sb.DensePolynomial(Z)
    stape, otape = tapes(sb, ell) if with_tape else (None, None)
    comm, blinds = sb.poly_commit(poly, big.view(ell), stape)
    want, want_blinds = pr.poly_commit(Z, ogens(ell), otape)
    assert comm.C == want.C
    assert ints(blinds) == [b % Q for b in want_blinds]
    assert comm.to_bytes() == pr.ser(want)
    if with_tape:
        assert same_tape(otape, stape)
    assert np.array_equal(poly.to_numpy(), Z)


JOINT = [(6, 1), (5, 2), (4, 3), (7, 5), (6, 8), (8, 64), (3, 5), (10, 33),   # rows inside the tables
         (2, 8), (2, 64), (0, 2), (1, 5)]                                         # rows across tables: the gathered merge


@pytest.mark.parametrize("m,k", JOINT)
@pytest.mark.parametrize("with_tape", [False, True])
def test_joint_commit_parity(sb, big, m, k, with_tape):
    c, ell = shape(m, k)
    Z = [table("joint-%d-%d-%d" % (m, k, j), 1 << m) for j in range(k)]
    polys = [sb.DensePolynomial(z) for z in Z]
    stape, otape = tapes(sb, 100 + ell) if with_tape else (None, None)
    sb.api.prof_enable(True)
    comm, blinds = sb.poly_commit(polys, big.view(ell), stape)
    n = launches(sb)
    sb.api.prof_enable(False)
    want, want_blinds = pr.poly_commit(sk.merge(Z), ogens(ell), otape)
    assert comm.C == want.C
    assert ints(blinds) == [b % Q for b in want_blinds]
    if with_tape:
        assert same_tape(otape, stape)
    if rows_in_tables(m, c):
        assert n == {"msm_rows": 0, "msm_rows_tables": 1, "bound_rows_many": 0}, n
    else:
        assert n["msm_rows_tables"] == 0 and n["bound_rows_many"] == 0, n
    for p, z in zip(polys, Z):
        assert np.array_equal(p.to_numpy(), z)


def random_table(rng, n):
    """n uniform-looking field elements (Montgomery limbs below 2^252 < q), cheap at 2^24"""
    a = rng.integers(0, 2 ** 63, size=(n, 4), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=(n, 4), dtype=np.uint64)
    a[:, 3] &= np.uint64((1 << 59) - 1)
    return a


@pytest.mark.parametrize("ell", [22, 24])
def test_commit_large_spot_rows(sb, ell):
    """first, last and 8 random rows of a 2^22 / 2^24 commitment against oc.commit_vec"""
    sb.release_cached_memory()
    rng = np.random.default_rng(ell)
    Z = random_table(rng, 1 << ell)
    g = sb.PolyCommitmentGens(ell, LABEL)
    poly = sb.DensePolynomial(Z)
    comm, _ = sb.poly_commit(poly, g)
    L, R = 1 << (ell // 2), 1 << (ell - ell // 2)
    gens_n = ogens(ell).gens.gens_n
    assert len(comm.C) == L
    for i in [0, L - 1] + list(rng.integers(1, L - 1, size=8)):
        assert comm.C[i] == oc.commit_vec(Z[i * R:(i + 1) * R], 0, gens_n).compress(), i
    del poly, g
    sb.release_cached_memory()


# ---------------------------------------------------------------------------------------------------- single openings
def point(tag, m):
    return oc.to_ints(table("r-" + tag, m)) if m else []


@pytest.mark.parametrize("ell", range(0, SMALL_VARS + 1))
def test_single_open_parity(sb, big, ell):
    """blinds and blind_Zr on or off (cycling with ell), Zr computed on the device"""
    with_blinds, with_bzr = ell % 2 == 1, ell % 4 >= 2
    Z = table("open-%d" % ell, 1 << ell)
    r = point("open-%d" % ell, ell)
    poly = sb.DensePolynomial(Z)
    g = big.view(ell)
    stape, otape = tapes(sb, 200 + ell)
    if with_blinds:
        _, blinds = sb.poly_commit(poly, g, stape)
        _, oblinds = pr.poly_commit(Z, ogens(ell), otape)
    bzr = oc.to_ints(table("bzr-%d" % ell, 1))[0] if with_bzr else None
    ot, st = transcripts(sb)
    proof, C_Zr, Zr = sb.PolyEvalProof.prove(poly, blinds if with_blinds else None, oc.to_arr(r), None, oc.to_arr([bzr])[0] if with_bzr else None,
                                             g, st, stape)
    Zr_want = oc.evaluate(Z, r)
    want, C_want = pr.PolyEvalProof.prove(Z, oblinds if with_blinds else None, r, Zr_want, bzr, ogens(ell), ot, otape)
    assert ints(Zr) == [Zr_want]
    assert proof.data == pr.ser(want)
    assert C_Zr == C_want
    assert same_transcript(ot, st) and same_tape(otape, stape)
    assert np.array_equal(poly.to_numpy(), Z)


def test_single_open_given_zr_parity(sb, big):
    """a caller-given Zr is used as given (here the right one) and returned"""
    ell = 9
    Z = table("given", 1 << ell)
    r = point("given", ell)
    Zr = oc.evaluate(Z, r)
    stape, otape = tapes(sb, 300)
    ot, st = transcripts(sb)
    proof, C_Zr, Zr_out = sb.PolyEvalProof.prove(sb.DensePolynomial(Z), None, oc.to_arr(r), oc.to_arr([Zr])[0], None, big.view(ell), st, stape)
    want, _ = pr.PolyEvalProof.prove(Z, None, r, Zr, None, ogens(ell), ot, otape)
    assert proof.data == pr.ser(want) and ints(Zr_out) == [Zr]
    assert same_transcript(ot, st) and same_tape(otape, stape)


@pytest.mark.parametrize("ell", [20, 22])
def test_single_open_large_oracle_verifies(sb, ell):
    sb.release_cached_memory()
    rng = np.random.default_rng(1000 + ell)
    Z = random_table(rng, 1 << ell)
    r = oc.to_ints(random_table(rng, ell))
    g = sb.PolyCommitmentGens(ell, LABEL)
    poly = sb.DensePolynomial(Z)
    stape = sb.RandomTape(sb.tape_seed(ell))
    comm, blinds = sb.poly_commit(poly, g, stape)
    st = sb.Transcript(LABEL)
    proof, C_Zr, Zr = sb.PolyEvalProof.prove(poly, blinds, oc.to_arr(r), None, None, g, st, stape)
    assert ints(Zr) == [oc.evaluate(Z, r)]
    ot = oc.Transcript(LABEL)
    pr.deser(pr.PolyEvalProof, proof.data)[0].verify(ogens(ell), ot, r, C_Zr, pr.PolyCommitment(comm.C))
    sb.PolyEvalProof(proof.data).verify(g, sb.Transcript(LABEL), oc.to_arr(r), C_Zr, comm)
    del poly, g
    sb.release_cached_memory()


# ---------------------------------------------------------------------------------------------------- joint openings
def oracle_joint_prove(Z, r, blinds, ell, ot, otape):
    """(proof, evaluations) of the oracle's DerefsEvalProof.prove; with the joint commitment's blinds (DerefsEvalProof.prove has none) the same
    steps with PolyEvalProof.prove given those blinds"""
    k = len(Z)
    c = shape(len(r), k)[0]
    evals = [oc.evaluate(z, r) for z in Z]
    merged = type("Merged", (), {"comb": sk.merge(Z)})
    if blinds is None:
        return sk.DerefsEvalProof.prove(merged, evals, [], r, ogens(ell), ot, otape).proof_derefs, evals
    ot.append_protocol_name(b"Derefs evaluation proof")
    ev = evals + [0] * (oc.next_pow2(k) - k)
    ot.append_scalars(b"evals_ops_val", ev)
    ch = ot.challenge_vector(b"challenge_combine_n_to_one", c)
    for i in reversed(range(c)):
        ev = oc.bound_bot_ints(ev, ch[i])
    ot.append_scalar(b"joint_claim_eval", ev[0])
    return pr.PolyEvalProof.prove(merged.comb, blinds, ch + r, ev[0], None, ogens(ell), ot, otape)[0], evals


@pytest.mark.parametrize("m,k", JOINT)
def test_joint_open_parity(sb, big, m, k):
    """parity with DerefsEvalProof.prove (the CPU model of test_pc_model.py is pinned to it), blinds of the joint commitment when k is odd"""
    c, ell = shape(m, k)
    Z = [table("jopen-%d-%d-%d" % (m, k, j), 1 << m) for j in range(k)]
    r = point("jopen-%d-%d" % (m, k), m)
    polys = [sb.DensePolynomial(z) for z in Z]
    g = big.view(ell)
    stape, otape = tapes(sb, 400 + 70 * m + k)
    if k % 2:
        comm, blinds = sb.poly_commit(polys, g, stape)
        pr.poly_commit(sk.merge(Z), ogens(ell), otape)
    else:
        comm, blinds = sb.poly_commit(polys, g)[0], None
    ot, st = transcripts(sb)
    st.append_message(b"protocol-name", b"Derefs evaluation proof")
    sb.api.prof_enable(True)
    proof, evals = sb.PolyEvalProof.prove_joint(polys, blinds, oc.to_arr(r), g, st, stape)
    n = launches(sb)
    sb.api.prof_enable(False)
    want, want_evals = oracle_joint_prove(Z, r, ints(blinds) if k % 2 else None, ell, ot, otape)
    assert ints(evals) == want_evals
    assert proof.data == pr.ser(want)
    assert same_transcript(ot, st) and same_tape(otape, stape)
    assert n["bound_rows_many"] == (1 if rows_in_tables(m, c) else 0) and n["msm_rows_tables"] == 0, n
    for p, z in zip(polys, Z):
        assert np.array_equal(p.to_numpy(), z)
    # the oracle's verifier accepts the proof against the commitment (blinded or not)
    ot2 = oc.Transcript(LABEL)
    ot2.append_message(b"app", b"prefix")
    sk.DerefsEvalProof(pr.deser(pr.PolyEvalProof, proof.data)[0]).verify(r, want_evals, [], ogens(ell), pr.PolyCommitment(comm.C), ot2)


# ---------------------------------------------------------------------------------------------------- verifiers
def oracle_rejects(fn):
    try:
        fn()
    except Exception:
        return True
    return False


def test_verifiers_accept_oracle_proofs_and_reject_mutants(sb, big):
    ell = 8
    Z = table("verify", 1 << ell)
    r = point("verify", ell)
    g, og = big.view(ell), ogens(ell)
    comm, _ = pr.poly_commit(Z, og, None)
    scomm = sb.PolyCommitment(comm.C)
    Zr = oc.evaluate(Z, r)
    ot, _ = transcripts(sb)
    proof, C_Zr = pr.PolyEvalProof.prove(Z, None, r, Zr, None, og, ot, oc.RandomTape(b"proof", 5))
    data = pr.ser(proof)

    def lib_verify(data, r, Zr=None, C=None, comm=scomm):
        st = sb.Transcript(LABEL)
        st.append_message(b"app", b"prefix")
        p = sb.PolyEvalProof(data)
        if Zr is not None:
            p.verify_plain(g, st, oc.to_arr(r), oc.to_arr([Zr])[0], comm)
        else:
            p.verify(g, st, oc.to_arr(r), C, comm)
        return st

    def ora_verify(data, r, Zr=None, C=None, comm=comm):
        ot = oc.Transcript(LABEL)
        ot.append_message(b"app", b"prefix")
        p = pr.deser(pr.PolyEvalProof, data)[0]
        if Zr is not None:
            p.verify_plain(og, ot, r, Zr, comm)
        else:
            p.verify(og, ot, r, C, comm)
        return ot

    ot, st = ora_verify(data, r, Zr=Zr), lib_verify(data, r, Zr=Zr)
    assert same_transcript(ot, st)
    ot, st = ora_verify(data, r, C=C_Zr), lib_verify(data, r, C=C_Zr)
    assert same_transcript(ot, st)
    row_swapped = pr.PolyCommitment([comm.C[1]] + comm.C[1:])
    not_a_point = pr.PolyCommitment([b"\xff" * 32] + comm.C[1:])
    mutants = [
        ("changed Zr", dict(data=data, r=r, Zr=(Zr + 1) % Q)),
        ("changed row", dict(data=data, r=r, Zr=Zr, comm=row_swapped)),
        ("row not a point", dict(data=data, r=r, Zr=Zr, comm=not_a_point)),
        ("wrong r", dict(data=data, r=[(x + 1) % Q for x in r], Zr=Zr)),
        ("truncated", dict(data=data[:-1], r=r, Zr=Zr)),
    ]
    codes = {}
    for name, kw in mutants:
        assert oracle_rejects(lambda: ora_verify(**kw)), name
        kw_lib = dict(kw)
        if "comm" in kw_lib:
            kw_lib["comm"] = sb.PolyCommitment(kw_lib["comm"].C)
        with pytest.raises(sb.ProofVerifyError) as e:
            lib_verify(**kw_lib)
        codes[name] = e.value.code
    assert codes == {"changed Zr": 9, "changed row": 9, "row not a point": 10, "wrong r": 9, "truncated": 9}, codes
    # the joint verifier on the oracle's DerefsEvalProof, and a changed evaluation
    k, m = 3, 6
    Zs = [table("vjoint-%d" % j, 1 << m) for j in range(k)]
    rj = point("vjoint", m)
    c, ellj = shape(m, k)
    jc, _ = pr.poly_commit(sk.merge(Zs), ogens(ellj), None)
    evals = [oc.evaluate(z, rj) for z in Zs]
    ot = oc.Transcript(LABEL)
    jp = sk.DerefsEvalProof.prove(type("M", (), {"comb": sk.merge(Zs)}), evals, [], rj, ogens(ellj), ot, oc.RandomTape(b"proof", 6)).proof_derefs
    for ev, ok in [(evals, True), ([evals[0], (evals[1] + 1) % Q, evals[2]], False)]:
        st = sb.Transcript(LABEL)
        st.append_message(b"protocol-name", b"Derefs evaluation proof")
        p = sb.PolyEvalProof(pr.ser(jp))
        if ok:
            p.verify_joint(big.view(ellj), st, oc.to_arr(rj), oc.to_arr(ev), sb.PolyCommitment(jc.C))
        else:
            with pytest.raises(sb.ProofVerifyError):
                p.verify_joint(big.view(ellj), st, oc.to_arr(rj), oc.to_arr(ev), sb.PolyCommitment(jc.C))


# ---------------------------------------------------------------------------------------------------- a sumcheck and its openings on one transcript
def test_commit_sumcheck_open_one_transcript(sb, big):
    m, k = 10, 3
    Z = [table("comp-%d" % j, 1 << m) for j in range(k)]
    c, ell = shape(m, k)
    g = big.view(ell)
    polys = [sb.DensePolynomial(z) for z in Z]
    stape = sb.RandomTape(sb.tape_seed(77))
    st = sb.Transcript(LABEL)
    comm, blinds = sb.poly_commit(polys, g, stape)
    comm.append_to_transcript(b"tables", st)
    claim = sum(a * b % Q * cc for a, b, cc in zip(*[oc.to_ints(z) for z in Z])) % Q
    work = [sb.DensePolynomial(z) for z in Z]   # the sumcheck binds its tables in place
    comp = sb.Composition([(oc.to_arr([1])[0], (0, 1, 2))])
    sc_proof, r, finals, e = sb.sumcheck_prove(work, comp, oc.to_arr([claim])[0], m, st)
    st.append_message(b"protocol-name", b"Derefs evaluation proof")
    proof, evals = sb.PolyEvalProof.prove_joint(polys, blinds, r, g, st, stape)
    assert np.array_equal(evals, finals)
    # the oracle replays the whole transcript and accepts both proofs
    ot = oc.Transcript(LABEL)
    pr.PolyCommitment(comm.C).append_to_transcript(b"tables", ot)
    e_o, r_o = pr.deser(pr.SumcheckInstanceProof, sc_proof)[0].verify(claim, m, 3, ot)
    fin = ints(finals)
    assert list(r_o) == ints(r) and e_o == fin[0] * fin[1] % Q * fin[2] % Q
    ot.append_protocol_name(b"Derefs evaluation proof")
    ev = fin + [0] * (oc.next_pow2(k) - k)
    ot.append_scalars(b"evals_ops_val", ev)
    ch = ot.challenge_vector(b"challenge_combine_n_to_one", c)
    for i in reversed(range(c)):
        ev = oc.bound_bot_ints(ev, ch[i])
    ot.append_scalar(b"joint_claim_eval", ev[0])
    # blinded commitment: verify against C_Zr = joint * G_1 (verify_plain), as the reference's DerefsEvalProof::verify does
    pr.deser(pr.PolyEvalProof, proof.data)[0].verify_plain(ogens(ell), ot, ch + list(r_o), ev[0], pr.PolyCommitment(comm.C))
    assert same_transcript(ot, st)


# ---------------------------------------------------------------------------------------------------- views
def test_view_proves_as_private_gens_and_holds_no_memory(sb, big):
    ell = 12
    Z = table("view", 1 << ell)
    r = oc.to_arr(point("view", ell))
    poly = sb.DensePolynomial(Z)
    before = sb.device_bytes_live()
    v = big.view(ell)
    assert sb.device_bytes_live() == before
    own = sb.PolyCommitmentGens(ell, LABEL)
    outs = []
    for g in (v, own):
        stape = sb.RandomTape(sb.tape_seed(9))
        comm, blinds = sb.poly_commit(poly, g, stape)
        proof, C_Zr, _ = sb.PolyEvalProof.prove(poly, blinds, r, None, None, g, sb.Transcript(LABEL), stape)
        outs.append((comm.C, proof.data, C_Zr))
    assert outs[0] == outs[1]
    with pytest.raises(sb.SpartanB200Error):
        own.view(ell + 1)


# ---------------------------------------------------------------------------------------------------- refusals leave everything as it was
def test_refusals_leave_inputs_alone(sb, big):
    import ctypes as C
    m = 6
    Z = [table("refuse-%d" % j, 1 << m) for j in range(3)]
    polys = [sb.DensePolynomial(z) for z in Z]
    short = sb.DensePolynomial(table("refuse-short", 1 << (m - 1)))
    other_ctx = sb.Context(0)
    foreign = sb.DensePolynomial(Z[0], ctx=other_ctx)
    g = big.view(m + 2)
    r = oc.to_arr(point("refuse", m))
    bad = np.array([2 ** 64 - 1] * 4, dtype=np.uint64)   # limbs >= q
    st, stape = sb.Transcript(LABEL), sb.RandomTape(sb.tape_seed(3))
    st0, tape0 = st.state.raw, stape.state.raw

    def refused(fn, exc, what):
        with pytest.raises(exc) as e:
            fn()
        assert what in str(e.value), str(e.value)
        assert st.state.raw == st0 and stape.state.raw == tape0
        for p, z in zip(polys, Z):
            assert np.array_equal(p.to_numpy(), z)

    refused(lambda: sb.poly_commit(polys, big.view(m), stape), sb.SpartanB200Error, "needs n = R")
    refused(lambda: sb.poly_commit(polys[:2] + [short], g, stape), sb.SpartanB200Error, "differ in length")
    refused(lambda: sb.poly_commit([], g, stape), sb.SpartanB200Error, "0 tables; 1 .. SP_PC_MAX_TABLES = 64")
    refused(lambda: sb.poly_commit((polys * 22)[:65], g, stape), sb.SpartanB200Error, "65 tables; 1 .. SP_PC_MAX_TABLES = 64")
    refused(lambda: sb.poly_commit(polys[:2] + [foreign], g, stape), sb.SpartanB200Error, "another context")
    refused(lambda: sb.PolyEvalProof.prove_joint(polys, None, np.vstack([r[:-1], bad]), g, st, stape), sb.R1CSError, "not reduced")
    refused(lambda: sb.PolyEvalProof.prove_joint(polys, np.tile(bad, (1 << ((m + 2) // 2), 1)), r, g, st, stape), sb.R1CSError, "not reduced")
    refused(lambda: sb.PolyEvalProof.prove(polys[0], None, r, bad, None, big.view(m), st, stape), sb.R1CSError, "not reduced")
    refused(lambda: sb.PolyEvalProof.prove(polys[0], None, r, None, bad, big.view(m), st, stape), sb.R1CSError, "not reduced")
    refused(lambda: sb.PolyEvalProof.prove(polys[0], None, r[:-1], None, None, big.view(m), st, stape), sb.SpartanB200Error, "|r|")
    refused(lambda: sb.PolyEvalProof.prove_joint(polys, None, r, big.view(m), st, stape), sb.SpartanB200Error, "needs n = R")
    refused(lambda: sb.PolyEvalProof.prove_joint(polys[:2] + [foreign], None, r, g, st, stape), sb.SpartanB200Error, "another context")
    # the status codes themselves, through the C ABI
    ctx = sb.default_context()
    out, n = C.POINTER(C.c_ubyte)(), C.c_size_t()
    arr = (C.c_void_p * 1)(polys[0].h)
    assert sb.lib.sp_pc_commit(ctx.h, g.h, arr, C.c_int(0), None, C.byref(out), C.byref(n), None) == 3
    assert sb.lib.sp_pc_commit(ctx.h, g.h, arr, C.c_int(65), None, C.byref(out), C.byref(n), None) == 3
    zr, c_zr = np.zeros(4, dtype=np.uint64), C.create_string_buffer(32)
    assert sb.lib.sp_pc_eval_prove_t(ctx.h, big.view(m).h, polys[0].h, None, bad.ctypes.data_as(C.c_void_p), C.c_size_t(m), None,
                                     None, st.state, stape.state, C.byref(out), C.byref(n), c_zr, zr.ctypes.data_as(C.c_void_p)) in (3, 5)
    assert st.state.raw == st0 and stape.state.raw == tape0
    del foreign, other_ctx


# ---------------------------------------------------------------------------------------------------- the parity cases under the memory-check mode
def test_parity_cases_under_memcheck(tmp_path):
    if os.environ.get("SP_MEMCHECK_OUT"):
        pytest.skip("already running under the memory-check mode")
    out = tmp_path / "memcheck.json"
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "tests"), ROOT] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    env["SP_MEMCHECK_OUT"] = str(out)
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "memcheck_plugin", "-p", "no:cacheprovider", "-k", "parity and not memcheck",
           os.path.join(ROOT, "tests", "test_gpu_poly_commit.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-20000:]
    tot = json.load(open(out))
    assert tot["violations"] == 0, tot
    assert tot["blocks_filled"] > 0 and tot["context_refills"] > 0, tot
