"""The host side of the caller's dot products beside their product circuits, on the CPU (the library loads for its host-only entries):
sp_prod_verify_dotp_t against proofs the oracle's ProductCircuitEvalProofBatched.prove(circuits, split dot products, T) makes after a caller
prefix (accepted with the oracle verify's rand, leaf claims, dotp claims and final transcript state), its rejection of a mutant of every dotp
claim and of every passed half sum with the transcript where the oracle's verify leaves it, its refusals, which leave the transcript alone, and
sp_prod_leaf_eval on the operand forms against the oracle's materialised operands at rand."""
import random

import numpy as np
import pytest

import spartan_b200 as sb
from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import spark as sk

Q = oc.Q
LABEL = b"prod-dotp-model"
NTABLES = 4
KKD = [(1, 1), (3, 2), (22, 1), (2, 11)]


def tables(m, tag):
    return [oc.prg_scalars("prod-dotp-model-%s-%d-%d" % (tag, m, j), 1 << m) for j in range(NTABLES)]


def materialise(desc, T, m):
    sources, idx, cst = desc
    vals = [oc.to_ints(t) for t in T]
    return oc.to_arr([(cst + idx * x + sum(c * vals[s][x] for s, c in sources)) % Q for x in range(1 << m)])


def operand_descs(rng, kd):
    """(left, right, weight) of each dot product, cycling over the operand kinds: a plain table, a three-source form, an index term, a constant
    weight of one, and one table read by several operands"""
    rs = lambda: rng.randrange(Q)
    kinds = [
        lambda: (([(0, 1)], 0, 0), ([(1, rs()), (2, rs()), (3, 1)], 0, rs()), ([], 0, 1)),
        lambda: (([], 1, 0), ([(2, 1)], 0, 0), ([(1, 1)], 0, 0)),
        lambda: (([(3, rs())], rs(), 0), ([(3, 1)], 0, rs()), ([(3, 1), (0, rs())], 0, 0)),
        lambda: (([(1, 1)], 0, 0), ([(0, 1)], 0, 0), ([], rs(), rs())),
    ]
    return [kinds[d % len(kinds)]() for d in range(kd)]


def leaf_descs(k):
    return [([(c % NTABLES, 1)], 0, 0) for c in range(k)]


def forms(descs):
    return [sb.ProductLeaves(s, index_coeff=i, const=c) for s, i, c in descs]


def both_transcripts(products, halves):
    """the oracle's and the library's transcript after the same caller prefix: a message, then the products and the half sums absorbed"""
    ot, st = oc.Transcript(LABEL), sb.Transcript(LABEL)
    for t in (ot, st):
        t.append_message(b"caller", b"prefix")
    for p in list(products) + list(halves):
        ot.append_scalar(b"claim", p)
        st.append_message(b"claim", oc.scalar_to_bytes(p))
    return ot, st


def same_state(ot, st):
    return ot.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64)


def oracle_case(m, k, kd, tag):
    """tables, descriptors, products, half sums, and the oracle's proof and rand"""
    T = tables(m, tag)
    ld, dd = leaf_descs(k), operand_descs(random.Random("%s-%d-%d-%d" % (tag, m, k, kd)), kd)
    cs = [sk.ProductCircuit(materialise(d, T, m)) for d in ld]
    dps = []
    for ops in dd:
        dps.extend(sk.DotProductCircuit(*[materialise(o, T, m) for o in ops]).split())
    products, halves = [c.evaluate() for c in cs], [d.evaluate() for d in dps]
    ot, _ = both_transcripts(products, halves)
    proof, rand = sk.ProductCircuitEvalProofBatched.prove(cs, dps, ot)
    return T, ld, dd, products, halves, proof, rand


def lib_verify(data, products, halves, m, st):
    return sb.ProductCircuitEvalProofBatched.verify_dotp(data, oc.to_arr(products), oc.to_arr(halves).reshape(-1, 2, 4), m, st)


@pytest.mark.parametrize("k,kd", KKD)
@pytest.mark.parametrize("m", [1, 2, 3, 8])
def test_verify_accepts_oracle_proofs(m, k, kd):
    T, _, dd, products, halves, proof, rand = oracle_case(m, k, kd, "acc")
    ot, st = both_transcripts(products, halves)
    claims_o, dotp_o, rand_o = proof.verify(products, halves, 1 << m, ot)
    assert rand_o == rand and len(dotp_o) == 3 * kd
    r, claims, dotp = lib_verify(pr.ser(proof), products, halves, m, st)
    assert oc.to_ints(r) == rand_o
    assert oc.to_ints(claims) == claims_o
    assert dotp.shape == (kd, 3, 4) and oc.to_ints(dotp.reshape(-1, 4)) == dotp_o
    assert same_state(ot, st)
    # the verifier's side of the operands: each form at rand from the tables' values there is the operand's evaluation, and the claim
    tev = oc.to_arr([oc.evaluate(t, rand_o) for t in T])
    for d, ops in enumerate(dd):
        got = oc.to_ints(sb.product_leaf_eval(forms(ops), tev, r))
        assert got == [oc.evaluate(materialise(o, T, m), rand_o) for o in ops]
        assert got == dotp_o[3 * d:3 * d + 3]


def check_rejected(data, products, halves, m, oracle_run):
    """the library rejects; its transcript then equals the oracle verify's after its assertion"""
    ot, st = both_transcripts(products, halves)
    with pytest.raises((pr.ProofVerifyError, AssertionError)):
        oracle_run(ot)
    with pytest.raises(sb.ProofVerifyError) as e:
        lib_verify(data, products, halves, m, st)
    assert e.value.code == 9
    assert same_state(ot, st), str(e.value)
    return str(e.value)


@pytest.mark.parametrize("m,k,kd", [(1, 1, 1), (2, 3, 2), (4, 2, 3)])
def test_verify_rejects_every_dotp_mutant(m, k, kd):
    _, _, _, products, halves, proof, _ = oracle_case(m, k, kd, "mut")
    cl, cr, cw = proof.claims_dotp
    sites = [(name, v, i) for name, v in (("left", cl), ("right", cr), ("weight", cw)) for i in range(len(v))]
    assert len(sites) == 3 * 2 * kd
    for what, vec, idx in sites:   # every final dotp claim of the proof
        old = vec[idx]
        vec[idx] = (old + 1) % Q
        msg = check_rejected(pr.ser(proof), products, halves, m, lambda t: proof.verify(products, halves, 1 << m, t))
        vec[idx] = old
        assert "product circuit layer" in msg, (what, msg)
    data = pr.ser(proof)
    for j in range(2 * kd):   # every half sum the verifier is given
        bad = list(halves)
        bad[j] = (bad[j] + 1) % Q
        msg = check_rejected(data, products, bad, m, lambda t: proof.verify(products, bad, 1 << m, t))
        assert "product circuit layer" in msg, (j, msg)


def test_verify_refusals_leave_the_transcript():
    m, k, kd = 3, 2, 2
    _, _, _, products, halves, proof, _ = oracle_case(m, k, kd, "refuse")
    data, P, H = pr.ser(proof), oc.to_arr(products), oc.to_arr(halves).reshape(-1, 2, 4)
    cases = [((P, H, 0), "m = 0"), ((P, H, 61), "m = 61"),
             ((P, np.zeros((0, 2, 4), dtype=np.uint64), m), "0 dot products next to 2 circuits"),
             ((np.vstack([P] * 12)[:23], H[:1], m), "1 dot products next to 23 circuits"),
             ((P, np.vstack([H] * 6)[:12], m), "12 dot products next to 2 circuits")]
    for (p, h, mm), what in cases:
        ot, st = both_transcripts(products, halves)
        with pytest.raises(sb.SpartanB200Error) as e:
            sb.ProductCircuitEvalProofBatched.verify_dotp(data, p, h, mm, st)
        assert what in str(e.value) and not isinstance(e.value, sb.ProofVerifyError), str(e.value)
        assert same_state(ot, st)
    bad = H.copy()
    bad[1, 0] = np.full(4, 2 ** 64 - 1, dtype=np.uint64)   # a half sum not reduced
    ot, st = both_transcripts(products, halves)
    with pytest.raises(sb.R1CSError) as e:
        sb.ProductCircuitEvalProofBatched.verify_dotp(data, P, bad, m, st)
    assert "dotp claim" in str(e.value)
    assert same_state(ot, st)


def test_product_only_verify_still_refuses_dotp_proofs():
    """sp_prod_verify_t keeps its contract: a proof with dotp claims is rejected there"""
    m, k, kd = 3, 2, 1
    _, _, _, products, halves, proof, _ = oracle_case(m, k, kd, "prodonly")
    st = both_transcripts(products, halves)[1]
    with pytest.raises(sb.ProofVerifyError) as e:
        sb.ProductCircuitEvalProofBatched.verify(pr.ser(proof), oc.to_arr(products), m, st)
    assert "dotp" in str(e.value)
