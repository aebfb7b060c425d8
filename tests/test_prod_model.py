"""The host side of the caller's product circuits, on the CPU (the library loads for its host-only entries): sp_prod_verify_t against proofs the
oracle's ProductCircuitEvalProofBatched.prove makes on a transcript with a caller prefix (accepted with the oracle verify's rand, leaf claims and
final transcript state), its rejection of mutants with the transcript where the oracle's verify leaves it, and sp_prod_leaf_eval against the
oracle's evaluation of the materialised leaf vectors."""
import random

import numpy as np
import pytest

import spartan_b200 as sb
from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import spark as sk

Q = oc.Q
LABEL = b"prod-model"


def tables(m, k, tag):
    return [oc.prg_scalars("prod-model-%s-%d-%d" % (tag, m, j), 1 << m) for j in range(k)]


def both_transcripts(products):
    """the oracle's and the library's transcript after the same caller prefix: a message, then the products absorbed"""
    ot, st = oc.Transcript(LABEL), sb.Transcript(LABEL)
    for t in (ot, st):
        t.append_message(b"caller", b"prefix")
    for p in products:
        ot.append_scalar(b"product", p)
        st.append_message(b"product", oc.scalar_to_bytes(p))
    return ot, st


def same_state(ot, st):
    return ot.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64)


def oracle_proof(m, k, tag):
    cs = [sk.ProductCircuit(t) for t in tables(m, k, tag)]
    products = [c.evaluate() for c in cs]
    ot, _ = both_transcripts(products)
    proof, rand = sk.ProductCircuitEvalProofBatched.prove(cs, [], ot)
    return products, proof, rand


@pytest.mark.parametrize("m", [1, 2, 3, 8, 12])
@pytest.mark.parametrize("k", [1, 2, 5, 24])
def test_verify_accepts_oracle_proofs(m, k):
    products, proof, rand = oracle_proof(m, k, "acc")
    ot, st = both_transcripts(products)
    claims_o, dotp_o, rand_o = proof.verify(products, [], 1 << m, ot)
    assert rand_o == rand and dotp_o == []
    r, claims = sb.ProductCircuitEvalProofBatched.verify(pr.ser(proof), oc.to_arr(products), m, st)
    assert oc.to_ints(r) == rand_o
    assert oc.to_ints(claims) == claims_o
    assert same_state(ot, st)


def scalar_sites(proof):
    """(description, setter) for every scalar field of the proof: round polynomial coefficients and the product claims of every layer"""
    sites = []
    for i, layer in enumerate(proof.proof):
        for j, cp in enumerate(layer.proof.compressed_polys):
            for c in range(len(cp.coeffs_except_linear_term)):
                sites.append(("layer %d round %d coeff %d" % (i, j, c), cp.coeffs_except_linear_term, c))
        for name in ("claims_prod_left", "claims_prod_right"):
            v = getattr(layer, name)
            for c in range(len(v)):
                sites.append(("layer %d %s[%d]" % (i, name, c), v, c))
    return sites


def check_rejected(proof_bytes, products, m, oracle_run):
    """the library rejects; its transcript then equals the oracle verify's after its assertion (oracle_run: the oracle's verify on its transcript)"""
    ot, st = both_transcripts(products)
    with pytest.raises((pr.ProofVerifyError, AssertionError)):
        oracle_run(ot)
    with pytest.raises(sb.ProofVerifyError) as e:
        sb.ProductCircuitEvalProofBatched.verify(proof_bytes, oc.to_arr(products), m, st)
    assert e.value.code == 9
    assert same_state(ot, st), str(e.value)
    return str(e.value)


@pytest.mark.parametrize("m,k", [(1, 2), (3, 2), (4, 3)])
def test_verify_rejects_every_scalar_mutant(m, k):
    products, proof, _ = oracle_proof(m, k, "mut")
    sites = scalar_sites(proof)
    assert sites
    for what, vec, idx in sites:
        old = vec[idx]
        vec[idx] = (old + 1) % Q
        msg = check_rejected(pr.ser(proof), products, m, lambda t: proof.verify(products, [], 1 << m, t))
        vec[idx] = old
        assert "product circuit layer" in msg, (what, msg)


def test_verify_rejects_wrong_product_depth_truncation_and_dotp_claims():
    m, k = 4, 3
    products, proof, _ = oracle_proof(m, k, "shape")
    good = pr.ser(proof)
    # a wrong product: the first layer's check fails
    bad = list(products)
    bad[1] = (bad[1] + 1) % Q
    assert "layer 0" in check_rejected(good, bad, m, lambda t: proof.verify(bad, [], 1 << m, t))
    # a wrong m, either way: the depth check, before the transcript is touched
    for mm in (m - 1, m + 1):
        assert "depth" in check_rejected(good, products, mm, lambda t: proof.verify(products, [], 1 << mm, t))
    # truncated bytes (and one byte too many) do not decode: the transcript stays as it was
    for cut in (good[:-1], good[:len(good) // 2], good[:7], good + b"\x00"):
        ot, st = both_transcripts(products)
        with pytest.raises(sb.ProofVerifyError):
            sb.ProductCircuitEvalProofBatched.verify(cut, oc.to_arr(products), m, st)
        assert same_state(ot, st)
    # non-empty dotp claims: refused at the last layer, where the reference reads a coefficient it never drew (it panics after absorbing the
    # first triple, so the transcripts are not compared here)
    proof.claims_dotp = ([1], [2], [3])
    st = both_transcripts(products)[1]
    with pytest.raises(sb.ProofVerifyError) as e:
        sb.ProductCircuitEvalProofBatched.verify(pr.ser(proof), oc.to_arr(products), m, st)
    assert "dotp" in str(e.value)
    with pytest.raises((IndexError, AssertionError, pr.ProofVerifyError)):
        proof.verify(products, [], 1 << m, both_transcripts(products)[0])


def test_verify_refusals_leave_the_transcript():
    products, proof, _ = oracle_proof(3, 2, "refuse")
    data = pr.ser(proof)
    arr = oc.to_arr(products)
    for args, what in [((arr, 0), "m = 0"), ((arr, 61), "m = 61"), ((np.zeros((0, 4), dtype=np.uint64), 3), "0 products"),
                       ((np.vstack([arr] * 13)[:25], 3), "25 products")]:
        ot, st = both_transcripts(products)
        with pytest.raises(sb.SpartanB200Error) as e:
            sb.ProductCircuitEvalProofBatched.verify(data, args[0], args[1], st)
        assert what in str(e.value) and not isinstance(e.value, sb.ProofVerifyError)
        assert same_state(ot, st)
    ot, st = both_transcripts(products)
    with pytest.raises(sb.R1CSError):
        sb.ProductCircuitEvalProofBatched.verify(data, np.vstack([arr[:1], np.full((1, 4), 2 ** 64 - 1, dtype=np.uint64)]), 3, st)
    assert same_state(ot, st)


# ---------------------------------------------------------------------------------------------------- leaf polynomials at rand
def random_leaves(rng, ntables, k):
    """descriptors of every kind: plain tables, fingerprints, index-only, constant-only, repeated sources, zero sources"""
    kinds = ["plain", "hash", "index", "const", "repeat", "empty", "mixed"]
    out = []
    for c in range(k):
        kind = kinds[c % len(kinds)]
        rs = lambda: rng.randrange(Q)
        if kind == "plain":
            out.append(([(rng.randrange(ntables), 1)], 0, 0))
        elif kind == "hash":
            r, g = rs(), rs()
            out.append(([(rng.randrange(ntables), r * r % Q), (rng.randrange(ntables), r), (rng.randrange(ntables), 1)], 0, (Q - g) % Q))
        elif kind == "index":
            out.append(([], rs(), 0))
        elif kind == "const":
            out.append(([], 0, rs()))
        elif kind == "repeat":
            t = rng.randrange(ntables)
            out.append(([(t, rs()), (t, rs()), (t, 1)], 1, rs()))
        elif kind == "empty":
            out.append(([], 0, 0))
        else:
            out.append(([(rng.randrange(ntables), rs())], rs(), rs()))
    return out


def materialise(desc, T, m):
    sources, idx, cst = desc
    vals = [oc.to_ints(t) for t in T]
    return [(cst + idx * x + sum(c * vals[s][x] for s, c in sources)) % Q for x in range(1 << m)]


@pytest.mark.parametrize("m", [1, 2, 5, 9])
def test_leaf_eval_matches_materialised_leaves(m):
    rng = random.Random(1000 + m)
    ntables = 4
    T = tables(m, ntables, "leaf")
    rand = oc.to_ints(oc.prg_scalars("prod-model-rand-%d" % m, m))
    table_evals = [oc.evaluate(t, rand) for t in T]
    descs = random_leaves(rng, ntables, 14)
    leaves = [sb.ProductLeaves(s, index_coeff=i, const=c) for s, i, c in descs]
    got = sb.product_leaf_eval(leaves, oc.to_arr(table_evals), oc.to_arr(rand))
    want = [oc.evaluate(oc.to_arr(materialise(d, T, m)), rand) for d in descs]
    assert oc.to_ints(got) == want
    # leaves None: circuit i is table i
    assert oc.to_ints(sb.product_leaf_eval(None, oc.to_arr(table_evals), oc.to_arr(rand))) == table_evals


def test_leaf_eval_refusals():
    ev, r = oc.to_arr([1, 2]), oc.to_arr([3, 4])
    cases = [
        ([sb.ProductLeaves([(2, 1)])], "table 2 >= ntables = 2"),
        ([sb.ProductLeaves([(0, 1)] * 4)], "4 sources; at most SP_PROD_MAX_SOURCES = 3"),
        ([], "0 circuits; 1 .. SP_PROD_MAX_CIRCUITS = 24"),
        ([sb.ProductLeaves([(0, 1)])] * 25, "25 circuits; 1 .. SP_PROD_MAX_CIRCUITS = 24"),
    ]
    for leaves, what in cases:
        with pytest.raises(sb.SpartanB200Error) as e:
            sb.product_leaf_eval(leaves, ev, r)
        assert what in str(e.value), str(e.value)
    bad = np.full(4, 2 ** 64 - 1, dtype=np.uint64)
    with pytest.raises(sb.R1CSError):
        sb.product_leaf_eval([sb.ProductLeaves([(0, bad)])], ev, r)
    with pytest.raises(sb.R1CSError):
        sb.product_leaf_eval([sb.ProductLeaves([], const=bad)], ev, r)
