"""A CPU model of the zero-knowledge sumcheck of a caller-defined polynomial (include/spartan_b200.h: sp_zk_sumcheck_prove_t): the oracle's
ZKSumcheckInstanceProof._prove (prove_quad / prove_cubic_with_additive_term) with its evaluation loop replaced by the round evaluations of any
sum of products, as test_sumcheck_poly_model.py computes them.  At A*B and A*B*C - A*D it is pinned byte for byte to the oracle's two provers;
at every other degree the oracle's generic verify must accept its proofs.  test_gpu_zk_sumcheck.py checks the GPU against it."""
import zlib

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from test_gpu_sumcheck_poly import from_evals, g_at  # noqa: E402
from test_sumcheck_poly_model import _distinct, as_table, comb_sum, hypercube_sum, mixed_composition, rand_ints, special_compositions  # noqa: E402

Q = oc.Q
LABEL_1, LABEL_N = b"zk-model-gens-1", b"zk-model-gens-n"


def zk_model_prove(tables, terms, claim, blind_claim, num_rounds, gens_1, gens_n, T, tape):
    """ZKSumcheckInstanceProof._prove with comb_func = sum_t c_t prod_{f in factors_t} tables[f] (a table object passed twice is one table,
    bound once).  Returns (proof, r, finals = tables[i][0] after the last bind for every index i, blind of the last comm_eval).  The caller's
    arrays are not changed."""
    seen, slot = _distinct([as_table(t) for t in tables])
    P = [np.array(t, copy=True) for t in seen]
    sterms = [(c % Q, tuple(slot[f] for f in fs)) for c, fs in terms]
    used = {f for _, fs in sterms for f in fs}
    d = max(len(fs) for _, fs in terms)
    assert gens_1.n == 1 and gens_n.n == d + 1
    blinds_poly = tape.random_vector(b"blinds_poly", num_rounds)
    blinds_evals = tape.random_vector(b"blinds_evals", num_rounds)
    claim_per_round = claim % Q
    comm_claim_per_round = oc.commit_scalar(claim_per_round, blind_claim, gens_1).compress()
    r, comm_polys, comm_evals, proofs = [], [], [], []
    for j in range(num_rounds):
        half = len(P[0]) // 2
        zero = oc.zeros(half)
        ev = []
        for t in [0] + list(range(2, d + 1)):
            x = [None if k not in used else p[:half] if t == 0 else oc.lincomb3(p[:half], p[half:], zero, (1 - t) % Q, t, 0)
                 for k, p in enumerate(P)]
            ev.append(comb_sum(x, sterms))
        poly = from_evals([ev[0], (claim_per_round - ev[0]) % Q] + ev[1:])
        comm_poly = oc.commit_vec(poly.coeffs, blinds_poly[j], gens_n).compress()
        T.append_point(b"comm_poly", comm_poly)
        comm_polys.append(comm_poly)
        r_j = T.challenge_scalar(b"challenge_nextround")
        P = [oc.bound_top(p, r_j) for p in P]
        e = poly.evaluate(r_j)
        comm_eval = oc.commit_scalar(e, blinds_evals[j], gens_1).compress()
        T.append_point(b"comm_claim_per_round", comm_claim_per_round)
        T.append_point(b"comm_eval", comm_eval)
        w = T.challenge_vector(b"combine_two_claims_to_one", 2)
        target = (w[0] * claim_per_round + w[1] * e) % Q
        blind_sc = blind_claim if j == 0 else blinds_evals[j - 1]
        blind = (w[0] * blind_sc + w[1] * blinds_evals[j]) % Q
        a = [(w[0] * (2 if k == 0 else 1) + w[1] * pow(r_j, k, Q)) % Q for k in range(d + 1)]
        proof, _, _ = pr.DotProductProof.prove(gens_1, gens_n, T, tape, poly.coeffs, blinds_poly[j], a, target, blind)
        proofs.append(proof)
        claim_per_round, comm_claim_per_round = e, comm_eval
        r.append(r_j)
        comm_evals.append(comm_eval)
    finals = [oc.arr_get(P[s], 0) for s in slot]
    return pr.ZKSumcheckInstanceProof(comm_polys, comm_evals, proofs), r, finals, blinds_evals[num_rounds - 1]


_GENS = {}


def gens(n, label):
    if (n, label) not in _GENS:
        _GENS[(n, label)] = oc.MultiCommitGens.new(n, label)
    return _GENS[(n, label)]


def states(tag, seed):
    """a transcript with a prefix and a seeded tape, twice"""
    out = []
    for _ in range(2):
        T = oc.Transcript(b"zk-model")
        T.append_message(b"app", tag)
        out.append((T, oc.RandomTape(b"proof", seed)))
    return out


def same_states(a, b):
    return all(x.challenge_bytes(b"after", 32) == y.challenge_bytes(b"after", 32) for x, y in ((a[0], b[0]), (a[1].tape, b[1].tape)))


# ---------------------------------------------------------------------------------------------------- the model is the oracle at A*B and A*B*C - A*D
@pytest.mark.parametrize("n", [1, 2, 5, 9])
def test_model_equals_prove_quad(n):
    rng = np.random.default_rng(n)
    A, B = (oc.prg_scalars("zkm-quad-%d-%d" % (n, j), 1 << n) for j in range(2))
    claim, blind = rand_ints(rng, 2)
    g1, g3 = gens(1, LABEL_1), gens(3, LABEL_N)
    s1, s2 = states(b"quad", 11 + n)
    want = pr.ZKSumcheckInstanceProof.prove_quad(claim, blind, n, A.copy(), B.copy(), g1, g3, *s1)
    got = zk_model_prove([A, B], [(1, (0, 1))], claim, blind, n, g1, g3, *s2)
    assert pr.ser(got[0]) == pr.ser(want[0])
    assert got[1:] == want[1:]
    assert same_states(s1, s2)


@pytest.mark.parametrize("n", [1, 2, 5, 9])
def test_model_equals_prove_cubic_with_additive_term(n):
    rng = np.random.default_rng(100 + n)
    A, B, Cc, D = (oc.prg_scalars("zkm-cubic-%d-%d" % (n, j), 1 << n) for j in range(4))
    claim, blind = rand_ints(rng, 2)
    g1, g4 = gens(1, LABEL_1), gens(4, LABEL_N)
    s1, s2 = states(b"cubic", 21 + n)
    want = pr.ZKSumcheckInstanceProof.prove_cubic_with_additive_term(claim, blind, n, A.copy(), B.copy(), Cc.copy(), D.copy(), g1, g4, *s1)
    got = zk_model_prove([A, B, Cc, D], [(1, (0, 1, 2)), (Q - 1, (0, 3))], claim, blind, n, g1, g4, *s2)
    assert pr.ser(got[0]) == pr.ser(want[0])
    assert got[1:] == want[1:]
    assert same_states(s1, s2)


# ---------------------------------------------------------------------------------------------------- other degrees: the oracle's verify accepts
def _prove_and_verify(tables, terms, num_rounds, tag, honest=True):
    d = max(len(fs) for _, fs in terms)
    rng = np.random.default_rng(zlib.crc32(tag))
    claim = hypercube_sum(tables, terms) if honest else rand_ints(rng, 1)[0]
    blind = rand_ints(rng, 1)[0]
    g1, gn = gens(1, LABEL_1), gens(d + 1, LABEL_N)
    (T, tape), (Tv, _) = states(tag, 7)
    proof, r, finals, blind_post = zk_model_prove(tables, terms, claim, blind, num_rounds, g1, gn, T, tape)
    proof = pr.deser(pr.ZKSumcheckInstanceProof, pr.ser(proof))[0]   # through the wire format
    comm_claim = oc.commit_scalar(claim, blind, g1).compress()
    comm_eval, vr = proof.verify(comm_claim, num_rounds, d, g1, gn, Tv)
    assert vr == r
    assert T.challenge_bytes(b"after", 32) == Tv.challenge_bytes(b"after", 32)
    if honest and num_rounds == oc.log_2(len(as_table(tables[0]))):
        assert comm_eval == oc.commit_scalar(g_at(terms, finals), blind_post, g1).compress()
    return proof, finals


@pytest.mark.parametrize("n", [1, 3, 6])
@pytest.mark.parametrize("D", [1, 2, 3, 4, 5, 6])
def test_oracle_verify_accepts_every_degree(D, n):
    rng = np.random.default_rng(10 * D + n)
    k, terms = mixed_composition(D, rng)
    tables = [oc.prg_scalars("zkm-deg-%d-%d-%d" % (D, n, j), 1 << n) for j in range(k)]
    proof, _ = _prove_and_verify(tables, terms, n, b"degree%d-%d" % (D, n))
    assert all(len(p.z) == D + 1 for p in proof.proofs)


@pytest.mark.parametrize("name", ["repeated_table", "unused_table", "cancelling_terms", "all_terms_cancel"])
def test_oracle_verify_accepts_special_compositions(name):
    n = 5
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    idx, terms = special_compositions(rng)[name]
    distinct = [oc.prg_scalars("zkm-%s-%d" % (name, j), 1 << n) for j in range(max(idx) + 1)]
    _, finals = _prove_and_verify([distinct[i] for i in idx], terms, n, name.encode())
    if name == "repeated_table":
        assert finals[0] == finals[1]


def test_oracle_verify_accepts_edge_tables_and_coefficients():
    """tables of zeros and of q - 1, a zero coefficient and a q - 1 coefficient, degree 6"""
    n = 4
    zeros, qm1 = [0] * (1 << n), [Q - 1] * (1 << n)
    t = oc.prg_scalars("zkm-edge", 1 << n)
    tables = [oc.to_arr(zeros), oc.to_arr(qm1), t]
    terms = [(0, (0, 1, 2)), (Q - 1, (1, 1, 1, 2, 2, 2)), (1, (2,)), (Q - 1, (0, 2))]
    _prove_and_verify(tables, terms, n, b"edge")


@pytest.mark.parametrize("num_rounds", [1, 3])
@pytest.mark.parametrize("D", [1, 4, 6])
def test_oracle_verify_accepts_fewer_rounds_than_variables(D, num_rounds):
    n = 6
    k, terms = mixed_composition(D, np.random.default_rng(D + num_rounds))
    tables = [oc.prg_scalars("zkm-rounds-%d-%d" % (D, j), 1 << n) for j in range(k)]
    _prove_and_verify(tables, terms, num_rounds, b"rounds%d-%d" % (D, num_rounds), honest=False)


def test_oracle_verify_rejects_a_dishonest_claim():
    n = 4
    k, terms = mixed_composition(5, np.random.default_rng(3))
    tables = [oc.prg_scalars("zkm-bad-%d" % j, 1 << n) for j in range(k)]
    g1, gn = gens(1, LABEL_1), gens(6, LABEL_N)
    (T, tape), (Tv, _) = states(b"bad", 9)
    claim = hypercube_sum(tables, terms)
    proof, _, _, _ = zk_model_prove(tables, terms, claim, 5, n, g1, gn, T, tape)
    with pytest.raises(pr.ProofVerifyError):
        proof.verify(oc.commit_scalar(claim + 1, 5, g1).compress(), n, 5, g1, gn, Tv)
