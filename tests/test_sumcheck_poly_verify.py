"""sp_sumcheck_verify_t without a GPU: SumcheckInstanceProof::verify (sumcheck.rs:27-62) on proofs the oracle's prove_cubic_batched makes and on
their mutants, with the oracle's verify as the judge of the verdict, the final claim, the challenges and the transcript left behind."""
import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr

LABEL = b"sumcheck-poly"


def _batched_proof(n, npar, nseq, seed):
    """an oracle prove_cubic_batched proof over n variables, its claim, and the state it was proved from (a transcript with a prefix absorbed)"""
    rng = np.random.default_rng(seed)

    def table():
        return oc.to_arr([int.from_bytes(rng.bytes(32), "little") % oc.Q for _ in range(1 << n)])
    A_par, B_par, C_par = [table() for _ in range(npar)], [table() for _ in range(npar)], table()
    A_seq, B_seq, C_seq = [table() for _ in range(nseq)], [table() for _ in range(nseq)], [table() for _ in range(nseq)]
    coeffs = [int.from_bytes(rng.bytes(32), "little") % oc.Q for _ in range(npar + nseq)]
    claim = sum(c * oc.dot3(a, b, cc) for c, a, b, cc in zip(coeffs, A_par + A_seq, B_par + B_seq, [C_par] * npar + C_seq)) % oc.Q
    T = oc.Transcript(LABEL)
    T.append_message(b"prefix", b"%d" % seed)
    proof, _, _, _ = pr.prove_cubic_batched(claim, n, (A_par, B_par, C_par), (A_seq, B_seq, C_seq), coeffs, T)
    return proof, claim


def _fresh_pair(seed):
    import spartan_b200 as sb
    ot, st = oc.Transcript(LABEL), sb.Transcript(LABEL)
    for t in (ot, st):
        t.append_message(b"prefix", b"%d" % seed)
    return ot, st


def _judge(proof_bytes, claim, num_rounds, degree, seed):
    """oracle verdict vs library verdict on the same bytes and the same starting transcript"""
    import spartan_b200 as sb
    ot, st = _fresh_pair(seed)
    try:
        want = pr.deser(pr.SumcheckInstanceProof, proof_bytes)[0].verify(claim, num_rounds, degree, ot)
    except (AssertionError, IndexError):
        want = None
    try:
        got = sb.sumcheck_verify(proof_bytes, oc.to_arr([claim])[0], num_rounds, degree, st)
    except sb.ProofVerifyError as err:
        assert err.code == sb.api.SP_ERR_VERIFY
        got = None
    assert (got is None) == (want is None), "library %s, oracle %s" % ("rejects" if got is None else "accepts", "rejects" if want is None else "accepts")
    if want is not None:
        e, r = want
        assert oc.to_ints(got[0].reshape(1, 4)) == [e]
        assert oc.to_ints(got[1]) == list(r)
    # the transcript is left where the oracle's verify left it, accepted or not
    assert st.challenge_bytes(b"after", 64) == ot.challenge_bytes(b"after", 64)
    return want


def _replace_polys(proof, polys):
    return pr.ser(pr.SumcheckInstanceProof(polys))


@pytest.mark.parametrize("n,npar,nseq", [(1, 1, 0), (3, 2, 1), (6, 3, 2), (9, 12, 0)])
def test_verify_matches_oracle_on_batched_proofs(n, npar, nseq):
    proof, claim = _batched_proof(n, npar, nseq, seed=n)
    assert _judge(pr.ser(proof), claim, n, 3, n) is not None


@pytest.mark.parametrize("n", [2, 5])
def test_verify_mutants_judged_by_oracle(n):
    proof, claim = _batched_proof(n, 2, 1, seed=100 + n)
    polys = proof.compressed_polys
    honest = _judge(pr.ser(proof), claim, n, 3, 100 + n)
    cases = []
    for j in range(n):   # a changed coefficient: accepted by verify (as by the reference), with another final claim
        for c in range(3):
            mutated = [pr.CompressedUniPoly(list(p.coeffs_except_linear_term)) for p in polys]
            mutated[j].coeffs_except_linear_term[c] = (mutated[j].coeffs_except_linear_term[c] + 1) % oc.Q
            cases.append(("coeff", _replace_polys(proof, mutated), claim, n, 3))
    cases.append(("dropped round", _replace_polys(proof, polys[:-1]), claim, n, 3))
    cases.append(("added round", _replace_polys(proof, polys + [polys[-1]]), claim, n, 3))
    cases.append(("rounds - 1", pr.ser(proof), claim, n - 1, 3))
    cases.append(("rounds + 1", pr.ser(proof), claim, n + 1, 3))
    cases.append(("degree - 1", pr.ser(proof), claim, n, 2))
    cases.append(("degree + 1", pr.ser(proof), claim, n, 4))
    short = [pr.CompressedUniPoly(list(p.coeffs_except_linear_term)) for p in polys]
    short[n // 2].coeffs_except_linear_term.pop()
    cases.append(("a round of degree 2", _replace_polys(proof, short), claim, n, 3))
    cases.append(("wrong claim", pr.ser(proof), (claim + 1) % oc.Q, n, 3))
    cases.append(("truncated", pr.ser(proof)[:-1], claim, n, 3))
    for name, data, cl, rounds, degree in cases:
        if name == "truncated":   # bytes that do not decode: the library rejects, the transcript is untouched
            import spartan_b200 as sb
            ot, st = _fresh_pair(100 + n)
            with pytest.raises(sb.ProofVerifyError):
                sb.sumcheck_verify(data, oc.to_arr([cl])[0], rounds, degree, st)
            assert st.challenge_bytes(b"after", 64) == ot.challenge_bytes(b"after", 64)
            continue
        want = _judge(data, cl, rounds, degree, 100 + n)
        if name in ("coeff", "wrong claim"):
            assert want is not None and want[0] != honest[0], name   # verify passes; the caller's final check e = g(finals) rejects it
        else:
            assert want is None, name


def test_verify_refuses_bad_arguments():
    import spartan_b200 as sb
    proof, claim = _batched_proof(2, 1, 0, seed=7)
    with pytest.raises(sb.SpartanB200Error, match="degree_bound"):
        sb.sumcheck_verify(pr.ser(proof), oc.to_arr([claim])[0], 2, 0, sb.Transcript(LABEL))
    with pytest.raises(sb.SpartanB200Error, match="not reduced"):
        sb.sumcheck_verify(pr.ser(proof), np.frombuffer(oc.Q.to_bytes(32, "little"), dtype=np.uint64), 2, 3, sb.Transcript(LABEL))


def test_new_symbols_are_exported():
    import spartan_b200 as sb
    for s in ["sp_sumcheck_prove_t", "sp_sumcheck_prove", "sp_sumcheck_verify_t"]:
        assert hasattr(sb.lib, s), s
    assert sb.Composition([(oc.to_arr([1])[0], (0, 0, 1)), (oc.to_arr([5])[0], (2,))]).degree == 3
