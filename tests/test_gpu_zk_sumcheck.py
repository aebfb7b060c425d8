"""Zero-knowledge sumchecks of caller-defined polynomials and the sigma protocols on the GPU (sp_zk_sumcheck_*_t, sp_knowledge_* ..
sp_dotproduct_*; ZKSumcheckInstanceProof, KnowledgeProof, EqualityProof, ProductProof, DotProductProof): byte parity with the oracle's
prove_quad / prove_cubic_with_additive_term and with the CPU model of test_zk_sumcheck_model.py at every degree, the transcript and tape states
after each call, both verifiers on every proof and on its mutants, the refusals, the launch count, and the parity cases again under the
memory-check mode."""
import json
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from test_sumcheck_poly_model import hypercube_sum, mixed_composition, rand_ints, special_compositions  # noqa: E402
from test_zk_sumcheck_model import zk_model_prove  # noqa: E402

pytestmark = pytest.mark.gpu
Q = oc.Q
LABEL = b"zk-gpu"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G1_LABEL, GN_LABEL = b"zk-gpu-gens-1", b"zk-gpu-gens-n"


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    sb.default_context()
    return sb


_GENS = {}


def gens(sb, n, label):
    """(library, oracle) MultiCommitGens::new(n, label)"""
    if (n, label) not in _GENS:
        _GENS[(n, label)] = (sb.MultiCommitGens(n, label), oc.MultiCommitGens.new(n, label))
    return _GENS[(n, label)]


def split_gens(sb, n, label):
    """DotProductProofGens::new(n, label) (nizk/mod.rs:414-418): gens_n, gens_1 = MultiCommitGens::new(n + 1, label).split_at(n), on the library
    side as from_points views; returns (lib gens_1, lib gens_n, oracle gens_1, oracle gens_n)"""
    key = ("split", n, label)
    if key not in _GENS:
        full = sb.MultiCommitGens(n + 1, label)
        pts = full.export()
        o = pr.DotProductProofGens(n, label)
        _GENS[key] = (sb.MultiCommitGens.from_points([pts[n], pts[n + 1]]), sb.MultiCommitGens.from_points(pts[:n] + [pts[n + 1]]), o.gens_1, o.gens_n)
    return _GENS[key]


def L(x):
    return oc.to_arr([x % Q])[0]


def ints(a):
    return oc.to_ints(np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4))


class States:
    """the oracle's and the library's transcript (with a prefix) and tape (one seed)"""

    def __init__(self, sb, tag, seed):
        self.ot, self.st = oc.Transcript(LABEL), sb.Transcript(LABEL)
        self.ot.append_message(b"app", tag)
        self.st.append_message(b"app", tag)
        self.otape = oc.RandomTape(b"proof", ints(sb.tape_seed(seed))[0])
        self.stape = sb.RandomTape(sb.tape_seed(seed))

    def raw(self):
        return self.st.state.raw, self.stape.state.raw

    def same(self):
        return (self.ot.challenge_bytes(b"after", 64) == self.st.challenge_bytes(b"after", 64)
                and self.otape.tape.challenge_bytes(b"after", 64) == self.stape.challenge_bytes(b"after", 64))


def verifier_transcripts(sb, tag):
    ot, st = oc.Transcript(LABEL), sb.Transcript(LABEL)
    ot.append_message(b"app", tag)
    st.append_message(b"app", tag)
    return ot, st


def lib_polys(sb, tables):
    """one DensePolynomial per distinct table object, repeated where the list repeats it"""
    made = {}
    return [made.setdefault(id(t), sb.DensePolynomial(t)) for t in tables]


def comp_of(sb, terms):
    return sb.Composition([(L(c), fs) for c, fs in terms])


def lib_prove(sb, tables, terms, claim, blind, num_rounds, g1, gn, S):
    polys = lib_polys(sb, tables)
    proof, r, finals, bp = sb.ZKSumcheckInstanceProof.prove(polys, comp_of(sb, terms), L(claim), L(blind), num_rounds, g1, gn, S.st, S.stape)
    return proof, ints(r), ints(finals), ints(bp)[0], polys


def check_verifiers(sb, proof_bytes, claim, blind, num_rounds, d, lg1, lgn, og1, ogn, tag):
    """on transcripts with the prover's prefix `tag`, the oracle's and the library's verify accept, return the same comm_eval and r, and leave
    the same transcript"""
    comm_claim = oc.commit_scalar(claim, blind, og1).compress()
    ot, st = verifier_transcripts(sb, tag)
    want_eval, want_r = pr.deser(pr.ZKSumcheckInstanceProof, proof_bytes)[0].verify(comm_claim, num_rounds, d, og1, ogn, ot)
    got_eval, got_r = sb.ZKSumcheckInstanceProof(proof_bytes).verify(comm_claim, num_rounds, d, lg1, lgn, st)
    assert got_eval == want_eval and ints(got_r) == list(want_r)
    assert ot.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64)
    return comm_claim


# ---------------------------------------------------------------------------------------------------- parity with the oracle's two provers
@pytest.mark.parametrize("n", [2, 5, 11, 16])
@pytest.mark.parametrize("kind", ["quad", "cubic"])
def test_parity_with_oracle_provers(sb, kind, n):
    rng = np.random.default_rng(zlib.crc32(kind.encode()) + n)
    k, d = (2, 2) if kind == "quad" else (4, 3)
    tables = [oc.prg_scalars("zk-gpu-%s-%d-%d" % (kind, n, j), 1 << n) for j in range(k)]
    claim, blind = rand_ints(rng, 2)
    lg1, og1 = gens(sb, 1, G1_LABEL)
    lgn, ogn = gens(sb, d + 1, GN_LABEL)
    S = States(sb, kind.encode(), n)
    if kind == "quad":
        want = pr.ZKSumcheckInstanceProof.prove_quad(claim, blind, n, *[t.copy() for t in tables], og1, ogn, S.ot, S.otape)
        terms = [(1, (0, 1))]
    else:
        want = pr.ZKSumcheckInstanceProof.prove_cubic_with_additive_term(claim, blind, n, *[t.copy() for t in tables], og1, ogn, S.ot, S.otape)
        terms = [(1, (0, 1, 2)), (Q - 1, (0, 3))]
    proof, r, finals, bp, polys = lib_prove(sb, tables, terms, claim, blind, n, lg1, lgn, S)
    assert proof.data == pr.ser(want[0])
    assert r == want[1] and finals == want[2] and bp == want[3]
    assert S.same()
    assert all(p.len() == 1 for p in polys)
    check_verifiers(sb, proof.data, claim, blind, n, d, lg1, lgn, og1, ogn, kind.encode())


# ---------------------------------------------------------------------------------------------------- parity with the model at every degree
def model_case(sb, tables, terms, num_rounds, tag, honest=True):
    d = max(len(fs) for _, fs in terms)
    rng = np.random.default_rng(zlib.crc32(tag))
    claim = hypercube_sum(tables, terms) if honest else rand_ints(rng, 1)[0]
    blind = rand_ints(rng, 1)[0]
    lg1, og1 = gens(sb, 1, G1_LABEL)
    lgn, ogn = gens(sb, d + 1, GN_LABEL)
    S = States(sb, tag, 3)
    want = zk_model_prove(tables, terms, claim, blind, num_rounds, og1, ogn, S.ot, S.otape)
    proof, r, finals, bp, polys = lib_prove(sb, tables, terms, claim, blind, num_rounds, lg1, lgn, S)
    assert proof.data == pr.ser(want[0])
    assert r == want[1] and finals == want[2] and bp == want[3]
    assert S.same()
    assert all(p.len() == len(tables[0]) >> num_rounds for p in polys)
    check_verifiers(sb, proof.data, claim, blind, num_rounds, d, lg1, lgn, og1, ogn, tag)
    return proof


@pytest.mark.parametrize("n", [3, 12, 16])
@pytest.mark.parametrize("D", [1, 2, 3, 4, 5, 6])
def test_parity_with_model_every_degree(sb, D, n):
    k, terms = mixed_composition(D, np.random.default_rng(10 * D + n))
    tables = [oc.prg_scalars("zk-gpu-deg-%d-%d-%d" % (D, n, j), 1 << n) for j in range(k)]
    model_case(sb, tables, terms, n, b"degree%d-%d" % (D, n))


@pytest.mark.parametrize("name", ["repeated_table", "unused_table", "cancelling_terms", "all_terms_cancel"])
def test_parity_with_model_special_compositions(sb, name):
    n = 6
    idx, terms = special_compositions(np.random.default_rng(zlib.crc32(name.encode())))[name]
    distinct = [oc.prg_scalars("zk-gpu-%s-%d" % (name, j), 1 << n) for j in range(max(idx) + 1)]
    model_case(sb, [distinct[i] for i in idx], terms, n, name.encode())


def test_parity_with_model_edge_tables_and_coefficients(sb):
    n = 5
    tables = [oc.to_arr([0] * (1 << n)), oc.to_arr([Q - 1] * (1 << n)), oc.prg_scalars("zk-gpu-edge", 1 << n)]
    terms = [(0, (0, 1, 2)), (Q - 1, (1, 1, 1, 2, 2, 2)), (1, (2,)), (Q - 1, (0, 2))]
    model_case(sb, tables, terms, n, b"edge")


@pytest.mark.parametrize("num_rounds", [1, 4])
@pytest.mark.parametrize("D", [1, 3, 6])
def test_parity_with_model_fewer_rounds_than_variables(sb, D, num_rounds):
    n = 8
    k, terms = mixed_composition(D, np.random.default_rng(D + num_rounds))
    tables = [oc.prg_scalars("zk-gpu-rounds-%d-%d" % (D, j), 1 << n) for j in range(k)]
    model_case(sb, tables, terms, num_rounds, b"rounds%d-%d" % (D, num_rounds), honest=False)


# ---------------------------------------------------------------------------------------------------- both verifiers reject every mutated field
def _mutants(obj):
    """(name, mutated proof) for every comm_poly, comm_eval and DotProductProof field of the first and the last round"""
    n = len(obj.comm_polys)
    other = lambda lst, i: lst[(i + 1) % len(lst)] if len(lst) > 1 else oc.commit_scalar(1, 1, oc.MultiCommitGens.new(1, b"x")).compress()  # noqa: E731
    out = []
    for i in sorted({0, n - 1}):
        for field in ("comm_polys", "comm_evals"):
            m = pr.deser(pr.ZKSumcheckInstanceProof, pr.ser(obj))[0]
            getattr(m, field)[i] = other(getattr(obj, field), i) if n > 1 else other([], 0)
            out.append(("%s[%d]" % (field, i), m))
        for field in ("delta", "beta", "z0", "zlast", "z_delta", "z_beta"):
            m = pr.deser(pr.ZKSumcheckInstanceProof, pr.ser(obj))[0]
            p = m.proofs[i]
            if field in ("delta", "beta"):
                setattr(p, field, obj.comm_polys[i])
            elif field == "z0":
                p.z[0] = (p.z[0] + 1) % Q
            elif field == "zlast":
                p.z[-1] = (p.z[-1] + 1) % Q
            else:
                setattr(p, field, (getattr(p, field) + 1) % Q)
            out.append(("proofs[%d].%s" % (i, field), m))
    return out


@pytest.mark.parametrize("D", [2, 5])
def test_verifiers_reject_mutants(sb, D):
    n = 4
    k, terms = mixed_composition(D, np.random.default_rng(50 + D))
    tables = [oc.prg_scalars("zk-gpu-mut-%d-%d" % (D, j), 1 << n) for j in range(k)]
    claim, blind = hypercube_sum(tables, terms), 77
    lg1, og1 = gens(sb, 1, G1_LABEL)
    lgn, ogn = gens(sb, D + 1, GN_LABEL)
    proof, _, _, _, _ = lib_prove(sb, tables, terms, claim, blind, n, lg1, lgn, States(sb, b"mut", 5))
    comm_claim = check_verifiers(sb, proof.data, claim, blind, n, D, lg1, lgn, og1, ogn, b"mut")
    obj = pr.deser(pr.ZKSumcheckInstanceProof, proof.data)[0]
    for name, m in _mutants(obj):
        ot, st = verifier_transcripts(sb, b"mut")
        with pytest.raises(pr.ProofVerifyError):
            m.verify(comm_claim, n, D, og1, ogn, ot)
        with pytest.raises(sb.ProofVerifyError) as e:
            sb.ZKSumcheckInstanceProof(pr.ser(m)).verify(comm_claim, n, D, lg1, lgn, st)
        assert e.value.code == sb.api.SP_ERR_VERIFY, name


# ---------------------------------------------------------------------------------------------------- the sigma protocols
def _sigma_cases(sb, n):
    """(name, library prove, oracle prove, library verify, oracle verify) over one States; the scalars are random with one zero and one q - 1"""
    rng = np.random.default_rng(n)
    x, rx, y, ry, rz = rand_ints(rng, 5)
    lg1, lgn, og1, ogn = split_gens(sb, n, b"zk-gpu-sigma")
    xs, a = [0] + rand_ints(rng, n - 2) + [Q - 1] if n >= 2 else [Q - 1], rand_ints(rng, n)
    dot = sum(i * j for i, j in zip(xs, a)) % Q
    return {
        "knowledge": (lambda S: sb.KnowledgeProof.prove(lg1, S.st, S.stape, L(x), L(rx)),
                      lambda S: pr.KnowledgeProof.prove(og1, S.ot, S.otape, x, rx),
                      lambda p, c, t: sb.KnowledgeProof(p).verify(lg1, t, *c),
                      lambda p, c, t: pr.deser(pr.KnowledgeProof, p)[0].verify(og1, t, *c), pr.KnowledgeProof),
        "equality": (lambda S: sb.EqualityProof.prove(lg1, S.st, S.stape, L(x), L(rx), L(x), L(ry)),
                     lambda S: pr.EqualityProof.prove(og1, S.ot, S.otape, x, rx, x, ry),
                     lambda p, c, t: sb.EqualityProof(p).verify(lg1, t, *c),
                     lambda p, c, t: pr.deser(pr.EqualityProof, p)[0].verify(og1, t, *c), pr.EqualityProof),
        "product": (lambda S: sb.ProductProof.prove(lg1, S.st, S.stape, L(x), L(rx), L(y), L(ry), L(x * y), L(rz)),
                    lambda S: pr.ProductProof.prove(og1, S.ot, S.otape, x, rx, y, ry, x * y % Q, rz),
                    lambda p, c, t: sb.ProductProof(p).verify(lg1, t, *c),
                    lambda p, c, t: pr.deser(pr.ProductProof, p)[0].verify(og1, t, *c), pr.ProductProof),
        "dotproduct": (lambda S: sb.DotProductProof.prove(lg1, lgn, S.st, S.stape, oc.to_arr(xs), L(rx), oc.to_arr(a), L(dot), L(ry)),
                       lambda S: pr.DotProductProof.prove(og1, ogn, S.ot, S.otape, xs, rx, a, dot, ry),
                       lambda p, c, t: sb.DotProductProof(p).verify(lg1, lgn, t, oc.to_arr(a), *c),
                       lambda p, c, t: pr.deser(pr.DotProductProof, p)[0].verify(og1, ogn, t, a, *c), pr.DotProductProof),
    }


def _field_mutants(tp, data):
    """one mutant per field of a sigma proof: a point replaced by another point of the proof or of the generators, a scalar plus one"""
    obj = pr.deser(tp, data)[0]
    pts = [getattr(obj, f) for f in ("alpha", "beta", "delta") if hasattr(obj, f)]
    spare = oc.MultiCommitGens.new(1, b"zk-gpu-spare").g(0).compress()
    out = []
    import dataclasses
    for f in dataclasses.fields(tp):
        v = getattr(obj, f.name)
        if isinstance(v, bytes):
            out.append((f.name, dataclasses.replace(obj, **{f.name: next((p for p in pts if p != v), spare)})))
        elif isinstance(v, int):
            out.append((f.name, dataclasses.replace(obj, **{f.name: (v + 1) % Q})))
        else:
            for i in sorted({0, len(v) - 1}):
                w = list(v)
                w[i] = (w[i] + 1) % Q
                out.append(("%s[%d]" % (f.name, i), dataclasses.replace(obj, **{f.name: type(v)(w)})))
    return out


@pytest.mark.parametrize("n", [1, 4, 7, 64])
@pytest.mark.parametrize("name", ["knowledge", "equality", "product", "dotproduct"])
def test_sigma_parity_and_verify(sb, name, n):
    if name != "dotproduct" and n != 1:
        pytest.skip("n is the dot product's length")
    lprove, oprove, lverify, overify, tp = _sigma_cases(sb, n)[name]
    S = States(sb, name.encode(), 40 + n)
    got, want = lprove(S), oprove(S)
    assert got[0].data == pr.ser(want[0])
    assert list(got[1:]) == list(want[1:])
    assert S.same()
    comms = list(want[1:])
    ot, st = verifier_transcripts(sb, name.encode())
    overify(got[0].data, comms, ot)
    lverify(pr.ser(want[0]), comms, st)
    assert ot.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64)
    for field, m in _field_mutants(tp, pr.ser(want[0])):
        ot, st = verifier_transcripts(sb, name.encode())
        with pytest.raises(pr.ProofVerifyError):
            overify(pr.ser(m), comms, ot)
        with pytest.raises(sb.ProofVerifyError):
            lverify(pr.ser(m), comms, st)
        assert ot.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64), field


# ---------------------------------------------------------------------------------------------------- refusals leave everything untouched
def test_refusals_leave_tables_transcript_and_tape(sb):
    n = 4
    A = sb.api
    lg1, _ = gens(sb, 1, G1_LABEL)
    lg3, _ = gens(sb, 3, GN_LABEL)
    lg4, _ = gens(sb, 4, GN_LABEL)
    other = sb.Context(lg1.ctx.device)
    foreign, foreign3 = sb.MultiCommitGens(1, G1_LABEL, ctx=other), sb.MultiCommitGens(3, GN_LABEL, ctx=other)
    tabs = [oc.prg_scalars("zk-gpu-refuse-%d" % j, 1 << n) for j in range(3)]
    polys = [sb.DensePolynomial(t) for t in tabs]
    quad, cubic = comp_of(sb, [(1, (0, 1))]), comp_of(sb, [(1, (0, 1, 2))])
    one, bad = L(1), np.frombuffer(Q.to_bytes(32, "little"), dtype=np.uint64)
    not_a_point = b"\xff" * 32
    C1 = oc.commit_scalar(1, 2, oc.MultiCommitGens.new(1, G1_LABEL)).compress()
    zk = sb.ZKSumcheckInstanceProof

    def zkp(ps=polys[:2], comp=quad, claim=one, rounds=n, g1=lg1, gn=lg3):
        return lambda S: zk.prove(ps, comp, claim, one, rounds, g1, gn, S.st, S.stape)

    cases = [
        (A.SP_ERR_INVALID_ARG, "gens_1.n = 3", zkp(g1=lg3)),
        (A.SP_ERR_INVALID_ARG, "gens_n.n = 4 but a round polynomial of degree 2 needs 3", zkp(gn=lg4)),
        (A.SP_ERR_INVALID_ARG, "gens_n.n = 3 but a round polynomial of degree 3 needs 4", zkp(ps=polys[:3], comp=cubic)),
        (A.SP_ERR_INVALID_ARG, "num_rounds = 5 outside", zkp(rounds=n + 1)),
        (A.SP_ERR_INVALID_ARG, "gens_1 belongs to another context", zkp(g1=foreign)),
        (A.SP_ERR_INVALID_SCALAR, "claim", zkp(claim=bad)),
        (A.SP_ERR_INVALID_ARG, "gens_n.n = 3", lambda S: sb.KnowledgeProof.prove(lg3, S.st, S.stape, one, one)),
        (A.SP_ERR_INVALID_SCALAR, "knowledge_prove: x", lambda S: sb.KnowledgeProof.prove(lg1, S.st, S.stape, bad, one)),
        (A.SP_ERR_INVALID_SCALAR, "equality_prove: s2", lambda S: sb.EqualityProof.prove(lg1, S.st, S.stape, one, one, one, bad)),
        (A.SP_ERR_INVALID_SCALAR, "product_prove: rZ", lambda S: sb.ProductProof.prove(lg1, S.st, S.stape, one, one, one, one, one, bad)),
        (A.SP_ERR_INVALID_ARG, "gens_n belongs to another context",
         lambda S: sb.DotProductProof.prove(lg1, foreign3, S.st, S.stape, oc.to_arr([1, 2, 3]), one, oc.to_arr([1, 2, 3]), one, one)),
        (A.SP_ERR_INVALID_ARG, "gens_n.n = 3 but vectors of length n = 2 needs 2",
         lambda S: sb.DotProductProof.prove(lg1, lg3, S.st, S.stape, oc.to_arr([1, 2]), one, oc.to_arr([1, 2]), one, one)),
        (A.SP_ERR_INVALID_ARG, "n = 65 outside 1 .. SP_DOTPROD_MAX_N = 64",
         lambda S: sb.DotProductProof.prove(lg1, lg3, S.st, S.stape, oc.to_arr([1] * 65), one, oc.to_arr([1] * 65), one, one)),
        (A.SP_ERR_INVALID_SCALAR, "dotproduct_prove: a_vec",
         lambda S: sb.DotProductProof.prove(lg1, lg3, S.st, S.stape, oc.to_arr([1, 2, 3]), one, np.stack([one, one, bad]), one, one)),
        (A.SP_ERR_INVALID_ARG, "gens_n.n = 4 but degree_bound = 2 needs 3", lambda S: zk(b"").verify(C1, 2, 2, lg1, lg4, S.st)),
        (A.SP_ERR_INVALID_ARG, "num_rounds must be >= 1", lambda S: zk(b"").verify(C1, 0, 2, lg1, lg3, S.st)),
        (A.SP_ERR_INVALID_POINT, "comm_claim", lambda S: zk(b"").verify(not_a_point, 2, 2, lg1, lg3, S.st)),
        (A.SP_ERR_INVALID_POINT, "knowledge_verify: C", lambda S: sb.KnowledgeProof(b"").verify(lg1, S.st, not_a_point)),
        (A.SP_ERR_INVALID_POINT, "equality_verify: C2", lambda S: sb.EqualityProof(b"").verify(lg1, S.st, C1, not_a_point)),
        (A.SP_ERR_INVALID_POINT, "product_verify: Z", lambda S: sb.ProductProof(b"").verify(lg1, S.st, C1, C1, not_a_point)),
        (A.SP_ERR_INVALID_POINT, "dotproduct_verify: Cx", lambda S: sb.DotProductProof(b"").verify(lg1, lg3, S.st, oc.to_arr([1, 2, 3]), not_a_point, C1)),
        (A.SP_ERR_INVALID_ARG, "n = 2 outside|gens_n.n = 3 but vectors of length n = 2",
         lambda S: sb.DotProductProof(b"").verify(lg1, lg3, S.st, oc.to_arr([1, 2]), C1, C1)),
    ]
    for code, msg, call in cases:
        S = States(sb, b"refuse", 1)
        before = S.raw()
        with pytest.raises(sb.SpartanB200Error, match=msg) as e:
            call(S)
        assert S.raw() == before, msg
        if code == A.SP_ERR_INVALID_ARG:
            assert "error %d" % code in str(e.value), msg
    for p, t in zip(polys, tabs):
        assert p.len() == 1 << n and np.array_equal(p.to_numpy(), t)


# ---------------------------------------------------------------------------------------------------- launches
def test_launches_one_per_round_plus_a_constant(sb):
    """a ZK sumcheck of n rounds makes n + c launches, c the same for every n and d: one per round (the first evaluation, n - 1 fused binds and
    evaluations, the last bind), the gather of the final entries, and the tape-only commitments (four row MSMs of two launches each on sets
    without a row table, one compression)"""
    extra = {}
    lg1, _ = gens(sb, 1, G1_LABEL)
    for D in (1, 3, 6):
        k, terms = mixed_composition(D, np.random.default_rng(D))
        lgn, _ = gens(sb, D + 1, GN_LABEL)
        for n in (3, 10, 16):
            polys = [sb.DensePolynomial(oc.prg_scalars("zk-gpu-launch-%d-%d" % (n, j), 1 << n)) for j in range(k)]
            S = States(sb, b"launch", 2)
            sb.ZKSumcheckInstanceProof.prove(polys, comp_of(sb, terms), L(0), L(0), 1, lg1, lgn, S.st, S.stape)   # host tables built
            polys = [sb.DensePolynomial(oc.prg_scalars("zk-gpu-launch-%d-%d" % (n, j), 1 << n)) for j in range(k)]
            before = sb.kernel_launches()
            sb.ZKSumcheckInstanceProof.prove(polys, comp_of(sb, terms), L(0), L(0), n, lg1, lgn, S.st, S.stape)
            extra[(D, n)] = sb.kernel_launches() - before - n
    print("launches beyond one per round:", extra)
    assert len(set(extra.values())) == 1, extra
    assert list(extra.values())[0] == 11, extra


# ---------------------------------------------------------------------------------------------------- the parity cases under the memory-check mode
def test_parity_cases_under_memcheck(tmp_path):
    if os.environ.get("SP_MEMCHECK_OUT"):
        pytest.skip("already running under the memory-check mode")
    out = tmp_path / "memcheck.json"
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "tests"), ROOT] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    env["SP_MEMCHECK_OUT"] = str(out)
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "memcheck_plugin", "-p", "no:cacheprovider", "-k",
           "parity_with_oracle_provers or sigma_parity", os.path.join(ROOT, "tests", "test_gpu_zk_sumcheck.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-20000:]
    tot = json.load(open(out))
    assert tot["violations"] == 0, tot
    assert tot["blocks_filled"] > 0 and tot["context_refills"] > 0, tot
