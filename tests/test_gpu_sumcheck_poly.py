"""Whole sumchecks of caller-defined polynomials on the GPU (sp_sumcheck_prove_t, Composition / sumcheck_prove): byte parity with the oracle's
prove_cubic_batched and with a plain-Python model of the generic round (below), the oracle's verify on large proofs, the library's verify, the
refusals, and one kernel launch per round."""
import ctypes as C
import zlib

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr

pytestmark = pytest.mark.gpu
Q = oc.Q
LABEL = b"sumcheck-poly"


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    sb.default_context()
    return sb


# ---------------------------------------------------------------------------------------------------- the model
def from_evals(evals):
    """UniPoly::from_evals (unipoly.rs:23-54) for 3 and 4 points, Lagrange interpolation over 0 .. n-1 otherwise"""
    if len(evals) in (3, 4):
        return pr.UniPoly.from_evals(evals)
    n = len(evals)
    coeffs = [0] * n
    for i in range(n):
        num, den = [1], 1
        for j in range(n):
            if j == i:
                continue
            num = [((num[k - 1] if k > 0 else 0) - j * (num[k] if k < len(num) else 0)) % Q for k in range(len(num) + 1)]
            den = den * (i - j) % Q
        w = evals[i] * oc.inv(den) % Q
        coeffs = [(c + a * w) % Q for c, a in zip(coeffs, num)]
    return pr.UniPoly(coeffs)


def g_at(terms, x):
    acc = 0
    for c, fs in terms:
        p = c
        for f in fs:
            p = p * x[f] % Q
        acc += p
    return acc % Q


def model_prove(tables, terms, claim, num_rounds, T):
    """the semantics of include/spartan_b200.h on Python integers: tables are lists (copies of a repeated table are bound separately, which is
    the same as binding the one table once); terms are (int coefficient, factor indices)"""
    P = [list(t) for t in tables]
    d = max(len(f) for _, f in terms)
    points = [0] + list(range(2, d + 1))
    e, r, polys = claim, [], []
    for _ in range(num_rounds):
        half = len(P[0]) // 2
        ev = []
        for t in points:
            s = 0
            for i in range(half):
                s += g_at(terms, [(p[i] + t * (p[half + i] - p[i])) % Q for p in P])
            ev.append(s % Q)
        poly = from_evals([ev[0], (e - ev[0]) % Q] + ev[1:])
        poly.append_to_transcript(b"poly", T)
        r_j = T.challenge_scalar(b"challenge_nextround")
        P = [[(p[i] + r_j * (p[half + i] - p[i])) % Q for i in range(half)] for p in P]
        e = poly.evaluate(r_j)
        polys.append(poly.compress())
        r.append(r_j)
    return pr.SumcheckInstanceProof(polys), r, P, e


def rand_ints(rng, n):
    return [int.from_bytes(rng.bytes(32), "little") % Q for _ in range(n)]


def comp_of(sb, terms):
    return sb.Composition([(oc.to_arr([c])[0], fs) for c, fs in terms])


def transcripts(sb, prefix=b"prefix"):
    ot, st = oc.Transcript(LABEL), sb.Transcript(LABEL)
    ot.append_message(b"app", prefix)
    st.append_message(b"app", prefix)
    return ot, st


def same_state(ot, st):
    return ot.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64)


def check_library_verify(sb, proof_bytes, claim, num_rounds, degree, prefix):
    """the library's verify accepts and leaves the oracle verify's transcript; returns its (e, r) as integers"""
    ot, st = transcripts(sb, prefix)
    want_e, want_r = pr.deser(pr.SumcheckInstanceProof, proof_bytes)[0].verify(claim, num_rounds, degree, ot)
    e, r = sb.sumcheck_verify(proof_bytes, oc.to_arr([claim])[0], num_rounds, degree, st)
    assert oc.to_ints(e.reshape(1, 4)) == [want_e] and oc.to_ints(r) == list(want_r)
    assert same_state(ot, st)
    return want_e, want_r


# ---------------------------------------------------------------------------------------------------- parity with prove_cubic_batched
@pytest.mark.parametrize("n", [1, 2, 5, 10, 11, 12, 13, 16, 18])
@pytest.mark.parametrize("npar,nseq", [(3, 0), (2, 1)])
def test_batched_parity_with_oracle(sb, n, npar, nseq):
    """sum_i c_i A_i B_i C_par + sum_j c'_j A'_j B'_j C'_j as one composition, the shared C_par one table"""
    rng = np.random.default_rng(1000 * n + 10 * npar + nseq)
    N = 1 << n

    def table(tag):
        return oc.prg_scalars("scpoly-%s-%d-%d-%d" % (tag, n, npar, nseq), N)
    A_par, B_par, C_par = [table("ap%d" % i) for i in range(npar)], [table("bp%d" % i) for i in range(npar)], table("cp")
    A_seq, B_seq, C_seq = [table("as%d" % i) for i in range(nseq)], [table("bs%d" % i) for i in range(nseq)], [table("cs%d" % i) for i in range(nseq)]
    coeffs = rand_ints(rng, npar + nseq)
    claim = sum(c * oc.dot3(a, b, cc) for c, a, b, cc in zip(coeffs, A_par + A_seq, B_par + B_seq, [C_par] * npar + C_seq)) % Q
    # tables: A_par..., B_par..., C_par, then (A', B', C') per seq instance
    arrays = A_par + B_par + [C_par]
    terms = [(coeffs[i], (i, npar + i, 2 * npar)) for i in range(npar)]
    for j in range(nseq):
        base = len(arrays)
        arrays += [A_seq[j], B_seq[j], C_seq[j]]
        terms.append((coeffs[npar + j], (base, base + 1, base + 2)))
    polys = [sb.DensePolynomial(a) for a in arrays]
    ot, st = transcripts(sb)
    oproof, orr, claims_prod, claims_dotp = pr.prove_cubic_batched(claim, n, ([a.copy() for a in A_par], [b.copy() for b in B_par], C_par.copy()),
                                                                   ([a.copy() for a in A_seq], [b.copy() for b in B_seq], [c.copy() for c in C_seq]),
                                                                   coeffs, ot)
    proof, r, finals, e = sb.sumcheck_prove(polys, comp_of(sb, terms), oc.to_arr([claim])[0], n, st)
    assert proof == pr.ser(oproof)
    assert oc.to_ints(r) == list(orr)
    want_finals = list(claims_prod[0]) + list(claims_prod[1]) + [claims_prod[2]]
    for j in range(nseq):
        want_finals += [claims_dotp[0][j], claims_dotp[1][j], claims_dotp[2][j]]
    assert oc.to_ints(finals) == want_finals
    assert same_state(ot, st)
    assert all(p.len() == 1 for p in polys)
    e_ver, _ = check_library_verify(sb, proof, claim, n, 3, b"prefix")
    assert oc.to_ints(e.reshape(1, 4)) == [e_ver]


# ---------------------------------------------------------------------------------------------------- general compositions against the model
def _c(rng):
    return rand_ints(rng, 1)[0]


GENERAL = {
    "degree1": lambda rng: (2, [(_c(rng), (0,)), (_c(rng), (1,))]),
    "degree2": lambda rng: (3, [(_c(rng), (0, 1)), (_c(rng), (2,))]),
    "degree3_AAB": lambda rng: (2, [(_c(rng), (0, 0, 1))]),
    "degree4": lambda rng: (4, [(_c(rng), (0, 1, 2, 3)), (_c(rng), (1, 1)), (1, (3,))]),
    "degree5": lambda rng: (3, [(1, (0, 1, 2, 0, 1)), (_c(rng), (2, 2, 2))]),
    "degree6": lambda rng: (6, [(_c(rng), (0, 1, 2, 3, 4, 5)), (_c(rng), (5, 5, 5, 5, 5, 5)), (_c(rng), (0, 3))]),
    "zero_coefficient": lambda rng: (3, [(0, (0, 1, 2)), (_c(rng), (1, 2))]),
    "linear_only": lambda rng: (3, [(_c(rng), (0,)), (_c(rng), (1,)), (1, (2,))]),
    "one_table_in_every_term": lambda rng: (4, [(_c(rng), (0, 1)), (_c(rng), (0, 2, 3)), (_c(rng), (0,)), (_c(rng), (3, 0, 0))]),
    "eight_tables": lambda rng: (8, [(_c(rng), (i, (i + 1) % 8, (i + 3) % 8)) for i in range(8)]),
}


@pytest.mark.parametrize("n", [1, 3, 8, 12])
@pytest.mark.parametrize("name", sorted(GENERAL))
def test_general_compositions_against_model(sb, name, n):
    rng = np.random.default_rng(zlib.crc32(name.encode()) + n)
    k, terms = GENERAL[name](rng)
    tables = [rand_ints(rng, 1 << n) for _ in range(k)]
    claim = _c(rng)   # not checked by the prover: any value gives a proof
    polys = [sb.DensePolynomial(oc.to_arr(t)) for t in tables]
    ot, st = transcripts(sb, name.encode())
    wproof, wr, _, we = model_prove(tables, terms, claim, n, ot)
    d = max(len(f) for _, f in terms)
    proof, r, finals, e = sb.sumcheck_prove(polys, comp_of(sb, terms), oc.to_arr([claim])[0], n, st)
    assert proof == pr.ser(wproof)
    assert all(len(p.coeffs_except_linear_term) == d for p in wproof.compressed_polys)
    assert oc.to_ints(r) == wr
    assert oc.to_ints(e.reshape(1, 4)) == [we]
    assert same_state(ot, st)
    # the final claim is g at the tables' final entries for an honest claim only; here the finals are each table at r
    assert oc.to_ints(finals) == [oc.evaluate(oc.to_arr(t), wr) for t in tables]
    check_library_verify(sb, proof, claim, n, d, name.encode())


@pytest.mark.parametrize("num_rounds", [1, 3, 7])
def test_fewer_rounds_than_variables(sb, num_rounds):
    n = 10
    rng = np.random.default_rng(num_rounds)
    terms = [(_c(rng), (0, 1, 1)), (_c(rng), (2, 0)), (_c(rng), (2,))]
    tables = [rand_ints(rng, 1 << n) for _ in range(3)]
    claim = _c(rng)
    polys = [sb.DensePolynomial(oc.to_arr(t)) for t in tables]
    ot, st = transcripts(sb)
    wproof, wr, wP, we = model_prove(tables, terms, claim, num_rounds, ot)
    proof, r, finals, e = sb.sumcheck_prove(polys, comp_of(sb, terms), oc.to_arr([claim])[0], num_rounds, st)
    assert proof == pr.ser(wproof) and oc.to_ints(r) == wr and oc.to_ints(e.reshape(1, 4)) == [we]
    assert same_state(ot, st)
    for p, w in zip(polys, wP):
        assert p.len() == 1 << (n - num_rounds)
        assert oc.to_ints(p.to_numpy()) == w
    assert oc.to_ints(finals) == [w[0] for w in wP]


def test_repeated_handle_is_bound_once(sb):
    """A*A*B with A passed twice: the handle is one table, bound once per round, and both indices report its final entry"""
    n = 6
    rng = np.random.default_rng(77)
    a, b = rand_ints(rng, 1 << n), rand_ints(rng, 1 << n)
    terms = [(_c(rng), (0, 1, 2)), (_c(rng), (1,))]
    A, B = sb.DensePolynomial(oc.to_arr(a)), sb.DensePolynomial(oc.to_arr(b))
    ot, st = transcripts(sb)
    wproof, wr, wP, we = model_prove([a, a, b], terms, 5, n, ot)
    proof, r, finals, e = sb.sumcheck_prove([A, A, B], comp_of(sb, terms), oc.to_arr([5])[0], n, st)
    assert proof == pr.ser(wproof) and A.len() == 1 and B.len() == 1
    assert oc.to_ints(finals) == [wP[0][0], wP[1][0], wP[2][0]]


def test_label_form_equals_fresh_transcript(sb):
    n = 5
    rng = np.random.default_rng(3)
    tabs = [oc.to_arr(rand_ints(rng, 1 << n)) for _ in range(2)]
    comp = comp_of(sb, [(_c(rng), (0, 1, 1, 0))])
    claim = oc.to_arr([9])[0]
    p1 = [sb.DensePolynomial(t) for t in tabs]
    want = sb.sumcheck_prove(p1, comp, claim, n, sb.Transcript(LABEL))[0]
    p2 = [sb.DensePolynomial(t) for t in tabs]
    ctx = p2[0].ctx
    out, ln = C.POINTER(C.c_ubyte)(), C.c_size_t()
    r, finals, e = np.zeros((n, 4), np.uint64), np.zeros((2, 4), np.uint64), np.zeros(4, np.uint64)
    terms = comp._c_terms()
    ctx.check(sb.lib.sp_sumcheck_prove(ctx.h, (C.c_void_p * 2)(*[p.h for p in p2]), 2, terms, 1, claim.ctypes.data_as(C.c_void_p), C.c_size_t(n),
                                       C.c_char_p(LABEL), C.c_size_t(len(LABEL)), C.byref(out), C.byref(ln), r.ctypes.data_as(C.c_void_p),
                                       finals.ctypes.data_as(C.c_void_p), e.ctypes.data_as(C.c_void_p)))
    got = C.string_at(out, ln.value)
    sb.lib.sp_free(out)
    assert got == want


# ---------------------------------------------------------------------------------------------------- large tables
@pytest.mark.parametrize("n", [20, 22])
@pytest.mark.parametrize("shape", ["cubic", "degree6"])
def test_large_tables_verify_with_oracle(sb, n, shape):
    N = 1 << n
    rng = np.random.default_rng(n)
    if shape == "cubic":
        k, terms = 3, [(1, (0, 1, 2))]
    else:
        k, terms = 4, [(_c(rng), (0, 0, 1, 2, 3, 3)), (_c(rng), (1, 2)), (_c(rng), (0,))]
    arrays = [oc.prg_scalars("scpoly-large-%s-%d-%d" % (shape, n, j), N) for j in range(k)]
    copies = [a.copy() for a in arrays]
    polys = [sb.DensePolynomial(a) for a in arrays]
    claim = 0   # an honest claim needs the whole sum; the checks below hold for any claim through e = s_n(r_n)
    if shape == "cubic":
        claim = oc.dot3(arrays[0], arrays[1], arrays[2])
    d = max(len(f) for _, f in terms)
    ot, st = transcripts(sb)
    before = sb.kernel_launches()
    proof, r, finals, e = sb.sumcheck_prove(polys, comp_of(sb, terms), oc.to_arr([claim])[0], n, st)
    launches = sb.kernel_launches() - before
    assert launches <= n + 2, launches   # one per round, then the last bind and the gather of the first entries
    oe, orr = pr.deser(pr.SumcheckInstanceProof, proof)[0].verify(claim, n, d, ot)
    assert oc.to_ints(r) == list(orr) and oc.to_ints(e.reshape(1, 4)) == [oe]
    fin = oc.to_ints(finals)
    for j in range(k):
        assert fin[j] == oc.evaluate(copies[j], list(orr))
    if shape == "cubic":   # an honest claim: the final check of the verifier's caller passes
        assert oe == g_at(terms, fin)
    st2 = sb.Transcript(LABEL)
    st2.append_message(b"app", b"prefix")
    sb.sumcheck_verify(proof, oc.to_arr([claim])[0], n, d, st2)
    assert st2.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64)


def test_honest_degree6_final_check(sb):
    """an honest claim of a degree-6 composition at a size that crosses the streaming / small-table switch: e = g(finals)"""
    n = 14
    rng = np.random.default_rng(6)
    tables = [rand_ints(rng, 1 << n) for _ in range(3)]
    terms = [(_c(rng), (0, 0, 1, 1, 2, 2)), (_c(rng), (0, 1, 2)), (_c(rng), (2,))]
    claim = sum(g_at(terms, [t[i] for t in tables]) for i in range(1 << n)) % Q
    polys = [sb.DensePolynomial(oc.to_arr(t)) for t in tables]
    ot, st = transcripts(sb)
    proof, r, finals, e = sb.sumcheck_prove(polys, comp_of(sb, terms), oc.to_arr([claim])[0], n, st)
    oe, _ = pr.deser(pr.SumcheckInstanceProof, proof)[0].verify(claim, n, 6, ot)
    assert oe == oc.to_ints(e.reshape(1, 4))[0] == g_at(terms, oc.to_ints(finals))


# ---------------------------------------------------------------------------------------------------- verifier mutants on a GPU proof
def test_library_verify_rejects_mutants(sb):
    n = 6
    rng = np.random.default_rng(5)
    tables = [oc.to_arr(rand_ints(rng, 1 << n)) for _ in range(3)]
    terms = [(_c(rng), (0, 1, 2, 2))]
    polys = [sb.DensePolynomial(t) for t in tables]
    proof, _, _, _ = sb.sumcheck_prove(polys, comp_of(sb, terms), oc.to_arr([1])[0], n, sb.Transcript(LABEL))
    honest_e, _ = sb.sumcheck_verify(proof, oc.to_arr([1])[0], n, 4, sb.Transcript(LABEL))
    p = pr.deser(pr.SumcheckInstanceProof, proof)[0]
    for data, rounds, degree in [(pr.ser(pr.SumcheckInstanceProof(p.compressed_polys[:-1])), n, 4),
                                 (pr.ser(pr.SumcheckInstanceProof(p.compressed_polys + p.compressed_polys[:1])), n, 4),
                                 (proof, n, 3), (proof, n, 5), (proof, n - 1, 4)]:
        with pytest.raises(sb.ProofVerifyError) as err:
            sb.sumcheck_verify(data, oc.to_arr([1])[0], rounds, degree, sb.Transcript(LABEL))
        assert err.value.code == sb.api.SP_ERR_VERIFY
    changed = [pr.CompressedUniPoly(list(c.coeffs_except_linear_term)) for c in p.compressed_polys]
    changed[2].coeffs_except_linear_term[1] = (changed[2].coeffs_except_linear_term[1] + 1) % Q
    e, _ = sb.sumcheck_verify(pr.ser(pr.SumcheckInstanceProof(changed)), oc.to_arr([1])[0], n, 4, sb.Transcript(LABEL))
    assert not np.array_equal(e, honest_e)   # as the reference's verify: accepted with another final claim, which the final check rejects
    e, _ = sb.sumcheck_verify(proof, oc.to_arr([2])[0], n, 4, sb.Transcript(LABEL))
    assert not np.array_equal(e, honest_e)


# ---------------------------------------------------------------------------------------------------- refusals
def test_refusals_leave_tables_unbound(sb):
    n = 4
    rng = np.random.default_rng(9)
    tabs = [oc.to_arr(rand_ints(rng, 1 << n)) for _ in range(9)]
    polys = [sb.DensePolynomial(t) for t in tabs]
    short = sb.DensePolynomial(tabs[0][: 1 << (n - 1)])
    other_ctx = sb.Context(polys[0].ctx.device)
    foreign = sb.DensePolynomial(tabs[1], ctx=other_ctx)
    one = oc.to_arr([1])[0]
    cubic = sb.Composition([(one, (0, 1, 2))])
    cases = [
        ("differ in length", polys[:2] + [short], cubic, n),
        ("num_rounds = 0", polys[:3], cubic, 0),
        ("num_rounds = %d" % (n + 1), polys[:3], cubic, n + 1),
        ("table index 3 >= k = 3", polys[:3], sb.Composition([(one, (0, 1, 3))]), n),
        ("has no factors", polys[:3], sb.Composition([(one, (0, 1, 2)), (one, ())]), n),
        ("7 factors", polys[:3], sb.Composition([(one, (0, 1, 2, 0, 1, 2, 0))]), n),
        ("9 tables", polys[:9], cubic, n),
        ("33 terms", polys[:3], sb.Composition([(one, (0, 1, 2))] * 33), n),
        ("another context", polys[:2] + [foreign], cubic, n),
    ]
    for msg, ps, comp, rounds in cases:
        t = sb.Transcript(LABEL)
        state = t.state.raw
        with pytest.raises(sb.SpartanB200Error, match="error %d: .*%s" % (sb.api.SP_ERR_INVALID_ARG, msg)):
            sb.sumcheck_prove(ps, comp, one, rounds, t)
        assert t.state.raw == state
    for p, t in zip(polys, tabs):
        assert p.len() == 1 << n and np.array_equal(p.to_numpy(), t)
    assert short.len() == 1 << (n - 1)
    assert foreign.len() == 1 << n and np.array_equal(foreign.to_numpy(), tabs[1])
    bad = np.frombuffer(Q.to_bytes(32, "little"), dtype=np.uint64)
    with pytest.raises(sb.R1CSError):
        sb.sumcheck_prove(polys[:3], cubic, bad, n, sb.Transcript(LABEL))
    with pytest.raises(sb.R1CSError):
        sb.sumcheck_prove(polys[:3], sb.Composition([(bad, (0, 1, 2))]), one, n, sb.Transcript(LABEL))
    for p, t in zip(polys, tabs):
        assert np.array_equal(p.to_numpy(), t)


# ---------------------------------------------------------------------------------------------------- launches
@pytest.mark.parametrize("n", [3, 12, 16])
def test_one_launch_per_round(sb, n):
    rng = np.random.default_rng(n)
    polys = [sb.DensePolynomial(oc.prg_scalars("scpoly-launch-%d-%d" % (n, j), 1 << n)) for j in range(4)]
    comp = comp_of(sb, [(_c(rng), (0, 1, 2, 3, 3)), (_c(rng), (1,))])
    before = sb.kernel_launches()
    sb.sumcheck_prove(polys, comp, oc.to_arr([0])[0], n, sb.Transcript(LABEL))
    assert sb.kernel_launches() - before <= n + 2
