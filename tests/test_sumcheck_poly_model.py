"""A vectorised CPU model of a whole sumcheck of a caller-defined polynomial (include/spartan_b200.h: sp_sumcheck_prove_t), on the oracle's C
vector operations, pinned byte for byte to the plain-Python model_prove of test_gpu_sumcheck_poly.py.  That model works on Python integers and
stops being usable near 2^12 entries; this one reaches the sizes at which the device kernels change shape (streaming rounds, multi-pass grids),
so test_gpu_sumcheck_poly_limits.py checks the GPU against it."""
import time
import zlib

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from test_gpu_sumcheck_poly import from_evals, g_at, model_prove  # noqa: E402

Q = oc.Q


# ---------------------------------------------------------------------------------------------------- the model
def _distinct(tables):
    """one slot per distinct table object (a table passed twice is one table, bound once), and each index's slot"""
    seen, slot = [], []
    for t in tables:
        at = next((j for j, s in enumerate(seen) if s is t), None)
        if at is None:
            at = len(seen)
            seen.append(t)
        slot.append(at)
    return seen, slot


_ONES = {}


def _ones(n):
    if n not in _ONES:
        _ONES[n] = np.repeat(oc.to_arr([1]), n, axis=0)
    return _ONES[n]


def as_table(t):
    return t if isinstance(t, np.ndarray) else oc.to_arr(t)


def comb_sum(x, terms):
    """sum over i of g(x_0[i], x_1[i], ..) for g = sum_t c_t prod_{f in factors_t} x_f; x holds (n, 4) arrays (None for a table no term reads).
    Each distinct product is formed once, its prefixes shared: the last factor goes into the dot product."""
    prods, sums = {}, {}

    def prod(key):
        if key not in prods:
            prods[key] = x[key[0]] if len(key) == 1 else oc.hadamard(prod(key[:-1]), x[key[-1]])
        return prods[key]

    acc = 0
    for c, fs in terms:
        if c % Q == 0:
            continue
        key = tuple(sorted(fs))
        if key not in sums:
            if len(key) == 1:
                sums[key] = oc.dot(x[key[0]], _ones(len(x[key[0]])))
            else:
                sums[key] = oc.dot(prod(key[:-1]), x[key[-1]])
        acc += c * sums[key]
    return acc % Q


def hypercube_sum(tables, terms):
    """the honest claim: g summed over every entry of the tables"""
    seen, slot = _distinct([as_table(t) for t in tables])
    return comb_sum(seen, [(c, tuple(slot[f] for f in fs)) for c, fs in terms])


def model_prove_fast(tables, terms, claim, num_rounds, T):
    """model_prove's semantics and signature on (n, 4) Montgomery arrays (lists of ints are converted): returns (SumcheckInstanceProof, r,
    the bound tables as arrays (one per index, a repeated table's entries the same array), e).  The caller's arrays are not changed."""
    seen, slot = _distinct([as_table(t) for t in tables])
    P = [np.array(t, copy=True) for t in seen]
    sterms = [(c % Q, tuple(slot[f] for f in fs)) for c, fs in terms]
    used = {f for _, fs in sterms for f in fs}
    d = max(len(fs) for _, fs in terms)
    e, r, polys = claim % Q, [], []
    for _ in range(num_rounds):
        half = len(P[0]) // 2
        zero = oc.zeros(half)
        ev = []
        for t in [0] + list(range(2, d + 1)):
            # x_k(t) = (1 - t) lo + t hi, the values the device reaches as lo + t (hi - lo)
            x = [None if k not in used else p[:half] if t == 0 else oc.lincomb3(p[:half], p[half:], zero, (1 - t) % Q, t, 0)
                 for k, p in enumerate(P)]
            ev.append(comb_sum(x, sterms))
        poly = from_evals([ev[0], (e - ev[0]) % Q] + ev[1:])
        poly.append_to_transcript(b"poly", T)
        r_j = T.challenge_scalar(b"challenge_nextround")
        P = [oc.bound_top(p, r_j) for p in P]
        e = poly.evaluate(r_j)
        polys.append(poly.compress())
        r.append(r_j)
    return pr.SumcheckInstanceProof(polys), r, [P[s] for s in slot], e


# ---------------------------------------------------------------------------------------------------- compositions shared with the GPU tests
def rand_ints(rng, n):
    return [int.from_bytes(rng.bytes(32), "little") % Q for _ in range(n)]


def mixed_composition(D, rng):
    """degree D over 3 or 4 tables: a degree-D term with a random coefficient, a term of degree max(1, D - 1) with coefficient q - 1, a linear
    term with coefficient 1 (the kernels skip the multiplication by a unit coefficient) and a term of degree about D/2"""
    k = 3 + D % 2
    f = lambda m: tuple(int(i) for i in rng.integers(0, k, m))   # noqa: E731
    terms = [(rand_ints(rng, 1)[0], tuple(j % k for j in range(D))),
             (Q - 1, f(max(1, D - 1))),
             (1, (k - 1,)),
             (rand_ints(rng, 1)[0], f((D + 1) // 2))]
    return k, terms


def limits_composition(rng):
    """the kernels' limits: 8 distinct tables and 32 terms of degree up to 6.  One term is a single table to the sixth power, one has coefficient
    0, two cancel each other (the same product with its factors in another order), the other 28 are random products of degree 1 .. 6 that
    between them read every table."""
    c = rand_ints(rng, 1)[0]
    terms = [(rand_ints(rng, 1)[0], (5,) * 6),
             (0, (0, 1, 2)),
             (c, (3, 6, 6, 1)),
             (Q - c, (6, 1, 3, 6))]
    for i in range(28):
        m = int(rng.integers(1, 7))
        coeff = 1 if i == 0 else Q - 1 if i == 1 else rand_ints(rng, 1)[0]
        terms.append((coeff, (i % 8,) + tuple(int(j) for j in rng.integers(0, 8, m - 1))))
    assert len(terms) == 32 and max(len(fs) for _, fs in terms) == 6
    return 8, terms


def special_compositions(rng):
    """(tables as indices into k distinct random tables, terms): a repeated table, an unused table, cancelling terms, all terms cancelling"""
    c = rand_ints(rng, 1)[0]
    return {
        "repeated_table": ([0, 0, 1], [(rand_ints(rng, 1)[0], (0, 1, 2)), (c, (1, 1)), (1, (2,))]),
        "unused_table": ([0, 1, 2, 3], [(rand_ints(rng, 1)[0], (0, 1, 2)), (c, (2, 0))]),
        "cancelling_terms": ([0, 1, 2], [(c, (0, 1, 2)), (Q - c, (2, 1, 0)), (rand_ints(rng, 1)[0], (1, 1))]),
        "all_terms_cancel": ([0, 1], [(c, (0, 1, 1)), (Q - c, (1, 0, 1)), (1, (0,)), (Q - 1, (0,))]),
    }


# ---------------------------------------------------------------------------------------------------- the fast model equals the plain one
def _both(tables, terms, claim, num_rounds, label):
    ot1, ot2 = oc.Transcript(b"sumcheck-poly-model"), oc.Transcript(b"sumcheck-poly-model")
    ot1.append_message(b"app", label)
    ot2.append_message(b"app", label)
    want = model_prove([oc.to_ints(t) for t in tables], terms, claim, num_rounds, ot1)
    got = model_prove_fast(tables, terms, claim, num_rounds, ot2)
    assert pr.ser(got[0]) == pr.ser(want[0])
    assert got[1] == want[1] and got[3] == want[3]
    assert [oc.to_ints(p) for p in got[2]] == want[2]
    assert ot1.challenge_bytes(b"after", 32) == ot2.challenge_bytes(b"after", 32)
    return got


@pytest.mark.parametrize("n", [1, 2, 5, 8])
@pytest.mark.parametrize("D", [1, 2, 3, 4, 5, 6])
def test_fast_model_equals_plain_model_at_every_degree(D, n):
    rng = np.random.default_rng(100 * D + n)
    k, terms = mixed_composition(D, rng)
    tables = [oc.prg_scalars("scpm-%d-%d-%d" % (D, n, j), 1 << n) for j in range(k)]
    proof, _, _, _ = _both(tables, terms, rand_ints(rng, 1)[0], n, b"degree%d" % D)
    assert all(len(p.coeffs_except_linear_term) == D for p in proof.compressed_polys)


@pytest.mark.parametrize("n", [1, 2, 5, 8])
@pytest.mark.parametrize("name", ["repeated_table", "unused_table", "cancelling_terms", "all_terms_cancel"])
def test_fast_model_equals_plain_model_on_special_compositions(name, n):
    rng = np.random.default_rng(zlib.crc32(name.encode()) + n)
    idx, terms = special_compositions(rng)[name]
    distinct = [oc.prg_scalars("scpm-%s-%d-%d" % (name, n, j), 1 << n) for j in range(max(idx) + 1)]
    tables = [distinct[i] for i in idx]
    claim = hypercube_sum(tables, terms)
    proof, r, bound, e = _both(tables, terms, claim, n, name.encode())
    assert e == g_at(terms, [oc.to_ints(b)[0] for b in bound])
    if name == "repeated_table":
        assert bound[0] is bound[1]
    if name == "all_terms_cancel":   # g is zero everywhere: so are the claim and every round polynomial
        assert claim == 0 and all(c == 0 for p in proof.compressed_polys for c in p.coeffs_except_linear_term)


@pytest.mark.parametrize("num_rounds", [1, 3, 7])
def test_fast_model_fewer_rounds_than_variables(num_rounds):
    n = 8
    rng = np.random.default_rng(num_rounds)
    k, terms = mixed_composition(5, rng)
    tables = [oc.prg_scalars("scpm-rounds-%d-%d" % (num_rounds, j), 1 << n) for j in range(k)]
    _, _, bound, _ = _both(tables, terms, rand_ints(rng, 1)[0], num_rounds, b"rounds")
    assert all(len(b) == 1 << (n - num_rounds) for b in bound)


def test_fast_model_leaves_the_callers_tables():
    rng = np.random.default_rng(4)
    k, terms = mixed_composition(3, rng)
    tables = [oc.prg_scalars("scpm-keep-%d" % j, 64) for j in range(k)]
    copies = [t.copy() for t in tables]
    model_prove_fast(tables, terms, 0, 6, oc.Transcript(b"keep"))
    assert all(np.array_equal(t, c) for t, c in zip(tables, copies))


def test_fast_model_time_at_the_largest_gpu_case():
    """the largest model-checked case of test_gpu_sumcheck_poly_limits.py (8 tables, 32 terms, degree 6, 2^17 entries), with an honest claim: the
    oracle's verify accepts and its final claim is g at the bound tables"""
    n = 17
    k, terms = limits_composition(np.random.default_rng(17))
    tables = [oc.prg_scalars("scpm-limits-%d" % j, 1 << n) for j in range(k)]
    t0 = time.perf_counter()
    claim = hypercube_sum(tables, terms)
    T = oc.Transcript(b"limits")
    proof, r, bound, e = model_prove_fast(tables, terms, claim, n, T)
    took = time.perf_counter() - t0
    print("fast model, 8 tables, 32 terms, degree 6, n = %d: %.1f s" % (n, took))
    ve, vr = proof.verify(claim, n, 6, oc.Transcript(b"limits"))
    assert (ve, vr) == (e, r)
    assert e == g_at(terms, [oc.to_ints(b)[0] for b in bound])
