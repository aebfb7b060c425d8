"""The caller-defined sumcheck kernels (kernels_sc.cu: k_scp_eval<D>, k_scp_fold_eval<D>, k_scp_fold_eval_small<D>) at every degree on both
fold paths, at the 8-table / 32-term / degree-6 limits, with few distinct tables at a high degree, on edge-valued tables, with unused and
repeated tables on the streaming path, with fewer rounds than variables, and between other calls on one context.  Every case goes through
sb.sumcheck_prove with a caller transcript and is checked against the vectorised model of test_sumcheck_poly_model.py: proof bytes, r, the
finals, e, the transcript afterwards, the library's and the oracle's verify, the tables left on the device; and every case asserts which kernel
families it launched, so a case that no longer reaches its path fails."""
import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from test_gpu_sumcheck_poly import check_library_verify, comp_of, g_at, same_state, transcripts  # noqa: E402
from test_sumcheck_poly_model import hypercube_sum, limits_composition, mixed_composition, model_prove_fast, rand_ints  # noqa: E402

pytestmark = pytest.mark.gpu
Q = oc.Q
SC_SMALL_MAX = 1024   # kernels_sc.cu: a fold of len-entry tables takes the small-table kernel once len/4 <= SC_SMALL_MAX
H100_SMS = 132


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    sb.default_context()
    return sb


def expected_launches(n, num_rounds):
    """the scp_* kernel families a sumcheck of 2^n-entry tables launches: the first round's evaluation, then one fold per later round, streaming
    while the tables being bound have more than 4 * SC_SMALL_MAX entries"""
    folds = [1 << (n - j) for j in range(num_rounds - 1)]
    stream = sum(1 for L in folds if L // 4 > SC_SMALL_MAX)
    want = {"scp_eval": 1, "scp_fold_eval": stream, "scp_fold_eval_small": len(folds) - stream}
    return {k: v for k, v in want.items() if v}


def handles_for(sb, tables):
    """one DensePolynomial per distinct array: an array passed at several indices is one handle passed several times"""
    made, polys = [], []
    for t in tables:
        at = next((p for a, p in made if a is t), None)
        if at is None:
            at = sb.DensePolynomial(t)
            made.append((t, at))
        polys.append(at)
    return polys


def prove_and_check(sb, tables, terms, num_rounds, label, reaches, claim=None):
    """prove on the GPU and compare everything with the model; claim None: the honest claim (the sum of g over the hypercube), which adds the
    final check e = g(finals), or e = the sum of g over the tables left when num_rounds < n"""
    n = len(tables[0]).bit_length() - 1
    honest = claim is None
    if honest:
        claim = hypercube_sum(tables, terms)
    d = max(len(fs) for _, fs in terms)
    polys = handles_for(sb, tables)
    ot, st = transcripts(sb, label)
    wproof, wr, wP, we = model_prove_fast(tables, terms, claim, num_rounds, ot)
    sb.api.prof_enable(True)
    try:
        proof, r, finals, e = sb.sumcheck_prove(polys, comp_of(sb, terms), oc.to_arr([claim])[0], num_rounds, st)
        prof = sb.api.prof_report()
    finally:
        sb.api.prof_enable(False)
    launched = {k: v["launches"] for k, v in prof.items() if k.startswith("scp_")}
    assert launched == expected_launches(n, num_rounds), launched
    for family in reaches:
        assert launched.get(family, 0) > 0, (family, launched)
    assert proof == pr.ser(wproof)
    assert all(len(p.coeffs_except_linear_term) == d for p in wproof.compressed_polys)
    assert oc.to_ints(r) == wr
    assert oc.to_ints(e.reshape(1, 4)) == [we]
    assert oc.to_ints(finals) == [oc.arr_get(w, 0) for w in wP]
    assert same_state(ot, st)
    left = []
    for p, w in zip(polys, wP):
        assert p.len() == len(w) == 1 << (n - num_rounds)
        if num_rounds < n:
            left.append(p.to_numpy())
            assert np.array_equal(left[-1], w)
    check_library_verify(sb, proof, claim, num_rounds, d, label)   # the oracle's verify and the library's accept, with the same e, r, state
    if honest:
        assert we == (g_at(terms, oc.to_ints(finals)) if num_rounds == n else hypercube_sum(left, terms))
    return proof, r, finals, e


def random_tables(tag, n, k):
    return [oc.prg_scalars("scp-limits-%s-%d-%d" % (tag, n, j), 1 << n) for j in range(k)]


ALL_PATHS = ("scp_eval", "scp_fold_eval", "scp_fold_eval_small")


# ---------------------------------------------------------------------------------------------------- 1. every degree on every kernel
@pytest.mark.parametrize("n", [13, 16])
@pytest.mark.parametrize("D", [1, 2, 3, 4, 5, 6])
def test_every_degree_on_every_kernel(sb, D, n):
    """n = 13: the streaming evaluation, one streaming fold, then small folds; n = 16: four streaming folds"""
    k, terms = mixed_composition(D, np.random.default_rng(10 * D + n))
    prove_and_check(sb, random_tables("deg%d" % D, n, k), terms, n, b"degree%d" % D, ALL_PATHS)


# ---------------------------------------------------------------------------------------------------- 2. the limits
@pytest.mark.parametrize("n", [3, 12, 13, 17, 18])
def test_eight_tables_thirty_two_terms_degree_six(sb, n):
    """the largest shared-memory column (2 * 8 tables * 128 threads * 32 B = 64 KB) and the most terms.  At n = 18 both the evaluation
    (2^17 indices) and the streaming folds (2^16 at the first) make several grid passes whatever the occupancy: 64 KB columns leave at most three
    blocks of 128 threads on each SM."""
    k, terms = limits_composition(np.random.default_rng(17))
    assert k == 8 and len(terms) == 32
    if n == 18:
        assert (1 << n) // 4 > H100_SMS * (228 // 64) * 128
    reaches = ALL_PATHS if n > 12 else ("scp_eval", "scp_fold_eval_small")
    prove_and_check(sb, random_tables("limits", n, k), terms, n, b"limits", reaches)


# ---------------------------------------------------------------------------------------------------- 3. few distinct tables at a high degree
FEW = {
    # name: (table index -> distinct table, terms)
    "A": ([0], [(5, (0,))]),
    "A^6": ([0], [(7, (0,) * 6)]),
    "AAAAB": ([0, 1], [(Q - 3, (0, 0, 0, 0, 1))]),
    "eight_handles_two_tables": ([0, 1, 0, 1, 0, 1, 0, 1], [(11, (0, 1, 2, 3, 4, 5)), (1, (6, 7)), (Q - 1, (2,))]),
}


@pytest.mark.parametrize("n", [1, 2, 3, 12, 13, 16])
@pytest.mark.parametrize("name", sorted(FEW))
def test_few_distinct_tables_high_degree(sb, name, n):
    """the small-table kernel sizes its block by the degree when D > 2 * (distinct tables): one warp per evaluation point outnumbers the two
    warps per table that bind.  A^6, A*A*A*A*B and eight handles of two tables reach that branch; A alone is the single-table composition."""
    idx, terms = FEW[name]
    D, distinct = max(len(fs) for _, fs in terms), max(idx) + 1
    assert name == "A" or D > 2 * distinct
    arrays = random_tables("few-%s" % name, n, distinct)
    reaches = ("scp_eval",) + (("scp_fold_eval_small",) if n >= 2 else ()) + (("scp_fold_eval",) if n > 12 else ())
    prove_and_check(sb, [arrays[i] for i in idx], terms, n, name.encode(), reaches)


# ---------------------------------------------------------------------------------------------------- 4. edge-valued tables
EDGES = [0, 1, 2, Q - 2, Q - 1, (Q - 1) // 2, (Q + 1) // 2, oc.R_MONT, oc.R_MONT * oc.R_MONT % Q]


def edge_tables(rng, n, k):
    """every entry one of EDGES, so every (lo, hi) pair of the first round is a pair of edge values"""
    vals = oc.to_arr(EDGES)
    return [np.ascontiguousarray(vals[rng.integers(0, len(EDGES), 1 << n)]) for _ in range(k)]


def paths(n):
    return ALL_PATHS if n > 12 else ("scp_eval", "scp_fold_eval_small")


@pytest.mark.parametrize("n", [5, 13])
@pytest.mark.parametrize("D", [1, 3, 6])
def test_edge_valued_tables(sb, D, n):
    rng = np.random.default_rng(1000 + 10 * D + n)
    k, terms = mixed_composition(D, rng)
    prove_and_check(sb, edge_tables(rng, n, k), terms, n, b"edges%d" % D, paths(n))


def round_constants(proof):
    """each round polynomial's constant term; asserts every other coefficient is zero (the linear one is implied by s(0) + s(1) = e)"""
    out = []
    for p in pr.deser(pr.SumcheckInstanceProof, proof)[0].compressed_polys:
        assert all(c == 0 for c in p.coeffs_except_linear_term[1:])
        out.append(p.coeffs_except_linear_term[0])
    return out


@pytest.mark.parametrize("n", [5, 13])
def test_all_zero_tables(sb, n):
    """every round polynomial is zero, and so are e and the finals"""
    k, terms = mixed_composition(6, np.random.default_rng(n))
    proof, _, finals, e = prove_and_check(sb, [oc.zeros(1 << n) for _ in range(k)], terms, n, b"zeros", paths(n))
    assert round_constants(proof) == [0] * n
    assert oc.to_ints(finals) == [0] * k and oc.to_ints(e.reshape(1, 4)) == [0]


@pytest.mark.parametrize("n", [5, 13])
@pytest.mark.parametrize("c", [Q - 1, (Q + 1) // 2, oc.R_MONT * oc.R_MONT % Q])
def test_constant_tables(sb, c, n):
    """tables constant at c: the claim is 2^n g(c), round j's polynomial is the constant 2^(n-j) g(c), the finals are c and e = g(c)"""
    k, terms = mixed_composition(6, np.random.default_rng(n + c % 1000))
    tables = [np.repeat(oc.to_arr([c]), 1 << n, axis=0) for _ in range(k)]
    gc = g_at(terms, [c] * k)
    assert hypercube_sum(tables, terms) == (1 << n) * gc % Q
    proof, _, finals, e = prove_and_check(sb, tables, terms, n, b"constant", paths(n))
    assert round_constants(proof) == [(1 << (n - 1 - j)) * gc % Q for j in range(n)]
    assert oc.to_ints(finals) == [c] * k and oc.to_ints(e.reshape(1, 4)) == [gc]


@pytest.mark.parametrize("n", [5, 13])
@pytest.mark.parametrize("D", [1, 3, 6])
def test_equal_halves_give_a_constant_first_round(sb, D, n):
    """hi == lo at every index of the first round: s_1 has degree 0, its constant half the claim"""
    rng = np.random.default_rng(2000 + 10 * D + n)
    k, terms = mixed_composition(D, rng)
    tables = [np.concatenate([t, t]) for t in edge_tables(rng, n - 1, k)]
    claim = hypercube_sum(tables, terms)
    proof, _, _, _ = prove_and_check(sb, tables, terms, n, b"halves", paths(n))
    p1 = pr.deser(pr.SumcheckInstanceProof, proof)[0].compressed_polys[0].coeffs_except_linear_term
    assert p1[0] == claim * oc.inv(2) % Q and all(v == 0 for v in p1[1:])


# ---------------------------------------------------------------------------------------------------- 5. unused and repeated tables, streaming
def test_unused_table_is_bound_on_the_streaming_path(sb):
    n = 14
    rng = np.random.default_rng(14)
    tables = random_tables("unused", n, 4)
    terms = [(rand_ints(rng, 1)[0], (0, 1, 2)), (rand_ints(rng, 1)[0], (2, 0)), (1, (1,))]
    _, r, finals, _ = prove_and_check(sb, tables, terms, n, b"unused", ALL_PATHS)
    assert oc.to_ints(finals)[3] == oc.evaluate(tables[3], oc.to_ints(r))


def test_handle_passed_three_times_on_the_streaming_path(sb):
    n = 14
    rng = np.random.default_rng(15)
    a, b = random_tables("thrice", n, 2)
    terms = [(rand_ints(rng, 1)[0], (0, 1, 2, 3)), (rand_ints(rng, 1)[0], (1, 3)), (1, (2,))]
    _, r, finals, _ = prove_and_check(sb, [a, a, a, b], terms, n, b"thrice", ALL_PATHS)
    fin = oc.to_ints(finals)
    assert fin[0] == fin[1] == fin[2] == oc.evaluate(a, oc.to_ints(r))


# ---------------------------------------------------------------------------------------------------- 6. fewer rounds than variables, large tables
@pytest.mark.parametrize("num_rounds", [1, 2, 3])
def test_fewer_rounds_than_variables_large_tables(sb, num_rounds):
    """n = 16: one round is k_scp_eval then fold_top alone; two and three rounds fold through k_scp_fold_eval once and twice.  The tables left
    on the device are compared entry for entry."""
    n = 16
    k, terms = mixed_composition(6, np.random.default_rng(num_rounds))
    reaches = ("scp_eval",) + (("scp_fold_eval",) if num_rounds > 1 else ())
    prove_and_check(sb, random_tables("rounds", n, k), terms, num_rounds, b"rounds", reaches)


# ---------------------------------------------------------------------------------------------------- 7. one context, many calls
def test_one_context_many_calls(sb):
    """the sumcheck shares the context's small buffers, reduction scratch, pinned result buffer and signal sequence with every other entry
    point: back to back, and between a variable-base MSM and a SNARK proof, every call gives what it gives alone (the MSM and the proof as
    pinned by the golden fixtures)"""
    from test_gpu_golden import GOLD, same

    rng = np.random.default_rng(7)
    specs = [(13, mixed_composition(3, rng), b"first"), (14, limits_composition(rng), b"second")]

    def run(i, check=False):
        n, (k, terms), label = specs[i]
        tables = random_tables("ctx%d" % i, n, k)
        if check:
            out = prove_and_check(sb, tables, terms, n, label, ALL_PATHS)
        else:
            _, st = transcripts(sb, label)
            out = sb.sumcheck_prove(handles_for(sb, tables), comp_of(sb, terms), oc.to_arr([hypercube_sum(tables, terms)])[0], n, st)
        return (out[0],) + tuple(np.ascontiguousarray(a).tobytes() for a in out[1:])

    alone = [run(0, check=True), run(1, check=True)]
    assert [run(0), run(1)] == alone

    mcase = next(c for c in GOLD["msm"] if c["n"] == 1024)
    g = sb.MultiCommitGens(mcase["n"], mcase["label"].encode())
    points = sb.api.Points(g.export()[:mcase["n"]])
    scalars = sb.prg_scalars("msm", mcase["n"], mcase["n"])
    scase = next(c for c in GOLD["snark"] if (c["num_cons"], c["num_vars"]) == (256, 256))
    nc, nv, ni, seed = scase["num_cons"], scase["num_vars"], scase["num_inputs"], scase["seed"]
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(nc, nv, ni, seed=seed)
    gens = sb.SNARKGens(nc, nv, ni, nc)
    comm = sb.SNARK.encode(inst, gens)
    label = GOLD["transcript_labels"]["snark"].encode()

    assert points.msm(scalars).hex() == mcase["result"]
    assert run(0) == alone[0]
    proof = sb.SNARK.prove(inst, comm, vars_, inputs, gens, label, sb.tape_seed(seed))
    assert same(proof.bytes, scase["proof"])
    assert run(1) == alone[1]
    assert points.msm(scalars).hex() == mcase["result"]
