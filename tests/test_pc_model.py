"""Models of the joint commitment and joint opening of k tables (sp_pc_commit, sp_pc_eval_prove_joint_t) built from oracle pieces, on the CPU:
the joint prove as the library runs it (evaluations from the bound rows of each table, the merge's bound rows as a combination of them) pinned
byte for byte to the oracle's DerefsEvalProof.prove, the factorisation it rests on for every shape up to 2^10 entries and 64 tables, and the
table-list row mapping of the joint commitment against oc.commit_rows on the merged table."""
import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import spark as sk

Q = oc.Q
MAX_TABLES = 64


def shape(m, k):
    """(c, ell, lv, R) of the merge of k tables of 2^m entries"""
    c = oc.log_2(oc.next_pow2(k))
    ell = m + c
    return c, ell, ell // 2, 1 << (ell - ell // 2)


def rows_in_tables(m, c):
    """a row of the merge lies inside one table (R <= 2^m): the library reads the tables where they are; otherwise it gathers the merge"""
    return (m + c + 1) // 2 <= m


def tables(m, k, tag):
    return [oc.prg_scalars("pc-model-%s-%d-%d" % (tag, m, j), 1 << m) for j in range(k)]


def points(m, tag):
    return oc.to_ints(oc.prg_scalars("pc-model-r-" + tag, m)) if m else []


def eval_rows_model(Z, r, k):
    """the library's first steps on the tables-in-place path: LZ_j = bound(Z_j, eq(r[..lv - c])) in one pass, eval_j = <LZ_j, eq(r[lv - c..])>"""
    m = len(r)
    c, ell, lv, R = shape(m, k)
    lt = lv - c
    Lt = oc.eq_evals(r[:lt])
    LZ = [oc.bound_rows(z, Lt, 1 << lt, R) for z in Z]
    Rv = oc.eq_evals(r[lt:])
    return LZ, [oc.dot(lz, Rv) for lz in LZ], Rv


def combine_lz(LZ, ch):
    """the merge's bound rows: sum_j eq(ch)_j LZ_j (a k x R combination; the padding tables are zero)"""
    eq_ch = oc.eq_evals(ch)
    return oc.bound_rows(np.concatenate(LZ), eq_ch[:len(LZ)], len(LZ), len(LZ[0]))


def joint_prove_model(Z, r, gens, T, tape):
    """sp_pc_eval_prove_joint_t (DerefsEvalProof::prove_single without its protocol name) the way the library computes it, from oracle pieces"""
    k = len(Z)
    c, ell, lv, R = shape(len(r), k)
    assert rows_in_tables(len(r), c)
    LZ, evals, Rv = eval_rows_model(Z, r, k)
    evals = evals + [0] * (oc.next_pow2(k) - k)
    T.append_scalars(b"evals_ops_val", evals)
    ch = T.challenge_vector(b"challenge_combine_n_to_one", c)
    pe = list(evals)
    for i in reversed(range(c)):
        pe = oc.bound_bot_ints(pe, ch[i])
    joint = pe[0]
    T.append_scalar(b"joint_claim_eval", joint)
    T.append_protocol_name(b"polynomial evaluation proof")
    proof, _, _ = pr.DotProductProofLog.prove(gens.gens, T, tape, combine_lz(LZ, ch), 0, Rv, joint, 0)
    return pr.PolyEvalProof(proof), evals[:k]


@pytest.mark.parametrize("m,k", [(4, 1), (5, 2), (6, 3), (7, 5), (8, 8), (9, 6)])
def test_joint_prove_model_is_derefs_eval_proof(m, k):
    """the protocol-name line plus the model gives the oracle's DerefsEvalProof.prove byte for byte (all k evaluations as its eval_row)"""
    Z = tables(m, k, "pin")
    r = points(m, "pin-%d-%d" % (m, k))
    c, ell, _, _ = shape(m, k)
    gens = pr.PolyCommitmentGens(ell, b"pc-model")
    seed = 7 * m + k
    T_ref, tape_ref = oc.Transcript(b"pc-model"), oc.RandomTape(b"proof", seed)
    evals = [oc.evaluate(z, r) for z in Z]
    derefs = type("Merged", (), {"comb": sk.merge(Z)})   # DerefsEvalProof.prove reads only the merge; all k evaluations go in as eval_row
    want = sk.DerefsEvalProof.prove(derefs, evals, [], r, gens, T_ref, tape_ref)
    T, tape = oc.Transcript(b"pc-model"), oc.RandomTape(b"proof", seed)
    T.append_protocol_name(b"Derefs evaluation proof")
    got, got_evals = joint_prove_model(Z, r, gens, T, tape)
    assert got_evals == evals
    assert pr.ser(got) == pr.ser(want.proof_derefs)
    assert T.challenge_bytes(b"after", 32) == T_ref.challenge_bytes(b"after", 32)
    assert tape.random_scalar(b"after") == tape_ref.random_scalar(b"after")


@pytest.mark.parametrize("m", range(0, 11))
def test_merged_bound_rows_factor_per_table(m):
    """for every k <= 64: where rows lie inside tables, sum_j eq(ch)_j bound(Z_j, eq(r[..lv - c])) = bound(merge(Z), eq(r_joint[..lv])) and
    <LZ_j, eq(r[lv - c..])> = Z_j(r); where they do not, the merge is small enough to gather (at most 2^12 entries)"""
    pool = tables(m, MAX_TABLES, "factor")
    r = points(m, "factor-%d" % m)
    for k in range(1, MAX_TABLES + 1):
        c, ell, lv, R = shape(m, k)
        if not rows_in_tables(m, c):
            assert lv < c and (1 << ell) <= 1 << 12
            continue
        Z = pool[:k]
        ch = points(c, "ch-%d-%d" % (m, k))
        LZ, evals, _ = eval_rows_model(Z, r, k)
        merged = sk.merge(Z)
        want = oc.bound_rows(merged, oc.eq_evals((ch + r)[:lv]), 1 << lv, R)
        assert np.array_equal(combine_lz(LZ, ch), want), (m, k)
        assert evals == [oc.evaluate(z, r) for z in Z], (m, k)


def table_list_rows(Z, m, k):
    """the row mapping of the table-list row MSM (dev::TableRows): row i is row i % rows_per_table of table i / rows_per_table, zero past k"""
    c, ell, lv, R = shape(m, k)
    rpt = (1 << m) // R
    rows = []
    for i in range(1 << lv):
        j = i // rpt
        rows.append(Z[j][(i % rpt) * R:(i % rpt + 1) * R] if j < k else oc.zeros(R))
    return np.concatenate(rows)


@pytest.mark.parametrize("m,k,blinded", [(2, 1, False), (3, 2, True), (4, 3, False), (5, 5, True), (6, 8, False), (5, 7, True), (4, 4, True), (8, 6, False)])
def test_table_list_rows_reproduce_commit_rows(m, k, blinded):
    """the rows the mapping reads, committed row by row, give oc.commit_rows of the merged table (padding rows: identity or blind only)"""
    c, ell, lv, R = shape(m, k)
    assert rows_in_tables(m, c)
    Z = tables(m, k, "rows")
    merged = sk.merge(Z)
    mapped = table_list_rows(Z, m, k)
    assert np.array_equal(mapped, merged)
    gens = pr.PolyCommitmentGens(ell, b"pc-model-rows").gens.gens_n
    blinds = oc.to_ints(oc.prg_scalars("pc-model-blinds-%d-%d" % (m, k), 1 << lv)) if blinded else [0] * (1 << lv)
    want = oc.commit_rows(merged, 1 << lv, R, blinds, gens)
    got = [oc.commit_rows(mapped[i * R:(i + 1) * R], 1, R, [blinds[i]], gens)[0] for i in range(1 << lv)]
    assert got == want
    if not blinded:   # a padding row without a blind is the identity
        assert all(c == bytes(32) for c in want[k * ((1 << m) // R):])


@pytest.mark.parametrize("sms,no_instance", [(114, ("window", 8, 4)), (132, None)])
def test_limit_shapes_reach_every_branch(sms, no_instance):
    """the chooser of test_gpu_poly_commit_limits.py finds a shape for every launch path of the joint commitment and every slab split of the
    joint opening on 114 and 132 SMs, and each chosen shape takes the path it was chosen for.  Two paths no power-of-two table list reaches
    while the set has its row table (the set skips it only when device memory is short, which a shared GPU cannot be made to be):
    GROUPS = 1 of the table-list per-window MSM, since the per-window form runs only up to 2^16 merged entries, where L (R + 1) stays below
    1024 per SM; and the per-window MSM's batches of 32768 rows, which need L > 32768, so ell >= 32.  On 114 SMs GROUPS = 8 with CPT = 4 is
    not reached either: the shapes with 8 groups have too few blocks for four column passes."""
    from test_gpu_poly_commit_limits import COMMIT_INSTANCES, OPEN_BRANCHES, choose_shapes, commit_branch, commit_shapes, open_branch
    from test_gpu_poly_commit_limits import dims
    commit, opening = choose_shapes(sms)
    instances = COMMIT_INSTANCES - {no_instance}
    assert {b[0] for b in commit} == instances
    for inst in instances:
        assert {b[1] for b in commit if b[0] == inst} == {"k = 1", "k = 2^c", "padded k"}, inst
    assert {b[2] for b in commit if b[0] == "row table"} == {False, True}
    for b, (m, k, bl) in commit.items():
        assert commit_branch(m, k, bl, sms) == b
    assert any(k == MAX_TABLES and commit_branch(m, k, bl, sms)[0] == "row table" for m, k, bl in commit_shapes(sms))
    assert set(opening) == OPEN_BRANCHES
    for b, (m, k) in opening.items():
        assert open_branch(m, k, sms) == b or (b == "k > 32" and k > 32), b
    # what stays unreached: no GROUPS = 1 on the per-window form of a table list, which a table list takes only up to 2^16 merged entries
    for m in range(0, 31):
        for k in range(1, MAX_TABLES + 1):
            for bl in (False, True):
                b = commit_branch(m, k, bl, sms)
                if b is not None and b[0] != "row table":
                    assert dims(m, k)[1] <= 16 and b[0][1] != 1, (m, k, bl, b)
