"""Joint commitments and joint openings of the caller's tables (sp_pc_commit, sp_pc_eval_prove_joint_t) on every launch path the shape selects:
the table-list row MSM on each per-window instance k_msm_rows<8|13|15, GROUPS, CPT, RowTables> and on the row-table path (k_msm_digits<RowTables>
and the kernels after it), each with one table, a power of two of them and a padded count, with and without blinds; and k_bound_rows_many on
each of its slab splits (one row per slab, even slabs of several rows, an uneven last slab, the 64-slab cap, a single row, one slab of many rows
written without k_sum_slabs) and with more than 32 tables.  Byte parity with the oracle up to 2^22 entries, a 2^25 opening checked by both
verifiers, and the parity cases again under the memory-check mode.

Which path a shape takes depends on the SM count, so the shapes are chosen by a mirror of the selection (prover.hpp pc_rows_in_tables;
kernels.cu msm_rows_use_row_table, msm_pick_groups, msm_pick_cpt, bound_rows_many_slabs) with this device's SM count.  Each case also checks on
the device that the path it was chosen for ran, by its kernel count: a commitment's launches tell the row-table MSM (four kernels) from the
per-window one (two), and a joint opening's launches, against those of a single opening with the same inner-product length on the same set,
tell one k_bound_rows_many from k_bound_rows_many and k_sum_slabs.

Every table carries the recodings' edge scalars at its first and last entries, so that a row read from the wrong table or offset changes the
commitment, and one table of each list of three or more is all zero.  Blinds of exactly 0 or q - 1 are not covered here: sp_pc_commit draws
its blinds from the random tape, so a caller cannot plant them (test_gpu_msm_instances.py plants them in the stride form of the same kernels)."""
import contextlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import spark as sk
from test_gpu_msm_instances import pick_cpt, pick_groups, uses_row_table, window_edges
from test_gpu_poly_commit import (LABEL, ints, launches, ogens, oracle_joint_prove, point, random_table, rows_in_tables, same_tape,
                                  same_transcript, shape, tapes, transcripts)
from test_row_msm import edge_scalars

pytestmark = pytest.mark.gpu
Q = oc.Q
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDTHS = ["8", "13", "15"]
COMMIT_VARS = 17    # one set per window width of 2^9 + 2 generators (>= 512: SP_MSM_WINDOW applies, and the set has its row table)
PARITY_VARS = 22    # every byte against the oracle up to 2^22 entries; above, the verifiers and spot-checked rows
MAX_K = 64
ROW_TABLE_EXTRA = [(11, 33), (11, 64)]   # 4 rows per table on the row-table path: 124 padding rows, and the last table index


# ---------------------------------------------------------------------------------------------------- mirror of the selection
def dims(m, k):
    """(c, ell, L, R) of the merge of k tables of 2^m entries"""
    c, ell = shape(m, k)
    return c, ell, 1 << (ell // 2), 1 << (ell - ell // 2)


def kclass(k):
    return "k = 1" if k == 1 else "k = 2^c" if k & (k - 1) == 0 else "padded k"


def commit_branch(m, k, blinds, sms):
    """the launch path of sp_pc_commit for a set with its row table: ("row table" | ("window", GROUPS, CPT), k class, blinds); None: gathered"""
    c, ell, L, R = dims(m, k)
    if not rows_in_tables(m, c):
        return None
    if uses_row_table(L, R):
        return ("row table", kclass(k), blinds)
    g = pick_groups(L, R, sms)
    return (("window", g, pick_cpt(L, R + (1 if blinds else 0), g, sms)), kclass(k), blinds)


def bound_rows_many_slabs(k, L_size, R_size, sms):
    """(slabs, rows per slab, slabs wanted before the caps) of k_bound_rows_many"""
    blocks, want = -(-R_size // 128) * k, sms * 16
    wanted = -(-want // blocks)
    n = max(min(wanted, 64, L_size), 1)
    rows = -(-L_size // n)
    return -(-L_size // rows), rows, wanted


def open_split(m, k, sms):
    """(Lt, RJ, slabs, rows per slab) of the joint opening's k_bound_rows_many launch"""
    c, ell, _, _ = dims(m, k)
    lv = ell // 2
    Lt, RJ = 1 << (lv - c), 1 << (ell - lv)
    return (Lt, RJ) + bound_rows_many_slabs(k, Lt, RJ, sms)[:2]


def open_branch(m, k, sms):
    """the slab split of sp_pc_eval_prove_joint_t's bound rows; None: the merge is gathered"""
    c, _, _, _ = dims(m, k)
    if not rows_in_tables(m, c):
        return None
    Lt, RJ, n, rows = open_split(m, k, sms)
    if Lt == 1:
        return "one row"
    if n == 1:
        return "one slab of many rows"
    if rows == 1:
        return "one row per slab"
    if bound_rows_many_slabs(k, Lt, RJ, sms)[2] > 64 and Lt > 64:
        return "64-slab cap"
    return "uneven last slab" if Lt % rows else "even slabs"


COMMIT_INSTANCES = {("window", 8, 1), ("window", 8, 4), ("window", 4, 1), ("window", 4, 4), "row table"}
OPEN_BRANCHES = {"one row per slab", "even slabs", "uneven last slab", "64-slab cap", "one row", "one slab of many rows", "k > 32"}


def choose_shapes(sms, max_m=24):
    """the cheapest shape (fewest merged entries, then fewest tables) reaching each branch: commitments {branch: (m, k, blinds)} within
    COMMIT_VARS, joint openings {branch: (m, k)} with "k > 32" (two dot_many launches for the evaluations) as a branch of its own"""
    commit, opening = {}, {}
    for m in range(0, max_m + 1):
        for k in range(1, MAX_K + 1):
            c, ell, L, R = dims(m, k)
            cost = (ell, k)
            for bl in (False, True):
                b = commit_branch(m, k, bl, sms)
                if b is not None and ell <= COMMIT_VARS and (b not in commit or cost < commit[b][0]):
                    commit[b] = (cost, m, k, bl)
            b = open_branch(m, k, sms)
            for key in ([b] + (["k > 32"] if k > 32 else [])) if b else []:
                if key not in opening or cost < opening[key][0]:
                    opening[key] = (cost, m, k)
    return {b: v[1:] for b, v in commit.items()}, {b: v[1:] for b, v in opening.items()}


def eq_launches(nvars):
    """kernels of dev::eq_evals: one up to 10 variables, two halves and their combination above"""
    return 1 if nvars <= 10 else 3


def commit_launches(m, k):
    """kernels of sp_pc_commit on the table-list path: k_msm_digits, k_msm_win, k_msm_chunks and k_msm_horner on the row table, or one
    k_msm_rows per 32768 rows and a reducer on the per-window tables; then k_compress"""
    c, ell, L, R = dims(m, k)
    return (4 if uses_row_table(L, R) else -(-L // 32768) + 1) + 1


def open_launches_over_single(m, k, sms):
    """kernels of sp_pc_eval_prove_joint_t minus those of sp_pc_eval_prove_t (Zr not given) of a table of 2^(2r - 1) entries on the same set,
    where RJ = 2^r.  Both run eq_evals of r variables, to_canonical, bound_rows (two kernels) and the inner-product proof on RJ entries.  The
    joint opening adds eq_evals of lt variables, k_bound_rows_many, k_sum_slabs when there is more than one slab, and one dot_many per 32
    tables; the single opening adds eq_evals of r - 1 variables and one dot"""
    Lt, RJ, slabs, _ = open_split(m, k, sms)
    r = RJ.bit_length() - 1
    return eq_launches(Lt.bit_length() - 1) + (1 if slabs == 1 else 2) + -(-k // 32) - eq_launches(max(2 * r - 1, 0) // 2) - 1


def commit_shapes(sms):
    """every chosen commitment shape, plus the row-table extras with and without blinds"""
    commit, _ = choose_shapes(sms)
    return sorted(set(commit.values()) | {(m, k, bl) for m, k in ROW_TABLE_EXTRA for bl in (False, True)})


# ---------------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    sb.default_context()
    return sb


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def shapes(sms):
    commit, opening = choose_shapes(sms)
    print("\ncaller-table commitments on %d SMs (window widths %s):" % (sms, "/".join(WIDTHS)))
    print("%-18s %-9s %6s %4s %3s %4s %5s %5s" % ("path", "k class", "blinds", "m", "k", "ell", "L", "R"))
    for m, k, bl in commit_shapes(sms):
        c, ell, L, R = dims(m, k)
        b = commit_branch(m, k, bl, sms)
        print("%-18s %-9s %6s %4d %3d %4d %5d %5d" % (b[0] if b[0] == "row table" else "window G%d C%d" % b[0][1:], b[1], bl, m, k, ell, L, R))
    print("joint openings (k_bound_rows_many):")
    print("%-22s %4s %3s %4s %5s %5s %6s %9s" % ("branch", "m", "k", "ell", "Lt", "RJ", "slabs", "rows/slab"))
    for b in sorted(opening):
        m, k = opening[b]
        print("%-22s %4d %3d %4d %5d %5d %6d %9d" % ((b, m, k, dims(m, k)[1]) + open_split(m, k, sms)))
    return commit, opening


@contextlib.contextmanager
def msm_window(w):
    """SP_MSM_WINDOW = w while generator sets are built"""
    old = os.environ.get("SP_MSM_WINDOW")
    os.environ["SP_MSM_WINDOW"] = w
    try:
        yield
    finally:
        if old is None:
            del os.environ["SP_MSM_WINDOW"]
        else:
            os.environ["SP_MSM_WINDOW"] = old


EDGES = [0, 1, 2, Q - 1, Q - 2, oc.R_MONT] + [e for W in (8, 13, 15) for e in window_edges(W)] + edge_scalars(16)


def tables(m, k, tag):
    """k tables of 2^m entries with the edge scalars at the start and at the end of each (rotated per table), and table 1 all zero when k >= 3"""
    n = 1 << m
    out = []
    for j in range(k):
        z = oc.prg_scalars("pc-limits-%s-%d-%d-%d" % (tag, m, k, j), n)
        if j == 1 and k >= 3:
            z[:] = 0
        else:
            rot = EDGES[j % len(EDGES):] + EDGES[:j % len(EDGES)]
            cnt = min(len(EDGES), max(1, n // 2))
            z[:cnt] = oc.to_arr(rot[:cnt])
            z[n - cnt:] = oc.to_arr(rot[-cnt:])
        out.append(z)
    return out


def seed_of(m, k, bl):
    return 1000 * m + 2 * k + (1 if bl else 0)


# ---------------------------------------------------------------------------------------------------- commitments
@pytest.fixture(scope="module")
def oracle_commits(sb, sms):
    """the oracle's commitment, blinds and tape state after them, of every shape, once for all window widths"""
    oc.lib.oracle_set_threads(max(1, (os.cpu_count() or 2) // 2))
    out = {}
    for m, k, bl in commit_shapes(sms):
        c, ell, L, R = dims(m, k)
        otape = tapes(sb, seed_of(m, k, bl))[1] if bl else None
        want, blinds = pr.poly_commit(sk.merge(tables(m, k, "commit")), ogens(ell), otape)
        out[(m, k, bl)] = (want, blinds, otape.tape.challenge_bytes(b"after", 64) if bl else None)
    return out


@pytest.mark.parametrize("window", WIDTHS)
def test_commit_parity_every_path(sb, sms, shapes, oracle_commits, window, monkeypatch):
    """each chosen shape committed through views of one set of COMMIT_VARS built under SP_MSM_WINDOW = window: the commitment's bytes, its
    blinds and the tape against the oracle, the tables left alone, one table-list row MSM that ran the kernels of the path the shape was chosen
    for; rows of the zero table and padding rows without blinds are the identity"""
    monkeypatch.setenv("SP_MSM_WINDOW", window)
    big = sb.PolyCommitmentGens(COMMIT_VARS, LABEL)
    try:
        for m, k, bl in commit_shapes(sms):
            c, ell, L, R = dims(m, k)
            what = "%s (m=%d, k=%d, blinds=%s, window %s)" % (commit_branch(m, k, bl, sms), m, k, bl, window)
            Z = tables(m, k, "commit")
            polys = [sb.DensePolynomial(z) for z in Z]
            stape = tapes(sb, seed_of(m, k, bl))[0] if bl else None
            g = big.view(ell)
            sb.api.prof_enable(True)
            l0 = sb.kernel_launches()
            comm, blinds = sb.poly_commit(polys, g, stape)
            kernels = sb.kernel_launches() - l0
            n = launches(sb)
            sb.api.prof_enable(False)
            want, want_blinds, tape_after = oracle_commits[(m, k, bl)]
            bad = [i for i in range(L) if comm.C[i] != want.C[i]]
            assert not bad, "%s: %d of %d rows differ from the oracle, first row %d" % (what, len(bad), L, bad[0])
            assert comm.to_bytes() == pr.ser(want), what
            if bl:
                assert ints(blinds) == [b % Q for b in want_blinds], what
                assert stape.challenge_bytes(b"after", 64) == tape_after, what
            else:
                rpt = (1 << m) // R
                zero_rows = list(range(rpt, 2 * rpt)) if k >= 3 else []
                assert all(comm.C[i] == bytes(32) for i in zero_rows + list(range(k * rpt, L))), what
            assert n == {"msm_rows": 0, "msm_rows_tables": 1, "bound_rows_many": 0}, (what, n)
            assert kernels == commit_launches(m, k), (what, kernels, commit_launches(m, k))
            for p, z in zip(polys, Z):
                assert np.array_equal(p.to_numpy(), z), what
    finally:
        del big


# ---------------------------------------------------------------------------------------------------- joint openings
_single = {}


def single_open_launches(sb, gset, RJ):
    """kernels of one sp_pc_eval_prove_t (Zr computed) on a view of gset whose rows have RJ entries (launch counts do not depend on values)"""
    key = (id(gset), RJ)
    if key not in _single:
        r = RJ.bit_length() - 1
        ell = max(2 * r - 1, 0)
        poly = sb.DensePolynomial(oc.zeros(1 << ell))
        l0 = sb.kernel_launches()
        sb.PolyEvalProof.prove(poly, None, oc.to_arr(point("single-%d" % ell, ell)), None, None, gset.view(ell), sb.Transcript(LABEL),
                               sb.RandomTape(sb.tape_seed(1)))
        _single[key] = sb.kernel_launches() - l0
    return _single[key]


def check_slab_kernels(sb, gset, m, k, sms, kernels, what):
    """the joint opening launched one kernel for its bound rows when the mirror says one slab, two (k_bound_rows_many, k_sum_slabs) otherwise"""
    Lt, RJ, slabs, _ = open_split(m, k, sms)
    single = single_open_launches(sb, gset, RJ)
    assert kernels - single == open_launches_over_single(m, k, sms), (what, "slabs", slabs, "kernels", kernels, "single opening", single)


@pytest.fixture(scope="module")
def open_gens(sb, shapes):
    """one set for the joint openings up to PARITY_VARS, 8-bit windows (its tables stay small at 2^11 generators)"""
    ell = max(dims(m, k)[1] for m, k in shapes[1].values() if dims(m, k)[1] <= PARITY_VARS)
    with msm_window("8"):
        g = sb.PolyCommitmentGens(max(ell, 1), LABEL)
    yield g
    del g


@pytest.mark.parametrize("blinded", [False, True])
def test_joint_open_parity_every_split(sb, sms, shapes, open_gens, blinded):
    """each slab split (and k > 32) up to PARITY_VARS, opened with or without the joint commitment's blinds: proof bytes, evaluations,
    transcript and tape against the oracle, one bound_rows_many with the kernel count of its split and no table-list MSM in the proof, the
    tables left alone, and the oracle's verifier accepting the proof against the library's commitment"""
    oc.lib.oracle_set_threads(max(1, (os.cpu_count() or 2) // 2))
    for branch, (m, k) in sorted(shapes[1].items()):
        c, ell, L, R = dims(m, k)
        if ell > PARITY_VARS:
            continue
        what = "%s (m=%d, k=%d, blinds=%s)" % (branch, m, k, blinded)
        Z = tables(m, k, "open")
        r = point("limits-%d-%d" % (m, k), m)
        polys = [sb.DensePolynomial(z) for z in Z]
        g = open_gens.view(ell)
        stape, otape = tapes(sb, 5000 + seed_of(m, k, blinded))
        comm, blinds = sb.poly_commit(polys, g, stape if blinded else None)
        oblinds = None
        if blinded:
            oblinds = otape.random_vector(b"poly_blinds", L)
            assert ints(blinds) == [b % Q for b in oblinds], what
        ot, st = transcripts(sb)
        st.append_message(b"protocol-name", b"Derefs evaluation proof")
        sb.api.prof_enable(True)
        l0 = sb.kernel_launches()
        proof, evals = sb.PolyEvalProof.prove_joint(polys, blinds if blinded else None, oc.to_arr(r), g, st, stape)
        kernels = sb.kernel_launches() - l0
        n = launches(sb)
        sb.api.prof_enable(False)
        want, want_evals = oracle_joint_prove(Z, r, oblinds, ell, ot, otape)
        assert ints(evals) == want_evals, what
        assert proof.data == pr.ser(want), what
        assert same_transcript(ot, st) and same_tape(otape, stape), what
        assert n["bound_rows_many"] == 1 and n["msm_rows_tables"] == 0, (what, n)   # (msm_rows: the inner-product rounds' blind terms)
        check_slab_kernels(sb, open_gens, m, k, sms, kernels, what)
        for p, z in zip(polys, Z):
            assert np.array_equal(p.to_numpy(), z), what
        ot2 = oc.Transcript(LABEL)   # blinded or not: the reference's DerefsEvalProof::verify checks against joint * G_1
        ot2.append_message(b"app", b"prefix")
        sk.DerefsEvalProof(pr.deser(pr.PolyEvalProof, proof.data)[0]).verify(r, want_evals, [], ogens(ell), pr.PolyCommitment(comm.C), ot2)


def test_joint_open_large_one_slab(sb, sms, shapes):
    """the splits whose cheapest shape lies above PARITY_VARS (on 132 SMs: one slab of many rows, m = 19 and k = 33, 2^25 merged entries) on
    a set with 8-bit windows: the kernel count of the split, the evaluations against oc.evaluate, the library's verify_joint and the oracle's
    DerefsEvalProof.verify accept the proof against the library's commitment, and that commitment's rows at every table boundary, in the
    padding, first and last against oc.commit_vec.  Prints the largest device_bytes_live() seen between the calls: a lower bound on the peak,
    since the scratch a call frees before it returns is not seen"""
    big = sorted((b, mk) for b, mk in shapes[1].items() if dims(*mk)[1] > PARITY_VARS)
    oc.lib.oracle_set_threads(max(1, (os.cpu_count() or 2) // 2))
    for branch, (m, k) in big:
        c, ell, L, R = dims(m, k)
        sb.release_cached_memory()
        live0, seen = sb.device_bytes_live(), 0
        rng = np.random.default_rng(ell)
        Z = [random_table(rng, 1 << m) for _ in range(k)]
        Z[1][:] = 0
        r = oc.to_ints(random_table(rng, m))
        with msm_window("8"):
            g = sb.PolyCommitmentGens(ell, LABEL)
        polys = [sb.DensePolynomial(z) for z in Z]
        seen = max(seen, sb.device_bytes_live())
        stape = sb.RandomTape(sb.tape_seed(ell))
        comm, blinds = sb.poly_commit(polys, g, stape)
        seen = max(seen, sb.device_bytes_live())
        st = sb.Transcript(LABEL)
        st.append_message(b"protocol-name", b"Derefs evaluation proof")
        sb.api.prof_enable(True)
        l0 = sb.kernel_launches()
        proof, evals = sb.PolyEvalProof.prove_joint(polys, blinds, oc.to_arr(r), g, st, stape)
        kernels = sb.kernel_launches() - l0
        n = launches(sb)
        sb.api.prof_enable(False)
        seen = max(seen, sb.device_bytes_live())
        print("\n%s: m=%d k=%d ell=%d, device_bytes_live() between the calls up to %.2f GB above the %.2f GB live before (a lower bound on the "
              "peak)" % (branch, m, k, ell, (seen - live0) / 1e9, live0 / 1e9))
        assert n["bound_rows_many"] == 1 and n["msm_rows_tables"] == 0, n
        check_slab_kernels(sb, g, m, k, sms, kernels, branch)
        want_evals = [oc.evaluate(z, r) for z in Z]
        assert ints(evals) == want_evals
        vt = sb.Transcript(LABEL)
        vt.append_message(b"protocol-name", b"Derefs evaluation proof")
        sb.PolyEvalProof(proof.data).verify_joint(g, vt, oc.to_arr(r), evals, comm)
        assert vt.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64)
        og = ogens(ell)
        sk.DerefsEvalProof(pr.deser(pr.PolyEvalProof, proof.data)[0]).verify(r, want_evals, [], og, pr.PolyCommitment(comm.C), oc.Transcript(LABEL))
        # the commitment's rows: both sides of every table boundary, padding rows (the blind term alone), first and last
        rpt = (1 << m) // R
        bl = ints(blinds)
        rows = sorted({0, L - 1} | {i for j in range(1, k) for i in (j * rpt - 1, j * rpt)} | {k * rpt, (k * rpt + L) // 2})
        zero_row = oc.zeros(R)
        for i in rows:
            j, o = divmod(i, rpt)
            x = Z[j][o * R:(o + 1) * R] if j < k else zero_row
            assert comm.C[i] == oc.commit_vec(x, bl[i], og.gens.gens_n).compress(), (branch, i)
        for p, z in zip(polys[:2], Z[:2]):
            assert np.array_equal(p.to_numpy(), z)
        del polys, g, comm, proof
        _single.clear()
        sb.release_cached_memory()


# ---------------------------------------------------------------------------------------------------- the parity cases under the memory-check mode
def test_parity_cases_under_memcheck(tmp_path):
    if os.environ.get("SP_MEMCHECK_OUT"):
        pytest.skip("already running under the memory-check mode")
    out = tmp_path / "memcheck.json"
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "tests"), ROOT] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    env["SP_MEMCHECK_OUT"] = str(out)
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "memcheck_plugin", "-p", "no:cacheprovider", "-k", "parity and not memcheck",
           os.path.join(ROOT, "tests", "test_gpu_poly_commit_limits.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-20000:]
    tot = json.load(open(out))
    assert tot["violations"] == 0, tot
    assert tot["blocks_filled"] > 0 and tot["context_refills"] > 0, tot
