"""GPU parity (operator level): every kernel family called through the C-ABI and compared bit for bit with the oracle
(oracle/ = CPU restatement of the reference) on the same seeded inputs.  Run on the GPU: pytest -m gpu."""
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle.spartan_ref import core as oc  # noqa: E402


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as m
    m.default_context()
    return m


def edge_table(n, tag):
    """seeded table with the field's edge values planted: 0, 1, q-1, R, R^2 (SURVEY §7 step 4)"""
    t = oc.prg_scalars(tag, n)
    edges = oc.to_arr([0, 1, oc.Q - 1, oc.R_MONT, oc.R_MONT * oc.R_MONT % oc.Q, 2, oc.Q - 2])
    for k in range(min(n, len(edges))):
        t[(k * 7) % n] = edges[k]
    return t


@pytest.mark.parametrize("logn", [1, 2, 3, 5, 8, 10, 13, 16])
def test_fold_top(sb, logn):
    from spartan_b200 import api
    n = 1 << logn
    tabs = [edge_table(n, "f%d" % k) for k in range(3)]
    r = oc.arr_get(oc.prg_scalars("r", 1, logn), 0)
    polys = [sb.DensePolynomial(t) for t in tabs]
    api.fold_top(polys, oc.to_arr([r])[0])
    for t, p in zip(tabs, polys):
        want = oc.bound_top(t.copy(), r)
        assert p.len() == n // 2
        assert np.array_equal(p.to_numpy(), want)


@pytest.mark.parametrize("kind,nt", [(0, 2), (1, 3), (2, 4)])
@pytest.mark.parametrize("logn", [1, 2, 4, 9, 12, 17])
def test_sumcheck_eval_and_fused_fold_eval(sb, kind, nt, logn):
    """sumcheck.rs:460-469 / :204-228 / :625-652 round polynomials, then the whole chain of rounds through the fused kernel"""
    from spartan_b200 import api
    n = 1 << logn
    tabs = [edge_table(n, "sc%d_%d" % (kind, k)) for k in range(nt)]
    polys = [sb.DensePolynomial(t) for t in tabs]

    def oracle_eval(ts):
        if kind == 0:
            e0, e2 = oc.sc_eval_quad(ts[0], ts[1])
            return [e0, e2, 0]
        return oc.sc_eval_cubic(ts[0], ts[1], ts[2], ts[3] if kind == 2 else None)
    got = oc.to_ints(api.sumcheck_eval(kind, polys))
    assert got == oracle_eval(tabs)
    cur = [t.copy() for t in tabs]
    for j in range(logn - 1):
        r = oc.arr_get(oc.prg_scalars("rr", 1, 100 * logn + j), 0)
        got = oc.to_ints(api.sumcheck_fold_eval(kind, polys, oc.to_arr([r])[0]))
        cur = [oc.bound_top(t, r) for t in cur]
        assert got == oracle_eval(cur), (logn, j)
        if j in (0, logn - 2):
            for p, t in zip(polys, cur):
                assert np.array_equal(p.to_numpy()[: len(t)], t)


@pytest.mark.parametrize("ell", [0, 1, 2, 5, 10, 11, 15, 18])
def test_eq_evals(sb, ell):
    r = oc.to_ints(oc.prg_scalars("eq", ell, ell)) if ell else []
    if ell >= 2:
        r[0], r[1] = 0, 1
    got = sb.DensePolynomial.eq_evals(oc.to_arr(r) if ell else np.zeros((0, 4), dtype=np.uint64)).to_numpy()
    assert np.array_equal(got, oc.eq_evals(r))


def test_known_answer_evaluate(sb):
    """dense_mlpoly.rs:434-452: Z = [1,2,1,4], r = [4,3] -> 28"""
    Z = oc.to_arr([1, 2, 1, 4])
    p = sb.DensePolynomial(Z)
    assert oc.to_ints(p.evaluate(oc.to_arr([4, 3]))[None, :]) == [28]


@pytest.mark.parametrize("ell", [2, 7, 12, 16])
def test_evaluate_bound_dot(sb, ell):
    n = 1 << ell
    Z = edge_table(n, "Z%d" % ell)
    r = oc.to_ints(oc.prg_scalars("pt", ell, ell))
    p = sb.DensePolynomial(Z)
    assert oc.to_ints(p.evaluate(oc.to_arr(r))[None, :]) == [oc.evaluate(Z, r)]
    lv = ell // 2
    L_size, R_size = 1 << lv, 1 << (ell - lv)
    Lv = oc.eq_evals(r[:lv])
    assert np.array_equal(p.bound(Lv).to_numpy(), oc.bound_rows(Z, Lv, L_size, R_size))
    W = oc.prg_scalars("W", n, ell)
    assert oc.to_ints(p.dot(sb.DensePolynomial(W))[None, :]) == [oc.dot(Z, W)]


def test_generators_and_point_codec(sb):
    """MultiCommitGens::new (commitments.rs:15-33): SHAKE256 -> one-way map on the device, compared as compressed points"""
    from spartan_b200 import api
    n = 70
    g = sb.MultiCommitGens(n, b"gens_r1cs_sat")
    mine = g.export()
    ref = oc.MultiCommitGens.new(n, b"gens_r1cs_sat")
    assert mine[:n] == [ref.g(i).compress() for i in range(n)]
    assert mine[n] == ref.h.compress()
    assert api.point_roundtrip(mine) == mine
    bad = [hashlib.sha256(b"bad%d" % i).digest() for i in range(64)] + [bytes(32), b"\x01" + bytes(31), b"\xff" * 32]
    assert api.point_decompress_check(bad) == [oc.Point.decompress(b) is not None for b in bad]


@pytest.mark.parametrize("n", [1, 2, 5, 33, 190, 1024, 4096])
def test_msm(sb, n):
    """vartime_multiscalar_mul (group.rs:98-117) through the fixed-base window kernel"""
    g = sb.MultiCommitGens(n, b"msm-test")
    ref = oc.MultiCommitGens.new(n, b"msm-test")
    sc = oc.prg_scalars("msm", n, n)
    sc[0] = 0
    if n > 4:
        sc[1] = oc.to_arr([1])[0]
        sc[2] = oc.to_arr([oc.Q - 1])[0]
        sc[3] = oc.to_arr([128])[0]          # window-carry edge of the signed 8-bit recoding
        sc[4] = oc.to_arr([(1 << 252) + 129])[0]
    assert g.msm(sc) == oc.msm(sc, ref.G).compress()
    small = oc.from_u64(np.arange(n, dtype=np.uint64) % 3)   # the 0/1/2-valued vectors that dominate in-protocol
    assert g.msm(small) == oc.msm(small, ref.G).compress()


@pytest.mark.parametrize("L,R", [(1, 4), (2, 2), (32, 32), (64, 128), (16, 1024)])
def test_commit_rows(sb, L, R):
    """DensePolynomial::commit_inner (dense_mlpoly.rs:148-177)"""
    g = sb.MultiCommitGens(R, b"rows-test")
    ref = oc.MultiCommitGens.new(R, b"rows-test")
    Z = edge_table(L * R, "rows%d_%d" % (L, R))
    blinds = oc.prg_scalars("bl", L, L * R)
    p = sb.DensePolynomial(Z)
    assert p.commit(g, L, R, blinds) == oc.commit_rows(Z, L, R, oc.to_ints(blinds), ref)
    assert p.commit(g, L, R, None) == oc.commit_rows(Z, L, R, [0] * L, ref)
    # linearity (size-independent property): commit(a)+commit(b) == commit(a+b) row-wise
    Z2 = oc.prg_scalars("rows-b", L * R, 1)
    Zs = oc.to_arr([(a + b) % oc.Q for a, b in zip(oc.to_ints(Z[: 4 * R if L >= 4 else L * R]), oc.to_ints(Z2[: 4 * R if L >= 4 else L * R]))])
    rows = len(Zs) // R
    ca = sb.DensePolynomial(Z[: rows * R]).commit(g, rows, R)
    cb = sb.DensePolynomial(Z2[: rows * R]).commit(g, rows, R)
    cs = sb.DensePolynomial(Zs).commit(g, rows, R)
    for a, b, s in zip(ca, cb, cs):
        assert (oc.Point.decompress(a) + oc.Point.decompress(b)).compress() == s


def test_gens_upload(sb):
    """sp_gens_upload: caller-supplied generators (here: the oracle's MultiCommitGens::scale output, commitments.rs:43-49) behave like derived ones"""
    from spartan_b200 import api
    n = 37
    ref = oc.MultiCommitGens.new(n, b"upload-test")
    k = 0x1234567890abcdef
    enc = [(ref.g(i) * k).compress() for i in range(n)] + [ref.h.compress()]
    g = sb.MultiCommitGens.from_points(enc)
    assert g.export() == enc
    sc = edge_table(n, "up")
    G = np.stack([oc.Point.decompress(e).buf for e in enc[:n]])
    assert g.msm(sc) == oc.msm(sc, G).compress()
    p = sb.DensePolynomial(edge_table(4 * 8, "upc"))
    blinds = oc.prg_scalars("upb", 4, 1)
    want = [(oc.msm(p.to_numpy()[8 * i:8 * i + 8], G) + oc.Point.decompress(enc[n]) * oc.to_ints(blinds)[i]).compress() for i in range(4)]
    assert p.commit(g, 4, 8, blinds) == want
    bad = list(enc)
    bad[3] = hashlib.sha256(b"bad0").digest()
    with pytest.raises(api.SpartanB200Error, match="error 8"):
        sb.MultiCommitGens.from_points(bad)


@pytest.mark.parametrize("ninst", [5, 24])
@pytest.mark.parametrize("logn", [2, 5, 11, 14, 16])
def test_sumcheck_batched(sb, logn, ninst):
    """prove_cubic_batched's loops (sumcheck.rs:290-357): 5 or 24 (SC_MAX_INST) instances, several of them sharing one C table (poly_C_par),
    whole chain of rounds; 25 instances are refused"""
    from spartan_b200 import api
    n = 1 << logn
    A = [edge_table(n, "ba%d" % i) for i in range(ninst)]
    B = [edge_table(n, "bb%d" % i) for i in range(ninst)]
    Cs = [edge_table(n, "bc%d" % i) for i in range(3)]
    cmap = [0, 0, 1, 0, 2] + [k % 3 for k in range(ninst - 5)]
    dA, dB = [sb.DensePolynomial(t) for t in A], [sb.DensePolynomial(t) for t in B]
    dC = [sb.DensePolynomial(t) for t in Cs]
    got = api.sumcheck_batched_eval(dA, dB, [dC[k] for k in cmap])
    for i in range(ninst):
        assert oc.to_ints(got[i]) == oc.sc_eval_cubic(A[i], B[i], Cs[cmap[i]], None)
    for j in range(logn - 1):
        r = oc.arr_get(oc.prg_scalars("br", 1, j), 0)
        A = [oc.bound_top(t, r) for t in A]; B = [oc.bound_top(t, r) for t in B]; Cs = [oc.bound_top(t, r) for t in Cs]
        got = api.sumcheck_batched_fold_eval(dA, dB, [dC[k] for k in cmap], oc.to_arr([r])[0])
        for i in range(ninst):
            assert oc.to_ints(got[i]) == oc.sc_eval_cubic(A[i], B[i], Cs[cmap[i]], None), (j, i)
        assert all(p.len() == len(A[0]) for p in dA + dB + dC)
    for t, p in zip(A + B + Cs, dA + dB + dC):
        assert np.array_equal(p.to_numpy(), t)
    with pytest.raises(api.SpartanB200Error):
        api.sumcheck_batched_eval([dA[0], dA[0]], dB[:2], dC[:2])
    over = [dA[k % ninst] for k in range(25)]
    with pytest.raises(api.SpartanB200Error):
        api.sumcheck_batched_eval(over, [dB[k % ninst] for k in range(25)], [dC[k % 3] for k in range(25)])
    with pytest.raises(api.SpartanB200Error):
        api.sumcheck_batched_fold_eval(over, [dB[k % ninst] for k in range(25)], [dC[k % 3] for k in range(25)], oc.to_arr([3])[0])


@pytest.mark.parametrize("n", [2, 32, 1024, 4096])
def test_bullet_reduction_operator_level(sb, n):
    """BulletReductionProof::prove (nizk/bullet.rs:32-132) driven from the host through sp_ipa_begin / sp_ipa_round_LR / sp_ipa_fold /
    sp_ipa_finish with the oracle's transcript: every L, R, the final a, b and G[0] equal the oracle's.  The rounds run the prover's own launches
    (IpaRound: k_ipa_msm_quad with its fused dot products, then k_ipa_fold_update; RowSum for G[0]).  n >= 512 runs the 13-bit-window
    instance of k_ipa_msm_quad (the generator set of the 2^20 proofs), n = 32 the 8-bit one."""
    from spartan_b200 import api
    from oracle.spartan_ref import protocol as pr
    lg = n.bit_length() - 1
    g = sb.MultiCommitGens(n, b"ipa-test")
    ref = oc.MultiCommitGens.new(n, b"ipa-test")
    a = oc.prg_scalars("ipa-a", n, n)
    b = oc.prg_scalars("ipa-b", n, n + 1)
    if n >= 32:
        a[0] = 0; a[1] = oc.to_arr([1])[0]; b[3] = 0
    blinds = [(int(x), int(y)) for x, y in zip(oc.to_ints(oc.prg_scalars("bl1", lg, n)), oc.to_ints(oc.prg_scalars("bl2", lg, n)))]
    Qp = ref.g(0) * 12345
    H = ref.h
    To = oc.Transcript(b"ipa")
    want, _, a_hat, b_hat, G_hat, _ = pr.BulletReductionProof.prove(To, Qp, ref.G, H, oc.to_ints(a), oc.to_ints(b), 7, blinds)
    T = oc.Transcript(b"ipa")
    red = api.BulletReduction(g, sb.DensePolynomial(a), sb.DensePolynomial(b))
    for k in range(lg):
        L, R = red.round_LR(Qp.compress(), H.compress(), oc.to_arr([blinds[k][0]])[0], oc.to_arr([blinds[k][1]])[0])
        assert (L, R) == (want.L_vec[k], want.R_vec[k]), "round %d" % k
        T.append_point(b"L", L); T.append_point(b"R", R)
        u = T.challenge_scalar(b"u")
        red.fold(oc.to_arr([u])[0], oc.to_arr([oc.inv(u)])[0])
    ga, gb, gG = red.finish()
    assert oc.to_ints(ga[None, :]) == [a_hat] and oc.to_ints(gb[None, :]) == [b_hat] and gG == G_hat.compress()
