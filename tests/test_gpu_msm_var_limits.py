"""The variable-base MSM (kernels_pip.cu, through sp_msm_var and sp_msm_var_resident) on every launch plan pip_plan makes: each default window
width from 2^13 to 2^23 points, each override width 2..16 over several tiles, lane groups G = 16 and 32 and the S cap, each under the scalar
distributions aimed at one branch (skewed, empty windows, the extreme digits, buckets of exactly S - 1 .. 2S + 1 entries).  Also the range
edges of a point set, one set reused by growing and shrinking plans, the launch count of a call, and the refusal of ranges whose offset + n
wraps past 2^64.

The plans come from the mirror in tests/test_pip_model.py, which the CPU suite checks branch by branch; here each case first asserts that the
library's own pip_plan (spd_pip_plan) is the plan the mirror picked.

Judge: point i of a set is P_idx[i] = a_idx[i] B, one of 2^16 points built by the oracle (the identity, B, and pairs a, q - a), uploaded from
one buffer of encodings.  The expected sum is (sum_i k_i a_idx[i] mod q) B: one oracle dot product per case at any n, with no bucket logic in
it.  The construction is tied to the oracle's own MSM at 2^14, and the skewed distributions are also checked against oc.msm on derived points.
Run on the GPU: pytest -m gpu."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from test_pip_model import CASES, all_digits, case_dists, plan

pytestmark = pytest.mark.gpu
Q = oc.Q
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NPTS = 1 << 16
PLAN_FIELDS = ("c", "nwin", "nb", "tile", "ntiles", "G", "S", "max_items", "scratch")
LAUNCHES = 9        # k_pip_prepare, k_pip_count, k_pip_scan, k_pip_scatter, k_pip_accumulate, k_pip_bucket_sum, k_pip_window, k_pip_final, k_compress
SP_ERR_INVALID_ARG = 3


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as m
    m.default_context()
    return m


@pytest.fixture(autouse=True)
def release_cache(sb):
    """every test returns the device blocks its point sets, scalars and sort workspaces leave in the pool's cache: up to 2^23 points, with
    sizes that differ from case to case, they would otherwise stay with this process and starve the next test's (or another process's)
    allocations"""
    yield
    sb.release_cached_memory()


@pytest.fixture(scope="module")
def dt():
    lib = C.CDLL(os.path.join(ROOT, "spartan_b200", "libsp_devtest.so"))
    lib.spd_last_error.restype = C.c_char_p
    return lib


@pytest.fixture(scope="module")
def table():
    """a_j (ints and Montgomery limbs), the encodings of a_j B and the oracle's points, for j < 2^16: a_0 = 0 (the identity), a_1 = 1, then
    pairs (x, q - x) along a random walk x += d_t over 256 random steps d_t (one oracle addition per point)"""
    rng = np.random.default_rng(16)
    B = oc.Point.decompress(oc.BASEPOINT_COMPRESSED)
    steps = [int.from_bytes(rng.bytes(32), "little") % Q for _ in range(256)]
    step_pts = [B * d for d in steps]
    a, pts = [0, 1], [oc.Point.identity(), B]
    x, X = 0, oc.Point.identity()
    for t in rng.integers(0, 256, size=(NPTS - 2) // 2):
        x, X = (x + steps[t]) % Q, X + step_pts[t]
        a += [x, (Q - x) % Q]
        pts += [X, oc.Point.identity() - X]
    enc = np.frombuffer(b"".join(p.compress() for p in pts), dtype=np.uint8).reshape(NPTS, 32)
    return dict(a=a, A=oc.to_arr(a), enc=enc, G=oc.points_array(pts), B=B)


def upload(sb, table, idx):
    """the point set P_idx[0], P_idx[1], ... through sp_points_upload from one contiguous buffer"""
    from spartan_b200 import api
    ctx = api.default_context()
    buf = np.ascontiguousarray(table["enc"][idx]).tobytes()
    h = C.c_void_p()
    ctx.check(api.lib.sp_points_upload(ctx.h, C.c_char_p(buf), C.c_size_t(len(idx)), C.byref(h)))
    P = api.Points.__new__(api.Points)
    P.ctx, P.h = ctx, h
    return P


def expected(table, K, idx):
    return (table["B"] * oc.dot(K, table["A"][idx])).compress()


def lib_plan(dt, n, c):
    out = (C.c_uint64 * 9)()
    assert dt.spd_pip_plan(C.c_size_t(n), C.c_int(c), out) == 0, dt.spd_last_error()
    return dict(zip(PLAN_FIELDS, (int(v) for v in out)))


def msm(sb, P, K, c=0, resident=False, offset=0):
    """P.msm under SP_PIP_WINDOW = c (0: the default width), and the launches it made"""
    from spartan_b200 import api
    arg = sb.DensePolynomial(K) if resident else K
    if c:
        os.environ["SP_PIP_WINDOW"] = str(c)
    try:
        before = api.kernel_launches()
        got = P.msm(arg, offset=offset)
        return got, api.kernel_launches() - before
    finally:
        os.environ.pop("SP_PIP_WINDOW", None)


# ---------------------------------------------------------------------------------------------------- scalar distributions
def mont_of(vals, pick):
    """Montgomery limbs of vals[pick[i]] (a few distinct canonical values, indexed at any n)"""
    return oc.to_arr(vals)[pick]


def scalars(dist, n, p, rng):
    """n Montgomery scalars of the named distribution for plan p"""
    c, nb, S = p["c"], p["nb"], p["S"]
    if dist == "random":
        t = rng.integers(0, np.iinfo(np.uint64).max, size=(n, 4), dtype=np.uint64, endpoint=True)
        t[:, 3] &= np.uint64(0x0FFFFFFFFFFFFFFF)              # < 2^252 < q: reduced Montgomery limbs of some scalar
        return t
    if dist == "zero_one":
        return oc.from_u64(rng.integers(0, 2, size=n, dtype=np.uint64))
    if dist == "zero_one_two":
        return oc.from_u64(rng.integers(0, 3, size=n, dtype=np.uint64))
    if dist == "u64":
        return oc.from_u64(rng.integers(0, np.iinfo(np.uint64).max, size=n, dtype=np.uint64, endpoint=True))
    if dist == "all_equal":                                   # one hot bucket per window, split into n / S items
        return mont_of([int.from_bytes(rng.bytes(31), "little")], np.zeros(n, dtype=np.int64))
    if dist in ("digit_min", "digit_max"):                   # every signed digit -2^(c-1) (bucket nb - 1) / 2^(c-1) - 1 (bucket nb - 2)
        pats = [[-nb]] if dist == "digit_min" else [[nb - 1], [nb - 1, -nb]]
        vals = sorted({k for pt in pats for top in (0, 1, 2, nb - 1, nb) for k in [all_digits(c, pt, top)] if 0 <= k < Q})
        return mont_of(vals, rng.integers(0, len(vals), size=n))
    if dist == "bucket_sizes":                               # window 0 buckets of exactly S + 1, 2S + 1, S, S - 1 and 2S entries, the rest 0
        sizes = [S + 1, 2 * S + 1, S, S - 1, 2 * S]
        vals = sorted(v for v in {1, 2, nb // 2, nb - 2, nb - 1} if 1 <= v < nb)   # scalars in [1, nb): digit k in window 0, bucket k - 1
        pick = np.zeros(n, dtype=np.int64)
        at = 0
        for j, v in enumerate(vals):
            assert at + sizes[j] <= n
            pick[at:at + sizes[j]] = j + 1
            at += sizes[j]
        return mont_of([0] + vals, rng.permutation(pick))
    if dist == "half_hot":
        K = scalars("random", n, p, rng)
        K[rng.permutation(n)[: n // 2]] = oc.to_arr([int.from_bytes(rng.bytes(32), "little") % Q])[0]
        return K
    if dist == "negated":                                    # q - v for small and 64-bit v
        v = [int(x) for x in rng.integers(0, 1 << 62, size=2048)] + list(range(2048))
        return mont_of([(Q - x) % Q for x in v], rng.integers(0, len(v), size=n))
    raise ValueError(dist)


# ---------------------------------------------------------------------------------------------------- every plan
@pytest.mark.parametrize("name,n,c", CASES, ids=[x[0].replace(" ", "_") for x in CASES])
def test_plan_parity(sb, dt, table, name, n, c):
    """the plan the mirror picked for the case is the library's, and every distribution of the case gives the judged sum through both entries"""
    p = plan(n, c)
    assert lib_plan(dt, n, c) == {k: p[k] for k in PLAN_FIELDS}
    rng = np.random.default_rng([n, c])
    idx = rng.integers(0, NPTS, size=n)
    P = upload(sb, table, idx)
    for j, dist in enumerate(case_dists(n, c)):
        K = scalars(dist, n, p, rng)
        want = expected(table, K, idx)
        for resident in ((False, True) if j == 0 else (j % 2 == 1,)):
            got, launched = msm(sb, P, K, c, resident)
            assert got == want, (name, dist, resident)
            assert launched == LAUNCHES, (name, dist, launched)


def test_judge_matches_oracle_msm(sb, table):
    """the table construction against oc.msm: 2^14 points of the table, random and skewed scalars"""
    n = 1 << 14
    rng = np.random.default_rng(14)
    idx = rng.integers(0, NPTS, size=n)
    idx[:4] = [0, 1, 2, 3]                                   # the identity, B and a pair a, q - a
    P = upload(sb, table, idx)
    G = table["G"][idx]
    for dist in ("random", "all_equal", "digit_min", "negated"):
        K = scalars(dist, n, plan(n), rng)
        want = oc.msm(K, G).compress()
        assert expected(table, K, idx) == want, dist
        assert msm(sb, P, K)[0] == want, dist


@pytest.mark.parametrize("c", [0, 3, 10, 16])
def test_skewed_vs_oracle_on_derived_points(sb, c):
    """2^16 points of the b"msm-skew" generator stream against oc.msm, under the skewed distributions, at the default width and at 3, 10, 16"""
    from spartan_b200 import api
    n = 1 << 16
    P = api.Points.derive(n, b"msm-skew")
    G = oc.MultiCommitGens.new(n, b"msm-skew").G
    p = plan(n, c)
    rng = np.random.default_rng(c)
    for dist in ("all_equal", "half_hot", "bucket_sizes", "digit_min", "digit_max", "zero_one_two"):
        K = scalars(dist, n, p, rng)
        assert msm(sb, P, K, c)[0] == oc.msm(K, G).compress(), (c, dist)


# ---------------------------------------------------------------------------------------------------- ranges, reuse, launches
def test_range_edges(sb, table):
    """offset + n == len through both entries, n = 0 at offset == len (the identity, one launch: k_compress), export at the end"""
    L = 100003
    rng = np.random.default_rng(3)
    idx = rng.integers(0, NPTS, size=L)
    P = upload(sb, table, idx)
    for m in (1, 33, 4097, L):
        K = scalars("random", m, plan(m), rng)
        want = expected(table, K, idx[L - m:])
        assert msm(sb, P, K, offset=L - m)[0] == want, m
        assert msm(sb, P, K, offset=L - m, resident=True)[0] == want, m
    assert msm(sb, P, oc.zeros(0), offset=L) == (bytes(32), 1)
    assert P.export(L - 3, 3) == [bytes(table["enc"][j]) for j in idx[L - 3:]]
    assert P.export(L, 0) == []


def test_scratch_reused_by_growing_and_shrinking_plans(sb, table):
    """one point set through plans that grow and shrink, with and without SP_PIP_WINDOW: its sort scratch is allocated when a plan needs more
    and otherwise reused as the last call left it, without clearing"""
    n_max = 1 << 20
    rng = np.random.default_rng(20)
    idx = rng.integers(0, NPTS, size=n_max)
    P = upload(sb, table, idx)
    steps = [(1 << 12, 0, "random"), (1 << 20, 0, "all_equal"), (1 << 14, 0, "u64"), (1 << 18, 16, "digit_min"), (5000, 2, "half_hot"),
             (1 << 20, 0, "random"), (1 << 13, 5, "bucket_sizes"), (1 << 17, 13, "zero_one"), (1 << 16, 0, "digit_max")]
    have, reused, grown = 0, 0, 0
    for j, (n, c, dist) in enumerate(steps):
        p = plan(n, c)
        grown += p["scratch"] > have
        reused += p["scratch"] <= have
        have = max(have, p["scratch"])
        off = int(rng.integers(0, n_max - n + 1))
        K = scalars(dist, n, p, rng)
        got, launched = msm(sb, P, K, c, resident=j % 2 == 1, offset=off)
        assert got == expected(table, K, idx[off:off + n]), (n, c, dist)
        assert launched == LAUNCHES
    assert grown >= 3 and reused >= 4, (grown, reused)


# ---------------------------------------------------------------------------------------------------- ranges that wrap
def test_wrapping_ranges_refused(sb, table):
    """offset + n past 2^64 is refused with SP_ERR_INVALID_ARG before any launch, by sp_msm_var, sp_msm_var_resident and sp_points_export, and
    the set still works afterwards"""
    from spartan_b200 import api
    L = 4096
    rng = np.random.default_rng(64)
    idx = rng.integers(0, NPTS, size=L)
    P = upload(sb, table, idx)
    ctx = P.ctx
    out = C.create_string_buffer(32 * 4)
    top = (1 << 64) - 1

    def refused(rc, what):
        assert rc == SP_ERR_INVALID_ARG, rc
        assert api.lib.sp_last_error(ctx.h).decode() == "%s: range outside the point set" % what

    for n in (1, 3, 64):
        K = scalars("random", n, plan(n), rng)
        poly = sb.DensePolynomial(K)
        for off in {top, ((1 << 64) - n + 1) % (1 << 64), L - n + 1} - {0}:   # 2^64 - n + 1: offset + n wraps to 1 (for n = 1 that is offset 0)
            before = api.kernel_launches()
            refused(api.lib.sp_msm_var(ctx.h, P.h, C.c_size_t(off), K.ctypes.data_as(C.c_void_p), C.c_size_t(n), out), "msm_var")
            refused(api.lib.sp_msm_var_resident(ctx.h, P.h, C.c_size_t(off), poly.h, out), "msm_var")
            refused(api.lib.sp_points_export(ctx.h, P.h, C.c_size_t(off), C.c_size_t(n), out), "points_export")
            assert api.kernel_launches() == before, off
    K = scalars("random", 1, plan(1), rng)
    poly = sb.DensePolynomial(K)
    before = api.kernel_launches()
    for arg in (K, poly):
        with pytest.raises(api.SpartanB200Error, match="error 3: msm_var: range outside the point set"):
            P.msm(arg, offset=-1)
    with pytest.raises(api.SpartanB200Error, match="error 3: points_export: range outside the point set"):
        P.export(offset=-1, n=1)
    assert api.kernel_launches() == before
    assert msm(sb, P, K, offset=L - 1)[0] == expected(table, K, idx[L - 1:])
