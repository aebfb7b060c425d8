"""Every entry of the generator tables, checked directly, and every generator reached at its extreme digits.

A commitment reads one table entry per generator, window and digit its scalars hit, so most entries of a large set are never read by any other
test.  Here (libsp_devtest.so, spd_gen_set_check) each production set is built through GenSet's own constructors and every entry it holds is
compared with its value computed from the generator itself (k_niels_check: doublings, double-and-add and one mixed addition per entry, compared
by cross-multiplication, coordinates required canonical): the per-window table at the width the set chose, the row table, and the radix-2^51
host copies the sigma protocols use, including those a smaller view adds later.  Every generator is compared with the oracle's encoding, and the
set's window width and row-table choice with prover.cpp's rule for the free memory at the build.  A self-test plants defects in a copy of a table
and requires the checker to name exactly the entries changed.  Last, commitments whose every non-top digit is an extreme of the recoding, for
every generator and the blind generator h, on the row-table path and on the per-window path at W = 8, 13 and 15, are compared with the oracle.

Sets are built one at a time and freed before the next; a case the free device memory cannot hold is skipped with the bytes it needs.
Run on the GPU: pytest -m gpu -s tests/test_gpu_gen_table_entries.py (-s shows the per-case report)."""
import ctypes as C
import os
import sys

import pytest

from oracle.spartan_ref import core as oc
from test_gen_table_digits import P, niels_bytes, niels_dbl, niels_from_bytes, niels_neg, nwin, table_scalars

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NIELS, GE = 96, 128
ROW_DEPTH = 1 << 15
CHECK_OUT = 24
_sz, _vp, _i64p, _u64p = C.c_size_t, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_uint64)


def depth(W):
    return 1 << (W - 1)


def table_bytes(n, W):
    return n * nwin(W) * depth(W) * NIELS


def row_bytes(n):
    return n * ROW_DEPTH * NIELS


def width_rule(n, free, forced):
    """GenSet::finish (prover.cpp): the row table for >= 512 generators when it fits in 65 % of the free bytes, then the widest window table that
    fits in 65 % of what is left (15 bits only from 2048 generators on); below 512 generators always 8 bits; SP_MSM_WINDOW forces a width"""
    row = n >= 512 and row_bytes(n) <= 0.65 * free
    left = free - (row_bytes(n) if row else 0)
    if n < 512:
        return 8, row
    if forced:
        return forced, row
    fits = lambda W: table_bytes(n, W) <= 0.65 * left  # noqa: E731
    return (15 if n >= 2048 and fits(15) else 13 if fits(13) else 8), row


# ---- host bases of the views (prover.cpp R1CSGens::host_bases, snark.cpp SparkDims::host_bases)
def log2_ceil(x):
    return (x - 1).bit_length()


def r1cs_host(nvp):
    ell = log2_ceil(nvp)
    n = 1 << (ell - ell // 2)
    return [0, 1, 2, 3, 4, n, n + 1]


def spark_host(num_cons, nvp, nnz):
    x, y, lgnz = log2_ceil(num_cons), log2_ceil(2 * nvp), log2_ceil(nnz)
    v = [lgnz + 4, max(x, y) + 1, lgnz + 3]
    return [b for k in v for b in ((1 << (k - k // 2)), (1 << (k - k // 2)) + 1)]


SAT, EVAL = b"gens_r1cs_sat", b"gens_r1cs_eval"
N20, N22 = 1 << 20, 1 << 22
# id: label, generators, forced width, host bases at the build, host bases views add later, the (width, row table) an 80 GB GPU gives
CASES = {
    "2p20_r1cs": (SAT, 1026, None, r1cs_host(N20), r1cs_host(1 << 16) + r1cs_host(1 << 18), (13, True)),
    "2p20_spark": (EVAL, 4098, None, spark_host(N20, N20, N20), spark_host(1 << 16, 1 << 16, 1 << 16), (13, True)),
    "2p22_r1cs": (SAT, 2050, None, r1cs_host(N22), r1cs_host(N20), (13, True)),
    "2p22_spark": (EVAL, 8194, None, spark_host(N22, N22, N22), spark_host(N20, N20, N20), (8, True)),
    "1026_w15": (SAT, 1026, 15, r1cs_host(N20), [], (15, True)),
    "513_w8": (EVAL, 513, 8, [0, 1, 511, 512], [2, 3, 4, 513, 700], (8, True)),
    "511": (EVAL, 511, None, [0, 1, 509, 510], [2, 3, 4, 511], (8, False)),
    "5": (SAT, 5, None, r1cs_host(4), [], (8, False)),
    "6": (SAT, 6, None, r1cs_host(16), r1cs_host(4), (8, False)),
    "18": (EVAL, 18, None, spark_host(128, 16, 16), spark_host(16, 16, 16), (8, False)),
}
UPLOAD_N = 520   # generators of the uploaded set, h included: above the row-table threshold


@pytest.fixture(scope="module")
def dt():
    lib = C.CDLL(os.path.join(ROOT, "spartan_b200", "libsp_devtest.so"))
    lib.spd_last_error.restype = C.c_char_p
    lib.spd_niels_table_check.argtypes = [_vp, _sz, C.c_int, _vp, _i64p, _u64p]
    lib.spd_gen_set_check.argtypes = [C.c_char_p, _sz, _sz, C.c_char_p, _i64p, _sz, _i64p, _sz, C.c_char_p, _i64p, _i64p, _u64p,
                                      C.POINTER(C.c_double)]
    lib.spd_gen_table_copy.argtypes = [C.c_char_p, _sz, _sz, C.c_int, _vp, _sz, _vp, _i64p]
    return lib


@pytest.fixture(scope="module")
def oracle_enc():
    """the oracle's generator encodings (G then h of MultiCommitGens::new) of the largest set of each label; smaller sets are prefixes"""
    oc.lib.oracle_set_threads(max(1, (os.cpu_count() or 2) // 2))
    out = {}
    for label, n in ((SAT, 2050), (EVAL, 8194)):
        g = oc.MultiCommitGens.new(n - 1, label)
        out[label] = [g.g(i).compress() for i in range(n - 1)] + [g.h.compress()]
    return out


def release_cached():
    """hand every cached device block of this process back to the driver, so that the free memory a case sees is the GPU's"""
    if "spartan_b200" in sys.modules:
        sys.modules["spartan_b200"].release_cached_memory()
    if "torch" in sys.modules and sys.modules["torch"].cuda.is_initialized():
        sys.modules["torch"].cuda.empty_cache()


def free_bytes():
    import torch
    release_cached()
    return torch.cuda.mem_get_info()[0]


def need_or_skip(what, need):
    free = free_bytes()
    if free < need:
        pytest.skip("%s needs %d bytes of free device memory, %d are free" % (what, need, free))


def i64(vals):
    return (C.c_int64 * max(1, len(vals)))(*vals)


def report(out):
    """the 24-word report of one check as a dict"""
    o = list(out)
    return {"entries": o[0], "bad": o[1], "ypx": o[2], "ymx": o[3], "t2d": o[4], "noncanon": o[5], "listed": o[8:8 + o[6]], "exact": o[7]}


def gen_set_check(dt, label, n, host, extra, enc=None):
    G_enc = C.create_string_buffer(32 * n)
    info = (C.c_int64 * 6)()
    checked = (C.c_int64 * max(1, len(host) + len(extra)))()
    out = (C.c_uint64 * (3 * CHECK_OUT))()
    ms = (C.c_double * 2)()
    rc = dt.spd_gen_set_check(label, len(label), n, b"".join(enc) if enc else None, i64(host), len(host), i64(extra), len(extra), G_enc, info,
                              checked, out, ms)
    assert rc == 0, (rc, dt.spd_last_error())
    reps = [report(out[k * CHECK_OUT:(k + 1) * CHECK_OUT]) for k in range(3)]
    return {"W": info[0], "row": bool(info[1]), "free": info[2], "total": info[3], "bytes": info[4], "checked": list(checked[:info[5]]),
            "G": [G_enc.raw[32 * i:32 * i + 32] for i in range(n)], "table": reps[0], "rows": reps[1], "host": reps[2], "ms": (ms[0], ms[1])}


def expected_host(n, host, extra):
    want = []
    for b in host + extra:
        if b < n and b not in want:
            want.append(b)
    return want


def check_set(dt, case_id, label, n, forced, host, extra, nominal, want_G, enc=None):
    r = gen_set_check(dt, label, n, host, extra, enc)
    W, row = r["W"], r["row"]
    print("\n%-11s nbases %5d  W %2d  row table %-3s  entries: window %11d  row %11d  host %7d (%d bases)  bad %d/%d/%d  build %.0f ms  check %.0f ms"
          % (case_id, n, W, "yes" if row else "no", r["table"]["entries"], r["rows"]["entries"], r["host"]["entries"], len(r["checked"]),
             r["table"]["bad"], r["rows"]["bad"], r["host"]["bad"], r["ms"][0], r["ms"][1]))
    rules = {width_rule(n, r["free"] * f, forced) for f in (0.99, 1.0, 1.01)}
    if len(rules) == 1:   # else the free memory at the build was within 1 % of a threshold of the rule: either choice is the rule's
        assert (W, row) == rules.pop(), (case_id, W, row, r["free"])
    assert (W, row) == nominal, "%s: width %d, row table %s on %d free bytes" % (case_id, W, row, r["free"])
    assert r["table"]["entries"] == n * nwin(W) * depth(W)
    assert r["rows"]["entries"] == (n * ROW_DEPTH if row else 0)
    assert r["checked"] == expected_host(n, host, extra)
    assert r["host"]["entries"] == len(r["checked"]) * 32 * 128
    for kind in ("table", "rows", "host"):
        assert r[kind]["bad"] == 0, "%s: %s: %s" % (case_id, kind, r[kind])
    assert r["bytes"] == n * GE + (r["table"]["entries"] + r["rows"]["entries"]) * NIELS
    bad = [i for i in range(n) if r["G"][i] != want_G[i]]
    assert not bad, "%s: %d generators differ from the oracle, first %d" % (case_id, len(bad), bad[0])


def case_need(n, forced, nominal):
    """free bytes under which the nominal choice cannot be made"""
    W, row = nominal
    rb = row_bytes(n) if row else 0
    if forced:
        return int(rb / 0.65) if rb else 0, rb + table_bytes(n, W) + (1 << 30)
    if n < 512 or W == 8:
        return int(rb / 0.65) + table_bytes(n, 8), 0
    return int(rb / 0.65), rb + int(table_bytes(n, W) / 0.65)


# ---------------------------------------------------------------------------------------------------- (a), (b): production sets
@pytest.mark.parametrize("case_id", list(CASES))
def test_production_set_entries(dt, oracle_enc, case_id, monkeypatch):
    """every entry of the per-window table, the row table and the host copies (the build's and a view's) of one production set is right, every
    generator is the oracle's, and the width and row table are prover.cpp's choice"""
    label, n, forced, host, extra, nominal = CASES[case_id]
    if forced:
        monkeypatch.setenv("SP_MSM_WINDOW", str(forced))
    else:
        monkeypatch.delenv("SP_MSM_WINDOW", raising=False)
    need_or_skip("%s (%d generators, W = %d%s)" % (case_id, n, nominal[0], ", row table" if nominal[1] else ""), max(case_need(n, forced, nominal)))
    check_set(dt, case_id, label, n, forced, host, extra, nominal, oracle_enc[label])


def test_uploaded_set_entries(dt, monkeypatch):
    """a set of caller generators through the upload constructor (sp_gens_upload's path): the oracle's MultiCommitGens::scale output, with host
    copies added afterwards"""
    monkeypatch.delenv("SP_MSM_WINDOW", raising=False)
    need_or_skip("the uploaded set", max(case_need(UPLOAD_N, None, (13, True))))
    ref = oc.MultiCommitGens.new(UPLOAD_N - 1, b"upload-entries").scale(0x1234567890abcdef)
    enc = [ref.g(i).compress() for i in range(UPLOAD_N - 1)] + [ref.h.compress()]
    check_set(dt, "upload", b"", UPLOAD_N, None, [], [0, 1, 2, 3, 4, UPLOAD_N - 2, UPLOAD_N - 1], (13, True), enc, enc)


# ---------------------------------------------------------------------------------------------------- (c): the checker can fail
SELF = {"window8": (6, 0, 8), "row": (513, 1, 0)}   # generators, which table, layout (0: row)
SELF_LABEL = b"table-self-test"


@pytest.mark.parametrize("layout", list(SELF))
def test_checker_names_each_planted_defect(dt, layout, monkeypatch):
    """a copy of a real table: clean, no bad entry; with one defect planted at the first and last generator (h), the first and last window and
    the first and last digit, exactly the entries changed are reported: an entry swapped with its neighbour, negated, taken from another generator,
    one coordinate off by p, and a whole window shifted by one doubling"""
    import torch
    n, row, W = SELF[layout]
    monkeypatch.setenv("SP_MSM_WINDOW", "8")
    nw, D = (nwin(W), depth(W)) if W else (1, ROW_DEPTH)
    entries = n * nw * D
    need_or_skip("the %s self-test" % layout, 3 * entries * NIELS + (row_bytes(n) if row else 0) + (1 << 30))
    tab = torch.empty((entries, NIELS), dtype=torch.uint8, device="cuda")
    G = torch.empty((n, GE), dtype=torch.uint8, device="cuda")
    info = (C.c_int64 * 2)()
    torch.cuda.synchronize()
    assert dt.spd_gen_table_copy(SELF_LABEL, len(SELF_LABEL), n, row, tab.data_ptr(), entries, G.data_ptr(), info) == 0, dt.spd_last_error()
    assert (info[0], info[1]) == (8, entries)
    clean = tab.clone()
    torch.cuda.synchronize()

    def check():
        torch.cuda.synchronize()
        out = (C.c_uint64 * CHECK_OUT)()
        assert dt.spd_niels_table_check(tab.data_ptr(), n, W, G.data_ptr(), None, out) == 0, dt.spd_last_error()
        return report(out)

    def idx(j, w, d):
        return (j * nw + w) * D + d - 1

    def get(i):
        return niels_from_bytes(bytes(tab[i].cpu().numpy()))

    def put(i, nl):
        tab[i] = torch.frombuffer(bytearray(niels_bytes(nl)), dtype=torch.uint8).to("cuda")

    r = check()
    assert r["entries"] == entries and r["bad"] == 0, r
    planted = 0
    for j in (0, n - 1):
        for w in sorted({0, nw - 1}):
            for d in (1, D):
                i = idx(j, w, d)
                nb = idx(j, w, d + 1 if d < D else d - 1)
                other = idx(j + 1 if j + 1 < n else j - 1, w, d)
                defects = {
                    "swap": lambda: (tab.index_copy_(0, torch.tensor([i, nb], device="cuda"), clean[[nb, i]]), [i, nb]),
                    "negated": lambda: (put(i, niels_neg(get(i))), [i]),
                    "other generator": lambda: (tab[i].copy_(clean[other]), [i]),
                    "off by p": lambda: (put(i, tuple(c + P if k == (j + w + d) % 3 else c for k, c in enumerate(get(i)))), [i]),
                }
                if d == 1:   # one per (generator, window)
                    def shift():
                        lo = idx(j, w, 1)
                        win = bytes(tab[lo:lo + D].cpu().numpy())
                        dbl = b"".join(niels_bytes(niels_dbl(niels_from_bytes(win[NIELS * k:NIELS * (k + 1)]))) for k in range(D))
                        tab[lo:lo + D] = torch.frombuffer(bytearray(dbl), dtype=torch.uint8).to("cuda").view(D, NIELS)
                        return None, list(range(lo, lo + D))
                    defects["window shifted by one doubling"] = shift
                for name, plant in defects.items():
                    tab.copy_(clean)
                    _, changed = plant()
                    r = check()
                    where = "%s at (j %d, w %d, d %d)" % (name, j, w, d)
                    assert r["bad"] == len(changed) and r["exact"] == 1, (where, r)
                    assert r["listed"] == sorted(changed)[:16], (where, r)
                    if name == "off by p":
                        assert r["noncanon"] == 1 and r["ypx"] == r["ymx"] == r["t2d"] == 0, (where, r)
                    planted += 1
    tab.copy_(clean)
    assert check()["bad"] == 0
    print("\nself-test %s: %d generators, %d entries, %d planted defects each reported at exactly the entries changed" % (layout, n, entries, planted))
    del tab, G, clean
    release_cached()


# ---------------------------------------------------------------------------------------------------- (d): every generator at its extreme digits
D_LABEL = b"gen-table-digits"
D_SIZES = (1024, 4096)


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as m
    m.default_context()
    return m


@pytest.fixture(scope="module")
def extreme_commitments():
    """the oracle's commitments of the extreme-digit tables: 64 rows of n (16-bit digits, the row tables) and 4 rows of n for W = 8, 13, 15"""
    oc.lib.oracle_set_threads(max(1, (os.cpu_count() or 2) // 2))
    out = {}
    for n in D_SIZES:
        ref = oc.MultiCommitGens.new(n, D_LABEL)
        for W, L in ((16, 64), (8, 4), (13, 4), (15, 4)):
            Z, blinds = table_scalars(W, L, n)
            Za = oc.to_arr(Z)
            out[(n, W)] = (Za, oc.to_arr(blinds), oc.commit_rows(Za, L, n, blinds, ref))
    return out


@pytest.mark.parametrize("n", D_SIZES)
@pytest.mark.parametrize("window", [8, 13, 15])
def test_every_generator_at_extreme_digits(sb, extreme_commitments, n, window, monkeypatch):
    """sp_gens_create(label, n) under SP_MSM_WINDOW = window; sp_commit_rows of 64 x n (the row-table path) and of 4 x n (k_msm_rows on the
    window tables) on the extreme-digit scalars, blinds on h, equal the oracle's commitments byte for byte"""
    monkeypatch.setenv("SP_MSM_WINDOW", str(window))
    need_or_skip("%d generators at W = %d" % (n + 1, window), row_bytes(n + 1) + table_bytes(n + 1, window) + (2 << 30))
    g = sb.MultiCommitGens(n, D_LABEL)
    try:
        for W, L in ((16, 64), (window, 4)):
            Z, blinds, want = extreme_commitments[(n, W)]
            got = sb.DensePolynomial(Z).commit(g, L, n, blinds)
            bad = [i for i in range(L) if got[i] != want[i]]
            assert not bad, "n %d, W %d, %d rows (%s): %d rows differ from the oracle, first %d" % (
                n, window, L, "row tables" if L == 64 else "window tables", len(bad), bad[0])
    finally:
        del g
        release_cached()
    print("\nextreme digits: %d generators + h, W %d: 64 x %d on the row tables and 4 x %d on the window tables equal the oracle" % (n, window, n, n))

