"""A mirror of the variable-base MSM's launch plan (kernels_pip.cu pip_plan) and an integer model of its whole bucket pipeline, on the CPU.

Group elements are replaced by their discrete logs: the point a*B is the integer a mod q, so a mixed addition is an addition mod q, a negated
point is q - a and a doubling is 2a.  The model runs the algorithm exactly as the kernels split it: the offset C and the signed digits with the
top window unsigned (k_pip_prepare, pip_digit), the per-bucket counts (k_pip_count), items of at most S entries and istart as k_pip_scan computes
them with its 1024 threads of `per` buckets, the per-item sums (k_pip_accumulate, with its binary search and `last = first + S` clamp), the bucket
sums (k_pip_bucket_sum), k_pip_window's 512 chunks of `per` buckets with the lo * run correction, the c*w doublings and k_pip_final.  Its result
is compared with sum k_i a_i mod q.

CASES are the launch shapes tests/test_gpu_msm_var_limits.py runs on the GPU; test_every_branch_reached prints the plan the mirror gives each of
them and asserts that together they reach every branch of the plan (each window width 2..16, each lane count G, the S cap, several tiles with and
without the opt-in shared-memory histogram, a scan and a window sum whose threads own several buckets).  The GPU file checks that the library's
own pip_plan agrees with this mirror for every case, so a change to pip_plan cannot move a case off its branch unnoticed."""
import ctypes as C
import os
import random

import pytest

from oracle.spartan_ref import core as oc

Q = oc.Q
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHM_DEFAULT = 48 * 1024     # bytes of dynamic shared memory a launch gets without the opt-in attribute
GE = 128                    # sizeof(ge): X, Y, Z, T of 32 bytes each


# ---------------------------------------------------------------------------------------------------- mirror of pip_plan
def plan(n, c_override=0):
    """pip_plan(n, c_override) field by field, plus what the kernels derive from it"""
    lg = 0
    while (2 << lg) <= n:
        lg += 1
    c = min(max(lg - 7, 6), 16)
    if c_override:
        c = c_override
    if c < 2 or c > 16:
        raise ValueError("MSM window width out of range")
    nb = 1 << (c - 1)
    tile = max(nb * 4, 8192)
    ntiles = max(-(-n // tile), 1)
    G = 32
    while G > 1 and (n // nb) // G < 64:
        G >>= 1
    S = max(2 * (n // nb), G * 64)
    S = -(-S // 32) * 32
    s_capped = S > 8192
    S = min(S, 8192)
    p = dict(n=n, c=c, nwin=253 // c + 1, nb=nb, tile=tile, ntiles=ntiles, G=G, S=S, max_items=n // S + nb + 1)
    p.update(s_capped=s_capped, optin=nb * 4 > SHM_DEFAULT, scan_per=-(-nb // 1024), window_per=-(-nb // 512), scratch=scratch_bytes(p))
    return p


def scratch_bytes(p):
    """pip_layout(p).total: the sort workspace a point set keeps between calls"""
    al = lambda b: -(-b // 256) * 256
    n, nwin, nb = p["n"], p["nwin"], p["nb"]
    parts = [8 * n * 4, nwin * n * 4, nwin * nb * 4, nwin * p["ntiles"] * nb * 4, nwin * nb * 4, nwin * nb * 4, nwin * (nb + 1) * 4, nwin * 4,
             nwin * p["max_items"] * GE, nwin * nb * GE, nwin * GE]
    return sum(al(b) for b in parts)


# ---------------------------------------------------------------------------------------------------- digits
def offset_C(c, nwin):
    """C = sum_{w < nwin-1} 2^(c-1 + c*w): added to every scalar so each signed digit depends on its own window only"""
    return sum(1 << (c - 1 + c * w) for w in range(nwin - 1))


def limbs(kp):
    return [(kp >> (32 * j)) & 0xFFFFFFFF for j in range(8)]


def pip_digit(kl, w, c, nwin):
    """pip_digit on the eight 32-bit limbs of k' = k + C: two limbs when the window crosses a limb boundary, the top window unsigned"""
    b = w * c
    limb, sh = b >> 5, b & 31
    v = kl[limb] >> sh
    if sh + c > 32 and limb + 1 < 8:
        v |= (kl[limb + 1] << (32 - sh)) & 0xFFFFFFFF
    v &= (1 << c) - 1
    return v - (1 << (c - 1)) if w + 1 < nwin else v


def digits(k, c, nwin):
    kl = limbs((k + offset_C(c, nwin)) & ((1 << 256) - 1))   # k_pip_prepare keeps 256 bits
    return [pip_digit(kl, w, c, nwin) for w in range(nwin)]


def from_digits(ds, c):
    return sum(d << (c * w) for w, d in enumerate(ds))


def all_digits(c, pattern, top):
    """the scalar whose signed digits repeat `pattern` below a top digit `top`"""
    nwin = 253 // c + 1
    return from_digits([pattern[w % len(pattern)] for w in range(nwin - 1)] + [top], c)


def edge_scalars(c):
    """0, 1, q-1, 2^(c-1) +- 1, 2^c - 1, and the scalars whose every signed digit is -2^(c-1), 2^(c-1) - 1 or alternates between the two, under
    the smallest and largest top digits, those that keep them in [0, q)"""
    h = 1 << (c - 1)
    out = [0, 1, Q - 1, h - 1, h + 1, (1 << c) - 1]
    for pattern in ([-h], [h - 1], [-h, h - 1], [h - 1, -h]):
        for top in sorted({0, 1, 2, h - 1, h, h + 1}):
            k = all_digits(c, pattern, top)
            if 0 <= k < Q:
                out.append(k)
    return out


# ---------------------------------------------------------------------------------------------------- the pipeline on discrete logs
def scan_model(cnt, S):
    """k_pip_scan: 1024 threads, thread t owns buckets [t*per, t*per + per); each sums its counts and item counts, an exclusive scan over the
    threads gives its base, and it writes start and istart of its buckets from there"""
    nb = len(cnt)
    per = -(-nb // 1024)
    sa, sb = [], []
    for t in range(1024):
        lo, hi = t * per, min(t * per + per, nb)
        sa.append(sum(cnt[lo:hi]))
        sb.append(sum((x + S - 1) // S for x in cnt[lo:hi]))
    start, istart = [0] * nb, [0] * (nb + 1)
    ra = rb = 0                                                  # the exclusive scan of sa, sb at thread t
    for t in range(1024):
        a, b = ra, rb
        for i in range(t * per, min(t * per + per, nb)):
            start[i], istart[i] = a, b
            a += cnt[i]
            b += (cnt[i] + S - 1) // S
        ra += sa[t]
        rb += sb[t]
    istart[nb] = rb
    return start, istart, rb


def item_range(item, istart, start, cnt, S):
    """k_pip_accumulate: the bucket b with istart[b] <= item < istart[b+1] (binary search), and the item's entries [first, last)"""
    lo, hi = 0, len(cnt)
    while hi - lo > 1:
        mid = (lo + hi) >> 1
        if istart[mid] <= item:
            lo = mid
        else:
            hi = mid
    b = lo
    first = start[b] + (item - istart[b]) * S
    last = min(start[b] + cnt[b], first + S)
    return b, first, last


def window_model(buckets, c, w):
    """k_pip_window: 512 threads of `per` buckets, running sums from the top of each chunk, + lo * run, the block sum, then c*w doublings"""
    nb = len(buckets)
    per = -(-nb // 512)
    acc_all = 0
    for t in range(512):
        lo, hi = t * per, min(t * per + per, nb)
        if lo >= nb:
            continue
        run = acc = 0
        for b in range(hi - 1, lo - 1, -1):
            run = (run + buckets[b]) % Q
            acc = (acc + run) % Q
        acc = (acc + lo * run) % Q
        acc_all += acc
    return (acc_all << (c * w)) % Q


def pipeline(ks, a, c_override=0, stats=None):
    """sum_i k_i (a_i B) as the kernels compute it, on discrete logs: returns the log of the result"""
    n = len(ks)
    p = plan(n, c_override)
    c, nwin, nb, S = p["c"], p["nwin"], p["nb"], p["S"]
    ds = [digits(k, c, nwin) for k in ks]
    total = 0
    for w in range(nwin):
        cnt = [0] * nb
        for i in range(n):
            d = ds[i][w]
            if d:
                cnt[abs(d) - 1] += 1
        start, istart, nitems = scan_model(cnt, S)
        assert nitems <= p["max_items"]
        cursor = list(start)                                   # k_pip_scatter: entry = point index with the sign
        sorted_ = [None] * sum(cnt)
        for i in range(n):
            d = ds[i][w]
            if d:
                b = abs(d) - 1
                sorted_[cursor[b]] = (i, d < 0)
                cursor[b] += 1
        partial = []
        for item in range(nitems):
            b, first, last = item_range(item, istart, start, cnt, S)
            assert first < last <= start[b] + cnt[b] and last - first <= S
            partial.append(sum(Q - a[i] if neg else a[i] for i, neg in sorted_[first:last]) % Q)
        buckets = [sum(partial[istart[b]:istart[b + 1]]) % Q for b in range(nb)]
        if stats is not None:
            stats["items"] = max(stats.get("items", 0), nitems)
            stats["empty_windows"] = stats.get("empty_windows", 0) + (nitems == 0)
            stats["top_bucket"] = stats.get("top_bucket", False) or cnt[nb - 1] > 0
            stats["max_items_per_bucket"] = max([stats.get("max_items_per_bucket", 0)] + [istart[b + 1] - istart[b] for b in range(nb)])
        total += window_model(buckets, c, w)
    return total % Q


# ---------------------------------------------------------------------------------------------------- the GPU cases (tests/test_gpu_msm_var_limits.py)
DISTS = ("random", "zero_one", "zero_one_two", "u64", "all_equal", "digit_min", "digit_max", "bucket_sizes", "half_hot", "negated")
# (name, n, c override): every default width from 2^13 to 2^23, every override 2..16 over at least two tiles, then G = 16, G = 32 and the S cap
CASES = ([("default 2^%d" % e, 1 << e, 0) for e in range(13, 24)]
         + [("default 2^17+12345", (1 << 17) + 12345, 0)]
         + [("window %d" % c, 1 << 18, c) for c in range(2, 17)]
         + [("G16", 1 << 19, 10), ("G32", 1 << 20, 10), ("S cap", 1 << 20, 8)])


def case_dists(n, c_override):
    """the scalar distributions a case runs: every one up to 2^20 points, the cheaper branch-aimed ones above"""
    if n <= 1 << 20:
        return DISTS
    return ("random", "zero_one", "all_equal", "digit_min", "bucket_sizes")


def branches(p):
    """the branches of the plan and of the kernels' loops that a plan reaches"""
    out = {("c", p["c"]), ("G", p["G"])}
    if p["s_capped"]:
        out.add(("S cap",))
    if p["ntiles"] > 1:
        out.add(("tiles", "opt-in" if p["optin"] else "default shm"))
    if p["scan_per"] >= 2:
        out.add(("scan per >= 2",))
    if p["window_per"] >= 2:
        out.add(("window per >= 2",))
    return out


WANTED = ({("c", c) for c in range(2, 17)} | {("G", g) for g in (1, 2, 4, 8, 16, 32)}
          | {("S cap",), ("tiles", "opt-in"), ("tiles", "default shm"), ("scan per >= 2",), ("window per >= 2",)})


def test_every_branch_reached():
    reached = set()
    print("\n%-20s %9s %3s %4s %6s %6s %6s %3s %5s %8s %6s %4s %4s" % ("case", "n", "c", "nwin", "nb", "tile", "ntiles", "G", "S", "max_items",
                                                                          "opt-in", "scan", "win"))
    for name, n, co in CASES:
        p = plan(n, co)
        reached |= branches(p)
        print("%-20s %9d %3d %4d %6d %6d %6d %3d %5d%s %8d %6s %4d %4d" % (name, n, p["c"], p["nwin"], p["nb"], p["tile"], p["ntiles"], p["G"], p["S"],
                                                                            "*" if p["s_capped"] else " ", p["max_items"], "yes" if p["optin"] else "no",
                                                                            p["scan_per"], p["window_per"]))
    print("(* = S capped at 8192; scan / win = buckets per thread of k_pip_scan / k_pip_window)")
    assert not WANTED - reached, "branches no GPU case reaches: %s" % sorted(WANTED - reached, key=str)
    assert all(plan(n, co)["nwin"] * n < 1 << 31 for _, n, co in CASES)


def test_mirror_equals_library_plan():
    """the mirror field by field against the library's pip_plan and pip_scratch_bytes (host code of libsp_devtest.so: no device needed) for
    every case and for n = 2^e - 1, 2^e, 2^e + 777 up to 2^26 under every width; widths 1 and 17 refused by both"""
    lib = C.CDLL(os.path.join(ROOT, "spartan_b200", "libsp_devtest.so"))
    lib.spd_last_error.restype = C.c_char_p
    out = (C.c_uint64 * 9)()
    fields = ("c", "nwin", "nb", "tile", "ntiles", "G", "S", "max_items", "scratch")
    shapes = [(n, co) for _, n, co in CASES] + [(n, co) for e in range(27) for n in ((1 << e) - 1, 1 << e, (1 << e) + 777) for co in [0] + list(range(2, 17))]
    for n, co in shapes:
        assert lib.spd_pip_plan(C.c_size_t(n), C.c_int(co), out) == 0, lib.spd_last_error()
        p = plan(n, co)
        assert list(out) == [p[k] for k in fields], (n, co)
    for co in (1, 17):
        assert lib.spd_pip_plan(C.c_size_t(1000), C.c_int(co), out) == -1
        assert b"window width out of range" in lib.spd_last_error()
        with pytest.raises(ValueError):
            plan(1000, co)


def test_default_width_and_plan_fields():
    """the default width is clamp(floor(log2 n) - 7, 6, 16); a few fields pinned by hand"""
    for e in range(0, 31):
        for n in (1 << e, (1 << e) + 1, (2 << e) - 1):
            assert plan(n)["c"] == min(max(e - 7, 6), 16), n
    assert plan(0)["c"] == 6 and plan(0)["ntiles"] == 1
    p = plan(1 << 24)
    assert (p["c"], p["nwin"], p["nb"], p["tile"], p["ntiles"], p["G"], p["S"], p["optin"]) == (16, 16, 1 << 15, 1 << 17, 128, 8, 1024, True)
    p = plan(1 << 23)
    assert (p["c"], p["G"], p["ntiles"], p["optin"]) == (16, 4, 64, True)
    p = plan(1 << 22)
    assert (p["c"], p["G"], p["ntiles"], p["optin"]) == (15, 4, 64, True)


@pytest.mark.parametrize("c", range(2, 17))
def test_digits_recompose(c):
    """sum_w d_w 2^(cw) = k, |d_w| <= nb (bucket |d| - 1 exists), the top digit >= 0, for the edge scalars and random ones; the digit
    patterns come back as built"""
    nwin, nb = 253 // c + 1, 1 << (c - 1)
    rnd = random.Random(c)
    ks = edge_scalars(c) + [rnd.randrange(Q) for _ in range(200)] + [Q - rnd.randrange(1 << 64) for _ in range(20)]
    assert len(ks) > 6 + 4                                  # every digit pattern gives at least one scalar below q
    for k in ks:
        ds = digits(k, c, nwin)
        assert from_digits(ds, c) == k, (c, k)
        assert all(abs(d) <= nb for d in ds), (c, k, ds)
        assert all(-nb <= d <= nb - 1 for d in ds[:-1]) and 0 <= ds[-1] <= nb, (c, k, ds)
    for pattern in ([-nb], [nb - 1], [-nb, nb - 1]):
        for top in sorted({0, 1, 2, nb - 1, nb, nb + 1}):
            k = all_digits(c, pattern, top)
            if 0 <= k < Q:
                assert digits(k, c, nwin) == [pattern[w % len(pattern)] for w in range(nwin - 1)] + [top]


@pytest.mark.parametrize("c", range(2, 17))
def test_pipeline_matches_dot(c):
    """the integer pipeline == sum k_i a_i mod q: random and edge scalars, one scalar repeated into a single oversized bucket, and the window
    extremes (bucket nb - 1 and bucket nb - 2 in every signed window)"""
    rnd = random.Random(100 + c)
    n = 3000
    p = plan(n, c)
    a = [rnd.randrange(Q) for _ in range(n)]
    a[0], a[1] = 0, Q - a[2]                                 # the identity and a point with its negation
    edges = edge_scalars(c)
    ks = [rnd.randrange(Q) for _ in range(n)]
    ks[:len(edges)] = edges
    stats = {}
    assert pipeline(ks, a, c, stats) == sum(k * x for k, x in zip(ks, a)) % Q
    assert stats["top_bucket"]
    hot = [all_digits(c, [-p["nb"]], 1)] * n                 # every signed digit -2^(c-1): bucket nb - 1 in every window but the top
    stats = {}
    assert pipeline(hot, a, c, stats) == sum(hot[0] * x for x in a) % Q
    assert stats["top_bucket"] and stats["max_items_per_bucket"] == -(-n // p["S"])
    assert stats["max_items_per_bucket"] >= 2 or p["S"] >= n
    small = [rnd.randrange(3) for _ in range(n)]             # 0/1/2: windows above the first have no items
    stats = {}
    assert pipeline(small, a, c, stats) == sum(k * x for k, x in zip(small, a)) % Q
    assert stats["empty_windows"] >= p["nwin"] - 2            # (c = 2: the digit of 2 is -2 with a carry of 1 into window 1)


def test_pipeline_large_windows_reduction_ranges():
    """c = 11..16 at a few thousand points: k_pip_window with per >= 2 (lo * run of a chunk > 0) and k_pip_scan with per >= 2, with the last
    bucket (weight nb) occupied"""
    rnd = random.Random(7)
    for c in (11, 12, 16):
        p = plan(4000, c)
        assert p["window_per"] >= 2 and (c < 12 or p["scan_per"] >= 2)
        a = [rnd.randrange(Q) for _ in range(4000)]
        ks = [rnd.randrange(Q) for _ in range(4000)]
        ks[::97] = [all_digits(c, [-p["nb"]], 1)] * len(ks[::97])
        stats = {}
        assert pipeline(ks, a, c, stats) == sum(k * x for k, x in zip(ks, a)) % Q
        assert stats["top_bucket"]


@pytest.mark.parametrize("n", [1, 100, 8191, 8192, 1 << 16, (1 << 20) + 3, 1 << 23, 1 << 24, 1 << 25])
def test_items_within_max_items(n):
    """sum_b ceil(count_b / S) <= max_items for every width: all entries in one bucket, spread evenly, and split into runs of S + 1"""
    for c in [0] + list(range(2, 17)):
        p = plan(n, c)
        nb, S = p["nb"], p["S"]
        worst = [
            [n] + [0] * (nb - 1),
            [n // nb + (b < n % nb) for b in range(nb)],
        ]
        runs = [0] * nb
        left = n
        for b in range(nb):
            runs[b] = min(left, S + 1)
            left -= runs[b]
        runs[0] += left
        worst.append(runs)
        for cnt in worst:
            assert sum(cnt) == n
            items = sum(-(-x // S) for x in cnt)
            assert items <= p["max_items"], (n, c, items, p["max_items"])
        if n <= 1 << 16 and c in (0, 2, 12, 16):
            for cnt in worst:                                 # the scan's own count, thread by thread
                assert scan_model(cnt, S)[2] == sum(-(-x // S) for x in cnt)
