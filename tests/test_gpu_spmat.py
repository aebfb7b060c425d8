"""Products of the caller's sparse matrices with vectors on the GPU (SparseMatPolynomial.multiply_vec / compute_eval_table_sparse,
SparseMatPolynomial.multi_products) bit for bit against the oracle's SparseMat, for b = 1 .. 8 matrices: square, wide and tall shapes, x = 0 and
y = 0, one row or one column holding 2^20 entries, duplicate entries, values 0, 1 and q - 1, unequal nnz across the batch, num_rows above and
below 2^x, and the tile-edge shapes of test_spmat_model.py at the kernel's tile.  Also the weighted eval table, host against device matrices,
refusals (nothing launched, allocated or changed), the fixed launch count, no table crossing PCIe, the outputs as tables of a caller sumcheck,
and one skewed batch under the memory-check mode."""
import ctypes as C
import zlib

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import r1cs as r1
from test_spmat_model import TILE, shape

pytestmark = pytest.mark.gpu
Q = oc.Q


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    sb.default_context()
    return sb


def canonical(ints_):
    return np.frombuffer(b"".join(oc.scalar_to_bytes(v) for v in ints_), dtype=np.uint8).reshape(-1, 32)


def entries(tag, x, y, n, pattern="random", nrows=None):
    """rows < nrows (default 2^x), cols < 2^y; values from the tag's stream with 0, 1 and q - 1 planted"""
    rng = np.random.default_rng(zlib.crc32(repr((tag, x, y, n, pattern)).encode()))
    rows = rng.integers(0, nrows or (1 << x), n, dtype=np.uint64)
    cols = rng.integers(0, 1 << y, n, dtype=np.uint64)
    if pattern == "row":
        rows[:] = (1 << x) - 1 if nrows is None else nrows - 1
    if pattern == "col":
        cols[:] = 0
    if pattern == "dup" and n > 8:
        rows[1:6], cols[1:6] = rows[0], cols[0]           # the same (row, col) six times
    vals = oc.to_ints(oc.prg_scalars("spmat-gpu-" + tag, n)) if n else []
    for i, v in enumerate((0, 1, Q - 1)):
        if i < n:
            vals[n - 1 - i] = v
    return rows, cols, vals


def pair(sb, x, y, ents, device=False):
    """the library's and the oracle's matrices of the same entries"""
    if device:
        torch = pytest.importorskip("torch")
        lib = [sb.SparseMatPolynomial.from_tensors(x, y, torch.tensor(r.astype(np.int64), device="cuda"), torch.tensor(c.astype(np.int64), device="cuda"),
                                                   torch.tensor(canonical(v), device="cuda")) for r, c, v in ents]
    else:
        lib = [sb.SparseMatPolynomial(x, y, r, c, canonical(v)) for r, c, v in ents]
    orc = [r1.SparseMat(x, y, r, c, oc.to_arr(v) if len(v) else oc.zeros(0)) for r, c, v in ents]
    return lib, orc


def vec(tag, n):
    v = oc.prg_scalars("spmat-gpu-vec-" + tag, n)
    v[0] = oc.to_arr([Q - 1])[0]
    return v


def check_products(sb, x, y, ents, num_rows, num_cols, tag, device=False):
    lib, orc = pair(sb, x, y, ents, device)
    P = sb.SparseMatPolynomial.multi_products(lib)
    z, e = vec("z-" + tag, num_cols), vec("e-" + tag, num_rows)
    got = P.multiply_vec(num_rows, num_cols, z)
    got_t = P.compute_eval_table_sparse(e, num_rows, num_cols)
    for m, M in enumerate(orc):
        assert got[m].to_numpy().tobytes() == M.multiply_vec(num_rows, num_cols, z).tobytes(), (tag, "M z", m)
        assert got_t[m].to_numpy().tobytes() == M.compute_eval_table_sparse(e, num_rows, num_cols).tobytes(), (tag, "M^T e", m)
    return P, got, got_t


# (tag, x, y, nnz per matrix, pattern, num_rows, num_cols); None: 2^x, 2^y
CASES = [
    ("b1-sq", 6, 6, [300], "random", None, None),
    ("b1-x0", 0, 7, [90], "random", None, None),
    ("b1-y0", 7, 0, [90], "random", None, None),
    ("b2-wide", 3, 9, [200, 1000], "random", None, None),
    ("b3-tall", 10, 4, [5000, 17, 3000], "dup", None, None),
    ("b4-unequal", 8, 8, [1, 0, 2500, 999], "random", None, None),
    ("b5-rows-above", 5, 5, [100, 200, 300, 50, 60], "random", 1000, 37),
    ("b6-rows-below", 9, 6, [40] * 6, "random", 300, 64),
    ("b7-col", 6, 6, [1500] * 7, "col", None, None),
    ("b8-row", 6, 6, [2100, 3, 1025, 1024, 1023, 0, 4096, 77], "row", None, None),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_products_match_the_oracle(sb, case):
    tag, x, y, nnzs, pattern, nr, ncl = case
    num_rows, num_cols = nr or (1 << x), ncl or (1 << y)
    bound = min(num_rows, 1 << x)
    ents = [entries("%s-%d" % (tag, i), x, y, n, pattern, nrows=bound) for i, n in enumerate(nnzs)]
    ents = [(r, np.minimum(c, num_cols - 1).astype(np.uint64), v) for r, c, v in ents]
    check_products(sb, x, y, ents, num_rows, num_cols, tag)


@pytest.mark.parametrize("name", ["one-row", "row-on-edge", "empty-runs", "single", "empty", "batch-mid-tile", "random"])
def test_tile_edge_shapes(sb, name):
    num_rows, num_cols, ents = shape(name, TILE)
    x, y = max(1, (num_rows - 1).bit_length()), max(1, (num_cols - 1).bit_length())
    full = []
    for i, (rows, cols) in enumerate(ents):
        n = len(rows)
        full.append((np.asarray(rows, dtype=np.uint64), np.asarray(cols, dtype=np.uint64), oc.to_ints(oc.prg_scalars("tile-%s-%d" % (name, i), n)) if n else []))
    check_products(sb, x, y, full, num_rows, num_cols, "tile-" + name)


@pytest.mark.parametrize("pattern", ["row", "col"])
def test_2p20_entries_on_one_row_or_column(sb, pattern):
    """the R1CS constant-column shape (and its transpose): one column or row holding 2^20 entries, beside a uniform matrix"""
    x = y = 20
    ents = [entries("big-" + pattern, x, y, 1 << 20, pattern), entries("big-u-" + pattern, x, y, 1 << 20)]
    check_products(sb, x, y, ents, 1 << x, 1 << y, "big-" + pattern)


def weights3():
    return oc.to_arr([0, 1, Q - 1])


def test_weighted_eval_table(sb):
    x, y = 7, 8
    ents = [entries("w-%d" % i, x, y, n, "row" if i == 1 else "random") for i, n in enumerate([700, 3000, 5])]
    lib, orc = pair(sb, x, y, ents)
    P = sb.SparseMatPolynomial.multi_products(lib)
    e = vec("we", 1 << x)
    for w in (weights3(), oc.prg_scalars("spmat-w", 3)):
        got = P.compute_eval_table_sparse(e, 1 << x, 1 << y, weights=w)
        tabs = [oc.to_ints(M.compute_eval_table_sparse(e, 1 << x, 1 << y)) for M in orc]
        wi = oc.to_ints(w)
        want = [sum(wi[m] * tabs[m][i] for m in range(3)) % Q for i in range(1 << y)]
        assert oc.to_ints(got.to_numpy()) == want


def test_single_matrix_methods_and_the_cached_device_form(sb):
    x, y = 5, 6
    r, c, v = entries("single", x, y, 400, "dup")
    (M,), (O,) = pair(sb, x, y, [(r, c, v)])
    z, e = vec("sz", 1 << y), vec("se", 1 << x)
    assert M.multiply_vec(1 << x, 1 << y, sb.DensePolynomial(z)).to_numpy().tobytes() == O.multiply_vec(1 << x, 1 << y, z).tobytes()
    handle = M._spmat
    assert M.compute_eval_table_sparse(e, 1 << x, 1 << y).to_numpy().tobytes() == O.compute_eval_table_sparse(e, 1 << x, 1 << y).tobytes()
    assert M._spmat is handle


def test_host_and_device_matrices_give_the_same_bytes(sb):
    x, y = 9, 7
    ents = [entries("hd-%d" % i, x, y, n, p) for i, (n, p) in enumerate([(3000, "col"), (100, "random"), (2048, "row")])]
    _, h, ht = check_products(sb, x, y, ents, 1 << x, 1 << y, "hd")
    _, d, dt = check_products(sb, x, y, ents, 1 << x, 1 << y, "hd", device=True)
    for a, b in zip(h + ht, d + dt):
        assert a.to_numpy().tobytes() == b.to_numpy().tobytes()


def test_creation_errors(sb):
    x, y = 4, 5
    r, c, v = entries("err", x, y, 50)
    good = (r, c, v)
    bad_row = (r.copy(), c, v)
    bad_row[0][17] = 1 << x
    bad_col = (r, c.copy(), v)
    bad_col[1][9] = 1 << y
    with pytest.raises(sb.R1CSError, match=r"InvalidIndex.*row out of range \(matrix 1, entry 17\)"):
        sb.SparseMatPolynomial.multi_products(pair(sb, x, y, [good, bad_row])[0])
    with pytest.raises(sb.R1CSError, match=r"InvalidIndex.*col out of range \(matrix 2, entry 9\)"):
        sb.SparseMatPolynomial.multi_products(pair(sb, x, y, [good, good, bad_col])[0])
    vals = canonical(v).copy()
    vals[3] = np.frombuffer(Q.to_bytes(32, "little"), dtype=np.uint8)
    with pytest.raises(sb.R1CSError, match=r"InvalidScalar.*\(matrix 0, entry 3\)"):
        sb.SparseMatPolynomial.multi_products([sb.SparseMatPolynomial(x, y, r, c, vals)])
    for b in (0, 9):
        with pytest.raises(sb.SpartanB200Error, match="SP_SPMAT_MAX_BATCH"):
            sb.SparseMatPolynomial.multi_products(pair(sb, x, y, [good] * b)[0])
    with pytest.raises(sb.SpartanB200Error, match="> 30"):
        sb.SparseMatPolynomial.multi_products([sb.SparseMatPolynomial(31, 2, r, c % 4, canonical(v))])


def _refused(sb, P, call, inputs, code):
    """`call(outs)` must fail with `code` before any launch: no output written, the inputs unchanged"""
    ctx = P.ctx
    before = [t.to_numpy().tobytes() for t in inputs]
    launches = sb.kernel_launches()
    outs = (C.c_void_p * P.batch_size)(*([0x1234] * P.batch_size))
    rc = call(outs)
    assert rc == code, (rc, sb.lib.sp_last_error(ctx.h).decode())
    assert sb.kernel_launches() == launches
    assert list(outs) == [0x1234] * P.batch_size
    assert [t.to_numpy().tobytes() for t in inputs] == before
    return sb.lib.sp_last_error(ctx.h).decode()


def test_refusals(sb):
    from spartan_b200 import api
    x, y = 6, 5
    ents = [entries("ref-%d" % i, x, y, 300) for i in range(3)]
    lib, _ = pair(sb, x, y, ents)
    P = sb.SparseMatPolynomial.multi_products(lib)
    ctx, lb = P.ctx, sb.lib
    nr, ncl = 1 << x, 1 << y
    max_row = int(max(r.max() for r, _, _ in ents))
    max_col = int(max(c.max() for _, c, _ in ents))
    z, e = sb.DensePolynomial(vec("rz", ncl)), sb.DensePolynomial(vec("re", nr))
    sz = C.c_size_t
    INV, SCAL = api.SP_ERR_INVALID_ARG, api.SP_ERR_INVALID_SCALAR

    def mv(rows, cols, zz, h=None):
        return lambda outs: lb.sp_spmat_multiply_vec(ctx.h, P.h if h is None else h, sz(rows), sz(cols), zz, outs)

    def et(rows, cols, ee, w=None, h=None):
        return lambda outs: lb.sp_spmat_eval_table(ctx.h, P.h if h is None else h, ee, sz(rows), sz(cols), w, outs)
    assert "len(z)" in _refused(sb, P, mv(nr, ncl + 1, z.h), [z], INV)
    assert "len(e)" in _refused(sb, P, et(nr - 1, ncl, e.h), [e], INV)
    assert "row" in _refused(sb, P, mv(max_row, ncl, z.h), [z], INV)
    assert "col" in _refused(sb, P, mv(nr, max_col, sb.DensePolynomial(vec("rz2", max_col)).h), [z], INV)
    assert "col" in _refused(sb, P, et(nr, max_col, e.h), [e], INV)
    assert "num_rows" in _refused(sb, P, mv(0, ncl, z.h), [z], INV)
    assert "NULL" in _refused(sb, P, mv(nr, ncl, None), [z], INV)
    assert "NULL" in _refused(sb, P, et(nr, ncl, e.h, h=C.c_void_p(0)), [e], INV)
    assert "NULL" in _refused(sb, P, lambda outs: lb.sp_spmat_multiply_vec(ctx.h, P.h, sz(nr), sz(ncl), z.h, None), [z], INV)
    w = weights3()
    w[1] = np.frombuffer(Q.to_bytes(32, "little"), dtype=np.uint64)   # limbs of q: not reduced
    assert "weights" in _refused(sb, P, et(nr, ncl, e.h, w=w.ctypes.data_as(C.c_void_p)), [e], SCAL)
    other = sb.Context()
    z_other = sb.DensePolynomial(vec("rz", ncl), ctx=other)
    assert "another context" in _refused(sb, P, mv(nr, ncl, z_other.h), [z], INV)
    P_other = sb.SparseMatPolynomial.multi_products(lib, ctx=other)
    assert "another context" in _refused(sb, P, mv(nr, ncl, z.h, h=P_other.h), [z], INV)


@pytest.mark.parametrize("pattern", ["random", "row", "col"])
def test_launch_count_and_no_host_traffic(sb, pattern):
    from spartan_b200 import api
    x, y = 14, 14
    ents = [entries("lc-%s-%d" % (pattern, i), x, y, n, pattern) for i, n in enumerate([1 << 16, 5000, 1 << 15])]
    lib, _ = pair(sb, x, y, ents)
    P = sb.SparseMatPolynomial.multi_products(lib)
    z, e = sb.DensePolynomial(vec("lz", 1 << y)), sb.DensePolynomial(vec("le", 1 << x))
    for call, extra in ((lambda: P.multiply_vec(1 << x, 1 << y, z), 0), (lambda: P.compute_eval_table_sparse(e, 1 << x, 1 << y), 0),
                        (lambda: P.compute_eval_table_sparse(e, 1 << x, 1 << y, weights=weights3()), 1)):
        io0, l0 = api.io_bytes(), sb.kernel_launches()
        call()
        io1 = api.io_bytes()
        assert sb.kernel_launches() - l0 == api.SP_SPMAT_PRODUCT_LAUNCHES + extra
        assert io1[0] - io0[0] < 4096 and io1[1] - io0[1] < 4096, (io0, io1)


def test_outputs_feed_a_caller_sumcheck(sb):
    x, y = 8, 9
    ents = [entries("sc-%d" % i, x, y, n) for i, n in enumerate([2000, 3000])]
    lib, orc = pair(sb, x, y, ents)
    P = sb.SparseMatPolynomial.multi_products(lib)
    z = vec("scz", 1 << y)
    Az, Bz = P.multiply_vec(1 << x, 1 << y, z)
    a, b = (oc.to_ints(M.multiply_vec(1 << x, 1 << y, z)) for M in orc)
    claim = sum(u * v for u, v in zip(a, b)) % Q
    comp = sb.Composition([(oc.to_arr([1])[0], (0, 1))])
    proof, r, finals, e = sb.sumcheck_prove([Az, Bz], comp, oc.to_arr([claim])[0], x, sb.Transcript(b"spmat-sc"))
    ri = oc.to_ints(r)
    assert oc.to_ints(finals) == [oc.evaluate(oc.to_arr(a), ri), oc.evaluate(oc.to_arr(b), ri)]
    ve, vr = sb.sumcheck_verify(proof, oc.to_arr([claim])[0], x, 2, sb.Transcript(b"spmat-sc"))
    assert vr.tobytes() == r.tobytes() and ve.tobytes() == e.tobytes()


def test_memcheck_b4_skewed(sb):
    sb.debug_memcheck(True)
    try:
        v0 = sb.debug_memcheck_report()["violations"]
        ctx = sb.Context()
        x, y = 11, 11
        ents = [entries("mc-%d" % i, x, y, n, p) for i, (n, p) in enumerate([(3000, "row"), (1, "random"), (5000, "col"), (1024, "dup")])]
        lib = [sb.SparseMatPolynomial(x, y, r, c, canonical(v)) for r, c, v in ents]
        orc = [r1.SparseMat(x, y, r, c, oc.to_arr(v)) for r, c, v in ents]
        P = sb.SparseMatPolynomial.multi_products(lib, ctx=ctx)
        z, e = vec("mz", 1 << y), vec("me", 1 << x)
        got = P.multiply_vec(1 << x, 1 << y, z)
        got_t = P.compute_eval_table_sparse(e, 1 << x, 1 << y)
        got_w = P.compute_eval_table_sparse(e, 1 << x, 1 << y, weights=oc.prg_scalars("mw", 4))
        for m, M in enumerate(orc):
            assert got[m].to_numpy().tobytes() == M.multiply_vec(1 << x, 1 << y, z).tobytes()
            assert got_t[m].to_numpy().tobytes() == M.compute_eval_table_sparse(e, 1 << x, 1 << y).tobytes()
        assert got_w.len() == 1 << y
        del got, got_t, got_w, P, ctx
        assert sb.debug_memcheck_scan() == 0
        rep = sb.debug_memcheck_report()
        assert rep["violations"] == v0, rep["last_violation"]
    finally:
        sb.debug_memcheck(False)


@pytest.mark.parametrize("nnzs", [[300, 1, 400], [1500, 2000, 1000], [9000, 7000, 500]], ids=["total-701", "total-4500", "total-16500"])
def test_memcheck_carry_scratch(sb, nnzs):
    """batches whose carry scratch has the most alignment padding for its size: 1 .. 1024 entries, and 4097 .. 5120 and 16385 .. 18432, where
    the pool's rounding of the request leaves no slack past it.  Every product's scratch is guarded, and a write past it is a violation"""
    sb.debug_memcheck(True)
    try:
        v0 = sb.debug_memcheck_report()["violations"]
        ctx = sb.Context()
        x, y = 10, 10
        ents = [entries("mcs-%d-%d" % (sum(nnzs), i), x, y, n, "row" if i == 0 else "random") for i, n in enumerate(nnzs)]
        lib = [sb.SparseMatPolynomial(x, y, r, c, canonical(v)) for r, c, v in ents]
        orc = [r1.SparseMat(x, y, r, c, oc.to_arr(v)) for r, c, v in ents]
        P = sb.SparseMatPolynomial.multi_products(lib, ctx=ctx)
        z, e = vec("mcz", 1 << y), vec("mce", 1 << x)
        got = P.multiply_vec(1 << x, 1 << y, z)
        got_t = P.compute_eval_table_sparse(e, 1 << x, 1 << y)
        got_w = P.compute_eval_table_sparse(e, 1 << x, 1 << y, weights=weights3())
        tabs = [oc.to_ints(M.compute_eval_table_sparse(e, 1 << x, 1 << y)) for M in orc]
        for m, M in enumerate(orc):
            assert got[m].to_numpy().tobytes() == M.multiply_vec(1 << x, 1 << y, z).tobytes()
            assert oc.to_ints(got_t[m].to_numpy()) == tabs[m]
        assert oc.to_ints(got_w.to_numpy()) == [(tabs[1][i] - tabs[2][i]) % Q for i in range(1 << y)]
        del got, got_t, got_w, P, ctx
        assert sb.debug_memcheck_scan() == 0
        rep = sb.debug_memcheck_report()
        assert rep["violations"] == v0, rep["last_violation"]
    finally:
        sb.debug_memcheck(False)
