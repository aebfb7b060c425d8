"""The tile / carry partition of the segmented matrix products (kernels_inst.cu: spmat_products) as a Python model, on the oracle alone (no
GPU): the entries of b matrices sorted by key, tiles of the kernel's size (read from the library through a host-only hook), direct stores of
the segments inside a tile, two carries per tile reduced by one more tiled level, and the last level in one serial pass.  The model stores
every output key at most once and equals the oracle's SparseMat.multiply_vec / compute_eval_table_sparse on the shapes where a tiling goes
wrong: one row spanning many tiles, a row ending on a tile edge, runs of empty rows at tile edges, a single entry, no entries, and batches whose
matrix boundary falls inside a tile.  Small tiles run the same cases through every carry level."""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import r1cs as r1

Q = oc.Q
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def hosttest():
    path = os.path.join(ROOT, "spartan_b200", "libsp_hosttest_portable.so")
    if not os.path.exists(path):
        import __graft_entry__ as ge
        ge.build_hosttest()
    lib = C.CDLL(path)
    lib.sph_spmat_tile.restype = C.c_size_t
    return lib


TILE = int(hosttest().sph_spmat_tile())


# ----------------------------------------------------------------------------- the model
def tile_pass(items, base, nt, store):
    """one tile of (key, value) items: stores the segments that start and end inside it; returns (kf, vf, kl, vl, single)"""
    first = None
    run, seen = 0, False
    for j in range(base, base + nt):
        k, v = items[j]
        if j > base and k != items[j - 1][0]:          # a head: the segment before it closes
            if seen:
                store(items[j - 1][0], run)
            else:
                first = (items[j - 1][0], run)
            run, seen = 0, True
        run = (run + v) % Q
    kl = items[base + nt - 1][0]
    if not seen:
        return kl, run, kl, run, True
    return first[0], first[1], kl, run, False


def tiled_level(items, tile, store):
    carries = []
    for base in range(0, len(items), tile):
        kf, vf, kl, vl, single = tile_pass(items, base, min(tile, len(items) - base), store)
        carries += [(kf, vf), (kl, 0 if single else vl)]
    return carries


def final_level(items, tile, store):
    open_, rk, rv = False, None, 0
    for base in range(0, len(items), tile):
        kf, vf, kl, vl, single = tile_pass(items, base, min(tile, len(items) - base), store)
        first = vf
        if open_ and rk == kf:
            first = (rv + first) % Q
        elif open_:
            store(rk, rv)
        if single:
            rk, rv = kf, first
        else:
            store(kf, first)
            rk, rv = kl, vl
        open_ = True
    if open_:
        store(rk, rv)


def model_products(mats, x, nout, tile, transpose=False):
    """out[m][key] = sum val * x[src] for matrices given as (rows, cols, vals as ints); key = row (M x) or col (M^T x)"""
    items = []
    for m, (rows, cols, vals) in enumerate(mats):
        keys, srcs = (cols, rows) if transpose else (rows, cols)
        order = sorted(range(len(keys)), key=lambda i: keys[i])          # stable, as the radix sort
        items += [((m << 32) | int(keys[i]), vals[i] * x[int(srcs[i])] % Q) for i in order]
    out = [[0] * nout for _ in mats]
    written = set()

    def store(k, v):
        assert k not in written, "key %x stored twice" % k
        written.add(k)
        out[k >> 32][k & 0xffffffff] = v
    final_level(tiled_level(tiled_level(items, tile, store), tile, store), tile, store)
    keys = {k for k, _ in items}
    assert written == keys, "keys with entries that were never stored"
    return out


# ----------------------------------------------------------------------------- shapes
def shape(name, tile):
    """(num_rows, num_cols, [(rows, cols)]) of one case at tile size `tile`"""
    rng = np.random.default_rng(zlib.crc32(("%s-%d" % (name, tile)).encode()))
    if name == "one-row":               # every entry on one row, spanning many tiles
        n = 5 * tile + 17
        return 64, 4096, [(np.full(n, 9), rng.integers(0, 4096, n))]
    if name == "row-on-edge":           # rows of exactly tile and 2 tile entries: segments ending on tile edges
        rows = np.concatenate([np.full(tile, 0), np.full(2 * tile, 3), np.full(tile - 1, 5), np.full(1, 6), np.arange(7, 7 + tile)])
        return 8 + tile, 512, [(rows, rng.integers(0, 512, len(rows)))]
    if name == "empty-runs":            # runs of empty rows where tiles meet
        rows = np.concatenate([np.arange(0, tile - 3), np.full(3, tile + 50), np.full(tile, 3 * tile), np.arange(5 * tile, 5 * tile + 10)])
        return 6 * tile + 64, 256, [(rows, rng.integers(0, 256, len(rows)))]
    if name == "single":
        return 1 << 10, 1 << 10, [(np.array([1023]), np.array([0]))]
    if name == "empty":
        return 16, 16, [(np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64))]
    if name == "batch-mid-tile":        # matrix boundaries inside tiles, one empty matrix, unequal nnz, the same row across the boundary
        sizes = [tile // 3, 0, tile + tile // 2, 7, 2 * tile + 1]
        mats = []
        for i, n in enumerate(sizes):
            rows = rng.integers(0, 40, n)
            rows[: n // 2] = 39                      # a long run on the last row, where the next matrix starts on row 39 again
            mats.append((rows, rng.integers(0, 300, n)))
        return 40, 300, mats
    if name == "random":
        n = 3 * tile + 5
        return 200, 100, [(rng.integers(0, 200, n), rng.integers(0, 100, n)), (rng.integers(0, 200, n // 2), rng.integers(0, 100, n // 2))]
    raise KeyError(name)


SHAPES = ["one-row", "row-on-edge", "empty-runs", "single", "empty", "batch-mid-tile", "random"]


def vals_for(tag, n):
    return oc.prg_scalars("spmat-model-" + tag, n) if n else oc.zeros(0)


@pytest.mark.parametrize("tile", [TILE, 4, 2])
@pytest.mark.parametrize("name", SHAPES)
def test_model_equals_oracle(name, tile):
    num_rows, num_cols, ents = shape(name, tile)
    omats, mats = [], []
    for i, (rows, cols) in enumerate(ents):
        v = vals_for("%s-%d-%d" % (name, tile, i), len(rows))
        vi = oc.to_ints(v) if len(rows) else []
        omats.append(r1.SparseMat(0, 0, np.asarray(rows, dtype=np.uint64), np.asarray(cols, dtype=np.uint64), v))
        mats.append((list(rows), list(cols), vi))
    z = vals_for("z-" + name, num_cols)
    e = vals_for("e-" + name, num_rows)
    zi, ei = oc.to_ints(z), oc.to_ints(e)
    got = model_products(mats, zi, num_rows, tile)
    got_t = model_products(mats, ei, num_cols, tile, transpose=True)
    for m, M in enumerate(omats):
        assert got[m] == oc.to_ints(M.multiply_vec(num_rows, num_cols, z)), (name, m)
        assert got_t[m] == oc.to_ints(M.compute_eval_table_sparse(e, num_rows, num_cols)), (name, m)


def test_kernel_tile_and_levels():
    """the kernel's tile is 256 threads x 4 entries, and two tiled levels leave at most 2^14 carries for the one-CTA pass below 2^32 entries"""
    assert TILE == 1024
    carries = lambda n: 2 * ((n + TILE - 1) // TILE)  # noqa: E731
    assert carries(carries((1 << 32) - 1)) <= 1 << 14


def test_carry_scratch_holds_its_layout():
    """the scratch spmat_products asks for holds the four carry regions it carves (values and keys of both levels, each at a 256-byte boundary),
    without overlap, for every total up to 40 tiles and around the sizes where the regions' padding adds up to most"""
    lib = hosttest()
    out = (C.c_size_t * 7)()
    totals = list(range(0, 40 * TILE + 2)) + [k * TILE + d for k in (127, 128, 129, 196, 197, 1024, 4096) for d in (-1, 0, 1)]
    totals += [(1 << 32) - 1]
    for total in totals:
        lib.sph_spmat_carries(C.c_size_t(total), out)
        n1, n2, cv1, cv2, ck1, ck2, nbytes = list(out)
        assert n1 == 2 * -(-total // TILE) and n2 == 2 * -(-n1 // TILE), total
        regions = sorted([(cv1, 32 * n1), (cv2, 32 * n2), (ck1, 8 * n1), (ck2, 8 * n2)])
        for (a, la), (b, _) in zip(regions, regions[1:]):
            assert a + la <= b, (total, regions)
        assert all(off % 256 == 0 for off, _ in regions), (total, regions)
        assert regions[-1][0] + regions[-1][1] <= nbytes, (total, regions, nbytes)
