"""The inputs of the generator-table tests (test_gpu_gen_table_entries.py), checked on the CPU.

Scalars whose every non-top signed W-bit digit is an extreme of the recoding (+2^(W-1), -(2^(W-1) - 1), +1, -1) and whose top window is as large
as q allows: a commitment of them reads, for every generator and every window, the last table entry, the one before it and the first, with both
signs.  The digits are checked through spt_signed_digits (the recoding of curve.cuh compiled for the host) for W = 8, 13 and 15 (the per-window
tables) and 16 (the row tables).  The oracle's generators of every set size the tables are built at are prefixes of one SHAKE stream per label,
so one expansion per label serves every size.  The plain-Python point helpers the self-test plants defects with are checked against the oracle."""
import ctypes as C
import hashlib
import os

import pytest

from oracle.spartan_ref import core as oc
from test_gpu_arith import D, P, ed_dbl, encode, from_uniform, niels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q = oc.Q
WIDTHS = (8, 13, 15, 16)
PATTERNS = 4
# every set size the GPU test checks, per label: the 2^20 / 2^22 R1CS sets, the 2^20 / 2^22 SPARK sets, the sets on both sides of the row-table
# threshold and the small sets of tiny circuits
SET_SIZES = {b"gens_r1cs_sat": (5, 6, 1026, 2050), b"gens_r1cs_eval": (18, 511, 513, 4098, 8194)}


def nwin(W):
    return -(-253 // W)


def extreme_digits(W):
    half = 1 << (W - 1)
    return (half, -(half - 1), 1, -1)


def extreme_scalar(W, pattern):
    """window w < nwin - 1 has digit extreme_digits(W)[(pattern + w) % 4]; the top window the largest digit that keeps the scalar below q"""
    ext = extreme_digits(W)
    low = sum(ext[(pattern + w) % PATTERNS] << (W * w) for w in range(nwin(W) - 1))
    top_shift = W * (nwin(W) - 1)
    top = (Q - 1 - low) >> top_shift
    return low + (top << top_shift), top


def table_scalars(W, L, R):
    """an L x R table and L blinds: column j of row r (the blind being column R, the generator h) takes pattern (r + j) mod 4, so that over any
    four consecutive rows every column meets every pattern in every window"""
    ks = [extreme_scalar(W, p)[0] for p in range(PATTERNS)]
    return [ks[(r + j) % PATTERNS] for r in range(L) for j in range(R)], [ks[(r + R) % PATTERNS] for r in range(L)]


@pytest.fixture(scope="module")
def hostlib():
    path = os.path.join(ROOT, "spartan_b200", "libsp_hosttest_portable.so")
    if not os.path.exists(path):
        import __graft_entry__ as ge
        ge.build_hosttest()
    return C.CDLL(path)


def signed_digits(hostlib, k, W):
    out = (C.c_int * 64)()
    n = hostlib.spt_signed_digits(C.c_char_p(k.to_bytes(32, "little")), W, out)
    assert n == nwin(W)
    return list(out[:n])


@pytest.mark.parametrize("W", WIDTHS)
def test_extreme_scalars_recode_to_their_digits(hostlib, W):
    """each pattern's scalar is below q, its top digit is the largest that keeps it there, and the recoding gives back exactly the planted digits"""
    ext = extreme_digits(W)
    top_shift = W * (nwin(W) - 1)
    for p in range(PATTERNS):
        k, top = extreme_scalar(W, p)
        assert 0 <= k < Q <= k + (1 << top_shift)
        assert 0 < top < 1 << (W - 1)
        d = signed_digits(hostlib, k, W)
        assert d[:-1] == [ext[(p + w) % PATTERNS] for w in range(nwin(W) - 1)], (W, p)
        assert d[-1] == top


@pytest.mark.parametrize("W,L,R", [(8, 4, 1024), (13, 4, 4096), (15, 4, 1024), (16, 64, 1024), (16, 64, 4096)])
def test_every_column_meets_every_extreme(hostlib, W, L, R):
    """the layouts of the GPU test (4 rows on the per-window tables, 64 rows on the row tables): in every non-top window every column, the blind
    column included, meets +2^(W-1), -(2^(W-1) - 1), +1 and -1"""
    Z, blinds = table_scalars(W, L, R)
    digits = {}
    for k in set(Z) | set(blinds):
        digits[k] = signed_digits(hostlib, k, W)
    want = set(extreme_digits(W))
    for j in range(R + 1):
        col = [blinds[r] if j == R else Z[r * R + j] for r in range(L)]
        for w in range(nwin(W) - 1):
            assert {digits[k][w] for k in col} == want, (j, w)


@pytest.mark.parametrize("label", sorted(SET_SIZES))
def test_oracle_sets_are_prefixes_of_one_stream(label):
    """MultiCommitGens::new(n - 1, label) (n generators counting h) is the first n points of the largest set's stream, for every size checked on
    the GPU, and its points are those the plain-Python from_uniform gives for the same SHAKE bytes"""
    big = max(SET_SIZES[label])
    full = oc.MultiCommitGens.new(big - 1, label)
    enc = [full.g(i).compress() for i in range(big - 1)] + [full.h.compress()]
    assert len(set(enc)) == big
    for n in SET_SIZES[label]:
        g = oc.MultiCommitGens.new(n - 1, label)
        assert [g.g(i).compress() for i in range(n - 1)] + [g.h.compress()] == enc[:n], n
    uni = hashlib.shake_256(label + oc.BASEPOINT_COMPRESSED).digest(64 * big)
    for i in (0, 1, big // 2, big - 1):
        assert encode(from_uniform(uni[64 * i:64 * i + 64])) == enc[i], i


# ---- plain-Python affine-niels helpers for planting defects in a table copy
def niels_bytes(n):
    return b"".join(c.to_bytes(32, "little") for c in n)


def niels_from_bytes(b):
    return tuple(int.from_bytes(b[32 * i:32 * i + 32], "little") for i in range(3))


def niels_to_ext(n):
    """(y + x, y - x, 2dxy) -> extended coordinates (x, y, 1, xy)"""
    inv2 = pow(2, -1, P)
    x, y = (n[0] - n[1]) * inv2 % P, (n[0] + n[1]) * inv2 % P
    return (x, y, 1, x * y % P)


def niels_neg(n):
    return (n[1], n[0], (-n[2]) % P)


def niels_dbl(n):
    return niels(ed_dbl(niels_to_ext(n)))


def test_niels_helpers():
    """niels_to_ext inverts niels, and doubling / negation in niels form are the oracle's on ristretto classes and exact on edwards25519"""
    uni = hashlib.shake_256(b"niels-helpers").digest(64 * 8)
    for i in range(8):
        pt = from_uniform(uni[64 * i:64 * i + 64])
        n = niels(pt)
        e = niels_to_ext(n)
        assert niels(e) == n and n[2] == 2 * D * e[3] % P
        o = oc.Point.decompress(encode(pt))
        assert encode(niels_to_ext(niels_dbl(n))) == (o + o).compress()
        assert encode(niels_to_ext(niels_neg(n))) == (oc.Point.identity() - o).compress()
        assert niels_dbl(niels_neg(n)) == niels_neg(niels_dbl(n))
        assert niels_from_bytes(niels_bytes(n)) == n
