"""Row commitments through the row tables (d * G_j, signed W-bit windows, per-window sums combined by Horner's rule): the recoding and the
Horner combination on the CPU (device formulation compiled for the host), the kernels on the GPU, both against the oracle."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

from oracle.spartan_ref import core as oc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q = oc.Q
ROW_WIDTHS = (16, 17)   # the row table's window width (16) and the 17-bit alternative measured in DESIGN.md §7: the GPU tests plant the edges of both


def edge_scalars(W):
    """scalars at the edges of the signed W-bit recoding"""
    every_carry = (1 << 252) - 1                                  # every window is 2^W - 1: each one carries into the next
    half_plus_one = sum(((1 << (W - 1)) + 1) << (W * w) for w in range(252 // W))   # every window just above the half
    return [0, 1, 2, Q - 1, (1 << (W - 1)) - 1, 1 << (W - 1), (1 << (W - 1)) + 1, (1 << W) - 1, 1 << W, every_carry, half_plus_one % Q,
            (1 << 252) + 5, (1 << 252) + (1 << (W - 1)), Q - (1 << (W - 1))]


@pytest.fixture(scope="module")
def hostlib():
    path = os.path.join(ROOT, "spartan_b200", "libsp_hosttest_portable.so")
    if not os.path.exists(path):
        import __graft_entry__ as ge
        ge.build_hosttest()
    return C.CDLL(path)


@pytest.mark.parametrize("W", [5, 8, 13, 16, 17])
def test_signed_digits(hostlib, W):
    rng = np.random.default_rng(W)
    out = (C.c_int * 64)()
    for k in edge_scalars(W) + [int.from_bytes(rng.bytes(32), "little") % Q for _ in range(50)]:
        nwin = hostlib.spt_signed_digits(C.c_char_p(k.to_bytes(32, "little")), W, out)
        assert nwin == -(-253 // W)
        d = list(out[:nwin])
        assert sum(x << (W * w) for w, x in enumerate(d)) == k, k
        assert all(-(1 << (W - 1)) < x <= (1 << (W - 1)) for x in d), (k, d)


@pytest.mark.parametrize("W", [5, 16, 17])
def test_row_sums_and_horner(hostlib, W):
    n = 6
    pts = [oc.Point.from_uniform_bytes(hashlib.sha512(b"row%d" % i).digest()) for i in range(n)]
    enc = b"".join(p.compress() for p in pts)
    edges = edge_scalars(W)
    out = C.create_string_buffer(32)
    for r in range(0, len(edges), n):
        ks = (edges[r:r + n] + [3] * n)[:n]
        want = oc.Point.identity()
        for k, p in zip(ks, pts):
            want = want + p * k
        assert hostlib.spt_row_msm(C.c_char_p(oc.to_arr(ks).tobytes()), C.c_char_p(enc), n, W, out) == 1
        assert out.raw == want.compress(), ks


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as m
    m.default_context()
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("L,R", [(64, 512), (96, 1024), (63, 512), (64, 511), (65, 600), (97, 767)])
def test_commit_rows_row_tables(sb, L, R):
    """DensePolynomial::commit_inner on both sides of the row-table selection (64 rows of 512 terms or more take the row tables), with a zero
    row, a zero column and the recoding's edge scalars planted; with and without blinds.  65 and 97 rows leave a Horner block with one live row;
    600 and 767 columns are not a multiple of the 256-column chunk, with the blind column and without"""
    g = sb.MultiCommitGens(R, b"row-msm-test")
    ref = oc.MultiCommitGens.new(R, b"row-msm-test")
    Z = oc.prg_scalars("row-msm%d_%d" % (L, R), L * R)
    Z[3 * R:4 * R] = 0                 # zero row
    Z[5::R] = 0                        # zero column
    edges = oc.to_arr([k for W in ROW_WIDTHS for k in edge_scalars(W)])
    Z[R + 7:R + 7 + len(edges)] = edges
    Z[2 * R - len(edges):2 * R] = edges   # ... and at the end of a row, next to the blind column
    blinds = oc.prg_scalars("row-msm-bl", L, L * R)
    blinds[1] = oc.to_arr([Q - 1])[0]
    blinds[2] = 0
    p = sb.DensePolynomial(Z)
    assert p.commit(g, L, R, blinds) == oc.commit_rows(Z, L, R, oc.to_ints(blinds), ref)
    assert p.commit(g, L, R, None) == oc.commit_rows(Z, L, R, [0] * L, ref)


@pytest.mark.gpu
def test_commit_rows_small_scalars(sb):
    """the 0/1/2-valued rows that dominate SPARK's committed tables: most windows of every scalar are zero and are skipped"""
    L, R = 64, 1024
    g = sb.MultiCommitGens(R, b"row-msm-small")
    ref = oc.MultiCommitGens.new(R, b"row-msm-small")
    Z = oc.from_u64(np.arange(L * R, dtype=np.uint64) % 3)
    assert sb.DensePolynomial(Z).commit(g, L, R) == oc.commit_rows(Z, L, R, [0] * L, ref)
