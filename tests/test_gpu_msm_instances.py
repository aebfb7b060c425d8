"""Every instance of the per-window fixed-base MSM, deterministically: k_msm_rows<WBITS, GROUPS, CPT> for window widths 8 / 13 / 15, each
(GROUPS, CPT) pair that msm_rows' selection can produce, both reducers (k_msm_reduce_small for <= 32 chunks, k_msm_reduce above), the blind column
and the batching of more than 32768 rows; k_ipa_msm_quad<8|13|15, .> through the inner-product rounds; and whole SNARK proofs under each width.

Which instance a commitment launches depends on its shape and on the SM count, so the shapes are chosen here by a mirror of the selection in
kernels.cu (msm_rows_use_row_table, msm_pick_groups, msm_pick_cpt) with this device's SM count.  The window width of a generator set is read
from SP_MSM_WINDOW when the set is built; below 512 generators it is always 8, so the sets here have more."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle.spartan_ref import core as oc  # noqa: E402
from test_gpu_ops import test_bullet_reduction_operator_level as bullet_reduction  # noqa: E402  (not collected again under this name)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q = oc.Q
GENS = 600          # generators per set: >= 512, so that SP_MSM_WINDOW applies; a row uses the first R <= GENS of them
WIDTHS = ["8", "13", "15"]
BATCH_SHAPE = (40000, 4, True)   # more than 32768 rows: msm_rows launches k_msm_rows once per batch of 32768


# ---- mirror of the per-window MSM's launch selection (kernels.cu)
def uses_row_table(L, R):
    return L >= 64 and R >= 512


def pick_groups(L, R, sms):
    cols, target = L * (R + 1), sms * 1024
    return 1 if cols >= target else 4 if cols * 4 >= target else 8


def pick_cpt(L, ncols, groups, sms):
    cols = 128 // groups
    blocks4 = L * -(-ncols // (4 * cols))
    return 4 if ncols >= 4 * cols and blocks4 >= sms * 4 else 1


def instance(L, R, blinds, sms):
    """(GROUPS, CPT, chunks per row, reducer, k_msm_rows launches) of msm_rows for L rows of R terms (+ the blind column)"""
    ncols = R + (1 if blinds else 0)
    g = pick_groups(L, R, sms)
    c = pick_cpt(L, ncols, g, sms)
    chunks = -(-ncols // ((128 // g) * c))
    return g, c, chunks, "k_msm_reduce_small" if chunks <= 32 else "k_msm_reduce", -(-L // 32768)


def choose_shapes(sms):
    """the cheapest (L, R, blinds) with R <= GENS, off the row-table path, for each (GROUPS, CPT) pair and for the large-chunk reducer"""
    best = {}
    Ls = sorted(set(range(2, 64)) | set(range(64, 2049, 8)))
    for R in range(2, GENS + 1):
        for L in Ls:
            if uses_row_table(L, R):
                continue
            for bl in (True, False):
                g, c, chunks, red, _ = instance(L, R, bl, sms)
                for key in [(g, c)] + ([red] if red == "k_msm_reduce" else []):
                    if key not in best or L * R < best[key][0] * best[key][1]:
                        best[key] = (L, R, bl)
    return best


@pytest.fixture(scope="module")
def shapes():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    best = choose_shapes(sms)
    chosen = sorted(set(best.values()) | {BATCH_SHAPE})
    table = [(L, R, bl) + instance(L, R, bl, sms) for L, R, bl in chosen]
    print("\nper-window MSM instances on %d SMs (window widths %s):" % (sms, "/".join(WIDTHS)))
    print("%8s %5s %6s %7s %4s %7s %-19s %s" % ("L", "R", "blind", "GROUPS", "CPT", "chunks", "reducer", "launches"))
    for row in table:
        print("%8d %5d %6s %7d %4d %7d %-19s %d" % row)
    return table


def test_selection_reaches_every_instance(shapes):
    """the chosen shapes launch every (GROUPS, CPT) pair, both reducers, the blind column and the row batching"""
    assert {(t[3], t[4]) for t in shapes} == {(g, c) for g in (1, 4, 8) for c in (1, 4)}
    assert {t[6] for t in shapes} == {"k_msm_reduce_small", "k_msm_reduce"}
    assert any(t[2] for t in shapes) and any(t[7] > 1 for t in shapes)


def window_edges(W):
    """scalars at the carries of the signed W-bit recoding, including a chain that carries only through the carry-in of each window"""
    half = 1 << (W - 1)
    return [half - 1, half, half + 1, (1 << W) - 1, 1 << W, (1 << 252) - 1, sum((half + 1) << (W * w) for w in range(252 // W)) % Q,
            ((half + 1) + sum(half << (W * w) for w in range(1, 252 // W))) % Q, (1 << 252) + half, Q - half]


def shape_scalars(L, R):
    Z = oc.prg_scalars("msm-inst%d_%d" % (L, R), L * R)
    edges = [0, 1, Q - 1, oc.R_MONT, oc.R_MONT * oc.R_MONT % Q, 2, Q - 2] + [k for W in (8, 13, 15) for k in window_edges(W)]
    e = oc.to_arr(edges)
    for k in range(len(edges)):                      # scattered over rows and columns: every thread position of a block meets some of them
        Z[(k * 7919 + 3) % (L * R)] = e[k]
    Z[:min(len(edges), L * R)] = e[:min(len(edges), L * R)]   # and a run at the start of row 0
    return Z


@pytest.fixture(scope="module")
def oracle_rows(shapes):
    """the oracle's commitments of every shape, computed once for all window widths"""
    oc.lib.oracle_set_threads(max(1, (os.cpu_count() or 2) // 2))
    ref = oc.MultiCommitGens.new(GENS, b"msm-instances")
    out = {}
    for L, R, bl, *_ in shapes:
        Z = shape_scalars(L, R)
        blinds = oc.prg_scalars("msm-inst-bl", L, L * R) if bl else None
        if bl:
            blinds[0] = oc.to_arr([Q - 1])[0]
            blinds[min(1, L - 1)] = 0
        out[(L, R, bl)] = (Z, blinds, oc.commit_rows(Z, L, R, oc.to_ints(blinds) if bl else [0] * L, ref))
    return out


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as m
    m.default_context()
    return m


@pytest.mark.parametrize("window", WIDTHS)
def test_msm_rows_every_instance(sb, shapes, oracle_rows, window, monkeypatch):
    """DensePolynomial::commit_inner on each chosen shape with a generator set of GENS bases built under SP_MSM_WINDOW = window"""
    monkeypatch.setenv("SP_MSM_WINDOW", window)
    g = sb.MultiCommitGens(GENS, b"msm-instances")
    try:
        for L, R, bl, groups, cpt, chunks, red, launches in shapes:
            Z, blinds, want = oracle_rows[(L, R, bl)]
            got = sb.DensePolynomial(Z).commit(g, L, R, blinds)
            bad = [i for i in range(L) if got[i] != want[i]]
            assert not bad, "k_msm_rows<%s,%d,%d> (L=%d, R=%d, blind=%s, %s): %d of %d rows differ from the oracle, first row %d" % (
                window, groups, cpt, L, R, bl, red, len(bad), L, bad[0])
    finally:
        del g


@pytest.mark.parametrize("window", WIDTHS)
def test_bullet_reduction_every_window(sb, window, monkeypatch):
    """k_ipa_msm_quad<8|13|15, .>: the operator-level inner-product rounds on a 512-generator set built under each window width"""
    monkeypatch.setenv("SP_MSM_WINDOW", window)
    bullet_reduction(sb, 512)


def test_snark_bytes_equal_under_every_window():
    """a 2^16 SNARK (its SPARK generator sets have 512 generators) proved once per window width, each in its own process: the same proof bytes"""
    shas = {}
    for w in WIDTHS:
        e = dict(os.environ)
        e["SP_MSM_WINDOW"] = w
        out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ab_prove.py"), "w" + w, "16", "1"], env=e, capture_output=True, text=True,
                             timeout=900)
        assert out.returncode == 0, out.stderr[-2000:]
        shas[w] = json.loads(out.stdout.strip().splitlines()[-1])["sha256"]
    assert len(set(shas.values())) == 1, shas
