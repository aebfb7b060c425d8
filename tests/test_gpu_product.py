"""Product circuits over the caller's tables and the batched proof of their products on the GPU (sp_prod_*, ProductCircuits /
ProductCircuitEvalProofBatched): products, proof bytes, rand, leaf evaluations and transcript states against the oracle's ProductCircuit and
ProductCircuitEvalProofBatched for plain and fingerprinted leaves on both sides of hadamard_many's 16-circuit group and of batched_prove's
eq-factored threshold, the tables left as they were, a 2^22 batch checked by the library's verifier, a read-only memory check on one transcript
with the oracle replaying it, the refusals, the launch counts, and the parity cases again under the memory-check mode.  The edge kind runs every
affine form k_prod_leaves distinguishes (no source, a coefficient of 0 or q - 1, a unit coefficient before or after non-unit ones, one table as
every source, index coefficients other than 0 and 1) on tables with zeros and runs of ones; 2^19 leaves take the kernel's grid-stride loop past
its first pass on 132 SMs."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import spark as sk

pytestmark = pytest.mark.gpu
Q = oc.Q
LABEL = b"prod-gpu"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MS = [1, 2, 3, 5, 10, 14, 15, 16, 17, 18]
KS = [1, 2, 3, 16, 17, 24]


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    sb.default_context()
    return sb


def ints(a):
    return oc.to_ints(np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4))


def transcripts(sb, products, label=LABEL):
    """the oracle's and the library's transcript after the same caller prefix and the products absorbed"""
    ot, st = oc.Transcript(label), sb.Transcript(label)
    for t in (ot, st):
        t.append_message(b"app", b"prefix")
    for p in products:
        ot.append_scalar(b"claim_product", p)
        st.append_message(b"claim_product", oc.scalar_to_bytes(p))
    return ot, st


def same_transcript(ot, st):
    return ot.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64)


_aux = {}


def ones_index(n):
    if n not in _aux:
        _aux[n] = (oc.from_u64(np.ones(n, dtype=np.uint64)), oc.from_u64(np.arange(n, dtype=np.uint64)))
    return _aux[n]


def leaf_vector(desc, T, n):
    """the leaves the library computes, materialised by the oracle: const + idx * x + sum coeff * T[source][x]"""
    sources, idx, cst = desc
    z = oc.zeros(n)
    arrs = [T[i] for i, _ in sources] + [z] * (3 - len(sources))
    cs = [c for _, c in sources] + [0] * (3 - len(sources))
    one, index = ones_index(n)
    return oc.lincomb3(oc.lincomb3(*arrs, *cs), one, index, 1, cst, idx)


def leaf_eval(desc, evals, rand):
    """the same form on the tables' values at rand (the verifier's side)"""
    sources, idx, cst = desc
    m = len(rand)
    ident = sum(pow(2, m - 1 - i) * r for i, r in enumerate(rand)) % Q
    return (cst + idx * ident + sum(c * evals[s] for s, c in sources)) % Q


def fingerprint_descs(k, r, g):
    """the memory check's hashes ts*r^2 + val*r + addr - g over groups of three tables (addr, val, ts): circuit c is init / read / write /
    audit (c % 4) of group c // 4; init and audit take the address from the index"""
    out, r2 = [], r * r % Q
    for c in range(k):
        a, v, t = 3 * (c // 4), 3 * (c // 4) + 1, 3 * (c // 4) + 2
        out.append([([(v, r)], 1, -g % Q), ([(t, r2), (v, r), (a, 1)], 0, -g % Q), ([(t, r2), (v, r), (a, 1)], 0, (r2 - g) % Q),
                    ([(t, r2), (v, r)], 1, -g % Q)][c % 4])
    return out, 3 * ((k + 3) // 4)


def edge_descs(k, r, g):
    """the forms k_prod_leaves tells apart, cycled over k circuits of three tables: no source (index only, with index coefficients 2, r and
    q - 1, or index and constant), a coefficient of 0 or q - 1, a unit coefficient at source 0 ahead of non-unit ones and the reverse, one table
    as all three sources, a constant of q - 1, and a table alone (its zeros make the product 0; so do the index-only forms at x = 0)"""
    forms = [([], 2, 0), ([], r, 0), ([], Q - 1, 0), ([], g, r),
             ([(0, 0), (1, r)], 0, g),
             ([(1, Q - 1), (2, r)], 1, 0),
             ([(0, 1), (1, r), (2, Q - 1)], 0, 0),
             ([(2, r), (1, Q - 1), (0, 1)], 2, g),
             ([(0, r), (0, 1), (0, g)], 0, 0),
             ([(1, r)], 0, Q - 1),
             ([(0, 1)], 0, 0)]
    return [forms[c % len(forms)] for c in range(k)], 3


def edge_tables(n, tag):
    """three tables with zeros, runs of ones and q - 1 planted at both ends and in the middle"""
    T = [oc.prg_scalars("prod-gpu-%s-%d" % (tag, j), n) for j in range(3)]
    zero, one, top = oc.to_arr([0, 1, Q - 1])
    run = max(1, min(8, n // 4))
    T[0][0] = T[0][n - 1] = T[0][n // 2] = zero
    T[0][n // 4:n // 4 + run] = one
    T[1][:run] = one
    T[1][n - 1] = top
    T[1][n // 2] = zero
    T[2][n - run:] = one
    T[2][0] = top
    return T


def case(sb, m, k, kind, tag):
    """tables, descriptors and the library's leaves argument (None for plain leaves: circuit i = table i)"""
    n = 1 << m
    if kind == "plain":
        descs, nt = [([(c, 1)], 0, 0) for c in range(k)], k
    else:
        r, g = oc.to_ints(oc.prg_scalars("prod-gpu-rg-%s-%d-%d" % (tag, m, k), 2))
        descs, nt = (fingerprint_descs if kind == "fingerprint" else edge_descs)(k, r, g)
    if kind == "edge":
        T = edge_tables(n, "%s-%d-%d" % (tag, m, k))
    else:
        T = [oc.prg_scalars("prod-gpu-%s-%d-%d-%d" % (tag, m, k, j), n) for j in range(nt)]
    leaves = None if kind == "plain" else [sb.ProductLeaves(s, index_coeff=i, const=c) for s, i, c in descs]
    return T, descs, leaves


def build_launches(m, k):
    """one k_prod_leaves launch (the leaves and layer 1), then layers 2 .. m-1 one hadamard_many launch per group of at most 16 circuits"""
    return 1 + -(-k // 16) * (m - 2) if m >= 2 else 1


def prove_launches(m):
    """batched_prove as implemented, single GPU, no dot-product circuits (so independent of k).  Layer l runs R = m-1-l rounds: R = 0 is one
    gather of the two heads; R = 1 is the eq extension, the evaluation, the bind and the heads gather (4); R >= 2 is R + 1: the eq extension or
    the first eq-factored evaluation, then one launch per round (each bind fused with the next evaluation, the switch out of the eq-factored
    rounds a bind plus an evaluation in place of one, and the last round bound on the host).  Every layer but the last processed (l > 0) then
    builds the next layer's eq table: eq_evals of R variables (one launch up to 10, three above) and, when the next layer has at least two
    eq-factored rounds (R >= 14), their suffix levels (one)."""
    total = 0
    for R in range(m):
        total += 1 if R == 0 else 4 if R == 1 else R + 1
        if R < m - 1:
            total += (1 if R <= 10 else 3) + (1 if R >= 14 else 0)
    return total


# ---------------------------------------------------------------------------------------------------- parity with the oracle
@pytest.mark.parametrize("kind", ["plain", "fingerprint", "edge"])
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("m", MS)
def test_build_prove_parity(sb, m, k, kind):
    build_prove_parity(sb, m, k, kind)


@pytest.mark.parametrize("kind", ["plain", "edge"])
@pytest.mark.parametrize("k", [1, 2, 17])
def test_build_prove_parity_second_grid_pass(sb, k, kind):
    """2^19 leaves: 2^18 leaf pairs are more threads than k_prod_leaves' grid holds on 132 SMs (4 CTAs of 256 per SM), so each thread takes a
    second pair"""
    build_prove_parity(sb, 19, k, kind)


def build_prove_parity(sb, m, k, kind):
    n = 1 << m
    T, descs, leaves = case(sb, m, k, kind, "par")
    polys = [sb.DensePolynomial(t) for t in T]
    pc = sb.ProductCircuits(polys, leaves)
    leafv = [leaf_vector(d, T, n) for d in descs]
    cs = [sk.ProductCircuit(v) for v in leafv]
    products = [c.evaluate() for c in cs]
    assert ints(pc.products) == products and pc.num_vars == m
    ot, st = transcripts(sb, products)
    proof, rand, evals = sb.ProductCircuitEvalProofBatched.prove(pc, st)
    want, orand = sk.ProductCircuitEvalProofBatched.prove(cs, [], ot)
    assert proof == pr.ser(want)
    assert ints(rand) == orand
    assert ints(evals) == [oc.evaluate(v, orand) for v in leafv]
    assert same_transcript(ot, st)
    for p, t in zip(polys, T):   # read, never modified
        assert np.array_equal(p.to_numpy(), t)
    if kind == "edge":   # the verifier's side of every form: sp_prod_leaf_eval on the host from the tables' values at rand
        tev = [oc.evaluate(t, orand) for t in T]
        want = [leaf_eval(d, tev, orand) for d in descs]
        assert ints(sb.product_leaf_eval(leaves, oc.to_arr(tev), rand)) == want
        assert ints(evals) == want
        assert 0 in products


def test_launch_counts(sb):
    for m in (1, 2, 3, 5, 11, 12, 15, 16, 17):
        for k in (1, 16, 17, 24):
            T, _, leaves = case(sb, m, k, "fingerprint", "launch")
            polys = [sb.DensePolynomial(t) for t in T]
            l0 = sb.kernel_launches()
            pc = sb.ProductCircuits(polys, leaves)
            l1 = sb.kernel_launches()
            ot, st = transcripts(sb, ints(pc.products))
            sb.ProductCircuitEvalProofBatched.prove(pc, st)
            l2 = sb.kernel_launches()
            assert (l1 - l0, l2 - l1) == (build_launches(m, k), prove_launches(m)), (m, k)


# ---------------------------------------------------------------------------------------------------- 2^22 leaves, checked by the library's verifier
def test_large_batch_verifies(sb):
    m, k = 22, 8
    n = 1 << m
    T, descs, leaves = case(sb, m, k, "fingerprint", "large")
    polys = [sb.DensePolynomial(t) for t in T]
    pc = sb.ProductCircuits(polys, leaves)
    products = ints(pc.products)
    ot, st = transcripts(sb, products)
    proof, rand, evals = sb.ProductCircuitEvalProofBatched.prove(pc, st)
    del pc
    _, vt = transcripts(sb, products)
    vrand, claims = sb.ProductCircuitEvalProofBatched.verify(proof, oc.to_arr(products), m, vt)
    assert np.array_equal(vrand, rand) and np.array_equal(claims, evals)
    assert vt.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64)
    for c, d in enumerate(descs):
        v = leaf_vector(d, T, n)
        assert sb.DensePolynomial(v).evaluate(rand).tolist() == evals[c].tolist()   # sp_poly_evaluate of the leaves, materialised separately
        while len(v) > 1:   # a host product of the leaves
            v = oc.hadamard(v[:len(v) // 2], v[len(v) // 2:])
        assert oc.arr_get(v, 0) == products[c]
    for p, t in zip(polys, T):
        assert np.array_equal(p.to_numpy(), t)


# ---------------------------------------------------------------------------------------------------- a read-only memory check on one transcript
def memory_tables(m, flip=False):
    """a memory of 2^m cells read 2^m times: ops tables addr, val, read_ts and memory tables mem, audit_ts (AddrTimestamps::new,
    sparse_mlpoly.rs:220-254); flip changes the memory's value in a cell that is read"""
    n = 1 << m
    rng = np.random.default_rng(11)
    mem = oc.prg_scalars("prod-gpu-mem", n)
    addr = rng.integers(0, n, size=n, dtype=np.uint64)
    read_ts, audit = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint64)
    for i, a in enumerate(addr):
        read_ts[i] = audit[a]
        audit[a] += 1
    val = np.ascontiguousarray(mem[addr.astype(np.int64)])
    if flip:
        mem = mem.copy()
        mem[int(addr[0])] = oc.to_arr([oc.arr_get(mem, int(addr[0])) + 1])[0]
    return [oc.from_u64(addr), val, oc.from_u64(read_ts), mem, oc.from_u64(audit)]


def memory_descs(r, g):
    """init, read, write, audit over tables addr (0), val (1), read_ts (2), mem (3), audit_ts (4)"""
    r2 = r * r % Q
    return [([(3, r)], 1, -g % Q), ([(2, r2), (1, r), (0, 1)], 0, -g % Q), ([(2, r2), (1, r), (0, 1)], 0, (r2 - g) % Q), ([(4, r2), (3, r)], 1, -g % Q)]


def test_read_only_memory_check_one_transcript(sb):
    m = 10
    n = 1 << m
    T = memory_tables(m)
    big = sb.PolyCommitmentGens(m + 2, LABEL)
    g_ops, g_mem = big, big.view(m + 1)
    og = pr.PolyCommitmentGens(m + 2, LABEL)   # n = 64 for both num_vars
    polys = [sb.DensePolynomial(t) for t in T]
    seed = ints(sb.tape_seed(21))[0]
    stape, otape = sb.RandomTape(sb.tape_seed(21)), oc.RandomTape(b"proof", seed)

    def head(t, comms, chal):
        """commitments absorbed, fingerprint challenges drawn"""
        t.append_message(b"app", b"memory check")
        for label, c in zip((b"comm_ops", b"comm_mem"), comms):
            c.append_to_transcript(label, t)
        return [oc.scalar_from_bytes_wide(chal(t)) for _ in range(2)]

    # the library, as a caller drives it
    st = sb.Transcript(LABEL)
    c_ops, _ = sb.poly_commit(polys[:3], g_ops)
    c_mem, _ = sb.poly_commit(polys[3:], g_mem)
    r, g = head(st, (c_ops, c_mem), lambda t: t.challenge_bytes(b"challenge_r_hash", 64))
    descs = memory_descs(r, g)
    leaves = [sb.ProductLeaves(s, index_coeff=i, const=c) for s, i, c in descs]
    pc = sb.ProductCircuits(polys, leaves)
    prods = ints(pc.products)
    assert prods[0] * prods[2] % Q == prods[1] * prods[3] % Q   # init * write == read * audit
    for p in prods:
        st.append_message(b"claim_product", oc.scalar_to_bytes(p))
    proof, rand, leaf_evals = sb.ProductCircuitEvalProofBatched.prove(pc, st)
    st.append_message(b"protocol-name", b"Derefs evaluation proof")
    p_ops, ev_ops = sb.PolyEvalProof.prove_joint(polys[:3], None, rand, g_ops, st, stape)
    st.append_message(b"protocol-name", b"Derefs evaluation proof")
    p_mem, ev_mem = sb.PolyEvalProof.prove_joint(polys[3:], None, rand, g_mem, st, stape)

    # the oracle runs the same sequence and makes the same bytes
    ot = oc.Transcript(LABEL)
    oc_ops, _ = pr.poly_commit(sk.merge(T[:3]), og)
    oc_mem, _ = pr.poly_commit(sk.merge(T[3:]), og)
    assert (oc_ops.C, oc_mem.C) == (c_ops.C, c_mem.C)
    assert head(ot, (oc_ops, oc_mem), lambda t: t.challenge_bytes(b"challenge_r_hash", 64)) == [r, g]
    leafv = [leaf_vector(d, T, n) for d in descs]
    cs = [sk.ProductCircuit(v) for v in leafv]
    assert [c.evaluate() for c in cs] == prods
    for p in prods:
        ot.append_scalar(b"claim_product", p)
    want, orand = sk.ProductCircuitEvalProofBatched.prove(cs, [], ot)
    assert proof == pr.ser(want) and ints(rand) == orand
    evals_o = [oc.evaluate(t, orand) for t in T]
    d_ops = sk.DerefsEvalProof.prove(type("M", (), {"comb": sk.merge(T[:3])}), evals_o[:3], [], orand, og, ot, otape)
    d_mem = sk.DerefsEvalProof.prove(type("M", (), {"comb": sk.merge(T[3:])}), evals_o[3:], [], orand, og, ot, otape)
    assert p_ops.data == pr.ser(d_ops.proof_derefs) and p_mem.data == pr.ser(d_mem.proof_derefs)
    assert ints(ev_ops) + ints(ev_mem) == evals_o
    assert same_transcript(ot, st)

    # the library's verifier accepts
    vt = sb.Transcript(LABEL)
    assert head(vt, (c_ops, c_mem), lambda t: t.challenge_bytes(b"challenge_r_hash", 64)) == [r, g]
    for p in prods:
        vt.append_message(b"claim_product", oc.scalar_to_bytes(p))
    vrand, claims = sb.ProductCircuitEvalProofBatched.verify(proof, pc.products, m, vt)
    vt.append_message(b"protocol-name", b"Derefs evaluation proof")
    p_ops.verify_joint(g_ops, vt, vrand, ev_ops, c_ops)
    vt.append_message(b"protocol-name", b"Derefs evaluation proof")
    p_mem.verify_joint(g_mem, vt, vrand, ev_mem, c_mem)
    assert np.array_equal(sb.product_leaf_eval(leaves, np.vstack([ev_ops, ev_mem]), vrand), claims)
    assert np.array_equal(claims, leaf_evals)
    # ... and so does the oracle's
    ot2 = oc.Transcript(LABEL)
    head(ot2, (oc_ops, oc_mem), lambda t: t.challenge_bytes(b"challenge_r_hash", 64))
    for p in prods:
        ot2.append_scalar(b"claim_product", p)
    oclaims, _, orand2 = pr.deser(sk.ProductCircuitEvalProofBatched, proof)[0].verify(prods, [], n, ot2)
    sk.DerefsEvalProof(pr.deser(pr.PolyEvalProof, p_ops.data)[0]).verify(orand2, evals_o[:3], [], og, oc_ops, ot2)
    sk.DerefsEvalProof(pr.deser(pr.PolyEvalProof, p_mem.data)[0]).verify(orand2, evals_o[3:], [], og, oc_mem, ot2)
    assert oclaims == [leaf_eval(d, evals_o, orand2) for d in descs]

    # one memory value flipped: the multiset check of the products fails
    Tf = memory_tables(m, flip=True)
    bad = ints(sb.ProductCircuits([sb.DensePolynomial(t) for t in Tf], leaves).products)
    assert bad[0] * bad[2] % Q != bad[1] * bad[3] % Q


# ---------------------------------------------------------------------------------------------------- refusals leave everything as it was
def test_refusals_leave_inputs_alone(sb):
    import ctypes as C
    m = 5
    T = [oc.prg_scalars("prod-gpu-refuse-%d" % j, 1 << m) for j in range(3)]
    polys = [sb.DensePolynomial(t) for t in T]
    short = sb.DensePolynomial(oc.prg_scalars("prod-gpu-refuse-short", 1 << (m - 1)))
    one = sb.DensePolynomial(oc.prg_scalars("prod-gpu-refuse-one", 1))
    odd = sb.DensePolynomial(oc.prg_scalars("prod-gpu-refuse-odd", 3))
    other_ctx = sb.Context(0)
    foreign = sb.DensePolynomial(T[0], ctx=other_ctx)
    bad = np.full(4, 2 ** 64 - 1, dtype=np.uint64)   # limbs >= q
    st = sb.Transcript(LABEL)
    st0 = st.state.raw
    plain = sb.ProductLeaves([(0, 1)])

    def refused(fn, exc, what, code=None):
        live = sb.device_bytes_live()
        l0 = sb.kernel_launches()
        with pytest.raises(exc) as e:
            fn()
        assert what in str(e.value), str(e.value)
        assert st.state.raw == st0
        assert sb.device_bytes_live() == live and sb.kernel_launches() == l0
        for p, t in zip(polys, T):
            assert np.array_equal(p.to_numpy(), t)

    E, S = sb.SpartanB200Error, sb.R1CSError
    refused(lambda: sb.ProductCircuits(polys, []), E, "0 circuits; 1 .. SP_PROD_MAX_CIRCUITS = 24")
    refused(lambda: sb.ProductCircuits(polys, [plain] * 25), E, "25 circuits; 1 .. SP_PROD_MAX_CIRCUITS = 24")
    refused(lambda: sb.ProductCircuits([], [plain]), E, "0 tables")
    refused(lambda: sb.ProductCircuits(polys[:2] + [short]), E, "differ in length")
    refused(lambda: sb.ProductCircuits([one]), E, "power of two >= 2")
    refused(lambda: sb.ProductCircuits([odd]), E, "power of two >= 2")
    refused(lambda: sb.ProductCircuits(polys, [sb.ProductLeaves([(3, 1)])]), E, "table 3 >= ntables = 3")
    refused(lambda: sb.ProductCircuits(polys, [sb.ProductLeaves([(0, 1)] * 4)]), E, "4 sources; at most SP_PROD_MAX_SOURCES = 3")
    refused(lambda: sb.ProductCircuits(polys[:2] + [foreign]), E, "another context")
    refused(lambda: sb.ProductCircuits(polys, [sb.ProductLeaves([(0, bad)])]), S, "not reduced")
    refused(lambda: sb.ProductCircuits(polys, [sb.ProductLeaves([(0, 1)], index_coeff=bad)]), S, "not reduced")
    refused(lambda: sb.ProductCircuits(polys, [sb.ProductLeaves([(0, 1)], const=bad)]), S, "not reduced")
    # the status codes, and what only the C ABI can pass
    ctx = sb.default_context()
    arr = (C.c_void_p * 3)(*[p.h for p in polys])
    h, prods = C.c_void_p(), np.zeros((25, 4), dtype=np.uint64)
    pp = prods.ctypes.data_as(C.c_void_p)
    live = sb.device_bytes_live()
    assert sb.lib.sp_prod_build(ctx.h, arr, C.c_int(3), None, C.c_int(2), C.byref(h), pp) == 3   # leaves NULL with k != ntables
    assert "k = ntables" in sb.lib.sp_last_error(ctx.h).decode()
    assert sb.lib.sp_prod_build(ctx.h, arr, C.c_int(3), None, C.c_int(0), C.byref(h), pp) == 3
    assert sb.lib.sp_prod_build(ctx.h, arr, C.c_int(0), None, C.c_int(0), C.byref(h), pp) == 3
    lv = sb.api._c_leaves([sb.ProductLeaves([(0, bad)])])
    assert sb.lib.sp_prod_build(ctx.h, arr, C.c_int(3), lv, C.c_int(1), C.byref(h), pp) == 5
    assert sb.device_bytes_live() == live and st.state.raw == st0
    out, n = C.POINTER(C.c_ubyte)(), C.c_size_t()
    rand, ev = np.zeros((m, 4), dtype=np.uint64), np.zeros((3, 4), dtype=np.uint64)
    rp, ep = rand.ctypes.data_as(C.c_void_p), ev.ctypes.data_as(C.c_void_p)
    assert sb.lib.sp_prod_prove_t(ctx.h, None, st.state, C.byref(out), C.byref(n), rp, ep) == 3   # NULL handle
    theirs = sb.ProductCircuits([foreign])
    assert sb.lib.sp_prod_prove_t(ctx.h, theirs.h, st.state, C.byref(out), C.byref(n), rp, ep) == 3   # handle of another context
    assert "another context" in sb.lib.sp_last_error(ctx.h).decode()
    assert st.state.raw == st0
    # a second proof on one handle is refused, with the transcript left alone
    pc = sb.ProductCircuits(polys)
    sb.ProductCircuitEvalProofBatched.prove(pc, sb.Transcript(LABEL))
    refused(lambda: sb.ProductCircuitEvalProofBatched.prove(pc, st), E, "consumed")
    del theirs, foreign, other_ctx


# ---------------------------------------------------------------------------------------------------- the parity cases under the memory-check mode
def test_parity_cases_under_memcheck(tmp_path):
    if os.environ.get("SP_MEMCHECK_OUT"):
        pytest.skip("already running under the memory-check mode")
    out = tmp_path / "memcheck.json"
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "tests"), ROOT] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    env["SP_MEMCHECK_OUT"] = str(out)
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "memcheck_plugin", "-p", "no:cacheprovider", "-k", "parity and not memcheck",
           os.path.join(ROOT, "tests", "test_gpu_product.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-20000:]
    tot = json.load(open(out))
    assert tot["violations"] == 0, tot
    assert tot["blocks_filled"] > 0 and tot["context_refills"] > 0, tot
