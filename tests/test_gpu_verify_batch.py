"""GPU tests for batch verification (SNARK.verify_batch / NIZK.verify_batch, sp_*_verify_batch[_t], csrc/verifier.cpp): every proof's status,
message and transcript must be what the single verify gives it, for proofs from this library and from the oracle; and the two new kernels,
the segmented variable-base MSM and k_ipa_srow, against the oracle.  Run on the GPU: pytest -m gpu."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import r1cs, spark
from test_gpu_verify import corruptions  # noqa: E402  (the single-byte flips the single-verify tests use)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(16, 16, 3, 0), (256, 256, 10, 1), (64, 256, 7, 3), (512, 32, 5, 4), (2, 2, 1, 5)]
_vp, _sz = C.c_void_p, C.c_size_t


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as m
    m.default_context()
    return m


def single(fn):
    """(status, message) of one single-proof verify call"""
    from spartan_b200 import api
    try:
        fn()
        return api.SP_OK, None
    except api.ProofVerifyError as e:
        return e.code, str(e)


def codes(results):
    from spartan_b200 import api
    return [api.SP_OK if r is None else r.code for r in results]


class Setup:
    """one statement, its gens, handles and proofs of both kinds"""

    def __init__(self, sb, nc, nv, ni, seed, nproofs):
        self.inst, self.vars, self.inputs = sb.Instance.produce_synthetic_r1cs(nc, nv, ni, seed=seed)
        self.ngens = sb.NIZKGens(nc, nv, ni)
        self.sgens = sb.SNARKGens(nc, nv, ni, nc)
        self.comm = sb.SNARK.encode(self.inst, self.sgens)
        self.nizk = [sb.NIZK.prove(self.inst, self.vars, self.inputs, self.ngens, b"batch", sb.tape_seed(seed + 17 * j)) for j in range(nproofs)]
        self.snark = [sb.SNARK.prove(self.inst, self.comm, self.vars, self.inputs, self.sgens, b"batch", sb.tape_seed(seed + 17 * j)) for j in range(nproofs)]


@pytest.mark.parametrize("nc,nv,ni,seed", SHAPES)
def test_accept(sb, nc, nv, ni, seed):
    """k = 1, 3 and 17 valid proofs are all accepted, with oracle proofs inside the batch and two commitments of the same gens mixed"""
    s = Setup(sb, nc, nv, ni, seed, 3)
    from spartan_b200 import api
    oi, ovars, oinputs = r1cs.Instance.produce_synthetic_r1cs(nc, nv, ni, seed)
    oi.digest = s.inst.digest
    onizk = sb.NIZK(r1cs.NIZK.prove(oi, ovars, oinputs, r1cs.NIZKGens(nc, nv, ni), oc.Transcript(b"batch"), r1cs.tape_seed(seed + 11)).ser())
    ogens = spark.SNARKGens(nc, nv, ni, nc)
    ocomm, odecomm = spark.SNARK.encode(oi, ogens)
    osnark = sb.SNARK(spark.SNARK.prove(oi, ocomm, odecomm, ovars, oinputs, ogens, oc.Transcript(b"batch"), r1cs.tape_seed(seed + 11)).ser())
    # a second statement of the same shape: its own commitment against the same gens
    inst2, vars2, inputs2 = sb.Instance.produce_synthetic_r1cs(nc, nv, ni, seed=seed + 100)
    comm2 = sb.SNARK.encode(inst2, s.sgens)
    p2 = sb.SNARK.prove(inst2, comm2, vars2, inputs2, s.sgens, b"batch", sb.tape_seed(seed))
    n2 = sb.NIZK.prove(inst2, vars2, inputs2, s.ngens, b"batch", sb.tape_seed(seed))
    comm_only = api.ComputationCommitment.from_bytes(s.comm.commitment_bytes())
    for k in (1, 3, 17):
        pn = [(s.nizk + [onizk])[j % 4] for j in range(k)]
        assert NIZK_all_none(sb.NIZK.verify_batch(pn, s.inst, [s.inputs] * k, b"batch", s.ngens))
        ps = [(s.snark + [osnark])[j % 4] for j in range(k)]
        assert NIZK_all_none(sb.SNARK.verify_batch(ps, s.comm, [s.inputs] * k, b"batch", s.sgens))
        # mixed statements: every third proof is the second statement's
        mixed = [(p2, comm2, inputs2) if j % 3 == 1 else (ps[j], comm_only if j % 2 else s.comm, s.inputs) for j in range(k)]
        assert NIZK_all_none(sb.SNARK.verify_batch([m[0] for m in mixed], [m[1] for m in mixed], [m[2] for m in mixed], b"batch", s.sgens))
        mixed = [(n2, inst2, inputs2) if j % 3 == 1 else (pn[j], s.inst, s.inputs) for j in range(k)]
        assert NIZK_all_none(sb.NIZK.verify_batch([m[0] for m in mixed], [m[1] for m in mixed], [m[2] for m in mixed], b"batch", s.ngens))


def NIZK_all_none(results):
    return all(r is None for r in results)


def _rejects(sb, s, kind):
    """about 40 (proof, statement, inputs, label) cases: valid proofs interleaved with byte flips, wrong inputs, a wrong label, a truncated proof,
    a trailing byte and a proof for another statement"""
    P = sb.SNARK if kind == "snark" else sb.NIZK
    proofs = s.snark if kind == "snark" else s.nizk
    stmt = s.comm if kind == "snark" else s.inst
    good = proofs[0].bytes
    bad_inputs = sb.Assignment(s.inputs.limbs.copy())
    bad_inputs.limbs[0, 0] ^= np.uint64(1)
    cases = []
    flips = [b for _, b in corruptions(good, 24, 7)]
    for j, b in enumerate(flips):
        cases.append((P(proofs[j % len(proofs)].bytes), stmt, s.inputs, b"batch"))
        cases.append((P(b), stmt, s.inputs, b"batch"))
    cases += [(P(good), stmt, bad_inputs, b"batch"), (P(good), stmt, s.inputs, b"another label"), (P(good[:-32]), stmt, s.inputs, b"batch"),
              (P(good + b"\x00"), stmt, s.inputs, b"batch"), (P(s.other.bytes), stmt, s.other_inputs, b"batch"), (P(proofs[1].bytes), stmt, s.inputs, b"batch")]
    return cases


@pytest.mark.parametrize("kind", ["snark", "nizk"])
def test_statuses(sb, kind):
    """each status equals the single call's code, the error message is the single call's for the first rejected proof, the call returns SP_ERR_VERIFY"""
    from spartan_b200 import api
    s = Setup(sb, 64, 256, 7, 3, 2)
    inst2, vars2, inputs2 = sb.Instance.produce_synthetic_r1cs(64, 256, 7, seed=77)
    if kind == "snark":
        comm2 = sb.SNARK.encode(inst2, s.sgens)
        s.other = sb.SNARK.prove(inst2, comm2, vars2, inputs2, s.sgens, b"batch", sb.tape_seed(1))
    else:
        s.other = sb.NIZK.prove(inst2, vars2, inputs2, s.ngens, b"batch", sb.tape_seed(1))
    s.other_inputs = inputs2
    gens = s.sgens if kind == "snark" else s.ngens
    cases = _rejects(sb, s, kind)
    assert len(cases) >= 40
    want = [single(lambda c=c: c[0].verify(c[1], c[2], c[3], gens)) for c in cases]
    P = sb.SNARK if kind == "snark" else sb.NIZK
    got = P.verify_batch([c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases], gens)
    assert codes(got) == [w[0] for w in want]
    assert any(w[0] == api.SP_ERR_DECOMPRESS for w in want) and any(w[0] == api.SP_ERR_VERIFY for w in want)
    first = next(i for i, w in enumerate(want) if w[0] != api.SP_OK)
    kind_prefix, msg = want[first][1].split(": ", 1)
    assert str(got[first]) == "%s: proof %d: %s" % (kind_prefix, first, msg)
    # the C return code
    k = len(cases)
    datas = [c[0].bytes for c in cases]
    limbs = [np.ascontiguousarray(c[2].limbs) for c in cases]
    stmts = (_vp * k)(*[c[1].h for c in cases])
    entry = api.lib.sp_snark_verify_batch if kind == "snark" else api.lib.sp_nizk_verify_batch
    status = (C.c_int * k)()
    rc = entry(sb.default_context().h, _sz(k), stmts, (_vp * k)(*[a.ctypes.data_as(_vp) for a in limbs]), (_sz * k)(*[len(a) for a in limbs]), gens.h,
               (C.c_char_p * k)(*[c[3] for c in cases]), (_sz * k)(*[len(c[3]) for c in cases]), (C.c_char_p * k)(*datas), (_sz * k)(*[len(d) for d in datas]),
               C.c_char_p(os.urandom(32)), status)
    assert rc == api.SP_ERR_VERIFY and list(status) == [w[0] for w in want]
    assert api.lib.sp_last_error(sb.default_context().h).decode() == "proof %d: %s" % (first, msg)
    # all valid: SP_OK; k = 0: SP_OK; a NULL seed: SP_ERR_INVALID_ARG
    ok = [c for c, w in zip(cases, want) if w[0] == api.SP_OK]
    assert NIZK_all_none(P.verify_batch([c[0] for c in ok], [c[1] for c in ok], [c[2] for c in ok], b"batch", gens))
    assert P.verify_batch([], [], [], b"batch", gens) == []
    rc = entry(sb.default_context().h, _sz(1), stmts, None, None, gens.h, None, None, None, None, None, status)
    assert rc == api.SP_ERR_INVALID_ARG


@pytest.mark.parametrize("kind", ["snark", "nizk"])
def test_transcripts(sb, kind):
    """_t forms: caller transcripts with data absorbed beforehand end as the single _t call leaves them, accepted or rejected"""
    s = Setup(sb, 16, 16, 3, 0, 2)
    P = sb.SNARK if kind == "snark" else sb.NIZK
    stmt, gens = (s.comm, s.sgens) if kind == "snark" else (s.inst, s.ngens)

    def fresh(j):
        t = sb.Transcript(b"outer")
        t.append_message(b"ctx", b"caller data %d" % j)
        return t
    # proofs made on such a transcript
    proofs = []
    for j in range(4):
        t = fresh(j)
        if kind == "snark":
            proofs.append(sb.SNARK.prove(s.inst, s.comm, s.vars, s.inputs, s.sgens, t, sb.tape_seed(j)))
        else:
            proofs.append(sb.NIZK.prove(s.inst, s.vars, s.inputs, s.ngens, t, sb.tape_seed(j)))
    flips = [b for _, b in corruptions(proofs[0].bytes, 6, 3)]
    batch = [p.bytes for p in proofs] + flips + [proofs[1].bytes]
    idx = list(range(4)) + [0] * len(flips) + [2]       # the last one is verified on another proof's transcript
    want_states, want_codes = [], []
    for b, j in zip(batch, idx):
        t = fresh(j)
        want_codes.append(single(lambda: P(b).verify(stmt, s.inputs, t, gens))[0])
        want_states.append(t.state.raw)
    ts = [fresh(j) for j in idx]
    got = P.verify_batch([P(b) for b in batch], stmt, [s.inputs] * len(batch), ts, gens)
    assert codes(got) == want_codes
    assert want_codes[:4] == [0] * 4 and all(c != 0 for c in want_codes[4:])
    assert [t.state.raw for t in ts] == want_states


def test_seeds(sb):
    """two seeds give the same statuses; one seed twice gives identical results"""
    s = Setup(sb, 64, 256, 7, 3, 2)
    flips = [b for _, b in corruptions(s.snark[0].bytes, 10, 5)]
    batch = [sb.SNARK(b) for b in [s.snark[0].bytes, s.snark[1].bytes] + flips]
    args = (s.comm, [s.inputs] * len(batch), b"batch", s.sgens)
    a = sb.SNARK.verify_batch(batch, *args, seed=b"\x01" * 32)
    b = sb.SNARK.verify_batch(batch, *args, seed=b"\x02" * 32)
    c = sb.SNARK.verify_batch(batch, *args, seed=b"\x01" * 32)
    assert codes(a) == codes(b) == codes(c)
    assert [str(x) for x in a] == [str(x) for x in c]
    assert codes(a)[:2] == [0, 0]


def test_batch_2p16(sb):
    """k = 8 SNARK proofs at 2^16 with one corrupted proof in the middle: only that proof is rejected"""
    n = 1 << 16
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=0)
    gens = sb.SNARKGens(n, n, 10, n)
    comm = sb.SNARK.encode(inst, gens)
    proofs = [sb.SNARK.prove(inst, comm, vars_, inputs, gens, b"v", sb.tape_seed(j)) for j in range(8)]
    b = bytearray(proofs[4].bytes)
    b[len(b) // 3] ^= 4
    proofs[4] = sb.SNARK(bytes(b))
    got = sb.SNARK.verify_batch(proofs, comm, [inputs] * 8, b"v", gens)
    assert [r is None for r in got] == [True] * 4 + [False] + [True] * 3
    assert got[4].code == single(lambda: proofs[4].verify(comm, inputs, b"v", gens))[0]


# ---- the kernels, through libsp_devtest.so
@pytest.fixture(scope="module")
def dt():
    lib = C.CDLL(os.path.join(ROOT, "spartan_b200", "libsp_devtest.so"))
    lib.spd_msm_var_segmented.argtypes = [_sz, _sz, _vp, _vp, _vp, _vp]
    lib.spd_ipa_srow.argtypes = [_sz] + [_vp] * 6 + [_sz, _vp]
    lib.spd_ristretto_decode.argtypes = [_sz, _vp, _vp, _vp]
    lib.spd_ristretto_encode.argtypes = [_sz, _vp, _vp]
    return lib


def _p(a):
    return a.ctypes.data_as(_vp)


def test_msm_var_segmented(sb, dt):
    """every segment against the oracle's ge_msm: sizes 0, 1, 2, 31, 300 and 4096, bases shared between segments, zero scalars, duplicate and
    identity points, and 1000 segments in one launch"""
    rng = np.random.default_rng(5)
    pool_n = 600
    G = oc.MultiCommitGens.new(pool_n, b"seg-msm")
    enc = [G.g(i).compress() for i in range(pool_n)] + [bytes(32)]       # the last one: the identity
    ident = pool_n
    sizes = [0, 1, 2, 31, 300, 4096, 0, 5] + [int(x) for x in rng.integers(0, 40, size=992)]
    idx, sc = [], []
    for k, m in enumerate(sizes):
        ii = [int(x) for x in rng.integers(0, pool_n, size=m)]
        if m >= 4:
            ii[1] = ii[0]          # a duplicate point
            ii[2] = ident          # the identity
        vals = [int.from_bytes(rng.bytes(32), "little") % oc.Q for _ in range(m)]
        if m >= 4:
            vals[3] = 0
        if m >= 6:
            vals[4], vals[5] = oc.Q - 1, 1
        idx.append(ii)
        sc.append(vals)
    flat_idx = [i for ii in idx for i in ii]
    flat_sc = [v for vals in sc for v in vals]
    n = len(flat_idx)
    raw = np.frombuffer(b"".join(enc[i] for i in flat_idx), dtype=np.uint32).reshape(n, 8).copy()
    pts = np.zeros((n, 32), dtype=np.uint32)
    ok = np.zeros(n, dtype=np.int32)
    assert dt.spd_ristretto_decode(_sz(n), _p(raw), _p(pts), _p(ok)) == 0 and ok.all()
    scal = np.frombuffer(b"".join(v.to_bytes(32, "little") for v in flat_sc), dtype=np.uint32).reshape(n, 8).copy()
    seg = np.zeros(len(sizes) + 1, dtype=np.uint32)
    seg[1:] = np.cumsum(sizes)
    K = len(sizes)
    out = np.zeros((K, 32), dtype=np.uint32)
    assert dt.spd_msm_var_segmented(_sz(K), _sz(n), _p(pts), _p(scal), _p(seg), _p(out)) == 0
    got = np.zeros((K, 8), dtype=np.uint32)
    assert dt.spd_ristretto_encode(_sz(K), _p(out), _p(got)) == 0
    ref_pts = np.concatenate([G.G[:pool_n], oc.Point.identity().buf[None, :]])
    for k in range(K):
        want = oc.msm(sc[k], ref_pts[idx[k]]).compress() if sizes[k] else bytes(32)
        assert got[k].tobytes() == want, "segment %d (%d points)" % (k, sizes[k])


def test_ipa_srow(sb, dt):
    """k_ipa_srow against the loop of DotProductProofLog::verify for lg n = 0 .. 12, writing and adding"""
    rng = np.random.default_rng(9)
    lgs = list(range(13))
    items = []
    off = 0
    for lg in lgs:
        for add in (0, 1):
            u = [int.from_bytes(rng.bytes(32), "little") % oc.Q or 1 for _ in range(lg)]
            scale = int.from_bytes(rng.bytes(32), "little") % oc.Q
            items.append((lg, add, u, scale, off))
            off += 1 << lg
    total = off
    init = [int.from_bytes(rng.bytes(32), "little") % oc.Q for _ in range(total)]
    rows = oc.to_arr(init)
    usq = np.zeros((len(items) * 32, 4), dtype=np.uint64)
    allinv, scales, want = [], [], list(init)
    for t, (lg, add, u, scale, o) in enumerate(items):
        u_sq = [x * x % oc.Q for x in u]
        ai = 1
        for x in u:
            ai = ai * oc.inv(x) % oc.Q
        if lg:
            usq[32 * t:32 * t + lg] = oc.to_arr(u_sq)
        allinv.append(ai)
        scales.append(scale)
        n = 1 << lg
        s = [0] * n
        s[0] = ai
        for i in range(1, n):
            lg_i = i.bit_length() - 1
            s[i] = s[i - (1 << lg_i)] * u_sq[(lg - 1) - lg_i] % oc.Q
        for i in range(n):
            v = s[i] * scale % oc.Q
            want[o + i] = (want[o + i] + v) % oc.Q if add else v
    # items of one launch write disjoint ranges
    lg_a = np.array([it[0] for it in items], dtype=np.uint32)
    add_a = np.array([it[1] for it in items], dtype=np.uint32)
    off_a = np.array([it[4] for it in items], dtype=np.uint64)
    rc = dt.spd_ipa_srow(_sz(len(items)), _p(lg_a), _p(add_a), _p(oc.to_arr(allinv)), _p(oc.to_arr(scales)), _p(usq), _p(off_a), _sz(total), _p(rows))
    assert rc == 0
    assert oc.to_ints(rows) == want


_NO_RERUN = r'''
import sys
sys.path.insert(0, sys.argv[1])
import spartan_b200 as sb
ctx = sb.default_context()
inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(256, 256, 10, seed=1)
sg = sb.SNARKGens(256, 256, 10, 256)
comm = sb.SNARK.encode(inst, sg)
ng = sb.NIZKGens(256, 256, 10)
ps = [sb.SNARK.prove(inst, comm, vars_, inputs, sg, b"t", sb.tape_seed(j)) for j in range(3)]
ns = [sb.NIZK.prove(inst, vars_, inputs, ng, b"t", sb.tape_seed(j)) for j in range(3)]
assert sb.SNARK.verify_batch(ps, comm, [inputs] * 3, b"t", sg) == [None] * 3
t = ctx.timings()
assert "fine:batch.final" in t and "fine:batch.rerun" not in t, t
assert sb.NIZK.verify_batch(ns, inst, [inputs] * 3, b"t", ng) == [None] * 3
t = ctx.timings()
assert "fine:batch.final" in t and "fine:batch.rerun" not in t, t
bad = bytearray(ps[1].bytes); bad[len(bad) // 2] ^= 1
assert sb.SNARK.verify_batch([ps[0], sb.SNARK(bytes(bad))], comm, [inputs] * 2, b"t", sg)[1] is not None
assert "fine:batch.rerun" in ctx.timings()
print("ok")
'''


def test_valid_proofs_pass_the_deferred_checks(sb):
    """valid proofs are accepted by the device pass itself, not by the re-run that gives a rejected proof its status (the phase timers of
    SP_FINE_TIMERS=1 show which ran; a process of its own, since the switch is read once)"""
    import subprocess
    import sys
    env = dict(os.environ, SP_FINE_TIMERS="1")
    r = subprocess.run([sys.executable, "-c", _NO_RERUN, ROOT], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr


# ---- the deferred checker on hand-made equations (spd_deferred_check: verifier.cpp's Deferred checker and final pass)
DC_LABEL, DC_BASES = b"deferred-check", 8


def _deferred(dt, proofs, seed=b"\x07" * 32):
    """proofs: list of equation lists; an equation is (lhs, rhs), a side a list of (k, j) with j a generator index (int) or a point (oc.Point)"""
    dt.spd_deferred_check.argtypes = [_sz] + [_vp] * 6 + [C.c_char_p, _sz, _sz, C.c_char_p, _vp]
    eq_start, term_start, side, gen, pts, ks = [0], [0], [], [], [], []
    for eqs in proofs:
        for lhs, rhs in eqs:
            for s_, terms in ((0, lhs), (1, rhs)):
                for k, x in terms:
                    side.append(s_)
                    gen.append(x if isinstance(x, int) else -1)
                    pts.append(bytes(32) if isinstance(x, int) else x.compress())
                    ks.append(k)
            term_start.append(len(side))
        eq_start.append(len(term_start) - 1)
    ok = np.zeros(len(proofs), dtype=np.int32)
    rc = dt.spd_deferred_check(_sz(len(proofs)), _p(np.array(eq_start, dtype=np.uint32)), _p(np.array(term_start, dtype=np.uint32)),
                               _p(np.array(side, dtype=np.int32)), _p(np.array(gen, dtype=np.int64)), _p(np.frombuffer(b"".join(pts) or bytes(32), dtype=np.uint8).copy()),
                               _p(oc.to_arr(ks) if ks else oc.zeros(1)), DC_LABEL, _sz(len(DC_LABEL)), _sz(DC_BASES), seed, _p(ok))
    assert rc == 0
    return [bool(x) for x in ok]


def test_deferred_checks(sb, dt):
    """all-true equations are accepted; one false equation is rejected; two false equations whose errors cancel (+D and -D) are rejected, within
    one proof and across two proofs of one batch, on the variable-base and on the fixed-base part"""
    Gs = oc.MultiCommitGens.new(DC_BASES, DC_LABEL)
    P = oc.MultiCommitGens.new(6, b"deferred-points")
    A, B, D, E = P.g(0), P.g(1), P.g(2), P.g(3)
    a, b, c = 12345678901234567, oc.Q - 5, 77
    true_eqs = [([(a * b % oc.Q, A)], [(a, A * b)]),                        # (ab) A == a (bA)
                ([(c, 3), (1, B)], [(1, Gs.g(3) * c + B)]),                 # c G3 + B == (c G3 + B)
                ([(a, 0), (b, 5)], [(1, Gs.g(0) * a + Gs.g(5) * b)])]
    one_false = true_eqs[:1] + [([(c, 3), (1, B)], [(1, Gs.g(3) * c + B + D)])] + true_eqs[2:]
    cancel = true_eqs + [([(1, A + D)], [(1, A)]), ([(1, B)], [(1, B + D)])]
    cancel_fixed = [([(c, 3)], [(1, Gs.g(3) * c + D)]), ([(1, E + D)], [(1, E)])] + true_eqs
    cancel_scaled = [([(a, A + D)], [(a, A)]), ([(a, B)], [(a, B + D)])]     # the same coefficient on both: cancels under any one weight
    across = ([([(1, A + D)], [(1, A)])], [([(1, B)], [(1, B + D)])])
    got = _deferred(dt, [true_eqs, one_false, cancel, cancel_fixed, cancel_scaled, across[0], across[1], true_eqs, []])
    assert got == [True, False, False, False, False, False, False, True, True]
    # another seed: the same verdicts
    assert _deferred(dt, [true_eqs, cancel, one_false], seed=b"\x09" * 32) == [True, False, False]


def _z_beta_offset(nizk_bytes):
    """byte offset of z_beta of the first DotProductProof of the first ZK sumcheck in bincode(NIZK) (wire.hpp: R1CSProof field order)"""
    u64 = lambda o: int.from_bytes(nizk_bytes[o:o + 8], "little")
    o = 0
    o += 8 + 32 * u64(o)                        # comm_vars.C
    o += 8 + 32 * u64(o)                        # sc_proof_phase1.comm_polys
    o += 8 + 32 * u64(o)                        # comm_evals
    assert u64(o) >= 1
    o += 8                                      # proofs: length
    o += 64                                     # delta, beta
    o += 8 + 32 * u64(o)                        # z
    o += 32                                     # z_delta
    return o


def test_one_unabsorbed_scalar(sb):
    """z_beta of a DotProductProof enters no transcript and only the proof's beta equation, so changing it makes exactly that equation false: the
    batch must reject the proof as the single verify does"""
    s = Setup(sb, 64, 256, 7, 3, 2)
    b = bytearray(s.nizk[0].bytes)
    o = _z_beta_offset(b)
    b[o + 1] ^= 1                               # Montgomery limbs: + or - 256, still reduced
    bad = sb.NIZK(bytes(b))
    code, msg = single(lambda: bad.verify(s.inst, s.inputs, b"batch", s.ngens))
    from spartan_b200 import api
    assert code == api.SP_ERR_VERIFY and msg.endswith("proof rejected: DotProductProof")
    got = sb.NIZK.verify_batch([s.nizk[1], bad, s.nizk[0]], s.inst, [s.inputs] * 3, b"batch", s.ngens)
    assert got[0] is None and got[2] is None and got[1].code == api.SP_ERR_VERIFY
    assert str(got[1]) == "InternalError: proof 1: proof rejected: DotProductProof"
