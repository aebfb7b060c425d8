"""DotProductProofLog of the caller's vectors on the GPU (sp_dotlog_*; DotProductProofGens, DotProductProofLog): byte parity with the oracle's
prove for n = 1 .. 2^16 (both sides of SP_DOTLOG_TABLE_MAX_N) and against the golden 2^18 / 2^20 proofs, the transcript and tape states after
each call, both verifiers on every proof and on its mutants, device and host vectors, edge values, the generator-fold kernel against the oracle's
MSM, the refusals, and the device memory each call leaves behind."""
import ctypes as C
import gc
import json
import os
import re

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import r1cs

pytestmark = pytest.mark.gpu
Q = oc.Q
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LABEL, GENS_LABEL = b"dotlog-gpu", b"dotlog-gpu-gens"
_sz, _vp = C.c_size_t, C.c_void_p


def header_define(name):
    src = open(os.path.join(ROOT, "include", "spartan_b200.h")).read()
    return int(eval(re.search(r"#define %s \(?([^/\n]*?)\)?\s*(/\*|\n)" % name, src).group(1).replace("u", "")))


TABLE_MAX_N = header_define("SP_DOTLOG_TABLE_MAX_N")
MAX_N = header_define("SP_DOTLOG_MAX_N")


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    sb.default_context()
    return sb


_GENS = {}


def gens(sb, n, label=GENS_LABEL):
    """(library, oracle) DotProductProofGens::new(n, label)"""
    if (n, label) not in _GENS:
        _GENS.clear()   # one size at a time: the large sets are big
        _GENS[(n, label)] = (sb.DotProductProofGens(n, label), pr.DotProductProofGens(n, label))
    return _GENS[(n, label)]


def L(x):
    return oc.to_arr([x % Q])[0]


def ints(a):
    return oc.to_ints(np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4))


class States:
    """the oracle's and the library's transcript and tape (one seed)"""

    def __init__(self, sb, seed, label=LABEL):
        self.ot, self.st = oc.Transcript(label), sb.Transcript(label)
        self.otape = oc.RandomTape(b"proof", r1cs.tape_seed(seed))
        self.stape = sb.RandomTape(sb.tape_seed(seed))

    def raw(self):
        return self.st.state.raw, self.stape.state.raw

    def same(self):
        return (self.ot.challenge_bytes(b"after", 64) == self.st.challenge_bytes(b"after", 64)
                and self.otape.tape.challenge_bytes(b"after", 64) == self.stape.challenge_bytes(b"after", 64))


def vectors(n, tag):
    return oc.prg_scalars("dotlog-%s-x-%d" % (tag, n), n), oc.prg_scalars("dotlog-%s-a-%d" % (tag, n), n)


def prove_both(sb, n, x, a, y=None, seed=1, blinds=(5, 7)):
    """the library's and the oracle's prove of the same statement; y None: <x, a> (the library computes it)"""
    lg, og = gens(sb, n)
    S = States(sb, seed)
    xi, ai = ints(x), ints(a)
    y_int = sum(p * q for p, q in zip(xi, ai)) % Q if y is None else y
    proof, Cx, Cy = sb.DotProductProofLog.prove(lg, S.st, S.stape, x, L(blinds[0]), a, None if y is None else L(y), L(blinds[1]))
    oproof, oCx, oCy = pr.DotProductProofLog.prove(og, S.ot, S.otape, xi, blinds[0], ai, y_int, blinds[1])
    return proof, (Cx, Cy), oproof, (oCx, oCy), S


def verify_both(sb, n, data, a, Cx, Cy, label=LABEL):
    """(oracle verdict, library verdict, transcripts after) on fresh transcripts of the label the proofs were made on: verdict True = accepted"""
    lg, og = gens(sb, n)
    ot, st = oc.Transcript(label), sb.Transcript(label)
    try:
        p, pos = pr.deser(pr.DotProductProofLog, data)
        ok_o = pos == len(data)
        if ok_o:
            p.verify(n, og, ot, ints(a), Cx, Cy)
    except (pr.ProofVerifyError, AssertionError, ValueError, IndexError):
        ok_o = False
    try:
        sb.DotProductProofLog(data).verify(n, lg, st, a, Cx, Cy)
        ok_l = True
    except sb.ProofVerifyError:
        ok_l = False
    return ok_o, ok_l, ot, st


# ---------------------------------------------------------------------------------------------------- bytes, states and both verifiers
@pytest.mark.parametrize("logn", list(range(17)))
def test_parity_with_oracle(sb, logn):
    n = 1 << logn
    x, a = vectors(n, "parity")
    proof, (Cx, Cy), oproof, (oCx, oCy), S = prove_both(sb, n, x, a, y=None if logn % 2 else 12345, seed=logn)
    assert proof.data == pr.ser(oproof), "n = %d" % n
    assert (Cx, Cy) == (oCx, oCy)
    assert S.same(), "transcript or tape after the prove"
    ok_o, ok_l, ot, st = verify_both(sb, n, proof.data, a, Cx, Cy)
    assert ok_l == ok_o == (logn % 2 == 1)   # a given y = 12345 is not <x, a>: both verifiers reject that proof
    assert ot.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64), "transcript after the verify"


@pytest.mark.parametrize("logn", [18, 20])
def test_golden(sb, logn):
    path = os.path.join(ROOT, "tests", "golden", "dotlog_golden.json")
    want = json.load(open(path)).get(str(logn))
    assert want is not None, "tests/golden/dotlog_golden.json has no 2^%d entry (tests/golden/make_dotlog_golden.py)" % logn
    n = 1 << logn
    lg = sb.DotProductProofGens(n, b"dotlog-golden")
    x = sb.DensePolynomial(oc.prg_scalars("dotlog-golden-x-%d" % logn, n))
    a = sb.DensePolynomial(oc.prg_scalars("dotlog-golden-a-%d" % logn, n))
    bx, by = oc.prg_scalars("dotlog-golden-blinds-%d" % logn, 2)
    T, tape = sb.Transcript(b"dotlog-golden"), sb.RandomTape(sb.tape_seed(logn))
    proof, Cx, Cy = sb.DotProductProofLog.prove(lg, T, tape, x, bx, a, None, by)
    assert proof.data.hex() == want["proof"]
    assert (Cx.hex(), Cy.hex()) == (want["Cx"], want["Cy"])
    assert T.challenge_bytes(b"after", 64).hex() == want["transcript_after"]
    assert tape.challenge_bytes(b"after", 64).hex() == want["tape_after"]
    T2 = sb.Transcript(b"dotlog-golden")
    proof.verify(n, lg, T2, a, Cx, Cy)


# ---------------------------------------------------------------------------------------------------- rejections, with the oracle as judge
def _pt_mutants(P, G):
    Pp = pr._unpack(P)
    return {"P+G": (Pp + G).compress(), "-P": (Pp * (Q - 1)).compress(), "identity": bytes(32), "undecodable": b"\xff" * 32}


def _encode(Ls, Rs, delta, beta, z1, z2):
    return pr.ser([bytes(v) for v in Ls]) + pr.ser([bytes(v) for v in Rs]) + delta + beta + oc.mont_bytes(z1) + oc.mont_bytes(z2)


@pytest.mark.parametrize("logn", [3, 8, 9, 11])
def test_rejections_match_oracle(sb, logn):
    n = 1 << logn
    x, a = vectors(n, "mutants")
    proof, (Cx, Cy), _, _, _ = prove_both(sb, n, x, a, seed=100 + logn)
    p, _ = pr.deser(pr.DotProductProofLog, proof.data)
    Ls, Rs = list(p.bullet_reduction_proof.L_vec), list(p.bullet_reduction_proof.R_vec)
    G = gens(sb, n)[1].gens_1.g(0)
    cases = {}
    for i in range(logn):
        for kind, v in _pt_mutants(Ls[i], G).items():
            cases["L[%d] %s" % (i, kind)] = _encode(Ls[:i] + [v] + Ls[i + 1:], Rs, p.delta, p.beta, p.z1, p.z2)
        for kind, v in _pt_mutants(Rs[i], G).items():
            cases["R[%d] %s" % (i, kind)] = _encode(Ls, Rs[:i] + [v] + Rs[i + 1:], p.delta, p.beta, p.z1, p.z2)
    cases["L and R swapped"] = _encode(Rs, Ls, p.delta, p.beta, p.z1, p.z2)
    cases["L short"] = _encode(Ls[:-1], Rs, p.delta, p.beta, p.z1, p.z2)
    cases["both short"] = _encode(Ls[:-1], Rs[:-1], p.delta, p.beta, p.z1, p.z2)
    cases["R long"] = _encode(Ls, Rs + [Rs[0]], p.delta, p.beta, p.z1, p.z2)
    cases["both long"] = _encode(Ls + [Ls[0]], Rs + [Rs[0]], p.delta, p.beta, p.z1, p.z2)
    for kind, v in _pt_mutants(p.delta, G).items():
        cases["delta " + kind] = _encode(Ls, Rs, v, p.beta, p.z1, p.z2)
    for kind, v in _pt_mutants(p.beta, G).items():
        cases["beta " + kind] = _encode(Ls, Rs, p.delta, v, p.z1, p.z2)
    cases["z1 + 1"] = _encode(Ls, Rs, p.delta, p.beta, p.z1 + 1, p.z2)
    cases["z2 + 1"] = _encode(Ls, Rs, p.delta, p.beta, p.z1, (p.z2 + 1) % Q)
    assert _encode(Ls, Rs, p.delta, p.beta, p.z1, p.z2) == proof.data
    for name, data in cases.items():
        ok_o, ok_l, ot, st = verify_both(sb, n, data, a, Cx, Cy)
        assert not ok_o and not ok_l, name
    # the statement: a wrong Cx, Cy or a
    for name, (cx, cy, aa) in {"Cx": ((pr._unpack(Cx) + G).compress(), Cy, a), "Cy": (Cx, (pr._unpack(Cy) + G).compress(), a),
                               "a": (Cx, Cy, oc.to_arr([(ints(a)[0] + 1) % Q] + ints(a)[1:]))}.items():
        ok_o, ok_l, ot, st = verify_both(sb, n, proof.data, aa, cx, cy)
        assert not ok_o and not ok_l, "wrong " + name
        assert ot.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64), "transcript after rejecting a wrong " + name
    # a proof made with a wrong y, and the right one
    y = sum(p_ * q for p_, q in zip(ints(x), ints(a))) % Q
    bad, (bCx, bCy), obad, _, _ = prove_both(sb, n, x, a, y=(y + 1) % Q, seed=200 + logn)
    assert bad.data == pr.ser(obad)
    assert verify_both(sb, n, bad.data, a, bCx, bCy)[:2] == (False, False)
    assert verify_both(sb, n, proof.data, a, Cx, Cy)[:2] == (True, True)


# ---------------------------------------------------------------------------------------------------- inputs
@pytest.mark.parametrize("logn", [8, 9])
def test_device_and_host_vectors(sb, logn):
    """host arrays and DensePolynomial.from_tensor give the same bytes; the caller's vectors are unchanged; y=None is <x, a>"""
    torch = pytest.importorskip("torch")
    n = 1 << logn
    x, a = vectors(n, "inputs")
    lg, _ = gens(sb, n)
    outs = []
    for kind in ("host", "device"):
        if kind == "host":
            xv, av = x, a
        else:
            canon = lambda v: torch.tensor(np.frombuffer(b"".join(int(i).to_bytes(32, "little") for i in ints(v)), dtype=np.uint8).reshape(-1, 32), device="cuda:0")
            xv, av = sb.DensePolynomial.from_tensor(canon(x)), sb.DensePolynomial.from_tensor(canon(a))
        S = States(sb, 7)
        proof, Cx, Cy = sb.DotProductProofLog.prove(lg, S.st, S.stape, xv, L(3), av, None, L(4))
        if kind == "device":
            assert np.array_equal(xv.to_numpy(), x) and np.array_equal(av.to_numpy(), a), "the caller's vectors changed"
        outs.append((proof.data, Cx, Cy, S.raw()))
    assert outs[0] == outs[1]
    y = sum(p * q for p, q in zip(ints(x), ints(a))) % Q
    S = States(sb, 7)
    proof_y, _, _ = sb.DotProductProofLog.prove(lg, S.st, S.stape, x, L(3), a, L(y), L(4))
    assert proof_y.data == outs[0][0]


@pytest.mark.parametrize("logn", [6, 10])
def test_edge_values(sb, logn):
    n = 1 << logn
    cases = {"x zero": ([0] * n, list(range(n))),
             "a with zeros": ([Q - 1 - i for i in range(n)], [0 if i % 3 else 1 for i in range(n)]),
             "ones and q-1": ([1 if i % 2 else Q - 1 for i in range(n)], [Q - 1 if i % 4 else 1 for i in range(n)])}
    for name, (xi, ai) in cases.items():
        proof, C_, oproof, oC, S = prove_both(sb, n, oc.to_arr(xi), oc.to_arr(ai), seed=logn)
        assert proof.data == pr.ser(oproof) and C_ == oC, name
        assert S.same(), name


# ---------------------------------------------------------------------------------------------------- the fold kernel by itself
@pytest.fixture(scope="module")
def dt():
    lib = C.CDLL(os.path.join(ROOT, "spartan_b200", "libsp_devtest.so"))
    lib.spd_dotlog_fold.argtypes = [_sz, C.c_int, C.c_int, _vp, _vp, _vp]
    lib.spd_ristretto_decode.argtypes = [_sz, _vp, _vp, _vp]
    lib.spd_ristretto_encode.argtypes = [_sz, _vp, _vp]
    return lib


def _p(a):
    return a.ctypes.data_as(_vp)


FOLD_NIELS, FOLD_GE = 0, 1


def test_fold_kernel(sb, dt):
    """H_L + k H_R against the oracle's msm([1, k], [H_L, H_R]) = u * msm([u^-1, u], [G_L, G_R]) for k = u^2: k = 0, 1, q - 1, 2^252 - 1 (every
    4-bit window carries into the next), 8 * (16^63 - 1) / 15 (every digit 8: no carry), a random u^2; every pair of formats"""
    m = 37
    G = oc.MultiCommitGens.new(2 * m, b"dotlog-fold")
    enc = [G.g(i).compress() for i in range(2 * m)]
    enc[3] = bytes(32)          # an identity on the left
    enc[m + 5] = bytes(32)      # and on the right
    enc[m + 6] = enc[6]         # a pair of equal points
    raw = np.frombuffer(b"".join(enc), dtype=np.uint32).reshape(2 * m, 8).copy()
    pts = np.zeros((2 * m, 32), dtype=np.uint32)
    ok = np.zeros(2 * m, dtype=np.int32)
    assert dt.spd_ristretto_decode(_sz(2 * m), _p(raw), _p(pts), _p(ok)) == 0 and ok.all()
    u = int.from_bytes(os.urandom(32), "little") % Q
    ks = [0, 1, Q - 1, 2 ** 252 - 1, 8 * (16 ** 63 - 1) // 15, u * u % Q]
    ref_pts = [oc.Point.decompress(e) if e != bytes(32) else oc.Point.identity() for e in enc]
    for k in ks:
        want = [oc.msm([1, k], oc.points_array([ref_pts[i], ref_pts[i + m]])).compress() for i in range(m)]
        kk = np.frombuffer(k.to_bytes(32, "little"), dtype=np.uint32).copy()
        for fin, fout in ((FOLD_NIELS, FOLD_NIELS), (FOLD_NIELS, FOLD_GE), (FOLD_GE, FOLD_GE)):
            out = np.zeros((m, 32), dtype=np.uint32)
            assert dt.spd_dotlog_fold(_sz(m), fin, fout, _p(pts), _p(kk), _p(out)) == 0
            got = np.zeros((m, 8), dtype=np.uint32)
            assert dt.spd_ristretto_encode(_sz(m), _p(out), _p(got)) == 0
            assert [got[i].tobytes() for i in range(m)] == want, "k = %#x, formats %d -> %d" % (k, fin, fout)


# ---------------------------------------------------------------------------------------------------- refusals
def test_refusals(sb):
    ctx = sb.default_context()
    lib = sb.lib
    for n in (0, 3, 6, 2 ** 20 + 2 ** 19, MAX_N * 2):
        h = _vp()
        before = sb.kernel_launches()
        assert lib.sp_dotlog_gens_create(ctx.h, _sz(n), C.c_char_p(b"x"), _sz(1), C.byref(h)) == sb.api.SP_ERR_INVALID_ARG, n
        assert sb.kernel_launches() == before and not h.value
    for n in (TABLE_MAX_N, 2 * TABLE_MAX_N):
        lg, _ = gens(sb, n)
        x, a = vectors(n, "refuse")
        X, A, short = sb.DensePolynomial(x), sb.DensePolynomial(a), sb.DensePolynomial(x[: n // 2])
        other = sb.Context(0)
        foreign = sb.DensePolynomial(x, other)
        lg_other = sb.DotProductProofGens(n, GENS_LABEL, ctx=other)
        bad = np.array([2 ** 64 - 1] * 4, dtype=np.uint64)
        S = States(sb, 3)
        raw = S.raw()

        def refused(code, fn):
            before, live = sb.kernel_launches(), sb.device_bytes_live()
            with pytest.raises(Exception) as e:
                fn()
            assert sb.kernel_launches() == before
            assert S.raw() == raw, "transcript or tape touched"
            assert sb.device_bytes_live() == live
            return e.value

        refused(None, lambda: sb.DotProductProofLog.prove(lg, S.st, S.stape, short, L(1), A, None, L(2)))
        refused(None, lambda: sb.DotProductProofLog.prove(lg, S.st, S.stape, X, L(1), short, None, L(2)))
        refused(None, lambda: sb.DotProductProofLog.prove(lg, S.st, S.stape, foreign, L(1), A, None, L(2)))
        refused(None, lambda: sb.DotProductProofLog.prove(lg_other, S.st, S.stape, X, L(1), A, None, L(2)))
        for args in ((bad, None, L(2)), (L(1), bad, L(2)), (L(1), None, bad)):
            e = refused(None, lambda: sb.DotProductProofLog.prove(lg, S.st, S.stape, X, args[0], A, args[1], args[2]))
            assert isinstance(e, sb.R1CSError) and "InvalidScalar" in str(e)
        lg_small, _ = gens(sb, n // 2)
        refused(None, lambda: sb.DotProductProofLog.prove(lg_small, S.st, S.stape, X, L(1), A, None, L(2)))
        lg, _ = gens(sb, n)
        proof, Cx, Cy = sb.DotProductProofLog.prove(lg, sb.Transcript(b"r"), sb.RandomTape(sb.tape_seed(0)), X, L(1), A, None, L(2))
        refused(None, lambda: proof.verify(n // 2, lg, S.st, A, Cx, Cy))
        refused(None, lambda: proof.verify(n, lg, S.st, short, Cx, Cy))
        refused(None, lambda: proof.verify(n, lg, S.st, foreign, Cx, Cy))
        refused(None, lambda: proof.verify(n, lg, S.st, A, b"\xff" * 32, Cy))
        del foreign, lg_other, other


# ---------------------------------------------------------------------------------------------------- memory
@pytest.mark.parametrize("logn", [8, 9, 17])
def test_memory_returns_to_baseline(sb, logn):
    """prove and verify leave device_bytes_live where it was; gens above the threshold hold the points and the two-generator set only"""
    n = 1 << logn
    gc.collect()   # objects of earlier tests (another context among them) must not be freed between two readings
    gc.disable()
    try:
        memory_case(sb, n)
    finally:
        gc.enable()


def memory_case(sb, n):
    sb.release_cached_memory()
    live0 = sb.device_bytes_live()
    lg = sb.DotProductProofGens(n, b"dotlog-mem")
    held = sb.device_bytes_live() - live0
    if n > TABLE_MAX_N:
        assert held <= 96 * n + (4 << 20), held   # niels points and {G_n, h} with its 8-bit tables, no window table per generator
    x, a = vectors(n, "mem")
    X, A = sb.DensePolynomial(x), sb.DensePolynomial(a)
    for rep in range(2):   # the first call may grow the context's persistent scratch
        base = sb.device_bytes_live()
        T = sb.Transcript(b"mem")
        proof, Cx, Cy = sb.DotProductProofLog.prove(lg, T, sb.RandomTape(sb.tape_seed(1)), X, L(1), A, None, L(2))
        assert rep == 0 or sb.device_bytes_live() == base
        base = sb.device_bytes_live()
        proof.verify(n, lg, sb.Transcript(b"mem"), A, Cx, Cy)
        assert rep == 0 or sb.device_bytes_live() == base
    if n <= 2 ** 16:
        og = pr.DotProductProofGens(n, b"dotlog-mem")
        ot, otape = oc.Transcript(b"mem"), oc.RandomTape(b"proof", r1cs.tape_seed(1))
        xi, ai = ints(x), ints(a)
        op, _, _ = pr.DotProductProofLog.prove(og, ot, otape, xi, 1, ai, sum(p * q for p, q in zip(xi, ai)) % Q, 2)
        assert proof.data == pr.ser(op)


def test_memory_cases_under_memcheck(tmp_path):
    if os.environ.get("SP_MEMCHECK_OUT"):
        pytest.skip("already running under the memory-check mode")
    import subprocess
    import sys
    out = tmp_path / "memcheck.json"
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "tests"), ROOT] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    env["SP_MEMCHECK_OUT"] = str(out)
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "memcheck_plugin", "-p", "no:cacheprovider", "-k",
           "memory_returns_to_baseline or fold_kernel", os.path.join(ROOT, "tests", "test_gpu_dotlog.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-20000:]
    tot = json.load(open(out))
    assert tot["violations"] == 0, tot
    assert tot["blocks_filled"] > 0 and tot["context_refills"] > 0, tot
