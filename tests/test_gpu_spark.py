"""SPARK on the caller's matrices on the GPU (SparseMatPolyCommitmentGens, SparseMatPolynomial.multi_commit / multi_evaluate,
SparseMatPolyEvalProof.prove / verify) against the oracle, for b = 1 .. 4 matrices on shapes with x = y, x < y (x = 0 included) and x > y,
entry counts on and off powers of two, one matrix far shorter than the others, all entries on one row or one column, entries at the maximum
index: commitment bytes, evaluations, proof bytes (the oracle's prove at b = 3, the generalisation in test_spark_model.py otherwise), transcript
and tape states, and both verifiers on each other's transcripts.  Then rejections, refusals, device input, one 2^20 case and the memory-check
mode."""
import zlib

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import r1cs as r1
from oracle.spartan_ref import spark as sk
from test_spark_model import spark_prove

pytestmark = pytest.mark.gpu
Q = oc.Q
LABEL = b"spark-gpu"


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    sb.default_context()
    return sb


def entries(tag, x, y, n, pattern):
    rng = np.random.default_rng(zlib.crc32(repr((tag, x, y, n, pattern)).encode()))
    rows = rng.integers(0, 1 << x, n, dtype=np.uint64)
    cols = rng.integers(0, 1 << y, n, dtype=np.uint64)
    if pattern == "row":
        rows[:] = (1 << x) - 1
    if pattern == "col":
        cols[:] = 0
    if n:
        rows[0], cols[0] = (1 << x) - 1, (1 << y) - 1    # the maximum index
    vals = oc.prg_scalars("spark-gpu-%s-%d" % (tag, n), n) if n else oc.zeros(0)
    return rows, cols, vals


def canonical(vals):
    return np.frombuffer(b"".join(oc.scalar_to_bytes(v) for v in oc.to_ints(vals)), dtype=np.uint8).reshape(-1, 32)


def build(sb, tag, x, y, nnzs, pattern="random"):
    ents = [entries("%s-%d" % (tag, i), x, y, n, pattern) for i, n in enumerate(nnzs)]
    b = len(nnzs)
    opolys = [r1.SparseMat(x, y, r, c, v) for r, c, v in ents]
    spolys = [sb.SparseMatPolynomial(x, y, r, c, canonical(v)) for r, c, v in ents]
    return ents, opolys, spolys, sb.SparseMatPolyCommitmentGens(LABEL, x, y, max(nnzs), b), sk.SparseMatPolyCommitmentGens(LABEL, x, y, max(nnzs), b)


def point(tag, x, y):
    rx = oc.prg_scalars("spark-gpu-rx-" + tag, x) if x else oc.zeros(0)
    ry = oc.prg_scalars("spark-gpu-ry-" + tag, y) if y else oc.zeros(0)
    return rx, ry, (oc.to_ints(rx) if x else []), (oc.to_ints(ry) if y else [])


def pair(sb, label=b"spark-gpu-t"):
    ot, st = oc.Transcript(label), sb.Transcript(label)
    for t in (ot, st):
        t.append_message(b"app", b"prefix")
    return ot, st


def state(t):
    return bytes(t.state.raw)


def same(ot, st):
    """the oracle's and the library's transcript (or tape) in the same state: they draw the same challenge"""
    return ot.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64)


CASES = [
    ("b1-sq", 5, 5, [37], "random"),
    ("b1-x0", 0, 6, [64], "random"),
    ("b2-xlty", 3, 7, [100, 5], "random"),
    ("b2-col", 6, 6, [128, 128], "col"),
    ("b3-xgty", 8, 5, [700, 1024, 3], "random"),
    ("b3-row", 6, 9, [513, 40, 200], "row"),
    ("b4-x0", 0, 7, [200, 50, 256, 1], "random"),
    ("b4-big", 10, 9, [1 << 12, 3000, 1 << 11, 17], "random"),
    ("b3-2p14", 12, 12, [1 << 14, 1 << 13, 9000], "random"),
]


@pytest.mark.parametrize("tag,x,y,nnzs,pattern", CASES, ids=[c[0] for c in CASES])
def test_against_the_oracle(sb, tag, x, y, nnzs, pattern):
    b = len(nnzs)
    _, opolys, spolys, gens, ogens = build(sb, tag, x, y, nnzs, pattern)
    comm, dense = sb.SparseMatPolynomial.multi_commit(spolys, gens)
    ocomm, odense = sk.multi_commit(opolys, ogens)
    assert comm.to_bytes() == ocomm.ser()
    assert sb.SparseMatPolyCommitment.from_bytes(comm.to_bytes()).to_bytes() == comm.to_bytes()
    rx, ry, rxi, ryi = point(tag, x, y)
    trx, try_ = oc.eq_evals(rxi), oc.eq_evals(ryi)
    oev = [p.evaluate_with_tables(trx, try_) for p in opolys]
    assert oc.to_ints(sb.SparseMatPolynomial.multi_evaluate(dense, rx, ry)) == oev
    # prove from the same transcript state and tape seed
    seed = oc.prg_scalars("spark-gpu-seed-" + tag, 1)
    ot, st = pair(sb)
    otape, stape = oc.RandomTape(b"proof", oc.to_ints(seed)[0]), sb.RandomTape(seed[0])
    proof, ev = sb.SparseMatPolyEvalProof.prove(dense, rx, ry, None, gens, st, stape)
    assert oc.to_ints(ev) == oev
    oproof = (sk.SparseMatPolyEvalProof.prove if b == 3 else spark_prove)(odense, rxi, ryi, oev, ogens, ot, otape)
    assert proof.data == pr.ser(oproof)
    assert same(ot, st)
    assert same(otape.tape, stape)
    # given (correct) evaluations give the same proof
    _, st2 = pair(sb)
    proof2, _ = sb.SparseMatPolyEvalProof.prove(dense, rx, ry, ev, gens, st2, sb.RandomTape(seed[0]))
    assert proof2.data == proof.data
    # both verifiers accept, and leave the same transcript
    ot, st = pair(sb)
    proof.verify(comm, rx, ry, ev, gens, st)
    oproof.verify(ocomm, rxi, ryi, oev, ogens, ot)
    assert same(ot, st)


def test_rejections(sb):
    tag, x, y, nnzs = "rej", 4, 6, [40, 64, 9, 33]
    _, _, spolys, gens, _ = build(sb, tag, x, y, nnzs)
    comm, dense = sb.SparseMatPolynomial.multi_commit(spolys, gens)
    rx, ry, _, _ = point(tag, x, y)
    proof, ev = sb.SparseMatPolyEvalProof.prove(dense, rx, ry, None, gens, b"t", sb.RandomTape(sb.tape_seed(1)))
    proof.verify(comm, rx, ry, ev, gens, b"t")

    def rejected(data=proof.data, c=comm, rx=rx, ry=ry, ev=ev):
        with pytest.raises(sb.ProofVerifyError) as e:
            sb.SparseMatPolyEvalProof(data).verify(c, rx, ry, ev, gens, b"t")
        return str(e.value)
    bad = ev.copy(); bad[2] = oc.prg_scalars("other", 1)[0]
    rejected(ev=bad)
    rx2 = rx.copy(); rx2[1] = oc.prg_scalars("other", 1)[0]
    rejected(rx=rx2)
    other = [sb.SparseMatPolynomial(x, y, *e[:2], canonical(e[2])) for e in (entries("rej-other-%d" % i, x, y, n, "random") for i, n in enumerate(nnzs))]
    rejected(c=sb.SparseMatPolynomial.multi_commit(other, gens)[0])
    for off in (40, 300, len(proof.data) // 3, len(proof.data) // 2, len(proof.data) - 100, len(proof.data) - 1):
        d = bytearray(proof.data); d[off] ^= 1
        rejected(data=bytes(d))
    # a commitment of another shape is refused before the transcript is touched
    c = sb.SparseMatPolyCommitment.from_bytes(comm.to_bytes()); c.num_mem_cells *= 2
    t = sb.Transcript(b"t"); before = state(t)
    with pytest.raises(sb.ProofVerifyError):
        proof.verify(c, rx, ry, ev, gens, t)
    assert state(t) == before


def expect(sb, fn, exc, words, *transcripts):
    before = [state(t) for t in transcripts]
    with pytest.raises(exc) as e:
        fn()
    assert all(w in str(e.value) for w in words), str(e.value)
    assert [state(t) for t in transcripts] == before


def test_refusals(sb):
    Err, R1 = sb.SpartanB200Error, sb.R1CSError
    expect(sb, lambda: sb.SparseMatPolyCommitmentGens(LABEL, 3, 3, 16, 5), Err, ["batch_size"])
    expect(sb, lambda: sb.SparseMatPolyCommitmentGens(LABEL, 3, 3, 16, 0), Err, ["batch_size"])
    expect(sb, lambda: sb.SparseMatPolyCommitmentGens(LABEL, 0, 0, 16, 1), Err, ["= 0"])
    expect(sb, lambda: sb.SparseMatPolyCommitmentGens(LABEL, 31, 2, 16, 1), Err, ["32-bit"])
    x, y = 3, 4
    gens = sb.SparseMatPolyCommitmentGens(LABEL, x, y, 16, 2)
    r, c, v = entries("ref", x, y, 16, "random")
    good = sb.SparseMatPolynomial(x, y, r, c, canonical(v))
    one = sb.SparseMatPolynomial(x, y, r[:1], c[:1], canonical(v[:1]))
    commit = sb.SparseMatPolynomial.multi_commit
    expect(sb, lambda: commit([good] * 5, gens), Err, ["matrices"])
    expect(sb, lambda: commit([one, one], gens), Err, ["at most one entry"])
    expect(sb, lambda: commit([good, good], sb.SparseMatPolyCommitmentGens(LABEL, x, y + 4, 16, 2)), Err, ["do not fit"])
    expect(sb, lambda: commit([good, sb.SparseMatPolynomial(x, y, r[:3], c[:3], canonical(v[:3]))], sb.SparseMatPolyCommitmentGens(LABEL, x, y, 64, 2)), Err,
           ["do not fit"])
    r2 = r.copy(); r2[5] = 1 << x
    c2 = c.copy(); c2[3] = 1 << y
    big = canonical(v).copy(); big[7] = 0xFF
    expect(sb, lambda: commit([good, sb.SparseMatPolynomial(x, y, r2, c2, canonical(v))], gens), R1, ["InvalidIndex", "col", "matrix 1, entry 3"])
    expect(sb, lambda: commit([sb.SparseMatPolynomial(x, y, r2, c, big), good], gens), R1, ["InvalidIndex", "row", "matrix 0, entry 5"])
    expect(sb, lambda: commit([good, sb.SparseMatPolynomial(x, y, r, c, big)], gens), R1, ["InvalidScalar"])
    comm, dense = commit([good, good], gens)
    rx, ry, _, _ = point("ref", x, y)
    t, tape = sb.Transcript(b"t"), sb.RandomTape(sb.tape_seed(2))
    prove = sb.SparseMatPolyEvalProof.prove
    ev = sb.SparseMatPolynomial.multi_evaluate(dense, rx, ry)
    bad = ev.copy(); bad[1] = ev[0] if oc.to_ints(ev[:1]) != oc.to_ints(ev[1:2]) else oc.prg_scalars("x", 1)[0]
    expect(sb, lambda: prove(dense, rx, ry, bad, gens, t, tape), Err, ["evals[1]"], t, tape)
    expect(sb, lambda: prove(dense, rx[:2], ry, None, gens, t, tape), Err, ["|rx| = 2"], t, tape)
    expect(sb, lambda: prove(dense, rx, ry, None, sb.SparseMatPolyCommitmentGens(LABEL, x, y, 16, 3), t, tape), Err, ["do not fit"], t, tape)
    other_gens = sb.SparseMatPolyCommitmentGens(LABEL, x, y, 16, 2, ctx=sb.Context())
    expect(sb, lambda: prove(dense, rx, ry, None, other_gens, t, tape), Err, ["another context"], t, tape)
    notred = rx.copy(); notred[0] = np.array([2**64 - 1] * 4, dtype=np.uint64)
    expect(sb, lambda: prove(dense, notred, ry, None, gens, t, tape), R1, ["InvalidScalar"], t, tape)
    proof, _ = prove(dense, rx, ry, None, gens, b"t", sb.RandomTape(sb.tape_seed(2)))
    expect(sb, lambda: proof.verify(comm, rx, ry, np.concatenate([ev, ev])[:5], gens, t), Err, ["evaluations"], t)
    expect(sb, lambda: proof.verify(comm, rx, ry, ev[:1], gens, t), sb.ProofVerifyError, ["batch size"], t)
    expect(sb, lambda: proof.verify(comm, notred, ry, ev, gens, t), R1, ["InvalidScalar"], t)


def test_device_input_equals_host_input(sb):
    import torch
    x, y, nnzs = 5, 7, [300, 77, 128]
    ents, _, spolys, gens, _ = build(sb, "dev", x, y, nnzs)
    comm, dense = sb.SparseMatPolynomial.multi_commit(spolys, gens)
    dpolys = [sb.SparseMatPolynomial.from_tensors(x, y, torch.tensor(r.astype(np.int64), device="cuda"), torch.tensor(c.astype(np.int64), device="cuda"),
                                                 torch.tensor(canonical(v), device="cuda")) for r, c, v in ents]
    dcomm, ddense = sb.SparseMatPolynomial.multi_commit(dpolys, gens)
    assert dcomm.to_bytes() == comm.to_bytes()
    rx, ry, _, _ = point("dev", x, y)
    p1, _ = sb.SparseMatPolyEvalProof.prove(dense, rx, ry, None, gens, b"t", sb.RandomTape(sb.tape_seed(3)))
    p2, _ = sb.SparseMatPolyEvalProof.prove(ddense, rx, ry, None, gens, b"t", sb.RandomTape(sb.tape_seed(3)))
    assert p1.data == p2.data
    bad = torch.tensor(np.array([1 << y], dtype=np.int64), device="cuda")
    one = torch.zeros(1, dtype=torch.int64, device="cuda")
    with pytest.raises(sb.R1CSError, match="col"):
        sb.SparseMatPolynomial.multi_commit([dpolys[0], sb.SparseMatPolynomial.from_tensors(x, y, one, bad, torch.zeros((1, 32), dtype=torch.uint8, device="cuda"))],
                                            sb.SparseMatPolyCommitmentGens(LABEL, x, y, 300, 2))


def test_scale_2p20(sb):
    x = y = 20
    n = 1 << 20
    gens = sb.SparseMatPolyCommitmentGens(LABEL, x, y, n, 3)
    polys = []
    for i in range(3):
        rng = np.random.default_rng(100 + i)
        vals = np.zeros((n, 32), dtype=np.uint8)
        vals[:, :31] = rng.integers(0, 256, (n, 31), dtype=np.uint8)
        polys.append(sb.SparseMatPolynomial(x, y, rng.integers(0, n, n, dtype=np.uint64), rng.integers(0, n, n, dtype=np.uint64), vals))
    comm, dense = sb.SparseMatPolynomial.multi_commit(polys, gens)
    rx, ry, _, _ = point("scale", x, y)
    proof, ev = sb.SparseMatPolyEvalProof.prove(dense, rx, ry, None, gens, b"t", sb.RandomTape(sb.tape_seed(4)))
    proof.verify(comm, rx, ry, ev, gens, b"t")


def test_memcheck_b4(sb):
    sb.debug_memcheck(True)
    try:
        v0 = sb.debug_memcheck_report()["violations"]
        ctx = sb.Context()
        x, y, nnzs = 3, 6, [33, 64, 7, 50]
        ents = [entries("mc-%d" % i, x, y, n, "random") for i, n in enumerate(nnzs)]
        gens = sb.SparseMatPolyCommitmentGens(LABEL, x, y, 64, 4, ctx=ctx)
        ogens = sk.SparseMatPolyCommitmentGens(LABEL, x, y, 64, 4)
        comm, dense = sb.SparseMatPolynomial.multi_commit([sb.SparseMatPolynomial(x, y, r, c, canonical(v)) for r, c, v in ents], gens)
        ocomm, odense = sk.multi_commit([r1.SparseMat(x, y, r, c, v) for r, c, v in ents], ogens)
        assert comm.to_bytes() == ocomm.ser()
        rx, ry, rxi, ryi = point("mc", x, y)
        seed = oc.prg_scalars("spark-gpu-seed-mc", 1)
        proof, ev = sb.SparseMatPolyEvalProof.prove(dense, rx, ry, None, gens, b"t", sb.RandomTape(seed[0]))
        oproof = spark_prove(odense, rxi, ryi, oc.to_ints(ev), ogens, oc.Transcript(b"t"), oc.RandomTape(b"proof", oc.to_ints(seed)[0]))
        assert proof.data == pr.ser(oproof)
        proof.verify(comm, rx, ry, ev, gens, b"t")
        del dense, gens, ctx
        assert sb.debug_memcheck_scan() == 0
        rep = sb.debug_memcheck_report()
        assert rep["violations"] == v0, rep["last_violation"]
    finally:
        sb.debug_memcheck(False)
