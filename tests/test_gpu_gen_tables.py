"""GPU tests for generator tables shared by gens views (sb.GeneratorTables, sp_gen_tables_*, sp_*_gens_create_from): views prove the golden
bytes, including small circuits on the wide windows and row tables of 2^20 tables; views hold no device memory of their own; views, private gens
and the oracle agree byte for byte and accept each other's proofs; views beyond the tables' sizes, of NIZK-only tables or on another context are
refused.  Run on the GPU: pytest -m gpu."""
import ctypes as C
import hashlib
import json
import os

import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import r1cs, spark
from test_gpu_verify_batch import SHAPES  # noqa: E402  (the shapes the batch verifier is tested on)

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLD = json.load(open(os.path.join(GOLDEN, "oracle_golden.json")))
N20 = 1 << 20


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as m
    m.default_context()
    return m


def same(b, d):
    return len(b) == d["len"] and hashlib.sha256(b).hexdigest() == d["sha256"] and b[:48].hex() == d["head"] and b[-48:].hex() == d["tail"]


def test_views_of_2p20_tables_prove_golden_bytes(sb):
    """one GeneratorTables(2^20, 2^20, 10, 2^20): SNARK views at 2^16, 2^18 and 2^20 give the golden commitments and proofs; NIZK and SNARK
    views for the oracle_golden.json cases (2 to 1024 constraints, inner products of n = 2 to 32 on the tables' 13/15-bit windows) give the
    golden bytes too"""
    fx = json.load(open(os.path.join(GOLDEN, "snark_proof_sha256.json")))
    tables = sb.GeneratorTables(N20, N20, 10, N20)
    for logn in (16, 18, 20):
        n = 1 << logn
        inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=0)
        gens = sb.SNARKGens(n, n, 10, n, tables=tables)
        comm = sb.SNARK.encode(inst, gens)
        assert hashlib.sha256(comm.commitment_bytes()).hexdigest() == fx["%d_commitment" % logn]
        proof = sb.SNARK.prove(inst, comm, sb.DensePolynomial(vars_.limbs), inputs, gens, b"example", sb.tape_seed(0))
        assert len(proof.bytes) == fx["%d_len" % logn]
        assert hashlib.sha256(proof.bytes).hexdigest() == fx[str(logn)]
        if logn == 20:
            assert proof.bytes == open(os.path.join(GOLDEN, "snark_2p20_proof.bin"), "rb").read()
        proof.verify(comm, inputs, b"example", gens)
        del inst, vars_, inputs, gens, comm, proof
    label = GOLD["transcript_labels"]["nizk"].encode()
    for case in GOLD["nizk"]:
        inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(case["num_cons"], case["num_vars"], case["num_inputs"], seed=case["seed"])
        inst.set_digest(case["digest"].encode())
        gens = sb.NIZKGens(case["num_cons"], case["num_vars"], case["num_inputs"], tables=tables)
        proof = sb.NIZK.prove(inst, vars_, inputs, gens, label, sb.tape_seed(case["seed"]))
        assert same(proof.bytes, case["proof"]), "%dx%d" % (case["num_cons"], case["num_vars"])
        proof.verify(inst, inputs, label, gens)
    label = GOLD["transcript_labels"]["snark"].encode()
    for case in GOLD["snark"]:
        nc, nv, ni, seed = case["num_cons"], case["num_vars"], case["num_inputs"], case["seed"]
        inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(nc, nv, ni, seed=seed)
        gens = sb.SNARKGens(nc, nv, ni, nc, tables=tables)
        comm = sb.SNARK.encode(inst, gens)
        assert same(comm.commitment_bytes(), case["commitment"]), "%dx%d" % (nc, nv)
        proof = sb.SNARK.prove(inst, comm, vars_, inputs, gens, label, sb.tape_seed(seed))
        assert same(proof.bytes, case["proof"]), "%dx%d" % (nc, nv)
        proof.verify(comm, inputs, label, gens)


def test_views_share_the_tables_memory(sb):
    """views for every batch-verify shape and for 2^16, 2^18 and 2^20 add no device bytes to the 2^20 tables; they keep the tables alive after the
    caller's reference is dropped, and freeing them all returns the library's live bytes to what they were before the tables"""
    live0 = sb.device_bytes_live()
    tables = sb.GeneratorTables(N20, N20, 10, N20)
    live1 = sb.device_bytes_live()
    info = tables.info()
    assert [(s["label"], s["nbases"]) for s in info] == [("gens_r1cs_sat", 1026), ("gens_r1cs_eval", 4098)]
    assert live1 - live0 >= sum(s["device_bytes"] for s in info) > 0
    views = []
    for nc, nv, ni, _ in SHAPES:
        views += [sb.NIZKGens(nc, nv, ni, tables=tables), sb.SNARKGens(nc, nv, ni, nc, tables=tables)]
    for logn in (16, 18, 20):
        n = 1 << logn
        views += [sb.NIZKGens(n, n, 10, tables=tables), sb.SNARKGens(n, n, 10, n, tables=tables)]
    assert sb.device_bytes_live() == live1
    del tables
    assert sb.device_bytes_live() == live1
    del views[:]
    assert sb.device_bytes_live() == live0


@pytest.fixture(scope="module")
def shape_tables(sb):
    """tables for the largest of SHAPES in every dimension"""
    return sb.GeneratorTables(max(s[0] for s in SHAPES), max(s[1] for s in SHAPES), max(s[2] for s in SHAPES), max(s[0] for s in SHAPES))


@pytest.mark.parametrize("nc,nv,ni,seed", SHAPES)
def test_views_match_private_gens_and_oracle(sb, shape_tables, nc, nv, ni, seed):
    """same tape seed: a view, private gens and the oracle give the same commitment and proof bytes; proofs made with either kind of gens are
    accepted through the other by single and batch verify; the oracle's verifier accepts the bytes"""
    label = b"gen tables"
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(nc, nv, ni, seed=seed)
    oi, ovars, oinputs = r1cs.Instance.produce_synthetic_r1cs(nc, nv, ni, seed)
    oi.digest = inst.digest
    # NIZK
    view, own = sb.NIZKGens(nc, nv, ni, tables=shape_tables), sb.NIZKGens(nc, nv, ni)
    ogens = r1cs.NIZKGens(nc, nv, ni)
    oproof = r1cs.NIZK.prove(oi, ovars.copy(), oinputs, ogens, oc.Transcript(label), r1cs.tape_seed(seed))
    a = sb.NIZK.prove(inst, vars_, inputs, view, label, sb.tape_seed(seed))
    b = sb.NIZK.prove(inst, vars_, inputs, own, label, sb.tape_seed(seed))
    assert a.bytes == b.bytes == oproof.ser()
    a.verify(inst, inputs, label, own)
    b.verify(inst, inputs, label, view)
    for g in (view, own):
        assert sb.NIZK.verify_batch([a, b], inst, [inputs] * 2, label, g) == [None, None]
    oproof.verify(oi, oinputs, oc.Transcript(label), ogens)
    # SNARK
    view, own = sb.SNARKGens(nc, nv, ni, nc, tables=shape_tables), sb.SNARKGens(nc, nv, ni, nc)
    ogens = spark.SNARKGens(nc, nv, ni, nc)
    ocomm, odecomm = spark.SNARK.encode(oi, ogens)
    cv, co = sb.SNARK.encode(inst, view), sb.SNARK.encode(inst, own)
    assert cv.commitment_bytes() == co.commitment_bytes() == ocomm.ser()
    want = spark.SNARK.prove(oi, ocomm, odecomm, ovars.copy(), oinputs, ogens, oc.Transcript(label), r1cs.tape_seed(seed)).ser()
    a = sb.SNARK.prove(inst, cv, vars_, inputs, view, label, sb.tape_seed(seed))
    b = sb.SNARK.prove(inst, co, vars_, inputs, own, label, sb.tape_seed(seed))
    assert a.bytes == b.bytes == want
    a.verify(co, inputs, label, own)
    b.verify(cv, inputs, label, view)
    assert sb.SNARK.verify_batch([a, b], co, [inputs] * 2, label, view) == [None, None]
    assert sb.SNARK.verify_batch([a, b], cv, [inputs] * 2, label, own) == [None, None]
    parsed, pos = pr.deser(spark.SNARK, a.bytes)
    assert pos == len(a.bytes)
    parsed.verify(ocomm, oinputs, oc.Transcript(label), ogens)


def _create(sb, ctx, tables, *dims):
    """(status, message) of sp_snark_gens_create_from (4 dims) or sp_nizk_gens_create_from (3 dims); a created view is freed"""
    h = C.c_void_p()
    fn, free = (sb.lib.sp_snark_gens_create_from, sb.lib.sp_snark_gens_free) if len(dims) == 4 else (sb.lib.sp_nizk_gens_create_from, sb.lib.sp_nizk_gens_free)
    rc = fn(ctx.h, tables.h, *[C.c_size_t(d) for d in dims], C.byref(h))
    if h.value:
        free(h)
    return rc, sb.lib.sp_last_error(ctx.h).decode()


def test_boundaries(sb):
    """(128, 16, 8, 16) is sized so that doubling any one dimension needs more generators of a set: a view at the tables' size is accepted, one
    a power of two above in any dimension is refused with SP_ERR_INVALID_ARG and leaves the live device bytes as they were"""
    from spartan_b200 import api
    ctx = sb.default_context()
    tables = sb.GeneratorTables(128, 16, 8, 16)
    assert [s["nbases"] for s in tables.info()] == [6, 18]   # max(2^ceil(4/2) + 2, 5); 2^ceil(8/2) + 2 for ops (16 entries) and mem (128 rows)
    assert _create(sb, ctx, tables, 128, 16, 8, 16)[0] == api.SP_OK
    assert _create(sb, ctx, tables, 128, 16, 8)[0] == api.SP_OK
    live = sb.device_bytes_live()
    for dims in [(256, 16, 8, 16), (128, 32, 8, 16), (128, 16, 16, 16), (128, 16, 8, 32)]:
        rc, msg = _create(sb, ctx, tables, *dims)
        assert rc == api.SP_ERR_INVALID_ARG, dims
        assert "gens_r1cs_sat needs" in msg and "gens_r1cs_eval needs" in msg, msg
    for dims in [(128, 32, 8), (128, 16, 16)]:
        rc, msg = _create(sb, ctx, tables, *dims)
        assert rc == api.SP_ERR_INVALID_ARG and "gens_r1cs_sat needs 10 generators, has 6" in msg, (dims, msg)
    assert sb.device_bytes_live() == live
    with pytest.raises(sb.SpartanB200Error, match="needs"):
        sb.SNARKGens(128, 32, 8, 16, tables=tables)
    # NIZK-only tables: NIZK views yes, SNARK views no
    nizk_only = sb.GeneratorTables(128, 16, 8)
    assert [s["label"] for s in nizk_only.info()] == ["gens_r1cs_sat"]
    assert _create(sb, ctx, nizk_only, 128, 16, 8)[0] == api.SP_OK
    rc, msg = _create(sb, ctx, nizk_only, 16, 16, 3, 16)
    assert rc == api.SP_ERR_INVALID_ARG and "without SNARK sizes" in msg, msg
    # tables of another context (another GPU when there is one, else a second context on this one)
    other = sb.Context(1 if sb.lib.sp_device_count() > 1 else 0)
    for dims in [(16, 16, 3), (16, 16, 3, 16)]:
        rc, msg = _create(sb, other, tables, *dims)
        assert rc == api.SP_ERR_INVALID_ARG and "another context" in msg, msg


def test_views_prove_after_the_tables_are_dropped(sb):
    """gens made from tables keep proving, with the golden bytes, after the caller drops its reference to the tables"""
    case = GOLD["nizk"][0]
    nc, nv, ni, seed = case["num_cons"], case["num_vars"], case["num_inputs"], case["seed"]
    tables = sb.GeneratorTables(nc, nv, ni, nc)
    ngens, sgens = sb.NIZKGens(nc, nv, ni, tables=tables), sb.SNARKGens(nc, nv, ni, nc, tables=tables)
    del tables
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(nc, nv, ni, seed=seed)
    inst.set_digest(case["digest"].encode())
    label = GOLD["transcript_labels"]["nizk"].encode()
    assert same(sb.NIZK.prove(inst, vars_, inputs, ngens, label, sb.tape_seed(seed)).bytes, case["proof"])
    scase = next(c for c in GOLD["snark"] if (c["num_cons"], c["num_vars"], c["num_inputs"]) == (nc, nv, ni))
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(nc, nv, ni, seed=scase["seed"])
    comm = sb.SNARK.encode(inst, sgens)
    assert same(comm.commitment_bytes(), scase["commitment"])
    label = GOLD["transcript_labels"]["snark"].encode()
    proof = sb.SNARK.prove(inst, comm, vars_, inputs, sgens, label, sb.tape_seed(scase["seed"]))
    assert same(proof.bytes, scase["proof"])
    proof.verify(comm, inputs, label, sgens)
