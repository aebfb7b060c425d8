"""SNARK and NIZK proofs of R1CS instances shaped like real circuits (tests/test_instance_shapes.py CASES): several entries per row, empty rows, a
heavy row and column, duplicate entries, nnz that differs per matrix and from num_cons, num_vars != num_cons, and dimensions that Instance::new pads.
They put the size, padding and routing decisions of snark.cpp and prover.cpp on branches produce_synthetic_r1cs never reaches (the mirror in that
file names them per case); every proof is diffed byte for byte against the oracle.

Per case: the instance's exported matrices equal the oracle's and it is satisfied; SNARK::encode commitment, SNARK and NIZK proof bytes equal the
oracle's; the library's verifiers accept both proofs and reject single-byte flips; the oracle's verifier accepts the SNARK up to 2^15.  Also the
SPARK generator-size buckets, and the single-op instance snark_encode refuses.  Sharded proving is not covered here (tests/test_gpu_sharded.py).
Run on the GPU: pytest -m gpu."""
import gc
import os
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle.spartan_ref import core as oc  # noqa: E402
from oracle.spartan_ref import protocol as pr  # noqa: E402
from oracle.spartan_ref import r1cs, spark  # noqa: E402
from test_instance_shapes import CASES, Spec, cached_instance, gens_widths, spec_plan  # noqa: E402

LABEL = b"instance shapes"
ORACLE_VERIFY_MAX = 1 << 15


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as m
    m.default_context()
    oc.lib.oracle_set_threads(max(1, (os.cpu_count() or 2) // 2))
    return m


@pytest.fixture(autouse=True)
def release_device_memory(sb):
    """each case builds generator sets of up to several GB whose blocks the library keeps cached for reuse after they are freed: hand them back to
    the driver, so that the tests after these, and the processes they start on the same GPU, find the memory free"""
    yield
    gc.collect()
    sb.release_cached_memory()


def first_diff(a, b):
    if len(a) != len(b):
        return "lengths %d != %d" % (len(a), len(b))
    return next((i for i in range(len(a)) if a[i] != b[i]), None)


def flips(data, n, seed):
    """n single-byte flips spread over the proof, the first and last byte included"""
    rng = np.random.default_rng(seed)
    for p in sorted({0, len(data) - 1} | {int(x) for x in rng.integers(0, len(data), size=n)}):
        b = bytearray(data)
        b[p] ^= 1 << int(rng.integers(0, 8))
        yield p, bytes(b)


def library_instance(sb, si):
    s = si.spec
    inst = sb.Instance.new(s.num_cons, s.num_vars, s.num_inputs, *si.triples)
    return inst, sb.Assignment(si.vars), sb.Assignment(oc.to_arr(si.inputs) if si.inputs else oc.zeros(0))


class Clock:
    def __init__(self):
        self.t = {"oracle": 0.0, "library": 0.0}

    def run(self, who, f, *a):
        t0 = time.perf_counter()
        out = f(*a)
        self.t[who] += time.perf_counter() - t0
        return out


@pytest.mark.parametrize("name", list(CASES))
def test_case_matches_oracle(sb, name):
    spec, _ = CASES[name]
    seed = 3
    clk = Clock()
    si = cached_instance(spec)
    oi = si.oracle
    plan = spec_plan(spec)
    inst, vars_, inputs = clk.run("library", library_instance, sb, si)
    for m, M in enumerate((oi.inst.A, oi.inst.B, oi.inst.C)):
        row, col, val = inst.export(m)
        assert np.array_equal(row, M.row) and np.array_equal(col, M.col) and np.array_equal(val, M.val), "matrix %d" % m
    assert (inst.num_cons, inst.num_vars) == (plan["num_cons"], plan["num_vars"])
    assert inst.is_sat(vars_, inputs)

    # SNARK
    nz = max(spec.nnz)
    ogens = clk.run("oracle", spark.SNARKGens, spec.num_cons, spec.num_vars, spec.num_inputs, nz)
    ocomm, odecomm = clk.run("oracle", spark.SNARK.encode, oi, ogens)
    assert ocomm.comm.num_ops == plan["N"] and ocomm.comm.num_mem_cells == plan["cells"]
    want = clk.run("oracle", lambda: spark.SNARK.prove(oi, ocomm, odecomm, si.vars, si.inputs, ogens, oc.Transcript(LABEL), r1cs.tape_seed(seed)).ser())
    gens = clk.run("library", sb.SNARKGens, spec.num_cons, spec.num_vars, spec.num_inputs, nz)
    comm = clk.run("library", sb.SNARK.encode, inst, gens)
    assert first_diff(comm.commitment_bytes(), ocomm.ser()) is None, "commitment: first differing byte %s" % first_diff(comm.commitment_bytes(), ocomm.ser())
    proof = clk.run("library", sb.SNARK.prove, inst, comm, vars_, inputs, gens, LABEL, sb.tape_seed(seed))
    d = first_diff(proof.bytes, want)
    assert d is None, "SNARK: first differing byte %s of %d" % (d, len(want))
    if name == "tall_sparse":
        # without the background commitment the dereferenced values are committed on the prover's stream, after ry is left-padded to rx's length
        ctx = sb.default_context()
        ctx.set_overlap(False)
        try:
            off = clk.run("library", sb.SNARK.prove, inst, comm, vars_, inputs, gens, LABEL, sb.tape_seed(seed))
        finally:
            ctx.set_overlap(True)
        d = first_diff(off.bytes, want)
        assert d is None, "SNARK with overlap off: first differing byte %s of %d" % (d, len(want))
    proof.verify(comm, inputs, LABEL, gens)
    for pos, bad in flips(proof.bytes, 4, seed):
        with pytest.raises(sb.ProofVerifyError):
            sb.SNARK(bad).verify(comm, inputs, LABEL, gens)
    if max(plan["N"], plan["cells"]) <= ORACLE_VERIFY_MAX:
        parsed, pos = pr.deser(spark.SNARK, proof.bytes)
        assert pos == len(proof.bytes)
        clk.run("oracle", parsed.verify, ocomm, si.inputs, oc.Transcript(LABEL), ogens)

    # NIZK
    inst.set_digest(oi.digest)
    onproof = clk.run("oracle", lambda: r1cs.NIZK.prove(oi, si.vars, si.inputs, r1cs.NIZKGens(spec.num_cons, spec.num_vars, spec.num_inputs),
                                                         oc.Transcript(LABEL), r1cs.tape_seed(seed)).ser())
    ngens = clk.run("library", sb.NIZKGens, spec.num_cons, spec.num_vars, spec.num_inputs)
    nproof = clk.run("library", sb.NIZK.prove, inst, vars_, inputs, ngens, LABEL, sb.tape_seed(seed))
    d = first_diff(nproof.bytes, onproof)
    assert d is None, "NIZK: first differing byte %s of %d" % (d, len(onproof))
    nproof.verify(inst, inputs, LABEL, ngens)
    for pos, bad in flips(nproof.bytes, 4, seed):
        with pytest.raises(sb.ProofVerifyError):
            sb.NIZK(bad).verify(inst, inputs, LABEL, ngens)
    print("\n%s: oracle %.1f s, library %.1f s (N = %d, cells = %d)" % (name, clk.t["oracle"], clk.t["library"], plan["N"], plan["cells"]))


BUCKET = Spec("buckets", 512, 512, 10, (1225, 700, 900))   # N = 2^11


def test_generator_size_buckets(sb):
    """SNARKGens sized for any nz in N's power-of-two bucket proves with the oracle's bytes; one bucket smaller or larger changes exactly one of the
    comb_ops / derefs generator widths and raises SP_ERR_INVALID_ARG from SNARK::encode (comb_ops) or SNARK::prove (derefs), never a proof"""
    si = cached_instance(BUCKET)
    s = BUCKET
    assert spec_plan(s)["N"] == 1 << 11
    ogens = spark.SNARKGens(s.num_cons, s.num_vars, s.num_inputs, 1 << 11)
    ocomm, odecomm = spark.SNARK.encode(si.oracle, ogens)
    want = spark.SNARK.prove(si.oracle, ocomm, odecomm, si.vars, si.inputs, ogens, oc.Transcript(LABEL), r1cs.tape_seed(0)).ser()
    inst, vars_, inputs = library_instance(sb, si)
    for nz in ((1 << 10) + 1, 1 << 11):
        gens = sb.SNARKGens(s.num_cons, s.num_vars, s.num_inputs, nz)
        comm = sb.SNARK.encode(inst, gens)
        assert comm.commitment_bytes() == ocomm.ser()
        assert sb.SNARK.prove(inst, comm, vars_, inputs, gens, LABEL, sb.tape_seed(0)).bytes == want
    base = gens_widths(s.num_cons, s.num_vars, s.num_inputs, 1 << 11)
    stages = set()
    for nz in (1 << 10, 1 << 12):
        w = gens_widths(s.num_cons, s.num_vars, s.num_inputs, nz)
        gens = sb.SNARKGens(s.num_cons, s.num_vars, s.num_inputs, nz)
        if w[0] != base[0]:
            with pytest.raises(sb.SpartanB200Error, match="error 3"):
                sb.SNARK.encode(inst, gens)
            stages.add("encode")
        else:
            assert w[2] != base[2]
            comm = sb.SNARK.encode(inst, gens)
            with pytest.raises(sb.SpartanB200Error, match="error 3"):
                sb.SNARK.prove(inst, comm, vars_, inputs, gens, LABEL, sb.tape_seed(0))
            stages.add("prove")
    assert stages == {"encode", "prove"}


def test_single_op_instance_is_refused(sb):
    """every matrix with at most one entry gives N = 1: product circuits without layers.  SNARK::encode refuses it with SP_ERR_INVALID_ARG before
    any device work (the oracle fails in its ProductCircuit), and SNARK::verify refuses a commitment that claims fewer than two ops"""
    one = (1).to_bytes(32, "little")
    A, B, Cm = [(0, 0, one)], [(0, 0, one)], [(0, 0, one)]
    inst = sb.Instance.new(2, 2, 1, A, B, Cm)
    gens = sb.SNARKGens(2, 2, 1, 1)
    with pytest.raises(sb.SpartanB200Error, match="error 3") as e:
        sb.SNARK.encode(inst, gens)
    assert not isinstance(e.value, sb.ProofVerifyError)
    oi = r1cs.Instance.new(2, 2, 1, A, B, Cm)
    ogens = spark.SNARKGens(2, 2, 1, 1)
    ocomm, odecomm = spark.SNARK.encode(oi, ogens)
    with pytest.raises(AssertionError):
        spark.SNARK.prove(oi, ocomm, odecomm, oc.to_arr([1, 0]), [0], ogens, oc.Transcript(LABEL), r1cs.tape_seed(0))

    from spartan_b200 import api
    si = cached_instance(CASES["many_inputs"][0])
    s = si.spec
    inst, vars_, inputs = library_instance(sb, si)
    gens = sb.SNARKGens(s.num_cons, s.num_vars, s.num_inputs, max(s.nnz))
    comm = sb.SNARK.encode(inst, gens)
    proof = sb.SNARK.prove(inst, comm, vars_, inputs, gens, LABEL, sb.tape_seed(0))
    raw = comm.commitment_bytes()
    api.SNARK(proof.bytes).verify(api.ComputationCommitment.from_bytes(raw), inputs, LABEL, gens)
    for num_ops in (1, 0):
        bad = raw[:32] + num_ops.to_bytes(8, "little") + raw[40:]     # num_cons, num_vars, num_inputs, batch_size, num_ops, ...
        with pytest.raises(sb.SpartanB200Error, match="error 3") as e:
            proof.verify(api.ComputationCommitment.from_bytes(bad), inputs, LABEL, gens)
        assert not isinstance(e.value, sb.ProofVerifyError)
