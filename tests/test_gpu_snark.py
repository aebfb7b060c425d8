"""GPU parity for the SNARK path (BASELINE.json configs[1]/[4] shape): SNARK::encode commitments and SNARK::prove proof bytes diffed
against the oracle from 2 constraints up to the bench configuration itself (2^16 and 2^20: the oracle proves 2^20 in well under a minute on
the box's host cores); the published structural lengths (README.md:362,371,374) must hold and the oracle's SNARK::verify must accept.
Run on the GPU: pytest -m gpu."""
import os
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle.spartan_ref import core as oc  # noqa: E402
from oracle.spartan_ref import protocol as pr  # noqa: E402
from oracle.spartan_ref import r1cs, spark  # noqa: E402


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as m
    m.default_context()
    return m


def parse_commitment(b):
    vals = [int.from_bytes(b[8 * i:8 * i + 8], "little") for i in range(6)]
    ops, pos = pr.deser(pr.PolyCommitment, b, 48)
    mem, pos = pr.deser(pr.PolyCommitment, b, pos)
    assert pos == len(b)
    return spark.R1CSCommitment(vals[0], vals[1], vals[2], spark.SparseMatPolyCommitment(vals[3], vals[4], vals[5], ops, mem))


@pytest.mark.parametrize("num_cons,num_vars,num_inputs,seed", [(16, 16, 3, 0), (256, 256, 10, 1), (1024, 1024, 10, 2), (64, 256, 7, 3), (512, 32, 5, 4), (2, 2, 1, 5)])
def test_snark_bytes_match_oracle(sb, num_cons, num_vars, num_inputs, seed):
    nz = num_cons
    oi, ovars, oinputs = r1cs.Instance.produce_synthetic_r1cs(num_cons, num_vars, num_inputs, seed)
    ogens = spark.SNARKGens(num_cons, num_vars, num_inputs, nz)
    ocomm, odecomm = spark.SNARK.encode(oi, ogens)
    oproof = spark.SNARK.prove(oi, ocomm, odecomm, ovars, oinputs, ogens, oc.Transcript(b"snark_example"), r1cs.tape_seed(seed))
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(num_cons, num_vars, num_inputs, seed=seed)
    gens = sb.SNARKGens(num_cons, num_vars, num_inputs, nz)
    comm = sb.SNARK.encode(inst, gens)
    assert comm.commitment_bytes() == ocomm.ser()
    proof = sb.SNARK.prove(inst, comm, vars_, inputs, gens, b"snark_example", sb.tape_seed(seed))
    want = oproof.ser()
    assert len(proof.bytes) == len(want)
    first = next((i for i in range(len(want)) if want[i] != proof.bytes[i]), None)
    assert first is None, "first differing byte at %d of %d" % (first, len(want))
    proof2 = sb.SNARK.prove(inst, comm, sb.DensePolynomial(vars_.limbs), inputs, gens, b"snark_example", sb.tape_seed(seed))
    assert proof2.bytes == want
    assert sb.SNARK.prove(inst, comm, vars_, inputs, gens, b"snark_example", sb.tape_seed(seed + 7)).bytes != want


def test_snark_padded_constraints(sb):
    """lib.rs:672-752 test_padded_constraints through the GPU prover, bytes equal to the oracle and accepted by its verifier"""
    def s32(v):
        return (v % oc.Q).to_bytes(32, "little")
    num_cons, num_vars, num_inputs, nz = 1, 0, 3, 3
    A = [(0, num_vars + 2, s32(1))]
    B = [(0, num_vars + 2, s32(1))]
    Cm = [(0, num_vars + 1, s32(1)), (0, num_vars, s32(-13)), (0, num_vars + 3, s32(-1))]
    inst = sb.Instance.new(num_cons, num_vars, num_inputs, A, B, Cm)
    vars_ = sb.Assignment([])
    inputs = sb.Assignment([s32(16), s32(1), s32(2)])
    assert inst.is_sat(vars_, inputs)
    gens = sb.SNARKGens(num_cons, num_vars, num_inputs, nz)
    comm = sb.SNARK.encode(inst, gens)
    proof = sb.SNARK.prove(inst, comm, vars_, inputs, gens, b"snark_example", sb.tape_seed(0))
    oi = r1cs.Instance.new(num_cons, num_vars, num_inputs, A, B, Cm)
    ogens = spark.SNARKGens(num_cons, num_vars, num_inputs, nz)
    ocomm, odecomm = spark.SNARK.encode(oi, ogens)
    assert comm.commitment_bytes() == ocomm.ser()
    oproof = spark.SNARK.prove(oi, ocomm, odecomm, oc.zeros(0), [16, 1, 2], ogens, oc.Transcript(b"snark_example"), r1cs.tape_seed(0))
    assert proof.bytes == oproof.ser()
    parsed, pos = pr.deser(spark.SNARK, proof.bytes)
    assert pos == len(proof.bytes)
    parsed.verify(ocomm, [16, 1, 2], oc.Transcript(b"snark_example"), ogens)


def first_diff(a, b):
    if len(a) != len(b):
        return "lengths %d != %d" % (len(a), len(b))
    return next((i for i in range(len(a)) if a[i] != b[i]), None)


@pytest.mark.parametrize("logn", [16, 20])
def test_snark_bench_configuration_bytes_match_oracle(sb, logn):
    """BASELINE.json configs[1] — exactly what bench.py times (2^20 constraints / variables / non-zeros, 10 inputs, instance seed 0, tape
    seed 0, transcript label b"example") — and the 2^16 sample: computation commitment and proof bytes identical to the oracle's, which runs
    on all host cores.  This puts the row-table MSM (k_msm_digits, k_msm_win, k_msm_chunks, k_msm_horner) of the big row commitments,
    k_ipa_msm_quad<13,5> (4098-generator sets) and the streaming sumcheck kernels under a byte diff inside a whole proof; every k_msm_rows instance
    is checked directly by test_gpu_msm_instances.py.  Also the reference's published structure at 2^20: 47,024 / 64,712 / 133,720 bytes
    (README.md:362,371,374)."""
    n = 1 << logn
    oc.lib.oracle_set_threads(max(1, (os.cpu_count() or 2) // 2))
    oi, ovars, oinputs = r1cs.Instance.produce_synthetic_r1cs(n, n, 10, 0)
    ogens = spark.SNARKGens(n, n, 10, n)
    ocomm, odecomm = spark.SNARK.encode(oi, ogens)
    oproof = spark.SNARK.prove(oi, ocomm, odecomm, ovars.copy(), oinputs, ogens, oc.Transcript(b"example"), r1cs.tape_seed(0))
    want = oproof.ser()
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=0)
    gens = sb.SNARKGens(n, n, 10, n)
    comm = sb.SNARK.encode(inst, gens)
    assert first_diff(comm.commitment_bytes(), ocomm.ser()) is None
    proof = sb.SNARK.prove(inst, comm, vars_, inputs, gens, b"example", sb.tape_seed(0))
    assert first_diff(proof.bytes, want) is None, "first differing byte (or length mismatch): %s" % first_diff(proof.bytes, want)
    # the device-resident entry point (bench.py's `value` leg) gives the same bytes
    assert sb.SNARK.prove(inst, comm, sb.DensePolynomial(vars_.limbs), inputs, gens, b"example", sb.tape_seed(0)).bytes == want
    if logn == 20:
        assert len(pr.ser(oproof.r1cs_sat_proof)) == 47024
        assert len(pr.ser(oproof.r1cs_eval_proof.poly_eval_network_proof.proof_prod_layer)) == 64712
        assert len(pr.ser(oproof.r1cs_eval_proof)) == 133720
    proof.verify(comm, inputs, b"example", gens)    # the library's own verifier
    if logn == 16:
        oproof.verify(ocomm, oinputs, oc.Transcript(b"example"), ogens)


def test_snark_2p22_fits_one_gpu_and_matches_golden(sb):
    """BASELINE.json configs[4]'s size, 2^22, on ONE 80 GB GPU: the generator tables fall back to narrower windows when the wide ones do not fit
    (prover.cpp GenSet::finish); commitment and proof bytes equal the oracle's golden ones (tests/golden/make_snark_golden.py)"""
    import hashlib, json
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    fx = json.load(open(os.path.join(golden, "snark_proof_sha256.json")))
    n = 1 << 22
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=0)
    gens = sb.SNARKGens(n, n, 10, n)
    comm = sb.SNARK.encode(inst, gens)
    assert hashlib.sha256(comm.commitment_bytes()).hexdigest() == fx["22_commitment"]
    proof = sb.SNARK.prove(inst, comm, sb.DensePolynomial(vars_.limbs), inputs, gens, b"example", sb.tape_seed(0))
    want = open(os.path.join(golden, "snark_2p22_proof.bin"), "rb").read()
    assert first_diff(proof.bytes, want) is None, "first differing byte (or length mismatch): %s" % first_diff(proof.bytes, want)


@pytest.mark.parametrize("logn", [14])
def test_snark_large_accepted_by_oracle_verifier(sb, logn):
    """a GPU proof parsed from its bytes is accepted by the oracle's SNARK::verify, and a tampered one is rejected"""
    n = 1 << logn
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=1)
    gens = sb.SNARKGens(n, n, 10, n)
    comm = sb.SNARK.encode(inst, gens)
    proof = sb.SNARK.prove(inst, comm, vars_, inputs, gens, b"snark_example", sb.tape_seed(1))
    parsed, pos = pr.deser(spark.SNARK, proof.bytes)
    assert pos == len(proof.bytes)
    if logn == 20:
        assert len(pr.ser(parsed.r1cs_sat_proof)) == 47024
        assert len(pr.ser(parsed.r1cs_eval_proof.poly_eval_network_proof.proof_prod_layer)) == 64712
        assert len(pr.ser(parsed.r1cs_eval_proof)) == 133720
    ocomm = parse_commitment(comm.commitment_bytes())
    ogens = spark.SNARKGens(n, n, 10, n)
    parsed.verify(ocomm, oc.to_ints(inputs.limbs), oc.Transcript(b"snark_example"), ogens)
    # tampering is rejected
    bad = bytearray(proof.bytes)
    bad[len(bad) // 2] ^= 1
    try:
        tampered, _ = pr.deser(spark.SNARK, bytes(bad))
        with pytest.raises((pr.ProofVerifyError, AssertionError)):
            tampered.verify(ocomm, oc.to_ints(inputs.limbs), oc.Transcript(b"snark_example"), ogens)
    except (AssertionError, ValueError):
        pass


def test_snark_caller_owned_transcript(sb):
    """`transcript: &mut Transcript` semantics (lib.rs:339-347, :423-429): the caller absorbs its own data first, passes the transcript, and keeps
    using it afterwards.  Proof bytes equal the oracle's, and the transcript is left in the state the oracle's is left in (same next challenge)."""
    n, seed = 256, 3
    oi, ovars, oinputs = r1cs.Instance.produce_synthetic_r1cs(n, n, 10, seed)
    ogens = spark.SNARKGens(n, n, 10, n)
    ocomm, odecomm = spark.SNARK.encode(oi, ogens)
    ot = oc.Transcript(b"application")
    ot.append_message(b"context", b"data the caller absorbed before proving")
    want = spark.SNARK.prove(oi, ocomm, odecomm, ovars, oinputs, ogens, ot, r1cs.tape_seed(seed)).ser()
    after = ot.challenge_bytes(b"after-prove", 32)
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=seed)
    gens = sb.SNARKGens(n, n, 10, n)
    comm = sb.SNARK.encode(inst, gens)
    t = sb.Transcript(b"application")
    t.append_message(b"context", b"data the caller absorbed before proving")
    proof = sb.SNARK.prove(inst, comm, vars_, inputs, gens, t, sb.tape_seed(seed))
    assert proof.bytes == want
    assert t.challenge_bytes(b"after-prove", 32) == after
    tv = sb.Transcript(b"application")
    tv.append_message(b"context", b"data the caller absorbed before proving")
    proof.verify(comm, inputs, tv, gens)
    ov = oc.Transcript(b"application")
    ov.append_message(b"context", b"data the caller absorbed before proving")
    parsed, _ = pr.deser(spark.SNARK, proof.bytes)
    parsed.verify(ocomm, oinputs, ov, ogens)
    assert tv.challenge_bytes(b"after-verify", 32) == ov.challenge_bytes(b"after-verify", 32)
    bad = sb.Transcript(b"application")
    bad.append_message(b"context", b"different caller data")
    with pytest.raises(sb.ProofVerifyError):
        proof.verify(comm, inputs, bad, gens)
    # a label is shorthand for a fresh transcript
    assert sb.SNARK.prove(inst, comm, vars_, inputs, gens, sb.Transcript(b"snark_example"), sb.tape_seed(seed)).bytes == \
        sb.SNARK.prove(inst, comm, vars_, inputs, gens, b"snark_example", sb.tape_seed(seed)).bytes


def test_overlap_does_not_change_bytes(sb):
    """The background-stream commitment of the dereferenced values (snark.cpp) only changes WHEN things are computed: with the overlap off the
    commitment runs on the prover's stream, and the proof bytes must equal the overlapped proof's."""
    from test_instance_shapes import plan
    n = 1 << 12
    assert plan(n, n, 10, (n, n, n))["early"]   # a shape that takes the background path when the overlap is on
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=0)
    gens = sb.SNARKGens(n, n, 10, n)
    comm = sb.SNARK.encode(inst, gens)
    ctx = sb.default_context()
    proofs = {}
    try:
        for overlap in (True, False):
            ctx.set_overlap(overlap)
            proofs[overlap] = sb.SNARK.prove(inst, comm, vars_, inputs, gens, b"example", sb.tape_seed(0)).bytes
    finally:
        ctx.set_overlap(True)
    assert proofs[True] == proofs[False]
