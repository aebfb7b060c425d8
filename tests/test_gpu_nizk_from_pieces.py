"""NIZK::prove (lib.rs:501-546, r1csproof.rs:144-349) rebuilt by a caller from the public pieces alone: the transcript head, poly_commit with the
tape, challenge_tau, the phase-one ZK sumcheck of eq(tau) * (Az * Bz - Cz) with gens_1 / gens_4, the tape's claim blinds, KnowledgeProof,
ProductProof, the four claim points, EqualityProof, the phase-two ZK sumcheck of z * (r_A A + r_B B + r_C C)(rx, .) with gens_1 / gens_3,
PolyEvalProof with blind_eval, and the second EqualityProof.  The bytes must be the library's own NIZK proof, and NIZK.verify must accept them:
this pins the tape order, the generator views (gens_1 is the split_at view [P_n, P_(n+1)] of the label's stream) and every caller entry at once.
Az, Bz, Cz and the phase-two evaluation table come from the oracle on the host."""
import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import r1cs
from test_gpu_instance_shapes import library_instance  # noqa: E402
from test_instance_shapes import CASES, cached_instance  # noqa: E402

pytestmark = pytest.mark.gpu
Q = oc.Q
GENS_LABEL = b"gens_r1cs_sat"   # NIZKGens::new -> R1CSGens::new(b"gens_r1cs_sat", ..) (lib.rs:475-481)


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    sb.default_context()
    return sb


# ---- the ProofTranscript steps (transcript.rs) a caller runs between the library's calls, on a Transcript / RandomTape state
def L(x):
    return oc.to_arr([x % Q])[0]


def ints(a):
    return oc.to_ints(np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4))


def append_protocol_name(T, name):
    T.append_message(b"protocol-name", name)


def append_scalars(T, label, xs):
    T.append_message(label, b"begin_append_vector")
    for x in xs:
        T.append_message(label, oc.scalar_to_bytes(x))
    T.append_message(label, b"end_append_vector")


def challenge_scalar(T, label):
    """also RandomTape::random_scalar (random.rs:19-21) on a tape"""
    return oc.scalar_from_bytes_wide(T.challenge_bytes(label, 64))


def vec_bytes(r):
    """bincode of a Vec<Scalar> given as Montgomery limbs"""
    r = np.ascontiguousarray(r, dtype=np.uint64).reshape(-1, 4)
    return len(r).to_bytes(8, "little") + r.tobytes()


def rebuild_nizk(sb, shape, digest, vars_arr, inputs, label, seed):
    """the bytes of NIZK::prove(inst, vars, inputs, gens, Transcript::new(label)) with RandomTape seed tape_seed(seed), from the public pieces"""
    num_cons, num_vars = shape.num_cons, shape.num_vars
    vars_p = r1cs.pad_vars(vars_arr, num_vars)
    T, tape = sb.Transcript(label), sb.RandomTape(sb.tape_seed(seed))
    append_protocol_name(T, b"Spartan NIZK proof")
    T.append_message(b"R1CSShapeDigest", digest)
    append_protocol_name(T, b"R1CS proof")
    append_scalars(T, b"input", inputs)

    # the generators: R1CSGens::new(label, num_cons, num_vars) (r1csproof.rs:61-74)
    gens_pc = sb.PolyCommitmentGens(oc.log_2(num_vars), GENS_LABEL)
    n = gens_pc.n
    pts = sb.MultiCommitGens(n + 1, GENS_LABEL).export()   # G[0..n+1) then h
    gens_1 = sb.MultiCommitGens.from_points([pts[n], pts[n + 1]])   # gens_pc.gens.gens_1
    gens_3, gens_4 = sb.MultiCommitGens(3, GENS_LABEL), sb.MultiCommitGens(4, GENS_LABEL)

    vpoly = sb.DensePolynomial(vars_p)
    comm_vars, blinds_vars = sb.poly_commit(vpoly, gens_pc, tape)
    comm_vars.append_to_transcript(b"poly_commitment", T)
    z = np.concatenate([vars_p, oc.to_arr([1] + list(inputs)), oc.zeros(num_vars - len(inputs) - 1)])
    num_rounds_x, num_rounds_y = oc.log_2(num_cons), oc.log_2(len(z))
    tau = [challenge_scalar(T, b"challenge_tau") for _ in range(num_rounds_x)]

    # phase one: eq(tau) * (Az * Bz - Cz) = A*B*C - A*D over [eq(tau), Az, Bz, Cz], claim 0 with blind 0
    Az, Bz, Cz = shape.multiply_vec(num_cons, len(z), z)
    tabs1 = [sb.DensePolynomial(t) for t in (oc.eq_evals(tau), Az, Bz, Cz)]
    comp1 = sb.Composition([(L(1), (0, 1, 2)), (L(Q - 1), (0, 3))])
    sc1, rx, fin1, bpost1 = sb.ZKSumcheckInstanceProof.prove(tabs1, comp1, L(0), L(0), num_rounds_x, gens_1, gens_4, T, tape)
    tau_c, Az_c, Bz_c, Cz_c = ints(fin1)
    blind_claim_postsc1 = ints(bpost1)[0]
    Az_b, Bz_b, Cz_b, prod_b = (challenge_scalar(tape, l) for l in (b"Az_blind", b"Bz_blind", b"Cz_blind", b"prod_Az_Bz_blind"))
    pok, C_Cz = sb.KnowledgeProof.prove(gens_1, T, tape, L(Cz_c), L(Cz_b))
    prod_proof, C_Az, C_Bz, C_prod = sb.ProductProof.prove(gens_1, T, tape, L(Az_c), L(Az_b), L(Bz_c), L(Bz_b), L(Az_c * Bz_c), L(prod_b))
    for lab, c in ((b"comm_Az_claim", C_Az), (b"comm_Bz_claim", C_Bz), (b"comm_Cz_claim", C_Cz), (b"comm_prod_Az_Bz_claims", C_prod)):
        T.append_message(lab, c)
    claim_post1 = (Az_c * Bz_c - Cz_c) * tau_c % Q
    eq1, _, _ = sb.EqualityProof.prove(gens_1, T, tape, L(claim_post1), L(tau_c * (prod_b - Cz_b)), L(claim_post1), L(blind_claim_postsc1))

    # phase two: z * (r_A A + r_B B + r_C C)(rx, .)
    r_A, r_B, r_C = (challenge_scalar(T, l) for l in (b"challenge_Az", b"challenge_Bz", b"challenge_Cz"))
    claim2 = (r_A * Az_c + r_B * Bz_c + r_C * Cz_c) % Q
    blind2 = (r_A * Az_b + r_B * Bz_b + r_C * Cz_b) % Q
    eA, eB, eC = shape.compute_eval_table_sparse(num_cons, len(z), oc.eq_evals(ints(rx)))
    tabs2 = [sb.DensePolynomial(z), sb.DensePolynomial(oc.lincomb3(eA, eB, eC, r_A, r_B, r_C))]
    sc2, ry, fin2, bpost2 = sb.ZKSumcheckInstanceProof.prove(tabs2, sb.Composition([(L(1), (0, 1))]), L(claim2), L(blind2), num_rounds_y, gens_1,
                                                             gens_3, T, tape)
    z_c, abc_c = ints(fin2)
    blind_eval = challenge_scalar(tape, b"blind_eval")
    pe, C_vars_at_ry, _ = sb.PolyEvalProof.prove(vpoly, blinds_vars, ry[1:], None, L(blind_eval), gens_pc, T, tape)
    ry0 = ints(ry)[0]
    claim_post2 = z_c * abc_c % Q
    eq2, _, _ = sb.EqualityProof.prove(gens_1, T, tape, L(claim_post2), L(abc_c * (1 - ry0) * blind_eval), L(claim_post2), L(ints(bpost2)[0]))

    r1cs_proof = (comm_vars.to_bytes() + sc1.data + C_Az + C_Bz + C_Cz + C_prod + pok.data + prod_proof.data + eq1.data + sc2.data + C_vars_at_ry
                  + pe.data + eq2.data)
    return r1cs_proof + vec_bytes(rx) + vec_bytes(ry)


def first_diff(a, b):
    if len(a) != len(b):
        return "lengths %d != %d" % (len(a), len(b))
    return next((i for i in range(len(a)) if a[i] != b[i]), None)


@pytest.mark.parametrize("seed", [0, 5])
def test_rebuilt_nizk_equals_library_proof_2p10(sb, seed):
    n, label = 1 << 10, b"nizk-from-pieces"
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=seed)
    oi, ovars, oinputs = r1cs.Instance.produce_synthetic_r1cs(n, n, 10, seed)
    gens = sb.NIZKGens(n, n, 10)
    want = sb.NIZK.prove(inst, vars_, inputs, gens, label, sb.tape_seed(seed)).bytes
    got = rebuild_nizk(sb, oi.inst, inst.digest, ovars, [int(x) for x in oinputs], label, seed)
    assert first_diff(got, want) is None, "first differing byte %s of %d" % (first_diff(got, want), len(want))
    sb.NIZK(got).verify(inst, inputs, label, gens)


def test_rebuilt_nizk_equals_library_proof_on_a_padded_shape(sb):
    """the padding case of test_gpu_instance_shapes.py: 3000 constraints and 5000 variables padded to 4096 and 8192, 37 inputs"""
    spec, _ = CASES["padding"]
    si = cached_instance(spec)
    oi = si.oracle
    inst, vars_, inputs = library_instance(sb, si)
    inst.set_digest(oi.digest)
    label, seed = b"nizk-from-pieces-padding", 7
    gens = sb.NIZKGens(spec.num_cons, spec.num_vars, spec.num_inputs)
    want = sb.NIZK.prove(inst, vars_, inputs, gens, label, sb.tape_seed(seed)).bytes
    got = rebuild_nizk(sb, oi.inst, oi.digest, si.vars, list(si.inputs), label, seed)
    assert first_diff(got, want) is None, "first differing byte %s of %d" % (first_diff(got, want), len(want))
    sb.NIZK(got).verify(inst, inputs, label, gens)
