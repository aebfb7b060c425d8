"""SNARK::prove (lib.rs:339-420) rebuilt by a caller from the public pieces alone, with no oracle code in the proving path: the matrices of
Instance.export as SparseMatPolynomials, their commitment by SparseMatPolynomial.multi_commit with the gens R1CSCommitmentGens::new builds
(SparseMatPolyCommitmentGens(b"gens_r1cs_eval", log2 num_cons, log2 2 num_vars, nnz, 3), r1cs.rs:33-47), the transcript head (the SNARK's
protocol name, then R1CSCommitment's absorption, r1cs.rs:58-65: num_cons, num_vars, num_inputs as u64s and the SPARK commitment), the R1CSProof
of the NIZK rebuild with Az, Bz, Cz from multiply_vec and the phase-two table from the weighted compute_eval_table_sparse, the three claims and
SparseMatPolyEvalProof.prove.  The bytes must be the library's own SNARK proof, the commitment the library's, and SNARK.verify must accept."""
import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from test_gpu_nizk_from_pieces import L, append_protocol_name, append_scalars, challenge_scalar, first_diff, ints  # noqa: E402

pytestmark = pytest.mark.gpu
Q = oc.Q
GENS_LABEL = b"gens_r1cs_sat"


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    sb.default_context()
    return sb


def matrices(sb, inst):
    """A, B, C of the instance (padded shape, input columns moved past num_vars) as host SparseMatPolynomials"""
    x, y = oc.log_2(inst.num_cons), oc.log_2(2 * inst.num_vars)
    out = []
    for m in range(3):
        row, col, val = inst.export(m)
        out.append(sb.SparseMatPolynomial(x, y, row, col, ints(val)))
    return out, max(len(p.rows) for p in out)


def rebuild_snark(sb, inst, nnz, vars_limbs, inputs, label, seed):
    """(commitment, proof bytes) of SNARK::encode / prove(inst, comm, vars, inputs, gens, Transcript::new(label)) with tape_seed(seed)"""
    num_cons, num_vars, num_inputs = inst.num_cons, inst.num_vars, inst.num_inputs
    mats, _ = matrices(sb, inst)
    spark_gens = sb.SparseMatPolyCommitmentGens(b"gens_r1cs_eval", oc.log_2(num_cons), oc.log_2(2 * num_vars), nnz, 3)
    comm, dense = sb.SparseMatPolynomial.multi_commit(mats, spark_gens)
    products = sb.SparseMatPolynomial.multi_products(mats)

    T, tape = sb.Transcript(label), sb.RandomTape(sb.tape_seed(seed))
    append_protocol_name(T, b"Spartan SNARK proof")
    for name, v in ((b"num_cons", num_cons), (b"num_vars", num_vars), (b"num_inputs", num_inputs)):
        T.append_message(name, int(v).to_bytes(8, "little"))
    comm.append_to_transcript(b"comm", T)
    append_protocol_name(T, b"R1CS proof")
    append_scalars(T, b"input", inputs)

    gens_pc = sb.PolyCommitmentGens(oc.log_2(num_vars), GENS_LABEL)
    n = gens_pc.n
    pts = sb.MultiCommitGens(n + 1, GENS_LABEL).export()
    gens_1 = sb.MultiCommitGens.from_points([pts[n], pts[n + 1]])
    gens_3, gens_4 = sb.MultiCommitGens(3, GENS_LABEL), sb.MultiCommitGens(4, GENS_LABEL)

    vars_p = np.concatenate([vars_limbs, oc.zeros(num_vars - len(vars_limbs))])
    vpoly = sb.DensePolynomial(vars_p)
    comm_vars, blinds_vars = sb.poly_commit(vpoly, gens_pc, tape)
    comm_vars.append_to_transcript(b"poly_commitment", T)
    z = np.concatenate([vars_p, oc.to_arr([1] + list(inputs)), oc.zeros(num_vars - len(inputs) - 1)])
    zpoly = sb.DensePolynomial(z)
    num_rounds_x, num_rounds_y = oc.log_2(num_cons), oc.log_2(len(z))
    tau = np.array([L(challenge_scalar(T, b"challenge_tau")) for _ in range(num_rounds_x)])

    Az, Bz, Cz = products.multiply_vec(num_cons, len(z), zpoly)
    tabs1 = [sb.DensePolynomial.eq_evals(tau), Az, Bz, Cz]
    comp1 = sb.Composition([(L(1), (0, 1, 2)), (L(Q - 1), (0, 3))])
    sc1, rx, fin1, bpost1 = sb.ZKSumcheckInstanceProof.prove(tabs1, comp1, L(0), L(0), num_rounds_x, gens_1, gens_4, T, tape)
    tau_c, Az_c, Bz_c, Cz_c = ints(fin1)
    blind_claim_postsc1 = ints(bpost1)[0]
    Az_b, Bz_b, Cz_b, prod_b = (challenge_scalar(tape, lab) for lab in (b"Az_blind", b"Bz_blind", b"Cz_blind", b"prod_Az_Bz_blind"))
    pok, C_Cz = sb.KnowledgeProof.prove(gens_1, T, tape, L(Cz_c), L(Cz_b))
    prod_proof, C_Az, C_Bz, C_prod = sb.ProductProof.prove(gens_1, T, tape, L(Az_c), L(Az_b), L(Bz_c), L(Bz_b), L(Az_c * Bz_c), L(prod_b))
    for lab, c in ((b"comm_Az_claim", C_Az), (b"comm_Bz_claim", C_Bz), (b"comm_Cz_claim", C_Cz), (b"comm_prod_Az_Bz_claims", C_prod)):
        T.append_message(lab, c)
    claim_post1 = (Az_c * Bz_c - Cz_c) * tau_c % Q
    eq1, _, _ = sb.EqualityProof.prove(gens_1, T, tape, L(claim_post1), L(tau_c * (prod_b - Cz_b)), L(claim_post1), L(blind_claim_postsc1))

    r_A, r_B, r_C = (challenge_scalar(T, lab) for lab in (b"challenge_Az", b"challenge_Bz", b"challenge_Cz"))
    claim2 = (r_A * Az_c + r_B * Bz_c + r_C * Cz_c) % Q
    blind2 = (r_A * Az_b + r_B * Bz_b + r_C * Cz_b) % Q
    evals_rx = sb.DensePolynomial.eq_evals(rx)
    abc = products.compute_eval_table_sparse(evals_rx, num_cons, len(z), weights=np.array([L(r_A), L(r_B), L(r_C)]))
    sc2, ry, fin2, bpost2 = sb.ZKSumcheckInstanceProof.prove([zpoly, abc], sb.Composition([(L(1), (0, 1))]), L(claim2), L(blind2), num_rounds_y,
                                                             gens_1, gens_3, T, tape)
    z_c, abc_c = ints(fin2)
    blind_eval = challenge_scalar(tape, b"blind_eval")
    pe, C_vars_at_ry, _ = sb.PolyEvalProof.prove(vpoly, blinds_vars, ry[1:], None, L(blind_eval), gens_pc, T, tape)
    ry0 = ints(ry)[0]
    claim_post2 = z_c * abc_c % Q
    eq2, _, _ = sb.EqualityProof.prove(gens_1, T, tape, L(claim_post2), L(abc_c * (1 - ry0) * blind_eval), L(claim_post2), L(ints(bpost2)[0]))
    r1cs_proof = (comm_vars.to_bytes() + sc1.data + C_Az + C_Bz + C_Cz + C_prod + pok.data + prod_proof.data + eq1.data + sc2.data + C_vars_at_ry
                  + pe.data + eq2.data)

    evals = sb.SparseMatPolynomial.multi_evaluate(dense, rx, ry)
    for lab, v in zip((b"Ar_claim", b"Br_claim", b"Cr_claim"), ints(evals)):
        T.append_message(lab, oc.scalar_to_bytes(v))
    eval_proof, _ = sb.SparseMatPolyEvalProof.prove(dense, rx, ry, evals, spark_gens, T, tape)
    return comm, r1cs_proof + np.ascontiguousarray(evals, dtype=np.uint64).tobytes() + eval_proof.data


def check(sb, inst, vars_, inputs, label, seed):
    nnz = matrices(sb, inst)[1]
    gens = sb.SNARKGens(inst.num_cons, inst.num_vars, inst.num_inputs, nnz)
    lcomm = sb.SNARK.encode(inst, gens)
    want = sb.SNARK.prove(inst, lcomm, vars_, inputs, gens, label, sb.tape_seed(seed)).bytes
    comm, got = rebuild_snark(sb, inst, nnz, vars_.limbs, ints(inputs.limbs), label, seed)
    dims = b"".join(int(v).to_bytes(8, "little") for v in (inst.num_cons, inst.num_vars, inst.num_inputs))
    assert lcomm.commitment_bytes() == dims + comm.to_bytes()
    assert first_diff(got, want) is None, "first differing byte %s of %d" % (first_diff(got, want), len(want))
    sb.SNARK(got).verify(lcomm, inputs, label, gens)


def test_rebuilt_snark_equals_library_proof_2p10(sb):
    n = 1 << 10
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=3)
    check(sb, inst, vars_, inputs, b"snark-from-pieces", 3)


def test_rebuilt_snark_on_a_padded_shape_with_a_dense_constant_column(sb):
    """3000 constraints over 5000 variables (padded to 4096 and 8192) and 37 inputs; every constraint reads the constant column in A, B and C:
    (a_i z_i + c_i) * 1 = a_i z_i + c_i"""
    num_cons, num_vars, num_inputs = 3000, 5000, 37
    a = oc.to_ints(oc.prg_scalars("snark-pieces-a", num_cons))
    c = oc.to_ints(oc.prg_scalars("snark-pieces-c", num_cons))
    one = oc.scalar_to_bytes(1)
    A, B, Cm = [], [], []
    for i in range(num_cons):
        A += [(i, i, oc.scalar_to_bytes(a[i])), (i, num_vars, oc.scalar_to_bytes(c[i]))]
        B.append((i, num_vars, one))
        Cm += [(i, num_vars, oc.scalar_to_bytes(c[i])), (i, i, oc.scalar_to_bytes(a[i]))]
    inst = sb.Instance.new(num_cons, num_vars, num_inputs, A, B, Cm)
    vars_ = sb.Assignment(oc.prg_scalars("snark-pieces-vars", num_vars))
    inputs = sb.Assignment(oc.prg_scalars("snark-pieces-inputs", num_inputs))
    assert inst.is_sat(vars_, inputs)
    check(sb, inst, vars_, inputs, b"snark-from-pieces-constant-column", 11)
