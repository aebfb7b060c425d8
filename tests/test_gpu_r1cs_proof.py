"""R1CSProof::prove / verify (r1csproof.rs:144-489) as a caller entry: on the caller's transcript and tape, over an Instance (its k_spmv products,
as NIZK.prove runs them) or a SparseMatProducts of A, B, C (the tiled products).  The proof, rx, ry and the transcript and tape states after the
call must be the oracle's; the proof must be the one NIZK.prove and SNARK.prove embed; the verifier must accept with the claims Instance.evaluate
and SparseMatPolynomial.multi_evaluate give, and reject what the oracle verifier rejects."""
import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import r1cs
from test_gpu_instance_shapes import library_instance  # noqa: E402
from test_instance_shapes import CASES, cached_instance  # noqa: E402

pytestmark = pytest.mark.gpu
Q = oc.Q
LABEL = b"r1cs-proof-test"
GENS_LABEL = b"gens_r1cs_sat"


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    sb.default_context()
    return sb


def ints(a):
    return oc.to_ints(np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4))


def L(x):
    return oc.to_arr([x % Q])[0]


def spmat_of(sb, inst):
    """A, B, C of a library Instance (its padded column space) as a SparseMatProducts"""
    x, y = inst.num_cons.bit_length() - 1, (2 * inst.num_vars).bit_length() - 1
    mats = []
    for m in range(3):
        row, col, val = inst.export(m)
        mats.append(sb.SparseMatPolynomial(x, y, row, col, ints(val)))
    return sb.SparseMatPolynomial.multi_products(mats)


def spmat_polys(sb, inst):
    x, y = inst.num_cons.bit_length() - 1, (2 * inst.num_vars).bit_length() - 1
    out = []
    for m in range(3):
        row, col, val = inst.export(m)
        out.append(sb.SparseMatPolynomial(x, y, row, col, ints(val)))
    return out


def ctx_device(sb):
    return sb.default_context().device


class States:
    """the oracle's and the library's transcript, both after the caller's own message, and tape of one seed"""

    def __init__(self, sb, tag, seed):
        self.ot, self.st = oc.Transcript(LABEL), sb.Transcript(LABEL)
        self.ot.append_message(b"app", tag)
        self.st.append_message(b"app", tag)
        self.otape = oc.RandomTape(b"proof", ints(sb.tape_seed(seed))[0])
        self.stape = sb.RandomTape(sb.tape_seed(seed))

    def same(self):
        return (self.ot.challenge_bytes(b"after", 64) == self.st.challenge_bytes(b"after", 64)
                and self.otape.tape.challenge_bytes(b"after", 64) == self.stape.challenge_bytes(b"after", 64))


def vars_poly(sb, vars_arr, n):
    return sb.DensePolynomial(r1cs.pad_vars(np.ascontiguousarray(vars_arr, dtype=np.uint64).reshape(-1, 4), n))


# ---------------------------------------------------------------------------------------------- parity with the oracle
def synthetic(sb, n, ni, seed):
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, ni, seed=seed)
    oi, ovars, oinputs = r1cs.Instance.produce_synthetic_r1cs(n, n, ni, seed)
    return inst, vars_.limbs, inputs.limbs, oi.inst, ovars, [int(v) for v in oinputs]


def shaped(sb, name):
    si = cached_instance(CASES[name][0])
    inst, vars_, inputs = library_instance(sb, si)
    return inst, vars_.limbs, inputs.limbs, si.oracle.inst, si.vars, list(si.inputs)


def check_against_oracle(sb, inst, vars_l, inputs_l, oshape, ovars, oinputs, label, seed):
    """the oracle's R1CSProof::prove and the library's, from both sources, on one transcript head and tape seed: same proof, rx, ry, and the
    same transcript and tape states after the call"""
    nc, nv = inst.num_cons, inst.num_vars
    assert (oshape.num_cons, oshape.num_vars) == (nc, nv)
    gens, ogens = sb.R1CSGens(label, nc, nv), pr.R1CSGens(label, nc, nv)
    O = States(sb, label, seed)
    oproof, orx, ory = pr.R1CSProof.prove(oshape, r1cs.pad_vars(ovars, nv), oinputs, ogens, O.ot, O.otape)
    want = pr.ser(oproof)
    v = vars_poly(sb, vars_l, nv)
    before = v.to_numpy().copy()
    raw = []
    for mats in (inst, spmat_of(sb, inst)):
        S = States(sb, label, seed)
        proof, rx, ry = sb.R1CSProof.prove(mats, v, inputs_l, gens, S.st, S.stape)
        assert proof.data == want, type(mats).__name__
        assert ints(rx) == list(orx) and ints(ry) == list(ory), type(mats).__name__
        assert np.array_equal(v.to_numpy(), before), "vars must be read only"
        raw.append((S.st.state.raw, S.stape.state.raw))
        last = S
    assert raw[0] == raw[1]
    last.ot, last.otape = O.ot, O.otape
    assert last.same()


@pytest.mark.parametrize("label", [GENS_LABEL, b"caller-r1cs-label"])
def test_synthetic_2p10_equals_oracle(sb, label):
    inst, vl, il, oshape, ovars, oin = synthetic(sb, 1 << 10, 10, 3)
    check_against_oracle(sb, inst, vl, il, oshape, ovars, oin, label, 4)


@pytest.mark.parametrize("name", ["padding", "many_inputs", "dense_rows"])
def test_instance_shapes_equal_oracle(sb, name):
    inst, vl, il, oshape, ovars, oin = shaped(sb, name)
    check_against_oracle(sb, inst, vl, il, oshape, ovars, oin, b"shape-" + name.encode(), 9)


# ---------------------------------------------------------------------------------------------- parity with NIZK.prove
def nizk_head(sb, inst, label):
    T = sb.Transcript(label)
    T.append_message(b"protocol-name", b"Spartan NIZK proof")
    T.append_message(b"R1CSShapeDigest", inst.digest)
    return T


def vec_bytes(r):
    r = np.ascontiguousarray(r, dtype=np.uint64).reshape(-1, 4)
    return len(r).to_bytes(8, "little") + r.tobytes()


@pytest.mark.parametrize("name", list(CASES))
def test_standalone_equals_nizk_inner_proof(sb, name):
    """every CASES shape, both sources: the proof NIZK.prove embeds, with its rx / ry (the Instance products are the ones NIZK.prove runs, and
    tests/test_gpu_instance_shapes.py pins NIZK.prove to the oracle on these shapes)"""
    spec = CASES[name][0]
    inst, vl, il, _, _, _ = shaped(sb, name)
    label, seed = b"nizk-" + name.encode(), 11
    ngens = sb.NIZKGens(spec.num_cons, spec.num_vars, spec.num_inputs)
    nizk = sb.NIZK.prove(inst, sb.Assignment(vl), sb.Assignment(il), ngens, label, sb.tape_seed(seed)).bytes
    gens = sb.R1CSGens.view(ngens, inst.num_cons, inst.num_vars)
    v = vars_poly(sb, vl, inst.num_vars)
    for mats in (inst, spmat_of(sb, inst)):
        T, tape = nizk_head(sb, inst, label), sb.RandomTape(sb.tape_seed(seed))
        proof, rx, ry = sb.R1CSProof.prove(mats, v, il, gens, T, tape)
        assert nizk == proof.data + vec_bytes(rx) + vec_bytes(ry), type(mats).__name__


# ---------------------------------------------------------------------------------------------- composition into SNARK.prove
def test_spmat_proof_and_spark_compose_to_snark(sb):
    n, ni, label, seed = 1 << 10, 10, b"snark-compose", 6
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, ni, seed=seed)
    sgens = sb.SNARKGens(n, n, ni, n)
    comm = sb.SNARK.encode(inst, sgens)
    want = sb.SNARK.prove(inst, comm, vars_, inputs, sgens, label, sb.tape_seed(seed)).bytes

    polys = spmat_polys(sb, inst)
    x, y = polys[0].num_vars_x, polys[0].num_vars_y
    spark_gens = sb.SparseMatPolyCommitmentGens(b"gens_r1cs_eval", x, y, n, 3)
    spark_comm, dense = sb.SparseMatPolynomial.multi_commit(polys, spark_gens)
    assert comm.commitment_bytes()[24:] == spark_comm.to_bytes()

    T, tape = sb.Transcript(label), sb.RandomTape(sb.tape_seed(seed))
    T.append_message(b"protocol-name", b"Spartan SNARK proof")
    for lab, v in ((b"num_cons", n), (b"num_vars", n), (b"num_inputs", ni)):
        T.append_message(lab, v.to_bytes(8, "little"))
    spark_comm.append_to_transcript(b"comm", T)
    proof, rx, ry = sb.R1CSProof.prove(sb.SparseMatPolynomial.multi_products(polys), vars_, inputs, sb.R1CSGens.view(sgens, n, n), T, tape)
    evals = sb.SparseMatPolynomial.multi_evaluate(dense, rx, ry)
    assert np.array_equal(evals, inst.evaluate(rx, ry))
    for lab, e in zip((b"Ar_claim", b"Br_claim", b"Cr_claim"), ints(evals)):
        T.append_message(lab, oc.scalar_to_bytes(e))
    ev_proof, _ = sb.SparseMatPolyEvalProof.prove(dense, rx, ry, evals, spark_gens, T, tape)
    got = proof.data + evals.tobytes() + ev_proof.data
    assert got == want
    sb.SNARK(got).verify(comm, inputs, label, sgens)


# ---------------------------------------------------------------------------------------------- verify
def verify_both(sb, proof, nc, nv, inputs, evals, label, seed_tag, ogens, gens):
    """(library verdict, oracle verdict, library (rx, ry), transcripts agree after)"""
    ot, st = oc.Transcript(LABEL), sb.Transcript(LABEL)
    ot.append_message(b"app", seed_tag)
    st.append_message(b"app", seed_tag)
    try:
        rx, ry = sb.R1CSProof(proof).verify(nv, nc, inputs, evals, st, gens)
        lib_ok = True
    except sb.ProofVerifyError:
        lib_ok, rx, ry = False, None, None
    try:
        op = pr.deser(pr.R1CSProof, proof)[0]
        op.verify(nv, nc, ints(inputs), tuple(ints(evals)), ot, ogens)
        o_ok = True
    except (pr.ProofVerifyError, AssertionError, ValueError, TypeError):
        o_ok = False
    return lib_ok, o_ok, (rx, ry), ot, st


def test_verify_accepts_and_rejects_as_the_oracle(sb):
    n, ni, label, seed = 1 << 10, 8, b"r1cs-verify", 2
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, ni, seed=seed)
    gens, ogens = sb.R1CSGens(label, n, n), pr.R1CSGens(label, n, n)
    S = States(sb, label, seed)
    proof, rx, ry = sb.R1CSProof.prove(spmat_of(sb, inst), vars_, inputs, gens, S.st, S.stape)
    ev_inst = inst.evaluate(rx, ry)
    polys = spmat_polys(sb, inst)
    spark_gens = sb.SparseMatPolyCommitmentGens(b"r1cs-verify-evals", polys[0].num_vars_x, polys[0].num_vars_y, n, 3)
    ev_spark = sb.SparseMatPolynomial.multi_evaluate(polys, rx, ry, spark_gens)
    assert np.array_equal(ev_inst, ev_spark)
    assert ints(ev_inst) == list(r1cs.Instance.produce_synthetic_r1cs(n, n, ni, seed)[0].inst.evaluate(ints(rx), ints(ry)))

    lib_ok, o_ok, (vrx, vry), ot, st = verify_both(sb, proof.data, n, n, inputs.limbs, ev_inst, label, label, ogens, gens)
    assert lib_ok and o_ok
    assert np.array_equal(vrx, rx) and np.array_equal(vry, ry)
    assert st.state.raw == S.st.state.raw, "the verifier leaves the prover's transcript state"
    assert ot.challenge_bytes(b"after", 64) == st.challenge_bytes(b"after", 64)

    for k in range(3):
        bad = ev_inst.copy()
        bad[k] = L(ints(ev_inst)[k] + 1)
        lib_ok, o_ok, _, ot, st = verify_both(sb, proof.data, n, n, inputs.limbs, bad, label, label, ogens, gens)
        assert not lib_ok and not o_ok, k
    bad_in = inputs.limbs.copy()
    bad_in[0] = L(ints(bad_in)[0] + 1)
    lib_ok, o_ok, _, _, _ = verify_both(sb, proof.data, n, n, bad_in, ev_inst, label, label, ogens, gens)
    assert not lib_ok and not o_ok
    lib_ok, o_ok, _, _, _ = verify_both(sb, proof.data, n, n, inputs.limbs, ev_inst, label, b"another head", ogens, gens)
    assert not lib_ok and not o_ok


# ---------------------------------------------------------------------------------------------- a heavy column at scale
def heavy_column_instance(sb, logn, seed):
    """A z = z_0 on every row (one column holds all of A), B = I, C = z_0 I: satisfiable for any vars"""
    torch = pytest.importorskip("torch")
    n = 1 << logn
    dev = torch.device("cuda", ctx_device(sb))
    vars_ = oc.prg_scalars("heavy-col", n, seed)
    i = torch.arange(n, dtype=torch.int64, device=dev)
    one = torch.zeros((n, 32), dtype=torch.uint8, device=dev)
    one[:, 0] = 1
    v0 = torch.tensor(list(oc.scalar_to_bytes(ints(vars_[:1])[0])), dtype=torch.uint8, device=dev).expand(n, 32).contiguous()
    A = (i, torch.zeros_like(i), one)
    B = (i, i, one)
    Cm = (i, i.clone(), v0)
    inst = sb.Instance.from_tensors(n, n, 0, A, B, Cm)
    return inst, vars_


def test_heavy_column_2p18(sb):
    inst, vars_ = heavy_column_instance(sb, 18, 1)
    n = 1 << 18
    assert inst.is_sat(sb.Assignment(vars_), sb.Assignment(oc.zeros(0)))
    gens = sb.R1CSGens(b"heavy-column", n, n)
    v = sb.DensePolynomial(vars_)
    out = []
    for mats in (spmat_of(sb, inst), inst):
        T, tape = sb.Transcript(LABEL), sb.RandomTape(sb.tape_seed(5))
        proof, rx, ry = sb.R1CSProof.prove(mats, v, oc.zeros(0), gens, T, tape)
        out.append((proof.data, rx.tobytes(), ry.tobytes(), T.state.raw, tape.state.raw))
    assert out[0] == out[1]
    proof, rx, ry = sb.R1CSProof(out[0][0]), np.frombuffer(out[0][1], dtype=np.uint64).reshape(-1, 4), np.frombuffer(out[0][2], dtype=np.uint64).reshape(-1, 4)
    T = sb.Transcript(LABEL)
    vrx, vry = proof.verify(n, n, oc.zeros(0), inst.evaluate(rx, ry), T, gens)
    assert np.array_equal(vrx, rx) and np.array_equal(vry, ry)


# ---------------------------------------------------------------------------------------------- refusals and memory
def test_refusals_touch_nothing(sb):
    import ctypes as C
    n, ni = 1 << 8, 4
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, ni, seed=1)
    gens = sb.R1CSGens(b"refusals", n, n)
    small = sb.R1CSGens(b"refusals", n, n // 4)
    spmat = spmat_of(sb, inst)
    other = sb.Instance.produce_synthetic_r1cs(2 * n, 2 * n, ni, seed=1)[0]
    two = sb.SparseMatPolynomial.multi_products(spmat_polys(sb, inst)[:2])
    v = sb.DensePolynomial(vars_.limbs)
    short = sb.DensePolynomial(vars_.limbs[: n // 2])
    ctx2 = sb.Context(ctx_device(sb))
    gens2 = sb.R1CSGens(b"refusals", n, n, ctx=ctx2)
    T, tape = sb.Transcript(LABEL), sb.RandomTape(sb.tape_seed(0))
    t0, p0 = T.state.raw, tape.state.raw
    too_many = oc.to_arr(list(range(1, n + 1)))
    ctx = gens.ctx
    launches = sb.kernel_launches()

    def refused(mats_inst, mats_spmat, nc, nv, vv, inp, g, code=3):
        out, ln = C.POINTER(C.c_ubyte)(), C.c_size_t()
        rx, ry = np.zeros((32, 4), dtype=np.uint64), np.zeros((32, 4), dtype=np.uint64)
        inp = np.ascontiguousarray(inp, dtype=np.uint64).reshape(-1, 4)
        rc = sb.lib.sp_r1cs_prove_t(ctx.h, mats_inst, mats_spmat, C.c_size_t(nc), C.c_size_t(nv), vv.h, inp.ctypes.data_as(C.c_void_p), C.c_size_t(len(inp)),
                                    g.h, T.state, tape.state, C.byref(out), C.byref(ln), rx.ctypes.data_as(C.c_void_p), ry.ctypes.data_as(C.c_void_p))
        assert rc == code, (rc, sb.lib.sp_last_error(ctx.h))
        assert T.state.raw == t0 and tape.state.raw == p0

    refused(inst.h, None, n - 1, n, v, inputs.limbs, gens)          # num_cons not a power of two
    refused(inst.h, None, n, n + 1, v, inputs.limbs, gens)          # num_vars not a power of two
    refused(inst.h, None, n, n, v, too_many, gens)                  # |inputs| + 1 > num_vars
    refused(inst.h, None, n, n, short, inputs.limbs, gens)          # vars of another length
    refused(None, two.h, n, n, v, inputs.limbs, gens)               # two matrices
    refused(None, spmat.h, 2 * n, n, v, inputs.limbs, gens)         # spmat of another shape
    refused(other.h, None, n, n, v, inputs.limbs, gens)             # instance of other dimensions
    refused(inst.h, spmat.h, n, n, v, inputs.limbs, gens)           # both sources
    refused(None, None, n, n, v, inputs.limbs, gens)                # neither
    refused(inst.h, None, n, n, v, inputs.limbs, small)             # gens for another num_vars
    refused(inst.h, None, n, n, v, np.full((1, 4), 2 ** 64 - 1, dtype=np.uint64), gens, code=5)   # unreduced input
    refused(inst.h, None, n, n, v, inputs.limbs, gens2)             # gens of another context
    assert sb.kernel_launches() == launches, "a refused call launches nothing"
    with pytest.raises(sb.SpartanB200Error):
        sb.R1CSGens(b"refusals", n, 3)
    with pytest.raises(sb.SpartanB200Error):
        sb.R1CSGens.view(sb.NIZKGens(n, n // 8, 0), n, n)           # a set too short for num_vars
    assert np.array_equal(v.to_numpy(), vars_.limbs)


def test_device_memory_returns_to_baseline(sb):
    n, ni = 1 << 10, 4
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, ni, seed=8)
    gens = sb.R1CSGens(b"memory", n, n)
    spmat = spmat_of(sb, inst)
    v = sb.DensePolynomial(vars_.limbs)
    sb.R1CSProof.prove(spmat, v, inputs, gens, sb.Transcript(LABEL), sb.RandomTape(sb.tape_seed(1)))   # warm every scratch pool
    base = sb.device_bytes_live()
    for mats in (spmat, inst):
        proof, rx, ry = sb.R1CSProof.prove(mats, v, inputs, gens, sb.Transcript(LABEL), sb.RandomTape(sb.tape_seed(1)))
        assert sb.device_bytes_live() == base
        proof.verify(n, n, inputs, inst.evaluate(rx, ry), sb.Transcript(LABEL), gens)
        assert sb.device_bytes_live() == base
