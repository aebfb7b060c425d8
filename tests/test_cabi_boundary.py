"""The C ABI's one error boundary: a transcript or tape state whose position bytes are out of range is refused with SP_ERR_INVALID_ARG by every
entry that reads one, the caller's buffer left as it was; host-only entries write their own message where sp_last_error(NULL) reads it; and the
Python layer maps a host-only call's status to the same exceptions as a context call's.  The first part needs no GPU."""
import ctypes as C

import numpy as np
import pytest

from oracle.spartan_ref import core as oc

LABEL = b"cabi-boundary"
SP_ERR_INVALID_ARG = 3
SP_ERR_INVALID_SCALAR = 5


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    return sb


def bad_state(sb):
    """a valid transcript state with its position byte (200) out of range"""
    t = sb.Transcript(LABEL)
    t.state[200] = b"\xff"
    return t


def limbs(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def last_host_error(sb):
    return sb.lib.sp_last_error(None).decode()


# ---------------------------------------------------------------------------------------------------- host-only entries (no GPU)
def test_host_verifiers_refuse_a_bad_state(sb):
    t = bad_state(sb)
    before = t.state.raw
    proof = b"\x00" * 8
    claim, e, r = limbs(oc.to_arr([1])[0]), np.zeros(4, dtype=np.uint64), np.zeros((2, 4), dtype=np.uint64)
    rc = sb.lib.sp_sumcheck_verify_t(None, C.c_char_p(proof), C.c_size_t(len(proof)), ptr(claim), C.c_size_t(2), C.c_size_t(3), t.state, ptr(e), ptr(r))
    assert rc == SP_ERR_INVALID_ARG
    assert "transcript state" in last_host_error(sb)
    assert t.state.raw == before
    products, rand, claims = limbs(oc.to_arr([5])), np.zeros((1, 4), dtype=np.uint64), np.zeros((1, 4), dtype=np.uint64)
    rc = sb.lib.sp_prod_verify_t(None, C.c_char_p(proof), C.c_size_t(len(proof)), ptr(products), C.c_int(1), C.c_size_t(1), t.state, ptr(rand), ptr(claims))
    assert rc == SP_ERR_INVALID_ARG
    assert "transcript state" in last_host_error(sb)
    assert t.state.raw == before


def test_transcript_entries_refuse_a_bad_state_with_their_own_message(sb):
    r, out = limbs(oc.to_arr([3])), np.zeros((2, 4), dtype=np.uint64)
    assert sb.lib.sp_prod_leaf_eval(None, C.c_int(2), None, C.c_int(2), ptr(r), C.c_size_t(1), ptr(out)) == SP_ERR_INVALID_ARG
    assert "prod_leaf_eval: NULL argument" in last_host_error(sb)
    t = bad_state(sb)
    before = t.state.raw
    assert sb.lib.sp_transcript_append_message(t.state, C.c_char_p(b"l"), C.c_size_t(1), C.c_char_p(b"m"), C.c_size_t(1)) == SP_ERR_INVALID_ARG
    assert "transcript state" in last_host_error(sb) and "prod_leaf_eval" not in last_host_error(sb)
    assert t.state.raw == before
    assert sb.lib.sp_prod_leaf_eval(None, C.c_int(2), None, C.c_int(2), ptr(r), C.c_size_t(1), ptr(out)) == SP_ERR_INVALID_ARG
    buf = C.create_string_buffer(32)
    assert sb.lib.sp_transcript_challenge_bytes(t.state, C.c_char_p(b"l"), C.c_size_t(1), buf, C.c_size_t(32)) == SP_ERR_INVALID_ARG
    assert "transcript state" in last_host_error(sb) and "prod_leaf_eval" not in last_host_error(sb)
    assert t.state.raw == before


def test_python_host_calls_raise_as_context_calls_do(sb):
    unreduced = np.frombuffer(oc.Q.to_bytes(32, "little"), dtype=np.uint64)
    with pytest.raises(sb.R1CSError, match="InvalidScalar: .*not reduced"):
        sb.sumcheck_verify(b"", unreduced, 0, 3, sb.Transcript(LABEL))
    t = bad_state(sb)
    with pytest.raises(sb.SpartanB200Error, match="error %d: .*transcript state" % SP_ERR_INVALID_ARG):
        t.append_message(b"label", b"message")
    with pytest.raises(sb.SpartanB200Error, match="error %d: .*transcript state" % SP_ERR_INVALID_ARG):
        t.challenge_bytes(b"label", 32)


# ---------------------------------------------------------------------------------------------------- entries with a context (GPU)
@pytest.mark.gpu
def test_context_entries_refuse_a_bad_state(sb):
    ctx = sb.default_context()
    n = 16
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 2, seed=5)
    out, ln = C.POINTER(C.c_ubyte)(), C.c_size_t()
    seed = limbs(sb.tape_seed(5))

    def refused(rc, *states):
        assert rc == SP_ERR_INVALID_ARG, rc
        assert "transcript state" in sb.lib.sp_last_error(ctx.h).decode()
        for s, raw in states:
            assert s.state.raw == raw

    t = bad_state(sb)
    st = (t, t.state.raw)
    nizk_gens = sb.NIZKGens(n, n, 2)
    proof = sb.NIZK.prove(inst, vars_, inputs, nizk_gens, LABEL, sb.tape_seed(5)).bytes
    refused(sb.lib.sp_nizk_verify_t(ctx.h, inst.h, ptr(inputs.limbs), C.c_size_t(len(inputs)), nizk_gens.h, t.state, C.c_char_p(proof),
                                    C.c_size_t(len(proof))), st)
    snark_gens = sb.SNARKGens(n, n, 2, n)
    comm = sb.SNARK.encode(inst, snark_gens)
    refused(sb.lib.sp_snark_prove_t(ctx.h, inst.h, comm.h, ptr(vars_.limbs), C.c_size_t(len(vars_)), ptr(inputs.limbs), C.c_size_t(len(inputs)),
                                    snark_gens.h, t.state, ptr(seed), C.byref(out), C.byref(ln)), st)

    m = 4
    tabs = [oc.prg_scalars("cabi-boundary-%d" % j, 1 << m) for j in range(3)]
    polys = [sb.DensePolynomial(x) for x in tabs]
    terms = sb.Composition([(oc.to_arr([1])[0], (0, 1, 2))])._c_terms()
    r, finals, e = np.zeros((m, 4), dtype=np.uint64), np.zeros((3, 4), dtype=np.uint64), np.zeros(4, dtype=np.uint64)
    claim = limbs(oc.to_arr([0])[0])
    refused(sb.lib.sp_sumcheck_prove_t(ctx.h, sb.api._handles(polys), C.c_int(3), terms, C.c_int(1), ptr(claim), C.c_size_t(m), t.state, C.byref(out),
                                       C.byref(ln), ptr(r), ptr(finals), ptr(e)), st)
    for p, x in zip(polys, tabs):   # not bound
        assert p.len() == 1 << m and np.array_equal(p.to_numpy(), x)

    gens = sb.PolyCommitmentGens(m, LABEL)
    point = limbs(oc.prg_scalars("cabi-boundary-r", m))
    c_zr, zr = C.create_string_buffer(32), np.zeros(4, dtype=np.uint64)
    good, tape = sb.Transcript(LABEL), sb.RandomTape(sb.tape_seed(5))
    bad_tape = bad_state(sb)
    states = [st] + [(s, s.state.raw) for s in (good, tape, bad_tape)]
    for strobe, tp in [(t, tape), (good, bad_tape)]:
        refused(sb.lib.sp_pc_eval_prove_t(ctx.h, gens.h, polys[0].h, None, ptr(point), C.c_size_t(m), None, None, strobe.state, tp.state, C.byref(out),
                                          C.byref(ln), c_zr, ptr(zr)), *states)

    circuits = sb.ProductCircuits(polys)
    rand, evals = np.zeros((m, 4), dtype=np.uint64), np.zeros((3, 4), dtype=np.uint64)
    refused(sb.lib.sp_prod_prove_t(ctx.h, circuits.h, t.state, C.byref(out), C.byref(ln), ptr(rand), ptr(evals)), st)
    sb.ProductCircuitEvalProofBatched.prove(circuits, sb.Transcript(LABEL))   # the refused call did not consume the circuits


@pytest.mark.gpu
def test_a_null_tape_is_refused_after_the_other_arguments(sb):
    """sp_pc_eval_prove_t and sp_pc_eval_prove_joint_t check every other argument before they look at the tape: a NULL tape next to an
    unreduced scalar reports the scalar, and alone it reports the tape, both leaving the transcript as it was"""
    ctx = sb.default_context()
    m, k = 4, 2
    polys = [sb.DensePolynomial(oc.prg_scalars("cabi-null-tape-%d" % j, 1 << m)) for j in range(k)]
    good_r = limbs(oc.prg_scalars("cabi-null-tape-r", m))
    bad_r = good_r.copy()
    bad_r[0] = np.frombuffer(oc.Q.to_bytes(32, "little"), dtype=np.uint64)
    out, ln = C.POINTER(C.c_ubyte)(), C.c_size_t()
    c_zr, zr, evals = C.create_string_buffer(32), np.zeros(4, dtype=np.uint64), np.zeros((k, 4), dtype=np.uint64)
    gens, joint_gens = sb.PolyCommitmentGens(m, LABEL), sb.PolyCommitmentGens(m + 1, LABEL)
    t = sb.Transcript(LABEL)
    before = t.state.raw

    def single(r):
        return sb.lib.sp_pc_eval_prove_t(ctx.h, gens.h, polys[0].h, None, ptr(r), C.c_size_t(m), None, None, t.state, None, C.byref(out),
                                         C.byref(ln), c_zr, ptr(zr))

    def joint(r):
        return sb.lib.sp_pc_eval_prove_joint_t(ctx.h, joint_gens.h, sb.api._handles(polys), C.c_int(k), None, ptr(r), C.c_size_t(m), t.state, None,
                                               C.byref(out), C.byref(ln), ptr(evals))

    for call, what in [(single, "pc_eval_prove"), (joint, "pc_eval_prove_joint")]:
        assert call(bad_r) == SP_ERR_INVALID_SCALAR
        assert sb.lib.sp_last_error(ctx.h).decode() == what + ": r: scalar limbs are not reduced modulo q"
        assert call(good_r) == SP_ERR_INVALID_ARG
        assert sb.lib.sp_last_error(ctx.h).decode() == what + ": tape state is NULL"
        assert t.state.raw == before
