"""The R1CSProof caller entries without a GPU: every entry the header declares is exported, the refusals that need no device are made before the
context is touched (so a NULL context reports them), and the claims (Ar, Br, Cr) the verifier takes are R1CSShape::evaluate, which the oracle's
verifier accepts and rejects as it should."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import r1cs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SP_ERR_INVALID_ARG = 3
Q = oc.Q
ENTRIES = ["sp_r1cs_gens_create", "sp_r1cs_gens_create_from", "sp_r1cs_gens_create_from_nizk", "sp_r1cs_gens_create_from_snark", "sp_r1cs_gens_free",
           "sp_r1cs_prove_t", "sp_r1cs_verify_t", "sp_instance_evaluate"]


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as sb
    return sb


def test_header_declares_and_library_exports_every_entry(sb):
    header = open(os.path.join(ROOT, "include", "spartan_b200.h")).read()
    for name in ENTRIES:
        assert re.search(r"\b%s\(" % name, header), name
        assert getattr(sb.lib, name) is not None, name
    assert hasattr(sb, "R1CSGens") and hasattr(sb, "R1CSProof") and hasattr(sb.Instance, "evaluate")


def last_error(sb):
    return sb.lib.sp_last_error(None).decode()


def prove_null_ctx(sb, num_cons, num_vars, ninputs, state, tape, inst=C.c_void_p(1), spmat=None):
    """sp_r1cs_prove_t on no context: only refusals that need no device can be reached"""
    out, n = C.POINTER(C.c_ubyte)(), C.c_size_t()
    inputs = np.zeros((max(ninputs, 1), 4), dtype=np.uint64)
    rx, ry = np.zeros((64, 4), dtype=np.uint64), np.zeros((64, 4), dtype=np.uint64)
    return sb.lib.sp_r1cs_prove_t(None, inst, spmat, C.c_size_t(num_cons), C.c_size_t(num_vars), None, inputs.ctypes.data_as(C.c_void_p), C.c_size_t(ninputs),
                                  None, state, tape, C.byref(out), C.byref(n), rx.ctypes.data_as(C.c_void_p), ry.ctypes.data_as(C.c_void_p))


def test_host_refusals_leave_the_states(sb):
    T, tape = sb.Transcript(b"r1cs-model"), sb.RandomTape(sb.tape_seed(0))
    t0, p0 = T.state.raw, tape.state.raw
    cases = [
        ((1 << 4, 1 << 4, 2, None, tape.state), "transcript state is NULL"),
        ((1 << 4, 1 << 4, 2, T.state, None), "tape state is NULL"),
        ((12, 1 << 4, 2, T.state, tape.state), "powers of two"),
        ((1 << 4, 24, 2, T.state, tape.state), "powers of two"),
        ((1, 1 << 4, 2, T.state, tape.state), "num_cons >= 2"),
        ((1 << 4, 1 << 4, 16, T.state, tape.state), "|inputs| + 1 = 17 > num_vars = 16"),
        ((1 << 4, 1 << 40, 0, T.state, tape.state), "supported"),
    ]
    for args, msg in cases:
        assert prove_null_ctx(sb, *args) == SP_ERR_INVALID_ARG, args
        assert msg in last_error(sb), (args, last_error(sb))
        assert T.state.raw == t0 and tape.state.raw == p0
    assert prove_null_ctx(sb, 16, 16, 2, T.state, tape.state, inst=None) == SP_ERR_INVALID_ARG
    assert "exactly one of inst and spmat" in last_error(sb)
    assert prove_null_ctx(sb, 16, 16, 2, T.state, tape.state, spmat=C.c_void_p(1)) == SP_ERR_INVALID_ARG
    assert "exactly one of inst and spmat" in last_error(sb)


def test_host_refusals_of_gens_and_verify(sb):
    h = C.c_void_p()
    assert sb.lib.sp_r1cs_gens_create(None, C.c_char_p(b"x"), C.c_size_t(1), C.c_size_t(16), C.c_size_t(12), C.byref(h)) == SP_ERR_INVALID_ARG
    assert "powers of two" in last_error(sb)
    assert sb.lib.sp_r1cs_gens_create(None, C.c_char_p(b"x"), C.c_size_t(1), C.c_size_t(16), C.c_size_t(16), None) == SP_ERR_INVALID_ARG
    assert "NULL argument" in last_error(sb)
    assert sb.lib.sp_r1cs_gens_create_from_nizk(None, None, C.c_size_t(16), C.c_size_t(16), C.byref(h)) == SP_ERR_INVALID_ARG
    T = sb.Transcript(b"r1cs-model")
    t0 = T.state.raw
    ev = np.zeros((3, 4), dtype=np.uint64)
    rx, ry = np.zeros((64, 4), dtype=np.uint64), np.zeros((64, 4), dtype=np.uint64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    for nc, nv, ni, msg in ((16, 12, 0, "powers of two"), (16, 4, 4, "|inputs| + 1 = 5 > num_vars = 4"), (16, 16, 0, "gens is NULL")):
        inputs = np.zeros((max(ni, 1), 4), dtype=np.uint64)
        rc = sb.lib.sp_r1cs_verify_t(None, C.c_char_p(b"\0" * 8), C.c_size_t(8), C.c_size_t(nc), C.c_size_t(nv), p(inputs), C.c_size_t(ni), p(ev), None,
                                     T.state, p(rx), p(ry))
        assert rc == SP_ERR_INVALID_ARG and msg in last_error(sb), (nc, nv, ni, last_error(sb))
        assert T.state.raw == t0


def brute_evaluate(shape, rx, ry):
    """sum over the entries of eq(rx, row) eq(ry, col) val, in integers"""
    ex, ey = oc.to_ints(oc.eq_evals(rx)), oc.to_ints(oc.eq_evals(ry))
    out = []
    for M in (shape.A, shape.B, shape.C):
        row, col, val = M.row, M.col, oc.to_ints(M.val) if isinstance(M.val, np.ndarray) and M.val.ndim == 2 else list(M.val)
        out.append(sum(ex[int(r)] * ey[int(c)] * int(v) for r, c, v in zip(row, col, val)) % Q)
    return out


def test_evals_are_the_shape_evaluation_the_oracle_verifier_needs(sb):
    n, ni, seed = 16, 3, 5
    oi, ovars, oinputs = r1cs.Instance.produce_synthetic_r1cs(n, n, ni, seed)
    shape = oi.inst
    label = b"r1cs-model-evals"
    gens = pr.R1CSGens(label, n, n)
    T, tape = oc.Transcript(label), oc.RandomTape(b"proof", 7)
    proof, rx, ry = pr.R1CSProof.prove(shape, r1cs.pad_vars(ovars, n), [int(v) for v in oinputs], gens, T, tape)
    evals = shape.evaluate(rx, ry)
    assert list(evals) == brute_evaluate(shape, rx, ry)
    vrx, vry = pr.R1CSProof.verify(proof, n, n, [int(v) for v in oinputs], tuple(evals), oc.Transcript(label), gens)
    assert list(vrx) == list(rx) and list(vry) == list(ry)
    for k in range(3):
        bad = list(evals)
        bad[k] = (bad[k] + 1) % Q
        with pytest.raises((pr.ProofVerifyError, AssertionError)):
            pr.R1CSProof.verify(proof, n, n, [int(v) for v in oinputs], tuple(bad), oc.Transcript(label), gens)
