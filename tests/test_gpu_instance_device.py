"""Instances and witnesses built on the device from CUDA tensors (Instance.from_tensors, DensePolynomial.from_tensor) against the host path.

Every shape tests/test_gpu_instance_shapes.py proves, the Instance::new padding case and an instance with more inputs than variables are built both
ways; the two instances must agree on bincode, digest, exported matrices and dimensions, on satisfiability, and give the same SNARK::encode
commitment and the same SNARK and NIZK proof bytes, which the library's verifiers accept.  The synthetic 2^18 instance rebuilt from its exported
matrices proves to the golden bytes.  Errors (bad rows, columns, scalars, several defects at once, tensors of the wrong kind) match the host path's
class and message; empty matrices, fewer than two constraints and address collisions in the memory-checking timestamps are covered too.
Run on the GPU: pytest -m gpu."""
import ctypes as C
import gc
import hashlib
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle.spartan_ref import core as oc  # noqa: E402
from oracle.spartan_ref import r1cs, spark  # noqa: E402
from test_instance_shapes import CASES, Spec, cached_instance  # noqa: E402

torch = pytest.importorskip("torch")

LABEL = b"device instances"
Q = oc.Q
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BUCKET = Spec("buckets", 512, 512, 10, (1225, 700, 900))   # the SNARKGens bucket case of test_gpu_instance_shapes.py


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as m
    m.default_context()
    return m


@pytest.fixture(autouse=True)
def release_device_memory(sb):
    yield
    gc.collect()
    sb.release_cached_memory()


def dev(sb):
    return "cuda:%d" % sb.default_context().device


def tensors(sb, triples):
    """(row, col, 32 bytes) triples -> (rows int64, cols int64, vals (n, 32) uint8) on the context's GPU; indices >= 2^63 wrap to negatives"""
    rows = np.array([r for r, _, _ in triples], dtype=np.uint64).view(np.int64)
    cols = np.array([c for _, c, _ in triples], dtype=np.uint64).view(np.int64)
    vals = np.frombuffer(b"".join(bytes(v) for _, _, v in triples), dtype=np.uint8).reshape(-1, 32).copy()
    return tuple(torch.from_numpy(a).to(dev(sb)) for a in (rows, cols, vals))


def canonical_tensor(sb, ints):
    return torch.from_numpy(np.frombuffer(b"".join(v.to_bytes(32, "little") for v in ints), dtype=np.uint8).reshape(-1, 32).copy()).to(dev(sb))


def unaligned(vals):
    """the same (n, 32) values as a contiguous view 8 bytes into its storage (not 16-byte aligned)"""
    flat = torch.zeros(vals.numel() + 8, dtype=torch.uint8, device=vals.device)
    flat[8:] = vals.reshape(-1)
    out = flat[8:].reshape(-1, 32)
    assert out.is_contiguous() and out.data_ptr() % 16 == 8
    return out


def both(sb, nc, nv, ni, triples):
    host = sb.Instance.new(nc, nv, ni, *triples)
    devi = sb.Instance.from_tensors(nc, nv, ni, *(tensors(sb, t) for t in triples))
    return host, devi


def same_shape(host, devi):
    assert (devi.num_cons, devi.num_vars, devi.num_inputs) == (host.num_cons, host.num_vars, host.num_inputs)
    for m in range(3):
        for a, b in zip(host.export(m), devi.export(m)):
            assert np.array_equal(a, b), "matrix %d" % m
    assert devi.bincode() == host.bincode()
    assert devi.digest == host.digest


class Case:
    def __init__(self, nc, nv, ni, triples, vars_, inputs):
        self.nc, self.nv, self.ni, self.triples, self.vars, self.inputs = nc, nv, ni, triples, vars_, inputs


def shape_case(spec):
    si = cached_instance(spec)
    return Case(spec.num_cons, spec.num_vars, spec.num_inputs, si.triples, si.vars, si.inputs)


def padding_case():
    """lib.rs:672-752 test_padded_constraints: one constraint, no variables, three inputs"""
    def s32(v):
        return (v % Q).to_bytes(32, "little")
    A = [(0, 2, s32(1))]
    B = [(0, 2, s32(1))]
    Cm = [(0, 1, s32(1)), (0, 0, s32(-13)), (0, 3, s32(-1))]
    return Case(1, 0, 3, [A, B, Cm], oc.zeros(0), [16, 1, 2])


CASE_IDS = list(CASES) + ["buckets", "padded_constraints"]


def make_case(name):
    if name == "padded_constraints":
        return padding_case()
    return shape_case(BUCKET if name == "buckets" else CASES[name][0])


def broken(sb, case):
    """the witness with one entry changed: the most used variable, or the first input when there are no variables"""
    vars_, inputs = case.vars.copy(), list(case.inputs)
    cols = np.array([c for t in case.triples for _, c, _ in t], dtype=np.int64)
    cols = cols[cols < case.nv]
    if len(cols):
        vars_[int(np.bincount(cols).argmax())] = oc.to_arr([12345])[0]
    else:
        inputs[0] = (inputs[0] + 1) % Q
    return sb.Assignment(vars_), sb.Assignment(oc.to_arr(inputs))


@pytest.mark.parametrize("name", CASE_IDS)
def test_device_instance_matches_host(sb, name):
    case = make_case(name)
    host, devi = both(sb, case.nc, case.nv, case.ni, case.triples)
    vars_, inputs = sb.Assignment(case.vars), sb.Assignment(oc.to_arr(case.inputs) if case.inputs else oc.zeros(0))
    seed = 5
    # SNARK first: the device instance proves before anything has asked for a host copy of its matrices
    nz = max(len(t) for t in case.triples)
    gens = sb.SNARKGens(case.nc, case.nv, case.ni, nz)
    comm_h, comm_d = sb.SNARK.encode(host, gens), sb.SNARK.encode(devi, gens)
    assert comm_d.commitment_bytes() == comm_h.commitment_bytes()
    proof_h = sb.SNARK.prove(host, comm_h, vars_, inputs, gens, LABEL, sb.tape_seed(seed))
    proof_d = sb.SNARK.prove(devi, comm_d, vars_, inputs, gens, LABEL, sb.tape_seed(seed))
    assert proof_d.bytes == proof_h.bytes
    proof_d.verify(comm_d, inputs, LABEL, gens)
    proof_d.verify(comm_h, inputs, LABEL, gens)
    del gens, comm_h, comm_d
    gc.collect()

    same_shape(host, devi)
    assert host.is_sat(vars_, inputs) and devi.is_sat(vars_, inputs)
    bad_vars, bad_inputs = broken(sb, case)
    assert not host.is_sat(bad_vars, bad_inputs) and not devi.is_sat(bad_vars, bad_inputs)

    ngens = sb.NIZKGens(case.nc, case.nv, case.ni)
    nproof_h = sb.NIZK.prove(host, vars_, inputs, ngens, LABEL, sb.tape_seed(seed))
    nproof_d = sb.NIZK.prove(devi, vars_, inputs, ngens, LABEL, sb.tape_seed(seed))
    assert nproof_d.bytes == nproof_h.bytes
    nproof_d.verify(devi, inputs, LABEL, ngens)
    nproof_d.verify(host, inputs, LABEL, ngens)


def test_synthetic_2p18_from_tensors_gives_golden_proof(sb):
    """the synthetic 2^18 instance exported, turned into canonical tensors and rebuilt by from_tensors proves to the golden bytes
    (tests/golden/snark_proof_sha256.json, "18": instance seed 0, 10 inputs, tape seed 0, label b"example")"""
    fx = json.load(open(os.path.join(GOLDEN, "snark_proof_sha256.json")))
    n = 1 << 18
    syn, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=0)
    mats = []
    for m in range(3):
        row, col, val = syn.export(m)
        mats.append((torch.from_numpy(row.view(np.int64)).to(dev(sb)), torch.from_numpy(col.view(np.int64)).to(dev(sb)), canonical_tensor(sb, oc.to_ints(val))))
    del syn
    inst = sb.Instance.from_tensors(n, n, 10, *mats)
    gens = sb.SNARKGens(n, n, 10, n)
    comm = sb.SNARK.encode(inst, gens)
    assert hashlib.sha256(comm.commitment_bytes()).hexdigest() == fx["18_commitment"]
    proof = sb.SNARK.prove(inst, comm, vars_, inputs, gens, b"example", sb.tape_seed(0))
    assert len(proof.bytes) == fx["18_len"] and hashlib.sha256(proof.bytes).hexdigest() == fx["18"]


# ---------------------------------------------------------------------------------------------------------------- errors
def s32(v):
    return int(v).to_bytes(32, "little")


def valid_triples(nc=4, nv=4, ni=2):
    rng = np.random.default_rng(7)
    return [[(int(rng.integers(0, nc)), int(rng.integers(0, nv + 1 + ni)), s32(rng.integers(0, 1 << 62))) for _ in range(n)] for n in (6, 5, 7)]


def with_defect(triples, m, k, row=None, col=None, val=None):
    t = [list(x) for x in triples]
    r, c, v = t[m][k]
    t[m][k] = (r if row is None else row, c if col is None else col, v if val is None else val)
    return t


def raised(f):
    with pytest.raises(Exception) as e:
        f()
    return e.value


def assert_same_error(sb, nc, nv, ni, triples, cls):
    eh = raised(lambda: sb.Instance.new(nc, nv, ni, *triples))
    ed = raised(lambda: sb.Instance.from_tensors(nc, nv, ni, *(tensors(sb, t) for t in triples)))
    assert type(eh) is cls and type(ed) is type(eh), (type(eh), type(ed))
    assert str(ed) == str(eh)
    return str(ed)


NC, NV, NI = 4, 4, 2
DEFECTS = {
    "row_eq_num_cons": ([(1, 3, dict(row=NC))], "(row)"),
    "col_eq_ncols": ([(0, 2, dict(col=NV + 1 + NI))], "(col)"),
    "row_2p63": ([(2, 0, dict(row=1 << 63))], "(row)"),
    "col_2p63": ([(2, 6, dict(col=1 << 63))], "(col)"),
    "val_q": ([(0, 0, dict(val=s32(Q)))], "InvalidScalar"),
    "val_q_plus_1": ([(1, 4, dict(val=s32(Q + 1)))], "InvalidScalar"),
    "val_2p256_minus_1": ([(2, 3, dict(val=b"\xff" * 32))], "InvalidScalar"),
    # several defects: the first in (matrix, entry) order wins, within one entry row before column before scalar
    "first_entry_wins": ([(0, 5, dict(row=NC)), (0, 3, dict(val=s32(Q))), (1, 0, dict(col=99))], "InvalidScalar"),
    "first_matrix_wins": ([(2, 0, dict(row=NC)), (1, 4, dict(col=NV + 1 + NI))], "(col)"),
    "col_before_scalar": ([(1, 2, dict(col=NV + 1 + NI, val=s32(Q)))], "(col)"),
    "row_before_col": ([(1, 2, dict(row=1 << 63, col=1 << 63, val=b"\xff" * 32))], "(row)"),
}


@pytest.mark.parametrize("name", list(DEFECTS))
def test_errors_match_host_path(sb, name):
    defects, want = DEFECTS[name]
    t = valid_triples(NC, NV, NI)
    for m, k, kw in defects:
        t = with_defect(t, m, k, **kw)
    msg = assert_same_error(sb, NC, NV, NI, t, sb.R1CSError)
    assert want in msg


def test_unaligned_and_strided_tensors(sb):
    """values that do not start on a 16-byte boundary, and non-contiguous index tensors, give the same instance"""
    t = valid_triples(NC, NV, NI)
    host = sb.Instance.new(NC, NV, NI, *t)
    mats = []
    for x in t:
        r, c, v = tensors(sb, x)
        rc = torch.stack([r, c], dim=1)               # rows and cols as strided columns of one tensor
        mats.append((rc[:, 0], rc[:, 1], unaligned(v)))
    assert not mats[0][0].is_contiguous()
    devi = sb.Instance.from_tensors(NC, NV, NI, *mats)
    same_shape(host, devi)
    t[2] = with_defect(t, 2, 1, val=s32(Q))[2]
    r, c, v = tensors(sb, t[2])
    mats[2] = (r, c, unaligned(v))
    with pytest.raises(sb.R1CSError, match="InvalidScalar"):
        sb.Instance.from_tensors(NC, NV, NI, *mats)


def test_tensor_kind_errors(sb):
    t = valid_triples(NC, NV, NI)
    good = [tensors(sb, x) for x in t]
    sb.Instance.from_tensors(NC, NV, NI, *good)
    cpu = tuple(x.cpu() for x in good[0])
    bad = {
        "cpu": [cpu, good[1], good[2]],
        "dtype": [good[0], (good[1][0].to(torch.int32), good[1][1], good[1][2]), good[2]],
        "val shape": [good[0], good[1], (good[2][0], good[2][1], good[2][2].reshape(-1))],
        "val width": [good[0], good[1], (good[2][0], good[2][1], good[2][2][:, :16])],
        "lengths": [(good[0][0][:-1], good[0][1], good[0][2]), good[1], good[2]],
        "not a triple": [good[0][:2], good[1], good[2]],
    }
    for what, mats in bad.items():
        with pytest.raises(sb.SpartanB200Error) as e:
            sb.Instance.from_tensors(NC, NV, NI, *mats)
        assert not isinstance(e.value, sb.R1CSError), what
    with pytest.raises(sb.SpartanB200Error):
        sb.DensePolynomial.from_tensor(canonical_tensor(sb, [1, 2]).cpu())
    with pytest.raises(sb.SpartanB200Error):
        sb.DensePolynomial.from_tensor(canonical_tensor(sb, [1, 2]).reshape(-1))


def test_c_abi_refuses_host_pointers(sb):
    """sp_instance_create_device / sp_poly_from_canonical_device check that every non-empty array is device memory of the context's GPU"""
    from spartan_b200 import api
    ctx = sb.default_context()
    rows = np.zeros(2, dtype=np.uint64)
    vals = np.zeros((2, 32), dtype=np.uint8)
    d_rows, d_cols, d_vals = tensors(sb, [(0, 0, s32(1)), (1, 1, s32(2))])
    h = C.c_void_p()
    p = api._p
    dv = [C.c_void_p(x.data_ptr()) for x in (d_rows, d_cols, d_vals)]
    for mats in ([p(rows), dv[1], dv[2]], [dv[0], p(rows), dv[2]], [dv[0], dv[1], p(vals)]):
        rc = api.lib.sp_instance_create_device(ctx.h, C.c_size_t(2), C.c_size_t(2), C.c_size_t(0), *mats, C.c_size_t(2), *dv, C.c_size_t(2), *dv,
                                               C.c_size_t(2), C.byref(h))
        assert rc == api.SP_ERR_INVALID_ARG, rc
        assert "device memory" in api.lib.sp_last_error(ctx.h).decode()
    rc = api.lib.sp_poly_from_canonical_device(ctx.h, p(vals), C.c_size_t(2), C.byref(h))
    assert rc == api.SP_ERR_INVALID_ARG
    rc = api.lib.sp_instance_create_device(ctx.h, C.c_size_t(2), C.c_size_t(2), C.c_size_t(0), *dv, C.c_size_t(2), *dv, C.c_size_t(2), *dv, C.c_size_t(2),
                                           C.byref(h))
    assert rc == api.SP_OK
    api.lib.sp_instance_free(h)


# ---------------------------------------------------------------------------------------------------------------- edge cases
def test_empty_matrices(sb):
    empty = [[], [], []]
    host, devi = both(sb, 4, 4, 2, empty)
    same_shape(host, devi)
    assert all(len(devi.export(m)[0]) == 0 for m in range(3))
    gens = sb.SNARKGens(4, 4, 2, 1)
    eh = raised(lambda: sb.SNARK.encode(host, gens))
    ed = raised(lambda: sb.SNARK.encode(devi, gens))
    assert type(ed) is type(eh) and str(ed) == str(eh)
    # one empty matrix among full ones
    t = valid_triples(NC, NV, NI)
    t[1] = []
    host, devi = both(sb, NC, NV, NI, t)
    same_shape(host, devi)


@pytest.mark.parametrize("num_cons", [0, 1])
def test_fewer_than_two_constraints(sb, num_cons):
    """Instance::new pads one constraint to two, and then appends (row i, column num_vars, 0) entries up to the padded count per matrix; zero
    constraints end up as one (0.next_power_of_two() = 1 overrides the two, lib.rs:143-156)"""
    host, devi = both(sb, num_cons, 3, 1, [[], [], []])
    same_shape(host, devi)
    padded = 2 if num_cons == 1 else 1
    assert devi.num_cons == padded and [len(devi.export(m)[0]) for m in range(3)] == [padded] * 3
    if num_cons == 1:
        t = [[(0, 1, s32(3))], [(0, 0, s32(Q - 1))], [(0, 3, s32(1))]]
        host, devi = both(sb, 1, 3, 1, t)
        same_shape(host, devi)
        gens = sb.SNARKGens(1, 3, 1, 2)
        assert sb.SNARK.encode(devi, gens).commitment_bytes() == sb.SNARK.encode(host, gens).commitment_bytes()
    else:
        assert_same_error(sb, 0, 3, 1, [[(0, 0, s32(1))], [], []], sb.R1CSError)


def test_timestamp_address_collisions(sb):
    """every entry of all three matrices at row 0, column 0: one address takes every read of both sides, so read_ts counts across matrices and
    positions; the commitment equals the oracle's SNARK::encode"""
    nc, nv, ni = 8, 8, 2
    rng = np.random.default_rng(11)
    t = [[(0, 0, s32(int(rng.integers(0, 1 << 62)) * 7919 % Q)) for _ in range(n)] for n in (16, 11, 9)]
    host, devi = both(sb, nc, nv, ni, t)
    same_shape(host, devi)
    gens = sb.SNARKGens(nc, nv, ni, 16)
    got = sb.SNARK.encode(devi, gens).commitment_bytes()
    assert got == sb.SNARK.encode(host, gens).commitment_bytes()
    oi = r1cs.Instance.new(nc, nv, ni, *t)
    ocomm, _ = spark.SNARK.encode(oi, spark.SNARKGens(nc, nv, ni, 16))
    assert got == ocomm.ser()


# ---------------------------------------------------------------------------------------------------------------- witness
def test_poly_from_tensor(sb):
    rng = np.random.default_rng(3)
    ints = [0, 1, Q - 1] + [int.from_bytes(rng.bytes(32), "little") % Q for _ in range(1000)]
    got = sb.DensePolynomial.from_tensor(canonical_tensor(sb, ints))
    assert got.len() == len(ints)
    assert np.array_equal(got.to_numpy(), sb.DensePolynomial(oc.to_arr(ints)).to_numpy())
    assert sb.DensePolynomial.from_tensor(canonical_tensor(sb, [])).len() == 0
    # a contiguous view whose storage starts 8 bytes into an allocation: the values are read bytewise
    assert np.array_equal(sb.DensePolynomial.from_tensor(unaligned(canonical_tensor(sb, ints))).to_numpy(), got.to_numpy())
    for bad in (Q, Q + 1, (1 << 256) - 1):
        with pytest.raises(sb.R1CSError) as e:
            sb.DensePolynomial.from_tensor(canonical_tensor(sb, ints[:10] + [bad] + ints[10:20]))
        assert "InvalidScalar" in str(e.value) and "entry 10" in str(e.value)


def test_prove_with_tensor_witness(sb):
    """SNARK and NIZK proofs with the witness given as a tensor equal those with the host assignment (a resident witness must already have
    num_vars entries: an instance whose num_vars is a power of two)"""
    case = shape_case(BUCKET)
    inst = sb.Instance.from_tensors(case.nc, case.nv, case.ni, *(tensors(sb, t) for t in case.triples))
    vars_, inputs = sb.Assignment(case.vars), sb.Assignment(oc.to_arr(case.inputs))
    wit = sb.DensePolynomial.from_tensor(canonical_tensor(sb, oc.to_ints(case.vars)))
    nz = max(len(t) for t in case.triples)
    gens = sb.SNARKGens(case.nc, case.nv, case.ni, nz)
    comm = sb.SNARK.encode(inst, gens)
    want = sb.SNARK.prove(inst, comm, vars_, inputs, gens, LABEL, sb.tape_seed(2)).bytes
    assert sb.SNARK.prove(inst, comm, wit, inputs, gens, LABEL, sb.tape_seed(2)).bytes == want
    ngens = sb.NIZKGens(case.nc, case.nv, case.ni)
    want = sb.NIZK.prove(inst, vars_, inputs, ngens, LABEL, sb.tape_seed(2)).bytes
    assert sb.NIZK.prove(inst, wit, inputs, ngens, LABEL, sb.tape_seed(2)).bytes == want
