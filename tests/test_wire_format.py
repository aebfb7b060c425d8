"""The proof wire format (spartan_b200/csrc/wire.hpp) without a GPU: the library's bincode Reader parses NIZK proofs, SNARK proofs and
computation commitments, and its Writer re-encodes them byte for byte; malformed inputs get the status code the C ABI returns for them.

A round trip cannot see a field order that is wrong on both sides alike: the GPU tests that verify oracle proofs and compare proof bytes
with the oracle's cover the layout itself."""
import ctypes as C
import os
import re

import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import r1cs, spark

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
NIZK, SNARK, COMMITMENT = 0, 1, 2


def _codes():
    with open(os.path.join(ROOT, "include", "spartan_b200.h")) as f:
        return {m.group(1): int(m.group(2)) for m in re.finditer(r"#define (SP_\w+) (\d+)", f.read())}


CODES = _codes()
SP_OK, SP_ERR_VERIFY, SP_ERR_INVALID_ARG = CODES["SP_OK"], CODES["SP_ERR_VERIFY"], CODES["SP_ERR_INVALID_ARG"]


@pytest.fixture(scope="module")
def lib():
    path = os.path.join(ROOT, "spartan_b200", "libsp_hosttest_fast.so")
    if not os.path.exists(path):
        import __graft_entry__ as ge
        ge.build_hosttest()
    l = C.CDLL(path)
    l.spt_wire_roundtrip.restype = C.c_int
    l.spt_wire_roundtrip.argtypes = [C.c_int, C.c_char_p, C.c_size_t, C.c_char_p, C.POINTER(C.c_size_t)]
    return l


def roundtrip(lib, kind, data):
    """(status code, re-encoded bytes or None)"""
    cap = len(data) + 64
    out = C.create_string_buffer(cap)
    n = C.c_size_t(cap)
    rc = lib.spt_wire_roundtrip(kind, data, len(data), out, C.byref(n))
    return rc, (out.raw[:n.value] if rc == SP_OK else None)


def assert_identical(lib, kind, data):
    rc, again = roundtrip(lib, kind, data)
    assert rc == SP_OK
    assert again == data


def _golden(name):
    with open(os.path.join(GOLDEN, name), "rb") as f:
        return f.read()


@pytest.fixture(scope="module")
def small_nizk():
    inst, vars_arr, inputs = r1cs.Instance.produce_synthetic_r1cs(2, 2, 1, 5)
    gens = r1cs.NIZKGens(2, 2, 1)
    return r1cs.NIZK.prove(inst, vars_arr, inputs, gens, oc.Transcript(b"nizk_example"), r1cs.tape_seed(5)).ser()


@pytest.fixture(scope="module")
def oracle_snark():
    """(proof bytes, commitment bytes) of the oracle's SNARK at 2^4 constraints"""
    n = 16
    inst, vars_arr, inputs = r1cs.Instance.produce_synthetic_r1cs(n, n, 10, 2)
    gens = spark.SNARKGens(n, n, 10, n)
    comm, decomm = spark.SNARK.encode(inst, gens)
    proof = spark.SNARK.prove(inst, comm, decomm, vars_arr, inputs, gens, oc.Transcript(b"snark_example"), r1cs.tape_seed(2))
    return proof.ser(), comm.ser()


@pytest.mark.parametrize("name", ["snark_2p20_proof.bin", "snark_2p22_proof.bin"])
def test_golden_snark_proofs_roundtrip(lib, name):
    assert_identical(lib, SNARK, _golden(name))


@pytest.mark.parametrize("num_cons,num_vars,num_inputs", [(16, 16, 3), (64, 256, 7), (2, 2, 1)])
def test_oracle_nizk_proofs_roundtrip(lib, num_cons, num_vars, num_inputs):
    inst, vars_arr, inputs = r1cs.Instance.produce_synthetic_r1cs(num_cons, num_vars, num_inputs, 5)
    gens = r1cs.NIZKGens(num_cons, num_vars, num_inputs)
    proof = r1cs.NIZK.prove(inst, vars_arr, inputs, gens, oc.Transcript(b"nizk_example"), r1cs.tape_seed(5)).ser()
    assert_identical(lib, NIZK, proof)


def test_oracle_snark_proof_and_commitment_roundtrip(lib, oracle_snark):
    proof, commitment = oracle_snark
    assert_identical(lib, SNARK, proof)
    assert_identical(lib, COMMITMENT, commitment)


def test_every_truncation_of_a_nizk_proof_is_rejected(lib, small_nizk):
    for k in range(len(small_nizk)):
        assert roundtrip(lib, NIZK, small_nizk[:k])[0] == SP_ERR_VERIFY, k


def test_truncations_of_the_2p20_snark_proof_are_rejected(lib):
    proof = _golden("snark_2p20_proof.bin")
    cuts = set(range(0, len(proof), 997)) | set(range(0, 600)) | set(range(len(proof) - 600, len(proof)))
    for k in sorted(cuts):
        assert roundtrip(lib, SNARK, proof[:k])[0] == SP_ERR_VERIFY, k


def test_trailing_byte_is_rejected(lib, small_nizk, oracle_snark):
    assert roundtrip(lib, NIZK, small_nizk + b"\0")[0] == SP_ERR_VERIFY
    assert roundtrip(lib, SNARK, _golden("snark_2p20_proof.bin") + b"\0")[0] == SP_ERR_VERIFY
    assert roundtrip(lib, COMMITMENT, oracle_snark[1] + b"\0")[0] == SP_ERR_INVALID_ARG


def test_unreduced_scalar_is_rejected(lib, small_nizk):
    """the last 32 bytes of either proof are a scalar (NIZK: the last entry of ry; SNARK: z2 of the derefs opening)"""
    q = oc.Q.to_bytes(32, "little")
    assert roundtrip(lib, NIZK, small_nizk[:-32] + q)[0] == SP_ERR_VERIFY
    proof = _golden("snark_2p20_proof.bin")
    assert roundtrip(lib, SNARK, proof[:-32] + q)[0] == SP_ERR_VERIFY
    assert roundtrip(lib, SNARK, proof[:-32] + (oc.Q - 1).to_bytes(32, "little"))[0] == SP_OK


def test_huge_length_prefix_is_rejected_before_allocating(lib, small_nizk, oracle_snark):
    """the first field of a proof is the length of comm_vars.C; the commitment's comm_comb_ops.C length follows six u64"""
    huge = (1 << 62).to_bytes(8, "little")
    assert roundtrip(lib, NIZK, huge + small_nizk[8:])[0] == SP_ERR_VERIFY
    assert roundtrip(lib, SNARK, huge + _golden("snark_2p20_proof.bin")[8:])[0] == SP_ERR_VERIFY
    commitment = oracle_snark[1]
    assert roundtrip(lib, COMMITMENT, commitment[:48] + huge + commitment[56:])[0] == SP_ERR_INVALID_ARG


def test_truncated_commitment_is_invalid_arg(lib, oracle_snark):
    commitment = oracle_snark[1]
    for k in range(len(commitment)):
        assert roundtrip(lib, COMMITMENT, commitment[:k])[0] == SP_ERR_INVALID_ARG, k
