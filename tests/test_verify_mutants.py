"""Structured mutants of whole proofs, judged by the oracle verifier (the CPU half of test_gpu_verify_mutants.py, which imports the machinery here).

A valid proof satisfies every equation the verifier tests, so an accepting test cannot see a check that was dropped or folded wrongly.  A
random byte flip cannot see it either: a flipped point almost never decodes, and a flipped value that is absorbed changes every later
challenge.  Here every field of a proof is walked in wire order (spartan_b200/csrc/wire.hpp states the same order) and mutated in place:
    scalars  x+1, q-1-x, swapped with the next element of the same vector or tuple;
    points   P+G (G a generator no proof uses), -P, the identity, a copy of another point of the proof, and one encoding per class the
             decoder rejects (s >= p, s negative, not square, t negative, y = 0);
    vectors  the last element removed or repeated (whole element spans, length prefix adjusted), L_vec[i] swapped with R_vec[i];
and the same point operators on the points of the computation commitment.  A malicious prover that permutes one leaf vector of the hash layer
reaches the four hash-layer checks, which nothing else can reach: the permutation leaves every product, so every earlier check, intact.

The oracle's verdict on the same bytes is the expected outcome: accept, DecompressionError, a ProofVerifyError label, or an AssertionError /
IndexError (where the reference panics).  This file checks the walker against the library's wire reader and the oracle's verdicts
themselves: every mutant is rejected except the listed divergences, and each oracle label the mapping table names is reached."""
import ctypes as C
import dataclasses
import os
import re
import typing

import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import r1cs, spark

Q = oc.Q
P_FIELD = 2**255 - 19
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------------- the field walker
@dataclasses.dataclass(frozen=True)
class Field:
    path: str          # e.g. r1cs_sat_proof.sc_proof_phase1.proofs[0].z[2]
    off: int           # byte offset in the encoding
    kind: str          # "scalar", "point" or "vec"
    span: int          # bytes, a vector's length prefix included
    elems: tuple = ()  # vec: (offset, span) of every element


def walk(tp, buf, pos=0, path="", out=None):
    """every scalar, point and vector of bincode(tp) in buf[pos:], as protocol.deser reads them: (end offset, [Field])"""
    out = [] if out is None else out
    origin = typing.get_origin(tp)
    if tp is int or tp is bytes:
        out.append(Field(path, pos, "scalar" if tp is int else "point", 32))
        return pos + 32, out
    if origin in (list, typing.List):
        (inner,) = typing.get_args(tp)
        n = int.from_bytes(buf[pos:pos + 8], "little")
        assert 8 * n <= len(buf) - pos, "length prefix at %d exceeds the input" % pos
        at, start = len(out), pos
        out.append(None)
        pos += 8
        elems = []
        for i in range(n):
            end, _ = walk(inner, buf, pos, "%s[%d]" % (path, i), out)
            elems.append((pos, end - pos))
            pos = end
        out[at] = Field(path, start, "vec", pos - start, tuple(elems))
        return pos, out
    if origin in (tuple, typing.Tuple):
        for i, inner in enumerate(typing.get_args(tp)):
            pos, _ = walk(inner, buf, pos, "%s[%d]" % (path, i), out)
        return pos, out
    if dataclasses.is_dataclass(tp):
        hints = typing.get_type_hints(tp)
        for f in dataclasses.fields(tp):
            pos, _ = walk(hints[f.name], buf, pos, (path + "." if path else "") + f.name, out)
        return pos, out
    raise TypeError(tp)


def walk_commitment(data):
    """the points of bincode(ComputationCommitment): six u64, then comm_comb_ops.C and comm_comb_mem.C"""
    out = []
    pos = 48
    for name in ("comm_comb_ops", "comm_comb_mem"):
        pos, _ = walk(pr.PolyCommitment, data, pos, "comm." + name, out)
    assert pos == len(data)
    return out


def parse_commitment(data):
    """bincode(ComputationCommitment) -> spark.R1CSCommitment"""
    u = [int.from_bytes(data[8 * i:8 * i + 8], "little") for i in range(6)]
    ops, pos = pr.deser(pr.PolyCommitment, data, 48)
    mem, pos = pr.deser(pr.PolyCommitment, data, pos)
    assert pos == len(data)
    return spark.R1CSCommitment(u[0], u[1], u[2], spark.SparseMatPolyCommitment(u[3], u[4], u[5], ops, mem))


# ---------------------------------------------------------------------------------------------------- mutation operators
MUTANT_GENERATOR = oc.MultiCommitGens.new(1, b"spartan-b200 verifier mutants").g(0)   # a point no proof uses


def invalid_encodings():
    """one encoding per class ristretto255 decoding rejects (RFC 9496 4.3.1), the late ones as test_gpu_arith.py finds them"""
    from test_gpu_arith import late_rejections
    late = late_rejections()
    return {"s >= p": (P_FIELD + 1).to_bytes(32, "little"), "s negative": (1).to_bytes(32, "little"), "not square": late["not square"],
            "t negative": late["t negative"], "y = 0": late["y = 0"]}


@dataclasses.dataclass
class Mutant:
    name: str          # "<path> <operator>"
    path: str
    op: str
    data: bytes        # the mutated proof, or the proof itself for a commitment mutant
    comm: bytes = None  # the mutated commitment (commitment mutants only)
    length: bool = False   # the vector's length changed


def _put(buf, off, b):
    return bytes(buf[:off]) + b + bytes(buf[off + len(b):])


def _point_ops(data, f, points, bad):
    """(operator, new 32 bytes) for the point field f of data"""
    cur = bytes(data[f.off:f.off + 32])
    P = oc.Point.decompress(cur)
    ops = [("P+G", (P + MUTANT_GENERATOR).compress()), ("-P", (oc.Point.identity() - P).compress()), ("identity", bytes(32))]
    other = next((p for p in points[points.index(cur) + 1:] + points if p != cur), None)
    if other is not None:
        ops.append(("copy", other))
    ops += [("invalid: " + k, v) for k, v in bad.items()]
    return [(op, b) for op, b in ops if b != cur]


def mutants(data, fields, pick=None):
    """every mutant of the proof `data` whose walk is `fields`; pick(field) -> bool keeps a subset (sampling at large shapes)"""
    bad = invalid_encodings()
    points = [bytes(data[f.off:f.off + 32]) for f in fields if f.kind == "point"]
    by_path = {f.path: f for f in fields}
    out = []
    for f in fields:
        if pick is not None and not pick(f):
            continue
        if f.kind == "scalar":
            x = oc.from_mont_bytes(data[f.off:f.off + 32])
            for op, y in (("x+1", (x + 1) % Q), ("q-1-x", (Q - 1 - x) % Q)):
                if y != x:
                    out.append(Mutant(f.path + " " + op, f.path, op, _put(data, f.off, oc.mont_bytes(y))))
            m = re.fullmatch(r"(.*)\[(\d+)\]", f.path)
            nb = by_path.get("%s[%d]" % (m.group(1), int(m.group(2)) + 1)) if m else None
            if nb is not None and nb.kind == "scalar" and data[nb.off:nb.off + 32] != data[f.off:f.off + 32]:
                swapped = _put(_put(data, f.off, bytes(data[nb.off:nb.off + 32])), nb.off, bytes(data[f.off:f.off + 32]))
                out.append(Mutant(f.path + " swap next", f.path, "swap next", swapped))
        elif f.kind == "point":
            for op, b in _point_ops(data, f, points, bad):
                out.append(Mutant(f.path + " " + op, f.path, op, _put(data, f.off, b)))
        elif f.elems:
            n = len(f.elems)
            (lo, ls) = f.elems[-1]
            dropped = data[:f.off] + (n - 1).to_bytes(8, "little") + data[f.off + 8:lo] + data[lo + ls:]
            repeated = data[:f.off] + (n + 1).to_bytes(8, "little") + data[f.off + 8:lo + ls] + data[lo:lo + ls] + data[lo + ls:]
            out.append(Mutant(f.path + " drop last", f.path, "drop last", bytes(dropped), length=True))
            out.append(Mutant(f.path + " repeat last", f.path, "repeat last", bytes(repeated), length=True))
            if f.path.endswith(".L_vec"):
                R = by_path[f.path[:-len("L_vec")] + "R_vec"]
                for i, ((lo_, _), (ro, _)) in enumerate(zip(f.elems, R.elems)):
                    swapped = _put(_put(data, lo_, bytes(data[ro:ro + 32])), ro, bytes(data[lo_:lo_ + 32]))
                    out.append(Mutant("%s[%d] swap R_vec[%d]" % (f.path, i, i), "%s[%d]" % (f.path, i), "swap L R", swapped))
    return out


def commitment_mutants(proof, comm, pick=None):
    """the point operators on comm_comb_ops.C and comm_comb_mem.C; the proof stays as it is"""
    bad = invalid_encodings()
    fields = walk_commitment(comm)
    points = [bytes(comm[f.off:f.off + 32]) for f in fields if f.kind == "point"]
    return [Mutant(f.path + " " + op, f.path, op, proof, comm=_put(comm, f.off, b)) for f in fields if f.kind == "point" and (pick is None or pick(f))
            for op, b in _point_ops(comm, f, points, bad)]


# ---------------------------------------------------------------------------------------------------- the malicious prover for the hash layer
HASH_TARGETS = [(side, leaf) for side in ("row", "col") for leaf in ("init", "read", "write", "audit")]


def hash_layer_proof(side, leaf, prove):
    """prove() with spark.build_hash_layer patched so that, on `side`, two unequal entries of the `leaf` vector (init, reads[1], writes[1] or
    audit) trade places before the product circuits are built.  Every product, so the prover's own assert, the subset check and every
    product-circuit proof, still hold; only the hash-layer check of that leaf can fail."""
    real = spark.build_hash_layer
    calls = []

    def permuted(*args):
        init, reads, writes, audit = real(*args)
        if len(calls) == ("row", "col").index(side):
            v = {"init": init, "read": reads[1], "write": writes[1], "audit": audit}[leaf]
            j = next(j for j in range(1, len(v)) if (v[j] != v[0]).any())
            v[[0, j]] = v[[j, 0]]
        calls.append(side)
        return init, reads, writes, audit
    with pytest.MonkeyPatch.context() as m:
        m.setattr(spark, "build_hash_layer", permuted)
        out = prove()
    assert len(calls) == 2
    return out


# ---------------------------------------------------------------------------------------------------- the oracle as judge
ACCEPT, DECOMPRESS = "accept", "DecompressionError"


def oracle_verdict(verify):
    """ACCEPT, DECOMPRESS, the ProofVerifyError label, or "panic: <exception type>" (the reference panics there)"""
    try:
        verify()
        return ACCEPT
    except pr.ProofVerifyError as e:
        return str(e)
    except (AssertionError, IndexError) as e:
        return "panic: " + type(e).__name__


class OracleStatement:
    """one statement on the oracle's side: verdict(kind, proof bytes, commitment bytes) for NIZK ("nizk") or SNARK ("snark") proofs"""

    def __init__(self, nc, nv, ni, seed, label, digest=None, kinds=("nizk", "snark")):
        self.inst, self.vars, self.inputs = r1cs.Instance.produce_synthetic_r1cs(nc, nv, ni, seed)
        if digest is not None:
            self.inst.digest = digest
        self.label = label
        if "nizk" in kinds:
            self.ngens = r1cs.NIZKGens(nc, nv, ni)
        if "snark" in kinds:
            self.sgens = spark.SNARKGens(nc, nv, ni, nc)
            self.comm, self.decomm = spark.SNARK.encode(self.inst, self.sgens)

    def prove(self, kind, seed):
        if kind == "nizk":
            return r1cs.NIZK.prove(self.inst, self.vars, self.inputs, self.ngens, oc.Transcript(self.label), r1cs.tape_seed(seed)).ser()
        return spark.SNARK.prove(self.inst, self.comm, self.decomm, self.vars, self.inputs, self.sgens, oc.Transcript(self.label), r1cs.tape_seed(seed)).ser()

    def verdict(self, kind, data, comm=None):
        if kind == "nizk":
            return oracle_verdict(lambda: _deser(r1cs.NIZK, data).verify(self.inst, self.inputs, oc.Transcript(self.label), self.ngens))
        c = self.comm if comm is None else parse_commitment(comm)
        return oracle_verdict(lambda: _deser(spark.SNARK, data).verify(c, self.inputs, oc.Transcript(self.label), self.sgens))


def _deser(tp, data):
    v, end = pr.deser(tp, data)
    assert end == len(data)
    return v


PROOF_TYPE = {"nizk": r1cs.NIZK, "snark": spark.SNARK}


# ---------------------------------------------------------------------------------------------------- the library's expected answer
# an oracle ProofVerifyError label -> the label the library's verifier (csrc/verifier.cpp) names for the same check
LABELS = [
    (r"KnowledgeProof", "KnowledgeProof"),
    (r"ProductProof", "ProductProof"),
    (r"EqualityProof", "EqualityProof"),
    (r"ZKSumcheck round \d+", "DotProductProof"),        # the DotProductProof of that round; an undecodable point of it too (sumcheck.rs:164-176)
    (r"DotProductProofLog", "DotProductProofLog"),
    (r"bullet size", "bullet reduction size"),
    (r"product circuit layer (\d+)", r"product circuit layer \1"),
    (r"subset check", "memory check: init * writes != reads * audit"),
    (r"dotp split", "dot product split"),
    (r"dotp claims", "dot product claims"),
    (r"hash init", "hash layer: init"),
    (r"hash read", "hash layer: read"),
    (r"hash write", "hash layer: write"),
    (r"hash audit", "hash layer: audit"),
]

# the library's shape checks: where the reference panics (the oracle's AssertionError / IndexError) the library rejects at one of these.  A
# vector whose length was changed may also meet one of them before the check the oracle fails at, which reads the vector past or short of
# its data.
SHAPE_LABELS = {"ZK sumcheck shape", "DotProductProof shape", "sumcheck rounds", "sumcheck degree", "bullet reduction size", "polynomial commitment size",
                "product circuit depth", "product circuit claims", "dotp claims shape", "product layer shape", "dotp shape", "hash layer shape",
                "claimed evaluation point"}

# mutants the oracle (so the reference) accepts and the library rejects, with why the library is right
DIVERGENCES = [
    (r"r1cs_sat_proof\.sc_proof_phase[12]\.proofs repeat last", "ZK sumcheck shape",
     "a ZK sumcheck with a DotProductProof beyond its rounds: sumcheck.rs:84-179 checks the lengths of comm_polys and comm_evals only, so the "
     "reference accepts two encodings of one proof; the library rejects the trailing proof to keep proofs non-malleable"),
    (r"r1cs_eval_proof\.poly_eval_network_proof\.proof_prod_layer\.proof_ops\.claims_dotp\[[12]\] repeat last", "dotp claims shape",
     "a trailing entry of dotp_right or dotp_weight: product_tree.rs:436-449 iterates over dotp_left only, so the reference ignores it; the "
     "library requires the three vectors to have one entry per dot-product claim, for the same reason"),
]

# checks of verifier.cpp that no parsed proof reaches, with the reason
UNREACHABLE = {
    "evaluation point differs from the sumcheck challenges": "the claimed rx, ry fix the instance evaluations, so a wrong point fails the phase-2 "
                                                             "EqualityProof first",
    "memory size": "2^|rx| is a function of the commitment's num_cons and num_vars, which check_commitment ties to num_mem_cells",
    "DotProductProofLog size": "the generators of every opening are sized from the statement, never from the proof",
    "polynomial commitment size": "every commitment is absorbed before it is opened, so one of another length changes the challenges and an "
                                  "earlier check fails",
    "claims shape": "batched_verify returns as many claims as it was given, and bounds the dot-product claims by their shape check",
    "product circuit randomness": "layer i of a product circuit has exactly i sumcheck rounds once the round count is checked",
    "number of inputs": "the inputs are the caller's, not part of the proof",
}

# every check verifier.cpp names (chk.equal sites and throw Reject), as the library reports it
LIBRARY_CHECKS = {
    "KnowledgeProof", "EqualityProof", "ProductProof", "DotProductProof", "DotProductProof shape", "ZK sumcheck shape", "sumcheck rounds", "sumcheck degree",
    "bullet reduction size", "DotProductProofLog size", "DotProductProofLog", "polynomial commitment size", "product circuit depth",
    "product circuit claims", "product circuit randomness", "dotp claims shape", "product circuit layer", "hash layer: init", "hash layer shape",
    "hash layer: read", "hash layer: write", "hash layer: audit", "memory size", "product layer shape", "memory check: init * writes != reads * audit",
    "dotp shape", "dot product split", "claims shape", "dot product claims", "number of inputs", "claimed evaluation point",
    "evaluation point differs from the sumcheck challenges",
}


def library_label(oracle_label):
    for pat, lib_label in LABELS:
        m = re.fullmatch(pat, oracle_label)
        if m:
            return m.expand(lib_label)
    raise AssertionError("oracle label %r has no entry in LABELS" % oracle_label)


def divergence(m):
    return next((d for d in DIVERGENCES if re.fullmatch(d[0], m.name)), None)


def check_name(label):
    """the check a library label names (the layer index dropped)"""
    return re.sub(r" \d+$", "", label)


# ---------------------------------------------------------------------------------------------------- CPU tests
def _library_reader():
    path = os.path.join(ROOT, "spartan_b200", "libsp_hosttest_fast.so")
    if not os.path.exists(path):
        import __graft_entry__ as ge
        ge.build_hosttest()
    lib = C.CDLL(path)
    lib.spt_wire_roundtrip.restype = C.c_int
    lib.spt_wire_roundtrip.argtypes = [C.c_int, C.c_char_p, C.c_size_t, C.c_char_p, C.POINTER(C.c_size_t)]

    def roundtrip(kind, data):
        out = C.create_string_buffer(len(data) + 64)
        n = C.c_size_t(len(data) + 64)
        rc = lib.spt_wire_roundtrip({"nizk": 0, "snark": 1}[kind], data, len(data), out, C.byref(n))
        return rc, out.raw[:n.value] if rc == 0 else None
    return roundtrip


CPU_SHAPES = [(2, 2, 1, 5), (16, 16, 3, 0), (32, 32, 4, 2)]


@pytest.fixture(scope="module")
def statements():
    return {s: OracleStatement(*s, b"mutants") for s in CPU_SHAPES}


@pytest.fixture(scope="module")
def proofs(statements):
    return {(s, kind): statements[s].prove(kind, s[3]) for s in CPU_SHAPES for kind in ("nizk", "snark")}


@pytest.mark.parametrize("kind", ["nizk", "snark"])
@pytest.mark.parametrize("shape", CPU_SHAPES)
def test_walker_follows_the_wire_format(proofs, shape, kind):
    """the walk ends at the proof's length, and the library's wire reader agrees on every field: q written over a scalar is refused as
    unreduced, the same bytes over a point are taken as they are, a length prefix one too large is refused"""
    data = proofs[(shape, kind)]
    end, fields = walk(PROOF_TYPE[kind], data)
    assert end == len(data)
    assert [f.off for f in fields if f.kind != "vec"] == sorted(f.off for f in fields if f.kind != "vec")
    roundtrip = _library_reader()
    assert roundtrip(kind, data) == (0, data)
    q = Q.to_bytes(32, "little")
    for f in fields:
        if f.kind == "vec":
            n = int.from_bytes(data[f.off:f.off + 8], "little")
            assert roundtrip(kind, _put(data, f.off, (n + 1).to_bytes(8, "little")))[0] != 0, f.path
            continue
        bad = _put(data, f.off, q)
        rc, again = roundtrip(kind, bad)
        if f.kind == "scalar":
            assert rc != 0, f.path
        else:
            assert (rc, again) == (0, bad), f.path


def test_walker_counts(proofs):
    """the field counts at 16 x 16 x 3: a SNARK proof has 316 scalars, 93 points and 89 length prefixes, a NIZK proof 146 fields in all"""
    _, f = walk(spark.SNARK, proofs[((16, 16, 3, 0), "snark")])
    assert [sum(x.kind == k for x in f) for k in ("scalar", "point", "vec")] == [316, 93, 89]
    _, f = walk(r1cs.NIZK, proofs[((16, 16, 3, 0), "nizk")])
    assert len(f) == 146


def _sample(k):
    """the fields whose every index is below 2 or a multiple of k: all field kinds, a bounded count at larger shapes"""
    def pick(f):
        idx = [int(i) for i in re.findall(r"\[(\d+)\]", f.path)]
        return all(i < 2 or i % k == 0 for i in idx)
    return pick


@pytest.mark.parametrize("kind", ["nizk", "snark"])
@pytest.mark.parametrize("shape", CPU_SHAPES[:2])
def test_oracle_rejects_every_mutant(statements, proofs, shape, kind):
    """every mutant is rejected, except those the divergence list names; the oracle labels reached include every entry of LABELS that a
    proof of this kind has (the hash layer's: test_malicious_prover_reaches_each_hash_check)"""
    st, data = statements[shape], proofs[(shape, kind)]
    _, fields = walk(PROOF_TYPE[kind], data)
    ms = mutants(data, fields)
    if kind == "snark":
        ms += commitment_mutants(data, st.comm.ser())
    seen = set()
    for m in ms:
        v = st.verdict(kind, m.data, m.comm)
        if divergence(m):
            assert v == ACCEPT, m.name
            continue
        assert v != ACCEPT, m.name
        if v != DECOMPRESS and not v.startswith("panic: "):
            seen.add(next(p for p, _ in LABELS if re.fullmatch(p, v)))
    assert {d[0] for d in DIVERGENCES if any(re.fullmatch(d[0], m.name) for m in ms)} == {d[0] for d in DIVERGENCES[:1 if kind == "nizk" else 2]}
    want = {"KnowledgeProof", "ProductProof", "EqualityProof", r"ZKSumcheck round \d+", "DotProductProofLog", "bullet size"}
    if kind == "snark":
        want |= {r"product circuit layer (\d+)", "subset check", "dotp split", "dotp claims"}
    assert want <= seen, want - seen


@pytest.mark.parametrize("side,leaf", HASH_TARGETS)
def test_malicious_prover_reaches_each_hash_check(statements, side, leaf):
    """a permuted leaf vector passes the prover's own checks and fails the oracle at exactly the hash check of that leaf"""
    st = statements[(16, 16, 3, 0)]
    data = hash_layer_proof(side, leaf, lambda: st.prove("snark", 0))
    assert st.verdict("snark", data) == "hash " + leaf
