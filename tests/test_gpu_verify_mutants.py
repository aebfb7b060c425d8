"""Both verifiers on structured mutants of whole proofs, with the oracle verifier as judge (the mutants, the oracle side and the label table:
test_verify_mutants.py).

For every mutant, the single verify (sp_*_verify, the immediate checker of csrc/verifier.cpp) must give the oracle's verdict on the same bytes:
SP_OK where it accepts, SP_ERR_DECOMPRESS for a DecompressionError, SP_ERR_VERIFY with the library label of the check the oracle names for a
ProofVerifyError, and SP_ERR_VERIFY with a shape label where the oracle raises AssertionError / IndexError (the reference panics).  The listed
divergences are the only mutants the oracle accepts.  Then every mutant goes through one verify_batch call (the deferred checker: all of a
proof's group equations weighted by random scalars and folded into one MSM), interleaved with valid proofs and with one mutant twice, and every
status must equal the single call's; a batch made only of mutants that each break one group equation catches a fold term dropped or mis-signed.
Last, the set of labels the mutants produced must be every check verifier.cpp has, except the few listed as unreachable.

Shapes, each for a path of its own: 2 x 2 x 1 (inner-product arguments of lg n = 1), 16 x 16 x 3 (every C_LZ on the host: at most 8 points),
32 x 32 x 4 SNARK (comm_derefs and comm_comb_ops of 16 points: the device C_LZ, decompress_batch + Pippenger) and a 1024 x 1024 x 10 NIZK
(comm_vars of 32 points), the last two on a sample of the fields.  Run on the GPU: pytest -m gpu."""
import os
import re
import subprocess
import sys

import pytest

from test_verify_mutants import (ACCEPT, DECOMPRESS, DIVERGENCES, HASH_TARGETS, LIBRARY_CHECKS, PROOF_TYPE, SHAPE_LABELS, UNREACHABLE, Mutant,
                                 OracleStatement, _sample, check_name, commitment_mutants, divergence, hash_layer_proof, library_label, mutants, walk)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LABEL = b"mutants"
# (name, num_cons, num_vars, num_inputs, seed, kinds, field sampler)
SHAPES = [("2x2x1", 2, 2, 1, 5, ("nizk", "snark"), None),
          ("16x16x3", 16, 16, 3, 0, ("nizk", "snark"), None),
          ("32x32x4", 32, 32, 4, 2, ("snark",), _sample(4)),
          ("1024x1024x10", 1024, 1024, 10, 2, ("nizk",), _sample(8))]
CASES = [(s[0], k) for s in SHAPES for k in s[5]]
# scalars that no transcript absorbs and that enter exactly one group equation
ONE_EQUATION = r".*(\.z1|\.z2|\.z|\.z_delta|\.z_beta|pok_claims_phase2\[1\]\.z\[[0134]\]) x\+1"


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as m
    m.default_context()
    return m


class Case:
    """one statement and one valid proof of it, both verifiers' view, and every mutant with the oracle's verdict and the single call's result"""

    def __init__(self, sb, name, kind):
        from spartan_b200 import api
        _, nc, nv, ni, seed, kinds, pick = next(s for s in SHAPES if s[0] == name)
        self.kind = kind
        self.inst, vars_, self.inputs = sb.Instance.produce_synthetic_r1cs(nc, nv, ni, seed=seed)
        self.oracle = OracleStatement(nc, nv, ni, seed, LABEL, digest=self.inst.digest, kinds=(kind,))
        if kind == "nizk":
            self.gens = sb.NIZKGens(nc, nv, ni)
            self.stmt = self.inst
            self.good = sb.NIZK.prove(self.inst, vars_, self.inputs, self.gens, LABEL, sb.tape_seed(seed)).bytes
        else:
            self.gens = sb.SNARKGens(nc, nv, ni, nc)
            self.stmt = sb.SNARK.encode(self.inst, self.gens)
            self.good = sb.SNARK.prove(self.inst, self.stmt, vars_, self.inputs, self.gens, LABEL, sb.tape_seed(seed)).bytes
            self.comm_bytes = self.stmt.commitment_bytes()
            assert self.comm_bytes == self.oracle.comm.ser()
        self.P = sb.NIZK if kind == "nizk" else sb.SNARK
        _, fields = walk(PROOF_TYPE[kind], self.good)
        self.mutants = mutants(self.good, fields, pick)
        if kind == "snark":
            self.mutants += commitment_mutants(self.good, self.comm_bytes, pick)
            if name == "16x16x3":
                self.mutants += [Mutant("hash layer %s %s permuted" % t, "hash layer", "permute", hash_layer_proof(*t, lambda: self.oracle.prove("snark", seed)))
                                 for t in HASH_TARGETS]
        self.comms = {}
        self.verdicts = [self.oracle.verdict(kind, m.data, m.comm) for m in self.mutants]
        self.results = [self.single(m) for m in self.mutants]
        self.api = api

    def statement(self, m):
        if m.comm is None:
            return self.stmt
        if m.comm not in self.comms:
            from spartan_b200 import api
            self.comms[m.comm] = api.ComputationCommitment.from_bytes(m.comm)
        return self.comms[m.comm]

    def single(self, m):
        """(status, label): the label is what follows "proof rejected: " in the message"""
        from spartan_b200 import api
        try:
            self.P(m.data).verify(self.statement(m), self.inputs, LABEL, self.gens)
            return api.SP_OK, None
        except api.ProofVerifyError as e:
            return e.code, str(e).split("proof rejected: ", 1)[1]


_cases = {}


def case(sb, name, kind):
    if (name, kind) not in _cases:
        _cases[(name, kind)] = Case(sb, name, kind)
    return _cases[(name, kind)]


def mismatch(api, m, verdict, code, label):
    """None when the single call's (code, label) is what the oracle's verdict asks for, else why not"""
    d = divergence(m)
    if d:
        ok = verdict == ACCEPT and code == api.SP_ERR_VERIFY and label == d[1]
    elif verdict == ACCEPT:
        ok = code == api.SP_OK
    elif verdict == DECOMPRESS:
        ok = code == api.SP_ERR_DECOMPRESS
    elif verdict.startswith("panic: "):
        ok = code == api.SP_ERR_VERIFY and label in SHAPE_LABELS
    else:
        ok = code == api.SP_ERR_VERIFY and (label == library_label(verdict) or (m.length and label in SHAPE_LABELS))
    return None if ok else "%s: oracle %r, library status %d %r" % (m.name, verdict, code, label)


@pytest.mark.parametrize("name,kind", CASES)
def test_single_verify_gives_the_oracle_verdict(sb, name, kind):
    c = case(sb, name, kind)
    bad = [x for x in (mismatch(c.api, m, v, *r) for m, v, r in zip(c.mutants, c.verdicts, c.results)) if x]
    assert not bad, "%d of %d mutants:\n" % (len(bad), len(c.mutants)) + "\n".join(bad[:30])
    assert c.single(Mutant("valid", "", "", c.good)) == (c.api.SP_OK, None)


@pytest.mark.parametrize("name,kind", CASES)
def test_batch_statuses_equal_the_single_calls(sb, name, kind):
    """every mutant in one batch, after every third a valid proof, and the first mutant again at the end"""
    c = case(sb, name, kind)
    valid = Mutant("valid", "", "", c.good)
    batch, want = [], []
    for j, (m, r) in enumerate(zip(c.mutants, c.results)):
        batch.append(m)
        want.append(r[0])
        if j % 3 == 2:
            batch.append(valid)
            want.append(c.api.SP_OK)
    batch.append(c.mutants[0])
    want.append(c.results[0][0])
    got = c.P.verify_batch([c.P(m.data) for m in batch], [c.statement(m) for m in batch], [c.inputs] * len(batch), LABEL, c.gens)
    codes = [c.api.SP_OK if g is None else g.code for g in got]
    bad = ["%s: batch %d, single %d" % (m.name, g, w) for m, g, w in zip(batch, codes, want) if g != w]
    assert not bad, "\n".join(bad[:30])


@pytest.mark.parametrize("name,kind", CASES)
def test_batch_of_one_equation_mutants(sb, name, kind):
    """only mutants that each make one group equation false and change no challenge: each must be rejected by the device pass of the
    batch and then by the re-run, as by the single call"""
    c = case(sb, name, kind)
    sel = [(m, r) for m, r in zip(c.mutants, c.results) if m.comm is None and re.fullmatch(ONE_EQUATION, m.name)]
    assert len(sel) >= 8
    assert all(r[0] == c.api.SP_ERR_VERIFY for _, r in sel)
    got = c.P.verify_batch([c.P(m.data) for m, _ in sel], c.stmt, [c.inputs] * len(sel), LABEL, c.gens)
    assert [g is not None and g.code == c.api.SP_ERR_VERIFY for g in got] == [True] * len(sel), [m.name for (m, _), g in zip(sel, got) if g is None]


def test_every_check_is_reached(sb):
    """the labels the mutants produced are every check verifier.cpp names, except those no parsed proof reaches; and each divergence
    from the reference was met"""
    labels, names = set(), set()
    for name, kind in CASES:
        c = case(sb, name, kind)
        labels |= {check_name(r[1]) for r in c.results if r[0] == c.api.SP_ERR_VERIFY}
        names |= {m.name for m in c.mutants}
    assert labels <= LIBRARY_CHECKS, labels - LIBRARY_CHECKS
    assert set(UNREACHABLE) <= LIBRARY_CHECKS
    assert labels == LIBRARY_CHECKS - set(UNREACHABLE), ("not reached", LIBRARY_CHECKS - set(UNREACHABLE) - labels)
    for pat, _, _ in DIVERGENCES:
        assert any(re.fullmatch(pat, n) for n in names), pat


_DEFERRED_ONLY = r'''
import sys
sys.path.insert(0, sys.argv[1])
import spartan_b200 as sb
ctx = sb.default_context()
for nc, nv, ni in ((2, 2, 1), (32, 32, 4)):
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(nc, nv, ni, seed=1)
    sg = sb.SNARKGens(nc, nv, ni, nc)
    comm = sb.SNARK.encode(inst, sg)
    ng = sb.NIZKGens(nc, nv, ni)
    ps = [sb.SNARK.prove(inst, comm, vars_, inputs, sg, b"t", sb.tape_seed(j)) for j in range(2)]
    ns = [sb.NIZK.prove(inst, vars_, inputs, ng, b"t", sb.tape_seed(j)) for j in range(2)]
    ctx.timings()
    assert sb.SNARK.verify_batch(ps, comm, [inputs] * 2, b"t", sg) == [None] * 2
    assert sb.NIZK.verify_batch(ns, inst, [inputs] * 2, b"t", ng) == [None] * 2
    t = ctx.timings()
    assert "fine:batch.final" in t and "fine:batch.rerun" not in t, (nc, t)
print("ok")
'''


def test_valid_proofs_pass_the_device_pass(sb):
    """at the two shapes that only these tests use (an IPA of lg n = 1, a device C_LZ), valid proofs are accepted by the deferred pass itself
    and not by the re-run a rejected proof gets: a deferred equation whose two sides do not cancel fails here, though the statuses stay right.
    A process of its own: SP_FINE_TIMERS=1 is read once."""
    env = dict(os.environ, SP_FINE_TIMERS="1")
    r = subprocess.run([sys.executable, "-c", _DEFERRED_ONLY, ROOT], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
