"""The memory-check mode (sp_debug_memcheck, spd_memcheck): every device block filled when it is handed out and guarded past its end, the
contexts' persistent scratch refilled at every call.  Under it, a kernel or proof that reads memory it did not write this call gets 0xFF field
elements or zero integers instead of the previous owner's (usually right) values, and a write past a buffer's end lands in a zero guard band that
is checked at free and by the scan.

  a. the mechanism on its own (spd_pool_selftest) and the per-call refill of a context's scratch;
  b. the oracle and golden comparisons of the GPU suite, rerun under the mode in a subprocess (tests/memcheck_plugin.py);
  c. one context through a sequence of changing shapes and entry points, each result against the fixtures or the oracle.

Run on the GPU: pytest -m gpu."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from oracle.spartan_ref import r1cs, spark

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def sb():
    import spartan_b200 as m
    return m


@pytest.fixture
def memcheck(sb):
    """the library's mode on for one test of this process, and off again after it (the rest of the suite runs without it)"""
    sb.debug_memcheck(True)
    try:
        yield sb
    finally:
        sb.debug_memcheck(False)


def counts(sb):
    return sb.debug_memcheck_report()


# ---------------------------------------------------------------------------------------------------- a. the mechanism
def test_pool_selftest():
    """through dev::pool_alloc of libsp_devtest.so's pool: fresh and reused u256 blocks read all 0xFF and a raw one zero, a byte written past the
    request (cudaMemset, inside the guard) is reported by the scan and at free, blocks from before the switch are not reused under it, and
    switching off restores the plain rounding"""
    lib = C.CDLL(os.path.join(ROOT, "spartan_b200", "libsp_devtest.so"))
    lib.spd_last_error.restype = C.c_char_p
    buf = C.create_string_buffer(4096)
    rc = lib.spd_pool_selftest(buf, C.c_size_t(len(buf)))
    assert rc == 0, lib.spd_last_error().decode()
    scan_msg, free_msg = buf.value.decode().split("\n")
    assert "1000 bytes requested, field elements / points" in scan_msg and "offset 1007 (7 bytes past the end)" in scan_msg, scan_msg
    assert "1000 bytes requested, raw / integer" in free_msg and "offset 1000 (0 bytes past the end)" in free_msg, free_msg


def test_context_scratch_refilled_every_call(memcheck):
    """two calls of each kind on one context see refilled scratch and small (the counters say so) and still give the oracle's values"""
    sb = memcheck
    before = counts(sb)
    ctx = sb.Context()
    n = 1 << 12
    a, b = oc.prg_scalars("memcheck-a", n, 1), oc.prg_scalars("memcheck-b", n, 2)
    pa, pb = sb.DensePolynomial(a, ctx), sb.DensePolynomial(b, ctx)
    want = oc.dot3(a, b, oc.to_arr([1] * n))
    r = oc.prg_scalars("memcheck-r", 12, 3)
    want_eval = oc.dot3(a, oc.eq_evals(oc.to_ints(r)), oc.to_arr([1] * n))
    for _ in range(2):
        assert oc.to_ints(pa.dot(pb).reshape(1, 4)) == [want]
        assert oc.to_ints(pa.evaluate(r).reshape(1, 4)) == [want_eval]
    after = counts(sb)
    assert after["context_refills"] - before["context_refills"] >= 6   # two uploads, two dots, two evaluations
    assert after["blocks_filled"] > before["blocks_filled"]
    assert sb.debug_memcheck_scan() == 0
    del pa, pb, ctx
    assert counts(sb)["violations"] == before["violations"], counts(sb)["last_violation"]


# ---------------------------------------------------------------------------------------------------- b. the suite under the mode
SUITE = ["test_gpu_kernels.py", "test_gpu_arith.py", "test_gpu_golden.py", "test_gpu_sumcheck_poly.py", "test_gpu_sumcheck_poly_limits.py",
         "test_gpu_msm_var.py", "test_gpu_msm_var_limits.py", "test_row_msm.py", "test_gpu_msm_instances.py", "test_gpu_verify_batch.py",
         "test_gpu_instance_device.py", "test_gpu_snark.py", "test_gpu_gen_tables.py", "test_gpu_instance_shapes.py"]
DESELECT = {
    # starts one process per MSM window width; those processes run without the mode (the window widths' kernels are each checked in-process by
    # test_msm_rows_every_instance)
    "test_gpu_msm_instances.py::test_snark_bytes_equal_under_every_window": "runs its proofs in subprocesses",
}


def test_suite_under_memcheck(tmp_path):
    out = tmp_path / "memcheck.json"
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "tests"), ROOT] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    env["SP_MEMCHECK_OUT"] = str(out)
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "memcheck_plugin", "-p", "no:cacheprovider", "--durations=15"]
    cmd += [os.path.join(ROOT, "tests", f) for f in SUITE]
    for nodeid in DESELECT:
        cmd += ["--deselect", os.path.join(ROOT, "tests", nodeid)]
    # its output passes through as it comes (visible with -s: the run takes minutes), the end of it goes into the failure message
    p = subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    lines = []
    for line in p.stdout:
        sys.stdout.write(line)
        sys.stdout.flush()
        lines = (lines + [line])[-200:]
    rc = p.wait()
    tail = "".join(lines)
    assert rc == 0, tail
    tot = json.load(open(out))
    assert tot["violations"] == 0, tot
    for k in ("blocks_filled", "blocks_refilled", "context_refills", "guard_bytes_checked"):
        assert tot[k] > 0, tot


# ---------------------------------------------------------------------------------------------------- c. one context, changing shapes
def test_one_context_changing_shapes(memcheck):
    """SNARK 2^16, NIZK 2^10, msm_var 2^18, sumcheck_prove, SNARK 2^12, SNARK 2^16 again, then batch verification of the proofs, all on one
    context under the mode: what each step leaves in the context's scratch and in the pool must not change the next one's result"""
    sb = memcheck
    from test_gpu_sumcheck_poly import comp_of, transcripts
    from oracle.spartan_ref import protocol as pr
    fx = json.load(open(os.path.join(GOLDEN, "snark_proof_sha256.json")))
    gold = json.load(open(os.path.join(GOLDEN, "oracle_golden.json")))
    v0 = counts(sb)["violations"]
    ctx = sb.Context()

    def scanned(what):
        assert sb.debug_memcheck_scan() == 0 and counts(sb)["violations"] == v0, "%s: %s" % (what, counts(sb)["last_violation"])

    def snark(logn):
        n = 1 << logn
        inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=0, ctx=ctx)
        gens = sb.SNARKGens(n, n, 10, n, ctx=ctx)
        comm = sb.SNARK.encode(inst, gens)
        proof = sb.SNARK.prove(inst, comm, vars_, inputs, gens, b"example", sb.tape_seed(0))
        return inst, inputs, gens, comm, proof

    s16 = snark(16)
    assert hashlib.sha256(s16[3].commitment_bytes()).hexdigest() == fx["16_commitment"]
    assert hashlib.sha256(s16[4].bytes).hexdigest() == fx["16"]
    scanned("SNARK 2^16")

    case = next(c for c in gold["nizk"] if c["num_cons"] == 1024)
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(case["num_cons"], case["num_vars"], case["num_inputs"], seed=case["seed"], ctx=ctx)
    inst.set_digest(case["digest"].encode())
    ngens = sb.NIZKGens(case["num_cons"], case["num_vars"], case["num_inputs"], ctx=ctx)
    label = gold["transcript_labels"]["nizk"].encode()
    nproof = sb.NIZK.prove(inst, vars_, inputs, ngens, label, sb.tape_seed(case["seed"]))
    assert len(nproof.bytes) == case["proof"]["len"] and hashlib.sha256(nproof.bytes).hexdigest() == case["proof"]["sha256"]
    scanned("NIZK 2^10")

    m = 1 << 18
    P = sb.api.Points.derive(m, b"msm-large", ctx)
    t = oc.prg_scalars("msm", m, 2)
    assert P.msm(t) == oc.msm(t, oc.MultiCommitGens.new(m, b"msm-large").G).compress()
    scanned("msm_var 2^18")

    k = 12
    tabs = [oc.prg_scalars("memcheck-sc%d" % i, 1 << k, i) for i in range(3)]
    claim = oc.dot3(*tabs)
    ot, st = transcripts(sb)
    oproof, orr, claims, _ = pr.prove_cubic_batched(claim, k, ([tabs[0].copy()], [tabs[1].copy()], tabs[2].copy()), ([], [], []), [1], ot)
    proof, r, finals, e = sb.sumcheck_prove([sb.DensePolynomial(x, ctx) for x in tabs], comp_of(sb, [(1, (0, 1, 2))]), oc.to_arr([claim])[0], k, st)
    assert proof == pr.ser(oproof) and oc.to_ints(r) == list(orr)
    scanned("sumcheck_prove 2^12")

    n = 1 << 12
    oi, ovars, oinputs = r1cs.Instance.produce_synthetic_r1cs(n, n, 10, 0)
    ogens = spark.SNARKGens(n, n, 10, n)
    ocomm, odecomm = spark.SNARK.encode(oi, ogens)
    want12 = spark.SNARK.prove(oi, ocomm, odecomm, ovars, oinputs, ogens, oc.Transcript(b"example"), r1cs.tape_seed(0)).ser()
    s12 = snark(12)
    assert s12[3].commitment_bytes() == ocomm.ser() and s12[4].bytes == want12
    scanned("SNARK 2^12")

    s16b = snark(16)
    assert s16b[4].bytes == s16[4].bytes
    scanned("SNARK 2^16 again")

    assert sb.SNARK.verify_batch([s16[4], s16b[4]], s16[3], [s16[1], s16b[1]], b"example", s16[2]) == [None, None]
    assert sb.SNARK.verify_batch([s12[4]], s12[3], [s12[1]], b"example", s12[2]) == [None]
    assert sb.NIZK.verify_batch([nproof], inst, [inputs], label, ngens) == [None]
    scanned("verify_batch")
