"""CPU-only checks of the drop-in boundary and the N>1 host logic: the C-ABI library loads and exports every symbol include/*.h
declares (no compute calls without a GPU), fails loudly without a device, and the multi-rank plumbing works under gloo (world_size 2)."""
import ctypes as C
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "spartan_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(sp_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    import spartan_b200 as sb
    syms = _declared_symbols()
    assert len(syms) >= 50
    for s in syms:
        assert hasattr(sb.lib, s), "missing export " + s


def test_every_export_cites_the_reference():
    text = open(os.path.join(ROOT, "include", "spartan_b200.h")).read()
    for needle in ["lib.rs:501", "lib.rs:339", "dense_mlpoly.rs:215-223", "sumcheck.rs:625-652", "group.rs:98-117", "dense_mlpoly.rs:148-177", "commitments.rs:15-33"]:
        assert needle in text or needle.split(":")[0] in text


def test_no_cpu_fallback():
    import spartan_b200 as sb
    if sb.lib.sp_device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(sb.SpartanB200Error):
        sb.Context()


def test_host_scalar_helpers_match_oracle():
    """the host-side scalar entry points (no GPU needed) against the oracle"""
    import spartan_b200 as sb
    from oracle.spartan_ref import core as oc
    rng = np.random.default_rng(11)
    for _ in range(50):
        a = int.from_bytes(rng.bytes(32), "little") % oc.Q
        b = int.from_bytes(rng.bytes(32), "little") % oc.Q
        A = sb.scalar_from_bytes(a.to_bytes(32, "little"))
        B = sb.scalar_from_bytes(b.to_bytes(32, "little"))
        assert A.tobytes() == oc.mont_bytes(a)
        out = np.zeros(4, dtype=np.uint64)
        sb.lib.sp_scalar_mul(A.ctypes.data_as(C.c_void_p), B.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
        assert oc.from_mont_bytes(out.tobytes()) == a * b % oc.Q
        assert sb.scalar_to_bytes(A) == a.to_bytes(32, "little")
    with pytest.raises(sb.R1CSError):
        sb.scalar_from_bytes(oc.Q.to_bytes(32, "little"))
    assert np.array_equal(sb.prg_scalars("Z", 5, 3), oc.prg_scalars("Z", 5, 3))


def test_product_does_not_import_oracle():
    """the product path must never route through the oracle"""
    for dirpath, _, files in os.walk(os.path.join(ROOT, "spartan_b200")):
        for f in files:
            if f.endswith((".py", ".cpp", ".cu", ".cuh", ".hpp", ".h")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "liboracle" not in text and "from oracle" not in text and "import oracle" not in text, f


WORKER = textwrap.dedent("""
    import os, sys
    sys.path.insert(0, %r)
    from spartan_b200 import dist as sd
    rank, world, local = sd.init("gloo")
    assert world == 2
    seed = sd.rank_seed(rank, 5)
    assert seed == 5 + rank
    sd.barrier()
    t = sd.max_over_ranks([1.0 + rank, 10.0 - rank])
    assert t == [2.0, 10.0], t
    thr = sd.aggregate_throughput(1 << 20, world, t[0])
    assert abs(thr - 2 * (1 << 20) / 2.0) < 1e-6
    sd.finalize()
    print("rank", rank, "ok")
""")


def test_two_rank_plumbing_under_gloo(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER % ROOT)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT="29533")
    procs = []
    for r in range(2):
        e = dict(env, RANK=str(r), WORLD_SIZE="2", LOCAL_RANK=str(r))
        procs.append(subprocess.Popen([sys.executable, str(script)], env=e, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=120)[0] for p in procs]
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, o
        assert "rank %d ok" % r in o


def test_transcript_state_helpers_match_merlin():
    """sp_transcript_* (the 203-byte STROBE state that crosses the ABI in place of `&mut Transcript`) against the oracle's Merlin, including the
    Merlin conformance vector and long messages that cross the 166-byte rate several times"""
    import spartan_b200 as sb
    from oracle.spartan_ref import core as oc
    t = sb.Transcript(b"test protocol")
    t.append_message(b"some label", b"some data")
    assert t.challenge_bytes(b"challenge", 32).hex() == "d5a21972d0d5fe320c0d263fac7fffb8145aa640af6e9bca177c03c7efcf0615"
    rng = np.random.default_rng(5)
    a, b = sb.Transcript(b"example"), oc.Transcript(b"example")
    for n in [0, 1, 31, 32, 165, 166, 167, 400, 5000]:
        msg = rng.bytes(n)
        a.append_message(b"lbl", msg); b.append_message(b"lbl", msg)
        assert a.challenge_bytes(b"c", 64) == b.challenge_bytes(b"c", 64)
        assert a.challenge_bytes(b"long", 700) == b.challenge_bytes(b"long", 700)
    assert len(a.state.raw) == 203 and a.state.raw[200] < 166

