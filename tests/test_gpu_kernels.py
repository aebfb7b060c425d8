"""The kernels that only whole proofs reach — the batched and eq-factored sumcheck rounds with and without host publication, the eq tables, the
SPARK layer kernels, the sparse products and the sharded table producers — launched one wrapper at a time through libsp_devtest.so (the hooks
link the very kernel objects of libspartan_b200.so) and diffed against the oracle at the shapes the protocol never produces: instance and table
counts up to the caps, lengths that are not powers of two, grids that make several passes, shared tables, every rank of a cyclic partition.
Expected values come from oracle/spartan_ref/core.py or, where it has no such function, plain Python integers mod q."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle.spartan_ref import core as oc
from test_gpu_ops import edge_table  # noqa: E402  (0, 1, q-1, R, R^2, 2, q-2 planted)
from test_shard_model import shard_eq_scale  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q = oc.Q
REFUSED = -1
NT = {0: 2, 1: 3, 2: 4}
_vp, _sz, _i = C.c_void_p, C.c_size_t, C.c_int


def _p(a):
    return None if a is None else a.ctypes.data_as(_vp)


def i32(v):
    return np.ascontiguousarray(np.asarray(v, dtype=np.int32))


def u32(v):
    return np.ascontiguousarray(np.asarray(v, dtype=np.uint32))


def cat(tables):
    return np.ascontiguousarray(np.concatenate(tables)) if tables else oc.zeros(0)


class Kern:
    """ctypes front of the kernel hooks of libsp_devtest.so (spartan_b200/csrc/devtest.cu)"""
    SIGS = dict(
        spd_sc_chain=[_i, _i, _sz, _i] + [_vp] * 4 + [_i, _vp, _i] + [_vp] * 7,
        spd_sc_g_chain=[_i, _sz, _vp, _vp, _vp, _i, _vp, _i] + [_vp] * 4,
        spd_eq_suffix=[_sz, _i, _vp, _vp], spd_eq_evals=[_i, _vp, _vp], spd_eq_extend_top=[_sz, _vp, _vp, _vp],
        spd_heads=[_i, _sz, _vp, _i, _vp, _vp, _vp], spd_fold_top=[_i, _sz, _vp, _vp],
        spd_spark_hash=[_sz] + [_vp] * 3 + [_i, _vp, _vp], spd_spark_hash_cyclic=[_sz, _i, _i] + [_vp] * 3 + [_i, _vp, _vp],
        spd_hadamard_many=[_i, _sz, _vp, _vp, _vp], spd_gather=[_sz, _vp, _sz, _vp, _vp], spd_dot3=[_sz] + [_vp] * 4,
        spd_dot_many=[_i, _sz, _vp, _vp, _vp], spd_lincomb3=[_sz] + [_vp] * 5, spd_bound_rows=[_sz, _sz, _vp, _vp, _vp],
        spd_to_canonical=[_sz, _vp, _vp], spd_spmv=[_sz, _sz, _vp, _vp, _vp, _sz, _vp, _vp],
        spd_spmv_cyclic=[_sz, _i, _i, _sz, _vp, _vp, _vp, _sz, _vp, _vp], spd_sparse_eval3=[_sz, _vp, _vp, _vp, _sz, _vp, _sz, _vp, _vp],
        spd_scale=[_sz, _vp, _vp], spd_take_cyclic=[_sz, _vp, _i, _i, _vp], spd_prof_enable=[_i], spd_prof_report=[C.c_char_p, _sz])

    def __init__(self, lib):
        self.lib = lib
        for name, args in self.SIGS.items():
            getattr(lib, name).argtypes = args
        lib.spd_last_error.restype = C.c_char_p
        lib.spd_launch_count.restype = C.c_ulonglong
        lib.spd_prof_report.restype = _sz

    def call(self, name, *args):
        rc = getattr(self.lib, name)(*args)
        assert rc == 0, "%s: error %d (%s)" % (name, rc, self.lib.spd_last_error().decode())

    def refused(self, name, *args):
        """the wrapper throws before it launches anything; the hook reports it as REFUSED"""
        before = self.launches()
        rc = getattr(self.lib, name)(*args)
        assert rc == REFUSED, "%s: expected a refusal, got %d" % (name, rc)
        return self.lib.spd_last_error().decode(), self.launches() - before

    def launches(self):
        return self.lib.spd_launch_count()

    def profiled(self, fn):
        """kernel family -> launches while fn() runs (the library's own CUDA-event profiler)"""
        self.lib.spd_prof_enable(1)
        try:
            fn()
            buf = C.create_string_buffer(1 << 16)
            self.lib.spd_prof_report(buf, len(buf))
        finally:
            self.lib.spd_prof_enable(0)
        fams = {}
        for rec in buf.value.decode().split(";"):
            if rec:
                name, launches = rec.split(":")[:2]
                fams[name] = int(launches)
        return fams


@pytest.fixture(scope="module")
def kern():
    path = os.path.join(ROOT, "spartan_b200", "libsp_devtest.so")
    assert os.path.exists(path), "libsp_devtest.so is not built: run __graft_entry__.build()"
    return Kern(C.CDLL(path))


def scalars(tag, n, seed=0):
    return oc.to_ints(oc.prg_scalars(tag, n, seed))


# ---------------------------------------------------------------------------------------------------- batched sumcheck rounds
class ScLayout:
    """the buffers of a batched sumcheck: A, B (, D) per instance; C private (i % 3 == 2) or shared by the instances i % 3 == g, whose first
    member folds it into a second buffer of the group (the prover's poly_C_par ping-pong)"""

    def __init__(self, kind, ninst, n, tag, tables=None, private=False):
        """tables(t, i): table t (0 = A, 1 = B, 2 = C, 3 = D) of instance i (private C) or of group i (shared C); default: edge tables"""
        self.kind, self.ninst, self.n = kind, ninst, n
        nt = NT[kind]
        self.bufs, self.groups = [], {}
        self.map = -np.ones((ninst, 4), dtype=np.int32)
        self.cbuf = -np.ones(ninst, dtype=np.int32)
        self.write_c = np.zeros(ninst, dtype=np.int32)
        mk = tables or (lambda t, i: edge_table(n, "%s%s%d" % (tag, "abcd"[t] if t != 2 or private or i % 3 == 2 else "s", i)))
        for i in range(ninst):
            self.map[i, 0] = self.add(mk(0, i))
            self.map[i, 1] = self.add(mk(1, i))
            if nt == 4:
                self.map[i, 3] = self.add(mk(3, i))
            if nt >= 3:
                g = 2 if private else i % 3
                if g == 2:
                    self.map[i, 2] = self.cbuf[i] = self.add(mk(2, i))
                    self.write_c[i] = 1
                else:
                    if g not in self.groups:
                        self.groups[g] = (self.add(mk(2, g)), self.add(oc.zeros(n)))
                        self.cbuf[i] = self.groups[g][1]
                        self.write_c[i] = 1
                    self.map[i, 2] = self.groups[g][0]

    def add(self, t):
        self.bufs.append(np.ascontiguousarray(t))
        return len(self.bufs) - 1

    def run(self, kern, rs, use_sig=True, bound=True):
        ninst, nf = self.ninst, len(rs)
        res = dict(out=oc.zeros(3 * ninst * (nf + 1)), host_out=oc.zeros(3 * ninst * (nf + 1)), flags=np.zeros(nf + 1, np.uint32),
                   dones=np.full(nf + 1, 0xdead, np.uint32), bound=oc.zeros(2 * NT[self.kind] * ninst), tables=oc.zeros(len(self.bufs) * self.n),
                   counters=np.full(64, 0xdead, np.uint32))
        kern.call("spd_sc_chain", self.kind, ninst, self.n, len(self.bufs), _p(cat(self.bufs)), _p(i32(self.map)), _p(i32(self.cbuf)),
                  _p(i32(self.write_c)), nf, _p(oc.to_arr(rs) if nf else oc.zeros(1)), int(use_sig), _p(res["out"]), _p(res["host_out"]),
                  _p(res["flags"]), _p(res["dones"]), _p(res["bound"]) if bound and use_sig else None, _p(res["tables"]), _p(res["counters"]))
        res["tables"] = res["tables"].reshape(len(self.bufs), self.n, 4)
        return res


def oracle_eval(kind, ts):
    if kind == 0:
        return oc.sc_eval_quad(ts[0], ts[1]) + [0]
    return oc.sc_eval_cubic(ts[0], ts[1], ts[2], ts[3] if kind == 2 else None)


def round_scalars(tag, nf):
    """the binding challenges, with 0, 1 and q-1 among them"""
    rs = scalars(tag, nf, nf)
    for k, v in zip(range(1, nf, 3), [Q - 1, 1, 0]):
        rs[k] = v
    return rs


def check_chain(lay, rs, res, use_sig):
    """every round's evaluations, the publication, the bound tables, and the shared C where the last round read it"""
    kind, ninst, nt = lay.kind, lay.ninst, NT[lay.kind]
    cur = {b: t.copy() for b, t in enumerate(lay.bufs)}
    prev = None
    for k in range(len(rs) + 1):
        if k:
            prev = {b: t.copy() for b, t in cur.items()}
            cur = {b: oc.bound_top(t.copy(), rs[k - 1]) for b, t in cur.items()}
        got = oc.to_ints(res["out"][3 * ninst * k:3 * ninst * (k + 1)])
        for i in range(ninst):
            assert got[3 * i:3 * i + 3] == oracle_eval(kind, [cur[lay.map[i, t]] for t in range(nt)]), "round %d, instance %d" % (k, i)
        if use_sig:
            assert np.array_equal(res["host_out"][3 * ninst * k:3 * ninst * (k + 1)], res["out"][3 * ninst * k:3 * ninst * (k + 1)]), "round %d" % k
            assert res["flags"][k] == k + 1, "round %d: flag %d" % (k, res["flags"][k])
            assert res["dones"][k] == 0, "round %d: completion counter left at %d" % (k, res["dones"][k])
    assert not res["counters"].any(), "ticket counters not reset: %s" % res["counters"][:ninst]
    m = len(cur[0])
    for i in range(ninst):
        for t in [t for t in range(nt) if t != 2]:
            b = lay.map[i, t]
            assert np.array_equal(res["tables"][b][:m], cur[b]), "instance %d table %d" % (i, t)
        if nt >= 3 and lay.write_c[i] and lay.cbuf[i] == lay.map[i, 2]:
            assert np.array_equal(res["tables"][lay.map[i, 2]][:m], cur[lay.map[i, 2]]), "private C of instance %d" % i
    for g, (ping, pong) in lay.groups.items():
        now, other = (pong, ping) if len(rs) % 2 else (ping, pong)
        assert np.array_equal(res["tables"][now][:m], cur[ping]), "shared C %d" % g
        if rs:
            assert np.array_equal(res["tables"][other][:2 * m], prev[ping]), "shared C %d: the last round wrote the buffer it read" % g
    if use_sig and m == 2 and rs:
        bound = oc.to_ints(res["bound"])
        for i in range(ninst):
            for t in range(nt):
                assert bound[2 * nt * i + 2 * t:2 * nt * i + 2 * t + 2] == oc.to_ints(cur[lay.map[i, t]]), "host_bound instance %d table %d" % (i, t)


SC_CASES = [(kind, ninst, logn, True) for kind in (0, 1, 2) for ninst in (1, 12, 18, 24) for logn in (12, 13)] + \
           [(kind, 12, 13, False) for kind in (0, 1, 2)]


@pytest.mark.parametrize("kind,ninst,logn,use_sig", SC_CASES)
def test_sc_batched_chain(kern, kind, ninst, logn, use_sig):
    """k_sc_eval, k_sc_fold_eval and k_sc_fold_eval_small with 1 .. SC_MAX_INST instances and a C shared by several of them (one instance folds it
    into the other ping-pong buffer, the others only read it): the whole chain of rounds down to two-entry tables, on both sides of the
    small / streaming switch (len/4 = 1024 vs 2048).  Signalled: every launch's host_out equals out, the flag holds this launch's sequence number,
    the completion counter `done` (gridDim.y = ninst > 1) is back to 0, the ticket counters are zero, and the fold to two-entry tables publishes
    the bound tables (host_bound).  The profiler shows which kernel family ran each fold."""
    n = 1 << logn
    lay = ScLayout(kind, ninst, n, "sc%d_%d_%d" % (kind, ninst, logn))
    rs = round_scalars("scr%d" % logn, logn - 1)
    res = {}
    fams = kern.profiled(lambda: res.update(lay.run(kern, rs, use_sig)))
    check_chain(lay, rs, res, use_sig)
    assert fams.get("sc_eval") == 1
    assert fams.get("sc_fold_eval", 0) == (1 if logn == 13 else 0)       # the streaming kernel: len/4 > 1024
    assert fams.get("sc_fold_eval_small") == logn - 1 - fams.get("sc_fold_eval", 0)


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_sc_batched_chain_multipass(kern, kind):
    """len 2^20: the capped grid of k_sc_eval / k_sc_fold_eval makes several passes per thread; four instances, two of them sharing C, then the
    small-table tail"""
    n = 1 << 20
    lay = ScLayout(kind, 4, n, "scbig%d" % kind)
    rs = round_scalars("scbigr", 19)
    check_chain(lay, rs, lay.run(kern, rs), True)


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_sc_shared_c_untouched(kern, kind):
    """one fold: instance 0 writes the folded shared C to its own buffer, the C every other instance reads stays byte for byte as it was"""
    n = 1 << 13
    lay = ScLayout(kind, 12, n, "scu%d" % kind)
    rs = [scalars("scur", 1)[0]]
    res = lay.run(kern, rs)
    check_chain(lay, rs, res, True)
    for g, (ping, pong) in lay.groups.items():
        assert np.array_equal(res["tables"][ping], lay.bufs[ping])
        assert np.array_equal(res["tables"][pong][:n // 2], oc.bound_top(lay.bufs[ping].copy(), rs[0]))


def test_sc_batch_refusals(kern):
    """25 instances (SC_MAX_INST = 24) are refused before any launch; host_bound without a HostSig is refused too"""
    lay = ScLayout(1, 25, 16, "sc25")
    args = lambda nf, sig, bound: (1, 25, 16, len(lay.bufs), _p(cat(lay.bufs)), _p(i32(lay.map)), _p(i32(lay.cbuf)), _p(i32(lay.write_c)), nf,  # noqa: E731
                                   _p(oc.to_arr([5] * 3)), sig, _p(oc.zeros(300)), _p(oc.zeros(300)), _p(np.zeros(4, np.uint32)),
                                   _p(np.zeros(4, np.uint32)), _p(oc.zeros(200)) if bound else None, _p(oc.zeros(len(lay.bufs) * 16)),
                                   _p(np.zeros(64, np.uint32)))
    msg, launched = kern.refused("spd_sc_chain", *args(2, 1, False))
    assert "too many" in msg and launched == 0
    small = ScLayout(1, 2, 4, "scb")
    rc = kern.lib.spd_sc_chain(1, 2, 4, len(small.bufs), _p(cat(small.bufs)), _p(i32(small.map)), _p(i32(small.cbuf)), _p(i32(small.write_c)), 1,
                               _p(oc.to_arr([3])), 0, _p(oc.zeros(12)), _p(oc.zeros(12)), _p(np.zeros(2, np.uint32)), _p(np.zeros(2, np.uint32)),
                               _p(oc.zeros(12)), _p(oc.zeros(len(small.bufs) * 4)), _p(np.zeros(64, np.uint32)))
    assert rc == REFUSED and "signalled" in kern.lib.spd_last_error().decode()


@pytest.mark.parametrize("logn", [2, 3])
def test_sc_host_bound_len4(kern, logn):
    """k_sc_fold_eval_small with host_bound at len 4: the published two-entry tables equal the bound tables, for every kind"""
    for kind in (0, 1, 2):
        lay = ScLayout(kind, 5, 1 << logn, "hb%d_%d" % (kind, logn))
        rs = scalars("hbr", logn - 1, kind)
        check_chain(lay, rs, lay.run(kern, rs), True)


@pytest.mark.parametrize("ninst,ntab", [(1, 1), (64, 64), (65, 65)])
def test_fold_top(kern, ninst, ntab):
    """k_fold_top over more than the 64 tables of one launch (several launches), at an odd multiple of the grid"""
    n = 2 * 777
    tabs = [edge_table(n, "ft%d_%d" % (ntab, k)) for k in range(ntab)]
    r = scalars("ftr", 1, ntab)[0]
    buf = cat(tabs)
    kern.call("spd_fold_top", ntab, n, _p(buf), _p(oc.to_arr([r])))
    buf = buf.reshape(ntab, n, 4)
    for k, t in enumerate(tabs):
        assert np.array_equal(buf[k][:n // 2], oc.bound_top(t.copy(), r)), k


# ---------------------------------------------------------------------------------------------------- eq-factored rounds
def run_g_chain(kern, ninst, logn, jG, use_sig, tag):
    n = 1 << logn
    tau = scalars(tag + "tau", logn, logn)
    A = [edge_table(n, "%sa%d" % (tag, i)) for i in range(ninst)]
    B = [edge_table(n, "%sb%d" % (tag, i)) for i in range(ninst)]
    rs = round_scalars(tag + "r", logn - 1)
    a, b = cat(A), cat(B)
    out, host_out = oc.zeros(3 * ninst * logn), oc.zeros(3 * ninst * logn)
    flags, dones = np.zeros(logn, np.uint32), np.full(logn, 0xdead, np.uint32)
    E0 = np.ascontiguousarray(oc.eq_evals(tau[1:]))
    args = (ninst, n, _p(a), _p(b), _p(E0), jG, _p(oc.to_arr(rs)), int(use_sig), _p(out), _p(host_out), _p(flags), _p(dones))
    return tau, A, B, rs, a.reshape(ninst, n, 4), b.reshape(ninst, n, 4), out, host_out, flags, dones, args


def diff(hi, lo):
    return oc.lincomb3(hi, lo, lo, 1, Q - 1, 0)


G_CASES = [(1, 15, 1, True), (12, 15, 2, True), (12, 15, 4, True), (1, 16, 3, False), (12, 16, 5, True), (2, 18, 7, True),
           (1, 20, 1, True), (1, 20, 2, True), (2, 20, 9, True)]


@pytest.mark.parametrize("ninst,logn,jG,use_sig", G_CASES)
def test_sc_g_chain(kern, ninst, logn, jG, use_sig):
    """k_eq_suffix, k_sc_eval_g and k_sc_fold_eval_g for rounds 0 .. jG-1, the switch (k_fold_top, then k_sc_eval on the last suffix level with
    instance 0 folding the shared C), then the standard rounds to two-entry tables, as batched_prove runs them.  In every eq-factored round q(0)
    and q(inf) equal sum E.A.B and sum E.dA.dB over the reference tables, and s_j(0), s_j(2), s_j(3), rebuilt from them exactly as batched_prove
    does (q(1) from the running claim, the prefix, eq(tau_j, t)), equal sc_eval_cubic on the reference tables with C = eq(tau); after the switch
    the standard evaluations times the prefix equal it too."""
    tau, A, B, rs, a, b, out, host_out, flags, dones, args = run_g_chain(kern, ninst, logn, jG, use_sig, "g%d_%d_%d" % (ninst, logn, jG))
    kern.call("spd_sc_g_chain", *args)
    Cq = oc.eq_evals(tau)
    claim = [oc.dot3(Cq, A[i], B[i]) for i in range(ninst)]
    prefix = 1
    curA, curB, curC = [t.copy() for t in A], [t.copy() for t in B], Cq.copy()
    for j in range(logn):
        if j:
            curA = [oc.bound_top(t.copy(), rs[j - 1]) for t in curA]
            curB = [oc.bound_top(t.copy(), rs[j - 1]) for t in curB]
            curC = oc.bound_top(curC.copy(), rs[j - 1])
        got = oc.to_ints(out[3 * ninst * j:3 * ninst * (j + 1)])
        if use_sig:
            assert np.array_equal(host_out[3 * ninst * j:3 * ninst * (j + 1)], out[3 * ninst * j:3 * ninst * (j + 1)]), j
            assert flags[j] == j + 1 and dones[j] == 0, (j, flags[j], dones[j])
        h = len(curA[0]) // 2
        Ej = oc.eq_evals(tau[j + 1:]) if j < jG else None
        t = tau[j]
        for i in range(ninst):
            want = oc.sc_eval_cubic(curA[i], curB[i], curC)
            if j < jG:
                q0, qinf = got[3 * i], got[3 * i + 1]
                assert q0 == oc.dot3(Ej, curA[i][:h], curB[i][:h]), "round %d instance %d: q(0)" % (j, i)
                assert qinf == oc.dot3(Ej, diff(curA[i][h:], curA[i][:h]), diff(curB[i][h:], curB[i][:h])), "round %d instance %d: q(inf)" % (j, i)
                q1 = (claim[i] - (1 - t) * q0) * oc.inv(t) % Q
                qb = (q1 - q0 - qinf) % Q
                q = lambda x: ((qinf * x + qb) * x + q0) % Q  # noqa: E731
                s = [prefix * ((1 - t) + x * (2 * t - 1)) % Q * q(x) % Q for x in (0, 2, 3)]
                assert s == want, "round %d instance %d: s_j" % (j, i)
                claim[i] = q(rs[j])
            else:
                assert [prefix * e % Q for e in got[3 * i:3 * i + 3]] == want, "round %d instance %d (standard)" % (j, i)
        if j < jG:
            prefix = prefix * ((1 - t) + rs[j] * (2 * t - 1)) % Q
    for i in range(ninst):
        assert np.array_equal(a[i][:2], curA[i]) and np.array_equal(b[i][:2], curB[i]), i


def test_sc_fold_eval_g_refuses_small_tables(kern):
    """sc_fold_eval_g is a streaming kernel: a launch at len/4 <= 1024 (len 4096) is refused; at 8192 it runs"""
    *_, args = run_g_chain(kern, 1, 12, 2, True, "gs")
    msg, launched = kern.refused("spd_sc_g_chain", *args)
    assert "streaming" in msg and launched == 2          # k_eq_suffix and round 0's k_sc_eval_g ran, the fold was refused
    *_, args = run_g_chain(kern, 1, 13, 2, True, "gs")
    kern.call("spd_sc_g_chain", *args)


@pytest.mark.parametrize("logn0,K", [(1, 1), (5, 3), (10, 9), (14, 1), (17, 8), (19, 12)])
def test_eq_suffix(kern, logn0, K):
    """k_eq_suffix: level k (1..K) = eq(tau[k+1..], .) from E0 = eq(tau[1..], .) of n0 = 2^logn0 entries"""
    tau = scalars("suf", logn0 + 1, logn0)
    n0 = 1 << logn0
    E0 = np.ascontiguousarray(oc.eq_evals(tau[1:]))
    levels = oc.zeros(sum(n0 >> k for k in range(1, K + 1)))
    kern.call("spd_eq_suffix", n0, K, _p(E0), _p(levels))
    off = 0
    for k in range(1, K + 1):
        assert np.array_equal(levels[off:off + (n0 >> k)], oc.eq_evals(tau[k + 1:])), k
        off += n0 >> k


# ---------------------------------------------------------------------------------------------------- eq tables and heads
@pytest.mark.parametrize("ell", [0, 1, 2, 7, 10, 11, 12, 17, 20])
def test_eq_evals(kern, ell):
    """k_eq_small alone (ell <= 10) and the two-level k_eq_small + k_eq_combine for odd and even ell > 10; r holds 0, 1 and q-1"""
    r = scalars("eqk", ell, ell)
    for k, v in zip(range(ell), [0, 1, Q - 1]):
        r[(3 * k + 1) % ell] = v
    out = oc.zeros(1 << ell)
    kern.call("spd_eq_evals", ell, _p(oc.to_arr(r) if ell else oc.zeros(1)), _p(out))
    assert np.array_equal(out, oc.eq_evals(r))


@pytest.mark.parametrize("n", [1, 257, 2 * 1056 * 256 + 17])
@pytest.mark.parametrize("r", [0, 1, Q - 1, "random"])
def test_eq_extend_top(kern, n, r):
    """k_eq_extend_top: [(1 - r) E | r E] from E, r in {0, 1, q-1, random}, n not a multiple of the grid (the last n several passes deep)"""
    r = scalars("ext", 1, n)[0] if r == "random" else r
    E = edge_table(n, "ext%d" % n)
    out = oc.zeros(2 * n)
    kern.call("spd_eq_extend_top", n, _p(E), _p(oc.to_arr([r])), _p(out))
    e = oc.to_ints(E)
    assert np.array_equal(out, oc.to_arr([(1 - r) * x % Q for x in e] + [r * x % Q for x in e]))


@pytest.mark.parametrize("count", [1, 63, 64])
@pytest.mark.parametrize("use_sig", [False, True])
def test_heads(kern, count, use_sig):
    """k_heads: the first entry of up to 64 tables, and with a HostSig the published copy and the flag"""
    tabs = [oc.prg_scalars("hd%d" % k, 3) for k in range(count)]
    for k, v in zip(range(0, count, 2), [0, 1, Q - 1, oc.R_MONT]):
        tabs[k][0] = oc.to_arr([v])[0]
    out, host_out, flag = oc.zeros(count), oc.zeros(count), np.zeros(1, np.uint32)
    kern.call("spd_heads", count, 3, _p(cat(tabs)), int(use_sig), _p(out), _p(host_out), _p(flag))
    assert np.array_equal(out, np.stack([t[0] for t in tabs]))
    if use_sig:
        assert np.array_equal(host_out, out) and flag[0] == 7


def test_heads_refuses_65(kern):
    tabs = cat([edge_table(1, "h65_%d" % k) for k in range(65)])
    msg, launched = kern.refused("spd_heads", 65, 1, _p(tabs), 1, _p(oc.zeros(65)), _p(oc.zeros(65)), _p(np.zeros(1, np.uint32)))
    assert "64" in msg and launched == 0


# ---------------------------------------------------------------------------------------------------- SPARK layer kernels
@pytest.mark.parametrize("with_addr", [True, False])
@pytest.mark.parametrize("with_ts", [True, False])
@pytest.mark.parametrize("plus_one", [0, 1])
def test_spark_hash(kern, with_addr, with_ts, plus_one):
    """k_spark_hash in all forms: out = ts r^2 + val r + addr - g, addr the index when null, ts zero when null, plus one when asked"""
    n = 777
    addr = edge_table(n, "sha") if with_addr else None
    ts = edge_table(n, "sht") if with_ts else None
    val = edge_table(n, "shv")
    r, g = scalars("shrg", 2)
    out = oc.zeros(n)
    kern.call("spd_spark_hash", n, _p(addr), _p(val), _p(ts), plus_one, _p(oc.to_arr([r, g])), _p(out))
    a = oc.to_ints(addr) if with_addr else list(range(n))
    t = oc.to_ints(ts) if with_ts else [0] * n
    want = [((ti + plus_one) * r * r + v * r + ai - g) % Q for ai, ti, v in zip(a, t, oc.to_ints(val))]
    assert oc.to_ints(out) == want


@pytest.mark.parametrize("count", [1, 16])
def test_hadamard_many(kern, count):
    """k_hadamard_many with 1 and 16 circuits at an odd length"""
    n = 1001
    a = [edge_table(n, "hma%d" % k) for k in range(count)]
    b = [edge_table(n, "hmb%d" % k) for k in range(count)]
    out = oc.zeros(count * n)
    kern.call("spd_hadamard_many", count, n, _p(cat(a)), _p(cat(b)), _p(out))
    assert np.array_equal(out, cat([oc.hadamard(x, y) for x, y in zip(a, b)]))


def test_hadamard_many_refuses_17(kern):
    t = cat([edge_table(3, "h17")] * 17)
    msg, launched = kern.refused("spd_hadamard_many", 17, 3, _p(t), _p(t), _p(oc.zeros(51)))
    assert "16" in msg and launched == 0


def test_gather(kern):
    """k_gather with indices 0 and cells-1, repeats, over a grid several passes deep"""
    cells = 4099
    mem = edge_table(cells, "gm")
    rng = np.random.default_rng(11)
    idx = rng.integers(0, cells, 300007).astype(np.uint32)
    idx[:6] = [0, cells - 1, 0, 0, cells - 1, 5]
    out = oc.zeros(len(idx))
    kern.call("spd_gather", cells, _p(mem), len(idx), _p(u32(idx)), _p(out))
    assert np.array_equal(out, mem[idx])


def big_table(n, tag):
    """an edge table of n entries without deriving n scalars: a seeded block repeated, edges planted at both ends"""
    base = edge_table(min(n, 65537), tag)
    t = np.ascontiguousarray(np.resize(base, (n, 4)))
    t[-1] = oc.to_arr([Q - 1])[0]
    return t


DOT_CASES = [(c, n) for c in (1, 21, 23, 32) for n in (1, 255, 257)] + [(1, 2**21 + 3), (23, 2**21 + 3)]


@pytest.mark.parametrize("count,n", DOT_CASES)
def test_dot_many(kern, count, n):
    """k_dot_many: up to 32 tables against one, lengths 1, 255, 257 and 2^21 + 3 (several passes of the capped grid, a ragged tail)"""
    b = big_table(n, "dmb%d" % n)
    base = big_table(n, "dma%d" % n)
    a = [np.roll(base, 5 * k, axis=0) for k in range(count)]
    out = oc.zeros(count)
    kern.call("spd_dot_many", count, n, _p(cat(a)), _p(b), _p(out))
    assert oc.to_ints(out) == [oc.dot(x, b) for x in a]


def test_dot_many_refuses_33(kern):
    t = cat([edge_table(2, "d33")] * 33)
    msg, launched = kern.refused("spd_dot_many", 33, 2, _p(t), _p(edge_table(2, "d33")), _p(oc.zeros(33)))
    assert "32" in msg and launched == 0


@pytest.mark.parametrize("n", [1, 255, 257, 2**20 + 3])
@pytest.mark.parametrize("third", [False, True])
def test_dot_and_dot3(kern, n, third):
    """k_dot with and without the third table"""
    a, b = big_table(n, "da"), np.roll(big_table(n, "db"), 3, axis=0)
    c = np.roll(big_table(n, "dc"), 7, axis=0) if third else None
    out = oc.zeros(1)
    kern.call("spd_dot3", n, _p(a), _p(b), _p(c), _p(out))
    assert oc.to_ints(out) == [oc.dot3(a, b, c) if third else oc.dot(a, b)]


def test_to_canonical(kern):
    """k_to_canonical: Montgomery limbs -> canonical little-endian integers (the transcript bytes)"""
    n = 3001
    t = edge_table(n, "canon")
    out = oc.zeros(n)
    kern.call("spd_to_canonical", n, _p(t), _p(out))
    assert [int.from_bytes(out[i].tobytes(), "little") for i in range(n)] == oc.to_ints(t)


# ---------------------------------------------------------------------------------------------------- sparse products
def csr_case(nrows, ncols, seed):
    """a CSR with empty rows (the first, the last, a run in between), one 4096-entry row and repeated columns"""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 9, nrows)
    lens[0] = lens[-1] = 0
    lens[nrows // 3:nrows // 3 + 5] = 0
    lens[nrows // 2] = 4096
    ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
    idx = rng.integers(0, ncols, int(ptr[-1])).astype(np.uint32)
    s = int(ptr[nrows // 2])
    idx[s:s + 5] = [ncols - 1, ncols - 1, 0, 0, ncols - 1]
    val = big_table(int(ptr[-1]), "csrv%d" % seed)
    return ptr, idx, val


def spmv_ref(ptr, idx, val, x, rows):
    v, xs = oc.to_ints(val), oc.to_ints(x)
    return [sum(v[k] * xs[idx[k]] for k in range(ptr[r], ptr[r + 1])) % Q for r in rows]


def test_spmv(kern):
    """k_spmv on a CSR with empty rows, one 4096-entry row and repeated columns"""
    nrows, ncols = 5000, 3001
    ptr, idx, val = csr_case(nrows, ncols, 1)
    x = edge_table(ncols, "spx")
    out = oc.zeros(nrows)
    kern.call("spd_spmv", nrows, len(idx), _p(ptr), _p(idx), _p(val), ncols, _p(x), _p(out))
    assert oc.to_ints(out) == spmv_ref(ptr, idx, val, x, range(nrows))


@pytest.mark.parametrize("nnz", [1, 255, 257, 2**20 + 3])
def test_sparse_eval3(kern, nnz):
    """k_sparse_eval3: sum trx[row] try[col] val over COO entries with duplicate (row, col) pairs and the largest row and column indices"""
    nr, ncl = 1 << 10, 1 << 11
    rng = np.random.default_rng(nnz)
    row = rng.integers(0, nr, nnz).astype(np.uint32)
    col = rng.integers(0, ncl, nnz).astype(np.uint32)
    row[0], col[0] = nr - 1, ncl - 1
    if nnz > 4:
        row[1:4], col[1:4] = nr - 1, ncl - 1      # the same (row, col) four times
        row[4], col[4] = 0, 0
    val = big_table(nnz, "sev%d" % nnz)
    trx, try_ = edge_table(nr, "sex"), edge_table(ncl, "sey")
    out = oc.zeros(1)
    kern.call("spd_sparse_eval3", nnz, _p(row), _p(col), _p(val), nr, _p(trx), ncl, _p(try_), _p(out))
    assert oc.to_ints(out) == [oc.dot3(np.ascontiguousarray(trx[row]), np.ascontiguousarray(try_[col]), val)]


def test_lincomb3(kern):
    """k_lincomb3: ra A + rb B + rc C with coefficients 1, q-1 and a random one, at a length that is not a multiple of the grid"""
    n = 4 * 132 * 256 * 2 + 5
    A, B, Cc = big_table(n, "lca"), np.roll(big_table(n, "lcb"), 1, axis=0), np.roll(big_table(n, "lcc"), 2, axis=0)
    for ra, rb, rc in [(1, Q - 1, scalars("lcr", 1)[0]), tuple(scalars("lcr3", 3))]:
        out = oc.zeros(n)
        kern.call("spd_lincomb3", n, _p(A), _p(B), _p(Cc), _p(oc.to_arr([ra, rb, rc])), _p(out))
        assert np.array_equal(out, oc.lincomb3(A, B, Cc, ra, rb, rc))


@pytest.mark.parametrize("L_size", [1, 3, 64, 65, 1000])
@pytest.mark.parametrize("R_size", [1, 127, 129, 4096])
def test_bound_rows(kern, L_size, R_size):
    """k_bound_rows_partial + k_sum_slabs: slab counts 1 .. 64 with a ragged last slab, column counts around the 128-thread block"""
    Z = big_table(L_size * R_size, "brz")
    L = edge_table(L_size, "brl%d" % L_size)
    out = oc.zeros(R_size)
    kern.call("spd_bound_rows", L_size, R_size, _p(Z), _p(L), _p(out))
    assert np.array_equal(out, oc.bound_rows(Z, L, L_size, R_size))


# ---------------------------------------------------------------------------------------------------- shard producers on one GPU
@pytest.mark.parametrize("W", [2, 4, 8])
def test_take_and_spark_hash_cyclic(kern, W):
    """k_take_cyclic and k_spark_hash_cyclic (every form) on every rank equal the unsharded result taken cyclically: out[j] = full[j W + rank]"""
    n = 8 * 1001
    full = edge_table(n, "tc")
    addr, val, ts = edge_table(n, "tca"), edge_table(n, "tcv"), edge_table(n, "tct")
    rg = oc.to_arr(scalars("tcrg", 2, W))
    for rank in range(W):
        out = oc.zeros(n // W)
        kern.call("spd_take_cyclic", n, _p(full), rank, W, _p(out))
        assert np.array_equal(out, full[rank::W]), rank
    for a, t, plus in [(addr, ts, 0), (None, None, 1), (addr, None, 1), (None, ts, 0)]:
        whole = oc.zeros(n)
        kern.call("spd_spark_hash", n, _p(a), _p(val), _p(t), plus, _p(rg), _p(whole))
        for rank in range(W):
            out = oc.zeros(n // W)
            kern.call("spd_spark_hash_cyclic", n, rank, W, _p(a), _p(val), _p(t), plus, _p(rg), _p(out))
            assert np.array_equal(out, whole[rank::W]), (rank, a is None, t is None, plus)
    r, g = oc.to_ints(rg)
    v, aa, tt = oc.to_ints(val), oc.to_ints(addr), oc.to_ints(ts)
    out = oc.zeros(n // W)
    kern.call("spd_spark_hash_cyclic", n, W - 1, W, _p(addr), _p(val), _p(ts), 1, _p(rg), _p(out))
    assert oc.to_ints(out) == [((tt[i] + 1) * r * r + v[i] * r + aa[i] - g) % Q for i in range(W - 1, n, W)]


@pytest.mark.parametrize("W", [2, 4, 8])
def test_spmv_cyclic(kern, W):
    """k_spmv_cyclic: rows j W + rank of a CSR with empty rows, a 4096-entry row and repeated columns, on every rank"""
    nrows, ncols = 8 * 613, 2049
    ptr, idx, val = csr_case(nrows, ncols, W)
    x = edge_table(ncols, "spcx")
    full = spmv_ref(ptr, idx, val, x, range(nrows))
    for rank in range(W):
        out = oc.zeros(nrows // W)
        kern.call("spd_spmv_cyclic", nrows, rank, W, len(idx), _p(ptr), _p(idx), _p(val), ncols, _p(x), _p(out))
        assert oc.to_ints(out) == full[rank::W], rank


@pytest.mark.parametrize("W", [2, 4, 8])
@pytest.mark.parametrize("ell", [6, 13])
def test_scale_to_eq_slice(kern, W, ell):
    """k_scale by c_rank turns eq(r[0 .. ell - log W), .) into rank `rank`'s cyclic slice of eq(r, .)"""
    logW = W.bit_length() - 1
    r = scalars("scq", ell, W)
    full = oc.eq_evals(r)
    for rank in range(W):
        t = np.ascontiguousarray(oc.eq_evals(r[:ell - logW]))
        kern.call("spd_scale", len(t), _p(t), _p(oc.to_arr([shard_eq_scale(r, W, rank)])))
        assert np.array_equal(t, full[rank::W]), rank


@pytest.mark.parametrize("W", [2, 4, 8])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_sumcheck_on_cyclic_shards(kern, W, kind):
    """sc_eval / sc_fold_eval on the W cyclic shards of one instance's tables (XRank world = 1, one instance per shard, private tables): the
    F_q sum of the shards' evaluations is the oracle's for the whole tables every round, and the folded shards reassemble into bound_top"""
    n = 1 << 15
    tabs = [edge_table(n, "cs%d_%d" % (kind, t)) for t in range(NT[kind])]
    lay = ScLayout(kind, W, n // W, "csh", tables=lambda t, rank: np.ascontiguousarray(tabs[t][rank::W]), private=True)
    nf = 14 - (W.bit_length() - 1)          # from 2^15 / W entries per shard down to two: streaming, then small-table folds
    rs = round_scalars("csr", nf)
    res = lay.run(kern, rs, use_sig=True, bound=False)
    cur = [t.copy() for t in tabs]
    for k in range(nf + 1):
        if k:
            cur = [oc.bound_top(t.copy(), rs[k - 1]) for t in cur]
        got = oc.to_ints(res["out"][3 * W * k:3 * W * (k + 1)])
        total = [sum(got[3 * i + e] for i in range(W)) % Q for e in range(3)]
        assert total == oracle_eval(kind, cur), "round %d" % k
    m = len(cur[0]) // W
    for t in range(NT[kind]):
        whole = oc.zeros(len(cur[0]))
        for rank in range(W):
            whole[rank::W] = res["tables"][lay.map[rank, t]][:m]
        assert np.array_equal(whole, cur[t]), "table %d" % t
