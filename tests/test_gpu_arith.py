"""The device arithmetic itself — field.cuh's inline-PTX carry chains and fq_fold_const, the generated multiplications of mul_ptx.cuh, curve.cuh
and the quad-lane point operations of quad.cuh — run elementwise on the GPU through libsp_devtest.so and compared with plain Python integers
mod q / mod p, a plain-Python RFC 9496 ristretto255 and the oracle's Point.

The CPU tests (test_host_math.py) check the portable formulation; on the device these functions compile to different code.  Random operands
almost never reach the carry paths that only operands within a few units of 2^256, p, 2p or q take, so every op also runs on directed edge
sets.  F_q results must be the canonical residue limb for limb (proof bytes are Montgomery limbs); F_p results must be congruent, and
fp_canon / the encodings exact.  Bulk random inputs: 2^20 per field op, 2^16 per exponentiation, a few thousand per point op."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

from oracle.spartan_ref import core as oc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2**255 - 19
Q = oc.Q
R = oc.R_MONT
RINV = pow(R, -1, Q)
M256 = (1 << 256) - 1
NBULK = 1 << 20
NEXP = 1 << 16

# ---------------------------------------------------------------------------------------------------- plain-Python ristretto255 (RFC 9496)
D = (-121665 * pow(121666, -1, P)) % P
SQRT_M1 = pow(2, (P - 1) // 4, P)
SQRT_AD_MINUS_ONE = 25063068953384623474111414158702152701244531502492656460079210482610430750235
INVSQRT_A_MINUS_D = 54469307008909316920995813868745141605393597292927456921205312896311721017578
ONE_MINUS_D_SQ = (1 - D * D) % P
D_MINUS_ONE_SQ = (D - 1) * (D - 1) % P


def is_neg(x):
    return (x % P) & 1


def fabs(x):
    x %= P
    return (P - x) % P if x & 1 else x


def sqrt_ratio_m1(u, v):
    """RFC 9496 4.2 SQRT_RATIO_M1 -> (was_square, r)"""
    u %= P
    v %= P
    v3 = v * v % P * v % P
    v7 = v3 * v3 % P * v % P
    r = u * v3 % P * pow(u * v7 % P, (P - 5) // 8, P) % P
    check = v * r % P * r % P
    correct, flipped, flipped_i = check == u, check == (-u) % P, check == (-u * SQRT_M1) % P
    if flipped or flipped_i:
        r = r * SQRT_M1 % P
    return correct or flipped, fabs(r)


def sqrt_branch(u, v):
    """which check of SQRT_RATIO_M1 holds for the candidate root: correct (v r^2 = u), flipped (= -u), flipped_i (= -u i) or none"""
    u, v = u % P, v % P
    v3 = v * v % P * v % P
    r = u * v3 % P * pow(u * v3 % P * v3 % P * v % P, (P - 5) // 8, P) % P
    check = v * r % P * r % P
    return "correct" if check == u else "flipped" if check == (-u) % P else "flipped_i" if check == (-u * SQRT_M1) % P else "none"


def decode_reason(b):
    """RFC 9496 4.3.1 Decode: ('ok', (X, Y, Z, T)) or (reason, None)"""
    s = int.from_bytes(b, "little")
    if s >= P:
        return "non-canonical", None
    if s & 1:
        return "negative", None
    ss = s * s % P
    u1, u2 = (1 - ss) % P, (1 + ss) % P
    u2_sqr = u2 * u2 % P
    v = (-(D * u1 % P * u1) - u2_sqr) % P
    was_square, invsqrt = sqrt_ratio_m1(1, v * u2_sqr)
    den_x = invsqrt * u2 % P
    den_y = invsqrt * den_x % P * v % P
    x = fabs(2 * s * den_x)
    y = u1 * den_y % P
    t = x * y % P
    if not was_square:
        return "not square", None
    if is_neg(t):
        return "t negative", None
    if y == 0:
        return "y = 0", None
    return "ok", (x, y, 1, t)


def encode(pt):
    """RFC 9496 4.3.2 Encode of extended coordinates (any representatives) -> 32 bytes"""
    X, Y, Z, T = (c % P for c in pt)
    u1 = (Z + Y) * (Z - Y) % P
    u2 = X * Y % P
    _, invsqrt = sqrt_ratio_m1(1, u1 * u2 % P * u2)
    den1, den2 = invsqrt * u1 % P, invsqrt * u2 % P
    z_inv = den1 * den2 % P * T % P
    ix0, iy0 = X * SQRT_M1 % P, Y * SQRT_M1 % P
    ench = den1 * INVSQRT_A_MINUS_D % P
    rotate = is_neg(T * z_inv)
    x, y, den_inv = (iy0, ix0, ench) if rotate else (X, Y, den2)
    if is_neg(x * z_inv):
        y = (-y) % P
    return fabs(den_inv * (Z - y)).to_bytes(32, "little")


def rmap(t):
    """RFC 9496 4.3.4 MAP"""
    t %= P
    r = SQRT_M1 * t % P * t % P
    u = (r + 1) * ONE_MINUS_D_SQ % P
    v = (-1 - r * D) * (r + D) % P
    was_square, s = sqrt_ratio_m1(u, v)
    s_prime = (-fabs(s * t)) % P
    c = P - 1
    if not was_square:
        s, c = s_prime, r
    N = (c * (r - 1) % P * D_MINUS_ONE_SQ - v) % P
    w0, w1 = 2 * s * v % P, N * SQRT_AD_MINUS_ONE % P
    w2, w3 = (1 - s * s) % P, (1 + s * s) % P
    return (w0 * w3 % P, w2 * w1 % P, w1 * w3 % P, w0 * w2 % P)


def from_uniform(b64):
    mask = (1 << 255) - 1
    return ed_add(rmap(int.from_bytes(b64[:32], "little") & mask), rmap(int.from_bytes(b64[32:], "little") & mask))


# edwards25519 (a = -1) in extended coordinates: the formulas of curve.cuh, evaluated exactly mod p
def ed_add(p, q):     # add-2008-hwcd-3
    A = (p[1] - p[0]) * (q[1] - q[0]) % P
    B = (p[1] + p[0]) * (q[1] + q[0]) % P
    Cc = p[3] * q[3] % P * 2 * D % P
    Dd = 2 * p[2] * q[2] % P
    E, F, G, H = B - A, Dd - Cc, Dd + Cc, B + A
    return (E * F % P, G * H % P, F * G % P, E * H % P)


def ed_dbl(p):        # dbl-2008-hwcd
    A, B, Cc = p[0] * p[0] % P, p[1] * p[1] % P, 2 * p[2] * p[2] % P
    E = ((p[0] + p[1]) ** 2 - A - B) % P
    G, H = (B - A) % P, (-A - B) % P
    F = (G - Cc) % P
    return (E * F % P, G * H % P, F * G % P, E * H % P)


def niels(p):         # (y + x, y - x, 2dxy), canonical
    zi = pow(p[2], P - 2, P)
    x, y = p[0] * zi % P, p[1] * zi % P
    return ((y + x) % P, (y - x) % P, 2 * D * x % P * y % P)


def ed_madd(p, n, neg):
    ypx, ymx, t2d = n
    if neg:
        ypx, ymx, t2d = ymx, ypx, (-t2d) % P
    A = (p[1] - p[0]) * ymx % P
    B = (p[1] + p[0]) * ypx % P
    Cc = p[3] * t2d % P
    Dd = 2 * p[2] % P
    E, F, G, H = B - A, Dd - Cc, Dd + Cc, B + A
    return (E * F % P, G * H % P, F * G % P, E * H % P)


IDENT = (0, 1, 1, 0)
TORSION = [(0, 1, 1, 0), (0, P - 1, 1, 0), (SQRT_M1, 0, 1, 0), (P - SQRT_M1, 0, 1, 0)]   # the 4-torsion of edwards25519


def same_point(a, b):
    """equal as points of edwards25519 (projective equality, not just the same ristretto class)"""
    return (a[0] * b[2] - b[0] * a[2]) % P == 0 and (a[1] * b[2] - b[1] * a[2]) % P == 0 and a[2] % P != 0 and b[2] % P != 0


def on_curve(p):
    X, Y, Z, T = (c % P for c in p)
    return Z != 0 and (-X * X + Y * Y - Z * Z - D * T * T) % P == 0 and (X * Y - Z * T) % P == 0


# ---------------------------------------------------------------------------------------------------- plumbing
def u256(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint32).reshape(-1, 8).copy()


def ints(arr):
    b = np.ascontiguousarray(arr).tobytes()
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


def ge_arr(pts):
    return u256([c for p in pts for c in p]).reshape(-1, 32)


def ge_ints(arr):
    v = ints(arr)
    return [tuple(v[i:i + 4]) for i in range(0, len(v), 4)]


def niels_arr(ns):
    return u256([c for n in ns for c in n]).reshape(-1, 24)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def rand_ints(rng, n, bits=256):
    b = rng.bytes(32 * n)
    mask = (1 << bits) - 1
    return [int.from_bytes(b[i:i + 32], "little") & mask for i in range(0, 32 * n, 32)]


def fmt(x):
    return "%#x" % x if isinstance(x, int) else repr(x)


def expect(op, got, want, operands, mod=None):
    """got[i] == want[i] (or congruent mod `mod`), else the first failures with their operands"""
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if (g != w if mod is None else (g - w) % mod)]
    assert len(got) == len(want)
    assert not bad, "%s: %d of %d results wrong%s; first: %s" % (
        op, len(bad), len(got), "" if mod is None else " mod p",
        "; ".join("operands (%s) -> got %s, want %s" % (", ".join(fmt(o[i]) for o in operands), fmt(got[i]), fmt(want[i])) for i in bad[:4]))


class Dev:
    """ctypes front of libsp_devtest.so (spartan_b200/csrc/devtest.cu); every call checks the CUDA status"""
    FQ = dict(mul=0, add=1, sub=2, neg=3, from_mont=4, to_mont=5, from_wide=6, from_u64=7, inv=8)
    FP = dict(mul=0, add=1, sub=2, neg=3, mul_small=4, canon=5, inv=6, pow22523=7)

    def __init__(self, lib):
        self.lib = lib
        for name in ["spd_fq", "spd_fp", "spd_ge"]:
            getattr(lib, name).argtypes = [C.c_int, C.c_size_t] + [C.c_void_p] * 3
        lib.spd_quad.argtypes = [C.c_int, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        lib.spd_ge_madd.argtypes = [C.c_size_t, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        for name in ["spd_fq_fold_const", "spd_fp_sqrt_ratio_i"]:
            getattr(lib, name).argtypes = [C.c_size_t] + [C.c_void_p] * 4
        for name in ["spd_ge_to_niels", "spd_ristretto_encode", "spd_ristretto_map"]:
            getattr(lib, name).argtypes = [C.c_size_t, C.c_void_p, C.c_void_p]
        for name in ["spd_ristretto_decode", "spd_ristretto_from_uniform"]:
            getattr(lib, name).argtypes = [C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
        for name in ["spd_signed_digits", "spd_window_digits"]:
            getattr(lib, name).argtypes = [C.c_size_t, C.c_void_p, C.c_int, C.c_void_p]

    @staticmethod
    def ok(rc, what):
        assert rc == 0, "%s: CUDA error %d" % (what, rc)

    def fq(self, op, a, b=None):
        A, B = u256(a), u256(b) if b is not None else None
        out = np.zeros_like(A)
        self.ok(self.lib.spd_fq(self.FQ[op], len(a), _ptr(A), _ptr(B), _ptr(out)), "fq_" + op)
        return ints(out)

    def fp(self, op, a, b=None):
        A, B = u256(a), u256(b) if b is not None else None
        out = np.zeros_like(A)
        self.ok(self.lib.spd_fp(self.FP[op], len(a), _ptr(A), _ptr(B), _ptr(out)), "fp_" + op)
        return ints(out)

    def fold_const(self, a0, a1, r_mont):
        A0, A1, Rm = u256(a0), u256(a1), u256([r_mont])
        out = np.zeros_like(A0)
        self.ok(self.lib.spd_fq_fold_const(len(a0), _ptr(A0), _ptr(A1), _ptr(Rm), _ptr(out)), "fq_fold_const")
        return ints(out)

    def sqrt_ratio_i(self, u, v):
        U, V = u256(u), u256(v)
        out, flag = np.zeros_like(U), np.zeros(len(u), dtype=np.int32)
        self.ok(self.lib.spd_fp_sqrt_ratio_i(len(u), _ptr(U), _ptr(V), _ptr(out), _ptr(flag)), "fp_sqrt_ratio_i")
        return [bool(f) for f in flag], ints(out)

    def ge(self, op, p, q=None):
        Pa, Qa = ge_arr(p), ge_arr(q) if q is not None else None
        out = np.zeros_like(Pa)
        self.ok(self.lib.spd_ge(0 if op == "add" else 1, len(p), _ptr(Pa), _ptr(Qa), _ptr(out)), "ge_" + op)
        return ge_ints(out)

    def madd(self, p, ns, neg):
        Pa, Na = ge_arr(p), niels_arr(ns)
        out = np.zeros_like(Pa)
        self.ok(self.lib.spd_ge_madd(len(p), _ptr(Pa), _ptr(Na), int(neg), _ptr(out)), "ge_madd")
        return ge_ints(out)

    def quad(self, op, p, q=None, ns=None, neg=False):
        Pa = ge_arr(p)
        Qa = ge_arr(q) if q is not None else None
        Na = niels_arr(ns) if ns is not None else None
        out = np.zeros_like(Pa)
        self.ok(self.lib.spd_quad(dict(add=0, madd=1, dbl=2)[op], len(p), _ptr(Pa), _ptr(Qa), _ptr(Na), int(neg), _ptr(out)), "quad_" + op)
        return ge_ints(out)

    def to_niels(self, p):
        Pa = ge_arr(p)
        out = np.zeros((len(p), 24), dtype=np.uint32)
        self.ok(self.lib.spd_ge_to_niels(len(p), _ptr(Pa), _ptr(out)), "ge_to_niels")
        v = ints(out)
        return [tuple(v[i:i + 3]) for i in range(0, len(v), 3)]

    def encode(self, p):
        Pa = ge_arr(p)
        out = np.zeros((len(p), 8), dtype=np.uint32)
        self.ok(self.lib.spd_ristretto_encode(len(p), _ptr(Pa), _ptr(out)), "ristretto_encode")
        return [x.to_bytes(32, "little") for x in ints(out)]

    def decode(self, encs):
        S = np.frombuffer(b"".join(encs), dtype=np.uint32).reshape(-1, 8).copy()
        out, ok = np.zeros((len(encs), 32), dtype=np.uint32), np.zeros(len(encs), dtype=np.int32)
        self.ok(self.lib.spd_ristretto_decode(len(encs), _ptr(S), _ptr(out), _ptr(ok)), "ristretto_decode")
        return [bool(x) for x in ok], ge_ints(out)

    def map(self, t):
        T = u256(t)
        out = np.zeros((len(t), 32), dtype=np.uint32)
        self.ok(self.lib.spd_ristretto_map(len(t), _ptr(T), _ptr(out)), "ristretto_map")
        return ge_ints(out)

    def from_uniform(self, b64s):
        lo = np.frombuffer(b"".join(b[:32] for b in b64s), dtype=np.uint32).reshape(-1, 8).copy()
        hi = np.frombuffer(b"".join(b[32:] for b in b64s), dtype=np.uint32).reshape(-1, 8).copy()
        out = np.zeros((len(b64s), 32), dtype=np.uint32)
        self.ok(self.lib.spd_ristretto_from_uniform(len(b64s), _ptr(lo), _ptr(hi), _ptr(out)), "ristretto_from_uniform")
        return ge_ints(out)

    def digits(self, fn, k, W):
        nwin = -(-253 // W)
        K = u256(k)
        out = np.zeros(len(k) * nwin, dtype=np.int32)
        self.ok(getattr(self.lib, fn)(len(k), _ptr(K), W, _ptr(out)), fn)
        return out.reshape(len(k), nwin).tolist()


@pytest.fixture(scope="module")
def dev():
    path = os.path.join(ROOT, "spartan_b200", "libsp_devtest.so")
    assert os.path.exists(path), "libsp_devtest.so is not built: run __graft_entry__.build()"
    return Dev(C.CDLL(path))


# ---------------------------------------------------------------------------------------------------- operand sets
def fq_core():
    """about 40 F_q values at the edges of the carry chains"""
    half = (Q - 1) // 2
    core = [0, 1, 2, Q - 1, Q - 2, half, half + 1, R, R * R % Q, RINV, 2**252, 2**252 - 1, 2**128, 2**64 - 1, 2**32 - 1, 2**32, 2**224,
            Q - 2**32, Q - 2**128, Q - 2**224, Q - 2**252, 2**253 % Q, M256 % Q]
    for i in range(8):                 # one 32-bit limb all ones and the rest zero, or the reverse, reduced
        core += [(0xffffffff << (32 * i)) % Q, (M256 ^ (0xffffffff << (32 * i))) % Q]
    return list(dict.fromkeys(core))


def fq_edges():
    e = fq_core()
    for k in range(253):
        e += [2**k, 2**k - 1, Q - 2**k]
    return list(dict.fromkeys(e))


def fq_pairs(rng):
    core, edges = fq_core(), fq_edges()
    a = [x for x in core for _ in core] + edges + edges
    b = [y for _ in core for y in core] + edges[::-1] + edges
    r = rand_ints(rng, 2 * NBULK)
    return a + [x % Q for x in r[:NBULK]], b + [x % Q for x in r[NBULK:]]


def fp_edges():
    e = list(range(41)) + list(range(P - 40, P + 41)) + list(range(2**255 - 40, 2**255 + 41)) + list(range(2 * P - 40, 2**256))
    for i in range(1, 8):              # limb boundaries
        e += [2**(32 * i) - 1, 2**(32 * i), 2**(32 * i) + 1]
    for i in range(8):
        e += [0xffffffff << (32 * i), M256 ^ (0xffffffff << (32 * i))]
    return list(dict.fromkeys(e))


def fp_pairs(rng):
    edges = fp_edges()                 # all pairs of the edge set
    a = [x for x in edges for _ in edges]
    b = [y for _ in edges for y in edges]
    r = rand_ints(rng, 2 * NBULK)
    return a + r[:NBULK], b + r[NBULK:]


# ---------------------------------------------------------------------------------------------------- F_q
FQ_BINARY = {"mul": lambda a, b: a * b * RINV % Q, "add": lambda a, b: (a + b) % Q, "sub": lambda a, b: (a - b) % Q}


@pytest.mark.gpu
@pytest.mark.parametrize("op", ["mul", "add", "sub"])
def test_fq_binary(dev, op):
    a, b = fq_pairs(np.random.default_rng(1))
    f = FQ_BINARY[op]
    expect("fq_" + op, dev.fq(op, a, b), [f(x, y) for x, y in zip(a, b)], [a, b])


@pytest.mark.gpu
def test_fq_unary(dev):
    rng = np.random.default_rng(2)
    a = fq_edges() + [x % Q for x in rand_ints(rng, NBULK)]
    expect("fq_neg", dev.fq("neg", a), [(-x) % Q for x in a], [a])
    expect("fq_from_mont", dev.fq("from_mont", a), [x * RINV % Q for x in a], [a])
    e = fq_edges() + [x % Q for x in rand_ints(rng, NEXP)]
    expect("fq_inv", dev.fq("inv", e), [pow(x * RINV % Q, -1, Q) * R % Q if x else 0 for x in e], [e])


@pytest.mark.gpu
def test_fq_to_mont_and_from_u64_full_range(dev):
    """to_mont accepts any 256-bit value (fq_to_mont: a < 2^256), including q .. 2^256 - 1"""
    rng = np.random.default_rng(3)
    high = [Q + k for k in range(41)] + [2 * Q - 1, 2 * Q, 2**253, 2**255, M256, M256 - 1, M256 - Q, 2**256 - 2**252]
    high += [M256 - 2**k for k in range(256)] + [(2**k - 1) << (256 - k) for k in range(1, 256)]
    a = fq_edges() + high + rand_ints(rng, NBULK)
    expect("fq_to_mont", dev.fq("to_mont", a), [x * R % Q for x in a], [a])
    u = [0, 1, 2, 2**32 - 1, 2**32, 2**63, 2**64 - 1] + [x & (2**64 - 1) for x in rand_ints(rng, 4096)]
    expect("fq_from_u64", dev.fq("from_u64", u), [x * R % Q for x in u], [u])


@pytest.mark.gpu
def test_fq_from_wide(dev):
    """Scalar::from_bytes_wide over the whole 512-bit range, 2^512 - 1 included"""
    rng = np.random.default_rng(4)
    edge = [0, 1, Q - 1, Q, 2**256 - 1, 2**256, 2**512 - 1, 2**512 - 2**256, Q * 2**256, Q * Q, Q * 2**256 + Q - 1, 2**511]
    edge += [2**k - 1 for k in range(1, 513, 7)] + [2**512 - 2**k for k in range(0, 512, 5)]
    w = edge + [lo | hi << 256 for lo, hi in zip(rand_ints(rng, NBULK), rand_ints(rng, NBULK))]
    lo, hi = [x & M256 for x in w], [x >> 256 for x in w]
    expect("fq_from_wide", dev.fq("from_wide", lo, hi), [x * R % Q for x in w], [w])


@pytest.mark.gpu
@pytest.mark.parametrize("r", [0, 1, Q - 1, 2**32, 2**224, 0x0BADC0FFEE0DDF00D5EED5EED5EED5EED5EED5EED5EED5EED5EED5EED5EED5E % Q],
                         ids=["0", "1", "q-1", "2^32", "2^224", "random"])
def test_fq_fold_const(dev, r):
    """a0 + r*(a1 - a0) through the host-built constant-multiplier table: triples from the core set with a1 < a0, a1 = a0, a1 > a0"""
    core = fq_core()
    a0 = [x for x in core for _ in core]
    a1 = [y for _ in core for y in core]
    rng = np.random.default_rng(5)
    rand = rand_ints(rng, 2 * NBULK // 4)
    a0 += [x % Q for x in rand[:NBULK // 4]] + fq_edges()
    a1 += [x % Q for x in rand[NBULK // 4:]] + fq_edges()[::-1]
    expect("fq_fold_const(r=%#x)" % r, dev.fold_const(a0, a1, r * R % Q), [(x + r * (y - x)) % Q for x, y in zip(a0, a1)], [a0, a1])


# ---------------------------------------------------------------------------------------------------- F_p
FP_BINARY = {"mul": lambda a, b: a * b % P, "add": lambda a, b: (a + b) % P, "sub": lambda a, b: (a - b) % P}


@pytest.mark.gpu
@pytest.mark.parametrize("op", ["mul", "add", "sub"])
def test_fp_binary(dev, op):
    """loose operands anywhere in [0, 2^256): all pairs of the edge set (p +- 40, 2^255 +- 40, 2p - 40 .. 2^256 - 1, limb boundaries) and
    2^20 random pairs; the second wrap of fp_add / fp_sub needs both operands near 2^256 (or one near 0)"""
    a, b = fp_pairs(np.random.default_rng(6))
    got = dev.fp(op, a, b)
    f = FP_BINARY[op]
    expect("fp_" + op, got, [f(x, y) for x, y in zip(a, b)], [a, b], mod=P)


@pytest.mark.gpu
def test_fp_unary(dev):
    rng = np.random.default_rng(7)
    a = fp_edges() + rand_ints(rng, NBULK)
    expect("fp_neg", dev.fp("neg", a), [(-x) % P for x in a], [a], mod=P)
    expect("fp_canon", dev.fp("canon", a), [x % P for x in a], [a])          # exact
    k = [0, 1, 2, 19, 38, 121666, 2**31, 2**32 - 1] + [x & 0xffffffff for x in rand_ints(rng, len(a) - 8)]
    expect("fp_mul_small", dev.fp("mul_small", a, k), [x * y % P for x, y in zip(a, k)], [a, k], mod=P)
    e = fp_edges() + rand_ints(rng, NEXP)
    expect("fp_inv", dev.fp("inv", e), [pow(x, P - 2, P) for x in e], [e], mod=P)
    expect("fp_pow22523", dev.fp("pow22523", e), [pow(x, (P - 5) // 8, P) for x in e], [e], mod=P)


@pytest.mark.gpu
def test_fp_chained(dev):
    """64 rounds fed with the device's own outputs: whatever loose values the kernels really produce go back in"""
    rng = np.random.default_rng(8)
    n = 1 << 12
    edges = fp_edges()
    x = edges + rand_ints(rng, n - len(edges))
    y = rand_ints(rng, n - len(edges)) + edges[::-1]
    for rnd in range(64):
        s, d = dev.fp("add", x, y), dev.fp("sub", x, y)
        expect("fp_add round %d" % rnd, s, [(a + b) % P for a, b in zip(x, y)], [x, y], mod=P)
        expect("fp_sub round %d" % rnd, d, [(a - b) % P for a, b in zip(x, y)], [x, y], mod=P)
        m = dev.fp("mul", s, d)
        expect("fp_mul round %d" % rnd, m, [a * b % P for a, b in zip(s, d)], [s, d], mod=P)
        ng = dev.fp("neg", m)
        expect("fp_neg round %d" % rnd, ng, [(-a) % P for a in m], [m], mod=P)
        k = [38] * n
        ms = dev.fp("mul_small", d, k)
        expect("fp_mul_small round %d" % rnd, ms, [a * 38 % P for a in d], [d], mod=P)
        expect("fp_canon round %d" % rnd, dev.fp("canon", ng), [a % P for a in ng], [ng])
        x, y = (ng, ms) if rnd % 2 else (m, s)


@pytest.mark.gpu
def test_fp_sqrt_ratio_i(dev):
    """RFC 9496 SQRT_RATIO_M1: every branch (u = 0, v = 0, u/v square, -u/v square, i*u/v square, neither); flag and root exact"""
    rng = np.random.default_rng(9)
    n = 4096
    xs, vs = rand_ints(rng, n), [v % P or 1 for v in rand_ints(rng, n)]
    nonsq = 2                                                       # 2 is not a square mod p
    cases = {"u=0": ([0] * n, vs), "v=0": (xs, [0] * n)}
    for name, c in [("u/v square", 1), ("-u/v square", P - 1), ("i*u/v square", SQRT_M1), ("-i*u/v square", P - SQRT_M1), ("neither", nonsq)]:
        cases[name] = ([c * x % P * x % P * v % P for x, v in zip(xs, vs)], vs)
    u = [x + P if x < 2**256 - P else x for x in rand_ints(rng, n)]   # loose operands too
    cases["random loose"] = (u, rand_ints(rng, n))
    branches = set()
    for name, (uu, vv) in cases.items():
        flags, roots = dev.sqrt_ratio_i(uu, vv)
        want = [sqrt_ratio_m1(a, b) for a, b in zip(uu, vv)]
        expect("fp_sqrt_ratio_i flag (%s)" % name, [int(f) for f in flags], [int(w[0]) for w in want], [uu, vv])
        expect("fp_sqrt_ratio_i root (%s)" % name, [r % P for r in roots], [w[1] for w in want], [uu, vv])
        branches |= {sqrt_branch(a, b) for a, b in zip(uu, vv)}
    assert branches == {"correct", "flipped", "flipped_i", "none"}, branches


# ---------------------------------------------------------------------------------------------------- group
BASE = decode_reason(oc.BASEPOINT_COMPRESSED)[1]


def rescale(p, lam, lift):
    """(lam X, lam Y, lam Z, lam T); lift: coordinates moved to the representative >= p where one exists below 2^256"""
    q = tuple(c * lam % P for c in p)
    return tuple(c + P if lift and c + P <= M256 else c for c in q)


def point_set(n_random):
    """small multiples 0..16 of the basepoint, their sums with the 4-torsion, mapped random points, and projective rescalings of them"""
    mult = [IDENT]
    for _ in range(16):
        mult.append(ed_add(mult[-1], BASE))
    rnd = [rmap(int.from_bytes(hashlib.sha256(b"devtest-pt%d" % i).digest(), "little")) for i in range(n_random)]
    pts = mult + [ed_add(m, t) for m in mult[:4] for t in TORSION[1:]] + rnd
    rng = np.random.default_rng(10)
    out = list(pts)
    for i, p in enumerate(pts):
        out.append(rescale(p, rand_ints(rng, 1)[0] % P or 1, lift=i % 2 == 0))
    out.append(rescale(BASE, P - 1, True))
    return mult, out


def check_points(op, got, want, operands):
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if not (same_point(g, w) and on_curve(g) and all((a - b) % P == 0 for a, b in zip(g, w)))]
    assert not bad, "%s: %d of %d results wrong; first: %s" % (op, len(bad), len(got), "; ".join(
        "operands %s -> got %s, want %s" % ([tuple(fmt(c) for c in o[i]) for o in operands], tuple(fmt(c) for c in got[i]), want[i]) for i in bad[:2]))


@pytest.mark.gpu
def test_point_ops_match_formulas(dev):
    """ge_add, ge_dbl, ge_madd (+/-), ge_to_niels and the quad-lane quad_add / quad_madd / quad_dbl give exactly the coordinates of their formulas
    (mod p) on identity, basepoint, multiples 0..16, P + P, P + (-P), 4-torsion sums and rescaled representatives with coordinates >= p"""
    mult, pts = point_set(2048)
    n = len(pts)
    rng = np.random.default_rng(11)
    perm = rng.permutation(n)
    ps = [mult[i] for i in range(17) for _ in range(17)] + pts
    qs = [mult[j] for _ in range(17) for j in range(17)] + [pts[k] for k in perm]
    ps += [BASE, BASE, pts[20]]
    qs += [BASE, (P - BASE[0], BASE[1], BASE[2], P - BASE[3]), (P - pts[20][0], pts[20][1], pts[20][2], P - pts[20][3])]   # P + P, P + (-P)
    want = [ed_add(p, q) for p, q in zip(ps, qs)]
    check_points("ge_add", dev.ge("add", ps, qs), want, [ps, qs])
    check_points("quad_add", dev.quad("add", ps, qs), want, [ps, qs])
    for p, q, w in zip(ps, qs, want):           # and the same points as the group law says
        assert same_point(w, ed_add(q, p))
    want = [ed_dbl(p) for p in pts]
    check_points("ge_dbl", dev.ge("dbl", pts), want, [pts])
    check_points("quad_dbl", dev.quad("dbl", pts), want, [pts])
    assert all(same_point(w, ed_add(p, p)) for w, p in zip(want, pts))
    ns = [niels(q) for q in qs]
    got = dev.to_niels(qs)
    bad = [i for i in range(len(qs)) if got[i] != ns[i]]
    assert not bad, "ge_to_niels: %d wrong; first operand %s got %s want %s" % (len(bad), qs[bad[0]], got[bad[0]], ns[bad[0]])
    for neg in (False, True):
        want = [ed_madd(p, nq, neg) for p, nq in zip(ps, ns)]
        check_points("ge_madd(neg=%d)" % neg, dev.madd(ps, ns, neg), want, [ps, qs])
        check_points("quad_madd(neg=%d)" % neg, dev.quad("madd", ps, ns=ns, neg=neg), want, [ps, qs])
        qq = [(P - q[0], q[1], q[2], P - q[3]) for q in qs] if neg else qs
        assert all(same_point(w, ed_add(p, q)) for w, p, q in zip(want, ps, qq))


@pytest.mark.gpu
def test_encode_cosets_and_oracle(dev):
    """ristretto_encode is the RFC encoding (plain-Python and the oracle's), is canonical, and does not change within a ristretto coset: P + T for
    each 4-torsion point T and every projective rescaling encode to the same bytes — the byte-identical proofs depend on it"""
    mult, pts = point_set(1024)
    got = dev.encode(pts)
    want = [encode(p) for p in pts]
    bad = [i for i in range(len(pts)) if got[i] != want[i]]
    assert not bad, "ristretto_encode: %d wrong; first operand %s got %s want %s" % (len(bad), pts[bad[0]], got[bad[0]].hex(), want[bad[0]].hex())
    B = oc.Point.decompress(oc.BASEPOINT_COMPRESSED)
    for k, m in enumerate(mult):
        assert dev.encode([m])[0] == (B * k).compress(), k
    for t in TORSION:
        tp = [ed_add(p, t) for p in pts]
        got_t = dev.encode(tp)
        bad = [i for i in range(len(pts)) if got_t[i] != want[i]]
        assert not bad, "encoding changed within the coset (T = %s): operand %s" % (t, pts[bad[0]])
        qt = dev.quad("add", pts, [t] * len(pts))     # through the device's own additions too
        assert dev.encode(qt) == want
    sums = dev.ge("add", pts[:256], pts[256:512])
    want = [(oc.Point.decompress(encode(p)) + oc.Point.decompress(encode(q))).compress() for p, q in zip(pts[:256], pts[256:512])]
    assert dev.encode(sums) == want


def late_rejections():
    """one encoding for each late rejection of ristretto_decode: found by classifying small even s with the plain-Python decode"""
    found = {"y = 0": (P - 1).to_bytes(32, "little")}
    s = 2
    while len(found) < 3:
        b = s.to_bytes(32, "little")
        reason, _ = decode_reason(b)
        if reason in ("not square", "t negative") and reason not in found:
            found[reason] = b
        s += 2
    assert decode_reason(found["y = 0"])[0] == "y = 0"
    return found


def rfc9496():
    with open(os.path.join(ROOT, "tests", "golden", "rfc9496.json")) as f:
        return json.load(f)


@pytest.mark.gpu
def test_decode(dev):
    """ristretto_decode on the RFC 9496 A.1 multiples and A.2 bad encodings, one encoding per late rejection (not square, t negative, y = 0) and
    random strings; the library's own k_decompress / k_compress (sp_point_decompress_check / sp_point_roundtrip) on the same vectors"""
    rfc = rfc9496()
    good = [bytes.fromhex(h) for h in rfc["multiples"]]
    late = late_rejections()
    bad = [bytes.fromhex(h) for h in rfc["bad_encodings"]] + list(late.values())
    rnd = [hashlib.sha256(b"devtest-dec%d" % i).digest() for i in range(4096)]
    rnd += [(int.from_bytes(r, "little") & ((1 << 255) - 2)).to_bytes(32, "little") for r in rnd[:2048]]   # top bit clear, even: more get far
    encs = good + bad + rnd
    ok, pts = dev.decode(encs)
    ref = [decode_reason(e) for e in encs]
    for e, o, p, (reason, rp) in zip(encs, ok, pts, ref):
        assert o == (reason == "ok"), "ristretto_decode(%s): device %s, RFC decode says %s" % (e.hex(), o, reason)
        if o:
            assert all((a - b) % P == 0 for a, b in zip(p, rp)), e.hex()
    assert ok[:len(good)] == [True] * len(good) and not any(ok[len(good):len(good) + len(bad)])
    assert dev.encode([p for p, o in zip(pts, ok) if o]) == [e for e, o in zip(encs, ok) if o]
    assert [o for o in ok[len(good) + len(bad):]] == [oc.Point.decompress(e) is not None for e in rnd]
    import spartan_b200 as sb
    from spartan_b200 import api
    sb.default_context()
    assert api.point_decompress_check(encs) == ok
    assert api.point_roundtrip([e for e, o in zip(encs, ok) if o]) == [e for e, o in zip(encs, ok) if o]


@pytest.mark.gpu
def test_map_and_from_uniform(dev):
    """ristretto_map gives the coordinates of RFC 9496 MAP (mod p); ristretto_from_uniform encodes like the oracle's from_uniform_bytes"""
    rng = np.random.default_rng(12)
    t = [0, 1, 2, P - 1, P, P + 1, 2**255 - 1, SQRT_M1, D, M256] + rand_ints(rng, 4096)
    got = dev.map(t)
    want = [rmap(x) for x in t]
    bad = [i for i in range(len(t)) if not all((a - b) % P == 0 for a, b in zip(got[i], want[i]))]
    assert not bad, "ristretto_map(%#x): got %s want %s" % (t[bad[0]], got[bad[0]], want[bad[0]])
    hs = [hashlib.sha512(b"devtest-uni%d" % i).digest() for i in range(2048)] + [b"\xff" * 64, bytes(64)]
    pts = dev.from_uniform(hs)
    assert all(same_point(p, from_uniform(h)) for p, h in zip(pts, hs))
    assert dev.encode(pts) == [oc.Point.from_uniform_bytes(h).compress() for h in hs]


# ---------------------------------------------------------------------------------------------------- recoding
def recode_scalars(W):
    half = 1 << (W - 1)
    nwin = -(-253 // W)
    every_carry = (1 << 252) - 1
    half_plus_one = sum((half + 1) << (W * w) for w in range(252 // W)) % Q
    half_chain = ((half + 1) + sum(half << (W * w) for w in range(1, 252 // W))) % Q   # each window = half: carries only when the carry comes in
    ks = [0, 1, 2, Q - 1, half - 1, half, half + 1, (1 << W) - 1, 1 << W, every_carry, half_plus_one, half_chain, (1 << 252) + 5,
          (1 << 252) + half, Q - half, Q - 1 - half]
    ks += [((1 << W) - 1) << (W * w) for w in range(nwin - 1)] + [half << (W * w) for w in range(nwin)]
    return [k % Q for k in ks] + [k % Q for k in fq_edges()] + [x % Q for x in rand_ints(np.random.default_rng(W), NEXP)]


def check_digits(op, k, digits, W):
    for x, d in zip(k, digits):
        assert sum(v << (W * w) for w, v in enumerate(d)) == x and all(-(1 << (W - 1)) < v <= (1 << (W - 1)) for v in d), \
            "%s W=%d: k = %#x -> digits %s" % (op, W, x, d)


@pytest.mark.gpu
@pytest.mark.parametrize("W", [8, 13, 15, 16, 17])
def test_signed_digits(dev, W):
    k = recode_scalars(W)
    check_digits("signed_digit", k, dev.digits("spd_signed_digits", k, W), W)


@pytest.mark.gpu
@pytest.mark.parametrize("W", [8, 13, 15])
def test_msm_window_with_carry_in(dev, W):
    """msm_window<W> and the carry into a thread's first window that k_msm_rows / k_ipa_msm_quad compute, for every first window"""
    k = recode_scalars(W)
    check_digits("msm_window", k, dev.digits("spd_window_digits", k, W), W)


# ---------------------------------------------------------------------------------------------------- the plain-Python reference itself (CPU)
def test_python_ristretto_reference_matches_oracle():
    """the plain-Python RFC 9496 code above agrees with the RFC vectors and the oracle, so that the device tests compare against a checked reference"""
    rfc = rfc9496()
    acc = IDENT
    for h in rfc["multiples"]:
        assert encode(acc).hex() == h
        reason, p = decode_reason(bytes.fromhex(h))
        assert reason == "ok" and encode(p).hex() == h
        acc = ed_add(acc, BASE)
    for h in rfc["bad_encodings"]:
        assert decode_reason(bytes.fromhex(h))[0] != "ok"
    late = late_rejections()
    assert sorted(late) == ["not square", "t negative", "y = 0"]
    for b in late.values():
        assert oc.Point.decompress(b) is None
    for i in range(64):
        h = hashlib.sha512(b"ref%d" % i).digest()
        p = from_uniform(h)
        assert on_curve(p) and encode(p) == oc.Point.from_uniform_bytes(h).compress()
        b = hashlib.sha256(b"refdec%d" % i).digest()
        assert (decode_reason(b)[0] == "ok") == (oc.Point.decompress(b) is not None)
    for t in TORSION:
        assert on_curve(t) and encode(ed_add(BASE, t)) == oc.BASEPOINT_COMPRESSED
    assert same_point(ed_dbl(BASE), ed_add(BASE, BASE))
    assert ed_madd(BASE, niels(BASE), True)[0] % P == 0     # P - P: the identity class
