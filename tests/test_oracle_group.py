"""ristretto255 restatement (oracle/csrc/ristretto.c) pinned against RFC 9496 appendix A vectors and,
as an independent differential oracle, libsodium (bundled with pyzmq) — SURVEY.md §8c item 3.
The reference holds no group-level known answers (its group is curve25519-dalek, a third-party crate)."""
import ctypes as C
import glob
import hashlib
import json
import os
import site

import numpy as np
import pytest

from oracle.spartan_ref import core as oc

# RFC 9496 A.1 (multiples 0..4 of the generator) and A.2 (bad encodings), shared with the device tests
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rfc9496.json")) as _f:
    RFC = json.load(_f)
RFC_MULTIPLES = RFC["multiples"]


def _sodium():
    cands = [p for sp in site.getsitepackages() for p in glob.glob(sp + "/pyzmq.libs/libsodium*")]
    if not cands:
        pytest.skip("libsodium not available")
    return C.CDLL(cands[0])


def test_rfc9496_basepoint_multiples():
    B = oc.Point.decompress(oc.BASEPOINT_COMPRESSED)
    acc = oc.Point.identity()
    for h in RFC_MULTIPLES:
        assert acc.compress().hex() == h
        acc = acc + B
    assert (B * 3).compress().hex() == RFC_MULTIPLES[3]


def test_decode_rejects_bad_encodings():
    # RFC 9496 A.2: non-canonical field encodings and negative field elements
    bad = RFC["bad_encodings"]
    for h in bad:
        assert oc.Point.decompress(bytes.fromhex(h)) is None


def test_differential_vs_libsodium():
    sod = _sodium()
    rng = np.random.default_rng(7)
    o = C.create_string_buffer(32)
    pts = []
    for i in range(40):
        h = hashlib.sha512(b"pt%d" % i).digest()
        sod.crypto_core_ristretto255_from_hash(o, C.c_char_p(h))
        mine = oc.Point.from_uniform_bytes(h)
        assert mine.compress() == o.raw
        assert oc.Point.decompress(o.raw).compress() == o.raw
        pts.append((mine, o.raw))
    for i in range(0, 40, 2):
        sod.crypto_core_ristretto255_add(o, C.c_char_p(pts[i][1]), C.c_char_p(pts[i + 1][1]))
        assert (pts[i][0] + pts[i + 1][0]).compress() == o.raw
        sod.crypto_core_ristretto255_sub(o, C.c_char_p(pts[i][1]), C.c_char_p(pts[i + 1][1]))
        assert (pts[i][0] - pts[i + 1][0]).compress() == o.raw
        k = int.from_bytes(rng.bytes(32), "little") % oc.Q
        assert sod.crypto_scalarmult_ristretto255(o, C.c_char_p(k.to_bytes(32, "little")), C.c_char_p(pts[i][1])) == 0
        assert (pts[i][0] * k).compress() == o.raw
    # validity of random byte strings agrees
    for i in range(300):
        b = hashlib.sha256(b"v%d" % i).digest()
        assert (oc.Point.decompress(b) is not None) == bool(sod.crypto_core_ristretto255_is_valid_point(C.c_char_p(b)))


@pytest.mark.parametrize("n", [1, 2, 5, 33, 189, 190, 600, 1024])
def test_msm_matches_naive(n):
    """vartime_multiscalar_mul (group.rs:98-117): Straus / Pippenger paths against sum of scalar mults"""
    gens = oc.MultiCommitGens.new(n, b"test-msm")
    sc = oc.prg_scalars("msm%d" % n, n)
    if n >= 3:
        sc[0] = 0
        sc[1] = oc.to_arr([1])[0]
        sc[2] = oc.to_arr([oc.Q - 1])[0]
    got = oc.msm(sc, gens.G)
    ints = oc.to_ints(sc)
    if n <= 33:
        acc = oc.Point.identity()
        for i in range(n):
            acc = acc + gens.g(i) * ints[i]
        assert got.compress() == acc.compress()
    # linearity: MSM(2s) == 2*MSM(s)
    got2 = oc.msm([(2 * v) % oc.Q for v in ints], gens.G)
    assert got2.compress() == (got + got).compress()


def test_msm_vs_libsodium():
    sod = _sodium()
    n = 16
    gens = oc.MultiCommitGens.new(n, b"sodium-msm")
    sc = oc.to_ints(oc.prg_scalars("s", n))
    o = C.create_string_buffer(32)
    acc = bytes(32)
    for i in range(n):
        sod.crypto_scalarmult_ristretto255(o, C.c_char_p(sc[i].to_bytes(32, "little")), C.c_char_p(gens.g(i).compress()))
        t = C.create_string_buffer(32)
        sod.crypto_core_ristretto255_add(t, C.c_char_p(acc), C.c_char_p(o.raw))
        acc = t.raw
    assert oc.msm(sc, gens.G).compress() == acc


def test_gens_prefix_sharing():
    """r1csproof.rs:48-58: gens_3 / gens_4 built from the same label share the SHAKE prefix of gens_n"""
    g5 = oc.MultiCommitGens.new(5, b"gens_r1cs_sat")
    g3 = oc.MultiCommitGens.new(3, b"gens_r1cs_sat")
    assert np.array_equal(g3.G, g5.G[:3])
    assert g3.h.compress() == g5.g(3).compress()
    # generator derivation is exactly the RFC one-way map of consecutive 64-byte SHAKE blocks (commitments.rs:15-33)
    stream = hashlib.shake_256(b"gens_r1cs_sat" + oc.BASEPOINT_COMPRESSED).digest(64 * 6)
    assert oc.Point.from_uniform_bytes(stream[64:128]).compress() == g5.g(1).compress()
    assert g5.h.compress() == oc.Point.from_uniform_bytes(stream[320:384]).compress()
