"""Host pieces of batch verification without a GPU (libsp_hosttest): the O(lg n) product that replaced the inner-product argument's n-term
a_hat sum, against that sum; and the weights of the deferred equations, against a hashlib restatement of their derivation."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

from oracle.spartan_ref import core as oc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    path = os.path.join(ROOT, "spartan_b200", "libsp_hosttest_fast.so")
    if not os.path.exists(path):
        import __graft_entry__ as ge
        ge.build_hosttest()
    l = C.CDLL(path)
    l.spt_batch_weight.argtypes = [C.c_char_p, C.c_uint64, C.c_uint64, C.c_char_p]
    l.spt_ipa_a_hat.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t, C.c_char_p]
    return l


@pytest.mark.parametrize("lg_n", [0, 1, 2, 3, 5, 8, 11])
def test_ipa_a_hat(lib, lg_n):
    rng = np.random.default_rng(lg_n)
    for _ in range(3):
        r = [int.from_bytes(rng.bytes(32), "little") % oc.Q for _ in range(lg_n)]
        u = [int.from_bytes(rng.bytes(32), "little") % oc.Q or 1 for _ in range(lg_n)]
        out = C.create_string_buffer(64)
        lib.spt_ipa_a_hat(b"".join(oc.mont_bytes(x) for x in r), b"".join(oc.mont_bytes(x) for x in u), lg_n, out)
        fast, slow = oc.from_mont_bytes(out.raw[:32]), oc.from_mont_bytes(out.raw[32:])
        assert fast == slow
        # and the closed form, in Python integers
        want = 1
        for rj, uj in zip(r, u):
            want = want * ((1 - rj) * oc.inv(uj) + rj * uj) % oc.Q
        assert fast == want


def test_batch_weight(lib):
    for seed in (bytes(32), bytes(range(32)), hashlib.sha256(b"s").digest()):
        for i, e in [(0, 0), (1, 0), (0, 1), (17, 123), (2**40 + 3, 2**33 + 5)]:
            out = C.create_string_buffer(32)
            lib.spt_batch_weight(seed, i, e, out)
            wide = hashlib.shake_256(b"spartan-b200/v1/batch-verify" + seed + i.to_bytes(8, "little") + e.to_bytes(8, "little")).digest(64)
            assert oc.from_mont_bytes(out.raw) == int.from_bytes(wide, "little") % oc.Q
