"""pytest plugin: run GPU tests under the memory-check mode of libspartan_b200.so and libsp_devtest.so (sp_debug_memcheck / spd_memcheck).

Not a conftest: load it explicitly, with tests/ on PYTHONPATH:

    PYTHONPATH=tests pytest -m gpu -p memcheck_plugin tests/test_gpu_kernels.py ...

Under the mode every device block either library hands out is filled first (field elements and points 0xFF, everything else zero), carries a
zero guard band past its end, and every context entry point refills the context's persistent scratch.  The tests' own oracle and golden
comparisons then fail on a read of memory the call did not write; a write past a buffer's end is a guard violation, which this plugin turns
into a failure of the test that caused it (found by the scan after its call, or at the free of the block in its teardown).  At the end of
the session it prints one line "memcheck {json}" with the counters of both libraries added up, and writes the same JSON to the file named
by SP_MEMCHECK_OUT when that is set.  Single GPU only.
"""
import ctypes as C
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

FIELDS = ("blocks_filled", "blocks_refilled", "context_refills", "guard_bytes_checked", "violations")


class _Devtest:
    """the mode of libsp_devtest.so's own copy of the pool (the same dlopen handle the kernel tests load)"""

    def __init__(self):
        self.lib = C.CDLL(os.path.join(ROOT, "spartan_b200", "libsp_devtest.so"))
        self.lib.spd_memcheck_scan.restype = C.c_ulonglong
        self.lib.spd_last_error.restype = C.c_char_p

    def enable(self, on):
        self.lib.spd_memcheck(C.c_int(1 if on else 0))

    def scan(self):
        n = int(self.lib.spd_memcheck_scan())
        if n == 2 ** 64 - 1:
            raise RuntimeError("spd_memcheck_scan: " + self.lib.spd_last_error().decode())
        return n

    def report(self):
        c = (C.c_ulonglong * 5)()
        buf = C.create_string_buffer(8192)
        assert self.lib.spd_memcheck_report(c, buf, C.c_size_t(len(buf))) == 0
        out = dict(zip(FIELDS, (int(x) for x in c)))
        out["first_violation"], _, out["last_violation"] = buf.value.decode().partition("\n")
        return out


class _Library:
    def __init__(self):
        import spartan_b200 as sb
        self.sb = sb

    def enable(self, on):
        self.sb.debug_memcheck(on)

    def scan(self):
        return self.sb.debug_memcheck_scan()

    def report(self):
        return self.sb.debug_memcheck_report()


class MemcheckPlugin:
    def __init__(self):
        self.libs = {"libspartan_b200.so": _Library(), "libsp_devtest.so": _Devtest()}
        for lib in self.libs.values():
            lib.enable(True)   # before any context or kernel-hook call exists
        self.seen = {name: lib.report()["violations"] for name, lib in self.libs.items()}

    def check(self, item, when, scan):
        """fail `item` when either library found a violation since the last check (the scan: its call's live blocks; the frees: its blocks)"""
        msgs = []
        for name, lib in self.libs.items():
            if scan:
                lib.scan()
            rep = lib.report()
            new = rep["violations"] - self.seen[name]
            self.seen[name] = rep["violations"]
            if new:
                msgs.append("%s: %d new guard violation(s), the latest: %s" % (name, new, rep["last_violation"]))
        if msgs:
            pytest.fail("memory check, %s of %s:\n%s" % (when, item.nodeid, "\n".join(msgs)), pytrace=False)

    @pytest.hookimpl(wrapper=True)
    def pytest_runtest_call(self, item):
        res = yield
        self.check(item, "after the call", scan=True)
        return res

    @pytest.hookimpl(wrapper=True)
    def pytest_runtest_teardown(self, item, nextitem):
        res = yield
        self.check(item, "in the teardown", scan=False)
        return res

    def totals(self):
        tot = dict.fromkeys(FIELDS, 0)
        for lib in self.libs.values():
            rep = lib.report()
            for k in FIELDS:
                tot[k] += rep[k]
        return tot

    def pytest_terminal_summary(self, terminalreporter):
        tot = self.totals()
        terminalreporter.write_line("memcheck " + json.dumps(tot, sort_keys=True))
        out = os.environ.get("SP_MEMCHECK_OUT")
        if out:
            with open(out, "w") as f:
                json.dump(tot, f)


def pytest_configure(config):
    config.pluginmanager.register(MemcheckPlugin(), "memcheck")
