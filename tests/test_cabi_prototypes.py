"""The Python layer states the C ABI only through include/spartan_b200.h: api.py takes every entry's prototype and every integer constant from
the header at import, so ctypes checks the arity and the types of each call, and api.py checks every status the library returns."""
import ast
import ctypes as C
import glob
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "spartan_b200.h")
API = os.path.join(ROOT, "spartan_b200", "api.py")
# the int-returning entries whose int is not a status: a count, a check scalar_from_bytes turns into R1CSError, one that raises on its own
NOT_A_STATUS = {"sp_device_count", "sp_scalar_from_bytes", "sp_debug_memcheck_report"}


def _header_text():
    return re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)


def _declared():
    return set(re.findall(r"\b(sp_\w+)\s*\(", _header_text()))


def test_hand_written_signatures():
    from spartan_b200 import api
    lib = api.lib
    assert list(lib.sp_poly_upload.argtypes) == [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    assert lib.sp_poly_upload.restype is C.c_int
    assert list(lib.sp_instance_synthetic.argtypes) == [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_uint64, C.c_void_p, C.c_void_p,
                                                        C.c_void_p]
    assert lib.sp_kernel_launches.restype is C.c_ulonglong
    assert lib.sp_last_error.restype is C.c_char_p
    assert lib.sp_free.restype is None
    assert lib.sp_poly_len.restype is C.c_size_t
    assert list(lib.sp_device_count.argtypes) == []
    assert list(lib.sp_comm_connect.argtypes) == [C.c_void_p, C.c_int, C.c_int, C.c_void_p]


@pytest.mark.parametrize("decl", ["float sp_free(void* p);", "int sp_free(long n);", "int sp_free();", "int sp_not_in_the_library(void);"])
def test_undeclarable_entries_fail_the_import(tmp_path, decl):
    """a type outside the mapping, an unnamed or missing parameter list, a name the library lacks: refused, not skipped"""
    from spartan_b200 import api
    header = tmp_path / "h.h"
    header.write_text("#define SP_X 1\n/* a comment sp_free(int); */\n%s\n" % decl)
    lib = C.CDLL(api._LIB_PATH)
    with pytest.raises(api.SpartanB200Error, match=re.escape(decl.rstrip(";"))):
        api._declare(lib, str(header))
    header.write_text("#define SP_X 1\n/* a comment sp_free(int); */\nvoid sp_free(void* p);\n")
    assert api._declare(lib, str(header)) == {"SP_X": 1} and list(lib.sp_free.argtypes) == [C.c_void_p]


def test_every_entry_has_a_prototype():
    from spartan_b200 import api
    declared = _declared()
    assert len(declared) >= 150
    for name in sorted(declared):
        assert getattr(api.lib, name).argtypes is not None, name


def test_python_layer_calls_only_declared_entries():
    used = set()
    for path in glob.glob(os.path.join(ROOT, "spartan_b200", "*.py")):
        used |= set(re.findall(r"\blib\.(sp_\w+)", open(path).read()))
    assert used and used <= _declared(), sorted(used - _declared())


def test_library_exports_only_declared_entries():
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm (binutils) is not installed")
    out = subprocess.run([nm, "-D", "--defined-only", os.path.join(ROOT, "spartan_b200", "libspartan_b200.so")], capture_output=True, text=True,
                         check=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.split() and line.split()[-1].startswith("sp_")}
    assert exported and exported <= _declared(), sorted(exported - _declared())


def test_ctypes_refuses_wrong_calls():
    """host-only entries: no device needed"""
    from spartan_b200 import api
    state = C.create_string_buffer(api.SP_TRANSCRIPT_STATE_BYTES)
    with pytest.raises(TypeError):
        api.lib.sp_transcript_new(b"x", 1)
    with pytest.raises(C.ArgumentError):
        api.lib.sp_transcript_new(b"x", "1", state)
    assert api.lib.sp_transcript_new(b"x", 1, state) == api.SP_OK


def test_str_labels_are_refused():
    import spartan_b200 as sb
    with pytest.raises(TypeError):
        sb.Transcript("x")
    with pytest.raises(TypeError):
        sb.Transcript(b"x").append_message("l", b"m")
    with pytest.raises(TypeError):
        sb.Transcript(b"x").challenge_bytes("l", 32)


def test_constants_come_from_the_header():
    from spartan_b200 import api
    defines = re.findall(r"^#define (SP_\w+) +(\d+) *$", _header_text(), re.M)
    assert len(defines) >= 20
    for name, value in defines:
        assert getattr(api, name) == int(value), name
    assert api.SP_TRANSCRIPT_STATE_BYTES == 203 and api.SP_ERR_INVALID_ARG == 3 and api.SP_PROD_MAX_SOURCES == 3


def test_every_status_is_checked():
    """an AST walk over api.py: every call of an int-returning lib.sp_* entry is the argument of ctx.check(...) or _check_host(...)"""
    from spartan_b200 import api

    def entry(node):
        f = node.func
        return f.attr if isinstance(f, ast.Attribute) and isinstance(f.value, ast.Name) and f.value.id == "lib" and f.attr.startswith("sp_") else None

    def checker(node):
        f = node.func
        return (isinstance(f, ast.Name) and f.id == "_check_host") or (isinstance(f, ast.Attribute) and f.attr == "check")

    calls = [n for n in ast.walk(ast.parse(open(API).read())) if isinstance(n, ast.Call)]
    checked = {id(a) for n in calls if checker(n) for a in n.args}
    unchecked, n_checked = [], 0
    for n in calls:
        name = entry(n)
        if name is None or getattr(api.lib, name).restype is not C.c_int:
            continue
        if id(n) in checked:
            n_checked += 1
        elif name not in NOT_A_STATUS:
            unchecked.append("%s (api.py:%d)" % (name, n.lineno))
    assert n_checked >= 100
    assert not unchecked, unchecked


@pytest.mark.gpu
def test_gpu_str_label_is_refused():
    import spartan_b200 as sb
    with pytest.raises(TypeError):
        sb.MultiCommitGens(4, "x")


@pytest.mark.gpu
def test_gpu_instance_export_refuses_a_bad_matrix():
    import spartan_b200 as sb
    inst, _, _ = sb.Instance.produce_synthetic_r1cs(256, 256, 10, seed=0)
    assert all(len(a) > 0 for a in inst.export(2))
    for m in (3, -1):
        with pytest.raises(sb.SpartanB200Error):
            inst.export(m)


@pytest.mark.gpu
def test_gpu_timings_after_a_snark_prove():
    import spartan_b200 as sb
    n = 1 << 12
    inst, vars_, inputs = sb.Instance.produce_synthetic_r1cs(n, n, 10, seed=0)
    gens = sb.SNARKGens(n, n, 10, n)
    comm = sb.SNARK.encode(inst, gens)
    sb.SNARK.prove(inst, comm, vars_, inputs, gens, b"example", sb.tape_seed(0))
    t = inst.ctx.timings()
    assert {"SNARK::prove", "R1CSProof::prove", "R1CSEvalProof::prove", "polycommit", "prove_sc_phase_one", "prove_sc_phase_two"} <= set(t), t
    assert all(v >= 0 for v in t.values())
