"""ctypes mirror of the reference's public API over libspartan_b200.so (see include/spartan_b200.h)."""
import ctypes as C
import hashlib
import os
import re
import zlib

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libspartan_b200.so")
_HEADER = os.path.join(_HERE, os.pardir, "include", "spartan_b200.h")


class SpartanB200Error(RuntimeError):
    pass


class ProofVerifyError(SpartanB200Error):
    """errors.rs:5-12: InternalError (a check failed) or DecompressionError (a point of the proof does not decompress).  `code`: the C status,
    SP_ERR_VERIFY or SP_ERR_DECOMPRESS"""

    def __init__(self, msg, code=None):
        super().__init__(msg)
        self.code = code


class R1CSError(SpartanB200Error):
    """errors.rs:28-41: InvalidIndex / InvalidScalar / InvalidNumberOfInputs"""


def _load():
    if not os.path.exists(_LIB_PATH):
        raise SpartanB200Error("libspartan_b200.so is not built (run `python -c 'import __graft_entry__ as g; g.build()'`); there is no CPU fallback")
    return C.CDLL(_LIB_PATH)


_RESTYPES = {"int": C.c_int, "void": None, "size_t": C.c_size_t, "unsigned long long": C.c_ulonglong, "const char*": C.c_char_p}
_ARGTYPES = {"int": C.c_int, "size_t": C.c_size_t, "uint64_t": C.c_uint64}


def _declare(lib, header):
    """Set restype and argtypes on `lib` for every sp_* function `header` declares, and return the header's `#define SP_<NAME> <decimal>`
    constants.  Pointer and array parameters become c_void_p, by-value ones map through _ARGTYPES, return types through _RESTYPES; any
    other type, or a declared name the library does not export, raises.  So ctypes refuses a call with too few arguments or an argument of
    the wrong type.  Two gaps remain: a call with extra trailing arguments is not refused (ctypes passes them on to a cdecl function), and a
    Python int too wide for a c_int parameter is truncated (2**40 arrives as 0), as C.c_int(2**40) truncates it."""
    with open(header) as f:
        text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", f.read(), flags=re.S)
    consts = {m[1]: int(m[2]) for m in re.finditer(r"^[ \t]*#[ \t]*define[ \t]+(SP_\w+)[ \t]+(\d+)[ \t]*$", text, re.M)}
    for decl in re.split(r"[;{}]", re.sub(r"^[ \t]*#.*$", " ", text, flags=re.M)):
        decl = " ".join(decl.split())
        if not re.search(r"\bsp_\w+ ?\(", decl):
            continue   # a typedef, a struct member, extern "C"
        m = re.fullmatch(r"(.+?) ?\b(sp_\w+) ?\((.*)\)", decl)
        try:
            fn = getattr(lib, m[2])
            fn.restype = _RESTYPES[m[1].replace(" *", "*")]
            params = [] if m[3] == "void" else [p.strip() for p in m[3].split(",")]
            fn.argtypes = [C.c_void_p if "*" in p or "[" in p else _ARGTYPES[p.rpartition(" ")[0]] for p in params]
        except (TypeError, KeyError, AttributeError):   # no match, a type outside the mapping, a name the library lacks
            raise SpartanB200Error("%s: cannot bind `%s` to %s" % (header, decl, _LIB_PATH)) from None
    return consts


lib = _load()
globals().update(_declare(lib, _HEADER))
_vp, _sz = C.c_void_p, C.c_size_t


def kernel_launches():
    return int(lib.sp_kernel_launches())


def release_cached_memory():
    """return the device blocks this process keeps for reuse to the driver (drop the Python objects first); bytes released"""
    return int(lib.sp_release_cached_memory())


class _MemcheckCounts(C.Structure):
    _fields_ = [(n, C.c_ulonglong) for n in ("blocks_filled", "blocks_refilled", "context_refills", "guard_bytes_checked", "violations")]


def debug_memcheck(on=True):
    """process-wide memory-check mode (sp_debug_memcheck, single GPU): every device block filled when handed out and guarded past its end, the
    contexts' persistent scratch refilled at every call.  Switch it on before the first Context is created"""
    lib.sp_debug_memcheck(1 if on else 0)


def debug_memcheck_scan():
    """synchronise the device and check every live block's guard band; returns the violations found"""
    n = int(lib.sp_debug_memcheck_scan())
    if n == 2 ** 64 - 1:
        raise SpartanB200Error("sp_debug_memcheck_scan: " + lib.sp_last_error(None).decode())
    return n


def debug_memcheck_report():
    """the mode's counters since load, and the first and the latest violation's message ("" when there was none)"""
    c = _MemcheckCounts()
    buf = C.create_string_buffer(8192)
    if lib.sp_debug_memcheck_report(C.byref(c), buf, len(buf)) != SP_OK:
        raise SpartanB200Error("sp_debug_memcheck_report: message longer than the buffer")
    out = {n: int(getattr(c, n)) for n, _ in _MemcheckCounts._fields_}
    first, _, last = buf.value.decode().partition("\n")
    out["first_violation"], out["last_violation"] = first, last
    return out


def _p(a):
    return a.ctypes.data_as(_vp) if isinstance(a, np.ndarray) else a


def _limbs(a):
    """(n,4) uint64 contiguous view of Montgomery limbs"""
    a = np.ascontiguousarray(a, dtype=np.uint64)
    return a.reshape(-1, 4)


def _status_error(rc, msg):
    """the exception for a failed call's status and message"""
    if rc == SP_ERR_INVALID_INDEX:
        return R1CSError("InvalidIndex: " + msg)
    if rc == SP_ERR_INVALID_SCALAR:
        return R1CSError("InvalidScalar: " + msg)
    if rc == SP_ERR_INVALID_INPUTS:
        return R1CSError("InvalidNumberOfInputs: " + msg)
    if rc == SP_ERR_VERIFY:
        return ProofVerifyError("InternalError: " + msg, rc)
    if rc == SP_ERR_DECOMPRESS:
        return ProofVerifyError("DecompressionError: " + msg, rc)
    return SpartanB200Error("spartan_b200 error %d: %s" % (rc, msg))


def _check_host(rc):
    """raises for a failed host-only call, whose message sp_last_error(NULL) holds"""
    if rc != SP_OK:
        raise _status_error(rc, lib.sp_last_error(None).decode())


def _string_out(check, entry, *args):
    """the string entry(*args, buf, buflen) writes, with the buffer doubled while the entry refuses it as too short (SP_ERR_INVALID_ARG);
    `check` raises for any other failure"""
    n = 4096
    while True:
        buf = C.create_string_buffer(n)
        rc = entry(*args, buf, n)
        if rc != SP_ERR_INVALID_ARG:
            check(rc)
            return buf.value.decode()
        n *= 2


class _Handle:
    """owner of one library object `h`, released by the class's `_free` when the Python object goes"""
    _free = None

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self._free(self.h)
                self.h = None
        except Exception:
            pass


class Context(_Handle):
    """One per GPU / host thread.  Fails loudly when no CUDA device is present."""
    _free = lib.sp_ctx_destroy

    def __init__(self, device=0):
        h = _vp()
        _check_host(lib.sp_ctx_create(device, C.byref(h)))
        self.h = h
        self.device = device

    def check(self, rc):
        if rc != SP_OK:
            raise _status_error(rc, lib.sp_last_error(self.h).decode())

    def connect_peers(self, rank, world, allgather):
        """Join `world` single-GPU processes into one sharded prover (sp_comm_export / sp_comm_connect).  `allgather(b: bytes) -> list[bytes]`
        is the host-side exchange (every rank contributes its handle, all get the list in rank order): spartan_b200.dist.allgather_bytes under
        torch.distributed.  Afterwards NIZK.prove / SNARK.prove must be called by every rank with the same arguments."""
        hb = lib.sp_comm_handle_bytes()
        mine = C.create_string_buffer(hb)
        self.check(lib.sp_comm_export(self.h, mine))
        handles = allgather(mine.raw)
        assert len(handles) == world and all(len(h) == hb for h in handles)
        self.check(lib.sp_comm_connect(self.h, rank, world, b"".join(handles)))
        self.rank, self.world = rank, world

    def set_sharding(self, enabled):
        """switch sharded proving off / on for a connected context (every rank must switch together)"""
        self.check(lib.sp_comm_set_enabled(self.h, 1 if enabled else 0))

    def set_overlap(self, enabled):
        """background-stream commitment of the dereferenced values in SNARK.prove on / off (off: every kernel on one stream, for per-kernel profiling)"""
        self.check(lib.sp_ctx_set_overlap(self.h, 1 if enabled else 0))

    def timings(self):
        out = {}
        for item in _string_out(self.check, lib.sp_timings, self.h).split(";"):
            if "=" in item:
                k, v = item.split("=")
                out[k] = float(v)
        return out


_default_ctx = None


def default_context():
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context(int(os.environ.get("LOCAL_RANK", "0")) if lib.sp_device_count() > 1 else 0)
    return _default_ctx


# ----------------------------------------------------------------------------- scalars
def scalar_from_bytes(b):
    """Scalar::from_bytes (ristretto255.rs:391): canonical 32 bytes -> Montgomery limbs; raises on non-canonical input"""
    out = np.zeros(4, dtype=np.uint64)
    if lib.sp_scalar_from_bytes(bytes(b), _p(out)) != SP_OK:
        raise R1CSError("InvalidScalar")
    return out


def scalar_to_bytes(limbs):
    out = C.create_string_buffer(32)
    lib.sp_scalar_to_bytes(_p(np.ascontiguousarray(limbs, dtype=np.uint64)), out)
    return out.raw


def prg_scalars(tag, n, seed=0):
    """DESIGN.md deterministic inputs: SHAKE256("spartan-b200/v1/" || tag || LE64(seed)) -> from_bytes_wide, as Montgomery limbs"""
    raw = hashlib.shake_256(b"spartan-b200/v1/" + tag.encode() + int(seed).to_bytes(8, "little")).digest(64 * n)
    out = np.zeros((n, 4), dtype=np.uint64)
    for i in range(n):
        lib.sp_scalar_from_bytes_wide(raw[64 * i:64 * i + 64], _p(out[i]))
    return out


def tape_seed(seed=0):
    """a DETERMINISTIC RandomTape seed (tests / benchmarks / byte-parity runs only): every blind of the proof becomes a public function
    of `seed`, so a proof made with it is not zero-knowledge.  Real proofs use random_tape_seed() (the default of NIZK.prove / SNARK.prove)."""
    return prg_scalars("tape", 1, seed)[0]


def random_tape_seed():
    """the scalar RandomTape::new draws from OsRng (random.rs:13-15): 64 bytes of OS randomness -> Scalar::from_bytes_wide"""
    out = np.zeros(4, dtype=np.uint64)
    lib.sp_scalar_from_bytes_wide(os.urandom(64), _p(out))
    return out


# ----------------------------------------------------------------------------- device arrays from torch
def _torch():
    import torch   # only the tensor entry points need torch: the module imports without it
    return torch


def _device_tensor(t, ctx, name, dtype, width=None):
    """t as a contiguous tensor of `dtype` on ctx.device: 1-D, or (n, width) when width is given"""
    torch = _torch()
    if not isinstance(t, torch.Tensor):
        raise SpartanB200Error("%s: expected a torch.Tensor, got %s" % (name, type(t).__name__))
    if t.device.type != "cuda" or t.device.index != ctx.device:
        raise SpartanB200Error("%s: expected a tensor on cuda:%d, got one on %s" % (name, ctx.device, t.device))
    if t.dtype != dtype:
        raise SpartanB200Error("%s: expected dtype %s, got %s" % (name, dtype, t.dtype))
    if (width is None and t.dim() != 1) or (width is not None and (t.dim() != 2 or t.shape[1] != width)):
        raise SpartanB200Error("%s: expected shape %s, got %s" % (name, "(n,)" if width is None else "(n, %d)" % width, tuple(t.shape)))
    return t.contiguous()


def _sync_torch(ctx):
    """the library reads the tensors on its own stream: whatever torch queued to write them must have finished"""
    torch = _torch()
    torch.cuda.current_stream(ctx.device).synchronize()


# ----------------------------------------------------------------------------- operator level
class DensePolynomial(_Handle):
    """dense_mlpoly.rs:18-22 with Z resident on the device"""
    _free = lib.sp_poly_free

    def __init__(self, Z, ctx=None):
        self.ctx = ctx or default_context()
        Z = _limbs(Z)
        h = _vp()
        self.ctx.check(lib.sp_poly_upload(self.ctx.h, _p(Z), len(Z), C.byref(h)))
        self.h = h

    @classmethod
    def _wrap(cls, ctx, h):
        o = cls.__new__(cls)
        o.ctx, o.h = ctx, h
        return o

    @classmethod
    def from_tensor(cls, vals, ctx=None):
        """Z from a (n, 32) uint8 CUDA tensor of canonical little-endian scalars on ctx.device (e.g. a witness computed by torch), converted to
        Montgomery form on the device; raises R1CSError (InvalidScalar) if a value is >= q"""
        ctx = ctx or default_context()
        vals = _device_tensor(vals, ctx, "vals", _torch().uint8, 32)
        _sync_torch(ctx)
        h = _vp()
        ctx.check(lib.sp_poly_from_canonical_device(ctx.h, _vp(vals.data_ptr()), vals.shape[0], C.byref(h)))
        return cls._wrap(ctx, h)

    def len(self):
        return int(lib.sp_poly_len(self.h))

    def to_numpy(self):
        out = np.zeros((self.len(), 4), dtype=np.uint64)
        self.ctx.check(lib.sp_poly_download(self.ctx.h, self.h, _p(out), len(out)))
        return out

    def bound_poly_var_top(self, r):
        arr = (_vp * 1)(self.h)
        self.ctx.check(lib.sp_fold_top(self.ctx.h, arr, 1, _p(np.ascontiguousarray(r, dtype=np.uint64))))

    def evaluate(self, r):
        r = _limbs(r)
        out = np.zeros(4, dtype=np.uint64)
        self.ctx.check(lib.sp_poly_evaluate(self.ctx.h, self.h, _p(r), len(r), _p(out)))
        return out

    def bound(self, L):
        L = _limbs(L)
        h = _vp()
        self.ctx.check(lib.sp_poly_bound_rows(self.ctx.h, self.h, _p(L), len(L), C.byref(h)))
        return DensePolynomial._wrap(self.ctx, h)

    def dot(self, other):
        out = np.zeros(4, dtype=np.uint64)
        self.ctx.check(lib.sp_dot(self.ctx.h, self.h, other.h, _p(out)))
        return out

    def commit(self, gens, L, R, blinds=None):
        """DensePolynomial::commit_inner (dense_mlpoly.rs:148-177) -> list of L compressed points"""
        out = C.create_string_buffer(32 * L)
        bl = _limbs(blinds) if blinds is not None else None
        self.ctx.check(lib.sp_commit_rows(self.ctx.h, gens.h, self.h, L, R, _p(bl) if bl is not None else None, out))
        return [out.raw[32 * i:32 * i + 32] for i in range(L)]

    @staticmethod
    def eq_evals(r, ctx=None):
        ctx = ctx or default_context()
        r = _limbs(r)
        h = _vp()
        ctx.check(lib.sp_eq_evals(ctx.h, _p(r), len(r), C.byref(h)))
        return DensePolynomial._wrap(ctx, h)


def sumcheck_eval(kind, polys):
    ctx = polys[0].ctx
    arr = (_vp * len(polys))(*[p.h for p in polys])
    out = np.zeros((3, 4), dtype=np.uint64)
    ctx.check(lib.sp_sumcheck_eval(ctx.h, kind, arr, _p(out)))
    return out


def sumcheck_fold_eval(kind, polys, r):
    ctx = polys[0].ctx
    arr = (_vp * len(polys))(*[p.h for p in polys])
    out = np.zeros((3, 4), dtype=np.uint64)
    ctx.check(lib.sp_sumcheck_fold_eval(ctx.h, kind, arr, _p(np.ascontiguousarray(r, dtype=np.uint64)), _p(out)))
    return out


def sumcheck_eval_sharded(kind, polys):
    """sumcheck_eval on cyclic shards held by the ranks of a connected context: returns the evaluations of the whole tables on every rank"""
    ctx = polys[0].ctx
    out = np.zeros((3, 4), dtype=np.uint64)
    ctx.check(lib.sp_sumcheck_eval_sharded(ctx.h, kind, (_vp * len(polys))(*[p.h for p in polys]), _p(out)))
    return out


def sumcheck_fold_eval_sharded(kind, polys, r):
    ctx = polys[0].ctx
    out = np.zeros((3, 4), dtype=np.uint64)
    ctx.check(lib.sp_sumcheck_fold_eval_sharded(ctx.h, kind, (_vp * len(polys))(*[p.h for p in polys]), _p(np.ascontiguousarray(r, dtype=np.uint64)), _p(out)))
    return out


def _handles(polys):
    return (_vp * len(polys))(*[p.h for p in polys])


def sumcheck_batched_eval(As, Bs, Cs):
    """prove_cubic_batched evaluation loops (sumcheck.rs:290-357) for len(As) instances of A*B*C; returns (ninst, 3, 4) limbs [e0, e2, e3]"""
    ctx = As[0].ctx
    out = np.zeros((len(As), 3, 4), dtype=np.uint64)
    ctx.check(lib.sp_sumcheck_batched_eval(ctx.h, len(As), _handles(As), _handles(Bs), _handles(Cs), _p(out)))
    return out


def sumcheck_batched_fold_eval(As, Bs, Cs, r):
    """bind the top variable of every table with r (a C shared by several instances once) and evaluate the next round"""
    ctx = As[0].ctx
    out = np.zeros((len(As), 3, 4), dtype=np.uint64)
    ctx.check(lib.sp_sumcheck_batched_fold_eval(ctx.h, len(As), _handles(As), _handles(Bs), _handles(Cs), _p(np.ascontiguousarray(r, dtype=np.uint64)), _p(out)))
    return out


def fold_top(polys, r):
    ctx = polys[0].ctx
    arr = (_vp * len(polys))(*[p.h for p in polys])
    ctx.check(lib.sp_fold_top(ctx.h, arr, len(polys), _p(np.ascontiguousarray(r, dtype=np.uint64))))


class _ScTerm(C.Structure):
    _fields_ = [("coeff_mont", C.c_uint64 * 4), ("nfactors", C.c_uint32), ("factor", C.c_uint32 * SP_SC_MAX_DEGREE)]


class Composition:
    """g = sum_t coeff_t * prod_{j in factors_t} P_j, the comb_func of a sumcheck as data: `terms` is a list of (coeff_limbs, (i, j, ..)) with
    coeff_limbs the coefficient's Montgomery limbs and (i, j, ..) table indices (a table may repeat: (0, 0, 1) is A*A*B)."""

    def __init__(self, terms):
        self.terms = [(np.ascontiguousarray(c, dtype=np.uint64).reshape(4), tuple(int(i) for i in f)) for c, f in terms]

    @property
    def degree(self):
        return max((len(f) for _, f in self.terms), default=0)

    def _c_terms(self):
        arr = (_ScTerm * max(len(self.terms), 1))()
        for t, (c, f) in enumerate(self.terms):
            arr[t].coeff_mont[:] = [int(x) for x in c]
            arr[t].nfactors = len(f)   # more than SP_SC_MAX_DEGREE factors: the count alone reaches the library, which refuses it
            for i, j in enumerate(f[:SP_SC_MAX_DEGREE]):
                arr[t].factor[i] = j
        return arr


def _transcript_state(transcript):
    """a Transcript object (advanced in place) or a label (Transcript::new(label), discarded afterwards)"""
    return transcript if isinstance(transcript, Transcript) else Transcript(bytes(transcript))


def sumcheck_prove(polys, comp, claim, num_rounds, transcript):
    """SumcheckInstanceProof::prove_cubic / prove_cubic_batched with comb_func = `comp` (a Composition) over the tables `polys`
    (DensePolynomials of one length, bound in place).  Returns (proof_bytes = bincode(SumcheckInstanceProof), r as (num_rounds, 4) limbs,
    finals = P_j[0] of every table as (k, 4) limbs, e = the final claim's limbs)."""
    ctx = polys[0].ctx
    t = _transcript_state(transcript)
    terms = comp._c_terms()
    out, n = C.POINTER(C.c_ubyte)(), _sz()
    r = np.zeros((num_rounds, 4), dtype=np.uint64)
    finals = np.zeros((len(polys), 4), dtype=np.uint64)
    e = np.zeros(4, dtype=np.uint64)
    ctx.check(lib.sp_sumcheck_prove_t(ctx.h, _handles(polys), len(polys), terms, len(comp.terms),
                                      _p(np.ascontiguousarray(claim, dtype=np.uint64)), num_rounds, t.state, C.byref(out), C.byref(n), _p(r),
                                      _p(finals), _p(e)))
    return _take_bytes(out, n), r, finals, e


def sumcheck_verify(proof, claim, num_rounds, degree_bound, transcript):
    """SumcheckInstanceProof::verify (sumcheck.rs:27-62), on the host: returns (e, r) as Montgomery limbs, raises ProofVerifyError.  The
    transcript (a Transcript object) is advanced as the reference's verify advances it, accepted or not."""
    t = _transcript_state(transcript)
    proof = bytes(proof)
    e = np.zeros(4, dtype=np.uint64)
    r = np.zeros((num_rounds, 4), dtype=np.uint64)
    _check_host(lib.sp_sumcheck_verify_t(None, proof, len(proof), _p(np.ascontiguousarray(claim, dtype=np.uint64)), num_rounds,
                                         degree_bound, t.state, _p(e), _p(r)))
    return e, r


class MultiCommitGens(_Handle):
    """commitments.rs:8-33"""
    _free = lib.sp_gens_free

    def __init__(self, n, label, ctx=None):
        self.ctx = ctx or default_context()
        self.n = n
        h = _vp()
        self.ctx.check(lib.sp_gens_create(self.ctx.h, bytes(label), len(label), n, C.byref(h)))
        self.h = h

    @classmethod
    def from_points(cls, compressed, ctx=None):
        """the caller's own generators: n+1 ristretto255 encodings, G[0..n) then h (e.g. a `scale`d MultiCommitGens, commitments.rs:43-49)"""
        o = cls.__new__(cls)
        o.ctx = ctx or default_context()
        o.n = len(compressed) - 1
        h = _vp()
        o.ctx.check(lib.sp_gens_upload(o.ctx.h, b"".join(compressed), o.n, C.byref(h)))
        o.h = h
        return o

    def export(self):
        out = C.create_string_buffer(32 * (self.n + 1))
        self.ctx.check(lib.sp_gens_export(self.ctx.h, self.h, out))
        return [out.raw[32 * i:32 * i + 32] for i in range(self.n + 1)]

    def msm(self, scalars):
        """GroupElement::vartime_multiscalar_mul(scalars, G).compress()"""
        s = _limbs(scalars)
        out = C.create_string_buffer(32)
        self.ctx.check(lib.sp_msm(self.ctx.h, self.h, _p(s), len(s), out))
        return out.raw


class BulletReduction(_Handle):
    """operator-level BulletReductionProof::prove (nizk/bullet.rs:32-132): the device keeps a, b and the (implicitly folded) generators, the
    caller keeps the transcript.  round_LR() -> (L, R) compressed; fold(u, u_inv); finish() -> (a_hat, b_hat, G_hat compressed)."""
    _free = lib.sp_ipa_free

    def __init__(self, gens, a_vec, b_vec):
        self.ctx = gens.ctx
        h = _vp()
        self.ctx.check(lib.sp_ipa_begin(self.ctx.h, gens.h, a_vec.h, b_vec.h, C.byref(h)))
        self.h = h

    def round_LR(self, Q, H, blind_L, blind_R):
        L, R = C.create_string_buffer(32), C.create_string_buffer(32)
        self.ctx.check(lib.sp_ipa_round_LR(self.ctx.h, self.h, bytes(Q), bytes(H), _p(np.ascontiguousarray(blind_L, dtype=np.uint64)),
                                           _p(np.ascontiguousarray(blind_R, dtype=np.uint64)), L, R))
        return L.raw, R.raw

    def fold(self, u, u_inv):
        self.ctx.check(lib.sp_ipa_fold(self.ctx.h, self.h, _p(np.ascontiguousarray(u, dtype=np.uint64)), _p(np.ascontiguousarray(u_inv, dtype=np.uint64))))

    def finish(self):
        a, b, g = np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64), C.create_string_buffer(32)
        self.ctx.check(lib.sp_ipa_finish(self.ctx.h, self.h, _p(a), _p(b), g))
        return a, b, g.raw


class Points(_Handle):
    """A caller-supplied `&[GroupElement]` (group.rs:8-9) resident on the device, for the variable-base MSM (bucket method, no tables)."""
    _free = lib.sp_points_free

    def __init__(self, compressed, ctx=None):
        """compressed: list of 32-byte ristretto255 encodings; raises if any does not decompress"""
        self.ctx = ctx or default_context()
        h = _vp()
        self.ctx.check(lib.sp_points_upload(self.ctx.h, b"".join(compressed), len(compressed), C.byref(h)))
        self.h = h

    @classmethod
    def derive(cls, n, label, ctx=None):
        """MultiCommitGens::new(n, label).G without window tables (commitments.rs:15-33)"""
        o = cls.__new__(cls)
        o.ctx = ctx or default_context()
        h = _vp()
        o.ctx.check(lib.sp_points_derive(o.ctx.h, bytes(label), len(label), n, C.byref(h)))
        o.h = h
        return o

    def __len__(self):
        return int(lib.sp_points_len(self.h))

    def export(self, offset=0, n=None):
        n = len(self) - offset if n is None else n
        out = C.create_string_buffer(32 * n + 1)
        self.ctx.check(lib.sp_points_export(self.ctx.h, self.h, offset, n, out))
        return [out.raw[32 * i:32 * i + 32] for i in range(n)]

    def msm(self, scalars, offset=0):
        """GroupElement::vartime_multiscalar_mul(scalars, points[offset:offset+len(scalars)]).compress()  (group.rs:98-117)"""
        out = C.create_string_buffer(32)
        if isinstance(scalars, DensePolynomial):
            self.ctx.check(lib.sp_msm_var_resident(self.ctx.h, self.h, offset, scalars.h, out))
        else:
            s = _limbs(scalars)
            self.ctx.check(lib.sp_msm_var(self.ctx.h, self.h, offset, _p(s), len(s), out))
        return out.raw

    def msm_sharded(self, scalars, offset=0):
        """this rank's slice of a vector split by index range over the ranks of a connected context -> encoding of the whole sum (on every rank)"""
        out = C.create_string_buffer(32)
        self.ctx.check(lib.sp_msm_var_sharded(self.ctx.h, self.h, offset, scalars.h, out))
        return out.raw


def point_roundtrip(points, ctx=None):
    ctx = ctx or default_context()
    n = len(points)
    out = C.create_string_buffer(32 * n)
    ctx.check(lib.sp_point_roundtrip(ctx.h, b"".join(points), n, out))
    return [out.raw[32 * i:32 * i + 32] for i in range(n)]


def point_decompress_check(points, ctx=None):
    ctx = ctx or default_context()
    n = len(points)
    ok = (C.c_int * n)()
    ctx.check(lib.sp_point_decompress_check(ctx.h, b"".join(points), n, ok))
    return [bool(x) for x in ok]


class Transcript:
    """merlin::Transcript as the caller-owned object the reference's prove / verify mutate (`transcript: &mut Transcript`, lib.rs:339-347):
    the 203-byte STROBE-128 state, advanced in place by NIZK.prove / SNARK.prove / verify when passed instead of a label."""

    def __init__(self, label):
        self.state = C.create_string_buffer(SP_TRANSCRIPT_STATE_BYTES)
        _check_host(lib.sp_transcript_new(bytes(label), len(label), self.state))

    def append_message(self, label, msg):
        msg = bytes(msg)
        _check_host(lib.sp_transcript_append_message(self.state, bytes(label), len(label), msg, len(msg)))

    def challenge_bytes(self, label, n):
        out = C.create_string_buffer(n)
        _check_host(lib.sp_transcript_challenge_bytes(self.state, bytes(label), len(label), out, n))
        return out.raw


# ----------------------------------------------------------------------------- polynomial commitments of the caller's tables
class PolyCommitmentGens(_Handle):
    """PolyCommitmentGens::new(num_vars, label) (dense_mlpoly.rs:29-36): the n = 2^(num_vars - num_vars/2) generators of gens_n, G_1 and h of the
    label's stream, with their device tables (footprint: include/spartan_b200.h, sp_pc_gens_create).  view(num_vars) gives the gens of a smaller
    num_vars of the same label as a view of these tables."""
    _free = lib.sp_pc_gens_free

    def __init__(self, num_vars, label, ctx=None):
        self.ctx = ctx or default_context()
        self.num_vars, self.n = num_vars, 1 << (num_vars - num_vars // 2)
        h = _vp()
        self.ctx.check(lib.sp_pc_gens_create(self.ctx.h, num_vars, bytes(label), len(label), C.byref(h)))
        self.h = h

    def view(self, num_vars):
        o = PolyCommitmentGens.__new__(PolyCommitmentGens)
        o.ctx, o.num_vars, o.n = self.ctx, num_vars, 1 << (num_vars - num_vars // 2)
        h = _vp()
        self.ctx.check(lib.sp_pc_gens_create_from(self.ctx.h, self.h, num_vars, C.byref(h)))
        o.h = h
        return o


class RandomTape(Transcript):
    """RandomTape::new(b"proof") (random.rs:10-17) as caller state (a merlin transcript, advanced in place by the calls that draw from it).
    seed=None draws the seed scalar from the OS, as the reference does; a given seed (Montgomery limbs, e.g. tape_seed(i)) makes every blind a
    public function of it: byte-parity tests only."""

    def __init__(self, seed=None):
        s = random_tape_seed() if seed is None else np.ascontiguousarray(seed, dtype=np.uint64).reshape(4)
        self.state = C.create_string_buffer(SP_TRANSCRIPT_STATE_BYTES)
        _check_host(lib.sp_random_tape_new(_p(s), self.state))


class PolyCommitment:
    """dense_mlpoly.rs:38-41: the L compressed row commitments"""

    def __init__(self, C_rows):
        self.C = list(C_rows)

    def to_bytes(self):
        """bincode(PolyCommitment)"""
        return len(self.C).to_bytes(8, "little") + b"".join(self.C)

    @classmethod
    def from_bytes(cls, data):
        data = bytes(data)
        n = int.from_bytes(data[:8], "little")
        if len(data) != 8 + 32 * n:
            raise SpartanB200Error("PolyCommitment: %d bytes do not hold %d points" % (len(data), n))
        return cls([data[8 + 32 * i:40 + 32 * i] for i in range(n)])

    def append_to_transcript(self, label, transcript):
        """dense_mlpoly.rs:292-300, on a Transcript"""
        transcript.append_message(label, b"poly_commitment_begin")
        for c in self.C:
            transcript.append_message(b"poly_commitment_share", c)
        transcript.append_message(label, b"poly_commitment_end")


def _poly_list(polys):
    return [polys] if isinstance(polys, DensePolynomial) else list(polys)


def _opt_limbs(x):
    return None if x is None else _p(np.ascontiguousarray(x, dtype=np.uint64))


def poly_commit(polys, gens, tape=None):
    """DensePolynomial::commit(gens, tape) (dense_mlpoly.rs:179-204) of one DensePolynomial, or of DensePolynomial::merge of a list of them
    (concatenated, zero-padded to a power of two; dense_mlpoly.rs:259-272).  tape: a RandomTape (advanced) or None (no blinds).
    Returns (PolyCommitment, blinds as (L, 4) Montgomery limbs)."""
    polys = _poly_list(polys)
    ctx = gens.ctx
    k = len(polys)
    ell = (max(polys[0].len(), 1).bit_length() - 1 + (k - 1).bit_length()) if k else 0   # log2 of the merge's length
    blinds = np.zeros((1 << (ell // 2), 4), dtype=np.uint64)
    out, n = C.POINTER(C.c_ubyte)(), _sz()
    ctx.check(lib.sp_pc_commit(ctx.h, gens.h, _handles(polys), k, tape.state if tape is not None else None, C.byref(out), C.byref(n), _p(blinds)))
    return PolyCommitment.from_bytes(_take_bytes(out, n)), blinds


class PolyEvalProof:
    """dense_mlpoly.rs:307-404, plus DerefsEvalProof::prove_single / verify_single (sparse_mlpoly.rs:80-176) as prove_joint / verify_joint.
    `data` = bincode(PolyEvalProof).  Transcripts: a Transcript (advanced in place) or a label (a fresh Transcript::new(label))."""

    def __init__(self, data):
        self.data = bytes(data)

    @staticmethod
    def prove(poly, blinds, r, Zr, blind_Zr, gens, transcript, tape):
        """PolyEvalProof::prove: returns (proof, C_Zr compressed, Zr limbs).  Zr=None: Z(r), computed on the device; blinds / blind_Zr None: zero"""
        ctx = poly.ctx
        t, r = _transcript_state(transcript), _limbs(r)
        out, n = C.POINTER(C.c_ubyte)(), _sz()
        c_zr, zr = C.create_string_buffer(32), np.zeros(4, dtype=np.uint64)
        ctx.check(lib.sp_pc_eval_prove_t(ctx.h, gens.h, poly.h, _opt_limbs(blinds), _p(r), len(r), _opt_limbs(Zr), _opt_limbs(blind_Zr), t.state,
                                         tape.state, C.byref(out), C.byref(n), c_zr, _p(zr)))
        return PolyEvalProof(_take_bytes(out, n)), c_zr.raw, zr

    def verify(self, gens, transcript, r, C_Zr, comm):
        """PolyEvalProof::verify against the commitment C_Zr (32 bytes); raises ProofVerifyError"""
        self._verify(gens, transcript, r, bytes(C_Zr), None, comm)

    def verify_plain(self, gens, transcript, r, Zr, comm):
        """PolyEvalProof::verify_plain against the evaluation Zr (limbs); raises ProofVerifyError"""
        self._verify(gens, transcript, r, None, _p(np.ascontiguousarray(Zr, dtype=np.uint64)), comm)

    def _verify(self, gens, transcript, r, c_zr, zr, comm):
        t, r, cb = _transcript_state(transcript), _limbs(r), comm.to_bytes()
        gens.ctx.check(lib.sp_pc_eval_verify_t(gens.ctx.h, gens.h, cb, len(cb), _p(r), len(r), c_zr, zr, t.state, self.data, len(self.data)))

    @staticmethod
    def prove_joint(polys, blinds, r, gens, transcript, tape):
        """k tables opened at one point r through their joint commitment (poly_commit of the same list): returns (proof, evals as (k, 4) limbs)"""
        polys = _poly_list(polys)
        ctx = polys[0].ctx
        t, r = _transcript_state(transcript), _limbs(r)
        out, n = C.POINTER(C.c_ubyte)(), _sz()
        evals = np.zeros((len(polys), 4), dtype=np.uint64)
        ctx.check(lib.sp_pc_eval_prove_joint_t(ctx.h, gens.h, _handles(polys), len(polys), _opt_limbs(blinds), _p(r), len(r), t.state,
                                               tape.state, C.byref(out), C.byref(n), _p(evals)))
        return PolyEvalProof(_take_bytes(out, n)), evals

    def verify_joint(self, gens, transcript, r, evals, comm):
        """DerefsEvalProof::verify_single for prove_joint's proof; raises ProofVerifyError"""
        t, r, ev, cb = _transcript_state(transcript), _limbs(r), _limbs(evals), comm.to_bytes()
        gens.ctx.check(lib.sp_pc_eval_verify_joint_t(gens.ctx.h, gens.h, cb, len(cb), _p(r), len(r), _p(ev), len(ev), t.state, self.data, len(self.data)))


# ----------------------------------------------------------------------------- zero-knowledge sumchecks and sigma protocols
def _scalar(x):
    return _p(np.ascontiguousarray(x, dtype=np.uint64).reshape(4))


def _point(c):
    c = bytes(c)
    if len(c) != 32:
        raise SpartanB200Error("a commitment is 32 bytes, got %d" % len(c))
    return c


class ZKSumcheckInstanceProof:
    """sumcheck.rs:64-776: the zero-knowledge sumcheck of a Composition over DensePolynomials (bound in place), every round polynomial and
    evaluation hidden in a Pedersen commitment and tied together by a DotProductProof.  `data` = bincode(ZKSumcheckInstanceProof).  Scalars are
    Montgomery limbs, commitments 32-byte encodings; gens_1 / gens_n are MultiCommitGens with n = 1 and n = degree + 1."""

    def __init__(self, data):
        self.data = bytes(data)

    @staticmethod
    def prove(polys, comp, claim, blind_claim, num_rounds, gens_1, gens_n, transcript, tape):
        """prove_quad / prove_cubic_with_additive_term for any composition: returns (proof, r as (num_rounds, 4) limbs, finals as (k, 4) limbs,
        blind_post = the blind of the last comm_eval)"""
        ctx = polys[0].ctx
        terms = comp._c_terms()
        out, n = C.POINTER(C.c_ubyte)(), _sz()
        r = np.zeros((num_rounds, 4), dtype=np.uint64)
        finals = np.zeros((len(polys), 4), dtype=np.uint64)
        blind_post = np.zeros(4, dtype=np.uint64)
        ctx.check(lib.sp_zk_sumcheck_prove_t(ctx.h, _handles(polys), len(polys), terms, len(comp.terms), _scalar(claim),
                                             _scalar(blind_claim), num_rounds, gens_1.h, gens_n.h, transcript.state, tape.state, C.byref(out),
                                             C.byref(n), _p(r), _p(finals), _p(blind_post)))
        return ZKSumcheckInstanceProof(_take_bytes(out, n)), r, finals, blind_post

    def verify(self, comm_claim, num_rounds, degree_bound, gens_1, gens_n, transcript):
        """sumcheck.rs:84-179: returns (comm_eval = the last round's commitment, r); raises ProofVerifyError"""
        ctx = gens_1.ctx
        comm_eval = C.create_string_buffer(32)
        r = np.zeros((max(num_rounds, 1), 4), dtype=np.uint64)
        ctx.check(lib.sp_zk_sumcheck_verify_t(ctx.h, self.data, len(self.data), _point(comm_claim), num_rounds, degree_bound,
                                              gens_1.h, gens_n.h, transcript.state, comm_eval, _p(r)))
        return comm_eval.raw, r[:num_rounds]


class KnowledgeProof:
    """nizk/mod.rs:16-75: knowledge of the opening (x, r) of C = x*G + r*h"""

    def __init__(self, data):
        self.data = bytes(data)

    @staticmethod
    def prove(gens_n, transcript, tape, x, r):
        """returns (proof, C)"""
        out, n, Cc = C.POINTER(C.c_ubyte)(), _sz(), C.create_string_buffer(32)
        gens_n.ctx.check(lib.sp_knowledge_prove_t(gens_n.ctx.h, gens_n.h, transcript.state, tape.state, _scalar(x), _scalar(r), C.byref(out), C.byref(n),
                                                  Cc))
        return KnowledgeProof(_take_bytes(out, n)), Cc.raw

    def verify(self, gens_n, transcript, C_):
        gens_n.ctx.check(lib.sp_knowledge_verify_t(gens_n.ctx.h, gens_n.h, transcript.state, _point(C_), self.data, len(self.data)))


class EqualityProof:
    """nizk/mod.rs:78-143: C1 = v*G + s1*h and C2 = v*G + s2*h open to the same v"""

    def __init__(self, data):
        self.data = bytes(data)

    @staticmethod
    def prove(gens_n, transcript, tape, v1, s1, v2, s2):
        """returns (proof, C1, C2)"""
        out, n, c1, c2 = C.POINTER(C.c_ubyte)(), _sz(), C.create_string_buffer(32), C.create_string_buffer(32)
        gens_n.ctx.check(lib.sp_equality_prove_t(gens_n.ctx.h, gens_n.h, transcript.state, tape.state, _scalar(v1), _scalar(s1), _scalar(v2), _scalar(s2),
                                                 C.byref(out), C.byref(n), c1, c2))
        return EqualityProof(_take_bytes(out, n)), c1.raw, c2.raw

    def verify(self, gens_n, transcript, C1, C2):
        gens_n.ctx.check(lib.sp_equality_verify_t(gens_n.ctx.h, gens_n.h, transcript.state, _point(C1), _point(C2), self.data, len(self.data)))


class ProductProof:
    """nizk/mod.rs:147-290: X, Y, Z commit to x, y and z = x*y"""

    def __init__(self, data):
        self.data = bytes(data)

    @staticmethod
    def prove(gens_n, transcript, tape, x, rX, y, rY, z, rZ):
        """returns (proof, X, Y, Z)"""
        out, n = C.POINTER(C.c_ubyte)(), _sz()
        X, Y, Z = C.create_string_buffer(32), C.create_string_buffer(32), C.create_string_buffer(32)
        gens_n.ctx.check(lib.sp_product_prove_t(gens_n.ctx.h, gens_n.h, transcript.state, tape.state, _scalar(x), _scalar(rX), _scalar(y), _scalar(rY),
                                                _scalar(z), _scalar(rZ), C.byref(out), C.byref(n), X, Y, Z))
        return ProductProof(_take_bytes(out, n)), X.raw, Y.raw, Z.raw

    def verify(self, gens_n, transcript, X, Y, Z):
        gens_n.ctx.check(lib.sp_product_verify_t(gens_n.ctx.h, gens_n.h, transcript.state, _point(X), _point(Y), _point(Z), self.data, len(self.data)))


class DotProductProof:
    """nizk/mod.rs:293-406: Cx commits to x_vec, Cy to y = <a_vec, x_vec>; vectors of gens_n.n <= SP_DOTPROD_MAX_N entries"""

    def __init__(self, data):
        self.data = bytes(data)

    @staticmethod
    def prove(gens_1, gens_n, transcript, tape, x_vec, blind_x, a_vec, y, blind_y):
        """returns (proof, Cx, Cy)"""
        x, a = _limbs(x_vec), _limbs(a_vec)
        if len(x) != len(a):
            raise SpartanB200Error("DotProductProof: x_vec has %d entries, a_vec %d" % (len(x), len(a)))
        out, n, cx, cy = C.POINTER(C.c_ubyte)(), _sz(), C.create_string_buffer(32), C.create_string_buffer(32)
        gens_1.ctx.check(lib.sp_dotproduct_prove_t(gens_1.ctx.h, gens_1.h, gens_n.h, transcript.state, tape.state, _p(x), _scalar(blind_x), _p(a),
                                                   len(x), _scalar(y), _scalar(blind_y), C.byref(out), C.byref(n), cx, cy))
        return DotProductProof(_take_bytes(out, n)), cx.raw, cy.raw

    def verify(self, gens_1, gens_n, transcript, a, Cx, Cy):
        a = _limbs(a)
        gens_1.ctx.check(lib.sp_dotproduct_verify_t(gens_1.ctx.h, gens_1.h, gens_n.h, transcript.state, _p(a), len(a), _point(Cx), _point(Cy),
                                                    self.data, len(self.data)))


class DotProductProofGens(_Handle):
    """DotProductProofGens::new(n, label) (nizk/mod.rs:414-419): gens_n = G[0..n), gens_1 = G[n], h = G[n+1] of the label's stream, for a power of
    two 1 <= n <= 2^24.  Up to SP_DOTLOG_TABLE_MAX_N (include/spartan_b200.h) the set holds window tables; above it only the points."""
    _free = lib.sp_dotlog_gens_free

    def __init__(self, n, label, ctx=None):
        self.ctx = ctx or default_context()
        self.n = n
        h = _vp()
        self.ctx.check(lib.sp_dotlog_gens_create(self.ctx.h, n, bytes(label), len(label), C.byref(h)))
        self.h = h


def _device_vec(v, ctx):
    """a DensePolynomial as it is, a host array of Montgomery limbs uploaded"""
    return v if isinstance(v, DensePolynomial) else DensePolynomial(v, ctx)


class DotProductProofLog:
    """nizk/mod.rs:407-583: Cx commits to x_vec, Cy to y = <a_vec, x_vec>, in a proof of O(log n) points (a bulletproofs inner-product argument).
    x_vec and a_vec: DensePolynomials (read, never modified) or host arrays of Montgomery limbs.  `data` = bincode(DotProductProofLog)."""

    def __init__(self, data):
        self.data = bytes(data)

    @staticmethod
    def prove(gens, transcript, tape, x_vec, blind_x, a_vec, y, blind_y):
        """returns (proof, Cx, Cy); y=None: y = <x_vec, a_vec>, computed on the device"""
        ctx = gens.ctx
        x, a = _device_vec(x_vec, ctx), _device_vec(a_vec, ctx)
        out, n, cx, cy = C.POINTER(C.c_ubyte)(), _sz(), C.create_string_buffer(32), C.create_string_buffer(32)
        y_out = np.zeros(4, dtype=np.uint64)
        ctx.check(lib.sp_dotlog_prove_t(ctx.h, gens.h, transcript.state, tape.state, x.h, _scalar(blind_x), a.h, None if y is None else _scalar(y),
                                        _scalar(blind_y), C.byref(out), C.byref(n), cx, cy, _p(y_out)))
        return DotProductProofLog(_take_bytes(out, n)), cx.raw, cy.raw

    def verify(self, n, gens, transcript, a, Cx, Cy):
        """raises ProofVerifyError"""
        ctx = gens.ctx
        a = _device_vec(a, ctx)
        ctx.check(lib.sp_dotlog_verify_t(ctx.h, gens.h, transcript.state, a.h, n, _point(Cx), _point(Cy), self.data, len(self.data)))


# ----------------------------------------------------------------------------- product circuits of the caller's tables
class _ProdLeaves(C.Structure):
    _fields_ = [("nsources", C.c_uint32), ("source", C.c_uint32 * SP_PROD_MAX_SOURCES), ("coeff_mont", (C.c_uint64 * 4) * SP_PROD_MAX_SOURCES),
                ("index_coeff_mont", C.c_uint64 * 4), ("const_mont", C.c_uint64 * 4)]


def _scalar_arg(x):
    """a Python int (< q) or Montgomery limbs -> limbs"""
    if isinstance(x, (int, np.integer)):
        return scalar_from_bytes(int(x).to_bytes(32, "little"))
    return np.ascontiguousarray(x, dtype=np.uint64).reshape(4)


class ProductLeaves:
    """One product circuit's leaves as an affine form of the tables and of the index x (sp_prod_leaves):
    leaf[x] = const + index_coeff * x + sum over sources (i, coeff) of coeff * tables[i][x].  Scalars: Python ints (< q) or Montgomery limbs.
    The memory check's hash(addr, val, ts) - gamma = ts*r^2 + val*r + addr - gamma (sparse_mlpoly.rs:542-591) is
    ProductLeaves([(ts, r^2), (val, r), (addr, 1)], const=-gamma), with index_coeff=1 instead of an addr table for init and audit."""

    def __init__(self, sources=(), index_coeff=0, const=0):
        self.sources = [(int(i), _scalar_arg(c)) for i, c in sources]
        self.index_coeff, self.const = _scalar_arg(index_coeff), _scalar_arg(const)

    def _fill(self, out):
        out.nsources = len(self.sources)   # more than SP_PROD_MAX_SOURCES: the count alone reaches the library, which refuses it
        for s, (i, c) in enumerate(self.sources[:SP_PROD_MAX_SOURCES]):
            out.source[s] = i
            out.coeff_mont[s][:] = [int(v) for v in c]
        out.index_coeff_mont[:] = [int(v) for v in self.index_coeff]
        out.const_mont[:] = [int(v) for v in self.const]


def _c_leaves(leaves):
    if leaves is None:
        return None
    arr = (_ProdLeaves * max(len(leaves), 1))()
    for l, a in zip(leaves, arr):
        l._fill(a)
    return arr


class ProductCircuits(_Handle):
    """ProductCircuit::new of k circuits, then ProductCircuit::evaluate (product_tree.rs:36-63), on the GPU: `tables` are DensePolynomials of
    one length 2^m (m >= 1), read and never modified; `leaves` a list of ProductLeaves (at most SP_PROD_MAX_CIRCUITS), or None for one circuit
    per table.  .products: the k products as (k, 4) limbs; .num_vars = m.  ProductCircuitEvalProofBatched.prove consumes the circuits.
    `dotps`: a list of kd (left, right, weight) triples of ProductLeaves, the dot products sum_x left[x] right[x] weight[x] to prove beside the
    circuits (k + 2 kd <= SP_PROD_MAX_CIRCUITS); .dotp_claims: the two half sums of each as (kd, 2, 4) limbs (claims_dotp_vec), and
    ProductCircuitEvalProofBatched.prove_dotp proves them."""
    _free = lib.sp_prod_free

    def __init__(self, tables, leaves=None, dotps=None):
        tables = _poly_list(tables)
        self.ctx = tables[0].ctx if tables else default_context()
        self.k = len(tables) if leaves is None else len(leaves)
        self.kd = 0 if dotps is None else len(dotps)
        products = np.zeros((max(self.k, 1), 4), dtype=np.uint64)
        claims = np.zeros((max(self.kd, 1), 2, 4), dtype=np.uint64)
        h = _vp()
        if dotps is None:
            self.ctx.check(lib.sp_prod_build(self.ctx.h, _handles(tables), len(tables), _c_leaves(leaves), self.k, C.byref(h), _p(products)))
        else:
            forms = _c_leaves([f for d in dotps for f in d])
            self.ctx.check(lib.sp_prod_build_dotp(self.ctx.h, _handles(tables), len(tables), _c_leaves(leaves), self.k, forms,
                                                  self.kd, C.byref(h), _p(products), _p(claims)))
        self.h = h
        self.products = products[:self.k]
        self.dotp_claims = claims[:self.kd]
        self.num_vars = tables[0].len().bit_length() - 1


class ProductCircuitEvalProofBatched:
    """product_tree.rs:250-485: prove / verify for product circuits alone, prove_dotp / verify_dotp with the caller's dot products.  Transcripts:
    a Transcript (advanced in place) or a label."""

    @staticmethod
    def prove(circuits, transcript):
        """ProductCircuitEvalProofBatched::prove(circuits, [], transcript) (product_tree.rs:259-383).  Absorb the products first: the proof does
        not.  Returns (proof bytes = bincode, rand as (m, 4) limbs, leaf_evals = each circuit's leaf polynomial at rand as (k, 4) limbs)."""
        ctx, t = circuits.ctx, _transcript_state(transcript)
        out, n = C.POINTER(C.c_ubyte)(), _sz()
        rand = np.zeros((circuits.num_vars, 4), dtype=np.uint64)
        evals = np.zeros((max(circuits.k, 1), 4), dtype=np.uint64)
        ctx.check(lib.sp_prod_prove_t(ctx.h, circuits.h, t.state, C.byref(out), C.byref(n), _p(rand), _p(evals)))
        return _take_bytes(out, n), rand, evals[:circuits.k]

    @staticmethod
    def verify(proof, products, num_vars, transcript):
        """ProductCircuitEvalProofBatched::verify(products, [], 2^num_vars, transcript) (product_tree.rs:385-485), on the host: returns (rand,
        leaf_claims) as limbs, raises ProofVerifyError.  The transcript is advanced as the reference's verify advances it, accepted or not."""
        t, proof, prods = _transcript_state(transcript), bytes(proof), _limbs(products)
        rand = np.zeros((max(num_vars, 1), 4), dtype=np.uint64)
        claims = np.zeros((max(len(prods), 1), 4), dtype=np.uint64)
        _check_host(lib.sp_prod_verify_t(None, proof, len(proof), _p(prods), len(prods), num_vars, t.state, _p(rand), _p(claims)))
        return rand[:num_vars], claims[:len(prods)]

    @staticmethod
    def prove_dotp(circuits, transcript):
        """ProductCircuitEvalProofBatched::prove(circuits, dotp halves, transcript) of ProductCircuits built with or without dotps.  Absorb the
        products (and what the caller's protocol absorbs of the half sums) first.  Returns (proof bytes, rand (m, 4), leaf_evals (k, 4),
        dotp_evals = (left, right, weight) of each dot product at rand as (kd, 3, 4) limbs)."""
        ctx, t = circuits.ctx, _transcript_state(transcript)
        out, n = C.POINTER(C.c_ubyte)(), _sz()
        rand = np.zeros((circuits.num_vars, 4), dtype=np.uint64)
        evals = np.zeros((max(circuits.k, 1), 4), dtype=np.uint64)
        dotp = np.zeros((max(circuits.kd, 1), 3, 4), dtype=np.uint64)
        ctx.check(lib.sp_prod_prove_dotp_t(ctx.h, circuits.h, t.state, C.byref(out), C.byref(n), _p(rand), _p(evals), _p(dotp)))
        return _take_bytes(out, n), rand, evals[:circuits.k], dotp[:circuits.kd]

    @staticmethod
    def verify_dotp(proof, products, dotp_claims, num_vars, transcript):
        """ProductCircuitEvalProofBatched::verify(products, dotp_claims, 2^num_vars, transcript) on the host, dotp_claims the (kd, 2, 4) half sums:
        returns (rand, leaf_claims, dotp_claims = (left, right, weight) of each dot product at rand as (kd, 3, 4) limbs), raises ProofVerifyError.
        The transcript is advanced as the reference's verify advances it, accepted or not."""
        t, proof, prods = _transcript_state(transcript), bytes(proof), _limbs(products)
        halves = _limbs(np.asarray(dotp_claims, dtype=np.uint64).reshape(-1, 4))
        kd = len(halves) // 2
        rand = np.zeros((max(num_vars, 1), 4), dtype=np.uint64)
        claims = np.zeros((max(len(prods), 1), 4), dtype=np.uint64)
        dotp = np.zeros((max(kd, 1), 3, 4), dtype=np.uint64)
        _check_host(lib.sp_prod_verify_dotp_t(None, proof, len(proof), _p(prods), len(prods), _p(halves), kd,
                                              num_vars, t.state, _p(rand), _p(claims), _p(dotp)))
        return rand[:num_vars], claims[:len(prods)], dotp[:kd]


def product_leaf_eval(leaves, table_evals, rand):
    """the leaf polynomials at rand from the tables' values there (sp_prod_leaf_eval), on the host: (k, 4) limbs.  leaves None: one circuit per
    table.  A verifier compares these with ProductCircuitEvalProofBatched.verify's leaf claims."""
    ev, r = _limbs(table_evals), _limbs(rand)
    k = len(ev) if leaves is None else len(leaves)
    out = np.zeros((max(k, 1), 4), dtype=np.uint64)
    _check_host(lib.sp_prod_leaf_eval(_c_leaves(leaves), k, _p(ev), len(ev), _p(r), len(r), _p(out)))
    return out[:k]


# ----------------------------------------------------------------------------- SPARK: the caller's sparse matrices
class _SparkEntries(C.Structure):
    _fields_ = [("row", _vp), ("col", _vp), ("val32", _vp), ("nnz", C.c_size_t)]


class SparseMatPolyCommitmentGens(_Handle):
    """SparseMatPolyCommitmentGens::new(label, num_vars_x, num_vars_y, num_nz_entries, batch_size) (sparse_mlpoly.rs:292-317): gens_ops, gens_mem
    and gens_derefs as views of one generator set of the label (footprint: include/spartan_b200.h, sp_spark_gens_create)."""
    _free = lib.sp_spark_gens_free

    def __init__(self, label, num_vars_x, num_vars_y, num_nz_entries, batch_size, ctx=None):
        self.ctx = ctx or default_context()
        self.num_vars_x, self.num_vars_y, self.batch_size = num_vars_x, num_vars_y, batch_size
        label = bytes(label)
        h = _vp()
        self.ctx.check(lib.sp_spark_gens_create(self.ctx.h, label, len(label), num_vars_x, num_vars_y, num_nz_entries, batch_size, C.byref(h)))
        self.h = h


class SparseMatPolyCommitment:
    """sparse_mlpoly.rs:319-341: batch_size, num_ops, num_mem_cells and the commitments to comb_ops and comb_mem"""

    def __init__(self, batch_size, num_ops, num_mem_cells, comm_comb_ops, comm_comb_mem):
        self.batch_size, self.num_ops, self.num_mem_cells = batch_size, num_ops, num_mem_cells
        self.comm_comb_ops, self.comm_comb_mem = comm_comb_ops, comm_comb_mem

    def to_bytes(self):
        """bincode(SparseMatPolyCommitment)"""
        return (self.batch_size.to_bytes(8, "little") + self.num_ops.to_bytes(8, "little") + self.num_mem_cells.to_bytes(8, "little")
                + self.comm_comb_ops.to_bytes() + self.comm_comb_mem.to_bytes())

    @classmethod
    def from_bytes(cls, data):
        data = bytes(data)
        if len(data) < 32:
            raise SpartanB200Error("SparseMatPolyCommitment: %d bytes are too few" % len(data))
        u = [int.from_bytes(data[8 * i:8 * i + 8], "little") for i in range(4)]
        n_ops = 32 + 32 * u[3]
        ops = PolyCommitment.from_bytes(data[24:n_ops])
        return cls(u[0], u[1], u[2], ops, PolyCommitment.from_bytes(data[n_ops:]))

    def append_to_transcript(self, label, transcript):
        """sparse_mlpoly.rs:329-341 on a Transcript (the reference ignores the label)"""
        for name, v in ((b"batch_size", self.batch_size), (b"num_ops", self.num_ops), (b"num_mem_cells", self.num_mem_cells)):
            transcript.append_message(name, int(v).to_bytes(8, "little"))
        self.comm_comb_ops.append_to_transcript(b"comm_comb_ops", transcript)
        self.comm_comb_mem.append_to_transcript(b"comm_comb_mem", transcript)


class SparseMatPolyDense(_Handle):
    """MultiSparseMatPolynomialAsDense (sparse_mlpoly.rs:274-282) on the device: what multi_commit returns beside the commitment"""
    _free = lib.sp_spark_dense_free

    def __init__(self, ctx, h, batch_size, num_vars_x, num_vars_y):
        self.ctx, self.h = ctx, h
        self.batch_size, self.num_vars_x, self.num_vars_y = batch_size, num_vars_x, num_vars_y


class SparseMatPolynomial:
    """SparseMatPolynomial (sparse_mlpoly.rs:31-37): 2^num_vars_x rows, 2^num_vars_y columns, entries (row, col, val).  vals: canonical 32-byte
    scalars as an (nnz, 32) uint8 array, a list of 32-byte strings or of ints (< q)."""

    def __init__(self, num_vars_x, num_vars_y, rows, cols, vals):
        self.num_vars_x, self.num_vars_y = num_vars_x, num_vars_y
        self.rows = np.ascontiguousarray(rows, dtype=np.uint64).reshape(-1)
        self.cols = np.ascontiguousarray(cols, dtype=np.uint64).reshape(-1)
        if isinstance(vals, np.ndarray):
            self.vals = np.ascontiguousarray(vals, dtype=np.uint8).reshape(-1, 32)
        else:
            self.vals = np.frombuffer(b"".join(int(v).to_bytes(32, "little") if isinstance(v, (int, np.integer)) else bytes(v) for v in vals),
                                      dtype=np.uint8).reshape(-1, 32)
        if not len(self.rows) == len(self.cols) == len(self.vals):
            raise SpartanB200Error("SparseMatPolynomial: rows, cols and vals differ in length")
        self.device = False

    @classmethod
    def from_tensors(cls, num_vars_x, num_vars_y, rows, cols, vals, ctx=None):
        """the entries as CUDA tensors on ctx.device: rows and cols int64 of length nnz, vals uint8 of shape (nnz, 32); multi_commit reads them there"""
        ctx = ctx or default_context()
        torch = _torch()
        o = cls.__new__(cls)
        o.num_vars_x, o.num_vars_y, o.ctx, o.device = num_vars_x, num_vars_y, ctx, True
        o.rows = _device_tensor(rows, ctx, "rows", torch.int64)
        o.cols = _device_tensor(cols, ctx, "cols", torch.int64)
        o.vals = _device_tensor(vals, ctx, "vals", torch.uint8, 32)
        if not o.rows.shape[0] == o.cols.shape[0] == o.vals.shape[0]:
            raise SpartanB200Error("rows, cols and vals differ in length (%d, %d, %d)" % (o.rows.shape[0], o.cols.shape[0], o.vals.shape[0]))
        return o

    def _entries(self):
        if self.device:
            return _SparkEntries(self.rows.data_ptr(), self.cols.data_ptr(), self.vals.data_ptr(), self.rows.shape[0])
        return _SparkEntries(self.rows.ctypes.data, self.cols.ctypes.data, self.vals.ctypes.data, len(self.rows))

    @staticmethod
    def _batch(polys, what):
        """(device, num_vars_x, num_vars_y, _SparkEntries array) of a batch that is all host or all device matrices of one shape; what: the
        method the refusals name"""
        device = bool(polys) and polys[0].device
        if any(p.device != device for p in polys):
            raise SpartanB200Error(what + ": mix of host and device matrices")
        if any((p.num_vars_x, p.num_vars_y) != (polys[0].num_vars_x, polys[0].num_vars_y) for p in polys):
            raise SpartanB200Error(what + ": matrices of different shapes")
        x, y = (polys[0].num_vars_x, polys[0].num_vars_y) if polys else (0, 0)
        return device, x, y, (_SparkEntries * max(len(polys), 1))(*[p._entries() for p in polys])

    @staticmethod
    def multi_commit(polys, gens):
        """SparseMatPolynomial::multi_commit (sparse_mlpoly.rs:483-503) of 1 .. SP_SPARK_MAX_BATCH matrices of one shape, all host or all device
        entries: returns (SparseMatPolyCommitment, SparseMatPolyDense)"""
        polys = list(polys)
        ctx = gens.ctx
        device, x, y, arr = SparseMatPolynomial._batch(polys, "multi_commit")
        if device:
            _sync_torch(ctx)
        h, out, n = _vp(), C.POINTER(C.c_ubyte)(), _sz()
        entry = lib.sp_spark_commit_device if device else lib.sp_spark_commit
        ctx.check(entry(ctx.h, gens.h, arr, len(polys), x, y, C.byref(h), C.byref(out), C.byref(n)))
        dense = SparseMatPolyDense(ctx, h, len(polys), x, y)
        return SparseMatPolyCommitment.from_bytes(_take_bytes(out, n)), dense

    @staticmethod
    def multi_evaluate(dense_or_polys, rx, ry, gens=None):
        """SparseMatPolynomial::multi_evaluate (sparse_mlpoly.rs:440-452) on the device: the b evaluations M_i(rx, ry) as (b, 4) limbs.  Takes a
        SparseMatPolyDense, or a list of SparseMatPolynomial together with gens that fit them (they are committed first)."""
        dense = dense_or_polys
        if not isinstance(dense, SparseMatPolyDense):
            if gens is None:
                raise SpartanB200Error("multi_evaluate of SparseMatPolynomials needs their gens")
            dense = SparseMatPolynomial.multi_commit(dense_or_polys, gens)[1]
        rx, ry = _limbs(rx), _limbs(ry)
        out = np.zeros((dense.batch_size, 4), dtype=np.uint64)
        dense.ctx.check(lib.sp_spark_evaluate(dense.ctx.h, dense.h, _p(rx), len(rx), _p(ry), len(ry), _p(out)))
        return out

    @staticmethod
    def multi_products(polys, ctx=None):
        """the device form of 1 .. SP_SPMAT_MAX_BATCH matrices of one shape, all host or all device entries, for their products with vectors
        (sp_spmat_create): a SparseMatProducts.  Host matrices go to ctx (default: the default context), device ones stay on theirs."""
        polys = list(polys)
        device, x, y, arr = SparseMatPolynomial._batch(polys, "multi_products")
        if device:
            ctx = polys[0].ctx
            if any(p.ctx is not ctx for p in polys):
                raise SpartanB200Error("multi_products: device matrices of different contexts")
            _sync_torch(ctx)
        ctx = ctx or default_context()
        h = _vp()
        entry = lib.sp_spmat_create_device if device else lib.sp_spmat_create
        ctx.check(entry(ctx.h, arr, len(polys), x, y, C.byref(h)))
        return SparseMatProducts(ctx, h, len(polys), x, y)

    def _products(self):
        if getattr(self, "_spmat", None) is None:
            self._spmat = SparseMatPolynomial.multi_products([self], self.ctx if self.device else None)
        return self._spmat

    def multiply_vec(self, num_rows, num_cols, z):
        """SparseMatPolynomial::multiply_vec (sparse_mlpoly.rs:454-464) on the device: M z as a DensePolynomial of num_rows entries.  z: a
        DensePolynomial or host Montgomery limbs of num_cols entries.  The device form is built on first use and kept on the object."""
        return self._products().multiply_vec(num_rows, num_cols, z)[0]

    def compute_eval_table_sparse(self, rx, num_rows, num_cols):
        """SparseMatPolynomial::compute_eval_table_sparse (sparse_mlpoly.rs:466-481) on the device: M^T rx as a DensePolynomial of num_cols
        entries.  rx is the eq table of num_rows entries (eq(r_x, .) as the reference passes it), not the point r_x; a DensePolynomial or host
        Montgomery limbs."""
        return self._products().compute_eval_table_sparse(rx, num_rows, num_cols)[0]


class SparseMatProducts(_Handle):
    """b matrices on the device, each sorted by row and by column (80 bytes per entry; include/spartan_b200.h, sp_spmat), for multiply_vec and
    compute_eval_table_sparse of all of them in one call"""
    _free = lib.sp_spmat_free

    def __init__(self, ctx, h, batch_size, num_vars_x=None, num_vars_y=None):
        self.ctx, self.h, self.batch_size = ctx, h, batch_size
        self.num_vars_x, self.num_vars_y = num_vars_x, num_vars_y

    def _vector(self, v):
        if isinstance(v, DensePolynomial):
            return v
        return DensePolynomial(v, self.ctx)

    def multiply_vec(self, num_rows, num_cols, z):
        """[M_m z for every matrix m]: b DensePolynomials of num_rows entries; len(z) must be num_cols"""
        z = self._vector(z)
        outs = (_vp * self.batch_size)()
        self.ctx.check(lib.sp_spmat_multiply_vec(self.ctx.h, self.h, num_rows, num_cols, z.h, outs))
        return [DensePolynomial._wrap(self.ctx, _vp(outs[i])) for i in range(self.batch_size)]

    def compute_eval_table_sparse(self, rx, num_rows, num_cols, weights=None):
        """[M_m^T rx for every matrix m], b DensePolynomials of num_cols entries, with rx the eq table of num_rows entries (not the point).  With
        weights (b scalars as Montgomery limbs): the one DensePolynomial sum_m weights[m] M_m^T rx."""
        rx = self._vector(rx)
        w = None if weights is None else _limbs(weights)
        if w is not None and len(w) != self.batch_size:
            raise SpartanB200Error("compute_eval_table_sparse: %d weights for %d matrices" % (len(w), self.batch_size))
        n = 1 if w is not None else self.batch_size
        outs = (_vp * n)()
        self.ctx.check(lib.sp_spmat_eval_table(self.ctx.h, self.h, rx.h, num_rows, num_cols, None if w is None else _p(w), outs))
        res = [DensePolynomial._wrap(self.ctx, _vp(outs[i])) for i in range(n)]
        return res[0] if w is not None else res


class SparseMatPolyEvalProof:
    """sparse_mlpoly.rs:1418-1557.  `data` = bincode(SparseMatPolyEvalProof).  Transcripts: a Transcript (advanced in place) or a label.  Neither
    prove nor verify absorbs the commitment or the evaluations: the caller does, before the call."""

    def __init__(self, data):
        self.data = bytes(data)

    @staticmethod
    def prove(dense, rx, ry, evals, gens, transcript, tape):
        """SparseMatPolyEvalProof::prove: returns (proof, evals as (b, 4) limbs).  evals=None: computed on the device; given evals must be
        M_i(rx, ry)."""
        ctx, t = dense.ctx, _transcript_state(transcript)
        rx, ry = _limbs(rx), _limbs(ry)
        out, n = C.POINTER(C.c_ubyte)(), _sz()
        ev = np.zeros((dense.batch_size, 4), dtype=np.uint64)
        ctx.check(lib.sp_spark_eval_prove_t(ctx.h, dense.h, gens.h, _p(rx), len(rx), _p(ry), len(ry),
                                            None if evals is None else _p(_limbs(evals)), t.state, tape.state, C.byref(out), C.byref(n), _p(ev)))
        return SparseMatPolyEvalProof(_take_bytes(out, n)), ev

    def verify(self, comm, rx, ry, evals, gens, transcript):
        """SparseMatPolyEvalProof::verify: raises ProofVerifyError; the transcript is advanced as the reference's verify advances it"""
        t, rx, ry, ev = _transcript_state(transcript), _limbs(rx), _limbs(ry), _limbs(evals)
        cb = comm.to_bytes() if isinstance(comm, SparseMatPolyCommitment) else bytes(comm)
        gens.ctx.check(lib.sp_spark_eval_verify_t(gens.ctx.h, gens.h, cb, len(cb), _p(rx), len(rx), _p(ry), len(ry), _p(ev),
                                                  len(ev), t.state, self.data, len(self.data)))


# ----------------------------------------------------------------------------- public API of lib.rs
class Assignment:
    """lib.rs:57-104: a vector of scalars given as canonical 32-byte strings"""

    def __init__(self, assignment):
        if isinstance(assignment, np.ndarray):
            self.limbs = _limbs(assignment).copy()
        else:
            self.limbs = np.zeros((len(assignment), 4), dtype=np.uint64)
            for i, b in enumerate(assignment):
                self.limbs[i] = scalar_from_bytes(b)  # raises R1CSError::InvalidScalar

    @staticmethod
    def new(assignment):
        return Assignment(assignment)

    def __len__(self):
        return len(self.limbs)


VarsAssignment = Assignment
InputsAssignment = Assignment


class Instance(_Handle):
    """lib.rs:111-274"""
    _free = lib.sp_instance_free

    def __init__(self, ctx, h):
        self.ctx, self.h = ctx, h
        nc, nv, ni = _sz(), _sz(), _sz()
        _check_host(lib.sp_instance_dims(h, C.byref(nc), C.byref(nv), C.byref(ni)))
        self.num_cons, self.num_vars, self.num_inputs = nc.value, nv.value, ni.value
        self._digest = None

    @staticmethod
    def new(num_cons, num_vars, num_inputs, A, B, Cm, ctx=None):
        """Instance::new (lib.rs:121-227); A/B/C: lists of (row, col, 32 canonical bytes)"""
        ctx = ctx or default_context()

        def split(t):
            rows = np.array([r for r, _, _ in t], dtype=np.uint64)
            cols = np.array([c for _, c, _ in t], dtype=np.uint64)
            vals = b"".join(bytes(v) for _, _, v in t)
            return rows, cols, vals, len(t)
        a, b, c = split(A), split(B), split(Cm)
        h = _vp()
        ctx.check(lib.sp_instance_create(ctx.h, num_cons, num_vars, num_inputs, _p(a[0]), _p(a[1]), a[2], a[3],
                                         _p(b[0]), _p(b[1]), b[2], b[3], _p(c[0]), _p(c[1]), c[2], c[3], C.byref(h)))
        return Instance(ctx, h)

    @staticmethod
    def from_tensors(num_cons, num_vars, num_inputs, A, B, Cm, ctx=None):
        """Instance::new from CUDA tensors on ctx.device, built there: A/B/C are (rows, cols, vals) with rows and cols int64 of length nnz and vals
        uint8 of shape (nnz, 32), canonical little-endian scalars.  Same checks, padding, errors and instance as Instance.new; the matrices stay
        on the device (bincode / digest / export download them on first use)."""
        ctx = ctx or default_context()
        torch = _torch()
        mats = []
        for mname, M in zip("ABC", (A, B, Cm)):
            if not isinstance(M, (tuple, list)) or len(M) != 3:
                raise SpartanB200Error("%s: expected a (rows, cols, vals) triple" % mname)
            rows = _device_tensor(M[0], ctx, mname + " rows", torch.int64)
            cols = _device_tensor(M[1], ctx, mname + " cols", torch.int64)
            vals = _device_tensor(M[2], ctx, mname + " vals", torch.uint8, 32)
            if not rows.shape[0] == cols.shape[0] == vals.shape[0]:
                raise SpartanB200Error("%s: rows, cols and vals differ in length (%d, %d, %d)" % (mname, rows.shape[0], cols.shape[0], vals.shape[0]))
            mats.append((rows, cols, vals))
        _sync_torch(ctx)
        args = []
        for rows, cols, vals in mats:
            args += [_vp(rows.data_ptr()), _vp(cols.data_ptr()), _vp(vals.data_ptr()), rows.shape[0]]
        h = _vp()
        ctx.check(lib.sp_instance_create_device(ctx.h, num_cons, num_vars, num_inputs, *args, C.byref(h)))
        return Instance(ctx, h)

    @staticmethod
    def produce_synthetic_r1cs(num_cons, num_vars, num_inputs, seed=0, ctx=None):
        """Instance::produce_synthetic_r1cs (lib.rs:262-274) with a seeded generator instead of OsRng"""
        ctx = ctx or default_context()
        h = _vp()
        vars_out = np.zeros((num_vars, 4), dtype=np.uint64)
        inputs_out = np.zeros((num_inputs, 4), dtype=np.uint64)
        ctx.check(lib.sp_instance_synthetic(ctx.h, num_cons, num_vars, num_inputs, seed, C.byref(h), _p(vars_out), _p(inputs_out)))
        return Instance(ctx, h), Assignment(vars_out), Assignment(inputs_out)

    def bincode(self):
        out, n = C.POINTER(C.c_ubyte)(), _sz()
        _check_host(lib.sp_instance_bincode(self.h, C.byref(out), C.byref(n)))
        return _take_bytes(out, n)

    @property
    def digest(self):
        """R1CSShape::get_digest (r1cs.rs:154-158): the caller-supplied bytes, else the library's miniz-level-6 zlib stream of bincode(shape)"""
        if self._digest is None:
            out, n = C.POINTER(C.c_ubyte)(), _sz()
            _check_host(lib.sp_instance_digest(self.h, C.byref(out), C.byref(n)))
            self._digest = _take_bytes(out, n)
        return self._digest

    def set_digest(self, digest):
        """absorb these bytes instead (e.g. the digest another compressor produced); b"" returns to the library's own"""
        _check_host(lib.sp_instance_set_digest(self.h, bytes(digest), len(digest)))
        self._digest = bytes(digest) if digest else None

    def export(self, matrix):
        n = _sz()
        _check_host(lib.sp_instance_nnz(self.h, matrix, C.byref(n)))
        row = np.zeros(n.value, dtype=np.uint64)
        col = np.zeros(n.value, dtype=np.uint64)
        val = np.zeros((n.value, 4), dtype=np.uint64)
        _check_host(lib.sp_instance_export(self.h, matrix, _p(row), _p(col), _p(val)))
        return row, col, val

    def is_sat(self, vars, inputs):
        sat = C.c_int()
        self.ctx.check(lib.sp_instance_is_sat(self.ctx.h, self.h, _p(vars.limbs), len(vars), _p(inputs.limbs), len(inputs), C.byref(sat)))
        return bool(sat.value)

    def evaluate(self, rx, ry):
        """R1CSShape::evaluate (r1cs.rs:300-303) on the device: (A(rx, ry), B(rx, ry), C(rx, ry)) as (3, 4) Montgomery limbs, the evals
        R1CSProof.verify takes.  rx: log2 num_cons scalars, ry: log2 (2 num_vars), of the padded dimensions."""
        rx, ry = _limbs(rx), _limbs(ry)
        nx, ny = self.num_cons.bit_length() - 1, (2 * self.num_vars).bit_length() - 1
        if len(rx) != nx or len(ry) != ny:
            raise SpartanB200Error("Instance.evaluate: |rx| = %d, |ry| = %d; this instance needs %d and %d" % (len(rx), len(ry), nx, ny))
        out = np.zeros((3, 4), dtype=np.uint64)
        self.ctx.check(lib.sp_instance_evaluate(self.ctx.h, self.h, _p(rx), _p(ry), _p(out)))
        return out


def _take_bytes(out, n):
    b = C.string_at(out, n.value)
    lib.sp_free(out)
    return b


class _GenSetInfo(C.Structure):
    _fields_ = [("label", C.c_char * 32), ("nbases", C.c_size_t), ("window_bits", C.c_int), ("has_row_table", C.c_int), ("device_bytes", C.c_size_t)]


class GeneratorTables(_Handle):
    """Generator tables sized once for the largest circuit a caller proves (sp_gen_tables): the gens_r1cs_sat set for circuits up to
    (num_cons, num_vars, num_inputs) and, if num_nz_entries > 0, the gens_r1cs_eval set up to that many non-zeros.  NIZKGens(..., tables=t)
    and SNARKGens(..., tables=t) for any circuit whose every dimension is <= these are views that share the tables' device memory and prove
    the same bytes as gens of their own.  Views keep the tables alive: `del` this object whenever convenient."""
    _free = lib.sp_gen_tables_free

    def __init__(self, num_cons, num_vars, num_inputs, num_nz_entries=0, ctx=None):
        self.ctx = ctx or default_context()
        h = _vp()
        self.ctx.check(lib.sp_gen_tables_create(self.ctx.h, num_cons, num_vars, num_inputs, num_nz_entries, C.byref(h)))
        self.h = h

    def info(self):
        """one dict per generator set: label, nbases, window_bits, has_row_table, device_bytes"""
        out, n = (_GenSetInfo * 2)(), _sz()
        self.ctx.check(lib.sp_gen_tables_info(self.h, out, 2, C.byref(n)))
        return [{"label": s.label.decode(), "nbases": int(s.nbases), "window_bits": int(s.window_bits), "has_row_table": bool(s.has_row_table),
                 "device_bytes": int(s.device_bytes)} for s in out[:n.value]]


def device_bytes_live():
    """device bytes in blocks the library holds for live objects (its cache of freed blocks excluded): unlike the driver's free-memory
    figure, other processes on the GPU do not change it"""
    return int(lib.sp_device_bytes_live())


class NIZKGens(_Handle):
    """lib.rs:468-486.  tables=GeneratorTables: a view into them instead of generator tables of its own"""
    _free = lib.sp_nizk_gens_free

    def __init__(self, num_cons, num_vars, num_inputs, ctx=None, tables=None):
        self.ctx = ctx or (tables.ctx if tables is not None else default_context())
        h = _vp()
        if tables is None:
            self.ctx.check(lib.sp_nizk_gens_create(self.ctx.h, num_cons, num_vars, num_inputs, C.byref(h)))
        else:
            self.ctx.check(lib.sp_nizk_gens_create_from(self.ctx.h, tables.h, num_cons, num_vars, num_inputs, C.byref(h)))
        self.h = h

    @staticmethod
    def new(num_cons, num_vars, num_inputs, ctx=None):
        return NIZKGens(num_cons, num_vars, num_inputs, ctx)


class R1CSGens(_Handle):
    """R1CSGens::new(label, num_cons, num_vars) (r1csproof.rs:61-74): gens_pc = PolyCommitmentGens::new(log2 num_vars, label) and the sumcheck
    gens gens_1, gens_3, gens_4 of the same label's stream, for a power-of-two num_vars.  view(gens, num_cons, num_vars) gives the same gens as a
    view of the gens_r1cs_sat set of NIZKGens, SNARKGens or GeneratorTables, without device memory of its own."""
    _free = lib.sp_r1cs_gens_free

    def __init__(self, label, num_cons, num_vars, ctx=None):
        self.ctx = ctx or default_context()
        self.num_cons, self.num_vars = num_cons, num_vars
        h = _vp()
        self.ctx.check(lib.sp_r1cs_gens_create(self.ctx.h, bytes(label), len(label), num_cons, num_vars, C.byref(h)))
        self.h = h

    @classmethod
    def view(cls, gens_or_tables, num_cons, num_vars):
        entry = {NIZKGens: lib.sp_r1cs_gens_create_from_nizk, SNARKGens: lib.sp_r1cs_gens_create_from_snark,
                 GeneratorTables: lib.sp_r1cs_gens_create_from}.get(type(gens_or_tables))
        if entry is None:
            raise SpartanB200Error("R1CSGens.view: expected NIZKGens, SNARKGens or GeneratorTables, got %s" % type(gens_or_tables).__name__)
        o = cls.__new__(cls)
        o.ctx, o.num_cons, o.num_vars = gens_or_tables.ctx, num_cons, num_vars
        h = _vp()
        o.ctx.check(entry(o.ctx.h, gens_or_tables.h, num_cons, num_vars, C.byref(h)))
        o.h = h
        return o


def _input_limbs(inputs):
    return inputs.limbs if isinstance(inputs, Assignment) else _limbs(inputs)


class R1CSProof:
    """r1csproof.rs:20-489: the proof NIZK and SNARK embed, on the caller's Transcript and RandomTape.  `data` = bincode(R1CSProof)."""

    def __init__(self, data):
        self.data = bytes(data)

    def to_bytes(self):
        return self.data

    @classmethod
    def from_bytes(cls, data):
        return cls(data)

    @staticmethod
    def prove(matrices, vars, inputs, gens, transcript, tape):
        """R1CSProof::prove(inst, vars, inputs, gens, transcript, random_tape): returns (proof, rx, ry) with rx, ry as Montgomery limbs.
        matrices: an Instance (its products as NIZK.prove runs them) or a SparseMatProducts of A, B, C (2^log2 num_cons rows, 2^log2 (2 num_vars)
        columns: the tiled products, whatever the rows' and columns' lengths).  vars: a DensePolynomial (read only) or host limbs, num_vars =
        len(vars) entries (the padded count); inputs: an Assignment or host limbs."""
        ctx = gens.ctx
        v = _device_vec(vars.limbs if isinstance(vars, Assignment) else vars, ctx)
        num_vars = v.len()
        if isinstance(matrices, Instance):
            inst, spmat, num_cons = matrices.h, None, matrices.num_cons
        elif isinstance(matrices, SparseMatProducts):
            if matrices.num_vars_x is None:
                raise SpartanB200Error("R1CSProof.prove: a SparseMatProducts of unknown shape (make it with SparseMatPolynomial.multi_products)")
            inst, spmat, num_cons = None, matrices.h, 1 << matrices.num_vars_x
        else:
            raise SpartanB200Error("R1CSProof.prove: matrices must be an Instance or a SparseMatProducts, got %s" % type(matrices).__name__)
        x = _input_limbs(inputs)
        out, n = C.POINTER(C.c_ubyte)(), _sz()
        rx = np.zeros((max(num_cons.bit_length() - 1, 1), 4), dtype=np.uint64)
        ry = np.zeros((max((2 * num_vars).bit_length() - 1, 1), 4), dtype=np.uint64)
        ctx.check(lib.sp_r1cs_prove_t(ctx.h, inst, spmat, num_cons, num_vars, v.h, _p(x), len(x), gens.h, transcript.state, tape.state,
                                      C.byref(out), C.byref(n), _p(rx), _p(ry)))
        return R1CSProof(_take_bytes(out, n)), rx[:num_cons.bit_length() - 1], ry[:(2 * num_vars).bit_length() - 1]

    def verify(self, num_vars, num_cons, inputs, evals, transcript, gens):
        """R1CSProof::verify(num_vars, num_cons, inputs, evals, transcript, gens) with evals = (Ar, Br, Cr) as (3, 4) limbs: returns (rx, ry),
        raises ProofVerifyError"""
        ctx = gens.ctx
        x, ev = _input_limbs(inputs), _limbs(evals)
        if len(ev) != 3:
            raise SpartanB200Error("R1CSProof.verify: %d evals; (Ar, Br, Cr) expected" % len(ev))
        nx, ny = max(num_cons, 1).bit_length() - 1, max(2 * num_vars, 1).bit_length() - 1
        rx, ry = np.zeros((max(nx, 1), 4), dtype=np.uint64), np.zeros((max(ny, 1), 4), dtype=np.uint64)
        ctx.check(lib.sp_r1cs_verify_t(ctx.h, self.data, len(self.data), num_cons, num_vars, _p(x), len(x), _p(ev), gens.h, transcript.state, _p(rx), _p(ry)))
        return rx[:nx], ry[:ny]


class NIZK:
    """lib.rs:488-591.  `bytes` = bincode::serialize(&NIZK)"""

    def __init__(self, data):
        self.bytes = data

    @staticmethod
    def prove(inst, vars, inputs, gens, transcript_label, seed=None):
        """NIZK::prove(&inst, vars, &inputs, &gens, &mut Transcript::new(transcript_label)).  `seed`: RandomTape seed scalar limbs; None (the
        default) draws it from the OS like the reference (random.rs:13-15).  Pass tape_seed(k) only for reproducible test / bench runs."""
        ctx = inst.ctx
        seed = random_tape_seed() if seed is None else np.ascontiguousarray(seed, dtype=np.uint64)
        out, n = C.POINTER(C.c_ubyte)(), _sz()
        if isinstance(transcript_label, Transcript):   # the caller's `&mut Transcript`: advanced in place
            v = vars.to_numpy() if isinstance(vars, DensePolynomial) else vars.limbs
            ctx.check(lib.sp_nizk_prove_t(ctx.h, inst.h, _p(v), len(v), _p(inputs.limbs), len(inputs), gens.h, transcript_label.state, _p(seed),
                                          C.byref(out), C.byref(n)))
        elif isinstance(vars, DensePolynomial):
            ctx.check(lib.sp_nizk_prove_resident(ctx.h, inst.h, vars.h, _p(inputs.limbs), len(inputs), gens.h, bytes(transcript_label),
                                                 len(transcript_label), _p(seed), C.byref(out), C.byref(n)))
        else:
            ctx.check(lib.sp_nizk_prove(ctx.h, inst.h, _p(vars.limbs), len(vars), _p(inputs.limbs), len(inputs), gens.h,
                                        bytes(transcript_label), len(transcript_label), _p(seed), C.byref(out), C.byref(n)))
        return NIZK(_take_bytes(out, n))

    def verify(self, inst, inputs, transcript_label, gens):
        """NIZK::verify(&self, &inst, &inputs, &mut Transcript::new(transcript_label), &gens): returns None, raises ProofVerifyError"""
        ctx = inst.ctx
        if isinstance(transcript_label, Transcript):
            ctx.check(lib.sp_nizk_verify_t(ctx.h, inst.h, _p(inputs.limbs), len(inputs), gens.h, transcript_label.state, bytes(self.bytes), len(self.bytes)))
            return
        ctx.check(lib.sp_nizk_verify(ctx.h, inst.h, _p(inputs.limbs), len(inputs), gens.h, bytes(transcript_label), len(transcript_label),
                                     bytes(self.bytes), len(self.bytes)))

    @staticmethod
    def verify_batch(proofs, inst, inputs, transcript_label, gens, seed=None):
        """NIZK::verify for k proofs in one call (sp_nizk_verify_batch): `inst` one Instance or a list of k, `inputs` a list of k assignments,
        `transcript_label` one label, k labels or k Transcript objects (advanced in place as NIZK.verify advances one).  Returns k entries: None
        (accepted) or a ProofVerifyError whose `.code` is the status the single verify gives that proof; the lowest rejected proof's error also
        carries the single verify's message, the others a generic one.  Rejections do not raise, bad arguments do.
        seed=None (the default) draws the seed of the batch weights from the OS; a known seed lets a false proof pass."""
        return _verify_batch(gens.ctx, lib.sp_nizk_verify_batch, lib.sp_nizk_verify_batch_t, inst, proofs, inputs, transcript_label, gens, seed)


class SNARKGens(_Handle):
    """lib.rs:277-309.  tables=GeneratorTables (built with num_nz_entries > 0): a view into them instead of generator tables of its own"""
    _free = lib.sp_snark_gens_free

    def __init__(self, num_cons, num_vars, num_inputs, num_nz_entries, ctx=None, tables=None):
        self.ctx = ctx or (tables.ctx if tables is not None else default_context())
        h = _vp()
        if tables is None:
            self.ctx.check(lib.sp_snark_gens_create(self.ctx.h, num_cons, num_vars, num_inputs, num_nz_entries, C.byref(h)))
        else:
            self.ctx.check(lib.sp_snark_gens_create_from(self.ctx.h, tables.h, num_cons, num_vars, num_inputs, num_nz_entries, C.byref(h)))
        self.h = h

    @staticmethod
    def new(num_cons, num_vars, num_inputs, num_nz_entries, ctx=None):
        return SNARKGens(num_cons, num_vars, num_inputs, num_nz_entries, ctx)


class ComputationCommitment(_Handle):
    """(ComputationCommitment, ComputationDecommitment) pair of SNARK::encode (lib.rs:44-55): the decommitment stays on the device"""
    _free = lib.sp_snark_encoding_free

    def __init__(self, ctx, h):
        self.ctx, self.h = ctx, h

    @classmethod
    def from_bytes(cls, data, ctx=None):
        """a verifier's view: bincode(ComputationCommitment) only (cannot be used to prove)"""
        ctx = ctx or default_context()
        h = _vp()
        ctx.check(lib.sp_snark_commitment_load(ctx.h, bytes(data), len(data), C.byref(h)))
        return cls(ctx, h)

    def commitment_bytes(self):
        out, n = C.POINTER(C.c_ubyte)(), _sz()
        _check_host(lib.sp_snark_commitment_bytes(self.h, C.byref(out), C.byref(n)))
        return _take_bytes(out, n)


class SNARK:
    """lib.rs:311-465.  `bytes` = bincode::serialize(&SNARK)"""

    def __init__(self, data):
        self.bytes = data

    @staticmethod
    def encode(inst, gens):
        """SNARK::encode (lib.rs:325-336) -> ComputationCommitment (holding the decommitment too)"""
        h = _vp()
        inst.ctx.check(lib.sp_snark_encode(inst.ctx.h, inst.h, gens.h, C.byref(h)))
        return ComputationCommitment(inst.ctx, h)

    @staticmethod
    def prove(inst, comm, vars, inputs, gens, transcript_label, seed=None):
        """SNARK::prove(&inst, &comm, &decomm, vars, &inputs, &gens, &mut Transcript::new(transcript_label)).  `seed` as in NIZK.prove:
        None = fresh OS randomness (zero-knowledge); tape_seed(k) = deterministic, for tests and benchmarks only."""
        ctx = inst.ctx
        seed = random_tape_seed() if seed is None else np.ascontiguousarray(seed, dtype=np.uint64)
        out, n = C.POINTER(C.c_ubyte)(), _sz()
        if isinstance(transcript_label, Transcript):   # the caller's `&mut Transcript`: advanced in place
            v = vars.to_numpy() if isinstance(vars, DensePolynomial) else vars.limbs
            ctx.check(lib.sp_snark_prove_t(ctx.h, inst.h, comm.h, _p(v), len(v), _p(inputs.limbs), len(inputs), gens.h, transcript_label.state, _p(seed),
                                           C.byref(out), C.byref(n)))
        elif isinstance(vars, DensePolynomial):
            ctx.check(lib.sp_snark_prove_resident(ctx.h, inst.h, comm.h, vars.h, _p(inputs.limbs), len(inputs), gens.h, bytes(transcript_label),
                                                  len(transcript_label), _p(seed), C.byref(out), C.byref(n)))
        else:
            ctx.check(lib.sp_snark_prove(ctx.h, inst.h, comm.h, _p(vars.limbs), len(vars), _p(inputs.limbs), len(inputs), gens.h,
                                         bytes(transcript_label), len(transcript_label), _p(seed), C.byref(out), C.byref(n)))
        return SNARK(_take_bytes(out, n))

    def verify(self, comm, inputs, transcript_label, gens):
        """SNARK::verify(&self, &comm, &inputs, &mut Transcript::new(transcript_label), &gens): returns None, raises ProofVerifyError"""
        ctx = comm.ctx
        if isinstance(transcript_label, Transcript):
            ctx.check(lib.sp_snark_verify_t(ctx.h, comm.h, _p(inputs.limbs), len(inputs), gens.h, transcript_label.state, bytes(self.bytes), len(self.bytes)))
            return
        ctx.check(lib.sp_snark_verify(ctx.h, comm.h, _p(inputs.limbs), len(inputs), gens.h, bytes(transcript_label), len(transcript_label),
                                      bytes(self.bytes), len(self.bytes)))

    @staticmethod
    def verify_batch(proofs, comm, inputs, transcript_label, gens, seed=None):
        """SNARK::verify for k proofs in one call (sp_snark_verify_batch): `comm` one ComputationCommitment or a list of k; otherwise as
        NIZK.verify_batch"""
        return _verify_batch(gens.ctx, lib.sp_snark_verify_batch, lib.sp_snark_verify_batch_t, comm, proofs, inputs, transcript_label, gens, seed)


def _verify_batch(ctx, entry, entry_t, handles, proofs, inputs, transcript_label, gens, seed):
    """the shared body of SNARK.verify_batch / NIZK.verify_batch: one sp_*_verify_batch(_t) call, statuses -> [None | ProofVerifyError]"""
    k = len(proofs)
    if len(inputs) != k:
        raise SpartanB200Error("verify_batch: %d proofs but %d input assignments" % (k, len(inputs)))
    if not isinstance(handles, (list, tuple)):
        handles = [handles] * k
    if len(handles) != k:
        raise SpartanB200Error("verify_batch: %d proofs but %d statements" % (k, len(handles)))
    if isinstance(transcript_label, (bytes, bytearray)):
        transcript_label = [bytes(transcript_label)] * k
    if len(transcript_label) != k:
        raise SpartanB200Error("verify_batch: %d proofs but %d transcripts" % (k, len(transcript_label)))
    seed = os.urandom(32) if seed is None else bytes(seed)
    if len(seed) != 32:
        raise SpartanB200Error("verify_batch: the weight seed is 32 bytes")
    datas = [bytes(p.bytes if hasattr(p, "bytes") else p) for p in proofs]
    limbs = [np.ascontiguousarray(a.limbs, dtype=np.uint64) for a in inputs]
    hs = (_vp * k)(*[h.h for h in handles])
    ins = (_vp * k)(*[_p(a) for a in limbs])
    nins = (_sz * k)(*[len(a) for a in limbs])
    pbuf = (C.c_char_p * k)(*datas)
    plens = (_sz * k)(*[len(d) for d in datas])
    status = (C.c_int * k)()
    if any(isinstance(t, Transcript) for t in transcript_label) and not all(isinstance(t, Transcript) for t in transcript_label):
        raise SpartanB200Error("verify_batch: transcript_label mixes Transcript objects and labels")
    if all(isinstance(t, Transcript) for t in transcript_label):
        states = (_vp * k)(*[C.cast(t.state, _vp) for t in transcript_label])
        rc = entry_t(ctx.h, k, hs, ins, nins, gens.h, states, pbuf, plens, seed, status)
    else:
        labels = [bytes(t) for t in transcript_label]
        lbuf = (C.c_char_p * k)(*labels)
        llens = (_sz * k)(*[len(t) for t in labels])
        rc = entry(ctx.h, k, hs, ins, nins, gens.h, lbuf, llens, pbuf, plens, seed, status)
    if rc not in (SP_OK, SP_ERR_VERIFY):
        ctx.check(rc)
    out = []
    for i in range(k):
        code = status[i]
        if code == SP_OK:
            out.append(None)
        else:
            kind = "DecompressionError" if code == SP_ERR_DECOMPRESS else "InternalError"
            out.append(ProofVerifyError("%s: proof %d rejected (status %d)" % (kind, i, code), code))
    if rc == SP_ERR_VERIFY:   # the message of the lowest rejected proof
        first = next(i for i in range(k) if status[i] != SP_OK)
        out[first] = ProofVerifyError(("DecompressionError: " if status[first] == SP_ERR_DECOMPRESS else "InternalError: ") +
                                      lib.sp_last_error(ctx.h).decode(), status[first])
    return out




# ----------------------------------------------------------------------------- measurement helpers (bench.py)
def io_bytes():
    a, b = C.c_ulonglong(), C.c_ulonglong()
    lib.sp_io_bytes(C.byref(a), C.byref(b))
    return int(a.value), int(b.value)


def prof_enable(on=True):
    lib.sp_prof_enable(1 if on else 0)


def prof_report():
    """{kernel family: {"launches", "ms", "bytes"}} measured with CUDA events on the launching stream"""
    out = {}
    for item in _string_out(_check_host, lib.sp_prof_report).split(";"):
        if item:
            name, n, ms, by, bb, bms = item.split(":")
            out[name] = {"launches": int(n), "ms": float(ms), "bytes": float(by), "largest_bytes": float(bb), "largest_ms": float(bms)}
    return out


def timer_start(ctx=None):
    ctx = ctx or default_context()
    ctx.check(lib.sp_timer_start(ctx.h))


def timer_stop_ms(ctx=None):
    ctx = ctx or default_context()
    ms = C.c_float()
    ctx.check(lib.sp_timer_stop_ms(ctx.h, C.byref(ms)))
    return float(ms.value)
