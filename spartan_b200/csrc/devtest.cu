// spartan_b200 — device test hooks, the GPU counterpart of hosttest.cpp.  Built with the kernels' nvcc flags, so the field and curve arithmetic
// here is the code the kernels run on the device (inline-PTX carry chains, generated multiplications, quad-lane point operations), not the portable
// formulation the CPU tests check.  Not linked into libspartan_b200.so; linked with the kernel objects of libspartan_b200.so instead, so the
// kernel hooks below (spd_sc_*, spd_eq_*, ...) launch the library's own kernels through the sp::dev wrappers of dev.hpp.
//
// Every arithmetic entry point takes host arrays of n elements, copies them to the device, runs one elementwise kernel (one thread per element, or
// one quad of lanes per point for the quad-lane operations), copies the results back and returns the CUDA status (0 = success).
//   u256:     8 little-endian 32-bit limbs.  F_q operands are Montgomery limbs, passed and returned unchanged; F_p operands may be any value < 2^256.
//   ge:       the four coordinates X, Y, Z, T as u256 (any representatives, not necessarily reduced or normalised).
//   ge_niels: y + x, y - x, 2dxy as u256.
// Every kernel hook also takes and returns host arrays (F_q values as Montgomery limbs), runs the wrappers on a stream of its own, frees its device
// and pinned buffers on return and returns 0, a CUDA status, or SPD_REFUSED when a wrapper threw (spd_last_error() then holds its message).
#include <cuda_runtime.h>
#include <string.h>
#include <algorithm>
#include <chrono>
#include <exception>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>
#include "kcommon.cuh"
#include "quad.cuh"
#include "snark.hpp"

using namespace sp;
using namespace sp::dev;

namespace {

constexpr int TPB = 128;
unsigned blocks_for(size_t threads) { return (unsigned)((threads + TPB - 1) / TPB); }

// device copies of one call's arrays, freed on return; the first failing CUDA call is kept and later steps are skipped.  Under the memory-check
// mode (spd_memcheck) the arrays come from the library's pool instead of cudaMalloc: filled by type and guarded, the guard checked on return.
struct Call {
  std::vector<void*> bufs;
  std::vector<bool> pooled;
  cudaError_t err = cudaSuccess;
  template <class T> T* alloc(size_t n) {
    void* d = nullptr;
    const bool mc = memcheck_on();
    if (err == cudaSuccess) {
      if (!mc) err = cudaMalloc(&d, n * sizeof(T));
      else try { d = pool_alloc(n * sizeof(T), pool_fill_of<T>()); } catch (const std::exception&) { err = cudaErrorMemoryAllocation; }
    }
    bufs.push_back(d);
    pooled.push_back(mc);
    return (T*)d;
  }
  template <class T> T* in(const T* h, size_t n) {
    T* d = alloc<T>(n);
    if (err == cudaSuccess) err = cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice);
    return d;
  }
  template <class T> void out(T* h, const T* d, size_t n) {
    if (err == cudaSuccess) err = cudaMemcpy(h, d, n * sizeof(T), cudaMemcpyDeviceToHost);
  }
  bool ok() const { return err == cudaSuccess; }
  void launched() { if (err == cudaSuccess) err = cudaGetLastError(); }
  ~Call() { for (size_t i = 0; i < bufs.size(); i++) if (bufs[i]) { if (pooled[i]) pool_free(bufs[i]); else cudaFree(bufs[i]); } }
};

// one call of a kernel hook: a Call whose wrappers run on a stream of its own (a blocking stream: ordered after the synchronous copies of in() and
// before those of out()), drained before the buffers go, plus zeroed device and pinned host buffers for scratch and the HostSig words.  Scratch
// counters and flag words start at zero by contract, also under the memory-check mode; pinned result arrays of field elements get 0xFF there.
constexpr int SPD_REFUSED = -1;
std::string g_last_error;
struct KCall : Call {
  cudaStream_t s = nullptr;
  std::vector<void*> pinned;
  KCall() { err = cudaStreamCreate(&s); }
  ~KCall() {
    if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); }
    for (void* p : pinned) if (p) cudaFreeHost(p);
  }
  template <class T> T* zeros(size_t n) {
    T* d = alloc<T>(n);
    if (err == cudaSuccess) err = cudaMemset(d, 0, n * sizeof(T));
    return d;
  }
  template <class T> T* host(size_t n) {
    void* p = nullptr;
    if (err == cudaSuccess) err = cudaMallocHost(&p, n * sizeof(T));
    if (err == cudaSuccess) memset(p, memcheck_on() && pool_fill_of<T>() == FILL_FF ? 0xFF : 0, n * sizeof(T));
    pinned.push_back(p);
    return (T*)p;
  }
  void sync() { if (err == cudaSuccess) err = cudaStreamSynchronize(s); }
};
// a wrapper's std::exception (a refused argument, a CUDA error it checked) becomes SPD_REFUSED; the KCall inside `f` is unwound first
template <class F> int guarded(F&& f) {
  try {
    return f();
  } catch (const std::exception& e) {
    g_last_error = e.what();
    return SPD_REFUSED;
  }
}
// reduction scratch of the dot / sparse kernels: [counters][partials], the same layout as the sumcheck kernels' (>= 32 tables)
size_t red_scratch_bytes() { return sc_scratch_bytes(32); }

enum FqOp { FQ_MUL, FQ_ADD, FQ_SUB, FQ_NEG, FQ_FROM_MONT, FQ_TO_MONT, FQ_FROM_WIDE, FQ_FROM_U64, FQ_INV };
enum FpOp { FP_MUL, FP_ADD, FP_SUB, FP_NEG, FP_MUL_SMALL, FP_CANON, FP_INV, FP_POW22523 };
enum GeOp { GE_ADD, GE_DBL };
enum QuadOp { QUAD_ADD, QUAD_MADD, QUAD_DBL };

__global__ void k_fq(int op, size_t n, const u256* a, const u256* b, u256* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u256 x = a[i], y = b ? b[i] : fq_zero();
  u256 r;
  switch (op) {
    case FQ_MUL: r = fq_mul(x, y); break;
    case FQ_ADD: r = fq_add(x, y); break;
    case FQ_SUB: r = fq_sub(x, y); break;
    case FQ_NEG: r = fq_neg(x); break;
    case FQ_FROM_MONT: r = fq_from_mont(x); break;
    case FQ_TO_MONT: r = fq_to_mont(x); break;
    case FQ_FROM_WIDE: r = fq_from_wide(x, y); break;                                   // x: low half, y: high half
    case FQ_FROM_U64: r = fq_from_u64((uint64_t)x.v[0] | ((uint64_t)x.v[1] << 32)); break;
    default: r = fq_inv(x); break;
  }
  out[i] = r;
}
__global__ void k_fq_fold_const(size_t n, const u256* a0, const u256* a1, const __grid_constant__ FqConst rc, u256* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = fq_fold_const(a0[i], a1[i], rc);
}
__global__ void k_fp(int op, size_t n, const u256* a, const u256* b, u256* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u256 x = a[i], y = b ? b[i] : fp_zero();
  u256 r;
  switch (op) {
    case FP_MUL: r = fp_mul(x, y); break;
    case FP_ADD: r = fp_add(x, y); break;
    case FP_SUB: r = fp_sub(x, y); break;
    case FP_NEG: r = fp_neg(x); break;
    case FP_MUL_SMALL: r = fp_mul_small(x, y.v[0]); break;                                // the multiplier is the low limb of b
    case FP_CANON: r = fp_canon(x); break;
    case FP_INV: r = fp_inv(x); break;
    default: r = fp_pow22523(x); break;
  }
  out[i] = r;
}
__global__ void k_fp_sqrt_ratio_i(size_t n, const u256* u, const u256* v, u256* out, int* flag) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  u256 r;
  flag[i] = fp_sqrt_ratio_i(r, u[i], v[i]) ? 1 : 0;
  out[i] = r;
}
__global__ void k_ge(int op, size_t n, const ge* p, const ge* q, ge* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = op == GE_ADD ? ge_add(p[i], q[i]) : ge_dbl(p[i]);
}
__global__ void k_ge_madd(size_t n, const ge* p, const ge_niels* q, int neg, ge* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = ge_madd(p[i], q[i], neg != 0);
}
__global__ void k_ge_to_niels(size_t n, const ge* p, ge_niels* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = ge_to_niels(p[i]);
}
__global__ void k_encode(size_t n, const ge* p, u256* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = ristretto_encode(p[i]);
}
__global__ void k_decode(size_t n, const u256* s, ge* out, int* ok) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  ge g = ge_identity();
  ok[i] = ristretto_decode(g, s[i]) ? 1 : 0;
  out[i] = g;
}
__global__ void k_map(size_t n, const u256* t, ge* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = ristretto_map(t[i]);
}
__global__ void k_from_uniform(size_t n, const u256* lo, const u256* hi, ge* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = ristretto_from_uniform(lo[i], hi[i]);
}
// four lanes per point, lane c holding coordinate c, as k_msm_horner and k_ipa_msm_quad run them.  The grid covers whole warps: lanes past the
// last point carry the identity and still take part in every shuffle.
__global__ void k_quad(int op, size_t n, const ge* p, const ge* q, const ge_niels* nq, int neg, ge* out) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x, i = t >> 2;
  const int lane = threadIdx.x & 31, c = lane & 3;
  const bool live = i < n;
  const u256 P = live ? reinterpret_cast<const u256*>(p + i)[c] : quad_identity(c);
  u256 r;
  if (op == QUAD_ADD) {
    r = quad_add(P, live ? reinterpret_cast<const u256*>(q + i)[c] : quad_identity(c), c, lane);
  } else if (op == QUAD_MADD) {
    u256 x = c == 3 ? fp_zero() : fp_one();                   // operand of +/-q per lane: (y - x, y + x, -, 2dxy), as k_ipa_msm_quad builds it
    if (live) {
      if (c == 0) x = neg ? nq[i].ypx : nq[i].ymx;
      else if (c == 1) x = neg ? nq[i].ymx : nq[i].ypx;
      else if (c == 3) { x = nq[i].t2d; if (neg) x = fp_neg(x); }
    }
    r = quad_madd(P, x, c, lane);
  } else {
    r = quad_dbl(P, c, lane);
  }
  if (live) reinterpret_cast<u256*>(out + i)[c] = r;
}
// signed W-bit digits of all windows (curve.cuh signed_digit, the recoding of k_msm_digits)
__global__ void k_signed_digits(size_t n, const u256* k, int wbits, int* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int nwin = (253 + wbits - 1) / wbits;
  const u256 x = k[i];
  uint32_t carry = 0;
  for (int w = 0; w < nwin; w++) out[i * nwin + w] = signed_digit(x, w, wbits, carry);
}
// digit w of the per-window MSMs (k_msm_rows, k_ipa_msm_quad) as computed by a thread whose first window is w: the carry into w from the recoding
// of the lower windows, then msm_window<W>(k, w) + carry, signed
template <int WBITS>
__global__ void k_window_digits(size_t n, const u256* k, int* out) {
  constexpr int NWIN = (253 + WBITS - 1) / WBITS;
  constexpr uint32_t HALF = 1u << (WBITS - 1);
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u256 x = k[i];
  for (int w0 = 0; w0 < NWIN; w0++) {
    uint32_t carry = 0;
    for (int w = 0; w < w0; w++) carry = (msm_window<WBITS>(x, w) + carry) > HALF ? 1u : 0u;
    const uint32_t v = msm_window<WBITS>(x, w0) + carry;
    out[i * NWIN + w0] = v > HALF ? (int)v - (int)(2 * HALF) : (int)v;
  }
}

// ---- generator-table checker.  An affine-niels table of nslots generators, entry (j, w, d) at (j nwin + w) depth + d - 1, must hold
// d 2^(W w) G_{base(j)}: per-window tables (W = 8, 13, 15: nwin = ceil(253 / W), depth = 2^(W-1)), row tables (nwin = 1, depth = 2^15), host copies
// (the 8-bit layout over a list of bases).  One thread per run of CHECK_RUN entries of one window computes B = 2^(W w) G by W w doublings and
// d0 B by double-and-add from G itself, never from the table, then walks the run with one mixed addition per entry and compares each stored entry
// with the extended point by cross-multiplication (ypx Z = Y + X, ymx Z = Y - X, t2d Z = 2d T mod p, both sides canonical) and requires every
// stored coordinate to be canonical (< p), as ge_to_niels leaves it.  A wrong entry is therefore reported at its own index and nowhere else.
constexpr size_t CHECK_RUN = 256;
constexpr unsigned CHECK_LIST = 1u << 16;   // bad indices kept for the report; past this the list is no longer the first ones in index order
enum { CK_SEEN, CK_BAD, CK_YPX, CK_YMX, CK_T2D, CK_NONCANON, CK_LISTED, CK_COUNTERS };
__global__ void __launch_bounds__(64) k_niels_check(const ge_niels* __restrict__ table, size_t nslots, int wbits, int nwin, size_t depth, const ge* __restrict__ G,
                                                    const int64_t* __restrict__ bases, unsigned long long* counters, unsigned long long* list) {
  const size_t runs = (depth + CHECK_RUN - 1) / CHECK_RUN;
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nslots * (size_t)nwin * runs) return;
  const size_t j = t / ((size_t)nwin * runs), r = t % runs;
  const int w = (int)((t / runs) % nwin);
  const ge* g = G + (bases ? (size_t)bases[j] : j);
  ge B;
  B.X = ld256_ro(&g->X); B.Y = ld256_ro(&g->Y); B.Z = ld256_ro(&g->Z); B.T = ld256_ro(&g->T);
  for (int k = 0; k < wbits * w; k++) B = ge_dbl(B);
  const ge_niels Bn = ge_to_niels(B);
  const size_t d0 = r * CHECK_RUN + 1, d1 = d0 + CHECK_RUN - 1 < depth ? d0 + CHECK_RUN - 1 : depth;
  u256 k0 = fq_zero();
  k0.v[0] = (uint32_t)d0;
  ge acc = ge_scalarmul(k0, B);
  const ge_niels* e = table + ((size_t)j * nwin + w) * depth;
  atomicAdd(&counters[CK_SEEN], (unsigned long long)(d1 - d0 + 1));
  for (size_t d = d0; d <= d1; d++) {
    if (d > d0) acc = ge_madd(acc, Bn, false);
    const u256 ypx = ld256_ro(&e[d - 1].ypx), ymx = ld256_ro(&e[d - 1].ymx), t2d = ld256_ro(&e[d - 1].t2d);
    const bool b_ypx = !fp_eq(fp_mul(ypx, acc.Z), fp_add(acc.Y, acc.X));
    const bool b_ymx = !fp_eq(fp_mul(ymx, acc.Z), fp_sub(acc.Y, acc.X));
    const bool b_t2d = !fp_eq(fp_mul(t2d, acc.Z), fp_mul(acc.T, fp_2D()));
    const bool b_canon = !fq_eq(fp_canon(ypx), ypx) || !fq_eq(fp_canon(ymx), ymx) || !fq_eq(fp_canon(t2d), t2d);
    if (!(b_ypx || b_ymx || b_t2d || b_canon)) continue;
    atomicAdd(&counters[CK_BAD], 1ull);
    if (b_ypx) atomicAdd(&counters[CK_YPX], 1ull);
    if (b_ymx) atomicAdd(&counters[CK_YMX], 1ull);
    if (b_t2d) atomicAdd(&counters[CK_T2D], 1ull);
    if (b_canon) atomicAdd(&counters[CK_NONCANON], 1ull);
    const unsigned long long slot = atomicAdd(&counters[CK_LISTED], 1ull);
    if (slot < CHECK_LIST) list[slot] = ((size_t)j * nwin + w) * depth + d - 1;
  }
}

// one check on c's stream.  out (24 words): entries the kernel compared, bad entries, ypx / ymx / t2d mismatches, entries with a non-canonical coordinate, the
// number of indices listed (<= 16), 1 when they are exactly the first bad entries in index order, then the listed entry indices, ascending
constexpr int CHECK_OUT = 24;
void niels_check(KCall& c, const ge_niels* table, size_t nslots, int wbits, const ge* G, const int64_t* d_bases, uint64_t* out) {
  memset(out, 0, CHECK_OUT * sizeof(uint64_t));
  const int nwin = wbits ? (253 + wbits - 1) / wbits : 1;
  const size_t depth = (size_t)1 << (wbits ? wbits - 1 : 15);
  unsigned long long* counters = c.zeros<unsigned long long>(CK_COUNTERS);
  unsigned long long* list = c.alloc<unsigned long long>(CHECK_LIST);
  const size_t threads = nslots * (size_t)nwin * ((depth + CHECK_RUN - 1) / CHECK_RUN);
  if (c.ok() && threads) k_niels_check<<<(unsigned)((threads + 63) / 64), 64, 0, c.s>>>(table, nslots, wbits, nwin, depth, G, d_bases, counters, list);
  c.launched();
  c.sync();
  unsigned long long h[CK_COUNTERS];
  c.out(h, counters, CK_COUNTERS);
  if (!c.ok()) return;
  const size_t kept = h[CK_LISTED] < CHECK_LIST ? h[CK_LISTED] : CHECK_LIST;
  std::vector<unsigned long long> idx(kept);
  c.out(idx.data(), list, kept);
  std::sort(idx.begin(), idx.end());
  for (int k = 0; k < 6; k++) out[k] = h[CK_SEEN + k];
  out[6] = kept < 16 ? kept : 16;
  out[7] = h[CK_LISTED] <= CHECK_LIST ? 1 : 0;
  for (size_t k = 0; k < out[6]; k++) out[8 + k] = idx[k];
}
// radix-2^51 host limbs -> the 256-bit value they stand for; limbs past 51 bits (never written by to_hniels) give all ones, which no canonical
// coordinate equals
u256 fe51_value(const fe51& a) {
  u256 r;
  for (int i = 0; i < 5; i++)
    if (a.v[i] >> 51) { for (int k = 0; k < 8; k++) r.v[k] = 0xffffffffu; return r; }
  const uint64_t w[4] = {a.v[0] | (a.v[1] << 51), (a.v[1] >> 13) | (a.v[2] << 38), (a.v[2] >> 26) | (a.v[3] << 25), (a.v[3] >> 39) | (a.v[4] << 12)};
  for (int k = 0; k < 4; k++) { r.v[2 * k] = (uint32_t)w[k]; r.v[2 * k + 1] = (uint32_t)(w[k] >> 32); }
  return r;
}
struct ReleaseCached { ~ReleaseCached() { pool_release_cached(); } };   // a set's freed tables go back to the device, not to this library's pool
// a generator set built as the library builds one: by label, or (enc non-null) from nbases encodings decoded on the device as sp_gens_upload does
std::unique_ptr<GenSet> make_set(Ctx& ctx, const uint8_t* label, size_t label_len, size_t nbases, const uint8_t* enc, const std::vector<size_t>& hb) {
  if (!enc) return std::unique_ptr<GenSet>(new GenSet(&ctx, std::string((const char*)label, label_len), nbases, hb));
  DevBuf<uint8_t> d_in(32 * nbases);
  DevBuf<ge> pts(nbases);
  DevBuf<int> d_ok(nbases);
  std::vector<int> ok(nbases);
  h2d(d_in.p, enc, 32 * nbases, ctx.stream);
  decompress_batch(pts.p, d_ok.p, d_in.p, nbases, ctx.stream);
  d2h(ok.data(), d_ok.p, sizeof(int) * nbases, ctx.stream);
  ctx.sync();
  for (size_t i = 0; i < nbases; i++) if (!ok[i]) throw std::runtime_error("encoding " + std::to_string(i) + " is not a ristretto255 point");
  return std::unique_ptr<GenSet>(new GenSet(&ctx, pts.p, nbases, hb));
}

}  // namespace

extern "C" {
int spd_fq(int op, size_t n, const u256* a, const u256* b, u256* out) {   // b: second operand of mul / add / sub, high half of from_wide; else unused
  if (op < FQ_MUL || op > FQ_INV) return (int)cudaErrorInvalidValue;
  if (!n) return 0;
  Call c;
  const bool two = op == FQ_MUL || op == FQ_ADD || op == FQ_SUB || op == FQ_FROM_WIDE;
  const u256* da = c.in(a, n);
  const u256* db = two ? c.in(b, n) : nullptr;
  u256* dout = c.alloc<u256>(n);
  if (c.ok()) k_fq<<<blocks_for(n), TPB>>>(op, n, da, db, dout);
  c.launched();
  c.out(out, dout, n);
  return (int)c.err;
}
// a0 + r*(a1 - a0) with the constant-multiplier table of r (Montgomery limbs) built on the host by fq_const_table and passed as a
// __grid_constant__ argument, as sc_fold_eval does
int spd_fq_fold_const(size_t n, const u256* a0, const u256* a1, const u256* r_mont, u256* out) {
  if (!n) return 0;
  const FqConst rc = fq_const_table(*r_mont);
  Call c;
  const u256* d0 = c.in(a0, n);
  const u256* d1 = c.in(a1, n);
  u256* dout = c.alloc<u256>(n);
  if (c.ok()) k_fq_fold_const<<<blocks_for(n), TPB>>>(n, d0, d1, rc, dout);
  c.launched();
  c.out(out, dout, n);
  return (int)c.err;
}
int spd_fp(int op, size_t n, const u256* a, const u256* b, u256* out) {   // b: second operand of mul / add / sub, multiplier of mul_small; else unused
  if (op < FP_MUL || op > FP_POW22523) return (int)cudaErrorInvalidValue;
  if (!n) return 0;
  Call c;
  const bool two = op == FP_MUL || op == FP_ADD || op == FP_SUB || op == FP_MUL_SMALL;
  const u256* da = c.in(a, n);
  const u256* db = two ? c.in(b, n) : nullptr;
  u256* dout = c.alloc<u256>(n);
  if (c.ok()) k_fp<<<blocks_for(n), TPB>>>(op, n, da, db, dout);
  c.launched();
  c.out(out, dout, n);
  return (int)c.err;
}
int spd_fp_sqrt_ratio_i(size_t n, const u256* u, const u256* v, u256* out, int* was_square) {
  if (!n) return 0;
  Call c;
  const u256* du = c.in(u, n);
  const u256* dv = c.in(v, n);
  u256* dout = c.alloc<u256>(n);
  int* dflag = c.alloc<int>(n);
  if (c.ok()) k_fp_sqrt_ratio_i<<<blocks_for(n), TPB>>>(n, du, dv, dout, dflag);
  c.launched();
  c.out(out, dout, n);
  c.out(was_square, dflag, n);
  return (int)c.err;
}
int spd_ge(int op, size_t n, const ge* p, const ge* q, ge* out) {   // GE_ADD: p + q, GE_DBL: 2p (q unused)
  if (op != GE_ADD && op != GE_DBL) return (int)cudaErrorInvalidValue;
  if (!n) return 0;
  Call c;
  const ge* dp = c.in(p, n);
  const ge* dq = op == GE_ADD ? c.in(q, n) : nullptr;
  ge* dout = c.alloc<ge>(n);
  if (c.ok()) k_ge<<<blocks_for(n), TPB>>>(op, n, dp, dq, dout);
  c.launched();
  c.out(out, dout, n);
  return (int)c.err;
}
int spd_ge_madd(size_t n, const ge* p, const ge_niels* q, int neg, ge* out) {
  if (!n) return 0;
  Call c;
  const ge* dp = c.in(p, n);
  const ge_niels* dq = c.in(q, n);
  ge* dout = c.alloc<ge>(n);
  if (c.ok()) k_ge_madd<<<blocks_for(n), TPB>>>(n, dp, dq, neg, dout);
  c.launched();
  c.out(out, dout, n);
  return (int)c.err;
}
int spd_ge_to_niels(size_t n, const ge* p, ge_niels* out) {
  if (!n) return 0;
  Call c;
  const ge* dp = c.in(p, n);
  ge_niels* dout = c.alloc<ge_niels>(n);
  if (c.ok()) k_ge_to_niels<<<blocks_for(n), TPB>>>(n, dp, dout);
  c.launched();
  c.out(out, dout, n);
  return (int)c.err;
}
int spd_ristretto_encode(size_t n, const ge* p, u256* out) {
  if (!n) return 0;
  Call c;
  const ge* dp = c.in(p, n);
  u256* dout = c.alloc<u256>(n);
  if (c.ok()) k_encode<<<blocks_for(n), TPB>>>(n, dp, dout);
  c.launched();
  c.out(out, dout, n);
  return (int)c.err;
}
int spd_ristretto_decode(size_t n, const u256* s, ge* out, int* ok) {
  if (!n) return 0;
  Call c;
  const u256* ds = c.in(s, n);
  ge* dout = c.alloc<ge>(n);
  int* dok = c.alloc<int>(n);
  if (c.ok()) k_decode<<<blocks_for(n), TPB>>>(n, ds, dout, dok);
  c.launched();
  c.out(out, dout, n);
  c.out(ok, dok, n);
  return (int)c.err;
}
int spd_ristretto_map(size_t n, const u256* t, ge* out) {
  if (!n) return 0;
  Call c;
  const u256* dt = c.in(t, n);
  ge* dout = c.alloc<ge>(n);
  if (c.ok()) k_map<<<blocks_for(n), TPB>>>(n, dt, dout);
  c.launched();
  c.out(out, dout, n);
  return (int)c.err;
}
int spd_ristretto_from_uniform(size_t n, const u256* lo, const u256* hi, ge* out) {
  if (!n) return 0;
  Call c;
  const u256* dl = c.in(lo, n);
  const u256* dh = c.in(hi, n);
  ge* dout = c.alloc<ge>(n);
  if (c.ok()) k_from_uniform<<<blocks_for(n), TPB>>>(n, dl, dh, dout);
  c.launched();
  c.out(out, dout, n);
  return (int)c.err;
}
// QUAD_ADD: p + q, QUAD_MADD: p +/- q with q in niels form (neg selects -q), QUAD_DBL: 2p
int spd_quad(int op, size_t n, const ge* p, const ge* q, const ge_niels* nq, int neg, ge* out) {
  if (op < QUAD_ADD || op > QUAD_DBL) return (int)cudaErrorInvalidValue;
  if (!n) return 0;
  Call c;
  const ge* dp = c.in(p, n);
  const ge* dq = op == QUAD_ADD ? c.in(q, n) : nullptr;
  const ge_niels* dn = op == QUAD_MADD ? c.in(nq, n) : nullptr;
  ge* dout = c.alloc<ge>(n);
  if (c.ok()) k_quad<<<blocks_for(4 * n), TPB>>>(op, n, dp, dq, dn, neg, dout);   // TPB is a multiple of 32: whole warps
  c.launched();
  c.out(out, dout, n);
  return (int)c.err;
}
// out[i * nwin + w]: signed wbits-bit digit w of canonical scalar k[i] (wbits in 2..24), nwin = ceil(253 / wbits)
int spd_signed_digits(size_t n, const u256* k, int wbits, int* out) {
  if (wbits < 2 || wbits > 24) return (int)cudaErrorInvalidValue;
  if (!n) return 0;
  const size_t nwin = (size_t)(253 + wbits - 1) / wbits;
  Call c;
  const u256* dk = c.in(k, n);
  int* dout = c.alloc<int>(n * nwin);
  if (c.ok()) k_signed_digits<<<blocks_for(n), TPB>>>(n, dk, wbits, dout);
  c.launched();
  c.out(out, dout, n * nwin);
  return (int)c.err;
}
// the same digits through msm_window<W> and the per-thread carry-in of the per-window MSM kernels; wbits in {8, 13, 15}
int spd_window_digits(size_t n, const u256* k, int wbits, int* out) {
  if (wbits != 8 && wbits != 13 && wbits != 15) return (int)cudaErrorInvalidValue;
  if (!n) return 0;
  const size_t nwin = (size_t)(253 + wbits - 1) / wbits;
  Call c;
  const u256* dk = c.in(k, n);
  int* dout = c.alloc<int>(n * nwin);
  if (c.ok()) {
    if (wbits == 8) k_window_digits<8><<<blocks_for(n), TPB>>>(n, dk, dout);
    else if (wbits == 13) k_window_digits<13><<<blocks_for(n), TPB>>>(n, dk, dout);
    else k_window_digits<15><<<blocks_for(n), TPB>>>(n, dk, dout);
  }
  c.launched();
  c.out(out, dout, n * nwin);
  return (int)c.err;
}

// ---------------------------------------------------------------------------------------------------- kernel hooks (the sp::dev wrappers)
const char* spd_last_error() { return g_last_error.c_str(); }
// ---- the memory-check mode of this library's own copy of the pool: the mirror of sp_debug_memcheck, sp_debug_memcheck_report and
// sp_debug_memcheck_scan.  counters: blocks filled, reused blocks refilled, context refills, guard bytes checked, violations
void spd_memcheck(int on) { memcheck_enable(on != 0); }
int spd_memcheck_report(unsigned long long counters[5], char* violations, size_t cap) {
  std::string first, last;
  const MemcheckStats s = memcheck_stats(&first, &last);
  const unsigned long long v[5] = {s.blocks_filled, s.blocks_refilled, s.context_refills, s.guard_bytes_checked, s.violations};
  memcpy(counters, v, sizeof v);
  const std::string text = first.empty() ? "" : first + "\n" + last;
  if (text.size() + 1 > cap) return SPD_REFUSED;
  memcpy(violations, text.c_str(), text.size() + 1);
  return 0;
}
unsigned long long spd_memcheck_scan() {
  try { return memcheck_scan(); } catch (const std::exception& e) { g_last_error = e.what(); return ~0ull; }
}
// The mode's mechanism on its own, through dev::pool_alloc: fresh and reused blocks read back as their fill class says, a block cached or live
// before the switch is not handed out under it, a byte written past the requested size is reported by the scan and at free, and switching the
// mode off restores the plain rounding.  0, or SPD_REFUSED with the failed check in spd_last_error(); `text` gets the messages of the two planted
// overruns.  The mode is left as it was found.
int spd_pool_selftest(char* text, size_t cap) {
  const bool was = memcheck_on();
  std::string notes;
  const int rc = guarded([&]() -> int {
    auto need = [](bool c, const char* what) { if (!c) throw std::runtime_error(std::string("pool self-test: ") + what); };
    auto cu = [](cudaError_t e) { if (e != cudaSuccess) throw std::runtime_error(std::string("pool self-test: ") + cudaGetErrorString(e)); };
    auto all = [&](const void* d, size_t n, uint8_t v) {
      std::vector<uint8_t> h(n);
      cu(cudaMemcpy(h.data(), d, n, cudaMemcpyDeviceToHost));
      for (uint8_t x : h) if (x != v) return false;
      return true;
    };
    auto stats = []() { return memcheck_stats(nullptr, nullptr); };
    auto last = []() { std::string l; memcheck_stats(nullptr, &l); return l; };
    const size_t B = 1000;   // far from a bucket edge: a 1 KiB block without the mode, 8 KiB with its 4 KiB guard
    memcheck_enable(false);
    void* before_cached = pool_alloc(B, FILL_FF);
    cu(cudaMemset(before_cached, 0x5A, B));
    pool_free(before_cached);
    void* before_live = pool_alloc(B, FILL_FF);
    cu(cudaMemset(before_live, 0x5A, B));
    memcheck_enable(true);
    const MemcheckStats s0 = stats();
    const size_t live0 = pool_live_bytes();
    uint8_t* a = (uint8_t*)pool_alloc(B, FILL_FF);
    need(pool_live_bytes() - live0 == 8192, "a 1000-byte block under the mode is not 8 KiB");
    need(stats().blocks_filled == s0.blocks_filled + 1 && stats().blocks_refilled == s0.blocks_refilled, "the block cached before the switch was handed out under it");
    need(all(a, B, 0xFF), "a fresh u256 block does not read back all 0xFF");
    need(all(a + B, 8192 - B, 0), "the guard band of a fresh block is not zero");
    pool_free(before_live);   // allocated before the switch: freed, not cached
    uint8_t* b = (uint8_t*)pool_alloc(B, FILL_FF);
    need(stats().blocks_refilled == s0.blocks_refilled, "a block allocated before the switch was reused under it");
    cu(cudaMemset(a, 0x11, B));
    pool_free(a);
    uint8_t* a2 = (uint8_t*)pool_alloc(B, FILL_FF);
    need(a2 == a && stats().blocks_refilled == s0.blocks_refilled + 1, "a freed block was not reused");
    need(all(a2, B, 0xFF), "a reused u256 block does not read back all 0xFF");
    uint8_t* raw = (uint8_t*)pool_alloc(B, FILL_ZERO);
    cu(cudaMemset(raw, 0x22, B));
    pool_free(raw);
    raw = (uint8_t*)pool_alloc(B, FILL_ZERO);
    need(stats().blocks_refilled == s0.blocks_refilled + 2, "a freed raw block was not reused");
    need(all(raw, B, 0), "a reused raw block does not read back zero");
    const unsigned long long v0 = stats().violations;
    cu(cudaMemset(a2 + B + 7, 1, 1));   // inside the guard, through the host API
    need(memcheck_scan() == 1, "the scan missed a byte written past the end");
    notes += last() + "\n";
    need(memcheck_scan() == 0, "the scan reported one overrun twice");
    cu(cudaMemset(raw + B, 1, 1));
    pool_free(raw);
    need(stats().violations == v0 + 2, "pool_free missed a byte written past the end");
    notes += last();
    pool_free(a2);
    pool_free(b);
    memcheck_enable(false);
    const size_t live1 = pool_live_bytes();
    void* c = pool_alloc(B, FILL_FF);
    const size_t plain = pool_live_bytes() - live1;
    pool_free(c);
    need(plain == 1024, "switching the mode off did not restore the plain rounding");
    return 0;
  });
  memcheck_enable(was);
  if (cap) { const size_t n = notes.size() < cap - 1 ? notes.size() : cap - 1; memcpy(text, notes.data(), n); text[n] = 0; }
  return rc;
}
unsigned long long spd_launch_count() { return launch_count(); }
void spd_prof_enable(int on) { prof_enable(on != 0); }
// "name:launches:total_ms:total_algorithmic_bytes;..." of the kernel families launched since spd_prof_enable(1), truncated to cap - 1 characters
size_t spd_prof_report(char* buf, size_t cap) {
  const std::string r = prof_report();
  if (cap) { const size_t n = r.size() < cap - 1 ? r.size() : cap - 1; memcpy(buf, r.data(), n); buf[n] = 0; }
  return r.size();
}

// A chain of batched sumcheck rounds: sc_eval on len entries, then nfold sc_fold_eval rounds with rs[0 .. nfold).  The tables live in nbuf
// buffers of len entries (`tables`, back to back); table t of instance i is buffer map[4 i + t] (-1: none), its folded C goes to buffer cbuf[i]
// when write_c[i].  A C shared by several instances is folded by one of them into a buffer of its own (cbuf[i] != map[4 i + 2]); after the round
// every instance that read it reads the folded copy, and the writer's next fold goes back to the first buffer, as the prover's ping-pong does.
// use_sig: every launch also publishes through a HostSig (seq = round + 1); host_out[round], flags[round] and dones[round] are the pinned results,
// the flag word and the device completion counter after the launch.  bound (use_sig, a fold to two-entry tables): the host_bound area of that
// fold.  On return: out[round] (ninst x 3 each), the buffers (tables_out) and the scratch's 64 ticket counters.
int spd_sc_chain(int kind, int ninst, size_t len, int nbuf, const u256* tables, const int* map, const int* cbuf, const int* write_c, int nfold,
                 const u256* rs, int use_sig, u256* out, u256* host_out, unsigned* flags, unsigned* dones, u256* bound, u256* tables_out,
                 unsigned* counters) {
  if (kind < SC_QUAD || kind > SC_CUBIC4 || ninst < 1 || ninst > 64 || nbuf < 1 || nfold < 0 || nfold > 40 || (nfold && (len >> nfold) < 2)) return (int)cudaErrorInvalidValue;
  return guarded([&] {
    KCall c;
    const int nt = kind == SC_QUAD ? 2 : kind == SC_CUBIC3 ? 3 : 4;
    u256* d = c.in(tables, (size_t)nbuf * len);
    void* scratch = c.zeros<char>(sc_scratch_bytes(ninst));
    u256* dout = c.zeros<u256>(3 * (size_t)ninst);
    HostSig sig;
    if (use_sig) { sig.host_out = c.host<u256>(3 * (size_t)ninst); sig.flag = c.host<unsigned>(1); sig.done = c.zeros<unsigned>(1); }
    u256* hb = bound ? c.host<u256>(2 * (size_t)nt * ninst) : nullptr;
    if (!c.ok()) return (int)c.err;
    std::vector<int> m(map, map + 4 * ninst), co(cbuf, cbuf + ninst);
    std::vector<ScInst> in(ninst);
    XRank xr;
    xr.world = 1;
    size_t cur = len;
    for (int k = 0; k <= nfold && c.ok(); k++) {
      for (int i = 0; i < ninst; i++) {
        for (int t = 0; t < 4; t++) in[i].t[t] = m[4 * i + t] >= 0 ? d + (size_t)m[4 * i + t] * len : nullptr;
        in[i].c_out = co[i] >= 0 ? d + (size_t)co[i] * len : nullptr;
        in[i].write_c = write_c[i];
      }
      sig.seq = (unsigned)k + 1;
      if (k == 0) {
        sc_eval((ScKind)kind, in.data(), ninst, cur, dout, scratch, c.s, sig, xr);
      } else {
        sc_fold_eval((ScKind)kind, in.data(), ninst, cur, rs[k - 1], dout, scratch, c.s, sig, xr, cur == 4 ? hb : nullptr);
        cur >>= 1;
      }
      c.sync();
      c.out(out + (size_t)k * 3 * ninst, dout, 3 * (size_t)ninst);
      if (use_sig && c.ok()) {
        memcpy(host_out + (size_t)k * 3 * ninst, sig.host_out, 3 * (size_t)ninst * sizeof(u256));
        flags[k] = *(volatile unsigned*)sig.flag;
        c.out(dones + k, sig.done, 1);
      }
      if (k > 0 && cur == 2 && hb && c.ok()) memcpy(bound, hb, 2 * (size_t)nt * ninst * sizeof(u256));
      if (k > 0 && nt > 2)
        for (int i = 0; i < ninst; i++) {
          const int old = m[4 * i + 2], nw = co[i];
          if (!write_c[i] || nw < 0 || nw == old) continue;
          for (int j = 0; j < ninst; j++) if (m[4 * j + 2] == old) m[4 * j + 2] = nw;
          co[i] = old;
        }
    }
    c.out(tables_out, d, (size_t)nbuf * len);
    c.out(counters, (unsigned*)scratch, 64);
    return (int)c.err;
  });
}

// The eq-factored chain of batched_prove on ninst instances of A * B * eq(tau, .): A_i, B_i of len = 2^n entries (a, b back to back), E0 =
// eq(tau[1..], .) (len/2 entries).  eq_suffix builds the levels E_1 .. E_{jG-1}; rounds 0 .. jG-1 run sc_eval_g / sc_fold_eval_g(rs[j-1]) on E_j
// (out[round][i] = q(0), q(inf), 0); round jG binds A and B with rs[jG-1] (fold_top) and runs sc_eval(SC_CUBIC3) on C = E_{jG-1}, instance 0
// folding the shared C into a ping-pong pair; rounds jG+1 .. n-1 run sc_fold_eval(SC_CUBIC3) down to two-entry tables.  use_sig as spd_sc_chain.
// On return a, b hold the bound tables (2 entries per instance, the first two of each table).
int spd_sc_g_chain(int ninst, size_t len, u256* a, u256* b, const u256* E0, int jG, const u256* rs, int use_sig, u256* out, u256* host_out,
                   unsigned* flags, unsigned* dones) {
  int n = 0;
  while (((size_t)1 << n) < len) n++;
  if (ninst < 1 || ninst > 64 || ((size_t)1 << n) != len || jG < 1 || jG >= n) return (int)cudaErrorInvalidValue;
  return guarded([&] {
    KCall c;
    u256* dA = c.in(a, (size_t)ninst * len);
    u256* dB = c.in(b, (size_t)ninst * len);
    const size_t n0 = len / 2;
    u256* dE0 = c.in(E0, n0);
    size_t nlev = 0;
    for (int k = 1; k < jG; k++) nlev += n0 >> k;
    u256* levels = c.alloc<u256>(nlev ? nlev : 1);
    const size_t chalf = (len >> jG) / 2;
    u256* cp[2] = {c.alloc<u256>(chalf), c.alloc<u256>(chalf)};
    void* scratch = c.zeros<char>(sc_scratch_bytes(ninst));
    u256* dout = c.zeros<u256>(3 * (size_t)ninst);
    HostSig sig;
    if (use_sig) { sig.host_out = c.host<u256>(3 * (size_t)ninst); sig.flag = c.host<unsigned>(1); sig.done = c.zeros<unsigned>(1); }
    if (!c.ok()) return (int)c.err;
    std::vector<u256*> E(jG);
    E[0] = dE0;
    for (size_t k = 1, off = 0; k < (size_t)jG; k++) { E[k] = levels + off; off += n0 >> k; }
    if (jG > 1) eq_suffix(levels, dE0, n0, jG - 1, c.s);
    std::vector<ScInst> in(ninst);
    std::vector<u256*> ab;
    for (int i = 0; i < ninst; i++) {
      in[i].t[0] = dA + (size_t)i * len; in[i].t[1] = dB + (size_t)i * len; in[i].t[2] = in[i].t[3] = nullptr;
      in[i].c_out = nullptr; in[i].write_c = 0;
      ab.push_back(in[i].t[0]); ab.push_back(in[i].t[1]);
    }
    XRank xr;
    xr.world = 1;
    size_t cur = len;
    for (int j = 0; j < n && c.ok(); j++) {
      sig.seq = (unsigned)j + 1;
      if (j == 0) sc_eval_g(in.data(), ninst, cur, E[0], dout, scratch, c.s, sig, xr);
      else if (j < jG) { sc_fold_eval_g(in.data(), ninst, cur, rs[j - 1], E[j], dout, scratch, c.s, sig, xr); cur >>= 1; }
      else if (j == jG) {
        fold_top(ab.data(), (int)ab.size(), cur, rs[j - 1], c.s);
        cur >>= 1;
        for (int i = 0; i < ninst; i++) { in[i].t[2] = E[jG - 1]; in[i].c_out = cp[0]; in[i].write_c = i == 0; }
        sc_eval(SC_CUBIC3, in.data(), ninst, cur, dout, scratch, c.s, sig, xr);
      } else {
        sc_fold_eval(SC_CUBIC3, in.data(), ninst, cur, rs[j - 1], dout, scratch, c.s, sig, xr);
        cur >>= 1;
        u256* folded = in[0].c_out;
        for (int i = 0; i < ninst; i++) { in[i].t[2] = folded; in[i].c_out = folded == cp[0] ? cp[1] : cp[0]; }
      }
      c.sync();
      c.out(out + (size_t)j * 3 * ninst, dout, 3 * (size_t)ninst);
      if (use_sig && c.ok()) {
        u256* h = host_out + (size_t)j * 3 * ninst;
        memcpy(h, sig.host_out, 3 * (size_t)ninst * sizeof(u256));
        // the eq-factored kernels publish q(0), q(inf) only: the third entry of their pinned slots is nobody's, and host_out says 0 there
        if (j < jG) for (int i = 0; i < ninst; i++) memset(&h[3 * (size_t)i + 2], 0, sizeof(u256));
        flags[j] = *(volatile unsigned*)sig.flag;
        c.out(dones + j, sig.done, 1);
      }
    }
    for (int i = 0; i < ninst; i++) {
      c.out(a + (size_t)i * len, dA + (size_t)i * len, 2);
      c.out(b + (size_t)i * len, dB + (size_t)i * len, 2);
    }
    return (int)c.err;
  });
}

// levels[k-1] (k = 1 .. K, n0 >> k entries each, back to back) from E0 (n0 entries)
int spd_eq_suffix(size_t n0, int K, const u256* E0, u256* levels) {
  return guarded([&] {
    KCall c;
    size_t total = 0;
    for (int k = 1; k <= K; k++) total += n0 >> k;
    const u256* dE = c.in(E0, n0);
    u256* dl = c.alloc<u256>(total ? total : 1);
    if (c.ok()) eq_suffix(dl, dE, n0, K, c.s);
    c.sync();
    c.out(levels, dl, total);
    return (int)c.err;
  });
}
// out (2^ell entries) = eq(r, .)
int spd_eq_evals(int ell, const u256* r, u256* out) {
  if (ell < 0 || ell > 30) return (int)cudaErrorInvalidValue;
  return guarded([&] {
    KCall c;
    const size_t n = (size_t)1 << ell;
    const u256* dr = c.in(r, ell ? (size_t)ell : 1);
    u256* dout = c.alloc<u256>(n);
    u256* small = c.alloc<u256>(eq_evals_scratch(ell));
    if (c.ok()) eq_evals(dout, dr, ell, small, c.s);
    c.sync();
    c.out(out, dout, n);
    return (int)c.err;
  });
}
// out (2n entries) = [(1 - r) E | r E] from E (n entries)
int spd_eq_extend_top(size_t n, const u256* E, const u256* r, u256* out) {
  return guarded([&] {
    KCall c;
    u256* d = c.alloc<u256>(2 * n);
    if (c.ok()) c.err = cudaMemcpy(d + n, E, n * sizeof(u256), cudaMemcpyHostToDevice);
    if (c.ok()) eq_extend_top(d, n, *r, c.s);
    c.sync();
    c.out(out, d, 2 * n);
    return (int)c.err;
  });
}
// out[k] = tables[k * n_each] for k < count; use_sig: host_out and *flag (seq 7) are the published copy
int spd_heads(int count, size_t n_each, const u256* tables, int use_sig, u256* out, u256* host_out, unsigned* flag) {
  return guarded([&] {
    KCall c;
    u256* d = c.in(tables, (size_t)count * n_each);
    u256* dout = c.zeros<u256>(64);
    HostSig sig;
    if (use_sig) { sig.host_out = c.host<u256>(64); sig.flag = c.host<unsigned>(1); sig.seq = 7; }
    if (!c.ok()) return (int)c.err;
    std::vector<const u256*> p(count);
    for (int k = 0; k < count; k++) p[k] = d + (size_t)k * n_each;
    heads(dout, p.data(), count, c.s, sig);
    c.sync();
    c.out(out, dout, (size_t)count);
    if (use_sig && c.ok()) { memcpy(host_out, sig.host_out, (size_t)count * sizeof(u256)); *flag = *(volatile unsigned*)sig.flag; }
    return (int)c.err;
  });
}
// fold_top of ntables tables of len entries (back to back, in place: the first len/2 entries of each are the result)
int spd_fold_top(int ntables, size_t len, u256* tables, const u256* r) {
  return guarded([&] {
    KCall c;
    u256* d = c.in(tables, (size_t)ntables * len);
    if (!c.ok()) return (int)c.err;
    std::vector<u256*> p(ntables);
    for (int k = 0; k < ntables; k++) p[k] = d + (size_t)k * len;
    fold_top(p.data(), ntables, len, *r, c.s);
    c.sync();
    c.out(tables, d, (size_t)ntables * len);
    return (int)c.err;
  });
}

// ---- batch verifier
// out[k] = sum over segment k of scalars[i] * pts[i] (msm_var_segmented); scalars canonical, seg_start: K+1 entries
int spd_msm_var_segmented(size_t K, size_t n, const ge* pts, const u256* scalars, const uint32_t* seg_start, ge* out) {
  return guarded([&] {
    KCall c;
    const ge* dp = c.in(pts, n ? n : 1);
    const u256* ds = c.in(scalars, n ? n : 1);
    const uint32_t* dseg = c.in(seg_start, K + 1);
    ge* dtmp = c.alloc<ge>(n ? n : 1);
    ge* dout = c.alloc<ge>(K ? K : 1);
    if (c.ok()) msm_var_segmented(dout, dp, ds, dseg, K, n, dtmp, c.s);
    c.sync();
    c.out(out, dout, K);
    return (int)c.err;
  });
}
// dotlog_fold of 2m points given as extended points: out[i] = pts[i] + k * pts[i + m] (k canonical).  in_fmt FOLD_NIELS converts the points to
// affine niels first (points_to_niels); a niels output comes back through niels_to_ge
int spd_dotlog_fold(size_t m, int in_fmt, int out_fmt, const ge* pts, const u256* k, ge* out) {
  return guarded([&] {
    KCall c;
    const ge* dp = c.in(pts, 2 * m);
    ge_niels* dn = c.alloc<ge_niels>(2 * m);
    ge_niels* don = c.alloc<ge_niels>(m);
    ge* dout = c.alloc<ge>(m);
    if (c.ok()) {
      const void* in = dp;
      if (in_fmt == FOLD_NIELS) { points_to_niels(dn, dp, 2 * m, c.s); in = dn; }
      if (out_fmt == FOLD_NIELS) {
        dotlog_fold(don, out_fmt, in, in_fmt, m, *k, c.s);
        niels_to_ge(dout, don, m, c.s);
      } else {
        dotlog_fold(dout, out_fmt, in, in_fmt, m, *k, c.s);
      }
    }
    c.sync();
    c.out(out, dout, m);
    return (int)c.err;
  });
}
// the launch plan msm_var runs for n points (pip_plan, c_override = 0: the default window width):
// out = {c, nwin, nb, tile, ntiles, G, S, max_items, pip_scratch_bytes}
int spd_pip_plan(size_t n, int c_override, uint64_t out[9]) {
  return guarded([&] {
    const PipPlan p = pip_plan(n, c_override);
    const uint64_t v[9] = {(uint64_t)p.c, (uint64_t)p.nwin, p.nb, p.tile, p.ntiles, (uint64_t)p.G, p.S, p.max_items, pip_scratch_bytes(p)};
    memcpy(out, v, sizeof(v));
    return 0;
  });
}
// ipa_srow over `nitems` rows packed back to back in rows[0 .. total) (in, out): item i writes or adds 2^lg_n[i] entries at row_off[i];
// u_sq: 32 scalars per item
int spd_ipa_srow(size_t nitems, const uint32_t* lg_n, const uint32_t* add, const u256* allinv, const u256* scale, const u256* u_sq, const uint64_t* row_off,
                 size_t total, u256* rows) {
  return guarded([&] {
    KCall c;
    u256* drows = c.in(rows, total);
    std::vector<IpaSRow> items(nitems);
    uint32_t max_lg = 0;
    for (size_t i = 0; i < nitems; i++) {
      memset(&items[i], 0, sizeof(IpaSRow));
      items[i].row = drows + row_off[i];
      items[i].lg_n = lg_n[i]; items[i].add = add[i]; items[i].allinv = allinv[i]; items[i].scale = scale[i];
      for (int j = 0; j < 32; j++) items[i].u_sq[j] = u_sq[32 * i + j];
      if (lg_n[i] > max_lg) max_lg = lg_n[i];
    }
    const IpaSRow* dit = c.in(items.data(), nitems ? nitems : 1);
    if (c.ok()) ipa_srow(dit, nitems, max_lg, c.s);
    c.sync();
    c.out(rows, drows, total);
    return (int)c.err;
  });
}

// the deferred checker of batch verification and its final pass (verifier.cpp deferred_check) on hand-made equations over a generator set of
// `nbases` points derived from `label`.  Proof i owns equations [eq_start[i], eq_start[i+1]); equation e owns terms [term_start[e],
// term_start[e+1]); term t: side[t] (0 lhs, 1 rhs), gen[t] (>= 0: that generator; < 0: the point pts[32 t .. 32 t + 32)), k[t] (Montgomery).
// ok[i] = 1 when the final pass accepts proof i.
int spd_deferred_check(size_t nproofs, const uint32_t* eq_start, const uint32_t* term_start, const int32_t* side, const int64_t* gen, const uint8_t* pts,
                       const u256* k, const uint8_t* label, size_t label_len, size_t nbases, const uint8_t* seed32, int* ok) {
  return guarded([&] {
    sp::Ctx ctx(0);
    sp::GenSet gs(&ctx, std::string((const char*)label, label_len), nbases, {});
    std::vector<std::vector<DeferredEq>> proofs(nproofs);
    for (size_t i = 0; i < nproofs; i++)
      for (uint32_t e = eq_start[i]; e < eq_start[i + 1]; e++) {
        DeferredEq eq;
        for (uint32_t t = term_start[e]; t < term_start[e + 1]; t++) {
          DeferredTerm x;
          x.k = Fq(k[t]); x.gen = (long)gen[t];
          memcpy(x.pt.b, pts + 32 * (size_t)t, 32);
          (side[t] ? eq.rhs : eq.lhs).push_back(x);
        }
        proofs[i].push_back(eq);
      }
    const std::vector<bool> r = deferred_check(ctx, gs, proofs, seed32);
    for (size_t i = 0; i < nproofs; i++) ok[i] = r[i] ? 1 : 0;
    return 0;
  });
}

// ---- generator tables
// Checks the affine-niels table in device memory d_table (k_niels_check): nslots generators in the per-window layout of wbits = 8, 13 or 15, or in
// the row layout (wbits = 0); slot j holds the multiples of d_G[bases[j]] (bases: nslots host entries, or null for slot j = generator j).  out: the
// 24-word report of niels_check.  d_table and d_G are only read.
int spd_niels_table_check(const void* d_table, size_t nslots, int wbits, const void* d_G, const int64_t* bases, uint64_t* out) {
  if ((wbits != 0 && wbits != 8 && wbits != 13 && wbits != 15) || nslots < 1) return (int)cudaErrorInvalidValue;
  return guarded([&] {
    KCall c;
    const int64_t* db = bases ? c.in(bases, nslots) : nullptr;
    niels_check(c, (const ge_niels*)d_table, nslots, wbits, (const ge*)d_G, db, out);
    return (int)c.err;
  });
}

// Builds one generator set through GenSet's production constructors (nbases generators of the SHAKE256 stream of `label`, or with enc non-null the
// nbases caller encodings) with the host copies of host_bases, adds those of extra_bases afterwards as a view does, and checks every entry the set
// holds: the per-window table at the width the set chose, the row table when it built one, and the host copies of every requested base below
// nbases (radix 2^51, taken back to 256-bit values) in the 8-bit layout against their generators.  out: three 24-word reports (niels_check) for the
// per-window table, the row table (all zero without one) and the host copies, whose slot j is base host_checked[j] (n_host + n_extra entries of
// room).  info: the window width, 1 when a row table was built, the free and total device bytes just before the build, the set's device bytes and
// the number of host copies checked.  G_enc: the nbases generators' encodings (k_compress).  ms: build and check wall times.  The set is freed and
// this library's cached blocks released before the call returns.
int spd_gen_set_check(const uint8_t* label, size_t label_len, size_t nbases, const uint8_t* enc, const int64_t* host_bases, size_t n_host,
                      const int64_t* extra_bases, size_t n_extra, uint8_t* G_enc, int64_t* info, int64_t* host_checked, uint64_t* out, double* ms) {
  if (nbases < 1) return (int)cudaErrorInvalidValue;
  return guarded([&] {
    ReleaseCached rel;
    pool_release_cached();
    Ctx ctx(0);
    const std::vector<size_t> hb(host_bases, host_bases + n_host), xb(extra_bases, extra_bases + n_extra);
    size_t free0 = 0, total0 = 0;
    mem_info(&free0, &total0);
    const auto t0 = std::chrono::steady_clock::now();
    std::unique_ptr<GenSet> gs = make_set(ctx, label, label_len, nbases, enc, hb);
    gs->add_host_tables(xb);
    ctx.sync();
    const auto t1 = std::chrono::steady_clock::now();
    std::vector<size_t> want;
    for (const std::vector<size_t>* v : {&hb, &xb})
      for (size_t b : *v)
        if (b < nbases && std::find(want.begin(), want.end(), b) == want.end()) want.push_back(b);
    for (size_t b : want) if (!gs->has_tab(b)) throw std::runtime_error("the set holds no host copy of base " + std::to_string(b));
    {
      KCall c;
      niels_check(c, gs->table.p, nbases, gs->wbits, gs->G.p, nullptr, out);
      if (gs->rows()) niels_check(c, gs->rows(), nbases, 0, gs->G.p, nullptr, out + CHECK_OUT);
      else memset(out + CHECK_OUT, 0, CHECK_OUT * sizeof(uint64_t));
      memset(out + 2 * CHECK_OUT, 0, CHECK_OUT * sizeof(uint64_t));
      if (!want.empty()) {
        const size_t per = 32 * 128;
        std::vector<ge_niels> h(want.size() * per);
        for (size_t i = 0; i < want.size(); i++) {
          const HostBaseTable& tb = gs->tab(want[i]);
          if (tb.e.size() != per) throw std::runtime_error("host copy of base " + std::to_string(want[i]) + " has " + std::to_string(tb.e.size()) + " entries");
          for (size_t e = 0; e < per; e++) h[i * per + e] = ge_niels{fe51_value(tb.e[e].ypx), fe51_value(tb.e[e].ymx), fe51_value(tb.e[e].t2d)};
        }
        const std::vector<int64_t> wb(want.begin(), want.end());
        const ge_niels* dh = c.in(h.data(), h.size());
        const int64_t* dwb = c.in(wb.data(), wb.size());
        niels_check(c, dh, want.size(), 8, gs->G.p, dwb, out + 2 * CHECK_OUT);
      }
      if (!c.ok()) return (int)c.err;
    }
    const auto t2 = std::chrono::steady_clock::now();
    DevBuf<uint8_t> comp(32 * nbases);
    compress_batch(comp.p, gs->G.p, nbases, ctx.stream);
    d2h(G_enc, comp.p, 32 * nbases, ctx.stream);
    ctx.sync();
    const int64_t v[6] = {gs->wbits, gs->rows() ? 1 : 0, (int64_t)free0, (int64_t)total0, (int64_t)gs->device_bytes(), (int64_t)want.size()};
    memcpy(info, v, sizeof v);
    for (size_t i = 0; i < want.size(); i++) host_checked[i] = (int64_t)want[i];
    ms[0] = std::chrono::duration<double, std::milli>(t1 - t0).count();
    ms[1] = std::chrono::duration<double, std::milli>(t2 - t1).count();
    return 0;
  });
}

// Builds the set of spd_gen_set_check by label (no host copies) and copies its per-window table (row = 0) or its row table (row = 1) into the
// caller's device buffer d_table (room for cap entries of 96 bytes), and its nbases generators into d_G (128 bytes each), so that a check can run
// on a copy the caller alters; the set's own tables are only read.  info: the window width and the entries copied.  SPD_REFUSED when the set has
// no row table or the table needs more than cap entries.
int spd_gen_table_copy(const uint8_t* label, size_t label_len, size_t nbases, int row, void* d_table, size_t cap, void* d_G, int64_t* info) {
  if (nbases < 1) return (int)cudaErrorInvalidValue;
  return guarded([&] {
    ReleaseCached rel;
    Ctx ctx(0);
    std::unique_ptr<GenSet> gs = make_set(ctx, label, label_len, nbases, nullptr, {});
    const DevBuf<ge_niels>& t = row ? gs->row_table : gs->table;
    if (!t.n) throw std::runtime_error("the set has no row table");
    if (t.n > cap) throw std::runtime_error("the table has " + std::to_string(t.n) + " entries, the buffer room for " + std::to_string(cap));
    d2d(d_table, t.p, t.n * sizeof(ge_niels), ctx.stream);
    d2d(d_G, gs->G.p, nbases * sizeof(ge), ctx.stream);
    ctx.sync();
    info[0] = gs->wbits;
    info[1] = (int64_t)t.n;
    return 0;
  });
}

// ---- SPARK layer and dense helpers
// out = ts * r^2 + val * r + addr - g over n entries; addr / ts null: the index / zero; rg = [r, g]
int spd_spark_hash(size_t n, const u256* addr, const u256* val, const u256* ts, int ts_plus_one, const u256* rg, u256* out) {
  return guarded([&] {
    KCall c;
    const u256* da = addr ? c.in(addr, n) : nullptr;
    const u256* dv = c.in(val, n);
    const u256* dt = ts ? c.in(ts, n) : nullptr;
    const u256* drg = c.in(rg, 2);
    u256* dout = c.alloc<u256>(n);
    if (c.ok()) spark_hash(dout, n, da, dv, dt, ts_plus_one, drg, c.s);
    c.sync();
    c.out(out, dout, n);
    return (int)c.err;
  });
}
// the same on rank `rank` of `world` (n / world local entries, global index j * world + rank) from the unsharded arrays
int spd_spark_hash_cyclic(size_t n, int rank, int world, const u256* addr, const u256* val, const u256* ts, int ts_plus_one, const u256* rg, u256* out) {
  if (world < 1 || rank < 0 || rank >= world || n % world) return (int)cudaErrorInvalidValue;
  return guarded([&] {
    KCall c;
    const u256* da = addr ? c.in(addr, n) : nullptr;
    const u256* dv = c.in(val, n);
    const u256* dt = ts ? c.in(ts, n) : nullptr;
    const u256* drg = c.in(rg, 2);
    u256* dout = c.alloc<u256>(n / world);
    if (c.ok()) spark_hash_cyclic(dout, n / world, rank, world, da, dv, dt, ts_plus_one, drg, c.s);
    c.sync();
    c.out(out, dout, n / world);
    return (int)c.err;
  });
}
// out[k] = a[k] o b[k] for count circuits of n entries (back to back)
int spd_hadamard_many(int count, size_t n, const u256* a, const u256* b, u256* out) {
  return guarded([&] {
    KCall c;
    const u256* da = c.in(a, (size_t)count * n);
    const u256* db = c.in(b, (size_t)count * n);
    u256* dout = c.alloc<u256>((size_t)count * n);
    if (!c.ok()) return (int)c.err;
    std::vector<u256*> po(count);
    std::vector<const u256*> pa(count), pb(count);
    for (int k = 0; k < count; k++) { po[k] = dout + (size_t)k * n; pa[k] = da + (size_t)k * n; pb[k] = db + (size_t)k * n; }
    hadamard_many(po.data(), pa.data(), pb.data(), count, n, c.s);
    c.sync();
    c.out(out, dout, (size_t)count * n);
    return (int)c.err;
  });
}
// out[i] = mem[idx[i]]
int spd_gather(size_t cells, const u256* mem, size_t n, const uint32_t* idx, u256* out) {
  return guarded([&] {
    KCall c;
    const u256* dm = c.in(mem, cells);
    const uint32_t* di = c.in(idx, n);
    u256* dout = c.alloc<u256>(n);
    if (c.ok()) gather(dout, dm, di, n, c.s);
    c.sync();
    c.out(out, dout, n);
    return (int)c.err;
  });
}
// *out = sum a b (c null: dot) or sum a b c (dot3)
int spd_dot3(size_t n, const u256* a, const u256* b, const u256* cc, u256* out) {
  return guarded([&] {
    KCall c;
    const u256* da = c.in(a, n);
    const u256* db = c.in(b, n);
    const u256* dc = cc ? c.in(cc, n) : nullptr;
    void* scratch = c.zeros<char>(red_scratch_bytes());
    u256* dout = c.zeros<u256>(1);
    if (c.ok()) { if (dc) dot3(dout, da, db, dc, n, scratch, c.s); else dot(dout, da, db, n, scratch, c.s); }
    c.sync();
    c.out(out, dout, 1);
    return (int)c.err;
  });
}
// out[k] = <a[k], b> for count tables of n entries (back to back)
int spd_dot_many(int count, size_t n, const u256* a, const u256* b, u256* out) {
  return guarded([&] {
    KCall c;
    const u256* da = c.in(a, (size_t)count * n);
    const u256* db = c.in(b, n);
    void* scratch = c.zeros<char>(red_scratch_bytes());
    u256* dout = c.zeros<u256>(count > 0 ? (size_t)count : 1);
    if (!c.ok()) return (int)c.err;
    std::vector<const u256*> pa(count);
    for (int k = 0; k < count; k++) pa[k] = da + (size_t)k * n;
    dot_many(dout, pa.data(), count, db, n, scratch, c.s);
    c.sync();
    c.out(out, dout, (size_t)count);
    return (int)c.err;
  });
}
// out = ra A + rb B + rc C, rabc = [ra, rb, rc]
int spd_lincomb3(size_t n, const u256* A, const u256* B, const u256* Cc, const u256* rabc, u256* out) {
  return guarded([&] {
    KCall c;
    const u256* da = c.in(A, n);
    const u256* db = c.in(B, n);
    const u256* dc = c.in(Cc, n);
    const u256* dr = c.in(rabc, 3);
    u256* dout = c.alloc<u256>(n);
    if (c.ok()) lincomb3(dout, da, db, dc, dr, n, c.s);
    c.sync();
    c.out(out, dout, n);
    return (int)c.err;
  });
}
// out[i] = sum_j L[j] Z[j R_size + i]
int spd_bound_rows(size_t L_size, size_t R_size, const u256* Z, const u256* L, u256* out) {
  return guarded([&] {
    KCall c;
    const u256* dz = c.in(Z, L_size * R_size);
    const u256* dl = c.in(L, L_size);
    u256* scratch = c.alloc<u256>(64 * R_size);
    u256* dout = c.alloc<u256>(R_size);
    if (c.ok()) bound_rows(dout, dz, dl, L_size, R_size, scratch, c.s);
    c.sync();
    c.out(out, dout, R_size);
    return (int)c.err;
  });
}
// Montgomery limbs -> canonical little-endian integers
int spd_to_canonical(size_t n, const u256* in, u256* out) {
  return guarded([&] {
    KCall c;
    const u256* di = c.in(in, n);
    u256* dout = c.alloc<u256>(n);
    if (c.ok()) to_canonical(dout, di, n, c.s);
    c.sync();
    c.out(out, dout, n);
    return (int)c.err;
  });
}

// ---- sparse products on caller CSR / COO arrays
int spd_spmv(size_t nrows, size_t nnz, const uint32_t* ptr, const uint32_t* idx, const u256* val, size_t ncols, const u256* x, u256* out) {
  return guarded([&] {
    KCall c;
    const uint32_t* dp = c.in(ptr, nrows + 1);
    const uint32_t* di = c.in(idx, nnz);
    const u256* dv = c.in(val, nnz);
    const u256* dx = c.in(x, ncols);
    u256* dout = c.alloc<u256>(nrows);
    if (c.ok()) spmv(dout, nrows, dp, di, dv, dx, c.s);
    c.sync();
    c.out(out, dout, nrows);
    return (int)c.err;
  });
}
// rows j * world + rank of the CSR (nrows / world of them)
int spd_spmv_cyclic(size_t nrows, int rank, int world, size_t nnz, const uint32_t* ptr, const uint32_t* idx, const u256* val, size_t ncols, const u256* x,
                    u256* out) {
  if (world < 1 || rank < 0 || rank >= world || nrows % world) return (int)cudaErrorInvalidValue;
  return guarded([&] {
    KCall c;
    const uint32_t* dp = c.in(ptr, nrows + 1);
    const uint32_t* di = c.in(idx, nnz);
    const u256* dv = c.in(val, nnz);
    const u256* dx = c.in(x, ncols);
    u256* dout = c.alloc<u256>(nrows / world);
    if (c.ok()) spmv_cyclic(dout, nrows / world, rank, world, dp, di, dv, dx, c.s);
    c.sync();
    c.out(out, dout, nrows / world);
    return (int)c.err;
  });
}
// *out = sum_k trx[row[k]] try[col[k]] val[k]
int spd_sparse_eval3(size_t nnz, const uint32_t* row, const uint32_t* col, const u256* val, size_t nrx, const u256* trx, size_t nry, const u256* try_,
                     u256* out) {
  return guarded([&] {
    KCall c;
    const uint32_t* dr = c.in(row, nnz);
    const uint32_t* dc = c.in(col, nnz);
    const u256* dv = c.in(val, nnz);
    const u256* dx = c.in(trx, nrx);
    const u256* dy = c.in(try_, nry);
    void* scratch = c.zeros<char>(red_scratch_bytes());
    u256* dout = c.zeros<u256>(1);
    if (c.ok()) sparse_eval3(dout, dr, dc, dv, nnz, dx, dy, scratch, c.s);
    c.sync();
    c.out(out, dout, 1);
    return (int)c.err;
  });
}

// ---- sharded table producers, on one GPU
int spd_scale(size_t n, u256* inout, const u256* cst) {
  return guarded([&] {
    KCall c;
    u256* d = c.in(inout, n);
    if (c.ok()) scale(d, *cst, n, c.s);
    c.sync();
    c.out(inout, d, n);
    return (int)c.err;
  });
}
// out[j] = full[j * world + rank], j < n / world
int spd_take_cyclic(size_t n, const u256* full, int rank, int world, u256* out) {
  if (world < 1 || rank < 0 || rank >= world || n % world) return (int)cudaErrorInvalidValue;
  return guarded([&] {
    KCall c;
    const u256* df = c.in(full, n);
    u256* dout = c.alloc<u256>(n / world);
    if (c.ok()) take_cyclic(dout, df, n / world, rank, world, c.s);
    c.sync();
    c.out(out, dout, n / world);
    return (int)c.err;
  });
}
}
