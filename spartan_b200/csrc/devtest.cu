// spartan_b200 — device test hooks, the GPU counterpart of hosttest.cpp.  Built with the kernels' nvcc flags, so the field and curve arithmetic
// here is the code the kernels run on the device (inline-PTX carry chains, generated multiplications, quad-lane point operations), not the portable
// formulation the CPU tests check.  Not linked into libspartan_b200.so.
//
// Every entry point takes host arrays of n elements, copies them to the device, runs one elementwise kernel (one thread per element, or one quad of
// lanes per point for the quad-lane operations), copies the results back and returns the CUDA status (0 = success).
//   u256:     8 little-endian 32-bit limbs.  F_q operands are Montgomery limbs, passed and returned unchanged; F_p operands may be any value < 2^256.
//   ge:       the four coordinates X, Y, Z, T as u256 (any representatives, not necessarily reduced or normalised).
//   ge_niels: y + x, y - x, 2dxy as u256.
#include <cuda_runtime.h>
#include <vector>
#include "kcommon.cuh"
#include "quad.cuh"

using namespace sp;
using namespace sp::dev;

namespace {

constexpr int TPB = 128;
unsigned blocks_for(size_t threads) { return (unsigned)((threads + TPB - 1) / TPB); }

// device copies of one call's arrays, freed on return; the first failing CUDA call is kept and later steps are skipped
struct Call {
  std::vector<void*> bufs;
  cudaError_t err = cudaSuccess;
  template <class T> T* alloc(size_t n) {
    void* d = nullptr;
    if (err == cudaSuccess) err = cudaMalloc(&d, n * sizeof(T));
    bufs.push_back(d);
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
  ~Call() { for (void* p : bufs) if (p) cudaFree(p); }
};

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
}
