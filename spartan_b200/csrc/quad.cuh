// spartan_b200 — window extraction of the fixed-base MSMs and the quad-lane point arithmetic, shared by the kernels (kernels.cu) and the
// device test harness (devtest.cu), so that the harness runs exactly the code the MSM kernels run.
#pragma once
#include "kcommon.cuh"

namespace sp {
namespace dev {

template <int WBITS>
__device__ __forceinline__ uint32_t msm_window(const u256& k, int w) {
  const int b = w * WBITS, limb = b >> 5, sh = b & 31;
  uint32_t v = k.v[limb] >> sh;
  if (sh + WBITS > 32 && limb + 1 < 8) v |= k.v[limb + 1] << (32 - sh);
  return v & ((1u << WBITS) - 1u);
}

// ---- quad-lane point arithmetic for latency-bound reductions.
// A lone warp gains nothing from the four independent field products of a point addition (9 products
// back to back), so a reduction tree of point additions costs 9 product latencies per level.  Here FOUR LANES share one point — lane c of a quad holds coordinate
// c (0: X, 1: Y, 2: Z, 3: T) — and run the products of add-2008-hwcd-3 side by side: three product latencies per addition (A | B | Z1 Z2 | T1 T2, then
// 2d on the T lane, then X3 | Y3 | Z3 | T3) and a few 8-word shuffles instead of nine products in a row.  Same formulas, same field values as
// ge_add / ge_madd; every lane of the warp must take part in every call (full-mask shuffles).
__device__ __forceinline__ u256 shfl_idx_256(const u256& x, int src) {
  u256 r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = __shfl_sync(0xffffffffu, x.v[i], src);
  return r;
}
__device__ __forceinline__ u256 shfl_xor_256(const u256& x, int m) {
  u256 r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = __shfl_xor_sync(0xffffffffu, x.v[i], m);
  return r;
}
__device__ __forceinline__ u256 quad_identity(int c) { return (c == 1 || c == 2) ? fp_one() : fp_zero(); }
// lane-dependent choice without a branch: the sums / differences below are computed by every lane and selected, because a divergent
// `if (c == k)` makes the warp run each arm one after the other
__device__ __forceinline__ u256 sel256(bool p, const u256& a, const u256& b) {
  u256 r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = p ? a.v[i] : b.v[i];
  return r;
}
// coordinates -> operands of the first products: lane 0: Y - X, lane 1: Y + X, lane 2: Z, lane 3: T
__device__ __forceinline__ u256 quad_prep(const u256& v, int c) {
  const u256 o = shfl_xor_256(v, 1);
  const u256 d = fp_sub(o, v), sm = fp_add(v, o);          // lane 0: Y - X = o - v; lane 1: Y + X
  return c >= 2 ? v : sel256(c == 0, d, sm);
}
// m = (A, B, D, C) on lanes 0..3  ->  the sum's coordinates (X3, Y3, Z3, T3) on lanes 0..3
static __device__ __noinline__ u256 quad_finish(u256 m, int c, int lane) {
  const u256 o = shfl_xor_256(m, 1);                       // lane 0 <- B, lane 1 <- A, lane 2 <- C, lane 3 <- D
  // lane 0: E = B - A = o - m, lane 1: H = B + A, lane 2: F = D - C = m - o, lane 3: G = D + C
  const u256 df = fp_sub(sel256(c == 0, o, m), sel256(c == 0, m, o)), sm = fp_add(m, o);
  const u256 w = sel256((c & 1) != 0, sm, df);
  const int base = lane & ~3;
  const u256 x = shfl_idx_256(w, base + ((0x2031 >> (4 * c)) & 3));   // lane 0 (E) <- H, lane 1 (H) <- G, lane 2 (F) <- E, lane 3 (G) <- F
  const u256 r = fp_mul(w, x);                             // lane 0: T3 = E H, lane 1: Y3 = H G, lane 2: X3 = F E, lane 3: Z3 = G F
  return shfl_idx_256(r, base + ((0x0312 >> (4 * c)) & 3));            // lane 0 <- X3 (lane 2), lane 1: Y3, lane 2 <- Z3 (lane 3), lane 3 <- T3 (lane 0)
}
static __device__ __noinline__ u256 quad_add(u256 p, u256 q, int c, int lane) {   // P + Q (ge_add)
  const u256 up = quad_prep(p, c), uq = quad_prep(q, c);
  const u256 m = fp_mul(up, uq);                           // A | B | Z1 Z2 | T1 T2
  const u256 m2 = fp_add(m, m);                            // D on lane 2
  const u256 mc = fp_mul(m, fp_2D());                      // C on lane 3 (every lane multiplies: one more product latency either way, no divergence)
  return quad_finish(c == 3 ? mc : (c == 2 ? m2 : m), c, lane);
}
// P + q for an affine niels operand given per lane as (y - x, y + x, -, 2d x y) of +/-q (ge_madd)
__device__ __forceinline__ u256 quad_madd(const u256& p, const u256& nq, int c, int lane) {
  const u256 up = quad_prep(p, c);
  const u256 m = fp_mul(up, nq);                           // A | B | (unused) | C
  const u256 m2 = fp_add(up, up);                          // D = 2 Z1 on lane 2
  return quad_finish(c == 2 ? m2 : m, c, lane);
}
// sum over the 8 quads of a warp -> quad 0
__device__ __forceinline__ u256 quad_warp_sum(u256 P, int c, int lane) {
#pragma unroll 1
  for (int d = 16; d >= 4; d >>= 1) P = quad_add(P, shfl_down_256(P, d), c, lane);
  return P;
}
// doubling: dbl-2008-hwcd (ge_dbl) on a quad, lane c holding coordinate c: one round of squarings (X^2 | Y^2 | Z^2 | (X+Y)^2), one of products
static __device__ __noinline__ u256 quad_dbl(u256 p, int c, int lane) {
  const int base = lane & ~3;
  const u256 x = shfl_idx_256(p, base), y = shfl_idx_256(p, base + 1);
  const u256 m = fp_sqr(sel256(c == 3, fp_add(x, y), p));
  const u256 A = shfl_idx_256(m, base), B = shfl_idx_256(m, base + 1), Z2 = shfl_idx_256(m, base + 2), S = shfl_idx_256(m, base + 3);
  const u256 C = fp_add(Z2, Z2), D = fp_neg(A);
  const u256 E = fp_sub(fp_sub(S, A), B), G = fp_add(D, B), F = fp_sub(G, C), H = fp_sub(D, B);
  // lane 0: X3 = E F, lane 1: Y3 = G H, lane 2: Z3 = F G, lane 3: T3 = E H
  return fp_mul(sel256(c == 1, G, sel256(c == 2, F, E)), sel256(c == 0, F, sel256(c == 2, G, H)));
}

}  // namespace dev
}  // namespace sp
