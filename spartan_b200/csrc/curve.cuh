// spartan_b200 — edwards25519 / ristretto255 group arithmetic for sm_90a (and the host, same source).
//
// Replaces what the reference reaches through curve25519-dalek: `GroupElement = RistrettoPoint`
// (/root/reference/src/group.rs:6), point add/sub/scalar-mul (group.rs:28-46), `compress`/`decompress`
// (e.g. dense_mlpoly.rs:173, sumcheck.rs:705) and `from_uniform_bytes` (commitments.rs:25).
// Encodings follow RFC 9496; any internal representative of a ristretto class encodes to the same 32 bytes,
// so results are bit-identical to dalek's regardless of addition order.
#pragma once
#include "field.cuh"

namespace sp {

struct ge {  // extended twisted-Edwards coordinates, a = -1: x = X/Z, y = Y/Z, T = XY/Z   (128 bytes)
  u256 X, Y, Z, T;
};
struct ge_niels {  // affine precomputed form for mixed addition: (y+x, y-x, 2d*x*y)              (96 bytes)
  u256 ypx, ymx, t2d;
};

SP_HD ge ge_identity() {
  ge r;
  r.X = fp_zero(); r.Y = fp_one(); r.Z = fp_one(); r.T = fp_zero();
  return r;
}
SP_HD ge_niels niels_identity() {
  ge_niels r;
  r.ypx = fp_one(); r.ymx = fp_one(); r.t2d = fp_zero();
  return r;
}

// add-2008-hwcd-3 (8M + 1 constant mul)
SP_HD ge ge_add(const ge& p, const ge& q) {
  u256 A = fp_mul(fp_sub(p.Y, p.X), fp_sub(q.Y, q.X));
  u256 B = fp_mul(fp_add(p.Y, p.X), fp_add(q.Y, q.X));
  u256 C = fp_mul(fp_mul(p.T, q.T), fp_2D());
  u256 D = fp_mul(p.Z, q.Z);
  D = fp_add(D, D);
  u256 E = fp_sub(B, A), F = fp_sub(D, C), G = fp_add(D, C), H = fp_add(B, A);
  ge r;
  r.X = fp_mul(E, F); r.Y = fp_mul(G, H); r.T = fp_mul(E, H); r.Z = fp_mul(F, G);
  return r;
}
// mixed addition with an affine niels point (7M); `neg` adds -q instead
SP_HD ge ge_madd(const ge& p, const ge_niels& q, bool neg) {
  u256 qa = neg ? q.ypx : q.ymx;  // (y-x) of +/-q
  u256 qb = neg ? q.ymx : q.ypx;
  u256 A = fp_mul(fp_sub(p.Y, p.X), qa);
  u256 B = fp_mul(fp_add(p.Y, p.X), qb);
  u256 C = fp_mul(p.T, q.t2d);
  if (neg) C = fp_neg(C);
  u256 D = fp_add(p.Z, p.Z);
  u256 E = fp_sub(B, A), F = fp_sub(D, C), G = fp_add(D, C), H = fp_add(B, A);
  ge r;
  r.X = fp_mul(E, F); r.Y = fp_mul(G, H); r.T = fp_mul(E, H); r.Z = fp_mul(F, G);
  return r;
}
// dbl-2008-hwcd (4M + 4S)
SP_HD ge ge_dbl(const ge& p) {
  u256 A = fp_sqr(p.X), B = fp_sqr(p.Y);
  u256 C = fp_sqr(p.Z);
  C = fp_add(C, C);
  u256 D = fp_neg(A);
  u256 t = fp_add(p.X, p.Y);
  u256 E = fp_sub(fp_sub(fp_sqr(t), A), B);
  u256 G = fp_add(D, B), F = fp_sub(G, C), H = fp_sub(D, B);
  ge r;
  r.X = fp_mul(E, F); r.Y = fp_mul(G, H); r.T = fp_mul(E, H); r.Z = fp_mul(F, G);
  return r;
}
SP_HD ge ge_neg(const ge& p) {
  ge r = p;
  r.X = fp_neg(p.X); r.T = fp_neg(p.T);
  return r;
}
SP_HD ge ge_sub(const ge& p, const ge& q) { return ge_add(p, ge_neg(q)); }
SP_HD bool ge_is_identity_class(const ge& p) {  // the ristretto identity class: X == 0 or Y == 0
  return fp_is_zero(p.X) || fp_is_zero(p.Y);
}

SP_HD ge_niels ge_to_niels(const ge& p) {  // one inversion
  u256 zi = fp_inv(p.Z);
  u256 x = fp_mul(p.X, zi), y = fp_mul(p.Y, zi);
  ge_niels r;
  r.ypx = fp_canon(fp_add(y, x));
  r.ymx = fp_canon(fp_sub(y, x));
  r.t2d = fp_canon(fp_mul(fp_mul(x, y), fp_2D()));
  return r;
}

// k*P, k given as canonical little-endian 256-bit integer limbs (not Montgomery); plain double-and-add, vartime
SP_HD ge ge_scalarmul(const u256& k, const ge& p) {
  ge acc = ge_identity();
  bool started = false;
  for (int i = 255; i >= 0; i--) {
    if (started) acc = ge_dbl(acc);
    if ((k.v[i >> 5] >> (i & 31)) & 1u) {
      acc = ge_add(acc, p);
      started = true;
    }
  }
  return acc;
}

// Signed W-bit recoding of a canonical scalar k < 2^253 (W <= 24): k = sum_w d_w * 2^(W*w) over ceil(253/W) windows, d_w in (-2^(W-1), 2^(W-1)].
// A window value above 2^(W-1) becomes v - 2^W and carries one into the next window; the top window never carries (its value is < 2^(W-1)).
SP_HD uint32_t scalar_window(const u256& k, int w, int wbits) {
  const int b = w * wbits, limb = b >> 5, sh = b & 31;
  if (limb >= 8) return 0;
  uint32_t v = k.v[limb] >> sh;
  if (sh + wbits > 32 && limb + 1 < 8) v |= k.v[limb + 1] << (32 - sh);
  return v & ((1u << wbits) - 1u);
}
SP_HD int signed_digit(const u256& k, int w, int wbits, uint32_t& carry) {   // the digit of window w, given the carry out of window w-1; updates carry
  const uint32_t half = 1u << (wbits - 1);
  const uint32_t v = scalar_window(k, w, wbits) + carry;
  carry = v > half ? 1u : 0u;
  return carry ? (int)v - (int)(2 * half) : (int)v;
}

// ---------------------------------------------------------------------------------------------- ristretto255
SP_HD u256 bytes_to_u256(const uint8_t* b) {
  u256 r;
  for (int i = 0; i < 8; i++)
    r.v[i] = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
  return r;
}
SP_HD void u256_to_bytes(uint8_t* b, const u256& a) {
  for (int i = 0; i < 8; i++) {
    b[4 * i] = (uint8_t)a.v[i]; b[4 * i + 1] = (uint8_t)(a.v[i] >> 8);
    b[4 * i + 2] = (uint8_t)(a.v[i] >> 16); b[4 * i + 3] = (uint8_t)(a.v[i] >> 24);
  }
}

// RFC 9496 4.3.2 Encode -> canonical field element s (caller stores its 32 little-endian bytes)
// RFC 9496 4.3.2 Encode, split around the inverse square root (see fp_sqrt_ratio_pre/post)
SP_HD u256 ristretto_encode_post(const ge& p, const u256& u1, const u256& u2, const u256& invsqrt) {
  u256 den1 = fp_mul(invsqrt, u1), den2 = fp_mul(invsqrt, u2);
  u256 z_inv = fp_mul(fp_mul(den1, den2), p.T);
  u256 ix0 = fp_mul(p.X, fp_SQRT_M1()), iy0 = fp_mul(p.Y, fp_SQRT_M1());
  u256 ench = fp_mul(den1, fp_INVSQRT_A_MINUS_D());
  bool rotate = fp_is_neg(fp_mul(p.T, z_inv));
  u256 x = rotate ? iy0 : p.X;
  u256 y = rotate ? ix0 : p.Y;
  u256 den_inv = rotate ? ench : den2;
  if (fp_is_neg(fp_mul(x, z_inv))) y = fp_neg(y);
  u256 s = fp_abs(fp_mul(den_inv, fp_sub(p.Z, y)));
  return fp_canon(s);
}
SP_HD u256 ristretto_encode(const ge& p) {
  u256 u1 = fp_mul(fp_add(p.Z, p.Y), fp_sub(p.Z, p.Y));
  u256 u2 = fp_mul(p.X, p.Y);
  u256 invsqrt;
  (void)fp_sqrt_ratio_i(invsqrt, fp_one(), fp_mul(u1, fp_sqr(u2)));
  return ristretto_encode_post(p, u1, u2, invsqrt);
}

// RFC 9496 4.3.1 Decode; false on a non-canonical / invalid encoding
SP_HD bool ristretto_decode(ge& out, const u256& sbytes) {
  if (sbytes.v[7] >> 31) return false;
  if (!fq_eq(fp_canon(sbytes), sbytes)) return false;  // non-canonical field element
  if (sbytes.v[0] & 1u) return false;                  // negative
  u256 s = sbytes;
  u256 ss = fp_sqr(s);
  u256 u1 = fp_sub(fp_one(), ss), u2 = fp_add(fp_one(), ss);
  u256 u2_sqr = fp_sqr(u2);
  u256 v = fp_sub(fp_neg(fp_mul(fp_D(), fp_sqr(u1))), u2_sqr);
  u256 invsqrt;
  bool was_square = fp_sqrt_ratio_i(invsqrt, fp_one(), fp_mul(v, u2_sqr));
  u256 den_x = fp_mul(invsqrt, u2);
  u256 den_y = fp_mul(fp_mul(invsqrt, den_x), v);
  u256 x = fp_abs(fp_mul(fp_add(s, s), den_x));
  u256 y = fp_mul(u1, den_y);
  u256 t = fp_mul(x, y);
  if (!was_square || fp_is_neg(t) || fp_is_zero(y)) return false;
  out.X = x; out.Y = y; out.Z = fp_one(); out.T = t;
  return true;
}

// RFC 9496 4.3.4 MAP (Elligator 2 for ristretto)
SP_HD ge ristretto_map(const u256& t) {
  u256 r = fp_mul(fp_SQRT_M1(), fp_sqr(t));
  u256 u = fp_mul(fp_add(r, fp_one()), fp_ONE_MINUS_D_SQ());
  u256 v = fp_mul(fp_sub(fp_neg(fp_one()), fp_mul(r, fp_D())), fp_add(r, fp_D()));
  u256 s;
  bool was_square = fp_sqrt_ratio_i(s, u, v);
  u256 s_prime = fp_neg(fp_abs(fp_mul(s, t)));
  u256 c = fp_neg(fp_one());
  if (!was_square) { s = s_prime; c = r; }
  u256 N = fp_sub(fp_mul(fp_mul(c, fp_sub(r, fp_one())), fp_D_MINUS_ONE_SQ()), v);
  u256 w0 = fp_mul(fp_add(s, s), v);
  u256 w1 = fp_mul(N, fp_SQRT_AD_MINUS_ONE());
  u256 s2 = fp_sqr(s);
  u256 w2 = fp_sub(fp_one(), s2), w3 = fp_add(fp_one(), s2);
  ge o;
  o.X = fp_mul(w0, w3); o.Y = fp_mul(w2, w1); o.Z = fp_mul(w1, w3); o.T = fp_mul(w0, w2);
  return o;
}
// RistrettoPoint::from_uniform_bytes: two maps of the masked 32-byte halves, added
SP_HD ge ristretto_from_uniform(const u256& lo, const u256& hi) {
  u256 a = lo, b = hi;
  a.v[7] &= 0x7fffffffu;
  b.v[7] &= 0x7fffffffu;
  return ge_add(ristretto_map(a), ristretto_map(b));
}

}  // namespace sp
