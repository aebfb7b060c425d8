// spartan_b200 — 256-bit modular arithmetic for sm_90a (and the host, same source).
//
// Two fields, both held as 8 x 32-bit little-endian limbs (one `uint4` pair = 32 bytes, so a table of
// scalars is loaded with two 128-bit LDGs per element):
//   Fq : the ristretto255 scalar field, q = 2^252 + 27742317777372353535851937790883648493, values in
//        Montgomery form with R = 2^256 and kept canonical in [0,q).  The byte layout of one element is
//        exactly the reference's `Scalar([u64;4])` (/root/reference/src/scalar/ristretto255.rs:195-199), so a
//        Rust `&[Scalar]` can be handed to the kernels without conversion.  mul = CIOS Montgomery product,
//        bit-identical to ristretto255.rs:690-714 + :642-686 because both return the canonical a*b*R^-1 mod q.
//   Fp : the curve field 2^255-19 (curve25519-dalek's FieldElement behind /root/reference/src/group.rs:6),
//        values kept "loose" in [0,2^256) modulo 2p = 2^256-38 and made canonical only when encoded.
//
// Everything is integer work on the INT32 pipe (IMAD.WIDE + IADD3 carry chains); there is no tensor-core
// formulation of a 256-bit modular product (see DESIGN.md).
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define SP_HD __host__ __device__ __forceinline__
#define SP_D __device__ __forceinline__
#else
#define SP_HD inline
#define SP_D inline
#endif

namespace sp {

struct alignas(16) u256 {
  uint32_t v[8];
};

// On the host (serial Fiat-Shamir tail: transcript-bound sigma protocols, a handful of fixed-base commitments per round)
// the two products use 64x64->128 multiplies over the same storage; the device uses the 32-bit IMAD formulation below.
// SP_FORCE_PORTABLE compiles the device formulation for the host too, so CPU-only tests can exercise it.
#if !defined(__CUDA_ARCH__) && !defined(SP_FORCE_PORTABLE) && defined(__SIZEOF_INT128__)
#define SP_HOST_FAST 1
inline u256 host_fq_mul(const u256& a, const u256& b);
inline u256 host_fp_mul(const u256& a, const u256& b);
#else
#define SP_HOST_FAST 0
#endif

// Constant multiplier of a sumcheck fold: a0 + r*(a1 - a0) with r fixed for a whole launch (dense_mlpoly.rs:215-223 binds every entry of every
// table with the same r).  k[8*j + i] = limb i of (r * 2^(32 j) mod q) with r taken OUT of Montgomery form, so that
//   a0 + sum_j d_j * K_j  =  a0 + r*d  (mod q)   for d = a1 - a0 given as eight 32-bit limbs d_j, all values staying in the Montgomery domain:
// the reduction of the shifted partial products is precomputed into the table (72 wide multiplications per fold instead of 112, and the
// addition of a0 rides in the first carry chain).  Built on the host once per round (fq_const_table) and passed as a kernel argument.
struct FqConst { uint32_t k[64]; };

}  // namespace sp
#include "mul_ptx.cuh"
namespace sp {

// ---------------------------------------------------------------------------------------------- Fq
// modulus / Montgomery constants (ristretto255.rs:248,304,307,315,323 split into 32-bit limbs)
#define SPQ0 0x5cf5d3edu
#define SPQ1 0x5812631au
#define SPQ2 0xa2f79cd6u
#define SPQ3 0x14def9deu
#define SPQ7 0x10000000u
#define SPQINV32 0x12547e1bu  // -(q^-1) mod 2^32 (low word of INV)

SP_HD u256 fq_zero() { u256 r; for (int i = 0; i < 8; i++) r.v[i] = 0; return r; }
SP_HD u256 fq_one() {  // R mod q
  u256 r = {{0x8d98951du, 0xd6ec3174u, 0x737dcf70u, 0xc6ef5bf4u, 0xfffffffeu, 0xffffffffu, 0xffffffffu, 0x0fffffffu}};
  return r;
}
SP_HD u256 fq_R2() {
  u256 r = {{0x449c0f01u, 0xa40611e3u, 0x68859347u, 0xd00e1ba7u, 0x17f5be65u, 0xceec73d2u, 0x7c309a3du, 0x0399411bu}};
  return r;
}
SP_HD u256 fq_R3() {
  u256 r = {{0x7b83a2dbu, 0x2a9e4968u, 0xaef7f3ecu, 0x278324e6u, 0x04ec5b65u, 0x8065dc6cu, 0x3599cec7u, 0x0e530b77u}};
  return r;
}
SP_HD uint32_t fq_modulus_limb(int i) {
  return i == 0 ? SPQ0 : i == 1 ? SPQ1 : i == 2 ? SPQ2 : i == 3 ? SPQ3 : i == 7 ? SPQ7 : 0u;
}

// r = a - q if a >= q else a   (a < 2q)
SP_HD u256 fq_cond_sub_q(const u256& a) {
  u256 d;
  int64_t borrow = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    int64_t t = (int64_t)a.v[i] - (int64_t)fq_modulus_limb(i) + borrow;
    d.v[i] = (uint32_t)t;
    borrow = t >> 32;  // 0 or -1
  }
  uint32_t keep = (uint32_t)borrow;  // all ones when a < q
  u256 r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = (a.v[i] & keep) | (d.v[i] & ~keep);
  return r;
}

#if defined(__CUDA_ARCH__)
// carry-chain forms for the device: one asm block per chain so the condition-code register never crosses statements
__device__ __forceinline__ u256 fq_csub_ptx(const u256& s) {   // s - q if s >= q else s   (s < 2q)
  u256 d, r;
  uint32_t borrow;
  asm("sub.cc.u32 %0, %9, %17;\n\tsubc.cc.u32 %1, %10, %18;\n\tsubc.cc.u32 %2, %11, %19;\n\tsubc.cc.u32 %3, %12, %20;\n\t"
      "subc.cc.u32 %4, %13, 0;\n\tsubc.cc.u32 %5, %14, 0;\n\tsubc.cc.u32 %6, %15, 0;\n\tsubc.cc.u32 %7, %16, %21;\n\tsubc.u32 %8, 0, 0;"
      : "=r"(d.v[0]), "=r"(d.v[1]), "=r"(d.v[2]), "=r"(d.v[3]), "=r"(d.v[4]), "=r"(d.v[5]), "=r"(d.v[6]), "=r"(d.v[7]), "=r"(borrow)
      : "r"(s.v[0]), "r"(s.v[1]), "r"(s.v[2]), "r"(s.v[3]), "r"(s.v[4]), "r"(s.v[5]), "r"(s.v[6]), "r"(s.v[7]),
        "r"(SPQ0), "r"(SPQ1), "r"(SPQ2), "r"(SPQ3), "r"(SPQ7));
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = borrow ? s.v[i] : d.v[i];   // borrow set <=> s < q
  return r;
}
__device__ __forceinline__ u256 fq_add_ptx(const u256& a, const u256& b) {
  u256 s, d;
  uint32_t borrow;
  asm("add.cc.u32 %0, %8, %16;\n\taddc.cc.u32 %1, %9, %17;\n\taddc.cc.u32 %2, %10, %18;\n\taddc.cc.u32 %3, %11, %19;\n\t"
      "addc.cc.u32 %4, %12, %20;\n\taddc.cc.u32 %5, %13, %21;\n\taddc.cc.u32 %6, %14, %22;\n\taddc.u32 %7, %15, %23;"
      : "=r"(s.v[0]), "=r"(s.v[1]), "=r"(s.v[2]), "=r"(s.v[3]), "=r"(s.v[4]), "=r"(s.v[5]), "=r"(s.v[6]), "=r"(s.v[7])
      : "r"(a.v[0]), "r"(a.v[1]), "r"(a.v[2]), "r"(a.v[3]), "r"(a.v[4]), "r"(a.v[5]), "r"(a.v[6]), "r"(a.v[7]),
        "r"(b.v[0]), "r"(b.v[1]), "r"(b.v[2]), "r"(b.v[3]), "r"(b.v[4]), "r"(b.v[5]), "r"(b.v[6]), "r"(b.v[7]));
  asm("sub.cc.u32 %0, %9, %17;\n\tsubc.cc.u32 %1, %10, %18;\n\tsubc.cc.u32 %2, %11, %19;\n\tsubc.cc.u32 %3, %12, %20;\n\t"
      "subc.cc.u32 %4, %13, 0;\n\tsubc.cc.u32 %5, %14, 0;\n\tsubc.cc.u32 %6, %15, 0;\n\tsubc.cc.u32 %7, %16, %21;\n\tsubc.u32 %8, 0, 0;"
      : "=r"(d.v[0]), "=r"(d.v[1]), "=r"(d.v[2]), "=r"(d.v[3]), "=r"(d.v[4]), "=r"(d.v[5]), "=r"(d.v[6]), "=r"(d.v[7]), "=r"(borrow)
      : "r"(s.v[0]), "r"(s.v[1]), "r"(s.v[2]), "r"(s.v[3]), "r"(s.v[4]), "r"(s.v[5]), "r"(s.v[6]), "r"(s.v[7]),
        "r"(SPQ0), "r"(SPQ1), "r"(SPQ2), "r"(SPQ3), "r"(SPQ7));
  u256 r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = borrow ? s.v[i] : d.v[i];   // borrow set <=> a + b < q
  return r;
}
__device__ __forceinline__ u256 fq_sub_ptx(const u256& a, const u256& b) {
  u256 d, r;
  uint32_t mask;
  asm("sub.cc.u32 %0, %9, %17;\n\tsubc.cc.u32 %1, %10, %18;\n\tsubc.cc.u32 %2, %11, %19;\n\tsubc.cc.u32 %3, %12, %20;\n\t"
      "subc.cc.u32 %4, %13, %21;\n\tsubc.cc.u32 %5, %14, %22;\n\tsubc.cc.u32 %6, %15, %23;\n\tsubc.cc.u32 %7, %16, %24;\n\tsubc.u32 %8, 0, 0;"
      : "=r"(d.v[0]), "=r"(d.v[1]), "=r"(d.v[2]), "=r"(d.v[3]), "=r"(d.v[4]), "=r"(d.v[5]), "=r"(d.v[6]), "=r"(d.v[7]), "=r"(mask)
      : "r"(a.v[0]), "r"(a.v[1]), "r"(a.v[2]), "r"(a.v[3]), "r"(a.v[4]), "r"(a.v[5]), "r"(a.v[6]), "r"(a.v[7]),
        "r"(b.v[0]), "r"(b.v[1]), "r"(b.v[2]), "r"(b.v[3]), "r"(b.v[4]), "r"(b.v[5]), "r"(b.v[6]), "r"(b.v[7]));
  uint32_t q0 = SPQ0 & mask, q1 = SPQ1 & mask, q2 = SPQ2 & mask, q3 = SPQ3 & mask, q7 = SPQ7 & mask;   // add q back on underflow
  asm("add.cc.u32 %0, %8, %16;\n\taddc.cc.u32 %1, %9, %17;\n\taddc.cc.u32 %2, %10, %18;\n\taddc.cc.u32 %3, %11, %19;\n\t"
      "addc.cc.u32 %4, %12, 0;\n\taddc.cc.u32 %5, %13, 0;\n\taddc.cc.u32 %6, %14, 0;\n\taddc.u32 %7, %15, %20;"
      : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]), "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7])
      : "r"(d.v[0]), "r"(d.v[1]), "r"(d.v[2]), "r"(d.v[3]), "r"(d.v[4]), "r"(d.v[5]), "r"(d.v[6]), "r"(d.v[7]),
        "r"(q0), "r"(q1), "r"(q2), "r"(q3), "r"(q7));
  return r;
}
#endif

SP_HD u256 fq_add(const u256& a, const u256& b) {  // ristretto255.rs:736-745
#if defined(__CUDA_ARCH__) && !defined(SP_NO_PTX)
  return fq_add_ptx(a, b);
#else
  u256 s;
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    c += (uint64_t)a.v[i] + b.v[i];
    s.v[i] = (uint32_t)c;
    c >>= 32;
  }
  return fq_cond_sub_q(s);  // a,b < q < 2^253: no carry out of limb 7
#endif
}

SP_HD u256 fq_sub(const u256& a, const u256& b) {  // ristretto255.rs:718-733
#if defined(__CUDA_ARCH__) && !defined(SP_NO_PTX)
  return fq_sub_ptx(a, b);
#else
  u256 d;
  int64_t borrow = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    int64_t t = (int64_t)a.v[i] - (int64_t)b.v[i] + borrow;
    d.v[i] = (uint32_t)t;
    borrow = t >> 32;
  }
  uint32_t mask = (uint32_t)borrow;  // all ones on underflow: add q back
  uint64_t c = 0;
  u256 r;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    c += (uint64_t)d.v[i] + (fq_modulus_limb(i) & mask);
    r.v[i] = (uint32_t)c;
    c >>= 32;
  }
  return r;
#endif
}

SP_HD u256 fq_neg(const u256& a) { return fq_sub(fq_zero(), a); }  // ristretto255.rs:749-765
SP_HD u256 fq_dbl(const u256& a) { return fq_add(a, a); }

SP_HD bool fq_is_zero(const u256& a) {
  uint32_t o = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) o |= a.v[i];
  return o == 0;
}
SP_HD bool fq_eq(const u256& a, const u256& b) {
  uint32_t o = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) o |= a.v[i] ^ b.v[i];
  return o == 0;
}

// Montgomery product a*b*2^-256 mod q, coarsely-integrated operand scanning on 32-bit limbs.
// The three zero limbs of q (4,5,6) drop out of the reduction at compile time.
#ifdef __CUDA_ARCH__
static __device__ __noinline__ u256 fq_mul_ni(u256 a, u256 b);
#endif
SP_HD u256 fq_mul_impl(const u256& a, const u256& b);
SP_HD u256 fq_mul(const u256& a, const u256& b) {
#ifdef __CUDA_ARCH__
  return fq_mul_ni(a, b);   // keeps the instruction footprint of the big fused kernels inside the instruction cache
#else
  return fq_mul_impl(a, b);
#endif
}
SP_HD u256 fq_mul_impl(const u256& a, const u256& b) {
#if SP_HOST_FAST
  return host_fq_mul(a, b);
#elif defined(__CUDA_ARCH__) && !defined(SP_NO_PTX)
  return fq_csub_ptx(fq_mul_ptx(a, b));   // generated carry-chain form (tools/gen_ptx_mul.py); the portable form below is the specification
#else
  uint32_t t[10];
#pragma unroll
  for (int i = 0; i < 10; i++) t[i] = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    uint64_t c = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      c += (uint64_t)a.v[j] * b.v[i] + t[j];
      t[j] = (uint32_t)c;
      c >>= 32;
    }
    c += t[8];
    t[8] = (uint32_t)c;
    t[9] = (uint32_t)(c >> 32);
    uint32_t m = t[0] * SPQINV32;
    c = ((uint64_t)m * SPQ0 + t[0]) >> 32;
    c += (uint64_t)m * SPQ1 + t[1]; t[0] = (uint32_t)c; c >>= 32;
    c += (uint64_t)m * SPQ2 + t[2]; t[1] = (uint32_t)c; c >>= 32;
    c += (uint64_t)m * SPQ3 + t[3]; t[2] = (uint32_t)c; c >>= 32;
    c += t[4]; t[3] = (uint32_t)c; c >>= 32;
    c += t[5]; t[4] = (uint32_t)c; c >>= 32;
    c += t[6]; t[5] = (uint32_t)c; c >>= 32;
    c += (uint64_t)m * SPQ7 + t[7]; t[6] = (uint32_t)c; c >>= 32;
    c += t[8]; t[7] = (uint32_t)c; c >>= 32;
    t[8] = t[9] + (uint32_t)c;
  }
  u256 r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = t[i];
  return fq_cond_sub_q(r);  // t < 2q and t[8] == 0
#endif
}
#ifdef __CUDA_ARCH__
static __device__ __noinline__ u256 fq_mul_ni(u256 a, u256 b) { return fq_mul_impl(a, b); }
#endif
SP_HD u256 fq_sqr(const u256& a) { return fq_mul(a, a); }

// out of Montgomery form: a * 1 * R^-1 (Scalar::to_bytes, ristretto255.rs:419-431) -> canonical integer limbs
SP_HD u256 fq_from_mont(const u256& a) {
  u256 one = fq_zero();
  one.v[0] = 1;
  return fq_mul(a, one);
}
SP_HD u256 fq_to_mont(const u256& a) { return fq_mul(a, fq_R2()); }  // a < 2^256 allowed (ristretto255.rs:449-462)
SP_HD u256 fq_from_u64(uint64_t x) {                                // From<u64>, ristretto255.rs:214-218
  u256 t = fq_zero();
  t.v[0] = (uint32_t)x;
  t.v[1] = (uint32_t)(x >> 32);
  return fq_to_mont(t);
}
// Scalar::from_bytes_wide (ristretto255.rs:435-466): lo*R2 + hi*R3
SP_HD u256 fq_from_wide(const u256& lo, const u256& hi) { return fq_add(fq_mul(lo, fq_R2()), fq_mul(hi, fq_R3())); }

// table for fq_fold_const: K_0 = r out of Montgomery form, K_{j+1} = K_j * 2^32 mod q  (one Montgomery product by 2^32*R each)
SP_HD FqConst fq_const_table(const u256& r_mont) {
  FqConst c;
  u256 kj = fq_from_mont(r_mont);
  const u256 two32 = fq_from_u64((uint64_t)1 << 32);
  for (int j = 0; j < 8; j++) {
    for (int i = 0; i < 8; i++) c.k[8 * j + i] = kj.v[i];
    kj = fq_mul(kj, two32);
  }
  return c;
}
// a0 + r*(a1 - a0), bit-identical to fq_add(a0, fq_mul(r, fq_sub(a1, a0))) (both are the canonical residue)
SP_HD u256 fq_fold_const(const u256& a0, const u256& a1, const FqConst& rc) {
#if defined(__CUDA_ARCH__) && !defined(SP_NO_PTX)
  // d = a1 - a0 + q in (0, 2q): two unconditional chains, no select
  u256 d;
  asm("sub.cc.u32 %0, %8, %16;\n\tsubc.cc.u32 %1, %9, %17;\n\tsubc.cc.u32 %2, %10, %18;\n\tsubc.cc.u32 %3, %11, %19;\n\t"
      "subc.cc.u32 %4, %12, %20;\n\tsubc.cc.u32 %5, %13, %21;\n\tsubc.cc.u32 %6, %14, %22;\n\tsubc.u32 %7, %15, %23;\n\t"
      "add.cc.u32 %0, %0, %24;\n\taddc.cc.u32 %1, %1, %25;\n\taddc.cc.u32 %2, %2, %26;\n\taddc.cc.u32 %3, %3, %27;\n\t"
      "addc.cc.u32 %4, %4, 0;\n\taddc.cc.u32 %5, %5, 0;\n\taddc.cc.u32 %6, %6, 0;\n\taddc.u32 %7, %7, %28;"
      : "=&r"(d.v[0]), "=&r"(d.v[1]), "=&r"(d.v[2]), "=&r"(d.v[3]), "=&r"(d.v[4]), "=&r"(d.v[5]), "=&r"(d.v[6]), "=&r"(d.v[7])
      : "r"(a1.v[0]), "r"(a1.v[1]), "r"(a1.v[2]), "r"(a1.v[3]), "r"(a1.v[4]), "r"(a1.v[5]), "r"(a1.v[6]), "r"(a1.v[7]),
        "r"(a0.v[0]), "r"(a0.v[1]), "r"(a0.v[2]), "r"(a0.v[3]), "r"(a0.v[4]), "r"(a0.v[5]), "r"(a0.v[6]), "r"(a0.v[7]),
        "r"(SPQ0), "r"(SPQ1), "r"(SPQ2), "r"(SPQ3), "r"(SPQ7));
  return fq_csub_ptx(fq_fold_const_ptx(a0, d, rc));
#else
  // portable specification: the same sum of partial products on 64-bit accumulators, then the fold through 2^252 = -c (mod q)
  uint32_t d[8];
  {
    int64_t borrow = 0;
    uint32_t t[8];
    for (int i = 0; i < 8; i++) { int64_t x = (int64_t)a1.v[i] - (int64_t)a0.v[i] + borrow; t[i] = (uint32_t)x; borrow = x >> 32; }
    uint64_t c = 0;
    for (int i = 0; i < 8; i++) { c += (uint64_t)t[i] + fq_modulus_limb(i); d[i] = (uint32_t)c; c >>= 32; }
  }
  uint32_t T[10];
  for (int i = 0; i < 8; i++) T[i] = a0.v[i];
  T[8] = 0; T[9] = 0;
  for (int j = 0; j < 8; j++) {
    uint64_t c = 0;
    for (int i = 0; i < 8; i++) { c += (uint64_t)d[j] * rc.k[8 * j + i] + T[i]; T[i] = (uint32_t)c; c >>= 32; }
    c += T[8]; T[8] = (uint32_t)c; c >>= 32;
    T[9] += (uint32_t)c;
  }
  // T < 2^288: hi = T >> 252 (36 bits)
  const uint64_t hi = ((uint64_t)T[8] << 4) | (T[7] >> 28);
  const uint32_t hi0 = (uint32_t)hi, hi1 = (uint32_t)(hi >> 32);
  uint32_t X[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  {
    uint64_t c = 0;
    for (int i = 0; i < 4; i++) { c += (uint64_t)hi0 * fq_modulus_limb(i); X[i] = (uint32_t)c; c >>= 32; }
    X[4] = (uint32_t)c;
    c = 0;
    for (int i = 0; i < 4; i++) { c += (uint64_t)hi1 * fq_modulus_limb(i) + X[i + 1]; X[i + 1] = (uint32_t)c; c >>= 32; }
    X[5] = (uint32_t)c;
  }
  u256 u;
  {
    uint64_t c = 0;
    for (int i = 0; i < 8; i++) { c += (uint64_t)(i == 7 ? (T[7] & 0x0fffffffu) : T[i]) + fq_modulus_limb(i); u.v[i] = (uint32_t)c; c >>= 32; }
    int64_t borrow = 0;
    for (int i = 0; i < 8; i++) { int64_t x = (int64_t)u.v[i] - (int64_t)X[i] + borrow; u.v[i] = (uint32_t)x; borrow = x >> 32; }
  }
  return fq_cond_sub_q(u);
#endif
}

// a^(q-2) by the reference's addition chain (ristretto255.rs:541-595); a == 0 -> 0
SP_HD u256 fq_inv(const u256& a) {
  u256 _1 = a, _10 = fq_sqr(_1), _100 = fq_sqr(_10), _11 = fq_mul(_10, _1), _101 = fq_mul(_10, _11), _111 = fq_mul(_10, _101),
       _1001 = fq_mul(_10, _111), _1011 = fq_mul(_10, _1001), _1111 = fq_mul(_100, _1011);
  u256 y = fq_mul(_1111, _1);
#define SP_SQMUL(n, x)                       \
  for (int _i = 0; _i < (n); _i++) y = fq_sqr(y); \
  y = fq_mul(y, x);
  SP_SQMUL(126, _101) SP_SQMUL(4, _11) SP_SQMUL(5, _1111) SP_SQMUL(5, _1111) SP_SQMUL(4, _1001) SP_SQMUL(2, _11)
  SP_SQMUL(5, _1111) SP_SQMUL(4, _101) SP_SQMUL(6, _101) SP_SQMUL(3, _111) SP_SQMUL(5, _1111) SP_SQMUL(5, _111)
  SP_SQMUL(4, _11) SP_SQMUL(5, _1011) SP_SQMUL(6, _1011) SP_SQMUL(10, _1001) SP_SQMUL(4, _11) SP_SQMUL(5, _11)
  SP_SQMUL(5, _11) SP_SQMUL(5, _1001) SP_SQMUL(4, _111) SP_SQMUL(6, _1111) SP_SQMUL(5, _1011) SP_SQMUL(3, _101)
  SP_SQMUL(6, _1111) SP_SQMUL(3, _101) SP_SQMUL(3, _11)
#undef SP_SQMUL
  return y;
}

// ---------------------------------------------------------------------------------------------- Fp = 2^255-19
SP_HD u256 fp_zero() { return fq_zero(); }
SP_HD u256 fp_one() { u256 r = fq_zero(); r.v[0] = 1; return r; }

// fold a carry-out word back: x + 38*c, repeated until no carry (value stays < 2^256)
SP_HD void fp_fold(u256& x, uint64_t c) {
#pragma unroll
  for (int rep = 0; rep < 2; rep++) {
    uint64_t k = c * 38;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      k += x.v[i];
      x.v[i] = (uint32_t)k;
      k >>= 32;
    }
    c = k;
  }
}

#if defined(__CUDA_ARCH__)
// carry-chain forms for the device (values stay loose in [0, 2^256), congruent mod p; 2^256 = 38 mod p)
__device__ __forceinline__ u256 fp_add_ptx(const u256& a, const u256& b) {
  u256 s, r;
  uint32_t c, c2;
  asm("add.cc.u32 %0, %9, %17;\n\taddc.cc.u32 %1, %10, %18;\n\taddc.cc.u32 %2, %11, %19;\n\taddc.cc.u32 %3, %12, %20;\n\t"
      "addc.cc.u32 %4, %13, %21;\n\taddc.cc.u32 %5, %14, %22;\n\taddc.cc.u32 %6, %15, %23;\n\taddc.cc.u32 %7, %16, %24;\n\taddc.u32 %8, 0, 0;"
      : "=r"(s.v[0]), "=r"(s.v[1]), "=r"(s.v[2]), "=r"(s.v[3]), "=r"(s.v[4]), "=r"(s.v[5]), "=r"(s.v[6]), "=r"(s.v[7]), "=r"(c)
      : "r"(a.v[0]), "r"(a.v[1]), "r"(a.v[2]), "r"(a.v[3]), "r"(a.v[4]), "r"(a.v[5]), "r"(a.v[6]), "r"(a.v[7]),
        "r"(b.v[0]), "r"(b.v[1]), "r"(b.v[2]), "r"(b.v[3]), "r"(b.v[4]), "r"(b.v[5]), "r"(b.v[6]), "r"(b.v[7]));
  uint32_t k = c * 38u;   // fold the carry-out back in
  asm("add.cc.u32 %0, %9, %17;\n\taddc.cc.u32 %1, %10, 0;\n\taddc.cc.u32 %2, %11, 0;\n\taddc.cc.u32 %3, %12, 0;\n\t"
      "addc.cc.u32 %4, %13, 0;\n\taddc.cc.u32 %5, %14, 0;\n\taddc.cc.u32 %6, %15, 0;\n\taddc.cc.u32 %7, %16, 0;\n\taddc.u32 %8, 0, 0;"
      : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]), "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7]), "=r"(c2)
      : "r"(s.v[0]), "r"(s.v[1]), "r"(s.v[2]), "r"(s.v[3]), "r"(s.v[4]), "r"(s.v[5]), "r"(s.v[6]), "r"(s.v[7]), "r"(k));
  r.v[0] += c2 * 38u;     // a second wrap leaves a value < 38*2, so this cannot carry
  return r;
}
__device__ __forceinline__ u256 fp_sub_ptx(const u256& a, const u256& b) {
  u256 d, r;
  uint32_t bw, bw2;
  asm("sub.cc.u32 %0, %9, %17;\n\tsubc.cc.u32 %1, %10, %18;\n\tsubc.cc.u32 %2, %11, %19;\n\tsubc.cc.u32 %3, %12, %20;\n\t"
      "subc.cc.u32 %4, %13, %21;\n\tsubc.cc.u32 %5, %14, %22;\n\tsubc.cc.u32 %6, %15, %23;\n\tsubc.cc.u32 %7, %16, %24;\n\tsubc.u32 %8, 0, 0;"
      : "=r"(d.v[0]), "=r"(d.v[1]), "=r"(d.v[2]), "=r"(d.v[3]), "=r"(d.v[4]), "=r"(d.v[5]), "=r"(d.v[6]), "=r"(d.v[7]), "=r"(bw)
      : "r"(a.v[0]), "r"(a.v[1]), "r"(a.v[2]), "r"(a.v[3]), "r"(a.v[4]), "r"(a.v[5]), "r"(a.v[6]), "r"(a.v[7]),
        "r"(b.v[0]), "r"(b.v[1]), "r"(b.v[2]), "r"(b.v[3]), "r"(b.v[4]), "r"(b.v[5]), "r"(b.v[6]), "r"(b.v[7]));
  uint32_t k = bw & 38u;  // wrapped by 2^256 = 38 (mod p): take 38 back out
  asm("sub.cc.u32 %0, %9, %17;\n\tsubc.cc.u32 %1, %10, 0;\n\tsubc.cc.u32 %2, %11, 0;\n\tsubc.cc.u32 %3, %12, 0;\n\t"
      "subc.cc.u32 %4, %13, 0;\n\tsubc.cc.u32 %5, %14, 0;\n\tsubc.cc.u32 %6, %15, 0;\n\tsubc.cc.u32 %7, %16, 0;\n\tsubc.u32 %8, 0, 0;"
      : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]), "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7]), "=r"(bw2)
      : "r"(d.v[0]), "r"(d.v[1]), "r"(d.v[2]), "r"(d.v[3]), "r"(d.v[4]), "r"(d.v[5]), "r"(d.v[6]), "r"(d.v[7]), "r"(k));
  r.v[0] -= bw2 & 38u;    // second wrap: the value is then >= 2^256 - 38, so this cannot borrow
  return r;
}
#endif

SP_HD u256 fp_add(const u256& a, const u256& b) {
#if defined(__CUDA_ARCH__) && !defined(SP_NO_PTX)
  return fp_add_ptx(a, b);
#else
  u256 s;
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    c += (uint64_t)a.v[i] + b.v[i];
    s.v[i] = (uint32_t)c;
    c >>= 32;
  }
  fp_fold(s, c);
  return s;
#endif
}
SP_HD u256 fp_sub(const u256& a, const u256& b) {
#if defined(__CUDA_ARCH__) && !defined(SP_NO_PTX)
  return fp_sub_ptx(a, b);
#else
  u256 d;
  int64_t borrow = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    int64_t t = (int64_t)a.v[i] - (int64_t)b.v[i] + borrow;
    d.v[i] = (uint32_t)t;
    borrow = t >> 32;
  }
  // wrapped by 2^256 = 38 (mod p): take 38 back out, twice at most
#pragma unroll
  for (int rep = 0; rep < 2; rep++) {
    int64_t k = borrow ? -38 : 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      int64_t t = (int64_t)d.v[i] + k;
      d.v[i] = (uint32_t)t;
      k = t >> 32;
    }
    borrow = k;
  }
  return d;
#endif
}
SP_HD u256 fp_neg(const u256& a) { return fp_sub(fp_zero(), a); }

SP_HD u256 fp_mul_impl(const u256& a, const u256& b);
SP_HD u256 fp_mul(const u256& a, const u256& b) { return fp_mul_impl(a, b); }
SP_HD u256 fp_mul_impl(const u256& a, const u256& b) {
#if SP_HOST_FAST
  return host_fp_mul(a, b);
#elif defined(__CUDA_ARCH__) && !defined(SP_NO_PTX)
  return fp_mul_ptx(a, b);
#else
  uint32_t t[16];
#pragma unroll
  for (int i = 0; i < 16; i++) t[i] = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    uint64_t c = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      c += (uint64_t)a.v[j] * b.v[i] + t[i + j];
      t[i + j] = (uint32_t)c;
      c >>= 32;
    }
    t[i + 8] = (uint32_t)c;
  }
  u256 r;
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    c += (uint64_t)t[i + 8] * 38u + t[i];
    r.v[i] = (uint32_t)c;
    c >>= 32;
  }
  fp_fold(r, c);
  return r;
#endif
}
#if defined(__CUDA_ARCH__)
static __device__ __noinline__ u256 fp_mul_ni(u256 a, u256 b) { return fp_mul_impl(a, b); }
#endif
SP_HD u256 fp_sqr(const u256& a) { return fp_mul(a, a); }
// out-of-line multiplication for the long exponentiation chains (inversion, square roots: ~265 multiplications each): there the call
// overhead is irrelevant and one shared body keeps compress/decompress kernels small
SP_HD u256 fp_mulc(const u256& a, const u256& b) {
#if defined(__CUDA_ARCH__)
  return fp_mul_ni(a, b);
#else
  return fp_mul_impl(a, b);
#endif
}
SP_HD u256 fp_sqrc(const u256& a) { return fp_mulc(a, a); }
SP_HD u256 fp_mul_small(const u256& a, uint32_t k) {
  u256 r;
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    c += (uint64_t)a.v[i] * k;
    r.v[i] = (uint32_t)c;
    c >>= 32;
  }
  fp_fold(r, c);
  return r;
}

// canonical representative in [0,p)
SP_HD u256 fp_canon(const u256& a) {
  u256 x = a;
  // bring below 2^255: x = (x mod 2^255) + 19*(x >> 255)
  uint64_t c = (uint64_t)(x.v[7] >> 31) * 19;
  x.v[7] &= 0x7fffffffu;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    c += x.v[i];
    x.v[i] = (uint32_t)c;
    c >>= 32;
  }
  // x < 2^255 + 19: subtract p if x >= p, i.e. if x + 19 has bit 255 set
  u256 y;
  c = 19;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    c += x.v[i];
    y.v[i] = (uint32_t)c;
    c >>= 32;
  }
  bool ge = (y.v[7] >> 31) != 0;
  y.v[7] &= 0x7fffffffu;
  return ge ? y : x;
}
SP_HD bool fp_is_zero(const u256& a) { return fq_is_zero(fp_canon(a)); }
SP_HD bool fp_eq(const u256& a, const u256& b) { return fq_eq(fp_canon(a), fp_canon(b)); }
SP_HD bool fp_is_neg(const u256& a) { return (fp_canon(a).v[0] & 1u) != 0; }
SP_HD u256 fp_abs(const u256& a) { return fp_is_neg(a) ? fp_neg(a) : a; }
SP_HD u256 fp_sqn(u256 a, int n) {
#pragma unroll 1
  for (int i = 0; i < n; i++) a = fp_sqrc(a);
  return a;
}

// z^(2^250-1) and z^11, shared by inversion and the square-root exponent
SP_HD void fp_pow250(const u256& z, u256& t250, u256& z11) {
  u256 z2 = fp_sqrc(z);
  u256 z9 = fp_mulc(fp_sqn(z2, 2), z);
  z11 = fp_mulc(z9, z2);
  u256 z_5_0 = fp_mulc(fp_sqrc(z11), z9);
  u256 z_10_0 = fp_mulc(fp_sqn(z_5_0, 5), z_5_0);
  u256 z_20_0 = fp_mulc(fp_sqn(z_10_0, 10), z_10_0);
  u256 z_40_0 = fp_mulc(fp_sqn(z_20_0, 20), z_20_0);
  u256 z_50_0 = fp_mulc(fp_sqn(z_40_0, 10), z_10_0);
  u256 z_100_0 = fp_mulc(fp_sqn(z_50_0, 50), z_50_0);
  u256 z_200_0 = fp_mulc(fp_sqn(z_100_0, 100), z_100_0);
  t250 = fp_mulc(fp_sqn(z_200_0, 50), z_50_0);
}
SP_HD u256 fp_inv(const u256& z) {
  u256 t250, z11;
  fp_pow250(z, t250, z11);
  return fp_mulc(fp_sqn(t250, 5), z11);
}
SP_HD u256 fp_pow22523(const u256& z) {
  u256 t250, z11;
  fp_pow250(z, t250, z11);
  return fp_mulc(fp_sqn(t250, 2), z);
}

// curve / ristretto constants (RFC 9496 section 4.1)
SP_HD u256 fp_D() { u256 r = {{0x135978a3u, 0x75eb4dcau, 0x4141d8abu, 0x00700a4du, 0x7779e898u, 0x8cc74079u, 0x2b6ffe73u, 0x52036ceeu}}; return r; }
SP_HD u256 fp_2D() { u256 r = {{0x26b2f159u, 0xebd69b94u, 0x8283b156u, 0x00e0149au, 0xeef3d130u, 0x198e80f2u, 0x56dffce7u, 0x2406d9dcu}}; return r; }
SP_HD u256 fp_SQRT_M1() { u256 r = {{0x4a0ea0b0u, 0xc4ee1b27u, 0xad2fe478u, 0x2f431806u, 0x3dfbd7a7u, 0x2b4d0099u, 0x4fc1df0bu, 0x2b832480u}}; return r; }
SP_HD u256 fp_SQRT_AD_MINUS_ONE() { u256 r = {{0x497b2e1bu, 0x7e97f6a0u, 0x1b7854bdu, 0xaf9d8e0cu, 0x31f5d1fdu, 0x0f3cfcc9u, 0x2b8348acu, 0x376931bfu}}; return r; }
SP_HD u256 fp_INVSQRT_A_MINUS_D() { u256 r = {{0x805d40eau, 0x99c8fdaau, 0x5a4172beu, 0x9d2f1617u, 0xfe01d840u, 0x16c27b91u, 0xcfaffca2u, 0x786c8905u}}; return r; }
SP_HD u256 fp_ONE_MINUS_D_SQ() { u256 r = {{0x945fc176u, 0xe27c09c1u, 0xcd5e350fu, 0x2c81a138u, 0xbe70dfe4u, 0x9994abddu, 0xb2b3e0d7u, 0x029072a8u}}; return r; }
SP_HD u256 fp_D_MINUS_ONE_SQ() { u256 r = {{0x44ed4d20u, 0x31ad5aaau, 0xb01e1999u, 0xd29e4a2cu, 0x529b4eebu, 0x4cdcd32fu, 0xf66c2241u, 0x5968b37au}}; return r; }

// RFC 9496 4.2 SQRT_RATIO_M1, split around its one exponentiation so that callers can run several exponentiations side by side
SP_HD u256 fp_sqrt_ratio_pre(const u256& u, const u256& v, u256& uv3) {   // returns u*v^7 (to be raised to (p-5)/8), sets uv3 = u*v^3
  u256 v3 = fp_mul(fp_sqr(v), v);
  u256 v7 = fp_mul(fp_sqr(v3), v);
  uv3 = fp_mul(u, v3);
  return fp_mul(u, v7);
}
SP_HD bool fp_sqrt_ratio_post(u256& out, const u256& u, const u256& v, const u256& uv3, const u256& pw) {
  u256 r = fp_mul(uv3, pw);
  u256 check = fp_mul(v, fp_sqr(r));
  u256 neg_u = fp_neg(u);
  bool correct = fp_eq(check, u);
  bool flipped = fp_eq(check, neg_u);
  bool flipped_i = fp_eq(check, fp_mul(neg_u, fp_SQRT_M1()));
  if (flipped || flipped_i) r = fp_mul(r, fp_SQRT_M1());
  out = fp_abs(r);
  return correct || flipped;
}
SP_HD bool fp_sqrt_ratio_i(u256& out, const u256& u, const u256& v) {
  u256 uv3;
  u256 base = fp_sqrt_ratio_pre(u, v, uv3);
  return fp_sqrt_ratio_post(out, u, v, uv3, fp_pow22523(base));
}

#if SP_HOST_FAST
inline u256 host_fq_mul(const u256& a, const u256& b) {   // CIOS Montgomery multiplication on 4x64-bit limbs (q has a zero limb: one product fewer per row)
  typedef unsigned __int128 u128;
  const uint64_t q0 = 0x5812631a5cf5d3edULL, q1 = 0x14def9dea2f79cd6ULL, q3 = 0x1000000000000000ULL;
  const uint64_t inv = 0xd2b51da312547e1bULL;
  uint64_t x[4], y[4];
  memcpy(x, a.v, 32); memcpy(y, b.v, 32);   // little-endian host: the 8x32-bit limbs are the 4x64-bit limbs
  uint64_t t0 = 0, t1 = 0, t2 = 0, t3 = 0, t4 = 0;
#if !defined(__CUDACC__)
#pragma GCC unroll 4
#endif
  for (int i = 0; i < 4; i++) {
    const uint64_t yi = y[i];
    u128 c = (u128)x[0] * yi + t0; t0 = (uint64_t)c; c >>= 64;
    c += (u128)x[1] * yi + t1; t1 = (uint64_t)c; c >>= 64;
    c += (u128)x[2] * yi + t2; t2 = (uint64_t)c; c >>= 64;
    c += (u128)x[3] * yi + t3; t3 = (uint64_t)c; c >>= 64;
    c += t4; t4 = (uint64_t)c; const uint64_t t5 = (uint64_t)(c >> 64);
    const uint64_t m = t0 * inv;
    c = ((u128)m * q0 + t0) >> 64;
    c += (u128)m * q1 + t1; t0 = (uint64_t)c; c >>= 64;
    c += t2; t1 = (uint64_t)c; c >>= 64;
    c += (u128)m * q3 + t3; t2 = (uint64_t)c; c >>= 64;
    c += t4; t3 = (uint64_t)c; c >>= 64;
    t4 = t5 + (uint64_t)c;
  }
  // result < 2q: subtract q once if needed
  u128 d = (u128)t0 - q0; uint64_t r0 = (uint64_t)d; uint64_t bw = (uint64_t)(d >> 64) & 1;
  d = (u128)t1 - q1 - bw; uint64_t r1 = (uint64_t)d; bw = (uint64_t)(d >> 64) & 1;
  d = (u128)t2 - bw; uint64_t r2 = (uint64_t)d; bw = (uint64_t)(d >> 64) & 1;
  d = (u128)t3 - q3 - bw; uint64_t r3 = (uint64_t)d; bw = (uint64_t)(d >> 64) & 1;
  const bool keep = bw && !t4;   // borrow out and no carry word: t < q
  uint64_t r[4] = {keep ? t0 : r0, keep ? t1 : r1, keep ? t2 : r2, keep ? t3 : r3};
  u256 o;
  memcpy(o.v, r, 32);
  return o;
}
inline u256 host_fp_mul(const u256& a, const u256& b) {
  typedef unsigned __int128 u128;
  uint64_t x[4], y[4], t[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 4; i++) { x[i] = (uint64_t)a.v[2 * i] | ((uint64_t)a.v[2 * i + 1] << 32); y[i] = (uint64_t)b.v[2 * i] | ((uint64_t)b.v[2 * i + 1] << 32); }
  for (int i = 0; i < 4; i++) {
    u128 c = 0;
    for (int j = 0; j < 4; j++) { c += (u128)x[j] * y[i] + t[i + j]; t[i + j] = (uint64_t)c; c >>= 64; }
    t[i + 4] = (uint64_t)c;
  }
  u128 c = 0;
  uint64_t r[4];
  for (int i = 0; i < 4; i++) { c += (u128)t[i + 4] * 38u + t[i]; r[i] = (uint64_t)c; c >>= 64; }
  for (int rep = 0; rep < 2; rep++) {
    u128 k = c * 38u;
    for (int i = 0; i < 4; i++) { k += r[i]; r[i] = (uint64_t)k; k >>= 64; }
    c = k;
  }
  u256 o;
  for (int i = 0; i < 4; i++) { o.v[2 * i] = (uint32_t)r[i]; o.v[2 * i + 1] = (uint32_t)(r[i] >> 32); }
  return o;
}
#endif

}  // namespace sp
