// spartan_b200 — host side of the prover: scalar wrapper, Merlin transcript, RandomTape, small fixed-base commitments.
//
// This is the part of the reference that stays on the CPU in a GPU deployment: the Fiat-Shamir transcript is a strict serial
// dependency between kernel launches (/root/reference/src/transcript.rs, src/random.rs), and the constant-size sigma protocols
// (src/nizk/mod.rs:27-405) commit to at most five scalars at a time.  The data-parallel work lives in kernels.cu.
#pragma once
#include <stdint.h>
#include <string.h>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>
#include "curve.cuh"
#include "field.cuh"
#include "host_fe51.hpp"
#include "../../include/spartan_b200.h"

namespace sp {

struct SpError : std::runtime_error {  // carries a C-ABI status code (include/spartan_b200.h)
  int code;
  SpError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

inline size_t log2_ceil(size_t x) { size_t l = 0; while (((size_t)1 << l) < x) l++; return l; }   // 0 for x <= 1
inline size_t next_pow2(size_t x) { return (size_t)1 << log2_ceil(x); }

// ------------------------------------------------------------------------------------------------ scalars
struct Fq {  // Montgomery-form element, same bytes as the reference's Scalar([u64;4])
  u256 m;
  Fq() : m(fq_zero()) {}
  explicit Fq(const u256& x) : m(x) {}
  static Fq zero() { return Fq(); }
  static Fq one() { return Fq(fq_one()); }
  static Fq from_u64(uint64_t x) { return Fq(fq_from_u64(x)); }
  static Fq from_bytes_wide(const uint8_t b[64]) { return Fq(fq_from_wide(bytes_to_u256(b), bytes_to_u256(b + 32))); }  // transcript.rs:26-30
  void to_bytes(uint8_t out[32]) const { u256_to_bytes(out, fq_from_mont(m)); }  // canonical LE (ristretto255.rs:419)
  u256 canonical() const { return fq_from_mont(m); }
  Fq operator+(const Fq& o) const { return Fq(fq_add(m, o.m)); }
  Fq operator-(const Fq& o) const { return Fq(fq_sub(m, o.m)); }
  Fq operator*(const Fq& o) const { return Fq(fq_mul(m, o.m)); }
  Fq operator-() const { return Fq(fq_neg(m)); }
  Fq& operator+=(const Fq& o) { m = fq_add(m, o.m); return *this; }
  Fq& operator-=(const Fq& o) { m = fq_sub(m, o.m); return *this; }
  Fq& operator*=(const Fq& o) { m = fq_mul(m, o.m); return *this; }
  bool operator==(const Fq& o) const { return fq_eq(m, o.m); }
  bool is_zero() const { return fq_is_zero(m); }
  Fq inv() const { return Fq(fq_inv(m)); }
  Fq sqr() const { return Fq(fq_sqr(m)); }
};
// Scalar::from_bytes acceptance test (ristretto255.rs:400-409): the little-endian integer must be < q
inline bool fq_bytes_canonical(const uint8_t b[32]) {
  static const uint8_t qb[32] = {0xed, 0xd3, 0xf5, 0x5c, 0x1a, 0x63, 0x12, 0x58, 0xd6, 0x9c, 0xf7, 0xa2, 0xde, 0xf9, 0xde, 0x14,
                                 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0x10};
  for (int i = 31; i >= 0; i--) {
    if (b[i] < qb[i]) return true;
    if (b[i] > qb[i]) return false;
  }
  return false;
}

// ------------------------------------------------------------------------------------------------ Keccak-f[1600] / STROBE-128 / Merlin
// merlin ^3.0.0 is a third-party crate (Cargo.toml:19); construction per the Merlin v1.0 / STROBE v1.0.2 specifications.
class Keccak {
 public:
  // Keccak-f[1600], lane-unrolled (theta / rho+pi / chi / iota per round); ~0.4 us per permutation on the host
  static void f1600(uint64_t A[25]) {
    static const uint64_t RC[24] = {0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808aULL, 0x8000000080008000ULL, 0x000000000000808bULL,
                                    0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL, 0x000000000000008aULL, 0x0000000000000088ULL,
                                    0x0000000080008009ULL, 0x000000008000000aULL, 0x000000008000808bULL, 0x800000000000008bULL, 0x8000000000008089ULL,
                                    0x8000000000008003ULL, 0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800aULL, 0x800000008000000aULL,
                                    0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};
#define SPK_ROL(v, n) (((v) << (n)) | ((v) >> (64 - (n))))
    uint64_t a00 = A[0], a01 = A[1], a02 = A[2], a03 = A[3], a04 = A[4], a05 = A[5], a06 = A[6], a07 = A[7], a08 = A[8], a09 = A[9], a10 = A[10], a11 = A[11],
             a12 = A[12], a13 = A[13], a14 = A[14], a15 = A[15], a16 = A[16], a17 = A[17], a18 = A[18], a19 = A[19], a20 = A[20], a21 = A[21], a22 = A[22],
             a23 = A[23], a24 = A[24];
    for (int rnd = 0; rnd < 24; rnd++) {
      uint64_t c0 = a00 ^ a05 ^ a10 ^ a15 ^ a20, c1 = a01 ^ a06 ^ a11 ^ a16 ^ a21, c2 = a02 ^ a07 ^ a12 ^ a17 ^ a22, c3 = a03 ^ a08 ^ a13 ^ a18 ^ a23,
               c4 = a04 ^ a09 ^ a14 ^ a19 ^ a24;
      uint64_t d0 = c4 ^ SPK_ROL(c1, 1), d1 = c0 ^ SPK_ROL(c2, 1), d2 = c1 ^ SPK_ROL(c3, 1), d3 = c2 ^ SPK_ROL(c4, 1), d4 = c3 ^ SPK_ROL(c0, 1);
      // rho + pi: b[y][2x+3y] = rot(a[x][y] ^ d[x], r[x][y]);  index = x + 5y
      uint64_t b00 = a00 ^ d0;
      uint64_t b10 = SPK_ROL(a01 ^ d1, 1), b20 = SPK_ROL(a02 ^ d2, 62), b05 = SPK_ROL(a03 ^ d3, 28), b15 = SPK_ROL(a04 ^ d4, 27);
      uint64_t b16 = SPK_ROL(a05 ^ d0, 36), b01 = SPK_ROL(a06 ^ d1, 44), b11 = SPK_ROL(a07 ^ d2, 6), b21 = SPK_ROL(a08 ^ d3, 55), b06 = SPK_ROL(a09 ^ d4, 20);
      uint64_t b07 = SPK_ROL(a10 ^ d0, 3), b17 = SPK_ROL(a11 ^ d1, 10), b02 = SPK_ROL(a12 ^ d2, 43), b12 = SPK_ROL(a13 ^ d3, 25), b22 = SPK_ROL(a14 ^ d4, 39);
      uint64_t b23 = SPK_ROL(a15 ^ d0, 41), b08 = SPK_ROL(a16 ^ d1, 45), b18 = SPK_ROL(a17 ^ d2, 15), b03 = SPK_ROL(a18 ^ d3, 21), b13 = SPK_ROL(a19 ^ d4, 8);
      uint64_t b14 = SPK_ROL(a20 ^ d0, 18), b24 = SPK_ROL(a21 ^ d1, 2), b09 = SPK_ROL(a22 ^ d2, 61), b19 = SPK_ROL(a23 ^ d3, 56), b04 = SPK_ROL(a24 ^ d4, 14);
      a00 = b00 ^ (~b01 & b02); a01 = b01 ^ (~b02 & b03); a02 = b02 ^ (~b03 & b04); a03 = b03 ^ (~b04 & b00); a04 = b04 ^ (~b00 & b01);
      a05 = b05 ^ (~b06 & b07); a06 = b06 ^ (~b07 & b08); a07 = b07 ^ (~b08 & b09); a08 = b08 ^ (~b09 & b05); a09 = b09 ^ (~b05 & b06);
      a10 = b10 ^ (~b11 & b12); a11 = b11 ^ (~b12 & b13); a12 = b12 ^ (~b13 & b14); a13 = b13 ^ (~b14 & b10); a14 = b14 ^ (~b10 & b11);
      a15 = b15 ^ (~b16 & b17); a16 = b16 ^ (~b17 & b18); a17 = b17 ^ (~b18 & b19); a18 = b18 ^ (~b19 & b15); a19 = b19 ^ (~b15 & b16);
      a20 = b20 ^ (~b21 & b22); a21 = b21 ^ (~b22 & b23); a22 = b22 ^ (~b23 & b24); a23 = b23 ^ (~b24 & b20); a24 = b24 ^ (~b20 & b21);
      a00 ^= RC[rnd];
    }
#undef SPK_ROL
    A[0] = a00; A[1] = a01; A[2] = a02; A[3] = a03; A[4] = a04; A[5] = a05; A[6] = a06; A[7] = a07; A[8] = a08; A[9] = a09; A[10] = a10; A[11] = a11; A[12] = a12;
    A[13] = a13; A[14] = a14; A[15] = a15; A[16] = a16; A[17] = a17; A[18] = a18; A[19] = a19; A[20] = a20; A[21] = a21; A[22] = a22; A[23] = a23; A[24] = a24;
  }
};

struct Shake256 {  // streaming SHAKE256 XOF (sha3's Shake256 + XofReader as used by commitments.rs:16-24): absorb once, squeeze in pieces
  uint64_t st[25];
  size_t pos = 0;
  Shake256(const uint8_t* in, size_t inlen) {
    memset(st, 0, sizeof st);
    uint8_t* sb = reinterpret_cast<uint8_t*>(st);
    const size_t rate = 136;
    while (inlen >= rate) { for (size_t i = 0; i < rate; i++) sb[i] ^= in[i]; Keccak::f1600(st); in += rate; inlen -= rate; }
    for (size_t i = 0; i < inlen; i++) sb[i] ^= in[i];
    sb[inlen] ^= 0x1f; sb[rate - 1] ^= 0x80;
    Keccak::f1600(st);
  }
  void squeeze(uint8_t* out, size_t n) {
    const uint8_t* sb = reinterpret_cast<const uint8_t*>(st);
    while (n) {
      if (pos == 136) { Keccak::f1600(st); pos = 0; }
      size_t m = n < 136 - pos ? n : 136 - pos;
      memcpy(out, sb + pos, m);
      out += m; n -= m; pos += m;
    }
  }
};

// Weight of equation e of proof i in a batch verification: from_bytes_wide(SHAKE256("spartan-b200/v1/batch-verify" || seed || LE64(i) || LE64(e))).
// Whoever knows the weights can make a bad proof pass, so `seed` must be fresh OS randomness on every call.
inline Fq batch_weight(const uint8_t seed[32], uint64_t i, uint64_t e) {
  static const char tag[] = "spartan-b200/v1/batch-verify";
  uint8_t in[sizeof(tag) - 1 + 32 + 16];
  memcpy(in, tag, sizeof(tag) - 1);
  memcpy(in + sizeof(tag) - 1, seed, 32);
  for (int b = 0; b < 8; b++) { in[sizeof(tag) - 1 + 32 + b] = (uint8_t)(i >> (8 * b)); in[sizeof(tag) - 1 + 40 + b] = (uint8_t)(e >> (8 * b)); }
  Shake256 x(in, sizeof in);
  uint8_t w[64];
  x.squeeze(w, 64);
  return Fq::from_bytes_wide(w);
}
// <eq(r, .), s> for the vector s of an inner-product argument with challenges u (s_i = prod_j u_j^-1 times u_j^2 for each bit j of i, the
// top bit first: bullet.rs:190-201): prod_j ((1 - r_j) u_j^-1 + r_j u_j), in O(lg n) instead of the n-term sum
inline Fq ipa_a_hat(const Fq* r, const Fq* u, const Fq* u_inv, size_t lg_n) {
  Fq acc = Fq::one();
  for (size_t j = 0; j < lg_n; j++) acc *= (Fq::one() - r[j]) * u_inv[j] + r[j] * u[j];
  return acc;
}

class Transcript {  // merlin::Transcript + ProofTranscript (transcript.rs:5-37)
 public:
  explicit Transcript(const std::string& label) {
    memset(st_, 0, sizeof st_);
    uint8_t* b = bytes();
    const uint8_t hdr[6] = {1, R + 2, 1, 0, 1, 96};
    memcpy(b, hdr, 6);
    memcpy(b + 6, "STROBEv1.0.2", 12);
    Keccak::f1600(st_);
    pos_ = 0; pos_begin_ = 0; cur_flags_ = 0;
    meta_ad((const uint8_t*)"Merlin v1.0", 11, false);
    append_message("dom-sep", (const uint8_t*)label.data(), label.size());
  }
  // The caller-owned `&mut Transcript` of the reference (lib.rs:339-347, :501-508) crosses the C ABI as merlin's whole STROBE-128 state:
  // the 200-byte Keccak state followed by pos, pos_begin and cur_flags (merlin/src/strobe.rs `Strobe128 { state, pos, pos_begin, cur_flags }`).
  static const size_t STATE_BYTES = 203;
  struct FromState {};
  Transcript(FromState, const uint8_t* in) {
    memcpy(st_, in, 200);
    pos_ = in[200]; pos_begin_ = in[201]; cur_flags_ = in[202];
    if (pos_ >= R || pos_begin_ > R) throw SpError(SP_ERR_INVALID_ARG, "spartan_b200: not a STROBE-128 transcript state (position out of range)");
  }
  void export_state(uint8_t* out) const { memcpy(out, st_, 200); out[200] = pos_; out[201] = pos_begin_; out[202] = cur_flags_; }
  void append_message(const char* label, const uint8_t* msg, size_t len) {
    uint8_t l4[4] = {(uint8_t)len, (uint8_t)(len >> 8), (uint8_t)(len >> 16), (uint8_t)(len >> 24)};
    meta_ad((const uint8_t*)label, strlen(label), false);
    meta_ad(l4, 4, true);
    ad(msg, len);
  }
  void append_message(const char* label, const char* msg) { append_message(label, (const uint8_t*)msg, strlen(msg)); }
  void append_u64(const char* label, uint64_t x) {
    uint8_t b[8];
    for (int i = 0; i < 8; i++) b[i] = (uint8_t)(x >> (8 * i));
    append_message(label, b, 8);
  }
  void challenge_bytes(const char* label, uint8_t* out, size_t n) {
    uint8_t l4[4] = {(uint8_t)n, (uint8_t)(n >> 8), (uint8_t)(n >> 16), (uint8_t)(n >> 24)};
    meta_ad((const uint8_t*)label, strlen(label), false);
    meta_ad(l4, 4, true);
    begin_op(FLAG_I | FLAG_A | FLAG_C, false);
    uint8_t* b = bytes();
    for (size_t i = 0; i < n; i++) { out[i] = b[pos_]; b[pos_] = 0; if (++pos_ == R) run_f(); }
  }
  // ProofTranscript
  void append_protocol_name(const char* name) { append_message("protocol-name", name); }
  void append_scalar(const char* label, const Fq& s) { uint8_t b[32]; s.to_bytes(b); append_message(label, b, 32); }
  void append_point(const char* label, const uint8_t p[32]) { append_message(label, p, 32); }
  Fq challenge_scalar(const char* label) { uint8_t b[64]; challenge_bytes(label, b, 64); return Fq::from_bytes_wide(b); }
  std::vector<Fq> challenge_vector(const char* label, size_t n) {
    std::vector<Fq> v(n);
    for (size_t i = 0; i < n; i++) v[i] = challenge_scalar(label);
    return v;
  }
  void append_scalars(const char* label, const Fq* v, size_t n) {  // AppendToTranscript for [Scalar], transcript.rs:49-57
    append_message(label, "begin_append_vector");
    for (size_t i = 0; i < n; i++) append_scalar(label, v[i]);
    append_message(label, "end_append_vector");
  }
  void append_scalars(const char* label, const std::vector<Fq>& v) { append_scalars(label, v.data(), v.size()); }
  // canonical 32-byte scalars already serialised (device-side to_bytes), same framing
  void append_scalar_bytes(const char* label, const uint8_t* canon32, size_t n) {
    append_message(label, "begin_append_vector");
    for (size_t i = 0; i < n; i++) append_message(label, canon32 + 32 * i, 32);
    append_message(label, "end_append_vector");
  }

 private:
  static const uint8_t R = 166, FLAG_I = 1, FLAG_A = 2, FLAG_C = 4, FLAG_M = 16, FLAG_K = 32;
  uint64_t st_[25];
  uint8_t pos_, pos_begin_, cur_flags_;
  uint8_t* bytes() { return reinterpret_cast<uint8_t*>(st_); }
  void run_f() {
    uint8_t* b = bytes();
    b[pos_] ^= pos_begin_;
    b[pos_ + 1] ^= 0x04;
    b[R + 1] ^= 0x80;
    Keccak::f1600(st_);
    pos_ = 0; pos_begin_ = 0;
  }
  void absorb(const uint8_t* d, size_t n) {
    uint8_t* b = bytes();
    while (n) {   // block-wise: up to the rate boundary at a time
      size_t room = (size_t)R - pos_, take = n < room ? n : room;
      uint8_t* dst = b + pos_;
      for (size_t i = 0; i < take; i++) dst[i] ^= d[i];
      pos_ = (uint8_t)(pos_ + take); d += take; n -= take;
      if (pos_ == R) run_f();
    }
  }
  void begin_op(uint8_t flags, bool more) {
    if (more) return;
    cur_flags_ = flags;
    uint8_t old_begin = pos_begin_;
    pos_begin_ = pos_ + 1;
    uint8_t hdr[2] = {old_begin, flags};
    absorb(hdr, 2);
    if ((flags & (FLAG_C | FLAG_K)) && pos_ != 0) run_f();
  }
  void meta_ad(const uint8_t* d, size_t n, bool more) { begin_op(FLAG_M | FLAG_A, more); absorb(d, n); }
  void ad(const uint8_t* d, size_t n) { begin_op(FLAG_A, false); absorb(d, n); }
};

class RandomTape {  // random.rs:6-28; the OsRng seed scalar is an explicit input here (SURVEY.md §8d)
 public:
  RandomTape(const std::string& name, const Fq& seed) : tape_(name) { tape_.append_scalar("init_randomness", seed); }
  // a tape is a merlin transcript: the caller's tape crosses the C ABI as its STROBE state, like a transcript
  explicit RandomTape(const Transcript& state) : tape_(state) {}
  const Transcript& state() const { return tape_; }
  Fq random_scalar(const char* label) { return tape_.challenge_scalar(label); }
  std::vector<Fq> random_vector(const char* label, size_t n) { return tape_.challenge_vector(label, n); }

 private:
  Transcript tape_;
};

// ------------------------------------------------------------------------------------------------ small host commitments
typedef uint8_t CompressedPoint[32];
struct Cp {  // CompressedGroup (group.rs:7)
  uint8_t b[32];
  bool operator==(const Cp& o) const { return memcmp(b, o.b, 32) == 0; }
};
inline Cp compress(const hge& p) { Cp c; uint8_t o[1][32]; hge_encode_n<1>(&p, o); memcpy(c.b, o[0], 32); return c; }
inline Cp compress(const ge& p) { return compress(to_hge(p)); }
// two encodings at once: the two 252-squaring exponentiations run in lockstep, so the CPU overlaps their dependency chains
inline void compress2(const hge& p, const hge& q, Cp& cp, Cp& cq) {
  hge pq[2] = {p, q};
  uint8_t o[2][32];
  hge_encode_n<2>(pq, o);
  memcpy(cp.b, o[0], 32); memcpy(cq.b, o[1], 32);
}
inline void compress2(const ge& p, const ge& q, Cp& cp, Cp& cq) { compress2(to_hge(p), to_hge(q), cp, cq); }

// 8-bit signed fixed-base windows for one generator: 32 windows x 128 affine-niels entries (copied from the device table)
struct HostBaseTable {
  std::vector<hniels> e;  // [w*128 + d-1], radix-2^51 limbs (host_fe51.hpp)
};
inline void host_fixed_mul_acc(hge& acc, const HostBaseTable& tb, const Fq& k) {
  if (k.is_zero()) return;
  u256 c = k.canonical();
  uint32_t carry = 0;
  for (int w = 0; w < 32; w++) {
    uint32_t v = ((c.v[w >> 2] >> ((w & 3) * 8)) & 0xffu) + carry;
    int d;
    if (v > 128u) { d = (int)v - 256; carry = 1; } else { d = (int)v; carry = 0; }
    if (d == 0) continue;
    int ad = d < 0 ? -d : d;
    acc = hge_madd(acc, tb.e[(size_t)w * 128 + ad - 1], d < 0);
  }
}

}  // namespace sp
