// spartan_b200 — CPU-only test hooks.  Compiled with -DSP_FORCE_PORTABLE so the *device* formulation of the field / curve
// arithmetic (32-bit limbs, the code the kernels run) executes on the host and can be checked against the oracle without a GPU.
// Not linked into libspartan_b200.so.
#include "host.hpp"
#include "engine.hpp"
#include "wire.hpp"
#include "snark.hpp"
using namespace sp;

namespace sp { void shake256(uint8_t* out, size_t outlen, const uint8_t* in, size_t inlen); }

static u256 in256(const uint8_t* b) { u256 r; memcpy(&r, b, 32); return r; }
static void out256(uint8_t* b, const u256& x) { memcpy(b, &x, 32); }

#include "deflate.cpp"   // host-only translation unit, pulled in here so the CPU tests can call it without the CUDA library

extern "C" {

// SparkDims of SparseMatPolyCommitmentGens::new(x, y, nz, b): out = v_ops, v_mem, v_derefs, n_ops, n_mem, n_der
void sph_spark_dims(size_t x, size_t y, size_t nz, size_t b, size_t out[6]) {
  const sp::SparkDims d(x, y, nz, b);
  const size_t v[6] = {d.v_ops, d.v_mem, d.v_derefs, d.n_ops, d.n_mem, d.n_der};
  for (int i = 0; i < 6; i++) out[i] = v[i];
}
// entries per tile of the segmented matrix products (kernels_inst.cu: spmat_products)
size_t sph_spmat_tile(void) { return sp::dev::SPMAT_TILE; }
// the carry layout of spmat_products for `total` entries: out = n1, n2, offsets of cv1, cv2, ck1, ck2, scratch bytes
void sph_spmat_carries(size_t total, size_t out[7]) {
  const sp::dev::SpmatCarries L(total);
  const size_t v[7] = {L.n1, L.n2, L.cv1, L.cv2, L.ck1, L.ck2, L.bytes};
  for (int i = 0; i < 7; i++) out[i] = v[i];
}
// R1CSShape digest compressor: zlib stream of miniz level 6 (deflate.cpp); returns the length (out must hold len + len/8 + 128 bytes)
size_t spt_zlib6(const uint8_t* in, size_t len, uint8_t* out) {
  std::vector<uint8_t> z = sp::miniz_zlib_level6(in, len);
  memcpy(out, z.data(), z.size());
  return z.size();
}
int spt_portable(void) {
#if SP_HOST_FAST
  return 0;
#else
  return 1;
#endif
}
void spt_fq_mul(const uint8_t* a, const uint8_t* b, uint8_t* r) { out256(r, fq_mul(in256(a), in256(b))); }
// the constant-multiplier fold of the sumcheck kernels (portable specification of fq_fold_const_ptx): table built from r, then a0 + r*(a1-a0)
void spt_fq_fold_const(const uint8_t* a0, const uint8_t* a1, const uint8_t* r, uint8_t* out) {
  FqConst rc = fq_const_table(in256(r));
  out256(out, fq_fold_const(in256(a0), in256(a1), rc));
}
void spt_fq_add(const uint8_t* a, const uint8_t* b, uint8_t* r) { out256(r, fq_add(in256(a), in256(b))); }
void spt_fq_sub(const uint8_t* a, const uint8_t* b, uint8_t* r) { out256(r, fq_sub(in256(a), in256(b))); }
void spt_fq_inv(const uint8_t* a, uint8_t* r) { out256(r, fq_inv(in256(a))); }
void spt_fq_from_wide(const uint8_t* w, uint8_t* r) { out256(r, fq_from_wide(in256(w), in256(w + 32))); }
void spt_fq_from_mont(const uint8_t* a, uint8_t* r) { out256(r, fq_from_mont(in256(a))); }
void spt_fq_from_u64(uint64_t x, uint8_t* r) { out256(r, fq_from_u64(x)); }
// Fp: inputs / outputs as canonical little-endian integers
void spt_fp_mul(const uint8_t* a, const uint8_t* b, uint8_t* r) { out256(r, fp_canon(fp_mul(in256(a), in256(b)))); }
void spt_fp_add(const uint8_t* a, const uint8_t* b, uint8_t* r) { out256(r, fp_canon(fp_add(in256(a), in256(b)))); }
void spt_fp_sub(const uint8_t* a, const uint8_t* b, uint8_t* r) { out256(r, fp_canon(fp_sub(in256(a), in256(b)))); }
void spt_fp_inv(const uint8_t* a, uint8_t* r) { out256(r, fp_canon(fp_inv(in256(a)))); }
void spt_fp_canon(const uint8_t* a, uint8_t* r) { out256(r, fp_canon(in256(a))); }
// group
int spt_decode_encode(const uint8_t* in32, uint8_t* out32) {
  ge g;
  if (!ristretto_decode(g, in256(in32))) return 0;
  out256(out32, ristretto_encode(g));
  return 1;
}
void spt_from_uniform(const uint8_t* in64, uint8_t* out32) { out256(out32, ristretto_encode(ristretto_from_uniform(in256(in64), in256(in64 + 32)))); }
int spt_add(const uint8_t* a32, const uint8_t* b32, uint8_t* out32) {
  ge a, b;
  if (!ristretto_decode(a, in256(a32)) || !ristretto_decode(b, in256(b32))) return 0;
  out256(out32, ristretto_encode(ge_add(a, b)));
  return 1;
}
int spt_dbl(const uint8_t* a32, uint8_t* out32) {
  ge a;
  if (!ristretto_decode(a, in256(a32))) return 0;
  out256(out32, ristretto_encode(ge_dbl(a)));
  return 1;
}
// compress2 (host.hpp): two encodings with interleaved exponentiations, of a+b and 2a (non-trivial Z)
int spt_compress2(const uint8_t* a32, const uint8_t* b32, uint8_t* out64) {
  ge a, b;
  if (!ristretto_decode(a, in256(a32)) || !ristretto_decode(b, in256(b32))) return 0;
  sp::Cp c1, c2;
  sp::compress2(ge_add(a, b), ge_dbl(a), c1, c2);   // the ge overload converts to radix 2^51 and encodes there
  memcpy(out64, c1.b, 32); memcpy(out64 + 32, c2.b, 32);
  return 1;
}
int spt_scalarmul(const uint8_t* k_canonical, const uint8_t* a32, uint8_t* out32) {
  ge a;
  if (!ristretto_decode(a, in256(a32))) return 0;
  out256(out32, ristretto_encode(ge_scalarmul(in256(k_canonical), a)));
  return 1;
}
// the fixed-base window path used by msm_rows / host_commit: build the 32x128 niels table of a point and multiply through it
int spt_fixed_base_mul(const uint8_t* k_mont, const uint8_t* a32, uint8_t* out32) {
  ge P;
  if (!ristretto_decode(P, in256(a32))) return 0;
  HostBaseTable tb;
  tb.e.resize(32 * 128);
  for (int w = 0; w < 32; w++) {
    ge acc = P;
    for (int d = 0; d < 128; d++) { tb.e[(size_t)w * 128 + d] = to_hniels(ge_to_niels(acc)); acc = ge_add(acc, P); }
    for (int k = 0; k < 8; k++) P = ge_dbl(P);
  }
  hge acc = hge_identity();
  Fq k; memcpy(&k.m, k_mont, 32);
  host_fixed_mul_acc(acc, tb, k);
  Cp c = compress(acc);
  memcpy(out32, c.b, 32);
  return 1;
}
// signed W-bit recoding of the row MSM (curve.cuh signed_digit) of a canonical scalar; returns the window count
int spt_signed_digits(const uint8_t* k_canonical, int wbits, int* out) {
  const u256 k = in256(k_canonical);
  const int nwin = (253 + wbits - 1) / wbits;
  uint32_t carry = 0;
  for (int w = 0; w < nwin; w++) out[w] = signed_digit(k, w, wbits, carry);
  return nwin;
}
// the row MSM's arithmetic on one row: per-window sums S_w = sum_j d_{j,w} * P_j (|d| * P_j standing in for the row-table entry), then
// out = sum_w 2^(W*w) S_w by Horner's rule with W doublings per window.  k_mont: n Montgomery scalars, pts: n encodings
int spt_row_msm(const uint8_t* k_mont, const uint8_t* pts, size_t n, int wbits, uint8_t* out32) {
  const int nwin = (253 + wbits - 1) / wbits;
  std::vector<ge> P(n);
  for (size_t j = 0; j < n; j++) if (!ristretto_decode(P[j], in256(pts + 32 * j))) return 0;
  std::vector<ge> S(nwin, ge_identity());
  for (size_t j = 0; j < n; j++) {
    const u256 km = in256(k_mont + 32 * j);
    if (fq_is_zero(km)) continue;
    const u256 k = fq_from_mont(km);
    uint32_t carry = 0;
    for (int w = 0; w < nwin; w++) {
      const int d = signed_digit(k, w, wbits, carry);
      if (d == 0) continue;
      u256 ad = fq_zero();
      ad.v[0] = (uint32_t)(d < 0 ? -d : d);
      const ge e = ge_scalarmul(ad, P[j]);
      S[w] = ge_add(S[w], d < 0 ? ge_neg(e) : e);
    }
  }
  ge acc = S[nwin - 1];
  for (int w = nwin - 2; w >= 0; w--) {
    for (int i = 0; i < wbits; i++) acc = ge_dbl(acc);
    acc = ge_add(acc, S[w]);
  }
  out256(out32, ristretto_encode(acc));
  return 1;
}
// radix-2^51 host arithmetic (host_fe51.hpp) against the 8x32-limb field code: mul, sqr, add, sub, freeze on raw 256-bit inputs
void spt_fe51_ops(const uint8_t* a32, const uint8_t* b32, uint8_t* out160) {
  fe51 a = fe_from_u256(in256(a32)), b = fe_from_u256(in256(b32));
  fe_to_bytes(out160, fe_mul(a, b));
  fe_to_bytes(out160 + 32, fe_sqr(a));
  fe_to_bytes(out160 + 64, fe_add(a, b));
  fe_to_bytes(out160 + 96, fe_sub(a, b));
  fe_to_bytes(out160 + 128, fe_mul(fe_sub(fe_add(a, b), fe_neg(a)), fe_add(fe_add(a, a), fe_add(b, b))));   // lazily-reduced operands
}
// hge (host_fe51.hpp): k*A by signed 4-bit windows, A+B, 2A -> encodings
int spt_hge_ops(const uint8_t* k_canonical, const uint8_t* a32, const uint8_t* b32, uint8_t* out96) {
  ge a, b;
  if (!ristretto_decode(a, in256(a32)) || !ristretto_decode(b, in256(b32))) return 0;
  Cp c1 = compress(hge_scalarmul(in256(k_canonical), to_hge(a)));
  Cp c2, c3;
  compress2(hge_add(to_hge(a), to_hge(b)), hge_dbl(to_hge(a)), c2, c3);
  memcpy(out96, c1.b, 32); memcpy(out96 + 32, c2.b, 32); memcpy(out96 + 64, c3.b, 32);
  return 1;
}
// transcript
void spt_transcript_kat(uint8_t* out32) {
  Transcript t("test protocol");
  t.append_message("some label", (const uint8_t*)"some data", 9);
  t.challenge_bytes("challenge", out32, 32);
}
void spt_transcript_run(const uint8_t* label, size_t llen, const uint8_t* msgs, const size_t* lens, size_t nmsgs, uint8_t* out64) {
  Transcript t(std::string((const char*)label, llen));
  size_t off = 0;
  for (size_t i = 0; i < nmsgs; i++) { t.append_message("m", msgs + off, lens[i]); off += lens[i]; }
  t.challenge_bytes("c", out64, 64);
}
void spt_shake256(uint8_t* out, size_t outlen, const uint8_t* in, size_t inlen) { sp::shake256(out, outlen, in, inlen); }
// batch verification: the weight of equation e of proof i (batch_weight), Montgomery limbs out
void spt_batch_weight(const uint8_t* seed32, uint64_t i, uint64_t e, uint8_t* out) { Fq w = batch_weight(seed32, i, e); memcpy(out, &w.m, 32); }
// <eq(r, .), s> of an inner-product argument two ways: ipa_a_hat's product (out) and the n-term sum over the vector s that
// DotProductProofLog::verify builds (out + 32); r, u: lg_n Montgomery scalars each
void spt_ipa_a_hat(const uint8_t* r_mont, const uint8_t* u_mont, size_t lg_n, uint8_t* out64) {
  std::vector<Fq> r(lg_n), u(lg_n), u_inv(lg_n), u_sq(lg_n);
  for (size_t j = 0; j < lg_n; j++) { memcpy(&r[j].m, r_mont + 32 * j, 32); memcpy(&u[j].m, u_mont + 32 * j, 32); }
  Fq allinv = Fq::one();
  for (size_t j = 0; j < lg_n; j++) { u_inv[j] = u[j].inv(); allinv *= u_inv[j]; u_sq[j] = u[j] * u[j]; }
  const Fq fast = ipa_a_hat(r.data(), u.data(), u_inv.data(), lg_n);
  // the reference's loop (bullet.rs:190-201): s[i] = s[i - 2^k] * u_sq[lg_n - 1 - k], k = floor(log2 i)
  const size_t n = (size_t)1 << lg_n;
  std::vector<Fq> s(n);
  s[0] = allinv;
  for (size_t i = 1; i < n; i++) {
    size_t lg_i = 0;
    while (((size_t)2 << lg_i) <= i) lg_i++;
    s[i] = s[i - ((size_t)1 << lg_i)] * u_sq[(lg_n - 1) - lg_i];
  }
  // a = eq(r, .) (EqPolynomial::evals: r[0] is the top bit of the index)
  Fq slow = Fq::zero();
  for (size_t i = 0; i < n; i++) {
    Fq a = Fq::one();
    for (size_t j = 0; j < lg_n; j++) a *= ((i >> (lg_n - 1 - j)) & 1) ? r[j] : Fq::one() - r[j];
    slow += a * s[i];
  }
  memcpy(out64, &fast.m, 32);
  memcpy(out64 + 32, &slow.m, 32);
}
// wire format (wire.hpp): parse one input with Reader under the status code the library uses for it, re-encode it with Writer.  kind 0: a NIZK
// proof, 1: a SNARK proof, 2: a ComputationCommitment.  *out_len: the capacity of out, then the length of the re-encoding.
int spt_wire_roundtrip(int kind, const uint8_t* in, size_t len, uint8_t* out, size_t* out_len) {
  try {
    std::vector<uint8_t> b;
    if (kind == 0) b = to_bincode(from_bincode<NizkProof>(in, len, SP_ERR_VERIFY, "proof"));
    else if (kind == 1) b = to_bincode(from_bincode<SnarkProof>(in, len, SP_ERR_VERIFY, "proof"));
    else if (kind == 2) b = to_bincode(from_bincode<ComputationCommitment>(in, len, SP_ERR_INVALID_ARG, "computation commitment"));
    else return SP_ERR_INVALID_ARG;
    if (b.size() > *out_len) return SP_ERR_INVALID_ARG;
    memcpy(out, b.data(), b.size());
    *out_len = b.size();
    return SP_OK;
  } catch (const SpError& e) { return e.code; }
}
}

namespace sp {
void shake256(uint8_t* out, size_t outlen, const uint8_t* in, size_t inlen) {
  uint64_t st[25];
  memset(st, 0, sizeof st);
  uint8_t* sb = reinterpret_cast<uint8_t*>(st);
  const size_t rate = 136;
  while (inlen >= rate) { for (size_t i = 0; i < rate; i++) sb[i] ^= in[i]; Keccak::f1600(st); in += rate; inlen -= rate; }
  for (size_t i = 0; i < inlen; i++) sb[i] ^= in[i];
  sb[inlen] ^= 0x1f; sb[rate - 1] ^= 0x80;
  Keccak::f1600(st);
  while (outlen) {
    size_t n = outlen < rate ? outlen : rate;
    memcpy(out, sb, n); out += n; outlen -= n;
    if (outlen) Keccak::f1600(st);
  }
}
}
