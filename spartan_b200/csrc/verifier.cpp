// spartan_b200 — NIZK::verify / SNARK::verify (SURVEY.md §8(f) row 4): the verifier side of the reference, so that a caller of this library
// can check the proofs it produces (or proofs produced by the reference: the wire format is bincode's).
//
// Follows /root/reference/src function by function: lib.rs:423-465 (SNARK::verify), :549-591 (NIZK::verify), r1csproof.rs:351-489,
// sumcheck.rs:27-62,84-179, nizk/mod.rs:54-75,118-143,245-290,372-405,527-583, nizk/bullet.rs:137-225, dense_mlpoly.rs:367-404,
// product_tree.rs:385-485, sparse_mlpoly.rs:151-211,837-1019,1228-1305,1356-1416,1516-1557.
// Every group equation a protocol step tests goes through a Checker (DESIGN.md "deferred checks"):
//   Immediate  evaluates it on the spot (host radix 2^51, generator-vector MSMs on the device) and throws at the first one that fails.  The
//              single-proof entries use it; it also gives a rejected proof of a batch its exact status and message.
//   Deferred   adds it, weighted by a fresh random scalar, to the proof's accumulator; one device pass over a whole batch then tests every
//              proof's sum against the identity (verify_batch below).
// Scalar checks and the group operations whose results the transcript absorbs run the same in both modes.  Failures map to
// ProofVerifyError::{InternalError, DecompressionError}.
#include <algorithm>
#include <unordered_map>
#include "../../include/spartan_b200.h"
#include "snark.hpp"

namespace sp {

namespace {

struct Reject : SpError { explicit Reject(const std::string& what) : SpError(SP_ERR_VERIFY, "proof rejected: " + what) {} };
struct BadPoint : SpError { explicit BadPoint(const std::string& what) : SpError(SP_ERR_DECOMPRESS, "proof rejected: " + what + " does not decompress") {} };

// ---- group helpers (host, radix 2^51)
hge unpack(const Cp& c, const char* what) {
  ge g;
  if (!ristretto_decode(g, bytes_to_u256(c.b))) throw BadPoint(what);
  return to_hge(g);
}
hge mul(const hge& p, const Fq& k) { return hge_scalarmul(k.canonical(), p); }
hge neg(const hge& p) { hge q = p; q.X = fe_neg(p.X); q.T = fe_neg(p.T); return q; }
bool same(const hge& a, const hge& b) { return compress(a) == compress(b); }
ge to_ge(const hge& p) {
  ge g;
  uint8_t b[32];
  fe_to_bytes(b, p.X); g.X = bytes_to_u256(b);
  fe_to_bytes(b, p.Y); g.Y = bytes_to_u256(b);
  fe_to_bytes(b, p.Z); g.Z = bytes_to_u256(b);
  fe_to_bytes(b, p.T); g.T = bytes_to_u256(b);
  return g;
}

// ---- group equations: sum lhs == sum rhs, each side a list of terms k * (a point of the proof | a point the verifier derived | a generator)
struct GTerm {
  Fq k;
  const Cp* cp = nullptr; const char* what = nullptr;   // a point of the proof, named for the DecompressionError message
  hge h;                                                 // else (cp, set null) a point the verifier derived
  const GenSet* set = nullptr; size_t base = 0;          // else generator `base` of `set`
};
GTerm P(const Fq& k, const Cp& c, const char* what) { GTerm t; t.k = k; t.cp = &c; t.what = what; return t; }
GTerm H(const Fq& k, const hge& h) { GTerm t; t.k = k; t.h = h; return t; }
GTerm G(const Fq& k, const CommitKey& key, size_t base) { GTerm t; t.k = k; t.set = key.set; t.base = base; return t; }
GTerm scaled(GTerm t, const Fq& k) { t.k = t.k * k; return t; }
typedef std::vector<GTerm> Side;
// scale * <s, gens_n.G> for the vector s of an inner-product argument: s_i = allinv * prod_{bit b of i} u_sq[lg_n - 1 - b]
struct IpaS {
  const CommitKey* gens_n;
  size_t lg_n;
  std::vector<Fq> u_sq;
  Fq allinv, scale;
};
dev::IpaSRow srow_item(u256* row, const IpaS& s, uint32_t add) {
  dev::IpaSRow it;
  memset(&it, 0, sizeof it);
  it.row = row; it.lg_n = (uint32_t)s.lg_n; it.add = add; it.allinv = s.allinv.m; it.scale = s.scale.m;
  for (size_t j = 0; j < s.lg_n; j++) it.u_sq[j] = s.u_sq[j].m;
  return it;
}

class Checker {
 public:
  explicit Checker(Ctx& c) : ctx(c) {}
  virtual ~Checker() {}
  Ctx& ctx;
  virtual hge point(const Cp& c, const char* what) = 0;   // a point of the proof, decompressed
  // sum lhs == sum rhs (+ the IPA term s on the right), else the proof is rejected with `what`
  virtual void equal(const Side& lhs, const Side& rhs, const char* what, const IpaS* s = nullptr) = 0;
};

class Immediate : public Checker {
 public:
  using Checker::Checker;
  hge point(const Cp& c, const char* what) override { return unpack(c, what); }
  void equal(const Side& lhs, const Side& rhs, const char* what, const IpaS* s) override {
    hge g_hat;
    if (s) g_hat = ipa_g_hat(*s);
    FineTimer ft(ctx, "verify.group_checks");
    hge l = eval(lhs), r = eval(rhs);
    if (s) r = hge_add(r, mul(g_hat, s->scale));
    if (!same(l, r)) throw Reject(what);
  }

 private:
  hge eval(const Side& side) {
    hge acc = hge_identity();
    for (const GTerm& t : side) {
      if (t.set) { host_fixed_mul_acc(acc, t.set->tab(t.base), t.k); continue; }
      const hge p = t.cp ? unpack(*t.cp, t.what) : t.h;
      acc = hge_add(acc, t.k == Fq::one() ? p : mul(p, t.k));
    }
    return acc;
  }
  // <s, G> through the device: s built by k_ipa_srow, summed against the generator tables
  hge ipa_g_hat(const IpaS& s) {
    FineTimer ft(ctx, "verify.ipa_g_hat");
    const size_t n = (size_t)1 << s.lg_n;
    DevBuf<u256> d(n);
    DevBuf<dev::IpaSRow> d_it(1);
    IpaS one = s;
    one.scale = Fq::one();
    const dev::IpaSRow it = srow_item(d.p, one, 0);
    dev::h2d(d_it.p, &it, sizeof it, ctx.stream);
    dev::ipa_srow(d_it.p, 1, (uint32_t)s.lg_n, ctx.stream);
    std::vector<Cp> out;
    commit_rows_and_compress(ctx, *s.gens_n, d.p, n, 1, n, nullptr, out);
    return unpack(out[0], "device MSM result");
  }
};

// one proof's deferred equations, weighted and summed: the proof is accepted when the sum is the identity
struct ProofAcc {
  std::vector<Fq> k;                              // variable-base part: k[j] * pts[j]
  std::vector<ge> pts;
  std::map<const GenSet*, std::vector<Fq>> rows;  // fixed-base part: one row of generator scalars per generator set
  std::vector<IpaS> ipa;                          // IPA terms, added into the rows on the device
};
struct CpHash { size_t operator()(const Cp& c) const { size_t x; memcpy(&x, c.b, sizeof x); return x; } };
typedef std::unordered_map<Cp, ge, CpHash> PointTable;   // the decompressed points of a batch's proofs

class Deferred : public Checker {
 public:
  Deferred(Ctx& c, const PointTable& pts, const uint8_t* seed, uint64_t proof, ProofAcc& acc) : Checker(c), pts_(pts), seed_(seed), proof_(proof), acc_(acc) {}
  hge point(const Cp& c, const char* what) override { return to_hge(lookup(c, what)); }
  void equal(const Side& lhs, const Side& rhs, const char*, const IpaS* s) override {
    const Fq rho = batch_weight(seed_, proof_, eq_++);
    add(lhs, rho);
    add(rhs, -rho);
    if (s) { acc_.ipa.push_back(*s); acc_.ipa.back().scale = -rho * s->scale; }
  }

 private:
  const PointTable& pts_;
  const uint8_t* seed_;
  uint64_t proof_, eq_ = 0;
  ProofAcc& acc_;
  ge lookup(const Cp& c, const char* what) {
    auto it = pts_.find(c);
    if (it != pts_.end()) return it->second;
    ge g;
    if (!ristretto_decode(g, bytes_to_u256(c.b))) throw BadPoint(what);
    return g;
  }
  void add(const Side& side, const Fq& w) {
    for (const GTerm& t : side) {
      const Fq k = w * t.k;
      if (t.set) {
        std::vector<Fq>& row = acc_.rows[t.set];
        if (row.empty()) row.assign(t.set->nbases, Fq::zero());
        row[t.base] += k;
      } else {
        acc_.k.push_back(k);
        acc_.pts.push_back(t.cp ? lookup(*t.cp, t.what) : to_ge(t.h));
      }
    }
  }
};

// The final pass of a batch: for every accumulator, its fixed-base rows (one msm_rows launch per generator set, one row per proof, with the IPA
// vectors added in by k_ipa_srow) plus its variable-base segment (one segmented MSM), compressed; ok[i] = the sum is the identity
std::vector<bool> deferred_final(Ctx& ctx, const std::vector<const ProofAcc*>& accs) {
  const size_t K = accs.size();
  std::vector<bool> ok(K, true);
  if (!K) return ok;
  std::vector<const GenSet*> sets;
  for (const ProofAcc* a : accs) {
    for (auto& r : a->rows) if (std::find(sets.begin(), sets.end(), r.first) == sets.end()) sets.push_back(r.first);
    for (auto& s : a->ipa) if (std::find(sets.begin(), sets.end(), s.gens_n->set) == sets.end()) sets.push_back(s.gens_n->set);
  }
  // variable-base segments
  size_t n = 0;
  for (const ProofAcc* a : accs) n += a->k.size();
  if (n >= ((size_t)1 << 32)) throw SpError(SP_ERR_INVALID_ARG, "verify_batch: more than 2^32 - 1 variable-base terms in one batch: split it");
  std::vector<uint32_t> seg(K + 1, 0);
  for (size_t i = 0; i < K; i++) seg[i + 1] = seg[i] + (uint32_t)accs[i]->k.size();
  std::vector<ge> pts(n);
  std::vector<u256> sc(n);
  for (size_t i = 0; i < K; i++)
    for (size_t j = 0; j < accs[i]->k.size(); j++) { pts[seg[i] + j] = accs[i]->pts[j]; sc[seg[i] + j] = accs[i]->k[j].canonical(); }
  DevBuf<ge> d_pts(std::max<size_t>(n, 1)), d_tmp(std::max<size_t>(n, 1)), total(K), part(K);
  DevBuf<u256> d_sc(std::max<size_t>(n, 1));
  DevBuf<uint32_t> d_seg(K + 1);
  dev::h2d(d_pts.p, pts.data(), n * sizeof(ge), ctx.stream);
  dev::h2d(d_sc.p, sc.data(), n * sizeof(u256), ctx.stream);
  dev::h2d(d_seg.p, seg.data(), (K + 1) * sizeof(uint32_t), ctx.stream);
  dev::msm_var_segmented(total.p, d_pts.p, d_sc.p, d_seg.p, K, n, d_tmp.p, ctx.stream);
  // fixed-base rows
  std::vector<std::vector<Fq>> host_rows(sets.size());
  std::vector<DevBuf<u256>> d_rows(sets.size());
  std::vector<DevBuf<dev::IpaSRow>> d_items(sets.size());
  for (size_t si = 0; si < sets.size(); si++) {
    const GenSet* gs = sets[si];
    const size_t R = gs->nbases;
    std::vector<Fq>& M = host_rows[si];
    M.assign(K * R, Fq::zero());
    d_rows[si].alloc(K * R);
    // the m-th IPA of every proof goes into launch m: the IPAs of one proof add into the same row, those of one launch must not
    std::vector<std::vector<dev::IpaSRow>> items;
    std::vector<uint32_t> max_lg;
    for (size_t i = 0; i < K; i++) {
      auto it = accs[i]->rows.find(gs);
      if (it != accs[i]->rows.end()) std::copy(it->second.begin(), it->second.end(), M.begin() + i * R);
      size_t m = 0;
      for (const IpaS& s : accs[i]->ipa) {
        if (s.gens_n->set != gs) continue;
        if (items.size() <= m) { items.emplace_back(); max_lg.push_back(0); }
        items[m].push_back(srow_item(d_rows[si].p + i * R + s.gens_n->off, s, 1));
        max_lg[m] = std::max(max_lg[m], (uint32_t)s.lg_n);
        m++;
      }
    }
    dev::h2d(d_rows[si].p, M.data(), K * R * sizeof(u256), ctx.stream);
    size_t nitems = 0;
    for (auto& v : items) nitems += v.size();
    d_items[si].alloc(std::max<size_t>(nitems, 1));
    for (size_t m = 0, at = 0; m < items.size(); at += items[m].size(), m++) {
      dev::h2d(d_items[si].p + at, items[m].data(), items[m].size() * sizeof(dev::IpaSRow), ctx.stream);
      dev::ipa_srow(d_items[si].p + at, items[m].size(), max_lg[m], ctx.stream);
    }
    ctx.ensure_scratch(dev::msm_scratch_bytes(K, R) + 64);
    dev::msm_rows(part.p, gs->table.p, gs->wbits, gs->rows(), d_rows[si].p, R, K, R, nullptr, 0, ctx.scratch.p, ctx.stream);
    dev::add_points(total.p, part.p, K, ctx.stream);
  }
  DevBuf<uint8_t> comp(32 * K);
  dev::compress_batch(comp.p, total.p, K, ctx.stream);
  std::vector<uint8_t> h(32 * K);
  dev::d2h(h.data(), comp.p, 32 * K, ctx.stream);
  ctx.sync();
  for (size_t i = 0; i < K; i++) ok[i] = std::all_of(h.begin() + 32 * i, h.begin() + 32 * (i + 1), [](uint8_t b) { return b == 0; });
  return ok;
}

// sum_i s_i * P_i for proof-supplied points: bucket MSM on the device, a plain loop when there are only a few
hge msm_points(Checker& chk, const std::vector<Cp>& pts, const std::vector<Fq>& s, const char* what) {
  Ctx& ctx = chk.ctx;
  FineTimer ft(ctx, "verify.c_lz");
  const size_t n = pts.size();
  if (n <= 8) {
    hge acc = hge_identity();
    for (size_t i = 0; i < n; i++) acc = hge_add(acc, mul(chk.point(pts[i], what), s[i]));
    return acc;
  }
  DevBuf<uint8_t> d_in(32 * n);
  DevBuf<ge> g(n), out(1);
  DevBuf<int> ok(n);
  DevBuf<ge_niels> nl(n);
  DevBuf<u256> d_s(n);
  dev::h2d(d_in.p, pts.data(), 32 * n, ctx.stream);
  dev::decompress_batch(g.p, ok.p, d_in.p, n, ctx.stream);
  std::vector<int> h_ok(n);
  dev::d2h(h_ok.data(), ok.p, sizeof(int) * n, ctx.stream);
  ctx.upload(d_s.p, s.data(), n);   // synchronises
  for (size_t i = 0; i < n; i++) if (!h_ok[i]) throw BadPoint(what);
  dev::points_to_niels(nl.p, g.p, n, ctx.stream);
  dev::PipPlan plan = dev::pip_plan(n, 0);
  DevBuf<uint8_t> scratch(dev::pip_scratch_bytes(plan));
  dev::msm_var(out.p, nl.p, d_s.p, plan, scratch.p, ctx.stream);
  ge r;
  dev::d2h(&r, out.p, sizeof(ge), ctx.stream);
  ctx.sync();
  return to_hge(r);
}

Fq eq_eval(const std::vector<Fq>& a, const std::vector<Fq>& b) {   // EqPolynomial::evaluate (dense_mlpoly.rs:57-66)
  Fq acc = Fq::one();
  for (size_t i = 0; i < a.size(); i++) acc *= a[i] * b[i] + (Fq::one() - a[i]) * (Fq::one() - b[i]);
  return acc;
}

// ---- sigma protocols
void knowledge_verify(Checker& chk, const KnowledgeProof& p, const CommitKey& g, Transcript& T, const Cp& C) {   // nizk/mod.rs:54-75
  T.append_protocol_name("knowledge proof");
  T.append_point("C", C.b);
  T.append_point("alpha", p.alpha.b);
  Fq c = T.challenge_scalar("c");
  chk.equal({G(p.z1, g, g.off), G(p.z2, g, g.h)}, {P(c, C, "C"), P(Fq::one(), p.alpha, "alpha")}, "KnowledgeProof");
}
// C1: a point the verifier derived (hge and its encoding), C2: a point of the proof
void equality_verify(Checker& chk, const EqualityProof& p, const CommitKey& g, Transcript& T, const hge& C1, const Cp& C1_c, const Cp& C2) {   // nizk/mod.rs:118-143
  T.append_protocol_name("equality proof");
  T.append_point("C1", C1_c.b);
  T.append_point("C2", C2.b);
  T.append_point("alpha", p.alpha.b);
  Fq c = T.challenge_scalar("c");
  chk.equal({G(p.z, g, g.h)}, {H(c, C1), P(-c, C2, "C2"), P(Fq::one(), p.alpha, "alpha")}, "EqualityProof");
}
void product_verify(Checker& chk, const ProductProof& p, const CommitKey& g, Transcript& T, const Cp& X, const Cp& Y, const Cp& Z) {   // nizk/mod.rs:245-290
  T.append_protocol_name("product proof");
  T.append_point("X", X.b); T.append_point("Y", Y.b); T.append_point("Z", Z.b);
  T.append_point("alpha", p.alpha.b); T.append_point("beta", p.beta.b); T.append_point("delta", p.delta.b);
  Fq c = T.challenge_scalar("c");
  const Fq one = Fq::one();
  chk.equal({P(c, X, "X"), P(one, p.alpha, "alpha")}, {G(p.z[0], g, g.off), G(p.z[1], g, g.h)}, "ProductProof");
  chk.equal({P(one, p.beta, "beta"), P(c, Y, "Y")}, {G(p.z[2], g, g.off), G(p.z[3], g, g.h)}, "ProductProof");
  // third check against the generators (X, h): z3*X + z5*h
  chk.equal({P(one, p.delta, "delta"), P(c, Z, "Z")}, {P(p.z[2], X, "X"), G(p.z[4], g, g.h)}, "ProductProof");
}
void dotproduct_verify(Checker& chk, const DotProductProof& p, const CommitKey& g1, const CommitKey& gn, Transcript& T, const std::vector<Fq>& a, const Cp& Cx,
                       const hge& Cy, const Cp& Cy_c) {   // nizk/mod.rs:372-405
  T.append_protocol_name("dot product proof");
  T.append_point("Cx", Cx.b);
  T.append_point("Cy", Cy_c.b);
  T.append_scalars("a", a);
  T.append_point("delta", p.delta.b);
  T.append_point("beta", p.beta.b);
  Fq c = T.challenge_scalar("c");
  if (p.z.size() != a.size() || a.size() != gn.n) throw Reject("DotProductProof shape");
  Side rhs;
  for (size_t i = 0; i < p.z.size(); i++) rhs.push_back(G(p.z[i], gn, gn.off + i));
  rhs.push_back(G(p.z_delta, gn, gn.h));
  chk.equal({P(c, Cx, "Cx"), P(Fq::one(), p.delta, "delta")}, rhs, "DotProductProof");
  Fq dz = Fq::zero();
  for (size_t i = 0; i < a.size(); i++) dz += p.z[i] * a[i];
  chk.equal({H(c, Cy), P(Fq::one(), p.beta, "beta")}, {G(dz, g1, g1.off), G(p.z_beta, g1, g1.h)}, "DotProductProof");
}

// ---- sumcheck verifiers
// ZKSumcheckInstanceProof::verify (sumcheck.rs:84-179); returns the last comm_eval.  comm_claim: the claim the verifier derived, and its encoding
Cp zk_sumcheck_verify(Checker& chk, const ZKSumcheckInstanceProof& p, const hge& comm_claim, const Cp& comm_claim_c, size_t num_rounds, size_t degree,
                      const CommitKey& g1, const CommitKey& gn, Transcript& T, std::vector<Fq>& r) {
  if (gn.n != degree + 1 || p.comm_polys.size() != num_rounds || p.comm_evals.size() != num_rounds || p.proofs.size() != num_rounds)
    throw Reject("ZK sumcheck shape");
  for (size_t i = 0; i < num_rounds; i++) {
    T.append_point("comm_poly", p.comm_polys[i].b);
    Fq r_i = T.challenge_scalar("challenge_nextround");
    const Cp& claim_c = i == 0 ? comm_claim_c : p.comm_evals[i - 1];
    T.append_point("comm_claim_per_round", claim_c.b);
    T.append_point("comm_eval", p.comm_evals[i].b);
    std::vector<Fq> w = T.challenge_vector("combine_two_claims_to_one", 2);
    const hge claim = i == 0 ? comm_claim : chk.point(claim_c, "comm_claim_per_round");
    hge target = hge_add(mul(claim, w[0]), mul(chk.point(p.comm_evals[i], "comm_eval"), w[1]));
    const std::vector<Fq> a = zk_round_weights(w, r_i, degree);
    try {
      dotproduct_verify(chk, p.proofs[i], g1, gn, T, a, p.comm_polys[i], target, compress(target));
    } catch (const BadPoint&) {   // the reference turns every error of the round's DotProductProof into InternalError (sumcheck.rs:164-176)
      throw Reject("DotProductProof");
    }
    r.push_back(r_i);
  }
  return p.comm_evals.back();
}
// SumcheckInstanceProof::verify (sumcheck.rs:27-62)
Fq sumcheck_verify(const SumcheckInstanceProof& p, Fq e, size_t num_rounds, size_t degree, Transcript& T, std::vector<Fq>& r) {
  if (p.compressed_polys.size() != num_rounds) throw Reject("sumcheck rounds");
  for (auto& cp : p.compressed_polys) {
    const auto& c = cp.coeffs_except_linear_term;
    if (c.size() != degree) throw Reject("sumcheck degree");
    // CompressedUniPoly::decompress (unipoly.rs:95-109): linear term from the hint e = p(0) + p(1)
    Fq lin = e - c[0] - c[0];
    for (size_t i = 1; i < c.size(); i++) lin -= c[i];
    UniPoly poly;
    poly.coeffs.push_back(c[0]); poly.coeffs.push_back(lin);
    for (size_t i = 1; i < c.size(); i++) poly.coeffs.push_back(c[i]);
    poly.append_to_transcript("poly", T);
    Fq r_i = T.challenge_scalar("challenge_nextround");
    r.push_back(r_i);
    e = poly.evaluate(r_i);
  }
  return e;
}

// ---- inner-product argument
// how the public vector a of a DotProductProofLog enters its verify: absorbed by the transcript, and a_hat = <a, s> from the challenges u
struct DotLogA {
  std::function<void(Transcript&)> absorb;
  std::function<Fq(const std::vector<Fq>& u, const std::vector<Fq>& u_inv, const IpaS& s)> a_hat;
};
// DotProductProofLog::verify (nizk/mod.rs:527-583) with BulletReductionProof::verify (nizk/bullet.rs:137-225) inlined, for vectors of n entries.
// g1: gens_1 (G_1 and h).  gens_n set: g_hat = <s, G> is the Checker's IPA term over its tables; else g_hat_of(s) computes it.  Cy: the claimed
// value's commitment as a term of coefficient one (a point of the proof, or Zr * G_1), and its encoding
void dotproduct_log_verify(Checker& chk, const DotProductProofLog& p, const CommitKey& g1, const CommitKey* gens_n, size_t n, Transcript& T, const DotLogA& a,
                           const hge& Cx, const Cp& Cx_c, const GTerm& Cy, const Cp& Cy_c, const std::function<hge(const IpaS&)>& g_hat_of = nullptr) {
  if (gens_n && gens_n->n != n) throw Reject("DotProductProofLog size");
  T.append_protocol_name("dot product proof (log)");
  T.append_point("Cx", Cx_c.b);
  T.append_point("Cy", Cy_c.b);
  a.absorb(T);
  Fq r = T.challenge_scalar("r");
  const auto& L = p.bullet_reduction_proof.L_vec;
  const auto& R = p.bullet_reduction_proof.R_vec;
  const size_t lg_n = L.size();
  if (lg_n >= 32 || n != ((size_t)1 << lg_n) || R.size() != lg_n) throw Reject("bullet reduction size");
  std::vector<Fq> u(lg_n), u_inv(lg_n), u_sq(lg_n), u_inv_sq(lg_n);
  for (size_t i = 0; i < lg_n; i++) {
    T.append_point("L", L[i].b);
    T.append_point("R", R[i].b);
    u[i] = T.challenge_scalar("u");
  }
  Fq allinv = Fq::one();
  for (size_t i = 0; i < lg_n; i++) { u_inv[i] = u[i].inv(); allinv *= u_inv[i]; u_sq[i] = u[i] * u[i]; u_inv_sq[i] = u_inv[i] * u_inv[i]; }
  const IpaS s{gens_n, lg_n, u_sq, allinv, p.z1};
  const Fq a_hat = a.a_hat(u, u_inv, s);
  T.append_point("delta", p.delta.b);
  T.append_point("beta", p.beta.b);
  Fq c = T.challenge_scalar("c");
  // lhs = a_hat*(c*Gamma_hat + beta) + delta, Gamma_hat = Cx + r*Cy + sum_i (u_i^2 L_i + u_i^-2 R_i)
  const Fq ac = a_hat * c;
  Side lhs = {H(ac, Cx), scaled(Cy, ac * r)};
  for (size_t i = 0; i < lg_n; i++) { lhs.push_back(P(ac * u_sq[i], L[i], "L")); lhs.push_back(P(ac * u_inv_sq[i], R[i], "R")); }
  lhs.push_back(P(a_hat, p.beta, "beta"));
  lhs.push_back(P(Fq::one(), p.delta, "delta"));
  // rhs = (g_hat + a_hat*(r*G1))*z1 + h*z2, g_hat = <s, G>
  Side rhs = {G(p.z1 * a_hat * r, g1, g1.off), G(p.z2, g1, g1.h)};
  if (gens_n) {
    chk.equal(lhs, rhs, "DotProductProofLog", &s);
    return;
  }
  rhs.push_back(H(p.z1, g_hat_of(s)));
  chk.equal(lhs, rhs, "DotProductProofLog");
}
// PolyEvalProof::verify (dense_mlpoly.rs:367-389).  It opens at a = eq(r_R, .), so a_hat = <a, s> is the O(lg n) product of ipa_a_hat
void polyeval_verify(Checker& chk, const PolyEvalProof& p, const PolyCommitmentGens& gens, Transcript& T, const std::vector<Fq>& r, const GTerm& C_Zr,
                     const Cp& C_Zr_c, const PolyCommitment& comm) {
  T.append_protocol_name("polynomial evaluation proof");
  size_t ell = r.size(), lv = ell / 2;
  const std::vector<Fq> r_R(r.begin() + lv, r.end());
  std::vector<Fq> Lv = host_eq_evals(std::vector<Fq>(r.begin(), r.begin() + lv)), Rv = host_eq_evals(r_R);
  if (comm.C.size() != Lv.size()) throw Reject("polynomial commitment size");
  hge C_LZ = msm_points(chk, comm.C, Lv, "polynomial commitment share");
  const DotLogA a{[&](Transcript& t) { t.append_scalars("a", Rv); },
                  [&](const std::vector<Fq>& u, const std::vector<Fq>& u_inv, const IpaS& s) { return ipa_a_hat(r_R.data(), u.data(), u_inv.data(), s.lg_n); }};
  dotproduct_log_verify(chk, p.proof, gens.gens_1, &gens.gens_n, Rv.size(), T, a, C_LZ, compress(C_LZ), C_Zr, C_Zr_c);
}
void polyeval_verify_plain(Checker& chk, const PolyEvalProof& p, const PolyCommitmentGens& gens, Transcript& T, const std::vector<Fq>& r, const Fq& Zr,
                           const PolyCommitment& comm) {   // dense_mlpoly.rs:391-404
  polyeval_verify(chk, p, gens, T, r, G(Zr, gens.gens_1, gens.gens_1.off), compress(commit1(gens.gens_1, Zr, Fq::zero())), comm);
}

// ---- R1CSProof::verify (r1csproof.rs:351-489)
void r1cs_verify(Checker& chk, const R1CSProof& p, size_t num_vars, size_t num_cons, const std::vector<Fq>& input, const Fq evals[3], Transcript& T,
                 const R1CSGens& gens, std::vector<Fq>& rx, std::vector<Fq>& ry) {
  T.append_protocol_name("R1CS proof");
  T.append_scalars("input", input);
  append_poly_commitment(T, "poly_commitment", p.comm_vars);
  const size_t num_rounds_x = log2_ceil(num_cons), num_rounds_y = log2_ceil(2 * num_vars);
  std::vector<Fq> tau = T.challenge_vector("challenge_tau", num_rounds_x);
  const hge claim_phase1 = commit1(gens.gens_1, Fq::zero(), Fq::zero());
  Cp comm_claim_post_phase1 = zk_sumcheck_verify(chk, p.sc_proof_phase1, claim_phase1, compress(claim_phase1), num_rounds_x, 3, gens.gens_1, gens.gens_4, T, rx);
  const Cp &comm_Az = p.claims_phase2[0], &comm_Bz = p.claims_phase2[1], &comm_Cz = p.claims_phase2[2], &comm_prod = p.claims_phase2[3];
  knowledge_verify(chk, p.pok_Cz, gens.gens_1, T, comm_Cz);
  product_verify(chk, p.proof_prod, gens.gens_1, T, comm_Az, comm_Bz, comm_prod);
  append_claims_phase2(T, p.claims_phase2);
  Fq taus_bound_rx = eq_eval(rx, tau);
  const hge expected1 = mul(hge_add(chk.point(comm_prod, "comm_prod"), neg(chk.point(comm_Cz, "comm_Cz"))), taus_bound_rx);
  equality_verify(chk, p.proof_eq_sc_phase1, gens.gens_1, T, expected1, compress(expected1), comm_claim_post_phase1);
  Fq r_A = T.challenge_scalar("challenge_Az"), r_B = T.challenge_scalar("challenge_Bz"), r_C = T.challenge_scalar("challenge_Cz");
  const hge comm_claim_phase2 = hge_add(hge_add(mul(chk.point(comm_Az, "comm_Az"), r_A), mul(chk.point(comm_Bz, "comm_Bz"), r_B)), mul(chk.point(comm_Cz, "comm_Cz"), r_C));
  Cp comm_claim_post_phase2 =
      zk_sumcheck_verify(chk, p.sc_proof_phase2, comm_claim_phase2, compress(comm_claim_phase2), num_rounds_y, 2, gens.gens_1, gens.gens_3, T, ry);
  polyeval_verify(chk, p.proof_eval_vars_at_ry, gens.gens_pc, T, std::vector<Fq>(ry.begin() + 1, ry.end()), P(Fq::one(), p.comm_vars_at_ry, "Cy"),
                  p.comm_vars_at_ry, p.comm_vars);
  // SparsePolynomial::evaluate over (0, 1), (i+1, input[i])   (r1csproof.rs:454-464, sparse_mlpoly.rs:1577-1593)
  const size_t nb = log2_ceil(num_vars);
  Fq poly_input_eval = Fq::zero();
  for (size_t e = 0; e <= input.size(); e++) {
    Fq chi = Fq::one();
    for (size_t k = 0; k < nb; k++) {
      bool bit = (e >> (nb - k - 1)) & 1;
      chi *= bit ? ry[1 + k] : Fq::one() - ry[1 + k];
    }
    poly_input_eval += chi * (e == 0 ? Fq::one() : input[e - 1]);
  }
  hge comm_eval_Z = hge_add(mul(chk.point(p.comm_vars_at_ry, "comm_vars_at_ry"), Fq::one() - ry[0]), mul(commit1(gens.gens_pc.gens_1, poly_input_eval, Fq::zero()), ry[0]));
  const hge expected2 = mul(comm_eval_Z, r_A * evals[0] + r_B * evals[1] + r_C * evals[2]);
  equality_verify(chk, p.proof_eq_sc_phase2, gens.gens_1, T, expected2, compress(expected2), comm_claim_post_phase2);
}

// ---- SPARK
// ProductCircuitEvalProofBatched::verify (product_tree.rs:385-485)
BatchedOut batched_verify(const ProductCircuitEvalProofBatched& p, const std::vector<Fq>& claims_prod, const std::vector<Fq>& claims_dotp, size_t len, Transcript& T) {
  const size_t num_layers = log2_ceil(len), np = claims_prod.size();
  if (p.proof.size() != num_layers) throw Reject("product circuit depth");
  BatchedOut o;
  std::vector<Fq> claims = claims_prod;
  for (size_t i = 0; i < num_layers; i++) {
    const bool last = i == num_layers - 1;
    if (last) claims.insert(claims.end(), claims_dotp.begin(), claims_dotp.end());
    std::vector<Fq> coeff = T.challenge_vector("rand_coeffs_next_layer", claims.size());
    Fq claim = Fq::zero();
    for (size_t k = 0; k < claims.size(); k++) claim += claims[k] * coeff[k];
    std::vector<Fq> rand_prod;
    Fq claim_last = sumcheck_verify(p.proof[i].proof, claim, i, 3, T, rand_prod);
    const auto &cpl = p.proof[i].claims_prod_left, &cpr = p.proof[i].claims_prod_right;
    if (cpl.size() != np || cpr.size() != np) throw Reject("product circuit claims");
    for (size_t k = 0; k < np; k++) { T.append_scalar("claim_prod_left", cpl[k]); T.append_scalar("claim_prod_right", cpr[k]); }
    if (o.rand.size() != rand_prod.size()) throw Reject("product circuit randomness");
    Fq eq = eq_eval(o.rand, rand_prod);
    Fq expected = Fq::zero();
    for (size_t k = 0; k < np; k++) expected += coeff[k] * (cpl[k] * cpr[k] * eq);
    if (last) {
      if (p.dotp_left.size() != claims_dotp.size() || p.dotp_right.size() != claims_dotp.size() || p.dotp_weight.size() != claims_dotp.size()) throw Reject("dotp claims shape");
      for (size_t k = 0; k < p.dotp_left.size(); k++) {
        T.append_scalar("claim_dotp_left", p.dotp_left[k]);
        T.append_scalar("claim_dotp_right", p.dotp_right[k]);
        T.append_scalar("claim_dotp_weight", p.dotp_weight[k]);
        expected += coeff[np + k] * p.dotp_left[k] * p.dotp_right[k] * p.dotp_weight[k];
      }
    }
    if (!(expected == claim_last)) throw Reject("product circuit layer " + std::to_string(i));
    Fq r_layer = T.challenge_scalar("challenge_r_layer");
    claims.resize(np);
    for (size_t k = 0; k < np; k++) claims[k] = cpl[k] + r_layer * (cpr[k] - cpl[k]);
    if (last)
      for (size_t k = 0; k < claims_dotp.size() / 2; k++) {
        o.claims_dotp.push_back(p.dotp_left[2 * k] + r_layer * (p.dotp_left[2 * k + 1] - p.dotp_left[2 * k]));
        o.claims_dotp.push_back(p.dotp_right[2 * k] + r_layer * (p.dotp_right[2 * k + 1] - p.dotp_right[2 * k]));
        o.claims_dotp.push_back(p.dotp_weight[2 * k] + r_layer * (p.dotp_weight[2 * k + 1] - p.dotp_weight[2 * k]));
      }
    std::vector<Fq> ext = {r_layer};
    ext.insert(ext.end(), rand_prod.begin(), rand_prod.end());
    o.rand = ext;
  }
  o.claims = claims;
  return o;
}
// HashLayerProof::verify_helper (sparse_mlpoly.rs:837-890)
void hash_helper(const std::vector<Fq>& rand_mem, const Fq& claim_init, const std::vector<Fq>& claim_read, const std::vector<Fq>& claim_write, const Fq& claim_audit,
                 const std::vector<Fq>& ops_val, const std::vector<Fq>& ops_addr, const std::vector<Fq>& read_ts, const Fq& audit_ts, const std::vector<Fq>& r,
                 const Fq& r_hash, const Fq& r_multiset) {
  const Fq r2 = r_hash * r_hash;
  auto h = [&](const Fq& addr, const Fq& val, const Fq& ts) { return ts * r2 + val * r_hash + addr - r_multiset; };
  const size_t ln = rand_mem.size();
  Fq init_addr = Fq::zero();   // IdentityPolynomial::evaluate (dense_mlpoly.rs:105-115)
  for (size_t i = 0; i < ln; i++) init_addr += Fq::from_u64((uint64_t)1 << (ln - i - 1)) * rand_mem[i];
  Fq init_val = eq_eval(r, rand_mem);
  if (!(h(init_addr, init_val, Fq::zero()) == claim_init)) throw Reject("hash layer: init");
  if (ops_addr.size() != ops_val.size() || read_ts.size() != ops_val.size() || claim_read.size() != ops_val.size() || claim_write.size() != ops_val.size())
    throw Reject("hash layer shape");
  for (size_t i = 0; i < ops_addr.size(); i++) {
    if (!(h(ops_addr[i], ops_val[i], read_ts[i]) == claim_read[i])) throw Reject("hash layer: read");
    if (!(h(ops_addr[i], ops_val[i], read_ts[i] + Fq::one()) == claim_write[i])) throw Reject("hash layer: write");
  }
  if (!(h(init_addr, init_val, audit_ts) == claim_audit)) throw Reject("hash layer: audit");
}
// SparseMatPolyEvalProof::verify (sparse_mlpoly.rs:1516-1557) -> PolyEvalNetworkProof::verify (:1356-1416)
void spark_verify(Checker& chk, const SparseMatPolyEvalProof& p, const SparseMatPolyCommitment& comm, std::vector<Fq> rx, std::vector<Fq> ry,
                  const std::vector<Fq>& evals, const SparkGens& gens, Transcript& T) {
  T.append_protocol_name("Sparse polynomial evaluation proof");
  equalize(rx, ry);
  if (((size_t)1 << rx.size()) != comm.num_mem_cells) throw Reject("memory size");
  append_derefs_commitment(T, p.comm_derefs);
  std::vector<Fq> r_mem = T.challenge_vector("challenge_r_hash", 2);
  const Fq &r_hash = r_mem[0], &r_multiset = r_mem[1];
  T.append_protocol_name("Sparse polynomial evaluation proof");      // PolyEvalNetworkProof::protocol_name is the same string
  const size_t ni = evals.size(), num_ops = next_pow2(comm.num_ops), num_cells = (size_t)1 << rx.size();
  // ---- ProductLayerProof::verify (sparse_mlpoly.rs:1228-1305)
  const ProductLayerProof& pl = p.proof_prod_layer;
  T.append_protocol_name("Sparse polynomial product layer proof");
  for (auto* v : {&pl.row_read, &pl.row_write, &pl.col_read, &pl.col_write})
    if (v->size() != ni) throw Reject("product layer shape");
  if (!append_memory_claims(T, pl)) throw Reject("memory check: init * writes != reads * audit");
  if (pl.eval_dotp_left.size() != ni || pl.eval_dotp_right.size() != ni) throw Reject("dotp shape");
  std::vector<Fq> claims_dotp_circuit;
  for (size_t i = 0; i < ni; i++) {
    if (!(pl.eval_dotp_left[i] + pl.eval_dotp_right[i] == evals[i])) throw Reject("dot product split");
    T.append_scalar("claim_eval_dotp_left", pl.eval_dotp_left[i]);
    T.append_scalar("claim_eval_dotp_right", pl.eval_dotp_right[i]);
    claims_dotp_circuit.push_back(pl.eval_dotp_left[i]); claims_dotp_circuit.push_back(pl.eval_dotp_right[i]);
  }
  std::vector<Fq> claims_prod;
  for (auto* v : {&pl.row_read, &pl.row_write, &pl.col_read, &pl.col_write}) claims_prod.insert(claims_prod.end(), v->begin(), v->end());
  BatchedOut ops = batched_verify(pl.proof_ops, claims_prod, claims_dotp_circuit, num_ops, T);
  BatchedOut mem = batched_verify(pl.proof_mem, {pl.row_init, pl.row_audit, pl.col_init, pl.col_audit}, {}, num_cells, T);
  if (mem.claims.size() != 4 || ops.claims.size() != 4 * ni || ops.claims_dotp.size() != 3 * ni) throw Reject("claims shape");
  std::vector<Fq> row_read(ops.claims.begin(), ops.claims.begin() + ni), row_write(ops.claims.begin() + ni, ops.claims.begin() + 2 * ni);
  std::vector<Fq> col_read(ops.claims.begin() + 2 * ni, ops.claims.begin() + 3 * ni), col_write(ops.claims.begin() + 3 * ni, ops.claims.end());
  const std::vector<Fq>&rand_mem = mem.rand, &rand_ops = ops.rand;
  // ---- HashLayerProof::verify (sparse_mlpoly.rs:892-1019)
  const HashLayerProof& hl = p.proof_hash_layer;
  T.append_protocol_name("Sparse polynomial hash layer proof");
  if (hl.derefs_row.size() != ni || hl.derefs_col.size() != ni || hl.eval_val.size() != ni) throw Reject("hash layer shape");
  Fq joint;
  {  // DerefsEvalProof::verify (sparse_mlpoly.rs:151-211)
    T.append_protocol_name("Derefs evaluation proof");
    const std::vector<Fq> r_joint = combine_to_one(T, hl, HashOpening::derefs, rand_ops, joint);
    polyeval_verify_plain(chk, hl.proof_derefs, gens.gens_derefs, T, r_joint, joint, p.comm_derefs);
  }
  for (size_t i = 0; i < ni; i++)
    if (!(ops.claims_dotp[3 * i] == hl.derefs_row[i]) || !(ops.claims_dotp[3 * i + 1] == hl.derefs_col[i]) || !(ops.claims_dotp[3 * i + 2] == hl.eval_val[i]))
      throw Reject("dot product claims");
  {
    const std::vector<Fq> r_joint = combine_to_one(T, hl, HashOpening::ops, rand_ops, joint);
    polyeval_verify_plain(chk, hl.proof_ops, gens.gens_ops, T, r_joint, joint, comm.comm_comb_ops);
  }
  {
    const std::vector<Fq> r_joint = combine_to_one(T, hl, HashOpening::mem, rand_mem, joint);
    polyeval_verify_plain(chk, hl.proof_mem, gens.gens_mem, T, r_joint, joint, comm.comm_comb_mem);
  }
  hash_helper(rand_mem, mem.claims[0], row_read, row_write, mem.claims[1], hl.derefs_row, hl.row_addr, hl.row_read_ts, hl.row_audit_ts, rx, r_hash, r_multiset);
  hash_helper(rand_mem, mem.claims[2], col_read, col_write, mem.claims[3], hl.derefs_col, hl.col_addr, hl.col_read_ts, hl.col_audit_ts, ry, r_hash, r_multiset);
}

bool pow2(size_t x) { return x && !(x & (x - 1)); }
// shape sanity shared by both verifiers: the padded dimensions the prover enforces (lib.rs:129-198, r1csproof.rs:156); without it a
// hand-made commitment with num_vars = 0 or num_cons <= 1 would leave the round vectors empty (`.back()`, `ry[0]`)
void check_dims(size_t num_cons, size_t num_vars, size_t num_inputs) {
  if (num_cons < 2 || num_vars < 1 || !pow2(num_cons) || !pow2(num_vars)) throw SpError(SP_ERR_INVALID_ARG, "verifier: num_cons >= 2 and num_vars >= 1 must be powers of two");
  if (!(num_inputs < num_vars)) throw SpError(SP_ERR_INVALID_ARG, "verifier: |input| + 1 must be at most the number of variables");
}
void check_commitment(const ComputationCommitment& comm) {
  check_dims(comm.num_cons, comm.num_vars, comm.num_inputs);
  // SparseMatPolyCommitment consistency (sparse_mlpoly.rs:366-420): 3 matrices, power-of-two op count of at least 2 (what snark_encode
  // produces: one op leaves the product circuits without layers), cells = max(num_cons, 2*num_vars)
  const size_t cells = std::max(comm.num_cons, 2 * comm.num_vars);
  if (comm.comm.batch_size != 3 || !pow2(comm.comm.num_ops) || comm.comm.num_ops < 2 || comm.comm.num_mem_cells != cells)
    throw SpError(SP_ERR_INVALID_ARG, "verifier: inconsistent computation commitment");
}

// NIZK::verify (lib.rs:549-591) after parsing
void nizk_replay(Checker& chk, const Instance& inst, const std::vector<Fq>& input, const R1CSGens& gens, Transcript& T, const NizkProof& p) {
  if (input.size() != inst.num_inputs) throw Reject("number of inputs");
  if (p.rx.size() != log2_ceil(inst.num_cons) || p.ry.size() != log2_ceil(2 * inst.num_vars)) throw Reject("claimed evaluation point");
  {
    FineTimer ft(chk.ctx, "verify.nizk_head");   // absorbs the R1CS shape digest
    append_nizk_head(T, inst);
  }
  Fq evals[3];
  {
    FineTimer ft(chk.ctx, "verify.instance_evaluate");
    instance_evaluate(chk.ctx, inst, p.rx, p.ry, evals);
  }
  std::vector<Fq> rx, ry;
  r1cs_verify(chk, p.r1cs_sat_proof, inst.num_vars, inst.num_cons, input, evals, T, gens, rx, ry);
  if (!(rx == p.rx) || !(ry == p.ry)) throw Reject("evaluation point differs from the sumcheck challenges");
}
// SNARK::verify (lib.rs:423-465) after parsing
void snark_replay(Checker& chk, const ComputationCommitment& comm, const std::vector<Fq>& input, const SnarkGens& gens, Transcript& T, const SnarkProof& p) {
  if (input.size() != comm.num_inputs) throw Reject("number of inputs");
  T.append_protocol_name("Spartan SNARK proof");
  append_computation_commitment(T, comm);
  const Fq* evals = p.inst_evals.data();
  std::vector<Fq> rx, ry;
  r1cs_verify(chk, p.r1cs_sat_proof, comm.num_vars, comm.num_cons, input, evals, T, *gens.gens_r1cs_sat, rx, ry);
  T.append_scalar("Ar_claim", evals[0]);
  T.append_scalar("Br_claim", evals[1]);
  T.append_scalar("Cr_claim", evals[2]);
  spark_verify(chk, p.r1cs_eval_proof, comm.comm, rx, ry, std::vector<Fq>(evals, evals + 3), gens.gens_r1cs_eval, T);
}

// every point a proof carries, in wire order (the fields io() lists)
struct PointLister {
  std::vector<Cp>& out;
  template <class... T> void operator()(T&... v) { (get(v), ...); }
  template <class T> void get(T& v) { v.io(*this); }
  void get(uint64_t&) {}
  void get(Fq&) {}
  void get(Cp& c) { out.push_back(c); }
  template <class T, size_t N> void get(std::array<T, N>& a) { for (auto& x : a) get(x); }
  template <class T> void get(std::vector<T>& v) { for (auto& x : v) get(x); }
};

bool is_rejection(const SpError& e) { return e.code == SP_ERR_VERIFY || e.code == SP_ERR_DECOMPRESS; }

// The batch driver (DESIGN.md "deferred checks"): parse, decompress every point of every proof in one launch, replay each proof's transcript
// with the deferred checker, test every accumulator in one device pass, then re-run each rejected proof with the immediate checker for its
// status, message and transcript state.  replay(chk, job, proof): the protocol after parsing; single(job, T): the whole single-proof verify.
// stmt_points(job, out): points of the statement that the replay decompresses on the host (msm_points' short path)
template <class Proof, class Replay, class Single, class StmtPoints>
void verify_batch(Ctx& ctx, std::vector<VerifyJob>& jobs, const uint8_t seed[32], Replay replay, Single single, StmtPoints stmt_points) {
  const size_t K = jobs.size();
  std::vector<Proof> proofs(K);
  std::vector<bool> alive(K, true);
  std::vector<Transcript> T_out;
  T_out.reserve(K);
  for (auto& j : jobs) T_out.push_back(j.T);
  PointTable table;
  {
    FineTimer ft(ctx, "batch.decompress");
    std::vector<std::vector<Cp>> pts(K);
    std::vector<Cp> all;
    for (size_t i = 0; i < K; i++) {
      try {
        proofs[i] = from_bincode<Proof>(jobs[i].proof, jobs[i].len, SP_ERR_VERIFY, "proof");
      } catch (const SpError& e) {
        if (!is_rejection(e)) throw;
        alive[i] = false;
        continue;
      }
      PointLister{pts[i]}(proofs[i]);
      all.insert(all.end(), pts[i].begin(), pts[i].end());
      stmt_points(jobs[i], all);   // a point that fails here stays out of the table: the replay's host decode then rejects the proof as the single call does
    }
    const size_t n = all.size();
    if (n) {
      DevBuf<uint8_t> d_in(32 * n);
      DevBuf<ge> g(n);
      DevBuf<int> ok(n);
      dev::h2d(d_in.p, all.data(), 32 * n, ctx.stream);
      dev::decompress_batch(g.p, ok.p, d_in.p, n, ctx.stream);
      std::vector<ge> h_g(n);
      std::vector<int> h_ok(n);
      dev::d2h(h_g.data(), g.p, sizeof(ge) * n, ctx.stream);
      dev::d2h(h_ok.data(), ok.p, sizeof(int) * n, ctx.stream);
      ctx.sync();
      std::unordered_map<Cp, bool, CpHash> bad;
      for (size_t m = 0; m < n; m++) {
        if (h_ok[m]) table.emplace(all[m], h_g[m]);
        else bad[all[m]] = true;
      }
      if (!bad.empty())
        for (size_t i = 0; i < K; i++)
          for (const Cp& c : pts[i]) if (bad.count(c)) { alive[i] = false; break; }
    }
  }
  std::vector<ProofAcc> accs(K);
  {
    FineTimer ft(ctx, "batch.replay");
    for (size_t i = 0; i < K; i++) {
      if (!alive[i]) continue;
      Deferred chk(ctx, table, seed, i, accs[i]);
      try {
        replay(chk, jobs[i], T_out[i], proofs[i]);
      } catch (const SpError& e) {
        if (!is_rejection(e)) throw;
        alive[i] = false;
      }
    }
  }
  {
    FineTimer ft(ctx, "batch.final");
    std::vector<const ProofAcc*> live;
    std::vector<size_t> idx;
    for (size_t i = 0; i < K; i++) if (alive[i]) { live.push_back(&accs[i]); idx.push_back(i); }
    const std::vector<bool> ok = deferred_final(ctx, live);
    for (size_t m = 0; m < idx.size(); m++) if (!ok[m]) alive[idx[m]] = false;
  }
  for (size_t i = 0; i < K; i++) {
    VerifyJob& j = jobs[i];
    if (alive[i]) { j.status = SP_OK; j.msg.clear(); j.T = T_out[i]; continue; }
    FineTimer ft(ctx, "batch.rerun");   // absent from the timings when no proof was re-run
    Transcript T = j.T;
    try {
      single(j, T);
      j.status = SP_OK;
      j.msg.clear();
    } catch (const SpError& e) {
      if (!is_rejection(e)) throw;
      j.status = e.code;
      j.msg = e.what();
    }
    j.T = T;
  }
}

}  // namespace

BatchedOut prod_verify(const uint8_t* proof, size_t len, const std::vector<Fq>& products, const std::vector<Fq>& dotp_claims, size_t m, Transcript& T) {
  const ProductCircuitEvalProofBatched p = from_bincode<ProductCircuitEvalProofBatched>(proof, len, SP_ERR_VERIFY, "product circuit proof");
  return batched_verify(p, products, dotp_claims, (size_t)1 << m, T);
}

Fq sumcheck_verify_bytes(const uint8_t* proof, size_t len, const Fq& claim, size_t num_rounds, size_t degree, Transcript& T, std::vector<Fq>& r) {
  const SumcheckInstanceProof p = from_bincode<SumcheckInstanceProof>(proof, len, SP_ERR_VERIFY, "sumcheck proof");
  return sumcheck_verify(p, claim, num_rounds, degree, T, r);
}

// the caller's sigma proofs and ZK sumchecks (sp_knowledge_verify_t .. sp_zk_sumcheck_verify_t)
void knowledge_verify_bytes(Ctx& ctx, const CommitKey& g, Transcript& T, const Cp& C, const uint8_t* proof, size_t len) {
  const KnowledgeProof p = from_bincode<KnowledgeProof>(proof, len, SP_ERR_VERIFY, "knowledge proof");
  Immediate chk(ctx);
  knowledge_verify(chk, p, g, T, C);
}
void equality_verify_bytes(Ctx& ctx, const CommitKey& g, Transcript& T, const Cp& C1, const Cp& C2, const uint8_t* proof, size_t len) {
  const EqualityProof p = from_bincode<EqualityProof>(proof, len, SP_ERR_VERIFY, "equality proof");
  Immediate chk(ctx);
  equality_verify(chk, p, g, T, unpack(C1, "C1"), C1, C2);
}
void product_verify_bytes(Ctx& ctx, const CommitKey& g, Transcript& T, const Cp& X, const Cp& Y, const Cp& Z, const uint8_t* proof, size_t len) {
  const ProductProof p = from_bincode<ProductProof>(proof, len, SP_ERR_VERIFY, "product proof");
  Immediate chk(ctx);
  product_verify(chk, p, g, T, X, Y, Z);
}
void dotproduct_verify_bytes(Ctx& ctx, const CommitKey& g1, const CommitKey& gn, Transcript& T, const std::vector<Fq>& a, const Cp& Cx, const Cp& Cy,
                             const uint8_t* proof, size_t len) {
  const DotProductProof p = from_bincode<DotProductProof>(proof, len, SP_ERR_VERIFY, "dot product proof");
  Immediate chk(ctx);
  dotproduct_verify(chk, p, g1, gn, T, a, Cx, unpack(Cy, "Cy"), Cy);
}
Cp zk_sumcheck_verify_bytes(Ctx& ctx, const uint8_t* proof, size_t len, const Cp& comm_claim, size_t num_rounds, size_t degree, const CommitKey& g1,
                            const CommitKey& gn, Transcript& T, std::vector<Fq>& r) {
  const ZKSumcheckInstanceProof p = from_bincode<ZKSumcheckInstanceProof>(proof, len, SP_ERR_VERIFY, "ZK sumcheck proof");
  Immediate chk(ctx);
  return zk_sumcheck_verify(chk, p, unpack(comm_claim, "comm_claim"), comm_claim, num_rounds, degree, g1, gn, T, r);
}

// NIZK::verify (lib.rs:549-591)
void nizk_verify(Ctx& ctx, const Instance& inst, const std::vector<Fq>& input, const R1CSGens& gens, Transcript& T, const uint8_t* proof, size_t len) {
  check_dims(inst.num_cons, inst.num_vars, inst.num_inputs);
  const NizkProof p = from_bincode<NizkProof>(proof, len, SP_ERR_VERIFY, "proof");
  Immediate chk(ctx);
  nizk_replay(chk, inst, input, gens, T, p);
}

// R1CSProof::verify (r1csproof.rs:351-489) of a caller's proof; the dimensions are checked by the caller
void r1cs_verify_bytes(Ctx& ctx, const uint8_t* proof, size_t len, size_t num_vars, size_t num_cons, const std::vector<Fq>& input, const Fq evals[3],
                       const R1CSGens& gens, Transcript& T, std::vector<Fq>& rx, std::vector<Fq>& ry) {
  const R1CSProof p = from_bincode<R1CSProof>(proof, len, SP_ERR_VERIFY, "R1CS proof");
  Immediate chk(ctx);
  r1cs_verify(chk, p, num_vars, num_cons, input, evals, T, gens, rx, ry);
}

// SNARK::verify (lib.rs:423-465); `enc` supplies the ComputationCommitment
void snark_verify(Ctx& ctx, const SnarkEncoding& enc, const std::vector<Fq>& input, const SnarkGens& gens, Transcript& T, const uint8_t* proof, size_t len) {
  check_commitment(enc.comm);
  const SnarkProof p = from_bincode<SnarkProof>(proof, len, SP_ERR_VERIFY, "proof");
  Immediate chk(ctx);
  snark_replay(chk, enc.comm, input, gens, T, p);
}

void check_spark_commitment(const SparseMatPolyCommitment& c, size_t nevals, size_t x, size_t y, const SparkGens& gens) {
  if (c.batch_size != nevals) throw Reject("commitment batch size " + std::to_string(c.batch_size) + " != " + std::to_string(nevals) + " evaluations");
  if (nevals < 1 || nevals > SP_SPARK_MAX_BATCH) throw Reject("batch size outside 1 .. SP_SPARK_MAX_BATCH");
  if (!pow2(c.num_ops) || c.num_ops < 2) throw Reject("commitment num_ops is not a power of two >= 2");
  if (std::max(x, y) >= 63 || c.num_mem_cells != ((size_t)1 << std::max(x, y))) throw Reject("commitment num_mem_cells != 2^max(|rx|, |ry|)");
  if (!SparkDims(x, y, c.num_ops, c.batch_size).fits(gens)) throw Reject("generators do not fit the commitment's sizes");
}
// SparseMatPolyEvalProof::verify (sparse_mlpoly.rs:1516-1557) of a caller's proof
void spark_eval_verify(Ctx& ctx, const SparseMatPolyCommitment& comm, const std::vector<Fq>& rx, const std::vector<Fq>& ry, const std::vector<Fq>& evals,
                       const SparkGens& gens, Transcript& T, const uint8_t* proof, size_t len) {
  const SparseMatPolyEvalProof p = from_bincode<SparseMatPolyEvalProof>(proof, len, SP_ERR_VERIFY, "proof");
  Immediate chk(ctx);
  spark_verify(chk, p, comm, rx, ry, evals, gens, T);
}

// PolyEvalProof::verify (dense_mlpoly.rs:367-389) against the caller's C_Zr, or verify_plain (:391-404) against Zr
void pc_eval_verify(Ctx& ctx, const PolyCommitmentGens& gens, const PolyCommitment& comm, const std::vector<Fq>& r, const Cp* C_Zr, const Fq* Zr, Transcript& T,
                    const uint8_t* proof, size_t len) {
  const PolyEvalProof p = from_bincode<PolyEvalProof>(proof, len, SP_ERR_VERIFY, "polynomial evaluation proof");
  Immediate chk(ctx);
  if (Zr) polyeval_verify_plain(chk, p, gens, T, r, *Zr, comm);
  else polyeval_verify(chk, p, gens, T, r, P(Fq::one(), *C_Zr, "C_Zr"), *C_Zr, comm);
}
// DotProductProofLog::verify of the caller's vectors (sp_dotlog_verify_t).  a_hat = <a, s>: on the host from n <= SP_DOTLOG_TABLE_MAX_N entries; on
// the folding path s is built on the device (k_ipa_srow), where a_hat = <a, s> and g_hat = <s, G> (bucket MSM over the gens' points) follow
void dotlog_verify_bytes(Ctx& ctx, const DotLogGens& gens, Transcript& T, const u256* d_a, const Cp& Cx, const Cp& Cy, const uint8_t* proof, size_t len) {
  const DotProductProofLog p = from_bincode<DotProductProofLog>(proof, len, SP_ERR_VERIFY, "dot product proof (log)");
  Immediate chk(ctx);
  const size_t n = gens.n;
  const std::vector<uint8_t> a_canon = canonical_bytes(ctx, d_a, n);
  hge g_hat;
  DotLogA a;
  a.absorb = [&](Transcript& t) { t.append_scalar_bytes("a", a_canon.data(), n); };
  if (!gens.folding()) {
    a.a_hat = [&](const std::vector<Fq>&, const std::vector<Fq>&, const IpaS& s) {   // bullet.rs:160-177
      const std::vector<Fq> av = ctx.download(d_a, n);
      std::vector<Fq> sv(n);
      sv[0] = s.allinv;
      Fq acc = av[0] * sv[0];
      for (size_t i = 1; i < n; i++) {
        const size_t lg_i = 63 - (size_t)__builtin_clzll((unsigned long long)i);
        sv[i] = sv[i - ((size_t)1 << lg_i)] * s.u_sq[s.lg_n - 1 - lg_i];
        acc += av[i] * sv[i];
      }
      return acc;
    };
  } else {
    a.a_hat = [&](const std::vector<Fq>&, const std::vector<Fq>&, const IpaS& s) {
      FineTimer ft(ctx, "verify.dotlog_s");
      DevBuf<u256> d_s(n);
      DevBuf<dev::IpaSRow> d_it(1);
      IpaS one = s;
      one.scale = Fq::one();
      const dev::IpaSRow it = srow_item(d_s.p, one, 0);
      dev::h2d(d_it.p, &it, sizeof it, ctx.stream);
      dev::ipa_srow(d_it.p, 1, (uint32_t)s.lg_n, ctx.stream);
      dev::dot(ctx.small.p + layout::SMALL_DOT.off, d_a, d_s.p, n, ctx.red.p, ctx.stream);
      g_hat = msm_var_host(ctx, gens.pts.p, d_s.p, n);   // synchronises
      Fq a_hat;
      ctx.get_small(layout::SMALL_DOT.off, &a_hat, 1);
      return a_hat;
    };
  }
  dotproduct_log_verify(chk, p, gens.g.gens_1, gens.folding() ? nullptr : &gens.g.gens_n, n, T, a, unpack(Cx, "Cx"), Cx, P(Fq::one(), Cy, "Cy"), Cy,
                        [&](const IpaS&) { return g_hat; });
}
// DerefsEvalProof::verify_single (sparse_mlpoly.rs:149-176)
void pc_eval_verify_joint(Ctx& ctx, const PolyCommitmentGens& gens, const PolyCommitment& comm, const std::vector<Fq>& r, const std::vector<Fq>& evals,
                          Transcript& T, const uint8_t* proof, size_t len) {
  const PolyEvalProof p = from_bincode<PolyEvalProof>(proof, len, SP_ERR_VERIFY, "polynomial evaluation proof");
  Fq joint;
  const std::vector<Fq> r_joint = combine_to_one(T, evals, r, "evals_ops_val", "challenge_combine_n_to_one", "joint_claim_eval", joint);
  Immediate chk(ctx);
  polyeval_verify_plain(chk, p, gens, T, r_joint, joint, comm);
}

void nizk_verify_batch(Ctx& ctx, const R1CSGens& gens, std::vector<VerifyJob>& jobs, const uint8_t seed[32]) {
  for (auto& j : jobs) check_dims(j.inst->num_cons, j.inst->num_vars, j.inst->num_inputs);
  verify_batch<NizkProof>(
      ctx, jobs, seed, [&](Checker& chk, const VerifyJob& j, Transcript& T, const NizkProof& p) { nizk_replay(chk, *j.inst, j.input, gens, T, p); },
      [&](const VerifyJob& j, Transcript& T) { nizk_verify(ctx, *j.inst, j.input, gens, T, j.proof, j.len); }, [](const VerifyJob&, std::vector<Cp>&) {});
}

void snark_verify_batch(Ctx& ctx, const SnarkGens& gens, std::vector<VerifyJob>& jobs, const uint8_t seed[32]) {
  for (auto& j : jobs) check_commitment(j.enc->comm);
  verify_batch<SnarkProof>(
      ctx, jobs, seed, [&](Checker& chk, const VerifyJob& j, Transcript& T, const SnarkProof& p) { snark_replay(chk, j.enc->comm, j.input, gens, T, p); },
      [&](const VerifyJob& j, Transcript& T) { snark_verify(ctx, *j.enc, j.input, gens, T, j.proof, j.len); },
      [](const VerifyJob& j, std::vector<Cp>& out) {
        for (const PolyCommitment* c : {&j.enc->comm.comm.comm_comb_ops, &j.enc->comm.comm.comm_comb_mem})
          if (c->C.size() <= 8) out.insert(out.end(), c->C.begin(), c->C.end());
      });
}

// The deferred checker and the final pass of a batch on hand-made equations (devtest.cu: spd_deferred_check): proof i's equations are recorded
// with proof i's weights, exactly as a replay records them, and ok[i] is what the final pass says of proof i
std::vector<bool> deferred_check(Ctx& ctx, const GenSet& gs, const std::vector<std::vector<DeferredEq>>& proofs, const uint8_t seed[32]) {
  PointTable table;
  std::vector<ProofAcc> accs(proofs.size());
  const CommitKey key{&gs, 0, gs.nbases, 0};
  for (size_t i = 0; i < proofs.size(); i++) {
    Deferred chk(ctx, table, seed, i, accs[i]);
    for (const DeferredEq& e : proofs[i]) {
      Side side[2];
      for (int k = 0; k < 2; k++)
        for (const DeferredTerm& t : k ? e.rhs : e.lhs) side[k].push_back(t.gen >= 0 ? G(t.k, key, (size_t)t.gen) : P(t.k, t.pt, "test point"));
      chk.equal(side[0], side[1], "test equation", nullptr);
    }
  }
  std::vector<const ProofAcc*> ptrs;
  for (auto& a : accs) ptrs.push_back(&a);
  return deferred_final(ctx, ptrs);
}

}  // namespace sp
