// spartan_b200 — NIZK::verify / SNARK::verify (SURVEY.md §8(f) row 4): the verifier side of the reference, so that a caller of this library
// can check the proofs it produces (or proofs produced by the reference: the wire format is bincode's).
//
// Follows /root/reference/src function by function: lib.rs:423-465 (SNARK::verify), :549-591 (NIZK::verify), r1csproof.rs:351-489,
// sumcheck.rs:27-62,84-179, nizk/mod.rs:54-75,118-143,245-290,372-405,527-583, nizk/bullet.rs:137-225, dense_mlpoly.rs:367-404,
// product_tree.rs:385-485, sparse_mlpoly.rs:151-211,837-1019,1228-1305,1356-1416,1516-1557.
// The multiexponentiations over generator vectors and over commitment vectors run on the device (fixed-base tables / bucket MSM); the
// constant-size group checks run on the host in radix 2^51.  Failures map to ProofVerifyError::{InternalError, DecompressionError}.
#include <algorithm>
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
// sum_i s_i * G[key.off + i] over the device tables (no blind)
hge msm_gens(Ctx& ctx, const CommitKey& key, const std::vector<Fq>& s) {
  DevBuf<u256> d(s.size());
  ctx.upload(d.p, s.data(), s.size());
  std::vector<Cp> out;
  commit_rows_and_compress(ctx, key, d.p, s.size(), 1, s.size(), nullptr, out);
  return unpack(out[0], "device MSM result");
}
// sum_i s_i * P_i for proof-supplied points: bucket MSM on the device, a plain loop when there are only a few
hge msm_points(Ctx& ctx, const std::vector<Cp>& pts, const std::vector<Fq>& s, const char* what) {
  const size_t n = pts.size();
  if (n <= 8) {
    hge acc = hge_identity();
    for (size_t i = 0; i < n; i++) acc = hge_add(acc, mul(unpack(pts[i], what), s[i]));
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
void knowledge_verify(const KnowledgeProof& p, const CommitKey& g, Transcript& T, const Cp& C) {   // nizk/mod.rs:54-75
  T.append_protocol_name("knowledge proof");
  T.append_point("C", C.b);
  T.append_point("alpha", p.alpha.b);
  Fq c = T.challenge_scalar("c");
  if (!same(commit1(g, p.z1, p.z2), hge_add(mul(unpack(C, "C"), c), unpack(p.alpha, "alpha")))) throw Reject("KnowledgeProof");
}
void equality_verify(const EqualityProof& p, const CommitKey& g, Transcript& T, const Cp& C1, const Cp& C2) {   // nizk/mod.rs:118-143
  T.append_protocol_name("equality proof");
  T.append_point("C1", C1.b);
  T.append_point("C2", C2.b);
  T.append_point("alpha", p.alpha.b);
  Fq c = T.challenge_scalar("c");
  hge Cd = hge_add(unpack(C1, "C1"), neg(unpack(C2, "C2")));
  Term t[1] = {{g.h, p.z}};
  if (!same(host_commit(*g.set, t, 1), hge_add(mul(Cd, c), unpack(p.alpha, "alpha")))) throw Reject("EqualityProof");
}
void product_verify(const ProductProof& p, const CommitKey& g, Transcript& T, const Cp& X, const Cp& Y, const Cp& Z) {   // nizk/mod.rs:245-290
  T.append_protocol_name("product proof");
  T.append_point("X", X.b); T.append_point("Y", Y.b); T.append_point("Z", Z.b);
  T.append_point("alpha", p.alpha.b); T.append_point("beta", p.beta.b); T.append_point("delta", p.delta.b);
  Fq c = T.challenge_scalar("c");
  hge Xp = unpack(X, "X");
  bool ok = same(hge_add(unpack(p.alpha, "alpha"), mul(Xp, c)), commit1(g, p.z[0], p.z[1]));
  ok = ok && same(hge_add(unpack(p.beta, "beta"), mul(unpack(Y, "Y"), c)), commit1(g, p.z[2], p.z[3]));
  // third check against the generators (X, h): z3*X + z5*h
  Term th[1] = {{g.h, p.z[4]}};
  ok = ok && same(hge_add(unpack(p.delta, "delta"), mul(unpack(Z, "Z"), c)), hge_add(mul(Xp, p.z[2]), host_commit(*g.set, th, 1)));
  if (!ok) throw Reject("ProductProof");
}
void dotproduct_verify(const DotProductProof& p, const CommitKey& g1, const CommitKey& gn, Transcript& T, const std::vector<Fq>& a, const Cp& Cx,
                       const hge& Cy, const Cp& Cy_c) {   // nizk/mod.rs:372-405
  T.append_protocol_name("dot product proof");
  T.append_point("Cx", Cx.b);
  T.append_point("Cy", Cy_c.b);
  T.append_scalars("a", a);
  T.append_point("delta", p.delta.b);
  T.append_point("beta", p.beta.b);
  Fq c = T.challenge_scalar("c");
  if (p.z.size() != a.size() || a.size() != gn.n) throw Reject("DotProductProof shape");
  bool ok = same(hge_add(mul(unpack(Cx, "Cx"), c), unpack(p.delta, "delta")), commitv(gn, p.z, p.z_delta));
  Fq dz = Fq::zero();
  for (size_t i = 0; i < a.size(); i++) dz += p.z[i] * a[i];
  ok = ok && same(hge_add(mul(Cy, c), unpack(p.beta, "beta")), commit1(g1, dz, p.z_beta));
  if (!ok) throw Reject("DotProductProof");
}

// ---- sumcheck verifiers
// ZKSumcheckInstanceProof::verify (sumcheck.rs:84-179); returns the last comm_eval
Cp zk_sumcheck_verify(const ZKSumcheckInstanceProof& p, const Cp& comm_claim, size_t num_rounds, size_t degree, const CommitKey& g1, const CommitKey& gn,
                      Transcript& T, std::vector<Fq>& r) {
  if (gn.n != degree + 1 || p.comm_polys.size() != num_rounds || p.comm_evals.size() != num_rounds || p.proofs.size() != num_rounds)
    throw Reject("ZK sumcheck shape");
  for (size_t i = 0; i < num_rounds; i++) {
    T.append_point("comm_poly", p.comm_polys[i].b);
    Fq r_i = T.challenge_scalar("challenge_nextround");
    const Cp& claim_c = i == 0 ? comm_claim : p.comm_evals[i - 1];
    T.append_point("comm_claim_per_round", claim_c.b);
    T.append_point("comm_eval", p.comm_evals[i].b);
    std::vector<Fq> w = T.challenge_vector("combine_two_claims_to_one", 2);
    hge target = hge_add(mul(unpack(claim_c, "comm_claim_per_round"), w[0]), mul(unpack(p.comm_evals[i], "comm_eval"), w[1]));
    const std::vector<Fq> a = zk_round_weights(w, r_i, degree);
    dotproduct_verify(p.proofs[i], g1, gn, T, a, p.comm_polys[i], target, compress(target));
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
// DotProductProofLog::verify (nizk/mod.rs:527-583) with BulletReductionProof::verify (nizk/bullet.rs:137-225) inlined
void dotproduct_log_verify(Ctx& ctx, const DotProductProofLog& p, const PolyCommitmentGens& gens, Transcript& T, const std::vector<Fq>& a, const hge& Cx,
                           const Cp& Cx_c, const Cp& Cy) {
  const size_t n = a.size();
  if (gens.n != n) throw Reject("DotProductProofLog size");
  T.append_protocol_name("dot product proof (log)");
  T.append_point("Cx", Cx_c.b);
  T.append_point("Cy", Cy.b);
  T.append_scalars("a", a);
  Fq r = T.challenge_scalar("r");
  hge Gamma = hge_add(Cx, mul(unpack(Cy, "Cy"), r));
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
  std::vector<Fq> s(n);
  s[0] = allinv;
  for (size_t i = 1; i < n; i++) {
    size_t lg_i = 0;
    while (((size_t)2 << lg_i) <= i) lg_i++;
    size_t k = (size_t)1 << lg_i;
    s[i] = s[i - k] * u_sq[(lg_n - 1) - lg_i];
  }
  hge g_hat = msm_gens(ctx, gens.gens_n, s);
  Fq a_hat = Fq::zero();
  for (size_t i = 0; i < n; i++) a_hat += a[i] * s[i];
  hge Gamma_hat = Gamma;
  for (size_t i = 0; i < lg_n; i++) Gamma_hat = hge_add(Gamma_hat, hge_add(mul(unpack(L[i], "L"), u_sq[i]), mul(unpack(R[i], "R"), u_inv_sq[i])));
  T.append_point("delta", p.delta.b);
  T.append_point("beta", p.beta.b);
  Fq c = T.challenge_scalar("c");
  hge lhs = hge_add(mul(hge_add(mul(Gamma_hat, c), unpack(p.beta, "beta")), a_hat), unpack(p.delta, "delta"));
  // rhs = (g_hat + a_hat*(r*G1))*z1 + h*z2
  Term t[2] = {{gens.gens_1.off, p.z1 * a_hat * r}, {gens.gens_1.h, p.z2}};
  hge rhs = hge_add(mul(g_hat, p.z1), host_commit(*gens.gens_1.set, t, 2));
  if (!same(lhs, rhs)) throw Reject("DotProductProofLog");
}
// PolyEvalProof::verify (dense_mlpoly.rs:367-389)
void polyeval_verify(Ctx& ctx, const PolyEvalProof& p, const PolyCommitmentGens& gens, Transcript& T, const std::vector<Fq>& r, const Cp& C_Zr,
                     const PolyCommitment& comm) {
  T.append_protocol_name("polynomial evaluation proof");
  size_t ell = r.size(), lv = ell / 2;
  std::vector<Fq> Lv = host_eq_evals(std::vector<Fq>(r.begin(), r.begin() + lv)), Rv = host_eq_evals(std::vector<Fq>(r.begin() + lv, r.end()));
  if (comm.C.size() != Lv.size()) throw Reject("polynomial commitment size");
  hge C_LZ = msm_points(ctx, comm.C, Lv, "polynomial commitment share");
  dotproduct_log_verify(ctx, p.proof, gens, T, Rv, C_LZ, compress(C_LZ), C_Zr);
}
void polyeval_verify_plain(Ctx& ctx, const PolyEvalProof& p, const PolyCommitmentGens& gens, Transcript& T, const std::vector<Fq>& r, const Fq& Zr,
                           const PolyCommitment& comm) {   // dense_mlpoly.rs:391-404
  polyeval_verify(ctx, p, gens, T, r, compress(commit1(gens.gens_1, Zr, Fq::zero())), comm);
}

// ---- R1CSProof::verify (r1csproof.rs:351-489)
void r1cs_verify(Ctx& ctx, const R1CSProof& p, size_t num_vars, size_t num_cons, const std::vector<Fq>& input, const Fq evals[3], Transcript& T,
                 const R1CSGens& gens, std::vector<Fq>& rx, std::vector<Fq>& ry) {
  T.append_protocol_name("R1CS proof");
  T.append_scalars("input", input);
  append_poly_commitment(T, "poly_commitment", p.comm_vars);
  const size_t num_rounds_x = log2_ceil(num_cons), num_rounds_y = log2_ceil(2 * num_vars);
  std::vector<Fq> tau = T.challenge_vector("challenge_tau", num_rounds_x);
  Cp claim_phase1 = compress(commit1(gens.gens_1, Fq::zero(), Fq::zero()));
  Cp comm_claim_post_phase1 = zk_sumcheck_verify(p.sc_proof_phase1, claim_phase1, num_rounds_x, 3, gens.gens_1, gens.gens_4, T, rx);
  const Cp &comm_Az = p.claims_phase2[0], &comm_Bz = p.claims_phase2[1], &comm_Cz = p.claims_phase2[2], &comm_prod = p.claims_phase2[3];
  knowledge_verify(p.pok_Cz, gens.gens_1, T, comm_Cz);
  product_verify(p.proof_prod, gens.gens_1, T, comm_Az, comm_Bz, comm_prod);
  append_claims_phase2(T, p.claims_phase2);
  Fq taus_bound_rx = eq_eval(rx, tau);
  Cp expected1 = compress(mul(hge_add(unpack(comm_prod, "comm_prod"), neg(unpack(comm_Cz, "comm_Cz"))), taus_bound_rx));
  equality_verify(p.proof_eq_sc_phase1, gens.gens_1, T, expected1, comm_claim_post_phase1);
  Fq r_A = T.challenge_scalar("challenge_Az"), r_B = T.challenge_scalar("challenge_Bz"), r_C = T.challenge_scalar("challenge_Cz");
  Cp comm_claim_phase2 = compress(hge_add(hge_add(mul(unpack(comm_Az, "comm_Az"), r_A), mul(unpack(comm_Bz, "comm_Bz"), r_B)), mul(unpack(comm_Cz, "comm_Cz"), r_C)));
  Cp comm_claim_post_phase2 = zk_sumcheck_verify(p.sc_proof_phase2, comm_claim_phase2, num_rounds_y, 2, gens.gens_1, gens.gens_3, T, ry);
  polyeval_verify(ctx, p.proof_eval_vars_at_ry, gens.gens_pc, T, std::vector<Fq>(ry.begin() + 1, ry.end()), p.comm_vars_at_ry, p.comm_vars);
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
  hge comm_eval_Z = hge_add(mul(unpack(p.comm_vars_at_ry, "comm_vars_at_ry"), Fq::one() - ry[0]), mul(commit1(gens.gens_pc.gens_1, poly_input_eval, Fq::zero()), ry[0]));
  Cp expected2 = compress(mul(comm_eval_Z, r_A * evals[0] + r_B * evals[1] + r_C * evals[2]));
  equality_verify(p.proof_eq_sc_phase2, gens.gens_1, T, expected2, comm_claim_post_phase2);
}

// ---- SPARK
struct BatchedOut { std::vector<Fq> claims, claims_dotp, rand; };
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
void spark_verify(Ctx& ctx, const SparseMatPolyEvalProof& p, const ComputationCommitment& comm, std::vector<Fq> rx, std::vector<Fq> ry,
                  const Fq evals[3], const SnarkGens& gens, Transcript& T) {
  T.append_protocol_name("Sparse polynomial evaluation proof");
  equalize(rx, ry);
  if (((size_t)1 << rx.size()) != comm.num_mem_cells) throw Reject("memory size");
  append_derefs_commitment(T, p.comm_derefs);
  std::vector<Fq> r_mem = T.challenge_vector("challenge_r_hash", 2);
  const Fq &r_hash = r_mem[0], &r_multiset = r_mem[1];
  T.append_protocol_name("Sparse polynomial evaluation proof");      // PolyEvalNetworkProof::protocol_name is the same string
  const size_t ni = 3, num_ops = next_pow2(comm.num_ops), num_cells = (size_t)1 << rx.size();
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
    polyeval_verify_plain(ctx, hl.proof_derefs, gens.gens_derefs, T, r_joint, joint, p.comm_derefs);
  }
  for (size_t i = 0; i < ni; i++)
    if (!(ops.claims_dotp[3 * i] == hl.derefs_row[i]) || !(ops.claims_dotp[3 * i + 1] == hl.derefs_col[i]) || !(ops.claims_dotp[3 * i + 2] == hl.eval_val[i]))
      throw Reject("dot product claims");
  {
    const std::vector<Fq> r_joint = combine_to_one(T, hl, HashOpening::ops, rand_ops, joint);
    polyeval_verify_plain(ctx, hl.proof_ops, gens.gens_ops, T, r_joint, joint, comm.comm_comb_ops);
  }
  {
    const std::vector<Fq> r_joint = combine_to_one(T, hl, HashOpening::mem, rand_mem, joint);
    polyeval_verify_plain(ctx, hl.proof_mem, gens.gens_mem, T, r_joint, joint, comm.comm_comb_mem);
  }
  hash_helper(rand_mem, mem.claims[0], row_read, row_write, mem.claims[1], hl.derefs_row, hl.row_addr, hl.row_read_ts, hl.row_audit_ts, rx, r_hash, r_multiset);
  hash_helper(rand_mem, mem.claims[2], col_read, col_write, mem.claims[3], hl.derefs_col, hl.col_addr, hl.col_read_ts, hl.col_audit_ts, ry, r_hash, r_multiset);
}

}  // namespace

static bool pow2(size_t x) { return x && !(x & (x - 1)); }
// shape sanity shared by both verifiers: the padded dimensions the prover enforces (lib.rs:129-198, r1csproof.rs:156); without it a
// hand-made commitment with num_vars = 0 or num_cons <= 1 would leave the round vectors empty (`.back()`, `ry[0]`)
static void check_dims(size_t num_cons, size_t num_vars, size_t num_inputs) {
  if (num_cons < 2 || num_vars < 1 || !pow2(num_cons) || !pow2(num_vars)) throw SpError(SP_ERR_INVALID_ARG, "verifier: num_cons >= 2 and num_vars >= 1 must be powers of two");
  if (!(num_inputs < num_vars)) throw SpError(SP_ERR_INVALID_ARG, "verifier: |input| + 1 must be at most the number of variables");
}

// NIZK::verify (lib.rs:549-591)
void nizk_verify(Ctx& ctx, const Instance& inst, const std::vector<Fq>& input, const R1CSGens& gens, Transcript& T, const uint8_t* proof, size_t len) {
  check_dims(inst.num_cons, inst.num_vars, inst.num_inputs);
  const NizkProof p = from_bincode<NizkProof>(proof, len, SP_ERR_VERIFY, "proof");
  if (input.size() != inst.num_inputs) throw Reject("number of inputs");
  if (p.rx.size() != log2_ceil(inst.num_cons) || p.ry.size() != log2_ceil(2 * inst.num_vars)) throw Reject("claimed evaluation point");
  append_nizk_head(T, inst);
  Fq evals[3];
  instance_evaluate(ctx, inst, p.rx, p.ry, evals);
  std::vector<Fq> rx, ry;
  r1cs_verify(ctx, p.r1cs_sat_proof, inst.num_vars, inst.num_cons, input, evals, T, gens, rx, ry);
  if (!(rx == p.rx) || !(ry == p.ry)) throw Reject("evaluation point differs from the sumcheck challenges");
}

// SNARK::verify (lib.rs:423-465); `enc` supplies the ComputationCommitment
void snark_verify(Ctx& ctx, const SnarkEncoding& enc, const std::vector<Fq>& input, const SnarkGens& gens, Transcript& T, const uint8_t* proof, size_t len) {
  const ComputationCommitment& comm = enc.comm;
  check_dims(comm.num_cons, comm.num_vars, comm.num_inputs);
  {  // SparseMatPolyCommitment consistency (sparse_mlpoly.rs:366-420): 3 matrices, power-of-two op count of at least 2 (what snark_encode
     // produces: one op leaves the product circuits without layers), cells = max(num_cons, 2*num_vars)
    const size_t cells = std::max(comm.num_cons, 2 * comm.num_vars);
    if (comm.batch_size != 3 || !pow2(comm.num_ops) || comm.num_ops < 2 || comm.num_mem_cells != cells)
      throw SpError(SP_ERR_INVALID_ARG, "verifier: inconsistent computation commitment");
  }
  const SnarkProof p = from_bincode<SnarkProof>(proof, len, SP_ERR_VERIFY, "proof");
  if (input.size() != comm.num_inputs) throw Reject("number of inputs");
  T.append_protocol_name("Spartan SNARK proof");
  append_computation_commitment(T, comm);
  const Fq* evals = p.inst_evals.data();
  std::vector<Fq> rx, ry;
  r1cs_verify(ctx, p.r1cs_sat_proof, comm.num_vars, comm.num_cons, input, evals, T, *gens.gens_r1cs_sat, rx, ry);
  T.append_scalar("Ar_claim", evals[0]);
  T.append_scalar("Br_claim", evals[1]);
  T.append_scalar("Cr_claim", evals[2]);
  spark_verify(ctx, p.r1cs_eval_proof, comm, rx, ry, evals, gens, T);
}

}  // namespace sp
