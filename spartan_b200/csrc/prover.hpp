// spartan_b200 — host prover: the GPU-driven R1CS / NIZK provers, and the protocol steps of theirs that the verifiers (verifier.cpp) run too.
// The proof structs and their bincode layout are in wire.hpp.
#pragma once
#include <functional>
#include <array>
#include <mutex>
#include "wire.hpp"

namespace sp {

// ---- generator bundles
struct PolyCommitmentGens {  // dense_mlpoly.rs:24-36 -> DotProductProofGens (nizk/mod.rs:407-419)
  size_t n = 0;              // gens_n.n = 2^ceil(ell/2)
  CommitKey gens_n, gens_1;
};
struct R1CSGens {  // r1csproof.rs:39-74
  std::shared_ptr<GenSet> set;   // the label's set this is a view into (gens_r1cs_sat of the tables, or a caller label's own set)
  PolyCommitmentGens gens_pc;
  CommitKey gens_1, gens_3, gens_4;
  // a view into tables.r1cs_sat for a num_vars (padded) circuit; SpError(SP_ERR_INVALID_ARG) when the set is too short or of another context
  R1CSGens(const Ctx* ctx, const GenTables& tables, size_t num_vars);
  // a view into a set of at least bases(num_vars) generators (checked by the caller); adds the host tables it needs
  R1CSGens(std::shared_ptr<GenSet> set, size_t num_vars);
  static size_t pc_n(size_t num_vars);                      // gens_pc.n
  static size_t bases(size_t num_vars);                     // generators of gens_r1cs_sat the view uses
  static std::vector<size_t> host_bases(size_t num_vars);   // the bases it needs host copies of
};
// num_vars as NIZKGens::new and SNARKGens::new pad it (lib.rs:288-294, :475-481)
inline size_t padded_num_vars(size_t num_vars, size_t num_inputs) { return next_pow2(std::max(num_vars, num_inputs + 1)); }

// ---- instance
struct SparseMatDev {  // one of A, B, C: COO (reference order), CSR and CSC on the device; a host copy of the COO only when asked for
  size_t nnz = 0;
  DevBuf<uint32_t> csr_ptr, csr_idx, csc_ptr, csc_idx, coo_row, coo_col;
  DevBuf<u256> csr_val, csc_val, coo_val;
  mutable std::vector<uint32_t> row, col;   // host COO: see Instance::host_coo
  mutable std::vector<Fq> val;
};
struct Instance {  // lib.rs:111-114 (R1CSShape + digest)
  size_t num_cons = 0, num_vars = 0, num_inputs = 0;
  SparseMatDev M[3];
  // R1CSShape::get_digest (r1cs.rs:154-158): zlib(level 6, miniz) of bincode(shape), computed on first use (deflate.cpp) unless the caller
  // supplied the bytes of its own compressor through sp_instance_set_digest
  mutable std::vector<uint8_t> digest;
  std::vector<uint8_t> shape_bincode() const;
  const std::vector<uint8_t>& shape_digest() const;
  // The device COO is authoritative.  The host copy is filled by one download on first use (the digest, export): a caller that only proves
  // SNARKs never moves the matrices to the host.  An instance built on the host (upload_coo) keeps its host copy from the start.
  void host_coo() const;
  void upload_coo(Ctx* ctx);   // host row / col / val -> device COO, nnz
  void finalize(Ctx* ctx);     // CSR and CSC from the device COO (returns once they are built)
 private:
  mutable bool host_ready = false;
  mutable std::mutex host_mu;
};

std::vector<uint8_t> miniz_zlib_level6(const uint8_t* data, size_t len);   // deflate.cpp

// The two products of the R1CS matrices A, B, C (num_cons x 2 num_vars, both powers of two) that R1CSProof::prove needs: inst.multiply_vec
// (r1cs.rs:268-282) in phase one and the weighted compute_eval_table_sparse (r1cs.rs:284-298) in phase two.  `sh`: the prover runs that phase's
// sumcheck on cyclic shards (Ctx::shard_table), and the outputs are this rank's n entries of each table.
struct R1csMatrices {
  size_t num_cons, num_vars;
  R1csMatrices(size_t nc, size_t nv) : num_cons(nc), num_vars(nv) {}
  virtual ~R1csMatrices() = default;
  // outs[m] = M_m z, z of 2 num_vars entries
  virtual void multiply_vec(Ctx& ctx, const u256* d_z, u256* const outs[3], size_t n, bool sh) const = 0;
  // out = w[0] A^T e + w[1] B^T e + w[2] C^T e, e of num_cons entries; d_w: 3 scalars of device scratch the weights may be staged in
  virtual void eval_table(Ctx& ctx, const u256* d_e, const Fq w[3], u256* d_w, u256* out, size_t n, bool sh) const = 0;
};
// an Instance's CSR / CSC copies through k_spmv (one thread per row or column), sharded when asked: the NIZK and SNARK provers' products
struct InstanceMatrices : R1csMatrices {
  const Instance& inst;
  explicit InstanceMatrices(const Instance& i);
  void multiply_vec(Ctx& ctx, const u256* d_z, u256* const outs[3], size_t n, bool sh) const override;
  void eval_table(Ctx& ctx, const u256* d_e, const Fq w[3], u256* d_w, u256* out, size_t n, bool sh) const override;
};

// R1CSProof::prove (r1csproof.rs:144-349).  d_vars: device array of num_vars Montgomery scalars (consumed read-only).
// hooks: called (when set) as soon as the first / the second sumcheck phase has produced its point, so that the caller can start work that
// depends only on rx / ry on another stream while the rest of the proof runs (SNARK::prove: the dereferenced SPARK values and their commitment)
struct R1csHooks { std::function<void(const std::vector<Fq>&)> on_rx, on_ry; };
void r1cs_prove(Ctx& ctx, const R1csMatrices& mats, const u256* d_vars, const std::vector<Fq>& input, const R1CSGens& gens, Transcript& T,
                RandomTape& tape, R1CSProof& proof, std::vector<Fq>& rx, std::vector<Fq>& ry, const R1csHooks* hooks = nullptr);
// R1CSProof::verify (r1csproof.rs:351-489) on bincode bytes with the Immediate checker (verifier.cpp): SpError(SP_ERR_VERIFY / SP_ERR_DECOMPRESS)
// naming the failing check.  evals: the claimed (A(rx, ry), B(rx, ry), C(rx, ry)).  Out: rx, ry
void r1cs_verify_bytes(Ctx& ctx, const uint8_t* proof, size_t len, size_t num_vars, size_t num_cons, const std::vector<Fq>& input, const Fq evals[3],
                       const R1CSGens& gens, Transcript& T, std::vector<Fq>& rx, std::vector<Fq>& ry);
// NIZK::prove (lib.rs:501-546)
void nizk_prove(Ctx& ctx, const Instance& inst, const u256* d_vars, const std::vector<Fq>& input, const R1CSGens& gens, Transcript& T,
                const Fq& tape_seed, NizkProof& out);

struct UniPoly {  // unipoly.rs
  std::vector<Fq> coeffs;
  static UniPoly from_evals(const std::vector<Fq>& e) {  // unipoly.rs:23-54
    static const Fq two_inv = Fq::from_u64(2).inv(), six_inv = Fq::from_u64(6).inv();
    UniPoly p;
    if (e.size() == 3) {
      Fq c = e[0];
      Fq a = two_inv * (e[2] - e[1] - e[1] + c);
      Fq b = e[1] - c - a;
      p.coeffs = {c, b, a};
    } else if (e.size() == 4) {
      Fq d = e[0];
      Fq a = six_inv * (e[3] - e[2] - e[2] - e[2] + e[1] + e[1] + e[1] - e[0]);
      Fq b = two_inv * (e[0] + e[0] - e[1] - e[1] - e[1] - e[1] - e[1] + e[2] + e[2] + e[2] + e[2] - e[3]);
      Fq c = e[1] - d - a - b;
      p.coeffs = {d, c, b, a};
    } else {
      p.coeffs = lagrange(e);
    }
    return p;
  }
  // the coefficients of the polynomial of degree < n through (i, e[i]), i = 0 .. n-1: sum_i e[i] prod_{j != i} (x - j) / (i - j).  It is unique, so
  // for n = 3, 4 it is what the closed forms above give
  static std::vector<Fq> lagrange(const std::vector<Fq>& e) {
    const size_t n = e.size();
    std::vector<Fq> out(n, Fq::zero());
    for (size_t i = 0; i < n; i++) {
      std::vector<Fq> num{Fq::one()};   // prod_{j != i} (x - j), lowest coefficient first
      Fq den = Fq::one();
      for (size_t j = 0; j < n; j++) {
        if (j == i) continue;
        const Fq fj = Fq::from_u64(j);
        std::vector<Fq> next(num.size() + 1, Fq::zero());
        for (size_t k = 0; k < num.size(); k++) { next[k + 1] += num[k]; next[k] -= num[k] * fj; }
        num.swap(next);
        den *= i > j ? Fq::from_u64(i - j) : -Fq::from_u64(j - i);
      }
      const Fq w = e[i] * den.inv();
      for (size_t k = 0; k < n; k++) out[k] += num[k] * w;
    }
    return out;
  }
  Fq evaluate(const Fq& r) const {  // unipoly.rs:72-80
    Fq ev = coeffs[0], power = r;
    for (size_t i = 1; i < coeffs.size(); i++) { ev += power * coeffs[i]; power *= r; }
    return ev;
  }
  CompressedUniPoly compress() const {  // unipoly.rs:82-88
    CompressedUniPoly c;
    c.coeffs_except_linear_term.push_back(coeffs[0]);
    for (size_t i = 2; i < coeffs.size(); i++) c.coeffs_except_linear_term.push_back(coeffs[i]);
    return c;
  }
  void append_to_transcript(const char* label, Transcript& T) const {  // unipoly.rs:112-120
    T.append_message(label, "UniPoly_begin");
    for (auto& c : coeffs) T.append_scalar("coeff", c);
    T.append_message(label, "UniPoly_end");
  }
};

void append_poly_commitment(Transcript& T, const char* label, const PolyCommitment& c);
// impl Commitments for Scalar / [Scalar] (commitments.rs:73-92): x*G + blind*h, sum x_i*G_i + blind*h, through the host tables (small n only)
hge commit1(const CommitKey& k, const Fq& x, const Fq& blind);
hge commitv(const CommitKey& k, const std::vector<Fq>& x, const Fq& blind);
// the weights a of round j's DotProductProof in a ZK sumcheck (sumcheck.rs:138-157, :535-554, :726-745): a_k = w0 * (k == 0 ? 2 : 1) + w1 * r_j^k, k = 0..degree
std::vector<Fq> zk_round_weights(const std::vector<Fq>& w, const Fq& r_j, size_t degree);
// the commitments to Az, Bz, Cz and Az*Bz at rx, absorbed after their sigma proofs (r1csproof.rs:245-248, :400-403)
void append_claims_phase2(Transcript& T, const std::array<Cp, 4>& c);
// NIZK::prove / verify before the R1CS proof: protocol name and R1CSShapeDigest (lib.rs:513-514, :558-559)
void append_nizk_head(Transcript& T, const Instance& inst);
// ---- sigma protocols (nizk/mod.rs), on the host over the host tables of the bases they commit against: g.off and g.h; DotProductProof also
// gn.off .. gn.off + n - 1.  Each returns the proof and, through the out-parameters, the commitments the reference returns alongside it.
KnowledgeProof knowledge_prove(const CommitKey& g, Transcript& T, RandomTape& tape, const Fq& x, const Fq& r, Cp& C_out);   // :27-52
EqualityProof equality_prove(const CommitKey& g, Transcript& T, RandomTape& tape, const Fq& v1, const Fq& s1, const Fq& v2, const Fq& s2,
                             Cp* C1_out = nullptr, Cp* C2_out = nullptr);   // :88-116
ProductProof product_prove(const CommitKey& g, Transcript& T, RandomTape& tape, const Fq& x, const Fq& rX, const Fq& y, const Fq& rY, const Fq& z,
                           const Fq& rZ, Cp& X, Cp& Y, Cp& Z);   // :159-229
// DotProductProof::prove (:311-370).  Cx_known: commit(x_vec; blind_x) when the caller already holds it.  pre: the tape draws made ahead of time
// in the reference's order, with the commitments that depend on the tape only (a ZK sumcheck's rounds)
struct DotPre { std::vector<Fq> d_vec; Fq r_delta, r_beta; Cp delta; hge r_beta_h; };
DotProductProof dotproduct_prove(const CommitKey& g1, const CommitKey& gn, Transcript& T, RandomTape& tape, const std::vector<Fq>& x_vec,
                                 const Fq& blind_x, const std::vector<Fq>& a_vec, const Fq& y, const Fq& blind_y, const Cp* Cx_known,
                                 const DotPre* pre = nullptr, Cp* Cx_out = nullptr, Cp* Cy_out = nullptr);
// their verifiers (verifier.cpp, the Immediate checker) on bincode bytes: SpError(SP_ERR_VERIFY / SP_ERR_DECOMPRESS) naming the failing check, the
// transcript advanced as the reference's verify advances it.  The caller's commitments (C, C1, .., Cy) must decompress.
void knowledge_verify_bytes(Ctx& ctx, const CommitKey& g, Transcript& T, const Cp& C, const uint8_t* proof, size_t len);
void equality_verify_bytes(Ctx& ctx, const CommitKey& g, Transcript& T, const Cp& C1, const Cp& C2, const uint8_t* proof, size_t len);
void product_verify_bytes(Ctx& ctx, const CommitKey& g, Transcript& T, const Cp& X, const Cp& Y, const Cp& Z, const uint8_t* proof, size_t len);
void dotproduct_verify_bytes(Ctx& ctx, const CommitKey& g1, const CommitKey& gn, Transcript& T, const std::vector<Fq>& a, const Cp& Cx, const Cp& Cy,
                             const uint8_t* proof, size_t len);
// ZKSumcheckInstanceProof::verify (sumcheck.rs:84-179): returns the last comm_eval, r the num_rounds (>= 1) challenges
Cp zk_sumcheck_verify_bytes(Ctx& ctx, const uint8_t* proof, size_t len, const Cp& comm_claim, size_t num_rounds, size_t degree, const CommitKey& g1,
                            const CommitKey& gn, Transcript& T, std::vector<Fq>& r);

// PolyEvalProof::prove (dense_mlpoly.rs:312-365) on a device-resident table.  Zr null: Zr = Z(r) = <LZ, eq(r[ell/2..])>, computed on the device
// from the bound rows (Z is not read again), and returned through Zr_out when that is set
void polyeval_prove(Ctx& ctx, const u256* d_Z, const std::vector<Fq>* blinds_opt, const std::vector<Fq>& r, const Fq* Zr, const Fq* blind_Zr_opt,
                    const PolyCommitmentGens& gens, Transcript& T, RandomTape& tape, PolyEvalProof& proof, Cp& C_Zr, Fq* Zr_out = nullptr);

// MultiCommitGens::new(n, label) (commitments.rs:15-33): point i is gens_from_uniform of bytes [64 i, 64 i + 64) of SHAKE256(label || basepoint).
// Points [0, n) are made in slabs of at most 2^18, so 2^24 points need no 1 GiB staging buffer.  They go to out[0, n) when out is given, else to
// a slab buffer of this call's; sink(i0, m, pts), when given, then receives points [i0, i0 + m) at pts on the device, valid until the sink's work
// on the context's stream has run.
void label_gens(Ctx& c, const std::string& label, size_t n, ge* out, const std::function<void(size_t i0, size_t m, const ge* pts)>& sink);

// ---- DotProductProofLog of the caller's vectors (sp_dotlog_*), on this rank's GPU alone
// DotProductProofGens::new(n, label) (nizk/mod.rs:414-419).  n <= SP_DOTLOG_TABLE_MAX_N: `set` holds the n + 2 generators with the window tables of
// sp_pc_gens_create's set and `g` views it, as PolyEvalProof's gens.  Larger n (folding()): `pts` holds G[0..n) as affine niels points, `set` the
// two generators {G_n, h} (host tables for the sigma terms), and g.gens_1 views it; g.gens_n is unused.
struct DotLogGens {
  Ctx* ctx;
  size_t n;
  std::unique_ptr<GenSet> set;
  PolyCommitmentGens g;
  DevBuf<ge_niels> pts;
  bool folding() const { return n > SP_DOTLOG_TABLE_MAX_N; }
  DotLogGens(Ctx& ctx, size_t n, const std::string& label);
};
// the largest half length whose round MSMs run as one segmented launch (msm_var_segmented, one thread per term) instead of the bucket MSM
constexpr size_t DOTLOG_SEG_MAX_HALF = 1024;
// DotProductProofLog::prove (nizk/mod.rs:440-525): d_x, d_a (n each) are read only; y null: <x, a> on the device.  Out: the proof, Cx, Cy, y_used
void dotlog_prove(Ctx& ctx, const DotLogGens& gens, Transcript& T, RandomTape& tape, const u256* d_x, const Fq& blind_x, const u256* d_a, const Fq* y,
                  const Fq& blind_y, DotProductProofLog& proof, Cp& Cx, Cp& Cy, Fq& y_used);
// DotProductProofLog::verify (nizk/mod.rs:527-583) on bincode bytes, with the Immediate checker (verifier.cpp): SpError(SP_ERR_VERIFY /
// SP_ERR_DECOMPRESS) naming the failing check.  d_a: the n entries of a on the device
void dotlog_verify_bytes(Ctx& ctx, const DotLogGens& gens, Transcript& T, const u256* d_a, const Cp& Cx, const Cp& Cy, const uint8_t* proof, size_t len);
// sum_i scalars[i] * pts[i] of n >= 1 terms (bucket MSM, Montgomery scalars on the device), to the host; synchronises
hge msm_var_host(Ctx& ctx, const ge_niels* pts, const u256* scalars, size_t n);
// a's entries as the canonical bytes the transcript absorbs (32 per entry), through the device
std::vector<uint8_t> canonical_bytes(Ctx& ctx, const u256* d_a, size_t n);

// ---- the caller's own tables (sp_pc_*): k tables of 2^m entries each, committed and opened as DensePolynomial::merge of them (dense_mlpoly.rs:259-272),
// on this rank's GPU alone
// PolyCommitmentGens::new(num_vars, label) (dense_mlpoly.rs:29-36): gens_n.n = 2^(num_vars - num_vars/2), n + 2 points of the label's stream
inline size_t pc_gens_n(size_t num_vars) { return (size_t)1 << (num_vars - num_vars / 2); }
PolyCommitmentGens pc_gens_view(GenSet& set, size_t num_vars);   // adds the host tables of bases n, n + 1 when missing
// The merge of k tables is 2^(m+c) entries, c = log2 next_pow2(k), split as a matrix of 2^floor((m+c)/2) rows of R = 2^ceil((m+c)/2).  A row lies
// inside one table when R <= 2^m: the device then reads the tables where they are.  Otherwise the merge has at most 2^12 entries (c <= 6) and is
// gathered into one buffer.
inline bool pc_rows_in_tables(size_t m, size_t c) { return (m + c + 1) / 2 <= m; }
// DensePolynomial::merge(tables).commit (dense_mlpoly.rs:179-204) with the row blinds `blinds` (L of them) or none (null)
PolyCommitment pc_commit(Ctx& ctx, const PolyCommitmentGens& gens, const u256* const* tables, int k, size_t m, const Fq* blinds);
// DerefsEvalProof::prove_single (sparse_mlpoly.rs:80-123), no protocol name: the k evaluations at r (out: evals) combined to one claim on the merge
// at (challenges || r), proved by PolyEvalProof::prove without blind_Zr.  blinds_opt: the merge's commitment blinds
void pc_eval_prove_joint(Ctx& ctx, const PolyCommitmentGens& gens, const u256* const* tables, int k, const std::vector<Fq>& r, const std::vector<Fq>* blinds_opt,
                         Transcript& T, RandomTape& tape, PolyEvalProof& proof, std::vector<Fq>& evals);
// the n-to-1 reduction of DerefsEvalProof / HashLayerProof (sparse_mlpoly.rs:80-123): evals padded to a power of two and absorbed, log2 of that many
// challenges, the evaluations folded by bound_poly_var_bot (last challenge first) into `joint`, which is absorbed; returns challenges || rand
std::vector<Fq> combine_to_one(Transcript& T, std::vector<Fq> evals, const std::vector<Fq>& rand, const char* label_evals, const char* label_challenge,
                               const char* label_joint, Fq& joint);
// PolyEvalProof::verify (C_Zr given) / verify_plain (Zr given) on bincode bytes, and DerefsEvalProof::verify_single (sparse_mlpoly.rs:149-176), with
// the Immediate checker (verifier.cpp): SpError(SP_ERR_VERIFY / SP_ERR_DECOMPRESS) naming the failing check
void pc_eval_verify(Ctx& ctx, const PolyCommitmentGens& gens, const PolyCommitment& comm, const std::vector<Fq>& r, const Cp* C_Zr, const Fq* Zr, Transcript& T,
                    const uint8_t* proof, size_t len);
void pc_eval_verify_joint(Ctx& ctx, const PolyCommitmentGens& gens, const PolyCommitment& comm, const std::vector<Fq>& r, const std::vector<Fq>& evals,
                          Transcript& T, const uint8_t* proof, size_t len);

// exposed pieces (C-ABI operator level and tests)
Cp commit_rows_and_compress(Ctx& ctx, const CommitKey& key, const u256* d_scalars, size_t stride, size_t L, size_t R, const Fq* blinds,
                            std::vector<Cp>& out, const std::function<const Fq*()>& blinds_late = nullptr);

// The device side of one inner-product round (bullet.rs:74-111) over the unfolded generators of `gs` (DESIGN.md "IPA without folding G"), run by
// DotProductProofLog's table layout (prover.cpp: DotLogTable) and by the operator-level sp_ipa_*.  launch() computes c_L = <a_L, b_R>, c_R = <a_R, b_L> and L' = <a_L, G_R>, R' = <a_R, G_L> in one
// kernel that publishes the two pairs to the host through separate flag words, so the host can work on c*Q while the MSM still runs.
// Scratch: >= ipa_msm_scratch_points(n, gs.wbits) points.
struct IpaRound {
  Ctx& ctx;
  const GenSet& gs;
  u256* a; u256* b;    // the current a, b (folded in place)
  u256* svec;          // the n running scalars of the unfolded generators
  size_t n;
  ge* pts;             // device copy of L', R'
  dev::HostSig sig_c, sig_lr;
  void launch(size_t cur);
  void wait_c(Fq& c_L, Fq& c_R);
  void wait_LR(ge& L, ge& R);
  void fold(size_t cur, const Fq& u, const Fq& u_inv);   // a, b, svec of the next round (bullet.rs:105-108)
};

// The device side of one sumcheck, or of a batch of instances proved together (prove_cubic_batched), run by zk_sumcheck_prove and batched_prove.
// An instance owns the tables t[0..4) that are set, except a t[2] it only reads (c_out != t[2]): a C shared by the batch, which one instance
// folds into c_out, where they all read it next round.  Sharded, the tables are this rank's cyclic shards until fold_eval leaves the sharded
// stage (DESIGN.md §6): once they are shorter than Ctx::SHARD_MIN_LOCAL it binds them, all-gathers them into replicated copies and evaluates there.
struct ScRounds {
  Ctx& ctx;
  dev::ScKind kind;
  std::vector<dev::ScInst> insts;
  size_t len;            // current length of the tables this rank holds
  bool sharded;
  u256* d_out;           // device result slot, 3 scalars per instance
  dev::HostSig sig;      // of the last launch that publishes evaluations
  void eval();                                              // evaluations of the current round
  void fold_eval(const Fq& r, u256* host_bound = nullptr);  // bind with r, evaluate the next round (host_bound: dev::sc_fold_eval)
  void fold(const Fq& r);                                   // bind the owned tables with r only
  std::vector<Fq> wait();                                   // the 3 ninst evaluations of the last launch
  std::vector<Fq> finals();                                 // t[k][0] of the first instance's tables t[0], t[1], .. (synchronises)
  dev::XRank xr();                                          // the cross-rank exchange of the next launch (none once replicated)
};

// A sumcheck of a caller-defined polynomial (sp_sumcheck_prove_t): SumcheckInstanceProof::prove_cubic (sumcheck.rs:183-252) with comb_func the
// sum of products P describes.  P.t: the distinct tables, `len` entries each, bound in place for num_rounds rounds.  Out: the proof, the challenges
// r, finals[k] = P.t[k][0] after the last bind, and the final claim e.  One launch per round (k_scp_eval, then k_scp_fold_eval as soon as r_j is
// drawn), then one bind and one gather of the first entries.  Single GPU.
void poly_sumcheck_prove(Ctx& ctx, const dev::ScPoly& P, size_t len, const Fq& claim, size_t num_rounds, Transcript& T, SumcheckInstanceProof& proof,
                         std::vector<Fq>& r, std::vector<Fq>& finals, Fq& e);
// The ZK sumcheck of the same polynomial (sp_zk_sumcheck_prove_t): ZKSumcheckInstanceProof::prove_quad / prove_cubic_with_additive_term
// (sumcheck.rs:428-776) with comb_func P, of degree d = P.degree, on the caller's transcript and tape.  g1: n = 1, gn: n = d + 1 (they may come from
// different generator sets); both need the host tables of the bases the rounds commit against (g1.off, g1.h, gn.off .. gn.off + d).  The rounds run
// on the device as poly_sumcheck_prove's do, one launch per round, with the host's sigma work of round j overlapping the launch of round j + 1.
// Out: the proof, r, finals as poly_sumcheck_prove's, blind_post = blinds_evals[num_rounds - 1].  Single GPU.
// the most rounds one ZK sumcheck stages its tape-only commitments for (a fixed pinned region of the context)
size_t zk_sumcheck_max_rounds();
void zk_poly_sumcheck_prove(Ctx& ctx, const dev::ScPoly& P, size_t len, const Fq& claim, const Fq& blind_claim, size_t num_rounds, const CommitKey& g1,
                            const CommitKey& gn, Transcript& T, RandomTape& tape, ZKSumcheckInstanceProof& proof, std::vector<Fq>& r,
                            std::vector<Fq>& finals, Fq& blind_post);
// SumcheckInstanceProof::verify (sumcheck.rs:27-62) on bincode bytes; SpError(SP_ERR_VERIFY) where the reference asserts or the bytes do not decode
Fq sumcheck_verify_bytes(const uint8_t* proof, size_t len, const Fq& claim, size_t num_rounds, size_t degree, Transcript& T, std::vector<Fq>& r);

// ---- product circuits (product.cpp): SPARK's memory check (snark_prove) and the caller's own (sp_prod_*)
// ProductCircuit (product_tree.rs:11-63): every layer kept; layer k has n/2^k entries (left half | right half).
// Single GPU: one 2n-scalar buffer, layer k at offset 2n - 2n/2^k.  Sharded over W ranks (cyclic partition: entry i of a layer on rank i mod W):
// the big layers [0, Ks) hold only this rank's n/(2^k W) entries (`loc`, same offset rule on the local sizes) — the Hadamard product that builds
// layer k+1 pairs i with i + len/2, which stay on one rank — and the layers from Ks on are replicated in `rep` (a circuit over n/2^Ks inputs).
struct ProdCircuit {
  DevBuf<u256> loc, rep;
  size_t n = 0, num_layers = 0, Ks = 0;
  int W = 1;
  void alloc(Ctx& ctx, size_t n_) {
    n = n_; num_layers = log2_ceil(n_); W = ctx.shard_world(); Ks = 0;
    // layer k's sumcheck runs on tables of n/2^(k+1) entries: shard it while those are worth sharding
    while (Ks + 1 < num_layers && ctx.shard_table((n >> Ks) / 2)) Ks++;
    if (Ks) loc.alloc(2 * (n / W));
    rep.alloc(2 * (n >> Ks));
  }
  bool sharded(size_t k) const { return k < Ks; }
  size_t layer_len(size_t k) const { return n >> k; }                                  // global entries
  size_t local_len(size_t k) const { return k < Ks ? (n >> k) / W : n >> k; }          // entries this rank holds
  u256* layer(size_t k) {
    if (k < Ks) { const size_t nl = n / W; return loc.p + (2 * nl - 2 * (nl >> k)); }
    const size_t nr = n >> Ks, kk = k - Ks;
    return rep.p + (2 * nr - 2 * (nr >> kk));
  }
};
// every layer after layer `from` of a group of at most 16 equally sized circuits whose layers up to `from` are built: one launch per layer
// (compute_layer, product_tree.rs:18-34); at the boundary between the sharded and the replicated layers the local products are all-gathered into
// every rank's copy
void build_circuits(Ctx& ctx, std::vector<ProdCircuit*> cs, size_t from = 0);
// DotProductCircuit (product_tree.rs:66-108) of `len` entries; the tables the sumcheck binds are this rank's cyclic shards when `sharded`
struct DotpCircuit { u256 *left, *right, *weight; size_t len; bool sharded; Fq claim; };
// ProductCircuitEvalProofBatched::prove (product_tree.rs:259-383) with SumcheckInstanceProof::prove_cubic_batched (sumcheck.rs:254-424) inlined.
// The product circuits' layers are bound in place.  rand_out: the point the proof ends on
void batched_prove(Ctx& ctx, std::vector<ProdCircuit*>& prods, std::vector<DotpCircuit>& dotps, Transcript& T, ProductCircuitEvalProofBatched& out,
                   std::vector<Fq>& rand_out);
// what ProductCircuitEvalProofBatched::verify (product_tree.rs:385-485; verifier.cpp: batched_verify) returns: the product circuits' claims about
// their leaf polynomials at rand, three claims per pair of dot-product circuits, and rand
struct BatchedOut { std::vector<Fq> claims, claims_dotp, rand; };
// ProductCircuitEvalProofBatched::verify(products, dotp_claims, 2^m, T) on bincode bytes (sp_prod_verify_t with no dotp claims,
// sp_prod_verify_dotp_t): SpError(SP_ERR_VERIFY) where the reference asserts or the bytes do not decode
BatchedOut prod_verify(const uint8_t* proof, size_t len, const std::vector<Fq>& products, const std::vector<Fq>& dotp_claims, size_t m, Transcript& T);
// the caller's dot products, each split into two DotpCircuits (d[2i], d[2i + 1]: the halves of dot product i) whose tables live in `ops`,
// [left | right | weight] of 2^m entries each per dot product; the claims are the halves' sums
struct ProdDotps { DevBuf<u256> ops; std::vector<DotpCircuit> d; };
// The caller's circuits (sp_prod_build, sp_prod_build_dotp): `leaves` without their layer pointers and `dotps` without their output pointers,
// k + 2 kd <= SP_PROD_MAX_CIRCUITS of them over tables of n = 2^m >= 2 entries, on this rank's GPU alone.  Allocates every circuit, writes the
// dot products' operands and half sums in one launch (dev::dotp_operands) when kd > 0, the leaves and the first product layer in one launch
// (dev::prod_leaves), the other layers with build_circuits in groups of at most 16, and returns the k products (ProductCircuit::evaluate)
std::vector<Fq> prod_build(Ctx& ctx, std::vector<dev::ProdLeaves> leaves, std::vector<dev::DotpOperands> dotps, size_t n,
                           std::vector<std::unique_ptr<ProdCircuit>>& out, ProdDotps& dout);
// ProductCircuitEvalProofBatched::prove(circuits, dotps, T) of the caller's circuits, on this rank's GPU alone; leaf_evals: each circuit's leaf
// polynomial at rand, the claims the verifier is left with; dotp_evals: (left, right, weight) at rand of each dot product (dotps holds its halves)
void prod_prove(Ctx& ctx, std::vector<ProdCircuit*>& cs, std::vector<DotpCircuit>& dotps, Transcript& T, ProductCircuitEvalProofBatched& out,
                std::vector<Fq>& rand, std::vector<Fq>& leaf_evals, std::vector<Fq>& dotp_evals);

// <x, G[0..n)> of one row of n scalars against the per-window table of `gs`, for latency.  For n >= 2 (even) it is the inner-product round kernel
// with a = (1, 1) and blocks of two generators: its "L" (odd j) and "R" (even j) reach the host through the kernel's own publication and are added
// there, one launch instead of msm_rows + reduce + compress + copy.  n = 1 runs msm_rows.  The constructor launches, collect() waits.
// Scratch: >= ipa_msm_scratch_points(n, gs.wbits) points, or msm_scratch_bytes(1, 1) bytes for n = 1.
struct RowSum {
  Ctx& ctx;
  size_t n;
  DevBuf<ge> pts;
  dev::HostSig sig;
  RowSum(Ctx& ctx, const GenSet& gs, const u256* d_x, size_t n);
  hge collect();
};
std::vector<Fq> host_eq_evals(const std::vector<Fq>& r);

}  // namespace sp
