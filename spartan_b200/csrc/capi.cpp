// spartan_b200 — extern "C" boundary (include/spartan_b200.h).  Every entry that can fail runs its body through guarded() or host_guarded(),
// which catch every exception and map it to a status code.
#include "../../include/spartan_b200.h"
#include <stdlib.h>
#include <algorithm>
#include <optional>
#include <sstream>
#include "prover.hpp"
#include "snark.hpp"

using namespace sp;

struct sp_ctx { Ctx c; explicit sp_ctx(int d) : c(d) {} };
struct sp_poly { Ctx* ctx; DevBuf<u256> d; size_t len; };
struct sp_gens { std::unique_ptr<GenSet> set; size_t n; };
struct sp_points { Ctx* ctx; DevBuf<ge_niels> pts; size_t n; mutable DevBuf<uint8_t> scratch; mutable size_t scratch_bytes = 0; };
struct sp_instance { Instance inst; };
struct sp_nizk_gens { std::unique_ptr<R1CSGens> g; };
struct sp_snark_gens { std::unique_ptr<SnarkGens> g; };
struct sp_snark_encoding { std::unique_ptr<SnarkEncoding> e; };
struct sp_gen_tables { std::unique_ptr<GenTables> t; };
struct sp_pc_gens {
  Ctx* ctx;
  std::shared_ptr<GenSet> set;   // shared by the views made from it
  size_t num_vars;
  PolyCommitmentGens g;
};
struct sp_dotlog_gens { Ctx* ctx; std::unique_ptr<DotLogGens> g; };
struct sp_spark_gens { Ctx* ctx; size_t x, y, nz, b; SparkGens g; };
struct sp_spark_dense { Ctx* ctx; SparkDense d; };
struct sp_prod_circuits {
  Ctx* ctx;
  size_t m;
  std::vector<std::unique_ptr<ProdCircuit>> cs;   // released by the proof
  bool spent;
  ProdDotps dotps;                                 // sp_prod_build_dotp's dot products, likewise
};

// the message sp_last_error(NULL) reads: of the last failed sp_ctx_create, or of the last failed host-only call made without a context
static std::string g_last_error;

// ---- the catch ladder.  host_guarded: entries without device work; the message goes to the context when one is given, else to g_last_error.
template <class F>
static int host_guarded(sp_ctx* ctx, const F& body) {
  std::string& err = ctx ? ctx->c.last_error : g_last_error;
  try {
    body();
    return SP_OK;
  } catch (const SpError& e) { err = e.what(); return e.code; }
  catch (const dev::CudaError& e) { err = e.what(); return SP_ERR_CUDA; }
  catch (const std::exception& e) { err = e.what(); return SP_ERR_INTERNAL; }
  catch (...) { err = "unknown error"; return SP_ERR_INTERNAL; }
}
// guarded: entries with a context, which start from refilled persistent scratch under the memory-check mode (Ctx::memcheck_refill)
template <class F>
static int guarded(sp_ctx* ctx, const F& body) {
  return host_guarded(ctx, [&] {
    if (ctx) ctx->c.memcheck_refill();
    body();
  });
}

// ---- scalars and results
static Fq fq_in(const uint64_t l[4]) { Fq f; memcpy(&f.m, l, 32); return f; }
static void fq_out(uint64_t l[4], const Fq& f) { memcpy(l, &f.m, 32); }
static std::vector<Fq> fq_vec(const uint64_t* l, size_t n) { std::vector<Fq> v(n); if (n) memcpy(v.data(), l, 32 * n); return v; }
// scalars that enter host arithmetic (public inputs, tape seed) must be reduced residues: limbs >= q are rejected at the boundary
static void require_reduced(const uint64_t* l, size_t n, const char* what) {
  for (size_t i = 0; i < n; i++)
    if (!fq_bytes_canonical(reinterpret_cast<const uint8_t*>(l + 4 * i))) throw SpError(SP_ERR_INVALID_SCALAR, std::string(what) + ": scalar limbs are not reduced modulo q");
}
// bytes handed to the caller, who releases them with sp_free
static void put_bytes(uint8_t** out, size_t* out_len, const std::vector<uint8_t>& v) {
  uint8_t* p = (uint8_t*)malloc(v.size() ? v.size() : 1);
  memcpy(p, v.data(), v.size());
  *out = p;
  *out_len = v.size();
}
static void put_scalars(uint64_t* out, const std::vector<Fq>& v) { if (!v.empty()) memcpy(out, v.data(), 32 * v.size()); }

// ---- argument checks shared by the caller-facing entries
static void require_count(const std::string& what, int k, const char* noun, const char* max_name, int max) {
  if (k < 1 || k > max)
    throw SpError(SP_ERR_INVALID_ARG, what + ": " + std::to_string(k) + " " + noun + "; 1 .. " + max_name + " = " + std::to_string(max) + " supported");
}
// a handle the call reads: not NULL, and made on this context
template <class H>
static void require_owned(const sp_ctx* ctx, const H* h, const std::string& what, const std::string& name) {
  if (!h) throw SpError(SP_ERR_INVALID_ARG, what + ": " + name + " is NULL");
  if (h->ctx != &ctx->c) throw SpError(SP_ERR_INVALID_ARG, what + ": " + name + " belongs to another context");
}
// the k >= 1 tables of one call: handles of this context, of one power-of-two length >= min_len
struct Tables { size_t len; std::vector<const u256*> d; };
static Tables caller_tables(const sp_ctx* ctx, sp_poly* const* polys, int k, const std::string& what, size_t min_len) {
  if (!polys) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL table array");
  Tables t{0, std::vector<const u256*>(k)};
  for (int i = 0; i < k; i++) {
    require_owned(ctx, polys[i], what, "table " + std::to_string(i));
    if (polys[i]->len != polys[0]->len) throw SpError(SP_ERR_INVALID_ARG, what + ": tables differ in length");
    t.d[i] = polys[i]->d.p;
  }
  t.len = polys[0]->len;
  if (t.len < min_len || (t.len & (t.len - 1)))
    throw SpError(SP_ERR_INVALID_ARG, what + ": the table length must be a power of two >= " + std::to_string(min_len) + ", got " + std::to_string(t.len));
  return t;
}

// ---- transcripts, tapes and witnesses of the proof entries
// The transcript and tape of a proof entry.  The transcript is a fresh Transcript::new(label) or (the _t entry points) the caller's STROBE state,
// updated in place; the tape, for the entries that draw from one, is the caller's tape state.  A NULL state is refused when this is made, before
// the entry's other checks; open() reads the states after those checks, and refuses one that is not a STROBE state.  The entries that take their
// tape later (the polynomial-evaluation and SPARK proofs, after their argument checks) pass it to open_tape() at that point instead, where a NULL or
// bad tape state is refused.  A prove writes both back with proved(), on success alone, so a refused prove leaves them as they were.  A verify
// opens with open_verify(): its transcript goes back to the caller on every exit, whether the proof is accepted or not.
class ProofStates {
 public:
  struct Label { const uint8_t* p; size_t n; };
  explicit ProofStates(Label label) : label_(label) {}
  explicit ProofStates(uint8_t* strobe_state) : state_(strobe_state) {
    if (!state_) throw SpError(SP_ERR_INVALID_ARG, "transcript state is NULL");
  }
  ProofStates(uint8_t* strobe_state, uint8_t* tape_state, const std::string& what) : ProofStates(strobe_state) {
    tape_state_ = checked_tape(tape_state, what);
  }
  // no transcript, and the caller's tape when one is given (sp_pc_commit: NULL draws no blinds)
  static ProofStates tape_only(uint8_t* tape_state) { return ProofStates(tape_state, false); }
  ProofStates(const ProofStates&) = delete;
  ~ProofStates() { if (verifying_) T_->export_state(state_); }

  void open() {
    if (transcript_) T_.emplace(state_ ? Transcript(Transcript::FromState(), state_) : Transcript(std::string((const char*)label_.p, label_.n)));
    if (tape_state_ && !tape_) tape_.emplace(Transcript(Transcript::FromState(), tape_state_));
  }
  void open_tape(uint8_t* tape_state, const std::string& what) {
    tape_state_ = checked_tape(tape_state, what);
    tape_.emplace(Transcript(Transcript::FromState(), tape_state_));
  }
  void open_verify() { open(); verifying_ = state_ != nullptr; }
  void proved() const {
    if (state_) T_->export_state(state_);
    if (tape_state_) tape_->state().export_state(tape_state_);
  }
  Transcript& T() { return *T_; }
  RandomTape& tape() { return *tape_; }

 private:
  ProofStates(uint8_t* tape_state, bool transcript) : transcript_(transcript), tape_state_(tape_state) {}
  static uint8_t* checked_tape(uint8_t* tape_state, const std::string& what) {
    if (!tape_state) throw SpError(SP_ERR_INVALID_ARG, what + ": tape state is NULL");
    return tape_state;
  }
  bool transcript_ = true, verifying_ = false;
  Label label_{nullptr, 0};
  uint8_t* state_ = nullptr;
  uint8_t* tape_state_ = nullptr;
  std::optional<Transcript> T_;
  std::optional<RandomTape> tape_;
};
static DevBuf<u256> upload_padded_vars(Ctx& c, const Instance& I, const uint64_t* vars, size_t nvars) {
  if (nvars > I.num_vars) throw SpError(SP_ERR_INVALID_INPUTS, "R1CSError::InvalidNumberOfInputs (vars)");
  DevBuf<u256> d(I.num_vars);
  dev::h2d(d.p, vars, nvars * 32, c.stream);
  if (nvars < I.num_vars) dev::dzero(d.p + nvars, (I.num_vars - nvars) * 32, c.stream);  // Assignment::pad (lib.rs:91-104)
  return d;
}
// the witness of a prove call: the caller's host limbs, padded on upload (Assignment::pad), or a resident poly already padded to num_vars
struct VarsArg { const uint64_t* host; size_t nvars; const sp_poly* resident; };
static const u256* vars_on_device(Ctx& c, const Instance& I, const VarsArg& v, DevBuf<u256>& upload) {
  if (!v.resident) { upload = upload_padded_vars(c, I, v.host, v.nvars); return upload.p; }
  if (v.resident->len != I.num_vars) throw SpError(SP_ERR_INVALID_INPUTS, "resident vars must already be padded to num_vars");
  return v.resident->d.p;
}
// The body NIZK and SNARK proofs share.  `transcript`: a ProofStates::Label or the caller's transcript state.  `prove(d_vars, inputs, T, seed)`
// runs the statement's own prover and returns the proof's bincode.
template <class Src, class Prove>
static void prove_statement(Ctx& c, const Instance& I, const VarsArg& vars, const uint64_t* inputs, size_t ninputs, const Src& transcript,
                            const uint64_t seed[4], uint8_t** proof, size_t* proof_len, const Prove& prove) {
  ProofStates st(transcript);
  DevBuf<u256> upload;
  const u256* d_vars = vars_on_device(c, I, vars, upload);
  if (ninputs != I.num_inputs) throw SpError(SP_ERR_INVALID_INPUTS, "R1CSError::InvalidNumberOfInputs");
  if (!seed) throw SpError(SP_ERR_INVALID_ARG, "tape seed is NULL: draw it from the OS RNG (random.rs:13-15); a fixed seed makes every blind public");
  require_reduced(inputs, ninputs, "inputs"); require_reduced(seed, 1, "tape seed");
  st.open();
  const std::vector<uint8_t> bytes = prove(d_vars, fq_vec(inputs, ninputs), st.T(), fq_in(seed));
  st.proved();
  put_bytes(proof, proof_len, bytes);
}
// SP_FINE_TIMERS=1: the sub-phase timers of the last verify call (single or batch) replace sp_timings, as a prove call's do
static void flush_fine(Ctx& c) {
  if (!FineTimer::enabled()) return;
  c.timings.clear();
  for (auto& f : c.fine) c.timings.push_back({"fine:" + f.first, f.second});
  c.fine.clear();
}
// The body NIZK and SNARK verification share.  `verify(inputs, T)` runs the statement's own verifier.
template <class Src, class Verify>
static int verify_statement(sp_ctx* ctx, const uint64_t* inputs, size_t ninputs, const Src& transcript, const Verify& verify) {
  return guarded(ctx, [&] {
    ProofStates st(transcript);
    require_reduced(inputs, ninputs, "inputs");
    st.open_verify();
    verify(fq_vec(inputs, ninputs), st.T());
    flush_fine(ctx->c);
  });
}

template <class Src>
static int nizk_prove_common(sp_ctx* ctx, const sp_instance* inst, const VarsArg& vars, const uint64_t* inputs, size_t ninputs, const sp_nizk_gens* gens,
                             const Src& transcript, const uint64_t seed[4], uint8_t** proof, size_t* proof_len) {
  return guarded(ctx, [&] {
    prove_statement(ctx->c, inst->inst, vars, inputs, ninputs, transcript, seed, proof, proof_len, [&](const u256* d_vars, const std::vector<Fq>& in, Transcript& T, const Fq& s) {
      NizkProof P;
      nizk_prove(ctx->c, inst->inst, d_vars, in, *gens->g, T, s, P);
      return to_bincode(P);
    });
  });
}
template <class Src>
static int snark_prove_common(sp_ctx* ctx, const sp_instance* inst, const sp_snark_encoding* enc, const VarsArg& vars, const uint64_t* inputs, size_t ninputs,
                              const sp_snark_gens* gens, const Src& transcript, const uint64_t seed[4], uint8_t** proof, size_t* proof_len) {
  return guarded(ctx, [&] {
    if (!enc->e->dense.comb_ops.p) throw SpError(SP_ERR_INVALID_ARG, "this handle holds a commitment only (sp_snark_commitment_load): proving needs sp_snark_encode");
    prove_statement(ctx->c, inst->inst, vars, inputs, ninputs, transcript, seed, proof, proof_len, [&](const u256* d_vars, const std::vector<Fq>& in, Transcript& T, const Fq& s) {
      SnarkProof P;
      snark_prove(ctx->c, inst->inst, *enc->e, d_vars, in, *gens->g, T, s, P);
      return to_bincode(P);
    });
  });
}
template <class Src>
static int nizk_verify_common(sp_ctx* ctx, const sp_instance* inst, const uint64_t* inputs, size_t ninputs, const sp_nizk_gens* gens, const Src& transcript,
                              const uint8_t* proof, size_t proof_len) {
  return verify_statement(ctx, inputs, ninputs, transcript, [&](const std::vector<Fq>& in, Transcript& T) { nizk_verify(ctx->c, inst->inst, in, *gens->g, T, proof, proof_len); });
}
template <class Src>
static int snark_verify_common(sp_ctx* ctx, const sp_snark_encoding* comm, const uint64_t* inputs, size_t ninputs, const sp_snark_gens* gens,
                               const Src& transcript, const uint8_t* proof, size_t proof_len) {
  return verify_statement(ctx, inputs, ninputs, transcript, [&](const std::vector<Fq>& in, Transcript& T) { snark_verify(ctx->c, *comm->e, in, *gens->g, T, proof, proof_len); });
}

// ---- batch verifiers: proof i is checked as the single call would check it (statement i, inputs i, label i or caller transcript i); the group
// equations of all of them are tested in one device pass (verifier.cpp, DESIGN.md "deferred checks")
struct BatchArgs {
  size_t k;
  const uint64_t* const* inputs; const size_t* ninputs;
  const uint8_t* const* labels; const size_t* label_lens;   // fresh transcripts, or
  uint8_t* const* states;                                    // the callers' transcripts (the _t forms)
  const uint8_t* const* proofs; const size_t* proof_lens;
  const uint8_t* seed; int* status;
};
static std::vector<VerifyJob> batch_jobs(const BatchArgs& a, const void* const* stmts) {
  const bool bad_transcripts = a.states ? false : (!a.labels || !a.label_lens);
  if (!stmts || !a.inputs || !a.ninputs || !a.proofs || !a.proof_lens || !a.status || bad_transcripts)
    throw SpError(SP_ERR_INVALID_ARG, "verify_batch: NULL array");
  std::vector<VerifyJob> jobs;
  jobs.reserve(a.k);
  for (size_t i = 0; i < a.k; i++) {
    const std::string at = "verify_batch: proof " + std::to_string(i) + ": ";
    if (!stmts[i]) throw SpError(SP_ERR_INVALID_ARG, at + "NULL statement handle");
    if (!a.proofs[i] && a.proof_lens[i]) throw SpError(SP_ERR_INVALID_ARG, at + "NULL proof");
    if (!a.inputs[i] && a.ninputs[i]) throw SpError(SP_ERR_INVALID_ARG, at + "NULL inputs");
    require_reduced(a.inputs[i], a.ninputs[i], "inputs");
    if (a.states && !a.states[i]) throw SpError(SP_ERR_INVALID_ARG, at + "transcript state is NULL");
    Transcript T = a.states ? Transcript(Transcript::FromState(), a.states[i]) : Transcript(std::string((const char*)a.labels[i], a.label_lens[i]));
    jobs.push_back(VerifyJob{nullptr, nullptr, fq_vec(a.inputs[i], a.ninputs[i]), T, a.proofs[i], a.proof_lens[i]});
  }
  return jobs;
}
// statuses and transcripts out; SP_ERR_VERIFY with the first rejection's message when any proof is rejected
static void batch_finish(Ctx& c, const BatchArgs& a, const std::vector<VerifyJob>& jobs) {
  size_t first = a.k;
  for (size_t i = 0; i < a.k; i++) {
    a.status[i] = jobs[i].status;
    if (a.states) jobs[i].T.export_state(a.states[i]);
    if (jobs[i].status != SP_OK && first == a.k) first = i;
  }
  flush_fine(c);
  if (first < a.k) throw SpError(SP_ERR_VERIFY, "proof " + std::to_string(first) + ": " + jobs[first].msg);
}
// The body NIZK and SNARK batch verification share.  `verify(jobs)` points the jobs at their statements and verifies them.
template <class Verify>
static int verify_batch(sp_ctx* ctx, const void* const* stmts, const void* gens, const BatchArgs& a, const Verify& verify) {
  return guarded(ctx, [&] {
    if (!a.seed) throw SpError(SP_ERR_INVALID_ARG, "verify_batch: weight seed is NULL: draw 32 bytes from the OS RNG on every call");
    if (!a.k) return;
    if (!gens) throw SpError(SP_ERR_INVALID_ARG, "verify_batch: NULL gens");
    std::vector<VerifyJob> jobs = batch_jobs(a, stmts);
    verify(jobs);
    batch_finish(ctx->c, a, jobs);
  });
}

// ---- polynomial commitments of the caller's tables
// gens of this context whose n is the row length R = 2^ceil(ell/2) of a table of 2^ell entries (commitments.rs:87-91 asserts gens_n.n == R)
static void pc_check_gens(const sp_ctx* ctx, const sp_pc_gens* g, size_t ell, const std::string& what) {
  require_owned(ctx, g, what, "gens handle");
  if (g->g.n != pc_gens_n(ell))
    throw SpError(SP_ERR_INVALID_ARG, what + ": gens for num_vars = " + std::to_string(g->num_vars) + " have n = " + std::to_string(g->g.n) +
                                          ", a table of 2^" + std::to_string(ell) + " entries needs n = R = " + std::to_string(pc_gens_n(ell)));
}
static const size_t PC_MAX_VARS = 60;

// ---- product circuits of the caller's tables
static const size_t PROD_MAX_VARS = 60;
// one circuit's leaf form, checked: leaf[x] = cst + idx * x + sum_s coeff[s] * table[src[s]][x]
struct LeafForm { uint32_t nsrc = 0; uint32_t src[SP_PROD_MAX_SOURCES] = {}; Fq coeff[SP_PROD_MAX_SOURCES], idx = Fq::zero(), cst = Fq::zero(); };
static void prod_counts(const sp_prod_leaves* leaves, int k, int ntables, const std::string& what) {
  require_count(what, k, "circuits", "SP_PROD_MAX_CIRCUITS", SP_PROD_MAX_CIRCUITS);
  if (ntables < 1) throw SpError(SP_ERR_INVALID_ARG, what + ": " + std::to_string(ntables) + " tables; at least one needed");
  if (!leaves && k != ntables)
    throw SpError(SP_ERR_INVALID_ARG, what + ": leaves NULL (circuit i = table i) needs k = ntables, got k = " + std::to_string(k) + ", ntables = " + std::to_string(ntables));
}
// the k forms of `leaves` checked: every count and source first (SP_ERR_INVALID_ARG), then every scalar (SP_ERR_INVALID_SCALAR).  name(c): what a
// message calls form c.  leaves NULL: form c is table c
template <class Name>
static std::vector<LeafForm> checked_forms(const sp_prod_leaves* leaves, int k, int ntables, const Name& name) {
  std::vector<LeafForm> f(k);
  for (int c = 0; c < k; c++) {
    if (!leaves) { f[c].nsrc = 1; f[c].src[0] = (uint32_t)c; f[c].coeff[0] = Fq::one(); continue; }
    const sp_prod_leaves& l = leaves[c];
    const std::string at = name(c);
    if (l.nsources > SP_PROD_MAX_SOURCES)
      throw SpError(SP_ERR_INVALID_ARG, at + " has " + std::to_string(l.nsources) + " sources; at most SP_PROD_MAX_SOURCES = " + std::to_string(SP_PROD_MAX_SOURCES));
    for (uint32_t s = 0; s < l.nsources; s++)
      if (l.source[s] >= (uint32_t)ntables)
        throw SpError(SP_ERR_INVALID_ARG, at + ": source " + std::to_string(s) + " is table " + std::to_string(l.source[s]) + " >= ntables = " + std::to_string(ntables));
  }
  if (leaves)
    for (int c = 0; c < k; c++) {
      const sp_prod_leaves& l = leaves[c];
      const std::string at = name(c);
      require_reduced(&l.coeff_mont[0][0], l.nsources, (at + ": coefficient").c_str());
      require_reduced(l.index_coeff_mont, 1, (at + ": index coefficient").c_str());
      require_reduced(l.const_mont, 1, (at + ": constant").c_str());
      f[c].nsrc = l.nsources;
      for (uint32_t s = 0; s < l.nsources; s++) { f[c].src[s] = l.source[s]; f[c].coeff[s] = fq_in(l.coeff_mont[s]); }
      f[c].idx = fq_in(l.index_coeff_mont);
      f[c].cst = fq_in(l.const_mont);
    }
  return f;
}
static std::vector<LeafForm> prod_forms(const sp_prod_leaves* leaves, int k, int ntables, const std::string& what) {
  prod_counts(leaves, k, ntables, what);
  return checked_forms(leaves, k, ntables, [&](int c) { return what + ": circuit " + std::to_string(c); });
}
// the caller's dot products next to k circuits: 1 <= kd and k + 2 kd <= SP_PROD_MAX_CIRCUITS (the circuits and both halves of every dot product
// are instances of one batched sumcheck launch)
static void dotp_counts(int k, int kd, const std::string& what) {
  if (kd < 1 || k + 2 * (int64_t)kd > SP_PROD_MAX_CIRCUITS)
    throw SpError(SP_ERR_INVALID_ARG, what + ": " + std::to_string(kd) + " dot products next to " + std::to_string(k) + " circuits; 1 <= kd and k + 2 kd <= SP_PROD_MAX_CIRCUITS = " +
                                          std::to_string(SP_PROD_MAX_CIRCUITS) + " supported");
}
static const char* const DOTP_OPERAND[3] = {"left", "right", "weight"};
// a checked form on the device: its sources resolved to the tables' device pointers
static dev::AffineForm device_form(const LeafForm& f, sp_poly* const* tables) {
  dev::AffineForm p;
  memset(static_cast<void*>(&p), 0, sizeof p);
  const Fq one = Fq::one();
  p.nsrc = f.nsrc;
  for (uint32_t s = 0; s < f.nsrc; s++) {
    p.src[s] = tables[f.src[s]]->d.p;
    p.coeff[s] = f.coeff[s].m;
    if (f.coeff[s] == one) p.flags |= dev::PROD_UNIT0 << s;
  }
  p.idx = f.idx.m; p.cst = f.cst.m;
  if (!f.idx.is_zero()) p.flags |= dev::PROD_IDX;
  if (!f.cst.is_zero()) p.flags |= dev::PROD_CST;
  return p;
}

// ---- the caller's sparse matrices
static void require_device(const Ctx& c, const void* p, size_t n, const char* what) {
  if (n && !dev::is_device_pointer(p, c.device))
    throw SpError(SP_ERR_INVALID_ARG, std::string(what) + ": not device memory of the context's GPU (device " + std::to_string(c.device) + ")");
}
// the word a checking kernel leaves: ~0 before `launch(err)` runs on the stream, read back after it (~0: nothing failed)
template <class Launch>
static unsigned long long first_fault(Ctx& c, const Launch& launch) {
  DevBuf<unsigned long long> err(1);
  dev::set_max_u64(err.p, c.stream);
  launch(err.p);
  unsigned long long first = 0;
  dev::d2h(&first, err.p, sizeof(first), c.stream);
  c.sync();
  return first;
}
// The entries of nmat matrices, host arrays (copied to the device as they are) or device arrays, through the ingestion kernel into out.  The caller's
// arrays are read by those copies (host) or by the kernel (device) only, and both have finished when this returns or throws.  A bad entry:
// refuse(matrix, entry, code) words the refusal of the first one in (matrix, entry) order, within it row, then column, then scalar (code:
// dev::INGEST_*), and throws.
template <class Refuse>
static void ingest(Ctx& c, dev::CooIn in, int nmat, bool on_host, const dev::CooOut& out, size_t num_rows, size_t num_cols, size_t num_vars, size_t shift,
                   const Refuse& refuse) {
  DevBuf<uint64_t> d_row[dev::INGEST_MAX_MATRICES], d_col[dev::INGEST_MAX_MATRICES];
  DevBuf<uint8_t> d_val[dev::INGEST_MAX_MATRICES];
  for (int m = 0; on_host && m < nmat; m++) {
    d_row[m].alloc(in.n[m]); d_col[m].alloc(in.n[m]); d_val[m].alloc(32 * in.n[m]);
    dev::h2d(d_row[m].p, in.row[m], in.n[m] * sizeof(uint64_t), c.stream);
    dev::h2d(d_col[m].p, in.col[m], in.n[m] * sizeof(uint64_t), c.stream);
    dev::h2d(d_val[m].p, in.val[m], 32 * in.n[m], c.stream);
    in.row[m] = d_row[m].p; in.col[m] = d_col[m].p; in.val[m] = d_val[m].p;
  }
  const unsigned long long first =
      first_fault(c, [&](unsigned long long* err) { dev::inst_ingest(in, nmat, out, num_rows, num_cols, num_vars, shift, err, c.stream); });
  if (first != ~0ull) refuse((size_t)(first >> 42), (size_t)((first >> 2) & ((1ull << 40) - 1)), (unsigned)(first & 3));
}
// the refusal of entry k of matrix m of a SPARK or product batch
[[noreturn]] static void refuse_entry(const std::string& what, size_t m, size_t k, unsigned code) {
  const std::string at = " (matrix " + std::to_string(m) + ", entry " + std::to_string(k) + ")";
  if (code == dev::INGEST_ROW) throw SpError(SP_ERR_INVALID_INDEX, what + ": row out of range" + at);
  if (code == dev::INGEST_COL) throw SpError(SP_ERR_INVALID_INDEX, what + ": col out of range" + at);
  throw SpError(SP_ERR_INVALID_SCALAR, what + ": value not a canonical scalar" + at);
}

extern "C" {

int sp_device_count(void) { return dev::device_count(); }
int sp_ctx_create(int device, sp_ctx** out) {
  try {
    if (dev::device_count() <= device) { g_last_error = "no CUDA device (spartan_b200 has no CPU fallback)"; return SP_ERR_NO_DEVICE; }
    *out = new sp_ctx(device);
    return SP_OK;
  } catch (const std::exception& e) { g_last_error = e.what(); return SP_ERR_CUDA; }
}
void sp_ctx_destroy(sp_ctx* ctx) { delete ctx; }
const char* sp_last_error(const sp_ctx* ctx) { return ctx ? ctx->c.last_error.c_str() : g_last_error.c_str(); }
unsigned long long sp_kernel_launches(void) { return dev::launch_count(); }
unsigned long long sp_release_cached_memory(void) { return dev::pool_release_cached(); }
void sp_debug_memcheck(int on) { dev::memcheck_enable(on != 0); }
int sp_debug_memcheck_report(sp_memcheck_counts* out, char* violations, size_t buflen) {
  std::string first, last;
  const dev::MemcheckStats s = dev::memcheck_stats(&first, &last);
  if (out) *out = sp_memcheck_counts{s.blocks_filled, s.blocks_refilled, s.context_refills, s.guard_bytes_checked, s.violations};
  if (!violations) return SP_OK;
  const std::string text = first.empty() ? "" : first + "\n" + last;
  if (text.size() + 1 > buflen) return SP_ERR_INVALID_ARG;
  memcpy(violations, text.c_str(), text.size() + 1);
  return SP_OK;
}
unsigned long long sp_debug_memcheck_scan(void) {
  try { return dev::memcheck_scan(); } catch (const std::exception& e) { g_last_error = e.what(); return ~0ull; }
}
int sp_timings(sp_ctx* ctx, char* buf, size_t buflen) {
  std::ostringstream os;
  for (auto& t : ctx->c.timings) os << t.first << "=" << t.second << ";";
  std::string s = os.str();
  if (s.size() + 1 > buflen) return SP_ERR_INVALID_ARG;
  memcpy(buf, s.c_str(), s.size() + 1);
  return SP_OK;
}

// ---- intra-proof sharding: one process per GPU, windows exchanged as CUDA IPC handles by whatever transport the host has
size_t sp_comm_handle_bytes(void) { return dev::ipc_handle_bytes(); }
int sp_comm_export(sp_ctx* ctx, uint8_t* handle_out) {
  return guarded(ctx, [&] {
    ctx->c.comm_create();
    if (ctx->c.comm->connected) throw SpError(SP_ERR_INVALID_ARG, "communicator already connected");
    ctx->c.comm->export_handle(handle_out);
  });
}
int sp_comm_connect(sp_ctx* ctx, int rank, int world, const uint8_t* handles) {
  return guarded(ctx, [&] {
    if (!ctx->c.comm) throw SpError(SP_ERR_INVALID_ARG, "sp_comm_export must be called first (it creates the window whose handle the peers map)");
    ctx->c.comm->connect(rank, world, handles);
  });
}
int sp_comm_set_enabled(sp_ctx* ctx, int enabled) { ctx->c.shard_enabled = enabled != 0; return SP_OK; }
int sp_ctx_set_overlap(sp_ctx* ctx, int enabled) { ctx->c.overlap = enabled != 0; return SP_OK; }
int sp_comm_info(const sp_ctx* ctx, int* rank, int* world) { *rank = ctx->c.rank(); *world = ctx->c.world(); return SP_OK; }

void sp_io_bytes(unsigned long long* h, unsigned long long* d) { dev::io_bytes(h, d); }
void sp_prof_enable(int on) { dev::prof_enable(on != 0); }
int sp_prof_report(char* buf, size_t buflen) {
  std::string s = dev::prof_report();
  if (s.size() + 1 > buflen) return SP_ERR_INVALID_ARG;
  memcpy(buf, s.c_str(), s.size() + 1);
  return SP_OK;
}
int sp_timer_start(sp_ctx* ctx) {
  return guarded(ctx, [&] {
    if (!ctx->c.ev_a) { ctx->c.ev_a = dev::event_create(); ctx->c.ev_b = dev::event_create(); }   // events belong to the context (device)
    dev::event_record(ctx->c.ev_a, ctx->c.stream);
    ctx->c.timer_running = true;
  });
}
int sp_timer_stop_ms(sp_ctx* ctx, float* ms) {
  return guarded(ctx, [&] {
    if (!ctx->c.timer_running) throw SpError(SP_ERR_INVALID_ARG, "sp_timer_stop_ms without sp_timer_start");
    dev::event_record(ctx->c.ev_b, ctx->c.stream);
    *ms = dev::event_elapsed_ms(ctx->c.ev_a, ctx->c.ev_b);
    ctx->c.timer_running = false;
  });
}

// ---- scalars
int sp_scalar_from_bytes(const uint8_t b[32], uint64_t out[4]) {
  Fq f(fq_to_mont(bytes_to_u256(b)));
  fq_out(out, f);
  return fq_bytes_canonical(b) ? SP_OK : SP_ERR_INVALID_SCALAR;
}
void sp_scalar_to_bytes(const uint64_t m[4], uint8_t out[32]) { fq_in(m).to_bytes(out); }
void sp_scalar_from_bytes_wide(const uint8_t w[64], uint64_t out[4]) { fq_out(out, Fq::from_bytes_wide(w)); }
void sp_scalar_mul(const uint64_t a[4], const uint64_t b[4], uint64_t out[4]) { fq_out(out, fq_in(a) * fq_in(b)); }
void sp_scalar_add(const uint64_t a[4], const uint64_t b[4], uint64_t out[4]) { fq_out(out, fq_in(a) + fq_in(b)); }
void sp_scalar_sub(const uint64_t a[4], const uint64_t b[4], uint64_t out[4]) { fq_out(out, fq_in(a) - fq_in(b)); }
int sp_scalar_invert(const uint64_t a[4], uint64_t out[4]) {
  Fq x = fq_in(a);
  fq_out(out, x.inv());
  return x.is_zero() ? SP_ERR_INVALID_SCALAR : SP_OK;
}

// ---- polys
int sp_poly_upload(sp_ctx* ctx, const uint64_t* limbs, size_t len, sp_poly** out) {
  return guarded(ctx, [&] {
    std::unique_ptr<sp_poly> p(new sp_poly{&ctx->c, DevBuf<u256>(len), len});
    dev::h2d(p->d.p, limbs, len * 32, ctx->c.stream);
    ctx->c.sync();
    *out = p.release();
  });
}
int sp_poly_download(sp_ctx* ctx, const sp_poly* p, uint64_t* limbs, size_t len) {
  return guarded(ctx, [&] {
    if (len > p->d.n) throw SpError(SP_ERR_INVALID_ARG, "download length exceeds allocation");
    dev::d2h(limbs, p->d.p, len * 32, ctx->c.stream);
    ctx->c.sync();
  });
}
size_t sp_poly_len(const sp_poly* p) { return p->len; }
void sp_poly_free(sp_poly* p) { delete p; }

static void check_same_len(sp_poly* const* polys, int k) {
  for (int i = 1; i < k; i++) if (polys[i]->len != polys[0]->len) throw SpError(SP_ERR_INVALID_ARG, "polynomials differ in length");
  if (polys[0]->len < 2 || (polys[0]->len & (polys[0]->len - 1))) throw SpError(SP_ERR_INVALID_ARG, "length must be a power of two >= 2");
}
int sp_fold_top(sp_ctx* ctx, sp_poly* const* polys, int k, const uint64_t r[4]) {
  return guarded(ctx, [&] {
    if (k < 1) throw SpError(SP_ERR_INVALID_ARG, "fold_top: no polynomials");
    check_same_len(polys, k);
    for (int i = 0; i < k; i++) for (int j = 0; j < i; j++) if (polys[i] == polys[j]) throw SpError(SP_ERR_INVALID_ARG, "fold_top: the same polynomial passed twice");
    Fq rr = fq_in(r);
    std::vector<u256*> t(k);
    for (int i = 0; i < k; i++) t[i] = polys[i]->d.p;
    dev::fold_top(t.data(), k, polys[0]->len, rr.m, ctx->c.stream);
    ctx->c.sync();
    for (int i = 0; i < k; i++) polys[i]->len /= 2;
  });
}
static int kind_tables(int kind) { return kind == 0 ? 2 : kind == 1 ? 3 : 4; }
static dev::ScInst make_inst(sp_poly* const* polys, int nt) {
  dev::ScInst in;
  for (int t = 0; t < 4; t++) in.t[t] = t < nt ? polys[t]->d.p : nullptr;
  in.c_out = in.t[2];
  in.write_c = 1;
  return in;
}
// sharded: the same calls on a connected context (sp_comm_connect), every rank passing its CYCLIC SHARDS of the tables (rank r holds the entries
// r, r+W, r+2W, ...): the kernels exchange their partial sums over NVLink and every rank receives the evaluations of the whole tables.
// Binding the top variable stays local as long as the local length is >= 2; shards must be of streaming size (>= 8192 entries) for fold_eval.
static int sumcheck_tables(Ctx& c, int kind, sp_poly* const* polys, bool sharded) {
  if (sharded && c.world() < 2) throw SpError(SP_ERR_INVALID_ARG, "not a connected multi-GPU context");
  if (kind < 0 || kind > 2) throw SpError(SP_ERR_INVALID_ARG, "bad sumcheck kind");
  const int nt = kind_tables(kind);
  check_same_len(polys, nt);
  return nt;
}
// sharded: the kernel's cross-rank completion counter and the next exchange (every rank issues it in the same order)
static dev::HostSig xr_sig(Ctx& c, bool sharded) { dev::HostSig s; if (sharded) s.done = c.sig_done.p + layout::SIG_DONE.off; return s; }
static int sumcheck_eval(sp_ctx* ctx, int kind, sp_poly* const* polys, uint64_t out[3][4], bool sharded) {
  return guarded(ctx, [&] {
    Ctx& c = ctx->c;
    const int nt = sumcheck_tables(c, kind, polys, sharded);
    dev::ScInst in = make_inst(polys, nt);
    dev::sc_eval((dev::ScKind)kind, &in, 1, polys[0]->len, c.small.p + layout::SMALL_ROUND.off, c.red.p, c.stream, xr_sig(c, sharded), sharded ? c.comm->next_xr() : dev::XRank());
    c.get_small(layout::SMALL_ROUND.off, reinterpret_cast<Fq*>(out), 3);
  });
}
static int sumcheck_fold_eval(sp_ctx* ctx, int kind, sp_poly* const* polys, const uint64_t r[4], uint64_t out[3][4], bool sharded) {
  return guarded(ctx, [&] {
    Ctx& c = ctx->c;
    const int nt = sumcheck_tables(c, kind, polys, sharded);
    if (polys[0]->len < (sharded ? Ctx::SHARD_MIN_LOCAL : 4))
      throw SpError(SP_ERR_INVALID_ARG, sharded ? "sharded fold_eval needs shards of at least 8192 entries (gather the shards and finish on one GPU)"
                                                : "fold_eval needs length >= 4");
    Fq rr = fq_in(r);
    dev::ScInst in = make_inst(polys, nt);
    dev::sc_fold_eval((dev::ScKind)kind, &in, 1, polys[0]->len, rr.m, c.small.p + layout::SMALL_ROUND.off, c.red.p, c.stream, xr_sig(c, sharded), sharded ? c.comm->next_xr() : dev::XRank());
    c.get_small(layout::SMALL_ROUND.off, reinterpret_cast<Fq*>(out), 3);
    for (int i = 0; i < nt; i++) polys[i]->len /= 2;
  });
}
int sp_sumcheck_eval(sp_ctx* ctx, int kind, sp_poly* const* polys, uint64_t out[3][4]) { return sumcheck_eval(ctx, kind, polys, out, false); }
int sp_sumcheck_fold_eval(sp_ctx* ctx, int kind, sp_poly* const* polys, const uint64_t r[4], uint64_t out[3][4]) {
  return sumcheck_fold_eval(ctx, kind, polys, r, out, false);
}
int sp_sumcheck_eval_sharded(sp_ctx* ctx, int kind, sp_poly* const* polys, uint64_t out[3][4]) { return sumcheck_eval(ctx, kind, polys, out, true); }
int sp_sumcheck_fold_eval_sharded(sp_ctx* ctx, int kind, sp_poly* const* polys, const uint64_t r[4], uint64_t out[3][4]) {
  return sumcheck_fold_eval(ctx, kind, polys, r, out, true);
}
// prove_cubic_batched's evaluation loops (sumcheck.rs:290-357): ninst instances of A*B*C; an sp_poly may serve as C of several instances
// (the shared eq table poly_C_par) — it is then bound once, through a temporary, and copied back
static void batched_insts(sp_ctx* ctx, int ninst, sp_poly* const* A, sp_poly* const* B, sp_poly* const* Cc, std::vector<dev::ScInst>& insts,
                          std::vector<std::pair<sp_poly*, std::unique_ptr<DevBuf<u256>>>>& shared, bool fold) {
  if (ninst < 1 || ninst > dev::SC_MAX_INST) throw SpError(SP_ERR_INVALID_ARG, "batched sumcheck: 1.." + std::to_string(dev::SC_MAX_INST) + " instances");
  const size_t len = A[0]->len;
  if (len < 2 || (len & (len - 1))) throw SpError(SP_ERR_INVALID_ARG, "length must be a power of two >= 2");
  for (int i = 0; i < ninst; i++) {
    if (A[i]->len != len || B[i]->len != len || Cc[i]->len != len) throw SpError(SP_ERR_INVALID_ARG, "polynomials differ in length");
    for (int j = 0; j < ninst; j++)
      if (A[i] == B[j] || A[i] == Cc[j] || B[i] == Cc[j] || (i != j && (A[i] == A[j] || B[i] == B[j])))
        throw SpError(SP_ERR_INVALID_ARG, "batched sumcheck: only the C table may be shared between instances");
  }
  insts.resize(ninst);
  for (int i = 0; i < ninst; i++) {
    dev::ScInst& in = insts[i];
    in.t[0] = A[i]->d.p; in.t[1] = B[i]->d.p; in.t[2] = Cc[i]->d.p; in.t[3] = nullptr;
    in.c_out = in.t[2]; in.write_c = 1;
    if (!fold) continue;
    int users = 0, first = -1;
    for (int j = 0; j < ninst; j++) if (Cc[j] == Cc[i]) { users++; if (first < 0) first = j; }
    if (users > 1) {
      DevBuf<u256>* tmp = nullptr;
      for (auto& sh : shared) if (sh.first == Cc[i]) tmp = sh.second.get();
      if (!tmp) { shared.push_back({Cc[i], std::unique_ptr<DevBuf<u256>>(new DevBuf<u256>(len / 2))}); tmp = shared.back().second.get(); }
      in.c_out = tmp->p;
      in.write_c = first == i;
    }
  }
  (void)ctx;
}
int sp_sumcheck_batched_eval(sp_ctx* ctx, int ninst, sp_poly* const* A, sp_poly* const* B, sp_poly* const* Cc, uint64_t* out) {
  return guarded(ctx, [&] {
    std::vector<dev::ScInst> insts;
    std::vector<std::pair<sp_poly*, std::unique_ptr<DevBuf<u256>>>> shared;
    batched_insts(ctx, ninst, A, B, Cc, insts, shared, false);
    DevBuf<u256> d_out(3 * ninst);
    dev::sc_eval(dev::SC_CUBIC3, insts.data(), ninst, A[0]->len, d_out.p, ctx->c.red.p, ctx->c.stream);
    dev::d2h(out, d_out.p, 96 * (size_t)ninst, ctx->c.stream);
    ctx->c.sync();
  });
}
int sp_sumcheck_batched_fold_eval(sp_ctx* ctx, int ninst, sp_poly* const* A, sp_poly* const* B, sp_poly* const* Cc, const uint64_t r[4], uint64_t* out) {
  return guarded(ctx, [&] {
    if (ninst < 1 || ninst > dev::SC_MAX_INST) throw SpError(SP_ERR_INVALID_ARG, "batched sumcheck: 1.." + std::to_string(dev::SC_MAX_INST) + " instances");
    if (A[0]->len < 4) throw SpError(SP_ERR_INVALID_ARG, "fold_eval needs length >= 4");
    std::vector<dev::ScInst> insts;
    std::vector<std::pair<sp_poly*, std::unique_ptr<DevBuf<u256>>>> shared;
    batched_insts(ctx, ninst, A, B, Cc, insts, shared, true);
    Fq rr = fq_in(r);
    DevBuf<u256> d_out(3 * ninst);
    const size_t len = A[0]->len;
    dev::sc_fold_eval(dev::SC_CUBIC3, insts.data(), ninst, len, rr.m, d_out.p, ctx->c.red.p, ctx->c.stream);
    for (auto& sh : shared) dev::d2d(sh.first->d.p, sh.second->p, (len / 2) * sizeof(u256), ctx->c.stream);
    dev::d2h(out, d_out.p, 96 * (size_t)ninst, ctx->c.stream);
    ctx->c.sync();
    std::vector<sp_poly*> seen;
    for (int i = 0; i < ninst; i++)
      for (sp_poly* p : {A[i], B[i], Cc[i]})
        if (std::find(seen.begin(), seen.end(), p) == seen.end()) { seen.push_back(p); p->len /= 2; }
  });
}
int sp_eq_evals(sp_ctx* ctx, const uint64_t* r, size_t ell, sp_poly** out) {
  return guarded(ctx, [&] {
    size_t n = (size_t)1 << ell;
    std::unique_ptr<sp_poly> p(new sp_poly{&ctx->c, DevBuf<u256>(n), n});
    DevBuf<u256> d_r(ell + 1), small(dev::eq_evals_scratch(ell));
    dev::h2d(d_r.p, r, ell * 32, ctx->c.stream);
    dev::eq_evals(p->d.p, d_r.p, (int)ell, small.p, ctx->c.stream);
    ctx->c.sync();
    *out = p.release();
  });
}
int sp_poly_evaluate(sp_ctx* ctx, const sp_poly* p, const uint64_t* r, size_t ell, uint64_t out[4]) {
  return guarded(ctx, [&] {
    if (p->len != (size_t)1 << ell) throw SpError(SP_ERR_INVALID_ARG, "evaluate: |r| != num_vars");
    DevBuf<u256> d_r(ell + 1), small(dev::eq_evals_scratch(ell)), eq(p->len);
    dev::h2d(d_r.p, r, ell * 32, ctx->c.stream);
    dev::eq_evals(eq.p, d_r.p, (int)ell, small.p, ctx->c.stream);
    dev::dot(ctx->c.small.p + layout::SMALL_DOT.off, p->d.p, eq.p, p->len, ctx->c.red.p, ctx->c.stream);
    Fq v;
    ctx->c.get_small(layout::SMALL_DOT.off, &v, 1);
    fq_out(out, v);
  });
}
int sp_poly_bound_rows(sp_ctx* ctx, const sp_poly* p, const uint64_t* Lm, size_t L_size, sp_poly** out) {
  return guarded(ctx, [&] {
    if (L_size == 0 || p->len % L_size) throw SpError(SP_ERR_INVALID_ARG, "bound: L does not divide the length");
    size_t R_size = p->len / L_size;
    std::unique_ptr<sp_poly> o(new sp_poly{&ctx->c, DevBuf<u256>(R_size), R_size});
    DevBuf<u256> d_L(L_size), tmp(64 * R_size);
    dev::h2d(d_L.p, Lm, L_size * 32, ctx->c.stream);
    dev::bound_rows(o->d.p, p->d.p, d_L.p, L_size, R_size, tmp.p, ctx->c.stream);
    ctx->c.sync();
    *out = o.release();
  });
}
int sp_dot(sp_ctx* ctx, const sp_poly* a, const sp_poly* b, uint64_t out[4]) {
  return guarded(ctx, [&] {
    if (a->len != b->len) throw SpError(SP_ERR_INVALID_ARG, "dot: length mismatch");
    dev::dot(ctx->c.small.p + layout::SMALL_DOT.off, a->d.p, b->d.p, a->len, ctx->c.red.p, ctx->c.stream);
    Fq v;
    ctx->c.get_small(layout::SMALL_DOT.off, &v, 1);
    fq_out(out, v);
  });
}

// ---- gens / commitments
int sp_gens_create(sp_ctx* ctx, const uint8_t* label, size_t label_len, size_t n, sp_gens** out) {
  return guarded(ctx, [&] {
    std::unique_ptr<sp_gens> g(new sp_gens);
    g->n = n;
    g->set.reset(new GenSet(&ctx->c, std::string((const char*)label, label_len), n + 1, {}));
    *out = g.release();
  });
}
// n ristretto255 encodings -> device points.  ok == null: an encoding that is not a point is an SP_ERR_INVALID_POINT naming its index
// (`what`); otherwise ok[i] tells whether encoding i is a point.
static DevBuf<ge> decode_points(Ctx& c, const uint8_t* in32, size_t n, const char* what, int* ok = nullptr) {
  DevBuf<uint8_t> d_in(32 * n + 1);
  DevBuf<ge> pts(n + 1);
  DevBuf<int> d_ok(n + 1);
  std::vector<int> h_ok(ok ? 0 : n);
  dev::h2d(d_in.p, in32, 32 * n, c.stream);
  dev::decompress_batch(pts.p, d_ok.p, d_in.p, n, c.stream);
  dev::d2h(ok ? ok : h_ok.data(), d_ok.p, sizeof(int) * n, c.stream);
  c.sync();
  for (size_t i = 0; i < h_ok.size(); i++)
    if (!h_ok[i]) throw SpError(SP_ERR_INVALID_POINT, std::string(what) + ": encoding " + std::to_string(i) + " is not a ristretto255 point");
  return pts;
}
int sp_gens_upload(sp_ctx* ctx, const uint8_t* compressed32, size_t n, sp_gens** out) {
  return guarded(ctx, [&] {
    DevBuf<ge> g = decode_points(ctx->c, compressed32, n + 1, "gens_upload");
    std::unique_ptr<sp_gens> G(new sp_gens);
    G->n = n;
    G->set.reset(new GenSet(&ctx->c, g.p, n + 1, {}));
    *out = G.release();
  });
}
void sp_gens_free(sp_gens* g) { delete g; }
int sp_gens_export(sp_ctx* ctx, const sp_gens* g, uint8_t* out32) {
  return guarded(ctx, [&] {
    DevBuf<uint8_t> comp(32 * (g->n + 1));
    dev::compress_batch(comp.p, g->set->G.p, g->n + 1, ctx->c.stream);
    dev::d2h(out32, comp.p, 32 * (g->n + 1), ctx->c.stream);
    ctx->c.sync();
  });
}
int sp_msm(sp_ctx* ctx, const sp_gens* g, const uint64_t* scalars, size_t n, uint8_t out32[32]) {
  return guarded(ctx, [&] {
    if (n > g->n) throw SpError(SP_ERR_INVALID_ARG, "msm: more scalars than generators");
    DevBuf<u256> d(n ? n : 1);
    dev::h2d(d.p, scalars, n * 32, ctx->c.stream);
    CommitKey key{g->set.get(), 0, g->n, g->n};
    std::vector<Cp> out;
    commit_rows_and_compress(ctx->c, key, d.p, n, 1, n, nullptr, out);
    memcpy(out32, out[0].b, 32);
  });
}
int sp_commit_rows(sp_ctx* ctx, const sp_gens* g, const sp_poly* p, size_t L, size_t R, const uint64_t* blinds, uint8_t* out32) {
  return guarded(ctx, [&] {
    if (L * R != p->len || R > g->n) throw SpError(SP_ERR_INVALID_ARG, "commit_rows: shape mismatch");
    CommitKey key{g->set.get(), 0, g->n, g->n};
    std::vector<Fq> bl;
    if (blinds) bl = fq_vec(blinds, L);
    std::vector<Cp> out;
    commit_rows_and_compress(ctx->c, key, p->d.p, R, L, R, blinds ? bl.data() : nullptr, out);
    memcpy(out32, out.data(), 32 * L);
  });
}
int sp_point_decompress_check(sp_ctx* ctx, const uint8_t* in32, size_t n, int* ok) {
  return guarded(ctx, [&] { decode_points(ctx->c, in32, n, nullptr, ok); });
}
int sp_point_roundtrip(sp_ctx* ctx, const uint8_t* in32, size_t n, uint8_t* out32) {
  return guarded(ctx, [&] {
    DevBuf<uint8_t> d_in(32 * n), d_out(32 * n);
    DevBuf<ge> pts(n);
    dev::h2d(d_in.p, in32, 32 * n, ctx->c.stream);
    dev::decompress_batch(pts.p, nullptr, d_in.p, n, ctx->c.stream);
    dev::compress_batch(d_out.p, pts.p, n, ctx->c.stream);
    dev::d2h(out32, d_out.p, 32 * n, ctx->c.stream);
    ctx->c.sync();
  });
}

// ---- inner-product argument, operator level: BulletReductionProof::prove (nizk/bullet.rs:32-132) with the host keeping the transcript.
// One handle per reduction: a_vec / b_vec (consumed), the generator set G (with its fixed-base tables) and the running scalars s of the
// unfolded-G formulation (DESIGN.md "IPA without folding G").  Per round: sp_ipa_round_LR (bullet.rs:78-97) -> transcript -> sp_ipa_fold (:105-111).
struct sp_ipa {
  Ctx* ctx; const GenSet* gs; size_t n, cur;
  DevBuf<u256> a, b, svec;
  DevBuf<ge> pts;
};
static hge point_in(const uint8_t p32[32], const char* what) {
  ge g;
  if (!ristretto_decode(g, bytes_to_u256(p32))) throw SpError(SP_ERR_INVALID_POINT, std::string(what) + " is not a ristretto255 point");
  return to_hge(g);
}
int sp_ipa_begin(sp_ctx* ctx, const sp_gens* gens, const sp_poly* a_vec, const sp_poly* b_vec, sp_ipa** out) {
  return guarded(ctx, [&] {
    const size_t n = a_vec->len;
    if (n < 1 || (n & (n - 1)) || b_vec->len != n || n > gens->n) throw SpError(SP_ERR_INVALID_ARG, "ipa: |a| = |b| = a power of two, at most the generator count");
    std::unique_ptr<sp_ipa> h(new sp_ipa);
    h->ctx = &ctx->c; h->gs = gens->set.get(); h->n = n; h->cur = n;
    h->a.alloc(n); h->b.alloc(n); h->svec.alloc(n); h->pts.alloc(2);
    dev::d2d(h->a.p, a_vec->d.p, n * sizeof(u256), ctx->c.stream);
    dev::d2d(h->b.p, b_vec->d.p, n * sizeof(u256), ctx->c.stream);
    dev::fill_one(h->svec.p, n, ctx->c.stream);
    // the fused round launch and, for n >= 2, the one-row sum of sp_ipa_finish run on ipa_msm scratch; n = 1 runs msm_rows
    ctx->c.ensure_scratch(std::max(dev::msm_scratch_bytes(1, n), dev::ipa_msm_scratch_points(n, gens->set->wbits) * sizeof(sp::ge)) + 64);
    ctx->c.sync();
    *out = h.release();
  });
}
void sp_ipa_free(sp_ipa* h) { delete h; }
static IpaRound ipa_round(sp_ipa* h) { return IpaRound{*h->ctx, *h->gs, h->a.p, h->b.p, h->svec.p, h->n, h->pts.p}; }
// L = <a_L, G_R> + c_L*Q + blind_L*H,  R = <a_R, G_L> + c_R*Q + blind_R*H  with c_L = <a_L, b_R>, c_R = <a_R, b_L>   (bullet.rs:74-97)
int sp_ipa_round_LR(sp_ctx* ctx, sp_ipa* h, const uint8_t Q32[32], const uint8_t H32[32], const uint64_t blind_L[4], const uint64_t blind_R[4], uint8_t L32[32],
                    uint8_t R32[32]) {
  return guarded(ctx, [&] {
    if (h->cur < 2) throw SpError(SP_ERR_INVALID_ARG, "ipa: the reduction is complete");
    const hge Q = point_in(Q32, "Q"), H = point_in(H32, "H");
    IpaRound rd = ipa_round(h);
    rd.launch(h->cur);
    Fq cc[2];
    rd.wait_c(cc[0], cc[1]);
    ge lr[2];
    rd.wait_LR(lr[0], lr[1]);
    const Fq bl[2] = {fq_in(blind_L), fq_in(blind_R)};
    Cp outp[2];
    hge full[2];
    for (int k = 0; k < 2; k++) full[k] = hge_add(to_hge(lr[k]), hge_add(hge_scalarmul(cc[k].canonical(), Q), hge_scalarmul(bl[k].canonical(), H)));
    compress2(full[0], full[1], outp[0], outp[1]);
    memcpy(L32, outp[0].b, 32); memcpy(R32, outp[1].b, 32);
  });
}
// a_L <- a_L*u + u^-1*a_R,  b_L <- b_L*u^-1 + u*b_R,  G_L <- u^-1*G_L + u*G_R (kept implicit in s)      (bullet.rs:105-108)
int sp_ipa_fold(sp_ctx* ctx, sp_ipa* h, const uint64_t u[4], const uint64_t u_inv[4]) {
  return guarded(ctx, [&] {
    if (h->cur < 2) throw SpError(SP_ERR_INVALID_ARG, "ipa: the reduction is complete");
    const Fq uu = fq_in(u), ui = fq_in(u_inv);
    if (!(uu * ui == Fq::one())) throw SpError(SP_ERR_INVALID_SCALAR, "ipa: u_inv is not the inverse of u");
    ipa_round(h).fold(h->cur, uu, ui);
    h->cur /= 2;
    ctx->c.sync();
  });
}
// a[0], b[0] and G[0] of the fully folded vectors (bullet.rs:113-122: the caller forms Gamma_hat from them)
int sp_ipa_finish(sp_ctx* ctx, sp_ipa* h, uint64_t a_hat[4], uint64_t b_hat[4], uint8_t G_hat32[32]) {
  return guarded(ctx, [&] {
    Ctx& c = ctx->c;
    if (h->cur != 1) throw SpError(SP_ERR_INVALID_ARG, "ipa: rounds remain");
    dev::d2h(a_hat, h->a.p, 32, c.stream);
    dev::d2h(b_hat, h->b.p, 32, c.stream);
    const Cp G = compress(RowSum(c, *h->gs, h->svec.p, h->n).collect());
    memcpy(G_hat32, G.b, 32);
  });
}

// ---- variable-base MSM (kernels_pip.cu)
static void points_from_ge(sp_ctx* ctx, sp_points* P, const ge* d_ge, size_t n) {
  P->ctx = &ctx->c; P->n = n;
  P->pts.alloc(n ? n : 1);
  dev::points_to_niels(P->pts.p, d_ge, n, ctx->c.stream);
}
int sp_points_upload(sp_ctx* ctx, const uint8_t* in32, size_t n, sp_points** out) {
  return guarded(ctx, [&] {
    DevBuf<ge> g = decode_points(ctx->c, in32, n, "points_upload");
    std::unique_ptr<sp_points> P(new sp_points);
    points_from_ge(ctx, P.get(), g.p, n);
    ctx->c.sync();
    *out = P.release();
  });
}
int sp_points_derive(sp_ctx* ctx, const uint8_t* label, size_t label_len, size_t n, sp_points** out) {
  return guarded(ctx, [&] {
    std::unique_ptr<sp_points> P(new sp_points);
    P->ctx = &ctx->c; P->n = n;
    P->pts.alloc(n ? n : 1);
    label_gens(ctx->c, std::string((const char*)label, label_len), n, nullptr,
               [&](size_t i0, size_t m, const ge* pts) { dev::points_to_niels(P->pts.p + i0, pts, m, ctx->c.stream); });
    *out = P.release();
  });
}
size_t sp_points_len(const sp_points* p) { return p->n; }
void sp_points_free(sp_points* p) { delete p; }
// [offset, offset + n) inside the point set, without forming offset + n (a caller's offset of 2^64 - 1 wraps it)
static void points_range(const sp_points* p, size_t offset, size_t n, const char* what) {
  if (offset > p->n || n > p->n - offset) throw SpError(SP_ERR_INVALID_ARG, std::string(what) + ": range outside the point set");
}
int sp_points_export(sp_ctx* ctx, const sp_points* p, size_t offset, size_t n, uint8_t* out32) {
  return guarded(ctx, [&] {
    points_range(p, offset, n, "points_export");
    if (n) {   // 1 * P_i through the MSM path's own mixed addition, then compress (no empty launch for n = 0)
      DevBuf<ge> g(n);
      DevBuf<uint8_t> comp(32 * n);
      dev::niels_to_ge(g.p, p->pts.p + offset, n, ctx->c.stream);
      dev::compress_batch(comp.p, g.p, n, ctx->c.stream);
      dev::d2h(out32, comp.p, 32 * n, ctx->c.stream);
      ctx->c.sync();
    }
  });
}
// sharded: the MSM split over the ranks of a connected context.  Every rank passes ITS slice of the points (offset, scalars->len) and of the
// scalars; the partial sums meet in a point-add all-reduce (all-gather of the W extended points into every window, W-term sum) and every rank
// returns the same encoding of the sum over all ranks.
static void msm_var_run(Ctx& c, const sp_points* p, size_t offset, const u256* d_scalars, size_t n, uint8_t out32[32], bool sharded) {
  if (sharded && c.world() < 2) throw SpError(SP_ERR_INVALID_ARG, "not a connected multi-GPU context");
  points_range(p, offset, n, "msm_var");
  DevBuf<ge> out(1), total;
  DevBuf<uint8_t> comp(32);
  if (n == 0) {
    ge id = ge_identity();
    dev::h2d(out.p, &id, sizeof(ge), c.stream);
  } else {
    const char* cenv = getenv("SP_PIP_WINDOW");
    dev::PipPlan plan = dev::pip_plan(n, cenv ? atoi(cenv) : 0);
    const size_t need = dev::pip_scratch_bytes(plan);
    if (need > p->scratch_bytes) { p->scratch.alloc(need); p->scratch_bytes = need; }   // the sort workspace stays with the point set
    else if (dev::memcheck_on()) dev::memcheck_fill(p->scratch.p, p->scratch.n, dev::FILL_ZERO);   // ... and is refilled like the context's
    dev::msm_var(out.p, p->pts.p + offset, d_scalars, plan, p->scratch.p, c.stream);
  }
  if (sharded) {
    total.alloc(1);
    dev::sum_points(total.p, reinterpret_cast<const ge*>(c.allgather_block(out.p, sizeof(ge))), c.world(), c.stream);
  }
  dev::compress_batch(comp.p, sharded ? total.p : out.p, 1, c.stream);
  dev::d2h(out32, comp.p, 32, c.stream);
  c.sync();
}
int sp_msm_var_sharded(sp_ctx* ctx, const sp_points* p, size_t offset, const sp_poly* scalars, uint8_t out32[32]) {
  return guarded(ctx, [&] { msm_var_run(ctx->c, p, offset, scalars->d.p, scalars->len, out32, true); });
}
int sp_msm_var(sp_ctx* ctx, const sp_points* p, size_t offset, const uint64_t* scalars, size_t n, uint8_t out32[32]) {
  return guarded(ctx, [&] {
    points_range(p, offset, n, "msm_var");   // before the scalars' upload
    DevBuf<u256> d(n ? n : 1);
    dev::h2d(d.p, scalars, n * 32, ctx->c.stream);
    msm_var_run(ctx->c, p, offset, d.p, n, out32, false);
  });
}
int sp_msm_var_resident(sp_ctx* ctx, const sp_points* p, size_t offset, const sp_poly* scalars, uint8_t out32[32]) {
  return guarded(ctx, [&] { msm_var_run(ctx->c, p, offset, scalars->d.p, scalars->len, out32, false); });
}

// ---- instances
// Instance::new (lib.rs:129-198) from the caller's arrays: padding rules, checks, input-column remap and Montgomery form on the device, then the
// CSR / CSC copies
static sp_instance* instance_from_coo(Ctx& c, size_t num_cons, size_t num_vars, size_t num_inputs, const dev::CooIn& in, bool on_host) {
  size_t num_vars_padded = next_pow2(std::max(num_vars, num_inputs + 1));
  size_t num_cons_padded = num_cons;
  if (num_cons_padded == 0 || num_cons_padded == 1) num_cons_padded = 2;
  if (next_pow2(num_cons) != num_cons) num_cons_padded = next_pow2(num_cons);
  std::unique_ptr<sp_instance> I(new sp_instance);
  I->inst.num_cons = num_cons_padded; I->inst.num_vars = num_vars_padded; I->inst.num_inputs = num_inputs;
  const bool pad = num_cons == 0 || num_cons == 1;   // lib.rs: fewer than two constraints get padding entries (row i, column num_vars, 0)
  dev::CooOut co;
  for (int m = 0; m < 3; m++) {
    SparseMatDev& M = I->inst.M[m];
    M.nnz = in.n[m] + (pad && in.n[m] < num_cons_padded ? num_cons_padded - in.n[m] : 0);
    M.coo_row.alloc(M.nnz); M.coo_col.alloc(M.nnz); M.coo_val.alloc(M.nnz);
    co.row[m] = M.coo_row.p; co.col[m] = M.coo_col.p; co.val[m] = M.coo_val.p;
  }
  ingest(c, in, 3, on_host, co, num_cons, num_vars + 1 + num_inputs, num_vars, num_vars_padded - num_vars, [](size_t, size_t, unsigned code) {
    if (code == dev::INGEST_ROW) throw SpError(SP_ERR_INVALID_INDEX, "R1CSError::InvalidIndex (row)");
    if (code == dev::INGEST_COL) throw SpError(SP_ERR_INVALID_INDEX, "R1CSError::InvalidIndex (col)");
    throw SpError(SP_ERR_INVALID_SCALAR, "R1CSError::InvalidScalar");
  });
  for (int m = 0; m < 3; m++)
    if (pad) dev::inst_pad_rows(co.row[m], co.col[m], co.val[m], in.n[m], I->inst.M[m].nnz, (uint32_t)num_vars, c.stream);
  I->inst.finalize(&c);
  return I.release();
}

int sp_instance_create(sp_ctx* ctx, size_t num_cons, size_t num_vars, size_t num_inputs, const uint64_t* A_row, const uint64_t* A_col, const uint8_t* A_val,
                       size_t nA, const uint64_t* B_row, const uint64_t* B_col, const uint8_t* B_val, size_t nB, const uint64_t* C_row, const uint64_t* C_col,
                       const uint8_t* C_val, size_t nC, sp_instance** out) {
  return guarded(ctx, [&] {
    const dev::CooIn in = {{A_row, B_row, C_row}, {A_col, B_col, C_col}, {A_val, B_val, C_val}, {nA, nB, nC}};
    *out = instance_from_coo(ctx->c, num_cons, num_vars, num_inputs, in, true);
  });
}
int sp_instance_create_device(sp_ctx* ctx, size_t num_cons, size_t num_vars, size_t num_inputs, const uint64_t* A_row, const uint64_t* A_col,
                              const uint8_t* A_val, size_t nA, const uint64_t* B_row, const uint64_t* B_col, const uint8_t* B_val, size_t nB,
                              const uint64_t* C_row, const uint64_t* C_col, const uint8_t* C_val, size_t nC, sp_instance** out) {
  return guarded(ctx, [&] {
    const dev::CooIn in = {{A_row, B_row, C_row}, {A_col, B_col, C_col}, {A_val, B_val, C_val}, {nA, nB, nC}};   // matrices past C: empty
    static const char* names[3][3] = {{"A_row", "A_col", "A_val"}, {"B_row", "B_col", "B_val"}, {"C_row", "C_col", "C_val"}};
    for (int m = 0; m < 3; m++) {
      require_device(ctx->c, in.row[m], in.n[m], names[m][0]);
      require_device(ctx->c, in.col[m], in.n[m], names[m][1]);
      require_device(ctx->c, in.val[m], in.n[m], names[m][2]);
    }
    *out = instance_from_coo(ctx->c, num_cons, num_vars, num_inputs, in, false);
  });
}

int sp_poly_from_canonical_device(sp_ctx* ctx, const uint8_t* d_canonical32, size_t n, sp_poly** out) {
  return guarded(ctx, [&] {
    Ctx& c = ctx->c;
    require_device(c, d_canonical32, n, "poly_from_canonical_device");
    std::unique_ptr<sp_poly> p(new sp_poly{&c, DevBuf<u256>(n), n});
    const unsigned long long first = first_fault(c, [&](unsigned long long* err) { dev::canonical_to_mont(p->d.p, d_canonical32, n, err, c.stream); });
    if (first != ~0ull) throw SpError(SP_ERR_INVALID_SCALAR, "R1CSError::InvalidScalar (entry " + std::to_string(first) + ")");
    *out = p.release();
  });
}

static std::vector<Fq> prg_scalars(const std::string& tag, size_t n, uint64_t seed) {
  // DESIGN.md "deterministic inputs": SHAKE256("spartan-b200/v1/" || tag || LE64(seed)), 64 bytes per scalar -> from_bytes_wide
  std::string s = "spartan-b200/v1/" + tag;
  std::vector<uint8_t> in(s.begin(), s.end());
  for (int i = 0; i < 8; i++) in.push_back((uint8_t)(seed >> (8 * i)));
  std::vector<uint8_t> raw(64 * n);
  shake256(raw.data(), raw.size(), in.data(), in.size());
  std::vector<Fq> out(n);
  for (size_t i = 0; i < n; i++) out[i] = Fq::from_bytes_wide(raw.data() + 64 * i);
  return out;
}

int sp_instance_synthetic(sp_ctx* ctx, size_t num_cons, size_t num_vars, size_t num_inputs, uint64_t seed, sp_instance** out, uint64_t* vars_out,
                          uint64_t* inputs_out) {
  return guarded(ctx, [&] {
    // R1CSShape::produce_synthetic_r1cs (r1cs.rs:160-238)
    if (next_pow2(num_cons) != num_cons || next_pow2(num_vars) != num_vars || !(num_inputs < num_vars)) throw SpError(SP_ERR_INVALID_ARG, "synthetic: sizes");
    size_t size_z = num_vars + num_inputs + 1;
    std::vector<Fq> Z = prg_scalars("Z", size_z, seed);
    Z[num_vars] = Fq::one();
    std::unique_ptr<sp_instance> I(new sp_instance);
    I->inst.num_cons = num_cons; I->inst.num_vars = num_vars; I->inst.num_inputs = num_inputs;
    SparseMatDev &A = I->inst.M[0], &B = I->inst.M[1], &Cm = I->inst.M[2];
    // batch inversion of the Z values used as C_val denominators
    std::vector<Fq> zinv(size_z), pref(size_z);
    Fq acc = Fq::one();
    for (size_t i = 0; i < size_z; i++) { pref[i] = acc; if (!Z[i].is_zero()) acc *= Z[i]; }
    Fq ainv = acc.inv();
    for (size_t i = size_z; i-- > 0;) { if (Z[i].is_zero()) { zinv[i] = Fq::zero(); continue; } zinv[i] = ainv * pref[i]; ainv *= Z[i]; }
    for (size_t i = 0; i < num_cons; i++) {
      size_t a = i % size_z, b = (i + 2) % size_z, c = (i + 3) % size_z;
      A.row.push_back((uint32_t)i); A.col.push_back((uint32_t)a); A.val.push_back(Fq::one());
      B.row.push_back((uint32_t)i); B.col.push_back((uint32_t)b); B.val.push_back(Fq::one());
      Fq ab = Z[a] * Z[b];
      Cm.row.push_back((uint32_t)i);
      if (Z[c].is_zero()) { Cm.col.push_back((uint32_t)num_vars); Cm.val.push_back(ab); }
      else { Cm.col.push_back((uint32_t)c); Cm.val.push_back(ab * zinv[c]); }
    }
    // the COO column index space is [vars | 1 | inputs] padded to 2*num_vars: columns >= num_vars need no shift here because
    // produce_synthetic_r1cs requires num_vars to be a power of two already (r1cs.rs:172-176)
    I->inst.upload_coo(&ctx->c);
    I->inst.finalize(&ctx->c);
    memcpy(vars_out, Z.data(), 32 * num_vars);
    memcpy(inputs_out, Z.data() + num_vars + 1, 32 * num_inputs);
    *out = I.release();
  });
}
void sp_instance_free(sp_instance* inst) { delete inst; }
int sp_instance_dims(const sp_instance* inst, size_t* nc, size_t* nv, size_t* ni) {
  *nc = inst->inst.num_cons; *nv = inst->inst.num_vars; *ni = inst->inst.num_inputs;
  return SP_OK;
}
int sp_instance_set_digest(sp_instance* inst, const uint8_t* digest, size_t len) { inst->inst.digest.assign(digest, digest + len); return SP_OK; }
int sp_instance_bincode(const sp_instance* inst, uint8_t** out, size_t* len) {
  return host_guarded(nullptr, [&] { put_bytes(out, len, inst->inst.shape_bincode()); });
}
// R1CSShape::get_digest (r1cs.rs:154-158): the bytes NIZK::prove / verify absorb (lib.rs:514) — the caller's (sp_instance_set_digest) or, by
// default, this library's miniz-level-6 zlib stream of bincode(shape), computed on first use
int sp_instance_digest(const sp_instance* inst, uint8_t** out, size_t* len) {
  return host_guarded(nullptr, [&] { put_bytes(out, len, inst->inst.shape_digest()); });
}
int sp_instance_nnz(const sp_instance* inst, int m, size_t* nnz) { if (m < 0 || m > 2) return SP_ERR_INVALID_ARG; *nnz = inst->inst.M[m].nnz; return SP_OK; }
int sp_instance_export(const sp_instance* inst, int m, uint64_t* row, uint64_t* col, uint64_t* val) {
  if (m < 0 || m > 2) return SP_ERR_INVALID_ARG;
  return host_guarded(nullptr, [&] {
    inst->inst.host_coo();
    const SparseMatDev& M = inst->inst.M[m];
    for (size_t k = 0; k < M.nnz; k++) { row[k] = M.row[k]; col[k] = M.col[k]; }
    if (M.nnz) memcpy(val, M.val.data(), 32 * M.nnz);
  });
}

int sp_instance_is_sat(sp_ctx* ctx, const sp_instance* inst, const uint64_t* vars, size_t nvars, const uint64_t* inputs, size_t ninputs, int* sat) {
  return guarded(ctx, [&] {
    const Instance& I = inst->inst;
    if (ninputs != I.num_inputs) throw SpError(SP_ERR_INVALID_INPUTS, "R1CSError::InvalidNumberOfInputs");
    Ctx& c = ctx->c;
    DevBuf<u256> d_vars = upload_padded_vars(c, I, vars, nvars);
    DevBuf<u256> z(2 * I.num_vars), Az(I.num_cons), Bz(I.num_cons), Cz(I.num_cons);
    dev::d2d(z.p, d_vars.p, I.num_vars * 32, c.stream);
    std::vector<Fq> tail(1 + ninputs);
    tail[0] = Fq::one();
    if (ninputs) memcpy(&tail[1], inputs, 32 * ninputs);
    dev::h2d(z.p + I.num_vars, tail.data(), tail.size() * 32, c.stream);
    dev::dzero(z.p + I.num_vars + tail.size(), (I.num_vars - tail.size()) * 32, c.stream);
    u256* outs[3] = {Az.p, Bz.p, Cz.p};
    for (int m = 0; m < 3; m++) dev::spmv(outs[m], I.num_cons, I.M[m].csr_ptr.p, I.M[m].csr_idx.p, I.M[m].csr_val.p, z.p, c.stream);
    DevBuf<u256> prod(I.num_cons);
    u256* prods[1] = {prod.p};
    const u256 *as[1] = {Az.p}, *bs[1] = {Bz.p};
    dev::hadamard_many(prods, as, bs, 1, I.num_cons, c.stream);
    std::vector<Fq> p = c.download(prod.p, I.num_cons), cz = c.download(Cz.p, I.num_cons);
    *sat = 1;
    for (size_t i = 0; i < I.num_cons; i++) if (!(p[i] == cz[i])) { *sat = 0; break; }   // r1cs.rs:265
  });
}

// ---- NIZK
// private gens: tables sized for this one circuit, then a view into them (the view holds the only reference)
int sp_nizk_gens_create(sp_ctx* ctx, size_t num_cons, size_t num_vars, size_t num_inputs, sp_nizk_gens** out) {
  return guarded(ctx, [&] {
    const GenTables t(&ctx->c, num_cons, num_vars, num_inputs, 0);
    std::unique_ptr<sp_nizk_gens> g(new sp_nizk_gens);
    g->g.reset(new R1CSGens(&ctx->c, t, padded_num_vars(num_vars, num_inputs)));  // lib.rs:475-481
    *out = g.release();
  });
}
int sp_nizk_gens_create_from(sp_ctx* ctx, const sp_gen_tables* tables, size_t num_cons, size_t num_vars, size_t num_inputs, sp_nizk_gens** out) {
  return guarded(ctx, [&] {
    (void)num_cons;
    std::unique_ptr<sp_nizk_gens> g(new sp_nizk_gens);
    g->g.reset(new R1CSGens(&ctx->c, *tables->t, padded_num_vars(num_vars, num_inputs)));
    *out = g.release();
  });
}
void sp_nizk_gens_free(sp_nizk_gens* g) { delete g; }

int sp_nizk_prove(sp_ctx* ctx, const sp_instance* inst, const uint64_t* vars, size_t nvars, const uint64_t* inputs, size_t ninputs, const sp_nizk_gens* gens,
                  const uint8_t* label, size_t label_len, const uint64_t seed[4], uint8_t** proof, size_t* proof_len) {
  return nizk_prove_common(ctx, inst, {vars, nvars, nullptr}, inputs, ninputs, gens, ProofStates::Label{label, label_len}, seed, proof, proof_len);
}
// NIZK::prove(&inst, vars, &inputs, &gens, transcript: &mut Transcript) with the caller's transcript state in / out (lib.rs:501-508)
int sp_nizk_prove_t(sp_ctx* ctx, const sp_instance* inst, const uint64_t* vars, size_t nvars, const uint64_t* inputs, size_t ninputs, const sp_nizk_gens* gens,
                    uint8_t* strobe_state, const uint64_t seed[4], uint8_t** proof, size_t* proof_len) {
  return nizk_prove_common(ctx, inst, {vars, nvars, nullptr}, inputs, ninputs, gens, strobe_state, seed, proof, proof_len);
}
int sp_nizk_prove_resident(sp_ctx* ctx, const sp_instance* inst, const sp_poly* vars, const uint64_t* inputs, size_t ninputs, const sp_nizk_gens* gens,
                           const uint8_t* label, size_t label_len, const uint64_t seed[4], uint8_t** proof, size_t* proof_len) {
  return nizk_prove_common(ctx, inst, {nullptr, 0, vars}, inputs, ninputs, gens, ProofStates::Label{label, label_len}, seed, proof, proof_len);
}

// ---- SNARK
int sp_snark_gens_create(sp_ctx* ctx, size_t num_cons, size_t num_vars, size_t num_inputs, size_t num_nz_entries, sp_snark_gens** out) {
  return guarded(ctx, [&] {
    // next_pow2(0) = next_pow2(1): tables for one non-zero entry are the tables num_nz_entries = 0 has always had, and they include gens_r1cs_eval
    const GenTables t(&ctx->c, num_cons, num_vars, num_inputs, std::max<size_t>(num_nz_entries, 1));
    std::unique_ptr<sp_snark_gens> g(new sp_snark_gens);
    g->g.reset(new SnarkGens(&ctx->c, t, num_cons, num_vars, num_inputs, num_nz_entries));
    *out = g.release();
  });
}
int sp_snark_gens_create_from(sp_ctx* ctx, const sp_gen_tables* tables, size_t num_cons, size_t num_vars, size_t num_inputs, size_t num_nz_entries,
                              sp_snark_gens** out) {
  return guarded(ctx, [&] {
    std::unique_ptr<sp_snark_gens> g(new sp_snark_gens);
    g->g.reset(new SnarkGens(&ctx->c, *tables->t, num_cons, num_vars, num_inputs, num_nz_entries));
    *out = g.release();
  });
}

// ---- generator tables shared by gens views
int sp_gen_tables_create(sp_ctx* ctx, size_t num_cons, size_t num_vars, size_t num_inputs, size_t num_nz_entries, sp_gen_tables** out) {
  return guarded(ctx, [&] {
    std::unique_ptr<sp_gen_tables> t(new sp_gen_tables);
    t->t.reset(new GenTables(&ctx->c, num_cons, num_vars, num_inputs, num_nz_entries));
    *out = t.release();
  });
}
void sp_gen_tables_free(sp_gen_tables* t) { delete t; }
int sp_gen_tables_info(const sp_gen_tables* t, sp_gen_set_info* out, size_t cap, size_t* n) {
  std::vector<const GenSet*> sets{t->t->r1cs_sat.get()};
  if (t->t->r1cs_eval) sets.push_back(t->t->r1cs_eval.get());
  *n = sets.size();
  if (cap < sets.size()) return SP_ERR_INVALID_ARG;
  for (size_t i = 0; i < sets.size(); i++) {
    sp_gen_set_info& o = out[i];
    memset(&o, 0, sizeof(o));
    memcpy(o.label, sets[i]->label.data(), std::min(sets[i]->label.size(), sizeof(o.label) - 1));
    o.nbases = sets[i]->nbases;
    o.window_bits = sets[i]->wbits;
    o.has_row_table = sets[i]->rows() != nullptr;
    o.device_bytes = sets[i]->device_bytes();
  }
  return SP_OK;
}
unsigned long long sp_device_bytes_live(void) { return dev::pool_live_bytes(); }
void sp_snark_gens_free(sp_snark_gens* g) { delete g; }
int sp_snark_encode(sp_ctx* ctx, const sp_instance* inst, const sp_snark_gens* gens, sp_snark_encoding** out) {
  return guarded(ctx, [&] {
    std::unique_ptr<sp_snark_encoding> e(new sp_snark_encoding);
    e->e.reset(new SnarkEncoding());
    snark_encode(ctx->c, inst->inst, *gens->g, *e->e);
    *out = e.release();
  });
}
void sp_snark_encoding_free(sp_snark_encoding* e) { delete e; }
int sp_snark_commitment_bytes(const sp_snark_encoding* e, uint8_t** out, size_t* len) {
  return host_guarded(nullptr, [&] { put_bytes(out, len, to_bincode(e->e->comm)); });
}
// a verifier holds only the ComputationCommitment: bincode(ComputationCommitment) -> a handle usable with sp_snark_verify (not with sp_snark_prove)
int sp_snark_commitment_load(sp_ctx* ctx, const uint8_t* bytes, size_t len, sp_snark_encoding** out) {
  return guarded(ctx, [&] {
    std::unique_ptr<sp_snark_encoding> E(new sp_snark_encoding);
    E->e.reset(new SnarkEncoding);
    E->e->comm = from_bincode<ComputationCommitment>(bytes, len, SP_ERR_INVALID_ARG, "computation commitment");
    *out = E.release();
  });
}
int sp_snark_prove(sp_ctx* ctx, const sp_instance* inst, const sp_snark_encoding* enc, const uint64_t* vars, size_t nvars, const uint64_t* inputs, size_t ninputs,
                   const sp_snark_gens* gens, const uint8_t* label, size_t label_len, const uint64_t seed[4], uint8_t** proof, size_t* proof_len) {
  return snark_prove_common(ctx, inst, enc, {vars, nvars, nullptr}, inputs, ninputs, gens, ProofStates::Label{label, label_len}, seed, proof, proof_len);
}
// SNARK::prove(..., transcript: &mut Transcript) with the caller's transcript state in / out (lib.rs:339-347)
int sp_snark_prove_t(sp_ctx* ctx, const sp_instance* inst, const sp_snark_encoding* enc, const uint64_t* vars, size_t nvars, const uint64_t* inputs, size_t ninputs,
                     const sp_snark_gens* gens, uint8_t* strobe_state, const uint64_t seed[4], uint8_t** proof, size_t* proof_len) {
  return snark_prove_common(ctx, inst, enc, {vars, nvars, nullptr}, inputs, ninputs, gens, strobe_state, seed, proof, proof_len);
}
int sp_snark_prove_resident(sp_ctx* ctx, const sp_instance* inst, const sp_snark_encoding* enc, const sp_poly* vars, const uint64_t* inputs, size_t ninputs,
                            const sp_snark_gens* gens, const uint8_t* label, size_t label_len, const uint64_t seed[4], uint8_t** proof, size_t* proof_len) {
  return snark_prove_common(ctx, inst, enc, {nullptr, 0, vars}, inputs, ninputs, gens, ProofStates::Label{label, label_len}, seed, proof, proof_len);
}

// ---- verifiers.  The _t forms verify on the caller's transcript state (lib.rs:423-429, :549-555).
int sp_nizk_verify(sp_ctx* ctx, const sp_instance* inst, const uint64_t* inputs, size_t ninputs, const sp_nizk_gens* gens, const uint8_t* label, size_t label_len,
                   const uint8_t* proof, size_t proof_len) {
  return nizk_verify_common(ctx, inst, inputs, ninputs, gens, ProofStates::Label{label, label_len}, proof, proof_len);
}
int sp_snark_verify(sp_ctx* ctx, const sp_snark_encoding* comm, const uint64_t* inputs, size_t ninputs, const sp_snark_gens* gens, const uint8_t* label,
                    size_t label_len, const uint8_t* proof, size_t proof_len) {
  return snark_verify_common(ctx, comm, inputs, ninputs, gens, ProofStates::Label{label, label_len}, proof, proof_len);
}
int sp_nizk_verify_t(sp_ctx* ctx, const sp_instance* inst, const uint64_t* inputs, size_t ninputs, const sp_nizk_gens* gens, uint8_t* strobe_state,
                     const uint8_t* proof, size_t proof_len) {
  return nizk_verify_common(ctx, inst, inputs, ninputs, gens, strobe_state, proof, proof_len);
}
int sp_snark_verify_t(sp_ctx* ctx, const sp_snark_encoding* comm, const uint64_t* inputs, size_t ninputs, const sp_snark_gens* gens, uint8_t* strobe_state,
                      const uint8_t* proof, size_t proof_len) {
  return snark_verify_common(ctx, comm, inputs, ninputs, gens, strobe_state, proof, proof_len);
}
// ---- a whole sumcheck of a caller-defined polynomial (prover.cpp: poly_sumcheck_prove).  Every argument is checked before the first launch, so a
// refused call leaves the tables as they were.
// The checked polynomial of the caller's tables and terms: P.t holds the distinct tables (a handle passed twice is one table, bound once per round),
// slot[i] the distinct table of index i
struct CallerPoly { dev::ScPoly P; size_t len; std::vector<sp_poly*> distinct; std::vector<uint8_t> slot; };
static CallerPoly caller_poly(const sp_ctx* ctx, sp_poly* const* tables, int k, const sp_sc_term* terms, int nterms, size_t num_rounds, const std::string& what) {
  require_count(what, k, "tables", "SP_SC_MAX_TABLES", SP_SC_MAX_TABLES);
  require_count(what, nterms, "terms", "SP_SC_MAX_TERMS", SP_SC_MAX_TERMS);
  CallerPoly cp;
  cp.len = caller_tables(ctx, tables, k, what, 2).len;
  const size_t m = log2_ceil(cp.len);
  if (num_rounds < 1 || num_rounds > m)
    throw SpError(SP_ERR_INVALID_ARG, what + ": num_rounds = " + std::to_string(num_rounds) + " outside 1 .. " + std::to_string(m) + " (the tables' variables)");
  dev::ScPoly& P = cp.P;
  memset(static_cast<void*>(&P), 0, sizeof P);
  cp.slot.resize(k);
  for (int i = 0; i < k; i++) {
    const size_t at = std::find(cp.distinct.begin(), cp.distinct.end(), tables[i]) - cp.distinct.begin();
    if (at == cp.distinct.size()) { cp.distinct.push_back(tables[i]); P.t[at] = tables[i]->d.p; }
    cp.slot[i] = (uint8_t)at;
  }
  P.ntables = (int)cp.distinct.size();
  P.nterms = nterms;
  const Fq one = Fq::one();
  const std::string coeff_what = what + ": coefficient";
  for (int t = 0; t < nterms; t++) {
    const sp_sc_term& tm = terms[t];
    const std::string at = what + ": term " + std::to_string(t);
    if (tm.nfactors == 0) throw SpError(SP_ERR_INVALID_ARG, at + " has no factors");
    if (tm.nfactors > SP_SC_MAX_DEGREE)
      throw SpError(SP_ERR_INVALID_ARG, at + " has " + std::to_string(tm.nfactors) + " factors; degree <= SP_SC_MAX_DEGREE = " + std::to_string(SP_SC_MAX_DEGREE) + " supported");
    for (uint32_t f = 0; f < tm.nfactors; f++) {
      if (tm.factor[f] >= (uint32_t)k) throw SpError(SP_ERR_INVALID_ARG, at + ": table index " + std::to_string(tm.factor[f]) + " >= k = " + std::to_string(k));
      P.fac[t][f] = cp.slot[tm.factor[f]];
    }
    require_reduced(tm.coeff_mont, 1, coeff_what.c_str());
    const Fq c = fq_in(tm.coeff_mont);
    P.coeff[t] = c.m;
    P.unit[t] = c == one;
    P.nfac[t] = (uint8_t)tm.nfactors;
    P.degree = std::max(P.degree, (int)tm.nfactors);
  }
  return cp;
}
// the body of sp_sumcheck_prove(_t), run inside guarded: the entry makes st, the first check of the call
static void sumcheck_prove_common(sp_ctx* ctx, sp_poly* const* tables, int k, const sp_sc_term* terms, int nterms, const uint64_t claim[4],
                                  size_t num_rounds, ProofStates&& st, uint8_t** proof, size_t* proof_len, uint64_t* r_out, uint64_t* finals_out,
                                  uint64_t e_out[4]) {
  const std::string what = "sumcheck_prove";
  if (!tables || !terms || !claim || !proof || !proof_len || !r_out || !finals_out || !e_out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
  const CallerPoly cp = caller_poly(ctx, tables, k, terms, nterms, num_rounds, what);
  require_reduced(claim, 1, "sumcheck_prove: claim");
  st.open();
  SumcheckInstanceProof pr;
  std::vector<Fq> r, finals;
  Fq e;
  poly_sumcheck_prove(ctx->c, cp.P, cp.len, fq_in(claim), num_rounds, st.T(), pr, r, finals, e);
  for (sp_poly* p : cp.distinct) p->len >>= num_rounds;
  st.proved();
  put_bytes(proof, proof_len, to_bincode(pr));
  put_scalars(r_out, r);
  for (int i = 0; i < k; i++) fq_out(finals_out + 4 * i, finals[cp.slot[i]]);
  fq_out(e_out, e);
}
int sp_sumcheck_prove_t(sp_ctx* ctx, sp_poly* const* tables, int k, const sp_sc_term* terms, int nterms, const uint64_t claim[4], size_t num_rounds,
                        uint8_t* strobe_state, uint8_t** proof, size_t* proof_len, uint64_t* r_out, uint64_t* finals_out, uint64_t e_out[4]) {
  return guarded(ctx, [&] {
    sumcheck_prove_common(ctx, tables, k, terms, nterms, claim, num_rounds, ProofStates(strobe_state), proof, proof_len, r_out, finals_out, e_out);
  });
}
int sp_sumcheck_prove(sp_ctx* ctx, sp_poly* const* tables, int k, const sp_sc_term* terms, int nterms, const uint64_t claim[4], size_t num_rounds,
                      const uint8_t* label, size_t label_len, uint8_t** proof, size_t* proof_len, uint64_t* r_out, uint64_t* finals_out, uint64_t e_out[4]) {
  return guarded(ctx, [&] {
    sumcheck_prove_common(ctx, tables, k, terms, nterms, claim, num_rounds, ProofStates(ProofStates::Label{label, label_len}), proof, proof_len, r_out,
                          finals_out, e_out);
  });
}
// host only: no device work, so ctx may be NULL (the message then goes where sp_last_error(NULL) reads it)
int sp_sumcheck_verify_t(sp_ctx* ctx, const uint8_t* proof, size_t proof_len, const uint64_t claim[4], size_t num_rounds, size_t degree_bound,
                         uint8_t* strobe_state, uint64_t e_out[4], uint64_t* r_out) {
  return host_guarded(ctx, [&] {
    ProofStates st(strobe_state);
    if (!claim || !e_out || (!r_out && num_rounds) || (!proof && proof_len)) throw SpError(SP_ERR_INVALID_ARG, "sumcheck_verify: NULL argument");
    if (degree_bound < 1) throw SpError(SP_ERR_INVALID_ARG, "sumcheck_verify: degree_bound must be >= 1");
    require_reduced(claim, 1, "sumcheck_verify: claim");
    st.open_verify();
    std::vector<Fq> r;
    fq_out(e_out, sumcheck_verify_bytes(proof, proof_len, fq_in(claim), num_rounds, degree_bound, st.T(), r));
    put_scalars(r_out, r);
  });
}

// ---- ZK sumchecks of a caller-defined polynomial and the sigma protocols (nizk/mod.rs), on the caller's transcript and tape and the caller's
// MultiCommitGens (sp_gens: G[0..n), h = G[n]).  Every argument is checked before the first launch, tape draw or transcript write, so a refused
// call leaves the tables, the transcript and the tape as they were.
static CommitKey gens_key(const sp_ctx* ctx, const sp_gens* g, const std::string& what, const char* name) {
  if (!g) throw SpError(SP_ERR_INVALID_ARG, what + ": " + name + " is NULL");
  if (g->set->ctx != &ctx->c) throw SpError(SP_ERR_INVALID_ARG, what + ": " + name + " belongs to another context");
  return CommitKey{g->set.get(), 0, g->n, g->n};
}
static void require_gens_n(const CommitKey& k, size_t n, const std::string& what, const char* name, const std::string& why) {
  if (k.n != n) throw SpError(SP_ERR_INVALID_ARG, what + ": " + name + ".n = " + std::to_string(k.n) + " but " + why + " needs " + std::to_string(n));
}
// the host copies of every generator and h of the sets the call commits against, built once per set (after the checks)
static void gens_host_tables(const sp_gens* g) {
  std::vector<size_t> b(g->n + 1);
  for (size_t i = 0; i <= g->n; i++) b[i] = i;
  g->set->add_host_tables(b);
}
static Cp cp_in(const uint8_t* p32, const std::string& what) {
  if (!p32) throw SpError(SP_ERR_INVALID_ARG, what + " is NULL");
  point_in(p32, what.c_str());   // SP_ERR_INVALID_POINT unless it decompresses
  Cp c;
  memcpy(c.b, p32, 32);
  return c;
}
static Fq scalar_in(const uint64_t* l, const std::string& what) {
  if (!l) throw SpError(SP_ERR_INVALID_ARG, what + " is NULL");
  require_reduced(l, 1, what.c_str());
  return fq_in(l);
}
static void cp_out(uint8_t* out32, const Cp& c) { if (out32) memcpy(out32, c.b, 32); }

int sp_zk_sumcheck_prove_t(sp_ctx* ctx, sp_poly* const* tables, int k, const sp_sc_term* terms, int nterms, const uint64_t claim[4],
                           const uint64_t blind_claim[4], size_t num_rounds, const sp_gens* gens_1, const sp_gens* gens_n, uint8_t* strobe_state,
                           uint8_t* tape_state, uint8_t** proof, size_t* proof_len, uint64_t* r_out, uint64_t* finals_out, uint64_t blind_post_out[4]) {
  return guarded(ctx, [&] {
    const std::string what = "zk_sumcheck_prove";
    ProofStates st(strobe_state, tape_state, what);
    if (!tables || !terms || !proof || !proof_len || !r_out || !finals_out || !blind_post_out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    const CallerPoly cp = caller_poly(ctx, tables, k, terms, nterms, num_rounds, what);
    if (num_rounds > zk_sumcheck_max_rounds())
      throw SpError(SP_ERR_INVALID_ARG, what + ": num_rounds = " + std::to_string(num_rounds) + " > " + std::to_string(zk_sumcheck_max_rounds()) +
                                            ", the rounds a ZK sumcheck stages");
    const CommitKey g1 = gens_key(ctx, gens_1, what, "gens_1"), gn = gens_key(ctx, gens_n, what, "gens_n");
    require_gens_n(g1, 1, what, "gens_1", "a claim's commitment");
    require_gens_n(gn, (size_t)cp.P.degree + 1, what, "gens_n", "a round polynomial of degree " + std::to_string(cp.P.degree));
    const Fq c = scalar_in(claim, what + ": claim"), bc = scalar_in(blind_claim, what + ": blind_claim");
    gens_host_tables(gens_1);
    gens_host_tables(gens_n);
    st.open();
    ZKSumcheckInstanceProof pr;
    std::vector<Fq> r, finals;
    Fq blind_post;
    zk_poly_sumcheck_prove(ctx->c, cp.P, cp.len, c, bc, num_rounds, g1, gn, st.T(), st.tape(), pr, r, finals, blind_post);
    for (sp_poly* p : cp.distinct) p->len >>= num_rounds;
    st.proved();
    put_bytes(proof, proof_len, to_bincode(pr));
    put_scalars(r_out, r);
    for (int i = 0; i < k; i++) fq_out(finals_out + 4 * i, finals[cp.slot[i]]);
    fq_out(blind_post_out, blind_post);
  });
}
int sp_zk_sumcheck_verify_t(sp_ctx* ctx, const uint8_t* proof, size_t proof_len, const uint8_t comm_claim32[32], size_t num_rounds, size_t degree_bound,
                            const sp_gens* gens_1, const sp_gens* gens_n, uint8_t* strobe_state, uint8_t comm_eval_out32[32], uint64_t* r_out) {
  return guarded(ctx, [&] {
    const std::string what = "zk_sumcheck_verify";
    ProofStates st(strobe_state);
    if ((!proof && proof_len) || !comm_eval_out32 || !r_out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    if (num_rounds < 1) throw SpError(SP_ERR_INVALID_ARG, what + ": num_rounds must be >= 1");
    if (degree_bound < 1 || degree_bound + 1 > SP_DOTPROD_MAX_N)
      throw SpError(SP_ERR_INVALID_ARG, what + ": degree_bound = " + std::to_string(degree_bound) + " outside 1 .. SP_DOTPROD_MAX_N - 1 = " + std::to_string(SP_DOTPROD_MAX_N - 1));
    const CommitKey g1 = gens_key(ctx, gens_1, what, "gens_1"), gn = gens_key(ctx, gens_n, what, "gens_n");
    require_gens_n(g1, 1, what, "gens_1", "a claim's commitment");
    require_gens_n(gn, degree_bound + 1, what, "gens_n", "degree_bound = " + std::to_string(degree_bound));
    const Cp cc = cp_in(comm_claim32, what + ": comm_claim");
    gens_host_tables(gens_1);
    gens_host_tables(gens_n);
    st.open_verify();
    std::vector<Fq> r;
    cp_out(comm_eval_out32, zk_sumcheck_verify_bytes(ctx->c, proof, proof_len, cc, num_rounds, degree_bound, g1, gn, st.T(), r));
    put_scalars(r_out, r);
  });
}

int sp_knowledge_prove_t(sp_ctx* ctx, const sp_gens* gens_n, uint8_t* strobe_state, uint8_t* tape_state, const uint64_t x[4], const uint64_t r[4],
                         uint8_t** proof, size_t* proof_len, uint8_t C_out32[32]) {
  return guarded(ctx, [&] {
    const std::string what = "knowledge_prove";
    ProofStates st(strobe_state, tape_state, what);
    if (!proof || !proof_len || !C_out32) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    const CommitKey g = gens_key(ctx, gens_n, what, "gens_n");
    require_gens_n(g, 1, what, "gens_n", "a scalar's commitment");
    const Fq fx = scalar_in(x, what + ": x"), fr = scalar_in(r, what + ": r");
    gens_host_tables(gens_n);
    st.open();
    Cp C;
    const KnowledgeProof p = knowledge_prove(g, st.T(), st.tape(), fx, fr, C);
    st.proved();
    put_bytes(proof, proof_len, to_bincode(p));
    cp_out(C_out32, C);
  });
}
int sp_knowledge_verify_t(sp_ctx* ctx, const sp_gens* gens_n, uint8_t* strobe_state, const uint8_t C32[32], const uint8_t* proof, size_t proof_len) {
  return guarded(ctx, [&] {
    const std::string what = "knowledge_verify";
    ProofStates st(strobe_state);
    if (!proof && proof_len) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    const CommitKey g = gens_key(ctx, gens_n, what, "gens_n");
    require_gens_n(g, 1, what, "gens_n", "a scalar's commitment");
    const Cp C = cp_in(C32, what + ": C");
    gens_host_tables(gens_n);
    st.open_verify();
    knowledge_verify_bytes(ctx->c, g, st.T(), C, proof, proof_len);
  });
}

int sp_equality_prove_t(sp_ctx* ctx, const sp_gens* gens_n, uint8_t* strobe_state, uint8_t* tape_state, const uint64_t v1[4], const uint64_t s1[4],
                        const uint64_t v2[4], const uint64_t s2[4], uint8_t** proof, size_t* proof_len, uint8_t C1_out32[32], uint8_t C2_out32[32]) {
  return guarded(ctx, [&] {
    const std::string what = "equality_prove";
    ProofStates st(strobe_state, tape_state, what);
    if (!proof || !proof_len || !C1_out32 || !C2_out32) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    const CommitKey g = gens_key(ctx, gens_n, what, "gens_n");
    require_gens_n(g, 1, what, "gens_n", "a scalar's commitment");
    const Fq a1 = scalar_in(v1, what + ": v1"), b1 = scalar_in(s1, what + ": s1"), a2 = scalar_in(v2, what + ": v2"), b2 = scalar_in(s2, what + ": s2");
    gens_host_tables(gens_n);
    st.open();
    Cp C1, C2;
    const EqualityProof p = equality_prove(g, st.T(), st.tape(), a1, b1, a2, b2, &C1, &C2);
    st.proved();
    put_bytes(proof, proof_len, to_bincode(p));
    cp_out(C1_out32, C1);
    cp_out(C2_out32, C2);
  });
}
int sp_equality_verify_t(sp_ctx* ctx, const sp_gens* gens_n, uint8_t* strobe_state, const uint8_t C1_32[32], const uint8_t C2_32[32], const uint8_t* proof,
                         size_t proof_len) {
  return guarded(ctx, [&] {
    const std::string what = "equality_verify";
    ProofStates st(strobe_state);
    if (!proof && proof_len) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    const CommitKey g = gens_key(ctx, gens_n, what, "gens_n");
    require_gens_n(g, 1, what, "gens_n", "a scalar's commitment");
    const Cp C1 = cp_in(C1_32, what + ": C1"), C2 = cp_in(C2_32, what + ": C2");
    gens_host_tables(gens_n);
    st.open_verify();
    equality_verify_bytes(ctx->c, g, st.T(), C1, C2, proof, proof_len);
  });
}

int sp_product_prove_t(sp_ctx* ctx, const sp_gens* gens_n, uint8_t* strobe_state, uint8_t* tape_state, const uint64_t x[4], const uint64_t rX[4],
                       const uint64_t y[4], const uint64_t rY[4], const uint64_t z[4], const uint64_t rZ[4], uint8_t** proof, size_t* proof_len,
                       uint8_t X_out32[32], uint8_t Y_out32[32], uint8_t Z_out32[32]) {
  return guarded(ctx, [&] {
    const std::string what = "product_prove";
    ProofStates st(strobe_state, tape_state, what);
    if (!proof || !proof_len || !X_out32 || !Y_out32 || !Z_out32) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    const CommitKey g = gens_key(ctx, gens_n, what, "gens_n");
    require_gens_n(g, 1, what, "gens_n", "a scalar's commitment");
    const Fq fx = scalar_in(x, what + ": x"), frX = scalar_in(rX, what + ": rX"), fy = scalar_in(y, what + ": y"), frY = scalar_in(rY, what + ": rY"),
             fz = scalar_in(z, what + ": z"), frZ = scalar_in(rZ, what + ": rZ");
    gens_host_tables(gens_n);
    st.open();
    Cp X, Y, Z;
    const ProductProof p = product_prove(g, st.T(), st.tape(), fx, frX, fy, frY, fz, frZ, X, Y, Z);
    st.proved();
    put_bytes(proof, proof_len, to_bincode(p));
    cp_out(X_out32, X);
    cp_out(Y_out32, Y);
    cp_out(Z_out32, Z);
  });
}
int sp_product_verify_t(sp_ctx* ctx, const sp_gens* gens_n, uint8_t* strobe_state, const uint8_t X32[32], const uint8_t Y32[32], const uint8_t Z32[32],
                        const uint8_t* proof, size_t proof_len) {
  return guarded(ctx, [&] {
    const std::string what = "product_verify";
    ProofStates st(strobe_state);
    if (!proof && proof_len) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    const CommitKey g = gens_key(ctx, gens_n, what, "gens_n");
    require_gens_n(g, 1, what, "gens_n", "a scalar's commitment");
    const Cp X = cp_in(X32, what + ": X"), Y = cp_in(Y32, what + ": Y"), Z = cp_in(Z32, what + ": Z");
    gens_host_tables(gens_n);
    st.open_verify();
    product_verify_bytes(ctx->c, g, st.T(), X, Y, Z, proof, proof_len);
  });
}

// the vectors of a DotProductProof: n = gens_n.n entries, 1 <= n <= SP_DOTPROD_MAX_N
static void dotproduct_len(const CommitKey& g1, const CommitKey& gn, size_t n, const std::string& what) {
  require_gens_n(g1, 1, what, "gens_1", "a scalar's commitment");
  if (n < 1 || n > SP_DOTPROD_MAX_N)
    throw SpError(SP_ERR_INVALID_ARG, what + ": n = " + std::to_string(n) + " outside 1 .. SP_DOTPROD_MAX_N = " + std::to_string(SP_DOTPROD_MAX_N) +
                                          " (longer vectors: PolyEvalProof)");
  require_gens_n(gn, n, what, "gens_n", "vectors of length n = " + std::to_string(n));
}
int sp_dotproduct_prove_t(sp_ctx* ctx, const sp_gens* gens_1, const sp_gens* gens_n, uint8_t* strobe_state, uint8_t* tape_state, const uint64_t* x_vec,
                          const uint64_t blind_x[4], const uint64_t* a_vec, size_t n, const uint64_t y[4], const uint64_t blind_y[4], uint8_t** proof,
                          size_t* proof_len, uint8_t Cx_out32[32], uint8_t Cy_out32[32]) {
  return guarded(ctx, [&] {
    const std::string what = "dotproduct_prove";
    ProofStates st(strobe_state, tape_state, what);
    if (!proof || !proof_len || !Cx_out32 || !Cy_out32 || !x_vec || !a_vec) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    const CommitKey g1 = gens_key(ctx, gens_1, what, "gens_1"), gn = gens_key(ctx, gens_n, what, "gens_n");
    dotproduct_len(g1, gn, n, what);
    require_reduced(x_vec, n, (what + ": x_vec").c_str());
    require_reduced(a_vec, n, (what + ": a_vec").c_str());
    const Fq bx = scalar_in(blind_x, what + ": blind_x"), fy = scalar_in(y, what + ": y"), by = scalar_in(blind_y, what + ": blind_y");
    gens_host_tables(gens_1);
    gens_host_tables(gens_n);
    st.open();
    Cp Cx, Cy;
    const DotProductProof p = dotproduct_prove(g1, gn, st.T(), st.tape(), fq_vec(x_vec, n), bx, fq_vec(a_vec, n), fy, by, nullptr, nullptr, &Cx, &Cy);
    st.proved();
    put_bytes(proof, proof_len, to_bincode(p));
    cp_out(Cx_out32, Cx);
    cp_out(Cy_out32, Cy);
  });
}
int sp_dotproduct_verify_t(sp_ctx* ctx, const sp_gens* gens_1, const sp_gens* gens_n, uint8_t* strobe_state, const uint64_t* a_vec, size_t n,
                           const uint8_t Cx32[32], const uint8_t Cy32[32], const uint8_t* proof, size_t proof_len) {
  return guarded(ctx, [&] {
    const std::string what = "dotproduct_verify";
    ProofStates st(strobe_state);
    if ((!proof && proof_len) || !a_vec) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    const CommitKey g1 = gens_key(ctx, gens_1, what, "gens_1"), gn = gens_key(ctx, gens_n, what, "gens_n");
    dotproduct_len(g1, gn, n, what);
    require_reduced(a_vec, n, (what + ": a_vec").c_str());
    const Cp Cx = cp_in(Cx32, what + ": Cx"), Cy = cp_in(Cy32, what + ": Cy");
    gens_host_tables(gens_1);
    gens_host_tables(gens_n);
    st.open_verify();
    dotproduct_verify_bytes(ctx->c, g1, gn, st.T(), fq_vec(a_vec, n), Cx, Cy, proof, proof_len);
  });
}

// ---- DotProductProofLog of the caller's vectors (prover.cpp: dotlog_*)
int sp_dotlog_gens_create(sp_ctx* ctx, size_t n, const uint8_t* label, size_t label_len, sp_dotlog_gens** out) {
  return guarded(ctx, [&] {
    const std::string what = "dotlog_gens_create";
    if (!out || (!label && label_len)) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    if (n < 1 || n > SP_DOTLOG_MAX_N || (n & (n - 1)))
      throw SpError(SP_ERR_INVALID_ARG, what + ": n = " + std::to_string(n) + " is not a power of two in 1 .. SP_DOTLOG_MAX_N = " + std::to_string(SP_DOTLOG_MAX_N));
    std::unique_ptr<sp_dotlog_gens> g(new sp_dotlog_gens{&ctx->c, nullptr});
    g->g.reset(new DotLogGens(ctx->c, n, std::string((const char*)label, label_len)));
    *out = g.release();
  });
}
void sp_dotlog_gens_free(sp_dotlog_gens* g) { delete g; }
// a vector of a DotProductProofLog: a handle of this context with gens' n entries
static const u256* dotlog_vec(const sp_ctx* ctx, const sp_poly* p, size_t n, const std::string& what, const char* name) {
  require_owned(ctx, p, what, name);
  if (p->len != n) throw SpError(SP_ERR_INVALID_ARG, what + ": " + name + " has " + std::to_string(p->len) + " entries, gens have n = " + std::to_string(n));
  return p->d.p;
}
int sp_dotlog_prove_t(sp_ctx* ctx, const sp_dotlog_gens* gens, uint8_t* strobe_state, uint8_t* tape_state, const sp_poly* x, const uint64_t blind_x[4],
                      const sp_poly* a, const uint64_t* y, const uint64_t blind_y[4], uint8_t** proof, size_t* proof_len, uint8_t Cx_out32[32],
                      uint8_t Cy_out32[32], uint64_t y_out[4]) {
  return guarded(ctx, [&] {
    const std::string what = "dotlog_prove";
    ProofStates st(strobe_state, tape_state, what);
    if (!proof || !proof_len || !Cx_out32 || !Cy_out32 || !y_out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    require_owned(ctx, gens, what, "gens");
    const size_t n = gens->g->n;
    const u256* dx = dotlog_vec(ctx, x, n, what, "x");
    const u256* da = dotlog_vec(ctx, a, n, what, "a");
    const Fq bx = scalar_in(blind_x, what + ": blind_x"), by = scalar_in(blind_y, what + ": blind_y");
    const Fq fy = y ? scalar_in(y, what + ": y") : Fq::zero();
    st.open();
    DotProductProofLog p;
    Cp Cx, Cy;
    Fq y_used;
    dotlog_prove(ctx->c, *gens->g, st.T(), st.tape(), dx, bx, da, y ? &fy : nullptr, by, p, Cx, Cy, y_used);
    st.proved();
    put_bytes(proof, proof_len, to_bincode(p));
    cp_out(Cx_out32, Cx);
    cp_out(Cy_out32, Cy);
    fq_out(y_out, y_used);
    flush_fine(ctx->c);
  });
}
int sp_dotlog_verify_t(sp_ctx* ctx, const sp_dotlog_gens* gens, uint8_t* strobe_state, const sp_poly* a, size_t n, const uint8_t Cx32[32],
                       const uint8_t Cy32[32], const uint8_t* proof, size_t proof_len) {
  return guarded(ctx, [&] {
    const std::string what = "dotlog_verify";
    ProofStates st(strobe_state);
    if (!proof && proof_len) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    require_owned(ctx, gens, what, "gens");
    if (n != gens->g->n) throw SpError(SP_ERR_INVALID_ARG, what + ": n = " + std::to_string(n) + " but gens have n = " + std::to_string(gens->g->n));
    const u256* da = dotlog_vec(ctx, a, n, what, "a");
    const Cp Cx = cp_in(Cx32, what + ": Cx"), Cy = cp_in(Cy32, what + ": Cy");
    st.open_verify();
    dotlog_verify_bytes(ctx->c, *gens->g, st.T(), da, Cx, Cy, proof, proof_len);
    flush_fine(ctx->c);
  });
}

// ---- polynomial commitments and evaluation proofs for the caller's tables (prover.cpp: pc_*).  Every argument is checked before the first
// launch and before the transcript or the tape is touched, so a refused call leaves the tables, the transcript and the tape as they were.
int sp_pc_gens_create(sp_ctx* ctx, size_t num_vars, const uint8_t* label, size_t label_len, sp_pc_gens** out) {
  return guarded(ctx, [&] {
    if (!out || (!label && label_len)) throw SpError(SP_ERR_INVALID_ARG, "pc_gens_create: NULL argument");
    if (num_vars > PC_MAX_VARS) throw SpError(SP_ERR_INVALID_ARG, "pc_gens_create: num_vars = " + std::to_string(num_vars) + " > " + std::to_string(PC_MAX_VARS));
    const size_t n = pc_gens_n(num_vars);
    std::unique_ptr<sp_pc_gens> g(new sp_pc_gens{&ctx->c, nullptr, num_vars, {}});
    g->set = std::make_shared<GenSet>(&ctx->c, std::string((const char*)label, label_len), n + 2, std::vector<size_t>{n, n + 1});
    g->g = pc_gens_view(*g->set, num_vars);
    *out = g.release();
  });
}
int sp_pc_gens_create_from(sp_ctx* ctx, const sp_pc_gens* larger, size_t num_vars, sp_pc_gens** out) {
  return guarded(ctx, [&] {
    const std::string what = "pc_gens_create_from";
    if (!out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    require_owned(ctx, larger, what, "gens handle");
    if (num_vars > larger->num_vars)
      throw SpError(SP_ERR_INVALID_ARG, what + ": num_vars = " + std::to_string(num_vars) + " > the larger gens' " + std::to_string(larger->num_vars));
    std::unique_ptr<sp_pc_gens> g(new sp_pc_gens{&ctx->c, larger->set, num_vars, {}});
    g->g = pc_gens_view(*g->set, num_vars);
    *out = g.release();
  });
}
void sp_pc_gens_free(sp_pc_gens* g) { delete g; }

// host only: no context
int sp_random_tape_new(const uint64_t seed[4], uint8_t* tape_state) {
  return host_guarded(nullptr, [&] {
    if (!seed || !tape_state) throw SpError(SP_ERR_INVALID_ARG, "random_tape_new: NULL argument");
    require_reduced(seed, 1, "random_tape_new: seed");
    RandomTape(std::string("proof"), fq_in(seed)).state().export_state(tape_state);   // random.rs:10-17
  });
}

int sp_pc_commit(sp_ctx* ctx, const sp_pc_gens* gens, sp_poly* const* polys, int k, uint8_t* tape_state, uint8_t** comm, size_t* comm_len, uint64_t* blinds_out) {
  return guarded(ctx, [&] {
    const std::string what = "pc_commit";
    if (!comm || !comm_len) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    require_count(what, k, "tables", "SP_PC_MAX_TABLES", SP_PC_MAX_TABLES);
    const Tables t = caller_tables(ctx, polys, k, what, 1);
    const size_t m = log2_ceil(t.len), ell = m + log2_ceil(next_pow2((size_t)k));
    pc_check_gens(ctx, gens, ell, what);
    const size_t L = (size_t)1 << (ell / 2);
    std::vector<Fq> blinds(L, Fq::zero());
    ProofStates st = ProofStates::tape_only(tape_state);
    st.open();
    if (tape_state) blinds = st.tape().random_vector("poly_blinds", L);   // dense_mlpoly.rs:185-189
    const std::vector<uint8_t> bytes = to_bincode(pc_commit(ctx->c, gens->g, t.d.data(), k, m, tape_state ? blinds.data() : nullptr));
    st.proved();
    put_bytes(comm, comm_len, bytes);
    if (blinds_out) put_scalars(blinds_out, blinds);
  });
}

int sp_pc_eval_prove_t(sp_ctx* ctx, const sp_pc_gens* gens, const sp_poly* poly, const uint64_t* blinds, const uint64_t* r, size_t ell, const uint64_t* Zr,
                       const uint64_t* blind_Zr, uint8_t* strobe_state, uint8_t* tape_state, uint8_t** proof, size_t* proof_len, uint8_t C_Zr32[32],
                       uint64_t Zr_out[4]) {
  return guarded(ctx, [&] {
    const std::string what = "pc_eval_prove";
    ProofStates st(strobe_state);
    if (!poly || !proof || !proof_len || !C_Zr32 || !Zr_out || (!r && ell)) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    sp_poly* const p = const_cast<sp_poly*>(poly);
    if (log2_ceil(caller_tables(ctx, &p, 1, what, 1).len) != ell || ell > PC_MAX_VARS)
      throw SpError(SP_ERR_INVALID_ARG, what + ": |r| = " + std::to_string(ell) + " but the table has " + std::to_string(poly->len) + " entries");
    pc_check_gens(ctx, gens, ell, what);
    const size_t L = (size_t)1 << (ell / 2);
    require_reduced(r, ell, "pc_eval_prove: r");
    if (Zr) require_reduced(Zr, 1, "pc_eval_prove: Zr");
    if (blind_Zr) require_reduced(blind_Zr, 1, "pc_eval_prove: blind_Zr");
    if (blinds) require_reduced(blinds, L, "pc_eval_prove: blinds");
    st.open_tape(tape_state, what);
    st.open();
    const std::vector<Fq> bl = blinds ? fq_vec(blinds, L) : std::vector<Fq>();
    const Fq Zr_in = Zr ? fq_in(Zr) : Fq::zero(), bZr = blind_Zr ? fq_in(blind_Zr) : Fq::zero();
    PolyEvalProof P;
    Cp C;
    Fq zr;
    polyeval_prove(ctx->c, poly->d.p, blinds ? &bl : nullptr, fq_vec(r, ell), Zr ? &Zr_in : nullptr, blind_Zr ? &bZr : nullptr, gens->g, st.T(), st.tape(), P, C, &zr);
    st.proved();
    put_bytes(proof, proof_len, to_bincode(P));
    memcpy(C_Zr32, C.b, 32);
    fq_out(Zr_out, zr);
  });
}

int sp_pc_eval_verify_t(sp_ctx* ctx, const sp_pc_gens* gens, const uint8_t* comm, size_t comm_len, const uint64_t* r, size_t ell, const uint8_t C_Zr32[32],
                        const uint64_t Zr[4], uint8_t* strobe_state, const uint8_t* proof, size_t proof_len) {
  return guarded(ctx, [&] {
    const std::string what = "pc_eval_verify";
    ProofStates st(strobe_state);
    if ((!comm && comm_len) || (!proof && proof_len) || (!r && ell)) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    if (!C_Zr32 == !Zr) throw SpError(SP_ERR_INVALID_ARG, what + ": give exactly one of C_Zr and Zr");
    if (ell > PC_MAX_VARS) throw SpError(SP_ERR_INVALID_ARG, what + ": |r| = " + std::to_string(ell) + " > " + std::to_string(PC_MAX_VARS));
    pc_check_gens(ctx, gens, ell, what);
    require_reduced(r, ell, "pc_eval_verify: r");
    if (Zr) require_reduced(Zr, 1, "pc_eval_verify: Zr");
    const PolyCommitment pc = from_bincode<PolyCommitment>(comm, comm_len, SP_ERR_INVALID_ARG, "polynomial commitment");
    Cp c;
    if (C_Zr32) memcpy(c.b, C_Zr32, 32);
    const Fq zr = Zr ? fq_in(Zr) : Fq::zero();
    st.open_verify();
    pc_eval_verify(ctx->c, gens->g, pc, fq_vec(r, ell), C_Zr32 ? &c : nullptr, Zr ? &zr : nullptr, st.T(), proof, proof_len);
  });
}

int sp_pc_eval_prove_joint_t(sp_ctx* ctx, const sp_pc_gens* gens, sp_poly* const* polys, int k, const uint64_t* blinds, const uint64_t* r, size_t m,
                             uint8_t* strobe_state, uint8_t* tape_state, uint8_t** proof, size_t* proof_len, uint64_t* evals_out) {
  return guarded(ctx, [&] {
    const std::string what = "pc_eval_prove_joint";
    ProofStates st(strobe_state);
    if (!proof || !proof_len || !evals_out || (!r && m)) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    require_count(what, k, "tables", "SP_PC_MAX_TABLES", SP_PC_MAX_TABLES);
    const Tables t = caller_tables(ctx, polys, k, what, 1);
    if (log2_ceil(t.len) != m || m > PC_MAX_VARS)
      throw SpError(SP_ERR_INVALID_ARG, what + ": |r| = " + std::to_string(m) + " but the tables have " + std::to_string(t.len) + " entries");
    const size_t ell = m + log2_ceil(next_pow2((size_t)k)), L = (size_t)1 << (ell / 2);
    pc_check_gens(ctx, gens, ell, what);
    require_reduced(r, m, "pc_eval_prove_joint: r");
    if (blinds) require_reduced(blinds, L, "pc_eval_prove_joint: blinds");
    st.open_tape(tape_state, what);
    st.open();
    const std::vector<Fq> bl = blinds ? fq_vec(blinds, L) : std::vector<Fq>();
    PolyEvalProof P;
    std::vector<Fq> evals;
    pc_eval_prove_joint(ctx->c, gens->g, t.d.data(), k, fq_vec(r, m), blinds ? &bl : nullptr, st.T(), st.tape(), P, evals);
    st.proved();
    put_bytes(proof, proof_len, to_bincode(P));
    put_scalars(evals_out, evals);
  });
}

int sp_pc_eval_verify_joint_t(sp_ctx* ctx, const sp_pc_gens* gens, const uint8_t* comm, size_t comm_len, const uint64_t* r, size_t m, const uint64_t* evals,
                              int k, uint8_t* strobe_state, const uint8_t* proof, size_t proof_len) {
  return guarded(ctx, [&] {
    const std::string what = "pc_eval_verify_joint";
    ProofStates st(strobe_state);
    if ((!comm && comm_len) || (!proof && proof_len) || (!r && m) || !evals) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    require_count(what, k, "evaluations", "SP_PC_MAX_TABLES", SP_PC_MAX_TABLES);
    if (m > PC_MAX_VARS) throw SpError(SP_ERR_INVALID_ARG, what + ": |r| = " + std::to_string(m) + " > " + std::to_string(PC_MAX_VARS));
    pc_check_gens(ctx, gens, m + log2_ceil(next_pow2((size_t)k)), what);
    require_reduced(r, m, "pc_eval_verify_joint: r");
    require_reduced(evals, (size_t)k, "pc_eval_verify_joint: evals");
    const PolyCommitment pc = from_bincode<PolyCommitment>(comm, comm_len, SP_ERR_INVALID_ARG, "polynomial commitment");
    st.open_verify();
    pc_eval_verify_joint(ctx->c, gens->g, pc, fq_vec(r, m), fq_vec(evals, (size_t)k), st.T(), proof, proof_len);
  });
}

// ---- product circuits of the caller's tables (product.cpp: prod_*).  Every argument is checked before the first launch or allocation and before
// the transcript is touched, so a refused call leaves the tables, the transcript and the device memory as they were.
// the body of sp_prod_build (dotp_forms NULL, kd = 0) and sp_prod_build_dotp
static void prod_build_entry(sp_ctx* ctx, sp_poly* const* tables, int ntables, const sp_prod_leaves* leaves, int k, const sp_prod_leaves* dotp_forms, int kd,
                             sp_prod_circuits** out, uint64_t* products_out, uint64_t* dotp_claims_out, const std::string& what) {
  if (!out || !products_out || (kd && (!dotp_forms || !dotp_claims_out))) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
  prod_counts(leaves, k, ntables, what);   // before any table is looked at
  if (dotp_forms) dotp_counts(k, kd, what);
  const size_t m = log2_ceil(caller_tables(ctx, tables, ntables, what, 2).len);
  const std::vector<LeafForm> f = prod_forms(leaves, k, ntables, what);
  const std::vector<LeafForm> g = checked_forms(dotp_forms, 3 * kd, ntables, [&](int c) {
    return what + ": dot product " + std::to_string(c / 3) + " " + DOTP_OPERAND[c % 3];
  });
  std::vector<dev::ProdLeaves> d(k);
  for (int c = 0; c < k; c++) d[c] = dev::ProdLeaves{device_form(f[c], tables), nullptr, nullptr};
  std::vector<dev::DotpOperands> dd(kd);
  for (int i = 0; i < kd; i++) dd[i] = dev::DotpOperands{{device_form(g[3 * i], tables), device_form(g[3 * i + 1], tables), device_form(g[3 * i + 2], tables)}, nullptr};
  std::unique_ptr<sp_prod_circuits> h(new sp_prod_circuits{&ctx->c, m, {}, false, {}});
  put_scalars(products_out, prod_build(ctx->c, d, dd, (size_t)1 << m, h->cs, h->dotps));
  for (size_t j = 0; j < h->dotps.d.size(); j++) fq_out(dotp_claims_out + 4 * j, h->dotps.d[j].claim);
  *out = h.release();
}

int sp_prod_build(sp_ctx* ctx, sp_poly* const* tables, int ntables, const sp_prod_leaves* leaves, int k, sp_prod_circuits** out, uint64_t* products_out) {
  return guarded(ctx, [&] { prod_build_entry(ctx, tables, ntables, leaves, k, nullptr, 0, out, products_out, nullptr, "prod_build"); });
}

int sp_prod_build_dotp(sp_ctx* ctx, sp_poly* const* tables, int ntables, const sp_prod_leaves* leaves, int k, const sp_prod_leaves* dotp_forms, int kd,
                       sp_prod_circuits** out, uint64_t* products_out, uint64_t* dotp_claims_out) {
  return guarded(ctx, [&] {
    const std::string what = "prod_build_dotp";
    if (!dotp_forms || !dotp_claims_out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    prod_build_entry(ctx, tables, ntables, leaves, k, dotp_forms, kd, out, products_out, dotp_claims_out, what);
  });
}

// the body of sp_prod_prove_t (dotp_evals_out NULL: refuses a handle with dot products) and sp_prod_prove_dotp_t
static void prod_prove_entry(sp_ctx* ctx, sp_prod_circuits* c, uint8_t* strobe_state, uint8_t** proof, size_t* proof_len, uint64_t* rand_out,
                             uint64_t* leaf_evals_out, uint64_t* dotp_evals_out, bool with_dotp, const std::string& what) {
  ProofStates st(strobe_state);
  if (!proof || !proof_len || !rand_out || !leaf_evals_out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
  require_owned(ctx, c, what, "circuits handle");
  if (c->spent) throw SpError(SP_ERR_INVALID_ARG, what + ": the circuits were consumed by an earlier proof (their layers are bound in place)");
  if (!c->dotps.d.empty() && !with_dotp)
    throw SpError(SP_ERR_INVALID_ARG, what + ": the circuits hold dot products, whose evaluations only sp_prod_prove_dotp_t returns");
  if (!c->dotps.d.empty() && !dotp_evals_out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
  std::vector<ProdCircuit*> cs;
  for (auto& p : c->cs) cs.push_back(p.get());
  st.open();
  c->spent = true;
  ProductCircuitEvalProofBatched P;
  std::vector<Fq> rand, evals, dotp_evals;
  prod_prove(ctx->c, cs, c->dotps.d, st.T(), P, rand, evals, dotp_evals);
  c->cs.clear();
  c->dotps = ProdDotps();
  st.proved();
  put_bytes(proof, proof_len, to_bincode(P));
  put_scalars(rand_out, rand);
  put_scalars(leaf_evals_out, evals);
  if (dotp_evals_out) put_scalars(dotp_evals_out, dotp_evals);
}

int sp_prod_prove_t(sp_ctx* ctx, sp_prod_circuits* c, uint8_t* strobe_state, uint8_t** proof, size_t* proof_len, uint64_t* rand_out, uint64_t* leaf_evals_out) {
  return guarded(ctx, [&] { prod_prove_entry(ctx, c, strobe_state, proof, proof_len, rand_out, leaf_evals_out, nullptr, false, "prod_prove"); });
}

int sp_prod_prove_dotp_t(sp_ctx* ctx, sp_prod_circuits* c, uint8_t* strobe_state, uint8_t** proof, size_t* proof_len, uint64_t* rand_out,
                         uint64_t* leaf_evals_out, uint64_t* dotp_evals_out) {
  return guarded(ctx, [&] { prod_prove_entry(ctx, c, strobe_state, proof, proof_len, rand_out, leaf_evals_out, dotp_evals_out, true, "prod_prove_dotp"); });
}

void sp_prod_free(sp_prod_circuits* c) { delete c; }

// the body of sp_prod_verify_t (kd = 0) and sp_prod_verify_dotp_t; host only
static void prod_verify_entry(const uint8_t* proof, size_t proof_len, const uint64_t* products, int k, const uint64_t* dotp_claims, int kd, size_t m,
                              uint8_t* strobe_state, uint64_t* rand_out, uint64_t* leaf_claims_out, uint64_t* dotp_claims_out, const std::string& what) {
  ProofStates st(strobe_state);
  if ((!proof && proof_len) || !products || !rand_out || !leaf_claims_out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
  require_count(what, k, "products", "SP_PROD_MAX_CIRCUITS", SP_PROD_MAX_CIRCUITS);
  if (dotp_claims) dotp_counts(k, kd, what);
  if (m < 1 || m > PROD_MAX_VARS) throw SpError(SP_ERR_INVALID_ARG, what + ": m = " + std::to_string(m) + "; 1 .. " + std::to_string(PROD_MAX_VARS) + " supported");
  require_reduced(products, (size_t)k, (what + ": product").c_str());
  require_reduced(dotp_claims, 2 * (size_t)kd, (what + ": dotp claim").c_str());
  st.open_verify();
  const BatchedOut o = prod_verify(proof, proof_len, fq_vec(products, (size_t)k), fq_vec(dotp_claims, 2 * (size_t)kd), m, st.T());
  put_scalars(rand_out, o.rand);
  put_scalars(leaf_claims_out, o.claims);
  if (dotp_claims_out) put_scalars(dotp_claims_out, o.claims_dotp);
}

// host only: no device work, so ctx may be NULL (the message then goes where sp_last_error(NULL) reads it)
int sp_prod_verify_t(sp_ctx* ctx, const uint8_t* proof, size_t proof_len, const uint64_t* products, int k, size_t m, uint8_t* strobe_state, uint64_t* rand_out,
                     uint64_t* leaf_claims_out) {
  return host_guarded(ctx, [&] {
    prod_verify_entry(proof, proof_len, products, k, nullptr, 0, m, strobe_state, rand_out, leaf_claims_out, nullptr, "prod_verify");
  });
}

int sp_prod_verify_dotp_t(sp_ctx* ctx, const uint8_t* proof, size_t proof_len, const uint64_t* products, int k, const uint64_t* dotp_claims, int kd, size_t m,
                          uint8_t* strobe_state, uint64_t* rand_out, uint64_t* leaf_claims_out, uint64_t* dotp_claims_out) {
  return host_guarded(ctx, [&] {
    const std::string what = "prod_verify_dotp";
    if (!dotp_claims || !dotp_claims_out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    prod_verify_entry(proof, proof_len, products, k, dotp_claims, kd, m, strobe_state, rand_out, leaf_claims_out, dotp_claims_out, what);
  });
}

// host only
int sp_prod_leaf_eval(const sp_prod_leaves* leaves, int k, const uint64_t* table_evals, int ntables, const uint64_t* rand, size_t m, uint64_t* out) {
  return host_guarded(nullptr, [&] {
    const std::string what = "prod_leaf_eval";
    if (!table_evals || !out || (!rand && m)) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    if (m > PROD_MAX_VARS) throw SpError(SP_ERR_INVALID_ARG, what + ": m = " + std::to_string(m) + " > " + std::to_string(PROD_MAX_VARS));
    const std::vector<LeafForm> f = prod_forms(leaves, k, ntables, what);
    require_reduced(table_evals, (size_t)ntables, "prod_leaf_eval: table evaluation");
    require_reduced(rand, m, "prod_leaf_eval: rand");
    Fq id = Fq::zero();   // IdentityPolynomial::evaluate (dense_mlpoly.rs:105-115): sum_i 2^(m-1-i) rand_i
    for (size_t i = 0; i < m; i++) id += Fq::from_u64((uint64_t)1 << (m - 1 - i)) * fq_in(rand + 4 * i);
    for (int c = 0; c < k; c++) {
      Fq v = f[c].cst + f[c].idx * id;
      for (uint32_t s = 0; s < f[c].nsrc; s++) v += f[c].coeff[s] * fq_in(table_evals + 4 * f[c].src[s]);
      fq_out(out + 4 * c, v);
    }
  });
}

// ---- SPARK of the caller's matrices (snark.cpp: spark_*).  Every argument is checked before the first allocation and before the transcript or
// the tape is touched, so a refused call leaves them as they were.
static const size_t SPARK_MAX_VARS = 30;   // 32-bit addresses, and fewer than 2^31 cells to sort
static void spark_shape(size_t x, size_t y, const std::string& what) {
  if (std::max(x, y) == 0) throw SpError(SP_ERR_INVALID_ARG, what + ": num_vars_x = num_vars_y = 0 (one memory cell) is not supported");
  if (std::max(x, y) > SPARK_MAX_VARS)
    throw SpError(SP_ERR_INVALID_ARG, what + ": max(num_vars_x, num_vars_y) = " + std::to_string(std::max(x, y)) + " > " + std::to_string(SPARK_MAX_VARS) +
                                          " (addresses are 32-bit)");
}
static void spark_check_gens(const sp_ctx* ctx, const sp_spark_gens* g, size_t x, size_t y, size_t N, size_t b, const std::string& what) {
  require_owned(ctx, g, what, "gens handle");
  if (!SparkDims(x, y, N, b).fits(g->g))
    throw SpError(SP_ERR_INVALID_ARG, what + ": gens for (x, y, nz, b) = (" + std::to_string(g->x) + ", " + std::to_string(g->y) + ", " + std::to_string(g->nz) +
                                          ", " + std::to_string(g->b) + ") do not fit (" + std::to_string(x) + ", " + std::to_string(y) + ", " + std::to_string(N) +
                                          ", " + std::to_string(b) + ")");
}
static void spark_commit_common(sp_ctx* ctx, const sp_spark_gens* gens, const sp_spark_entries* mats, int b, size_t x, size_t y, sp_spark_dense** dense,
                                uint8_t** comm, size_t* comm_len, bool device) {
  const std::string what = device ? "spark_commit_device" : "spark_commit";
  Ctx& c = ctx->c;
  if (!dense || !comm || !comm_len || !mats) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
  require_count(what, b, "matrices", "SP_SPARK_MAX_BATCH", SP_SPARK_MAX_BATCH);
  spark_shape(x, y, what);
  size_t N = 1;
  for (int m = 0; m < b; m++) {
    const sp_spark_entries& e = mats[m];
    if (e.nnz && (!e.row || !e.col || !e.val32)) throw SpError(SP_ERR_INVALID_ARG, what + ": matrix " + std::to_string(m) + ": NULL array");
    if (e.nnz >= ((size_t)1 << 31)) throw SpError(SP_ERR_INVALID_ARG, what + ": matrix " + std::to_string(m) + ": 2^31 or more entries");
    if (device) {
      const std::string at = "matrix " + std::to_string(m);
      require_device(c, e.row, e.nnz, (at + " row").c_str());
      require_device(c, e.col, e.nnz, (at + " col").c_str());
      require_device(c, e.val32, e.nnz, (at + " val").c_str());
    }
    N = std::max(N, next_pow2(e.nnz));
  }
  if (N < 2) throw SpError(SP_ERR_INVALID_ARG, what + ": every matrix has at most one entry (num_ops = 1 leaves the product circuits without layers)");
  spark_check_gens(ctx, gens, x, y, N, (size_t)b, what);
  // the caller's entries meet the checks of sp_instance_create: row < 2^x, col < 2^y, val < q
  DevBuf<uint32_t> row[SP_SPARK_MAX_BATCH], col[SP_SPARK_MAX_BATCH];
  DevBuf<u256> val[SP_SPARK_MAX_BATCH];
  dev::CooIn in{};
  dev::CooOut co{};
  SparkMatrix sm[SP_SPARK_MAX_BATCH];
  for (int m = 0; m < b; m++) {
    const sp_spark_entries& e = mats[m];
    in.row[m] = e.row; in.col[m] = e.col; in.val[m] = e.val32; in.n[m] = e.nnz;
    row[m].alloc(e.nnz); col[m].alloc(e.nnz); val[m].alloc(e.nnz);
    co.row[m] = row[m].p; co.col[m] = col[m].p; co.val[m] = val[m].p;
    sm[m] = SparkMatrix{row[m].p, col[m].p, val[m].p, e.nnz};
  }
  const size_t ncols = (size_t)1 << y;
  ingest(c, in, b, !device, co, (size_t)1 << x, ncols, ncols, 0, [&](size_t m, size_t k, unsigned code) { refuse_entry(what, m, k, code); });
  std::unique_ptr<sp_spark_dense> d(new sp_spark_dense{&c, {}});
  SparseMatPolyCommitment cm;
  spark_commit(c, sm, (size_t)b, x, y, gens->g, d->d, cm);
  put_bytes(comm, comm_len, to_bincode(cm));
  *dense = d.release();
}
// rx, ry of a dense's shape
static void spark_point(const sp_spark_dense* d, const uint64_t* rx, size_t x, const uint64_t* ry, size_t y, const std::string& what) {
  if ((!rx && x) || (!ry && y)) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
  if (x != d->d.x || y != d->d.y)
    throw SpError(SP_ERR_INVALID_ARG, what + ": |rx| = " + std::to_string(x) + ", |ry| = " + std::to_string(y) + " but the matrices have 2^" + std::to_string(d->d.x) +
                                          " rows and 2^" + std::to_string(d->d.y) + " columns");
  require_reduced(rx, x, (what + ": rx").c_str());
  require_reduced(ry, y, (what + ": ry").c_str());
}

int sp_spark_gens_create(sp_ctx* ctx, const uint8_t* label, size_t label_len, size_t x, size_t y, size_t nz, size_t b, sp_spark_gens** out) {
  return guarded(ctx, [&] {
    const std::string what = "spark_gens_create";
    if (!out || (!label && label_len)) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    if (b < 1 || b > SP_SPARK_MAX_BATCH)
      throw SpError(SP_ERR_INVALID_ARG, what + ": batch_size = " + std::to_string(b) + "; 1 .. SP_SPARK_MAX_BATCH = " + std::to_string(SP_SPARK_MAX_BATCH) + " supported");
    spark_shape(x, y, what);
    if (nz > ((size_t)1 << 31)) throw SpError(SP_ERR_INVALID_ARG, what + ": num_nz_entries > 2^31");
    const SparkDims d(x, y, nz, b);
    auto set = std::make_shared<GenSet>(&ctx->c, std::string((const char*)label, label_len), d.bases(), d.host_bases());
    std::unique_ptr<sp_spark_gens> g(new sp_spark_gens{&ctx->c, x, y, nz, b, SparkGens(set, d)});
    *out = g.release();
  });
}
void sp_spark_gens_free(sp_spark_gens* g) { delete g; }
int sp_spark_commit(sp_ctx* ctx, const sp_spark_gens* gens, const sp_spark_entries* matrices, int b, size_t x, size_t y, sp_spark_dense** dense, uint8_t** comm,
                    size_t* comm_len) {
  return guarded(ctx, [&] { spark_commit_common(ctx, gens, matrices, b, x, y, dense, comm, comm_len, false); });
}
int sp_spark_commit_device(sp_ctx* ctx, const sp_spark_gens* gens, const sp_spark_entries* matrices, int b, size_t x, size_t y, sp_spark_dense** dense,
                           uint8_t** comm, size_t* comm_len) {
  return guarded(ctx, [&] { spark_commit_common(ctx, gens, matrices, b, x, y, dense, comm, comm_len, true); });
}
void sp_spark_dense_free(sp_spark_dense* d) { delete d; }
int sp_spark_evaluate(sp_ctx* ctx, const sp_spark_dense* dense, const uint64_t* rx, size_t x, const uint64_t* ry, size_t y, uint64_t* out) {
  return guarded(ctx, [&] {
    const std::string what = "spark_evaluate";
    if (!out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    require_owned(ctx, dense, what, "dense handle");
    spark_point(dense, rx, x, ry, y, what);
    std::vector<Fq> ev(dense->d.b);
    spark_evaluate(ctx->c, dense->d, fq_vec(rx, x), fq_vec(ry, y), ev.data());
    put_scalars(out, ev);
  });
}
int sp_spark_eval_prove_t(sp_ctx* ctx, const sp_spark_dense* dense, const sp_spark_gens* gens, const uint64_t* rx, size_t x, const uint64_t* ry, size_t y,
                          const uint64_t* evals, uint8_t* strobe_state, uint8_t* tape_state, uint8_t** proof, size_t* proof_len, uint64_t* evals_out) {
  return guarded(ctx, [&] {
    const std::string what = "spark_eval_prove";
    ProofStates st(strobe_state);
    if (!proof || !proof_len || !evals_out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    require_owned(ctx, dense, what, "dense handle");
    const SparkDense& d = dense->d;
    spark_check_gens(ctx, gens, d.x, d.y, d.N, d.b, what);
    spark_point(dense, rx, x, ry, y, what);
    if (evals) require_reduced(evals, d.b, (what + ": evals").c_str());
    st.open_tape(tape_state, what);
    const std::vector<Fq> vx = fq_vec(rx, x), vy = fq_vec(ry, y);
    std::vector<Fq> ev(d.b);
    spark_evaluate(ctx->c, d, vx, vy, ev.data());
    if (evals)
      for (size_t m = 0; m < d.b; m++)
        if (!(fq_in(evals + 4 * m) == ev[m])) throw SpError(SP_ERR_INVALID_ARG, what + ": evals[" + std::to_string(m) + "] is not M_" + std::to_string(m) + "(rx, ry)");
    st.open();
    ctx->c.timings.clear();
    SparseMatPolyEvalProof P;
    spark_eval_prove(ctx->c, d, vx, vy, ev, gens->g, st.T(), st.tape(), P);
    st.proved();
    put_bytes(proof, proof_len, to_bincode(P));
    put_scalars(evals_out, ev);
  });
}
int sp_spark_eval_verify_t(sp_ctx* ctx, const sp_spark_gens* gens, const uint8_t* comm, size_t comm_len, const uint64_t* rx, size_t x, const uint64_t* ry,
                           size_t y, const uint64_t* evals, int b, uint8_t* strobe_state, const uint8_t* proof, size_t proof_len) {
  return guarded(ctx, [&] {
    const std::string what = "spark_eval_verify";
    ProofStates st(strobe_state);
    if ((!comm && comm_len) || (!proof && proof_len) || (!rx && x) || (!ry && y) || !evals) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    require_count(what, b, "evaluations", "SP_SPARK_MAX_BATCH", SP_SPARK_MAX_BATCH);
    require_owned(ctx, gens, what, "gens handle");
    if (std::max(x, y) > SPARK_MAX_VARS) throw SpError(SP_ERR_INVALID_ARG, what + ": max(|rx|, |ry|) > " + std::to_string(SPARK_MAX_VARS));
    require_reduced(rx, x, (what + ": rx").c_str());
    require_reduced(ry, y, (what + ": ry").c_str());
    require_reduced(evals, (size_t)b, (what + ": evals").c_str());
    const SparseMatPolyCommitment cm = from_bincode<SparseMatPolyCommitment>(comm, comm_len, SP_ERR_VERIFY, "sparse polynomial commitment");
    check_spark_commitment(cm, (size_t)b, x, y, gens->g);
    st.open_verify();
    spark_eval_verify(ctx->c, cm, fq_vec(rx, x), fq_vec(ry, y), fq_vec(evals, (size_t)b), gens->g, st.T(), proof, proof_len);
  });
}

// ---- batch verifiers
// ---- products of the caller's matrices (kernels_inst.cu: spmat_products).  Every argument is checked before the first allocation or launch.
static_assert(SP_SPMAT_MAX_BATCH == SP_SC_MAX_TABLES, "the b products of one call are the tables of one caller sumcheck");
static_assert(SP_SPMAT_MAX_BATCH >= SP_SPARK_MAX_BATCH, "a SPARK batch's matrices fit one product call");
struct SpmatOrder {   // one matrix sorted by key: row order (key = row, src = col) or column order (key = col, src = row)
  DevBuf<uint32_t> key, src;
  DevBuf<u256> val;
};
struct sp_spmat {
  Ctx* ctx;
  int b;
  size_t x, y, total;
  size_t nnz[SP_SPMAT_MAX_BATCH];
  SpmatOrder by_row[SP_SPMAT_MAX_BATCH], by_col[SP_SPMAT_MAX_BATCH];
  uint64_t max_row, max_col;   // over every entry; meaningful when total > 0
};
static const size_t SPMAT_MAX_VARS = 30;
static void spmat_create_common(sp_ctx* ctx, const sp_spark_entries* mats, int b, size_t x, size_t y, sp_spmat** out, bool device) {
  const std::string what = device ? "spmat_create_device" : "spmat_create";
  Ctx& c = ctx->c;
  if (!out || !mats) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
  require_count(what, b, "matrices", "SP_SPMAT_MAX_BATCH", SP_SPMAT_MAX_BATCH);
  if (std::max(x, y) > SPMAT_MAX_VARS)
    throw SpError(SP_ERR_INVALID_ARG, what + ": max(num_vars_x, num_vars_y) = " + std::to_string(std::max(x, y)) + " > " + std::to_string(SPMAT_MAX_VARS));
  size_t total = 0;
  for (int m = 0; m < b; m++) {
    const sp_spark_entries& e = mats[m];
    const std::string at = what + ": matrix " + std::to_string(m);
    if (e.nnz && (!e.row || !e.col || !e.val32)) throw SpError(SP_ERR_INVALID_ARG, at + ": NULL array");
    if (device) {
      require_device(c, e.row, e.nnz, (at + " row").c_str());
      require_device(c, e.col, e.nnz, (at + " col").c_str());
      require_device(c, e.val32, e.nnz, (at + " val").c_str());
    }
    total += e.nnz;
    if (e.nnz >= ((size_t)1 << 32) || total >= ((size_t)1 << 32)) throw SpError(SP_ERR_INVALID_ARG, what + ": 2^32 or more entries in all");
  }
  std::unique_ptr<sp_spmat> S(new sp_spmat{&c, b, x, y, total, {}, {}, {}, 0, 0});
  // matrix by matrix: the entries meet the checks of sp_instance_create (row < 2^x, col < 2^y, val < q) on the device, then both sorts
  for (int m = 0; m < b; m++) {
    const sp_spark_entries& e = mats[m];
    const size_t n = e.nnz;
    S->nnz[m] = n;
    if (!n) continue;
    dev::CooIn in{};
    in.row[0] = e.row; in.col[0] = e.col; in.val[0] = e.val32; in.n[0] = n;
    DevBuf<uint32_t> row(n), col(n);
    DevBuf<u256> val(n);
    dev::CooOut co{};
    co.row[0] = row.p; co.col[0] = col.p; co.val[0] = val.p;
    // the matrices are ingested in order, so a bad entry here is the first in (matrix, entry) order
    ingest(c, in, 1, !device, co, (size_t)1 << x, (size_t)1 << y, (size_t)1 << y, 0, [&](size_t, size_t k, unsigned code) { refuse_entry(what, m, k, code); });
    DevBuf<uint8_t> scratch(dev::spmat_sort_scratch_bytes(n));
    SpmatOrder& R = S->by_row[m];
    SpmatOrder& C = S->by_col[m];
    R.key.alloc(n); R.src.alloc(n); R.val.alloc(n);
    C.key.alloc(n); C.src.alloc(n); C.val.alloc(n);
    dev::spmat_sort(R.key.p, R.src.p, R.val.p, row.p, col.p, val.p, (size_t)1 << x, n, scratch.p, c.stream);
    dev::spmat_sort(C.key.p, C.src.p, C.val.p, col.p, row.p, val.p, (size_t)1 << y, n, scratch.p, c.stream);
    uint32_t last[2] = {0, 0};   // the largest row and column: the last keys of the two orders
    dev::d2h(&last[0], R.key.p + n - 1, 4, c.stream);
    dev::d2h(&last[1], C.key.p + n - 1, 4, c.stream);
    c.sync();
    S->max_row = std::max<uint64_t>(S->max_row, last[0]);
    S->max_col = std::max<uint64_t>(S->max_col, last[1]);
  }
  *out = S.release();
}
// outs[m] = M_m x (row order) or M_m^T x (transpose: column order), nout entries each, for every matrix m of S
static void spmat_run(Ctx& c, const sp_spmat& S, bool transpose, const u256* x, u256* const* outs, size_t nout) {
  dev::SpmatBatch B{};
  B.b = S.b;
  for (int m = 0; m < S.b; m++) {
    const SpmatOrder& o = transpose ? S.by_col[m] : S.by_row[m];
    B.key[m] = o.key.p; B.src[m] = o.src.p; B.val[m] = o.val.p; B.nnz[m] = S.nnz[m];
    B.out[m] = outs[m];
  }
  DevBuf<uint8_t> scratch(dev::spmat_products_scratch_bytes(S.total));
  dev::spmat_products(B, x, nout, scratch.p, c.stream);
}
// out = sum_m w[m] M_m^T e (nout entries), from the b tables in scratch
static void spmat_weighted(Ctx& c, const sp_spmat& S, const u256* e, const u256* w, u256* out, size_t nout) {
  DevBuf<u256> tables(nout * S.b);
  u256* t[SP_SPMAT_MAX_BATCH];
  for (int m = 0; m < S.b; m++) t[m] = tables.p + nout * m;
  spmat_run(c, S, true, e, t, nout);
  dev::LincombTables lt{};
  lt.b = S.b;
  for (int m = 0; m < S.b; m++) { lt.t[m] = t[m]; lt.w[m] = w[m]; }
  dev::lincomb_many(out, lt, nout, c.stream);
}
// M_m z (transpose = false: row order, z of num_cols entries, outputs of num_rows) or M_m^T e (column order, e of num_rows, outputs of num_cols)
static void spmat_product(sp_ctx* ctx, const sp_spmat* S, const sp_poly* x, size_t num_rows, size_t num_cols, const uint64_t* weights, sp_poly** outs,
                          bool transpose) {
  const std::string what = transpose ? "spmat_eval_table" : "spmat_multiply_vec";
  const char* xname = transpose ? "e" : "z";
  Ctx& c = ctx->c;
  if (!outs) throw SpError(SP_ERR_INVALID_ARG, what + ": outs is NULL");
  require_owned(ctx, S, what, "matrices");
  require_owned(ctx, x, what, xname);
  const size_t lim = (size_t)1 << 32;
  if (num_rows < 1 || num_rows > lim) throw SpError(SP_ERR_INVALID_ARG, what + ": num_rows = " + std::to_string(num_rows) + "; 1 .. 2^32 supported");
  if (num_cols < 1 || num_cols > lim) throw SpError(SP_ERR_INVALID_ARG, what + ": num_cols = " + std::to_string(num_cols) + "; 1 .. 2^32 supported");
  const size_t want = transpose ? num_rows : num_cols;
  if (x->len != want)
    throw SpError(SP_ERR_INVALID_ARG, what + ": len(" + xname + ") = " + std::to_string(x->len) + " but " + (transpose ? "num_rows" : "num_cols") + " = " +
                                          std::to_string(want));
  if (S->total && S->max_row >= num_rows)
    throw SpError(SP_ERR_INVALID_ARG, what + ": num_rows = " + std::to_string(num_rows) + " but an entry has row " + std::to_string(S->max_row));
  if (S->total && S->max_col >= num_cols)
    throw SpError(SP_ERR_INVALID_ARG, what + ": num_cols = " + std::to_string(num_cols) + " but an entry has col " + std::to_string(S->max_col));
  if (weights) require_reduced(weights, (size_t)S->b, (what + ": weights").c_str());
  const size_t nout = transpose ? num_cols : num_rows;
  const int nres = weights ? 1 : S->b;
  std::vector<std::unique_ptr<sp_poly>> res(nres);
  for (int i = 0; i < nres; i++) res[i].reset(new sp_poly{&c, DevBuf<u256>(nout), nout});
  if (weights) {
    spmat_weighted(c, *S, x->d.p, reinterpret_cast<const u256*>(weights), res[0]->d.p, nout);
  } else {
    u256* o[SP_SPMAT_MAX_BATCH];
    for (int m = 0; m < S->b; m++) o[m] = res[m]->d.p;
    spmat_run(c, *S, transpose, x->d.p, o, nout);
  }
  for (int i = 0; i < nres; i++) outs[i] = res[i].release();
}

int sp_spmat_create(sp_ctx* ctx, const sp_spark_entries* matrices, int b, size_t num_vars_x, size_t num_vars_y, sp_spmat** out) {
  return guarded(ctx, [&] { spmat_create_common(ctx, matrices, b, num_vars_x, num_vars_y, out, false); });
}
int sp_spmat_create_device(sp_ctx* ctx, const sp_spark_entries* matrices, int b, size_t num_vars_x, size_t num_vars_y, sp_spmat** out) {
  return guarded(ctx, [&] { spmat_create_common(ctx, matrices, b, num_vars_x, num_vars_y, out, true); });
}
void sp_spmat_free(sp_spmat* m) { delete m; }
int sp_spmat_multiply_vec(sp_ctx* ctx, const sp_spmat* mats, size_t num_rows, size_t num_cols, const sp_poly* z, sp_poly** outs) {
  return guarded(ctx, [&] { spmat_product(ctx, mats, z, num_rows, num_cols, nullptr, outs, false); });
}
int sp_spmat_eval_table(sp_ctx* ctx, const sp_spmat* mats, const sp_poly* e, size_t num_rows, size_t num_cols, const uint64_t* weights_mont, sp_poly** outs) {
  return guarded(ctx, [&] { spmat_product(ctx, mats, e, num_rows, num_cols, weights_mont, outs, true); });
}

// ---- R1CSProof of the caller's matrices (prover.cpp: r1cs_prove, verifier.cpp: r1cs_verify_bytes), on this rank's GPU alone
struct sp_r1cs_gens { Ctx* ctx; size_t num_vars; std::unique_ptr<R1CSGens> g; };
static const size_t R1CS_MAX_LOG = 32;   // num_cons and 2 num_vars: the tiled products index rows and columns with 32 bits
static bool is_pow2(size_t x) { return x && !(x & (x - 1)); }
// num_cons >= 2 and num_vars >= 1 powers of two (the verifier's check_dims), with both sumchecks short enough to stage
static void r1cs_dims(size_t num_cons, size_t num_vars, const std::string& what) {
  if (num_cons < 2 || !is_pow2(num_cons) || !is_pow2(num_vars))
    throw SpError(SP_ERR_INVALID_ARG, what + ": num_cons = " + std::to_string(num_cons) + " and num_vars = " + std::to_string(num_vars) +
                                          " must be powers of two, num_cons >= 2");
  const size_t lx = log2_ceil(num_cons), ly = log2_ceil(2 * num_vars);
  if (std::max(lx, ly) > std::min(R1CS_MAX_LOG, zk_sumcheck_max_rounds()))
    throw SpError(SP_ERR_INVALID_ARG, what + ": log2 num_cons = " + std::to_string(lx) + " and log2 (2 num_vars) = " + std::to_string(ly) + "; at most " +
                                          std::to_string(std::min(R1CS_MAX_LOG, zk_sumcheck_max_rounds())) + " supported");
}
// the view of `set` for num_vars, after the checks every gens entry shares
static void r1cs_gens_out(sp_ctx* ctx, std::shared_ptr<GenSet> set, size_t num_vars, sp_r1cs_gens** out, const std::string& what) {
  if (set->ctx != &ctx->c) throw SpError(SP_ERR_INVALID_ARG, what + ": the generators belong to another context");
  const size_t need = R1CSGens::bases(num_vars);
  if (set->nbases < need)
    throw SpError(SP_ERR_INVALID_ARG, what + ": num_vars = " + std::to_string(num_vars) + " needs " + std::to_string(need) + " generators of " + set->label +
                                          ", the set has " + std::to_string(set->nbases));
  std::unique_ptr<sp_r1cs_gens> g(new sp_r1cs_gens{&ctx->c, num_vars, nullptr});
  g->g.reset(new R1CSGens(std::move(set), num_vars));
  *out = g.release();
}
static void r1cs_gens_args(sp_r1cs_gens** out, size_t num_cons, size_t num_vars, const std::string& what) {
  if (!out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
  r1cs_dims(num_cons, num_vars, what);
}
int sp_r1cs_gens_create(sp_ctx* ctx, const uint8_t* label, size_t label_len, size_t num_cons, size_t num_vars, sp_r1cs_gens** out) {
  return guarded(ctx, [&] {
    const std::string what = "r1cs_gens_create";
    if (!label && label_len) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    r1cs_gens_args(out, num_cons, num_vars, what);
    r1cs_gens_out(ctx, std::make_shared<GenSet>(&ctx->c, std::string((const char*)label, label_len), R1CSGens::bases(num_vars), R1CSGens::host_bases(num_vars)),
                  num_vars, out, what);
  });
}
int sp_r1cs_gens_create_from(sp_ctx* ctx, const sp_gen_tables* tables, size_t num_cons, size_t num_vars, sp_r1cs_gens** out) {
  return guarded(ctx, [&] {
    const std::string what = "r1cs_gens_create_from";
    if (!tables) throw SpError(SP_ERR_INVALID_ARG, what + ": tables is NULL");
    r1cs_gens_args(out, num_cons, num_vars, what);
    r1cs_gens_out(ctx, tables->t->r1cs_sat, num_vars, out, what);
  });
}
int sp_r1cs_gens_create_from_nizk(sp_ctx* ctx, const sp_nizk_gens* gens, size_t num_cons, size_t num_vars, sp_r1cs_gens** out) {
  return guarded(ctx, [&] {
    const std::string what = "r1cs_gens_create_from_nizk";
    if (!gens) throw SpError(SP_ERR_INVALID_ARG, what + ": gens is NULL");
    r1cs_gens_args(out, num_cons, num_vars, what);
    r1cs_gens_out(ctx, gens->g->set, num_vars, out, what);
  });
}
int sp_r1cs_gens_create_from_snark(sp_ctx* ctx, const sp_snark_gens* gens, size_t num_cons, size_t num_vars, sp_r1cs_gens** out) {
  return guarded(ctx, [&] {
    const std::string what = "r1cs_gens_create_from_snark";
    if (!gens) throw SpError(SP_ERR_INVALID_ARG, what + ": gens is NULL");
    r1cs_gens_args(out, num_cons, num_vars, what);
    r1cs_gens_out(ctx, gens->g->gens_r1cs_sat->set, num_vars, out, what);
  });
}
void sp_r1cs_gens_free(sp_r1cs_gens* g) { delete g; }

// the dimensions, the gens and the inputs of a prove or verify call
static void r1cs_common(const sp_ctx* ctx, size_t num_cons, size_t num_vars, const uint64_t* inputs, size_t ninputs, const sp_r1cs_gens* gens,
                        const std::string& what) {
  r1cs_dims(num_cons, num_vars, what);
  if (!inputs && ninputs) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
  if (!(ninputs < num_vars))   // r1csproof.rs:156
    throw SpError(SP_ERR_INVALID_ARG, what + ": |inputs| + 1 = " + std::to_string(ninputs + 1) + " > num_vars = " + std::to_string(num_vars));
  require_owned(ctx, gens, what, "gens");
  if (gens->g->gens_pc.n != R1CSGens::pc_n(num_vars))
    throw SpError(SP_ERR_INVALID_ARG, what + ": gens for num_vars = " + std::to_string(gens->num_vars) + " do not fit num_vars = " + std::to_string(num_vars));
  require_reduced(inputs, ninputs, (what + ": inputs").c_str());
}
// the three matrices of an sp_spmat as R1CS matrices: the tiled products of sp_spmat_multiply_vec / sp_spmat_eval_table, never sharded
struct SpmatMatrices : R1csMatrices {
  const sp_spmat& S;
  SpmatMatrices(const sp_spmat& s, size_t nc, size_t nv) : R1csMatrices(nc, nv), S(s) {}
  void multiply_vec(Ctx& ctx, const u256* d_z, u256* const outs[3], size_t n, bool sh) const override {
    if (sh) throw SpError(SP_ERR_INTERNAL, "r1cs_prove: sp_spmat products do not shard");
    spmat_run(ctx, S, false, d_z, outs, n);
  }
  void eval_table(Ctx& ctx, const u256* d_e, const Fq w[3], u256*, u256* out, size_t n, bool sh) const override {
    if (sh) throw SpError(SP_ERR_INTERNAL, "r1cs_prove: sp_spmat products do not shard");
    const u256 wm[3] = {w[0].m, w[1].m, w[2].m};
    spmat_weighted(ctx, S, d_e, wm, out, n);
  }
};
int sp_r1cs_prove_t(sp_ctx* ctx, const sp_instance* inst, const sp_spmat* spmat, size_t num_cons, size_t num_vars, const sp_poly* vars, const uint64_t* inputs,
                    size_t ninputs, const sp_r1cs_gens* gens, uint8_t* strobe_state, uint8_t* tape_state, uint8_t** proof, size_t* proof_len, uint64_t* rx_out,
                    uint64_t* ry_out) {
  return guarded(ctx, [&] {
    const std::string what = "r1cs_prove";
    ProofStates st(strobe_state, tape_state, what);
    if (!proof || !proof_len || !rx_out || !ry_out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    if (!inst == !spmat) throw SpError(SP_ERR_INVALID_ARG, what + ": pass exactly one of inst and spmat");
    r1cs_common(ctx, num_cons, num_vars, inputs, ninputs, gens, what);
    std::optional<InstanceMatrices> im;
    std::optional<SpmatMatrices> sm;
    if (inst) {
      const Instance& I = inst->inst;
      require_device(ctx->c, I.M[0].csr_ptr.p, 1, (what + ": inst").c_str());   // the instance's matrices live on this context's device
      if (I.num_cons != num_cons || I.num_vars != num_vars)
        throw SpError(SP_ERR_INVALID_ARG, what + ": the instance is " + std::to_string(I.num_cons) + " x " + std::to_string(I.num_vars) + " (padded), not " +
                                              std::to_string(num_cons) + " x " + std::to_string(num_vars));
      im.emplace(I);
    } else {
      require_owned(ctx, spmat, what, "spmat");
      const size_t x = log2_ceil(num_cons), y = log2_ceil(2 * num_vars);
      if (spmat->b != 3 || spmat->x != x || spmat->y != y)
        throw SpError(SP_ERR_INVALID_ARG, what + ": spmat holds " + std::to_string(spmat->b) + " matrices of 2^" + std::to_string(spmat->x) + " x 2^" +
                                              std::to_string(spmat->y) + ", R1CS needs 3 of 2^" + std::to_string(x) + " x 2^" + std::to_string(y));
      sm.emplace(*spmat, num_cons, num_vars);
    }
    require_owned(ctx, vars, what, "vars");
    if (vars->len != num_vars)
      throw SpError(SP_ERR_INVALID_ARG, what + ": vars has " + std::to_string(vars->len) + " entries, num_vars = " + std::to_string(num_vars));
    st.open();
    ctx->c.timings.clear();
    R1CSProof P;
    std::vector<Fq> rx, ry;
    r1cs_prove(ctx->c, im ? static_cast<const R1csMatrices&>(*im) : *sm, vars->d.p, fq_vec(inputs, ninputs), *gens->g, st.T(), st.tape(), P, rx, ry);
    st.proved();
    put_bytes(proof, proof_len, to_bincode(P));
    put_scalars(rx_out, rx);
    put_scalars(ry_out, ry);
  });
}
int sp_r1cs_verify_t(sp_ctx* ctx, const uint8_t* proof, size_t proof_len, size_t num_cons, size_t num_vars, const uint64_t* inputs, size_t ninputs,
                     const uint64_t* evals, const sp_r1cs_gens* gens, uint8_t* strobe_state, uint64_t* rx_out, uint64_t* ry_out) {
  return guarded(ctx, [&] {
    const std::string what = "r1cs_verify";
    ProofStates st(strobe_state);
    if ((!proof && proof_len) || !evals || !rx_out || !ry_out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    r1cs_common(ctx, num_cons, num_vars, inputs, ninputs, gens, what);
    require_reduced(evals, 3, (what + ": evals").c_str());
    const std::vector<Fq> ev = fq_vec(evals, 3);
    st.open_verify();
    std::vector<Fq> rx, ry;
    r1cs_verify_bytes(ctx->c, proof, proof_len, num_vars, num_cons, fq_vec(inputs, ninputs), ev.data(), *gens->g, st.T(), rx, ry);
    put_scalars(rx_out, rx);
    put_scalars(ry_out, ry);
  });
}
// R1CSShape::evaluate (r1cs.rs:300-303) through the instance's COO on the device
int sp_instance_evaluate(sp_ctx* ctx, const sp_instance* inst, const uint64_t* rx, const uint64_t* ry, uint64_t* out) {
  return guarded(ctx, [&] {
    const std::string what = "instance_evaluate";
    if (!inst || !rx || !ry || !out) throw SpError(SP_ERR_INVALID_ARG, what + ": NULL argument");
    const Instance& I = inst->inst;
    const size_t x = log2_ceil(I.num_cons), y = log2_ceil(2 * I.num_vars);
    require_reduced(rx, x, (what + ": rx").c_str());
    require_reduced(ry, y, (what + ": ry").c_str());
    Fq ev[3];
    instance_evaluate(ctx->c, I, fq_vec(rx, x), fq_vec(ry, y), ev);
    for (int m = 0; m < 3; m++) fq_out(out + 4 * m, ev[m]);
  });
}

static int nizk_verify_batch_common(sp_ctx* ctx, const sp_instance* const* insts, const sp_nizk_gens* gens, const BatchArgs& a) {
  return verify_batch(ctx, reinterpret_cast<const void* const*>(insts), gens, a, [&](std::vector<VerifyJob>& jobs) {
    for (size_t i = 0; i < a.k; i++) jobs[i].inst = &insts[i]->inst;
    nizk_verify_batch(ctx->c, *gens->g, jobs, a.seed);
  });
}
static int snark_verify_batch_common(sp_ctx* ctx, const sp_snark_encoding* const* comms, const sp_snark_gens* gens, const BatchArgs& a) {
  return verify_batch(ctx, reinterpret_cast<const void* const*>(comms), gens, a, [&](std::vector<VerifyJob>& jobs) {
    for (size_t i = 0; i < a.k; i++) jobs[i].enc = comms[i]->e.get();
    snark_verify_batch(ctx->c, *gens->g, jobs, a.seed);
  });
}
int sp_nizk_verify_batch(sp_ctx* ctx, size_t k, const sp_instance* const* insts, const uint64_t* const* inputs_mont, const size_t* ninputs,
                         const sp_nizk_gens* gens, const uint8_t* const* labels, const size_t* label_lens, const uint8_t* const* proofs,
                         const size_t* proof_lens, const uint8_t weight_seed[32], int* status) {
  return nizk_verify_batch_common(ctx, insts, gens, {k, inputs_mont, ninputs, labels, label_lens, nullptr, proofs, proof_lens, weight_seed, status});
}
int sp_snark_verify_batch(sp_ctx* ctx, size_t k, const sp_snark_encoding* const* comms, const uint64_t* const* inputs_mont, const size_t* ninputs,
                          const sp_snark_gens* gens, const uint8_t* const* labels, const size_t* label_lens, const uint8_t* const* proofs,
                          const size_t* proof_lens, const uint8_t weight_seed[32], int* status) {
  return snark_verify_batch_common(ctx, comms, gens, {k, inputs_mont, ninputs, labels, label_lens, nullptr, proofs, proof_lens, weight_seed, status});
}
int sp_nizk_verify_batch_t(sp_ctx* ctx, size_t k, const sp_instance* const* insts, const uint64_t* const* inputs_mont, const size_t* ninputs,
                           const sp_nizk_gens* gens, uint8_t* const* strobe_states, const uint8_t* const* proofs, const size_t* proof_lens,
                           const uint8_t weight_seed[32], int* status) {
  return nizk_verify_batch_common(ctx, insts, gens, {k, inputs_mont, ninputs, nullptr, nullptr, strobe_states, proofs, proof_lens, weight_seed, status});
}
int sp_snark_verify_batch_t(sp_ctx* ctx, size_t k, const sp_snark_encoding* const* comms, const uint64_t* const* inputs_mont, const size_t* ninputs,
                            const sp_snark_gens* gens, uint8_t* const* strobe_states, const uint8_t* const* proofs, const size_t* proof_lens,
                            const uint8_t weight_seed[32], int* status) {
  return snark_verify_batch_common(ctx, comms, gens, {k, inputs_mont, ninputs, nullptr, nullptr, strobe_states, proofs, proof_lens, weight_seed, status});
}

// merlin::Transcript for hosts without merlin (tests, C callers): the state buffer is the whole object
int sp_transcript_new(const uint8_t* label, size_t label_len, uint8_t* strobe_state) {
  return host_guarded(nullptr, [&] { Transcript(std::string((const char*)label, label_len)).export_state(strobe_state); });
}
int sp_transcript_append_message(uint8_t* strobe_state, const uint8_t* label, size_t label_len, const uint8_t* msg, size_t msg_len) {
  return host_guarded(nullptr, [&] {
    Transcript T(Transcript::FromState(), strobe_state);
    T.append_message(std::string((const char*)label, label_len).c_str(), msg, msg_len);
    T.export_state(strobe_state);
  });
}
int sp_transcript_challenge_bytes(uint8_t* strobe_state, const uint8_t* label, size_t label_len, uint8_t* out, size_t n) {
  return host_guarded(nullptr, [&] {
    Transcript T(Transcript::FromState(), strobe_state);
    T.challenge_bytes(std::string((const char*)label, label_len).c_str(), out, n);
    T.export_state(strobe_state);
  });
}

void sp_free(void* p) { free(p); }

}  // extern "C"
