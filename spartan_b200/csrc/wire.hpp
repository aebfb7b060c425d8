// spartan_b200 — the proof wire format: bincode 1.x (default config) of the reference's proof structs.
// Struct and field names follow the reference's src/ so the layout (SURVEY.md Appendix B) can be checked line by line.  Each struct states its
// field order once, in io(): Writer and Reader both walk that list, so the encoder and the decoder cannot disagree.
// Host-only: no device memory, so the CPU tests can include it.
#pragma once
#include <array>
#include <string>
#include <type_traits>
#include <vector>
#include "../../include/spartan_b200.h"
#include "engine.hpp"

namespace sp {

// A vector's element type gives the fewest bytes one element can take on the wire, so that Reader can refuse a length prefix before
// allocating: 32 for points and scalars, MIN_BYTES of a struct
template <class T> constexpr size_t wire_min_bytes() {
  if constexpr (std::is_same_v<T, Fq> || std::is_same_v<T, Cp>) return 32;
  else return T::MIN_BYTES;
}

struct Writer {
  std::vector<uint8_t> out;
  void u64(uint64_t x) { for (int i = 0; i < 8; i++) out.push_back((uint8_t)(x >> (8 * i))); }
  void scalar(const Fq& s) { uint8_t b[32]; u256_to_bytes(b, s.m); out.insert(out.end(), b, b + 32); }  // Montgomery limbs, not canonical bytes
  void point(const Cp& c) { out.insert(out.end(), c.b, c.b + 32); }
  template <class... T> void operator()(const T&... v) { (put(v), ...); }
  // io() takes its fields by non-const reference so that Reader can fill them; a Writer only reads them
  template <class T> void put(const T& v) { const_cast<T&>(v).io(*this); }
  void put(const uint64_t& x) { u64(x); }
  void put(const Fq& s) { scalar(s); }
  void put(const Cp& c) { point(c); }
  template <class T, size_t N> void put(const std::array<T, N>& a) { for (auto& x : a) put(x); }
  template <class T> void put(const std::vector<T>& v) { u64(v.size()); for (auto& x : v) put(x); }
};

// The inverse of Writer.  Every malformed input throws SpError(code): a truncation, a vector length longer than the rest of the input could
// hold, a scalar whose limbs are not reduced modulo q, and bytes left over after the value.
struct Reader {
  const uint8_t* p;
  size_t n, pos = 0;
  int code;
  const char* what;   // names the input in error messages
  Reader(const uint8_t* b, size_t len, int code_, const char* what_) : p(b), n(len), code(code_), what(what_) {}
  [[noreturn]] void fail(const char* why) { throw SpError(code, std::string(what) + " rejected: " + why); }
  void need(size_t k) { if (n - pos < k) fail("truncated"); }
  uint64_t u64() { need(8); uint64_t x = 0; for (int i = 0; i < 8; i++) x |= (uint64_t)p[pos + i] << (8 * i); pos += 8; return x; }
  // a Scalar on the wire is its four Montgomery limbs (serde derive on `Scalar([u64;4])`): the reference accepts any limbs, but every host
  // routine here assumes a reduced residue, so limbs >= q are rejected instead of being carried into fq_mul / fq_eq (no malleability either)
  Fq scalar() { need(32); if (!fq_bytes_canonical(p + pos)) fail("scalar limbs are not reduced modulo q"); Fq f; memcpy(&f.m, p + pos, 32); pos += 32; return f; }
  Cp point() { need(32); Cp c; memcpy(c.b, p + pos, 32); pos += 32; return c; }
  template <class... T> void operator()(T&... v) { (get(v), ...); }
  template <class T> void get(T& v) { v.io(*this); }
  void get(uint64_t& x) { x = u64(); }
  void get(Fq& s) { s = scalar(); }
  void get(Cp& c) { c = point(); }
  template <class T, size_t N> void get(std::array<T, N>& a) { for (auto& x : a) get(x); }
  template <class T> void get(std::vector<T>& v) {
    const uint64_t k = u64();
    if (k > (n - pos) / wire_min_bytes<T>()) fail("vector length exceeds the input");
    v.resize(k);
    for (auto& x : v) get(x);
  }
};
static_assert(std::is_same_v<size_t, uint64_t>, "bincode lengths and the commitment's sizes are u64 on the wire");

template <class T> std::vector<uint8_t> to_bincode(const T& v) { Writer w; w(v); return std::move(w.out); }
// the whole input must be one T
template <class T> T from_bincode(const uint8_t* b, size_t len, int code, const char* what) {
  Reader r(b, len, code, what);
  T v;
  r(v);
  if (r.pos != len) r.fail("trailing bytes");
  return v;
}

// ---- nizk/mod.rs
struct KnowledgeProof { Cp alpha; Fq z1, z2; template <class A> void io(A& a) { a(alpha, z1, z2); } };
struct EqualityProof { Cp alpha; Fq z; template <class A> void io(A& a) { a(alpha, z); } };
struct ProductProof { Cp alpha, beta, delta; std::array<Fq, 5> z; template <class A> void io(A& a) { a(alpha, beta, delta, z); } };
struct DotProductProof {
  static constexpr size_t MIN_BYTES = 160;
  Cp delta, beta; std::vector<Fq> z; Fq z_delta, z_beta;
  template <class A> void io(A& a) { a(delta, beta, z, z_delta, z_beta); }
};
struct BulletReductionProof { std::vector<Cp> L_vec, R_vec; template <class A> void io(A& a) { a(L_vec, R_vec); } };
struct DotProductProofLog {
  BulletReductionProof bullet_reduction_proof; Cp delta, beta; Fq z1, z2;
  template <class A> void io(A& a) { a(bullet_reduction_proof, delta, beta, z1, z2); }
};
// ---- dense_mlpoly.rs
struct PolyCommitment { std::vector<Cp> C; template <class A> void io(A& a) { a(C); } };
struct PolyEvalProof { DotProductProofLog proof; template <class A> void io(A& a) { a(proof); } };
// ---- sumcheck.rs
struct ZKSumcheckInstanceProof {
  std::vector<Cp> comm_polys, comm_evals; std::vector<DotProductProof> proofs;
  template <class A> void io(A& a) { a(comm_polys, comm_evals, proofs); }
};
struct CompressedUniPoly {
  static constexpr size_t MIN_BYTES = 8;
  std::vector<Fq> coeffs_except_linear_term;
  template <class A> void io(A& a) { a(coeffs_except_linear_term); }
};
struct SumcheckInstanceProof { std::vector<CompressedUniPoly> compressed_polys; template <class A> void io(A& a) { a(compressed_polys); } };
// ---- r1csproof.rs:21-37
struct R1CSProof {
  PolyCommitment comm_vars;
  ZKSumcheckInstanceProof sc_proof_phase1;
  std::array<Cp, 4> claims_phase2;
  KnowledgeProof pok_Cz; ProductProof proof_prod;  // pok_claims_phase2
  EqualityProof proof_eq_sc_phase1;
  ZKSumcheckInstanceProof sc_proof_phase2;
  Cp comm_vars_at_ry;
  PolyEvalProof proof_eval_vars_at_ry;
  EqualityProof proof_eq_sc_phase2;
  template <class A> void io(A& a) {
    a(comm_vars, sc_proof_phase1, claims_phase2, pok_Cz, proof_prod, proof_eq_sc_phase1, sc_proof_phase2, comm_vars_at_ry, proof_eval_vars_at_ry,
      proof_eq_sc_phase2);
  }
};
// ---- product_tree.rs / sparse_mlpoly.rs
struct LayerProofBatched {
  static constexpr size_t MIN_BYTES = 8;
  SumcheckInstanceProof proof; std::vector<Fq> claims_prod_left, claims_prod_right;
  template <class A> void io(A& a) { a(proof, claims_prod_left, claims_prod_right); }
};
struct ProductCircuitEvalProofBatched {
  std::vector<LayerProofBatched> proof; std::vector<Fq> dotp_left, dotp_right, dotp_weight;
  template <class A> void io(A& a) { a(proof, dotp_left, dotp_right, dotp_weight); }
};
struct ProductLayerProof {
  Fq row_init; std::vector<Fq> row_read, row_write; Fq row_audit;
  Fq col_init; std::vector<Fq> col_read, col_write; Fq col_audit;
  std::vector<Fq> eval_dotp_left, eval_dotp_right;
  ProductCircuitEvalProofBatched proof_mem, proof_ops;
  template <class A> void io(A& a) {
    a(row_init, row_read, row_write, row_audit, col_init, col_read, col_write, col_audit, eval_dotp_left, eval_dotp_right, proof_mem, proof_ops);
  }
};
struct HashLayerProof {
  std::vector<Fq> row_addr, row_read_ts; Fq row_audit_ts;
  std::vector<Fq> col_addr, col_read_ts; Fq col_audit_ts;
  std::vector<Fq> eval_val, derefs_row, derefs_col;
  PolyEvalProof proof_ops, proof_mem, proof_derefs;
  template <class A> void io(A& a) {
    a(row_addr, row_read_ts, row_audit_ts, col_addr, col_read_ts, col_audit_ts, eval_val, derefs_row, derefs_col, proof_ops, proof_mem, proof_derefs);
  }
};
struct SparseMatPolyEvalProof {  // = R1CSEvalProof.proof
  PolyCommitment comm_derefs;    // DerefsCommitment.comm_ops_val
  ProductLayerProof proof_prod_layer;
  HashLayerProof proof_hash_layer;
  template <class A> void io(A& a) { a(comm_derefs, proof_prod_layer, proof_hash_layer); }
};

// ---- lib.rs
struct NizkProof { R1CSProof r1cs_sat_proof; std::vector<Fq> rx, ry; template <class A> void io(A& a) { a(r1cs_sat_proof, rx, ry); } };
struct SnarkProof {  // lib.rs:313-317
  R1CSProof r1cs_sat_proof;
  std::array<Fq, 3> inst_evals;
  SparseMatPolyEvalProof r1cs_eval_proof;
  template <class A> void io(A& a) { a(r1cs_sat_proof, inst_evals, r1cs_eval_proof); }
};
// SparseMatPolyCommitment (sparse_mlpoly.rs:319-327)
struct SparseMatPolyCommitment {
  size_t batch_size = 0, num_ops = 0, num_mem_cells = 0;
  PolyCommitment comm_comb_ops, comm_comb_mem;
  template <class A> void io(A& a) { a(batch_size, num_ops, num_mem_cells, comm_comb_ops, comm_comb_mem); }
};
// ComputationCommitment { R1CSCommitment { .., SparseMatPolyCommitment } } (r1cs.rs:49-55): bincode has no framing, so the nesting adds no bytes
struct ComputationCommitment {
  size_t num_cons = 0, num_vars = 0, num_inputs = 0;
  SparseMatPolyCommitment comm;
  template <class A> void io(A& a) { a(num_cons, num_vars, num_inputs, comm); }
};

}  // namespace sp
