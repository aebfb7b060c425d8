// spartan_b200 — SPARK, the sparse-polynomial commitment and evaluation proof (src/sparse_mlpoly.rs, src/product_tree.rs) driven on the device,
// for the caller's matrices and for the SNARK, its caller with the three R1CS matrices.
#pragma once
#include "prover.hpp"
#include <chrono>

namespace sp {

// SparseMatPolyCommitmentGens::new(label, num_vars_x, num_vars_y, num_nz_entries, batch_size) (sparse_mlpoly.rs:292-317): the variable counts of
// the ops, mem and derefs polynomials and their PolyCommitmentGens sizes.  The SNARK's is (log2 num_cons, log2 2*num_vars_padded, nz, 3)
// (R1CSCommitmentGens::new, r1cs.rs:34-47).
struct SparkGens;
struct SparkDims {
  size_t v_ops, v_mem, v_derefs, n_ops, n_mem, n_der;
  SparkDims(size_t x, size_t y, size_t num_nz_entries, size_t b) {
    const size_t lgnz = log2_ceil(next_pow2(num_nz_entries));
    v_ops = lgnz + log2_ceil(next_pow2(b * 5)); v_mem = std::max(x, y) + 1; v_derefs = lgnz + log2_ceil(next_pow2(b * 2));
    n_ops = (size_t)1 << (v_ops - v_ops / 2); n_mem = (size_t)1 << (v_mem - v_mem / 2); n_der = (size_t)1 << (v_derefs - v_derefs / 2);
  }
  size_t bases() const { return std::max(n_ops, std::max(n_mem, n_der)) + 2; }   // generators of the label's set the three views use
  std::vector<size_t> host_bases() const { return {n_ops, n_ops + 1, n_mem, n_mem + 1, n_der, n_der + 1}; }
  bool fits(const SparkGens& g) const;   // the three views of g have these n
};
static_assert(6 * SP_SPARK_MAX_BATCH <= dev::SC_MAX_INST, "the ops product proof batches 4b product and 2b dot-product circuits in one launch per round");

// ops / mem / derefs generators: views of one set, prefixes of the label's one SHAKE stream
struct SparkGens {
  std::shared_ptr<GenSet> set;
  PolyCommitmentGens gens_ops, gens_mem, gens_derefs;
  SparkGens() = default;
  SparkGens(std::shared_ptr<GenSet> set, const SparkDims& d);   // adds the host tables the views need
};
inline bool SparkDims::fits(const SparkGens& g) const { return g.gens_ops.n == n_ops && g.gens_mem.n == n_mem && g.gens_derefs.n == n_der; }

struct SnarkGens {  // lib.rs:277-309
  std::unique_ptr<R1CSGens> gens_r1cs_sat;
  SparkGens gens_r1cs_eval;   // label "gens_r1cs_eval", batch size 3
  // a view into both sets of `tables`; SpError(SP_ERR_INVALID_ARG) when either is too short or missing, or the tables are of another context
  SnarkGens(const Ctx* ctx, const GenTables& tables, size_t num_cons, size_t num_vars, size_t num_inputs, size_t num_nz_entries);
};

// b <= SP_SPARK_MAX_BATCH sparse matrices of 2^x rows and 2^y columns as device COO (entries with value 0 allowed)
struct SparkMatrix { const uint32_t* row; const uint32_t* col; const u256* val; size_t nnz; };
// MultiSparseMatPolynomialAsDense (sparse_mlpoly.rs:274-282, :366-420) on the device.  N = max_i next_pow2(nnz_i), cells = 2^max(x, y).
//   comb_ops = row.ops_addr[b] | row.read_ts[b] | col.ops_addr[b] | col.read_ts[b] | val[b] | zero pad to next_pow2(5b) N   (DensePolynomial::merge)
//   comb_mem = row.audit_ts | col.audit_ts
// Matrix i's entries are zero-padded to N: address 0, value 0.
struct SparkDense {
  size_t x = 0, y = 0, b = 0, N = 0, cells = 0;
  DevBuf<u256> comb_ops, comb_mem;
  std::vector<DevBuf<uint32_t>> row_idx, col_idx;   // ops_addr of each matrix as indices, N entries each
  const u256* row_addr(size_t m) const { return comb_ops.p + m * N; }
  const u256* row_ts(size_t m) const { return comb_ops.p + (b + m) * N; }
  const u256* col_addr(size_t m) const { return comb_ops.p + (2 * b + m) * N; }
  const u256* col_ts(size_t m) const { return comb_ops.p + (3 * b + m) * N; }
  const u256* val(size_t m) const { return comb_ops.p + (4 * b + m) * N; }
  const u256* row_audit() const { return comb_mem.p; }
  const u256* col_audit() const { return comb_mem.p + cells; }
};
struct SnarkEncoding {  // ComputationCommitment + ComputationDecommitment (lib.rs:44-55; sparse_mlpoly.rs:274-327)
  ComputationCommitment comm;   // alone in an encoding loaded from commitment bytes, which can verify but not prove
  SparkDense dense;
};

// SparseMatPolynomial::multi_commit (sparse_mlpoly.rs:483-503).  SpError(SP_ERR_INVALID_ARG) for N < 2 (the product circuits would have no layer)
// or gens of other sizes; SP_ERR_INVALID_INDEX for an address >= 2^max(x, y).  Argument ranges (b, x, y) are the caller's to check.
void spark_commit(Ctx& ctx, const SparkMatrix* mats, size_t b, size_t x, size_t y, const SparkGens& gens, SparkDense& dense, SparseMatPolyCommitment& comm);
// SparseMatPolynomial::multi_evaluate (sparse_mlpoly.rs:440-452) of b matrices: out[i] = M_i(rx, ry)
void sparse_evaluate(Ctx& ctx, const SparkMatrix* mats, size_t b, const std::vector<Fq>& rx, const std::vector<Fq>& ry, Fq* out);
void spark_evaluate(Ctx& ctx, const SparkDense& dense, const std::vector<Fq>& rx, const std::vector<Fq>& ry, Fq* out);
// The dereferenced values and their commitment, made by the caller ahead of the proof (SNARK::prove: on the background stream, during the R1CS proof)
struct SparkDerefs { const u256* derefs; const u256* mem_rx; const u256* mem_ry; PolyCommitment comm_derefs; };
// SparseMatPolyEvalProof::prove (sparse_mlpoly.rs:1447-1514) for b = dense.b matrices.  At b = 3 this is the reference's proof; for other b the
// generalisation its ProductLayerProof::prove leaves as a TODO (:1121-1122): ops circuits row.read[b], row.write[b], col.read[b], col.write[b] and
// dot-product circuits left_0, right_0, left_1, right_1, ..., the order its verifier assumes (:1264-1270).  Absorbs neither the commitment nor
// the evaluations.  pre null: the dereferenced values are computed and committed here.
void spark_eval_prove(Ctx& ctx, const SparkDense& dense, const std::vector<Fq>& rx, const std::vector<Fq>& ry, const std::vector<Fq>& evals,
                      const SparkGens& gens, Transcript& T, RandomTape& tape, SparseMatPolyEvalProof& out, const SparkDerefs* pre = nullptr);

void snark_encode(Ctx& ctx, const Instance& inst, const SnarkGens& gens, SnarkEncoding& out);
void snark_prove(Ctx& ctx, const Instance& inst, const SnarkEncoding& enc, const u256* d_vars, const std::vector<Fq>& input, const SnarkGens& gens,
                 Transcript& T, const Fq& tape_seed, SnarkProof& out);

// ---- protocol steps SNARK::prove and SNARK::verify share
void append_computation_commitment(Transcript& T, const ComputationCommitment& c);   // r1cs.rs:58-65
void append_sparse_commitment(Transcript& T, const SparseMatPolyCommitment& c);      // sparse_mlpoly.rs:329-341
void append_derefs_commitment(Transcript& T, const PolyCommitment& c);              // sparse_mlpoly.rs:204-210
// ProductLayerProof's memory-check claims, row side then column side (sparse_mlpoly.rs:1060-1088, :1246-1277): a side is absorbed only when
// init * prod(writes) == prod(reads) * audit; returns false, with that side not absorbed, at the first side where it does not hold
bool append_memory_claims(Transcript& T, const ProductLayerProof& pl);
// left-pad the shorter of rx, ry with zeros (sparse_mlpoly.rs:1429-1445)
void equalize(std::vector<Fq>& rx, std::vector<Fq>& ry);
// HashLayerProof opens three committed polynomials at one point each (sparse_mlpoly.rs:80-123, :766-824).  The claims it makes about one of
// them, padded with zeros to a power of two, are absorbed, combined into one joint claim by the challenges drawn next, and the joint claim is
// absorbed.  Sets `joint`; returns the point it is claimed at: the challenges followed by `rand` (rand_ops for derefs and ops, rand_mem for mem).
enum class HashOpening { derefs, ops, mem };
std::vector<Fq> combine_to_one(Transcript& T, const HashLayerProof& hl, HashOpening which, const std::vector<Fq>& rand, Fq& joint);
// inst.evaluate(rx, ry) (r1cs.rs:300-303 -> sparse_mlpoly.rs:440-452) on the device
void instance_evaluate(Ctx& ctx, const Instance& inst, const std::vector<Fq>& rx, const std::vector<Fq>& ry, Fq out[3]);
// the checks SparseMatPolyEvalProof::verify's asserts stand for, on a caller's commitment: batch_size = |evals| in 1 .. SP_SPARK_MAX_BATCH,
// num_ops a power of two >= 2, num_mem_cells = 2^max(x, y), and gens whose views fit (x, y, num_ops, batch_size).  SpError(SP_ERR_VERIFY) otherwise.
void check_spark_commitment(const SparseMatPolyCommitment& c, size_t nevals, size_t x, size_t y, const SparkGens& gens);

// ---- verifiers (verifier.cpp): throw SpError with code SP_ERR_VERIFY / SP_ERR_DECOMPRESS when the proof is rejected
void nizk_verify(Ctx& ctx, const Instance& inst, const std::vector<Fq>& input, const R1CSGens& gens, Transcript& T, const uint8_t* proof, size_t len);
void snark_verify(Ctx& ctx, const SnarkEncoding& enc, const std::vector<Fq>& input, const SnarkGens& gens, Transcript& T, const uint8_t* proof, size_t len);
// SparseMatPolyEvalProof::verify (sparse_mlpoly.rs:1516-1557) of a caller's proof, after check_spark_commitment
void spark_eval_verify(Ctx& ctx, const SparseMatPolyCommitment& comm, const std::vector<Fq>& rx, const std::vector<Fq>& ry, const std::vector<Fq>& evals,
                       const SparkGens& gens, Transcript& T, const uint8_t* proof, size_t len);
// Batch verification with deferred group checks (DESIGN.md "deferred checks").  Every job ends as the single verify leaves it: `status`
// SP_OK / SP_ERR_VERIFY / SP_ERR_DECOMPRESS, `msg` its message, `T` its transcript.  Throws (no job written) on bad arguments or device errors.
// `seed`: 32 bytes of fresh OS randomness (batch_weight).
struct VerifyJob {
  const Instance* inst = nullptr;        // NIZK
  const SnarkEncoding* enc = nullptr;    // SNARK
  std::vector<Fq> input;
  Transcript T;
  const uint8_t* proof = nullptr;
  size_t len = 0;
  int status = SP_OK;
  std::string msg;
};
void nizk_verify_batch(Ctx& ctx, const R1CSGens& gens, std::vector<VerifyJob>& jobs, const uint8_t seed[32]);
void snark_verify_batch(Ctx& ctx, const SnarkGens& gens, std::vector<VerifyJob>& jobs, const uint8_t seed[32]);
// the deferred checker on hand-made equations, for the tests: a term is k * (generator `gen` of `gs` if gen >= 0, else the point `pt`)
struct DeferredTerm { Fq k; long gen = -1; Cp pt; };
struct DeferredEq { std::vector<DeferredTerm> lhs, rhs; };
std::vector<bool> deferred_check(Ctx& ctx, const GenSet& gs, const std::vector<std::vector<DeferredEq>>& proofs, const uint8_t seed[32]);

}  // namespace sp
