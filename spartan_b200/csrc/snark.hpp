// spartan_b200 — SNARK path: SPARK sparse-polynomial commitment (src/sparse_mlpoly.rs, src/product_tree.rs) driven on the device.
#pragma once
#include "prover.hpp"
#include <chrono>

namespace sp {

// R1CSCommitmentGens::new (r1cs.rs:34-47) -> SparseMatPolyCommitmentGens::new(label, x, y, nz, 3) (sparse_mlpoly.rs:292-317): the variable counts of
// the ops, mem and derefs polynomials and their PolyCommitmentGens sizes
struct SparkDims {
  size_t v_ops, v_mem, v_derefs, n_ops, n_mem, n_der;
  SparkDims(size_t num_cons, size_t num_vars_padded, size_t num_nz_entries);
  size_t bases() const { return std::max(n_ops, std::max(n_mem, n_der)) + 2; }   // generators of gens_r1cs_eval the three views use
  std::vector<size_t> host_bases() const { return {n_ops, n_ops + 1, n_mem, n_mem + 1, n_der, n_der + 1}; }
};

struct SnarkGens {  // lib.rs:277-309
  std::unique_ptr<R1CSGens> gens_r1cs_sat;
  std::shared_ptr<GenSet> eval_set;  // label "gens_r1cs_eval": ops / mem / derefs generators share one SHAKE stream (sparse_mlpoly.rs:292-317)
  PolyCommitmentGens gens_ops, gens_mem, gens_derefs;
  // a view into both sets of `tables`; SpError(SP_ERR_INVALID_ARG) when either is too short or missing, or the tables are of another context
  SnarkGens(const Ctx* ctx, const GenTables& tables, size_t num_cons, size_t num_vars, size_t num_inputs, size_t num_nz_entries);
};

struct AddrTimestampsDev {  // sparse_mlpoly.rs:213-272
  std::vector<DevBuf<uint32_t>> ops_addr_idx;  // per instance, N entries
  std::vector<DevBuf<u256>> ops_addr, read_ts; // as field elements
  DevBuf<u256> audit_ts;
};
struct SnarkEncoding {  // ComputationCommitment + ComputationDecommitment (lib.rs:44-55; sparse_mlpoly.rs:274-327)
  ComputationCommitment comm;     // alone in an encoding loaded from commitment bytes, which can verify but not prove
  std::vector<DevBuf<u256>> val;  // dense.val
  AddrTimestampsDev row, col;
  DevBuf<u256> comb_ops, comb_mem;
};

void snark_encode(Ctx& ctx, const Instance& inst, const SnarkGens& gens, SnarkEncoding& out);
void snark_prove(Ctx& ctx, const Instance& inst, const SnarkEncoding& enc, const u256* d_vars, const std::vector<Fq>& input, const SnarkGens& gens,
                 Transcript& T, const Fq& tape_seed, SnarkProof& out);

// ---- protocol steps SNARK::prove and SNARK::verify share
void append_computation_commitment(Transcript& T, const ComputationCommitment& c);   // r1cs.rs:58-65, sparse_mlpoly.rs:329-341
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

// ---- verifiers (verifier.cpp): throw SpError with code SP_ERR_VERIFY / SP_ERR_DECOMPRESS when the proof is rejected
void nizk_verify(Ctx& ctx, const Instance& inst, const std::vector<Fq>& input, const R1CSGens& gens, Transcript& T, const uint8_t* proof, size_t len);
void snark_verify(Ctx& ctx, const SnarkEncoding& enc, const std::vector<Fq>& input, const SnarkGens& gens, Transcript& T, const uint8_t* proof, size_t len);
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
