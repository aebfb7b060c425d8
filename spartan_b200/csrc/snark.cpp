// spartan_b200 — SPARK (src/sparse_mlpoly.rs, src/product_tree.rs) driven on the device: the commitment to b sparse matrices and the proof of
// their evaluations, for the caller's matrices and for SNARK::encode / SNARK::prove (src/lib.rs:325-420), its caller with the three R1CS
// matrices.  Every table of the memory-checking network (hash layers, 4b + 4 product trees with all their layers, dereferenced values) lives in
// HBM; the host only runs the transcript.
#include "snark.hpp"
#include <cstdlib>
#include <algorithm>
#include <optional>
#include "../../include/spartan_b200.h"

namespace sp {

static PolyCommitmentGens pc_view(const GenSet* set, size_t num_vars) {  // PolyCommitmentGens::new (dense_mlpoly.rs:31-35)
  PolyCommitmentGens g;
  g.n = (size_t)1 << (num_vars - num_vars / 2);
  g.gens_n = CommitKey{set, 0, g.n, g.n + 1};
  g.gens_1 = CommitKey{set, g.n, 1, g.n + 1};
  return g;
}

SparkGens::SparkGens(std::shared_ptr<GenSet> s, const SparkDims& d) : set(std::move(s)) {
  set->add_host_tables(d.host_bases());
  gens_ops = pc_view(set.get(), d.v_ops);
  gens_mem = pc_view(set.get(), d.v_mem);
  gens_derefs = pc_view(set.get(), d.v_derefs);
}
static SparkDims snark_dims(size_t num_cons, size_t nvp, size_t num_nz_entries) { return SparkDims(log2_ceil(num_cons), log2_ceil(2 * nvp), num_nz_entries, 3); }

GenTables::GenTables(Ctx* c, size_t num_cons, size_t num_vars, size_t num_inputs, size_t num_nz_entries) : ctx(c) {
  const size_t nvp = padded_num_vars(num_vars, num_inputs);
  r1cs_sat = std::make_shared<GenSet>(ctx, "gens_r1cs_sat", R1CSGens::bases(nvp), R1CSGens::host_bases(nvp));
  if (num_nz_entries) {
    const SparkDims d = snark_dims(num_cons, nvp, num_nz_entries);
    r1cs_eval = std::make_shared<GenSet>(ctx, "gens_r1cs_eval", d.bases(), d.host_bases());
  }
}
void GenTables::require(const Ctx* c, size_t r1cs_bases, size_t eval_bases) const {
  if (c != ctx) throw SpError(SP_ERR_INVALID_ARG, "generator tables belong to another context: a view must be made on the context (device) that built them");
  if (eval_bases && !r1cs_eval)
    throw SpError(SP_ERR_INVALID_ARG, "generator tables were built without SNARK sizes (num_nz_entries = 0): a SNARKGens view needs their gens_r1cs_eval set");
  if (r1cs_bases <= r1cs_sat->nbases && (!eval_bases || eval_bases <= r1cs_eval->nbases)) return;
  std::string m = "generator tables too small for this circuit: gens_r1cs_sat needs " + std::to_string(r1cs_bases) + " generators, has " + std::to_string(r1cs_sat->nbases);
  if (eval_bases) m += "; gens_r1cs_eval needs " + std::to_string(eval_bases) + ", has " + std::to_string(r1cs_eval->nbases);
  throw SpError(SP_ERR_INVALID_ARG, m);
}

SnarkGens::SnarkGens(const Ctx* ctx, const GenTables& tables, size_t num_cons, size_t num_vars, size_t num_inputs, size_t num_nz_entries) {
  const size_t nvp = padded_num_vars(num_vars, num_inputs);  // lib.rs:288-294
  const SparkDims d = snark_dims(num_cons, nvp, num_nz_entries);
  tables.require(ctx, R1CSGens::bases(nvp), d.bases());     // both sets before either view: the message names both
  gens_r1cs_sat.reset(new R1CSGens(ctx, tables, nvp));
  gens_r1cs_eval = SparkGens(tables.r1cs_eval, d);
}

static void commit_poly(Ctx& ctx, const u256* d_Z, size_t len, const PolyCommitmentGens& gens, PolyCommitment& out) {  // DensePolynomial::commit, no blinds
  size_t ell = log2_ceil(len);
  size_t L = (size_t)1 << (ell / 2), R = (size_t)1 << (ell - ell / 2);
  if (R != gens.n) throw SpError(SP_ERR_INVALID_ARG, "polynomial size does not match the commitment generators (num_nz_entries too small?)");
  commit_rows_and_compress(ctx, gens.gens_n, d_Z, R, L, R, nullptr, out.C);
}


// ================================================================================================ multi_commit
void spark_commit(Ctx& ctx, const SparkMatrix* mats, size_t b, size_t x, size_t y, const SparkGens& gens, SparkDense& d, SparseMatPolyCommitment& c) {
  // SparseMatPolynomial::multi_commit -> multi_sparse_to_dense_rep (sparse_mlpoly.rs:366-420, :483-503)
  size_t N = 1;
  for (size_t m = 0; m < b; m++) N = std::max(N, next_pow2(mats[m].nnz));
  // every product circuit of the memory check has log2(N) layers and the proof binds its last one: with at most one entry per matrix there is
  // none (the reference panics in ProductCircuit::evaluate)
  if (N < 2) throw SpError(SP_ERR_INVALID_ARG, "SPARK needs a matrix with at least two entries (num_ops = 1 leaves the product circuits without layers)");
  const size_t cells = (size_t)1 << std::max(x, y), ops = next_pow2(5 * b) * N;
  d.x = x; d.y = y; d.b = b; d.N = N; d.cells = cells;
  c.batch_size = b; c.num_ops = N; c.num_mem_cells = cells;
  d.comb_ops.alloc(ops);
  d.comb_mem.alloc(2 * cells);
  dev::dzero(d.comb_ops.p, ops * sizeof(u256), ctx.stream);
  DevBuf<uint8_t> scratch(dev::spark_ts_scratch_bytes(b, N, cells));
  DevBuf<unsigned int> bad(1);
  dev::dzero(bad.p, sizeof(unsigned int), ctx.stream);
  for (int side = 0; side < 2; side++) {  // AddrTimestamps::new (sparse_mlpoly.rs:220-254), row then col
    std::vector<DevBuf<uint32_t>>& idx = side == 0 ? d.row_idx : d.col_idx;
    idx.resize(b);
    dev::SparkAddrs sa;
    sa.b = (int)b;
    for (size_t m = 0; m < b; m++) {
      idx[m].alloc(N);
      sa.src[m] = side == 0 ? mats[m].row : mats[m].col;
      sa.nnz[m] = mats[m].nnz;
      sa.idx[m] = idx[m].p;
    }
    // ops_addr[b] | read_ts[b] of this side are contiguous in comb_ops: position m*N + i of the loop's order is element m*N + i of each block
    dev::spark_timestamps(sa, d.comb_ops.p + side * 2 * b * N, d.comb_ops.p + (side * 2 + 1) * b * N, d.comb_mem.p + side * cells, N, cells, scratch.p,
                          bad.p, ctx.stream);
  }
  for (size_t m = 0; m < b; m++) dev::d2d(d.comb_ops.p + (4 * b + m) * N, mats[m].val, mats[m].nnz * sizeof(u256), ctx.stream);
  unsigned int out_of_range = 0;
  dev::d2h(&out_of_range, bad.p, sizeof(unsigned int), ctx.stream);
  ctx.sync();
  if (out_of_range) throw SpError(SP_ERR_INVALID_INDEX, "address out of range");
  commit_poly(ctx, d.comb_ops.p, ops, gens.gens_ops, c.comm_comb_ops);
  commit_poly(ctx, d.comb_mem.p, 2 * cells, gens.gens_mem, c.comm_comb_mem);
}

// ================================================================================================ SNARK::encode
void snark_encode(Ctx& ctx, const Instance& inst, const SnarkGens& gens, SnarkEncoding& e) {
  ComputationCommitment& c = e.comm;
  c.num_cons = inst.num_cons; c.num_vars = inst.num_vars; c.num_inputs = inst.num_inputs;
  SparkMatrix mats[3];
  for (int m = 0; m < 3; m++) mats[m] = SparkMatrix{inst.M[m].coo_row.p, inst.M[m].coo_col.p, inst.M[m].coo_val.p, inst.M[m].nnz};
  spark_commit(ctx, mats, 3, log2_ceil(inst.num_cons), log2_ceil(2 * inst.num_vars), gens.gens_r1cs_eval, e.dense, c.comm);
}

// ================================================================================================ steps the verifiers share
void append_sparse_commitment(Transcript& T, const SparseMatPolyCommitment& c) {
  T.append_u64("batch_size", c.batch_size); T.append_u64("num_ops", c.num_ops); T.append_u64("num_mem_cells", c.num_mem_cells);
  append_poly_commitment(T, "comm_comb_ops", c.comm_comb_ops);
  append_poly_commitment(T, "comm_comb_mem", c.comm_comb_mem);
}
void append_computation_commitment(Transcript& T, const ComputationCommitment& c) {
  T.append_u64("num_cons", c.num_cons); T.append_u64("num_vars", c.num_vars); T.append_u64("num_inputs", c.num_inputs);
  append_sparse_commitment(T, c.comm);
}
void append_derefs_commitment(Transcript& T, const PolyCommitment& c) {
  T.append_message("derefs_commitment", "begin_derefs_commitment");
  append_poly_commitment(T, "comm_poly_row_col_ops_val", c);
  T.append_message("derefs_commitment", "end_derefs_commitment");
}
bool append_memory_claims(Transcript& T, const ProductLayerProof& pl) {
  for (int side = 0; side < 2; side++) {
    const Fq& init = side ? pl.col_init : pl.row_init;
    const Fq& audit = side ? pl.col_audit : pl.row_audit;
    const std::vector<Fq>& read = side ? pl.col_read : pl.row_read;
    const std::vector<Fq>& write = side ? pl.col_write : pl.row_write;
    Fq ws = Fq::one(), rs = Fq::one();
    for (auto& w : write) ws *= w;
    for (auto& r : read) rs *= r;
    if (!(init * ws == rs * audit)) return false;
    T.append_scalar(side ? "claim_col_eval_init" : "claim_row_eval_init", init);
    T.append_scalars(side ? "claim_col_eval_read" : "claim_row_eval_read", read);
    T.append_scalars(side ? "claim_col_eval_write" : "claim_row_eval_write", write);
    T.append_scalar(side ? "claim_col_eval_audit" : "claim_row_eval_audit", audit);
  }
  return true;
}
void equalize(std::vector<Fq>& rx, std::vector<Fq>& ry) {
  if (rx.size() < ry.size()) rx.insert(rx.begin(), ry.size() - rx.size(), Fq::zero());
  if (ry.size() < rx.size()) ry.insert(ry.begin(), rx.size() - ry.size(), Fq::zero());
}
std::vector<Fq> combine_to_one(Transcript& T, std::vector<Fq> evals, const std::vector<Fq>& rand, const char* label_evals,
                               const char* label_challenge, const char* label_joint, Fq& joint) {
  evals.resize(next_pow2(evals.size()), Fq::zero());
  T.append_scalars(label_evals, evals);
  std::vector<Fq> r_joint = T.challenge_vector(label_challenge, log2_ceil(evals.size()));
  for (size_t k = r_joint.size(); k-- > 0;) {   // bound_poly_var_bot (dense_mlpoly.rs:225-233), last challenge first
    const size_t n = evals.size() / 2;
    for (size_t i = 0; i < n; i++) evals[i] = evals[2 * i] + r_joint[k] * (evals[2 * i + 1] - evals[2 * i]);
    evals.resize(n);
  }
  joint = evals[0];
  T.append_scalar(label_joint, joint);
  r_joint.insert(r_joint.end(), rand.begin(), rand.end());
  return r_joint;
}
std::vector<Fq> combine_to_one(Transcript& T, const HashLayerProof& hl, HashOpening which, const std::vector<Fq>& rand, Fq& joint) {
  const char* n_to_one = "challenge_combine_n_to_one";
  std::vector<Fq> evals;
  switch (which) {
    case HashOpening::derefs:   // DerefsEvalProof (sparse_mlpoly.rs:80-123)
      for (auto* v : {&hl.derefs_row, &hl.derefs_col}) evals.insert(evals.end(), v->begin(), v->end());
      return combine_to_one(T, evals, rand, "evals_ops_val", n_to_one, "joint_claim_eval", joint);
    case HashOpening::ops:
      for (auto* v : {&hl.row_addr, &hl.row_read_ts, &hl.col_addr, &hl.col_read_ts, &hl.eval_val}) evals.insert(evals.end(), v->begin(), v->end());
      return combine_to_one(T, evals, rand, "claim_evals_ops", n_to_one, "joint_claim_eval_ops", joint);
    case HashOpening::mem:
      return combine_to_one(T, {hl.row_audit_ts, hl.col_audit_ts}, rand, "claim_evals_mem", "challenge_combine_two_to_one", "joint_claim_eval_mem", joint);
  }
  throw SpError(SP_ERR_INTERNAL, "unknown hash-layer opening");
}
void sparse_evaluate(Ctx& ctx, const SparkMatrix* mats, size_t b, const std::vector<Fq>& rx, const std::vector<Fq>& ry, Fq* out) {
  DevBuf<u256> d_chal(rx.size() + ry.size() + 2), trx((size_t)1 << rx.size()), try_((size_t)1 << ry.size());
  DevBuf<u256> eq_small(dev::eq_evals_scratch(std::max(rx.size(), ry.size())));
  dev::h2d(d_chal.p, rx.data(), rx.size() * sizeof(u256), ctx.stream);
  dev::eq_evals(trx.p, d_chal.p, (int)rx.size(), eq_small.p, ctx.stream);
  dev::h2d(d_chal.p + rx.size(), ry.data(), ry.size() * sizeof(u256), ctx.stream);
  dev::eq_evals(try_.p, d_chal.p + rx.size(), (int)ry.size(), eq_small.p, ctx.stream);
  for (size_t m = 0; m < b; m++)
    dev::sparse_eval3(ctx.small.p + layout::SMALL_ABC.off + m, mats[m].row, mats[m].col, mats[m].val, mats[m].nnz, trx.p, try_.p, ctx.red.p, ctx.stream);
  ctx.get_small(layout::SMALL_ABC.off, out, b);
}
void instance_evaluate(Ctx& ctx, const Instance& inst, const std::vector<Fq>& rx, const std::vector<Fq>& ry, Fq out[3]) {
  SparkMatrix mats[3];
  for (int m = 0; m < 3; m++) mats[m] = SparkMatrix{inst.M[m].coo_row.p, inst.M[m].coo_col.p, inst.M[m].coo_val.p, inst.M[m].nnz};
  sparse_evaluate(ctx, mats, 3, rx, ry, out);
}
// the padding entries of the dense representation are (0, 0, value 0): they add nothing
void spark_evaluate(Ctx& ctx, const SparkDense& d, const std::vector<Fq>& rx, const std::vector<Fq>& ry, Fq* out) {
  SparkMatrix mats[SP_SPARK_MAX_BATCH];
  for (size_t m = 0; m < d.b; m++) mats[m] = SparkMatrix{d.row_idx[m].p, d.col_idx[m].p, d.val(m), d.N};
  sparse_evaluate(ctx, mats, d.b, rx, ry, out);
}

static void mark(Ctx& ctx, const char* name, std::chrono::steady_clock::time_point t0) {
  ctx.timings.push_back({name, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count()});
}

// ================================================================================================ SparseMatPolyEvalProof::prove
void spark_eval_prove(Ctx& ctx, const SparkDense& dv, const std::vector<Fq>& rx, const std::vector<Fq>& ry, const std::vector<Fq>& evals,
                      const SparkGens& gens, Transcript& T, RandomTape& tape, SparseMatPolyEvalProof& ep, const SparkDerefs* pre) {
  const size_t b = dv.b, N = dv.N, cells = dv.cells;
  const size_t lgN = log2_ceil(N), lgC = log2_ceil(cells);
  if (evals.size() != b) throw SpError(SP_ERR_INTERNAL, "SPARK: one evaluation per matrix");
  if (rx.size() != dv.x || ry.size() != dv.y) throw std::runtime_error("spartan_b200: unexpected evaluation point lengths");
  DevBuf<u256> d_chal(64), eq_small(dev::eq_evals_scratch(std::max(lgN + 4, lgC + 1)));
  T.append_protocol_name("Sparse polynomial evaluation proof");

  // ---- dereferenced values and their commitment (sparse_mlpoly.rs:507-512, :213-219): comb = row_ops_val[b] | col_ops_val[b] | zero pad
  const u256 *mem_rx, *mem_ry, *derefs_p;
  u256 *row_val[SP_SPARK_MAX_BATCH], *col_val[SP_SPARK_MAX_BATCH];
  DevBuf<u256> own_rx, own_ry, own_derefs;
  {
    auto tc = std::chrono::steady_clock::now();
    if (pre) {
      mem_rx = pre->mem_rx; mem_ry = pre->mem_ry; derefs_p = pre->derefs;
      ep.comm_derefs = pre->comm_derefs;
    } else {
      const size_t nd = next_pow2(2 * b) * N;
      own_rx.alloc(cells); own_ry.alloc(cells); own_derefs.alloc(nd);
      if (nd > 2 * b * N) dev::dzero(own_derefs.p + 2 * b * N, (nd - 2 * b * N) * sizeof(u256), ctx.stream);
      std::vector<Fq> rx_ext = rx, ry_ext = ry;
      equalize(rx_ext, ry_ext);
      dev::h2d(d_chal.p, rx_ext.data(), rx_ext.size() * sizeof(u256), ctx.stream);
      dev::eq_evals(own_rx.p, d_chal.p, (int)rx_ext.size(), eq_small.p, ctx.stream);
      dev::h2d(d_chal.p + 32, ry_ext.data(), ry_ext.size() * sizeof(u256), ctx.stream);
      dev::eq_evals(own_ry.p, d_chal.p + 32, (int)ry_ext.size(), eq_small.p, ctx.stream);
      for (size_t m = 0; m < b; m++) {
        dev::gather(own_derefs.p + m * N, own_rx.p, dv.row_idx[m].p, N, ctx.stream);
        dev::gather(own_derefs.p + (b + m) * N, own_ry.p, dv.col_idx[m].p, N, ctx.stream);
      }
      commit_poly(ctx, own_derefs.p, nd, gens.gens_derefs, ep.comm_derefs);
      mem_rx = own_rx.p; mem_ry = own_ry.p; derefs_p = own_derefs.p;
    }
    for (size_t m = 0; m < b; m++) { row_val[m] = const_cast<u256*>(derefs_p) + m * N; col_val[m] = const_cast<u256*>(derefs_p) + (b + m) * N; }
    append_derefs_commitment(T, ep.comm_derefs);
    mark(ctx, "commit_nondet_witness", tc);
  }
  std::vector<Fq> r_mem_check = T.challenge_vector("challenge_r_hash", 2);

  // ---- build_layered_network: hash layers (sparse_mlpoly.rs:529-604) written straight into layer 0 of the 4b + 4 product circuits
  auto tb = std::chrono::steady_clock::now();
  dev::h2d(d_chal.p, r_mem_check.data(), 2 * sizeof(u256), ctx.stream);
  struct Side { ProdCircuit init, audit, read[SP_SPARK_MAX_BATCH], write[SP_SPARK_MAX_BATCH]; } S[2];
  const int W = ctx.shard_world(), rk = ctx.rank();
  auto hash_into = [&](ProdCircuit& c, size_t n, const u256* addr, const u256* val, const u256* ts, int plus_one) {
    c.alloc(ctx, n);
    if (c.sharded(0)) dev::spark_hash_cyclic(c.layer(0), n / W, rk, W, addr, val, ts, plus_one, d_chal.p, ctx.stream);   // this rank's entries of the hash layer
    else dev::spark_hash(c.layer(0), n, addr, val, ts, plus_one, d_chal.p, ctx.stream);
  };
  for (int side = 0; side < 2; side++) {
    Side& s = S[side];
    const u256* mem = side == 0 ? mem_rx : mem_ry;
    hash_into(s.init, cells, nullptr, mem, nullptr, 0);
    hash_into(s.audit, cells, nullptr, mem, side == 0 ? dv.row_audit() : dv.col_audit(), 0);
    for (size_t m = 0; m < b; m++) {
      const u256* addr = side == 0 ? dv.row_addr(m) : dv.col_addr(m);
      const u256* ts = side == 0 ? dv.row_ts(m) : dv.col_ts(m);
      const u256* val = side == 0 ? row_val[m] : col_val[m];
      hash_into(s.read[m], N, addr, val, ts, 0);
      hash_into(s.write[m], N, addr, val, ts, 1);
    }
  }
  // the ops circuits in the order ProductLayerProof::prove batches them: row.read[b], row.write[b], col.read[b], col.write[b]
  std::vector<ProdCircuit*> prods;
  for (int side = 0; side < 2; side++) {
    for (size_t m = 0; m < b; m++) prods.push_back(&S[side].read[m]);
    for (size_t m = 0; m < b; m++) prods.push_back(&S[side].write[m]);
  }
  // every layer of the 4 memory-sized and the 4b ops-sized product trees: one launch per layer and group (product_tree.rs:36-56; 4b <= 16)
  build_circuits(ctx, {&S[0].init, &S[0].audit, &S[1].init, &S[1].audit});
  build_circuits(ctx, prods);
  ctx.sync();
  mark(ctx, "build_layered_network", tb);

  // ---- PolyEvalNetworkProof::prove (sparse_mlpoly.rs:1318-1354)
  auto tn = std::chrono::steady_clock::now();
  T.append_protocol_name("Sparse polynomial evaluation proof");
  ProductLayerProof& pl = ep.proof_prod_layer;
  T.append_protocol_name("Sparse polynomial product layer proof");  // ProductLayerProof::prove (sparse_mlpoly.rs:1035-1226)
  // ProductCircuit::evaluate of all 4b + 4 circuits (product_tree.rs:58-63): the two entries of every last layer through one gather kernel that
  // publishes them to the host, instead of one copy and stream synchronise per circuit
  const size_t per_side = 2 + 2 * b;
  std::vector<Fq> roots(2 * per_side);
  {
    std::vector<const u256*> hp;
    for (int side = 0; side < 2; side++) {
      Side& s = S[side];
      std::vector<ProdCircuit*> cs = {&s.init, &s.audit};
      for (size_t m = 0; m < b; m++) cs.push_back(&s.read[m]);
      for (size_t m = 0; m < b; m++) cs.push_back(&s.write[m]);
      for (auto* c : cs) { hp.push_back(c->layer(c->num_layers - 1)); hp.push_back(c->layer(c->num_layers - 1) + 1); }
    }
    DevBuf<u256> d_roots(hp.size());
    dev::HostSig hs = ctx.next_sig();
    dev::heads(d_roots.p, hp.data(), (int)hp.size(), ctx.stream, hs);
    ctx.wait_sig(hs);
    std::vector<Fq> v(hp.size());
    memcpy(v.data(), ctx.host_res + layout::RES_OUT.off, sizeof(Fq) * v.size());
    for (size_t c = 0; c < roots.size(); c++) roots[c] = v[2 * c] * v[2 * c + 1];
  }
  for (int side = 0; side < 2; side++) {
    const Fq* r = roots.data() + side * per_side;
    (side ? pl.col_init : pl.row_init) = r[0];
    (side ? pl.col_audit : pl.row_audit) = r[1];
    (side ? pl.col_read : pl.row_read).assign(r + 2, r + 2 + b);
    (side ? pl.col_write : pl.row_write).assign(r + 2 + b, r + 2 + 2 * b);
  }
  if (!append_memory_claims(T, pl)) throw SpError(SP_ERR_INTERNAL, "memory-check subset test failed (sparse_mlpoly.rs:1060)");
  // dot-product circuits: clones of (row_ops_val, col_ops_val, val), split in halves (sparse_mlpoly.rs:1090-1117), left_0, right_0, left_1, ...
  // Their claims are taken on the full tables; the copies the sumcheck binds are this rank's cyclic shards when the ops circuits are sharded.
  const bool sh_dotp = S[0].read[0].sharded(0);
  const size_t hN = N / 2, hloc = sh_dotp ? hN / W : hN;
  DevBuf<u256> dotp_buf(6 * b * hloc);
  std::vector<DotpCircuit> dotps;
  for (size_t m = 0; m < b; m++) {
    const u256* srcs[3] = {row_val[m], col_val[m], dv.val(m)};
    u256* d_lr2 = ctx.small.p + layout::SMALL_DOTP.off;
    dev::dot3(d_lr2, srcs[0], srcs[1], srcs[2], hN, ctx.red.p, ctx.stream);
    dev::dot3(d_lr2 + 1, srcs[0] + hN, srcs[1] + hN, srcs[2] + hN, hN, ctx.red.p, ctx.stream);
    Fq lr2[2];
    ctx.get_small(layout::SMALL_DOTP.off, lr2, 2);
    T.append_scalar("claim_eval_dotp_left", lr2[0]);
    T.append_scalar("claim_eval_dotp_right", lr2[1]);
    if (!(lr2[0] + lr2[1] == evals[m])) throw SpError(SP_ERR_INTERNAL, "dot-product circuit does not evaluate to the claimed matrix evaluation");
    pl.eval_dotp_left.push_back(lr2[0]); pl.eval_dotp_right.push_back(lr2[1]);
    for (int part = 0; part < 2; part++) {
      u256* base = dotp_buf.p + (6 * m + 3 * part) * hloc;
      for (int t = 0; t < 3; t++) {
        if (sh_dotp) dev::take_cyclic(base + t * hloc, srcs[t] + part * hN, hloc, rk, W, ctx.stream);
        else dev::d2d(base + t * hloc, srcs[t] + part * hN, hN * sizeof(u256), ctx.stream);
      }
      dotps.push_back(DotpCircuit{base, base + hloc, base + 2 * hloc, hloc, sh_dotp, lr2[part]});
    }
  }
  std::vector<Fq> rand_ops, rand_mem;
  {
    auto tq = std::chrono::steady_clock::now();
    batched_prove(ctx, prods, dotps, T, pl.proof_ops, rand_ops);
    mark(ctx, "  product_layer_ops(4b trees + 2b dotp)", tq);
    tq = std::chrono::steady_clock::now();
    std::vector<ProdCircuit*> mems = {&S[0].init, &S[0].audit, &S[1].init, &S[1].audit};
    std::vector<DotpCircuit> none;
    batched_prove(ctx, mems, none, T, pl.proof_mem, rand_mem);
    mark(ctx, "  product_layer_mem(4 trees)", tq);
  }
  auto th = std::chrono::steady_clock::now();

  // ---- HashLayerProof::prove (sparse_mlpoly.rs:722-835)
  HashLayerProof& hl = ep.proof_hash_layer;
  T.append_protocol_name("Sparse polynomial hash layer proof");
  {
    DevBuf<u256> eq_ops(N), eq_mem(cells);
    dev::h2d(d_chal.p, rand_ops.data(), rand_ops.size() * sizeof(u256), ctx.stream);
    dev::eq_evals(eq_ops.p, d_chal.p, (int)rand_ops.size(), eq_small.p, ctx.stream);
    dev::h2d(d_chal.p + 32, rand_mem.data(), rand_mem.size() * sizeof(u256), ctx.stream);
    dev::eq_evals(eq_mem.p, d_chal.p + 32, (int)rand_mem.size(), eq_small.p, ctx.stream);
    // 7b evaluations at rand_ops, 2 at rand_mem
    std::vector<const u256*> tabs;
    for (size_t m = 0; m < b; m++) tabs.push_back(row_val[m]);
    for (size_t m = 0; m < b; m++) tabs.push_back(col_val[m]);
    for (size_t m = 0; m < b; m++) tabs.push_back(dv.row_addr(m));
    for (size_t m = 0; m < b; m++) tabs.push_back(dv.row_ts(m));
    for (size_t m = 0; m < b; m++) tabs.push_back(dv.col_addr(m));
    for (size_t m = 0; m < b; m++) tabs.push_back(dv.col_ts(m));
    for (size_t m = 0; m < b; m++) tabs.push_back(dv.val(m));
    dev::dot_many(ctx.small.p + layout::SMALL_BATCH.off, tabs.data(), (int)tabs.size(), eq_ops.p, N, ctx.red.p, ctx.stream);
    const u256* mt[2] = {dv.row_audit(), dv.col_audit()};
    dev::dot_many(ctx.small.p + layout::SMALL_BATCH.off + tabs.size(), mt, 2, eq_mem.p, cells, ctx.red.p, ctx.stream);
    std::vector<Fq> ev(7 * b + 2);
    ctx.get_small(layout::SMALL_BATCH.off, ev.data(), ev.size());
    auto block = [&](size_t k) { return std::vector<Fq>(ev.begin() + k * b, ev.begin() + (k + 1) * b); };
    hl.derefs_row = block(0); hl.derefs_col = block(1);
    hl.row_addr = block(2); hl.row_read_ts = block(3);
    hl.col_addr = block(4); hl.col_read_ts = block(5);
    hl.eval_val = block(6);
    hl.row_audit_ts = ev[7 * b]; hl.col_audit_ts = ev[7 * b + 1];
  }
  mark(ctx, "  hash_layer_evaluations", th);
  th = std::chrono::steady_clock::now();
  Cp dummy;
  Fq joint;
  {  // DerefsEvalProof::prove (sparse_mlpoly.rs:125-149, prove_single :80-123)
    T.append_protocol_name("Derefs evaluation proof");
    const std::vector<Fq> r_joint = combine_to_one(T, hl, HashOpening::derefs, rand_ops, joint);
    polyeval_prove(ctx, derefs_p, nullptr, r_joint, &joint, nullptr, gens.gens_derefs, T, tape, hl.proof_derefs, dummy);
  }
  mark(ctx, "  polyeval_derefs", th);
  th = std::chrono::steady_clock::now();
  {  // ops decommitment (sparse_mlpoly.rs:766-797)
    const std::vector<Fq> r_joint = combine_to_one(T, hl, HashOpening::ops, rand_ops, joint);
    polyeval_prove(ctx, dv.comb_ops.p, nullptr, r_joint, &joint, nullptr, gens.gens_ops, T, tape, hl.proof_ops, dummy);
  }
  mark(ctx, "  polyeval_ops", th);
  th = std::chrono::steady_clock::now();
  {  // mem decommitment (sparse_mlpoly.rs:799-824)
    const std::vector<Fq> r_joint = combine_to_one(T, hl, HashOpening::mem, rand_mem, joint);
    polyeval_prove(ctx, dv.comb_mem.p, nullptr, r_joint, &joint, nullptr, gens.gens_mem, T, tape, hl.proof_mem, dummy);
  }
  mark(ctx, "  polyeval_mem", th);
  mark(ctx, "evalproof_layered_network", tn);
}

// ================================================================================================ SNARK::prove
void snark_prove(Ctx& ctx, const Instance& inst, const SnarkEncoding& enc, const u256* d_vars, const std::vector<Fq>& input, const SnarkGens& gens,
                 Transcript& T, const Fq& tape_seed, SnarkProof& out) {
  ctx.timings.clear();
  ShardScope shard(ctx);   // on a connected multi-GPU context every rank runs this same function on the same inputs (see DESIGN.md "Multi-GPU")
  auto t_start = std::chrono::steady_clock::now();
  RandomTape tape("proof", tape_seed);                    // lib.rs:352
  T.append_protocol_name("Spartan SNARK proof");          // lib.rs:354
  append_computation_commitment(T, enc.comm);

  const SparkDense& dv = enc.dense;
  const SparkGens& eg = gens.gens_r1cs_eval;
  const size_t N = dv.N, cells = dv.cells, b = dv.b;

  // ---- dereferenced values and their commitment (sparse_mlpoly.rs:507-512, :213-219), started EARLY on the background stream.
  // comb = row_ops_val[3] | col_ops_val[3] | zero pad, committed as an L x R matrix (dense_mlpoly.rs:165-177).  row_ops_val depends only on rx
  // (known after the first sumcheck phase), col_ops_val only on ry (after the second), and the transcript needs the commitment only after the
  // whole R1CS proof: the two 3N-term MSMs (ALU-bound, the longest kernels of the proof) run on ctx.stream2 underneath the latency-bound rounds
  // of phase two and of the witness evaluation proof, which keep the greatest stream priority.  Same values, same bytes, different timing.
  // Without the overlap spark_eval_prove computes them inline.
  const size_t nd = next_pow2(2 * b) * N;
  const size_t ell_d = log2_ceil(nd), L_d = (size_t)1 << (ell_d / 2), R_d = (size_t)1 << (ell_d - ell_d / 2);
  if (R_d != eg.gens_derefs.n) throw SpError(SP_ERR_INVALID_ARG, "polynomial size does not match the commitment generators (num_nz_entries too small?)");
  const bool early = ctx.overlap && N % R_d == 0;                 // each of the two parts is a whole number of matrix rows
  const size_t n_part = early ? b * N / R_d : 0;                  // rows per part; rows [2 n_part, L_d) are zero: the identity, 32 zero bytes
  const size_t Wd = (size_t)ctx.shard_world();
  const bool shard_rows = early && Wd > 1 && n_part % Wd == 0;    // rank r commits rows [r n_part/W, (r+1) n_part/W) of either part
  const size_t cnt = shard_rows ? n_part / Wd : n_part;
  const size_t nx = dv.x, ny = dv.y, nxy = std::max(nx, ny);
  DevBuf<u256> mem_rx, mem_ry, derefs;
  DevBuf<u256> d_chal2, eq_small2;
  DevBuf<ge> early_rows;
  DevBuf<uint8_t> early_comp;
  struct ForkGuard {   // an exception between fork and join must not release buffers the background stream still works on
    Ctx& c; bool forked = false;
    ~ForkGuard() { if (forked) { try { dev::stream_sync(c.stream2); } catch (...) {} } }
  } fork_guard{ctx};
  // a 60 KB shared-memory pad: three resident MSM CTAs per SM instead of four leave a quarter of every register file to the prover's stream
  // (DESIGN.md §3 has the H100 A/B)
  const size_t early_smem_pad = 60 << 10;
  if (early) {
    if (nxy * sizeof(u256) > layout::PIN_XY_PART) throw SpError(SP_ERR_INVALID_ARG, "instance with too many variables for the staged evaluation points");
    mem_rx.alloc(cells); mem_ry.alloc(cells); derefs.alloc(nd);
    if (nd > 2 * b * N) dev::dzero(derefs.p + 2 * b * N, (nd - 2 * b * N) * sizeof(u256), ctx.stream);
    d_chal2.alloc(64); eq_small2.alloc(dev::eq_evals_scratch(std::max(log2_ceil(N) + 4, log2_ceil(cells) + 1))); early_rows.alloc(2 * cnt); early_comp.alloc(64 * cnt);
    const size_t need = dev::msm_scratch_bytes(cnt, R_d) + 64;
    if (ctx.scratch2.n < need) { dev::stream_sync(ctx.stream2); ctx.scratch2.alloc(need); }
  }
  auto early_part = [&](int part, const std::vector<Fq>& pt) {   // part 0: rows from rx, part 1: columns from ry
    // equalize (sparse_mlpoly.rs:1429-1445): left-pad the shorter point with zeros; staged in pinned memory so that the copy never waits for the stream
    Fq* ext = reinterpret_cast<Fq*>(ctx.pinned + layout::PIN_XY.off + (size_t)part * layout::PIN_XY_PART);
    for (size_t i = 0; i < nxy - pt.size(); i++) ext[i] = Fq::zero();
    for (size_t i = 0; i < pt.size(); i++) ext[nxy - pt.size() + i] = pt[i];
    dev::event_record(ctx.ev_fork, ctx.stream);
    dev::stream_wait_event(ctx.stream2, ctx.ev_fork);
    fork_guard.forked = true;
    cudaStream_t s2 = ctx.stream2;
    u256* chal = d_chal2.p + 32 * part;
    u256* mem = part ? mem_ry.p : mem_rx.p;
    dev::h2d(chal, ext, nxy * sizeof(u256), s2);
    dev::eq_evals(mem, chal, (int)nxy, eq_small2.p, s2);
    for (size_t m = 0; m < b; m++) dev::gather(derefs.p + (part * b + m) * N, mem, (part ? dv.col_idx : dv.row_idx)[m].p, N, s2);
    const size_t first = (size_t)part * n_part + (shard_rows ? (size_t)ctx.rank() * cnt : 0);
    const CommitKey& key = eg.gens_derefs.gens_n;
    dev::msm_rows(early_rows.p + (size_t)part * cnt, key.set->table.p, key.set->wbits, key.set->rows(), derefs.p + first * R_d, R_d, cnt, R_d, nullptr, key.h, ctx.scratch2.p, s2, early_smem_pad);
    dev::compress_batch(early_comp.p + 32 * (size_t)part * cnt, early_rows.p + (size_t)part * cnt, cnt, s2);
  };
  R1csHooks hooks;
  if (early) {
    hooks.on_rx = [&](const std::vector<Fq>& p) { early_part(0, p); };
    hooks.on_ry = [&](const std::vector<Fq>& p) { early_part(1, p); };
  }

  std::vector<Fq> rx, ry;
  r1cs_prove(ctx, InstanceMatrices(inst), d_vars, input, *gens.gens_r1cs_sat, T, tape, out.r1cs_sat_proof, rx, ry, early ? &hooks : nullptr);

  auto t0 = std::chrono::steady_clock::now();
  const std::array<Fq, 3>& inst_evals = out.inst_evals;
  instance_evaluate(ctx, inst, rx, ry, out.inst_evals.data());
  T.append_scalar("Ar_claim", inst_evals[0]);
  T.append_scalar("Br_claim", inst_evals[1]);
  T.append_scalar("Cr_claim", inst_evals[2]);
  mark(ctx, "eval_sparse_polys", t0);

  // ---- R1CSEvalProof::prove -> SparseMatPolyEvalProof::prove (sparse_mlpoly.rs:1447-1514)
  auto t_eval = std::chrono::steady_clock::now();
  if (nx != rx.size() || ny != ry.size()) throw std::runtime_error("spartan_b200: unexpected sumcheck point lengths");
  std::optional<SparkDerefs> pre;
  if (early) {
    // join: the prover's stream continues after the background commitments; gather the rank shares when the rows were split
    dev::event_record(ctx.ev_join, ctx.stream2);
    dev::stream_wait_event(ctx.stream, ctx.ev_join);
    std::vector<uint8_t> hb(64 * cnt * (shard_rows ? Wd : 1));
    if (shard_rows) dev::d2h(hb.data(), ctx.allgather_block(early_comp.p, 64 * cnt), hb.size(), ctx.stream);
    else dev::d2h(hb.data(), early_comp.p, hb.size(), ctx.stream);
    ctx.sync();
    fork_guard.forked = false;
    pre.emplace(SparkDerefs{derefs.p, mem_rx.p, mem_ry.p, PolyCommitment{}});
    pre->comm_derefs.C.assign(L_d, Cp{});                                 // value-initialised: 32 zero bytes = the identity's encoding
    for (size_t r = 0; r < (shard_rows ? Wd : 1); r++)
      for (int part = 0; part < 2; part++)
        memcpy(pre->comm_derefs.C[(size_t)part * n_part + r * cnt].b, hb.data() + (r * 2 + part) * 32 * cnt, 32 * cnt);
  }
  spark_eval_prove(ctx, dv, rx, ry, std::vector<Fq>(inst_evals.begin(), inst_evals.end()), eg, T, tape, out.r1cs_eval_proof, pre ? &*pre : nullptr);
  mark(ctx, "R1CSEvalProof::prove", t_eval);
  mark(ctx, "SNARK::prove", t_start);
  for (auto& f : ctx.fine) ctx.timings.push_back({"fine:" + f.first, f.second});
  ctx.fine.clear();
}

}  // namespace sp
