// spartan_b200 — SNARK path: SNARK::encode / SNARK::prove (src/lib.rs:325-420) with the SPARK sparse-polynomial evaluation proof
// (src/sparse_mlpoly.rs:1447-1514, src/product_tree.rs:259-383) driven on the device.  Every table of the memory-checking network
// (hash layers, 16 product trees with all their layers, dereferenced values) lives in HBM; the host only runs the transcript.
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

SparkDims::SparkDims(size_t num_cons, size_t nvp, size_t num_nz_entries) {
  size_t x = log2_ceil(num_cons), y = log2_ceil(2 * nvp), lgnz = log2_ceil(next_pow2(num_nz_entries));
  v_ops = lgnz + log2_ceil(next_pow2(3 * 5)); v_mem = std::max(x, y) + 1; v_derefs = lgnz + log2_ceil(next_pow2(3 * 2));
  n_ops = (size_t)1 << (v_ops - v_ops / 2); n_mem = (size_t)1 << (v_mem - v_mem / 2); n_der = (size_t)1 << (v_derefs - v_derefs / 2);
}

GenTables::GenTables(Ctx* c, size_t num_cons, size_t num_vars, size_t num_inputs, size_t num_nz_entries) : ctx(c) {
  const size_t nvp = padded_num_vars(num_vars, num_inputs);
  r1cs_sat = std::make_shared<GenSet>(ctx, "gens_r1cs_sat", R1CSGens::bases(nvp), R1CSGens::host_bases(nvp));
  if (num_nz_entries) {
    const SparkDims d(num_cons, nvp, num_nz_entries);
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
  const SparkDims d(num_cons, nvp, num_nz_entries);
  tables.require(ctx, R1CSGens::bases(nvp), d.bases());     // both sets before either view: the message names both
  gens_r1cs_sat.reset(new R1CSGens(ctx, tables, nvp));
  eval_set = tables.r1cs_eval;
  eval_set->add_host_tables(d.host_bases());
  gens_ops = pc_view(eval_set.get(), d.v_ops);
  gens_mem = pc_view(eval_set.get(), d.v_mem);
  gens_derefs = pc_view(eval_set.get(), d.v_derefs);
}

static void commit_poly(Ctx& ctx, const u256* d_Z, size_t len, const PolyCommitmentGens& gens, PolyCommitment& out) {  // DensePolynomial::commit, no blinds
  size_t ell = log2_ceil(len);
  size_t L = (size_t)1 << (ell / 2), R = (size_t)1 << (ell - ell / 2);
  if (R != gens.n) throw SpError(SP_ERR_INVALID_ARG, "polynomial size does not match the commitment generators (num_nz_entries too small?)");
  commit_rows_and_compress(ctx, gens.gens_n, d_Z, R, L, R, nullptr, out.C);
}

// ================================================================================================ SNARK::encode
void snark_encode(Ctx& ctx, const Instance& inst, const SnarkGens& gens, SnarkEncoding& e) {
  // SparseMatPolynomial::multi_commit -> multi_sparse_to_dense_rep (sparse_mlpoly.rs:366-420, :483-503)
  ComputationCommitment& c = e.comm;
  c.num_cons = inst.num_cons; c.num_vars = inst.num_vars; c.num_inputs = inst.num_inputs;
  c.batch_size = 3;
  size_t N = 1;
  for (int m = 0; m < 3; m++) N = std::max(N, next_pow2(inst.M[m].nnz));
  // every product circuit of the memory check has log2(N) layers and the proof binds its last one: with at most one entry per matrix there is
  // none (the reference panics in ProductCircuit::evaluate)
  if (N < 2) throw SpError(SP_ERR_INVALID_ARG, "SNARK::encode needs a matrix with at least two entries (num_ops = 1 leaves the product circuits without layers)");
  size_t x = log2_ceil(inst.num_cons), y = log2_ceil(2 * inst.num_vars);
  size_t cells = (size_t)1 << std::max(x, y);
  c.num_ops = N; c.num_mem_cells = cells;
  e.comb_ops.alloc(16 * N);   // row.ops_addr[3] | row.read_ts[3] | col.ops_addr[3] | col.read_ts[3] | val[3] | zero pad  (DensePolynomial::merge)
  e.comb_mem.alloc(2 * cells);
  dev::dzero(e.comb_ops.p, 16 * N * sizeof(u256), ctx.stream);
  DevBuf<uint8_t> scratch(dev::spark_ts_scratch_bytes(N, cells));
  DevBuf<unsigned int> bad(1);
  dev::dzero(bad.p, sizeof(unsigned int), ctx.stream);
  for (int side = 0; side < 2; side++) {  // AddrTimestamps::new (sparse_mlpoly.rs:220-254), row then col
    AddrTimestampsDev& at = side == 0 ? e.row : e.col;
    at.ops_addr_idx.resize(3);
    dev::SparkAddrs sa;
    for (int m = 0; m < 3; m++) {
      at.ops_addr_idx[m].alloc(N);
      sa.src[m] = side == 0 ? inst.M[m].coo_row.p : inst.M[m].coo_col.p;
      sa.nnz[m] = inst.M[m].nnz;
      sa.idx[m] = at.ops_addr_idx[m].p;
    }
    // ops_addr[3] | read_ts[3] of this side are contiguous in comb_ops: position m*N + i of the loop's order is element m*N + i of each block
    dev::spark_timestamps(sa, e.comb_ops.p + (size_t)side * 6 * N, e.comb_ops.p + (size_t)(side * 6 + 3) * N, e.comb_mem.p + (size_t)side * cells, N, cells,
                          scratch.p, bad.p, ctx.stream);
  }
  for (int m = 0; m < 3; m++) dev::d2d(e.comb_ops.p + (size_t)(12 + m) * N, inst.M[m].coo_val.p, inst.M[m].nnz * sizeof(u256), ctx.stream);
  unsigned int out_of_range = 0;
  dev::d2h(&out_of_range, bad.p, sizeof(unsigned int), ctx.stream);
  ctx.sync();
  if (out_of_range) throw SpError(SP_ERR_INVALID_INDEX, "address out of range");
  commit_poly(ctx, e.comb_ops.p, 16 * N, gens.gens_ops, c.comm_comb_ops);
  commit_poly(ctx, e.comb_mem.p, 2 * cells, gens.gens_mem, c.comm_comb_mem);
}

// views into the dense representation
struct DenseView {
  size_t N, cells;
  const u256 *row_addr[3], *row_ts[3], *col_addr[3], *col_ts[3], *val[3], *row_audit, *col_audit;
  explicit DenseView(const SnarkEncoding& e) : N(e.comm.num_ops), cells(e.comm.num_mem_cells) {
    for (int m = 0; m < 3; m++) {
      row_addr[m] = e.comb_ops.p + (size_t)m * N; row_ts[m] = e.comb_ops.p + (size_t)(3 + m) * N;
      col_addr[m] = e.comb_ops.p + (size_t)(6 + m) * N; col_ts[m] = e.comb_ops.p + (size_t)(9 + m) * N;
      val[m] = e.comb_ops.p + (size_t)(12 + m) * N;
    }
    row_audit = e.comb_mem.p; col_audit = e.comb_mem.p + cells;
  }
};

// ================================================================================================ steps SNARK::verify shares
void append_computation_commitment(Transcript& T, const ComputationCommitment& c) {
  T.append_u64("num_cons", c.num_cons); T.append_u64("num_vars", c.num_vars); T.append_u64("num_inputs", c.num_inputs);
  T.append_u64("batch_size", c.batch_size); T.append_u64("num_ops", c.num_ops); T.append_u64("num_mem_cells", c.num_mem_cells);
  append_poly_commitment(T, "comm_comb_ops", c.comm_comb_ops);
  append_poly_commitment(T, "comm_comb_mem", c.comm_comb_mem);
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
void instance_evaluate(Ctx& ctx, const Instance& inst, const std::vector<Fq>& rx, const std::vector<Fq>& ry, Fq out[3]) {
  DevBuf<u256> d_chal(rx.size() + ry.size() + 2), trx((size_t)1 << rx.size()), try_((size_t)1 << ry.size());
  DevBuf<u256> eq_small(dev::eq_evals_scratch(std::max(rx.size(), ry.size())));
  dev::h2d(d_chal.p, rx.data(), rx.size() * sizeof(u256), ctx.stream);
  dev::eq_evals(trx.p, d_chal.p, (int)rx.size(), eq_small.p, ctx.stream);
  dev::h2d(d_chal.p + rx.size(), ry.data(), ry.size() * sizeof(u256), ctx.stream);
  dev::eq_evals(try_.p, d_chal.p + rx.size(), (int)ry.size(), eq_small.p, ctx.stream);
  for (int m = 0; m < 3; m++)
    dev::sparse_eval3(ctx.small.p + layout::SMALL_ABC.off + m, inst.M[m].coo_row.p, inst.M[m].coo_col.p, inst.M[m].coo_val.p, inst.M[m].nnz, trx.p, try_.p, ctx.red.p, ctx.stream);
  ctx.get_small(layout::SMALL_ABC.off, out, 3);
}

// ================================================================================================ SNARK::prove
void snark_prove(Ctx& ctx, const Instance& inst, const SnarkEncoding& enc, const u256* d_vars, const std::vector<Fq>& input, const SnarkGens& gens,
                 Transcript& T, const Fq& tape_seed, SnarkProof& out) {
  ctx.timings.clear();
  ShardScope shard(ctx);   // on a connected multi-GPU context every rank runs this same function on the same inputs (see DESIGN.md "Multi-GPU")
  auto t_start = std::chrono::steady_clock::now();
  auto mark = [&](const char* name, std::chrono::steady_clock::time_point t0) {
    ctx.timings.push_back({name, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count()});
  };
  RandomTape tape("proof", tape_seed);                    // lib.rs:352
  T.append_protocol_name("Spartan SNARK proof");          // lib.rs:354
  append_computation_commitment(T, enc.comm);

  const DenseView dv(enc);
  const size_t N = dv.N, cells = dv.cells;
  const size_t lgN = log2_ceil(N), lgC = log2_ceil(cells);
  DevBuf<u256> d_chal(64), eq_small(dev::eq_evals_scratch(std::max(lgN + 4, lgC + 1)));

  // ---- dereferenced values and their commitment (sparse_mlpoly.rs:507-512, :213-219), started EARLY on the background stream.
  // comb = row_ops_val[3] | col_ops_val[3] | zero pad, committed as an L x R matrix (dense_mlpoly.rs:165-177).  row_ops_val depends only on rx
  // (known after the first sumcheck phase), col_ops_val only on ry (after the second), and the transcript needs the commitment only after the
  // whole R1CS proof: the two 3N-term MSMs (ALU-bound, the longest kernels of the proof) run on ctx.stream2 underneath the latency-bound rounds
  // of phase two and of the witness evaluation proof, which keep the greatest stream priority.  Same values, same bytes, different timing.
  DevBuf<u256> mem_rx(cells), mem_ry(cells), derefs(8 * N);
  dev::dzero(derefs.p + 6 * N, 2 * N * sizeof(u256), ctx.stream);
  u256 *row_val[3], *col_val[3];
  for (int m = 0; m < 3; m++) { row_val[m] = derefs.p + (size_t)m * N; col_val[m] = derefs.p + (size_t)(3 + m) * N; }
  const size_t ell_d = log2_ceil(8 * N), L_d = (size_t)1 << (ell_d / 2), R_d = (size_t)1 << (ell_d - ell_d / 2);
  if (R_d != gens.gens_derefs.n) throw SpError(SP_ERR_INVALID_ARG, "polynomial size does not match the commitment generators (num_nz_entries too small?)");
  const bool early = ctx.overlap && N % R_d == 0;                 // each of the two parts is a whole number of matrix rows
  const size_t n_part = early ? 3 * N / R_d : 0;                  // rows per part; rows [2 n_part, L_d) are zero: the identity, 32 zero bytes
  const size_t Wd = (size_t)ctx.shard_world();
  const bool shard_rows = early && Wd > 1 && n_part % Wd == 0;    // rank r commits rows [r n_part/W, (r+1) n_part/W) of either part
  const size_t cnt = shard_rows ? n_part / Wd : n_part;
  const size_t nx = log2_ceil(inst.num_cons), ny = log2_ceil(2 * inst.num_vars), nxy = std::max(nx, ny);
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
    d_chal2.alloc(64); eq_small2.alloc(eq_small.n); early_rows.alloc(2 * cnt); early_comp.alloc(64 * cnt);
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
    for (int m = 0; m < 3; m++) dev::gather(part ? col_val[m] : row_val[m], mem, (part ? enc.col : enc.row).ops_addr_idx[m].p, N, s2);
    const size_t first = (size_t)part * n_part + (shard_rows ? (size_t)ctx.rank() * cnt : 0);
    const CommitKey& key = gens.gens_derefs.gens_n;
    dev::msm_rows(early_rows.p + (size_t)part * cnt, key.set->table.p, key.set->wbits, key.set->rows(), derefs.p + first * R_d, R_d, cnt, R_d, nullptr, key.h, ctx.scratch2.p, s2, early_smem_pad);
    dev::compress_batch(early_comp.p + 32 * (size_t)part * cnt, early_rows.p + (size_t)part * cnt, cnt, s2);
  };
  R1csHooks hooks;
  if (early) {
    hooks.on_rx = [&](const std::vector<Fq>& p) { early_part(0, p); };
    hooks.on_ry = [&](const std::vector<Fq>& p) { early_part(1, p); };
  }

  std::vector<Fq> rx, ry;
  r1cs_prove(ctx, inst, d_vars, input, *gens.gens_r1cs_sat, T, tape, out.r1cs_sat_proof, rx, ry, early ? &hooks : nullptr);

  auto t0 = std::chrono::steady_clock::now();
  const std::array<Fq, 3>& inst_evals = out.inst_evals;
  instance_evaluate(ctx, inst, rx, ry, out.inst_evals.data());
  T.append_scalar("Ar_claim", inst_evals[0]);
  T.append_scalar("Br_claim", inst_evals[1]);
  T.append_scalar("Cr_claim", inst_evals[2]);
  mark("eval_sparse_polys", t0);

  // ---- R1CSEvalProof::prove -> SparseMatPolyEvalProof::prove (sparse_mlpoly.rs:1447-1514)
  auto t_eval = std::chrono::steady_clock::now();
  SparseMatPolyEvalProof& ep = out.r1cs_eval_proof;
  T.append_protocol_name("Sparse polynomial evaluation proof");
  if (nx != rx.size() || ny != ry.size()) throw std::runtime_error("spartan_b200: unexpected sumcheck point lengths");
  {
    auto tc = std::chrono::steady_clock::now();
    if (early) {
      // join: the prover's stream continues after the background commitments; gather the rank shares when the rows were split
      dev::event_record(ctx.ev_join, ctx.stream2);
      dev::stream_wait_event(ctx.stream, ctx.ev_join);
      std::vector<uint8_t> hb(64 * cnt * (shard_rows ? Wd : 1));
      if (shard_rows) dev::d2h(hb.data(), ctx.allgather_block(early_comp.p, 64 * cnt), hb.size(), ctx.stream);
      else dev::d2h(hb.data(), early_comp.p, hb.size(), ctx.stream);
      ctx.sync();
      fork_guard.forked = false;
      ep.comm_derefs.C.assign(L_d, Cp{});                                  // value-initialised: 32 zero bytes = the identity's encoding
      for (size_t r = 0; r < (shard_rows ? Wd : 1); r++)
        for (int part = 0; part < 2; part++)
          memcpy(ep.comm_derefs.C[(size_t)part * n_part + r * cnt].b, hb.data() + (r * 2 + part) * 32 * cnt, 32 * cnt);
    } else {
      std::vector<Fq> rx_ext = rx, ry_ext = ry;
      equalize(rx_ext, ry_ext);
      dev::h2d(d_chal.p, rx_ext.data(), rx_ext.size() * sizeof(u256), ctx.stream);
      dev::eq_evals(mem_rx.p, d_chal.p, (int)rx_ext.size(), eq_small.p, ctx.stream);
      dev::h2d(d_chal.p + 32, ry_ext.data(), ry_ext.size() * sizeof(u256), ctx.stream);
      dev::eq_evals(mem_ry.p, d_chal.p + 32, (int)ry_ext.size(), eq_small.p, ctx.stream);
      for (int m = 0; m < 3; m++) {
        dev::gather(row_val[m], mem_rx.p, enc.row.ops_addr_idx[m].p, N, ctx.stream);
        dev::gather(col_val[m], mem_ry.p, enc.col.ops_addr_idx[m].p, N, ctx.stream);
      }
      commit_poly(ctx, derefs.p, 8 * N, gens.gens_derefs, ep.comm_derefs);
    }
    append_derefs_commitment(T, ep.comm_derefs);
    mark("commit_nondet_witness", tc);
  }
  std::vector<Fq> r_mem_check = T.challenge_vector("challenge_r_hash", 2);

  // ---- build_layered_network: hash layers (sparse_mlpoly.rs:529-604) written straight into layer 0 of the 16 product circuits
  auto tb = std::chrono::steady_clock::now();
  dev::h2d(d_chal.p, r_mem_check.data(), 2 * sizeof(u256), ctx.stream);
  struct Side { ProdCircuit init, audit, read[3], write[3]; } S[2];
  const int W = ctx.shard_world(), rk = ctx.rank();
  auto hash_into = [&](ProdCircuit& c, size_t n, const u256* addr, const u256* val, const u256* ts, int plus_one) {
    c.alloc(ctx, n);
    if (c.sharded(0)) dev::spark_hash_cyclic(c.layer(0), n / W, rk, W, addr, val, ts, plus_one, d_chal.p, ctx.stream);   // this rank's entries of the hash layer
    else dev::spark_hash(c.layer(0), n, addr, val, ts, plus_one, d_chal.p, ctx.stream);
  };
  for (int side = 0; side < 2; side++) {
    Side& s = S[side];
    const u256* mem = side == 0 ? mem_rx.p : mem_ry.p;
    hash_into(s.init, cells, nullptr, mem, nullptr, 0);
    hash_into(s.audit, cells, nullptr, mem, side == 0 ? dv.row_audit : dv.col_audit, 0);
    for (int m = 0; m < 3; m++) {
      const u256* addr = side == 0 ? dv.row_addr[m] : dv.col_addr[m];
      const u256* ts = side == 0 ? dv.row_ts[m] : dv.col_ts[m];
      const u256* val = side == 0 ? row_val[m] : col_val[m];
      hash_into(s.read[m], N, addr, val, ts, 0);
      hash_into(s.write[m], N, addr, val, ts, 1);
    }
  }
  // every layer of the 4 memory-sized and the 12 ops-sized product trees: one launch per layer (product_tree.rs:36-56)
  build_circuits(ctx, {&S[0].init, &S[0].audit, &S[1].init, &S[1].audit});
  build_circuits(ctx, {&S[0].read[0], &S[0].read[1], &S[0].read[2], &S[0].write[0], &S[0].write[1], &S[0].write[2],
                       &S[1].read[0], &S[1].read[1], &S[1].read[2], &S[1].write[0], &S[1].write[1], &S[1].write[2]});
  ctx.sync();
  mark("build_layered_network", tb);

  // ---- PolyEvalNetworkProof::prove (sparse_mlpoly.rs:1318-1354)
  auto tn = std::chrono::steady_clock::now();
  T.append_protocol_name("Sparse polynomial evaluation proof");
  ProductLayerProof& pl = ep.proof_prod_layer;
  T.append_protocol_name("Sparse polynomial product layer proof");  // ProductLayerProof::prove (sparse_mlpoly.rs:1035-1226)
  // ProductCircuit::evaluate of all 16 circuits (product_tree.rs:58-63): the two entries of every last layer through one gather kernel that
  // publishes them to the host, instead of 16 copies each followed by a stream synchronise
  Fq roots[2][8];
  {
    std::vector<const u256*> hp;
    for (int side = 0; side < 2; side++) {
      Side& s = S[side];
      ProdCircuit* cs[8] = {&s.init, &s.audit, &s.read[0], &s.read[1], &s.read[2], &s.write[0], &s.write[1], &s.write[2]};
      for (auto* c : cs) { hp.push_back(c->layer(c->num_layers - 1)); hp.push_back(c->layer(c->num_layers - 1) + 1); }
    }
    DevBuf<u256> d_roots(hp.size());
    dev::HostSig hs = ctx.next_sig();
    dev::heads(d_roots.p, hp.data(), (int)hp.size(), ctx.stream, hs);
    ctx.wait_sig(hs);
    Fq v[32];
    memcpy(v, ctx.host_res + layout::RES_OUT.off, sizeof v);
    for (int side = 0; side < 2; side++) for (int c = 0; c < 8; c++) roots[side][c] = v[16 * side + 2 * c] * v[16 * side + 2 * c + 1];
  }
  const Fq* rr = roots[0];
  pl.row_init = rr[0]; pl.row_audit = rr[1]; pl.row_read = {rr[2], rr[3], rr[4]}; pl.row_write = {rr[5], rr[6], rr[7]};
  const Fq* rc = roots[1];
  pl.col_init = rc[0]; pl.col_audit = rc[1]; pl.col_read = {rc[2], rc[3], rc[4]}; pl.col_write = {rc[5], rc[6], rc[7]};
  if (!append_memory_claims(T, pl)) throw SpError(SP_ERR_INTERNAL, "memory-check subset test failed (sparse_mlpoly.rs:1060)");
  // dot-product circuits: clones of (row_ops_val, col_ops_val, val), split in halves (sparse_mlpoly.rs:1090-1117).  Their claims are taken on the
  // full tables; the copies the sumcheck binds are this rank's cyclic shards when the ops circuits are sharded.
  const bool sh_dotp = S[0].read[0].sharded(0);
  const size_t hN = N / 2, hloc = sh_dotp ? hN / W : hN;
  DevBuf<u256> dotp_buf(18 * hloc);
  std::vector<DotpCircuit> dotps;
  for (int m = 0; m < 3; m++) {
    const u256* srcs[3] = {row_val[m], col_val[m], dv.val[m]};
    u256* d_lr2 = ctx.small.p + layout::SMALL_DOTP.off;
    dev::dot3(d_lr2, srcs[0], srcs[1], srcs[2], hN, ctx.red.p, ctx.stream);
    dev::dot3(d_lr2 + 1, srcs[0] + hN, srcs[1] + hN, srcs[2] + hN, hN, ctx.red.p, ctx.stream);
    Fq lr2[2];
    ctx.get_small(layout::SMALL_DOTP.off, lr2, 2);
    T.append_scalar("claim_eval_dotp_left", lr2[0]);
    T.append_scalar("claim_eval_dotp_right", lr2[1]);
    if (!(lr2[0] + lr2[1] == inst_evals[m])) throw SpError(SP_ERR_INTERNAL, "dot-product circuit does not evaluate to the claimed matrix evaluation");
    pl.eval_dotp_left.push_back(lr2[0]); pl.eval_dotp_right.push_back(lr2[1]);
    for (int part = 0; part < 2; part++) {
      u256* base = dotp_buf.p + (size_t)(6 * m + 3 * part) * hloc;
      for (int t = 0; t < 3; t++) {
        if (sh_dotp) dev::take_cyclic(base + t * hloc, srcs[t] + part * hN, hloc, rk, W, ctx.stream);
        else dev::d2d(base + t * hloc, srcs[t] + part * hN, hN * sizeof(u256), ctx.stream);
      }
      dotps.push_back(DotpCircuit{base, base + hloc, base + 2 * hloc, hloc, sh_dotp, lr2[part]});
    }
  }
  std::vector<Fq> rand_ops, rand_mem;
  {
    std::vector<ProdCircuit*> prods = {&S[0].read[0], &S[0].read[1], &S[0].read[2], &S[0].write[0], &S[0].write[1], &S[0].write[2],
                                       &S[1].read[0], &S[1].read[1], &S[1].read[2], &S[1].write[0], &S[1].write[1], &S[1].write[2]};
    auto tq = std::chrono::steady_clock::now();
    batched_prove(ctx, prods, dotps, T, pl.proof_ops, rand_ops);
    mark("  product_layer_ops(12 trees + 6 dotp)", tq);
    tq = std::chrono::steady_clock::now();
    std::vector<ProdCircuit*> mems = {&S[0].init, &S[0].audit, &S[1].init, &S[1].audit};
    std::vector<DotpCircuit> none;
    batched_prove(ctx, mems, none, T, pl.proof_mem, rand_mem);
    mark("  product_layer_mem(4 trees)", tq);
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
    // 21 evaluations at rand_ops, 2 at rand_mem
    std::vector<const u256*> tabs;
    for (int m = 0; m < 3; m++) tabs.push_back(row_val[m]);
    for (int m = 0; m < 3; m++) tabs.push_back(col_val[m]);
    for (int m = 0; m < 3; m++) tabs.push_back(dv.row_addr[m]);
    for (int m = 0; m < 3; m++) tabs.push_back(dv.row_ts[m]);
    for (int m = 0; m < 3; m++) tabs.push_back(dv.col_addr[m]);
    for (int m = 0; m < 3; m++) tabs.push_back(dv.col_ts[m]);
    for (int m = 0; m < 3; m++) tabs.push_back(dv.val[m]);
    dev::dot_many(ctx.small.p + layout::SMALL_BATCH.off, tabs.data(), (int)tabs.size(), eq_ops.p, N, ctx.red.p, ctx.stream);
    const u256* mt[2] = {dv.row_audit, dv.col_audit};
    dev::dot_many(ctx.small.p + layout::SMALL_BATCH.off + tabs.size(), mt, 2, eq_mem.p, cells, ctx.red.p, ctx.stream);
    std::vector<Fq> ev(23);
    ctx.get_small(layout::SMALL_BATCH.off, ev.data(), 23);
    hl.derefs_row.assign(ev.begin(), ev.begin() + 3);
    hl.derefs_col.assign(ev.begin() + 3, ev.begin() + 6);
    hl.row_addr.assign(ev.begin() + 6, ev.begin() + 9);
    hl.row_read_ts.assign(ev.begin() + 9, ev.begin() + 12);
    hl.col_addr.assign(ev.begin() + 12, ev.begin() + 15);
    hl.col_read_ts.assign(ev.begin() + 15, ev.begin() + 18);
    hl.eval_val.assign(ev.begin() + 18, ev.begin() + 21);
    hl.row_audit_ts = ev[21]; hl.col_audit_ts = ev[22];
  }
  mark("  hash_layer_evaluations", th);
  th = std::chrono::steady_clock::now();
  Cp dummy;
  Fq joint;
  {  // DerefsEvalProof::prove (sparse_mlpoly.rs:125-149, prove_single :80-123)
    T.append_protocol_name("Derefs evaluation proof");
    const std::vector<Fq> r_joint = combine_to_one(T, hl, HashOpening::derefs, rand_ops, joint);
    polyeval_prove(ctx, derefs.p, nullptr, r_joint, &joint, nullptr, gens.gens_derefs, T, tape, hl.proof_derefs, dummy);
  }
  mark("  polyeval_derefs(2^23)", th);
  th = std::chrono::steady_clock::now();
  {  // ops decommitment (sparse_mlpoly.rs:766-797)
    const std::vector<Fq> r_joint = combine_to_one(T, hl, HashOpening::ops, rand_ops, joint);
    polyeval_prove(ctx, enc.comb_ops.p, nullptr, r_joint, &joint, nullptr, gens.gens_ops, T, tape, hl.proof_ops, dummy);
  }
  mark("  polyeval_ops(2^24)", th);
  th = std::chrono::steady_clock::now();
  {  // mem decommitment (sparse_mlpoly.rs:799-824)
    const std::vector<Fq> r_joint = combine_to_one(T, hl, HashOpening::mem, rand_mem, joint);
    polyeval_prove(ctx, enc.comb_mem.p, nullptr, r_joint, &joint, nullptr, gens.gens_mem, T, tape, hl.proof_mem, dummy);
  }
  mark("  polyeval_mem(2^22)", th);
  mark("evalproof_layered_network", tn);
  mark("R1CSEvalProof::prove", t_eval);
  mark("SNARK::prove", t_start);
  for (auto& f : ctx.fine) ctx.timings.push_back({"fine:" + f.first, f.second});
  ctx.fine.clear();
}

}  // namespace sp
