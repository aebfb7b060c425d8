// spartan_b200 — host prover for the R1CS satisfiability proof (NIZK path), driving the sm_90a kernels.
// Follows the exact Fiat-Shamir schedule of /root/reference/src/r1csproof.rs:144-349 (SURVEY.md Appendix A) so that the
// proof bytes equal the reference's for identical instance, assignment, transcript label and RandomTape seed.
#include "prover.hpp"
#include "../../include/spartan_b200.h"
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <functional>

namespace sp {

// ================================================================================================ plumbing
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

Ctx::Ctx(int dev_) : device(dev_) {
  if (dev::device_count() <= dev_) throw std::runtime_error("spartan_b200: no CUDA device " + std::to_string(dev_) + " (the prover has no CPU fallback)");
  dev::set_device(dev_);
  stream = dev::stream_create_prio(+1);
  stream2 = dev::stream_create_prio(-1);
  ev_fork = dev::event_create(); ev_join = dev::event_create();
  pinned = (uint8_t*)dev::hmalloc_pinned(layout::PINNED_BYTES);
  if (dev::memcheck_on()) memset(pinned, 0xFF, layout::PINNED_BYTES);   // before the flag words are zeroed
  host_res = reinterpret_cast<u256*>(pinned + layout::PIN_RES.off);
  host_flag = reinterpret_cast<unsigned int*>(pinned + layout::PIN_FLAG.off);
  host_flag_c = reinterpret_cast<unsigned int*>(pinned + layout::PIN_FLAG_C.off);
  *host_flag = 0;
  *host_flag_c = 0;
  sig_done.alloc(layout::SIG_WORDS);
  dev::dzero(sig_done.p, layout::SIG_WORDS * sizeof(unsigned int), stream);
  small.alloc(layout::SMALL_SCALARS);
  dev::fill_one(small.p + layout::SMALL_ONES.off, layout::SMALL_ONES.cap, stream);   // ones()
  scratch.alloc(1 << 20);
  red.alloc(dev::sc_scratch_bytes(dev::SC_MAX_INST));
  dev::dzero(red.p, red.n, stream);
  sync();
}
void Ctx::comm_create() {
  if (comm) return;
  dev::set_device(device);
  comm.reset(new Comm());
  dev::dzero(comm->ticket.p, 16, stream);
  sync();
}
Ctx::~Ctx() {
  try { sync(); } catch (...) {}
  try { dev::stream_sync(stream2); } catch (...) {}
  scratch.release(); scratch2.release(); red.release(); small.release();
  dev::event_destroy(ev_fork); dev::event_destroy(ev_join);
  dev::stream_destroy(stream2);
  if (ev_a) { dev::event_destroy(ev_a); dev::event_destroy(ev_b); }
  dev::hfree_pinned(pinned);
  dev::stream_destroy(stream);
}
void Ctx::memcheck_refill() {
  if (!dev::memcheck_on()) return;
  sync();
  dev::stream_sync(stream2);
  dev::memcheck_fill(scratch.p, scratch.n, dev::FILL_ZERO);
  dev::memcheck_fill(scratch2.p, scratch2.n, dev::FILL_ZERO);
  // all of small but ones(), which nobody writes after Ctx::Ctx (a fill_one here would add a kernel launch to every call)
  dev::memcheck_fill(small.p, layout::SMALL_ONES.off * sizeof(u256), dev::FILL_FF);
  dev::memcheck_fill(small.p + layout::SMALL_ONES.end(), (small.n - layout::SMALL_ONES.end()) * sizeof(u256), dev::FILL_FF);
  for (const layout::Region& r : {layout::PIN_STAGE, layout::PIN_ZKPRE, layout::PIN_RES, layout::PIN_XY}) memset(pinned + r.off, 0xFF, r.cap);
  sync();
  dev::memcheck_count_refill();
}
void Ctx::wait_sig(const dev::HostSig& s) {
  volatile unsigned int* f = s.flag;
  auto t0 = std::chrono::steady_clock::now();
  unsigned long spins = 0;
  while ((int)(*f - s.seq) < 0) {   // sequence numbers only grow (one stream): a later signal also satisfies an earlier wait
    if ((++spins & 0xffff) == 0 && std::chrono::steady_clock::now() - t0 > std::chrono::seconds(5)) {
      sync();   // throws on a CUDA error; otherwise the kernel has finished and the flag must be visible
      if ((int)(*f - s.seq) < 0) throw std::runtime_error("spartan_b200: kernel completed without publishing its result flag");
    }
  }
  std::atomic_thread_fence(std::memory_order_acquire);
}
// ---- communicator
Comm::Comm() {
  win[0] = (uint8_t*)dev::win_alloc(window_bytes());
  ticket.alloc(4);
}
Comm::~Comm() {
  for (int p = 0; p < SP_MAX_RANKS; p++) {
    if (!win[p]) continue;
    if (p == rank) dev::win_free(win[p]); else dev::ipc_close(win[p]);
  }
}
void Comm::connect(int rank_, int world_, const uint8_t* handles) {
  if (connected) throw SpError(SP_ERR_INVALID_ARG, "communicator already connected");
  if (world_ < 1 || world_ > SP_MAX_RANKS || (world_ & (world_ - 1)) || rank_ < 0 || rank_ >= world_) throw SpError(SP_ERR_INVALID_ARG, "sharding needs a power-of-two world of at most 8 ranks");
  uint8_t* own = win[0];
  win[0] = nullptr;
  rank = rank_; world = world_;
  const size_t hb = dev::ipc_handle_bytes();
  for (int p = 0; p < world; p++) win[p] = p == rank ? own : (uint8_t*)dev::ipc_open(handles + (size_t)p * hb);
  connected = true;
}
const uint8_t* Ctx::allgather_block(const void* src, size_t bytes) {
  Comm& c = *comm;
  if ((size_t)c.world * bytes > SP_WIN_HALF_BYTES) throw std::runtime_error("spartan_b200: all-gather larger than the window");
  const size_t off = c.next_half_off();
  dev::push_block(c.devview(), src, bytes, off, c.bseq, c.ticket.p, stream);
  dev::wait_peers(c.devview(), c.bseq, stream);
  return c.win[c.rank] + off;
}
u256* Ctx::allgather_cyclic(const u256* const* tables, int ntables, size_t n_local) {
  Comm& c = *comm;
  if ((size_t)ntables * n_local * c.world * sizeof(u256) > SP_WIN_HALF_BYTES) throw std::runtime_error("spartan_b200: all-gather larger than the window");
  const size_t off = c.next_half_off();
  dev::push_cyclic(c.devview(), tables, ntables, n_local, off, c.bseq, c.ticket.p, stream);
  dev::wait_peers(c.devview(), c.bseq, stream);
  return reinterpret_cast<u256*>(c.win[c.rank] + off);
}

void Ctx::get_small(size_t slot, Fq* v, size_t k) {
  uint8_t* stage = pinned + layout::PIN_STAGE.off;
  dev::d2h(stage, small.p + slot, k * sizeof(u256), stream);
  sync();
  memcpy(v, stage, k * sizeof(u256));
}
void Ctx::upload(u256* d, const Fq* h, size_t n) { dev::h2d(d, h, n * sizeof(u256), stream); sync(); }
std::vector<Fq> Ctx::download(const u256* d, size_t n) {
  std::vector<Fq> v(n);
  dev::d2h(v.data(), d, n * sizeof(u256), stream);
  sync();
  return v;
}

void label_gens(Ctx& c, const std::string& label, size_t n, ge* out, const std::function<void(size_t i0, size_t m, const ge* pts)>& sink) {
  static const uint8_t basepoint[32] = {0xe2, 0xf2, 0xae, 0x0a, 0x6a, 0xbc, 0x4e, 0x71, 0xa8, 0x84, 0xa9, 0x61, 0xc5, 0x00, 0x51, 0x5f,
                                        0x58, 0xe3, 0x0b, 0x6a, 0xa5, 0x82, 0xdd, 0x8d, 0xb6, 0xa6, 0x59, 0x45, 0xe0, 0x8d, 0x2d, 0x76};
  std::vector<uint8_t> seed(label.begin(), label.end());
  seed.insert(seed.end(), basepoint, basepoint + 32);
  Shake256 xof(seed.data(), seed.size());
  const size_t slab = std::min<size_t>((size_t)1 << 18, std::max<size_t>(n, 1));
  std::vector<uint8_t> uni(64 * slab);
  DevBuf<uint8_t> d_uni(uni.size());
  DevBuf<ge> own(out ? 0 : slab);
  for (size_t i0 = 0; i0 < n; i0 += slab) {
    const size_t m = std::min(slab, n - i0);
    ge* pts = out ? out + i0 : own.p;
    xof.squeeze(uni.data(), 64 * m);
    dev::h2d(d_uni.p, uni.data(), 64 * m, c.stream);
    dev::gens_from_uniform(pts, d_uni.p, m, c.stream);
    if (sink) sink(i0, m, pts);
    c.sync();
  }
}
GenSet::GenSet(Ctx* c, const std::string& label_, size_t nbases_, const std::vector<size_t>& host_bases) : ctx(c), label(label_), nbases(nbases_) {
  G.alloc(nbases);
  label_gens(*ctx, label, nbases, G.p, nullptr);
  finish(host_bases);
}
GenSet::GenSet(Ctx* c, const ge* d_points, size_t nbases_, const std::vector<size_t>& host_bases) : ctx(c), label("<uploaded>"), nbases(nbases_) {
  G.alloc(nbases);
  dev::d2d(G.p, d_points, nbases * sizeof(ge), ctx->stream);
  finish(host_bases);
}
void GenSet::finish(const std::vector<size_t>& host_bases) {
  // large sets first get a row table (d * G_j only, 3.1 MB per generator at 16 bits): the big row commitments run on it with 16 additions per
  // term and a doubling tail per row.  It comes first because it serves the largest MSMs; it is skipped only when it would not fit.
  if (nbases >= 512) {
    size_t free_b = 0, total_b = 0;
    dev::mem_info(&free_b, &total_b);
    if ((double)dev::row_table_entries(nbases) * sizeof(ge_niels) <= 0.65 * (double)free_b) {
      row_table.alloc(dev::row_table_entries(nbases));
      dev::build_row_table(row_table.p, G.p, nbases, ctx->stream);
    }
  }
  // the per-window table serves the inner-product rounds and the small commitments.  Large generator sets get 13-bit windows (20 additions per
  // term instead of 32; 7.9 MB of table per generator); SP_MSM_WINDOW=15 trades 26.7 MB per generator for 17 additions per term
  const char* wenv = getenv("SP_MSM_WINDOW");
  if (nbases < 512) wbits = 8;
  else if (wenv) wbits = atoi(wenv);
  else {
    // the widest window whose table fits comfortably in what is free now: 15 bits (17 instead of 20 additions per term) only for sets of >= 2048
    // generators, where the MSM is long enough to pay for tripled tables, and only where memory allows; 8 bits (393 KB per generator) when even
    // the 13-bit table does not fit: the 8194 generators of a 2^22 SNARK take 64 GB at 13 bits
    size_t free_b = 0, total_b = 0;
    dev::mem_info(&free_b, &total_b);
    auto fits = [&](int w) { return (double)dev::table_entries(nbases, w) * sizeof(ge_niels) <= 0.65 * (double)free_b; };
    wbits = nbases >= 2048 && fits(15) ? 15 : (fits(13) ? 13 : 8);
  }
  if (wbits != 8 && wbits != 13 && wbits != 15) throw std::runtime_error("spartan_b200: SP_MSM_WINDOW must be 8, 13 or 15");
  table.alloc(dev::table_entries(nbases, wbits));
  dev::build_tables(table.p, G.p, nbases, wbits, ctx->stream);
  add_host_tables(host_bases);
  ctx->sync();
}
void GenSet::add_host_tables(const std::vector<size_t>& bases) {
  // host copies (8-bit windows) of the few generators the sigma protocols commit against
  std::vector<size_t> hb;
  for (size_t b : bases) if (b < nbases && !has_tab(b) && std::find(hb.begin(), hb.end(), b) == hb.end()) hb.push_back(b);
  if (hb.empty()) return;
  DevBuf<ge> sel(hb.size());
  for (size_t i = 0; i < hb.size(); i++) dev::d2d(sel.p + i, G.p + hb[i], sizeof(ge), ctx->stream);
  DevBuf<ge_niels> small(dev::table_entries(hb.size(), 8));
  dev::build_tables(small.p, sel.p, hb.size(), 8, ctx->stream);
  for (size_t i = 0; i < hb.size(); i++) {
    std::vector<ge_niels> raw(32 * 128);
    dev::d2h(raw.data(), small.p + i * 32 * 128, sizeof(ge_niels) * 32 * 128, ctx->stream);
    ctx->sync();
    HostBaseTable t;
    t.e.resize(32 * 128);
    for (size_t e = 0; e < raw.size(); e++) t.e[e] = to_hniels(raw[e]);
    std::lock_guard<std::mutex> lk(host_mu);
    host_tab.emplace(hb[i], std::move(t));   // a concurrent view may have added the same base: its copy is the same table
  }
}
hge host_commit(const GenSet& gs, const Term* terms, size_t nterms) {
  hge acc = hge_identity();
  for (size_t i = 0; i < nterms; i++) host_fixed_mul_acc(acc, gs.tab(terms[i].base), terms[i].k);
  return acc;
}

size_t R1CSGens::pc_n(size_t num_vars) {
  // R1CSGens::new (r1csproof.rs:68-73) -> PolyCommitmentGens::new(log2 num_vars) (dense_mlpoly.rs:31-35) ->
  // DotProductProofGens::new(2^ceil(ell/2)) = MultiCommitGens::new(n+1).split_at(n) (nizk/mod.rs:414-418)
  const size_t ell = log2_ceil(num_vars);
  return (size_t)1 << (ell - ell / 2);
}
size_t R1CSGens::bases(size_t num_vars) { return std::max<size_t>(pc_n(num_vars) + 2, 5); }   // gens_4 draws 5 points of the same stream
std::vector<size_t> R1CSGens::host_bases(size_t num_vars) { const size_t n = pc_n(num_vars); return {0, 1, 2, 3, 4, n, n + 1}; }

R1CSGens::R1CSGens(const Ctx* ctx, const GenTables& tables, size_t num_vars) : R1CSGens((tables.require(ctx, bases(num_vars), 0), tables.r1cs_sat), num_vars) {}
R1CSGens::R1CSGens(std::shared_ptr<GenSet> s, size_t num_vars) : set(std::move(s)) {
  set->add_host_tables(host_bases(num_vars));
  const size_t n = pc_n(num_vars);
  gens_pc.n = n;
  gens_pc.gens_n = CommitKey{set.get(), 0, n, n + 1};
  gens_pc.gens_1 = CommitKey{set.get(), n, 1, n + 1};
  gens_1 = gens_pc.gens_1;                       // R1CSSumcheckGens::new clones gens_pc.gens.gens_1 (r1csproof.rs:48-58)
  gens_3 = CommitKey{set.get(), 0, 3, 3};        // MultiCommitGens::new(3, label): same SHAKE prefix, h = 4th point
  gens_4 = CommitKey{set.get(), 0, 4, 4};
}

// ================================================================================================ small host protocol pieces
hge commit1(const CommitKey& k, const Fq& x, const Fq& blind) {
  Term t[2] = {{k.off, x}, {k.h, blind}};
  return host_commit(*k.set, t, 2);
}
hge commitv(const CommitKey& k, const std::vector<Fq>& x, const Fq& blind) {
  std::vector<Term> t;
  for (size_t i = 0; i < x.size(); i++) t.push_back({k.off + i, x[i]});
  t.push_back({k.h, blind});
  return host_commit(*k.set, t.data(), t.size());
}
std::vector<Fq> zk_round_weights(const std::vector<Fq>& w, const Fq& r_j, size_t degree) {
  std::vector<Fq> a(degree + 1);
  Fq rpow = Fq::one();
  for (size_t k = 0; k <= degree; k++) {
    a[k] = w[0] * (k == 0 ? Fq::from_u64(2) : Fq::one()) + w[1] * rpow;
    rpow *= r_j;
  }
  return a;
}
void append_claims_phase2(Transcript& T, const std::array<Cp, 4>& c) {
  T.append_point("comm_Az_claim", c[0].b);
  T.append_point("comm_Bz_claim", c[1].b);
  T.append_point("comm_Cz_claim", c[2].b);
  T.append_point("comm_prod_Az_Bz_claims", c[3].b);
}
void append_nizk_head(Transcript& T, const Instance& inst) {
  T.append_protocol_name("Spartan NIZK proof");
  const std::vector<uint8_t>& digest = inst.shape_digest();   // computed here unless the caller supplied its own (r1cs.rs:154-158)
  T.append_message("R1CSShapeDigest", digest.data(), digest.size());
}

KnowledgeProof knowledge_prove(const CommitKey& g, Transcript& T, RandomTape& tape, const Fq& x, const Fq& r, Cp& C_out) {  // nizk/mod.rs:27-52
  T.append_protocol_name("knowledge proof");
  Fq t1 = tape.random_scalar("t1"), t2 = tape.random_scalar("t2");
  C_out = compress(commit1(g, x, r));
  T.append_point("C", C_out.b);
  KnowledgeProof p;
  p.alpha = compress(commit1(g, t1, t2));
  T.append_point("alpha", p.alpha.b);
  Fq c = T.challenge_scalar("c");
  p.z1 = x * c + t1;
  p.z2 = r * c + t2;
  return p;
}
EqualityProof equality_prove(const CommitKey& g, Transcript& T, RandomTape& tape, const Fq& v1, const Fq& s1, const Fq& v2, const Fq& s2, Cp* C1_out,
                             Cp* C2_out) {  // :88-116
  T.append_protocol_name("equality proof");
  Fq r = tape.random_scalar("r");
  Cp C1 = compress(commit1(g, v1, s1)); T.append_point("C1", C1.b);
  Cp C2 = compress(commit1(g, v2, s2)); T.append_point("C2", C2.b);
  if (C1_out) *C1_out = C1;
  if (C2_out) *C2_out = C2;
  EqualityProof p;
  Term t[1] = {{g.h, r}};
  p.alpha = compress(host_commit(*g.set, t, 1));  // r * h
  T.append_point("alpha", p.alpha.b);
  Fq c = T.challenge_scalar("c");
  p.z = c * (s1 - s2) + r;
  return p;
}
ProductProof product_prove(const CommitKey& g, Transcript& T, RandomTape& tape, const Fq& x, const Fq& rX, const Fq& y, const Fq& rY, const Fq& z,
                           const Fq& rZ, Cp& X, Cp& Y, Cp& Z) {  // nizk/mod.rs:159-229
  T.append_protocol_name("product proof");
  Fq b1 = tape.random_scalar("b1"), b2 = tape.random_scalar("b2"), b3 = tape.random_scalar("b3"), b4 = tape.random_scalar("b4"), b5 = tape.random_scalar("b5");
  X = compress(commit1(g, x, rX)); T.append_point("X", X.b);
  Y = compress(commit1(g, y, rY)); T.append_point("Y", Y.b);
  Z = compress(commit1(g, z, rZ)); T.append_point("Z", Z.b);
  ProductProof p;
  p.alpha = compress(commit1(g, b1, b2)); T.append_point("alpha", p.alpha.b);
  p.beta = compress(commit1(g, b3, b4)); T.append_point("beta", p.beta.b);
  // delta = b3*X + b5*h with X = x*G + rX*h (nizk/mod.rs:199-206): same group element as (b3*x)*G + (b3*rX + b5)*h
  p.delta = compress(commit1(g, b3 * x, b3 * rX + b5));
  T.append_point("delta", p.delta.b);
  Fq c = T.challenge_scalar("c");
  p.z = {b1 + c * x, b2 + c * rX, b3 + c * y, b4 + c * rY, b5 + c * (rZ - rX * y)};
  return p;
}
DotProductProof dotproduct_prove(const CommitKey& g1, const CommitKey& gn, Transcript& T, RandomTape& tape, const std::vector<Fq>& x_vec,
                                 const Fq& blind_x, const std::vector<Fq>& a_vec, const Fq& y, const Fq& blind_y, const Cp* Cx_known, const DotPre* pre,
                                 Cp* Cx_out, Cp* Cy_out) {
  T.append_protocol_name("dot product proof");
  size_t n = x_vec.size();
  std::vector<Fq> d_vec = pre ? pre->d_vec : tape.random_vector("d_vec", n);
  Fq r_delta = pre ? pre->r_delta : tape.random_scalar("r_delta"), r_beta = pre ? pre->r_beta : tape.random_scalar("r_beta");
  Cp Cx = Cx_known ? *Cx_known : compress(commitv(gn, x_vec, blind_x));
  T.append_point("Cx", Cx.b);
  Cp Cy = compress(commit1(g1, y, blind_y));
  T.append_point("Cy", Cy.b);
  if (Cx_out) *Cx_out = Cx;
  if (Cy_out) *Cy_out = Cy;
  T.append_scalars("a", a_vec);
  DotProductProof p;
  p.delta = pre ? pre->delta : compress(commitv(gn, d_vec, r_delta));
  T.append_point("delta", p.delta.b);
  Fq dot = Fq::zero();
  for (size_t i = 0; i < n; i++) dot += a_vec[i] * d_vec[i];
  if (pre) { Term t1[1] = {{g1.off, dot}}; p.beta = compress(hge_add(host_commit(*g1.set, t1, 1), pre->r_beta_h)); }
  else p.beta = compress(commit1(g1, dot, r_beta));
  T.append_point("beta", p.beta.b);
  Fq c = T.challenge_scalar("c");
  p.z.resize(n);
  for (size_t i = 0; i < n; i++) p.z[i] = c * x_vec[i] + d_vec[i];
  p.z_delta = c * blind_x + r_delta;
  p.z_beta = c * blind_y + r_beta;
  return p;
}

std::vector<Fq> host_eq_evals(const std::vector<Fq>& r) {  // EqPolynomial::evals (dense_mlpoly.rs:68-84)
  size_t ell = r.size();
  std::vector<Fq> ev((size_t)1 << ell, Fq::one());
  size_t size = 1;
  for (size_t j = 0; j < ell; j++) {
    size *= 2;
    for (size_t i = size - 1;; i -= 2) {
      Fq s = ev[i / 2];
      ev[i] = s * r[j];
      ev[i - 1] = s - ev[i];
      if (i == 1) break;
    }
  }
  return ev;
}

// ================================================================================================ sumcheck rounds on the device
// the tables fold_top binds, in instance order: every set t[k] but a t[2] the instance only reads; with shared_c, that shared C follows once
static std::vector<u256*> owned_tables(const std::vector<dev::ScInst>& insts, bool shared_c) {
  std::vector<u256*> tabs;
  u256* shared = nullptr;
  for (const dev::ScInst& in : insts)
    for (int k = 0; k < 4; k++)
      if (k == 2 && in.c_out != in.t[2]) shared = in.t[2];
      else if (in.t[k]) tabs.push_back(in.t[k]);
  if (shared_c && shared) tabs.push_back(shared);
  return tabs;
}
dev::XRank ScRounds::xr() { return sharded ? ctx.comm->next_xr() : dev::XRank(); }
void ScRounds::eval() {
  sig = ctx.next_sig();
  dev::sc_eval(kind, insts.data(), (int)insts.size(), len, d_out, ctx.red.p, ctx.stream, sig, xr());
}
void ScRounds::fold_eval(const Fq& r, u256* host_bound) {
  if (sharded && len < Ctx::SHARD_MIN_LOCAL) {
    // leave the sharded stage: bind locally, all-gather every table into replicated copies (in the window), evaluate the next round there
    std::vector<u256*> tabs = owned_tables(insts, true);
    dev::fold_top(tabs.data(), (int)tabs.size(), len, r.m, ctx.stream);
    const size_t glen = (len / 2) * (size_t)ctx.shard_world();
    u256* g = ctx.allgather_cyclic(tabs.data(), (int)tabs.size(), len / 2);
    for (dev::ScInst& in : insts) {
      const bool own_c = in.c_out == in.t[2];
      for (int k = 0; k < 4; k++)
        if (in.t[k]) in.t[k] = g + (size_t)(std::find(tabs.begin(), tabs.end(), in.t[k]) - tabs.begin()) * glen;
      if (own_c) in.c_out = in.t[2];
    }
    sharded = false;
    len = glen;
    eval();
    return;
  }
  sig = ctx.next_sig();
  dev::sc_fold_eval(kind, insts.data(), (int)insts.size(), len, r.m, d_out, ctx.red.p, ctx.stream, sig, xr(), host_bound);
  len >>= 1;
  for (dev::ScInst& in : insts) in.t[2] = in.c_out;   // a shared C is read from where it was folded to
}
void ScRounds::fold(const Fq& r) {
  std::vector<u256*> tabs = owned_tables(insts, false);
  dev::fold_top(tabs.data(), (int)tabs.size(), len, r.m, ctx.stream);
  len >>= 1;
}
std::vector<Fq> ScRounds::wait() {
  ctx.wait_sig(sig);
  std::vector<Fq> ev(3 * insts.size());
  memcpy(static_cast<void*>(ev.data()), ctx.host_res + layout::RES_OUT.off, ev.size() * sizeof(u256));
  return ev;
}

std::vector<Fq> ScRounds::finals() {
  const dev::ScInst& in = insts[0];
  int nt = 0;
  while (nt < 4 && in.t[nt]) nt++;
  uint8_t* stage = ctx.pinned + layout::PIN_STAGE.off;
  for (int k = 0; k < nt; k++) dev::d2h(stage + 32 * k, in.t[k], 32, ctx.stream);   // the replicated copies after a shard exit
  ctx.sync();
  std::vector<Fq> f(nt);
  memcpy(static_cast<void*>(f.data()), stage, 32 * nt);
  return f;
}

// The device side of a sumcheck of a caller-defined polynomial: the operations of ScRounds over P (k_scp_eval, k_scp_fold_eval), single GPU
struct ScPolyRounds {
  Ctx& ctx;
  const dev::ScPoly& P;
  size_t len;
  u256* d_out = ctx.small.p + layout::SMALL_ROUND.off;   // the d evaluations of a round
  dev::HostSig sig;
  void eval() { sig = ctx.next_sig(); dev::scp_eval(P, len, d_out, ctx.red.p, ctx.stream, sig); }
  void fold_eval(const Fq& r) { sig = ctx.next_sig(); dev::scp_fold_eval(P, len, r.m, d_out, ctx.red.p, ctx.stream, sig); len >>= 1; }
  void fold(const Fq& r) { dev::fold_top(P.t, P.ntables, len, r.m, ctx.stream); len >>= 1; }
  std::vector<Fq> published(size_t k) {   // the first k results of the last launch
    ctx.wait_sig(sig);
    std::vector<Fq> v(k);
    memcpy(static_cast<void*>(v.data()), ctx.host_res + layout::RES_OUT.off, k * sizeof(u256));
    return v;
  }
  std::vector<Fq> wait() { return published(P.degree); }   // s(0), s(2) .. s(d)
  std::vector<Fq> finals() {   // P.t[k][0] of every table, in one launch
    sig = ctx.next_sig();
    dev::heads(ctx.small.p + layout::SMALL_HEADS.off, P.t, P.ntables, ctx.stream, sig);
    return published(P.ntables);
  }
};

void poly_sumcheck_prove(Ctx& ctx, const dev::ScPoly& P, size_t len, const Fq& claim, size_t num_rounds, Transcript& T, SumcheckInstanceProof& proof,
                         std::vector<Fq>& r, std::vector<Fq>& finals, Fq& e) {
  const size_t d = (size_t)P.degree;
  ScPolyRounds sc{ctx, P, len};
  sc.eval();
  e = claim;
  for (size_t j = 0; j < num_rounds; j++) {
    const std::vector<Fq> ev = sc.wait();
    std::vector<Fq> evals(d + 1);   // s_j(0), s_j(1) = e - s_j(0), s_j(2) .. s_j(d)
    evals[0] = ev[0];
    evals[1] = e - ev[0];
    for (size_t t = 2; t <= d; t++) evals[t] = ev[t - 1];
    UniPoly poly = UniPoly::from_evals(evals);
    poly.append_to_transcript("poly", T);
    const Fq r_j = T.challenge_scalar("challenge_nextround");
    if (j + 1 < num_rounds) sc.fold_eval(r_j);   // bind and evaluate the next round while the host finishes this one
    else sc.fold(r_j);
    e = poly.evaluate(r_j);
    proof.compressed_polys.push_back(poly.compress());
    r.push_back(r_j);
  }
  finals = sc.finals();
}

// ================================================================================================ ZK sumcheck on the device
// prove_quad (sumcheck.rs:428-586) and prove_cubic_with_additive_term (sumcheck.rs:588-776).
// tables: NT device arrays of length 2^num_rounds, folded in place (their first element holds the final evaluation).
// Everything of a ZK sumcheck that depends on the random tape only (RandomTape is independent of the transcript): the blinds of the round polynomials and
// evaluations, the per-round randomness of DotProductProof::prove (nizk/mod.rs:329-331) in the reference's order, and the commitments to them —
//   delta_j = commit(d_vec_j; r_delta_j) and the blind halves blinds_poly[j]*h, blinds_evals[j]*h, r_beta_j*h — in four batched device MSMs.
// enqueue() draws and launches (no synchronisation: the results travel to pinned host memory), finish() converts them once the stream has been synchronised.
// the staging area holds, per round, delta_j's encoding and three points
size_t zk_sumcheck_max_rounds() { return layout::PIN_ZKPRE.cap / (32 + 3 * sizeof(ge)); }
struct ZkPre {
  size_t num_rounds = 0, nco = 0;
  std::vector<Fq> blinds_poly, blinds_evals;
  std::vector<DotPre> pre;
  std::vector<hge> bp_h, be_h;
  DevBuf<u256> d_s, d_b;
  DevBuf<ge> d_pts;
  DevBuf<uint8_t> d_c;
  uint8_t* stage = nullptr;   // pinned: 32*num_rounds encodings, then 3*num_rounds points
  void enqueue(Ctx& ctx, int degree, size_t rounds, const CommitKey& g1, const CommitKey& gn, RandomTape& tape) {
    if (rounds > zk_sumcheck_max_rounds()) throw std::runtime_error("spartan_b200: ZK sumcheck with too many rounds for the staging area");
    num_rounds = rounds; nco = (size_t)degree + 1;
    blinds_poly = tape.random_vector("blinds_poly", num_rounds);
    blinds_evals = tape.random_vector("blinds_evals", num_rounds);
    pre.resize(num_rounds);
    std::vector<Fq> dmat(num_rounds * nco), rdel(num_rounds), rbet(num_rounds);
    for (size_t j = 0; j < num_rounds; j++) {
      pre[j].d_vec = tape.random_vector("d_vec", nco);
      pre[j].r_delta = tape.random_scalar("r_delta");
      pre[j].r_beta = tape.random_scalar("r_beta");
      for (size_t i = 0; i < nco; i++) dmat[j * nco + i] = pre[j].d_vec[i];
      rdel[j] = pre[j].r_delta; rbet[j] = pre[j].r_beta;
    }
    stage = ctx.pinned + layout::PIN_ZKPRE.off;
    d_s.alloc(num_rounds * nco); d_b.alloc(4 * num_rounds); d_pts.alloc(4 * num_rounds); d_c.alloc(32 * num_rounds);
    // pageable sources: the copies snapshot them before returning
    dev::h2d(d_s.p, dmat.data(), dmat.size() * sizeof(u256), ctx.stream);
    dev::h2d(d_b.p, rdel.data(), num_rounds * sizeof(u256), ctx.stream);
    dev::h2d(d_b.p + num_rounds, rbet.data(), num_rounds * sizeof(u256), ctx.stream);
    dev::h2d(d_b.p + 2 * num_rounds, blinds_poly.data(), num_rounds * sizeof(u256), ctx.stream);
    dev::h2d(d_b.p + 3 * num_rounds, blinds_evals.data(), num_rounds * sizeof(u256), ctx.stream);
    if (ctx.scratch.n < dev::msm_scratch_bytes(num_rounds, nco) + 64) ctx.ensure_scratch(dev::msm_scratch_bytes(num_rounds, nco) + 64);
    // each blind term against the h of its own key: gens_1 and gens_n may be different generator sets (the caller's)
    const GenSet &s1 = *g1.set, &sn = *gn.set;
    dev::msm_rows(d_pts.p, sn.table.p, sn.wbits, sn.rows(), d_s.p, nco, num_rounds, nco, d_b.p, gn.h, ctx.scratch.p, ctx.stream);                    // delta_j
    dev::compress_batch(d_c.p, d_pts.p, num_rounds, ctx.stream);
    dev::msm_rows(d_pts.p + num_rounds, s1.table.p, s1.wbits, s1.rows(), d_s.p, 0, num_rounds, 0, d_b.p + num_rounds, g1.h, ctx.scratch.p, ctx.stream);      // r_beta_j * h
    dev::msm_rows(d_pts.p + 2 * num_rounds, sn.table.p, sn.wbits, sn.rows(), d_s.p, 0, num_rounds, 0, d_b.p + 2 * num_rounds, gn.h, ctx.scratch.p, ctx.stream);  // blinds_poly[j] * h
    dev::msm_rows(d_pts.p + 3 * num_rounds, s1.table.p, s1.wbits, s1.rows(), d_s.p, 0, num_rounds, 0, d_b.p + 3 * num_rounds, g1.h, ctx.scratch.p, ctx.stream);  // blinds_evals[j] * h
    dev::d2h(stage, d_c.p, 32 * num_rounds, ctx.stream);
    dev::d2h(stage + 32 * num_rounds, d_pts.p + num_rounds, 3 * num_rounds * sizeof(ge), ctx.stream);
  }
  void finish() {   // the stream must have been synchronised after enqueue()
    bp_h.resize(num_rounds); be_h.resize(num_rounds);
    const ge* pts = reinterpret_cast<const ge*>(stage + 32 * num_rounds);
    for (size_t j = 0; j < num_rounds; j++) {
      memcpy(pre[j].delta.b, stage + 32 * j, 32);
      pre[j].r_beta_h = to_hge(pts[j]); bp_h[j] = to_hge(pts[num_rounds + j]); be_h[j] = to_hge(pts[2 * num_rounds + j]);
    }
    d_s.release(); d_b.release(); d_pts.release(); d_c.release();
  }
};

// The host side of a ZK sumcheck's rounds, shared by both drivers below.  commit(): round j's polynomial from the device's evaluations, comm_poly,
// r_j.  The driver then launches the bind with r_j (fused with the next round's evaluation), and prove() runs the rest of the round — comm_eval, the
// two weights and the DotProductProof — while that kernel runs.
struct ZkRounds {
  const CommitKey &g1, &gn;
  Transcript& T;
  RandomTape& tape;
  const ZkPre& zp;
  ZKSumcheckInstanceProof& proof;
  size_t degree;
  Fq claim_per_round;
  const Fq blind_claim;
  Cp comm_claim_per_round;
  UniPoly poly;
  Cp comm_poly;
  ZkRounds(const CommitKey& g1_, const CommitKey& gn_, Transcript& T_, RandomTape& tape_, const ZkPre& zp_, ZKSumcheckInstanceProof& proof_,
           size_t degree_, const Fq& claim, const Fq& blind_claim_)
      : g1(g1_), gn(gn_), T(T_), tape(tape_), zp(zp_), proof(proof_), degree(degree_), claim_per_round(claim), blind_claim(blind_claim_),
        comm_claim_per_round(compress(commit1(g1_, claim, blind_claim_))) {}
  // ev: s_j(0), s_j(2) .. s_j(degree); s_j(1) = claim - s_j(0)
  Fq commit(size_t j, const Fq* ev) {
    std::vector<Fq> evals = {ev[0], claim_per_round - ev[0]};
    for (size_t t = 2; t <= degree; t++) evals.push_back(ev[t - 1]);
    poly = UniPoly::from_evals(evals);
    std::vector<Term> t;   // commit(coeffs; blinds_poly[j]; gens_n) = sum coeff_i*G_i + (blinds_poly[j]*h)
    for (size_t i = 0; i < poly.coeffs.size(); i++) t.push_back({gn.off + i, poly.coeffs[i]});
    comm_poly = compress(hge_add(host_commit(*gn.set, t.data(), t.size()), zp.bp_h[j]));
    T.append_point("comm_poly", comm_poly.b);
    proof.comm_polys.push_back(comm_poly);
    return T.challenge_scalar("challenge_nextround");
  }
  void prove(size_t j, const Fq& r_j) {
    Fq eval = poly.evaluate(r_j);
    Term te[1] = {{g1.off, eval}};
    Cp comm_eval = compress(hge_add(host_commit(*g1.set, te, 1), zp.be_h[j]));   // eval*G + blinds_evals[j]*h
    T.append_point("comm_claim_per_round", comm_claim_per_round.b);
    T.append_point("comm_eval", comm_eval.b);
    std::vector<Fq> w = T.challenge_vector("combine_two_claims_to_one", 2);
    Fq target = w[0] * claim_per_round + w[1] * eval;
    const Fq& blind_sc = j == 0 ? blind_claim : zp.blinds_evals[j - 1];
    Fq blind = w[0] * blind_sc + w[1] * zp.blinds_evals[j];
    // (the reference also recomputes comm_target from the two decompressed commitments and asserts equality, sumcheck.rs:531/:722;
    //  it is a self-check with no effect on the transcript)
    const std::vector<Fq> a = zk_round_weights(w, r_j, degree);
    proof.proofs.push_back(dotproduct_prove(g1, gn, T, tape, poly.coeffs, zp.blinds_poly[j], a, target, blind, &comm_poly, &zp.pre[j]));
    claim_per_round = eval;
    comm_claim_per_round = comm_eval;
    proof.comm_evals.push_back(comm_claim_per_round);
  }
};

// The ZK sumcheck of degree `degree` over the device side `sc` (ScRounds or ScPolyRounds), its tables bound in place for num_rounds rounds.  The
// tape-only commitments (ZkPre) are enqueued ahead of the first evaluation and converted once the stream has run them; then each round's bind
// (fused with the next round's evaluation) is launched as soon as r_j is drawn, and the host runs the round's sigma protocol while it runs.
// Out: the proof, r, finals = the tables' first entries after the last bind, blind_post = blinds_evals[num_rounds - 1].
template <class Rounds>
static void zk_sumcheck_prove(Ctx& ctx, Rounds& sc, size_t degree, const Fq& claim, const Fq& blind_claim, size_t num_rounds, const CommitKey& g1,
                              const CommitKey& gn, Transcript& T, RandomTape& tape, ZKSumcheckInstanceProof& proof, std::vector<Fq>& r,
                              std::vector<Fq>& finals, Fq& blind_post) {
  ZkPre zp;
  zp.enqueue(ctx, (int)degree, num_rounds, g1, gn, tape);
  sc.eval();
  ctx.sync();
  zp.finish();
  ZkRounds zr(g1, gn, T, tape, zp, proof, degree, claim, blind_claim);
  for (size_t j = 0; j < num_rounds; j++) {
    FineTimer fw(ctx, "zk wait evals");
    const std::vector<Fq> e = sc.wait();
    fw.stop();
    FineTimer fh(ctx, "zk host commit_poly+challenge");
    const Fq r_j = zr.commit(j, e.data());
    if (j + 1 < num_rounds) sc.fold_eval(r_j);
    else sc.fold(r_j);
    fh.stop();
    FineTimer fs(ctx, "zk host sigma (overlaps kernel)");
    zr.prove(j, r_j);
    r.push_back(r_j);
  }
  finals = sc.finals();
  blind_post = zp.blinds_evals[num_rounds - 1];
}

void zk_poly_sumcheck_prove(Ctx& ctx, const dev::ScPoly& P, size_t len, const Fq& claim, const Fq& blind_claim, size_t num_rounds, const CommitKey& g1,
                            const CommitKey& gn, Transcript& T, RandomTape& tape, ZKSumcheckInstanceProof& proof, std::vector<Fq>& r,
                            std::vector<Fq>& finals, Fq& blind_post) {
  ScPolyRounds sc{ctx, P, len};
  zk_sumcheck_prove(ctx, sc, (size_t)P.degree, claim, blind_claim, num_rounds, g1, gn, T, tape, proof, r, finals, blind_post);
}

// One instance of a fixed-kind sumcheck over the nt tables (2^num_rounds entries, bound in place), for R1CS phase one (SC_CUBIC4) and two (SC_QUAD).
// sharded: `tables` are this rank's cyclic shards (length 2^num_rounds / world).  The first rounds then run on the shards — the fused kernels
// exchange their partial sums over NVLink before handing the round's evaluations to the host — until the local tables drop below streaming size;
// the shards are then all-gathered into replicated tables (in the window) and the latency-bound tail runs on every rank alike.
static ScRounds one_instance(Ctx& ctx, dev::ScKind kind, u256* const* tables, int nt, size_t num_rounds, bool sharded) {
  const bool sh = sharded && ctx.shard_world() > 1;
  dev::ScInst inst;
  for (int t = 0; t < 4; t++) inst.t[t] = t < nt ? tables[t] : nullptr;
  inst.c_out = inst.t[2];
  inst.write_c = 1;
  return ScRounds{ctx, kind, {inst}, ((size_t)1 << num_rounds) / (sh ? ctx.shard_world() : 1), sh, ctx.small.p + layout::SMALL_ROUND.off};
}

// ================================================================================================ polynomial commitment / evaluation proof
Cp commit_rows_and_compress(Ctx& ctx, const CommitKey& key, const u256* d_scalars, size_t stride, size_t L, size_t R, const Fq* blinds,
                            std::vector<Cp>& out, const std::function<const Fq*()>& blinds_late) {
  // DensePolynomial::commit_inner (dense_mlpoly.rs:148-177): C_i = (MSM(Z[iR..(i+1)R], G) + blinds[i]*h).compress()
  // blinds_late (instead of blinds): called AFTER the rows' MSM is in flight, so that the host draws the blinds from the random tape (0.8 us per
  // scalar of Keccak) while the device works; the blind terms blinds[i]*h are then a second, tiny launch added onto the rows.
  if (key.off != 0 || R > key.n) throw std::runtime_error("spartan_b200: commit_rows key mismatch");
  const bool blind_on_host = !blinds || blinds[0].is_zero() || key.set->has_tab(key.h);   // the blind term needs the host copy of h's table
  if (L == 1 && R >= 2 && R % 2 == 0 && !blinds_late && ctx.shard_world() == 1 && blind_on_host) {
    // one row (the Cx commitment of DotProductProofLog, nizk/mod.rs:466): a latency problem.  The row's sum reaches the host, which adds the
    // blind term and encodes, instead of a 265-product chain on one GPU thread; the blind term is computed while the kernel runs
    ctx.ensure_scratch(std::max(dev::msm_scratch_bytes(1, R), dev::ipa_msm_scratch_points(R, key.set->wbits) * sizeof(ge)) + 64);
    RowSum row(ctx, *key.set, d_scalars, R);
    hge acc = hge_identity();
    if (blinds && !blinds[0].is_zero()) { Term t[1] = {{key.h, blinds[0]}}; acc = host_commit(*key.set, t, 1); }
    out.resize(1);
    out[0] = compress(hge_add(row.collect(), acc));
    return out[0];
  }
  ctx.ensure_scratch(dev::msm_scratch_bytes(L, R) + 64);
  DevBuf<ge> rows(L), bh;
  DevBuf<u256> d_bl;
  if (blinds) { d_bl.alloc(L); dev::h2d(d_bl.p, blinds, L * sizeof(u256), ctx.stream); }
  DevBuf<uint8_t> comp(32 * L);
  out.resize(L);
  const size_t W = (size_t)ctx.shard_world();
  // rows are independent MSMs over the same generators: when sharded, rank r commits rows [r*L/W, (r+1)*L/W) and the 32-byte encodings are all-gathered
  const bool split = W > 1 && L >= 2 * W && L % W == 0;
  const size_t Lr = split ? L / W : L, row0 = split ? (size_t)ctx.rank() * Lr : 0;
  dev::msm_rows(rows.p, key.set->table.p, key.set->wbits, key.set->rows(), d_scalars + row0 * stride, stride, Lr, R, blinds ? d_bl.p + row0 : nullptr, key.h, ctx.scratch.p, ctx.stream);
  if (!blinds && blinds_late) {
    const Fq* bl = blinds_late();
    d_bl.alloc(L); bh.alloc(Lr);
    dev::h2d(d_bl.p, bl, L * sizeof(u256), ctx.stream);
    dev::msm_rows(bh.p, key.set->table.p, key.set->wbits, key.set->rows(), d_scalars, 0, Lr, 0, d_bl.p + row0, key.h, ctx.scratch.p, ctx.stream);   // blinds[i]*h (rows without generator terms)
    dev::add_points(rows.p, bh.p, Lr, ctx.stream);
  }
  dev::compress_batch(comp.p, rows.p, Lr, ctx.stream);
  if (split) dev::d2h(out.data(), ctx.allgather_block(comp.p, 32 * Lr), 32 * L, ctx.stream);
  else dev::d2h(out.data(), comp.p, 32 * L, ctx.stream);
  ctx.sync();
  return out.empty() ? Cp() : out[0];
}

void append_poly_commitment(Transcript& T, const char* label, const PolyCommitment& c) {  // dense_mlpoly.rs:292-300
  T.append_message(label, "poly_commitment_begin");
  for (auto& p : c.C) T.append_point("poly_commitment_share", p.b);
  T.append_message(label, "poly_commitment_end");
}

void IpaRound::launch(size_t cur) {
  // the dot products ride in the MSM's launch (two extra blocks with their own flag word, host_flag_c, and completion counter)
  sig_c.host_out = ctx.host_res + layout::RES_IPA_C.off; sig_c.flag = ctx.host_flag_c; sig_c.done = ctx.sig_done.p + layout::SIG_DONE_C.off; sig_c.seq = ++ctx.sigc_seq;
  sig_lr = ctx.next_sig();
  sig_lr.host_out = ctx.host_res + layout::RES_POINTS.off;
  dev::ipa_msm(pts, gs.table.p, gs.wbits, a, svec, cur, n, ctx.scratch.p, ctx.sig_done.p + layout::SIG_MSM_TICKET.off, ctx.stream, sig_lr, b,
               ctx.small.p + layout::SMALL_IPA_C.off, sig_c);
}
void IpaRound::wait_c(Fq& c_L, Fq& c_R) {
  ctx.wait_sig(sig_c);
  const u256* c = ctx.host_res + layout::RES_IPA_C.off;
  memcpy(&c_L, c, 32); memcpy(&c_R, c + 1, 32);
}
void IpaRound::wait_LR(ge& L, ge& R) {
  ctx.wait_sig(sig_lr);
  const ge* lr = reinterpret_cast<const ge*>(ctx.host_res + layout::RES_POINTS.off);
  memcpy(&L, lr, sizeof(ge)); memcpy(&R, lr + 1, sizeof(ge));
}
void IpaRound::fold(size_t cur, const Fq& u, const Fq& u_inv) { dev::ipa_fold_update(a, b, svec, cur / 2, n, u.m, u_inv.m, ctx.stream); }

RowSum::RowSum(Ctx& c, const GenSet& gs, const u256* d_x, size_t n_) : ctx(c), n(n_), pts(2) {
  if (n >= 2) {
    sig = ctx.next_sig();
    sig.host_out = ctx.host_res + layout::RES_POINTS.off;
    dev::ipa_msm(pts.p, gs.table.p, gs.wbits, ctx.ones(), d_x, 2, n, ctx.scratch.p, ctx.sig_done.p + layout::SIG_MSM_TICKET.off, ctx.stream, sig);
  } else {
    dev::msm_rows(pts.p, gs.table.p, gs.wbits, gs.rows(), d_x, n, 1, n, nullptr, 0, ctx.scratch.p, ctx.stream);
    dev::d2h(ctx.host_res + layout::RES_POINTS.off, pts.p, sizeof(ge), ctx.stream);
  }
}
hge RowSum::collect() {
  ge p[2];
  if (n < 2) {
    ctx.sync();
    memcpy(&p[0], ctx.host_res + layout::RES_POINTS.off, sizeof(ge));
    return to_hge(p[0]);
  }
  ctx.wait_sig(sig);
  memcpy(p, ctx.host_res + layout::RES_POINTS.off, 2 * sizeof(ge));
  return hge_add(to_hge(p[0]), to_hge(p[1]));
}

// ================================================================================================ DotProductProofLog
// the tape draws of DotProductProofLog::prove (nizk/mod.rs:452-467), in the reference's order
struct DotLogTape { Fq d, r_delta, r_beta; std::vector<std::pair<Fq, Fq>> blinds_vec; };
static DotLogTape dotlog_tape(RandomTape& tape, size_t n) {
  DotLogTape t;
  t.d = tape.random_scalar("d");
  t.r_delta = tape.random_scalar("r_delta");
  t.r_beta = tape.random_scalar("r_delta");  // sic: the reference reuses the label (nizk/mod.rs:459)
  const size_t lg_n = log2_ceil(n);
  std::vector<Fq> v1 = tape.random_vector("blinds_vec_1", lg_n), v2 = tape.random_vector("blinds_vec_2", lg_n);
  for (size_t i = 0; i < lg_n; i++) t.blinds_vec.push_back({v1[i], v2[i]});
  return t;
}
// DotProductProofLog::prove after the reduction (nizk/mod.rs:491-524): g1 = gens_1 (G_1 and h), the reduction's x_hat, a_hat, g_hat and the
// final blind rhat_Gamma (blind_y's share included)
static void dotlog_finish(Transcript& T, const CommitKey& g1, const DotLogTape& t, const Fq& r, const Fq& x_hat, const Fq& a_hat, const hge& g_hat,
                          const Fq& rhat_Gamma, DotProductProofLog& proof) {
  Fq y_hat = x_hat * a_hat;
  // delta = d*g_hat + r_delta*h (gens_hat, nizk/mod.rs:497-505)
  Term th[1] = {{g1.h, t.r_delta}};
  proof.delta = compress(hge_add(hge_scalarmul(t.d.canonical(), g_hat), host_commit(*g1.set, th, 1)));
  T.append_point("delta", proof.delta.b);
  // beta = d*(r*G1) + r_beta*h (gens_1_scaled, nizk/mod.rs:507)
  proof.beta = compress(commit1(g1, t.d * r, t.r_beta));
  T.append_point("beta", proof.beta.b);
  Fq c = T.challenge_scalar("c");
  proof.z1 = t.d + c * y_hat;
  proof.z2 = a_hat * (c * rhat_Gamma + t.r_beta) + t.r_delta;
}

// DotProductProofLog::prove (nizk/mod.rs:440-525) with BulletReductionProof::prove (nizk/bullet.rs:32-132) inlined, Q = r*G_1 and H = h folded into
// host fixed-base terms.  `dv` is the device side of one generator layout (DotLogTable, DotLogFold): it holds x and a (n each, folded in place) and
// runs commit_x, the rounds' setup, each round's launch / wait_c / wait_LR / add_blinds / fold, and finish.  a_canon: the canonical bytes of a, which
// the transcript absorbs while the device computes round 0 (same transcript order as nizk/mod.rs:475-477).
template <class Dev>
static void dotlog_body(Ctx& ctx, Dev& dv, const CommitKey& g1, Transcript& T, RandomTape& tape, const Fq& blind_x, const std::vector<uint8_t>& a_canon,
                        const Fq& y, const Fq& blind_y, DotProductProofLog& proof, Cp& Cx, Cp& Cy) {
  const size_t n = dv.n;
  T.append_protocol_name("dot product proof (log)");
  const DotLogTape t = dotlog_tape(tape, n);
  FineTimer f0(ctx, "dotlog Cx");
  Cx = dv.commit_x(blind_x);
  f0.stop();
  T.append_point("Cx", Cx.b);
  Cy = compress(commit1(g1, y, blind_y));
  T.append_point("Cy", Cy.b);
  Fq r = Fq::zero();
  auto absorb_a = [&]() {
    FineTimer fa(ctx, "dotlog absorb a");
    T.append_scalar_bytes("a", a_canon.data(), n);
    r = T.challenge_scalar("r");
  };
  FineTimer fr(ctx, "dotlog rounds");
  dv.setup(t.blinds_vec);
  // blind_Gamma = blind_x + r*blind_y enters the reduction only through the final blind, which is linear in it: start from blind_x, add r*blind_y after
  Fq blind_final = blind_x;
  BulletReductionProof& bullet = proof.bullet_reduction_proof;
  size_t k = 0;
  for (size_t m = n / 2; m >= 1; m /= 2, k++) {
    FineTimer f1(ctx, "dotlog round launch");
    dv.launch(m);
    f1.stop();
    if (k == 0) absorb_a();
    Fq c_L, c_R;
    ge Lg, Rg;
    FineTimer f2(ctx, "dotlog round wait");
    dv.wait_c(c_L, c_R);
    f2.stop();
    FineTimer f3(ctx, "dotlog round host");
    // + c_L*Q + blind_L*H with Q = r*G_1 (nizk/mod.rs:479-480), H = h   (bullet.rs:83-97), while the
    // table layout's MSM still computes L', R' (its wait counts as host time here)
    const Term tl[1] = {{g1.off, c_L * r}}, tr[1] = {{g1.off, c_R * r}};
    hge hl = host_commit(*g1.set, tl, 1), hr = host_commit(*g1.set, tr, 1);
    dv.add_blinds(k, hl, hr);
    dv.wait_LR(Lg, Rg);
    Cp Lc, Rc;
    compress2(hge_add(to_hge(Lg), hl), hge_add(to_hge(Rg), hr), Lc, Rc);
    T.append_point("L", Lc.b);
    T.append_point("R", Rc.b);
    const Fq u = T.challenge_scalar("u"), u_inv = u.inv();
    f3.stop();
    dv.fold(m, u, u_inv);   // bullet.rs:105-108
    blind_final = blind_final + t.blinds_vec[k].first * u * u + t.blinds_vec[k].second * u_inv * u_inv;  // bullet.rs:111
    bullet.L_vec.push_back(Lc);
    bullet.R_vec.push_back(Rc);
  }
  if (k == 0) absorb_a();
  Fq x_hat, a_hat;
  hge g_hat;
  dv.finish(x_hat, a_hat, g_hat);
  fr.stop();
  dotlog_finish(T, g1, t, r, x_hat, a_hat, g_hat, blind_final + r * blind_y, proof);
}

// The table layout (PolyEvalProof's gens, and DotLogGens up to SP_DOTLOG_TABLE_MAX_N): Cx through commit_rows_and_compress's one-row path, the
// rounds through IpaRound over the unfolded generators and their n running scalars svec (DESIGN.md "IPA without folding G"), every round's
// blind_L*H and blind_R*H in one batched launch up front, and g_hat = <svec, G> at the end.  x, a: device x_vec and a_vec (n each, consumed).
struct DotLogTable {
  Ctx& ctx;
  const PolyCommitmentGens& gens;
  u256 *x, *a;
  size_t n;
  DevBuf<u256> svec, lr, d_bl;
  DevBuf<ge> pts, d_bh;
  std::vector<ge> bh;   // blind_L[k]*H, blind_R[k]*H
  IpaRound rd;
  DotLogTable(Ctx& c, const PolyCommitmentGens& g, u256* x_, u256* a_, size_t n_)
      : ctx(c), gens(g), x(x_), a(a_), n(n_), rd{c, *g.gens_n.set, x_, a_, nullptr, n_, nullptr} {
    if (gens.n != n) throw std::runtime_error("spartan_b200: DotProductProofLog size mismatch");
  }
  Cp commit_x(const Fq& blind_x) {
    std::vector<Cp> cx;
    return commit_rows_and_compress(ctx, gens.gens_n, x, n, 1, n, &blind_x, cx);
  }
  void setup(const std::vector<std::pair<Fq, Fq>>& blinds_vec) {
    const GenSet& gs = *gens.gens_n.set;
    const size_t rounds = blinds_vec.size();
    svec.alloc(n); lr.alloc(2 * n); d_bl.alloc(2 * rounds + 1);
    pts.alloc(2); d_bh.alloc(2 * rounds + 1);
    dev::fill_one(svec.p, n, ctx.stream);
    ctx.ensure_scratch(dev::msm_scratch_bytes(2 * rounds + 2, n) + 64);
    // the blind terms depend on the tape only: rows with no generator terms, just the blind
    bh.resize(2 * rounds);
    if (rounds) {
      std::vector<Fq> bl(2 * rounds);
      for (size_t k = 0; k < rounds; k++) { bl[2 * k] = blinds_vec[k].first; bl[2 * k + 1] = blinds_vec[k].second; }
      dev::h2d(d_bl.p, bl.data(), bl.size() * sizeof(u256), ctx.stream);
      dev::msm_rows(d_bh.p, gs.table.p, gs.wbits, gs.rows(), lr.p, 0, 2 * rounds, 0, d_bl.p, gens.gens_n.h, ctx.scratch.p, ctx.stream);
      dev::d2h(bh.data(), d_bh.p, bh.size() * sizeof(ge), ctx.stream);   // pageable target: completes before the call returns
    }
    rd.svec = svec.p;
    rd.pts = pts.p;
  }
  void launch(size_t m) { rd.launch(2 * m); }
  void wait_c(Fq& c_L, Fq& c_R) { rd.wait_c(c_L, c_R); }
  void wait_LR(ge& L, ge& R) { rd.wait_LR(L, R); }
  void add_blinds(size_t k, hge& hl, hge& hr) { hl = hge_add(hl, to_hge(bh[2 * k])); hr = hge_add(hr, to_hge(bh[2 * k + 1])); }
  void fold(size_t m, const Fq& u, const Fq& u_inv) { rd.fold(2 * m, u, u_inv); }
  void finish(Fq& x_hat, Fq& a_hat, hge& g_hat) {   // g_hat = G_final[0] = <s, G>
    uint8_t* stage = ctx.pinned + layout::PIN_STAGE.off;
    dev::d2h(stage, x, 32, ctx.stream);
    dev::d2h(stage + 32, a, 32, ctx.stream);
    g_hat = RowSum(ctx, *gens.gens_n.set, svec.p, n).collect();
    ctx.sync();   // x_hat, a_hat
    memcpy(&x_hat, stage, 32); memcpy(&a_hat, stage + 32, 32);
  }
};

// ================================================================================================ DotProductProofLog of the caller's vectors
DotLogGens::DotLogGens(Ctx& c, size_t n_, const std::string& label) : ctx(&c), n(n_) {
  if (!folding()) {   // the set sp_pc_gens_create builds for n = 2^k (PolyCommitmentGens::new(2k, label) has this n)
    set.reset(new GenSet(&c, label, n + 2, {n, n + 1}));
    g = pc_gens_view(*set, 2 * log2_ceil(n));
    return;
  }
  // the label's n + 2 points: G[0..n) as niels into pts, G_n and h into the small set
  pts.alloc(n);
  DevBuf<ge> last(2);
  label_gens(c, label, n + 2, nullptr, [&](size_t i0, size_t m, const ge* gbuf) {
    const size_t in_g = i0 < n ? std::min(m, n - i0) : 0;
    dev::points_to_niels(pts.p + i0, gbuf, in_g, c.stream);
    if (m > in_g) dev::d2d(last.p + (i0 + in_g - n), gbuf + in_g, (m - in_g) * sizeof(ge), c.stream);
  });
  set.reset(new GenSet(&c, last.p, 2, {0, 1}));
  g.n = n;
  g.gens_1 = CommitKey{set.get(), 0, 1, 1};
}

std::vector<uint8_t> canonical_bytes(Ctx& ctx, const u256* d_a, size_t n) {
  DevBuf<u256> c(n);
  dev::to_canonical(c.p, d_a, n, ctx.stream);
  std::vector<uint8_t> out(32 * n);
  dev::d2h(out.data(), c.p, 32 * n, ctx.stream);
  ctx.sync();
  return out;
}

hge msm_var_host(Ctx& ctx, const ge_niels* pts, const u256* scalars, size_t n) {
  const dev::PipPlan plan = dev::pip_plan(n, 0);
  DevBuf<uint8_t> scratch(dev::pip_scratch_bytes(plan));
  DevBuf<ge> out(1);
  dev::msm_var(out.p, pts, scalars, plan, scratch.p, ctx.stream);
  ge g;
  dev::d2h(&g, out.p, sizeof(ge), ctx.stream);
  ctx.sync();
  return to_hge(g);
}

// The folding layout (DotLogGens above SP_DOTLOG_TABLE_MAX_N): Cx is one bucket MSM over G[0..n).  The folded vector is kept as G_k = c_k * H_k:
// a round folds H' = H_L + u^2 H_R (dev::dotlog_fold) and c' = c * u^-1, and its MSMs take the scalars c * x.  Halves of at most
// DOTLOG_SEG_MAX_HALF terms run both MSMs as one segmented launch over extended points; longer halves run the bucket MSM over niels points.  The
// blind terms are host fixed-base terms against h, and g_hat = c * H_final[0].  x, a: device x_vec and a_vec (n each, consumed).
struct DotLogFold {
  Ctx& ctx;
  const DotLogGens& gens;
  u256 *x, *a;
  size_t n;
  const std::vector<std::pair<Fq, Fq>>* blinds = nullptr;
  // folded points: niels while the next round's halves take the bucket MSM (n/2 of them at most), extended from there on (and G itself when
  // round 0 already takes the segmented MSM)
  DevBuf<ge_niels> hn;
  DevBuf<ge> hg, pts, seg_tmp;
  DevBuf<u256> w;
  DevBuf<uint8_t> scratch;
  DevBuf<uint32_t> d_seg;   // {0, m, 2m} of every segmented round
  const void* cur = nullptr;
  int fmt = dev::FOLD_NIELS;
  Fq c = Fq::one();
  size_t seg_at = 0;
  uint8_t* stage() const { return ctx.pinned + layout::PIN_STAGE.off; }
  Cp commit_x(const Fq& blind_x) {
    const Term tb[1] = {{gens.g.gens_1.h, blind_x}};
    return compress(hge_add(msm_var_host(ctx, gens.pts.p, x, n), host_commit(*gens.g.gens_1.set, tb, 1)));
  }
  void setup(const std::vector<std::pair<Fq, Fq>>& blinds_vec) {
    const size_t S = DOTLOG_SEG_MAX_HALF;
    blinds = &blinds_vec;
    if (n / 2 > 2 * S) hn.alloc(n / 2);
    hg.alloc(std::min(n, 2 * S)); pts.alloc(2); seg_tmp.alloc(std::min(n, 2 * S));
    w.alloc(n);
    size_t scratch_bytes = 0;
    std::vector<uint32_t> seg;
    for (size_t m = n / 2; m >= 1; m /= 2)
      if (m > S) scratch_bytes = std::max(scratch_bytes, dev::pip_scratch_bytes(dev::pip_plan(m, 0)));
      else seg.insert(seg.end(), {0u, (uint32_t)m, (uint32_t)(2 * m)});
    scratch.alloc(std::max<size_t>(scratch_bytes, 1));
    d_seg.alloc(std::max<size_t>(seg.size(), 1));
    dev::h2d(d_seg.p, seg.data(), seg.size() * sizeof(uint32_t), ctx.stream);
    cur = gens.pts.p;
    if (n / 2 <= S) { dev::niels_to_ge(hg.p, gens.pts.p, n, ctx.stream); cur = hg.p; fmt = dev::FOLD_GE; }
  }
  void launch(size_t m) {
    cudaStream_t s = ctx.stream;
    u256* c_dev = ctx.small.p + layout::SMALL_IPA_C.off;
    dev::dot(c_dev, x, a + m, m, ctx.red.p, s);       // c_L = <x_L, a_R>
    dev::dot(c_dev + 1, x + m, a, m, ctx.red.p, s);   // c_R = <x_R, a_L>
    const bool segmented = m <= DOTLOG_SEG_MAX_HALF;
    dev::dotlog_scalars(w.p, x, m, c.m, segmented, s);   // [c x_R | c x_L]
    if (segmented) {   // pts[0] = c <x_R, H_L> = R', pts[1] = c <x_L, H_R> = L'
      dev::msm_var_segmented(pts.p, static_cast<const ge*>(cur), w.p, d_seg.p + seg_at, 2, 2 * m, seg_tmp.p, s);
      seg_at += 3;
    } else {
      const dev::PipPlan plan = dev::pip_plan(m, 0);
      const ge_niels* H = static_cast<const ge_niels*>(cur);
      dev::msm_var(pts.p, H, w.p, plan, scratch.p, s);
      dev::msm_var(pts.p + 1, H + m, w.p + m, plan, scratch.p, s);
    }
    dev::d2h(stage(), c_dev, 2 * sizeof(u256), s);
    dev::d2h(stage() + 2 * sizeof(u256), pts.p, 2 * sizeof(ge), s);
  }
  void wait_c(Fq& c_L, Fq& c_R) {   // c_L, c_R, R', L' arrive together
    ctx.sync();
    memcpy(&c_L, stage(), 32); memcpy(&c_R, stage() + 32, 32);
  }
  void wait_LR(ge& L, ge& R) { memcpy(&R, stage() + 64, sizeof(ge)); memcpy(&L, stage() + 64 + sizeof(ge), sizeof(ge)); }
  void add_blinds(size_t k, hge& hl, hge& hr) {
    const CommitKey& g1 = gens.g.gens_1;
    host_fixed_mul_acc(hl, g1.set->tab(g1.h), (*blinds)[k].first);
    host_fixed_mul_acc(hr, g1.set->tab(g1.h), (*blinds)[k].second);
  }
  void fold(size_t m, const Fq& u, const Fq& u_inv) {
    dev::ipa_fold_update(x, a, nullptr, m, 2 * m, u.m, u_inv.m, ctx.stream);   // bullet.rs:106-107
    const int out_fmt = m > 2 * DOTLOG_SEG_MAX_HALF ? dev::FOLD_NIELS : dev::FOLD_GE;
    void* out = out_fmt == dev::FOLD_NIELS ? static_cast<void*>(hn.p) : static_cast<void*>(hg.p);
    dev::dotlog_fold(out, out_fmt, cur, fmt, m, (u * u).canonical(), ctx.stream);   // bullet.rs:108 over H
    cur = out;
    fmt = out_fmt;
    c = c * u_inv;
  }
  void finish(Fq& x_hat, Fq& a_hat, hge& g_hat) {   // g_hat = G_final[0] = c * H_final[0]
    dev::d2h(stage(), x, 32, ctx.stream);
    dev::d2h(stage() + 32, a, 32, ctx.stream);
    dev::d2h(stage() + 64, cur, sizeof(ge), ctx.stream);
    ctx.sync();
    ge h0;
    memcpy(&x_hat, stage(), 32); memcpy(&a_hat, stage() + 32, 32); memcpy(&h0, stage() + 64, sizeof(ge));
    g_hat = hge_scalarmul(c.canonical(), to_hge(h0));
  }
};

void dotlog_prove(Ctx& ctx, const DotLogGens& gens, Transcript& T, RandomTape& tape, const u256* d_x, const Fq& blind_x, const u256* d_a, const Fq* y,
                  const Fq& blind_y, DotProductProofLog& proof, Cp& Cx, Cp& Cy, Fq& y_used) {
  const size_t n = gens.n;
  DevBuf<u256> x(n), a(n);   // the caller's vectors are read only: the rounds fold these copies
  dev::d2d(x.p, d_x, n * sizeof(u256), ctx.stream);
  dev::d2d(a.p, d_a, n * sizeof(u256), ctx.stream);
  if (y) y_used = *y;
  else {
    dev::dot(ctx.small.p + layout::SMALL_DOT.off, x.p, a.p, n, ctx.red.p, ctx.stream);
    ctx.get_small(layout::SMALL_DOT.off, &y_used, 1);
  }
  const std::vector<uint8_t> a_canon = canonical_bytes(ctx, a.p, n);
  if (gens.folding()) {
    DotLogFold dv{ctx, gens, x.p, a.p, n};
    dotlog_body(ctx, dv, gens.g.gens_1, T, tape, blind_x, a_canon, y_used, blind_y, proof, Cx, Cy);
  } else {
    DotLogTable dv(ctx, gens.g, x.p, a.p, n);
    dotlog_body(ctx, dv, gens.g.gens_1, T, tape, blind_x, a_canon, y_used, blind_y, proof, Cx, Cy);
  }
}

// PolyEvalProof::prove (dense_mlpoly.rs:312-365).  d_Z: device table of 2^|r| scalars (read-only).
void polyeval_prove(Ctx& ctx, const u256* d_Z, const std::vector<Fq>* blinds_opt, const std::vector<Fq>& r, const Fq* Zr, const Fq* blind_Zr_opt,
                    const PolyCommitmentGens& gens, Transcript& T, RandomTape& tape, PolyEvalProof& proof, Cp& C_Zr, Fq* Zr_out) {
  T.append_protocol_name("polynomial evaluation proof");
  FineTimer fp(ctx, "polyeval pre (eq, bound_rows)");
  size_t ell = r.size(), lv = ell / 2;
  size_t L_size = (size_t)1 << lv, R_size = (size_t)1 << (ell - lv);
  // compute_factored_evals (dense_mlpoly.rs:90-98) on the device; the R half is also needed as canonical bytes (the transcript absorbs a_vec)
  DevBuf<u256> d_r(r.size() + 1), d_L(L_size), d_R(R_size), d_Rc(R_size), d_LZ(R_size), tmp(64 * R_size), eqs(dev::eq_evals_scratch(ell - lv));
  dev::h2d(d_r.p, r.data(), r.size() * sizeof(u256), ctx.stream);
  dev::eq_evals(d_L.p, d_r.p, (int)lv, eqs.p, ctx.stream);
  dev::eq_evals(d_R.p, d_r.p + lv, (int)(ell - lv), eqs.p, ctx.stream);
  dev::to_canonical(d_Rc.p, d_R.p, R_size, ctx.stream);
  std::vector<uint8_t> a_canon(32 * R_size);
  dev::d2h(a_canon.data(), d_Rc.p, 32 * R_size, ctx.stream);
  dev::bound_rows(d_LZ.p, d_Z, d_L.p, L_size, R_size, tmp.p, ctx.stream);  // DensePolynomial::bound (dense_mlpoly.rs:206-213)
  Fq Zr_dev;
  if (!Zr) {   // Z(r) = <bound(Z, L), R>: the bound rows already hold everything Z contributes
    dev::dot(ctx.small.p + layout::SMALL_DOT.off, d_LZ.p, d_R.p, R_size, ctx.red.p, ctx.stream);
    ctx.get_small(layout::SMALL_DOT.off, &Zr_dev, 1);
  }
  const Fq& Zr_used = Zr ? *Zr : Zr_dev;
  if (Zr_out) *Zr_out = Zr_used;
  Fq LZ_blind = Fq::zero();
  if (blinds_opt) {
    std::vector<Fq> Lev = ctx.download(d_L.p, L_size);
    for (size_t i = 0; i < L_size; i++) LZ_blind += (*blinds_opt)[i] * Lev[i];
  }
  ctx.sync();
  Fq blind_Zr = blind_Zr_opt ? *blind_Zr_opt : Fq::zero();
  fp.stop();
  DotLogTable dv(ctx, gens, d_LZ.p, d_R.p, R_size);
  Cp Cx;
  dotlog_body(ctx, dv, gens.gens_1, T, tape, LZ_blind, a_canon, Zr_used, blind_Zr, proof.proof, Cx, C_Zr);
}

// ================================================================================================ the caller's tables (sp_pc_*)
PolyCommitmentGens pc_gens_view(GenSet& set, size_t num_vars) {
  const size_t n = pc_gens_n(num_vars);
  if (set.nbases < n + 2)
    throw SpError(SP_ERR_INVALID_ARG, "PolyCommitmentGens for num_vars = " + std::to_string(num_vars) + " needs " + std::to_string(n + 2) + " generators, the set has " +
                                          std::to_string(set.nbases));
  set.add_host_tables({n, n + 1});
  PolyCommitmentGens g;   // DotProductProofGens::new (nizk/mod.rs:414-418): MultiCommitGens::new(n + 1, label).split_at(n)
  g.n = n;
  g.gens_n = CommitKey{&set, 0, n, n + 1};
  g.gens_1 = CommitKey{&set, n, 1, n + 1};
  return g;
}

// the merge of k tables of 2^m entries gathered into one zero-padded buffer (the shapes whose rows straddle tables: at most 2^12 entries)
static DevBuf<u256> pc_gather(Ctx& ctx, const u256* const* tables, int k, size_t m) {
  const size_t len = (size_t)1 << m, used = (size_t)k * len, total = next_pow2((size_t)k) * len;
  DevBuf<u256> z(total);
  for (int j = 0; j < k; j++) dev::d2d(z.p + j * len, tables[j], len * sizeof(u256), ctx.stream);
  if (total > used) dev::dzero(z.p + used, (total - used) * sizeof(u256), ctx.stream);
  return z;
}

PolyCommitment pc_commit(Ctx& ctx, const PolyCommitmentGens& gens, const u256* const* tables, int k, size_t m, const Fq* blinds) {
  const size_t c = log2_ceil(next_pow2((size_t)k)), ell = m + c, L = (size_t)1 << (ell / 2), R = (size_t)1 << (ell - ell / 2);
  if (gens.n != R) throw SpError(SP_ERR_INVALID_ARG, "poly commit: gens.n != R");
  PolyCommitment comm;
  if (!pc_rows_in_tables(m, c)) {
    DevBuf<u256> merged = pc_gather(ctx, tables, k, m);
    commit_rows_and_compress(ctx, gens.gens_n, merged.p, R, L, R, blinds, comm.C);
    return comm;
  }
  // every row of every table (and the blind-only padding rows) in one launch, reading the tables where they are
  const CommitKey& key = gens.gens_n;
  ctx.ensure_scratch(dev::msm_scratch_bytes(L, R) + 64);
  DevBuf<ge> rows(L);
  DevBuf<u256> d_bl;
  if (blinds) { d_bl.alloc(L); dev::h2d(d_bl.p, blinds, L * sizeof(u256), ctx.stream); }
  dev::TableRows tr;
  for (int j = 0; j < k; j++) tr.t[j] = tables[j];
  tr.ntables = k;
  tr.rows_per_table = ((size_t)1 << m) / R;
  tr.row_len = R;
  dev::msm_rows_tables(rows.p, key.set->table.p, key.set->wbits, key.set->rows(), tr, L, R, blinds ? d_bl.p : nullptr, key.h, ctx.scratch.p, ctx.stream);
  DevBuf<uint8_t> comp(32 * L);
  dev::compress_batch(comp.p, rows.p, L, ctx.stream);
  comm.C.resize(L);
  dev::d2h(comm.C.data(), comp.p, 32 * L, ctx.stream);
  ctx.sync();
  return comm;
}

void pc_eval_prove_joint(Ctx& ctx, const PolyCommitmentGens& gens, const u256* const* tables, int k, const std::vector<Fq>& r, const std::vector<Fq>* blinds_opt,
                         Transcript& T, RandomTape& tape, PolyEvalProof& proof, std::vector<Fq>& evals) {
  const size_t m = r.size(), c = log2_ceil(next_pow2((size_t)k)), ell = m + c, lv = ell / 2;
  DevBuf<u256> d_r(m + 1), d_ev(k);
  dev::h2d(d_r.p, r.data(), m * sizeof(u256), ctx.stream);
  // evals[j] = <rows[j], eq> (dot_many takes 32 tables a launch)
  auto evaluate = [&](const u256* const* rows, const u256* d_eq, size_t n) {
    for (int j0 = 0; j0 < k; j0 += 32) dev::dot_many(d_ev.p + j0, rows + j0, std::min(32, k - j0), d_eq, n, ctx.red.p, ctx.stream);
    evals = ctx.download(d_ev.p, k);
  };
  Fq joint;
  if (!pc_rows_in_tables(m, c)) {
    const size_t len = (size_t)1 << m;
    DevBuf<u256> merged = pc_gather(ctx, tables, k, m), d_eq(len), eqs(dev::eq_evals_scratch(m));
    dev::eq_evals(d_eq.p, d_r.p, (int)m, eqs.p, ctx.stream);
    evaluate(tables, d_eq.p, len);
    const std::vector<Fq> r_joint = combine_to_one(T, evals, r, "evals_ops_val", "challenge_combine_n_to_one", "joint_claim_eval", joint);
    Cp C_Zr;
    polyeval_prove(ctx, merged.p, blinds_opt, r_joint, &joint, nullptr, gens, T, tape, proof, C_Zr);
    return;
  }
  // The merge's row split puts the table index in the top c of its lv row bits, so its left eq factor is eq(ch) (x) eq(r[..lv - c]) and its bound
  // rows are sum_j eq(ch)_j LZ_j with LZ_j = bound(Z_j, eq(r[..lv - c])) (tables past k are zero).  The LZ_j need only r: one pass over the tables
  // gives them, the evaluations <LZ_j, eq(r[lv - c..])> follow, and the challenges only combine k rows of R_J entries.
  const size_t lt = lv - c, Lt = (size_t)1 << lt, RJ = (size_t)1 << (ell - lv);
  DevBuf<u256> d_Lt(Lt), d_R(RJ), eqs(dev::eq_evals_scratch(std::max(lt, ell - lv))), LZs((size_t)k * RJ),
      tmp(std::max(dev::bound_rows_many_scratch(k, Lt, RJ), (size_t)k * RJ));
  dev::eq_evals(d_Lt.p, d_r.p, (int)lt, eqs.p, ctx.stream);
  dev::eq_evals(d_R.p, d_r.p + lt, (int)(ell - lv), eqs.p, ctx.stream);
  dev::bound_rows_many(LZs.p, tables, k, d_Lt.p, Lt, RJ, tmp.p, ctx.stream);
  std::vector<const u256*> lz(k);
  for (int j = 0; j < k; j++) lz[j] = LZs.p + (size_t)j * RJ;
  evaluate(lz.data(), d_R.p, RJ);
  const std::vector<Fq> r_joint = combine_to_one(T, evals, r, "evals_ops_val", "challenge_combine_n_to_one", "joint_claim_eval", joint);
  const std::vector<Fq> eq_ch = host_eq_evals(std::vector<Fq>(r_joint.begin(), r_joint.begin() + c));
  DevBuf<u256> d_eqch(k), d_LZ(RJ), d_Rc(RJ);
  dev::h2d(d_eqch.p, eq_ch.data(), (size_t)k * sizeof(u256), ctx.stream);
  dev::bound_rows(d_LZ.p, LZs.p, d_eqch.p, (size_t)k, RJ, tmp.p, ctx.stream);
  Fq LZ_blind = Fq::zero();
  if (blinds_opt) {
    const std::vector<Fq> Lv = host_eq_evals(std::vector<Fq>(r_joint.begin(), r_joint.begin() + lv));
    for (size_t i = 0; i < Lv.size(); i++) LZ_blind += (*blinds_opt)[i] * Lv[i];
  }
  // the rest of PolyEvalProof::prove (dense_mlpoly.rs:312-365), as polyeval_prove runs it
  T.append_protocol_name("polynomial evaluation proof");
  dev::to_canonical(d_Rc.p, d_R.p, RJ, ctx.stream);
  std::vector<uint8_t> a_canon(32 * RJ);
  dev::d2h(a_canon.data(), d_Rc.p, 32 * RJ, ctx.stream);
  ctx.sync();
  DotLogTable dv(ctx, gens, d_LZ.p, d_R.p, RJ);
  Cp Cx, C_Zr;
  dotlog_body(ctx, dv, gens.gens_1, T, tape, LZ_blind, a_canon, joint, Fq::zero(), proof.proof, Cx, C_Zr);
}

// ================================================================================================ instance
template <class T>
static void up(Ctx* ctx, DevBuf<T>& d, const std::vector<T>& h) { d.alloc(h.size()); dev::h2d(d.p, h.data(), h.size() * sizeof(T), ctx->stream); }
static void up(Ctx* ctx, DevBuf<u256>& d, const std::vector<Fq>& h) { d.alloc(h.size()); dev::h2d(d.p, h.data(), h.size() * sizeof(u256), ctx->stream); }

void Instance::host_coo() const {
  std::lock_guard<std::mutex> lk(host_mu);
  if (host_ready) return;
  for (int m = 0; m < 3; m++) {   // finalize has synchronised the stream that wrote the COO: a blocking copy outside its order is safe
    const SparseMatDev& S = M[m];
    S.row.resize(S.nnz); S.col.resize(S.nnz); S.val.resize(S.nnz);
    dev::d2h_sync(S.row.data(), S.coo_row.p, S.nnz * sizeof(uint32_t));
    dev::d2h_sync(S.col.data(), S.coo_col.p, S.nnz * sizeof(uint32_t));
    dev::d2h_sync(S.val.data(), S.coo_val.p, S.nnz * sizeof(u256));
  }
  host_ready = true;
}
void Instance::upload_coo(Ctx* ctx) {
  for (int m = 0; m < 3; m++) {
    SparseMatDev& S = M[m];
    S.nnz = S.row.size();
    up(ctx, S.coo_row, S.row); up(ctx, S.coo_col, S.col); up(ctx, S.coo_val, S.val);
  }
  host_ready = true;
}

std::vector<uint8_t> Instance::shape_bincode() const {
  // bincode(R1CSShape{num_cons,num_vars,num_inputs,A,B,C}), SparseMatPolynomial{num_vars_x,num_vars_y,M:Vec<{row,col,val}>} (r1cs.rs:19-26, sparse_mlpoly.rs:19-37)
  host_coo();
  Writer w;
  w.u64(num_cons); w.u64(num_vars); w.u64(num_inputs);
  const size_t nx = log2_ceil(num_cons), ny = log2_ceil(2 * num_vars);
  for (int m = 0; m < 3; m++) {
    w.out.reserve(w.out.size() + 24 + 48 * M[m].row.size());
    w.u64(nx); w.u64(ny); w.u64(M[m].row.size());
    for (size_t k = 0; k < M[m].row.size(); k++) { w.u64(M[m].row[k]); w.u64(M[m].col[k]); w.scalar(M[m].val[k]); }
  }
  return std::move(w.out);
}
const std::vector<uint8_t>& Instance::shape_digest() const {
  if (digest.empty()) { std::vector<uint8_t> raw = shape_bincode(); digest = miniz_zlib_level6(raw.data(), raw.size()); }
  return digest;
}

void Instance::finalize(Ctx* ctx) {
  const size_t ncols = 2 * num_vars;
  size_t scratch = 0;
  for (int m = 0; m < 3; m++)
    scratch = std::max(scratch, std::max(dev::compress_scratch_bytes(num_cons, M[m].nnz), dev::compress_scratch_bytes(ncols, M[m].nnz)));
  DevBuf<uint8_t> tmp(scratch);
  for (int m = 0; m < 3; m++) {
    SparseMatDev& S = M[m];
    S.csr_ptr.alloc(num_cons + 1); S.csr_idx.alloc(S.nnz); S.csr_val.alloc(S.nnz);
    S.csc_ptr.alloc(ncols + 1); S.csc_idx.alloc(S.nnz); S.csc_val.alloc(S.nnz);
    dev::build_compressed(S.csr_ptr.p, S.csr_idx.p, S.csr_val.p, num_cons, S.coo_row.p, S.coo_col.p, S.coo_val.p, S.nnz, tmp.p, ctx->stream);
    dev::build_compressed(S.csc_ptr.p, S.csc_idx.p, S.csc_val.p, ncols, S.coo_col.p, S.coo_row.p, S.coo_val.p, S.nnz, tmp.p, ctx->stream);
  }
  ctx->sync();
}

// ================================================================================================ R1CSProof::prove
struct PhaseTimer {
  Ctx& ctx; const char* name; std::chrono::steady_clock::time_point t0;
  PhaseTimer(Ctx& c, const char* n) : ctx(c), name(n), t0(std::chrono::steady_clock::now()) {}
  ~PhaseTimer() { ctx.timings.push_back({name, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count()}); }
};

InstanceMatrices::InstanceMatrices(const Instance& i) : R1csMatrices(i.num_cons, i.num_vars), inst(i) {}
void InstanceMatrices::multiply_vec(Ctx& ctx, const u256* d_z, u256* const outs[3], size_t n, bool sh) const {
  const int W = ctx.shard_world(), rk = ctx.rank();
  for (int m = 0; m < 3; m++) {
    const SparseMatDev& S = inst.M[m];
    if (sh) dev::spmv_cyclic(outs[m], n, rk, W, S.csr_ptr.p, S.csr_idx.p, S.csr_val.p, d_z, ctx.stream);   // this rank's rows
    else dev::spmv(outs[m], n, S.csr_ptr.p, S.csr_idx.p, S.csr_val.p, d_z, ctx.stream);
  }
}
void InstanceMatrices::eval_table(Ctx& ctx, const u256* d_e, const Fq w[3], u256* d_w, u256* out, size_t n, bool sh) const {
  const int W = ctx.shard_world(), rk = ctx.rank();
  DevBuf<u256> eA(n), eB(n), eC(n);
  u256* outs[3] = {eA.p, eB.p, eC.p};
  for (int m = 0; m < 3; m++) {
    const SparseMatDev& S = inst.M[m];
    if (sh) dev::spmv_cyclic(outs[m], n, rk, W, S.csc_ptr.p, S.csc_idx.p, S.csc_val.p, d_e, ctx.stream);   // this rank's columns
    else dev::spmv(outs[m], n, S.csc_ptr.p, S.csc_idx.p, S.csc_val.p, d_e, ctx.stream);
  }
  dev::h2d(d_w, w, 3 * sizeof(u256), ctx.stream);
  dev::lincomb3(out, eA.p, eB.p, eC.p, d_w, n, ctx.stream);
}

void r1cs_prove(Ctx& ctx, const R1csMatrices& mats, const u256* d_vars, const std::vector<Fq>& input, const R1CSGens& gens, Transcript& T,
                RandomTape& tape, R1CSProof& proof, std::vector<Fq>& rx, std::vector<Fq>& ry, const R1csHooks* hooks) {
  PhaseTimer t_all(ctx, "R1CSProof::prove");
  T.append_protocol_name("R1CS proof");
  const size_t num_vars = mats.num_vars, num_cons = mats.num_cons;
  if (!(input.size() < num_vars)) throw std::runtime_error("spartan_b200: |input| + 1 must be at most the number of variables");  // r1csproof.rs:156
  T.append_scalars("input", input);

  const size_t ell = log2_ceil(num_vars);
  const size_t L_size = (size_t)1 << (ell / 2), R_size = (size_t)1 << (ell - ell / 2);
  std::vector<Fq> blinds_vars;
  {
    PhaseTimer t(ctx, "polycommit");
    // dense_mlpoly.rs:193-196; the blinds are the tape's first draw and are made while the rows' MSM already runs
    // (phase one's tape-only commitments are not queued behind the rows' MSM: their small kernels would lengthen this commitment's chain by
    //  what they save phase one, whose rounds are host-bound anyway)
    commit_rows_and_compress(ctx, gens.gens_pc.gens_n, d_vars, R_size, L_size, R_size, nullptr, proof.comm_vars.C,
                             [&]() { blinds_vars = tape.random_vector("poly_blinds", L_size); return blinds_vars.data(); });
    append_poly_commitment(T, "poly_commitment", proof.comm_vars);
  }

  // z = vars || 1 || input || 0...                                          (r1csproof.rs:177-185)
  const size_t zlen = 2 * num_vars;
  DevBuf<u256> d_z(zlen);
  const size_t num_rounds_x = log2_ceil(num_cons), num_rounds_y = log2_ceil(zlen);
  const int W = ctx.shard_world(), rk = ctx.rank(), logW = (int)log2_ceil(W);
  const bool sh1 = ctx.shard_table(num_cons), sh2 = ctx.shard_table(zlen);   // sumcheck tables as cyclic shards (rank r holds the indices = r mod W)
  const size_t n1 = sh1 ? num_cons / W : num_cons, n2 = sh2 ? zlen / W : zlen;
  DevBuf<u256> d_tau(num_cons), d_Az(n1), d_Bz(n1), d_Cz(n1), d_chal(64), eq_small(dev::eq_evals_scratch(std::max(num_rounds_x, num_rounds_y)));
  Fq blind_claim_postsc1;
  std::vector<Fq> claims1;
  {
    PhaseTimer t(ctx, "prove_sc_phase_one");
    dev::d2d(d_z.p, d_vars, num_vars * sizeof(u256), ctx.stream);
    std::vector<Fq> tail(1 + input.size());
    tail[0] = Fq::one();
    for (size_t i = 0; i < input.size(); i++) tail[1 + i] = input[i];
    dev::h2d(d_z.p + num_vars, tail.data(), tail.size() * sizeof(u256), ctx.stream);
    dev::dzero(d_z.p + num_vars + tail.size(), (num_vars - tail.size()) * sizeof(u256), ctx.stream);
    std::vector<Fq> tau = T.challenge_vector("challenge_tau", num_rounds_x);
    dev::h2d(d_chal.p, tau.data(), tau.size() * sizeof(u256), ctx.stream);
    if (sh1) {
      // this rank's slice of eq(tau, .): eq over the leading variables times the factor its low index bits fix; its rows of A z, B z, C z
      dev::eq_evals(d_tau.p, d_chal.p, (int)num_rounds_x - logW, eq_small.p, ctx.stream);
      dev::scale(d_tau.p, shard_eq_scale(tau, W, rk).m, n1, ctx.stream);
    } else {
      dev::eq_evals(d_tau.p, d_chal.p, (int)num_rounds_x, eq_small.p, ctx.stream);
    }
    // inst.multiply_vec (r1cs.rs:268-282)
    u256* const outs[3] = {d_Az.p, d_Bz.p, d_Cz.p};
    mats.multiply_vec(ctx, d_z.p, outs, n1, sh1);
    u256* tabs[4] = {d_tau.p, d_Az.p, d_Bz.p, d_Cz.p};
    ScRounds sc = one_instance(ctx, dev::SC_CUBIC4, tabs, 4, num_rounds_x, sh1);
    zk_sumcheck_prove(ctx, sc, 3, Fq::zero(), Fq::zero(), num_rounds_x, gens.gens_1, gens.gens_4, T, tape, proof.sc_proof_phase1, rx, claims1,
                      blind_claim_postsc1);
  }
  if (hooks && hooks->on_rx) hooks->on_rx(rx);
  const Fq tau_claim = claims1[0], Az_claim = claims1[1], Bz_claim = claims1[2], Cz_claim = claims1[3];
  Fq Az_blind = tape.random_scalar("Az_blind"), Bz_blind = tape.random_scalar("Bz_blind"), Cz_blind = tape.random_scalar("Cz_blind"),
     prod_Az_Bz_blind = tape.random_scalar("prod_Az_Bz_blind");
  Cp comm_Cz_claim, comm_Az_claim, comm_Bz_claim, comm_prod;
  proof.pok_Cz = knowledge_prove(gens.gens_1, T, tape, Cz_claim, Cz_blind, comm_Cz_claim);
  Fq prod = Az_claim * Bz_claim;
  proof.proof_prod = product_prove(gens.gens_1, T, tape, Az_claim, Az_blind, Bz_claim, Bz_blind, prod, prod_Az_Bz_blind, comm_Az_claim, comm_Bz_claim, comm_prod);
  proof.claims_phase2 = {comm_Az_claim, comm_Bz_claim, comm_Cz_claim, comm_prod};
  append_claims_phase2(T, proof.claims_phase2);
  Fq blind_expected_claim_postsc1 = tau_claim * (prod_Az_Bz_blind - Cz_blind);
  Fq claim_post_phase1 = (Az_claim * Bz_claim - Cz_claim) * tau_claim;
  proof.proof_eq_sc_phase1 = equality_prove(gens.gens_1, T, tape, claim_post_phase1, blind_expected_claim_postsc1, claim_post_phase1, blind_claim_postsc1);

  Fq blind_claim_postsc2;
  std::vector<Fq> claims2;
  {
    PhaseTimer t(ctx, "prove_sc_phase_two");
    Fq rabc[3] = {T.challenge_scalar("challenge_Az"), T.challenge_scalar("challenge_Bz"), T.challenge_scalar("challenge_Cz")};
    Fq claim_phase2 = rabc[0] * Az_claim + rabc[1] * Bz_claim + rabc[2] * Cz_claim;
    Fq blind_claim_phase2 = rabc[0] * Az_blind + rabc[1] * Bz_blind + rabc[2] * Cz_blind;
    // evals_rx = eq(rx, .), then the three transposed SpMVs of compute_eval_table_sparse (r1cs.rs:284-298), then r_A*A + r_B*B + r_C*C
    dev::h2d(d_chal.p, rx.data(), rx.size() * sizeof(u256), ctx.stream);
    dev::eq_evals(d_tau.p, d_chal.p, (int)num_rounds_x, eq_small.p, ctx.stream);
    DevBuf<u256> d_ABC(n2), d_zloc;
    mats.eval_table(ctx, d_tau.p, rabc, d_chal.p + 32, d_ABC.p, n2, sh2);
    if (sh2) { d_zloc.alloc(n2); dev::take_cyclic(d_zloc.p, d_z.p, n2, rk, W, ctx.stream); }
    u256* tabs[2] = {sh2 ? d_zloc.p : d_z.p, d_ABC.p};
    ScRounds sc = one_instance(ctx, dev::SC_QUAD, tabs, 2, num_rounds_y, sh2);
    zk_sumcheck_prove(ctx, sc, 2, claim_phase2, blind_claim_phase2, num_rounds_y, gens.gens_1, gens.gens_3, T, tape, proof.sc_proof_phase2, ry, claims2,
                      blind_claim_postsc2);
  }
  if (hooks && hooks->on_ry) hooks->on_ry(ry);
  {
    PhaseTimer t(ctx, "polyeval");
    // eval_vars_at_ry = poly_vars.evaluate(ry[1..]) (dense_mlpoly.rs:236-242)
    std::vector<Fq> ry1(ry.begin() + 1, ry.end());
    DevBuf<u256> d_eq(num_vars);
    dev::h2d(d_chal.p, ry1.data(), ry1.size() * sizeof(u256), ctx.stream);
    dev::eq_evals(d_eq.p, d_chal.p, (int)ry1.size(), eq_small.p, ctx.stream);
    dev::dot(ctx.small.p + layout::SMALL_DOT.off, d_vars, d_eq.p, num_vars, ctx.red.p, ctx.stream);
    Fq eval_vars_at_ry;
    ctx.get_small(layout::SMALL_DOT.off, &eval_vars_at_ry, 1);
    Fq blind_eval = tape.random_scalar("blind_eval");
    polyeval_prove(ctx, d_vars, &blinds_vars, ry1, &eval_vars_at_ry, &blind_eval, gens.gens_pc, T, tape, proof.proof_eval_vars_at_ry, proof.comm_vars_at_ry);
    Fq blind_eval_Z_at_ry = (Fq::one() - ry[0]) * blind_eval;
    Fq blind_expected_claim_postsc2 = claims2[1] * blind_eval_Z_at_ry;
    Fq claim_post_phase2 = claims2[0] * claims2[1];
    proof.proof_eq_sc_phase2 = equality_prove(gens.gens_pc.gens_1, T, tape, claim_post_phase2, blind_expected_claim_postsc2, claim_post_phase2, blind_claim_postsc2);
  }
}

void nizk_prove(Ctx& ctx, const Instance& inst, const u256* d_vars, const std::vector<Fq>& input, const R1CSGens& gens, Transcript& T, const Fq& tape_seed,
                NizkProof& out) {
  ctx.timings.clear();
  ShardScope shard(ctx);
  PhaseTimer t(ctx, "NIZK::prove");
  RandomTape tape("proof", tape_seed);                                   // lib.rs:511
  append_nizk_head(T, inst);
  r1cs_prove(ctx, InstanceMatrices(inst), d_vars, input, gens, T, tape, out.r1cs_sat_proof, out.rx, out.ry);
}

}  // namespace sp
