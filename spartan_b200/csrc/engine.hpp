// spartan_b200 — device context, buffers and generator sets shared by the host prover.
#pragma once
#include <chrono>
#include <cstdlib>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>
#include "dev.hpp"
#include "host.hpp"

namespace sp {

void shake256(uint8_t* out, size_t outlen, const uint8_t* in, size_t inlen);

template <class T>
struct DevBuf {  // owning device allocation
  T* p = nullptr;
  size_t n = 0;
  DevBuf() {}
  explicit DevBuf(size_t count) { alloc(count); }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept { if (this != &o) { release(); p = o.p; n = o.n; o.p = nullptr; o.n = 0; } return *this; }
  ~DevBuf() { release(); }
  void alloc(size_t count) { release(); p = (T*)dev::pool_alloc(count * sizeof(T), dev::pool_fill_of<T>()); n = count; }
  void release() { if (p) dev::pool_free(p); p = nullptr; n = 0; }
};

// Intra-proof sharding (SURVEY.md §8e): this rank's window, the peers' windows mapped through CUDA IPC, and the sequence counters every rank
// advances in lock step (all ranks run the same prover code on the same transcript, so they issue the same collectives in the same order).
struct Comm {
  int world = 1, rank = 0;
  uint8_t* win[SP_MAX_RANKS] = {};     // win[rank]: own allocation; others: cudaIpcOpenMemHandle mappings
  bool connected = false;
  unsigned int xseq = 0, bseq = 0;     // per-round partial-sum exchanges / bulk all-gathers issued so far
  DevBuf<unsigned int> ticket;         // block counter of the push kernels (zeroed once, self-resetting)
  Comm();
  ~Comm();
  Comm(const Comm&) = delete;
  Comm& operator=(const Comm&) = delete;
  static size_t window_bytes() { return SP_WIN_CTRL_BYTES + 2 * SP_WIN_HALF_BYTES; }
  void export_handle(uint8_t* out) const { dev::ipc_export(win[rank], out); }   // valid before connect(): rank is 0 then, win[0] is the own window
  void connect(int rank_, int world_, const uint8_t* handles);                   // handles: world x ipc_handle_bytes(), in rank order
  dev::XRank next_xr() {
    dev::XRank x; x.world = world; x.rank = rank; x.seq = ++xseq;
    for (int p = 0; p < world; p++) x.win[p] = reinterpret_cast<dev::WinCtrl*>(win[p]);
    return x;
  }
  dev::CommDev devview() const { dev::CommDev c; c.world = world; c.rank = rank; for (int p = 0; p < world; p++) c.win[p] = win[p]; return c; }
  // data half of the next bulk all-gather (alternating: a half is reused only after every rank has passed the collective in between)
  size_t next_half_off() { ++bseq; return SP_WIN_CTRL_BYTES + (size_t)(bseq & 1) * SP_WIN_HALF_BYTES; }
};

// Layout of the context's fixed scratch buffers: Ctx::small, Ctx::pinned (host_res and the flag words lie inside it) and Ctx::sig_done.  A region
// is an offset and a capacity in its buffer's unit, and this is the one place to add one: the asserts keep the regions of a buffer apart and
// inside it, and every capacity at the worst case its users reach.  Regions marked "shared" serve several users on purpose: those all run on the
// prover's stream and each reads its result back before the next is enqueued, so no two of them are ever in flight together.
namespace layout {
struct Region { size_t off, cap; constexpr size_t end() const { return off + cap; } };
// Ctx::small (device memory), in scalars
constexpr size_t SMALL_SCALARS = 4096;
constexpr Region SMALL_ROUND{0, 8};      // shared: a sumcheck round's evaluations, 3 of one instance (ZK sumcheck, sp_sumcheck_*) or one per degree (poly_sumcheck_prove)
constexpr Region SMALL_HEADS{8, 8};      // the final table heads of poly_sumcheck_prove
constexpr Region SMALL_IPA_C{16, 16};    // c_L, c_R of an inner-product round
constexpr Region SMALL_DOT{32, 8};       // shared: one dot product (r1cs_prove, sp_dot, sp_poly_evaluate)
constexpr Region SMALL_ABC{40, 8};       // the matrices at (rx, ry) (sparse_evaluate)
constexpr Region SMALL_DOTP{48, 16};     // the two halves of a dot-product circuit's claim (snark_prove)
constexpr Region SMALL_BATCH{64, 128};   // shared: batched_prove's 3 evaluations per instance; after it, spark_eval_prove's 7b + 2 hash-layer evaluations;
                                         // before it, prod_build's two half sums per dot product
constexpr Region SMALL_ONES{4000, 2};    // Ctx::ones()
// Ctx::pinned (mapped host memory), in bytes
constexpr size_t PINNED_BYTES = 1 << 20;
constexpr size_t PIN_XY_PART = 4096;
constexpr Region PIN_STAGE{0, 4096};                // shared: small copies to the host, each synchronised and read at once (get_small, a_hat | b_hat, the ZK sumcheck's
                                                    // final table heads, the two last-layer entries of each of batched_prove's product circuits)
constexpr Region PIN_ZKPRE{384 << 10, 96 << 10};    // ZkPre's encodings and points, read when its sumcheck starts
constexpr Region PIN_RES{512 << 10, 256 << 10};     // Ctx::host_res: what kernels publish through dev::HostSig (the RES_ regions)
constexpr Region PIN_FLAG{768 << 10, 64};           // Ctx::host_flag: the flag word of next_sig(), on a cache line of its own
constexpr Region PIN_FLAG_C{PIN_FLAG.end(), 64};    // Ctx::host_flag_c: the second flag word of an inner-product round, likewise
constexpr Region PIN_XY{960 << 10, 2 * PIN_XY_PART};   // snark_prove's equalized rx | ry, read by the background stream: PIN_XY_PART bytes each
// Ctx::host_res, in scalars
constexpr Region RES_OUT{0, 512};        // shared by the users of next_sig(): a sumcheck round's evaluations (3 per instance, batched_prove's 6 bound entries per
                                         // instance behind them) and the values of dev::heads
constexpr Region RES_IPA_C{0, 2};        // c_L, c_R of an inner-product round; inside RES_OUT, like RES_POINTS: no sumcheck runs during an inner-product argument
constexpr Region RES_POINTS{8, 8};       // shared: L', R' of an inner-product round, in flight together with RES_IPA_C, and RowSum's one or two points
// Ctx::sig_done (device memory), in words
constexpr size_t SIG_WORDS = 4;
constexpr Region SIG_DONE{0, 1};         // completion counter of next_sig()
constexpr Region SIG_MSM_TICKET{1, 1};   // block ticket of dev::ipa_msm
constexpr Region SIG_DONE_C{2, 1};       // completion counter of the second flag word

#define SP_APART(a, b) static_assert(a.end() <= b.off, #a " runs into " #b)
#define SP_HOLDS(a, n) static_assert(size_t(n) <= a.cap, #a " cannot hold " #n)
SP_APART(SMALL_ROUND, SMALL_HEADS); SP_APART(SMALL_HEADS, SMALL_IPA_C); SP_APART(SMALL_IPA_C, SMALL_DOT); SP_APART(SMALL_DOT, SMALL_ABC);
SP_APART(SMALL_ABC, SMALL_DOTP); SP_APART(SMALL_DOTP, SMALL_BATCH); SP_APART(SMALL_BATCH, SMALL_ONES);
static_assert(SMALL_ONES.end() <= SMALL_SCALARS, "SMALL_ONES ends outside Ctx::small");
SP_HOLDS(SMALL_ROUND, 3); SP_HOLDS(SMALL_ROUND, SP_SC_MAX_DEGREE); SP_HOLDS(SMALL_HEADS, SP_SC_MAX_TABLES); SP_HOLDS(SMALL_IPA_C, 2); SP_HOLDS(SMALL_DOT, 1);
SP_HOLDS(SMALL_ABC, SP_SPARK_MAX_BATCH); SP_HOLDS(SMALL_DOTP, 2); SP_HOLDS(SMALL_BATCH, 3 * dev::SC_MAX_INST); SP_HOLDS(SMALL_BATCH, 7 * SP_SPARK_MAX_BATCH + 2); SP_HOLDS(SMALL_BATCH, 2 * dev::PROD_MAX_DOTP); SP_HOLDS(SMALL_ONES, 2);
SP_APART(PIN_STAGE, PIN_ZKPRE); SP_APART(PIN_ZKPRE, PIN_RES); SP_APART(PIN_RES, PIN_FLAG); SP_APART(PIN_FLAG, PIN_FLAG_C); SP_APART(PIN_FLAG_C, PIN_XY);
static_assert(PIN_XY.end() <= PINNED_BYTES, "PIN_XY ends outside Ctx::pinned");
SP_HOLDS(PIN_STAGE, SMALL_BATCH.cap * sizeof(u256));   // get_small of any whole region of Ctx::small
SP_HOLDS(PIN_STAGE, 2 * sizeof(u256) * dev::SC_MAX_INST); SP_HOLDS(PIN_STAGE, 4 * sizeof(u256));   // batched_prove's entries; a ZK sumcheck's 4 tables
SP_HOLDS(PIN_STAGE, 2 * sizeof(u256) * SP_PROD_MAX_CIRCUITS);   // prod_build's two last-layer entries per circuit and two half sums per dot product
SP_HOLDS(PIN_RES, RES_OUT.end() * sizeof(u256));
SP_APART(RES_IPA_C, RES_POINTS);
static_assert(RES_POINTS.end() <= RES_OUT.end(), "RES_POINTS ends outside RES_OUT");
SP_HOLDS(RES_OUT, (3 + 6) * dev::SC_MAX_INST); SP_HOLDS(RES_OUT, 3 * dev::SC_MAX_INST /* batched_prove's heads: two per product instance, three per dot-product instance */); SP_HOLDS(RES_OUT, 2 * 2 * (2 + 2 * SP_SPARK_MAX_BATCH) /* spark_eval_prove heads */); SP_HOLDS(RES_POINTS, 2 * sizeof(ge) / sizeof(u256));
SP_APART(SIG_DONE, SIG_MSM_TICKET); SP_APART(SIG_MSM_TICKET, SIG_DONE_C);
static_assert(SIG_DONE_C.end() <= SIG_WORDS, "SIG_DONE_C ends outside Ctx::sig_done");
#undef SP_APART
#undef SP_HOLDS
}  // namespace layout

struct Ctx {
  int device = 0;
  std::unique_ptr<Comm> comm;          // null: single-GPU context
  int world() const { return comm && comm->connected ? comm->world : 1; }
  int rank() const { return comm && comm->connected ? comm->rank : 0; }
  // all-gather helpers (no-ops' worth of work when world() == 1 is the caller's business: they require a connected communicator)
  // every rank contributes `bytes` from device memory `src`; returns a device pointer (inside the own window) to world x bytes, rank-major
  const uint8_t* allgather_block(const void* src, size_t bytes);
  // every rank contributes `ntables` tables of n_local elements (cyclic shards); returns the window copy: table t = ptr + t*n_local*world, global order
  u256* allgather_cyclic(const u256* const* tables, int ntables, size_t n_local);
  void comm_create();                  // allocate the window (idempotent); connect through comm->connect
  // Sharding is switched on per prove call (ShardScope): operator-level entry points stay single-GPU even on a connected context, because a
  // collective needs every rank to make the same call.
  bool sharding = false;
  bool shard_enabled = true;           // sp_comm_set_enabled: a connected context can also prove on its own GPU only (every rank must agree)
  int shard_world() const { return sharding ? world() : 1; }
  // a table of `global_len` elements is worth sharding when every rank keeps at least one streaming-size fused round (see sc_fold_eval)
  static constexpr size_t SHARD_MIN_LOCAL = 8192;
  bool shard_table(size_t global_len) const { return shard_world() > 1 && global_len >= 2 * SHARD_MIN_LOCAL * (size_t)shard_world(); }
  cudaStream_t stream = nullptr;       // the prover's stream (greatest priority: its kernels are short and the transcript waits for each of them)
  // background stream (least priority) for throughput work whose inputs are known early and whose result the transcript needs late: the commitment
  // to the dereferenced SPARK values runs there under the second sumcheck phase and the witness evaluation proof (snark.cpp)
  cudaStream_t stream2 = nullptr;
  bool overlap = true;                 // sp_ctx_set_overlap: 0 keeps every kernel on the prover's stream (profiling: per-kernel event times free of concurrent work)
  void* ev_fork = nullptr; void* ev_join = nullptr;
  DevBuf<uint8_t> scratch2;        // MSM partial sums of the background stream
  uint8_t* pinned = nullptr;       // small host<->device exchanges (layout::PIN_*)
  DevBuf<uint8_t> scratch;         // MSM partial sums (growable)
  DevBuf<uint8_t> red;             // reduction tickets + per-block partials (fixed size, tickets zeroed once and self-resetting)
  DevBuf<u256> small;              // challenges, results (device side: layout::SMALL_*)
  const u256* ones() const { return small.p + layout::SMALL_ONES.off; }   // two Montgomery ones
  std::string last_error;
  // per-phase timers (profile feature of the reference, src/timer.rs): label -> milliseconds of the last prove
  std::vector<std::pair<std::string, double>> timings;
  std::map<std::string, double> fine;   // accumulated sub-phase timers (SP_FINE_TIMERS=1), flushed into `timings` by the prove entry points

  void* ev_a = nullptr; void* ev_b = nullptr; bool timer_running = false;   // sp_timer_start / sp_timer_stop_ms
  explicit Ctx(int dev);
  ~Ctx();
  // host-polled kernel results (mapped pinned memory): see dev::HostSig
  u256* host_res = nullptr;
  unsigned int* host_flag = nullptr;
  unsigned int* host_flag_c = nullptr;   // second flag word: the dot products fused into the inner-product MSM launch
  DevBuf<unsigned int> sig_done;
  unsigned int sig_seq = 0;
  unsigned int sigc_seq = 0;           // sequence of the second flag word
  dev::HostSig next_sig() {
    dev::HostSig s; s.host_out = host_res + layout::RES_OUT.off; s.flag = host_flag; s.done = sig_done.p + layout::SIG_DONE.off; s.seq = ++sig_seq; return s;
  }
  void wait_sig(const dev::HostSig& s);   // spins on the flag; falls back to a stream synchronise to surface CUDA errors
  void sync() { dev::stream_sync(stream); }
  void ensure_scratch(size_t bytes) { if (scratch.n < bytes) { sync(); scratch.alloc(bytes); } }
  // memory-check mode (dev::memcheck_on): refill the scratch that persists between calls, at the start of every device entry point, as the
  // allocator fills a block it hands out: scratch and scratch2 zero, small 0xFF (all but ones()), the pinned staging regions 0xFF.  The flag
  // words, sig_done and the tickets in red keep their contract (zero or self-resetting) and are not touched.
  void memcheck_refill();
  void get_small(size_t slot, Fq* v, size_t k);  // download k scalars from small[slot..]; synchronises
  void upload(u256* d, const Fq* h, size_t n);
  std::vector<Fq> download(const u256* d, size_t n);
};

struct ShardScope {   // RAII: sharded proving for the duration of one prove call on a connected context
  Ctx& ctx; bool prev;
  explicit ShardScope(Ctx& c) : ctx(c), prev(c.sharding) { c.sharding = c.world() > 1 && c.shard_enabled; }
  ~ShardScope() { ctx.sharding = prev; }
};
// eq(r, j*W + rank) = c * eq(r[0 .. ell-log2 W), j): the factor contributed by the last log2(W) variables, which the rank fixes
inline Fq shard_eq_scale(const std::vector<Fq>& r, int W, int rank) {
  const int logW = (int)log2_ceil(W);
  Fq c = Fq::one();
  for (int k = 0; k < logW; k++) {
    const Fq& rj = r[r.size() - logW + k];
    c *= ((rank >> (logW - 1 - k)) & 1) ? rj : Fq::one() - rj;
  }
  return c;
}

// One SHAKE256 generator stream (a `label` of MultiCommitGens::new, commitments.rs:15-33) expanded to `nbases` points,
// with the fixed-base window table on the device and host copies of the tables of a few named bases.
struct FineTimer {  // host wall-clock accumulator for latency hunting; a no-op unless SP_FINE_TIMERS is set
  Ctx& ctx; const char* name; std::chrono::steady_clock::time_point t0; bool on;
  static bool enabled() { static const bool e = getenv("SP_FINE_TIMERS") != nullptr; return e; }
  FineTimer(Ctx& c, const char* n) : ctx(c), name(n), on(enabled()) { if (on) t0 = std::chrono::steady_clock::now(); }
  void stop() { if (on) { ctx.fine[name] += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(); on = false; } }
  ~FineTimer() { stop(); }
};

// The device tables never change once built: views (GenTables) hand out raw pointers into them.  Only the host copies grow, when a view needs
// the copy of a base no earlier view needed; they are added under `host_mu` and never removed, so a reference from tab() stays valid.
struct GenSet {
  Ctx* ctx;
  std::string label;
  size_t nbases;
  DevBuf<ge> G;
  DevBuf<ge_niels> table;
  int wbits = 8;               // window width of `table` (host copies are always 8-bit)
  DevBuf<ge_niels> row_table;  // d * G_j for the row MSM of large sets (dev::build_row_table); empty for small sets
  const ge_niels* rows() const { return row_table.n ? row_table.p : nullptr; }
  GenSet(Ctx* c, const std::string& label, size_t nbases, const std::vector<size_t>& host_bases);
  GenSet(Ctx* c, const ge* d_points, size_t nbases, const std::vector<size_t>& host_bases);   // caller-supplied generators (device array)
  void finish(const std::vector<size_t>& host_bases);   // window tables + host copies, once G is filled
  // host copies of the bases < nbases among `bases` that have none yet, built on ctx's stream through staging buffers that are freed on return
  void add_host_tables(const std::vector<size_t>& bases);
  const HostBaseTable& tab(size_t base) const {
    std::lock_guard<std::mutex> lk(host_mu);
    auto it = host_tab.find(base);
    if (it == host_tab.end()) throw std::runtime_error("spartan_b200: no host table for generator " + std::to_string(base));
    return it->second;
  }
  bool has_tab(size_t base) const { std::lock_guard<std::mutex> lk(host_mu); return host_tab.count(base) != 0; }
  size_t device_bytes() const { return G.n * sizeof(ge) + (table.n + row_table.n) * sizeof(ge_niels); }
 private:
  std::map<size_t, HostBaseTable> host_tab;
  mutable std::mutex host_mu;
};

// Generator tables sized once for the largest circuit a caller proves (sp_gen_tables): the "gens_r1cs_sat" set and, when SPARK sizes are given, the
// "gens_r1cs_eval" set.  MultiCommitGens::new(n, label) of any n is a prefix of the label's SHAKE stream (commitments.rs:15-33), so every
// R1CSGens / SnarkGens for a circuit up to those sizes is a view into them, holding a reference to the sets it uses.
struct GenTables {
  Ctx* ctx;
  std::shared_ptr<GenSet> r1cs_sat, r1cs_eval;   // r1cs_eval: null when num_nz_entries was 0
  // set sizes (R1CSGens::bases, SparkDims::bases) and build order (R1CS first) as the private gens of one circuit have always used
  GenTables(Ctx* ctx, size_t num_cons, size_t num_vars, size_t num_inputs, size_t num_nz_entries);
  // SpError(SP_ERR_INVALID_ARG) unless a view on `c` fits: r1cs_bases of gens_r1cs_sat and (eval_bases > 0) eval_bases of gens_r1cs_eval
  void require(const Ctx* c, size_t r1cs_bases, size_t eval_bases) const;
};

// A MultiCommitGens view (commitments.rs:8-12): G = set.G[off .. off+n), h = set.G[h]
struct CommitKey {
  const GenSet* set = nullptr;
  size_t off = 0, n = 0, h = 0;
};

struct Term { size_t base; Fq k; };
// sum of k_i * G_{base_i} over host tables
hge host_commit(const GenSet& gs, const Term* terms, size_t nterms);

}  // namespace sp
