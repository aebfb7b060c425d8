// spartan_b200 — hand-written sm_90a kernels for the Spartan prover hot path.
//
// Kernel families (SURVEY.md §2b):
//   K1/K2  sc_eval / sc_fold_eval / fold_top : dense-multilinear sumcheck rounds
//          (reference loops: /root/reference/src/sumcheck.rs:460-469, :204-228, :296-355, :625-652 and
//           src/dense_mlpoly.rs:215-223).  Streaming scans: 128-bit coalesced loads, per-thread field accumulators,
//           warp-shuffle + shared-memory segmented reduction, last-block finalisation (no second launch).
//   K3/K4  msm_rows : Pedersen commitments sum_j s_j*G_j (+ blind*h) for L rows sharing one generator set
//          (reference: dalek vartime_multiscalar_mul behind src/group.rs:98-117, called from src/commitments.rs:80-92 and
//           src/dense_mlpoly.rs:165-177).  Generators are fixed per `Gens`, so the kernel is a fixed-base comb: 8-bit signed
//           windows, 128-entry affine-niels tables per (generator, window) resident in HBM, 7M mixed additions.  Many long rows
//           use 16-bit row tables (d * G_j only) instead: per-window sums, then a doubling tail per row.
//   K6     compress_batch / decompress_batch / gens_from_uniform (RFC 9496).
//   K7     eq_evals, dot, bound_rows, lincomb3, hadamard, spmv, SPARK hash layer, IPA helpers.
// All arithmetic is exact 256-bit integer work on the INT32 pipe; no tensor-core formulation exists (DESIGN.md).
#include <cuda_runtime.h>
#include <algorithm>
#include <stdexcept>
#include <string>
#include <map>
#include <mutex>
#include <atomic>
#include <vector>
#include "dev.hpp"
#include "kcommon.cuh"
#include "quad.cuh"

namespace sp {
namespace dev {

std::atomic<unsigned long long> g_launches{0};
unsigned long long launch_count() { return g_launches.load(); }
static std::atomic<unsigned long long> g_h2d{0}, g_d2h{0};
void io_bytes(unsigned long long* h2d_b, unsigned long long* d2h_b) { *h2d_b = g_h2d.load(); *d2h_b = g_d2h.load(); }

// ---- per-kernel-family CUDA-event profiler (bench.py roofline leg).  Off by default: one branch per wrapper.
bool g_prof = false;
std::vector<ProfRec> g_recs;
static std::vector<cudaEvent_t> g_event_pool;
cudaEvent_t prof_event() {
  if (!g_event_pool.empty()) { cudaEvent_t e = g_event_pool.back(); g_event_pool.pop_back(); return e; }
  cudaEvent_t e; cudaEventCreate(&e); return e;
}
void prof_enable(bool on) {
  g_prof = on;
  for (auto& r : g_recs) { g_event_pool.push_back(r.a); g_event_pool.push_back(r.b); }
  g_recs.clear();
}
// "name:launches:total_ms:total_algorithmic_bytes:largest_launch_bytes:largest_launch_ms;" per family, after a device synchronise
std::string prof_report() {
  cudaDeviceSynchronize();
  struct Agg { double ms = 0, bytes = 0, big_bytes = 0, big_ms = 0; unsigned long long n = 0; };
  std::vector<std::pair<std::string, Agg>> aggs;
  for (auto& r : g_recs) {
    float ms = 0;
    cudaEventElapsedTime(&ms, r.a, r.b);
    size_t k = 0;
    for (; k < aggs.size(); k++) if (aggs[k].first == r.name) break;
    if (k == aggs.size()) aggs.push_back({r.name, Agg()});
    aggs[k].second.ms += ms; aggs[k].second.bytes += r.bytes; aggs[k].second.n++;
    if (r.bytes > aggs[k].second.big_bytes) { aggs[k].second.big_bytes = r.bytes; aggs[k].second.big_ms = ms; }
  }
  std::string out;
  for (auto& a : aggs)
    out += a.first + ":" + std::to_string(a.second.n) + ":" + std::to_string(a.second.ms) + ":" + std::to_string(a.second.bytes) + ":" +
           std::to_string(a.second.big_bytes) + ":" + std::to_string(a.second.big_ms) + ";";
  return out;
}

void ck(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw CudaError(std::string("spartan_b200 CUDA error in ") + what + ": " + cudaGetErrorString(e));
}
void check(const char* what) { ck(cudaGetLastError(), what); }
int device_count() { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; } return n; }
void set_device(int d) { ck(cudaSetDevice(d), "cudaSetDevice"); }
// level > 0: the device's greatest priority (the transcript-serialised stream of small kernels), level < 0: its least (background MSMs)
cudaStream_t stream_create_prio(int level) {
  int least = 0, greatest = 0;
  ck(cudaDeviceGetStreamPriorityRange(&least, &greatest), "cudaDeviceGetStreamPriorityRange");
  cudaStream_t s;
  ck(cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, level > 0 ? greatest : (level < 0 ? least : (least + greatest) / 2)), "cudaStreamCreateWithPriority");
  return s;
}
void stream_wait_event(cudaStream_t s, void* ev) { ck(cudaStreamWaitEvent(s, (cudaEvent_t)ev, 0), "cudaStreamWaitEvent"); }
void stream_destroy(cudaStream_t s) { cudaStreamDestroy(s); }
void stream_sync(cudaStream_t s) { ck(cudaStreamSynchronize(s), "cudaStreamSynchronize"); }
namespace {
constexpr size_t UNGUARDED = ~(size_t)0;
struct LiveBlock {
  int dev; size_t size;           // device, rounded size
  size_t req;                     // requested bytes of a block handed out under the memory-check mode (guard: [req, size)); UNGUARDED otherwise
  int fill; unsigned long long seq;   // its fill class and allocation number under the mode
};
std::mutex g_pool_mu;
std::multimap<std::pair<int, size_t>, void*> g_pool_free;  // (device, rounded size) -> cached block
std::map<void*, LiveBlock> g_pool_live;                    // block -> what pool_alloc handed out
std::atomic<bool> g_memcheck{false};
struct {   // memory-check counters and messages, under g_pool_mu
  MemcheckStats st;
  unsigned long long seq = 0;
  std::string first, last;
} g_mc;
size_t pool_round(size_t b) {
  if (b < 256) b = 256;
  if (b <= (1u << 20)) { size_t r = 256; while (r < b) r <<= 1; return r; }
  const size_t g = 2u << 20;                   // 2 MiB granularity above 1 MiB
  return (b + g - 1) / g * g;
}
size_t drop_cached_locked() {   // caller holds g_pool_mu
  size_t bytes = 0;
  for (auto& kv : g_pool_free) { bytes += kv.first.second; cudaFree(kv.second); }
  g_pool_free.clear();
  return bytes;
}
// the guard band [req, size) of a block handed out under the memory-check mode must still be zero.  Caller holds g_pool_mu and has synchronised
// the device.  A dirty guard is reported once: it is zeroed again after the report.
void guard_check_locked(void* p, const LiveBlock& b) {
  const size_t n = b.size - b.req;
  std::vector<uint8_t> h(n);
  uint8_t* guard = (uint8_t*)p + b.req;
  std::string msg;
  if (cudaMemcpy(h.data(), guard, n, cudaMemcpyDeviceToHost) != cudaSuccess) {
    msg = std::string("guard band unreadable (") + cudaGetErrorString(cudaGetLastError()) + ")";
  } else {
    g_mc.st.guard_bytes_checked += n;
    size_t k = 0;
    while (k < n && !h[k]) k++;
    if (k == n) return;
    msg = "first dirty guard byte at offset " + std::to_string(b.req + k) + " (" + std::to_string(k) + " bytes past the end)";
    cudaMemset(guard, 0, n);
  }
  g_mc.st.violations++;
  g_mc.last = "write past the end of device allocation #" + std::to_string(b.seq) + " (" + std::to_string(b.req) + " bytes requested, " +
              (b.fill == FILL_FF ? "field elements / points" : "raw / integer") + "): " + msg;
  if (g_mc.first.empty()) g_mc.first = g_mc.last;
}
}  // namespace
size_t pool_release_cached() {
  std::lock_guard<std::mutex> lk(g_pool_mu);
  return drop_cached_locked();
}
size_t pool_live_bytes() {
  std::lock_guard<std::mutex> lk(g_pool_mu);
  size_t bytes = 0;
  for (auto& kv : g_pool_live) bytes += kv.second.size;
  return bytes;
}
void* pool_alloc(size_t bytes, int fill) {
  const bool mc = g_memcheck.load(std::memory_order_relaxed);
  size_t r = pool_round(mc ? bytes + MEMCHECK_GUARD : bytes);
  if (mc) ck(cudaDeviceSynchronize(), "cudaDeviceSynchronize (memory check)");   // whoever used a cached block last has finished with it
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lk(g_pool_mu);
  auto it = g_pool_free.find({dev, r});
  void* p;
  const bool reused = it != g_pool_free.end();
  if (reused) { p = it->second; g_pool_free.erase(it); }
  else {
    cudaError_t e = cudaMalloc(&p, r);
    if (e != cudaSuccess) {  // out of memory: drop the cache and retry once
      cudaGetLastError();
      drop_cached_locked();
      ck(cudaMalloc(&p, r), "cudaMalloc");
    }
  }
  if (!mc) { g_pool_live[p] = {dev, r, UNGUARDED, fill, 0}; return p; }
  g_pool_live[p] = {dev, r, bytes, fill, ++g_mc.seq};
  ck(cudaMemset(p, fill == FILL_FF ? 0xFF : 0, bytes), "cudaMemset (memory check)");
  ck(cudaMemset((uint8_t*)p + bytes, 0, r - bytes), "cudaMemset (memory check guard)");
  ck(cudaDeviceSynchronize(), "cudaDeviceSynchronize (memory check)");   // the legacy-stream fills are unordered with the library's streams
  g_mc.st.blocks_filled++;
  if (reused) g_mc.st.blocks_refilled++;
  return p;
}
void pool_free(void* p) {
  if (!p) return;
  std::lock_guard<std::mutex> lk(g_pool_mu);
  auto it = g_pool_live.find(p);
  if (it == g_pool_live.end()) { cudaFree(p); return; }
  const LiveBlock b = it->second;
  g_pool_live.erase(it);
  if (b.req != UNGUARDED) {   // no throw here: pool_free runs in destructors
    if (cudaDeviceSynchronize() != cudaSuccess) cudaGetLastError();
    guard_check_locked(p, b);
  }
  // blocks of tens of GB (generator tables) are long-lived: do not hoard them.  Per-proof buffers stay cached even when they pass 1 GiB (2^22 constraints: the
  // 1.2 GB dot-product circuit buffer) — a cudaFree synchronises the device, i.e. waits for the background stream's MSM, and the cudaMalloc of the next proof
  // would then make the proof time depend on whether that MSM had finished.  Under the memory-check mode, a block from before the switch is not cached.
  if (b.size > ((size_t)8 << 30) || (g_memcheck.load(std::memory_order_relaxed) && b.req == UNGUARDED)) cudaFree(p);
  else g_pool_free.insert({{b.dev, b.size}, p});
}
void memcheck_enable(bool on) {
  std::lock_guard<std::mutex> lk(g_pool_mu);
  if (g_memcheck.load() == on) return;
  drop_cached_locked();   // a cached block is never handed out across the switch
  g_memcheck.store(on);
}
bool memcheck_on() { return g_memcheck.load(std::memory_order_relaxed); }
MemcheckStats memcheck_stats(std::string* first_violation, std::string* last_violation) {
  std::lock_guard<std::mutex> lk(g_pool_mu);
  if (first_violation) *first_violation = g_mc.first;
  if (last_violation) *last_violation = g_mc.last;
  return g_mc.st;
}
unsigned long long memcheck_scan() {
  std::lock_guard<std::mutex> lk(g_pool_mu);
  const unsigned long long before = g_mc.st.violations;
  bool synced = false;
  for (auto& kv : g_pool_live) {
    if (kv.second.req == UNGUARDED) continue;
    if (!synced) { ck(cudaDeviceSynchronize(), "cudaDeviceSynchronize (memory check scan)"); synced = true; }
    guard_check_locked(kv.first, kv.second);
  }
  return g_mc.st.violations - before;
}
void memcheck_fill(void* d, size_t bytes, int fill) {
  if (!bytes) return;
  ck(cudaDeviceSynchronize(), "cudaDeviceSynchronize (memory check)");
  ck(cudaMemset(d, fill == FILL_FF ? 0xFF : 0, bytes), "cudaMemset (memory check)");
  ck(cudaDeviceSynchronize(), "cudaDeviceSynchronize (memory check)");
}
void memcheck_count_refill() { std::lock_guard<std::mutex> lk(g_pool_mu); g_mc.st.context_refills++; }
void* hmalloc_pinned(size_t b) { void* p = nullptr; ck(cudaMallocHost(&p, b ? b : 16), "cudaMallocHost"); return p; }
void hfree_pinned(void* p) { if (p) cudaFreeHost(p); }
void h2d(void* d, const void* h, size_t b, cudaStream_t s) { g_h2d += b; if (b) ck(cudaMemcpyAsync(d, h, b, cudaMemcpyHostToDevice, s), "h2d"); }
void d2h(void* h, const void* d, size_t b, cudaStream_t s) { g_d2h += b; if (b) ck(cudaMemcpyAsync(h, d, b, cudaMemcpyDeviceToHost, s), "d2h"); }
void d2d(void* dst, const void* src, size_t b, cudaStream_t s) { if (b) ck(cudaMemcpyAsync(dst, src, b, cudaMemcpyDeviceToDevice, s), "d2d"); }
void dzero(void* d, size_t b, cudaStream_t s) { if (b) ck(cudaMemsetAsync(d, 0, b, s), "memset"); }
int sm_count() {
  static int n = 0;
  if (!n) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); if (n <= 0) n = 132; }
  return n;
}
void mem_info(size_t* free_bytes, size_t* total_bytes) { ck(cudaMemGetInfo(free_bytes, total_bytes), "cudaMemGetInfo"); }
void* event_create() { cudaEvent_t e; ck(cudaEventCreate(&e), "cudaEventCreate"); return (void*)e; }
void event_record(void* ev, cudaStream_t s) { ck(cudaEventRecord((cudaEvent_t)ev, s), "cudaEventRecord"); }
float event_elapsed_ms(void* a, void* b) {
  float ms = 0;
  ck(cudaEventSynchronize((cudaEvent_t)b), "cudaEventSynchronize");
  ck(cudaEventElapsedTime(&ms, (cudaEvent_t)a, (cudaEvent_t)b), "cudaEventElapsedTime");
  return ms;
}
void event_destroy(void* ev) { cudaEventDestroy((cudaEvent_t)ev); }

unsigned int grid_for(size_t work, int threads, int per_sm) {
  size_t blocks = (work + threads - 1) / threads;
  size_t cap = (size_t)sm_count() * per_sm;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (unsigned int)blocks;
}


// =============================================================================================== dense helpers
// eq(r, .) table (dense_mlpoly.rs:68-84): out[i] = prod_j (bit_j(i) ? r_j : 1 - r_j), bit 0 of r = most significant bit of i.
// Two-level: small tables for the high / low halves of the variables, then one product per output element.
__global__ void k_eq_small(u256* out, const u256* __restrict__ r, int nv) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ((size_t)1 << nv)) return;
  u256 acc = fq_one();
  for (int j = 0; j < nv; j++) {
    u256 rj = ld256_ro(r + j);
    bool bit = (i >> (nv - 1 - j)) & 1;
    acc = fq_mul(acc, bit ? rj : fq_sub(fq_one(), rj));
  }
  st256(out + i, acc);
}
__global__ void k_eq_combine(u256* out, const u256* __restrict__ hi, const u256* __restrict__ lo, int nlo, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    st256(out + i, fq_mul(ld256_ro(hi + (i >> nlo)), ld256_ro(lo + (i & (((size_t)1 << nlo) - 1)))));
}
void eq_evals(u256* out, const u256* d_r, int ell, u256* small, cudaStream_t s) {
  ProfScope ps("eq_evals", 32.0 * (double)((size_t)1 << ell), s);
  if (ell <= 10) {
    size_t n = (size_t)1 << ell;
    k_eq_small<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(out, d_r, ell);
    SP_LAUNCHED(); check("eq_small");
    return;
  }
  int nhi = ell / 2, nlo = ell - nhi;
  u256* thi = small; u256* tlo = small + ((size_t)1 << nhi);
  k_eq_small<<<(unsigned)((((size_t)1 << nhi) + 127) / 128), 128, 0, s>>>(thi, d_r, nhi);
  k_eq_small<<<(unsigned)((((size_t)1 << nlo) + 127) / 128), 128, 0, s>>>(tlo, d_r + nhi, nlo);
  size_t n = (size_t)1 << ell;
  k_eq_combine<<<grid_for(n, 256, 8), 256, 0, s>>>(out, thi, tlo, nlo, n);
  SP_LAUNCHED(); SP_LAUNCHED(); SP_LAUNCHED(); check("eq_evals");
}
__global__ void k_eq_extend_top(u256* out, size_t n, const u256 r) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const u256 e = ld256(out + n + i), hi = fq_mul(e, r);
    st256(out + i, fq_sub(e, hi));   // (1 - r) e as e - r e: the same canonical residue
    st256(out + n + i, hi);
  }
}
void eq_extend_top(u256* out, size_t n, const u256& r, cudaStream_t s) {
  ProfScope ps("eq_evals", 96.0 * (double)n, s);
  k_eq_extend_top<<<grid_for(n, 256, 8), 256, 0, s>>>(out, n, r);
  SP_LAUNCHED(); check("eq_extend_top");
}

__global__ void __launch_bounds__(256) k_dot(const u256* __restrict__ a, const u256* __restrict__ b, const u256* __restrict__ c, size_t n,
                                            u256* partials, unsigned int* counters, u256* out) {
  u256 acc[1] = {fq_zero()};
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    u256 m = fq_mul(ld256_ro(a + i), ld256_ro(b + i));
    if (c) m = fq_mul(m, ld256_ro(c + i));
    acc[0] = fq_add(acc[0], m);
  }
  block_reduce_finish<1>(acc, partials, counters, out, 1);
}
void dot3(u256* out, const u256* a, const u256* b, const u256* c, size_t n, void* scratch, cudaStream_t s) {
  ProfScope ps("dot", (c ? 96.0 : 64.0) * (double)n, s);
  unsigned int* counters = (unsigned int*)scratch;
  u256* partials = (u256*)((char*)scratch + 256);
  dim3 grid(grid_for(n, 256, 2), 1);
  k_dot<<<grid, 256, 0, s>>>(a, b, c, n, partials, counters, out);
  SP_LAUNCHED(); check("dot");
}
void dot(u256* out, const u256* a, const u256* b, size_t n, void* scratch, cudaStream_t s) { dot3(out, a, b, nullptr, n, scratch, s); }

// out[k] = <a_k, b> for up to 32 tables sharing b (the 21 + 2 evaluations of HashLayerProof::prove, sparse_mlpoly.rs:696-764, all at one point)
struct DotBatch { const u256* a[32]; };
__global__ void __launch_bounds__(256) k_dot_many(DotBatch batch, const u256* __restrict__ b, size_t n, u256* partials, unsigned int* counters, u256* out) {
  const u256* a = batch.a[blockIdx.y];
  u256 acc[1] = {fq_zero()};
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    acc[0] = fq_add(acc[0], fq_mul(ld256_ro(a + i), ld256_ro(b + i)));
  block_reduce_finish<1>(acc, partials, counters, out, 1);
}
void dot_many(u256* out, const u256* const* a_list, int count, const u256* b, size_t n, void* scratch, cudaStream_t s) {
  ProfScope ps("dot_many", 32.0 * (double)n * (count + 1), s);
  if (count > 32) throw std::runtime_error("spartan_b200: dot_many supports at most 32 tables");
  DotBatch db;
  for (int i = 0; i < count; i++) db.a[i] = a_list[i];
  unsigned int* counters = (unsigned int*)scratch;
  u256* partials = (u256*)((char*)scratch + 256);
  dim3 grid(grid_for(n, 256, 1), count);
  k_dot_many<<<grid, 256, 0, s>>>(db, b, n, partials, counters, out);
  SP_LAUNCHED(); check("dot_many");
}

// first elements of up to 64 tables -> one contiguous array (+ the host, through HostSig): the layer claims of the batched product proofs
struct HeadBatch { const u256* p[HEADS_PER_LAUNCH]; };
__global__ void __launch_bounds__(HEADS_PER_LAUNCH) k_heads(HeadBatch hb, int count, u256* out, HostSig sig) {
  if ((int)threadIdx.x < count) {
    u256 v = ld256(hb.p[threadIdx.x]);
    st256(out + threadIdx.x, v);
    if (sig.host_out) st256(sig.host_out + threadIdx.x, v);
  }
  if (sig.flag) {
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) { __threadfence_system(); *((volatile unsigned int*)sig.flag) = sig.seq; }
  }
}
void heads(u256* out, const u256* const* tables, int count, cudaStream_t s, HostSig sig) {
  if (count > HEADS_PER_LAUNCH) throw std::runtime_error("spartan_b200: heads supports at most " + std::to_string(HEADS_PER_LAUNCH) + " tables");
  HeadBatch hb;
  for (int i = 0; i < count; i++) hb.p[i] = tables[i];
  k_heads<<<1, HEADS_PER_LAUNCH, 0, s>>>(hb, count, out, sig);
  SP_LAUNCHED(); check("heads");
}

// DensePolynomial::bound (dense_mlpoly.rs:206-213): out[i] = sum_j L[j]*Z[j*R+i].  Column-per-thread (coalesced over i),
// rows split into gridDim.y slabs whose partial sums land in scratch and are combined by a second tiny kernel.
__global__ void __launch_bounds__(128) k_bound_rows_partial(u256* part, const u256* __restrict__ Z, const u256* __restrict__ L, size_t L_size,
                                                           size_t R_size, size_t rows_per_slab) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R_size) return;
  size_t j0 = (size_t)blockIdx.y * rows_per_slab, j1 = j0 + rows_per_slab;
  if (j1 > L_size) j1 = L_size;
  u256 acc = fq_zero();
  for (size_t j = j0; j < j1; j++) acc = fq_add(acc, fq_mul(ld256_ro(L + j), ld256_ro(Z + j * R_size + i)));
  st256(part + (size_t)blockIdx.y * R_size + i, acc);
}
__global__ void k_sum_slabs(u256* out, const u256* __restrict__ part, size_t R_size, int nslabs) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R_size) return;
  u256 acc = fq_zero();
  for (int k = 0; k < nslabs; k++) acc = fq_add(acc, ld256_ro(part + (size_t)k * R_size + i));
  st256(out + i, acc);
}
void bound_rows(u256* out, const u256* Z, const u256* L, size_t L_size, size_t R_size, u256* scratch, cudaStream_t s) {
  ProfScope ps("bound_rows", 32.0 * (double)L_size * (double)R_size, s);
  int nslabs = 64;
  while (nslabs > 1 && (size_t)nslabs > L_size) nslabs >>= 1;
  size_t rows_per_slab = (L_size + nslabs - 1) / nslabs;
  dim3 grid((unsigned)((R_size + 127) / 128), nslabs);
  k_bound_rows_partial<<<grid, 128, 0, s>>>(scratch, Z, L, L_size, R_size, rows_per_slab);
  k_sum_slabs<<<(unsigned)((R_size + 127) / 128), 128, 0, s>>>(out, scratch, R_size, nslabs);
  SP_LAUNCHED(); SP_LAUNCHED(); check("bound_rows");
}
// bound_rows of k tables against one L in one pass over the tables: blockIdx.z is the table, and table j's partial sums of slab y land at
// part[(y * k + j) * R_size + i], so that k_sum_slabs over k * R_size entries leaves table j's result at out[j * R_size ..]
struct TablePtrs { const u256* t[SP_PC_MAX_TABLES]; };
__global__ void __launch_bounds__(128) k_bound_rows_many(u256* part, TablePtrs tp, const u256* __restrict__ L, size_t L_size, size_t R_size,
                                                        size_t rows_per_slab) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R_size) return;
  const u256* __restrict__ Z = tp.t[blockIdx.z];
  const size_t j0 = (size_t)blockIdx.y * rows_per_slab, j1 = j0 + rows_per_slab < L_size ? j0 + rows_per_slab : L_size;
  u256 acc = fq_zero();
  for (size_t j = j0; j < j1; j++) acc = fq_add(acc, fq_mul(ld256_ro(L + j), ld256_ro(Z + j * R_size + i)));
  st256(part + ((size_t)blockIdx.y * gridDim.z + blockIdx.z) * R_size + i, acc);
}
// enough slabs for about 16 CTAs per SM over all tables, at most 64 and at most one per row
static size_t bound_rows_many_slabs(int k, size_t L_size, size_t R_size) {
  const size_t blocks = ((R_size + 127) / 128) * (size_t)k, want = (size_t)sm_count() * 16;
  size_t nslabs = std::min<size_t>(std::min<size_t>((want + blocks - 1) / blocks, 64), L_size);
  nslabs = std::max<size_t>(nslabs, 1);
  const size_t rows_per_slab = (L_size + nslabs - 1) / nslabs;
  return (L_size + rows_per_slab - 1) / rows_per_slab;
}
size_t bound_rows_many_scratch(int k, size_t L_size, size_t R_size) {
  const size_t nslabs = bound_rows_many_slabs(k, L_size, R_size);
  return nslabs > 1 ? nslabs * (size_t)k * R_size : 1;
}
void bound_rows_many(u256* out, const u256* const* tables, int k, const u256* L, size_t L_size, size_t R_size, u256* scratch, cudaStream_t s) {
  ProfScope ps("bound_rows_many", 32.0 * (double)k * (double)L_size * (double)R_size, s);
  if (k < 1 || k > SP_PC_MAX_TABLES) throw std::runtime_error("spartan_b200: bound_rows_many supports 1 .. SP_PC_MAX_TABLES tables");
  TablePtrs tp;
  for (int j = 0; j < k; j++) tp.t[j] = tables[j];
  const size_t nslabs = bound_rows_many_slabs(k, L_size, R_size), rows_per_slab = (L_size + nslabs - 1) / nslabs;
  const unsigned bx = (unsigned)((R_size + 127) / 128);
  k_bound_rows_many<<<dim3(bx, (unsigned)nslabs, (unsigned)k), 128, 0, s>>>(nslabs > 1 ? scratch : out, tp, L, L_size, R_size, rows_per_slab);
  SP_LAUNCHED();
  if (nslabs > 1) {
    const size_t n = (size_t)k * R_size;
    k_sum_slabs<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(out, scratch, n, (int)nslabs);
    SP_LAUNCHED();
  }
  check("bound_rows_many");
}

__global__ void k_lincomb3(u256* out, const u256* __restrict__ A, const u256* __restrict__ B, const u256* __restrict__ C,
                           const u256* __restrict__ rabc, size_t n) {
  u256 ra = ld256_ro(rabc), rb = ld256_ro(rabc + 1), rc = ld256_ro(rabc + 2);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    st256(out + i, fq_add(fq_add(fq_mul(ra, ld256_ro(A + i)), fq_mul(rb, ld256_ro(B + i))), fq_mul(rc, ld256_ro(C + i))));
}
void lincomb3(u256* out, const u256* A, const u256* B, const u256* C, const u256* d_rabc, size_t n, cudaStream_t s) {
  ProfScope ps("lincomb3", 128.0 * (double)n, s);
  k_lincomb3<<<grid_for(n, 256, 4), 256, 0, s>>>(out, A, B, C, d_rabc, n);
  SP_LAUNCHED(); check("lincomb3");
}
// one product-tree layer of up to 16 circuits of equal size in one launch (blockIdx.y = circuit)
struct HadBatch { u256* out[16]; const u256* a[16]; const u256* b[16]; };
__global__ void k_hadamard_many(HadBatch hb, size_t n) {
  u256* out = hb.out[blockIdx.y]; const u256* a = hb.a[blockIdx.y]; const u256* b = hb.b[blockIdx.y];
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    st256(out + i, fq_mul(ld256(a + i), ld256(b + i)));
}
void hadamard_many(u256* const* outs, const u256* const* as, const u256* const* bs, int count, size_t n, cudaStream_t s) {
  ProfScope ps("hadamard", 96.0 * (double)n * count, s);
  if (count > 16) throw std::runtime_error("spartan_b200: hadamard_many supports at most 16 tables");
  HadBatch hb;
  for (int i = 0; i < count; i++) { hb.out[i] = outs[i]; hb.a[i] = as[i]; hb.b[i] = bs[i]; }
  dim3 grid(grid_for(n, 256, 4), count);
  k_hadamard_many<<<grid, 256, 0, s>>>(hb, n);
  SP_LAUNCHED(); check("hadamard_many");
}
// The descriptors of SP_PROD_MAX_CIRCUITS circuits (about 5 KB) travel as one kernel parameter: the large parameter space of sm_70+ with
// CUDA >= 12.1 (up to 32764 bytes), so the launch needs no descriptor upload, no device allocation and no copy ahead of it.
struct ProdBatch { ProdLeaves c[SP_PROD_MAX_CIRCUITS]; };
static_assert(sizeof(ProdBatch) + sizeof(size_t) <= 32764, "k_prod_leaves: the descriptors exceed the kernel parameter space");
// idx * R^2, so that idx * x in Montgomery form is one product with the plain integer x
__device__ __forceinline__ u256 form_idx_r2(const AffineForm& f) { return f.flags & PROD_IDX ? fq_mul(f.idx, fq_R2()) : fq_zero(); }
// the form at entry x: cst + idx * x + sum_s coeff[s] * src[s][x]
__device__ __forceinline__ u256 form_at(const AffineForm& f, const u256& idx_r2, size_t x) {
  u256 v = f.flags & PROD_CST ? f.cst : fq_zero();
  if (f.flags & PROD_IDX) {
    u256 xi = fq_zero();
    xi.v[0] = (uint32_t)x; xi.v[1] = (uint32_t)(x >> 32);
    v = fq_add(v, fq_mul(idx_r2, xi));
  }
#pragma unroll
  for (int s = 0; s < SP_PROD_MAX_SOURCES; s++) {
    if ((uint32_t)s >= f.nsrc) break;
    const u256 t = ld256_ro(f.src[s] + x);
    v = fq_add(v, (f.flags >> s) & PROD_UNIT0 ? t : fq_mul(f.coeff[s], t));
  }
  return v;
}
// a thread owns the pair (x, x + n/2): both leaves, and their product, the entry x of the first product layer
__global__ void __launch_bounds__(256) k_prod_leaves(const ProdBatch b, size_t half) {
  const ProdLeaves& d = b.c[blockIdx.y];
  const u256 idx_r2 = form_idx_r2(d.f);
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < half; x += (size_t)gridDim.x * blockDim.x) {
    const u256 lo = form_at(d.f, idx_r2, x), hi = form_at(d.f, idx_r2, x + half);
    st256(d.layer0 + x, lo);
    st256(d.layer0 + x + half, hi);
    if (d.layer1) st256(d.layer1 + x, fq_mul(lo, hi));
  }
}
void prod_leaves(const ProdLeaves* circuits, int k, size_t n, cudaStream_t s) {
  if (k < 1 || k > SP_PROD_MAX_CIRCUITS || n < 2) throw std::runtime_error("spartan_b200: prod_leaves takes 1 .. SP_PROD_MAX_CIRCUITS circuits of >= 2 leaves");
  double bytes = 0;
  ProdBatch b;
  for (int i = 0; i < k; i++) { b.c[i] = circuits[i]; bytes += (double)n * (32.0 * (circuits[i].f.nsrc + 1) + (circuits[i].layer1 ? 16.0 : 0.0)); }
  ProfScope ps("prod_leaves", bytes, s);
  dim3 grid(grid_for(n / 2, 256, 4), k);
  k_prod_leaves<<<grid, 256, 0, s>>>(b, n / 2);
  SP_LAUNCHED(); check("prod_leaves");
}
struct DotpBatch { DotpOperands d[PROD_MAX_DOTP]; };
static_assert(sizeof(DotpBatch) + 2 * sizeof(void*) + 2 * sizeof(size_t) <= 32764, "k_dotp_operands: the descriptors exceed the kernel parameter space");
// a thread owns the pair (x, x + n/2): the three operands at both entries, and left * right * weight added to the sum of its half
__global__ void __launch_bounds__(256) k_dotp_operands(const DotpBatch b, size_t half, u256* partials, unsigned int* counters, u256* out) {
  const DotpOperands& d = b.d[blockIdx.y];
  const size_t n = 2 * half;
  u256 idx_r2[3];
#pragma unroll
  for (int o = 0; o < 3; o++) idx_r2[o] = form_idx_r2(d.f[o]);
  u256 acc[2] = {fq_zero(), fq_zero()};
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < half; x += (size_t)gridDim.x * blockDim.x) {
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const size_t at = x + h * half;
      u256 prod = fq_one();
#pragma unroll
      for (int o = 0; o < 3; o++) {
        const u256 v = form_at(d.f[o], idx_r2[o], at);
        st256(d.out + o * n + at, v);
        prod = o ? fq_mul(prod, v) : v;
      }
      acc[h] = fq_add(acc[h], prod);
    }
  }
  block_reduce_finish<2>(acc, partials, counters, out, 2);
}
void dotp_operands(const DotpOperands* dotps, int kd, size_t n, u256* half_sums, void* scratch, cudaStream_t s) {
  if (kd < 1 || kd > PROD_MAX_DOTP || n < 2) throw std::runtime_error("spartan_b200: dotp_operands takes 1 .. PROD_MAX_DOTP dot products of >= 2 entries");
  double bytes = 96.0 * (double)n * kd;   // the operands written; each distinct source table read once
  const u256* seen[3 * PROD_MAX_DOTP * SP_PROD_MAX_SOURCES];
  int ns = 0;
  DotpBatch b;
  for (int i = 0; i < kd; i++) {
    b.d[i] = dotps[i];
    for (int o = 0; o < 3; o++)
      for (uint32_t t = 0; t < dotps[i].f[o].nsrc; t++) {
        const u256* p = dotps[i].f[o].src[t];
        if (std::find(seen, seen + ns, p) == seen + ns) { seen[ns++] = p; bytes += 32.0 * (double)n; }
      }
  }
  ProfScope ps("dotp_operands", bytes, s);
  // the partial sums of every block, two per block and dot product, in the reduction scratch the sumcheck rounds use
  const size_t cap = (sc_scratch_bytes(SC_MAX_INST) - 256) / (2 * sizeof(u256) * (size_t)kd);
  dim3 grid(std::min<size_t>(grid_for(n / 2, 256, 4), cap), kd);
  unsigned int* counters = (unsigned int*)scratch;
  u256* partials = (u256*)((char*)scratch + 256);
  k_dotp_operands<<<grid, 256, 0, s>>>(b, n / 2, partials, counters, half_sums);
  SP_LAUNCHED(); check("dotp_operands");
}
__global__ void k_to_canonical(u256* out, const u256* __restrict__ in, size_t n) {   // Scalar::to_bytes (ristretto255.rs:419) for a whole vector
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) st256(out + i, fq_from_mont(ld256_ro(in + i)));
}
void to_canonical(u256* out, const u256* in, size_t n, cudaStream_t s) {
  k_to_canonical<<<grid_for(n, 128, 8), 128, 0, s>>>(out, in, n);
  SP_LAUNCHED(); check("to_canonical");
}
__global__ void k_gather(u256* out, const u256* __restrict__ mem, const uint32_t* __restrict__ idx, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) st256(out + i, ld256_ro(mem + idx[i]));
}
void gather(u256* out, const u256* mem, const uint32_t* idx, size_t n, cudaStream_t s) {
  ProfScope ps("gather", 68.0 * (double)n, s);
  k_gather<<<grid_for(n, 256, 8), 256, 0, s>>>(out, mem, idx, n);
  SP_LAUNCHED(); check("gather");
}
__global__ void k_spark_hash(u256* out, size_t n, const u256* __restrict__ addr, const u256* __restrict__ val, const u256* __restrict__ ts,
                             int ts_plus_one, const u256* __restrict__ rg) {
  u256 r = ld256_ro(rg), g = ld256_ro(rg + 1), r2 = fq_sqr(r);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    u256 a = addr ? ld256_ro(addr + i) : fq_from_u64((uint64_t)i);
    u256 t = ts ? ld256_ro(ts + i) : fq_zero();
    if (ts_plus_one) t = fq_add(t, fq_one());
    u256 h = fq_add(fq_add(fq_mul(t, r2), fq_mul(ld256_ro(val + i), r)), a);
    st256(out + i, fq_sub(h, g));
  }
}
void spark_hash(u256* out, size_t n, const u256* addr, const u256* val, const u256* ts, int ts_plus_one, const u256* d_rg, cudaStream_t s) {
  ProfScope ps("spark_hash", 128.0 * (double)n, s);
  k_spark_hash<<<grid_for(n, 256, 4), 256, 0, s>>>(out, n, addr, val, ts, ts_plus_one, d_rg);
  SP_LAUNCHED(); check("spark_hash");
}
__global__ void k_fill_one(u256* out, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) st256(out + i, fq_one());
}
void fill_one(u256* out, size_t n, cudaStream_t s) {
  k_fill_one<<<grid_for(n, 256, 8), 256, 0, s>>>(out, n);
  SP_LAUNCHED(); check("fill_one");
}

// ---- IPA helpers (nizk/bullet.rs:72-119)
// both updates of an inner-product round in one launch: rows of blocks y = 0: s[j] *= u^(+-1); y = 1: fold a; y = 2: fold b (one or two products per thread)
__global__ void k_ipa_fold_update(u256* a, u256* b, u256* sv, size_t half, size_t n_full, const u256 u, const u256 ui) {
  const size_t t0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  if (blockIdx.y == 0) {
    for (size_t j = t0; sv && j < n_full; j += step) {
      const bool right = (j & (2 * half - 1)) >= half;
      st256(sv + j, fq_mul(ld256(sv + j), right ? u : ui));   // bullet.rs:108 on the unfolded generators
    }
  } else if (blockIdx.y == 1) {
    for (size_t i = t0; i < half; i += step) st256(a + i, fq_add(fq_mul(ld256(a + i), u), fq_mul(ui, ld256(a + i + half))));   // bullet.rs:106
  } else {
    for (size_t i = t0; i < half; i += step) st256(b + i, fq_add(fq_mul(ld256(b + i), ui), fq_mul(u, ld256(b + i + half))));   // bullet.rs:107
  }
}
void ipa_fold_update(u256* a, u256* b, u256* svec, size_t half, size_t n_full, const u256& u, const u256& uinv, cudaStream_t s) {
  ProfScope ps("ipa_fold_ab", 192.0 * (double)half + 64.0 * (double)n_full, s);
  dim3 grid(grid_for(n_full, 128, 8), 3);
  k_ipa_fold_update<<<grid, 128, 0, s>>>(a, b, svec, half, n_full, u, uinv);
  SP_LAUNCHED(); check("ipa_fold_update");
}

// ---- sparse
__global__ void k_spmv(u256* out, size_t nrows, const uint32_t* __restrict__ ptr, const uint32_t* __restrict__ idx, const u256* __restrict__ val,
                       const u256* __restrict__ x) {
  for (size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (size_t)gridDim.x * blockDim.x) {
    u256 acc = fq_zero();
    for (uint32_t k = ptr[r]; k < ptr[r + 1]; k++) acc = fq_add(acc, fq_mul(ld256_ro(val + k), ld256_ro(x + idx[k])));
    st256(out + r, acc);
  }
}
void spmv(u256* out, size_t nrows, const uint32_t* ptr, const uint32_t* idx, const u256* val, const u256* x, cudaStream_t s) {
  ProfScope ps("spmv", 100.0 * (double)nrows, s);
  k_spmv<<<grid_for(nrows, 128, 8), 128, 0, s>>>(out, nrows, ptr, idx, val, x);
  SP_LAUNCHED(); check("spmv");
}
__global__ void __launch_bounds__(256) k_sparse_eval3(const uint32_t* __restrict__ row, const uint32_t* __restrict__ col, const u256* __restrict__ val,
                                                     size_t nnz, const u256* __restrict__ trx, const u256* __restrict__ try_, u256* partials,
                                                     unsigned int* counters, u256* out) {
  u256 acc[1] = {fq_zero()};
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < nnz; k += (size_t)gridDim.x * blockDim.x)
    acc[0] = fq_add(acc[0], fq_mul(fq_mul(ld256_ro(trx + row[k]), ld256_ro(try_ + col[k])), ld256_ro(val + k)));
  block_reduce_finish<1>(acc, partials, counters, out, 1);
}
void sparse_eval3(u256* out, const uint32_t* row, const uint32_t* col, const u256* val, size_t nnz, const u256* trx, const u256* try_,
                  void* scratch, cudaStream_t s) {
  unsigned int* counters = (unsigned int*)scratch;
  u256* partials = (u256*)((char*)scratch + 256);
  dim3 grid(grid_for(nnz, 256, 2), 1);
  k_sparse_eval3<<<grid, 256, 0, s>>>(row, col, val, nnz, trx, try_, partials, counters, out);
  SP_LAUNCHED(); check("sparse_eval3");
}

// =============================================================================================== group kernels
__device__ __forceinline__ ge ld_ge(const ge* p) {
  ge r;
  r.X = ld256(&p->X); r.Y = ld256(&p->Y); r.Z = ld256(&p->Z); r.T = ld256(&p->T);
  return r;
}
__device__ __forceinline__ void st_ge(ge* p, const ge& g) { st256(&p->X, g.X); st256(&p->Y, g.Y); st256(&p->Z, g.Z); st256(&p->T, g.T); }

__global__ void k_gens_from_uniform(ge* out, const uint8_t* __restrict__ uni, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u256* p = reinterpret_cast<const u256*>(uni + 64 * i);
  st_ge(out + i, ristretto_from_uniform(ld256_ro(p), ld256_ro(p + 1)));
}
void gens_from_uniform(ge* out, const uint8_t* d_uniform64, size_t n, cudaStream_t s) {
  k_gens_from_uniform<<<(unsigned)((n + 63) / 64), 64, 0, s>>>(out, d_uniform64, n);
  SP_LAUNCHED(); check("gens_from_uniform");
}
__global__ void k_decompress(ge* out, int* ok, const uint8_t* __restrict__ in, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  ge g = ge_identity();
  bool good = ristretto_decode(g, ld256_ro(reinterpret_cast<const u256*>(in + 32 * i)));
  st_ge(out + i, g);
  if (ok) ok[i] = good ? 1 : 0;
}
void decompress_batch(ge* out, int* ok, const uint8_t* in32, size_t n, cudaStream_t s) {
  k_decompress<<<(unsigned)((n + 63) / 64), 64, 0, s>>>(out, ok, in32, n);
  SP_LAUNCHED(); check("decompress");
}
__global__ void k_compress(uint8_t* out, const ge* __restrict__ in, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  st256(reinterpret_cast<u256*>(out + 32 * i), ristretto_encode(ld_ge(in + i)));
}
void compress_batch(uint8_t* out32, const ge* in, size_t n, cudaStream_t s) {
  ProfScope ps("compress_batch", 160.0 * (double)n, s);
  k_compress<<<(unsigned)((n + 63) / 64), 64, 0, s>>>(out32, in, n);
  SP_LAUNCHED(); check("compress");
}

// ---- fixed-base window tables: entry (j, w, d-1) = d * 2^(W*w) * G_j, affine niels.  W = 8 (32 windows x 128 entries, 393 KB per
// generator) for small generator sets and the host-side copies; W = 13 (20 windows x 4096 entries, 7.9 MB per generator) for the large sets:
// 8 GB per thousand generators buys 37% fewer point additions per term (20 instead of 32); W = 15 (26.7 MB per generator) where memory allows.
static inline int msm_nwin(int wbits) { return (253 + wbits - 1) / wbits; }
static inline size_t msm_depth(int wbits) { return (size_t)1 << (wbits - 1); }
size_t table_entries(size_t nbases, int wbits) { return nbases * (size_t)msm_nwin(wbits) * msm_depth(wbits); }
__global__ void __launch_bounds__(64) k_build_tables(ge_niels* table, const ge* __restrict__ G, size_t nbases, int wbits, int nwin, int depth) {
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nbases * (size_t)nwin) return;
  size_t j = t / nwin;
  int w = (int)(t % nwin);
  ge P = ld_ge(G + j);
  for (int k = 0; k < wbits * w; k++) P = ge_dbl(P);
  ge acc = P;
  ge_niels* dst = table + t * (size_t)depth;
  for (int d = 0; d < depth; d++) {
    ge_niels nl = ge_to_niels(acc);  // the a=-1 addition law is complete: Z never vanishes
    st256(&dst[d].ypx, nl.ypx); st256(&dst[d].ymx, nl.ymx); st256(&dst[d].t2d, nl.t2d);
    acc = ge_add(acc, P);
  }
}
void build_tables(ge_niels* table, const ge* G, size_t nbases, int wbits, cudaStream_t s) {
  size_t threads = nbases * (size_t)msm_nwin(wbits);
  k_build_tables<<<(unsigned)((threads + 63) / 64), 64, 0, s>>>(table, G, nbases, wbits, msm_nwin(wbits), (int)msm_depth(wbits));
  SP_LAUNCHED(); check("build_tables");
}
// ---- row tables: entry (j, d-1) = d * G_j, d = 1 .. 2^(ROW_W-1), affine niels, no per-window copies (3.1 MB per generator at ROW_W = 16).  The row MSM
// sums the entries of each window separately and pays the window shift once per row (k_msm_horner).  One thread per (generator, run of 64 entries).
constexpr int ROW_W = 16, ROW_NWIN = (253 + ROW_W - 1) / ROW_W;   // 17 bits measured level with 16 (DESIGN.md §7)
constexpr size_t ROW_DEPTH = (size_t)1 << (ROW_W - 1);
constexpr int ROW_BUILD_RUN = 64;
size_t row_table_entries(size_t nbases) { return nbases * ROW_DEPTH; }
__global__ void __launch_bounds__(64) k_build_row_table(ge_niels* rt, const ge* __restrict__ G, size_t nbases) {
  constexpr size_t RUNS = ROW_DEPTH / ROW_BUILD_RUN;
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nbases * RUNS) return;
  const size_t j = t / RUNS, d0 = (t % RUNS) * ROW_BUILD_RUN;
  const ge P = ld_ge(G + j);
  u256 k = fq_zero();
  k.v[0] = (uint32_t)(d0 + 1);
  ge acc = ge_scalarmul(k, P);
  ge_niels* dst = rt + j * ROW_DEPTH + d0;
  for (int i = 0; i < ROW_BUILD_RUN; i++) {
    const ge_niels nl = ge_to_niels(acc);
    st256(&dst[i].ypx, nl.ypx); st256(&dst[i].ymx, nl.ymx); st256(&dst[i].t2d, nl.t2d);
    acc = ge_add(acc, P);
  }
}
void build_row_table(ge_niels* rt, const ge* G, size_t nbases, cudaStream_t s) {
  const size_t threads = nbases * (ROW_DEPTH / ROW_BUILD_RUN);
  k_build_row_table<<<(unsigned)((threads + 63) / 64), 64, 0, s>>>(rt, G, nbases);
  SP_LAUNCHED(); check("build_row_table");
}

// ---- multi-row fixed-base MSM
// grid = (chunks, L); block = 128 threads = COLS columns x GROUPS window-groups of one row.  A thread owns one scalar and the windows
// [g*WPT, (g+1)*WPT) of it; signed W-bit digits, zero digits are skipped (vartime, like the reference's vartime_multiscalar_mul).
// Partial sums are tree-reduced through shared memory.  At most 128 registers per thread (4 CTAs of 128 threads per SM).
__device__ __forceinline__ ge shfl_down_ge(const ge& p, int delta) {
  ge r;
  r.X = shfl_down_256(p.X, delta); r.Y = shfl_down_256(p.Y, delta); r.Z = shfl_down_256(p.Z, delta); r.T = shfl_down_256(p.T, delta);
  return r;
}
// block-wide point sum: shuffle tree inside each warp (no barriers, so a warp that runs out of non-zero digits early reduces at once),
// then the four warp leaders through shared memory
__device__ __forceinline__ ge block_sum_ge_128(ge acc) {
#pragma unroll 1
  for (int d = 16; d > 0; d >>= 1) acc = ge_add(acc, shfl_down_ge(acc, d));
  __shared__ ge sm[4];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) { acc = ge_add(acc, sm[1]); acc = ge_add(acc, ge_add(sm[2], sm[3])); }
  return acc;
}
// Where the MSM's rows come from.  RowStride: row r at scalars + r * stride.  RowTables (dev::TableRows): row r is row r % rows_per_table of
// table r / rows_per_table; the rows of tables at or past ntables are zero and are never read (PADDED: row() may return null for them).
struct RowStride {
  const u256* scalars;
  size_t stride;
  static constexpr bool PADDED = false;
  __device__ __forceinline__ const u256* row(size_t r) const { return scalars + r * stride; }
  RowStride skip(size_t rows) const { return RowStride{scalars + rows * stride, stride}; }
};
struct RowTables {
  const u256* t[SP_PC_MAX_TABLES];
  int ntables, rpt_log, len_log;   // rows per table and scalars per row are powers of two: shifts, no division in the kernels
  size_t first;                    // rows skipped by the launch's grid (gridDim.y limit)
  static constexpr bool PADDED = true;
  __device__ __forceinline__ const u256* row(size_t r) const {
    r += first;
    const size_t j = r >> rpt_log;
    return j < (size_t)ntables ? t[j] + ((r - (j << rpt_log)) << len_log) : nullptr;
  }
  RowTables skip(size_t rows) const { RowTables o = *this; o.first += rows; return o; }
};
template <int WBITS, int GROUPS, int CPT, class Src>
__global__ void __launch_bounds__(128, 4) k_msm_rows(ge* partial, const ge_niels* __restrict__ table, const Src src, size_t R,
                                                     const u256* __restrict__ blinds, size_t blind_base) {
  constexpr int NWIN = (253 + WBITS - 1) / WBITS;
  constexpr int WPT = (NWIN + GROUPS - 1) / GROUPS;   // windows per thread
  constexpr int COLS = 128 / GROUPS;                  // columns per block per pass; CPT passes amortise the reduction tree
  constexpr uint32_t HALF = 1u << (WBITS - 1);
  constexpr size_t DEPTH = (size_t)1 << (WBITS - 1);
  const size_t row = blockIdx.y;
  const size_t ncols = R + (blinds ? 1 : 0);
  const int g = threadIdx.x % GROUPS;
  ge acc = ge_identity();
#pragma unroll 1
  for (int pass = 0; pass < CPT; pass++) {
    const size_t col = ((size_t)blockIdx.x * CPT + pass) * COLS + threadIdx.x / GROUPS;
    if (col >= ncols) break;
    u256 k;
    size_t base;
    if (col < R) {
      const u256* rp = src.row(row);
      if (Src::PADDED && !rp) continue;
      k = ld256_ro(rp + col); base = col;
    } else { k = ld256_ro(blinds + row); base = blind_base; }
    if (fq_is_zero(k)) continue;
    k = fq_from_mont(k);  // group.rs:110-113: scalars leave Montgomery form before the MSM
    // carry into this thread's first window from the signed recoding of the lower windows
    uint32_t carry = 0;
    for (int w = 0; w < g * WPT; w++) carry = (msm_window<WBITS>(k, w) + carry) > HALF ? 1u : 0u;
    const int w_end = (g + 1) * WPT < NWIN ? (g + 1) * WPT : NWIN;
    const ge_niels* tb = table + (base * NWIN + (size_t)g * WPT) * DEPTH;
#pragma unroll 1
    for (int w = g * WPT; w < w_end; w++, tb += DEPTH) {
      uint32_t v = msm_window<WBITS>(k, w) + carry;
      int d;
      if (v > HALF) { d = (int)v - (int)(2 * HALF); carry = 1; } else { d = (int)v; carry = 0; }
      if (d == 0) continue;
      int ad = d < 0 ? -d : d;
      const ge_niels* e = tb + (ad - 1);
      ge_niels nl;
      nl.ypx = ld256_ro(&e->ypx); nl.ymx = ld256_ro(&e->ymx); nl.t2d = ld256_ro(&e->t2d);
      acc = ge_madd(acc, nl, d < 0);
    }
  }
  acc = block_sum_ge_128(acc);
  if (threadIdx.x == 0) st_ge(partial + row * gridDim.x + blockIdx.x, acc);
}
__global__ void __launch_bounds__(128) k_msm_reduce(ge* out, const ge* __restrict__ partial, int chunks) {
  const size_t row = blockIdx.x;
  ge acc = ge_identity();
  for (int c = threadIdx.x; c < chunks; c += 128) acc = ge_add(acc, ld_ge(partial + row * chunks + c));
  acc = block_sum_ge_128(acc);
  if (threadIdx.x == 0) st_ge(out + row, acc);
}
__global__ void __launch_bounds__(32) k_msm_reduce_small(ge* out, const ge* __restrict__ partial, int chunks) {   // chunks <= 32: one warp per row
  const size_t row = blockIdx.x;
  ge acc = (int)threadIdx.x < chunks ? ld_ge(partial + row * chunks + threadIdx.x) : ge_identity();
  for (int d = 16; d > 0; d >>= 1) if (d < 2 * chunks) acc = ge_add(acc, shfl_down_ge(acc, d));
  if (threadIdx.x == 0) st_ge(out + row, acc);
}
__global__ void __launch_bounds__(128) k_ge_add_arrays(ge* a, const ge* __restrict__ b, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) st_ge(a + i, ge_add(ld_ge(a + i), ld_ge(b + i)));
}
// a[i] += b[i] (the blind term of a row commitment, added after the row's MSM: the blinds are drawn on the host while the MSM runs)
void add_points(ge* a, const ge* b, size_t n, cudaStream_t s) {
  if (!n) return;
  k_ge_add_arrays<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(a, b, n);
  SP_LAUNCHED(); check("add_points");
}
// out[0] = sum of n <= 32 points (the "point-add allreduce" of a sharded MSM, after the all-gather of the partial results)
void sum_points(ge* out, const ge* in, int n, cudaStream_t s) {
  if (n < 1 || n > 32) throw std::runtime_error("spartan_b200: sum_points supports 1..32 points");
  k_msm_reduce_small<<<1, 32, 0, s>>>(out, in, n);
  SP_LAUNCHED(); check("sum_points");
}
// ---- the two MSMs of one inner-product round in a single launch (bullet.rs:83-97 with unfolded generators).  G is never folded on the device:
// after k rounds G_k[i] = sum_{j = i mod n_k} s[j]*G[j], so the round's L = <a_L, G_R> and R = <a_R, G_L> are full-length fixed-base MSMs in which
// every generator j carries exactly one non-zero scalar, a[.]*s[j], for L (j in the right half of its n_cur-block) or for R (left half).
// Quad-lane formulation: grid = (chunks, 2 sides), IPAQ_THREADS
// threads = IPAQ_THREADS/4 quads; a quad owns WPQ adjacent windows of one scalar and chains their table entries by mixed additions (two product
// latencies each), then 3 tree levels inside the warp, one gather + 3 levels across the warps, and the last block to finish sums the blocks' partial
// points of both sides.  WPQ balances the two costs: a lone warp already keeps much of its
// sub-partition's multiply pipe busy, so two windows per quad (4608 warps for 4096 generators) are throughput-bound; six or seven windows
// per quad need a quarter of the warps and add only a few mixed additions to the dependent chain.
constexpr int IPAQ_THREADS = 256;
constexpr int IPAQ_SPLIT = 4;   // window groups per scalar (17 windows -> 5 per quad)
template <int WBITS, int WPQ>
__global__ void __launch_bounds__(IPAQ_THREADS, 2) k_ipa_msm_quad(ge* partial, const ge_niels* __restrict__ table, const u256* __restrict__ a, const u256* __restrict__ sv,
                                                                  size_t n_cur, size_t n_full, unsigned int* ticket, ge* out, HostSig sig,
                                                                  const u256* __restrict__ b, u256* c_out, HostSig sigc) {
  if (blockIdx.y == 2) {
    // fused dot products of the round (bullet.rs:78-79), two blocks beside the MSM's: c_L = <a_L, b_R> (block 0), c_R = <a_R, b_L> (block 1); published
    // through their own flag word (sigc), long before the MSM finishes: the host turns them into c*Q while the MSM runs
    if (blockIdx.x >= 2) return;
    const size_t hn = n_cur >> 1;
    const u256* pa = a + (blockIdx.x == 0 ? 0 : hn);
    const u256* pb = b + (blockIdx.x == 0 ? hn : 0);
    u256 acc = fq_zero();
    for (size_t i = threadIdx.x; i < hn; i += IPAQ_THREADS) acc = fq_add(acc, fq_mul(ld256_ro(pa + i), ld256_ro(pb + i)));
    acc = warp_sum_fq(acc);
    __shared__ u256 ds[IPAQ_THREADS / 32];
    if ((threadIdx.x & 31) == 0) ds[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
      u256 v = threadIdx.x < IPAQ_THREADS / 32 ? ds[threadIdx.x] : fq_zero();
      v = warp_sum_fq(v);
      if (threadIdx.x == 0) {
        st256(c_out + blockIdx.x, v);
        if (sigc.host_out) st256(sigc.host_out + blockIdx.x, v);
        __threadfence_system();
        if (atomicAdd(sigc.done, 1u) == 1u) {                 // the second of the two blocks publishes
          *sigc.done = 0;
          if (sigc.flag) { __threadfence_system(); *((volatile unsigned int*)sigc.flag) = sigc.seq; }
        }
      }
    }
    return;
  }
  constexpr int NWIN = (253 + WBITS - 1) / WBITS;
  constexpr int QPS = (NWIN + WPQ - 1) / WPQ;              // quads per scalar
  constexpr int QPB = IPAQ_THREADS / 4, NWARP = IPAQ_THREADS / 32;   // quads per block, warps per block
  constexpr uint32_t HALF = 1u << (WBITS - 1);
  constexpr size_t DEPTH = (size_t)1 << (WBITS - 1);
  const int side = blockIdx.y, tid = threadIdx.x, lane = tid & 31, c = lane & 3, warp = tid >> 5;
  const size_t half = n_cur >> 1, total = n_full >> 1;
  const size_t total_quads = total * QPS, stride = (size_t)gridDim.x * QPB;
  u256 P = quad_identity(c);
  // grid-stride over the (scalar, window group) work items with the same trip count in every quad (the shuffles inside quad_madd need the whole
  // warp)
  for (size_t g0 = (size_t)blockIdx.x * QPB; g0 < total_quads; g0 += stride) {
    const size_t gq = g0 + (tid >> 2);
    const size_t t = gq / QPS;
    const int w0 = WPQ * (int)(gq - t * QPS);
    const bool live = t < total;                           // uniform inside a quad
    u256 k = fq_zero();
    size_t j = 0;
    if (live) {
      const size_t blk = t / half, off = t - blk * half;
      j = blk * n_cur + off + (side == 0 ? half : 0);
      k = fq_mul(ld256_ro(a + (side == 0 ? off : off + half)), ld256_ro(sv + j));
      if (!fq_is_zero(k)) k = fq_from_mont(k);
    }
    uint32_t carry = 0;
    for (int w = 0; w < w0; w++) carry = (msm_window<WBITS>(k, w) + carry) > HALF ? 1u : 0u;
    const ge_niels* tb = table + (j * NWIN + (size_t)w0) * DEPTH;
    // all WPQ table entries are fetched up front (independent gathers from a table of up to 110 GB: DRAM + TLB latency paid once, not once per
    // link of the chain); a zero digit or a window past the top contributes the identity as a niels operand: (y - x, y + x, -, 2dxy) = (1, 1, -, 0)
    u256 x[WPQ];
#pragma unroll
    for (int h = 0; h < WPQ; h++) {
      x[h] = c == 3 ? fp_zero() : fp_one();
      if (live && w0 + h < NWIN) {
        uint32_t v = msm_window<WBITS>(k, w0 + h) + carry;
        int d;
        if (v > HALF) { d = (int)v - (int)(2 * HALF); carry = 1; } else { d = (int)v; carry = 0; }
        if (d != 0) {
          const ge_niels* e = tb + (size_t)h * DEPTH + ((d < 0 ? -d : d) - 1);
          if (c == 0) x[h] = ld256_ro(d < 0 ? &e->ypx : &e->ymx);          // y - x of +/-q
          else if (c == 1) x[h] = ld256_ro(d < 0 ? &e->ymx : &e->ypx);     // y + x of +/-q
          else if (c == 3) { x[h] = ld256_ro(&e->t2d); if (d < 0) x[h] = fp_neg(x[h]); }
        }
      }
    }
#pragma unroll
    for (int h = 0; h < WPQ; h++) P = quad_madd(P, x[h], c, lane);
  }
  P = quad_warp_sum(P, c, lane);
  __shared__ u256 sm[NWARP][4];
  __shared__ bool is_last;
  if (lane < 4) sm[warp][c] = P;
  __syncthreads();
  if (warp == 0) {
    const int q = lane >> 2;                               // NWARP = 8: one warp's sum per quad
    P = q < NWARP ? sm[q][c] : quad_identity(c);
    P = quad_warp_sum(P, c, lane);
    if (lane < 4) { st256(reinterpret_cast<u256*>(partial + (size_t)side * gridDim.x + blockIdx.x) + c, P); __threadfence(); }
    __syncwarp();
    if (lane == 0) is_last = atomicAdd(ticket, 1u) == 2 * gridDim.x - 1;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // last block: the first half of its quads finishes L, the second half R
  constexpr int QH = QPB / 2;
  const int s2 = (tid >> 2) / QH, qq = (tid >> 2) % QH;
  const unsigned int nparts = gridDim.x;
  P = quad_identity(c);
  for (unsigned int base = 0; base < nparts; base += QH) {   // same trip count for every quad; out-of-range slots contribute the identity
    const unsigned int idx = base + qq;
    u256 Q = quad_identity(c);
    if (idx < nparts) Q = ld256_cg(reinterpret_cast<const u256*>(partial + (size_t)s2 * nparts + idx) + c);
    P = base == 0 ? Q : quad_add(P, Q, c, lane);
  }
  P = quad_warp_sum(P, c, lane);
  if (lane < 4) sm[warp][c] = P;
  __syncthreads();
  if (warp == 0 || warp == NWARP / 2) {                    // NWARP/2 = 4 warp sums per side
    const int q = lane >> 2;
    P = q < NWARP / 2 ? sm[warp + q][c] : quad_identity(c);
    P = quad_warp_sum(P, c, lane);
    if (lane < 4) {
      st256(reinterpret_cast<u256*>(out + s2) + c, P);
      if (sig.host_out) { st256(sig.host_out + 4 * s2 + c, P); __threadfence_system(); }
    }
  }
  __syncthreads();
  if (tid == 0) {
    *ticket = 0;
    if (sig.flag) { __threadfence_system(); *((volatile unsigned int*)sig.flag) = sig.seq; }
  }
}
// windows per quad: the window count split into three groups (17 -> 6, 20 -> 7, 32 -> 11)
template <int WBITS> struct IpaQ { static constexpr int NWIN = (253 + WBITS - 1) / WBITS, WPQ = (NWIN + IPAQ_SPLIT - 1) / IPAQ_SPLIT, QPS = (NWIN + WPQ - 1) / WPQ; };
template <int WBITS>
static void ipa_msm_quad_launch(ge* out, const ge_niels* table, const u256* a, const u256* svec, size_t n_cur, size_t n_full, void* scratch, unsigned int* ticket,
                                cudaStream_t s, HostSig sig, const u256* b, u256* c_out, HostSig sigc) {
  const size_t quads = (n_full / 2) * IpaQ<WBITS>::QPS, qpb = IPAQ_THREADS / 4;
  dim3 grid((unsigned)((quads + qpb - 1) / qpb), 2);
  if (b) { grid.y = 3; if (grid.x < 2) grid.x = 2; }        // a third row of blocks, of which two compute the round's dot products
  k_ipa_msm_quad<WBITS, IpaQ<WBITS>::WPQ><<<grid, IPAQ_THREADS, 0, s>>>((ge*)scratch, table, a, svec, n_cur, n_full, ticket, out, sig, b, c_out, sigc);
}
size_t ipa_msm_scratch_points(size_t n_full, int wbits) {   // partial points of the quad-lane kernel (>= 2 blocks per side when the dots are fused)
  const size_t nwin = (size_t)msm_nwin(wbits), total = n_full / 2, wpq = (nwin + IPAQ_SPLIT - 1) / IPAQ_SPLIT, qps = (nwin + wpq - 1) / wpq;
  return 2 * std::max<size_t>((total * qps + IPAQ_THREADS / 4 - 1) / (IPAQ_THREADS / 4), 2);
}
void ipa_msm(ge* out, const ge_niels* table, int wbits, const u256* a, const u256* svec, size_t n_cur, size_t n_full, void* scratch, unsigned int* ticket,
             cudaStream_t s, HostSig sig, const u256* b, u256* c_out, HostSig sigc) {
  ProfScope ps("ipa_msm", 64.0 * (double)n_full, s);
  if (wbits == 8) ipa_msm_quad_launch<8>(out, table, a, svec, n_cur, n_full, scratch, ticket, s, sig, b, c_out, sigc);
  else if (wbits == 13) ipa_msm_quad_launch<13>(out, table, a, svec, n_cur, n_full, scratch, ticket, s, sig, b, c_out, sigc);
  else if (wbits == 15) ipa_msm_quad_launch<15>(out, table, a, svec, n_cur, n_full, scratch, ticket, s, sig, b, c_out, sigc);
  else throw std::runtime_error("spartan_b200: unsupported MSM window width");
  SP_LAUNCHED(); check("ipa_msm_quad");
}

// ---- row MSM over the row tables, for many long rows (the witness commitment, the dereferenced SPARK values).  Per term it does ROW_NWIN mixed
// additions instead of the per-window tables' 20 (13-bit windows), at the price of (ROW_NWIN - 1) * ROW_W doublings per row:
//   k_msm_digits   signed ROW_W-bit digits of every scalar, once: digits[(row * ROW_NWIN + w) * ncols + col]
//   k_msm_win      four lanes own window w of one row and one chunk of ROW_CHUNK columns; lane i adds the table entries of columns i, i + 4, ...
//                  of the chunk into one accumulator, then two shuffle levels give the chunk's part of S[row, w] = sum_col d[row, w, col] * G_col
//   k_msm_chunks   S[row, w] = the sum over the chunks
//   k_msm_horner   out[row] = sum_w 2^(ROW_W * w) S[row, w] by Horner's rule, four lanes per row (quad_dbl / quad_add)
// A CTA makes ROW_CHUNK / 4 = 64 mixed additions per lane and retires, about as many as a CTA of k_msm_rows makes.  Short-lived CTAs matter when the
// MSM runs on the background stream: a kernel of the prover's stream that does not fit beside the resident MSM CTAs starts only when some of them
// retire, and one lane owning a whole 4096-column row (256 additions) delayed the inner-product rounds running beside it by 2 ms per proof.
// The doubling tail runs quad_dbl (quad.cuh).
template <class Src>
__global__ void __launch_bounds__(128) k_msm_digits(int* digits, const Src src, size_t L, size_t R, const u256* __restrict__ blinds) {
  const size_t ncols = R + (blinds ? 1 : 0);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < L * ncols; i += (size_t)gridDim.x * blockDim.x) {
    const size_t row = i / ncols, col = i - row * ncols;
    u256 k;
    if (col < R) {
      const u256* rp = src.row(row);
      k = Src::PADDED && !rp ? fq_zero() : ld256_ro(rp + col);
    } else k = ld256_ro(blinds + row);
    int* dst = digits + row * ROW_NWIN * ncols + col;
    const bool zero = fq_is_zero(k);
    if (!zero) k = fq_from_mont(k);  // group.rs:110-113: scalars leave Montgomery form before the MSM
    uint32_t carry = 0;
#pragma unroll
    for (int w = 0; w < ROW_NWIN; w++) {
      const int d = signed_digit(k, w, ROW_W, carry);
      dst[(size_t)w * ncols] = zero ? 0 : d;
    }
  }
}
constexpr size_t ROW_CHUNK = 256;
// grid = (groups / 32, chunks): CTA (x, y) sums columns [y * ROW_CHUNK, (y + 1) * ROW_CHUNK) of the 32 (row, window) groups [32 x, 32 x + 32)
__global__ void __launch_bounds__(128, 4) k_msm_win(ge* part, const ge_niels* __restrict__ rt, const int* __restrict__ digits, size_t groups, size_t ncols,
                                                    size_t R, size_t blind_base) {
  const size_t g = (size_t)blockIdx.x * 32 + threadIdx.x / 4;   // (row, window) = (g / ROW_NWIN, g % ROW_NWIN)
  const int lane = threadIdx.x % 4;
  const size_t c0 = (size_t)blockIdx.y * ROW_CHUNK, c1 = c0 + ROW_CHUNK < ncols ? c0 + ROW_CHUNK : ncols;
  ge acc = ge_identity();
  if (g < groups) {
    const int* dg = digits + g * ncols;
#pragma unroll 1
    for (size_t col = c0 + lane; col < c1; col += 4) {
      const int d = __ldg(dg + col);
      if (d == 0) continue;
      const size_t base = col < R ? col : blind_base;
      const ge_niels* e = rt + base * ROW_DEPTH + ((d < 0 ? -d : d) - 1);
      ge_niels nl;
      nl.ypx = ld256_ro(&e->ypx); nl.ymx = ld256_ro(&e->ymx); nl.t2d = ld256_ro(&e->t2d);
      acc = ge_madd(acc, nl, d < 0);
    }
  }
  acc = ge_add(acc, shfl_down_ge(acc, 2));   // the four lanes of a group are adjacent and 4-aligned in the warp
  acc = ge_add(acc, shfl_down_ge(acc, 1));
  if (lane == 0 && g < groups) st_ge(part + g * gridDim.y + blockIdx.y, acc);
}
__global__ void __launch_bounds__(128) k_msm_chunks(ge* sums, const ge* __restrict__ part, size_t groups, int chunks) {
  const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= groups) return;
  ge acc = ld_ge(part + g * chunks);
  for (int c = 1; c < chunks; c++) acc = ge_add(acc, ld_ge(part + g * chunks + c));
  st_ge(sums + g, acc);
}
__global__ void __launch_bounds__(32) k_msm_horner(ge* out, const ge* __restrict__ sums, size_t L) {
  const int lane = threadIdx.x & 31, c = lane & 3;
  const size_t row = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
  const bool live = row < L;                                 // every lane takes part in the shuffles; rows past L carry the identity
  const u256* S = reinterpret_cast<const u256*>(sums + (live ? row : 0) * ROW_NWIN) + c;   // coordinate c of S[row, w] at S[4 w]
  u256 P = live ? ld256(S + 4 * (ROW_NWIN - 1)) : quad_identity(c);
#pragma unroll 1
  for (int w = ROW_NWIN - 2; w >= 0; w--) {
#pragma unroll 1
    for (int i = 0; i < ROW_W; i++) P = quad_dbl(P, c, lane);
    P = quad_add(P, live ? ld256(S + 4 * w) : quad_identity(c), c, lane);
  }
  if (live) st256(reinterpret_cast<u256*>(out + row) + c, P);
}
static size_t row_msm_chunks(size_t ncols) { return (ncols + ROW_CHUNK - 1) / ROW_CHUNK; }
static size_t row_msm_points_bytes(size_t L, size_t ncols) { return (L * ROW_NWIN * (row_msm_chunks(ncols) + 1) * sizeof(ge) + 255) / 256 * 256; }
static size_t row_msm_scratch_bytes(size_t L, size_t ncols) { return row_msm_points_bytes(L, ncols) + L * ROW_NWIN * ncols * sizeof(int); }
template <class Src>
static void msm_rows_win(ge* out, const ge_niels* rt, const Src& src, size_t L, size_t R, const u256* blinds, size_t blind_base, void* scratch,
                         cudaStream_t s, size_t smem_pad) {
  const size_t ncols = R + (blinds ? 1 : 0), groups = L * ROW_NWIN, chunks = row_msm_chunks(ncols);
  ge* sums = (ge*)scratch;
  ge* part = sums + groups;
  int* digits = (int*)((char*)scratch + row_msm_points_bytes(L, ncols));
  k_msm_digits<<<grid_for(L * ncols, 128, 16), 128, 0, s>>>(digits, src, L, R, blinds);
  if (smem_pad > (48u << 10)) cudaFuncSetAttribute(k_msm_win, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_pad);
  k_msm_win<<<dim3((unsigned)((groups + 31) / 32), (unsigned)chunks), 128, smem_pad, s>>>(part, rt, digits, groups, ncols, R, blind_base);
  k_msm_chunks<<<(unsigned)((groups + 127) / 128), 128, 0, s>>>(sums, part, groups, (int)chunks);
  k_msm_horner<<<(unsigned)((L * 4 + 31) / 32), 32, 0, s>>>(out, sums, L);
  SP_LAUNCHED(); SP_LAUNCHED(); SP_LAUNCHED(); SP_LAUNCHED(); check("msm_rows_win");
}
// many rows of many terms: the doubling tail is shared by a row's terms and runs beside the other rows.  Short rows, few rows (the blind and delta
// batches of the ZK sumchecks, single-row commitments) stay on the per-window tables, which need no doublings.
static bool msm_rows_use_row_table(size_t L, size_t R) { return L >= 64 && R >= 512; }

static int msm_pick_groups(size_t L, size_t R) {
  // enough threads to fill the chip: one thread per scalar once L*R is large (least reduction work), else split the windows
  size_t cols = L * (R + 1);
  size_t target = (size_t)sm_count() * 1024;
  if (cols >= target) return 1;
  if (cols * 4 >= target) return 4;
  return 8;
}
static int msm_pick_cpt(size_t L, size_t ncols, int groups) {
  // several column passes per thread amortise the block reduction, as long as the grid still oversubscribes the chip
  size_t cols = 128 / groups;
  size_t blocks4 = L * ((ncols + 4 * cols - 1) / (4 * cols));
  return (ncols >= 4 * cols && blocks4 >= (size_t)sm_count() * 4) ? 4 : 1;
}
static size_t msm_chunks(size_t R1, int groups, int cpt) { size_t cols = (128 / groups) * (size_t)cpt; return (R1 + cols - 1) / cols; }
size_t msm_scratch_bytes(size_t L, size_t R) {
  const size_t per_window = L * msm_chunks(R + 1, 8, 1) * sizeof(ge);
  return msm_rows_use_row_table(L, R) ? std::max(per_window, row_msm_scratch_bytes(L, R + 1)) : per_window;
}
template <int WBITS, int GROUPS, class Src>
static void msm_launch2(int cpt, dim3 grid, cudaStream_t s, ge* pp, const ge_niels* table, const Src& src, size_t R, const u256* bl, size_t blind_base,
                        size_t smem_pad) {
  // smem_pad: unused dynamic shared memory that only lowers the number of resident CTAs per SM (a background MSM leaves room for the
  // latency-bound kernels of the main stream)
  if (cpt == 4) {
    if (smem_pad > (48u << 10)) cudaFuncSetAttribute(k_msm_rows<WBITS, GROUPS, 4, Src>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_pad);
    k_msm_rows<WBITS, GROUPS, 4, Src><<<grid, 128, smem_pad, s>>>(pp, table, src, R, bl, blind_base);
  } else {
    if (smem_pad > (48u << 10)) cudaFuncSetAttribute(k_msm_rows<WBITS, GROUPS, 1, Src>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_pad);
    k_msm_rows<WBITS, GROUPS, 1, Src><<<grid, 128, smem_pad, s>>>(pp, table, src, R, bl, blind_base);
  }
}
template <int WBITS, class Src>
static void msm_launch(int groups, int cpt, dim3 grid, cudaStream_t s, ge* pp, const ge_niels* table, const Src& src, size_t R, const u256* bl,
                       size_t blind_base, size_t smem_pad) {
  if (groups == 1) msm_launch2<WBITS, 1>(cpt, grid, s, pp, table, src, R, bl, blind_base, smem_pad);
  else if (groups == 4) msm_launch2<WBITS, 4>(cpt, grid, s, pp, table, src, R, bl, blind_base, smem_pad);
  else msm_launch2<WBITS, 8>(cpt, grid, s, pp, table, src, R, bl, blind_base, smem_pad);
}
template <class Src>
static void msm_rows_src(ge* out, const ge_niels* table, int wbits, const ge_niels* row_table, const Src& src, size_t L, size_t R, const u256* blinds,
                         size_t blind_base, void* scratch, cudaStream_t s, size_t smem_pad) {
  if (row_table && msm_rows_use_row_table(L, R)) {
    msm_rows_win(out, row_table, src, L, R, blinds, blind_base, scratch, s, smem_pad);
    return;
  }
  const size_t ncols = R + (blinds ? 1 : 0);
  int groups = msm_pick_groups(L, R);
  int cpt = msm_pick_cpt(L, ncols, groups);
  size_t chunks = msm_chunks(ncols, groups, cpt);
  ge* partial = (ge*)scratch;
  for (size_t row0 = 0; row0 < L; row0 += 32768) {   // gridDim.y limit 65535
    size_t rows = L - row0 < 32768 ? L - row0 : 32768;
    dim3 grid((unsigned)chunks, (unsigned)rows);
    const Src sc = src.skip(row0);
    const u256* bl = blinds ? blinds + row0 : nullptr;
    ge* pp = partial + row0 * chunks;
    if (wbits == 8) msm_launch<8>(groups, cpt, grid, s, pp, table, sc, R, bl, blind_base, smem_pad);
    else if (wbits == 13) msm_launch<13>(groups, cpt, grid, s, pp, table, sc, R, bl, blind_base, smem_pad);
    else if (wbits == 15) msm_launch<15>(groups, cpt, grid, s, pp, table, sc, R, bl, blind_base, smem_pad);
    else throw std::runtime_error("spartan_b200: unsupported MSM window width");
    SP_LAUNCHED();
  }
  if (chunks <= 32) k_msm_reduce_small<<<(unsigned)L, 32, 0, s>>>(out, partial, (int)chunks);
  else k_msm_reduce<<<(unsigned)L, 128, 0, s>>>(out, partial, (int)chunks);
  SP_LAUNCHED(); check("msm_rows");
}
void msm_rows(ge* out, const ge_niels* table, int wbits, const ge_niels* row_table, const u256* scalars, size_t stride, size_t L, size_t R,
              const u256* blinds, size_t blind_base, void* scratch, cudaStream_t s, size_t smem_pad) {
  ProfScope ps("msm_rows", 32.0 * (double)L * (double)R + 32.0 * (double)R, s);
  msm_rows_src(out, table, wbits, row_table, RowStride{scalars, stride}, L, R, blinds, blind_base, scratch, s, smem_pad);
}
void msm_rows_tables(ge* out, const ge_niels* table, int wbits, const ge_niels* row_table, const TableRows& tr, size_t L, size_t R, const u256* blinds,
                     size_t blind_base, void* scratch, cudaStream_t s) {
  // only the rows of the tables are read: 32 bytes per scalar of ntables * rows_per_table rows, plus the generators' R
  ProfScope ps("msm_rows_tables", 32.0 * (double)std::min<size_t>(L, (size_t)tr.ntables * tr.rows_per_table) * (double)R + 32.0 * (double)R, s);
  const bool pow2 = tr.rows_per_table && !(tr.rows_per_table & (tr.rows_per_table - 1)) && R && !(R & (R - 1));
  if (tr.row_len != R || tr.ntables < 1 || tr.ntables > SP_PC_MAX_TABLES || !pow2) throw std::runtime_error("spartan_b200: msm_rows_tables: inconsistent table list");
  RowTables src;
  for (int j = 0; j < tr.ntables; j++) src.t[j] = tr.t[j];
  src.ntables = tr.ntables;
  src.rpt_log = __builtin_ctzll(tr.rows_per_table);
  src.len_log = __builtin_ctzll(R);
  src.first = 0;
  msm_rows_src(out, table, wbits, row_table, src, L, R, blinds, blind_base, scratch, s, 0);
}

}  // namespace dev
}  // namespace sp
