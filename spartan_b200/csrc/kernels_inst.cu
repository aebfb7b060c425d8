// spartan_b200 — instance ingestion on the device: the checks and conversions of Instance::new (lib.rs:129-198) over caller arrays in device
// memory, the CSR / CSC copies of every matrix, the memory-checking timestamps of SNARK::encode (sparse_mlpoly.rs:220-254), and canonical
// scalars -> Montgomery form for a device-computed witness.  All O(nnz) passes; the two sorts are CUB's stable radix sort, so the compressed
// copies keep every row's entries in COO order and the timestamps count earlier positions exactly as the reference's serial loop does.
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#include <algorithm>
#include <stdexcept>
#include <string>
#include "dev.hpp"
#include "kcommon.cuh"

namespace sp {
namespace dev {

static int key_bits(size_t nkeys) {   // radix bits that cover the keys 0 .. nkeys-1 (at least one: CUB wants a non-empty bit range)
  int b = 1;
  while (b < 32 && ((size_t)1 << b) < nkeys) b++;
  return b;
}

bool is_device_pointer(const void* p, int device) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeDevice && a.device == device;
}
void set_max_u64(unsigned long long* w, cudaStream_t s) { ck(cudaMemsetAsync(w, 0xff, sizeof(unsigned long long), s), "memset"); }
void d2h_sync(void* h, const void* d, size_t b) {
  if (b) ck(cudaMemcpy(h, d, b, cudaMemcpyDeviceToHost), "d2h_sync");
}

// Scalar::from_bytes acceptance (ristretto255.rs:400-409): the little-endian integer must be < q
__device__ __forceinline__ bool fq_canonical(const u256& x) {
  int64_t borrow = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) borrow = ((int64_t)x.v[i] - (int64_t)fq_modulus_limb(i) + borrow) >> 32;
  return borrow != 0;
}
// 32 bytes at p: two 128-bit loads when the caller's array is 16-byte aligned (a torch view may start anywhere), bytes otherwise
__device__ __forceinline__ u256 ld_bytes32(const uint8_t* p, bool aligned) {
  if (aligned) return ld256_ro(reinterpret_cast<const u256*>(p));
  u256 r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = (uint32_t)p[4 * i] | ((uint32_t)p[4 * i + 1] << 8) | ((uint32_t)p[4 * i + 2] << 16) | ((uint32_t)p[4 * i + 3] << 24);
  return r;
}

// ---- Instance::new entries (or a caller's SPARK matrices): one pass over every matrix
__global__ void k_inst_ingest(CooIn in, CooOut out, size_t total, uint64_t num_rows, uint64_t num_cols, uint64_t num_vars, uint64_t shift, int aligned,
                              unsigned long long* err) {
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    int m = 0;
    size_t k = t;
#pragma unroll
    for (int j = 0; j < INGEST_MAX_MATRICES - 1; j++)
      if (m == j && k >= in.n[j]) { k -= in.n[j]; m = j + 1; }
    const uint64_t r = in.row[m][k], c = in.col[m][k];
    const u256 x = ld_bytes32(in.val[m] + 32 * k, aligned);
    // the host path's order within one entry: row, column, scalar
    const unsigned code = r >= num_rows ? INGEST_ROW : c >= num_cols ? INGEST_COL : !fq_canonical(x) ? INGEST_SCALAR : 3u;
    if (code != 3u) { atomicMin(err, ((((unsigned long long)m << 40) | k) << 2) | code); continue; }
    out.row[m][k] = (uint32_t)r;
    out.col[m][k] = (uint32_t)(c >= num_vars ? c + shift : c);
    st256(out.val[m] + k, fq_to_mont(x));
  }
}
void inst_ingest(const CooIn& in, int nmat, const CooOut& out, size_t num_rows, size_t num_cols, size_t num_vars, size_t shift, unsigned long long* err,
                 cudaStream_t s) {
  CooIn a = in;   // the matrices past nmat are empty: the kernel's matrix search never reaches them
  size_t total = 0;
  bool aligned = true;
  for (int m = 0; m < INGEST_MAX_MATRICES; m++) {
    if (m >= nmat) a.n[m] = 0;
    total += a.n[m];
    aligned = aligned && (a.n[m] == 0 || ((uintptr_t)a.val[m] & 15) == 0);
  }
  if (!total) return;
  k_inst_ingest<<<grid_for(total, 256, 8), 256, 0, s>>>(a, out, total, num_rows, num_cols, num_vars, shift, aligned ? 1 : 0, err);
  SP_LAUNCHED(); check("inst_ingest");
}
__global__ void k_inst_pad_rows(uint32_t* row, uint32_t* col, u256* val, size_t from, size_t to, uint32_t pad_col) {
  for (size_t i = from + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < to; i += (size_t)gridDim.x * blockDim.x) {
    row[i] = (uint32_t)i; col[i] = pad_col; st256(val + i, fq_zero());
  }
}
void inst_pad_rows(uint32_t* row, uint32_t* col, u256* val, size_t from, size_t to, uint32_t pad_col, cudaStream_t s) {
  if (to <= from) return;
  k_inst_pad_rows<<<1, 32, 0, s>>>(row, col, val, from, to, pad_col);
  SP_LAUNCHED(); check("inst_pad_rows");
}

// ---- canonical scalars -> Montgomery form (Assignment::new on a device array); err: smallest index of a non-canonical value
__global__ void k_canonical_to_mont(u256* out, const uint8_t* in, size_t n, int aligned, unsigned long long* err) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const u256 x = ld_bytes32(in + 32 * i, aligned);
    if (!fq_canonical(x)) { atomicMin(err, (unsigned long long)i); continue; }
    st256(out + i, fq_to_mont(x));
  }
}
void canonical_to_mont(u256* out, const uint8_t* in32, size_t n, unsigned long long* err, cudaStream_t s) {
  if (!n) return;
  k_canonical_to_mont<<<grid_for(n, 256, 8), 256, 0, s>>>(out, in32, n, ((uintptr_t)in32 & 15) == 0 ? 1 : 0, err);
  SP_LAUNCHED(); check("canonical_to_mont");
}

// ---- shared pieces of the two counting sorts: a histogram of the keys and the positions 0..n-1 as sort payload
__global__ void k_hist_iota(const uint32_t* __restrict__ key, size_t n, uint32_t nkeys, uint32_t* cnt, uint32_t* iota, unsigned int* bad) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t k = key[i];
    if (k < nkeys) atomicAdd(&cnt[k], 1u);
    else if (bad) atomicOr(bad, 1u);
    iota[i] = (uint32_t)i;
  }
}
static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
static size_t sort_temp_bytes(size_t n) {
  size_t b = 0;
  ck(cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n), "sort size");
  return b;
}
static size_t scan_temp_bytes(size_t n) {
  size_t b = 0;
  ck(cub::DeviceScan::ExclusiveSum(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n), "scan size");
  return b;
}
// carves [cnt: ncnt | keys_out, iota, perm: n each | cub temp] out of one scratch block
struct SortScratch {
  uint32_t *cnt, *keys_out, *iota, *perm;
  void* temp;
  size_t temp_bytes;
  static size_t bytes(size_t ncnt, size_t n) { return align256(4 * ncnt) + 3 * align256(4 * n) + align256(std::max(sort_temp_bytes(n), scan_temp_bytes(ncnt))); }
  SortScratch(void* scratch, size_t ncnt, size_t n) {
    char* p = (char*)scratch;
    cnt = (uint32_t*)p; p += align256(4 * ncnt);
    keys_out = (uint32_t*)p; p += align256(4 * n);
    iota = (uint32_t*)p; p += align256(4 * n);
    perm = (uint32_t*)p; p += align256(4 * n);
    temp = p;
    temp_bytes = std::max(sort_temp_bytes(n), scan_temp_bytes(ncnt));
  }
};
static void check_items(size_t n) { if (n >= ((size_t)1 << 31)) throw std::runtime_error("spartan_b200: more than 2^31 - 1 entries to sort"); }

// ---- CSR / CSC: ptr = exclusive scan of the histogram of `major`, entries in stable order of `major` (the host counting sort's layout)
size_t compress_scratch_bytes(size_t nmajor, size_t nnz) { check_items(nnz); check_items(nmajor + 1); return SortScratch::bytes(nmajor + 1, nnz); }
__global__ void k_gather_compressed(const uint32_t* __restrict__ perm, const uint32_t* __restrict__ minor, const u256* __restrict__ val, size_t n, uint32_t* idx,
                                    u256* v) {
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (size_t)gridDim.x * blockDim.x) {
    const uint32_t k = perm[p];
    idx[p] = minor[k];
    st256(v + p, ld256_ro(val + k));
  }
}
void build_compressed(uint32_t* ptr, uint32_t* idx, u256* v, size_t nmajor, const uint32_t* major, const uint32_t* minor, const u256* val, size_t nnz,
                      void* scratch, cudaStream_t s) {
  ProfScope ps("build_compressed", 80.0 * (double)nnz + 8.0 * (double)nmajor, s);
  SortScratch w(scratch, nmajor + 1, nnz);
  ck(cudaMemsetAsync(w.cnt, 0, 4 * (nmajor + 1), s), "memset");
  if (nnz) {
    k_hist_iota<<<grid_for(nnz, 256, 8), 256, 0, s>>>(major, nnz, (uint32_t)nmajor, w.cnt, w.iota, nullptr);
    SP_LAUNCHED(); check("hist_iota");
    size_t tb = w.temp_bytes;
    ck(cub::DeviceRadixSort::SortPairs(w.temp, tb, major, w.keys_out, w.iota, w.perm, (int)nnz, 0, key_bits(nmajor), s), "sort");
    k_gather_compressed<<<grid_for(nnz, 256, 8), 256, 0, s>>>(w.perm, minor, val, nnz, idx, v);
    SP_LAUNCHED(); check("gather_compressed");
  }
  size_t tb = w.temp_bytes;
  ck(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.cnt, ptr, (int)(nmajor + 1), s), "scan");   // cnt[nmajor] = 0, so ptr[nmajor] = nnz
}

// ---- the caller's matrices in one sorted order: keys sorted stably (CUB radix sort), src and val gathered along
size_t spmat_sort_scratch_bytes(size_t nnz) { check_items(nnz); return 2 * align256(4 * nnz) + align256(sort_temp_bytes(nnz)); }
void spmat_sort(uint32_t* key_out, uint32_t* src_out, u256* val_out, const uint32_t* key, const uint32_t* src, const u256* val, size_t nkeys, size_t nnz,
                void* scratch, cudaStream_t s) {
  if (!nnz) return;
  ProfScope ps("spmat_sort", 80.0 * (double)nnz, s);
  char* p = (char*)scratch;
  uint32_t* iota = (uint32_t*)p; p += align256(4 * nnz);
  uint32_t* perm = (uint32_t*)p; p += align256(4 * nnz);
  k_hist_iota<<<grid_for(nnz, 256, 8), 256, 0, s>>>(key, nnz, 0, nullptr, iota, nullptr);   // nkeys = 0: the positions only, no histogram
  SP_LAUNCHED(); check("hist_iota");
  size_t tb = sort_temp_bytes(nnz);
  ck(cub::DeviceRadixSort::SortPairs(p, tb, key, key_out, iota, perm, (int)nnz, 0, key_bits(nkeys), s), "sort");
  k_gather_compressed<<<grid_for(nnz, 256, 8), 256, 0, s>>>(perm, src, val, nnz, src_out, val_out);
  SP_LAUNCHED(); check("gather_compressed");
}

// ---- segmented products out_m[key] = sum val * x[src] over the entries of b matrices, each sorted by key (merge-based SpMV, Merrill & Garland):
// every CTA takes SPMAT_TILE consecutive entries of the concatenated batch whatever the rows' lengths.  An entry's segment key is (m << 32 | key),
// so a segment never crosses a matrix boundary.  Inside a tile, runs of equal key are summed in registers and joined across threads by a
// segmented scan (warp shuffles, then the warps' carries through shared memory).  A segment that starts and ends inside the tile is stored
// directly: the entries are sorted, so no other tile holds its key.  The tile's first and last segments go to a carry array of (key, partial)
// pairs (two per tile; a tile of one segment pairs it with a zero of the same key), which is again sorted by key and reduced the same way: one
// more tiled pass leaves 2 ceil(2 ceil(n / TILE) / TILE) carries, at most 2^14 for n < 2^32, which one CTA finishes.  Every output key is
// stored exactly once; the keys no entry has keep the zero the outputs start from.
struct SegOut { u256* out[SP_SPMAT_MAX_BATCH]; };
struct SegEnds { unsigned long long kf, kl; u256 vf, vl; int single; };
__device__ __forceinline__ void seg_store(const SegOut& o, unsigned long long k, const u256& v) { st256(o.out[k >> 32] + (uint32_t)k, v); }
__device__ __forceinline__ u256 shfl_up_256(const u256& x, int delta) {
  u256 r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = __shfl_up_sync(0xffffffffu, x.v[i], delta);
  return r;
}
// level 0: the matrices' entries; an entry's value is val * x[src]
struct SegEntries {
  const uint32_t* key[SP_SPMAT_MAX_BATCH];
  const uint32_t* src[SP_SPMAT_MAX_BATCH];
  const u256* val[SP_SPMAT_MAX_BATCH];
  unsigned long long start[SP_SPMAT_MAX_BATCH + 1];   // matrix m holds the global entries start[m] .. start[m + 1]
  const u256* x;
  int b;
  __device__ __forceinline__ void load(size_t t, unsigned long long& k, u256& v) const {
    int m = 0;
#pragma unroll
    for (int j = 1; j < SP_SPMAT_MAX_BATCH; j++) m += (j < b && t >= start[j]) ? 1 : 0;
    const size_t i = t - start[m];
    k = ((unsigned long long)m << 32) | key[m][i];
    v = fq_mul(ld256_ro(val[m] + i), ld256_ro(x + src[m][i]));
  }
};
// levels 1 and 2: the carries of the level below
struct SegCarries {
  const unsigned long long* k;
  const u256* v;
  __device__ __forceinline__ void load(size_t t, unsigned long long& key, u256& val) const { key = k[t]; val = ld256(v + t); }
};

// one tile of nt <= SPMAT_TILE items from `base`: stores the segments inside it, returns its first and last segments in `ends` (all threads)
template <class Src>
__device__ __forceinline__ void seg_tile(const Src& src, size_t base, int nt, const SegOut& o, SegEnds& ends) {
  __shared__ unsigned long long skey[SPMAT_TILE];
  __shared__ u256 wv[SPMAT_THREADS / 32];
  __shared__ int wf[SPMAT_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, j0 = tid * SPMAT_ITEMS;
  const int nitems = max(0, min(SPMAT_ITEMS, nt - j0));
  unsigned long long k[SPMAT_ITEMS];
  u256 p[SPMAT_ITEMS];
#pragma unroll
  for (int j = 0; j < SPMAT_ITEMS; j++) {
    k[j] = 0; p[j] = fq_zero();
    if (j < nitems) { src.load(base + j0 + j, k[j], p[j]); skey[j0 + j] = k[j]; }
  }
  __syncthreads();
  // head: an item, not the tile's first, whose key differs from its predecessor's.  Scan value: the sum since the thread's last head (all of it
  // without one), flagged when the thread has a head
  bool head[SPMAT_ITEMS];
  int f = 0;
  u256 v = fq_zero();
#pragma unroll
  for (int j = 0; j < SPMAT_ITEMS; j++) {
    head[j] = j < nitems && j0 + j > 0 && k[j] != (j ? k[j - 1] : skey[j0 - 1]);
    if (head[j]) { f = 1; v = fq_zero(); }
    if (j < nitems) v = fq_add(v, p[j]);
  }
  // inclusive segmented scan over the warp: (fa, va) + (fb, vb) = (fa | fb, fb ? vb : va + vb)
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const u256 vo = shfl_up_256(v, d);
    const int fo = __shfl_up_sync(0xffffffffu, f, d);
    if (lane >= d) {
      if (!f) v = fq_add(vo, v);
      f |= fo;
    }
  }
  if (lane == 31) { wv[warp] = v; wf[warp] = f; }
  // exclusive within the warp
  u256 ce = shfl_up_256(v, 1);
  int fe = __shfl_up_sync(0xffffffffu, f, 1);
  if (lane == 0) { ce = fq_zero(); fe = 0; }
  __syncthreads();
  // the earlier warps' carry: their aggregates back to the nearest flagged one
  u256 cw = fq_zero();
  int fw = 0;
  for (int w = warp - 1; w >= 0; w--) {
    cw = fq_add(wv[w], cw);
    if (wf[w]) { fw = 1; break; }
  }
  u256 run = fe ? ce : fq_add(cw, ce);   // the open segment's sum at the thread's first item
  int seen = fw | fe;                    // a head earlier in the tile: the open segment is not the tile's first
#pragma unroll
  for (int j = 0; j < SPMAT_ITEMS; j++) {
    if (head[j]) {
      const unsigned long long kp = j ? k[j - 1] : skey[j0 - 1];
      if (seen) seg_store(o, kp, run);
      else { ends.kf = kp; ends.vf = run; }
      run = fq_zero();
      seen = 1;
    }
    if (j < nitems) run = fq_add(run, p[j]);
  }
  if (nitems > 0 && j0 + nitems == nt) {   // the tile's last item
    ends.kl = k[nitems - 1]; ends.vl = run; ends.single = !seen;
    if (!seen) { ends.kf = ends.kl; ends.vf = run; }
  }
  __syncthreads();
}
template <class Src>
__global__ void __launch_bounds__(SPMAT_THREADS) k_seg_tiles(Src src, size_t n, SegOut o, unsigned long long* ck, u256* cv) {
  __shared__ SegEnds ends;
  const size_t base = (size_t)blockIdx.x * SPMAT_TILE;
  if (base >= n) return;
  seg_tile(src, base, (int)min((size_t)SPMAT_TILE, n - base), o, ends);
  if (threadIdx.x == 0) {
    ck[2 * blockIdx.x] = ends.kf; st256(cv + 2 * blockIdx.x, ends.vf);
    ck[2 * blockIdx.x + 1] = ends.kl; st256(cv + 2 * blockIdx.x + 1, ends.single ? fq_zero() : ends.vl);
  }
}
// the last level in one CTA: the tiles in order, the segment open at a tile's end carried into the next
__global__ void __launch_bounds__(SPMAT_THREADS) k_seg_final(SegCarries src, size_t n, SegOut o) {
  __shared__ SegEnds ends;
  unsigned long long rk = 0;
  u256 rv = fq_zero();
  bool open = false;
  for (size_t base = 0; base < n; base += SPMAT_TILE) {
    seg_tile(src, base, (int)min((size_t)SPMAT_TILE, n - base), o, ends);
    if (threadIdx.x == 0) {
      u256 first = ends.vf;
      if (open && rk == ends.kf) first = fq_add(rv, first);
      else if (open) seg_store(o, rk, rv);
      if (ends.single) { rk = ends.kf; rv = first; }
      else { seg_store(o, ends.kf, first); rk = ends.kl; rv = ends.vl; }
      open = true;
    }
  }
  if (threadIdx.x == 0 && open) seg_store(o, rk, rv);
}
size_t spmat_products_scratch_bytes(size_t total) { return SpmatCarries(total).bytes; }
void spmat_products(const SpmatBatch& B, const u256* x, size_t nout, void* scratch, cudaStream_t s) {
  SegEntries e{};
  SegOut o{};
  size_t total = 0;
  for (int m = 0; m < B.b; m++) {
    e.key[m] = B.key[m]; e.src[m] = B.src[m]; e.val[m] = B.val[m]; e.start[m] = total;
    o.out[m] = B.out[m];
    total += B.nnz[m];
    dzero(B.out[m], 32 * nout, s);
  }
  for (int m = B.b; m <= SP_SPMAT_MAX_BATCH; m++) e.start[m] = total;
  e.x = x; e.b = B.b;
  const SpmatCarries L(total);
  const size_t n1 = L.n1, n2 = L.n2;
  ProfScope ps("spmat_products", 72.0 * (double)total + 32.0 * (double)nout * B.b, s);
  char* p = (char*)scratch;
  u256* cv1 = (u256*)(p + L.cv1);
  u256* cv2 = (u256*)(p + L.cv2);
  unsigned long long* ck1 = (unsigned long long*)(p + L.ck1);
  unsigned long long* ck2 = (unsigned long long*)(p + L.ck2);
  // a fixed three launches (SP_SPMAT_PRODUCT_LAUNCHES) for every shape; the grids of empty levels run one CTA that returns at once
  k_seg_tiles<<<(unsigned)std::max<size_t>(1, n1 / 2), SPMAT_THREADS, 0, s>>>(e, total, o, ck1, cv1);
  k_seg_tiles<<<(unsigned)std::max<size_t>(1, n2 / 2), SPMAT_THREADS, 0, s>>>(SegCarries{ck1, cv1}, n1, o, ck2, cv2);
  k_seg_final<<<1, SPMAT_THREADS, 0, s>>>(SegCarries{ck2, cv2}, n2, o);
  SP_LAUNCHED(); SP_LAUNCHED(); SP_LAUNCHED(); check("spmat_products");
}
// out = sum_m w[m] * t[m] (the weighted eval table: k_lincomb3 for b tables)
__global__ void k_lincomb_many(u256* out, LincombTables lt, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    u256 acc = fq_mul(lt.w[0], ld256_ro(lt.t[0] + i));
    for (int m = 1; m < lt.b; m++) acc = fq_add(acc, fq_mul(lt.w[m], ld256_ro(lt.t[m] + i)));
    st256(out + i, acc);
  }
}
void lincomb_many(u256* out, const LincombTables& lt, size_t n, cudaStream_t s) {
  ProfScope ps("lincomb_many", 32.0 * (double)n * (lt.b + 1), s);
  k_lincomb_many<<<grid_for(n, 256, 4), 256, 0, s>>>(out, lt, n);
  SP_LAUNCHED(); check("lincomb_many");
}

// ---- AddrTimestamps::new (sparse_mlpoly.rs:220-254) for one side: b N positions in the reference loop's order (matrix-major, zero-padded to N);
// read_ts of a position = earlier positions with its address = its rank within its run after a stable sort by address; audit = run lengths
size_t spark_ts_scratch_bytes(size_t b, size_t N, size_t cells) {
  check_items(b * N); check_items(cells);
  return align256(4 * b * N) + align256(4 * cells) + SortScratch::bytes(cells, b * N);
}
__global__ void k_ts_addrs(SparkAddrs sa, size_t N, uint32_t* keys, u256* addr_f) {
  for (size_t pos = (size_t)blockIdx.x * blockDim.x + threadIdx.x; pos < (size_t)sa.b * N; pos += (size_t)gridDim.x * blockDim.x) {
    const int m = (int)(pos / N);
    const size_t i = pos - (size_t)m * N;
    const uint32_t a = i < sa.nnz[m] ? sa.src[m][i] : 0u;
    keys[pos] = a;
    sa.idx[m][i] = a;
    st256(addr_f + pos, fq_from_u64(a));
  }
}
__global__ void k_ts_ranks(const uint32_t* __restrict__ skey, const uint32_t* __restrict__ spos, const uint32_t* __restrict__ off, size_t n, uint32_t cells,
                           u256* ts_f) {
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (size_t)gridDim.x * blockDim.x) {
    const uint32_t a = skey[p];
    if (a < cells) st256(ts_f + spos[p], fq_from_u64((uint64_t)(p - off[a])));
  }
}
__global__ void k_u32_to_fq(u256* out, const uint32_t* __restrict__ v, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) st256(out + i, fq_from_u64(v[i]));
}
void spark_timestamps(const SparkAddrs& sa, u256* addr_f, u256* ts_f, u256* audit_f, size_t N, size_t cells, void* scratch, unsigned int* bad, cudaStream_t s) {
  const size_t n = (size_t)sa.b * N;
  ProfScope ps("spark_timestamps", (double)n * (32 + 32 + 32) + 40.0 * cells, s);
  uint32_t* keys = (uint32_t*)scratch;
  uint32_t* off = (uint32_t*)((char*)scratch + align256(4 * n));
  SortScratch w((char*)scratch + align256(4 * n) + align256(4 * cells), cells, n);
  ck(cudaMemsetAsync(w.cnt, 0, 4 * cells, s), "memset");
  k_ts_addrs<<<grid_for(n, 256, 8), 256, 0, s>>>(sa, N, keys, addr_f);
  k_hist_iota<<<grid_for(n, 256, 8), 256, 0, s>>>(keys, n, (uint32_t)cells, w.cnt, w.iota, bad);
  SP_LAUNCHED(); SP_LAUNCHED(); check("ts_addrs");
  size_t tb = w.temp_bytes;
  ck(cub::DeviceRadixSort::SortPairs(w.temp, tb, keys, w.keys_out, w.iota, w.perm, (int)n, 0, key_bits(cells), s), "sort");
  tb = w.temp_bytes;
  ck(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.cnt, off, (int)cells, s), "scan");
  k_ts_ranks<<<grid_for(n, 256, 8), 256, 0, s>>>(w.keys_out, w.perm, off, n, (uint32_t)cells, ts_f);
  k_u32_to_fq<<<grid_for(cells, 256, 8), 256, 0, s>>>(audit_f, w.cnt, cells);
  SP_LAUNCHED(); SP_LAUNCHED(); check("ts_ranks");
}

}  // namespace dev
}  // namespace sp
