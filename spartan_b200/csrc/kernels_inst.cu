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
