// spartan_b200 — intra-proof sharding over NVLink peer memory: window allocation / CUDA IPC mapping, the bulk all-gathers that write
// straight into every peer's window, and the sharded table producers.  One process per GPU; no NCCL on this path: every collective is a
// kernel that stores into peer-mapped memory and publishes a sequence number, so the transfer is part of the producing kernel
// (the per-round exchange of partial sums lives in block_reduce_finish / xrank_exchange, kcommon.cuh).
// Replaces nothing in the reference (libspartan is single-process); the loops being sharded are dense_mlpoly.rs:215-223 (fold),
// sumcheck.rs:290-357 / :460-469 / :625-652 (round evaluations), dense_mlpoly.rs:165-177 (row commitments), product_tree.rs:18-56.
#include <cuda_runtime.h>
#include <stdexcept>
#include <string>
#include "dev.hpp"
#include "kcommon.cuh"

namespace sp {
namespace dev {

// ---- windows
void* win_alloc(size_t bytes) {   // plain cudaMalloc (IPC-exportable), zero-filled
  void* p = nullptr;
  ck(cudaMalloc(&p, bytes), "cudaMalloc(window)");
  ck(cudaMemset(p, 0, bytes), "cudaMemset(window)");
  ck(cudaDeviceSynchronize(), "window init");
  return p;
}
void win_free(void* p) { if (p) cudaFree(p); }
size_t ipc_handle_bytes() { return sizeof(cudaIpcMemHandle_t); }
void ipc_export(void* devptr, uint8_t* out) {
  cudaIpcMemHandle_t h;
  ck(cudaIpcGetMemHandle(&h, devptr), "cudaIpcGetMemHandle");
  memcpy(out, &h, sizeof h);
}
void* ipc_open(const uint8_t* handle) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof h);
  void* p = nullptr;
  ck(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle (peer window)");
  return p;
}
void ipc_close(void* p) { if (p) cudaIpcCloseMemHandle(p); }

// ---- bulk all-gathers
__device__ __forceinline__ void push_done(const CommDev& c, unsigned int seq, unsigned int* ticket, unsigned int nblocks) {
  __threadfence_system();                       // every thread: its peer stores are performed before the ticket
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int t = atomicAdd(ticket, 1u);
    if (t == nblocks - 1) {
      *ticket = 0;
      __threadfence_system();
      for (int p = 0; p < c.world; p++)
        if (p != c.rank) st_release_sys(&reinterpret_cast<WinCtrl*>(c.win[p])->bflag[c.rank], seq);
    }
  }
}
__global__ void __launch_bounds__(256) k_push_block(const __grid_constant__ CommDev c, const uint4* __restrict__ src, size_t n16, size_t dst_off, unsigned int seq,
                                                    unsigned int* ticket) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) {
    const uint4 v = src[i];
    for (int p = 0; p < c.world; p++) reinterpret_cast<uint4*>(c.win[p] + dst_off + (size_t)c.rank * n16 * 16)[i] = v;
  }
  push_done(c, seq, ticket, gridDim.x);
}
void push_block(const CommDev& c, const void* src, size_t bytes, size_t dst_off, unsigned int seq, unsigned int* ticket, cudaStream_t s) {
  if (bytes % 16 || dst_off % 16) throw std::runtime_error("spartan_b200: push_block needs 16-byte granularity");
  const size_t n16 = bytes / 16;
  k_push_block<<<grid_for(n16 ? n16 : 1, 256, 2), 256, 0, s>>>(c, (const uint4*)src, n16, dst_off, seq, ticket);
  SP_LAUNCHED(); check("push_block");
}
struct PushTables { const u256* t[64]; };
__global__ void __launch_bounds__(256) k_push_cyclic(const __grid_constant__ CommDev c, const __grid_constant__ PushTables tabs, size_t n_local, size_t dst_off,
                                                     unsigned int seq, unsigned int* ticket) {
  const u256* T = tabs.t[blockIdx.y];
  const size_t base = (size_t)blockIdx.y * n_local * c.world;
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < n_local; j += (size_t)gridDim.x * blockDim.x) {
    const u256 v = ld256(T + j);
    const size_t idx = base + j * c.world + c.rank;
    for (int p = 0; p < c.world; p++) st256(reinterpret_cast<u256*>(c.win[p] + dst_off) + idx, v);
  }
  push_done(c, seq, ticket, gridDim.x * gridDim.y);
}
void push_cyclic(const CommDev& c, const u256* const* tables, int ntables, size_t n_local, size_t dst_off, unsigned int seq, unsigned int* ticket, cudaStream_t s) {
  if (ntables < 1 || ntables > 64) throw std::runtime_error("spartan_b200: push_cyclic supports 1..64 tables");
  PushTables pt;
  for (int i = 0; i < ntables; i++) pt.t[i] = tables[i];
  dim3 grid(grid_for(n_local, 256, 1), ntables);
  k_push_cyclic<<<grid, 256, 0, s>>>(c, pt, n_local, dst_off, seq, ticket);
  SP_LAUNCHED(); check("push_cyclic");
}
__global__ void __launch_bounds__(32) k_wait_peers(const __grid_constant__ CommDev c, unsigned int seq) {
  const int p = threadIdx.x;
  if (p < c.world && p != c.rank) wait_flag_sys(&reinterpret_cast<WinCtrl*>(c.win[c.rank])->bflag[p], seq);
}
void wait_peers(const CommDev& c, unsigned int seq, cudaStream_t s) {
  k_wait_peers<<<1, 32, 0, s>>>(c, seq);
  SP_LAUNCHED(); check("wait_peers");
}

// ---- sharded table producers (cyclic partition: rank r holds global index j*world + r at local index j)
__global__ void k_scale(u256* x, const u256 c, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) st256(x + i, fq_mul(ld256(x + i), c));
}
void scale(u256* inout, const u256& c, size_t n, cudaStream_t s) {
  k_scale<<<grid_for(n, 256, 4), 256, 0, s>>>(inout, c, n);
  SP_LAUNCHED(); check("scale");
}
__global__ void k_take_cyclic(u256* out, const u256* __restrict__ full, size_t n_local, int rank, int world) {
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < n_local; j += (size_t)gridDim.x * blockDim.x) st256(out + j, ld256_ro(full + j * world + rank));
}
void take_cyclic(u256* out, const u256* full, size_t n_local, int rank, int world, cudaStream_t s) {
  k_take_cyclic<<<grid_for(n_local, 256, 8), 256, 0, s>>>(out, full, n_local, rank, world);
  SP_LAUNCHED(); check("take_cyclic");
}
__global__ void k_spmv_cyclic(u256* out, size_t nrows_local, int rank, int world, const uint32_t* __restrict__ ptr, const uint32_t* __restrict__ idx,
                              const u256* __restrict__ val, const u256* __restrict__ x) {
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < nrows_local; j += (size_t)gridDim.x * blockDim.x) {
    const size_t r = j * world + rank;
    u256 acc = fq_zero();
    for (uint32_t k = ptr[r]; k < ptr[r + 1]; k++) acc = fq_add(acc, fq_mul(ld256_ro(val + k), ld256_ro(x + idx[k])));
    st256(out + j, acc);
  }
}
void spmv_cyclic(u256* out, size_t nrows_local, int rank, int world, const uint32_t* ptr, const uint32_t* idx, const u256* val, const u256* x, cudaStream_t s) {
  ProfScope ps("spmv", 100.0 * (double)nrows_local, s);
  k_spmv_cyclic<<<grid_for(nrows_local, 128, 8), 128, 0, s>>>(out, nrows_local, rank, world, ptr, idx, val, x);
  SP_LAUNCHED(); check("spmv_cyclic");
}
__global__ void k_spark_hash_cyclic(u256* out, size_t n_local, int rank, int world, const u256* __restrict__ addr, const u256* __restrict__ val,
                                    const u256* __restrict__ ts, int ts_plus_one, const u256* __restrict__ rg) {
  u256 r = ld256_ro(rg), g = ld256_ro(rg + 1), r2 = fq_sqr(r);
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < n_local; j += (size_t)gridDim.x * blockDim.x) {
    const size_t i = j * world + rank;
    u256 a = addr ? ld256_ro(addr + i) : fq_from_u64((uint64_t)i);
    u256 t = ts ? ld256_ro(ts + i) : fq_zero();
    if (ts_plus_one) t = fq_add(t, fq_one());
    u256 h = fq_add(fq_add(fq_mul(t, r2), fq_mul(ld256_ro(val + i), r)), a);
    st256(out + j, fq_sub(h, g));
  }
}
void spark_hash_cyclic(u256* out, size_t n_local, int rank, int world, const u256* addr, const u256* val, const u256* ts, int ts_plus_one, const u256* d_rg,
                       cudaStream_t s) {
  ProfScope ps("spark_hash", 128.0 * (double)n_local, s);
  k_spark_hash_cyclic<<<grid_for(n_local, 256, 4), 256, 0, s>>>(out, n_local, rank, world, addr, val, ts, ts_plus_one, d_rg);
  SP_LAUNCHED(); check("spark_hash_cyclic");
}

}  // namespace dev
}  // namespace sp
