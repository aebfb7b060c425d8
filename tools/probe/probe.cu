// Latency / throughput probes for the building blocks of the prover kernels (dev tool, not part of the library).
// Build: tools/probe/build.sh   Run on the GPU: tools/probe/probe
// Every latency probe runs ONE warp for ITER dependent operations and reports clock64 cycles per operation; throughput probes fill the chip
// with W warps per SM sub-partition and report operations per second.
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>
#include "../../spartan_b200/csrc/field.cuh"
#include "../../spartan_b200/csrc/curve.cuh"
using namespace sp;

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

__device__ __forceinline__ u256 shfl_down_dummy(const u256& x) { u256 r; for (int i = 0; i < 8; i++) r.v[i] = __shfl_down_sync(0xffffffffu, x.v[i], 1); return r; }
__device__ __forceinline__ u256 mk(uint32_t s) { u256 r; for (int i = 0; i < 8; i++) r.v[i] = s * (i + 1) + 12345u * i; r.v[7] &= 0x0fffffffu; return r; }

template <int OP>
__global__ void k_lat(long long* cycles, u256* sink, int iters, const __grid_constant__ FqConst rc) {
  u256 a = mk(threadIdx.x + 1), b = mk(threadIdx.x + 77);
  ge P = ge_identity(); P.X = a; P.Y = b; P.T = fp_mul(a, b);
  ge Q = P; Q.X = b; Q.Y = a;
  ge_niels N; N.ypx = a; N.ymx = b; N.t2d = fp_mul(a, b);
  long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < iters; i++) {
    if (OP == 0) a = fq_mul_impl(a, b);           // inline F_q Montgomery product
    if (OP == 1) a = fq_mul(a, b);                // as the kernels call it (out of line)
    if (OP == 2) a = fp_mul(a, b);
    if (OP == 3) P = ge_madd(P, N, false);
    if (OP == 4) P = ge_add(P, Q);
    if (OP == 5) a = fq_add(a, b);
    if (OP == 6) a = fq_fold_const(a, b, rc);     // a + r*(b-a) with the per-round constant table
    if (OP == 7) { ge R; R.X = shfl_down_dummy(P.X); R.Y = shfl_down_dummy(P.Y); R.Z = shfl_down_dummy(P.Z); R.T = shfl_down_dummy(P.T); P = ge_add(P, R); }
  }
  long long t1 = clock64();
  if (threadIdx.x == 0) cycles[0] = t1 - t0;
  a = fq_add(a, fq_add(P.X, fq_add(P.Y, fq_add(P.Z, P.T))));
  sink[threadIdx.x] = a;
}

// throughput: every thread runs CH independent chains of `iters` operations
template <int OP, int CH>
__global__ void __launch_bounds__(256) k_tput(u256* sink, int iters, const __grid_constant__ FqConst rc) {
  u256 a[CH], b = mk(threadIdx.x + 77 + blockIdx.x);
#pragma unroll
  for (int c = 0; c < CH; c++) a[c] = mk(threadIdx.x + 1 + c * 131 + blockIdx.x);
#pragma unroll 1
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < CH; c++) {
      if (OP == 0) a[c] = fq_mul_impl(a[c], b);
      if (OP == 1) a[c] = fq_mul(a[c], b);
      if (OP == 2) a[c] = fp_mul(a[c], b);
      if (OP == 6) a[c] = fq_fold_const(a[c], b, rc);
    }
  }
  u256 s = a[0];
#pragma unroll
  for (int c = 1; c < CH; c++) s = fq_add(s, a[c]);
  sink[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int OP>
static void lat(const char* name, long long* d_cyc, u256* sink, FqConst rc) {
  const int iters = 2000;
  k_lat<OP><<<1, 32>>>(d_cyc, sink, 10, rc);
  k_lat<OP><<<1, 32>>>(d_cyc, sink, iters, rc);
  CK(cudaDeviceSynchronize());
  long long c; CK(cudaMemcpy(&c, d_cyc, 8, cudaMemcpyDeviceToHost));
  printf("latency  %-28s %8.1f cycles/op (one warp, dependent chain)\n", name, (double)c / iters);
}
template <int OP, int CH>
static void tput(const char* name, u256* sink, int blocks_per_sm, int threads, FqConst rc) {
  int sms = 0, khz = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
  const int iters = 400;
  const double hz = khz * 1e3;
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  k_tput<OP, CH><<<sms * blocks_per_sm, threads>>>(sink, 10, rc);
  cudaEventRecord(e0);
  k_tput<OP, CH><<<sms * blocks_per_sm, threads>>>(sink, iters, rc);
  cudaEventRecord(e1);
  CK(cudaDeviceSynchronize());
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  double ops = (double)sms * blocks_per_sm * threads * CH * iters;
  printf("tput     %-22s chains/thread %d  warps/SM %3d : %8.2f Gop/s  (%.1f cycles per warp-op per SMSP at %.3f GHz)\n", name, CH, blocks_per_sm * threads / 32,
         ops / ms / 1e6, hz * 4 * sms / (ops / 32 / (ms / 1e3)), hz / 1e9);
}

int main() {
  long long* d_cyc; u256* sink;
  CK(cudaMalloc(&d_cyc, 64)); CK(cudaMalloc(&sink, sizeof(u256) * 256 * 16 * 256));   // up to 256 SMs x 16 CTAs x 256 threads
  u256 r; for (int i = 0; i < 8; i++) r.v[i] = 0x9e3779b9u * (i + 3); r.v[7] &= 0x0fffffffu;
  FqConst rc = fq_const_table(r);
  lat<0>("fq_mul (inline)", d_cyc, sink, rc);
  lat<1>("fq_mul (as called)", d_cyc, sink, rc);
  lat<2>("fp_mul", d_cyc, sink, rc);
  lat<3>("ge_madd (7M)", d_cyc, sink, rc);
  lat<4>("ge_add (9M)", d_cyc, sink, rc);
  lat<5>("fq_add", d_cyc, sink, rc);
  lat<6>("fq_fold_const a+r(b-a)", d_cyc, sink, rc);
  lat<7>("shfl(32 regs) + ge_add", d_cyc, sink, rc);
  for (int bps : {1, 2, 3, 4, 6, 8}) tput<1, 1>("fq_mul as called", sink, bps, 256, rc);
  for (int bps : {1, 2, 3, 4, 6, 8}) tput<0, 1>("fq_mul inline", sink, bps, 256, rc);
  for (int bps : {1, 2, 4}) tput<0, 2>("fq_mul inline", sink, bps, 256, rc);
  for (int bps : {1, 2, 4}) tput<0, 4>("fq_mul inline", sink, bps, 256, rc);
  for (int bps : {1, 2, 3, 4, 6, 8}) tput<6, 1>("fq_fold_const", sink, bps, 256, rc);
  for (int bps : {1, 2, 4}) tput<6, 2>("fq_fold_const", sink, bps, 256, rc);
  for (int bps : {1, 2, 4}) tput<6, 4>("fq_fold_const", sink, bps, 256, rc);
  for (int bps : {1, 2, 4, 8}) tput<2, 1>("fp_mul", sink, bps, 256, rc);
  for (int bps : {1, 2, 4}) tput<2, 2>("fp_mul", sink, bps, 256, rc);
  for (int bps : {1, 2, 4}) tput<2, 4>("fp_mul", sink, bps, 256, rc);
  return 0;
}
