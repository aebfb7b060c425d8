// spartan_b200 — sumcheck-round kernels (K1/K2 of SURVEY.md §2b), their own translation unit so the two .cu files build in parallel.
#include "kcommon.cuh"

namespace sp {
namespace dev {

// =============================================================================================== sumcheck rounds
struct ScBatch {   // a kernel parameter: SC_MAX_INST (dev.hpp) instances
  ScInst inst[SC_MAX_INST];
};

template <int KIND>
__device__ __forceinline__ u256 sc_comb(const u256& a, const u256& b, const u256& c, const u256& d) {
  if (KIND == SC_QUAD) return fq_mul(a, b);                        // r1csproof.rs:122-123
  if (KIND == SC_CUBIC3) return fq_mul(fq_mul(a, b), c);           // product_tree.rs:283-286
  return fq_mul(a, fq_sub(fq_mul(b, c), d));                       // r1csproof.rs:87-91
}

template <int KIND>
__device__ __forceinline__ void sc_accumulate(u256 (&acc)[3], const u256 (&lo)[4], const u256 (&hi)[4]) {
  constexpr int NT = KIND == SC_QUAD ? 2 : (KIND == SC_CUBIC3 ? 3 : 4);
  u256 x[4], dl[4];
#pragma unroll
  for (int t = 0; t < 4; t++) { x[t] = fq_zero(); dl[t] = fq_zero(); }
  // t = 0 : low halves                                             (sumcheck.rs:463 / :627)
  acc[0] = fq_add(acc[0], sc_comb<KIND>(lo[0], lo[1], lo[2], lo[3]));
  // t = 2 : 2*hi - lo = hi + (hi - lo)                              (sumcheck.rs:466-468 / :630-639)
#pragma unroll
  for (int t = 0; t < NT; t++) { dl[t] = fq_sub(hi[t], lo[t]); x[t] = fq_add(hi[t], dl[t]); }
  acc[1] = fq_add(acc[1], sc_comb<KIND>(x[0], x[1], x[2], x[3]));
  if (KIND != SC_QUAD) {
    // t = 3 : previous point + (hi - lo)                            (sumcheck.rs:642-651)
#pragma unroll
    for (int t = 0; t < NT; t++) x[t] = fq_add(x[t], dl[t]);
    acc[2] = fq_add(acc[2], sc_comb<KIND>(x[0], x[1], x[2], x[3]));
  }
}

template <int KIND>
__global__ void __launch_bounds__(256, 2) k_sc_eval(ScBatch batch, size_t len, u256* partials, unsigned int* counters, u256* out, HostSig sig,
                                                                   const __grid_constant__ XRank xr) {
  constexpr int NT = KIND == SC_QUAD ? 2 : (KIND == SC_CUBIC3 ? 3 : 4);
  const ScInst& in = batch.inst[blockIdx.y];
  const size_t half = len >> 1;
  u256 acc[3] = {fq_zero(), fq_zero(), fq_zero()};
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
    u256 lo[4], hi[4];
#pragma unroll
    for (int t = 0; t < 4; t++) { lo[t] = fq_zero(); hi[t] = fq_zero(); }
#pragma unroll
    for (int t = 0; t < NT; t++) { lo[t] = ld256(in.t[t] + i); hi[t] = ld256(in.t[t] + i + half); }
    sc_accumulate<KIND>(acc, lo, hi);
  }
  block_reduce_finish<3>(acc, partials, counters, out, 3, sig, xr);
}

// Fused: bind the top variable with r (len -> len/2) and evaluate the next round's polynomial on the folded table.
// Thread i owns elements {i, i+len/4, i+len/2, i+3len/4} of every table: in-place update is race-free.
// The bind is the constant-multiplier fold (fq_fold_const: table of r*2^(32j) mod q in uniform registers, 72 wide products and no separate
// modular addition) instead of sub + Montgomery product + add; same canonical values.
template <int KIND>
__global__ void __launch_bounds__(256, 2) k_sc_fold_eval(ScBatch batch, size_t len, const __grid_constant__ FqConst rc, u256* partials,
                                                       unsigned int* counters, u256* out, HostSig sig, const __grid_constant__ XRank xr) {
  constexpr int NT = KIND == SC_QUAD ? 2 : (KIND == SC_CUBIC3 ? 3 : 4);
  const ScInst& in = batch.inst[blockIdx.y];
  const size_t half = len >> 1, quarter = len >> 2;
  u256 acc[3] = {fq_zero(), fq_zero(), fq_zero()};
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < quarter; i += (size_t)gridDim.x * blockDim.x) {
    u256 lo[4], hi[4];
#pragma unroll
    for (int t = 0; t < 4; t++) { lo[t] = fq_zero(); hi[t] = fq_zero(); }
#pragma unroll
    for (int t = 0; t < NT; t++) {
      u256 a0 = ld256(in.t[t] + i), a1 = ld256(in.t[t] + i + half);
      u256 b0 = ld256(in.t[t] + i + quarter), b1 = ld256(in.t[t] + i + quarter + half);
      lo[t] = fq_fold_const(a0, a1, rc);   // dense_mlpoly.rs:218
      hi[t] = fq_fold_const(b0, b1, rc);
      if (t == 2) {
        if (in.write_c) { st256(in.c_out + i, lo[t]); st256(in.c_out + i + quarter, hi[t]); }
      } else {
        st256(in.t[t] + i, lo[t]); st256(in.t[t] + i + quarter, hi[t]);
      }
    }
    sc_accumulate<KIND>(acc, lo, hi);
  }
  block_reduce_finish<3>(acc, partials, counters, out, 3, sig, xr);
}

// ---- eq-factored rounds of the batched product-circuit sumchecks (prove_cubic_batched with the shared C = eq(tau, .): product_tree.rs:279-286).
// The round polynomial of sum_x eq(tau, x) A(x) B(x) factors: s_j(t) = prefix_j * eq(tau_j, t) * q_j(t) with prefix_j = prod_{i<j} eq(tau_i, r_i) and
//   q_j(t) = sum_{x'} E_j[x'] * A(t, x') * B(t, x'),   E_j = eq(tau[j+1..], .)  (the suffix table: half the length, never bound, never written),
// a QUADRATIC whose value at 1 follows from the running claim (q_j(1) = (c_j - (1 - tau_j) q_j(0)) / tau_j, c_{j+1} = q_j(r_j)), so a round needs
// q_j(0) and the leading coefficient q_j(inf) only: 4 field products per index (a0 b0, da db, and the two weights) instead of the 6 of the three
// cubic evaluations, no C table to bind, 2 values per instance to reduce.  The host rebuilds s_j(0), s_j(2), s_j(3) — the field elements the
// reference computes (sumcheck.rs:296-355) — so the proof bytes do not change.  Streaming rounds only; the small-table tail runs the standard
// kernels on C = prefix * eq(tau[j..], .).   out[3*inst + 0] = q(0), out[3*inst + 1] = q(inf).
__global__ void __launch_bounds__(256, 2) k_sc_eval_g(ScBatch batch, size_t len, const u256* __restrict__ E, u256* partials, unsigned int* counters,
                                                              u256* out, HostSig sig, const __grid_constant__ XRank xr) {
  const ScInst& in = batch.inst[blockIdx.y];
  const size_t half = len >> 1;
  u256 acc[2] = {fq_zero(), fq_zero()};
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
    const u256 a0 = ld256(in.t[0] + i), a1 = ld256(in.t[0] + i + half), b0 = ld256(in.t[1] + i), b1 = ld256(in.t[1] + i + half);
    const u256 w = ld256_ro(E + i);
    acc[0] = fq_add(acc[0], fq_mul(w, fq_mul(a0, b0)));
    acc[1] = fq_add(acc[1], fq_mul(w, fq_mul(fq_sub(a1, a0), fq_sub(b1, b0))));
  }
  block_reduce_finish<2>(acc, partials, counters, out, 3, sig, xr);
}
// fused: bind A and B with r (len -> len/2, in place, constant-multiplier fold) and evaluate the next round's q(0), q(inf) with the weights
// E = eq(tau[j+2..], .) of len/4 entries
__global__ void __launch_bounds__(256, 2) k_sc_fold_eval_g(ScBatch batch, size_t len, const __grid_constant__ FqConst rc, const u256* __restrict__ E,
                                                                   u256* partials, unsigned int* counters, u256* out, HostSig sig, const __grid_constant__ XRank xr) {
  const ScInst& in = batch.inst[blockIdx.y];
  const size_t half = len >> 1, quarter = len >> 2;
  u256 acc[2] = {fq_zero(), fq_zero()};
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < quarter; i += (size_t)gridDim.x * blockDim.x) {
    u256 lo[2], hi[2];
#pragma unroll
    for (int t = 0; t < 2; t++) {
      const u256 a0 = ld256(in.t[t] + i), a1 = ld256(in.t[t] + i + half), b0 = ld256(in.t[t] + i + quarter), b1 = ld256(in.t[t] + i + quarter + half);
      lo[t] = fq_fold_const(a0, a1, rc);   // dense_mlpoly.rs:218
      hi[t] = fq_fold_const(b0, b1, rc);
      st256(in.t[t] + i, lo[t]); st256(in.t[t] + i + quarter, hi[t]);
    }
    const u256 w = ld256_ro(E + i);
    acc[0] = fq_add(acc[0], fq_mul(w, fq_mul(lo[0], lo[1])));
    acc[1] = fq_add(acc[1], fq_mul(w, fq_mul(fq_sub(hi[0], lo[0]), fq_sub(hi[1], lo[1]))));
  }
  block_reduce_finish<2>(acc, partials, counters, out, 3, sig, xr);
}
// suffix tables below E0 = eq(tau[1..], .) (n0 entries): level k (1 <= k <= K) = eq(tau[k+1..], .) = sum over the top k index bits of E0
// (eq(tau_i, 0) + eq(tau_i, 1) = 1), n0 >> k entries, stored back to back in `levels`
__global__ void __launch_bounds__(256) k_eq_suffix(u256* levels, const u256* __restrict__ E0, size_t n0, int K) {
  size_t total = 0;
  for (int k = 1; k <= K; k++) total += n0 >> k;
  for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (size_t)gridDim.x * blockDim.x) {
    size_t off = 0, y = g;
    int k = 1;
    while (y >= (n0 >> k)) { y -= n0 >> k; off += n0 >> k; k++; }
    const size_t sz = n0 >> k;
    u256 acc = fq_zero();
    for (size_t b = 0; b < ((size_t)1 << k); b++) acc = fq_add(acc, ld256_ro(E0 + b * sz + y));
    st256(levels + off + y, acc);
  }
}

// Small tables (len/4 <= SC_SMALL_MAX): the round's latency, not its throughput, is what the prover waits for, so the work of one index is
// spread over 2*NT threads for the bind step (one multiplication deep) and 3 threads for the evaluations (two deep), exchanging the bound
// values through shared memory, instead of one thread running all 14 multiplications back to back.  Same arithmetic, same results.
#define SC_SMALL_Q 64
#define SC_SMALL_MAX 1024
// host_bound (len == 4 only): the bound two-entry tables also go to the host, host_bound[inst * 2 NT + 2 t + h] = table t's entry h, ordered before
// the flag like the evaluations, so the host can bind the last variable itself and skip a fold and a gather launch and their round trip.
template <int KIND>
__global__ void __launch_bounds__(SC_SMALL_Q * 8) k_sc_fold_eval_small(ScBatch batch, size_t len, const __grid_constant__ FqConst rc, u256* partials,
                                                                     unsigned int* counters, u256* out, HostSig sig, u256* host_bound) {
  constexpr int NT = KIND == SC_QUAD ? 2 : (KIND == SC_CUBIC3 ? 3 : 4);
  constexpr int NP = KIND == SC_QUAD ? 2 : 3;   // evaluation points 0, 2 (, 3)
  __shared__ u256 sh[NT][2][SC_SMALL_Q];
  const ScInst& in = batch.inst[blockIdx.y];
  const size_t half = len >> 1, quarter = len >> 2;
  const int e = threadIdx.x % SC_SMALL_Q, th = threadIdx.x / SC_SMALL_Q;
  const size_t i = (size_t)blockIdx.x * SC_SMALL_Q + e;
  const bool valid = i < quarter;
  if (valid && th < 2 * NT) {
    const int t = th >> 1, h = th & 1;
    const size_t idx = i + (h ? quarter : 0);
    u256 x0 = ld256(in.t[t] + idx), x1 = ld256(in.t[t] + idx + half);
    u256 v = fq_fold_const(x0, x1, rc);   // dense_mlpoly.rs:218
    if (t == 2) { if (in.write_c) st256(in.c_out + idx, v); }
    else st256(in.t[t] + idx, v);
    if (host_bound) st256(&host_bound[(size_t)blockIdx.y * 2 * NT + 2 * t + h], v);
    sh[t][h][e] = v;
  }
  __syncthreads();
  u256 val = fq_zero();
  if (valid && th < NP) {
    u256 x[4];
#pragma unroll
    for (int t = 0; t < 4; t++) x[t] = fq_zero();
#pragma unroll
    for (int t = 0; t < NT; t++) {
      u256 lo = sh[t][0][e], hi = sh[t][1][e];
      if (th == 0) x[t] = lo;                                            // t = 0
      else {
        u256 dl = fq_sub(hi, lo);
        x[t] = fq_add(hi, dl);                                           // t = 2: 2*hi - lo
        if (th == 2) x[t] = fq_add(x[t], dl);                            // t = 3
      }
    }
    val = sc_comb<KIND>(x[0], x[1], x[2], x[3]);
  }
  // Reduction: point p lives in warps 2p, 2p+1 (SC_SMALL_Q = 64), so one value per thread; blocks of one instance meet through the
  // ticket counter as in block_reduce_finish, and the last block of the last instance publishes the flag.
  __shared__ u256 ws[8];
  __shared__ bool is_last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, tid = threadIdx.x;
  if (warp < 2 * NP) { u256 v = warp_sum_fq(val); if (lane == 0) ws[warp] = v; }
  __syncthreads();
  u256 res = fq_zero();
  if (tid < NP) res = fq_add(ws[2 * tid], ws[2 * tid + 1]);
  if (gridDim.x > 1) {
    if (tid < 3) { st256(&partials[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 3 + tid], res); __threadfence(); }
    __syncthreads();
    if (tid == 0) is_last = atomicAdd(&counters[blockIdx.y], 1u) == gridDim.x - 1;
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    if (warp < 3) {   // warp k sums value k over the blocks (gridDim.x <= 16 here: one load per lane)
      u256 v = fq_zero();
      for (unsigned int b = lane; b < gridDim.x; b += 32) v = fq_add(v, ld256_cg(&partials[((size_t)blockIdx.y * gridDim.x + b) * 3 + warp]));
      v = warp_sum_fq(v);
      if (lane == 0) ws[warp] = v;
    }
    __syncthreads();
    if (tid < 3) res = ws[tid];
  }
  if (tid < 3) {
    st256(&out[(size_t)blockIdx.y * 3 + tid], res);
    if (sig.host_out) st256(&sig.host_out[(size_t)blockIdx.y * 3 + tid], res);
  }
  __syncthreads();
  if (tid == 0) {
    if (gridDim.x > 1) counters[blockIdx.y] = 0;
    if (sig.flag) {
      __threadfence_system();   // cumulative: orders the three stores above (joined through the barrier) before the flag
      bool publish = true;
      if (gridDim.y > 1) {
        unsigned int done = atomicAdd(sig.done, 1u) + 1;
        publish = done == gridDim.y;
        if (publish) { *sig.done = 0; __threadfence_system(); }
      }
      if (publish) *((volatile unsigned int*)sig.flag) = sig.seq;
    }
  }
}

// ---- sumcheck of a caller-defined polynomial (dev.hpp: ScPoly).  The factor indices are runtime values, and registers cannot be indexed at
// run time without going to local memory, so a thread keeps the bound points of every table (x_k, advanced point by point) and their steps
// d_k = hi - lo in its own column of dynamic shared memory, [x | d][ntables][SCP_THREADS]; the D accumulators (one per evaluation point) stay in
// registers.  Columns are private to their thread: no barrier.
#define SCP_THREADS 128
__device__ __forceinline__ u256 scp_comb(const ScPoly& P, const u256* x) {
  u256 sum = fq_zero();
  for (int t = 0; t < P.nterms; t++) {
    u256 prod = ld256(x + P.fac[t][0] * SCP_THREADS);
    for (int f = 1; f < P.nfac[t]; f++) prod = fq_mul(prod, ld256(x + P.fac[t][f] * SCP_THREADS));
    if (!P.unit[t]) prod = fq_mul(prod, P.coeff[t]);
    sum = fq_add(sum, prod);
  }
  return sum;
}
// x holds the low halves (t = 0) on entry; the points t = 2, 3, .., D follow as x + t*d, built by additions like sumcheck.rs:209-221
template <int D>
__device__ __forceinline__ void scp_accumulate(u256 (&acc)[D], const ScPoly& P, u256* x, const u256* d) {
  acc[0] = fq_add(acc[0], scp_comb(P, x));
#pragma unroll
  for (int p = 1; p < D; p++) {
    for (int k = 0; k < P.ntables; k++) {
      const u256 dk = ld256(d + k * SCP_THREADS);
      u256 xk = fq_add(ld256(x + k * SCP_THREADS), dk);
      if (p == 1) xk = fq_add(xk, dk);   // from t = 0 straight to t = 2
      st256(x + k * SCP_THREADS, xk);
    }
    acc[p] = fq_add(acc[p], scp_comb(P, x));
  }
}
template <int D>
__global__ void __launch_bounds__(SCP_THREADS, 4) k_scp_eval(const __grid_constant__ ScPoly P, size_t len, u256* partials, unsigned int* counters,
                                                            u256* out, HostSig sig) {
  extern __shared__ uint4 scp_sh[];
  u256* x = reinterpret_cast<u256*>(scp_sh) + threadIdx.x;
  u256* d = x + P.ntables * SCP_THREADS;
  const size_t half = len >> 1;
  u256 acc[D];
#pragma unroll
  for (int p = 0; p < D; p++) acc[p] = fq_zero();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
    for (int k = 0; k < P.ntables; k++) {
      const u256 lo = ld256(P.t[k] + i), hi = ld256(P.t[k] + i + half);
      st256(x + k * SCP_THREADS, lo);
      st256(d + k * SCP_THREADS, fq_sub(hi, lo));
    }
    scp_accumulate<D>(acc, P, x, d);
  }
  block_reduce_finish<D>(acc, partials, counters, out, D, sig);
}
// fused: bind every table with r (len -> len/2, in place) and evaluate the next round, with k_sc_fold_eval's ownership of four elements per thread
template <int D>
__global__ void __launch_bounds__(SCP_THREADS, 4) k_scp_fold_eval(const __grid_constant__ ScPoly P, size_t len, const __grid_constant__ FqConst rc,
                                                                 u256* partials, unsigned int* counters, u256* out, HostSig sig) {
  extern __shared__ uint4 scp_sh[];
  u256* x = reinterpret_cast<u256*>(scp_sh) + threadIdx.x;
  u256* d = x + P.ntables * SCP_THREADS;
  const size_t half = len >> 1, quarter = len >> 2;
  u256 acc[D];
#pragma unroll
  for (int p = 0; p < D; p++) acc[p] = fq_zero();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < quarter; i += (size_t)gridDim.x * blockDim.x) {
    for (int k = 0; k < P.ntables; k++) {
      u256* T = P.t[k];
      const u256 lo = fq_fold_const(ld256(T + i), ld256(T + i + half), rc);   // dense_mlpoly.rs:218
      const u256 hi = fq_fold_const(ld256(T + i + quarter), ld256(T + i + quarter + half), rc);
      st256(T + i, lo); st256(T + i + quarter, hi);
      st256(x + k * SCP_THREADS, lo);
      st256(d + k * SCP_THREADS, fq_sub(hi, lo));
    }
    scp_accumulate<D>(acc, P, x, d);
  }
  block_reduce_finish<D>(acc, partials, counters, out, D, sig);
}
// Small tables (len/4 <= SC_SMALL_MAX), latency-bound as in k_sc_fold_eval_small: 32 indices per block; warp 2k + h binds half h of table k
// (one fold per thread), then warp p evaluates point p (t = 0 for p = 0, else p + 1) from the bound values in shared memory.
#define SCP_SMALL_Q 32
__device__ __forceinline__ u256 scp_small_point(const u256 (&sh)[SP_SC_MAX_TABLES][2][SCP_SMALL_Q], int k, int e, int tp) {
  const u256 lo = sh[k][0][e];
  if (tp == 0) return lo;
  const u256 hi = sh[k][1][e], dk = fq_sub(hi, lo);
  u256 v = hi;
  for (int s = 1; s < tp; s++) v = fq_add(v, dk);
  return v;
}
template <int D>
__global__ void __launch_bounds__(SCP_SMALL_Q * 2 * SP_SC_MAX_TABLES) k_scp_fold_eval_small(const __grid_constant__ ScPoly P, size_t len,
                                                                                           const __grid_constant__ FqConst rc, u256* partials,
                                                                                           unsigned int* counters, u256* out, HostSig sig) {
  __shared__ u256 sh[SP_SC_MAX_TABLES][2][SCP_SMALL_Q];
  const size_t half = len >> 1, quarter = len >> 2;
  const int e = threadIdx.x % SCP_SMALL_Q, th = threadIdx.x / SCP_SMALL_Q;
  const size_t i = (size_t)blockIdx.x * SCP_SMALL_Q + e;
  const bool valid = i < quarter;
  if (valid && th < 2 * P.ntables) {
    const int k = th >> 1, h = th & 1;
    const size_t idx = i + (h ? quarter : 0);
    const u256 v = fq_fold_const(ld256(P.t[k] + idx), ld256(P.t[k] + idx + half), rc);   // dense_mlpoly.rs:218
    st256(P.t[k] + idx, v);
    sh[k][h][e] = v;
  }
  __syncthreads();
  u256 acc[D];
#pragma unroll
  for (int p = 0; p < D; p++) acc[p] = fq_zero();
  if (valid && th < D) {
    const int tp = th == 0 ? 0 : th + 1;
    u256 sum = fq_zero();
    for (int t = 0; t < P.nterms; t++) {
      u256 prod = scp_small_point(sh, P.fac[t][0], e, tp);
      for (int f = 1; f < P.nfac[t]; f++) prod = fq_mul(prod, scp_small_point(sh, P.fac[t][f], e, tp));
      if (!P.unit[t]) prod = fq_mul(prod, P.coeff[t]);
      sum = fq_add(sum, prod);
    }
#pragma unroll
    for (int p = 0; p < D; p++)
      if (p == th) acc[p] = sum;
  }
  block_reduce_finish<D>(acc, partials, counters, out, D, sig);
}

struct FoldBatch {
  u256* t[64];
};
__global__ void __launch_bounds__(256) k_fold_top(FoldBatch tabs, size_t len, const __grid_constant__ FqConst rc) {
  const size_t half = len >> 1;
  u256* T = tabs.t[blockIdx.y];
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
    u256 a0 = ld256(T + i), a1 = ld256(T + i + half);
    st256(T + i, fq_fold_const(a0, a1, rc));   // dense_mlpoly.rs:218
  }
}

// scratch layout: [counters: 64 x u32][partials]
static const size_t SC_MAX_BLOCKS = 132 * 6 + 64;   // 6 CTAs on each of an H100's 132 SMs; larger grids are capped to it
size_t sc_scratch_bytes(int ninst) { return 256 + (size_t)ninst * SC_MAX_BLOCKS * 3 * sizeof(u256); }

// algorithmic bytes of one launch: every DISTINCT table is streamed once (a C table shared by several instances of a batched sumcheck counts
// once, not once per instance): `per_elem` bytes per entry (32 for an evaluation pass, 48 for the fused bind + evaluate: read 32, write 16 per input entry)
static double sc_bytes(const ScInst* insts, int ninst, ScKind kind, size_t len, double per_elem) {
  const int nt = kind == SC_QUAD ? 2 : kind == SC_CUBIC3 ? 3 : 4;
  const u256* seen[SC_MAX_INST * 4];
  int ns = 0;
  if (ninst > SC_MAX_INST) return 0.0;   // fill_batch rejects the launch
  for (int i = 0; i < ninst; i++)
    for (int t = 0; t < nt; t++) {
      bool dup = false;
      for (int k = 0; k < ns; k++) dup = dup || seen[k] == insts[i].t[t];
      if (!dup) seen[ns++] = insts[i].t[t];
    }
  return (double)ns * (double)len * per_elem;
}
static void fill_batch(ScBatch& b, const ScInst* insts, int ninst) {
  if (ninst > SC_MAX_INST) throw std::runtime_error("spartan_b200: too many sumcheck instances in one batch");
  for (int i = 0; i < ninst; i++) b.inst[i] = insts[i];
}

void sc_eval(ScKind kind, const ScInst* insts, int ninst, size_t len, u256* out, void* scratch, cudaStream_t s, HostSig sig, const XRank& xr) {
  ProfScope ps("sc_eval", sc_bytes(insts, ninst, kind, len, 32.0), s);
  ScBatch b; fill_batch(b, insts, ninst);
  unsigned int* counters = (unsigned int*)scratch;
  u256* partials = (u256*)((char*)scratch + 256);
  dim3 grid(grid_for(len / 2, 256, 2), ninst);
  if (grid.x > SC_MAX_BLOCKS) grid.x = SC_MAX_BLOCKS;
  switch (kind) {
    case SC_QUAD: k_sc_eval<SC_QUAD><<<grid, 256, 0, s>>>(b, len, partials, counters, out, sig, xr); break;
    case SC_CUBIC3: k_sc_eval<SC_CUBIC3><<<grid, 256, 0, s>>>(b, len, partials, counters, out, sig, xr); break;
    default: k_sc_eval<SC_CUBIC4><<<grid, 256, 0, s>>>(b, len, partials, counters, out, sig, xr); break;
  }
  SP_LAUNCHED(); check("sc_eval");
}
void sc_fold_eval(ScKind kind, const ScInst* insts, int ninst, size_t len, const u256& r, u256* out, void* scratch, cudaStream_t s, HostSig sig, const XRank& xr,
                  u256* host_bound) {
  if (xr.world > 1 && (len / 4 <= SC_SMALL_MAX || !sig.done)) throw std::runtime_error("spartan_b200: a sharded sumcheck round needs a streaming-size table and a completion counter");
  if (host_bound && (len != 4 || !sig.flag)) throw std::runtime_error("spartan_b200: only a signalled fold to two-entry tables publishes them");
  // two kernels, two profiler families: the streaming kernel (HBM roofline) and the latency-bound small-table kernel (k_sc_fold_eval_small)
  const bool small = len / 4 <= SC_SMALL_MAX && len >= 4;
  ProfScope ps(small ? "sc_fold_eval_small" : "sc_fold_eval", sc_bytes(insts, ninst, kind, len, 48.0), s);
  ScBatch b; fill_batch(b, insts, ninst);
  unsigned int* counters = (unsigned int*)scratch;
  u256* partials = (u256*)((char*)scratch + 256);
  const FqConst rc = fq_const_table(r);
  if (small) {
    dim3 grid((unsigned)((len / 4 + SC_SMALL_Q - 1) / SC_SMALL_Q), ninst);
    switch (kind) {
      case SC_QUAD: k_sc_fold_eval_small<SC_QUAD><<<grid, SC_SMALL_Q * 4, 0, s>>>(b, len, rc, partials, counters, out, sig, host_bound); break;
      case SC_CUBIC3: k_sc_fold_eval_small<SC_CUBIC3><<<grid, SC_SMALL_Q * 6, 0, s>>>(b, len, rc, partials, counters, out, sig, host_bound); break;
      default: k_sc_fold_eval_small<SC_CUBIC4><<<grid, SC_SMALL_Q * 8, 0, s>>>(b, len, rc, partials, counters, out, sig, host_bound); break;
    }
    SP_LAUNCHED(); check("sc_fold_eval_small");
    return;
  }
  dim3 grid(grid_for(len / 4, 256, 2), ninst);
  if (grid.x > SC_MAX_BLOCKS) grid.x = SC_MAX_BLOCKS;
  switch (kind) {
    case SC_QUAD: k_sc_fold_eval<SC_QUAD><<<grid, 256, 0, s>>>(b, len, rc, partials, counters, out, sig, xr); break;
    case SC_CUBIC3: k_sc_fold_eval<SC_CUBIC3><<<grid, 256, 0, s>>>(b, len, rc, partials, counters, out, sig, xr); break;
    default: k_sc_fold_eval<SC_CUBIC4><<<grid, 256, 0, s>>>(b, len, rc, partials, counters, out, sig, xr); break;
  }
  SP_LAUNCHED(); check("sc_fold_eval");
}
void sc_eval_g(const ScInst* insts, int ninst, size_t len, const u256* E, u256* out, void* scratch, cudaStream_t s, HostSig sig, const XRank& xr) {
  ProfScope ps("sc_eval", (double)ninst * 2.0 * (double)len * 32.0 + (double)len * 16.0, s);
  ScBatch b; fill_batch(b, insts, ninst);
  unsigned int* counters = (unsigned int*)scratch;
  u256* partials = (u256*)((char*)scratch + 256);
  dim3 grid(grid_for(len / 2, 256, 2), ninst);
  if (grid.x > SC_MAX_BLOCKS) grid.x = SC_MAX_BLOCKS;
  k_sc_eval_g<<<grid, 256, 0, s>>>(b, len, E, partials, counters, out, sig, xr);
  SP_LAUNCHED(); check("sc_eval_g");
}
void sc_fold_eval_g(const ScInst* insts, int ninst, size_t len, const u256& r, const u256* E, u256* out, void* scratch, cudaStream_t s, HostSig sig, const XRank& xr) {
  if (len / 4 <= SC_SMALL_MAX) throw std::runtime_error("spartan_b200: sc_fold_eval_g is a streaming kernel");
  if (xr.world > 1 && !sig.done) throw std::runtime_error("spartan_b200: a sharded sumcheck round needs a completion counter");
  ProfScope ps("sc_fold_eval", (double)ninst * 2.0 * (double)len * 48.0 + (double)len * 8.0, s);
  ScBatch b; fill_batch(b, insts, ninst);
  unsigned int* counters = (unsigned int*)scratch;
  u256* partials = (u256*)((char*)scratch + 256);
  const FqConst rc = fq_const_table(r);
  dim3 grid(grid_for(len / 4, 256, 2), ninst);
  if (grid.x > SC_MAX_BLOCKS) grid.x = SC_MAX_BLOCKS;
  k_sc_fold_eval_g<<<grid, 256, 0, s>>>(b, len, rc, E, partials, counters, out, sig, xr);
  SP_LAUNCHED(); check("sc_fold_eval_g");
}
// rc == null: the first round (k_scp_eval); else the fused bind + evaluate, in its small-table form for len/4 <= SC_SMALL_MAX
template <int D>
static void scp_launch(const ScPoly& P, size_t len, const FqConst* rc, u256* out, void* scratch, cudaStream_t s, HostSig sig) {
  unsigned int* counters = (unsigned int*)scratch;
  u256* partials = (u256*)((char*)scratch + 256);
  if (rc && len / 4 <= SC_SMALL_MAX) {
    const int nth = 2 * P.ntables > D ? 2 * P.ntables : D;
    k_scp_fold_eval_small<D><<<(unsigned)((len / 4 + SCP_SMALL_Q - 1) / SCP_SMALL_Q), SCP_SMALL_Q * nth, 0, s>>>(P, len, *rc, partials, counters, out, sig);
    return;
  }
  const size_t smem = 2 * (size_t)P.ntables * SCP_THREADS * sizeof(u256);   // up to 64 KB: above the default 48 KB opt-in
  const void* fn = rc ? (const void*)k_scp_fold_eval<D> : (const void*)k_scp_eval<D>;
  if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) check("scp shared memory");
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, SCP_THREADS, smem) != cudaSuccess) check("scp occupancy");
  dim3 grid(grid_for(rc ? len / 4 : len / 2, SCP_THREADS, per_sm > 0 ? per_sm : 1));
  if (grid.x > SC_MAX_BLOCKS) grid.x = SC_MAX_BLOCKS;
  if (rc) k_scp_fold_eval<D><<<grid, SCP_THREADS, smem, s>>>(P, len, *rc, partials, counters, out, sig);
  else k_scp_eval<D><<<grid, SCP_THREADS, smem, s>>>(P, len, partials, counters, out, sig);
}
static void scp_dispatch(const ScPoly& P, size_t len, const FqConst* rc, u256* out, void* scratch, cudaStream_t s, HostSig sig) {
  if (P.ntables < 1 || P.ntables > SP_SC_MAX_TABLES || P.nterms < 1 || P.nterms > SP_SC_MAX_TERMS)
    throw std::runtime_error("spartan_b200: sumcheck polynomial outside the kernel's limits");
  switch (P.degree) {
    case 1: scp_launch<1>(P, len, rc, out, scratch, s, sig); break;
    case 2: scp_launch<2>(P, len, rc, out, scratch, s, sig); break;
    case 3: scp_launch<3>(P, len, rc, out, scratch, s, sig); break;
    case 4: scp_launch<4>(P, len, rc, out, scratch, s, sig); break;
    case 5: scp_launch<5>(P, len, rc, out, scratch, s, sig); break;
    case 6: scp_launch<6>(P, len, rc, out, scratch, s, sig); break;
    default: throw std::runtime_error("spartan_b200: sumcheck polynomial degree outside 1.." + std::to_string(SP_SC_MAX_DEGREE));
  }
  SP_LAUNCHED();
}
void scp_eval(const ScPoly& p, size_t len, u256* out, void* scratch, cudaStream_t s, HostSig sig) {
  ProfScope ps("scp_eval", (double)p.ntables * (double)len * 32.0, s);
  scp_dispatch(p, len, nullptr, out, scratch, s, sig);
  check("scp_eval");
}
void scp_fold_eval(const ScPoly& p, size_t len, const u256& r, u256* out, void* scratch, cudaStream_t s, HostSig sig) {
  if (len < 4) throw std::runtime_error("spartan_b200: scp_fold_eval needs tables of at least four entries");
  ProfScope ps(len / 4 <= SC_SMALL_MAX ? "scp_fold_eval_small" : "scp_fold_eval", (double)p.ntables * (double)len * 48.0, s);
  const FqConst rc = fq_const_table(r);
  scp_dispatch(p, len, &rc, out, scratch, s, sig);
  check("scp_fold_eval");
}
static size_t eq_suffix_entries(size_t n0, int K) { size_t t = 0; for (int k = 1; k <= K; k++) t += n0 >> k; return t; }
void eq_suffix(u256* levels, const u256* E0, size_t n0, int K, cudaStream_t s) {
  if (K < 1) return;
  ProfScope ps("eq_evals", 64.0 * (double)n0, s);
  k_eq_suffix<<<grid_for(eq_suffix_entries(n0, K), 256, 4), 256, 0, s>>>(levels, E0, n0, K);
  SP_LAUNCHED(); check("eq_suffix");
}
void fold_top(u256* const* tables, int ntables, size_t len, const u256& r, cudaStream_t s) {
  ProfScope ps("fold_top", (double)ntables * len * 48.0, s);
  const FqConst rc = fq_const_table(r);
  for (int base = 0; base < ntables; base += 64) {
    FoldBatch fb; int n = ntables - base < 64 ? ntables - base : 64;
    for (int i = 0; i < n; i++) fb.t[i] = tables[base + i];
    dim3 grid(grid_for(len / 2, 256, 4), n);
    k_fold_top<<<grid, 256, 0, s>>>(fb, len, rc);
    SP_LAUNCHED();
  }
  check("fold_top");
}

}  // namespace dev
}  // namespace sp
