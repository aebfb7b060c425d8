// spartan_b200 — variable-base multiscalar multiplication on arbitrary ristretto points (bucket method), sm_90a.
//
// Replaces GroupElement::vartime_multiscalar_mul (/root/reference/src/group.rs:98-117) -> dalek Pippenger for inputs that are NOT a fixed
// generator set (BASELINE config "standalone MSM, N = 2^24"; SURVEY.md §8 a7/(d) config 3).  The prover itself commits against fixed
// generators and uses the window tables of kernels.cu; this path is for callers that bring their own points.
//
// Pipeline for N points, c-bit signed windows (NB = 2^(c-1) buckets per window, NWIN = floor(253/c)+1 windows):
//   k_pip_prepare    scalars leave Montgomery form (group.rs:110-113); k' = k + C with C = sum_{w<NWIN-1} 2^(c-1+cw) makes every window's
//                    signed digit independent of its neighbours: d_w = ((k' >> cw) & (2^c-1)) - 2^(c-1); the top window stays unsigned.
//                    k' is stored limb-major (8 arrays of N words) so every later pass reads it coalesced.
//   k_pip_count      grid (tiles, NWIN): shared-memory histogram of |d_w| per tile, flushed with one global atomic per non-empty bucket
//   k_pip_scan       per window: exclusive scan of bucket sizes -> bucket start, and of ceil(size/S) -> first work item of the bucket
//   k_pip_scatter    same tiling: reserve a range per (tile,bucket) with one global atomic, then rank inside the tile with shared atomics;
//                    writes point index | sign<<31.  Order inside a bucket is arbitrary — point addition commutes and the final
//                    ristretto encoding is canonical, so the output bytes are deterministic.
//   k_pip_accumulate one warp per work item (<= S consecutive entries of one bucket): coalesced index loads, 96-byte affine-niels gathers,
//                    7M mixed additions per lane, shuffle-tree over the warp
//   k_pip_bucket_sum one warp per bucket sums its items' partial points
//   k_pip_window     per window: sum_b (b+1)*B_b by chunked running sums (+ a <=15-bit scalar multiple per chunk), then c*w doublings
//   k_pip_final      sum of the window points
// HBM traffic: 32 B (scalar) + NWIN * (4 B index + 96 B point) per term; the kernel is ALU-bound (NWIN mixed additions per term).
#include "field.cuh"
#include "curve.cuh"
#include "kcommon.cuh"

namespace sp {
namespace dev {

void check(const char* what);

__device__ __forceinline__ ge ld_ge_p(const ge* p) {
  ge r;
  r.X = ld256(&p->X); r.Y = ld256(&p->Y); r.Z = ld256(&p->Z); r.T = ld256(&p->T);
  return r;
}
__device__ __forceinline__ void st_ge_p(ge* p, const ge& g) { st256(&p->X, g.X); st256(&p->Y, g.Y); st256(&p->Z, g.Z); st256(&p->T, g.T); }
__device__ __forceinline__ ge shfl_down_ge_p(const ge& p, int delta) {
  ge r;
  r.X = shfl_down_256(p.X, delta); r.Y = shfl_down_256(p.Y, delta); r.Z = shfl_down_256(p.Z, delta); r.T = shfl_down_256(p.T, delta);
  return r;
}
__device__ __forceinline__ ge warp_sum_ge(ge acc) {
#pragma unroll 1
  for (int d = 16; d > 0; d >>= 1) acc = ge_add(acc, shfl_down_ge_p(acc, d));
  return acc;
}

__global__ void k_points_to_niels(ge_niels* out, const ge* __restrict__ in, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  ge_niels q = ge_to_niels(ld_ge_p(in + i));
  st256(&out[i].ypx, q.ypx); st256(&out[i].ymx, q.ymx); st256(&out[i].t2d, q.t2d);
}
void points_to_niels(ge_niels* out, const ge* in, size_t n, cudaStream_t s) {
  if (!n) return;
  k_points_to_niels<<<(unsigned)((n + 63) / 64), 64, 0, s>>>(out, in, n);
  SP_LAUNCHED(); check("points_to_niels");
}

__global__ void k_niels_to_ge(ge* out, const ge_niels* __restrict__ in, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  ge_niels nl;
  nl.ypx = ld256_ro(&in[i].ypx); nl.ymx = ld256_ro(&in[i].ymx); nl.t2d = ld256_ro(&in[i].t2d);
  st_ge_p(out + i, ge_madd(ge_identity(), nl, false));
}
void niels_to_ge(ge* out, const ge_niels* in, size_t n, cudaStream_t s) {
  if (!n) return;
  k_niels_to_ge<<<(unsigned)((n + 63) / 64), 64, 0, s>>>(out, in, n);
  SP_LAUNCHED(); check("niels_to_ge");
}

PipPlan pip_plan(size_t n, int c_override) {
  PipPlan p;
  p.n = n;
  int lg = 0;
  while (((size_t)2 << lg) <= n) lg++;          // floor(log2 n) for n >= 1
  int c = lg - 7;
  if (c < 6) c = 6;
  if (c > 16) c = 16;
  if (c_override) c = c_override;
  if (c < 2 || c > 16) throw std::runtime_error("spartan_b200: MSM window width out of range");
  p.c = c;
  p.nwin = 253 / c + 1;
  p.nb = 1u << (c - 1);
  // tiles of 4*nb scalars (for c = 13..16: many blocks in flight beat amortising the nb-word flush further)
  size_t tile = (size_t)p.nb * 4;
  if (tile < 8192) tile = 8192;
  p.tile = tile;
  p.ntiles = (n + tile - 1) / tile;
  if (!p.ntiles) p.ntiles = 1;
  // work items: at most S consecutive entries of one bucket, summed by G lanes.  G is sized so a lane gets ~64 additions from an average
  // bucket (n/nb entries), S so that an oversized bucket (skewed scalars) is split across items
  int G = 32;
  while (G > 1 && (n / p.nb) / (size_t)G < 64) G >>= 1;
  p.G = G;
  size_t S = 2 * (n / p.nb);
  if (S < (size_t)G * 64) S = (size_t)G * 64;
  S = (S + 31) / 32 * 32;
  if (S > 8192) S = 8192;
  p.S = S;
  p.max_items = n / S + p.nb + 1;
  return p;
}
static size_t al256(size_t b) { return (b + 255) / 256 * 256; }
struct PipLayout {
  size_t kp, sorted, counts, tile_hist, start, cursor, istart, nitems, partial, buckets, wins, total;
};
static PipLayout pip_layout(const PipPlan& p) {
  PipLayout L;
  size_t o = 0;
  L.kp = o; o += al256(8 * p.n * 4);
  L.sorted = o; o += al256((size_t)p.nwin * p.n * 4);
  L.counts = o; o += al256((size_t)p.nwin * p.nb * 4);
  L.tile_hist = o; o += al256((size_t)p.nwin * p.ntiles * p.nb * 4);
  L.start = o; o += al256((size_t)p.nwin * p.nb * 4);
  L.cursor = o; o += al256((size_t)p.nwin * p.nb * 4);
  L.istart = o; o += al256((size_t)p.nwin * (p.nb + 1) * 4);
  L.nitems = o; o += al256((size_t)p.nwin * 4);
  L.partial = o; o += al256((size_t)p.nwin * p.max_items * sizeof(ge));
  L.buckets = o; o += al256((size_t)p.nwin * p.nb * sizeof(ge));
  L.wins = o; o += al256((size_t)p.nwin * sizeof(ge));
  L.total = o;
  return L;
}
size_t pip_scratch_bytes(const PipPlan& p) { return pip_layout(p).total; }

__global__ void __launch_bounds__(256) k_pip_prepare(uint32_t* __restrict__ kp, const u256* __restrict__ scalars, size_t n, const u256 C) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  u256 k = fq_from_mont(ld256_ro(scalars + i));
  uint64_t carry = 0;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    uint64_t t = (uint64_t)k.v[j] + C.v[j] + carry;
    kp[(size_t)j * n + i] = (uint32_t)t;
    carry = t >> 32;
  }
}

constexpr int PIP_UNROLL = 8;
// signed digit of window w: 0 = skip, else bucket |d|-1 and sign
__device__ __forceinline__ int pip_digit(const uint32_t* __restrict__ kp, size_t n, size_t i, int w, int c, int nwin) {
  const int b = w * c, limb = b >> 5, sh = b & 31;
  uint32_t v = kp[(size_t)limb * n + i] >> sh;
  if (sh + c > 32 && limb + 1 < 8) v |= kp[(size_t)(limb + 1) * n + i] << (32 - sh);
  v &= (1u << c) - 1u;
  return w + 1 < nwin ? (int)v - (1 << (c - 1)) : (int)v;
}

__global__ void __launch_bounds__(1024) k_pip_count(uint32_t* __restrict__ counts, uint32_t* __restrict__ tile_hist, const uint32_t* __restrict__ kp, size_t n,
                                                   size_t tile, int c, int nwin, uint32_t nb) {
  extern __shared__ uint32_t hist[];
  const int w = blockIdx.y;
  for (uint32_t b = threadIdx.x; b < nb; b += blockDim.x) hist[b] = 0;
  __syncthreads();
  const size_t lo = (size_t)blockIdx.x * tile, hi = lo + tile < n ? lo + tile : n;
  for (size_t i0 = lo + threadIdx.x; i0 < hi; i0 += (size_t)PIP_UNROLL * blockDim.x) {   // PIP_UNROLL independent loads in flight per thread
    int d[PIP_UNROLL];
#pragma unroll
    for (int u = 0; u < PIP_UNROLL; u++) { size_t i = i0 + (size_t)u * blockDim.x; d[u] = i < hi ? pip_digit(kp, n, i, w, c, nwin) : 0; }
#pragma unroll
    for (int u = 0; u < PIP_UNROLL; u++) if (d[u]) atomicAdd(&hist[(d[u] < 0 ? -d[u] : d[u]) - 1], 1u);
  }
  __syncthreads();
  uint32_t* th = tile_hist + ((size_t)w * gridDim.x + blockIdx.x) * nb;   // kept for the scatter pass (saves recounting the tile)
  for (uint32_t b = threadIdx.x; b < nb; b += blockDim.x) {
    uint32_t h = hist[b];
    th[b] = h;
    if (h) atomicAdd(&counts[(size_t)w * nb + b], h);
  }
}

// one block per window: start[b] = sum_{b'<b} counts[b'], istart[b] = sum_{b'<b} ceil(counts[b']/S); cursor = start; nitems = total items
__global__ void __launch_bounds__(1024) k_pip_scan(uint32_t* __restrict__ start, uint32_t* __restrict__ cursor, uint32_t* __restrict__ istart,
                                                  uint32_t* __restrict__ nitems, const uint32_t* __restrict__ counts, uint32_t nb, uint32_t S) {
  __shared__ uint32_t sa[1024], sb[1024];
  const int w = blockIdx.x, t = threadIdx.x;
  const uint32_t per = (nb + 1023) / 1024;
  const uint32_t lo = t * per, hi = lo + per < nb ? lo + per : nb;
  const uint32_t* cw = counts + (size_t)w * nb;
  uint32_t a = 0, b = 0;
  for (uint32_t i = lo; i < hi; i++) { uint32_t x = cw[i]; a += x; b += (x + S - 1) / S; }
  sa[t] = a; sb[t] = b;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {   // Hillis-Steele inclusive scan
    uint32_t xa = t >= d ? sa[t - d] : 0, xb = t >= d ? sb[t - d] : 0;
    __syncthreads();
    sa[t] += xa; sb[t] += xb;
    __syncthreads();
  }
  uint32_t ra = sa[t] - a, rb = sb[t] - b;   // exclusive
  for (uint32_t i = lo; i < hi; i++) {
    uint32_t x = cw[i];
    start[(size_t)w * nb + i] = ra; cursor[(size_t)w * nb + i] = ra; istart[(size_t)w * (nb + 1) + i] = rb;
    ra += x; rb += (x + S - 1) / S;
  }
  if (t == 1023) { istart[(size_t)w * (nb + 1) + nb] = sb[1023]; nitems[w] = sb[1023]; }
}

__global__ void __launch_bounds__(1024) k_pip_scatter(uint32_t* __restrict__ sorted, uint32_t* __restrict__ cursor, const uint32_t* __restrict__ tile_hist,
                                                     const uint32_t* __restrict__ kp, size_t n, size_t tile, int c, int nwin, uint32_t nb) {
  extern __shared__ uint32_t hist[];
  const int w = blockIdx.y;
  const uint32_t* th = tile_hist + ((size_t)w * gridDim.x + blockIdx.x) * nb;
  for (uint32_t b = threadIdx.x; b < nb; b += blockDim.x) {
    uint32_t h = th[b];
    hist[b] = h ? atomicAdd(&cursor[(size_t)w * nb + b], h) : 0u;   // this tile's range inside the bucket
  }
  __syncthreads();
  const size_t lo = (size_t)blockIdx.x * tile, hi = lo + tile < n ? lo + tile : n;
  uint32_t* out = sorted + (size_t)w * n;
  for (size_t i0 = lo + threadIdx.x; i0 < hi; i0 += (size_t)PIP_UNROLL * blockDim.x) {
    int d[PIP_UNROLL];
#pragma unroll
    for (int u = 0; u < PIP_UNROLL; u++) { size_t i = i0 + (size_t)u * blockDim.x; d[u] = i < hi ? pip_digit(kp, n, i, w, c, nwin) : 0; }
#pragma unroll
    for (int u = 0; u < PIP_UNROLL; u++) if (d[u]) {
      uint32_t pos = atomicAdd(&hist[(d[u] < 0 ? -d[u] : d[u]) - 1], 1u);
      out[pos] = (uint32_t)(i0 + (size_t)u * blockDim.x) | (d[u] < 0 ? 0x80000000u : 0u);
    }
  }
}

// G = lanes per work item (power of two <= 32): few lanes when buckets are small, so the shuffle tree (log2 G additions) stays a small
// fraction of the item's mixed additions
__global__ void __launch_bounds__(128, 4) k_pip_accumulate(ge* __restrict__ partial, const ge_niels* __restrict__ pts, const uint32_t* __restrict__ sorted,
                                                                  const uint32_t* __restrict__ start, const uint32_t* __restrict__ counts,
                                                                  const uint32_t* __restrict__ istart, const uint32_t* __restrict__ nitems, size_t n, uint32_t nb,
                                                                  uint32_t S, size_t max_items, int G) {
  const int w = blockIdx.y;
  const uint32_t per_block = 128 / G;
  const uint32_t item = blockIdx.x * per_block + threadIdx.x / G;
  const int sub = threadIdx.x & (G - 1);
  const uint32_t total = nitems[w];
  if ((blockIdx.x * per_block + (threadIdx.x & ~31u) / G) >= total) return;   // whole warp past the end
  const bool valid = item < total;
  uint32_t first = 0, last = 0;
  if (valid) {
    const uint32_t* is = istart + (size_t)w * (nb + 1);
    uint32_t lo = 0, hi = nb;   // the bucket b with is[b] <= item < is[b+1]
    while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (is[mid] <= item) lo = mid; else hi = mid; }
    const uint32_t b = lo;
    const uint32_t k = item - is[b];
    first = start[(size_t)w * nb + b] + k * S;
    last = start[(size_t)w * nb + b] + counts[(size_t)w * nb + b];
    if (first + S < last) last = first + S;
  }
  const uint32_t* so = sorted + (size_t)w * n;
  ge acc = ge_identity();
  uint32_t vnext = first + sub < last ? so[first + sub] : 0u;
#pragma unroll 1
  for (uint32_t e = first + sub; e < last; e += G) {
    const uint32_t v = vnext;
    if (e + G < last) {
      vnext = so[e + G];
      const char* nq = reinterpret_cast<const char*>(pts + (vnext & 0x7fffffffu));
      asm volatile("prefetch.global.L2 [%0];" ::"l"(nq));
      asm volatile("prefetch.global.L2 [%0];" ::"l"(nq + 64));
    }
    const ge_niels* q = pts + (v & 0x7fffffffu);
    ge_niels nl;
    nl.ypx = ld256_ro(&q->ypx); nl.ymx = ld256_ro(&q->ymx); nl.t2d = ld256_ro(&q->t2d);
    acc = ge_madd(acc, nl, (v >> 31) != 0);
  }
#pragma unroll 1
  for (int d = G >> 1; d > 0; d >>= 1) acc = ge_add(acc, shfl_down_ge_p(acc, d));   // lane 0 of each group only ever reads inside its group
  if (valid && sub == 0) st_ge_p(partial + (size_t)w * max_items + item, acc);
}

__global__ void __launch_bounds__(128) k_pip_bucket_sum(ge* __restrict__ buckets, const ge* __restrict__ partial, const uint32_t* __restrict__ istart, uint32_t nb,
                                                       size_t max_items) {
  const int w = blockIdx.y, lane = threadIdx.x & 31;
  const uint32_t b = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (b >= nb) return;
  const uint32_t i0 = istart[(size_t)w * (nb + 1) + b], i1 = istart[(size_t)w * (nb + 1) + b + 1];
  const ge* pw = partial + (size_t)w * max_items;
  ge acc = ge_identity();
  if (i1 - i0 == 1) { if (lane == 0) st_ge_p(buckets + (size_t)w * nb + b, ld_ge_p(pw + i0)); return; }
#pragma unroll 1
  for (uint32_t i = i0 + lane; i < i1; i += 32) acc = ge_add(acc, ld_ge_p(pw + i));
  if (i1 - i0 > 1) acc = warp_sum_ge(acc);
  if (lane == 0) st_ge_p(buckets + (size_t)w * nb + b, acc);
}

// one block per window: sum_b (b+1) * B_b, then multiply by 2^(c*w)
__global__ void __launch_bounds__(512) k_pip_window(ge* __restrict__ wins, const ge* __restrict__ buckets, uint32_t nb, int c) {
  __shared__ ge sm[16];
  const int w = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const uint32_t per = (nb + 511) / 512;
  const uint32_t lo = t * per, hi = lo + per < nb ? lo + per : nb;
  ge run = ge_identity(), acc = ge_identity();
  if (lo < nb) {
#pragma unroll 1
    for (uint32_t b = hi; b-- > lo;) { run = ge_add(run, ld_ge_p(buckets + (size_t)w * nb + b)); acc = ge_add(acc, run); }
    // acc = sum (b - lo + 1) B_b ; add lo * run
    if (lo) {
      ge m = ge_identity();
      int top = 31 - __clz(lo);
#pragma unroll 1
      for (int bit = top; bit >= 0; bit--) { m = ge_dbl(m); if ((lo >> bit) & 1u) m = ge_add(m, run); }
      acc = ge_add(acc, m);
    }
  }
  acc = warp_sum_ge(acc);
  if (lane == 0) sm[warp] = acc;
  __syncthreads();
  if (warp == 0) {
    acc = warp_sum_ge(lane < 16 ? sm[lane] : ge_identity());
    if (lane == 0) {
#pragma unroll 1
      for (int i = 0; i < c * w; i++) acc = ge_dbl(acc);
      st_ge_p(wins + w, acc);
    }
  }
}
__global__ void __launch_bounds__(32) k_pip_final(ge* out, const ge* __restrict__ wins, int nwin) {
  ge acc = ge_identity();
  for (int i = threadIdx.x; i < nwin; i += 32) acc = ge_add(acc, ld_ge_p(wins + i));
  acc = warp_sum_ge(acc);
  if (threadIdx.x == 0) st_ge_p(out, acc);
}

void msm_var(ge* out, const ge_niels* pts, const u256* scalars, const PipPlan& p, void* scratch, cudaStream_t s) {
  ProfScope ps("msm_var", 32.0 * (double)p.n + (double)p.nwin * 100.0 * (double)p.n, s);
  if (p.n >= ((size_t)1 << 31)) throw std::runtime_error("spartan_b200: msm_var supports at most 2^31-1 points");
  const PipLayout L = pip_layout(p);
  uint8_t* base = (uint8_t*)scratch;
  uint32_t* kp = (uint32_t*)(base + L.kp);
  uint32_t* sorted = (uint32_t*)(base + L.sorted);
  uint32_t* counts = (uint32_t*)(base + L.counts);
  uint32_t* tile_hist = (uint32_t*)(base + L.tile_hist);
  uint32_t* start = (uint32_t*)(base + L.start);
  uint32_t* cursor = (uint32_t*)(base + L.cursor);
  uint32_t* istart = (uint32_t*)(base + L.istart);
  uint32_t* nitems = (uint32_t*)(base + L.nitems);
  ge* partial = (ge*)(base + L.partial);
  ge* buckets = (ge*)(base + L.buckets);
  ge* wins = (ge*)(base + L.wins);
  if (p.nb * 4 > 48 * 1024) {   // per device and cheap: set whenever the histogram needs the opt-in shared-memory size
    cudaFuncSetAttribute(k_pip_count, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024);
    cudaFuncSetAttribute(k_pip_scatter, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024);
  }
  // C = sum_{w < nwin-1} 2^(c-1 + c*w)
  u256 C;
  for (int j = 0; j < 8; j++) C.v[j] = 0;
  for (int w = 0; w + 1 < p.nwin; w++) { int bit = p.c - 1 + p.c * w; C.v[bit >> 5] |= 1u << (bit & 31); }
  const size_t n = p.n;
  {
    ProfScope p1("pip_sort", 32.0 * (double)n + 3.0 * 4.0 * (double)p.nwin * (double)n, s);
    cudaMemsetAsync(counts, 0, (size_t)p.nwin * p.nb * 4, s);
    k_pip_prepare<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(kp, scalars, n, C);
    SP_LAUNCHED();
    dim3 tg((unsigned)p.ntiles, (unsigned)p.nwin);
    const size_t shm = (size_t)p.nb * 4;
    k_pip_count<<<tg, 1024, shm, s>>>(counts, tile_hist, kp, n, p.tile, p.c, p.nwin, p.nb);
    SP_LAUNCHED();
    k_pip_scan<<<p.nwin, 1024, 0, s>>>(start, cursor, istart, nitems, counts, p.nb, (uint32_t)p.S);
    SP_LAUNCHED();
    k_pip_scatter<<<tg, 1024, shm, s>>>(sorted, cursor, tile_hist, kp, n, p.tile, p.c, p.nwin, p.nb);
    SP_LAUNCHED();
  }
  {
    ProfScope p2("pip_accumulate", 100.0 * (double)p.nwin * (double)n, s);
    const size_t per_block = 128 / p.G;
    dim3 ag((unsigned)((p.max_items + per_block - 1) / per_block), (unsigned)p.nwin);
    k_pip_accumulate<<<ag, 128, 0, s>>>(partial, pts, sorted, start, counts, istart, nitems, n, p.nb, (uint32_t)p.S, p.max_items, p.G);
    SP_LAUNCHED();
  }
  {
    ProfScope p3("pip_reduce", 128.0 * (double)p.nwin * ((double)p.max_items + (double)p.nb), s);
    dim3 bg((p.nb + 3) / 4, (unsigned)p.nwin);
    k_pip_bucket_sum<<<bg, 128, 0, s>>>(buckets, partial, istart, p.nb, p.max_items);
    SP_LAUNCHED();
    k_pip_window<<<p.nwin, 512, 0, s>>>(wins, buckets, p.nb, p.c);
    SP_LAUNCHED();
    k_pip_final<<<1, 32, 0, s>>>(out, wins, p.nwin);
  }
  SP_LAUNCHED(); check("msm_var");
}

// ---- segmented variable-base MSM of the batch verifier: K independent sums over ragged segments of a few hundred points each.  Every point's
// multiple is one thread's double-and-add (no shared buckets: a segment is too short to fill them), then one block per segment adds its multiples.
__global__ void __launch_bounds__(128) k_seg_scalarmul(ge* __restrict__ out, const ge* __restrict__ pts, const u256* __restrict__ scalars, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  st_ge_p(out + i, ge_scalarmul(ld256_ro(scalars + i), ld_ge_p(pts + i)));
}
__global__ void __launch_bounds__(128) k_seg_sum(ge* __restrict__ out, const ge* __restrict__ terms, const uint32_t* __restrict__ seg_start) {
  __shared__ ge sm[4];
  const uint32_t k = blockIdx.x, lo = seg_start[k], hi = seg_start[k + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  ge acc = ge_identity();
#pragma unroll 1
  for (uint32_t i = lo + threadIdx.x; i < hi; i += blockDim.x) acc = ge_add(acc, ld_ge_p(terms + i));
  acc = warp_sum_ge(acc);
  if (lane == 0) sm[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) st_ge_p(out + k, ge_add(ge_add(sm[0], sm[1]), ge_add(sm[2], sm[3])));
}
void msm_var_segmented(ge* out, const ge* pts, const u256* scalars, const uint32_t* seg_start, size_t K, size_t n, ge* scratch, cudaStream_t s) {
  if (!K) return;
  if (n >= ((size_t)1 << 32)) throw std::runtime_error("spartan_b200: msm_var_segmented supports fewer than 2^32 points");
  ProfScope ps("msm_var_segmented", 160.0 * (double)n, s);
  if (n) {
    k_seg_scalarmul<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(scratch, pts, scalars, n);
    SP_LAUNCHED();
  }
  k_seg_sum<<<(unsigned)K, 128, 0, s>>>(out, scratch, seg_start);
  SP_LAUNCHED(); check("msm_var_segmented");
}

// ---- the scalars s_i = allinv * scale * prod_{bit b of i} u_sq[lg_n - 1 - b] of an inner-product argument's unfolded generators
// (bullet.rs:190-201), one row per item; blockIdx.y = item
__global__ void __launch_bounds__(256) k_ipa_srow(const IpaSRow* __restrict__ items) {
  const IpaSRow& it = items[blockIdx.y];
  const size_t n = (size_t)1 << it.lg_n;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  u256 v = fq_mul(it.allinv, it.scale);
  for (uint32_t b = 0; b < it.lg_n; b++)
    if ((i >> b) & 1) v = fq_mul(v, it.u_sq[it.lg_n - 1 - b]);
  if (it.add) v = fq_add(v, ld256(it.row + i));
  st256(it.row + i, v);
}
void ipa_srow(const IpaSRow* d_items, size_t nitems, uint32_t max_lg_n, cudaStream_t s) {
  if (max_lg_n >= 32) throw std::runtime_error("spartan_b200: ipa_srow: rows of at most 2^31 entries");
  for (size_t at = 0; at < nitems; at += 65535) {   // gridDim.y limit
    dim3 g((unsigned)((((size_t)1 << max_lg_n) + 255) / 256), (unsigned)(nitems - at < 65535 ? nitems - at : 65535));
    k_ipa_srow<<<g, 256, 0, s>>>(d_items + at);
    SP_LAUNCHED();
  }
  check("ipa_srow");
}

// ---- the generator fold of DotProductProofLog's folding path.  Every thread multiplies its own point by the same scalar, so the signed digits are
// recoded once on the host and every thread walks the same digit sequence: no divergence, and a table of the multiples 1..8 of the point.
struct FoldDigits { int8_t d[FOLD_NWIN]; };
template <int FMT> __device__ __forceinline__ ge fold_load(const void* p, size_t i) {
  if (FMT == FOLD_GE) return ld_ge_p(static_cast<const ge*>(p) + i);
  const ge_niels* q = static_cast<const ge_niels*>(p) + i;
  ge_niels nl;
  nl.ypx = ld256(&q->ypx); nl.ymx = ld256(&q->ymx); nl.t2d = ld256(&q->t2d);
  return ge_madd(ge_identity(), nl, false);
}
template <int IN, int OUT>
__global__ void __launch_bounds__(128) k_dotlog_fold(void* out, const void* in, size_t m, const FoldDigits dg) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  ge t[8];   // t[j] = (j + 1) * H_R[i]
  t[0] = fold_load<IN>(in, i + m);
  t[1] = ge_dbl(t[0]);
  t[2] = ge_add(t[1], t[0]);
  t[3] = ge_dbl(t[1]);
  t[4] = ge_add(t[3], t[0]);
  t[5] = ge_dbl(t[2]);
  t[6] = ge_add(t[5], t[0]);
  t[7] = ge_dbl(t[3]);
  ge acc = ge_identity();
  bool started = false;   // the same for every thread
#pragma unroll 1
  for (int w = FOLD_NWIN - 1; w >= 0; w--) {
    if (started) { acc = ge_dbl(acc); acc = ge_dbl(acc); acc = ge_dbl(acc); acc = ge_dbl(acc); }
    const int d = dg.d[w];
    if (d) {
      const ge& q = t[(d < 0 ? -d : d) - 1];
      acc = started ? ge_add(acc, d < 0 ? ge_neg(q) : q) : (d < 0 ? ge_neg(q) : q);
      started = true;
    }
  }
  acc = ge_add(acc, fold_load<IN>(in, i));
  if (OUT == FOLD_GE) {
    st_ge_p(static_cast<ge*>(out) + i, acc);
  } else {
    const ge_niels q = ge_to_niels(acc);   // one inversion per point: about a tenth of the multiplication's field products
    ge_niels* o = static_cast<ge_niels*>(out) + i;
    st256(&o->ypx, q.ypx); st256(&o->ymx, q.ymx); st256(&o->t2d, q.t2d);
  }
}
void dotlog_fold(void* out, int out_fmt, const void* in, int in_fmt, size_t m, const u256& k, cudaStream_t s) {
  if (!m) return;
  ProfScope ps("dotlog_fold", (in_fmt == FOLD_GE ? 256.0 : 192.0) * (double)m + (out_fmt == FOLD_GE ? 128.0 : 96.0) * (double)m, s);
  FoldDigits dg;
  uint32_t carry = 0;
  for (int w = 0; w < FOLD_NWIN; w++) dg.d[w] = (int8_t)signed_digit(k, w, FOLD_WBITS, carry);
  if (carry) throw std::runtime_error("spartan_b200: dotlog_fold: scalar not reduced");
  const unsigned blocks = (unsigned)((m + 127) / 128);
  if (in_fmt == FOLD_NIELS && out_fmt == FOLD_NIELS) k_dotlog_fold<FOLD_NIELS, FOLD_NIELS><<<blocks, 128, 0, s>>>(out, in, m, dg);
  else if (in_fmt == FOLD_NIELS) k_dotlog_fold<FOLD_NIELS, FOLD_GE><<<blocks, 128, 0, s>>>(out, in, m, dg);
  else if (out_fmt == FOLD_GE) k_dotlog_fold<FOLD_GE, FOLD_GE><<<blocks, 128, 0, s>>>(out, in, m, dg);
  else throw std::runtime_error("spartan_b200: dotlog_fold: extended input needs extended output");
  SP_LAUNCHED(); check("dotlog_fold");
}

__global__ void __launch_bounds__(256) k_dotlog_scalars(u256* __restrict__ out, const u256* __restrict__ a, size_t m, const u256 c, int canonical) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * m) return;
  const u256 v = fq_mul(c, ld256_ro(a + (i < m ? i + m : i - m)));
  st256(out + i, canonical ? fq_from_mont(v) : v);
}
void dotlog_scalars(u256* out, const u256* a, size_t m, const u256& c, int canonical, cudaStream_t s) {
  if (!m) return;
  ProfScope ps("dotlog_scalars", 64.0 * (double)m, s);
  k_dotlog_scalars<<<(unsigned)((2 * m + 255) / 256), 256, 0, s>>>(out, a, m, c, canonical);
  SP_LAUNCHED(); check("dotlog_scalars");
}

}  // namespace dev
}  // namespace sp
