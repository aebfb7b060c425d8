// spartan_b200 — launch wrappers around the sm_90a kernels (kernels.cu).  Plain C++ signatures so the host
// prover (prover.cpp, compiled by g++) never sees CUDA syntax.  All pointers are DEVICE pointers unless named h_*.
// Every wrapper enqueues on `stream` and returns immediately; errors surface through sp::dev::check().
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <stdexcept>
#include <string>
#include <type_traits>
#include "field.cuh"
#include "curve.cuh"
#include "../../include/spartan_b200.h"

struct CUstream_st;
typedef CUstream_st* cudaStream_t;

namespace sp {
namespace dev {

// ---- runtime plumbing
struct CudaError : std::runtime_error {  // a failed CUDA call; the C ABI returns SP_ERR_CUDA for it
  using std::runtime_error::runtime_error;
};
void check(const char* what);  // throws CudaError on a pending CUDA error
#ifdef __CUDACC__
void ck(cudaError_t e, const char* what);  // throws CudaError unless e is cudaSuccess
#endif
int device_count();
void set_device(int dev);
cudaStream_t stream_create_prio(int level);   // > 0: greatest priority of the device, < 0: least
void stream_wait_event(cudaStream_t s, void* ev);
void stream_destroy(cudaStream_t s);
void stream_sync(cudaStream_t s);
// size-bucketed caching allocator on top of cudaMalloc: a prove call allocates the same multi-hundred-MB buffers every time, and
// cudaMalloc / cudaFree (which synchronises the device) would otherwise cost milliseconds per proof
// `fill`: what a block holds when it is handed out under the memory-check mode (below); ignored otherwise
enum PoolFill { FILL_ZERO = 0, FILL_FF = 1 };
// field elements and points get 0xFF bytes: above both moduli and not a point, so a read of an entry nobody wrote shows in the result.  Every
// other buffer (raw scratch, indices, counters, structs) gets zero, what fresh memory holds: an index read from it stays in range
template <class T> constexpr int pool_fill_of() { return std::is_same<T, u256>::value || std::is_same<T, ge>::value || std::is_same<T, ge_niels>::value ? FILL_FF : FILL_ZERO; }
void* pool_alloc(size_t bytes, int fill = FILL_ZERO);
void pool_free(void* p);
size_t pool_release_cached();   // cudaFree every cached free block; returns their bytes
size_t pool_live_bytes();       // rounded bytes of the blocks handed out and not yet freed, every device
// ---- memory-check mode (sp_debug_memcheck; single GPU: sharded windows are not pool memory).  While it is on, every block is filled when it is
// handed out, fresh or reused (after a device synchronise, so the previous owner has finished), and carries a zero guard band of at least
// MEMCHECK_GUARD bytes past the requested size; a non-zero guard byte found at pool_free or by memcheck_scan is a violation.  Switching it on or
// off drops the free cache, and a block allocated before the switch is never cached under it.
constexpr size_t MEMCHECK_GUARD = 4096;
struct MemcheckStats { unsigned long long blocks_filled = 0, blocks_refilled = 0, context_refills = 0, guard_bytes_checked = 0, violations = 0; };
void memcheck_enable(bool on);
bool memcheck_on();
MemcheckStats memcheck_stats(std::string* first_violation, std::string* last_violation);
unsigned long long memcheck_scan();   // synchronises the device and checks the guard of every live block; returns the violations it found
void memcheck_fill(void* d, size_t bytes, int fill);   // device memory, between two device synchronises
void memcheck_count_refill();         // one context's persistent scratch refilled at an entry point
void* hmalloc_pinned(size_t bytes);
void hfree_pinned(void* p);
void h2d(void* d, const void* h, size_t bytes, cudaStream_t s);
void d2h(void* h, const void* d, size_t bytes, cudaStream_t s);
void d2d(void* dst, const void* src, size_t bytes, cudaStream_t s);
void dzero(void* d, size_t bytes, cudaStream_t s);
int sm_count();
void mem_info(size_t* free_bytes, size_t* total_bytes);
// event timing of the kernels launched through these wrappers (bench.py roofline leg)
void* event_create();
void event_record(void* ev, cudaStream_t s);
float event_elapsed_ms(void* a, void* b);
void event_destroy(void* ev);
unsigned long long launch_count();  // kernels launched by this library since load
void io_bytes(unsigned long long* h2d_bytes, unsigned long long* d2h_bytes);  // bytes moved through h2d()/d2h() since load
void prof_enable(bool on);          // CUDA-event timing around every kernel family (clears previous records)
std::string prof_report();          // "name:launches:total_ms:total_algorithmic_bytes;..."

// ---- sumcheck rounds (K1/K2 of SURVEY.md §2b)
enum ScKind { SC_QUAD = 0 /*A*B*/, SC_CUBIC3 = 1 /*A*B*C*/, SC_CUBIC4 = 2 /*A*(B*C-D)*/ };
struct ScInst {        // one sumcheck instance: up to four tables of the same current length
  u256* t[4];          // A, B, C, D (unused entries null)
  u256* c_out;         // where the folded C goes (== t[2] for private C; a ping-pong buffer when C is shared)
  int write_c;         // 1: this instance stores the folded C
};
constexpr int SC_MAX_INST = 24;   // instances of one batched launch: sc_eval and its siblings refuse more
// Optional host notification of a reduction kernel: results are also stored to `host_out` (mapped pinned memory) and `seq` is then
// published in `*flag`; `done` is a zero-initialised device counter (instances of a batched launch finish independently).
struct HostSig {
  u256* host_out = nullptr;
  unsigned int* flag = nullptr;
  unsigned int* done = nullptr;
  unsigned int seq = 0;
};
// ---- intra-proof sharding over NVLink peer memory (comm.cu).  One process per GPU; every rank owns a "window" (plain cudaMalloc memory
// exported with cudaIpcGetMemHandle and mapped by every peer), laid out as [control | data half 0 | data half 1]:
//   control: per-source flag words and mailboxes for the per-round exchange of partial sums, flag words for the bulk all-gathers, an error word
//   data   : destination of the bulk all-gathers (alternating halves), read in place by the kernels that follow
// All ranks execute the same sequence of collectives, so a sequence number identifies an operation on every rank.
#define SP_MAX_RANKS 8
#define SP_XR_SLOTS 4
#define SP_XR_CAP 80                                   // u256 per (slot, source): a full batch's 3 evaluations per instance fit
#define SP_WIN_CTRL_BYTES ((size_t)1 << 20)
#define SP_WIN_HALF_BYTES ((size_t)96 << 20)
static_assert(SP_XR_CAP >= 3 * SC_MAX_INST, "SP_XR_CAP: a mailbox must hold the 3 evaluations of each of SC_MAX_INST instances");
struct WinCtrl {                                        // at offset 0 of every window
  unsigned int xflag[SP_MAX_RANKS];                     // [source]: sequence number of the last partial-sum message from `source`
  unsigned int bflag[SP_MAX_RANKS];                     // [source]: sequence number of the last bulk all-gather contribution from `source`
  unsigned int err;                                     // set by a kernel whose peer wait timed out
  unsigned int pad[15];
  u256 mbox[SP_XR_SLOTS][SP_MAX_RANKS][SP_XR_CAP];      // [seq % SP_XR_SLOTS][source][value]
};
// Cross-rank completion of a reduction kernel: the finishing warp stores this rank's totals into every peer's mailbox (NVLink stores), publishes
// the sequence number, waits for the peers' messages and adds them up in rank order (exact field arithmetic: every rank gets identical bytes),
// then hands the sums to the host.  world <= 1: no exchange.
struct XRank {
  int world = 1, rank = 0;
  unsigned int seq = 0;
  WinCtrl* win[SP_MAX_RANKS] = {};                      // this process's mapping of every rank's window (win[rank] = own)
};

// scratch: >= sc_scratch_bytes(); out: ninst*3 scalars [e0,e2,e3] (e3 = 0 for SC_QUAD), device memory
size_t sc_scratch_bytes(int ninst);
// out[i] = tables[i][0] for count <= HEADS_PER_LAUNCH tables (the kernel parameter holds that many pointers)
constexpr int HEADS_PER_LAUNCH = 64;
void heads(u256* out, const u256* const* tables, int count, cudaStream_t s, HostSig sig = HostSig());
void sc_eval(ScKind kind, const ScInst* d_insts, int ninst, size_t len, u256* out, void* scratch, cudaStream_t s, HostSig sig = HostSig(), const XRank& xr = XRank());
// fold every table of every instance by r (len -> len/2, in place) and evaluate the next round on the result; r travels as a kernel argument.
// host_bound (len == 4, signalled launch): the bound two-entry tables also go to the host, host_bound[i * 2 NT + 2 t + h] = entry h of table t of
// instance i (NT = 2, 3 or 4 tables per instance), published with the evaluations
void sc_fold_eval(ScKind kind, const ScInst* d_insts, int ninst, size_t len, const u256& r, u256* out, void* scratch, cudaStream_t s,
                  HostSig sig = HostSig(), const XRank& xr = XRank(), u256* host_bound = nullptr);
// ---- eq-factored streaming rounds of a batched A*B*eq sumcheck (kernels_sc.cu: k_sc_eval_g): instances use t[0] = A, t[1] = B; E: the suffix eq table
// of the round (len/2 entries for sc_eval_g, len/4 for sc_fold_eval_g); out[3*i + 0] = q(0), out[3*i + 1] = q(inf) of instance i
void sc_eval_g(const ScInst* d_insts, int ninst, size_t len, const u256* E, u256* out, void* scratch, cudaStream_t s, HostSig sig = HostSig(), const XRank& xr = XRank());
void sc_fold_eval_g(const ScInst* d_insts, int ninst, size_t len, const u256& r, const u256* E, u256* out, void* scratch, cudaStream_t s, HostSig sig = HostSig(),
                    const XRank& xr = XRank());
// ---- rounds of a sumcheck of a caller-defined polynomial g = sum_t coeff[t] * prod_f t[fac[t][f]] (kernels_sc.cu: k_scp_*).  The tables are
// distinct (each is bound once per round); out = the `degree` evaluations at t = 0, 2, 3, .., degree (just t = 0 for degree 1)
struct ScPoly {
  u256* t[SP_SC_MAX_TABLES];
  u256 coeff[SP_SC_MAX_TERMS];                          // Montgomery form
  uint8_t fac[SP_SC_MAX_TERMS][SP_SC_MAX_DEGREE];       // table indices < ntables
  uint8_t nfac[SP_SC_MAX_TERMS];                        // 1 .. degree
  uint8_t unit[SP_SC_MAX_TERMS];                        // 1: coeff is one, the product is not multiplied by it
  int ntables, nterms, degree;
};
void scp_eval(const ScPoly& p, size_t len, u256* out, void* scratch, cudaStream_t s, HostSig sig);
// bind every table with r (len -> len/2, in place; len >= 4) and evaluate the next round on the result
void scp_fold_eval(const ScPoly& p, size_t len, const u256& r, u256* out, void* scratch, cudaStream_t s, HostSig sig);
// levels[k-1] (k = 1..K, back to back, n0 >> k entries each) = eq(tau[k+1..], .) from E0 = eq(tau[1..], .) of n0 entries
void eq_suffix(u256* levels, const u256* E0, size_t n0, int K, cudaStream_t s);
// fold only (bound_poly_var_top, dense_mlpoly.rs:215-223): tables[k][i] += r*(tables[k][i+len/2]-tables[k][i])
void fold_top(u256* const* d_tables, int ntables, size_t len, const u256& r, cudaStream_t s);

// ---- dense polynomial helpers (K7)
void eq_evals(u256* out, const u256* d_r, int ell, u256* scratch_small /* >= eq_evals_scratch(ell) */, cudaStream_t s);
inline size_t eq_evals_scratch(size_t ell) { return 2 * ((size_t)1 << ((ell + 1) / 2)) + 8; }   // scalars
// out[n .. 2n) holds E = eq(r', .); rewrite out[0 .. 2n) as eq((r, r'), .) = [(1 - r) E | r E] in one pass
void eq_extend_top(u256* out, size_t n, const u256& r, cudaStream_t s);
void dot(u256* out, const u256* a, const u256* b, size_t n, void* scratch, cudaStream_t s);
void dot_many(u256* out, const u256* const* a_list, int count, const u256* b, size_t n, void* scratch, cudaStream_t s);
void dot3(u256* out, const u256* a, const u256* b, const u256* c, size_t n, void* scratch, cudaStream_t s);
void bound_rows(u256* out, const u256* Z, const u256* L, size_t L_size, size_t R_size, u256* scratch /* >= 64*R_size */, cudaStream_t s);
// out[j * R_size + i] = sum_r L[r] * tables[j][r * R_size + i] for k <= SP_PC_MAX_TABLES tables of L_size x R_size entries: bound_rows of every
// table, each table read once, in one launch (plus a sum of the slabs when the rows are split)
size_t bound_rows_many_scratch(int k, size_t L_size, size_t R_size);   // scalars
void bound_rows_many(u256* out, const u256* const* tables, int k, const u256* L, size_t L_size, size_t R_size, u256* scratch, cudaStream_t s);
void lincomb3(u256* out, const u256* A, const u256* B, const u256* C, const u256* d_rabc /*3*/, size_t n, cudaStream_t s);
void hadamard_many(u256* const* outs, const u256* const* as, const u256* const* bs, int count, size_t n, cudaStream_t s);
// ---- the leaves of the caller's product circuits (sp_prod_build) and the operands of their dot products (sp_prod_build_dotp): affine forms
// form[x] = cst + idx * x + sum_{s < nsrc} coeff[s] * src[s][x] of the caller's tables, which are only read
enum { PROD_UNIT0 = 1 /* bit s: coeff[s] is one */, PROD_IDX = 8 /* idx != 0 */, PROD_CST = 16 /* cst != 0 */ };
struct AffineForm {
  const u256* src[SP_PROD_MAX_SOURCES];
  u256 coeff[SP_PROD_MAX_SOURCES], idx, cst;   // Montgomery form
  uint32_t nsrc, flags;
};
// a circuit's leaves: the form for x < n written to layer0 (n entries), and layer1[x] = leaf[x] * leaf[x + n/2] for x < n/2 (the first product
// layer) when layer1 is set
struct ProdLeaves {
  AffineForm f;
  u256* layer0;
  u256* layer1;
};
// k <= SP_PROD_MAX_CIRCUITS circuits of n >= 2 leaves each, in one launch (blockIdx.y = circuit)
void prod_leaves(const ProdLeaves* circuits, int k, size_t n, cudaStream_t s);
// a dot product sum_x left[x] right[x] weight[x]: its three operand forms, written for x < n to out = [left | right | weight] (3n entries)
constexpr int PROD_MAX_DOTP = (SP_PROD_MAX_CIRCUITS - 1) / 2;   // one circuit and the two halves of each dot product in one batched sumcheck
struct DotpOperands {
  AffineForm f[3];   // left, right, weight
  u256* out;
};
// kd <= PROD_MAX_DOTP dot products of n >= 2 entries each in one launch (blockIdx.y = dot product): the operands, and half_sums[2d + h] = the sum
// of left * right * weight over half h (entries [h n/2, (h + 1) n/2)) of dot product d.  scratch: Ctx::red (>= sc_scratch_bytes(SC_MAX_INST))
void dotp_operands(const DotpOperands* dotps, int kd, size_t n, u256* half_sums, void* scratch, cudaStream_t s);
void to_canonical(u256* out, const u256* in, size_t n, cudaStream_t s);   // Montgomery -> canonical little-endian integers (transcript bytes)
void gather(u256* out, const u256* mem, const uint32_t* idx, size_t n, cudaStream_t s);
// hash layer of the SPARK memory check: out = ts*r^2 + val*r + addr - g  (sparse_mlpoly.rs:545-600)
// addr == null: addr = index i;  ts == null: ts = 0;  ts_plus_one adds one.   d_rg = [r_hash, r_multiset]
void spark_hash(u256* out, size_t n, const u256* addr, const u256* val, const u256* ts, int ts_plus_one, const u256* d_rg, cudaStream_t s);
// the folds of an inner-product round (bullet.rs:105-108) in one launch: a[i] = a[i]*u + uinv*a[i+half], b[i] = b[i]*uinv + u*b[i+half], and the
// running scalars s[j] of the unfolded generators (DESIGN.md "IPA without folding G") times uinv (left half of their block) or u (right half);
// svec null: a and b only
void ipa_fold_update(u256* a, u256* b, u256* svec, size_t n_cur_half, size_t n_full, const u256& u, const u256& uinv, cudaStream_t s);
void fill_one(u256* out, size_t n, cudaStream_t s);

// windows: IPC-exportable device allocations and their mappings in the peers
void* win_alloc(size_t bytes);
void win_free(void* p);
size_t ipc_handle_bytes();
void ipc_export(void* devptr, uint8_t* out);
void* ipc_open(const uint8_t* handle);
void ipc_close(void* p);
// ---- sharded table producers: rank `rank` of `world` holds the global indices i = j*world + rank (cyclic partition) at local index j
void scale(u256* inout, const u256& c, size_t n, cudaStream_t s);                                        // x[i] *= c
void take_cyclic(u256* out, const u256* full, size_t n_local, int rank, int world, cudaStream_t s);      // out[j] = full[j*world + rank]
void spmv_cyclic(u256* out, size_t nrows_local, int rank, int world, const uint32_t* ptr, const uint32_t* idx, const u256* val, const u256* x, cudaStream_t s);
void spark_hash_cyclic(u256* out, size_t n_local, int rank, int world, const u256* addr, const u256* val, const u256* ts, int ts_plus_one, const u256* d_rg, cudaStream_t s);
// ---- bulk all-gathers into every rank's window (comm.cu); `dst_off`: byte offset inside the window, the same on every rank
struct CommDev {                                        // device-side view of the communicator
  int world = 1, rank = 0;
  uint8_t* win[SP_MAX_RANKS] = {};
};
// every rank's `bytes` land at dst_off + source*bytes of every window
void push_block(const CommDev& c, const void* src, size_t bytes, size_t dst_off, unsigned int seq, unsigned int* ticket, cudaStream_t s);
// table t of rank `source`, element j  ->  window element (dst_off/32) + t*(n_local*world) + j*world + source
void push_cyclic(const CommDev& c, const u256* const* tables, int ntables, size_t n_local, size_t dst_off, unsigned int seq, unsigned int* ticket, cudaStream_t s);
void wait_peers(const CommDev& c, unsigned int seq, cudaStream_t s);   // returns (on the stream) once every peer's contribution `seq` has landed

// ---- sparse matrix-vector products on CSR (row-major) / CSC (column-major) copies of the COO triples
void spmv(u256* out, size_t nrows, const uint32_t* ptr, const uint32_t* idx, const u256* val, const u256* x, cudaStream_t s);
// sum_k trx[row_k]*try[col_k]*val_k
void sparse_eval3(u256* out, const uint32_t* row, const uint32_t* col, const u256* val, size_t nnz, const u256* trx, const u256* try_, void* scratch, cudaStream_t s);

// ---- instance ingestion (kernels_inst.cu)
bool is_device_pointer(const void* p, int device);   // memory allocated on `device` (cudaMemoryTypeDevice)
void set_max_u64(unsigned long long* w, cudaStream_t s);
void d2h_sync(void* h, const void* d, size_t bytes);  // blocking copy outside any stream's order (data no pending work writes)
// Instance::new (lib.rs:129-198) entries of A, B, C, or of a caller's SPARK matrices, from caller arrays: `nmat` matrices, row < num_rows,
// col < num_cols, value < q; columns from num_vars on move up by `shift` (the R1CS input columns; num_vars = num_cols: none); values to
// Montgomery form.  The first bad entry in (matrix, entry, row/col/scalar) order wins: *err = min over bad entries of ((m << 40 | k) << 2) | code
// (*err = ~0 beforehand: none)
enum { INGEST_ROW = 0, INGEST_COL = 1, INGEST_SCALAR = 2 };
constexpr int INGEST_MAX_MATRICES = SP_SPARK_MAX_BATCH;   // >= 3, the R1CS matrices
struct CooIn { const uint64_t* row[INGEST_MAX_MATRICES]; const uint64_t* col[INGEST_MAX_MATRICES]; const uint8_t* val[INGEST_MAX_MATRICES]; size_t n[INGEST_MAX_MATRICES]; };
struct CooOut { uint32_t* row[INGEST_MAX_MATRICES]; uint32_t* col[INGEST_MAX_MATRICES]; u256* val[INGEST_MAX_MATRICES]; };
void inst_ingest(const CooIn& in, int nmat, const CooOut& out, size_t num_rows, size_t num_cols, size_t num_vars, size_t shift, unsigned long long* err,
                 cudaStream_t s);
// entries [from, to) = (row i, column pad_col, value 0): the padding of an instance with fewer than two constraints
void inst_pad_rows(uint32_t* row, uint32_t* col, u256* val, size_t from, size_t to, uint32_t pad_col, cudaStream_t s);
// n canonical 32-byte scalars -> Montgomery form; *err = smallest index of a value >= q (*err = ~0 beforehand: none)
void canonical_to_mont(u256* out, const uint8_t* in32, size_t n, unsigned long long* err, cudaStream_t s);
// CSR (major = row) or CSC (major = column) copy of a COO matrix: ptr[nmajor + 1], idx / v[nnz] in stable order of the major index
size_t compress_scratch_bytes(size_t nmajor, size_t nnz);
void build_compressed(uint32_t* ptr, uint32_t* idx, u256* v, size_t nmajor, const uint32_t* major, const uint32_t* minor, const u256* val, size_t nnz,
                      void* scratch, cudaStream_t s);
// ---- the caller's matrices as products (sp_spmat): every matrix in row order (key = row, src = col) and in column order (key = col, src = row)
// sorted copy of nnz entries by key < nkeys, stable (equal keys keep their input order); scratch >= spmat_sort_scratch_bytes(nnz)
size_t spmat_sort_scratch_bytes(size_t nnz);
void spmat_sort(uint32_t* key_out, uint32_t* src_out, u256* val_out, const uint32_t* key, const uint32_t* src, const u256* val, size_t nkeys, size_t nnz,
                void* scratch, cudaStream_t s);
// out[m][key] = sum over the entries of matrix m with that key of val * x[src], for m < b; every out[m] has nout entries (zero where no entry has the
// key; every key < nout).  Tiles of SPMAT_TILE entries of the batch whatever the rows' lengths, and three launches for every shape
// (kernels_inst.cu); scratch >= spmat_products_scratch_bytes(sum of nnz)
constexpr int SPMAT_THREADS = 256, SPMAT_ITEMS = 4, SPMAT_TILE = SPMAT_THREADS * SPMAT_ITEMS;
struct SpmatBatch {
  const uint32_t* key[SP_SPMAT_MAX_BATCH];
  const uint32_t* src[SP_SPMAT_MAX_BATCH];
  const u256* val[SP_SPMAT_MAX_BATCH];
  size_t nnz[SP_SPMAT_MAX_BATCH];
  u256* out[SP_SPMAT_MAX_BATCH];
  int b;
};
// the carries of spmat_products in its scratch: n1 = 2 per tile of the entries (level 1), n2 = 2 per tile of those (level 2); values (32 B) and
// keys (8 B) of each level, every region at a 256-byte boundary.  The one layout both the size and the carving read
struct SpmatCarries {
  size_t n1, n2, cv1, cv2, ck1, ck2, bytes;   // carry counts, byte offsets of the four regions, total bytes
  static size_t carries(size_t n) { return 2 * ((n + SPMAT_TILE - 1) / SPMAT_TILE); }
  static size_t up256(size_t b) { return (b + 255) & ~(size_t)255; }
  explicit SpmatCarries(size_t total) : n1(carries(total)), n2(carries(n1)) {
    cv1 = 0;
    cv2 = cv1 + up256(32 * n1);
    ck1 = cv2 + up256(32 * n2);
    ck2 = ck1 + up256(8 * n1);
    bytes = ck2 + 8 * n2;
  }
};
size_t spmat_products_scratch_bytes(size_t total);   // SpmatCarries(total).bytes
void spmat_products(const SpmatBatch& B, const u256* x, size_t nout, void* scratch, cudaStream_t s);
// out[i] = sum_{m < b} w[m] * t[m][i] (w: Montgomery form)
struct LincombTables { const u256* t[SP_SPMAT_MAX_BATCH]; u256 w[SP_SPMAT_MAX_BATCH]; int b; };
void lincomb_many(u256* out, const LincombTables& lt, size_t n, cudaStream_t s);
// AddrTimestamps::new (sparse_mlpoly.rs:220-254), one side of b <= SP_SPARK_MAX_BATCH matrices: the addresses src[m][0..nnz[m]) zero-padded to N
// -> idx[m] (N each) and, as field elements over the b N positions (matrix-major, the reference loop's order), addr_f, ts_f (read_ts) and audit_f
// (cells, counts over all b matrices); *bad |= 1 when an address is >= cells
struct SparkAddrs { const uint32_t* src[SP_SPARK_MAX_BATCH]; size_t nnz[SP_SPARK_MAX_BATCH]; uint32_t* idx[SP_SPARK_MAX_BATCH]; int b; };
size_t spark_ts_scratch_bytes(size_t b, size_t N, size_t cells);
void spark_timestamps(const SparkAddrs& sa, u256* addr_f, u256* ts_f, u256* audit_f, size_t N, size_t cells, void* scratch, unsigned int* bad, cudaStream_t s);

// ---- group: generators, fixed-base window tables, multi-row MSM, compression (K3/K4/K6)
void gens_from_uniform(ge* out, const uint8_t* d_uniform64, size_t n, cudaStream_t s);
void decompress_batch(ge* out, int* ok, const uint8_t* in32, size_t n, cudaStream_t s);
void compress_batch(uint8_t* out32, const ge* in, size_t n, cudaStream_t s);
// table[(j*NWIN + w)*2^(W-1) + (d-1)] = d * 2^(W*w) * G_j in affine-niels form; W (wbits) is 8 or 13, NWIN = ceil(253 / W)
size_t table_entries(size_t nbases, int wbits);
void build_tables(ge_niels* table, const ge* G, size_t nbases, int wbits, cudaStream_t s);
// row table: rt[j*2^(W-1) + (d-1)] = d * G_j for every base; W = ROW_W = 16 (kernels.cu)
size_t row_table_entries(size_t nbases);
void build_row_table(ge_niels* rt, const ge* G, size_t nbases, cudaStream_t s);
// out[row] = sum_{j<R} scalars[row*stride + j] * G_j  (+ blinds[row] * G_{blind_base} when blinds != null)
// scalars are Montgomery-form; partial: scratch >= msm_scratch_bytes(L, R).  Many long rows run on `row_table` when the set has one (null: none),
// every other shape on the per-window `table`.
size_t msm_scratch_bytes(size_t L, size_t R);
// smem_pad: bytes of unused dynamic shared memory per CTA, which cap the resident CTAs per SM (an MSM that runs in the background of
// latency-bound work leaves them room)
void msm_rows(ge* out, const ge_niels* table, int wbits, const ge_niels* row_table, const u256* scalars, size_t stride, size_t L, size_t R,
              const u256* blinds, size_t blind_base, void* scratch, cudaStream_t s, size_t smem_pad = 0);
// The table-list form: row i of the L rows is row i % rows_per_table of table t[i / rows_per_table] (row_len = R scalars per row, rows back to
// back); the rows of tables at or past ntables are zero and are not read, so they give the identity, or blinds[i] * G_blind_base alone.  The
// rows of k tables concatenated and zero-padded (DensePolynomial::merge) without a copy.  Same kernels, scratch and launch shapes as msm_rows.
struct TableRows {
  const u256* t[SP_PC_MAX_TABLES];
  int ntables;
  size_t rows_per_table, row_len;
};
void msm_rows_tables(ge* out, const ge_niels* table, int wbits, const ge_niels* row_table, const TableRows& tr, size_t L, size_t R, const u256* blinds,
                     size_t blind_base, void* scratch, cudaStream_t s);

void add_points(ge* a, const ge* b, size_t n, cudaStream_t s);   // a[i] += b[i]
void sum_points(ge* out, const ge* in, int n, cudaStream_t s);   // out[0] = in[0] + ... + in[n-1], n <= 32
// both MSMs of an inner-product round (L, R -> out[0], out[1]) over unfolded generators: scalar of generator j is a[.]*svec[j].
// scratch >= ipa_msm_scratch_points(n_full, wbits) points; ticket: one zero-initialised word (self-resetting)
size_t ipa_msm_scratch_points(size_t n_full, int wbits);
void ipa_msm(ge* out, const ge_niels* table, int wbits, const u256* a, const u256* svec, size_t n_cur, size_t n_full, void* scratch, unsigned int* ticket,
             cudaStream_t s, HostSig sig = HostSig(),
             // b != null: the same launch also computes c_out[0] = <a_L, b_R>, c_out[1] = <a_R, b_L> of the round and
             // publishes them through sigc (its own flag word and completion counter), long before the MSM finishes
             const u256* b = nullptr, u256* c_out = nullptr, HostSig sigc = HostSig());

// ---- variable-base MSM on arbitrary points (bucket method; kernels_pip.cu).  pts: affine-niels form of the caller's points.
struct PipPlan { size_t n = 0; int c = 0, nwin = 0, G = 32; uint32_t nb = 0; size_t tile = 0, ntiles = 0, S = 0, max_items = 0; };
PipPlan pip_plan(size_t n, int c_override);   // c_override = 0: pick the window width from n
size_t pip_scratch_bytes(const PipPlan& p);
void points_to_niels(ge_niels* out, const ge* in, size_t n, cudaStream_t s);
void niels_to_ge(ge* out, const ge_niels* in, size_t n, cudaStream_t s);
// out = sum_i scalars[i] * pts[i]   (scalars Montgomery-form, device-resident; scratch >= pip_scratch_bytes(p))
void msm_var(ge* out, const ge_niels* pts, const u256* scalars, const PipPlan& p, void* scratch, cudaStream_t s);
// out[k] = sum_{seg_start[k] <= i < seg_start[k+1]} scalars[i] * pts[i] for k < K (an empty segment gives the identity).  scalars: canonical
// integers (not Montgomery form); seg_start: K+1 entries, non-decreasing, seg_start[K] = n; scratch >= n points
void msm_var_segmented(ge* out, const ge* pts, const u256* scalars, const uint32_t* seg_start, size_t K, size_t n, ge* scratch, cudaStream_t s);

// ---- the generator scalars of an inner-product argument: row[i] (+)= allinv * scale * prod_{bit b of i} u_sq[lg_n - 1 - b] for i < 2^lg_n, the
// vector s of DotProductProofLog::verify (bullet.rs:190-201) times `scale`.  Montgomery form; add = 0 writes, 1 adds.  The items of one launch
// must write disjoint entries
struct IpaSRow {
  u256* row;
  uint32_t lg_n, add;
  u256 allinv, scale;
  u256 u_sq[32];
};
void ipa_srow(const IpaSRow* d_items, size_t nitems, uint32_t max_lg_n, cudaStream_t s);

// ---- the folding path of DotProductProofLog (prover.cpp: dotlog_fold_prove).  The generator vector G_k = c_k * H_k is kept as H_k and one common
// scalar c_k, so a round folds H' = H_L + u^2 * H_R (bullet.rs:108 divided by c' = c * u^-1): one variable-base multiplication per pair.
// A point buffer holds affine niels points (FOLD_NIELS, the input of msm_var) or extended points (FOLD_GE, the input of msm_var_segmented).
enum FoldFmt { FOLD_NIELS = 0, FOLD_GE = 1 };
constexpr int FOLD_WBITS = 4, FOLD_NWIN = (253 + FOLD_WBITS - 1) / FOLD_WBITS;   // signed 4-bit digits of the fold scalar
// out[i] = in[i] + k * in[i + m] for i < m; k canonical (< q).  out may be in itself when both have the same format (thread i writes only entry i)
void dotlog_fold(void* out, int out_fmt, const void* in, int in_fmt, size_t m, const u256& k, cudaStream_t s);
// the scalars of a round's two MSMs, halves swapped: out = [c * a[m .. 2m) | c * a[0 .. m)], Montgomery form, or canonical integers (canonical = 1)
void dotlog_scalars(u256* out, const u256* a, size_t m, const u256& c, int canonical, cudaStream_t s);

}  // namespace dev
}  // namespace sp
