/*
 * spartan_b200 — C ABI of the H100-native Spartan prover (libspartan_b200.so).
 *
 * Drop-in boundary for the prover hot path of microsoft/Spartan (libspartan 0.9.0).  The reference has no FFI of its own
 * (pure Rust, single crate); these are the entry points a `libspartan-sys` shim would bind, each naming the Rust item it
 * replaces (paths relative to /root/reference).  Conventions:
 *   - every function returns an int status: SP_OK or an SP_ERR_* code; sp_last_error() gives the message.  No exception or
 *     panic crosses the boundary (the reference panics on misuse, e.g. src/r1csproof.rs:156).
 *   - a transcript or tape state whose position bytes are out of range is refused with SP_ERR_INVALID_ARG.
 *   - scalars cross as `uint64_t[4]` little-endian limbs in MONTGOMERY form = the in-memory layout of `Scalar`
 *     (src/scalar/ristretto255.rs:195-199), so a Rust `&[Scalar]` is passed as-is (`as_ptr() as *const u64`).
 *     Where the reference API takes canonical bytes (`[u8;32]`, src/lib.rs:64,121) so does this ABI.
 *   - group elements cross only as 32-byte ristretto255 encodings (`CompressedRistretto::as_bytes`).
 *   - handles are opaque and own device memory; one sp_ctx per host thread / per GPU.
 *   - there is NO CPU fallback: sp_ctx_create fails with SP_ERR_NO_DEVICE when no CUDA device is present.
 */
#ifndef SPARTAN_B200_H
#define SPARTAN_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SP_OK 0
#define SP_ERR_NO_DEVICE 1
#define SP_ERR_CUDA 2
#define SP_ERR_INVALID_ARG 3
#define SP_ERR_INVALID_INDEX 4     /* R1CSError::InvalidIndex            src/errors.rs:28-41 */
#define SP_ERR_INVALID_SCALAR 5    /* R1CSError::InvalidScalar */
#define SP_ERR_INVALID_INPUTS 6    /* R1CSError::InvalidNumberOfInputs */
#define SP_ERR_INTERNAL 7
#define SP_ERR_VERIFY 9            /* ProofVerifyError::InternalError: the proof was rejected                    src/errors.rs:5-12 */
#define SP_ERR_DECOMPRESS 10       /* ProofVerifyError::DecompressionError: a point of the proof does not decompress */
#define SP_ERR_INVALID_POINT 8     /* CompressedRistretto::decompress() == None (ProofVerifyError::DecompressionError, src/errors.rs:10) */

typedef struct sp_ctx sp_ctx;
typedef struct sp_poly sp_poly;           /* DensePolynomial.Z on the device          src/dense_mlpoly.rs:18-22 */
typedef struct sp_gens sp_gens;           /* MultiCommitGens + fixed-base tables      src/commitments.rs:8-12 */
typedef struct sp_points sp_points;       /* a caller-supplied &[GroupElement] on the device   src/group.rs:8-9 */
typedef struct sp_instance sp_instance;   /* Instance (R1CSShape + digest)            src/lib.rs:111-114 */
typedef struct sp_nizk_gens sp_nizk_gens; /* NIZKGens                                 src/lib.rs:468-486 */
typedef struct sp_snark_gens sp_snark_gens;     /* SNARKGens                          src/lib.rs:277-309 */
typedef struct sp_snark_encoding sp_snark_encoding; /* (ComputationCommitment, ComputationDecommitment)  src/lib.rs:44-55 */

/* ---- context */
int sp_device_count(void);
int sp_ctx_create(int device, sp_ctx** out);
void sp_ctx_destroy(sp_ctx* ctx);
const char* sp_last_error(const sp_ctx* ctx);  /* ctx may be NULL: message of the last failed sp_ctx_create or host-only call made without one */
unsigned long long sp_kernel_launches(void);   /* kernels launched by this library since load */
/* device blocks freed by the library are kept for reuse by later proofs of this process; this returns them to the driver (e.g. before another
 * process on the same GPU needs the memory) and gives their size in bytes.  Buffers still held by live objects are not touched. */
unsigned long long sp_release_cached_memory(void);
/* Memory-check mode, process-wide, single GPU (a debugging aid: slower, never for production).  While it is on, every device block the library
 * hands out is filled first, fresh or reused: field elements and points with 0xFF bytes (above both moduli, not a point), everything else with
 * zero; every block carries a zero guard band of at least 4 KiB past the requested size; and every entry point refills the context's persistent
 * scratch (and a point set's sort workspace) before it starts.  So a read of memory the call did not write changes its result, and a write past a
 * buffer's end lands in the guard, where the block's free or sp_debug_memcheck_scan reports it.  Switching the mode drops the cache of freed
 * blocks; a block allocated before the switch is never reused under it.  Switch it on before the first context is created. */
void sp_debug_memcheck(int on);
typedef struct sp_memcheck_counts {
  unsigned long long blocks_filled;        /* blocks handed out under the mode */
  unsigned long long blocks_refilled;      /* ... of them, cached blocks reused */
  unsigned long long context_refills;      /* entry points that refilled a context's persistent scratch */
  unsigned long long guard_bytes_checked;
  unsigned long long violations;           /* dirty guard bands found */
} sp_memcheck_counts;
/* the counters since load and, when there were violations, the first one's message, a newline and the latest one's ("" otherwise) */
int sp_debug_memcheck_report(sp_memcheck_counts* out, char* violations, size_t buflen);
/* synchronise the device and check the guard band of every live block; returns the violations found (~0 on a CUDA error) */
unsigned long long sp_debug_memcheck_scan(void);

/* ---- one proof over several GPUs (SURVEY.md 8(e); the reference is single-process, the loops being sharded are dense_mlpoly.rs:215-223,
 * sumcheck.rs:290-357 / :460-469 / :625-652, dense_mlpoly.rs:165-177, product_tree.rs:18-56).  One process per GPU, one context per process.
 * Every rank calls sp_comm_export, the hosts exchange the sp_comm_handle_bytes()-byte handles by any transport (MPI, a socket, torch.distributed),
 * every rank calls sp_comm_connect with all handles in rank order (world = 2, 4 or 8 GPUs of one NVLink domain).  From then on sp_nizk_prove* and
 * sp_snark_prove* must be called by EVERY rank with identical arguments: each call is one sharded proof, every rank returns the same proof bytes —
 * the bytes the single-GPU prover returns.  Operator-level entry points, encode and the verifiers stay single-GPU. */
size_t sp_comm_handle_bytes(void);
int sp_comm_export(sp_ctx* ctx, uint8_t* handle_out);
int sp_comm_connect(sp_ctx* ctx, int rank, int world, const uint8_t* handles /* world x sp_comm_handle_bytes() */);
int sp_comm_info(const sp_ctx* ctx, int* rank, int* world);
int sp_comm_set_enabled(sp_ctx* ctx, int enabled);   /* 0: the next prove calls run on this rank's GPU alone (all ranks must switch together) */
/* 1 (default): SNARK::prove commits to the dereferenced SPARK values on a background stream underneath the latency-bound rounds that precede the
 * commitment in the transcript (same bytes, shorter proof); 0: every kernel on the context's stream, one after the other (per-kernel profiling) */
int sp_ctx_set_overlap(sp_ctx* ctx, int enabled);
/* phase timings of the last prove call, the labels of the reference's `profile` feature (src/timer.rs; src/r1csproof.rs:152-298) */
int sp_timings(sp_ctx* ctx, char* buf, size_t buflen);
/* bytes moved host->device / device->host by this library since load (bench.py e2e leg) */
void sp_io_bytes(unsigned long long* h2d_bytes, unsigned long long* d2h_bytes);
/* CUDA-event timing of every kernel family on the launching stream (bench.py roofline leg).  sp_prof_enable(1) clears and starts;
 * sp_prof_report writes "name:launches:total_ms:total_algorithmic_bytes;..." after synchronising the device */
void sp_prof_enable(int on);
int sp_prof_report(char* buf, size_t buflen);
/* device-side stopwatch on the context's stream (CUDA events) */
int sp_timer_start(sp_ctx* ctx);
int sp_timer_stop_ms(sp_ctx* ctx, float* ms);

/* ---- scalar field helpers (host side, for harnesses) */
int sp_scalar_from_bytes(const uint8_t canonical[32], uint64_t out_mont[4]);        /* Scalar::from_bytes       ristretto255.rs:391 */
void sp_scalar_to_bytes(const uint64_t mont[4], uint8_t out_canonical[32]);         /* Scalar::to_bytes         ristretto255.rs:419 */
void sp_scalar_from_bytes_wide(const uint8_t wide[64], uint64_t out_mont[4]);       /* Scalar::from_bytes_wide  ristretto255.rs:435 */
void sp_scalar_mul(const uint64_t a[4], const uint64_t b[4], uint64_t out[4]);      /* Mul for Scalar           ristretto255.rs:690 */
void sp_scalar_add(const uint64_t a[4], const uint64_t b[4], uint64_t out[4]);      /* ristretto255.rs:736 */
void sp_scalar_sub(const uint64_t a[4], const uint64_t b[4], uint64_t out[4]);      /* ristretto255.rs:718 */
int sp_scalar_invert(const uint64_t a[4], uint64_t out[4]);                         /* Scalar::invert           ristretto255.rs:541 */

/* ---- dense multilinear polynomials on the device */
int sp_poly_upload(sp_ctx* ctx, const uint64_t* limbs_mont, size_t len, sp_poly** out);   /* DensePolynomial::new   dense_mlpoly.rs:121 */
int sp_poly_download(sp_ctx* ctx, const sp_poly* p, uint64_t* limbs_mont, size_t len);
/* n canonical little-endian 32-byte scalars in DEVICE memory of the context's GPU (e.g. a witness computed there) -> a polynomial in Montgomery
 * form, for sp_*_prove_resident.  SP_ERR_INVALID_SCALAR if a value is >= q, SP_ERR_INVALID_ARG if the pointer is not device memory of the
 * context's device.  Same synchronisation rules as sp_instance_create_device. */
int sp_poly_from_canonical_device(sp_ctx* ctx, const uint8_t* d_canonical32, size_t n, sp_poly** out);
size_t sp_poly_len(const sp_poly* p);
void sp_poly_free(sp_poly* p);
/* bound_poly_var_top on k polynomials of equal length                                      dense_mlpoly.rs:215-223 */
int sp_fold_top(sp_ctx* ctx, sp_poly* const* polys, int k, const uint64_t r_mont[4]);
/* one sumcheck round evaluation: kind 0 = A*B (sumcheck.rs:460-469), 1 = A*B*C (sumcheck.rs:204-228), 2 = A*(B*C-D) (sumcheck.rs:625-652).
 * out = [e(0), e(2), e(3)] as Montgomery limbs (e(3) = 0 for kind 0) */
int sp_sumcheck_eval(sp_ctx* ctx, int kind, sp_poly* const* polys, uint64_t out[3][4]);
/* fused: bind the top variable of every table to r, then evaluate the next round on the folded tables */
int sp_sumcheck_fold_eval(sp_ctx* ctx, int kind, sp_poly* const* polys, const uint64_t r_mont[4], uint64_t out[3][4]);
/* the same two calls on a connected context, on CYCLIC SHARDS (rank r holds entries r, r+W, ...): partial sums are exchanged over NVLink inside
 * the kernel ("scalar-add all-reduce"), every rank gets the evaluations of the whole tables; shards of >= 8192 entries for fold_eval */
int sp_sumcheck_eval_sharded(sp_ctx* ctx, int kind, sp_poly* const* polys, uint64_t out[3][4]);
int sp_sumcheck_fold_eval_sharded(sp_ctx* ctx, int kind, sp_poly* const* polys, const uint64_t r[4], uint64_t out[3][4]);
/* SumcheckInstanceProof::prove_cubic_batched evaluation loops (sumcheck.rs:290-357): ninst instances of comb = A*B*C (product_tree.rs:283-286).
 * out = ninst x [e0, e2, e3] Montgomery limbs.  The same sp_poly may be passed as C of several instances (poly_C_par); A and B must be distinct. */
int sp_sumcheck_batched_eval(sp_ctx* ctx, int ninst, sp_poly* const* A, sp_poly* const* B, sp_poly* const* C, uint64_t* out /* ninst*3*4 */);
/* bound_poly_var_top(r) on every table (each shared C once) fused with the next round's evaluations */
int sp_sumcheck_batched_fold_eval(sp_ctx* ctx, int ninst, sp_poly* const* A, sp_poly* const* B, sp_poly* const* C, const uint64_t r_mont[4],
                                  uint64_t* out /* ninst*3*4 */);
/* ---- a whole sumcheck of a caller-defined polynomial (SumcheckInstanceProof::prove_cubic / prove_cubic_batched with any comb_func that is a
 * sum of products of the tables, sumcheck.rs:183-424).  Inputs: k tables P_0 .. P_{k-1} of one length 2^m (the same handle may appear more
 * than once), the composition g = sum_t coeff_t * prod_{j in factor_t} P_j (a factor may repeat: A*A*B), the claim and num_rounds (1 <= num_rounds
 * <= m).  The degree is d = max_t nfactors_t.  Round j: s_j(t) = sum_x g(P(t, x)) at t = 0, 2, 3, .., d (bound points lo + t*(hi - lo));
 * s_j(1) = e - s_j(0); the d+1 coefficients by interpolation over 0..d (UniPoly::from_evals for d = 2, 3, unipoly.rs:23-54); the transcript
 * absorbs the polynomial (label "poly") and draws r_j ("challenge_nextround"); every distinct table is bound with r_j once, in place
 * (bound_poly_var_top); e = s_j(r_j).  Outputs: *proof = bincode(SumcheckInstanceProof) (free with sp_free), r_out = the num_rounds challenges,
 * finals_out = P_j[0] for every j < k after the last bind, e_out = the final e.  Every handle's sp_poly_len is then 2^(m - num_rounds).  Round
 * polynomials always carry d+1 coefficients.  The claim is not checked (neither does the reference).
 * SP_ERR_INVALID_ARG, with the tables untouched: unequal lengths or a length that is not a power of two >= 2, num_rounds out of range, a factor
 * index >= k, a term without factors, d > SP_SC_MAX_DEGREE, k > SP_SC_MAX_TABLES, nterms outside 1..SP_SC_MAX_TERMS, a handle of another
 * context.  SP_ERR_INVALID_SCALAR: a coefficient or the claim is not reduced.  One kernel launch per round plus a constant.  On a connected
 * multi-GPU context the call runs on this rank's GPU alone. */
#define SP_SC_MAX_DEGREE 6
#define SP_SC_MAX_TABLES 8
#define SP_SC_MAX_TERMS 32
typedef struct { uint64_t coeff_mont[4]; uint32_t nfactors; uint32_t factor[SP_SC_MAX_DEGREE]; } sp_sc_term;
int sp_sumcheck_prove_t(sp_ctx* ctx, sp_poly* const* tables, int k, const sp_sc_term* terms, int nterms, const uint64_t claim_mont[4], size_t num_rounds,
                        uint8_t* strobe_state /* in, out */, uint8_t** proof, size_t* proof_len, uint64_t* r_out /* num_rounds x 4 */,
                        uint64_t* finals_out /* k x 4 */, uint64_t e_out[4]);
/* the same on Transcript::new(label) */
int sp_sumcheck_prove(sp_ctx* ctx, sp_poly* const* tables, int k, const sp_sc_term* terms, int nterms, const uint64_t claim_mont[4], size_t num_rounds,
                      const uint8_t* label, size_t label_len, uint8_t** proof, size_t* proof_len, uint64_t* r_out, uint64_t* finals_out, uint64_t e_out[4]);
/* SumcheckInstanceProof::verify(claim, num_rounds, degree_bound, transcript) (sumcheck.rs:27-62), host only: ctx may be NULL (sp_last_error(NULL)
 * then holds the message).  SP_ERR_VERIFY where the reference asserts (round count, degree of a round polynomial, s(0) + s(1) = e) or the bytes
 * do not decode; the transcript is left as the reference's verify leaves it, accepted or not.  On success e_out = the final claim, r_out = the
 * num_rounds challenges.  degree_bound must be >= 1. */
int sp_sumcheck_verify_t(sp_ctx* ctx, const uint8_t* proof, size_t proof_len, const uint64_t claim_mont[4], size_t num_rounds, size_t degree_bound,
                         uint8_t* strobe_state /* in, out */, uint64_t e_out[4], uint64_t* r_out /* num_rounds x 4 */);
int sp_eq_evals(sp_ctx* ctx, const uint64_t* r_mont, size_t ell, sp_poly** out);           /* EqPolynomial::evals   dense_mlpoly.rs:68-84 */
int sp_poly_evaluate(sp_ctx* ctx, const sp_poly* p, const uint64_t* r_mont, size_t ell, uint64_t out[4]); /* DensePolynomial::evaluate :236 */
int sp_poly_bound_rows(sp_ctx* ctx, const sp_poly* p, const uint64_t* L_mont, size_t L_size, sp_poly** out); /* DensePolynomial::bound :206 */
int sp_dot(sp_ctx* ctx, const sp_poly* a, const sp_poly* b, uint64_t out[4]);              /* compute_dotproduct   nizk/mod.rs:435 */

/* ---- Pedersen generators and commitments */
/* MultiCommitGens::new(n, label): G[0..n), h = G[n]  (n+1 points drawn)                    commitments.rs:15-33 */
int sp_gens_create(sp_ctx* ctx, const uint8_t* label, size_t label_len, size_t n, sp_gens** out);
/* the caller's own MultiCommitGens (e.g. after `scale`, commitments.rs:43-49): n+1 encodings, G[0..n) then h; SP_ERR_INVALID_POINT if one fails */
int sp_gens_upload(sp_ctx* ctx, const uint8_t* compressed32, size_t n, sp_gens** out);
void sp_gens_free(sp_gens* g);
int sp_gens_export(sp_ctx* ctx, const sp_gens* g, uint8_t* out32 /* (n+1)*32: G then h */);
/* GroupElement::vartime_multiscalar_mul(scalars, G[0..n)) compressed                       group.rs:98-117 */
int sp_msm(sp_ctx* ctx, const sp_gens* g, const uint64_t* scalars_mont, size_t n, uint8_t out32[32]);
/* DensePolynomial::commit_inner: L rows of R scalars; out[i] = (MSM(row_i, G) + blinds[i]*h).compress(); blinds may be NULL (zero)
 *                                                                                          dense_mlpoly.rs:148-177 */
int sp_commit_rows(sp_ctx* ctx, const sp_gens* g, const sp_poly* p, size_t L, size_t R, const uint64_t* blinds_mont, uint8_t* out32);
int sp_point_decompress_check(sp_ctx* ctx, const uint8_t* in32, size_t n, int* ok);        /* CompressedRistretto::decompress */
int sp_point_roundtrip(sp_ctx* ctx, const uint8_t* in32, size_t n, uint8_t* out32);        /* decompress().compress() on the device */

/* ---- variable-base MSM on caller-supplied points (bucket method; no precomputed tables — for point sets that are used once or are too
 * large for window tables, e.g. the 2^24-point standalone MSM of BASELINE.json).                                   group.rs:98-117 */
/* points cross as n 32-byte encodings; SP_ERR_INVALID_POINT if any fails to decompress */
int sp_points_upload(sp_ctx* ctx, const uint8_t* compressed32, size_t n, sp_points** out);
/* MultiCommitGens::new(n, label).G (the h generator is not kept)                                                   commitments.rs:15-33 */
int sp_points_derive(sp_ctx* ctx, const uint8_t* label, size_t label_len, size_t n, sp_points** out);
size_t sp_points_len(const sp_points* p);
void sp_points_free(sp_points* p);
int sp_points_export(sp_ctx* ctx, const sp_points* p, size_t offset, size_t n, uint8_t* out32);
/* GroupElement::vartime_multiscalar_mul(scalars[0..n), points[offset..offset+n)).compress(); SP_ERR_INVALID_ARG, before any launch, when
 * [offset, offset + n) is not inside the set (an offset + n that wraps past 2^64 included), here and in sp_points_export */
int sp_msm_var(sp_ctx* ctx, const sp_points* p, size_t offset, const uint64_t* scalars_mont, size_t n, uint8_t out32[32]);
int sp_msm_var_resident(sp_ctx* ctx, const sp_points* p, size_t offset, const sp_poly* scalars, uint8_t out32[32]);
/* every rank of a connected context passes its slice of the points and of the scalars; point-add all-reduce of the W partial sums; every rank
 * returns the encoding of the whole sum (group.rs:98-117 on a vector split by index range) */
int sp_msm_var_sharded(sp_ctx* ctx, const sp_points* p, size_t offset, const sp_poly* scalars, uint8_t out32[32]);

/* ---- polynomial commitments and evaluation proofs for the caller's own tables: the Hyrax-style commitment of dense_mlpoly.rs (a table of 2^ell
 * entries is an L x R matrix, L = 2^floor(ell/2) rows of R = 2^ceil(ell/2), each row committed with one Pedersen vector commitment) and its
 * opening by PolyEvalProof (a bulletproofs inner-product argument), bytes identical to the reference's for the same transcript and tape.  Use:
 * commit before a sumcheck, absorb the commitment, run sp_sumcheck_prove_t, then open every table at its r with sp_pc_eval_prove_joint_t on the
 * same transcript.  Every entry below runs on this rank's GPU alone, also on a connected multi-GPU context.  Tables are read, never modified.
 *
 * PolyCommitmentGens::new(num_vars, label) (dense_mlpoly.rs:29-36) = DotProductProofGens::new(n, label), n = 2^(num_vars - num_vars/2)
 * (nizk/mod.rs:414-418): n + 2 points of the label's SHAKE256 stream, gens_n = G[0..n) and gens_1 = G[n], both with h = G[n+1].  Device
 * footprint (read it with sp_device_bytes_live): the n + 2 points and a fixed-base window table, of 8-bit windows (393 KB per generator) for
 * n <= 256; for larger n a 16-bit row table (3.1 MB per generator) and 13-bit windows (7.9 MB per generator; 15-bit, 26.7 MB, from n = 2048),
 * each only if it fits in 65% of the free device memory (else no row table, narrower windows: same bytes, slower).  num_vars = 20: n = 1024,
 * about 11 GB; num_vars = 24: n = 4096, about 32 GB of window table plus 12.7 GB of row table. */
typedef struct sp_pc_gens sp_pc_gens;
#define SP_PC_MAX_TABLES 64
int sp_pc_gens_create(sp_ctx* ctx, size_t num_vars, const uint8_t* label, size_t label_len, sp_pc_gens** out);
/* PolyCommitmentGens::new(num_vars, label) for num_vars <= larger's, as a view of `larger`'s tables (MultiCommitGens::new of any size is a prefix of
 * the label's stream): proves and verifies byte for byte as sp_pc_gens_create(num_vars, label) would, and holds no device memory of its own.  The
 * tables live until the last of the handles that share them is freed.  SP_ERR_INVALID_ARG for a larger num_vars or a handle of another context. */
int sp_pc_gens_create_from(sp_ctx* ctx, const sp_pc_gens* larger, size_t num_vars, sp_pc_gens** out);
void sp_pc_gens_free(sp_pc_gens* g);
/* RandomTape::new(b"proof") (random.rs:10-17) with its seed scalar, as a 203-byte STROBE state like a transcript's (SP_TRANSCRIPT_STATE_BYTES),
 * so that one tape can be threaded through a commitment and later proofs.  The sp_transcript_* helpers work on it.  seed_mont must be FRESH OS
 * RANDOMNESS (Scalar::from_bytes_wide of 64 random bytes, as RandomTape::new draws it): every blind is a function of it. */
int sp_random_tape_new(const uint64_t seed_mont[4], uint8_t* tape_state /* out */);
/* DensePolynomial::merge(polys).commit(gens, tape) (dense_mlpoly.rs:179-204, :259-272): with k = 1 DensePolynomial::commit of the table; with
 * k > 1 the commitment to the k tables concatenated and zero-padded to the next power of two.  *comm = bincode(PolyCommitment) (free with
 * sp_free).  tape_state NULL: no blinds, blinds_out (L scalars) gets zeros; else the tape draws random_vector("poly_blinds", L) and is advanced.
 * blinds_out may be NULL.  SP_ERR_INVALID_ARG, nothing written: k outside 1 .. SP_PC_MAX_TABLES, lengths unequal or not a power of two, gens'
 * n != R of the merged table (the reference asserts gens_n.n == R, commitments.rs:87-91), a handle of another context. */
int sp_pc_commit(sp_ctx* ctx, const sp_pc_gens* gens, sp_poly* const* polys, int k, uint8_t* tape_state /* in, out; NULL = no blinds */, uint8_t** comm,
                 size_t* comm_len, uint64_t* blinds_out /* L x 4 or NULL */);
/* PolyEvalProof::prove(poly, blinds, r, Zr, blind_Zr, gens, transcript, tape) (dense_mlpoly.rs:312-365) on the caller's transcript and tape
 * (both advanced).  ell = |r| = log2 of the table's length, 0 allowed.  blinds: the L blinds of the table's commitment or NULL (zero).  Zr NULL:
 * computed on the device as Z(r); a given Zr is not checked (neither does the reference): the verifier rejects the proof.  blind_Zr NULL: zero.
 * Out: *proof = bincode(PolyEvalProof) (free with sp_free), C_Zr32 = the commitment to Zr the proof is against, Zr_out = the Zr used.
 * SP_ERR_INVALID_ARG: |r| != log2 length, gens' n != R; SP_ERR_INVALID_SCALAR: r, Zr, blind_Zr or a blind not reduced. */
int sp_pc_eval_prove_t(sp_ctx* ctx, const sp_pc_gens* gens, const sp_poly* poly, const uint64_t* blinds_mont, const uint64_t* r_mont, size_t ell,
                       const uint64_t* Zr_mont, const uint64_t* blind_Zr_mont, uint8_t* strobe_state /* in, out */, uint8_t* tape_state /* in, out */,
                       uint8_t** proof, size_t* proof_len, uint8_t C_Zr32[32], uint64_t Zr_out[4]);
/* PolyEvalProof::verify(gens, transcript, r, C_Zr, comm) (dense_mlpoly.rs:367-389) when C_Zr32 is given, verify_plain(.., Zr, ..) (:391-404) when
 * Zr_mont is given (exactly one of them).  comm = bincode(PolyCommitment).  SP_OK = accepted; SP_ERR_VERIFY / SP_ERR_DECOMPRESS = rejected,
 * sp_last_error names the failing check; the transcript is advanced as the reference's verify advances it, accepted or not (an argument
 * refused with SP_ERR_INVALID_ARG / SP_ERR_INVALID_SCALAR leaves it untouched).  Needs the device (<s, G>). */
int sp_pc_eval_verify_t(sp_ctx* ctx, const sp_pc_gens* gens, const uint8_t* comm, size_t comm_len, const uint64_t* r_mont, size_t ell,
                        const uint8_t C_Zr32[32], const uint64_t Zr_mont[4], uint8_t* strobe_state /* in, out */, const uint8_t* proof, size_t proof_len);
/* k tables of 2^m entries opened at one point r (m scalars) through one commitment to their merge (sp_pc_commit of the same k tables):
 * DerefsEvalProof::prove_single (sparse_mlpoly.rs:80-123) without a protocol name (absorb b"Derefs evaluation proof" first to match
 * DerefsEvalProof::prove).  evals_j = P_j(r) are computed on the device, padded with zeros to k' = next_pow2(k) and absorbed as "evals_ops_val";
 * log2 k' challenges "challenge_combine_n_to_one" fold them (bound_poly_var_bot, last challenge first) into "joint_claim_eval"; the merge is proved
 * at (challenges || r) by PolyEvalProof::prove without blind_Zr.  blinds: the joint commitment's L blinds or NULL.  Out: the proof, evals_out =
 * the k evaluations.  After sp_sumcheck_prove_t over the same tables, r = its r_out and evals_out equals its finals_out.  Errors as sp_pc_commit. */
int sp_pc_eval_prove_joint_t(sp_ctx* ctx, const sp_pc_gens* gens, sp_poly* const* polys, int k, const uint64_t* blinds_mont, const uint64_t* r_mont,
                             size_t m, uint8_t* strobe_state /* in, out */, uint8_t* tape_state /* in, out */, uint8_t** proof, size_t* proof_len,
                             uint64_t* evals_out /* k x 4 */);
/* DerefsEvalProof::verify_single (sparse_mlpoly.rs:149-176) for sp_pc_eval_prove_joint_t's proof: evals = the k claimed evaluations */
int sp_pc_eval_verify_joint_t(sp_ctx* ctx, const sp_pc_gens* gens, const uint8_t* comm, size_t comm_len, const uint64_t* r_mont, size_t m,
                              const uint64_t* evals_mont, int k, uint8_t* strobe_state /* in, out */, const uint8_t* proof, size_t proof_len);

/* ---- zero-knowledge sumchecks of a caller-defined polynomial and the sigma protocols that tie committed claims together (sumcheck.rs:64-776,
 * nizk/mod.rs:16-406), on the caller's transcript and tape (both advanced, and written back only when a prove succeeds) and the caller's
 * MultiCommitGens: gens_1 has n = 1, gens_n the n the proof needs; the two may be different sets (sp_gens_create, or sp_gens_upload of the
 * split_at views the reference uses, e.g. gens_pc.gens.gens_1 = [G_n, h]).  Commitments cross as 32-byte ristretto255 encodings.  Bytes equal
 * the reference's for the same transcript, tape and generators.  Every argument is checked before the first launch, tape draw or transcript
 * write, so a refused call leaves the tables, the transcript and the tape byte-identical.  SP_ERR_INVALID_ARG: gens_1.n != 1, a gens_n.n other
 * than the proof's length, a handle of another context, a NULL argument; SP_ERR_INVALID_SCALAR: an unreduced scalar; SP_ERR_INVALID_POINT: a
 * commitment given to a verify that does not decompress.  The verifies return SP_OK when they accept, SP_ERR_VERIFY / SP_ERR_DECOMPRESS when they
 * reject (sp_last_error names the check), and leave the transcript where the reference's verify leaves it.  The sigma protocols commit on the
 * host; each set's host tables are built at its first such use.  On a connected multi-GPU context every entry runs on this rank's GPU alone. */
/* DotProductProof is linear in n: n <= SP_DOTPROD_MAX_N (a ZK sumcheck's rounds need d + 1 <= 7); longer vectors belong to DotProductProofLog
 * (sp_dotlog_prove_t) */
#define SP_DOTPROD_MAX_N 64
/* ZKSumcheckInstanceProof::prove_quad / prove_cubic_with_additive_term (sumcheck.rs:428-776) generalised to the composition of
 * sp_sumcheck_prove_t (same tables, terms, num_rounds and refusals; degree d = max nfactors, 1 <= d <= SP_SC_MAX_DEGREE).  The tape draws
 * blinds_poly and blinds_evals (num_rounds each), then per round d_vec, r_delta, r_beta.  Round j: s_j(0), s_j(2) .. s_j(d) on the device, s_j(1) =
 * claim_j - s_j(0), coefficients as sp_sumcheck_prove_t's; comm_poly = commit(coeffs; blinds_poly[j]; gens_n) absorbed, r_j drawn, then
 * comm_claim_per_round, comm_eval = commit(s_j(r_j); blinds_evals[j]; gens_1), the weights w ("combine_two_claims_to_one") and
 * DotProductProof::prove with a = w0 (2, 1, .., 1) + w1 (1, r_j, .., r_j^d).  At d = 2 with A*B, and at d = 3 with A*B*C - A*D, the bytes are the
 * reference's two provers'.  gens_n.n must be d + 1.  Out: *proof = bincode(ZKSumcheckInstanceProof) (free with sp_free), r_out, finals_out as
 * sp_sumcheck_prove_t's, blind_post_out = blinds_evals[num_rounds - 1] (the blind of the last comm_eval).  One kernel launch per round plus a
 * constant, once gens_1 and gens_n have their host tables (the first call on a set builds them, with launches of their own); no table data
 * reaches the host.  num_rounds is also capped by the pinned area that stages the rounds' tape-only commitments (SP_ERR_INVALID_ARG names the
 * limit, over 200 rounds). */
int sp_zk_sumcheck_prove_t(sp_ctx* ctx, sp_poly* const* tables, int k, const sp_sc_term* terms, int nterms, const uint64_t claim_mont[4],
                           const uint64_t blind_claim_mont[4], size_t num_rounds, const sp_gens* gens_1, const sp_gens* gens_n,
                           uint8_t* strobe_state /* in, out */, uint8_t* tape_state /* in, out */, uint8_t** proof, size_t* proof_len,
                           uint64_t* r_out /* num_rounds x 4 */, uint64_t* finals_out /* k x 4 */, uint64_t blind_post_out[4]);
/* ZKSumcheckInstanceProof::verify(comm_claim, num_rounds, degree_bound, gens_1, gens_n, transcript) (sumcheck.rs:84-179): num_rounds >= 1,
 * gens_n.n = degree_bound + 1 <= SP_DOTPROD_MAX_N.  On success comm_eval_out32 = the last comm_eval, r_out = the num_rounds challenges. */
int sp_zk_sumcheck_verify_t(sp_ctx* ctx, const uint8_t* proof, size_t proof_len, const uint8_t comm_claim32[32], size_t num_rounds, size_t degree_bound,
                            const sp_gens* gens_1, const sp_gens* gens_n, uint8_t* strobe_state /* in, out */, uint8_t comm_eval_out32[32],
                            uint64_t* r_out /* num_rounds x 4 */);
/* KnowledgeProof::prove(gens_n, transcript, tape, x, r) -> (proof, C)  /  ::verify(gens_n, transcript, C)        nizk/mod.rs:27-75; gens_n.n = 1 */
int sp_knowledge_prove_t(sp_ctx* ctx, const sp_gens* gens_n, uint8_t* strobe_state, uint8_t* tape_state, const uint64_t x_mont[4], const uint64_t r_mont[4],
                         uint8_t** proof, size_t* proof_len, uint8_t C_out32[32]);
int sp_knowledge_verify_t(sp_ctx* ctx, const sp_gens* gens_n, uint8_t* strobe_state, const uint8_t C32[32], const uint8_t* proof, size_t proof_len);
/* EqualityProof::prove(gens_n, transcript, tape, v1, s1, v2, s2) -> (proof, C1, C2)  /  ::verify(gens_n, transcript, C1, C2)   :88-143; n = 1 */
int sp_equality_prove_t(sp_ctx* ctx, const sp_gens* gens_n, uint8_t* strobe_state, uint8_t* tape_state, const uint64_t v1_mont[4], const uint64_t s1_mont[4],
                        const uint64_t v2_mont[4], const uint64_t s2_mont[4], uint8_t** proof, size_t* proof_len, uint8_t C1_out32[32], uint8_t C2_out32[32]);
int sp_equality_verify_t(sp_ctx* ctx, const sp_gens* gens_n, uint8_t* strobe_state, const uint8_t C1_32[32], const uint8_t C2_32[32], const uint8_t* proof,
                         size_t proof_len);
/* ProductProof::prove(gens_n, transcript, tape, x, rX, y, rY, z, rZ) -> (proof, X, Y, Z)  /  ::verify(gens_n, transcript, X, Y, Z)
 *                                                                                                                     :159-290; n = 1 */
int sp_product_prove_t(sp_ctx* ctx, const sp_gens* gens_n, uint8_t* strobe_state, uint8_t* tape_state, const uint64_t x_mont[4], const uint64_t rX_mont[4],
                       const uint64_t y_mont[4], const uint64_t rY_mont[4], const uint64_t z_mont[4], const uint64_t rZ_mont[4], uint8_t** proof,
                       size_t* proof_len, uint8_t X_out32[32], uint8_t Y_out32[32], uint8_t Z_out32[32]);
int sp_product_verify_t(sp_ctx* ctx, const sp_gens* gens_n, uint8_t* strobe_state, const uint8_t X32[32], const uint8_t Y32[32], const uint8_t Z32[32],
                        const uint8_t* proof, size_t proof_len);
/* DotProductProof::prove(gens_1, gens_n, transcript, tape, x_vec, blind_x, a_vec, y, blind_y) -> (proof, Cx, Cy)  /
 * ::verify(gens_1, gens_n, transcript, a_vec, Cx, Cy)                              :311-405; vectors of n = gens_n.n <= SP_DOTPROD_MAX_N entries */
int sp_dotproduct_prove_t(sp_ctx* ctx, const sp_gens* gens_1, const sp_gens* gens_n, uint8_t* strobe_state, uint8_t* tape_state, const uint64_t* x_vec_mont,
                          const uint64_t blind_x_mont[4], const uint64_t* a_vec_mont, size_t n, const uint64_t y_mont[4], const uint64_t blind_y_mont[4],
                          uint8_t** proof, size_t* proof_len, uint8_t Cx_out32[32], uint8_t Cy_out32[32]);
int sp_dotproduct_verify_t(sp_ctx* ctx, const sp_gens* gens_1, const sp_gens* gens_n, uint8_t* strobe_state, const uint64_t* a_vec_mont, size_t n,
                           const uint8_t Cx32[32], const uint8_t Cy32[32], const uint8_t* proof, size_t proof_len);

/* ---- inner products of the caller's committed vectors in logarithmic size: DotProductProofLog (nizk/mod.rs:407-583, nizk/bullet.rs:32-225), the
 * proof that Cx = <x, G> + blind_x * h commits to a vector x whose inner product with a public vector a is the y of Cy = y * G_n + blind_y * h.
 * Conventions of the sigma protocols above (transcript and tape advanced and written back only when a prove succeeds, every argument checked
 * before the first launch, tape draw or transcript write, this rank's GPU alone).  x and a are sp_poly handles of n entries, read and never
 * modified: the prover folds copies.  Bytes equal the reference's for the same transcript, tape and vectors.
 *
 * Two layouts of the generators, chosen by n alone:
 *   n <= SP_DOTLOG_TABLE_MAX_N: the set sp_pc_gens_create builds for this n (n + 2 points and 8-bit window tables, 393 KB per generator: at most
 *     about 100 MB); the proof runs the inner-product rounds of PolyEvalProof over the unfolded generators.  256 is the largest n whose n + 2
 *     generators stay under the 512 from which a set gets a row table and wider windows, gigabytes an inner-product proof never reads.
 *   larger n: G[0..n) as affine niels points (96 B each, no window tables; 2^24 points take 1.6 GB) and a two-generator set {G_n, h}.  Every
 *     round folds the generators on the device (H' = H_L + u^2 H_R with G = c * H, one variable-base multiplication per pair) and computes L and
 *     R by MSMs over the folded halves.  A prove also holds copies of x and a and the round's MSM scalars (32 B per entry each), n/2 folded points
 *     (96 B each) and the bucket MSM's scratch for n terms (about 100 B per term at n = 2^24): about 3 GB at n = 2^24; a verify holds the vector s
 *     (32 B per entry) and the same MSM scratch.  All of it is released on return.  DESIGN.md ("Inner products of the caller's vectors") has the numbers. */
#define SP_DOTLOG_MAX_N (1u << 24)
#define SP_DOTLOG_TABLE_MAX_N 256
typedef struct sp_dotlog_gens sp_dotlog_gens;
/* DotProductProofGens::new(n, label) (nizk/mod.rs:414-419) = MultiCommitGens::new(n + 1, label).split_at(n): gens_n = G[0..n), gens_1 = G[n], both
 * with h = G[n + 1].  SP_ERR_INVALID_ARG, before any allocation, unless n is a power of two with 1 <= n <= SP_DOTLOG_MAX_N. */
int sp_dotlog_gens_create(sp_ctx* ctx, size_t n, const uint8_t* label, size_t label_len, sp_dotlog_gens** out);
void sp_dotlog_gens_free(sp_dotlog_gens* g);
/* DotProductProofLog::prove(gens, transcript, tape, x_vec, blind_x, a_vec, y, blind_y) -> (proof, Cx, Cy)   nizk/mod.rs:440-525.
 * y NULL: y = <x, a>, computed on the device; a given y is not checked (neither does the reference): the verifier rejects the proof.  Out: *proof =
 * bincode(DotProductProofLog) (free with sp_free), Cx, Cy and y_out = the y used.  SP_ERR_INVALID_ARG: a NULL argument, x or a of another context
 * or of a length other than gens' n; SP_ERR_INVALID_SCALAR: blind_x, y or blind_y not reduced. */
int sp_dotlog_prove_t(sp_ctx* ctx, const sp_dotlog_gens* gens, uint8_t* strobe_state /* in, out */, uint8_t* tape_state /* in, out */, const sp_poly* x,
                      const uint64_t blind_x_mont[4], const sp_poly* a, const uint64_t* y_mont /* NULL: <x, a> */, const uint64_t blind_y_mont[4],
                      uint8_t** proof, size_t* proof_len, uint8_t Cx_out32[32], uint8_t Cy_out32[32], uint64_t y_out[4]);
/* DotProductProofLog::verify(n, gens, transcript, a, Cx, Cy) with BulletReductionProof::verify (nizk/mod.rs:527-583, bullet.rs:137-225): SP_OK =
 * accepted; SP_ERR_VERIFY / SP_ERR_DECOMPRESS = rejected, sp_last_error names the check (an L_vec or R_vec of a length other than log2 n, or of 32
 * or more, is SP_ERR_VERIFY), the transcript left where the reference's verify leaves it.  SP_ERR_INVALID_ARG: a NULL argument, n != gens' n, a of
 * another context or length; SP_ERR_INVALID_POINT: Cx or Cy does not decompress; a refused call leaves the transcript untouched. */
int sp_dotlog_verify_t(sp_ctx* ctx, const sp_dotlog_gens* gens, uint8_t* strobe_state /* in, out */, const sp_poly* a, size_t n, const uint8_t Cx32[32],
                       const uint8_t Cy32[32], const uint8_t* proof, size_t proof_len);

/* ---- product circuits over the caller's tables and the batched proof of their products: the grand-product argument of the reference's memory
 * check (ProductCircuit, ProductCircuitEvalProofBatched, product_tree.rs), bytes identical to the reference's for the same transcript.  Use, e.g.
 * for an offline memory check, multiset equality or a lookup argument: commit to the tuple tables (sp_pc_commit), draw the fingerprint
 * challenges, build one circuit per fingerprinted multiset (sp_prod_build), absorb the products, prove them (sp_prod_prove_t), and open the
 * tables at the point the proof ends on (sp_pc_eval_prove_joint_t); the verifier checks the leaf claims with sp_prod_leaf_eval.  Every entry runs
 * on this rank's GPU alone, also on a connected multi-GPU context.  sp_prod_build / sp_prod_prove_t / sp_prod_verify_t prove products alone
 * (the reference's prove with dotp_circuit_vec empty: the proof's claims_dotp are three empty vectors); the _dotp entries below also prove dot
 * products batched into the last layer's sumcheck.
 *
 * Circuit c's leaf at index x < 2^m is an affine form of up to SP_PROD_MAX_SOURCES of the tables and of x itself:
 *   leaf_c[x] = const_c + index_coeff_c * x + sum_{s < nsources_c} coeff_{c,s} * tables[source_{c,s}][x]
 * A plain table is one source with coefficient one.  The memory check's hash(addr, val, ts) - r_multiset = ts*r^2 + val*r + addr - gamma
 * (sparse_mlpoly.rs:542-591) is sources (ts, r^2), (val, r), (addr, 1) and const -gamma; for init / audit addr is the index (index_coeff = 1), and
 * the write set's ts + 1 moves r^2 into the constant.  All scalars are Montgomery limbs and must be reduced (< q).
 *
 * Device footprint (32 bytes per scalar): 2^(m+1) scalars per circuit, every layer kept, from sp_prod_build until sp_prod_prove_t or sp_prod_free;
 * sp_prod_prove_t adds 2^m scalars of eq tables (poly_C_par and its two ping-pong halves) plus O(2^(m/2)) scalars, released on return.  At
 * m = 20: 64 MiB per circuit and 32 MiB for the proof. */
#define SP_PROD_MAX_CIRCUITS 24   /* = the instances of one batched sumcheck launch: one launch per round */
#define SP_PROD_MAX_SOURCES 3
typedef struct {
  uint32_t nsources;                          /* 0 .. SP_PROD_MAX_SOURCES */
  uint32_t source[SP_PROD_MAX_SOURCES];       /* indices into the tables array */
  uint64_t coeff_mont[SP_PROD_MAX_SOURCES][4];
  uint64_t index_coeff_mont[4];               /* times x: IdentityPolynomial (dense_mlpoly.rs:101-117) */
  uint64_t const_mont[4];
} sp_prod_leaves;
typedef struct sp_prod_circuits sp_prod_circuits;
/* ProductCircuit::new of each of k circuits of 2^m leaves, then ProductCircuit::evaluate (product_tree.rs:36-63).  tables: ntables handles of one
 * length 2^m, m >= 1 (the reference panics without a product layer); the same handle may appear twice.  leaves NULL: k = ntables and circuit i's
 * leaves are table i.  Out: *out, and products_out = the k products.  The tables are read, never modified.  One launch builds the leaves and the
 * first product layer of every circuit; each further layer is one launch per group of at most 16 circuits: 1 + ceil(k/16) (m - 2) launches for
 * m >= 2, one for m = 1.
 * SP_ERR_INVALID_ARG: k outside 1 .. SP_PROD_MAX_CIRCUITS, ntables < 1, a NULL table or one of another context, unequal lengths or a length that
 * is not a power of two >= 2, nsources > SP_PROD_MAX_SOURCES or a source >= ntables, leaves NULL with k != ntables.  SP_ERR_INVALID_SCALAR: a
 * coefficient or constant not reduced.  A refused call allocates and launches nothing. */
int sp_prod_build(sp_ctx* ctx, sp_poly* const* tables, int ntables, const sp_prod_leaves* leaves, int k, sp_prod_circuits** out,
                  uint64_t* products_out /* k x 4 */);
/* ProductCircuitEvalProofBatched::prove(circuits, [], transcript) (product_tree.rs:259-383) on the caller's transcript.  The proof does not absorb
 * the products: absorb them first, as ProductLayerProof::prove does (sparse_mlpoly.rs:1061-1064).  Out: *proof = bincode(ProductCircuitEvalProofBatched)
 * (free with sp_free), rand_out = the m scalars of the point the proof ends on, leaf_evals_out = each circuit's leaf polynomial at rand (the
 * last claims_to_verify: the values sp_prod_verify_t returns as leaf claims).  Consumes the circuits: their layers are bound in place and released,
 * and a second call on the handle is refused (SP_ERR_INVALID_ARG), as are a NULL handle, one of another context and one made by
 * sp_prod_build_dotp with dot products (prove it with sp_prod_prove_dotp_t; the handle is then not consumed); a refused call leaves the
 * transcript untouched.  Launches, independent of k: one per sumcheck round plus a few per layer (tests/test_gpu_product.py states the count). */
int sp_prod_prove_t(sp_ctx* ctx, sp_prod_circuits* c, uint8_t* strobe_state /* in, out */, uint8_t** proof, size_t* proof_len,
                    uint64_t* rand_out /* m x 4 */, uint64_t* leaf_evals_out /* k x 4 */);
void sp_prod_free(sp_prod_circuits* c);
/* ProductCircuitEvalProofBatched::verify(products, [], 2^m, transcript) (product_tree.rs:385-485), host only: ctx may be NULL (sp_last_error(NULL)
 * then holds the message).  SP_OK: accepted, rand_out = the m scalars, leaf_claims_out = the k claims about the leaf polynomials at rand.
 * SP_ERR_VERIFY: rejected (wrong depth, claim shapes, a layer check, non-empty dotp claims, bytes that do not decode), the transcript left as the
 * reference's verify leaves it.  SP_ERR_INVALID_ARG: k outside 1 .. SP_PROD_MAX_CIRCUITS or m outside 1 .. 60; SP_ERR_INVALID_SCALAR: a product
 * not reduced; either leaves the transcript untouched. */
int sp_prod_verify_t(sp_ctx* ctx, const uint8_t* proof, size_t proof_len, const uint64_t* products_mont, int k, size_t m,
                     uint8_t* strobe_state /* in, out */, uint64_t* rand_out /* m x 4 */, uint64_t* leaf_claims_out /* k x 4 */);
/* host only: each circuit's leaf polynomial at rand (m scalars) from the tables' values there (e.g. sp_pc_eval_prove_joint_t's evals_out):
 * const + index_coeff * sum_i 2^(m-1-i) rand_i + sum_s coeff_s * table_evals[source_s].  The verifier compares it with sp_prod_verify_t's leaf
 * claims.  leaves NULL: circuit i is table i (k = ntables).  Refusals as sp_prod_build's. */
int sp_prod_leaf_eval(const sp_prod_leaves* leaves, int k, const uint64_t* table_evals_mont, int ntables, const uint64_t* rand_mont, size_t m,
                      uint64_t* out /* k x 4 */);

/* ---- dot products beside the product circuits: ProductCircuitEvalProofBatched::prove(prod_circuit_vec, dotp_circuit_vec, transcript) with the
 * caller's dot products sum_x left[x] * right[x] * weight[x] over x < 2^m, batched into the sumcheck of the circuits' last layer (product_tree.rs:
 * 259-485).  SPARK proves a sparse evaluation this way from its dereferenced values (sparse_mlpoly.rs:1090-1117); a caller's own memory check
 * proves the value its reads add up to.  Each operand is an affine form of the tables, exactly as a circuit's leaves (sp_prod_leaves): a plain
 * table, a fingerprint, the index or a constant (weight = 1 is const = one).  The library splits each dot product into its halves
 * [0, 2^(m-1)) and [2^(m-1), 2^m) (DotProductCircuit::split) and batches them as the reference's verifier pairs them: dotp_circuit_vec =
 * half 0 of dot product 0, half 1 of dot product 0, half 0 of dot product 1, ..  So `let (l, r) = d.split(); dotp_vec.push(l); dotp_vec.push(r)`
 * is one dot product here, and claims_dotp_vec is the 2 kd half sums sp_prod_build_dotp returns.
 * Limits: 1 <= k, 1 <= kd and k + 2 kd <= SP_PROD_MAX_CIRCUITS (the circuits and both halves of every dot product are instances of one batched
 * sumcheck launch).  Device footprint: 3 * 2^m scalars per dot product (its operands, bound in place by the proof), from sp_prod_build_dotp until
 * sp_prod_prove_dotp_t or sp_prod_free; at m = 20, 96 MiB per dot product. */
/* sp_prod_build with kd dot products: dotp_forms holds 3 kd forms, (left, right, weight) of each dot product.  One more launch than sp_prod_build
 * writes every dot product's operands and sums each half.  Out: as sp_prod_build's, and dotp_claims_out = the two half sums of each dot product
 * (claims_dotp_vec, DotProductCircuit::evaluate of each half).  Refusals as sp_prod_build's, also for the dot products' counts, sources, reduced
 * coefficients and constants, and NULL dotp_forms or dotp_claims_out; a refused call allocates and launches nothing. */
int sp_prod_build_dotp(sp_ctx* ctx, sp_poly* const* tables, int ntables, const sp_prod_leaves* leaves, int k, const sp_prod_leaves* dotp_forms /* 3 kd */,
                       int kd, sp_prod_circuits** out, uint64_t* products_out /* k x 4 */, uint64_t* dotp_claims_out /* 2 kd x 4 */);
/* sp_prod_prove_t for a handle of either build: the proof carries the dot products' final claims, and dotp_evals_out = (left, right, weight) at
 * rand of each dot product (the values sp_prod_verify_dotp_t returns as dotp claims).  dotp_evals_out may be NULL for a handle without dot
 * products.  Consumes the circuits, and refuses as sp_prod_prove_t.  Launches: sp_prod_prove_t's, plus one per eq-factored round of the last
 * layer (rounds whose tables hold >= 2^14 entries: the dot-product instances take a second launch there), plus, when the last layer's tables
 * (two per circuit, six per dot product) exceed 64, one at m = 1 and m >= 15 and two at m = 2 (the gather of its final claims at m <= 2 and
 * the bind of its one round at m = 2 or of the switch out of its eq-factored rounds at m >= 15 take 64 tables per launch;
 * tests/test_gpu_product_dotp.py states the count). */
int sp_prod_prove_dotp_t(sp_ctx* ctx, sp_prod_circuits* c, uint8_t* strobe_state /* in, out */, uint8_t** proof, size_t* proof_len,
                         uint64_t* rand_out /* m x 4 */, uint64_t* leaf_evals_out /* k x 4 */, uint64_t* dotp_evals_out /* 3 kd x 4 */);
/* ProductCircuitEvalProofBatched::verify(products, dotp_claims, 2^m, transcript), host only (ctx may be NULL): dotp_claims = the 2 kd half sums.
 * SP_OK: accepted, rand_out and leaf_claims_out as sp_prod_verify_t's, and dotp_claims_out = (left, right, weight) at rand of each dot product: the
 * verifier checks them with sp_prod_leaf_eval on the operand forms.  SP_ERR_VERIFY, SP_ERR_INVALID_ARG and SP_ERR_INVALID_SCALAR as
 * sp_prod_verify_t's, also for kd (the limits above), NULL dotp_claims or dotp_claims_out and half sums not reduced. */
int sp_prod_verify_dotp_t(sp_ctx* ctx, const uint8_t* proof, size_t proof_len, const uint64_t* products_mont, int k, const uint64_t* dotp_claims_mont /* 2 kd x 4 */,
                          int kd, size_t m, uint8_t* strobe_state /* in, out */, uint64_t* rand_out /* m x 4 */, uint64_t* leaf_claims_out /* k x 4 */,
                          uint64_t* dotp_claims_out /* 3 kd x 4 */);

/* ---- SPARK: commitments to the caller's sparse matrices and proofs of their evaluations (SparseMatPolyCommitmentGens, SparseMatPolynomial::
 * multi_commit / multi_evaluate, SparseMatPolyEvalProof::{prove, verify}, src/sparse_mlpoly.rs), for b = 1 .. SP_SPARK_MAX_BATCH matrices of
 * 2^num_vars_x rows and 2^num_vars_y columns each (x != y allowed; the memory has 2^max(x, y) cells).  SNARK::encode / prove / verify run
 * through the same code with the three R1CS matrices.  Every entry runs on this rank's GPU alone, also on a connected multi-GPU context.
 *
 * b = 3: commitment and proof bytes are the reference's.  Other b: the reference's ProductLayerProof::prove asserts b = 3 (sparse_mlpoly.rs:
 * 1121-1122, a TODO); its verifier is general in b.  The proof is the generalisation the TODO implies: the ops product proof batches the circuits
 * row.read[0..b), row.write[0..b), col.read[0..b), col.write[0..b) with the dot-product circuits left_0, right_0, left_1, right_1, .. (the order
 * the verifier's claims_dotp_circuit assumes, :1264-1270), and the reference's verify accepts it.  b <= 4 because those 6b circuits go in one
 * batched sumcheck launch per round (24 instances). */
#define SP_SPARK_MAX_BATCH 4
typedef struct sp_spark_gens sp_spark_gens;
typedef struct sp_spark_dense sp_spark_dense;   /* MultiSparseMatPolynomialAsDense on the device (sparse_mlpoly.rs:274-282) */
/* SparseMatPolyCommitmentGens::new(label, num_vars_x, num_vars_y, num_nz_entries, batch_size) (sparse_mlpoly.rs:292-317): gens_ops, gens_mem and
 * gens_derefs as views of one set of the label's SHAKE stream, of num_vars_ops = log2 next_pow2(nz) + log2 next_pow2(5b), num_vars_mem =
 * max(x, y) + 1, num_vars_derefs = log2 next_pow2(nz) + log2 next_pow2(2b).  Device footprint as sp_pc_gens_create's for the largest of the three
 * n = 2^(v - v/2): nz = 2^20 with b = 4 gives n_ops = 8192, whose full-width tables do not fit beside a prover, so the set falls back to narrower
 * windows (same bytes, speed not measured).  SP_ERR_INVALID_ARG: batch_size outside 1 .. SP_SPARK_MAX_BATCH, max(x, y) = 0 or > 30. */
int sp_spark_gens_create(sp_ctx* ctx, const uint8_t* label, size_t label_len, size_t num_vars_x, size_t num_vars_y, size_t num_nz_entries, size_t batch_size,
                         sp_spark_gens** out);
void sp_spark_gens_free(sp_spark_gens* g);
/* one matrix's entries: nnz (row, col, canonical 32-byte value) */
typedef struct { const uint64_t* row; const uint64_t* col; const uint8_t* val32; size_t nnz; } sp_spark_entries;
/* SparseMatPolynomial::multi_commit(polys, gens) (sparse_mlpoly.rs:483-503) of b matrices.  *dense: the decommitment, on the device (free with
 * sp_spark_dense_free): comb_ops (next_pow2(5b) N scalars), comb_mem (2 * 2^max(x, y)) and 2b N address indices, N = max_i next_pow2(nnz_i);
 * 32 bytes per scalar, so nz = 2^20, b = 3 holds 512 MiB of comb_ops.  *comm = bincode(SparseMatPolyCommitment) (free with sp_free).
 * SP_ERR_INVALID_INDEX: a row >= 2^x ("row") or col >= 2^y ("col"); SP_ERR_INVALID_SCALAR: a value >= q; the first bad entry in (matrix, entry,
 * row/col/scalar) order is reported.  SP_ERR_INVALID_ARG, before anything is allocated: b outside 1 .. SP_SPARK_MAX_BATCH, N < 2 (every matrix
 * has at most one entry: the product circuits would have no layer), max(x, y) = 0 or > 30 (32-bit addresses), gens of other sizes (their three
 * views' n against those of (x, y, N, b)), a handle of another context, NULL arrays with nnz > 0. */
int sp_spark_commit(sp_ctx* ctx, const sp_spark_gens* gens, const sp_spark_entries* matrices, int b, size_t num_vars_x, size_t num_vars_y,
                    sp_spark_dense** dense, uint8_t** comm, size_t* comm_len);
/* the same with every array in DEVICE memory of the context's GPU: the synchronisation rules and pointer checks of sp_instance_create_device */
int sp_spark_commit_device(sp_ctx* ctx, const sp_spark_gens* gens, const sp_spark_entries* matrices, int b, size_t num_vars_x, size_t num_vars_y,
                           sp_spark_dense** dense, uint8_t** comm, size_t* comm_len);
void sp_spark_dense_free(sp_spark_dense* d);
/* SparseMatPolynomial::multi_evaluate (sparse_mlpoly.rs:440-452) on the device: out[i] = M_i(rx, ry), |rx| = x, |ry| = y */
int sp_spark_evaluate(sp_ctx* ctx, const sp_spark_dense* dense, const uint64_t* rx_mont, size_t x, const uint64_t* ry_mont, size_t y,
                      uint64_t* out /* b x 4 */);
/* SparseMatPolyEvalProof::prove(dense, rx, ry, evals, gens, transcript, tape) (sparse_mlpoly.rs:1447-1514) on the caller's transcript and tape
 * (both advanced).  Like the reference's, the proof absorbs neither the commitment nor the evaluations: the caller absorbs them first, as
 * SNARK::prove absorbs Ar/Br/Cr_claim.  evals NULL: computed on the device; given evals that differ from M_i(rx, ry) are refused.  Out: *proof =
 * bincode(SparseMatPolyEvalProof) (free with sp_free), evals_out = the b evaluations.  SP_ERR_INVALID_ARG: |rx| != x or |ry| != y of the dense,
 * gens that do not fit it, a wrong evaluation, a handle of another context; SP_ERR_INVALID_SCALAR: rx, ry or evals not reduced.  A refused call
 * leaves the transcript and the tape untouched. */
int sp_spark_eval_prove_t(sp_ctx* ctx, const sp_spark_dense* dense, const sp_spark_gens* gens, const uint64_t* rx_mont, size_t x, const uint64_t* ry_mont,
                          size_t y, const uint64_t* evals_mont /* b x 4 or NULL */, uint8_t* strobe_state /* in, out */, uint8_t* tape_state /* in, out */,
                          uint8_t** proof, size_t* proof_len, uint64_t* evals_out /* b x 4 */);
/* SparseMatPolyEvalProof::verify(comm, rx, ry, evals, gens, transcript) (sparse_mlpoly.rs:1516-1557).  comm = bincode(SparseMatPolyCommitment).
 * SP_OK: accepted.  SP_ERR_VERIFY / SP_ERR_DECOMPRESS: rejected, sp_last_error names the check, the transcript advanced as the reference's verify
 * advances it.  A commitment that does not decode or does not fit the call (batch_size != b, num_ops not a power of two >= 2, num_mem_cells !=
 * 2^max(x, y), gens whose views do not fit) is SP_ERR_VERIFY with the transcript untouched.  SP_ERR_INVALID_ARG: b outside 1 ..
 * SP_SPARK_MAX_BATCH, NULL arguments; SP_ERR_INVALID_SCALAR: rx, ry or evals not reduced; both leave the transcript untouched. */
int sp_spark_eval_verify_t(sp_ctx* ctx, const sp_spark_gens* gens, const uint8_t* comm, size_t comm_len, const uint64_t* rx_mont, size_t x,
                           const uint64_t* ry_mont, size_t y, const uint64_t* evals_mont, int b, uint8_t* strobe_state /* in, out */, const uint8_t* proof,
                           size_t proof_len);

/* ---- products of the caller's sparse matrices with vectors on the device: SparseMatPolynomial::multiply_vec (src/sparse_mlpoly.rs:454-464) and
 * compute_eval_table_sparse (:466-481), for b = 1 .. SP_SPMAT_MAX_BATCH matrices of one shape (2^num_vars_x rows, 2^num_vars_y columns, x, y
 * <= 30, fewer than 2^32 entries in all, nnz = 0 allowed).  b <= 8 = SP_SC_MAX_TABLES: the outputs are the tables of one caller sumcheck.
 *
 * sp_spmat holds every matrix twice on the device, sorted by row and sorted by column (stable: equal keys keep the caller's order), each entry as
 * a 32-bit key, a 32-bit source index and a 32-byte Montgomery value: 80 bytes per entry, so 2^22 entries hold 320 MiB.  Building it also needs
 * about 56 bytes per entry of the largest matrix, released on return: 40 for the ingested copy (row, column, value) and 16 for the sort (positions,
 * permutation, and CUB's alternate key and value buffers); host arrays are staged on the device first, 48 bytes per entry more.  It records the
 * largest row and column of all its entries, so a product call checks its bounds without reading the device.
 *
 * Every product runs on tiles of 1024 entries of the whole batch, whatever the rows' lengths: one row or column holding most entries costs what
 * the same number of entries spread over many rows costs.  One call launches SP_SPMAT_PRODUCT_LAUNCHES kernels for every shape and skew (the
 * weighted eval table one more), plus one memset per output; no table crosses PCIe.  Field addition is exact, so the outputs are the reference's
 * bytes. */
#define SP_SPMAT_MAX_BATCH 8
#define SP_SPMAT_PRODUCT_LAUNCHES 3
typedef struct sp_spmat sp_spmat;
/* the b matrices' entries (sp_spark_entries of host arrays).  SP_ERR_INVALID_INDEX: a row >= 2^x ("row") or col >= 2^y ("col");
 * SP_ERR_INVALID_SCALAR: a value >= q; the first bad entry in (matrix, entry, row/col/scalar) order is reported.  SP_ERR_INVALID_ARG, before
 * anything is allocated: b outside 1 .. SP_SPMAT_MAX_BATCH, x or y > 30, 2^32 or more entries in all, NULL arrays with nnz > 0. */
int sp_spmat_create(sp_ctx* ctx, const sp_spark_entries* matrices, int b, size_t num_vars_x, size_t num_vars_y, sp_spmat** out);
/* the same with every array in DEVICE memory of the context's GPU: the synchronisation rules and pointer checks of sp_instance_create_device */
int sp_spmat_create_device(sp_ctx* ctx, const sp_spark_entries* matrices, int b, size_t num_vars_x, size_t num_vars_y, sp_spmat** out);
void sp_spmat_free(sp_spmat* m);
/* multiply_vec of every matrix: outs[m] = M_m z, a new polynomial of num_rows entries (free each with sp_poly_free).  As in the reference,
 * len(z) = num_cols, and num_rows, num_cols >= 1 may be any sizes (not only 2^x, 2^y, nor powers of two) that hold every entry: rows past the
 * last entry read zero.  SP_ERR_INVALID_ARG where the reference panics (len(z) != num_cols, a row >= num_rows, a col >= num_cols), and for
 * num_rows or num_cols of 0 or above 2^32, NULL arguments, handles of another context.  A refused call launches nothing, allocates no output
 * and leaves z and outs untouched. */
int sp_spmat_multiply_vec(sp_ctx* ctx, const sp_spmat* mats, size_t num_rows, size_t num_cols, const sp_poly* z, sp_poly** outs /* b */);
/* compute_eval_table_sparse of every matrix: outs[m] = M_m^T e, num_cols entries, with e the eq table of len(e) = num_rows entries (not the
 * point).  weights != NULL: the one table outs[0] = sum_m w_m M_m^T e (the R1CS prover's r_A, r_B, r_C combination), from the b tables in
 * scratch and one more launch.  Refusals as sp_spmat_multiply_vec's (len(e) != num_rows instead of len(z)), and SP_ERR_INVALID_SCALAR for a
 * weight that is not reduced; e, the weights and outs are left untouched. */
int sp_spmat_eval_table(sp_ctx* ctx, const sp_spmat* mats, const sp_poly* e, size_t num_rows, size_t num_cols, const uint64_t* weights_mont /* b x 4 or NULL */,
                        sp_poly** outs /* b, or 1 with weights */);

/* ---- R1CSProof of the caller's matrices: R1CSGens::new (src/r1csproof.rs:61-74), R1CSProof::prove (:144-349) and ::verify (:351-489) on the
 * caller's transcript and tape, on this rank's GPU alone (a connected multi-GPU context does not shard these calls).  The proof is the one
 * NIZK::prove and SNARK::prove embed; the verifier takes the three claimed evaluations (A(rx, ry), B(rx, ry), C(rx, ry)) instead of the matrices,
 * so a caller can prove those with its own argument (sp_spark_*, or a closed form of structured matrices).
 *
 * num_cons >= 2 and num_vars >= 1 are powers of two (the padded sizes), log2 num_cons and log2 (2 num_vars) at most 32.  z = vars || 1 || inputs ||
 * 0.. has 2 num_vars entries, and |inputs| + 1 <= num_vars (r1csproof.rs:156). */
typedef struct sp_r1cs_gens sp_r1cs_gens;
/* R1CSGens::new(label, num_cons, num_vars): gens_pc = PolyCommitmentGens::new(log2 num_vars, label) and the sumcheck gens gens_1 (= gens_pc's),
 * gens_3 and gens_4, all prefixes of the label's one stream: max(2^ceil(log2(num_vars) / 2) + 2, 5) generators with the device tables and
 * footprint of sp_pc_gens_create's set.  NIZKGens / SNARKGens use the label "gens_r1cs_sat". */
int sp_r1cs_gens_create(sp_ctx* ctx, const uint8_t* label, size_t label_len, size_t num_cons, size_t num_vars, sp_r1cs_gens** out);
/* the same gens as a view of an existing gens_r1cs_sat set: of generator tables, of NIZK gens or of SNARK gens.  No device memory is added; the
 * view keeps the set alive.  SP_ERR_INVALID_ARG: a set shorter than num_vars needs, or of another context */
int sp_r1cs_gens_create_from(sp_ctx* ctx, const struct sp_gen_tables* tables /* sp_gen_tables, below */, size_t num_cons, size_t num_vars, sp_r1cs_gens** out);
int sp_r1cs_gens_create_from_nizk(sp_ctx* ctx, const sp_nizk_gens* gens, size_t num_cons, size_t num_vars, sp_r1cs_gens** out);
int sp_r1cs_gens_create_from_snark(sp_ctx* ctx, const sp_snark_gens* gens, size_t num_cons, size_t num_vars, sp_r1cs_gens** out);
void sp_r1cs_gens_free(sp_r1cs_gens* g);
/* R1CSProof::prove(inst, vars, inputs, gens, transcript, random_tape): the matrices are exactly one of
 *   inst   an instance of num_cons x num_vars (padded): its products run as NIZK::prove's, one thread per row or column (k_spmv), so one row or
 *          column holding most entries costs seconds at 2^20 (DESIGN.md "Products of the caller's matrices");
 *   spmat  an sp_spmat of exactly 3 matrices A, B, C of 2^log2(num_cons) rows and 2^log2(2 num_vars) columns: the tiled products of
 *          sp_spmat_multiply_vec / sp_spmat_eval_table, whose time does not depend on how the entries spread over rows and columns.
 * vars: num_vars entries, read only.  The transcript and the tape (sp_random_tape_new) advance as the reference's do, and are written back only
 * on success.  *proof = bincode(R1CSProof), released with sp_free; rx_out: log2 num_cons scalars, ry_out: log2 (2 num_vars).
 * SP_ERR_INVALID_ARG, with nothing launched and the states untouched: dimensions as above, |inputs| + 1 > num_vars, both or neither of inst and
 * spmat, an instance of other dimensions, an spmat of another shape, vars of another length, gens for another num_vars, NULL arguments, handles
 * of another context; SP_ERR_INVALID_SCALAR: inputs not reduced. */
int sp_r1cs_prove_t(sp_ctx* ctx, const sp_instance* inst, const sp_spmat* spmat, size_t num_cons, size_t num_vars, const sp_poly* vars,
                    const uint64_t* inputs_mont, size_t ninputs, const sp_r1cs_gens* gens, uint8_t* strobe_state /* in, out */,
                    uint8_t* tape_state /* in, out */, uint8_t** proof, size_t* proof_len, uint64_t* rx_out, uint64_t* ry_out);
/* R1CSProof::verify(num_vars, num_cons, inputs, evals, transcript, gens) with evals = (Ar, Br, Cr): SP_ERR_VERIFY / SP_ERR_DECOMPRESS naming the
 * failing check; the transcript is advanced as the reference's verify advances it, accepted or not.  rx_out / ry_out as sp_r1cs_prove_t's.
 * Refusals as sp_r1cs_prove_t's, and SP_ERR_INVALID_SCALAR for evals not reduced; a refused call leaves the transcript untouched. */
int sp_r1cs_verify_t(sp_ctx* ctx, const uint8_t* proof, size_t proof_len, size_t num_cons, size_t num_vars, const uint64_t* inputs_mont, size_t ninputs,
                     const uint64_t evals_mont[12], const sp_r1cs_gens* gens, uint8_t* strobe_state /* in, out */, uint64_t* rx_out, uint64_t* ry_out);

/* ---- inner-product argument, operator level: BulletReductionProof::prove (src/nizk/bullet.rs:32-132) for a host that keeps the transcript and
 * the orchestration.  sp_ipa_begin copies a_vec / b_vec; the generator vector G is `gens` (G[0..n)).  Each round: sp_ipa_round_LR returns the
 * compressed L, R of bullet.rs:83-97 (c_L, c_R are formed inside; Q and H are the caller's points), the host appends them and derives u
 * (bullet.rs:99-103), sp_ipa_fold applies bullet.rs:105-108.  After lg n rounds sp_ipa_finish returns a[0], b[0] and G[0] (bullet.rs:113-122). */
typedef struct sp_ipa sp_ipa;
int sp_ipa_begin(sp_ctx* ctx, const sp_gens* gens, const sp_poly* a_vec, const sp_poly* b_vec, sp_ipa** out);
void sp_ipa_free(sp_ipa* h);
int sp_ipa_round_LR(sp_ctx* ctx, sp_ipa* h, const uint8_t Q32[32], const uint8_t H32[32], const uint64_t blind_L_mont[4], const uint64_t blind_R_mont[4],
                    uint8_t L32[32], uint8_t R32[32]);
int sp_ipa_fold(sp_ctx* ctx, sp_ipa* h, const uint64_t u_mont[4], const uint64_t u_inv_mont[4]);
int sp_ipa_finish(sp_ctx* ctx, sp_ipa* h, uint64_t a_hat_mont[4], uint64_t b_hat_mont[4], uint8_t G_hat32[32]);

/* ---- instances                                                                           lib.rs:111-274 */
/* Instance::new: entries are (row, col, canonical 32-byte value); rows < num_cons, cols < num_vars + 1 + num_inputs */
int sp_instance_create(sp_ctx* ctx, size_t num_cons, size_t num_vars, size_t num_inputs, const uint64_t* A_row, const uint64_t* A_col, const uint8_t* A_val32,
                       size_t nA, const uint64_t* B_row, const uint64_t* B_col, const uint8_t* B_val32, size_t nB, const uint64_t* C_row, const uint64_t* C_col,
                       const uint8_t* C_val32, size_t nC, sp_instance** out);
/* the same with every array in DEVICE memory on the context's GPU (e.g. CUDA tensors, a Rust caller's own device buffers): same padding, input-column
 * remap, error codes and messages; the first bad entry in (matrix, entry) order is reported, row before column before scalar.  A pointer that is
 * not device memory of the context's device (an array with zero entries is not looked at) gives SP_ERR_INVALID_ARG.  The arrays must be fully
 * written before the call (synchronise the stream that wrote them); the call returns only after it has finished reading them.  The instance
 * keeps no host copy of the matrices until sp_instance_bincode / sp_instance_digest / sp_instance_export asks for one. */
int sp_instance_create_device(sp_ctx* ctx, size_t num_cons, size_t num_vars, size_t num_inputs, const uint64_t* A_row, const uint64_t* A_col,
                              const uint8_t* A_val32, size_t nA, const uint64_t* B_row, const uint64_t* B_col, const uint8_t* B_val32, size_t nB,
                              const uint64_t* C_row, const uint64_t* C_col, const uint8_t* C_val32, size_t nC, sp_instance** out);
/* Instance::produce_synthetic_r1cs with the OsRng replaced by the seeded SHAKE256 generator of DESIGN.md.
 * vars_out: num_vars*4 limbs, inputs_out: num_inputs*4 limbs (Montgomery) */
int sp_instance_synthetic(sp_ctx* ctx, size_t num_cons, size_t num_vars, size_t num_inputs, uint64_t seed, sp_instance** out, uint64_t* vars_out,
                          uint64_t* inputs_out);
void sp_instance_free(sp_instance* inst);
int sp_instance_dims(const sp_instance* inst, size_t* num_cons, size_t* num_vars, size_t* num_inputs);
/* R1CSShape::get_digest (r1cs.rs:154-158): NIZK::prove / verify absorb zlib(bincode(shape)) (lib.rs:514).  The reference compresses with flate2's
 * miniz_oxide backend at level 6; this library computes the same stream with its own restatement of miniz's compressor (csrc/deflate.cpp, bit-identical
 * to C miniz level 6) on first use.  A caller that wants its own compressor's bytes absorbed instead passes them with sp_instance_set_digest. */
int sp_instance_set_digest(sp_instance* inst, const uint8_t* digest, size_t len);
int sp_instance_digest(const sp_instance* inst, uint8_t** out, size_t* len);   /* free with sp_free */
/* bincode(R1CSShape) — the bytes the reference deflates to obtain the digest (r1cs.rs:154-158) */
int sp_instance_bincode(const sp_instance* inst, uint8_t** out, size_t* len);
/* COO export in the reference's entry order: matrix 0/1/2 = A/B/C; vals are Montgomery limbs */
int sp_instance_nnz(const sp_instance* inst, int matrix, size_t* nnz);
int sp_instance_export(const sp_instance* inst, int matrix, uint64_t* row, uint64_t* col, uint64_t* val_mont);
int sp_instance_is_sat(sp_ctx* ctx, const sp_instance* inst, const uint64_t* vars_mont, size_t nvars, const uint64_t* inputs_mont, size_t ninputs, int* sat);
/* R1CSShape::evaluate(rx, ry) (r1cs.rs:300-303): out = (A(rx, ry), B(rx, ry), C(rx, ry)), the claims sp_r1cs_verify_t takes.  rx: log2 num_cons
 * scalars, ry: log2 (2 num_vars), of the padded dimensions.  SP_ERR_INVALID_SCALAR: rx or ry not reduced. */
int sp_instance_evaluate(sp_ctx* ctx, const sp_instance* inst, const uint64_t* rx_mont, const uint64_t* ry_mont, uint64_t out_mont[12]);

/* ---- NIZK                                                                                lib.rs:468-591 */
int sp_nizk_gens_create(sp_ctx* ctx, size_t num_cons, size_t num_vars, size_t num_inputs, sp_nizk_gens** out);
void sp_nizk_gens_free(sp_nizk_gens* g);
/* NIZK::prove(inst, vars, inputs, gens, &mut Transcript::new(transcript_label)); tape_seed = the scalar RandomTape::new draws from OsRng
 * (random.rs:13-15).  vars are HOST Montgomery limbs and are copied to the device inside the call.  *proof = bincode::serialize(&NIZK),
 * released with sp_free. */
int sp_nizk_prove(sp_ctx* ctx, const sp_instance* inst, const uint64_t* vars_mont, size_t nvars, const uint64_t* inputs_mont, size_t ninputs,
                  const sp_nizk_gens* gens, const uint8_t* transcript_label, size_t label_len, const uint64_t tape_seed_mont[4], uint8_t** proof,
                  size_t* proof_len);
/* same with the assignment already resident on the device (bench "value" leg) */
int sp_nizk_prove_resident(sp_ctx* ctx, const sp_instance* inst, const sp_poly* vars, const uint64_t* inputs_mont, size_t ninputs, const sp_nizk_gens* gens,
                           const uint8_t* transcript_label, size_t label_len, const uint64_t tape_seed_mont[4], uint8_t** proof, size_t* proof_len);

/* ---- SNARK                                                                               lib.rs:277-465 */
int sp_snark_gens_create(sp_ctx* ctx, size_t num_cons, size_t num_vars, size_t num_inputs, size_t num_nz_entries, sp_snark_gens** out);
void sp_snark_gens_free(sp_snark_gens* g);

/* ---- generator tables shared by several gens.  sp_nizk_gens_create / sp_snark_gens_create each build their own generator sets; a NIZKGens
 * or SNARKGens made from tables is a view into the tables' sets and holds no device memory of its own, so gens for any number of circuits
 * up to the tables' sizes share one copy.  MultiCommitGens::new(n, label) of any n is a prefix of the label's SHAKE stream
 * (commitments.rs:15-33): a view proves and verifies byte for byte as the private gens of its circuit do.  Tables, the gens made from them
 * and encodings may be freed in any order; the device memory goes back to the library's cache when the last holder is freed. */
typedef struct sp_gen_tables sp_gen_tables;
/* the gens_r1cs_sat set for circuits up to (num_cons, num_vars, num_inputs) and, if num_nz_entries > 0, the gens_r1cs_eval set up to that
 * many non-zeros (commitments.rs:15-33, r1csproof.rs:68-73, sparse_mlpoly.rs:292-317); widths chosen as for private gens (DESIGN.md §2) */
int sp_gen_tables_create(sp_ctx* ctx, size_t num_cons, size_t num_vars, size_t num_inputs, size_t num_nz_entries, sp_gen_tables** out);
void sp_gen_tables_free(sp_gen_tables* t);       /* drops the caller's reference; views keep the tables alive */
typedef struct { char label[32]; size_t nbases; int window_bits; int has_row_table; size_t device_bytes; } sp_gen_set_info;
/* one entry per set (gens_r1cs_sat, then gens_r1cs_eval if built); *n = the number of sets; SP_ERR_INVALID_ARG (nothing written) if cap < *n */
int sp_gen_tables_info(const sp_gen_tables* t, sp_gen_set_info* out, size_t cap, size_t* n);
/* views for a circuit whose every dimension is <= the tables' (NIZKGens::new lib.rs:475-481, SNARKGens::new lib.rs:288-309).  SP_ERR_INVALID_ARG
 * when a set is too short (the message gives needed vs available generators per set), when a SNARK view is asked of tables built with
 * num_nz_entries = 0, or when the tables were built on another context.  Host copies of the few generators the sigma protocols use are added
 * to the tables if missing; no device memory stays allocated. */
int sp_nizk_gens_create_from(sp_ctx* ctx, const sp_gen_tables* tables, size_t num_cons, size_t num_vars, size_t num_inputs, sp_nizk_gens** out);
int sp_snark_gens_create_from(sp_ctx* ctx, const sp_gen_tables* tables, size_t num_cons, size_t num_vars, size_t num_inputs, size_t num_nz_entries,
                              sp_snark_gens** out);
/* device bytes in blocks this library holds for live objects, on every device (its cache of freed blocks excluded): a footprint that other
 * processes on the GPU cannot change, unlike cudaMemGetInfo */
unsigned long long sp_device_bytes_live(void);

int sp_snark_encode(sp_ctx* ctx, const sp_instance* inst, const sp_snark_gens* gens, sp_snark_encoding** out);   /* SNARK::encode lib.rs:325 */
void sp_snark_encoding_free(sp_snark_encoding* e);
/* bincode::serialize(&ComputationCommitment) */
int sp_snark_commitment_bytes(const sp_snark_encoding* e, uint8_t** out, size_t* len);
int sp_snark_prove(sp_ctx* ctx, const sp_instance* inst, const sp_snark_encoding* enc, const uint64_t* vars_mont, size_t nvars, const uint64_t* inputs_mont,
                   size_t ninputs, const sp_snark_gens* gens, const uint8_t* transcript_label, size_t label_len, const uint64_t tape_seed_mont[4],
                   uint8_t** proof, size_t* proof_len);
int sp_snark_prove_resident(sp_ctx* ctx, const sp_instance* inst, const sp_snark_encoding* enc, const sp_poly* vars, const uint64_t* inputs_mont,
                            size_t ninputs, const sp_snark_gens* gens, const uint8_t* transcript_label, size_t label_len,
                            const uint64_t tape_seed_mont[4], uint8_t** proof, size_t* proof_len);

/* bincode(ComputationCommitment) (as written by sp_snark_commitment_bytes or by the reference) -> a commitment-only handle for sp_snark_verify */
int sp_snark_commitment_load(sp_ctx* ctx, const uint8_t* bytes, size_t len, sp_snark_encoding** out);

/* ---- verifiers: SP_OK = accepted; SP_ERR_VERIFY / SP_ERR_DECOMPRESS = rejected (sp_last_error names the failing check).  `proof` is
 * bincode::serialize(&NIZK) / (&SNARK), as produced by sp_*_prove or by the reference. */
/* NIZK::verify(&self, &Instance, &InputsAssignment, &mut Transcript, &NIZKGens)                         lib.rs:549-591 */
int sp_nizk_verify(sp_ctx* ctx, const sp_instance* inst, const uint64_t* inputs_mont, size_t ninputs, const sp_nizk_gens* gens, const uint8_t* label,
                   size_t label_len, const uint8_t* proof, size_t proof_len);
/* SNARK::verify(&self, &ComputationCommitment, &InputsAssignment, &mut Transcript, &SNARKGens)          lib.rs:423-465
 * (`comm`: a handle from sp_snark_encode or from sp_snark_commitment_load; only its commitment part is read) */
int sp_snark_verify(sp_ctx* ctx, const sp_snark_encoding* comm, const uint64_t* inputs_mont, size_t ninputs, const sp_snark_gens* gens, const uint8_t* label,
                    size_t label_len, const uint8_t* proof, size_t proof_len);

/* ---- the caller-owned transcript.  The reference's prove / verify take `transcript: &mut Transcript` (src/lib.rs:339-347, :423-429, :501-508,
 * :549-555): the caller may have absorbed its own data before the call and may keep using the transcript afterwards.  The *_t entry points take
 * merlin's whole STROBE-128 state instead of a label — SP_TRANSCRIPT_STATE_BYTES = 200 bytes of Keccak state, then pos, pos_begin, cur_flags
 * (merlin::strobe::Strobe128) — and leave it exactly as the reference's call leaves the caller's transcript.  sp_*_prove / sp_*_verify with a
 * label are the shorthand for a transcript the caller has just created with Transcript::new(label) and does not reuse (benches/snark.rs:56). */
#define SP_TRANSCRIPT_STATE_BYTES 203
int sp_nizk_prove_t(sp_ctx* ctx, const sp_instance* inst, const uint64_t* vars_mont, size_t nvars, const uint64_t* inputs_mont, size_t ninputs,
                    const sp_nizk_gens* gens, uint8_t* strobe_state /* in, out */, const uint64_t tape_seed[4], uint8_t** proof, size_t* proof_len);
int sp_snark_prove_t(sp_ctx* ctx, const sp_instance* inst, const sp_snark_encoding* enc, const uint64_t* vars_mont, size_t nvars, const uint64_t* inputs_mont,
                     size_t ninputs, const sp_snark_gens* gens, uint8_t* strobe_state /* in, out */, const uint64_t tape_seed[4], uint8_t** proof, size_t* proof_len);
int sp_nizk_verify_t(sp_ctx* ctx, const sp_instance* inst, const uint64_t* inputs_mont, size_t ninputs, const sp_nizk_gens* gens, uint8_t* strobe_state /* in, out */,
                     const uint8_t* proof, size_t proof_len);
int sp_snark_verify_t(sp_ctx* ctx, const sp_snark_encoding* comm, const uint64_t* inputs_mont, size_t ninputs, const sp_snark_gens* gens,
                      uint8_t* strobe_state /* in, out */, const uint8_t* proof, size_t proof_len);

/* ---- batch verification: k proofs in one call.  Proof i is checked against comms[i] / insts[i] (one handle may repeat; every handle's sizes must
 * match `gens`), inputs i (ninputs[i] scalars) and a fresh transcript labels[i] (label_lens[i] bytes) or, in the _t forms, the caller's transcript
 * strobe_states[i] (in, out).  Each proof's group equations are weighted by random scalars and tested together with the other proofs' in one
 * device pass (DESIGN.md "deferred checks"); a proof that fails any check is re-run as the single call would run it.  So:
 *   status[i]   = what sp_*_verify / sp_*_verify_t returns for proof i (SP_OK, SP_ERR_VERIFY or SP_ERR_DECOMPRESS);
 *   strobe_states[i] is left exactly as the single _t call leaves it, whether proof i is accepted or rejected;
 *   sp_last_error = "proof <i>: " + the single call's message, for the lowest rejected i;
 *   returns SP_OK when every proof is accepted, SP_ERR_VERIFY when one or more is rejected, or the usual code for bad arguments (NULL arrays,
 *   a NULL seed, inputs not reduced, an inconsistent commitment) or device errors, in which case `status` and the states are not written.
 *   k = 0 returns SP_OK.  A batch may hold up to 2^32 - 1 variable-base terms in all (a few hundred per proof); a larger one is refused with
 *   SP_ERR_INVALID_ARG: split it.
 * weight_seed: 32 bytes of FRESH OS RANDOMNESS on every call (like tape_seed): the weight of equation e of proof i is
 * from_bytes_wide(SHAKE256("spartan-b200/v1/batch-verify" || seed || LE64(i) || LE64(e))), and anyone who knows the weights before the call can
 * build a false proof that passes.  On a connected multi-GPU context the batch runs on this rank's GPU alone (no collectives). */
int sp_snark_verify_batch(sp_ctx* ctx, size_t k, const sp_snark_encoding* const* comms, const uint64_t* const* inputs_mont, const size_t* ninputs,
                          const sp_snark_gens* gens, const uint8_t* const* labels, const size_t* label_lens, const uint8_t* const* proofs,
                          const size_t* proof_lens, const uint8_t weight_seed[32], int* status /* k, out */);
int sp_nizk_verify_batch(sp_ctx* ctx, size_t k, const sp_instance* const* insts, const uint64_t* const* inputs_mont, const size_t* ninputs,
                         const sp_nizk_gens* gens, const uint8_t* const* labels, const size_t* label_lens, const uint8_t* const* proofs,
                         const size_t* proof_lens, const uint8_t weight_seed[32], int* status /* k, out */);
int sp_snark_verify_batch_t(sp_ctx* ctx, size_t k, const sp_snark_encoding* const* comms, const uint64_t* const* inputs_mont, const size_t* ninputs,
                            const sp_snark_gens* gens, uint8_t* const* strobe_states /* k x 203, in, out */, const uint8_t* const* proofs,
                            const size_t* proof_lens, const uint8_t weight_seed[32], int* status /* k, out */);
int sp_nizk_verify_batch_t(sp_ctx* ctx, size_t k, const sp_instance* const* insts, const uint64_t* const* inputs_mont, const size_t* ninputs,
                           const sp_nizk_gens* gens, uint8_t* const* strobe_states /* k x 203, in, out */, const uint8_t* const* proofs,
                           const size_t* proof_lens, const uint8_t weight_seed[32], int* status /* k, out */);

/* merlin::Transcript::{new, append_message, challenge_bytes} on such a state buffer (transcript.rs:13-30), for hosts without merlin and for the tests */
int sp_transcript_new(const uint8_t* label, size_t label_len, uint8_t* strobe_state /* out */);
int sp_transcript_append_message(uint8_t* strobe_state, const uint8_t* label, size_t label_len, const uint8_t* msg, size_t msg_len);
int sp_transcript_challenge_bytes(uint8_t* strobe_state, const uint8_t* label, size_t label_len, uint8_t* out, size_t n);

void sp_free(void* p);

#ifdef __cplusplus
}
#endif
#endif
