/* b2kyber.h -- C ABI of the H100 batch group-arithmetic engine (libb2kyber.so).
 *
 * This is the drop-in boundary under dedis/kyber's kyber.Group/Point/Scalar and pairing.Suite
 * (reference: group.go:23-194, pairing/pairing.go:8-20).  The reference has NO batch entry point
 * and no FFI; every function below names the reference call site(s) whose Go loop / single-op method
 * it replaces.  A Go adapter (pairing/bls12381/b200, shaped like pairing/bls12381/kilic) binds these
 * with cgo -- see INTEGRATION.md.
 *
 * Conventions
 *   - all buffers are caller-owned, contiguous, fixed stride; nothing is retained after return
 *   - scalars: 32 bytes big-endian, canonical (< group order) = mod.Int.MarshalBinary
 *     (group/mod/int.go:334-349); a scalar >= order yields B2K_ERR_SCALAR_RANGE, like
 *     mod.Int.UnmarshalBinary (int.go:359-372)
 *   - operand points: affine coordinates, big-endian canonical field elements, all-zero = infinity
 *       BLS12-381 G1: x||y            (96 B)     G2: x.c1||x.c0||y.c1||y.c0 (192 B)
 *       bn254     G1: x||y            (64 B)
 *   - result points: the reference's MarshalBinary bytes
 *       BLS12-381 G1: 48 B ZCash compressed (kilic/g1.go:119-124)   G2: 96 B (kilic/g2.go:118-123)
 *       bn254     G1: 64 B x||y, infinity all-zero (pairing/bn254/point.go:113-132)
 *   - return value: 0 = ok, negative = B2K_ERR_*; no exceptions, no callbacks
 *   - a context owns one CUDA stream and its scratch memory; calls on one context are serialised by
 *     the caller (one context per goroutine/thread), several contexts may be used concurrently
 *   - there is NO CPU fallback: without a usable sm_90 device b2k_create fails
 *   - operand points are re-validated where that is cheap: canonical coordinates (< p, where the reference's Unmarshal checks
 *     that: BLS12-381, bn254) and the curve equation; a violation -> B2K_ERR_POINT (the point is treated as infinity).  Membership
 *     in the order-r subgroup is NOT re-checked (a scalar multiplication per point): like in the reference that is the job of
 *     UnmarshalBinary, i.e. of b2k_*_decompress / b2k_*_unmarshal_check; the endomorphism paths (G1 Mul / MSM) assume it
 *   - *_dev variants take DEVICE pointers (same layouts) and only enqueue work on the context's
 *     stream; they exist so a caller that keeps batches resident in HBM pays no PCIe traffic;
 *     data errors of enqueued work (scalar >= order, malformed point) are collected by b2k_wait
 */
#ifndef B2KYBER_H
#define B2KYBER_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b2k_ctx b2k_ctx;

enum {
  B2K_OK = 0,
  B2K_ERR_CUDA = -1,          /* a CUDA runtime call failed; see b2k_last_error */
  B2K_ERR_ARG = -2,           /* null pointer / size out of range */
  B2K_ERR_SCALAR_RANGE = -3,  /* some scalar >= group order */
  B2K_ERR_NO_DEVICE = -4,     /* no sm_90 device */
  B2K_ERR_POINT = -5,         /* some operand point is malformed (coordinate >= p or not on curve) */
  B2K_ERR_COMM = -6           /* multi-GPU exchange: a peer rank did not arrive (b2k_comm_*), reported by b2k_wait */
};

/* ---- lifetime ------------------------------------------------------------------------------ */
int b2k_create(int device, b2k_ctx** out);
void b2k_destroy(b2k_ctx* ctx);
const char* b2k_last_error(const b2k_ctx* ctx);
const char* b2k_version(void);
/* Use an existing CUDA stream (cudaStream_t passed as void*) instead of the context's own. */
int b2k_set_stream(b2k_ctx* ctx, void* cuda_stream);
int b2k_synchronize(b2k_ctx* ctx);
/* Device-side durations (ms, CUDA events on the context's stream) of the stages of the LAST MSM call:
 * [0] load/convert points  [1] digits+histogram  [2] scan  [3] scatter  [4] bucket accumulate
 * [5] chunk reduce  [6] window sum  [7] final (Horner + encode)  [8] whole pipeline
 * [9] fix-up of buckets cut by slice boundaries ([4] is the accumulate pass alone: affine rounds + XYZZ slices)
 * [10] the affine pair-tree rounds inside [4] (0 when they are off).
 * Returns the number of entries written (<= max). Synchronises the stream. */
int b2k_last_timings(b2k_ctx* ctx, float* ms, int max);
/* Parameters the LAST MSM of this context ran with: [0] window bits c  [1] windows W  [2] buckets per window
 * [3] reduction chunk  [4] slice length of the XYZZ pass  [5] affine pair-tree rounds R  [6..13] additions per thread of
 * round 0..7  [14] 1 when the endomorphism split was used  [15] 1 when the rounds ran as three kernels each.
 * Returns the number of entries written. */
int b2k_last_msm_plan(const b2k_ctx* ctx, int* out, int max);
/* Override the MSM window size (0 = automatic).  Testing / tuning aid. */
int b2k_set_msm_window(b2k_ctx* ctx, int c);
/* Slice length of the balanced bucket-accumulate (0 = automatic) and the accumulate variant
 * (0 = balanced slices [default], 1 = one thread per bucket).  Testing / tuning aids. */
int b2k_set_msm_slice(b2k_ctx* ctx, int slice_len);
int b2k_set_msm_variant(b2k_ctx* ctx, int one_thread_per_bucket);
/* Window groups of an experimental overlapped MSM tail (default 1 = off; measured slower, see DESIGN.md): the windows are accumulated in `groups` launches, top
 * group first, and the bucket reduction of each group runs on a second, high-priority stream while the next
 * group accumulates.  1 = strictly serial pipeline, in which b2k_last_timings reports every stage separately;
 * with groups > 1, [4] spans all accumulate launches, [9] is the exposed remainder of the reduction, [5],[6] ~ 0. */
int b2k_set_msm_groups(b2k_ctx* ctx, int groups);
/* BLS12-381 G1 MSM front end: 1 (default) = split every scalar with the curve endomorphism (k P = k1 P + k2 (-phi P),
 * 127-bit k1, k2: half the windows), 0 = plain 255-bit pipeline.  Same results; kept switchable for A/B timing. */
int b2k_set_msm_glv(b2k_ctx* ctx, int on);
/* Affine pair-tree rounds in front of the XYZZ bucket slices (BLS12-381 G1 MSM): every round replaces the operands of
 * each bucket by the sums of neighbouring pairs, computed as batched AFFINE additions (6 field products each instead of
 * 10) around one inversion per thread.  rounds: -1 = automatic (default), 0 = off, 1..8; batch: additions per thread
 * (8..64 fused / ..1024 split, 0 = automatic).  Same result bytes either way; kept switchable for A/B timing. */
int b2k_set_msm_affine(b2k_ctx* ctx, int rounds, int batch);
/* 1 (default) = every affine round runs as three kernels (forward prefix products, one inversion per thread, backward
 * additions; batch up to 1024), 0 = one fused kernel per round (batch up to 64, prefix products in local memory).  A/B aid. */
int b2k_set_msm_affine_split(b2k_ctx* ctx, int split);
/* Affine rounds with the operands of the next output staged global -> shared memory by cp.async: backward pass bit 0 = the first
 * (gathering) round, bit 1 = the later rounds; forward pass bits 2 and 3 likewise.  Same bytes out; A/B aid. */
int b2k_set_msm_staging(b2k_ctx* ctx, int mask);
/* Register cap of the inversion kernel of the affine rounds: 4 [default] = uncapped; 5 = 96 registers, so that its single wave
 * leaves one block slot per SM for a product kernel of another MSM in flight (measured: no gain; kept for A/B).  (The 5/6-block variants of the XYZZ kernel
 * measured slower than 4 and were removed.) */
int b2k_set_msm_occupancy(b2k_ctx* ctx, int blocks_per_sm);
/* Resident blocks per SM of the BLS12-381 G1 Point.Mul batch kernel.  The constrained variants measured 0.6-0.7x of the
 * compiler's own allocation and were removed: accepted, ignored. */
int b2k_set_mul_occupancy(b2k_ctx* ctx, int blocks_per_sm);
/* Buckets per thread in the chunked bucket reduction (power of two, 0 = automatic).  Tuning aid. */
int b2k_set_msm_chunk(b2k_ctx* ctx, int m);
/* Bucket reduction in one level (chunks of m buckets, a small scalar multiplication per chunk) or two (the scalar
 * multiplications move to the second level, which has m1 times fewer operands).  levels: 0 = automatic, 1, 2; m1, m2 = chunk
 * sizes of the two levels (powers of two, 0 = default 8 and 4).  Same result bytes either way; A/B and tuning aid. */
int b2k_set_msm_reduce(b2k_ctx* ctx, int levels, int m1, int m2);
/* code layout of the field products inside the G1 MSM / Point.Mul kernels (b2k_bls12381_g1_msm_dev, _mul_batch*_dev):
 * 0 = one out-of-line body called by value (instruction-cache friendly; the library default), 1 = inlined at every use
 * (the round-1 layout); identical results, A/B aid. */
int b2k_set_msm_layout(b2k_ctx* ctx, int layout);
/* Number of kernels launched by this context so far. */
uint64_t b2k_launch_count(const b2k_ctx* ctx);

/* ---- BLS12-381 G1 ------------------------------------------------------------------------------ */
/* out[i] = scalars[i] * points[i]    -- n independent Point.Mul
 * replaces: kilic.G1Elt.Mul, pairing/bls12381/kilic/g1.go:110-116 called in loops such as
 * sign/bdn/mask.go:58-61 and util/test/group.go:118-122 */
int b2k_bls12381_g1_mul_batch(b2k_ctx* ctx, size_t n, const uint8_t* scalars /*[n][32]*/,
                              const uint8_t* points /*[n][96]*/, uint8_t* out /*[n][48]*/);
int b2k_bls12381_g1_mul_batch_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points,
                                  void* d_out);
/* Same, but results in OPERAND form (96 B affine x||y, all-zero = infinity): what the adapter keeps
 * in a G1Elt between operations (MarshalBinary is applied only when bytes are asked for). */
int b2k_bls12381_g1_mul_batch_affine(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points,
                                     uint8_t* out /*[n][96]*/);
int b2k_bls12381_g1_mul_batch_affine_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points,
                                         void* d_out);
/* out = sum_i scalars[i] * points[i]    -- Pippenger MSM
 * replaces the Mul+Add loops of share.RecoverCommit (share/poly.go:461-473) and
 * bdn.AggregateSignatures (sign/bdn/bdn.go:126-161) */
int b2k_bls12381_g1_msm(b2k_ctx* ctx, size_t n, const uint8_t* scalars /*[n][32]*/,
                        const uint8_t* points /*[n][96]*/, uint8_t* out /*[48]*/);
int b2k_bls12381_g1_msm_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points,
                            void* d_out);
/* Same with the sum in OPERAND form (96 B): the partial a rank contributes to a multi-GPU MSM. */
int b2k_bls12381_g1_msm_affine_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points,
                                   void* d_out /*[96]*/);

/* ---- multi-GPU MSM by partial-bucket exchange (the shape BASELINE.json's north_star names; SURVEY.md 8e shape 1) ----
 * A sharded MSM (each rank holds n of the pairs of one sum, e.g. the 2^24-term aggregate of config C5) as three
 * device-side steps around two collectives issued by the host (kyber_b200/multi.py: msm_bucket_exchange):
 *   msm_buckets_dev         this rank's pairs -> its W x 2^(c-1) PARTIAL buckets, raw Montgomery limbs
 *                           (plan[3] bytes per bucket: XYZZ coordinates, 4 x 48 B), window-major
 *   ncclAllToAll            rank g receives windows [g W/G, (g+1) W/G) of every rank  (= reduce-scatter without the
 *                           reduction: NCCL cannot add curve points)
 *   msm_reduce_windows_dev  d_recv = [parts][w_cnt][2^(c-1)] buckets; the bucket-wise EC addition of the `parts`
 *                           partials is fused into the running-sum reduction; d_wsum = [w_cnt] window sums
 *   ncclAllGather           all W window sums on every rank
 *   msm_finish_dev          Horner over the windows, affine, wire bytes (48 B compressed, or 96 B operand form)
 * Replaces the same Mul+Add loops as b2k_bls12381_g1_msm (share/poly.go:461-473, sign/bdn/bdn.go:126-161) when the
 * terms live on several GPUs.  plan = {c, W, buckets per window, bytes per bucket}; all ranks must obtain the same
 * plan (same n and switches), which bucket_plan lets the host check before sizing its buffers. */
int b2k_bls12381_g1_msm_bucket_plan(b2k_ctx* ctx, size_t n, int* plan /*[4]*/);
int b2k_bls12381_g1_msm_buckets_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points,
                                    void* d_buckets, size_t cap_bytes, int* plan /*[4], may be NULL*/);
int b2k_bls12381_g1_msm_reduce_windows_dev(b2k_ctx* ctx, int c, int w_cnt, int parts, const void* d_recv,
                                           void* d_wsum /*[w_cnt][plan[3]]*/);
int b2k_bls12381_g1_msm_finish_dev(b2k_ctx* ctx, int c, int W, const void* d_wsum, void* d_out, int affine_out);

/* ---- the sharded MSM as ONE call per rank: the `b2k_msm_multi_gpu` of SURVEY.md 8(b), and 8(e) ------------------------
 * Replaces the same loops (share/poly.go:461-473, sign/bdn/bdn.go:126-161) when the terms of one sum are partitioned over
 * the GPUs of a box (BASELINE.json configs[4]: 2^24 pairs, 2^21 per GPU).  A communicator belongs to one context (= one
 * rank) and owns that rank's EXCHANGE SLAB, a stable device allocation every peer maps (peer access inside one process,
 * CUDA IPC across processes).  A step then needs no host-side collective at all:
 *   partial buckets into the own slab -> release-store of the step number into every peer's flag word -> spin on the own
 *   flag words -> ONE kernel pulls windows [g W/G, (g+1) W/G) of every rank out of the peers' slabs over NVLink and fuses
 *   the G-way EC addition into the running-sum reduction -> window sums pushed to every peer -> Horner on every rank.
 * All of it is enqueued on the context's stream; ranks must issue their steps on a communicator in the same order.  A peer
 * that never arrives makes the waiting kernel give up after ~10 s and b2k_wait return B2K_ERR_COMM (no device hang).
 * Wiring:  one process per GPU (torchrun, MPI):  create -> export -> all-gather the blobs out of band -> connect;
 *          one process, ngpu contexts (the cgo adapter):  create x ngpu -> connect_local.
 * b2k_comm_use_nccl swaps the transport of the bucket exchange for NCCL (grouped ncclSend/ncclRecv = all-to-all, then
 * ncclAllGather of the window sums; libnccl.so.2 is resolved at run time with dlopen; one rank per process; the 128-byte id
 * comes from b2k_nccl_unique_id on rank 0 and travels out of band) -- the shape north_star words literally, kept for A/B.
 * shape: 0 = partial-bucket exchange (W must be a multiple of the rank count), 1 = result exchange (every rank finishes
 * its MSM, 96-byte results are pushed to every peer and added; any rank count; peer transport only). */
#define B2K_MAX_RANKS 16
#define B2K_COMM_BLOB_BYTES 128
typedef struct b2k_comm b2k_comm;
int b2k_comm_create(b2k_ctx* ctx, int nranks, int rank, b2k_comm** out);
int b2k_comm_export(b2k_comm* comm, uint8_t* blob /*[B2K_COMM_BLOB_BYTES]*/);
int b2k_comm_connect(b2k_comm* comm, const uint8_t* blobs /*[nranks][B2K_COMM_BLOB_BYTES], rank order*/);
int b2k_comm_connect_local(b2k_comm** comms /*[nranks], rank order*/, int nranks);
int b2k_nccl_unique_id(uint8_t* id /*[128]*/);
int b2k_comm_use_nccl(b2k_comm* comm, const uint8_t* id /*[128]*/);
void b2k_comm_destroy(b2k_comm* comm);
int b2k_comm_last_plan(const b2k_comm* comm, int* plan /*[4]: c, W, buckets per window, bytes per bucket*/);
/* this rank's n pairs (DEVICE buffers) -> the 48-byte sum over ALL ranks in d_out on every rank; enqueue only */
int b2k_bls12381_g1_msm_sharded_dev(b2k_comm* comm, size_t n, const void* d_scalars, const void* d_points,
                                    void* d_out /*[48]*/, int shape);
/* the same from (page-locked) HOST buffers, result to host; enqueue only, collect with b2k_wait(ctx of the communicator) */
int b2k_bls12381_g1_msm_sharded_async(b2k_comm* comm, size_t n, const uint8_t* scalars, const uint8_t* points,
                                      uint8_t* out /*[48]*/);
/* one process driving ngpu ranks: partitions the n pairs contiguously, runs the sharded MSM on every communicator, waits */
int b2k_bls12381_g1_msm_multi_gpu(b2k_comm** comms /*[ngpu], rank order*/, int ngpu, size_t n, const uint8_t* scalars /*[n][32]*/,
                                  const uint8_t* points /*[n][96]*/, uint8_t* out /*[48]*/);

/* ---- BLS12-381 G2 ------------------------------------------------------------------------------------ */
/* replaces: kilic.G2Elt.Mul, pairing/bls12381/kilic/g2.go:109-115 (public keys / signatures on G2:
 * bdn.NewMask terms sign/bdn/mask.go:58-61, bdn.AggregateSignatures on G2).  Operands 192 B
 * (x.c1||x.c0||y.c1||y.c0), results 96 B ZCash compressed (kilic/g2.go:118-123). */
int b2k_bls12381_g2_mul_batch(b2k_ctx* ctx, size_t n, const uint8_t* scalars /*[n][32]*/,
                              const uint8_t* points /*[n][192]*/, uint8_t* out /*[n][96]*/);
int b2k_bls12381_g2_mul_batch_affine(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points,
                                     uint8_t* out /*[n][192]*/);
int b2k_bls12381_g2_mul_batch_affine_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points,
                                         void* d_out);
int b2k_bls12381_g2_msm(b2k_ctx* ctx, size_t n, const uint8_t* scalars /*[n][32]*/,
                        const uint8_t* points /*[n][192]*/, uint8_t* out /*[96]*/);
int b2k_bls12381_g2_msm_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points, void* d_out);

/* MSM with the sum in OPERAND form (G1 96 B / G2 192 B), host buffers: what the adapter's Point.Add / Sub use
 * (unit scalars) so that results stay in operand form between operations. */
int b2k_bls12381_g1_msm_affine(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out /*[96]*/);
/* Asynchronous form of b2k_bls12381_g1_msm: the H2D copies, the MSM and the D2H copy of the result are ENQUEUED on the
 * context's stream and the call returns.  scalars, points and out must stay valid until b2k_wait(ctx) returns (and should
 * be page-locked, otherwise the copies do not overlap anything).  b2k_wait blocks until everything enqueued on the
 * context is done and returns the deferred status of the last MSM (B2K_ERR_SCALAR_RANGE ...).  Two contexts used
 * alternately (async on A, async on B, wait A, async on A, ...) keep the PCIe copies of one batch under the kernels
 * of the other: this is how a caller with a stream of batches (goroutines verifying aggregates, share/poly recoveries)
 * should drive the library; the blocking form is this followed by b2k_wait.
 * b2k_wait is also the status query after *_dev calls (which only enqueue and therefore cannot report data errors themselves):
 * the device status word is sticky across them; b2k_wait synchronises, returns B2K_ERR_SCALAR_RANGE / B2K_ERR_POINT if any
 * call since the previous b2k_wait (or host-buffer call) saw such an operand, and clears it. */
int b2k_bls12381_g1_msm_async(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out);
int b2k_wait(b2k_ctx* ctx);
int b2k_bls12381_g2_msm_affine(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out /*[192]*/);

/* ---- BLS12-381 UnmarshalBinary (decompress + subgroup check) --------------------------------------------- */
/* out[i] = operand form of the ZCash-compressed input, ok[i] = 1, or ok[i] = 0 (out[i] zeroed) when the
 * reference's UnmarshalBinary would return an error: wrong flag bits, x >= p, not on the curve, not in the
 * r-torsion subgroup.   replaces: kilic.G1Elt.UnmarshalBinary -> FromCompressed (kilic/g1.go:127-131),
 * kilic.G2Elt.UnmarshalBinary (kilic/g2.go:126-130); behaviour pinned by the 34 ZCash fixtures.
 * (Wrong LENGTH is the caller's check: the stride is fixed.) */
int b2k_bls12381_g1_decompress(b2k_ctx* ctx, size_t n, const uint8_t* in /*[n][48]*/, uint8_t* out /*[n][96]*/,
                               uint8_t* ok /*[n]*/);
int b2k_bls12381_g1_decompress_dev(b2k_ctx* ctx, size_t n, const void* d_in, void* d_out, void* d_ok);
int b2k_bls12381_g2_decompress(b2k_ctx* ctx, size_t n, const uint8_t* in /*[n][96]*/, uint8_t* out /*[n][192]*/,
                               uint8_t* ok /*[n]*/);
int b2k_bls12381_g2_decompress_dev(b2k_ctx* ctx, size_t n, const void* d_in, void* d_out, void* d_ok);

/* ---- BLS12-381 hash-to-G1 and signature verification ------------------------------------------------- */
/* out[i] = hash_to_curve(msgs[offsets[i] .. offsets[i+1]), dst) in operand form (96 B), RFC 9380 suite
 * BLS12381G1_XMD:SHA-256_SSWU_RO_.   replaces: kilic.G1Elt.Hash, pairing/bls12381/kilic/g1.go:161-170
 * (default DST "BLS_SIG_BLS12381G1_XMD:SHA-256_SSWU_RO_NUL_", g1.go:17; suite override suite.go:32-46).
 * offsets are n+1 uint32 byte offsets into msgs; 0 < dst_len <= 255. */
int b2k_bls12381_hash_to_g1(b2k_ctx* ctx, size_t n, const uint8_t* msgs, const uint32_t* offsets /*[n+1]*/,
                            const uint8_t* dst, uint32_t dst_len, uint8_t* out /*[n][96]*/);
int b2k_bls12381_hash_to_g1_dev(b2k_ctx* ctx, size_t n, const void* d_msgs, const void* d_offsets, const void* d_dst,
                                uint32_t dst_len, void* d_out);
/* ok[i] = 1 iff bls.Verify(pk_i, msg_i, sig_i) == nil for the scheme with signatures on G1
 * (bls.NewSchemeOnG1, sign/bls/bls.go:33-44,82-96): UnmarshalBinary of the 96-byte compressed G2 key and
 * the 48-byte compressed G1 signature (subgroup checks included), H(msg), then
 * ValidatePairing(H(m), pk, sig, G2 generator) (kilic/suite.go:57-68).  One call = n independent
 * verifications = the loop of util/test/benchmark.go:62-71 (BLSBenchVerify). */
int b2k_bls12381_verify_g1sig(b2k_ctx* ctx, size_t n, const uint8_t* pks /*[n][96]*/, const uint8_t* msgs,
                              const uint32_t* offsets /*[n+1]*/, const uint8_t* dst, uint32_t dst_len,
                              const uint8_t* sigs /*[n][48]*/, uint8_t* ok /*[n]*/);
int b2k_bls12381_verify_g1sig_dev(b2k_ctx* ctx, size_t n, const void* d_pks, const void* d_msgs, const void* d_offsets,
                                  const void* d_dst, uint32_t dst_len, const void* d_sigs, void* d_ok);

/* Same for the scheme with signatures on G2 and keys on G1 (bls.NewSchemeOnG2, sign/bls/bls.go:48-59; the drand
 * default): hash_to_curve onto G2, suite BLS12381G2_XMD:SHA-256_SSWU_RO_ (kilic.G2Elt.Hash, kilic/g2.go:160-169,
 * default DST "BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_NUL_" g2.go:18), out 192 B operand form; verification is
 * ValidatePairing(G1 base, sig, pk, H(m)), keys 48 B compressed, signatures 96 B compressed. */
int b2k_bls12381_hash_to_g2(b2k_ctx* ctx, size_t n, const uint8_t* msgs, const uint32_t* offsets /*[n+1]*/,
                            const uint8_t* dst, uint32_t dst_len, uint8_t* out /*[n][192]*/);
int b2k_bls12381_hash_to_g2_dev(b2k_ctx* ctx, size_t n, const void* d_msgs, const void* d_offsets, const void* d_dst,
                                uint32_t dst_len, void* d_out);
int b2k_bls12381_verify_g2sig(b2k_ctx* ctx, size_t n, const uint8_t* pks /*[n][48]*/, const uint8_t* msgs,
                              const uint32_t* offsets /*[n+1]*/, const uint8_t* dst, uint32_t dst_len,
                              const uint8_t* sigs /*[n][96]*/, uint8_t* ok /*[n]*/);
int b2k_bls12381_verify_g2sig_dev(b2k_ctx* ctx, size_t n, const void* d_pks, const void* d_msgs, const void* d_offsets,
                                  const void* d_dst, uint32_t dst_len, const void* d_sigs, void* d_ok);

/* ---- BLS12-381 pairings ---------------------------------------------------------------------------- */
/* gt[i] = e(g1[i], g2[i]); g2 operands are 192 B: x.c1||x.c0||y.c1||y.c0.  GT = 576 B, 12 x 48 B
 * big-endian, highest tower coefficient first (kilic/gt.go:115-117), final exponent 3 (p^12-1)/r as in the
 * reference's back-ends.  An infinity operand gives the GT identity.   replaces: kilic.Suite.Pair, kilic/suite.go:70-75
 * Byte order and exponent are pinned by the reference vector encrypt/ibe/ibe_test.go:202-245 (see tests/). */
int b2k_bls12381_pair(b2k_ctx* ctx, size_t n, const uint8_t* g1 /*[n][96]*/, const uint8_t* g2 /*[n][192]*/,
                      uint8_t* gt /*[n][576]*/);
int b2k_bls12381_pair_dev(b2k_ctx* ctx, size_t n, const void* d_g1, const void* d_g2, void* d_gt);
/* ok[i] = ( e(a1[i], a2[i]) == e(b1[i], b2[i]) ) as 1/0 -- one 2-pair Miller loop + one final
 * exponentiation per element.   replaces: kilic.Suite.ValidatePairing(p1,p2,inv1,inv2),
 * kilic/suite.go:57-68, as called by bls.Verify (sign/bls/bls.go:82-96). */
int b2k_bls12381_pairing_check(b2k_ctx* ctx, size_t n, const uint8_t* a1 /*[n][96]*/, const uint8_t* a2 /*[n][192]*/,
                               const uint8_t* b1 /*[n][96]*/, const uint8_t* b2 /*[n][192]*/, uint8_t* ok /*[n]*/);
int b2k_bls12381_pairing_check_dev(b2k_ctx* ctx, size_t n, const void* d_a1, const void* d_a2, const void* d_b1,
                                   const void* d_b2, void* d_ok);
/* gt[i] = e(g1[i], g2) for ONE g2 operand: its Miller-loop lines are computed once and shared by every element (the kernel
 * b2k_bls12381_ibe_decrypt_cca_g1 runs above the cooperative size).  Same bytes as b2k_bls12381_pair with g2 repeated n times. */
int b2k_bls12381_pair_fixed_g2(b2k_ctx* ctx, size_t n, const uint8_t* g1 /*[n][96]*/, const uint8_t* g2 /*[192]*/,
                               uint8_t* gt /*[n][576]*/);

/* ---- encrypt/ibe: Boneh-Franklin CCA encryption on BLS12-381 ---------------------------------------------------------------
 * One key (or master key and identity) and n messages of one length len, 0 <= len <= 32 (s.Hash().Size(), SHA-256); points are
 * compressed kyber wire bytes.  With len bytes of each hash:
 *   H2(g) = SHA256("IBE-H2" || GT.MarshalBinary(g)),  H4(sigma) = SHA256("IBE-H4" || sigma),
 *   H3(sigma, msg): buf = SHA256("IBE-H3" || sigma || msg); for i = 1 .. 65534: h = SHA256(LE16(i) || buf), h[0] >>= 1, the
 *   first h < r read big-endian.
 * Decrypt: sigma = V xor H2(e(U, priv)) (OnG2: e(priv, U)), msg = W xor H4(sigma), accepted when H3(sigma, msg) Base == U.
 * status[i]: B2K_IBE_OK, B2K_IBE_PROOF (the reference's "invalid proof: rP check failed"; U at infinity gives this), or
 * B2K_IBE_POINT (U does not decode with the checks of b2k_bls12381_g1/g2_decompress); msg[i] is zeroed unless OK.
 * Encrypt: Gid = e(master, Q_id) (OnG2: e(Q_id, master)) with Q_id = hash_to_g2(id) (OnG2: hash_to_g1), dst NULL = the default
 * DST of that hash; for each message r = H3(sigma, msg), U = r Base, V = sigma xor H2(Gid^r), W = msg xor H4(sigma).  sigma is
 * the caller's randomness (crypto/rand in the reference).
 * A key that does not decode -> B2K_ERR_POINT; len > 32, n = 0 or a null pointer -> B2K_ERR_ARG.  Blocking, host buffers.
 *   replaces: DecryptCCAonG1 ibe.go:99-134, DecryptCCAonG2 ibe.go:196-231, EncryptCCAonG1 ibe.go:51-97, EncryptCCAonG2 ibe.go:148-194 */
enum { B2K_IBE_OK = 0, B2K_IBE_PROOF = 1, B2K_IBE_POINT = 2 };
int b2k_bls12381_ibe_decrypt_cca_g1(b2k_ctx* ctx, const uint8_t* priv /*[96]*/, size_t n, const uint8_t* u /*[n][48]*/, size_t len,
                                    const uint8_t* v /*[n][len]*/, const uint8_t* w /*[n][len]*/, uint8_t* msg /*[n][len]*/,
                                    uint8_t* status /*[n]*/);
int b2k_bls12381_ibe_decrypt_cca_g2(b2k_ctx* ctx, const uint8_t* priv /*[48]*/, size_t n, const uint8_t* u /*[n][96]*/, size_t len,
                                    const uint8_t* v /*[n][len]*/, const uint8_t* w /*[n][len]*/, uint8_t* msg /*[n][len]*/,
                                    uint8_t* status /*[n]*/);
int b2k_bls12381_ibe_encrypt_cca_g1(b2k_ctx* ctx, const uint8_t* master /*[48]*/, const uint8_t* id, size_t id_len, const uint8_t* dst,
                                    size_t dst_len, size_t n, size_t len, const uint8_t* msgs /*[n][len]*/,
                                    const uint8_t* sigmas /*[n][len]*/, uint8_t* u /*[n][48]*/, uint8_t* v /*[n][len]*/,
                                    uint8_t* w /*[n][len]*/);
int b2k_bls12381_ibe_encrypt_cca_g2(b2k_ctx* ctx, const uint8_t* master /*[96]*/, const uint8_t* id, size_t id_len, const uint8_t* dst,
                                    size_t dst_len, size_t n, size_t len, const uint8_t* msgs /*[n][len]*/,
                                    const uint8_t* sigmas /*[n][len]*/, uint8_t* u /*[n][96]*/, uint8_t* v /*[n][len]*/,
                                    uint8_t* w /*[n][len]*/);

/* ---- the target group as a kyber.Group, Miller / Finalize, products of pairings, G1 / G2 Add ------------------------------
 * GT is written additively in kyber: Add = Fp12 product, Neg = inverse, Mul = exponentiation, Null = 1
 * (pairing/bls12381/kilic/gt.go:33-83; pairing/bn254/point.go:560-623).  Elements travel as their MarshalBinary bytes
 * (BLS12-381: 576 B, kilic/gt.go:115-117; bn254/bn256: 384 B, pairing/bn254/point.go:625-656); a coefficient >= p raises
 * B2K_ERR_POINT where the reference's Unmarshal range-checks (BLS12-381, bn254).  gt_exp takes 32-byte big-endian scalars
 * below the group order and is valid for any Fp12 element (plain square-and-multiply).  gt_inv maps the zero element (all
 * coefficients 0, not a member of GT) to zero, as the field inversion underneath maps 0 to 0.
 * miller / final_exp (finalize): pointGT.Miller and pointGT.Finalize (pairing/bn254/point.go:768-786) -- exported by the
 * reference so that a caller can multiply several Miller values and pay ONE final exponentiation; miller(...) output fed to
 * final_exp(...) equals pair(...).  An operand at infinity gives 1 (pairing/bn254/optate.go:267-269).
 * pairing_product_check: ok[0] = ( prod_i e(g1[i], g2[i]) == 1 ), n Miller loops, a product tree, ONE final exponentiation
 * (SURVEY.md 8e); Suite.ValidatePairing(p1, p2, q1, q2) is the n = 2 case with q1 negated (kilic/suite.go:57-68).
 * pairing_product: the same product as GT bytes (e.g. n-signer aggregate checks that compare against a stored value).
 * g{1,2}_add_batch: out[i] = a[i] + b[i] (negate_b = 0) or a[i] - b[i] (negate_b = 1), operand form in and out, every
 * exceptional case of the group law handled (kilic/g1.go:92-108, g2.go:91-107: Point.Add / Sub / Neg, one at a time in Go). */
int b2k_bls12381_gt_mul(b2k_ctx* ctx, size_t n, const uint8_t* a /*[n][576]*/, const uint8_t* b /*[n][576]*/, uint8_t* out /*[n][576]*/);
int b2k_bls12381_gt_inv(b2k_ctx* ctx, size_t n, const uint8_t* a /*[n][576]*/, uint8_t* out /*[n][576]*/);
int b2k_bls12381_gt_exp(b2k_ctx* ctx, size_t n, const uint8_t* scalars /*[n][32]*/, const uint8_t* a /*[n][576]*/, uint8_t* out /*[n][576]*/);
int b2k_bn254_gt_mul(b2k_ctx* ctx, size_t n, const uint8_t* a /*[n][384]*/, const uint8_t* b /*[n][384]*/, uint8_t* out /*[n][384]*/);
int b2k_bn254_gt_inv(b2k_ctx* ctx, size_t n, const uint8_t* a /*[n][384]*/, uint8_t* out /*[n][384]*/);
int b2k_bn254_gt_exp(b2k_ctx* ctx, size_t n, const uint8_t* scalars /*[n][32]*/, const uint8_t* a /*[n][384]*/, uint8_t* out /*[n][384]*/);
int b2k_bls12381_miller(b2k_ctx* ctx, size_t n, const uint8_t* g1 /*[n][96]*/, const uint8_t* g2 /*[n][192]*/, uint8_t* out /*[n][576]*/);
int b2k_bls12381_final_exp(b2k_ctx* ctx, size_t n, const uint8_t* in /*[n][576]*/, uint8_t* out /*[n][576]*/);
int b2k_bls12381_pairing_product_check(b2k_ctx* ctx, size_t n, const uint8_t* g1 /*[n][96]*/, const uint8_t* g2 /*[n][192]*/, uint8_t* ok /*[1]*/);
int b2k_bls12381_pairing_product(b2k_ctx* ctx, size_t n, const uint8_t* g1 /*[n][96]*/, const uint8_t* g2 /*[n][192]*/, uint8_t* gt /*[576]*/);
int b2k_bn254_miller(b2k_ctx* ctx, size_t n, const uint8_t* g1 /*[n][64]*/, const uint8_t* g2 /*[n][128]*/, uint8_t* out /*[n][384]*/);
int b2k_bn254_finalize(b2k_ctx* ctx, size_t n, const uint8_t* in /*[n][384]*/, uint8_t* out /*[n][384]*/);
int b2k_bn254_pairing_product_check(b2k_ctx* ctx, size_t n, const uint8_t* g1 /*[n][64]*/, const uint8_t* g2 /*[n][128]*/, uint8_t* ok /*[1]*/);
int b2k_bn256_miller(b2k_ctx* ctx, size_t n, const uint8_t* g1 /*[n][64]*/, const uint8_t* g2 /*[n][128]*/, uint8_t* out /*[n][384]*/);
int b2k_bn256_finalize(b2k_ctx* ctx, size_t n, const uint8_t* in /*[n][384]*/, uint8_t* out /*[n][384]*/);
int b2k_bn256_pairing_product_check(b2k_ctx* ctx, size_t n, const uint8_t* g1 /*[n][64]*/, const uint8_t* g2 /*[n][128]*/, uint8_t* ok /*[1]*/);
int b2k_bls12381_g1_add_batch(b2k_ctx* ctx, size_t n, const uint8_t* a /*[n][96]*/, const uint8_t* b /*[n][96]*/, int negate_b, uint8_t* out /*[n][96]*/);
int b2k_bls12381_g2_add_batch(b2k_ctx* ctx, size_t n, const uint8_t* a /*[n][192]*/, const uint8_t* b /*[n][192]*/, int negate_b, uint8_t* out /*[n][192]*/);

/* ---- bn254 G1 (share.RecoverCommit config: t = 1024 over bn254 G1) ------------------------------ */
/* replaces bn254 curvePoint.Mul, pairing/bn254/curve.go:196-218 */
int b2k_bn254_g1_mul_batch(b2k_ctx* ctx, size_t n, const uint8_t* scalars /*[n][32]*/,
                           const uint8_t* points /*[n][64]*/, uint8_t* out /*[n][64]*/);
int b2k_bn254_g1_msm(b2k_ctx* ctx, size_t n, const uint8_t* scalars /*[n][32]*/,
                     const uint8_t* points /*[n][64]*/, uint8_t* out /*[64]*/);
int b2k_bn254_g1_msm_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points, void* d_out);
/* out = sum_i lambda_i * points[i] with lambda_i = prod_{j!=i} x_j / (x_j - x_i) mod r, x_i = indices[i] + 1:
 * the whole of share.RecoverCommit (share/poly.go:449-476) after xyCommit's sort/selection (poly.go:418-445):
 * Lagrange weights (t^2 scalar products + t inversions) and the t-term MSM both run on the device.
 * Duplicate indices -> B2K_ERR_ARG. */
int b2k_bn254_recover_commit(b2k_ctx* ctx, size_t t, const uint32_t* indices /*[t]*/, const uint8_t* points /*[t][64]*/,
                             uint8_t* out /*[64]*/);

/* ---- threshold BLS on BLS12-381: share.RecoverCommit and share.PubPoly.Eval --------------------------------- */
/* RecoverCommit over G1 (points [t][96], out 48 B) or G2 ([t][192], out 96 B): Lagrange weights and MSM on the
 * device, exactly as b2k_bn254_recover_commit.  replaces: share.RecoverCommit (share/poly.go:449-476) as called by
 * tbls.Recover (sign/tbls/tbls.go:141) on the signature group. */
int b2k_bls12381_g1_recover_commit(b2k_ctx* ctx, size_t t, const uint32_t* indices /*[t]*/, const uint8_t* points /*[t][96]*/,
                                   uint8_t* out /*[48]*/);
int b2k_bls12381_g2_recover_commit(b2k_ctx* ctx, size_t t, const uint32_t* indices /*[t]*/, const uint8_t* points /*[t][192]*/,
                                   uint8_t* out /*[96]*/);
/* out[i] = sum_j (indices[i] + 1)^j * commits[j]  (Horner), operand form in and out.
 * replaces: share.PubPoly.Eval / Shares (share/poly.go:340-357) -- t Point.Mul + t Add per index -- the
 * per-partial-signature cost of tbls.Recover (sign/tbls/tbls.go:126) and of DKG/VSS share verification. */
int b2k_bls12381_g1_pubpoly_eval(b2k_ctx* ctx, size_t t, const uint8_t* commits /*[t][96]*/, size_t n,
                                 const uint32_t* indices /*[n]*/, uint8_t* out /*[n][96]*/);
int b2k_bls12381_g2_pubpoly_eval(b2k_ctx* ctx, size_t t, const uint8_t* commits /*[t][192]*/, size_t n,
                                 const uint32_t* indices /*[n]*/, uint8_t* out /*[n][192]*/);

/* share.RecoverPubPoly (share/poly.go:480-508; lagrangeBasis :513-545): the WHOLE public polynomial from t public shares
 * (the first t by index, like recover_commit): commits_out[k] = sum_j L_j[k] * points[j], k = 0..t-1, operand form.
 * commits_out[0] equals recover_commit's result (as compressed / operand bytes of the same point).  1 <= t <= 4096.
 * PriPoly.Commit (poly.go:143-149): out[i] = scalars[i] * base for ONE base point (NULL = the group's generator) -- the
 * fixed-base batch a dealer runs over its coefficient vector (callers no longer replicate the generator n times). */
int b2k_bls12381_g1_recover_pubpoly(b2k_ctx* ctx, size_t t, const uint32_t* indices /*[t]*/, const uint8_t* points /*[t][96]*/,
                                    uint8_t* commits_out /*[t][96]*/);
int b2k_bls12381_g2_recover_pubpoly(b2k_ctx* ctx, size_t t, const uint32_t* indices /*[t]*/, const uint8_t* points /*[t][192]*/,
                                    uint8_t* commits_out /*[t][192]*/);
int b2k_bn254_recover_pubpoly(b2k_ctx* ctx, size_t t, const uint32_t* indices /*[t]*/, const uint8_t* points /*[t][64]*/,
                              uint8_t* commits_out /*[t][64]*/);
int b2k_bls12381_g1_commit_batch(b2k_ctx* ctx, size_t n, const uint8_t* scalars /*[n][32]*/, const uint8_t* base /*[96] or NULL*/,
                                 uint8_t* out /*[n][96]*/);
int b2k_bls12381_g2_commit_batch(b2k_ctx* ctx, size_t n, const uint8_t* scalars /*[n][32]*/, const uint8_t* base /*[192] or NULL*/,
                                 uint8_t* out /*[n][192]*/);
int b2k_bn254_commit_batch(b2k_ctx* ctx, size_t n, const uint8_t* scalars /*[n][32]*/, const uint8_t* base /*[64] or NULL*/,
                           uint8_t* out /*[n][64]*/);

/* ---- share.PubPoly.Check over a batch of deals: the verification loops of share/vss and share/dkg ---------------------
 * For dealer d (m of them) with commitments commits[d][0..t) and private shares (indices[d][k], shares[d][k]), k < n:
 *     ok[d][k] = ( sum_j (indices[d][k] + 1)^j commits[d][j]  ==  shares[d][k] * B ),   B = the group's base point.
 * One thread per (d, k): Horner evaluation, base-point multiplication and a projective comparison on the device.
 * shares: 32-byte big-endian scalars; a share not below the group order gives ok = 0 (the reference drops such a deal
 * at UnmarshalBinary).  commits in operand form ([96] / [192] / [64] bytes), ok: one byte per check.
 * replaces: PubPoly.Check (share/poly.go:405-409) = Eval + Mul + Equal, run once per received deal / response /
 * justification in share/vss/pedersen/vss.go:636-645 and share/dkg/pedersen/dkg.go:489-494, 826-834, 965 -- an
 * n x n x t scalar-multiplication workload at key generation / resharing time, sequential in the reference. */
int b2k_bls12381_g1_pubpoly_check(b2k_ctx* ctx, size_t m, size_t t, const uint8_t* commits /*[m][t][96]*/, size_t n,
                                  const uint32_t* indices /*[m][n]*/, const uint8_t* shares /*[m][n][32]*/, uint8_t* ok /*[m][n]*/);
int b2k_bls12381_g2_pubpoly_check(b2k_ctx* ctx, size_t m, size_t t, const uint8_t* commits /*[m][t][192]*/, size_t n,
                                  const uint32_t* indices /*[m][n]*/, const uint8_t* shares /*[m][n][32]*/, uint8_t* ok /*[m][n]*/);
int b2k_bn254_pubpoly_check(b2k_ctx* ctx, size_t m, size_t t, const uint8_t* commits /*[m][t][64]*/, size_t n,
                            const uint32_t* indices /*[m][n]*/, const uint8_t* shares /*[m][n][32]*/, uint8_t* ok /*[m][n]*/);

/* ---- bn254 G2 and pairing --------------------------------------------------------------------------------- */
/* G2 operands/results: 128 B x.imag||x.real||y.imag||y.real, infinity all-zero (pairing/bn254/point.go:428-455).
 * replaces: bn254 twistPoint.Mul, pairing/bn254/twist.go:167-181 */
int b2k_bn254_g2_mul_batch(b2k_ctx* ctx, size_t n, const uint8_t* scalars /*[n][32]*/, const uint8_t* points /*[n][128]*/,
                           uint8_t* out /*[n][128]*/);
int b2k_bn254_g2_msm(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out /*[128]*/);
/* gt[i] = e(g1[i], g2[i]) as the 384-byte GT MarshalBinary (pairing/bn254/point.go:625-656); an infinity operand
 * gives the identity.  replaces: bn254 Suite.Pair -> optimalAte -> miller + finalExponentiation,
 * pairing/bn254/suite.go:133-136, optate.go:124-271.  GT bytes are source-pinned (the in-tree Go fixes them). */
int b2k_bn254_pair(b2k_ctx* ctx, size_t n, const uint8_t* g1 /*[n][64]*/, const uint8_t* g2 /*[n][128]*/,
                   uint8_t* gt /*[n][384]*/);
/* ok[i] = ( e(a1,a2) == e(b1,b2) ).  replaces: bn254 Suite.ValidatePairing, pairing/bn254/suite.go:138-144 */
int b2k_bn254_pairing_check(b2k_ctx* ctx, size_t n, const uint8_t* a1 /*[n][64]*/, const uint8_t* a2 /*[n][128]*/,
                            const uint8_t* b1, const uint8_t* b2, uint8_t* ok /*[n]*/);

/* ---- bn256 (pairing/bn256: the curve of the reference's byte-exact BDN fixtures) --------------------------- */
/* G1 64 B x||y, G2 128 B x.imag||x.real||y.imag||y.real (pairing/bn256/point.go:170-192, :423-452), operands
 * and results alike.  replaces: bn256 curvePoint.Mul (curve.go:189-203), twistPoint.Mul (twist.go:162-175) and the
 * Mul+Add loops of sign/bdn (bdn.go:126-181, mask.go:57-61) on this curve. */
int b2k_bn256_g1_mul_batch(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out /*[n][64]*/);
int b2k_bn256_g1_msm(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out /*[64]*/);
int b2k_bn256_g2_mul_batch(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out /*[n][128]*/);
int b2k_bn256_g2_msm(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out /*[128]*/);
/* bn256 pairing: the twin of the bn254 one (pairing/bn256/optate.go:126-274, suite.go:99-109); GT 384 B. */
int b2k_bn256_pair(b2k_ctx* ctx, size_t n, const uint8_t* g1 /*[n][64]*/, const uint8_t* g2 /*[n][128]*/, uint8_t* gt /*[n][384]*/);
int b2k_bn256_pairing_check(b2k_ctx* ctx, size_t n, const uint8_t* a1, const uint8_t* a2, const uint8_t* b1,
                            const uint8_t* b2, uint8_t* ok /*[n]*/);

/* ---- UnmarshalBinary validation for whole batches of BN points (wire-format gate of the Mul / MSM / pairing entry points)
 * ok[i] = 1 when the reference's UnmarshalBinary would accept in[i] (all-zero = the point at infinity is accepted):
 *   bn254 G1: coordinates below p, on y^2 = x^3 + 3                      pairing/bn254/point.go:146-185, gfp.go:101-119
 *   bn254 G2: coordinates below p, on the twist, killed by the group order  point.go:473-514, twist.go:50-66
 *   bn256 G1/G2: NO range check (values reduce mod p), on the curve / twist, no order check
 *                                                                        pairing/bn256/point.go:206-238, 469-506 */
int b2k_bn254_g1_unmarshal_check(b2k_ctx* ctx, size_t n, const uint8_t* in /*[n][64]*/, uint8_t* ok /*[n]*/);
int b2k_bn254_g2_unmarshal_check(b2k_ctx* ctx, size_t n, const uint8_t* in /*[n][128]*/, uint8_t* ok /*[n]*/);
int b2k_bn256_g1_unmarshal_check(b2k_ctx* ctx, size_t n, const uint8_t* in /*[n][64]*/, uint8_t* ok /*[n]*/);
int b2k_bn256_g2_unmarshal_check(b2k_ctx* ctx, size_t n, const uint8_t* in /*[n][128]*/, uint8_t* ok /*[n]*/);

/* Launch shape / code layout of the BLS12-381 pairing kernels: variant = shape + 4 * layout, shape 0..2 = (64 threads, 4 / 8 / 6
 * blocks per SM), layout 0 = out-of-line by-value field products (default), 1 = inlined;
 * 16 + 2 m + f = Miller loop and final exponentiation as two kernels (m, f: 0 = 128 registers, 1 = 255).  Tuning aid. */
int b2k_set_pairing_variant(b2k_ctx* ctx, int variant);
/* Batches of at most max_n pairings / pairing checks (BLS12-381, bn254, bn256) run on the warp-cooperative kernels (one warp per
 * element: a single BLS12-381 Suite.Pair takes 2.0 ms instead of one thread's 20 ms, a single ValidatePairing 2.3 instead of 26 ms;
 * bn254 / bn256: 2.1 / 2.5 ms instead of 12-23 ms; GT.Mul on BLS12-381 and bn254, batches up to 4096: 2.5 instead of 22 ms); larger
 * batches use the one-per-thread kernels.  Default 10240 (the measured
 * break-even on BLS12-381; the Barreto-Naehrig curves cap it at 8192), 0 = never.  Same bytes either way. */
int b2k_set_pairing_coop(b2k_ctx* ctx, int max_n);

/* ---- edwards25519 ---------------------------------------------------------------------------------------- */
/* out[i] = scalars[i] * points[i] on edwards25519, as geScalarMult computes it.  scalars: RAW 256-bit little-endian
 * integers (the reference does not reduce on UnmarshalBinary, group/edwards25519/scalar.go:226-233), read as 64 signed
 * nibbles; a top nibble e63 above 8 (possible only from 2^255 on) selects nothing, so the product is then
 * (k - e63 2^252) P; below 2^255 it is k P.  Points and results: 32-byte compressed (ge.go:99-150; non-canonical y
 * accepted).  A point that does not decode -> B2K_ERR_POINT
 * (its output zeroed).   replaces: point.Mul, group/edwards25519/point.go:235-258 (geScalarMult, ge.go:443-502)
 * in loops such as util/test/group.go:118-122. */
int b2k_ed25519_mul_batch(b2k_ctx* ctx, size_t n, const uint8_t* scalars /*[n][32] LE*/,
                          const uint8_t* points /*[n][32]*/, uint8_t* out /*[n][32]*/);
int b2k_ed25519_mul_batch_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points, void* d_out);

/* ---- edwards25519 MSM and share/poly -------------------------------------------------------------------------------------
 * Points: 32-byte compressed, decoded like FromBytes (ge.go:110-150, non-canonical y accepted); a point that does not decode
 * -> B2K_ERR_POINT and its term counts as the identity.  Results: the canonical ToBytes encoding.  The identity is 01 00..00;
 * all-zero bytes decode to a point of order 4, NOT to the identity.
 * Scalars: 32-byte little-endian, read as the reference's Point.Mul reads them (geScalarMult, ge.go:443-502): the plain integer
 * (no reduction mod l, so torsion parts of the points count), except when the top digit e63 = (k >> 252) + carry of its
 * signed-nibble recoding exceeds 8: selectCached (ge.go:419-433) then selects nothing and the term is (k - e63 2^252) P.
 * Indices: x = index + 1 (index 0xffffffff gives 2^32), as in the other groups' share entry points.
 * b2k_last_msm_plan [0..4] and b2k_last_timings report the last MSM / RecoverCommit ([0] includes the point decoding). */
/* out = sum_i scalars[i] * points[i].  replaces: the Point.Mul + Add loops over edwards25519 (share/poly.go:461-473,
 * sign/cosi's aggregate of commitments), one call instead of n Mul. */
int b2k_ed25519_msm(b2k_ctx* ctx, size_t n, const uint8_t* scalars /*[n][32] LE*/, const uint8_t* points /*[n][32]*/,
                    uint8_t* out /*[32]*/);
/* device pointers; enqueue only: data errors (B2K_ERR_POINT) arrive at b2k_wait */
int b2k_ed25519_msm_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points, void* d_out);
/* out = sum_i lambda_i points[i], lambda_i = prod_{j != i} x_j / (x_j - x_i) mod l: share.RecoverCommit (share/poly.go:449-476,
 * also pvss.RecoverSecret pvss.go:322 and DKG resharing dkg.go:965) after xyCommit's selection.  Duplicate indices -> B2K_ERR_ARG. */
int b2k_ed25519_recover_commit(b2k_ctx* ctx, size_t t, const uint32_t* indices /*[t]*/, const uint8_t* points /*[t][32]*/,
                               uint8_t* out /*[32]*/);
/* out[i] = sum_j (indices[i] + 1)^j commits[j] (Horner): share.PubPoly.Eval (share/poly.go:340-357) for n indices. */
int b2k_ed25519_pubpoly_eval(b2k_ctx* ctx, size_t t, const uint8_t* commits /*[t][32]*/, size_t n, const uint32_t* indices /*[n]*/,
                             uint8_t* out /*[n][32]*/);
/* ok[d][k] = ( sum_j (indices[d][k] + 1)^j commits[d][j] == shares[d][k] * B ), B the base point, one byte per check:
 * share.PubPoly.Check (share/poly.go:405-409) as run once per deal, response and justification in
 * share/vss/pedersen/vss.go:636-645 and share/dkg/pedersen/dkg.go:489-494, 826-834.  shares: 32-byte little-endian, read
 * like the scalars above (Check's Mul(s.V, p.b) goes through geScalarMult). */
int b2k_ed25519_pubpoly_check(b2k_ctx* ctx, size_t m, size_t t, const uint8_t* commits /*[m][t][32]*/, size_t n,
                              const uint32_t* indices /*[m][n]*/, const uint8_t* shares /*[m][n][32] LE*/, uint8_t* ok /*[m][n]*/);

/* ---- edwards25519 DLEQ proofs and PVSS ----------------------------------------------------------------------------------
 * One status byte per proof, in the reference's order of failure:
 *   B2K_DLEQ_POINT      an operand (point argument, VG or VH) does not decode like FromBytes: the reference could not have
 *                       built this input
 *   B2K_DLEQ_CHALLENGE  C differs from the expected challenge as raw bytes (Scalar.Equal, scalar.go:37-45): a C congruent to
 *                       it but not canonical fails here
 *   B2K_DLEQ_INVALID    VG != R G + C xG or VH != R H + C xH (dleq.Proof.Verify, proof/dleq/dleq.go:161-172)
 * Proofs are 128 bytes C || R || VG || VH.  C and R are 32-byte little-endian, read raw as Point.Mul reads them (no reduction
 * mod l; a top signed nibble above 8 selects nothing, as in b2k_ed25519_msm).  Points decode like FromBytes (non-canonical y
 * accepted; all-zero bytes are the point of order 4).  Challenges hash MarshalTo of the DECODED points (their canonical
 * encodings), SHA-256, then Scalar.Pick from blake2xb.New(digest) (the digest is the BLAKE2b key).
 * Bad data is never a call error, only a status; B2K_ERR_ARG means a null pointer, a zero size, or m n or m t >= 2^31. */
enum { B2K_DLEQ_OK = 0, B2K_DLEQ_CHALLENGE = 1, B2K_DLEQ_INVALID = 2, B2K_DLEQ_POINT = 3 };
/* status[i] of dleq.Proof.Verify(g[i], h[i], xg[i], xh[i]) for n proofs (OK, INVALID or POINT).
 * replaces: dleq.Proof.Verify called once per proof (dleq.go:161-172). */
int b2k_ed25519_dleq_verify(b2k_ctx* ctx, size_t n, const uint8_t* g /*[n][32]*/, const uint8_t* h /*[n][32]*/,
                            const uint8_t* xg /*[n][32]*/, const uint8_t* xh /*[n][32]*/, const uint8_t* proofs /*[n][128]*/,
                            uint8_t* status /*[n]*/);
/* device pointers; enqueue only */
int b2k_ed25519_dleq_verify_dev(b2k_ctx* ctx, size_t n, const void* d_g, const void* d_h, const void* d_xg, const void* d_xh,
                                const void* d_proofs, void* d_status);
/* pvss.VerifyEncShareBatch (share/pvss/pvss.go:168-194) for m deals of n encrypted shares each, threshold t: deal d has the
 * base h[d], the commitments commits[d][0..t), and per share i the key x[d][i], the caller's sH sh[d][i], the encrypted share
 * v[d][i] and its proof.  The deal's challenge is Pick(XOF(SHA-256(coms[0..n) || V[0..n) || VG[0..n) || VH[0..n)))) with
 * coms[i] = sum_j (i + 1)^j commits[d][j] at the POSITION i (pvss.go:94-149); each share then checks C against it and
 * Verify(h, x, sh, v).  A deal whose h, a commitment, a V, VG or VH does not decode gives B2K_DLEQ_POINT for every share; an x or
 * sh that does not decode only for its share.  K and E of the reference are the shares with status B2K_DLEQ_OK. */
int b2k_ed25519_pvss_verify_enc_shares(b2k_ctx* ctx, size_t m, size_t t, size_t n, const uint8_t* h /*[m][32]*/,
                                       const uint8_t* commits /*[m][t][32]*/, const uint8_t* x /*[m][n][32]*/,
                                       const uint8_t* sh /*[m][n][32]*/, const uint8_t* v /*[m][n][32]*/,
                                       const uint8_t* proofs /*[m][n][128]*/, uint8_t* status /*[m][n]*/);
/* pvss.VerifyDecShareBatch (pvss.go:281-299): per share, C against Pick(XOF(SHA-256(x || enc_v || VG || VH))), then
 * Verify(g, dec_v, x, enc_v) (VerifyDecShare, pvss.go:248-277).  pvss.RecoverSecret is this call followed by
 * b2k_ed25519_recover_commit on the shares with status B2K_DLEQ_OK (sorted by index, the first t). */
int b2k_ed25519_pvss_verify_dec_shares(b2k_ctx* ctx, size_t n, const uint8_t* g /*[32]*/, const uint8_t* x /*[n][32]*/,
                                       const uint8_t* enc_v /*[n][32]*/, const uint8_t* dec_v /*[n][32]*/,
                                       const uint8_t* proofs /*[n][128]*/, uint8_t* status /*[n]*/);

/* ---- edwards25519 Neff shuffle verification (shuffle/) ------------------------------------------------------------------
 * One status byte per shuffle, in the reference's order of failure:
 *   B2K_SHUFFLE_POINT   an input point (g, h, x, y, xbar, ybar) or a proof point does not decode like FromBytes: the proof's Get
 *                       fails (point.go:65) before any equation is checked
 *   B2K_SHUFFLE_SIMPLE  a thver check of SimpleShuffle.Verify fails: "incorrect SimpleShuffleProof" (shuffle/simple.go:186-254)
 *   B2K_SHUFFLE_PAIR    (33), (34) or (35) of PairShuffle.Verify fails: "invalid PairShuffleProof" (shuffle/pair.go:291-309)
 * A proof is the fixbuf encoding of the prover's messages, fields in declaration order, no length prefixes, 32 bytes per item:
 *   ega1 Gamma, A[k], C[k], U[k], W[k], Lambda1, Lambda2 | ega3 D[k] | ega5 Zsigma[k], Ztau | ssa0 X[k], Y[k] | ssa2 Theta[2k] |
 *   ssa4 Zalpha[2k - 1]   = 32 (12k + 3) bytes.
 * The transcript is proof.HashVerify's (proof/hash.go:92-142) with suite edwards25519.NewBlakeSHA256Ed25519: blake2xb.New(proto);
 * each PubRand Reseeds (128 stream bytes -> New(them), xof/blake2xb/blake.go:55-75) and absorbs the RAW proof bytes read since the
 * last one (ega1; ega3; ega5 || ssa0; ssa2 -- ssa4 and the inputs are not hashed); scalars are Scalar.Pick draws.  Proof
 * scalars (Zsigma, Ztau, Zalpha) are read raw (no reduction mod l, scalar.go:226-232; a top signed nibble above 8 selects
 * nothing, as in b2k_ed25519_msm).  Non-canonical point encodings are accepted; equality is exact point equality.
 * The transcript runs on host threads inside the call (it needs the proof bytes on the host, so there is no _dev form).
 * Bad data is never a call error, only a status.  B2K_ERR_ARG: a null pointer (proto may be null when proto_len = 0), k < 2,
 * or m, k or m k above B2K_SHUFFLE_MAX_PAIRS. */
#define B2K_SHUFFLE_MAX_PAIRS ((size_t)1 << 22)
enum { B2K_SHUFFLE_OK = 0, B2K_SHUFFLE_SIMPLE = 1, B2K_SHUFFLE_PAIR = 2, B2K_SHUFFLE_POINT = 3 };
/* status[s] of proof.HashVerify(suite, proto, shuffle.Verifier(suite, G, H, X[s], Y[s], Xbar[s], Ybar[s]), proofs[s]) for m
 * shuffles of k >= 2 pairs (proof/hash.go:168-175, shuffle/pair.go:369-377); g, h: NULL = the base point, else [m][32].
 * replaces: proof.HashVerify of one shuffle proof at a time (e.g. examples/neff_shuffle_test.go). */
int b2k_ed25519_shuffle_verify(b2k_ctx* ctx, size_t m, size_t k, const uint8_t* g /*[m][32] or NULL*/,
                               const uint8_t* h /*[m][32] or NULL*/, const uint8_t* x /*[m][k][32]*/, const uint8_t* y /*[m][k][32]*/,
                               const uint8_t* xbar /*[m][k][32]*/, const uint8_t* ybar /*[m][k][32]*/,
                               const uint8_t* proofs /*[m][32 (12k + 3)]*/, const uint8_t* proto, uint32_t proto_len,
                               uint8_t* status /*[m]*/);
/* shuffle.GetSequenceVerifiable (shuffle/sequences.go:155-190): x_up[i] = sum_j e[j] x[j][i], and y_up, x_down (xbar), y_down
 * (ybar) likewise, as canonical encodings.  e [nq][32] little-endian, read raw like any Point.Mul scalar.  A point that does not
 * decode -> B2K_ERR_POINT.  B2K_ERR_ARG: a null pointer, nq or k zero, or nq, k or nq k above B2K_SHUFFLE_MAX_PAIRS. */
int b2k_ed25519_shuffle_sequence_verifiable(b2k_ctx* ctx, size_t nq, size_t k, const uint8_t* x /*[nq][k][32]*/,
                                            const uint8_t* y /*[nq][k][32]*/, const uint8_t* xbar /*[nq][k][32]*/,
                                            const uint8_t* ybar /*[nq][k][32]*/, const uint8_t* e /*[nq][32]*/,
                                            uint8_t* x_up /*[k][32]*/, uint8_t* y_up /*[k][32]*/, uint8_t* x_down /*[k][32]*/,
                                            uint8_t* y_down /*[k][32]*/);

/* ---- edwards25519 ring signatures (sign/anon) --------------------------------------------------------------------------
 * status[j] of anon.Verify(suite, msg_j, ring, linkable ? scope : nil, sigs[j]) for m signatures over ONE ring and ONE
 * scope; suite = edwards25519.NewBlakeSHA256Ed25519 (XOF = blake2xb).  sig_j = C0 || S_0..S_{n-1} [|| Tag] (32 (n + 1 +
 * linkable) bytes; the caller cuts longer buffers and answers shorter ones itself, as fixbuf would).  tags (may be NULL):
 * the canonical Tag of every OK linkable signature, zero otherwise.  A ring key that does not decode -> B2K_ERR_POINT;
 * m == 0 or a null pointer -> B2K_ERR_ARG; n == 0 is legal (the reference's loop does not run).  Blocking, host buffers.
 *   B2K_ANON_INVALID  the final challenge differs from C0: "invalid signature" (sig.go:242-244)
 *   B2K_ANON_POINT    the Tag does not decode: "invalid Ed25519 curve point" (fixbuf's read of the Tag)
 * Scalars are read raw (no reduction mod l; a top signed nibble above 8 selects nothing, as geScalarMult and
 * geScalarMultBase do); C0 is compared as raw bytes (Scalar.Equal), so a C0 >= l never verifies when n >= 1.  A non-canonical
 * Tag encoding that decodes is accepted; H1 hashes, and tags returns, its canonical encoding.  One signature is one thread's
 * n-step chain: the batch is the use.  msgs/offsets as in b2k_ed25519_verify; ring may be NULL when n = 0, scope when
 * scope_len = 0 or unlinkable.  B2K_ERR_ARG also for m, n, m (n + 2) or scope_len above B2K_ANON_MAX.
 *   replaces: anon.Verify (sign/anon/sig.go:192-248) called once per signature */
#define B2K_ANON_MAX ((size_t)1 << 30)
enum { B2K_ANON_OK = 0, B2K_ANON_INVALID = 1, B2K_ANON_POINT = 2 };
int b2k_ed25519_anon_verify(b2k_ctx* ctx, size_t n, const uint8_t* ring /*[n][32]*/, int linkable,
                            const uint8_t* scope, size_t scope_len, size_t m, const uint8_t* msgs,
                            const uint32_t* offsets /*[m+1]*/, const uint8_t* sigs, uint8_t* status /*[m]*/,
                            uint8_t* tags /*[m][32] or NULL*/);

/* ---- edwards25519 ECIES (encrypt/ecies, hash SHA-256) -------------------------------------------------------------------
 * Byte for byte ecies.Encrypt / ecies.Decrypt (encrypt/ecies/ecies.go:23-112) on edwards25519 with sha256.New, the calls of
 * the Pedersen DKG's Deals (share/dkg/pedersen/dkg.go:364-385) and ProcessDeals (:470-494).  A ciphertext is
 * R (32) || AES-256-GCM(body) || tag (16); the AES key and the GCM nonce are HKDF-SHA256(dh.MarshalBinary(), salt nil,
 * info nil)[0:32] and [32:44]; no AAD.  R and the public keys decode like FromBytes (non-canonical y and small-order points
 * accepted, all-zero bytes are the point of order 4).  Scalars (priv, r) are 32 raw little-endian bytes read as
 * geScalarMult / geScalarMultBase read them: no reduction mod l, and a top signed digit above 8 selects nothing (see
 * b2k_ed25519_msm).  Constant time on the secrets (key, r, dh, the derived key, AES and GHASH state, plaintext): no
 * data-dependent branch or address on the device.  One length per call; bad data is only a status, never a call error.
 * B2K_ERR_ARG: a null pointer, n == 0, len out of range, or n len too large.  Blocking, host buffers, staged through the
 * context's input arena, which is cleared before the call returns.
 *   B2K_ECIES_POINT  R (decrypt) or the public key (encrypt) does not decode: "invalid Ed25519 curve point"
 *   B2K_ECIES_AUTH   the GCM tag does not match: "cipher: message authentication failed"
 * A reference ciphertext shorter than 48 bytes never reaches these calls: below 32 bytes it is "invalid ecies cipher"; from
 * 32 to 47 bytes the caller decodes R first ("invalid Ed25519 curve point"), then GCM Open fails on the short body.
 *   replaces: ecies.Decrypt / ecies.Encrypt called once per ciphertext */
#define B2K_ECIES_OK    0
#define B2K_ECIES_POINT 1
#define B2K_ECIES_AUTH  2
#define B2K_ECIES_MAX_LEN ((size_t)1 << 16)
/* len = ciphertext body incl. tag, 16 <= len <= B2K_ECIES_MAX_LEN + 16; msg[i] zeroed unless OK */
int b2k_ed25519_ecies_decrypt(b2k_ctx* ctx, const uint8_t* priv /*[32] LE*/, size_t n, size_t len,
                              const uint8_t* ctxt /*[n][32 + len]*/, uint8_t* msg /*[n][len - 16]*/, uint8_t* status /*[n]*/);
/* len = plaintext length, 0 <= len <= B2K_ECIES_MAX_LEN; ctxt[i] zeroed unless OK */
int b2k_ed25519_ecies_encrypt(b2k_ctx* ctx, size_t n, const uint8_t* pubs /*[n][32]*/, const uint8_t* r /*[n][32] LE*/,
                              size_t len, const uint8_t* msg /*[n][len]*/, uint8_t* ctxt /*[n][32 + len + 16]*/,
                              uint8_t* status /*[n]*/);

/* ---- BLS12-381 ECIES, keys on G1 or on G2 (encrypt/ecies, hash SHA-256) ---------------------------------------------------
 * Byte for byte ecies.Encrypt / ecies.Decrypt (encrypt/ecies/ecies.go:23-131) with the suite's G1 or G2 as the group and
 * sha256.New: the Pedersen DKG's Deals (share/dkg/pedersen/dkg.go:377) and ProcessDeals (:478) when its key group is BLS12-381
 * (keys on G1, or on G2).  A ciphertext is R.MarshalBinary() (48 bytes on G1, 96 on G2, ZCash compressed, kilic/g1.go:119-124,
 * g2.go:118-123) || AES-256-GCM(body) || tag (16); the AES key and the GCM nonce are HKDF-SHA256(dh.MarshalBinary(), salt nil,
 * info nil)[0:32] and [32:44] (an ikm of 48 or 96 bytes); no AAD.  R and the public keys decode as UnmarshalBinary does
 * (compressed form, x < p, on the curve, in the subgroup; infinity only as 0xC0 || 0...).  Scalars (priv, r) are mod.Int bytes:
 * 32 bytes big-endian; 0 is valid (dh and R are then infinity).  A scalar >= r fails the whole call with B2K_ERR_SCALAR_RANGE
 * before anything is staged; that check runs on the host as a borrow chain over all 32 bytes of every scalar, without an early
 * exit.  Bad data is only a status, never a call error.  B2K_ERR_ARG: a null pointer, n == 0, len out of range, or n len too
 * large.  Blocking, host buffers, staged through the context's input arena, which is cleared before the call returns.
 *   B2K_ECIES_POINT  R (decrypt) or the public key (encrypt) does not decode (UnmarshalBinary's error); ctxt/msg zeroed
 *   B2K_ECIES_AUTH   the GCM tag does not match: "cipher: message authentication failed"; msg zeroed
 * Constant time on the secrets (key, r, dh, R before it is returned, the derived key, AES and GHASH state, plaintext): no
 * data-dependent branch or address on the device.
 *   - scalar multiplication: 65 signed radix-16 digits, every digit reads all 8 table entries 1..8 P and keeps one with masks,
 *     then one complete addition (Renes-Costello-Batina, projective, no case for the identity or P = +-Q), 4 doublings between
 *     digits; no endomorphism split.  r G runs the same walk over 1..8 G.
 *   - compression of dh and R: Fermat inversion (on G2 of the norm), sign flag and infinity encoding chosen by masks.
 *   - AES without tables, GHASH with masks, the tag compared over all 16 bytes (as for edwards25519).
 * A reference ciphertext shorter than the point length is "invalid ecies cipher"; one too short for a tag fails GCM Open.
 *   replaces: ecies.Decrypt / ecies.Encrypt called once per ciphertext */
/* len = ciphertext body incl. tag, 16 <= len <= B2K_ECIES_MAX_LEN + 16; msg[i] zeroed unless OK */
int b2k_bls12381_g1_ecies_decrypt(b2k_ctx* ctx, const uint8_t* priv /*[32] BE*/, size_t n, size_t len,
                                  const uint8_t* ctxt /*[n][48 + len]*/, uint8_t* msg /*[n][len - 16]*/, uint8_t* status /*[n]*/);
int b2k_bls12381_g2_ecies_decrypt(b2k_ctx* ctx, const uint8_t* priv /*[32] BE*/, size_t n, size_t len,
                                  const uint8_t* ctxt /*[n][96 + len]*/, uint8_t* msg /*[n][len - 16]*/, uint8_t* status /*[n]*/);
/* len = plaintext length, 0 <= len <= B2K_ECIES_MAX_LEN; ctxt[i] zeroed unless OK */
int b2k_bls12381_g1_ecies_encrypt(b2k_ctx* ctx, size_t n, const uint8_t* pubs /*[n][48]*/, const uint8_t* r /*[n][32] BE*/,
                                  size_t len, const uint8_t* msg /*[n][len]*/, uint8_t* ctxt /*[n][48 + len + 16]*/,
                                  uint8_t* status /*[n]*/);
int b2k_bls12381_g2_ecies_encrypt(b2k_ctx* ctx, size_t n, const uint8_t* pubs /*[n][96]*/, const uint8_t* r /*[n][32] BE*/,
                                  size_t len, const uint8_t* msg /*[n][len]*/, uint8_t* ctxt /*[n][96 + len + 16]*/,
                                  uint8_t* status /*[n]*/);

/* status[i] = 0 iff eddsa.VerifyWithChecks(pks[i], msg_i, sigs[i]) == nil (sign/eddsa/eddsa.go:149-229), else the code of
 * the FIRST check that fails, in the reference's order:
 *   1 s >= l (scalar.IsCanonical)              -> ErrSignatureNotCanonical
 *   2 R's y >= p (point.IsCanonical)           -> ErrPointRNotCanonical
 *   3 R does not decode                        -> ErrPointRInvalid
 *   4 R has order 1, 2, 4 or 8 (HasSmallOrder) -> ErrPointRSmallOrder
 *   5, 6, 7 the same three checks on the key   -> ErrPKNotCanonical, ErrPKInvalid, ErrPKSmallOrder
 *   8 encode(s B) != encode(R + h A), h = SHA-512(R || pk || msg) mod l, cofactorless -> ErrSignatureRecNotEqual
 * Signatures (R || s) and keys have a fixed stride, so the reference's length errors are the caller's checks;
 * ErrSchnorrInvalidScalar cannot occur for 32 bytes.  msgs/offsets as in b2k_bls12381_verify_g1sig (decreasing offsets ->
 * B2K_ERR_ARG from the host form).  Bad data is never a call error, only a status.  The host form stages every input in
 * one device allocation and synchronises; the _dev form takes device pointers and only enqueues.
 * replaces: eddsa.Verify / VerifyWithChecks called in a loop (e.g. sign/dss/dss.go:216). */
enum { B2K_ED_OK = 0, B2K_ED_SIG_NOT_CANONICAL = 1, B2K_ED_R_NOT_CANONICAL = 2, B2K_ED_R_INVALID = 3,
       B2K_ED_R_SMALL_ORDER = 4, B2K_ED_PK_NOT_CANONICAL = 5, B2K_ED_PK_INVALID = 6, B2K_ED_PK_SMALL_ORDER = 7,
       B2K_ED_NOT_EQUAL = 8 };
int b2k_ed25519_verify(b2k_ctx* ctx, size_t n, const uint8_t* pks /*[n][32]*/, const uint8_t* msgs,
                       const uint32_t* offsets /*[n+1]*/, const uint8_t* sigs /*[n][64] R||s*/, uint8_t* status /*[n]*/);
int b2k_ed25519_verify_dev(b2k_ctx* ctx, size_t n, const void* d_pks, const void* d_msgs, const void* d_offsets,
                           const void* d_sigs, void* d_status);

/* ---- hash-to-G1 on the BN curves ------------------------------------------------------------------------- */
/* out[i] = Hash(msg_i) as 64 bytes x||y; msgs/offsets as in b2k_bls12381_hash_to_g1 (offsets[n+1], msg_i =
 * msgs[offsets[i] .. offsets[i+1])).
 * bn254: expand_message_xmd(Keccak-256) -> 2 field elements -> Shallue-van de Woestijne map -> add; dst as given
 *   (the suite default is "BN254G1_XMD:KECCAK-256_SVDW_RO_", pairing/bn254/suite.go:43).
 *   replaces: pointG1.Hash / hashToPoint, pairing/bn254/point.go:208-285 (per message in bls.Sign/Verify on bn254)
 * bn256: x = SHA-256(m) mod p, try-and-increment, y = (x^3+3)^((p+1)/4).
 *   replaces: pointG1.Hash / hashToPoint, pairing/bn256/point.go:261-312 (per message in sign/bls, sign/bdn on bn256) */
int b2k_bn254_hash_to_g1(b2k_ctx* ctx, size_t n, const uint8_t* msgs, const uint32_t* offsets, const uint8_t* dst,
                         uint32_t dst_len, uint8_t* out /*[n][64]*/);
int b2k_bn254_hash_to_g1_dev(b2k_ctx* ctx, size_t n, const void* d_msgs, const void* d_offsets, const void* d_dst,
                             uint32_t dst_len, void* d_out);
int b2k_bn256_hash_to_g1(b2k_ctx* ctx, size_t n, const uint8_t* msgs, const uint32_t* offsets, uint8_t* out /*[n][64]*/);
int b2k_bn256_hash_to_g1_dev(b2k_ctx* ctx, size_t n, const void* d_msgs, const void* d_offsets, void* d_out);
/* bn256 HashG1 (pairing/bn256/hash.go:10-110): t = 48 bytes of HKDF-SHA256(secret = msg, salt = dst, info = "H2C" 0 1) mod p
 * (gfp.go:46-67), then the Shallue-van de Woestijne map.  dst may be NULL / 0 (the reference's own vectors use a nil dst:
 * hash_test.go:11-19, reproduced in tests/).  Output 64 B x||y. */
int b2k_bn256_hash_g1(b2k_ctx* ctx, size_t n, const uint8_t* msgs, const uint32_t* offsets /*[n+1]*/, const uint8_t* dst,
                      uint32_t dst_len, uint8_t* out /*[n][64]*/);
int b2k_bn256_hash_g1_dev(b2k_ctx* ctx, size_t n, const void* d_msgs, const void* d_offsets, const void* d_dst, uint32_t dst_len,
                          void* d_out);

/* ---- sign/bdn: rogue-key coefficients (HOST function: no context, no device work) ------------------------- */
/* out[i] = c_i (+1 if add_one) as a 32-byte big-endian scalar, where c_0..c_{n-1} are the first 16 n bytes of
 * BLAKE2Xs (unkeyed, output length unknown) over pubs[0] || ... || pubs[n-1], 16 bytes per key read little-endian
 * (= reversed + SetBytes on the big-endian mod.Int of every pairing suite).  c_i < 2^128 < group order: no reduction.
 * replaces: bdn.hashPointToR, sign/bdn/bdn.go:29-63; with add_one = 1 the factors (c_i + 1) of the loops
 * bdn.AggregateSignatures (bdn.go:126-161) and NewMask (mask.go:57-61), whose sums are the *_msm entry points above
 * applied to (factors, signatures) / (factors, public keys) of the enabled participants.
 * The absorb phase is one sequential hash chain, so it runs on the host exactly as in the reference. */
int b2k_bdn_coefficients(size_t n, const uint8_t* pubs /*[n][pub_len] MarshalBinary bytes*/, size_t pub_len, int add_one,
                         uint8_t* out /*[n][32] BE*/);

/* ---- sign/bdn: masked aggregation and batch verification ----------------------------------------------------------------
 * The verifier's workload: many aggregate signatures over ONE roster, each with its own participation mask.  Three key groups:
 *   bls12381_g2  bdn.NewSchemeOnG1 (keys on G2, signatures on G1): keys 96 B compressed, terms 192 B operand form
 *   bls12381_g1  bdn.NewSchemeOnG2 (keys on G1, signatures on G2): keys 48 B compressed, terms 96 B operand form
 *   bn256_g2     bdn.NewSchemeOnG1(bn256.NewSuite()): keys and terms 128 B (bn256 has no hash onto G2: no second scheme)
 * Terms (NewMask, sign/bdn/mask.go:34-64): terms[i] = (c_i + 1) PK_i, with c_i = b2k_bdn_coefficients over the keys'
 *   MarshalBinary bytes -- the input bytes for BLS12-381, the canonical re-encoding (coordinates reduced mod p) for bn256,
 *   whose Unmarshal does not range-check.  Keys decode like UnmarshalBinary (BLS12-381: b2k_bls12381_g{1,2}_decompress,
 *   subgroup check included; bn256: b2k_bn256_g2_unmarshal_check); a key that does not decode -> B2K_ERR_POINT.
 *   Compute them once per roster.
 * Aggregate keys (AggregatePublicKeys, bdn.go:166-181, once per mask): out[k] = sum of terms[i] over the bits i < n set in
 *   masks[k] (bit i of byte i/8, least significant bit first: mask.go:88-97); bits at positions >= n are ignored; an empty mask
 *   gives infinity (all zeros).  Masks have a fixed stride of (n + 7) / 8 bytes, so the reference's "mismatching mask lengths"
 *   is the caller's check.  A pure sum of cached terms: no scalar multiplication.  Terms are re-validated like every operand
 *   (canonical coordinates where the curve's Unmarshal checks them, the curve equation): a violation -> B2K_ERR_POINT.
 * Verification (bls.Verify under each aggregate key, sign/bls/bls.go:82-96): status[k] in the reference's order
 *   B2K_BDN_SIG      the signature does not decode: "bls: unmarshalling signature point"
 *   B2K_BDN_INVALID  the pairing equation fails: "bls: invalid signature"
 *   msgs/offsets as in b2k_bls12381_verify_g1sig (offsets[m+1]); 0 < dst_len <= 255; bn256 hashes like b2k_bn256_hash_to_g1
 *   (try-and-increment, no dst).  Bad signature data is never a call error; an empty mask with the infinity signature is OK,
 *   as in the reference (e(H(m), O) = e(O, B) = 1).
 * B2K_ERR_ARG: a null pointer, n == 0 or m == 0, n above B2K_BDN_MAX_N, m above B2K_BDN_MAX_M, dst_len out of range, decreasing
 *   offsets (host forms).  The *_dev forms take device pointers and only enqueue; B2K_ERR_POINT then arrives at b2k_wait.
 * Not here: AggregateSignatures (the aggregator's side, one *_msm call each) and sign.Policy (the caller pop-counts its own
 * mask bytes).
 *   replaces: bdn.AggregatePublicKeys + bdn.Verify called once per aggregate signature */
#define B2K_BDN_MAX_N ((size_t)1 << 20)
#define B2K_BDN_MAX_M ((size_t)1 << 20)
enum { B2K_BDN_OK = 0, B2K_BDN_SIG = 1, B2K_BDN_INVALID = 2 };
int b2k_bls12381_g2_bdn_terms(b2k_ctx* ctx, size_t n, const uint8_t* pubs /*[n][96]*/, uint8_t* terms /*[n][192]*/);
int b2k_bls12381_g1_bdn_terms(b2k_ctx* ctx, size_t n, const uint8_t* pubs /*[n][48]*/, uint8_t* terms /*[n][96]*/);
int b2k_bn256_g2_bdn_terms(b2k_ctx* ctx, size_t n, const uint8_t* pubs /*[n][128]*/, uint8_t* terms /*[n][128]*/);
int b2k_bls12381_g2_bdn_aggregate_keys(b2k_ctx* ctx, size_t n, const uint8_t* terms /*[n][192]*/, size_t m,
                                       const uint8_t* masks /*[m][(n+7)/8]*/, uint8_t* out /*[m][192]*/);
int b2k_bls12381_g2_bdn_aggregate_keys_dev(b2k_ctx* ctx, size_t n, const void* d_terms, size_t m, const void* d_masks,
                                           void* d_out);
int b2k_bls12381_g1_bdn_aggregate_keys(b2k_ctx* ctx, size_t n, const uint8_t* terms /*[n][96]*/, size_t m,
                                       const uint8_t* masks /*[m][(n+7)/8]*/, uint8_t* out /*[m][96]*/);
int b2k_bls12381_g1_bdn_aggregate_keys_dev(b2k_ctx* ctx, size_t n, const void* d_terms, size_t m, const void* d_masks,
                                           void* d_out);
int b2k_bn256_g2_bdn_aggregate_keys(b2k_ctx* ctx, size_t n, const uint8_t* terms /*[n][128]*/, size_t m,
                                    const uint8_t* masks /*[m][(n+7)/8]*/, uint8_t* out /*[m][128]*/);
int b2k_bls12381_bdn_verify_g1sig(b2k_ctx* ctx, size_t n, const uint8_t* terms /*[n][192]*/, size_t m,
                                  const uint8_t* masks /*[m][(n+7)/8]*/, const uint8_t* msgs, const uint32_t* offsets /*[m+1]*/,
                                  const uint8_t* dst, uint32_t dst_len, const uint8_t* sigs /*[m][48]*/, uint8_t* status /*[m]*/);
int b2k_bls12381_bdn_verify_g1sig_dev(b2k_ctx* ctx, size_t n, const void* d_terms, size_t m, const void* d_masks,
                                      const void* d_msgs, const void* d_offsets, const void* d_dst, uint32_t dst_len,
                                      const void* d_sigs, void* d_status);
int b2k_bls12381_bdn_verify_g2sig(b2k_ctx* ctx, size_t n, const uint8_t* terms /*[n][96]*/, size_t m,
                                  const uint8_t* masks /*[m][(n+7)/8]*/, const uint8_t* msgs, const uint32_t* offsets /*[m+1]*/,
                                  const uint8_t* dst, uint32_t dst_len, const uint8_t* sigs /*[m][96]*/, uint8_t* status /*[m]*/);
int b2k_bls12381_bdn_verify_g2sig_dev(b2k_ctx* ctx, size_t n, const void* d_terms, size_t m, const void* d_masks,
                                      const void* d_msgs, const void* d_offsets, const void* d_dst, uint32_t dst_len,
                                      const void* d_sigs, void* d_status);
int b2k_bn256_bdn_verify_g1sig(b2k_ctx* ctx, size_t n, const uint8_t* terms /*[n][128]*/, size_t m,
                               const uint8_t* masks /*[m][(n+7)/8]*/, const uint8_t* msgs, const uint32_t* offsets /*[m+1]*/,
                               const uint8_t* sigs /*[m][64]*/, uint8_t* status /*[m]*/);

/* ---- sign/schnorr over BLS12-381 keys on G1 or on G2 ------------------------------------------------------------------------
 * status[i] = 0 iff schnorr.VerifyWithChecks(suite.G1() or suite.G2(), pks[i], msg_i, sigs[i]) == nil
 * (sign/schnorr/schnorr.go:89-183), else the code of the FIRST check that fails, in the reference's order:
 *   1 B2K_SCHNORR_R        R (the first 48 / 96 bytes of sig) does not decode: kilic's UnmarshalBinary error (ZCash flags,
 *                          x < p, on the curve, in the order-r subgroup: b2k_bls12381_g{1,2}_decompress)
 *   2 B2K_SCHNORR_S        s (the last 32 bytes, big-endian) >= r: mod.Int's "UnmarshalBinary: value out of range"
 *   3 B2K_SCHNORR_PK       the key does not decode: "schnorr: error unmarshalling public key"
 *   4 B2K_SCHNORR_INVALID  s B != R + h public, h = SHA-512(R || public || msg) read big-endian mod r: "schnorr: invalid signature"
 * The reference's "point not in correct group" (R.IsInCorrectGroup) cannot fail on this backend: UnmarshalBinary already
 * refused every point outside the subgroup.  Neither kilic's points nor mod.Int have IsCanonical / HasSmallOrder, so those
 * checks do not apply.  The digest hashes the input bytes of R and of the key: the decoders accept only encodings that are
 * their own MarshalBinary.  Infinity is a valid R and a valid key, as in the reference: with the key at infinity a signature
 * is valid iff s B = R, and (R, s, key) = (O, 0, O) is accepted.
 * Signatures (R || s: 80 bytes with keys on G1, 128 on G2) and keys have a fixed stride, so the reference's length error is
 * the caller's check.  msgs/offsets as in b2k_ed25519_verify.  Bad data is never a call error, only a status; n == 0, a null
 * pointer or decreasing offsets (host forms) -> B2K_ERR_ARG.  The host forms stage every input in one device allocation and
 * synchronise; the _dev forms take device pointers and only enqueue.
 * replaces: schnorr.Verify / VerifyWithChecks called once per packet, e.g. dkg.VerifyPacketSignature
 * (share/dkg/pedersen/structs.go:293-348, protocol.go:275-281), share/vss/pedersen vss.go:439, 675, share/vss/rabin
 * vss.go:485, 677, share/dkg/rabin dkg.go:454, 494, 563.  On edwards25519, b2k_ed25519_verify is the device path: the two
 * schemes accept exactly the same signatures there. */
enum { B2K_SCHNORR_OK = 0, B2K_SCHNORR_R = 1, B2K_SCHNORR_S = 2, B2K_SCHNORR_PK = 3, B2K_SCHNORR_INVALID = 4 };
int b2k_bls12381_g1_schnorr_verify(b2k_ctx* ctx, size_t n, const uint8_t* pks /*[n][48]*/, const uint8_t* msgs,
                                   const uint32_t* offsets /*[n+1]*/, const uint8_t* sigs /*[n][80] R||s*/, uint8_t* status /*[n]*/);
int b2k_bls12381_g1_schnorr_verify_dev(b2k_ctx* ctx, size_t n, const void* d_pks, const void* d_msgs, const void* d_offsets,
                                       const void* d_sigs, void* d_status);
int b2k_bls12381_g2_schnorr_verify(b2k_ctx* ctx, size_t n, const uint8_t* pks /*[n][96]*/, const uint8_t* msgs,
                                   const uint32_t* offsets /*[n+1]*/, const uint8_t* sigs /*[n][128] R||s*/, uint8_t* status /*[n]*/);
int b2k_bls12381_g2_schnorr_verify_dev(b2k_ctx* ctx, size_t n, const void* d_pks, const void* d_msgs, const void* d_offsets,
                                       const void* d_sigs, void* d_status);

#ifdef __cplusplus
}
#endif
#endif /* B2KYBER_H */
