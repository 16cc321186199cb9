// msm_host.cuh -- host-side launch templates shared by the translation units of libb2kyber.so
// (plan selection, scratch layout, stage timing, enqueue of the MSM pipeline and of mul_batch).
#pragma once
#include <cuda_runtime.h>
#include <cstring>
#include <string>
#include "../../include/b2kyber.h"
#include "b2k_ctx.h"
#include "kernels.cuh"

namespace b2k_host {
using namespace b2k;
constexpr int N_EV = B2K_N_EV;

#define CK(call)                                                                       \
  do {                                                                                 \
    cudaError_t e_ = (call);                                                           \
    if (e_ != cudaSuccess) {                                                           \
      ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_);                   \
      return B2K_ERR_CUDA;                                                             \
    }                                                                                  \
  } while (0)

inline int arena_reserve(b2k_ctx* ctx, size_t bytes) { return b2k_arena_reserve(ctx, bytes); }
template <class T>
T* arena_take(b2k_ctx* ctx, size_t count) { return reinterpret_cast<T*>(b2k_arena_take(ctx, count * sizeof(T))); }
inline size_t pad256(size_t b) { return (b + 255) & ~size_t(255); }
inline int pick_window(size_t n, int scalar_bits) {
  // minimise  W * (10 n + 40 * 2^(c-1))  field multiplications (mixed add ~10, bucket reduce ~40/bucket)
  int best = 4;
  double bestc = 1e300;
  for (int c = 4; c <= 16; c++) {
    int W = (scalar_bits + c) / c;
    double cost = (double)W * (10.0 * (double)n + 40.0 * (double)(1u << (c - 1)));
    if (cost < bestc) { bestc = cost; best = c; }
  }
  return best;
}

// scalar_bits = bit length of the group order: signed-digit recoding needs windows for scalar_bits + 1 bits
inline MsmPlan make_plan(size_t n, int force_c, int scalar_bits, int force_m = 0) {
  MsmPlan pl;
  pl.c = force_c ? force_c : pick_window(n, scalar_bits);
  pl.W = (scalar_bits + pl.c) / pl.c;
  pl.nb = 1 << (pl.c - 1);
  size_t total = (size_t)pl.W * pl.nb;
  int m = 1;
  while (m < 64 && m * 2 <= pl.nb && total / (size_t)(m * 2) >= 32768) m *= 2;   // >= 32k reduction threads (measured best)
  if (force_m > 0 && force_m <= pl.nb && (force_m & (force_m - 1)) == 0) m = force_m;
  pl.m = m;
  memset(pl.K, 0, sizeof pl.K);
  for (int w = 0; w < pl.W; w++) {
    int bit = pl.c * w + pl.c - 1;
    pl.K[bit >> 5] |= 1u << (bit & 31);
  }
  return pl;
}

// slice length of the balanced accumulate: 64 additions per thread when there is enough work to fill
// the chip (>= 128k slices), shorter slices for small problems
inline uint32_t slice_len_entries(size_t e, int force_L) {
  if (force_L > 0) return (uint32_t)force_L;
  size_t L = e / 131072;
  if (L > 64) L = 64;
  if (L < 4) L = 4;
  return (uint32_t)L;
}
inline uint32_t slice_len(size_t n, const MsmPlan& pl, int force_L) { return slice_len_entries(n * (size_t)pl.W, force_L); }


// ---- bucket reduction: one level (chunks of pl.m buckets, a small scalar multiplication per chunk) or two levels
// (msm.cuh: msm_reduce_l1 / msm_reduce_l2: the scalar multiplications move to the level with m1 times fewer operands) ----
struct ReducePlan {
  int levels = 1;
  int m1 = 1, m2 = 1, log2_m1 = 0;
  int T1 = 0;      // level-1 chunks (= run sums) per window
  int TP = 0;      // partials per window that the window sum adds up
};
inline ReducePlan reduce_plan(const b2k_ctx* ctx, int nb, int single_m) {
  ReducePlan rp;
  // defaults chosen by A/B at C2 (b2k_set_msm_reduce): (8, 4) beat one level for the pipelined MSM
  int m1 = ctx->reduce_m1 > 0 ? ctx->reduce_m1 : 8, m2 = ctx->reduce_m2 > 0 ? ctx->reduce_m2 : 4;
  const bool fits = nb >= 4096 && nb % (m1 * m2) == 0;
  const bool two = ctx->reduce_levels == 2 ? (nb % (m1 * m2) == 0 && nb / (m1 * m2) >= 1) : (ctx->reduce_levels == 0 && fits);
  if (two) {
    rp.levels = 2; rp.m1 = m1; rp.m2 = m2;
    while ((1 << rp.log2_m1) < m1) rp.log2_m1++;
    rp.T1 = nb / m1;
    rp.TP = rp.T1 + rp.T1 / m2;
  } else {
    rp.m1 = single_m; rp.T1 = nb / single_m; rp.TP = rp.T1;
  }
  return rp;
}
// sub-blocks of the two-level window sum: S blocks of TP / S partials each
inline int window_sum_split(int TP) {
  int S = 1;
  if (TP >= 1024) {
    S = TP / 512;
    if (S > 128) S = 128;
    while (S > 1 && TP % S) S--;
  }
  return S;
}

inline int check_flags(b2k_ctx* ctx) {
  uint32_t f = *ctx->h_flags;
  if (f & FLAG_SCALAR_RANGE) { ctx->err = "scalar not below the group order"; return B2K_ERR_SCALAR_RANGE; }
  if (f & FLAG_POINT) { ctx->err = "malformed operand point"; return B2K_ERR_POINT; }
  if (f & FLAG_COMM_TIMEOUT) { ctx->err = "multi-GPU exchange: a peer rank did not arrive within 10 s"; return B2K_ERR_COMM; }
  return B2K_OK;
}

// message offsets of the host entry points: non-decreasing (ADVICE r1: a decreasing pair would make a kernel read ~4 GiB)
inline int check_offsets(b2k_ctx* ctx, size_t n, const uint32_t* offsets) {
  for (size_t i = 0; i < n; i++)
    if (offsets[i + 1] < offsets[i]) { ctx->err = "message offsets must be non-decreasing"; return B2K_ERR_ARG; }
  return B2K_OK;
}

// host-buffer entry points: the device status word is cleared in front of the call's work, fetched AND cleared behind it
// (a failed call must not leave a stale bit for a later *_dev sequence + b2k_wait)
inline int status_begin(b2k_ctx* ctx) {
  CK(cudaMemsetAsync(ctx->d_flags, 0, 4, ctx->stream));
  return B2K_OK;
}
inline int status_fetch_async(b2k_ctx* ctx) {
  CK(cudaMemcpyAsync(ctx->h_flags, ctx->d_flags, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemsetAsync(ctx->d_flags, 0, 4, ctx->stream));
  return B2K_OK;
}
inline int status_finish(b2k_ctx* ctx) {
  int rc = status_fetch_async(ctx);
  if (rc) return rc;
  CK(cudaStreamSynchronize(ctx->stream));
  return check_flags(ctx);
}

// ---- GLV front end: which curves have it, and the problem the pipeline then sees ----------------------------------
template <class CV> struct GlvTraits { static constexpr bool enabled = false; static constexpr int bits = 0; };
template <> struct GlvTraits<Bls381G1> { static constexpr bool enabled = true; static constexpr int bits = GLV_BITS_BLS381; };

template <class CV>
inline bool msm_uses_glv(const b2k_ctx* ctx, size_t n) { return GlvTraits<CV>::enabled && ctx->use_glv && n < (size_t(1) << 30); }
// number of (scalar, point) pairs the sort/accumulate stages process
template <class CV>
inline size_t msm_virtual_n(const b2k_ctx* ctx, size_t n) { return msm_uses_glv<CV>(ctx, n) ? 2 * n : n; }
template <class CV>
inline MsmPlan msm_plan(const b2k_ctx* ctx, size_t n) {
  const bool g = msm_uses_glv<CV>(ctx, n);
  return make_plan(g ? 2 * n : n, ctx->force_c, g ? GlvTraits<CV>::bits : CV::SCALAR_BITS, ctx->force_m);
}

// ---- affine pair-tree rounds in front of the XYZZ slices (msm_affine.cuh): which curves, how many, how wide ----------
template <class CV> struct AffineTraits { static constexpr bool enabled = false; };
template <> struct AffineTraits<Bls381G1> { static constexpr bool enabled = true; };
constexpr int PT_MAX_ROUNDS = 8;
struct AffinePlan {
  int R = 0;                            // rounds
  uint32_t B[PT_MAX_ROUNDS] = {};       // outputs per thread
  size_t bound[PT_MAX_ROUNDS + 1] = {}; // host-side upper bound of the operand count before round r (bound[R]: what the slices see)
  uint32_t T[PT_MAX_ROUNDS] = {};       // threads of round r (multiple of the block size)
  size_t pre_elems = 0;                 // split rounds: field elements of the prefix-product array (max over the rounds)
  uint32_t max_T = 0;
};
// n = pairs the pipeline processes (msm_virtual_n)
template <class CV>
inline AffinePlan affine_plan(const b2k_ctx* ctx, size_t n, const MsmPlan& pl) {
  AffinePlan ap;
  ap.bound[0] = n * (size_t)pl.W;
  if (!AffineTraits<CV>::enabled || ctx->use_v1 || ctx->msm_groups > 1) return ap;
  const size_t total = (size_t)pl.W * pl.nb;
  int R = ctx->affine_rounds;
  // automatic: no rounds.  Measured on H100 at C2 (64 operands per bucket; profiles/h100_kernels_*.txt, h100_rounds_*.txt):
  // every round costs about the XYZZ slice time it saves (round 0: 0.94 + 0.14 + 2.38 ms of forward / inversion / backward
  // against 3.37 ms of slices), so 0..3 rounds land within 1.5 % of each other in kernel time, none ahead of R = 0, and no
  // batch width 16..256 beat the automatic one; without rounds the MSM also needs ~1.6 GB less scratch (round outputs and
  // prefix products).  b2k_set_msm_affine still forces them.
  if (R < 0) R = 0;
  if (R > PT_MAX_ROUNDS) R = PT_MAX_ROUNDS;
  ap.R = R;
  for (int r = 0; r < R; r++) {
    ap.bound[r + 1] = (ap.bound[r] + total) / 2 + 1;   // ceil(k/2) summed over the buckets
    size_t B = ctx->affine_batch > 0 ? (size_t)ctx->affine_batch : ap.bound[r + 1] / ((size_t)ctx->sm_count * 512);   // 512 threads per SM
    if (ctx->affine_batch <= 0 && B < 32) B = 32;       // one inversion per thread: keep it amortised
    if (B < 1) B = 1;
    const size_t bmax = ctx->affine_split ? 1024 : (size_t)PT_MAXB;    // the fused kernel keeps B prefix products in local memory
    if (B > bmax) B = bmax;
    ap.B[r] = (uint32_t)B;
    ap.T[r] = (uint32_t)(((ap.bound[r + 1] + B - 1) / B + 127) / 128 * 128);
    if ((size_t)ap.T[r] * B > ap.pre_elems) ap.pre_elems = (size_t)ap.T[r] * B;
    if (ap.T[r] > ap.max_T) ap.max_T = ap.T[r];
  }
  return ap;
}

// ------------------------------------------------------------------------------------------------
// Resident blocks per SM of the slice kernels (register cap 65536 / (128 * MINB)): the most at which sm_90a still compiles their
// field products without spills (tools/codegen_check.py, tests/test_codegen.py): 4 up to 10-limb fields, 3 for BLS12-381's 12 limbs;
// Fp2 points need the uncapped 255 registers.  A spilling product lengthens every addition of the pass.
template <class CV>
constexpr int slice_minb() { return sizeof(typename CV::F) > 48 ? 1 : sizeof(typename CV::F) > 40 ? 3 : 4; }

// n = number of pairs the pipeline processes (msm_virtual_n)
template <class CV>
size_t msm_scratch_bytes(const b2k_ctx* ctx, size_t n, const MsmPlan& pl) {
  const int force_L = ctx->force_L;
  using F = typename CV::F;
  size_t total = (size_t)pl.W * pl.nb;
  size_t T = pl.nb / pl.m;
  size_t b = 0;
  b += pad256(n * sizeof(Affine<F>));
  b += pad256(n * (size_t)pl.W * 2);              // digit columns (int16, window-major)
  b += pad256((total + 1) * 4) * 3;               // counts, offs, cursor
  b += pad256(n * (size_t)pl.W * sizeof(SortRec)); // coarse-partitioned (entry, bucket) records of the bucket sort
  b += pad256(n * (size_t)pl.W * 4);              // entries
  b += pad256(total * sizeof(Xyzz<F>));           // buckets
  b += pad256((size_t)pl.W * T * sizeof(Xyzz<F>));  // partials
  {
    const ReducePlan rp = reduce_plan(ctx, pl.nb, pl.m);
    b += pad256((size_t)pl.W * (size_t)(rp.TP + rp.T1) * sizeof(Xyzz<F>));   // two-level partials + run sums
  }
  b += pad256((size_t)pl.W * (1 + 128) * sizeof(Xyzz<F>));    // window sums + their sub-block partials
  size_t smax = (n * (size_t)pl.W) / (size_t)slice_len(n, pl, force_L) + 2;
  const AffinePlan ap = affine_plan<CV>(ctx, n, pl);
  if (ap.R > 0) {                                 // the slices after the rounds may be shorter, hence more numerous
    size_t sa = ap.bound[ap.R] / (size_t)slice_len_entries(ap.bound[ap.R], force_L) + 2;
    if (sa > smax) smax = sa;
  }
  b += pad256(2 * smax * sizeof(Xyzz<F>));        // slice partials (worst case: smallest automatic L)
  b += pad256((total + 1) * 4) + pad256(4096 * (size_t)(1 + ap.R));   // big-bucket list, block sums (one page per scanned column)
  if (ap.R > 0) {
    b += pad256((size_t)ap.R * (total + 1) * 4);  // bucket offsets after each round
    b += pad256(ap.bound[1] * sizeof(Affine<F>));
    if (ap.R > 1) b += pad256(ap.bound[2] * sizeof(Affine<F>));
    if (ctx->affine_split) b += pad256(ap.pre_elems * sizeof(F)) + pad256((size_t)ap.max_T * sizeof(F));
  }
  return b + 8192;
}

// Enqueue the whole MSM on ctx->stream. d_scalars/d_points/d_out are device pointers; scratch must
// already be reserved (arena) for msm_scratch_bytes(msm_virtual_n(n)) and pl must come from msm_plan(n).
template <class CV>
int msm_enqueue(b2k_ctx* ctx, size_t n_in, const MsmPlan& pl, const uint8_t* d_scalars_in, const uint8_t* d_points,
                uint8_t* d_out, int affine_out = 0, Xyzz<typename CV::F>* ext_buckets = nullptr) {
  using F = typename CV::F;
  cudaStream_t st = ctx->stream;
  const bool glv = msm_uses_glv<CV>(ctx, n_in);
  const size_t n = glv ? 2 * n_in : n_in;          // pairs seen by the digit / sort / accumulate stages
  size_t total = (size_t)pl.W * pl.nb;
  int T = pl.nb / pl.m;
  auto* pts = arena_take<Affine<F>>(ctx, n);
  auto* digits = arena_take<int16_t>(ctx, n * (size_t)pl.W);
  auto* counts = arena_take<uint32_t>(ctx, total + 1);
  auto* offs = arena_take<uint32_t>(ctx, total + 1);
  auto* cursor = arena_take<uint32_t>(ctx, total + 1);
  auto* recs = arena_take<SortRec>(ctx, n * (size_t)pl.W);
  auto* entries = arena_take<uint32_t>(ctx, n * (size_t)pl.W);
  auto* own_buckets = arena_take<Xyzz<F>>(ctx, total);
  // bucket exchange (multi-GPU shape 1): the pipeline stops after the fix-up and leaves the W x 2^(c-1) buckets in the caller's buffer
  auto* buckets = ext_buckets ? ext_buckets : own_buckets;
  const ReducePlan rp = reduce_plan(ctx, pl.nb, pl.m);
  auto* partials = arena_take<Xyzz<F>>(ctx, (size_t)pl.W * (size_t)(rp.TP > T ? rp.TP : T));
  auto* runs = arena_take<Xyzz<F>>(ctx, (size_t)pl.W * rp.T1);
  auto* wsum = arena_take<Xyzz<F>>(ctx, pl.W);
  // window sum in two levels when a window has many chunk partials: S sub-blocks of >= 512 partials each
  const int S = window_sum_split(rp.TP);
  auto* wpart = arena_take<Xyzz<F>>(ctx, (size_t)pl.W * 128);
  if (!wpart) { ctx->err = "scratch arena too small"; return B2K_ERR_ARG; }
  if (!pts || !digits || !counts || !offs || !cursor || !recs || !entries || !own_buckets || !partials || !runs || !wsum) {
    ctx->err = "scratch arena too small";
    return B2K_ERR_ARG;
  }
  const uint32_t L = slice_len(n, pl, ctx->force_L);
  const uint32_t smax = (uint32_t)((n * (size_t)pl.W + L - 1) / L) + 1;
  const AffinePlan ap = affine_plan<CV>(ctx, n, pl);
  const uint32_t La = ap.R > 0 ? slice_len_entries(ap.bound[ap.R], ctx->force_L) : L;
  const uint32_t sa = ap.R > 0 ? (uint32_t)((ap.bound[ap.R] + La - 1) / La) + 1 : 0;      // slices after the affine rounds
  auto* spart = arena_take<Xyzz<F>>(ctx, 2 * (size_t)(sa > smax ? sa : smax));
  auto* big_list = arena_take<uint32_t>(ctx, total + 1);
  auto* bsum = arena_take<uint32_t>(ctx, 1024 * (size_t)(1 + ap.R));   // block sums of the scan, 1024 words per column
  if (!spart || !big_list || !bsum || total > 1024u * 1024u || (pl.nb >> sort_shift(pl.c)) > PART_BPW) {
    ctx->err = "scratch arena too small / too many buckets";
    return B2K_ERR_ARG;
  }
  // bucket offsets after round r + 1: offs_rt + r (total + 1), written by the stage-2 scan (columns 1..R)
  uint32_t* offs_rt = nullptr;
  Affine<F>* aff_rt[2] = {nullptr, nullptr};
  if (ap.R > 0) {
    offs_rt = arena_take<uint32_t>(ctx, (size_t)ap.R * (total + 1));
    aff_rt[0] = arena_take<Affine<F>>(ctx, ap.bound[1]);
    if (ap.R > 1) aff_rt[1] = arena_take<Affine<F>>(ctx, ap.bound[2]);
    if (!offs_rt || !aff_rt[0] || (ap.R > 1 && !aff_rt[1])) { ctx->err = "scratch arena too small"; return B2K_ERR_ARG; }
  }
  F* pt_pre = nullptr;
  F* pt_accs = nullptr;
  if (ap.R > 0 && ctx->affine_split) {
    pt_pre = arena_take<F>(ctx, ap.pre_elems);
    pt_accs = arena_take<F>(ctx, ap.max_T);
    if (!pt_pre || !pt_accs) { ctx->err = "scratch arena too small"; return B2K_ERR_ARG; }
  }
  {
    int* lp = ctx->last_plan;
    lp[0] = pl.c; lp[1] = pl.W; lp[2] = pl.nb; lp[3] = pl.m;
    lp[4] = (int)La;
    lp[5] = ap.R;
    for (int r = 0; r < PT_MAX_ROUNDS; r++) lp[6 + r] = r < ap.R ? (int)ap.B[r] : 0;
    lp[14] = glv ? 1 : 0;
    lp[15] = (ap.R > 0 && ctx->affine_split) ? 1 : 0;
    lp[16] = rp.levels; lp[17] = rp.m1; lp[18] = rp.levels == 2 ? rp.m2 : 0;
  }
  uint32_t* big_count = bsum + 1023;      // last word of the block-sum page is never a block sum (<= 1023 blocks used)
  unsigned gb_n = (unsigned)((n + 255) / 256);
  unsigned sblocks = (unsigned)((total + 1023) / 1024);
  int nl = 0;
  CK(cudaEventRecord(ctx->ev[0], st));
  CK(cudaMemsetAsync(counts, 0, (total + 1) * 4, st));
  if (ctx->h2d_chunks > 1 && !glv) CK(cudaStreamWaitEvent(st, ctx->gev[ctx->h2d_chunks], 0));   // (not reached: msm_host chunks GLV calls only)
  if constexpr (GlvTraits<CV>::enabled) {
    if (glv && ctx->h2d_chunks > 1) {
      // host-buffer call: the inputs arrive in chunks on the copy stream (msm_host); every chunk is prepared as soon as it has landed,
      // so that only the last chunk's front-end work is left when the copy ends
      const size_t per = (n_in + ctx->h2d_chunks - 1) / ctx->h2d_chunks;
      for (int k = 0; k < ctx->h2d_chunks; k++) {
        const size_t i0 = (size_t)k * per;
        if (i0 >= n_in) break;
        const size_t cnt = (n_in - i0 < per) ? n_in - i0 : per;
        CK(cudaStreamWaitEvent(st, ctx->gev[1 + k], 0));
        k_glv_prepare_bls381<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(n_in, i0, cnt, d_scalars_in, d_points, pts, pl, digits, counts, ctx->d_flags);
      }
    } else if (glv) k_glv_prepare_bls381<<<(unsigned)((n_in + 255) / 256), 256, 0, st>>>(n_in, 0, n_in, d_scalars_in, d_points, pts, pl, digits, counts, ctx->d_flags);
    else k_msm_load<CV><<<gb_n, 256, 0, st>>>(n, d_scalars_in, d_points, pts, pl, digits, counts, ctx->d_flags);
  } else {
    k_msm_load<CV><<<gb_n, 256, 0, st>>>(n, d_scalars_in, d_points, pts, pl, digits, counts, ctx->d_flags);
  }
  nl++;
  CK(cudaEventRecord(ctx->ev[1], st));             // the digits and the histogram come out of the load pass: ev[1..2] is empty
  CK(cudaEventRecord(ctx->ev[2], st));
  {
    const dim3 cols(sblocks, 1 + ap.R), tops(1, 1 + ap.R);     // the histogram + the bucket sizes after each affine round
    k_scan_blocks<<<cols, 1024, 0, st>>>((uint32_t)total, counts, offs, offs_rt, bsum);
    k_scan_tops<<<tops, 1024, 0, st>>>(sblocks, (uint32_t)total, bsum, offs, offs_rt);
    k_scan_finish<<<cols, 1024, 0, st>>>((uint32_t)total, bsum, offs, offs_rt, cursor); nl += 3;
  }
  CK(cudaEventRecord(ctx->ev[3], st));
  {
    const int S = sort_shift(pl.c);
    const size_t nrec = n * (size_t)pl.W;
    k_msm_partition<<<(unsigned)((n + PART_TILE - 1) / PART_TILE), PART_T, 0, st>>>((uint32_t)n, pl, S, digits, cursor, recs);
    k_msm_bin_sort<<<(unsigned)((nrec + BSORT_TILE - 1) / BSORT_TILE), BSORT_T, 0, st>>>((uint32_t)total, S, recs, offs, counts, entries);
    nl += 2;
  }
  const int G = (!ext_buckets && !ctx->use_v1 && ctx->msm_groups > 1 && pl.W >= 2 * ctx->msm_groups && ctx->stream2) ? ctx->msm_groups : 1;
  if (G > 1) {
    // ---- overlapped tail: groups of windows, top group first; reduction of group g on stream2 while the main
    //      stream accumulates group g-1.  ms[4] = all accumulate launches, ms[5] = what is left after them.
    cudaStream_t s2 = ctx->stream2;
    uint32_t* ranges = bsum + 900;                 // G+1 words
    uint32_t* bigc = bsum + 920;                   // one counter per group
    CK(cudaMemsetAsync(buckets, 0, total * sizeof(Xyzz<F>), st));
    CK(cudaMemsetAsync(bigc, 0, 64, st));
    k_msm_group_ranges<<<1, 32, 0, st>>>(G, pl.W, pl.nb, L, (uint32_t)total, offs, ranges); nl++;
    CK(cudaEventRecord(ctx->ev[4], st));
    CK(cudaEventRecord(ctx->ev[10], st));
    for (int g = G - 1; g >= 0; g--) {
      const int w_lo = g * pl.W / G, w_hi = (g + 1) * pl.W / G, w_cnt = w_hi - w_lo;
      k_msm_accumulate_slices_range<CV><<<(smax + 127) / 128, 128, 0, st>>>(ranges, g, L, (uint32_t)total, pts, offs, entries, buckets, spart); nl++;
      CK(cudaEventRecord(ctx->gev[g], st));
      CK(cudaStreamWaitEvent(s2, ctx->gev[g], 0));
      const uint32_t gid_lo = (uint32_t)((size_t)w_lo * pl.nb), gid_hi = (uint32_t)((size_t)w_hi * pl.nb);
      k_msm_fixup_range<CV><<<(gid_hi - gid_lo + 127) / 128, 128, 0, s2>>>(gid_lo, gid_hi, L, offs, buckets, spart, bigc + g, big_list + gid_lo);
      k_msm_fixup_big<CV><<<64, 128, 0, s2>>>(L, offs, buckets, spart, bigc + g, big_list + gid_lo);
      size_t nch = (size_t)w_cnt * T;
      k_msm_reduce_chunks_range<CV><<<(unsigned)((nch + 127) / 128), 128, 0, s2>>>(pl, w_lo, w_cnt, buckets, partials);
      k_msm_window_sum<CV><<<w_cnt, 128, 0, s2>>>(T, partials, wsum, w_lo); nl += 4;
    }
    CK(cudaEventRecord(ctx->ev[9], st));           // end of the accumulate launches
    CK(cudaEventRecord(ctx->gev[G], s2));
    CK(cudaStreamWaitEvent(st, ctx->gev[G], 0));
    CK(cudaEventRecord(ctx->ev[5], st));
    CK(cudaEventRecord(ctx->ev[6], st));
    CK(cudaEventRecord(ctx->ev[7], st));
    k_msm_final<CV><<<1, 128, 0, st>>>(pl, wsum, d_out, affine_out); nl++;
    CK(cudaEventRecord(ctx->ev[8], st));
  } else {
  if (ctx->use_v1) {
    CK(cudaEventRecord(ctx->ev[4], st));
    CK(cudaEventRecord(ctx->ev[10], st));
    k_msm_accumulate<CV><<<(unsigned)((total + 127) / 128), 128, 0, st>>>(total, pts, offs, entries, buckets); nl++;
    CK(cudaEventRecord(ctx->ev[9], st));
  } else {
    CK(cudaMemsetAsync(buckets, 0, total * sizeof(Xyzz<F>), st));
    CK(cudaMemsetAsync(big_count, 0, 4, st));
    CK(cudaEventRecord(ctx->ev[4], st));
    if (ap.R > 0) {
      if constexpr (AffineTraits<CV>::enabled) {
        // ---- affine pair-tree rounds: operands of every bucket halve per round; the slices below finish the rest
        const uint32_t* offs_cur = offs;
        const Affine<F>* in_cur = pts;
        for (int r = 0; r < ap.R; r++) {
          const uint32_t* offs_nxt = offs_rt + (size_t)r * (total + 1);
          Affine<F>* out = aff_rt[r & 1];
          const unsigned grid = ap.T[r] / 128;
          if (ctx->affine_split) {
            constexpr size_t fstage_bytes = 128 * 4 * sizeof(F);              // two 2-coordinate buffers per thread (24 KB for G1)
            if (fstage_bytes <= 48 * 1024 && ((ctx->pt_stage >> (r == 0 ? 2 : 3)) & 1)) {
              if (r == 0) k_pt_forward_staged<CV, true><<<grid, 128, fstage_bytes, st>>>(ap.B[r], (uint32_t)total, in_cur, entries, offs_cur, offs_nxt, pt_pre, pt_accs);
              else k_pt_forward_staged<CV, false><<<grid, 128, fstage_bytes, st>>>(ap.B[r], (uint32_t)total, in_cur, nullptr, offs_cur, offs_nxt, pt_pre, pt_accs);
            } else {
              if (r == 0) k_pt_forward<CV, true><<<grid, 128, 0, st>>>(ap.B[r], (uint32_t)total, in_cur, entries, offs_cur, offs_nxt, pt_pre, pt_accs);
              else k_pt_forward<CV, false><<<grid, 128, 0, st>>>(ap.B[r], (uint32_t)total, in_cur, nullptr, offs_cur, offs_nxt, pt_pre, pt_accs);
            }
            if (ctx->acc_minb == 5) k_pt_invert<F, 5><<<grid, 128, 0, st>>>(ap.B[r], (uint32_t)total, offs_nxt, pt_accs);
            else k_pt_invert<F, 4><<<grid, 128, 0, st>>>(ap.B[r], (uint32_t)total, offs_nxt, pt_accs);
            constexpr size_t stage_bytes = 128 * (4 * sizeof(Affine<F>) + sizeof(F));   // per thread two 2-point buffers + one prefix product (54 KB for G1)
            const bool staged = stage_bytes <= 56 * 1024 && ((ctx->pt_stage >> (r == 0 ? 0 : 1)) & 1);
            if (staged) {
              if (!ctx->pt_stage_opted) {                     // more than 48 KB of dynamic shared memory needs the opt-in (per device: kept per context)
                CK(cudaFuncSetAttribute(k_pt_backward_staged<CV, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)stage_bytes));
                CK(cudaFuncSetAttribute(k_pt_backward_staged<CV, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)stage_bytes));
                ctx->pt_stage_opted = true;
              }
              if (r == 0) k_pt_backward_staged<CV, true><<<grid, 128, stage_bytes, st>>>(ap.B[r], (uint32_t)total, in_cur, entries, offs_cur, offs_nxt, pt_pre, pt_accs, out);
              else k_pt_backward_staged<CV, false><<<grid, 128, stage_bytes, st>>>(ap.B[r], (uint32_t)total, in_cur, nullptr, offs_cur, offs_nxt, pt_pre, pt_accs, out);
            } else {
              if (r == 0) k_pt_backward<CV, true><<<grid, 128, 0, st>>>(ap.B[r], (uint32_t)total, in_cur, entries, offs_cur, offs_nxt, pt_pre, pt_accs, out);
              else k_pt_backward<CV, false><<<grid, 128, 0, st>>>(ap.B[r], (uint32_t)total, in_cur, nullptr, offs_cur, offs_nxt, pt_pre, pt_accs, out);
            }
            nl += 3;
          } else {
            if (r == 0) k_msm_pairtree_round<CV, true><<<grid, 128, 0, st>>>(ap.B[r], (uint32_t)total, in_cur, entries, offs_cur, offs_nxt, out);
            else k_msm_pairtree_round<CV, false><<<grid, 128, 0, st>>>(ap.B[r], (uint32_t)total, in_cur, nullptr, offs_cur, offs_nxt, out);
            nl += 1;
          }
          offs_cur = offs_nxt;
          in_cur = out;
        }
        CK(cudaEventRecord(ctx->ev[10], st));        // end of the rounds
        k_msm_accumulate_slices_direct<CV, slice_minb<CV>()><<<(sa + 127) / 128, 128, 0, st>>>(sa, La, (uint32_t)total, in_cur, offs_cur, buckets, spart);
        nl++;
        CK(cudaEventRecord(ctx->ev[9], st));
        k_msm_fixup<CV><<<(unsigned)((total + 127) / 128), 128, 0, st>>>((uint32_t)total, La, offs_cur, buckets, spart, big_count, big_list);
        k_msm_fixup_big<CV><<<256, 128, 0, st>>>(La, offs_cur, buckets, spart, big_count, big_list); nl += 2;
      }
    } else {
    CK(cudaEventRecord(ctx->ev[10], st));
    // slice_minb resident blocks per SM (above); b2k_set_msm_occupancy is ignored.
    k_msm_accumulate_slices<CV, slice_minb<CV>()><<<(smax + 127) / 128, 128, 0, st>>>(smax, L, (uint32_t)total, pts, offs, entries, buckets, spart);
    nl++;
    CK(cudaEventRecord(ctx->ev[9], st));
    k_msm_fixup<CV><<<(unsigned)((total + 127) / 128), 128, 0, st>>>((uint32_t)total, L, offs, buckets, spart, big_count, big_list);
    k_msm_fixup_big<CV><<<256, 128, 0, st>>>(L, offs, buckets, spart, big_count, big_list); nl += 2;
    }
  }
  CK(cudaEventRecord(ctx->ev[5], st));
  if (ext_buckets) {                       // the tail runs after the exchange (msm_reduce_windows_dev / msm_finish_dev)
    CK(cudaEventRecord(ctx->ev[6], st));
    CK(cudaEventRecord(ctx->ev[7], st));
    CK(cudaEventRecord(ctx->ev[8], st));
    CK(cudaGetLastError());
    ctx->launches += (uint64_t)nl;
    ctx->timings_valid = true;
    return B2K_OK;
  }
  if (rp.levels == 2) {
    const size_t n1 = (size_t)pl.W * rp.T1, n2 = (size_t)pl.W * (rp.T1 / rp.m2);
    k_msm_reduce_l1<CV><<<(unsigned)((n1 + 127) / 128), 128, 0, st>>>(pl.nb, rp.m1, rp.m2, pl.W, 1, buckets, partials, runs);
    k_msm_reduce_l2<CV><<<(unsigned)((n2 + 127) / 128), 128, 0, st>>>(pl.nb, rp.m1, rp.m2, rp.log2_m1, pl.W, runs, partials); nl += 2;
  } else {
    size_t nchunks = (size_t)pl.W * T;
    k_msm_reduce_chunks<CV><<<(unsigned)((nchunks + 127) / 128), 128, 0, st>>>(pl, buckets, partials); nl++;
  }
  CK(cudaEventRecord(ctx->ev[6], st));
  if (S > 1) {
    k_msm_window_sum<CV><<<pl.W * S, 128, 0, st>>>(rp.TP / S, partials, wpart);      // (w, s) -> wpart[w S + s]
    k_msm_window_sum<CV><<<pl.W, 128, 0, st>>>(S, wpart, wsum); nl += 2;
  } else {
    k_msm_window_sum<CV><<<pl.W, 128, 0, st>>>(rp.TP, partials, wsum); nl++;
  }
  CK(cudaEventRecord(ctx->ev[7], st));
  k_msm_final<CV><<<1, 128, 0, st>>>(pl, wsum, d_out, affine_out); nl++;
  CK(cudaEventRecord(ctx->ev[8], st));
  }
  CK(cudaGetLastError());
  ctx->launches += (uint64_t)nl;
  ctx->timings_valid = true;
  return B2K_OK;
}

// sorted-entry positions are 32-bit (offs[], cursor, entries, slice bounds): a problem whose pairs x windows reach 2^32 is refused
template <class CV>
inline bool msm_too_large(b2k_ctx* ctx, size_t n, const MsmPlan& pl) {
  if ((unsigned long long)msm_virtual_n<CV>(ctx, n) * (unsigned long long)pl.W < (1ull << 32)) return false;
  ctx->err = "MSM too large for one call: pairs x windows must stay below 2^32 (split the batch or use the sharded entry points)";
  return true;
}

template <class CV>
int msm_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points, void* d_out, int affine_out = 0) {
  if (!ctx || !d_scalars || !d_points || !d_out || n == 0 || n >= (size_t(1) << 31)) {
    if (ctx) ctx->err = "bad argument";
    return B2K_ERR_ARG;
  }
  CK(cudaSetDevice(ctx->device));
  MsmPlan pl = msm_plan<CV>(ctx, n);
  if (msm_too_large<CV>(ctx, n, pl)) return B2K_ERR_ARG;
  int rc = arena_reserve(ctx, msm_scratch_bytes<CV>(ctx, msm_virtual_n<CV>(ctx, n), pl));
  if (rc) return rc;
  return msm_enqueue<CV>(ctx, n, pl, (const uint8_t*)d_scalars, (const uint8_t*)d_points, (uint8_t*)d_out, affine_out);
}

// ---- multi-GPU bucket exchange (SURVEY 8e shape 1) ---------------------------------------------------------------------
// Three device-side steps around the two collectives the host issues (kyber_b200/multi.py: msm_bucket_exchange):
//   msm_buckets_dev        pairs of this rank -> its W x 2^(c-1) partial buckets (raw Xyzz limbs, Montgomery form)
//   [ncclAllToAll]         rank g receives windows [g W/G, (g+1) W/G) of every rank
//   msm_reduce_windows_dev sum of the G partials fused into the chunk reduction, then the window sums of these windows
//   [ncclAllGather]        W window sums (W x sizeof(Xyzz)) on every rank
//   msm_finish_dev         Horner over the windows, affine, wire bytes
// plan_out = {c, W, buckets per window, bytes per bucket}; every rank must run the same plan (same n class, same switches).
template <class CV>
int msm_buckets_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points, void* d_buckets, size_t cap_bytes, int* plan_out) {
  using X = Xyzz<typename CV::F>;
  if (!ctx || !d_scalars || !d_points || !d_buckets || n == 0 || n >= (size_t(1) << 31)) {
    if (ctx) ctx->err = "bad argument";
    return B2K_ERR_ARG;
  }
  CK(cudaSetDevice(ctx->device));
  MsmPlan pl = msm_plan<CV>(ctx, n);
  if (msm_too_large<CV>(ctx, n, pl)) return B2K_ERR_ARG;
  if (plan_out) { plan_out[0] = pl.c; plan_out[1] = pl.W; plan_out[2] = pl.nb; plan_out[3] = (int)sizeof(X); }
  if (cap_bytes < (size_t)pl.W * pl.nb * sizeof(X) || (reinterpret_cast<uintptr_t>(d_buckets) & 15)) {
    ctx->err = "bucket buffer too small or not 16-byte aligned";
    return B2K_ERR_ARG;
  }
  int rc = arena_reserve(ctx, msm_scratch_bytes<CV>(ctx, msm_virtual_n<CV>(ctx, n), pl));
  if (rc) return rc;
  return msm_enqueue<CV>(ctx, n, pl, (const uint8_t*)d_scalars, (const uint8_t*)d_points, nullptr, 0, reinterpret_cast<X*>(d_buckets));
}

// The same from HOST buffers (page-locked for the copies to overlap other contexts' kernels): the rank's shard is staged in the
// context's arena and the whole sequence is only enqueued.  Used by the sharded entry points of b2k_multi.cu.
template <class CV>
int msm_buckets_host(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, void* d_buckets, size_t cap_bytes, int* plan_out) {
  using X = Xyzz<typename CV::F>;
  if (!ctx || !scalars || !points || !d_buckets || n == 0 || n >= (size_t(1) << 31)) {
    if (ctx) ctx->err = "bad argument";
    return B2K_ERR_ARG;
  }
  CK(cudaSetDevice(ctx->device));
  MsmPlan pl = msm_plan<CV>(ctx, n);
  if (msm_too_large<CV>(ctx, n, pl)) return B2K_ERR_ARG;
  if (plan_out) { plan_out[0] = pl.c; plan_out[1] = pl.W; plan_out[2] = pl.nb; plan_out[3] = (int)sizeof(X); }
  if (cap_bytes < (size_t)pl.W * pl.nb * sizeof(X) || (reinterpret_cast<uintptr_t>(d_buckets) & 15)) {
    ctx->err = "bucket buffer too small or not 16-byte aligned";
    return B2K_ERR_ARG;
  }
  const size_t in_bytes = pad256(n * 32) + pad256(n * (size_t)CV::IN_BYTES) + 256;
  int rc = arena_reserve(ctx, msm_scratch_bytes<CV>(ctx, msm_virtual_n<CV>(ctx, n), pl) + in_bytes);
  if (rc) return rc;
  auto* d_s = arena_take<uint8_t>(ctx, n * 32);
  auto* d_p = arena_take<uint8_t>(ctx, n * (size_t)CV::IN_BYTES);
  CK(cudaMemcpyAsync(d_s, scalars, n * 32, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(d_p, points, n * (size_t)CV::IN_BYTES, cudaMemcpyHostToDevice, ctx->stream));
  return msm_enqueue<CV>(ctx, n, pl, d_s, d_p, nullptr, 0, reinterpret_cast<X*>(d_buckets));
}

// bucket-count query for sizing the exchange buffers before the first call
template <class CV>
int msm_bucket_plan(b2k_ctx* ctx, size_t n, int* plan_out) {
  if (!ctx || !plan_out || n == 0) return B2K_ERR_ARG;
  MsmPlan pl = msm_plan<CV>(ctx, n);
  plan_out[0] = pl.c; plan_out[1] = pl.W; plan_out[2] = pl.nb; plan_out[3] = (int)sizeof(Xyzz<typename CV::F>);
  return B2K_OK;
}

template <class CV>
int msm_reduce_windows_dev(b2k_ctx* ctx, int c, int w_cnt, int parts, const void* d_recv, void* d_wsum) {
  using X = Xyzz<typename CV::F>;
  if (!ctx || !d_recv || !d_wsum || c < 2 || c > 16 || w_cnt < 1 || w_cnt > 64 || parts < 1 || parts > 64) {
    if (ctx) ctx->err = "bad argument";
    return B2K_ERR_ARG;
  }
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const int nb = 1 << (c - 1);
  int m = 1;                                       // single-level chunk: keep >= 16k reduction threads for the few windows of one rank
  while (m < 64 && m * 2 <= nb && ((size_t)w_cnt * nb) / (size_t)(m * 2) >= 16384) m *= 2;
  if (ctx->force_m > 0 && ctx->force_m <= nb && (ctx->force_m & (ctx->force_m - 1)) == 0) m = ctx->force_m;
  const ReducePlan rp = reduce_plan(ctx, nb, m);
  const int S = window_sum_split(rp.TP);
  int rc = arena_reserve(ctx, pad256((size_t)w_cnt * rp.TP * sizeof(X)) + pad256((size_t)w_cnt * rp.T1 * sizeof(X)) +
                                  pad256((size_t)w_cnt * 128 * sizeof(X)) + 4096);
  if (rc) return rc;
  auto* partials = arena_take<X>(ctx, (size_t)w_cnt * rp.TP);
  auto* runs = arena_take<X>(ctx, (size_t)w_cnt * rp.T1);
  auto* wpart = arena_take<X>(ctx, (size_t)w_cnt * 128);
  if (!partials || !runs || !wpart) { ctx->err = "scratch arena too small"; return B2K_ERR_ARG; }
  const X* recv = reinterpret_cast<const X*>(d_recv);
  if (rp.levels == 2) {
    const size_t n1 = (size_t)w_cnt * rp.T1, n2 = (size_t)w_cnt * (rp.T1 / rp.m2);
    k_msm_reduce_l1<CV><<<(unsigned)((n1 + 127) / 128), 128, 0, st>>>(nb, rp.m1, rp.m2, w_cnt, parts, recv, partials, runs);
    k_msm_reduce_l2<CV><<<(unsigned)((n2 + 127) / 128), 128, 0, st>>>(nb, rp.m1, rp.m2, rp.log2_m1, w_cnt, runs, partials);
    ctx->launches += 2;
  } else {
    const size_t nchunks = (size_t)w_cnt * rp.T1;
    k_msm_reduce_chunks_parts<CV><<<(unsigned)((nchunks + 127) / 128), 128, 0, st>>>(nb, m, w_cnt, parts, recv, partials);
    ctx->launches += 1;
  }
  if (S > 1) {
    k_msm_window_sum<CV><<<w_cnt * S, 128, 0, st>>>(rp.TP / S, partials, wpart);
    k_msm_window_sum<CV><<<w_cnt, 128, 0, st>>>(S, wpart, reinterpret_cast<X*>(d_wsum));
    ctx->launches += 2;
  } else {
    k_msm_window_sum<CV><<<w_cnt, 128, 0, st>>>(rp.TP, partials, reinterpret_cast<X*>(d_wsum));
    ctx->launches += 1;
  }
  CK(cudaGetLastError());
  return B2K_OK;
}

template <class CV>
int msm_finish_dev(b2k_ctx* ctx, int c, int W, const void* d_wsum, void* d_out, int affine_out) {
  using X = Xyzz<typename CV::F>;
  if (!ctx || !d_wsum || !d_out || c < 2 || c > 16 || W < 1 || W > 128) {
    if (ctx) ctx->err = "bad argument";
    return B2K_ERR_ARG;
  }
  CK(cudaSetDevice(ctx->device));
  MsmPlan pl;
  memset(&pl, 0, sizeof pl);
  pl.c = c; pl.W = W; pl.nb = 1 << (c - 1); pl.m = 1;
  k_msm_final<CV><<<1, 128, 0, ctx->stream>>>(pl, reinterpret_cast<const X*>(d_wsum), (uint8_t*)d_out, affine_out);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return B2K_OK;
}

// the context's copy stream (created on first use; nullptr if that fails: the caller copies on the main stream instead)
inline cudaStream_t copy_stream(b2k_ctx* ctx) {
  if (!ctx->copy_stream && cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); ctx->copy_stream = nullptr; }
  return ctx->copy_stream;
}

// Host-buffer MSM.  wait = false: everything (H2D copies, pipeline, D2H of the result and of the status word) is only
// ENQUEUED on the context's stream; the caller collects the status with msm_wait() (b2k_wait).  With page-locked host
// buffers the copies of one context overlap the kernels of another: two contexts alternate to keep PCIe and the SMs busy.
template <class CV>
int msm_host(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out, int affine_out = 0, bool wait = true) {
  if (!ctx || !scalars || !points || !out || n == 0 || n >= (size_t(1) << 31)) {
    if (ctx) ctx->err = "bad argument";
    return B2K_ERR_ARG;
  }
  CK(cudaSetDevice(ctx->device));
  MsmPlan pl = msm_plan<CV>(ctx, n);
  if (msm_too_large<CV>(ctx, n, pl)) return B2K_ERR_ARG;
  size_t in_bytes = pad256(n * 32) + pad256(n * (size_t)CV::IN_BYTES) + 256;
  int rc = arena_reserve(ctx, msm_scratch_bytes<CV>(ctx, msm_virtual_n<CV>(ctx, n), pl) + in_bytes);
  if (rc) return rc;
  auto* d_s = arena_take<uint8_t>(ctx, n * 32);
  auto* d_p = arena_take<uint8_t>(ctx, n * (size_t)CV::IN_BYTES);
  auto* d_o = arena_take<uint8_t>(ctx, 256);
  CK(cudaMemsetAsync(ctx->d_flags, 0, 4, ctx->stream));
  // Large G1 batches: the H2D copy goes in 8 chunks on its own stream and the front end (k_glv_prepare: range and curve checks, the
  // endomorphism split, 8 field products per pair) runs chunk by chunk under it -- a blocking call no longer holds every kernel back until the
  // last byte has arrived (VERDICT r1 weak 6).  gev[0] orders the copies behind whatever still reads the arena, gev[1..8] hand the chunks over.
  const bool chunked = msm_uses_glv<CV>(ctx, n) && ctx->msm_groups <= 1 && n >= (size_t(1) << 18) && copy_stream(ctx);
  if (chunked) {
    constexpr int K = 8;
    const size_t per = (n + K - 1) / K;
    CK(cudaEventRecord(ctx->gev[0], ctx->stream));
    CK(cudaStreamWaitEvent(ctx->copy_stream, ctx->gev[0], 0));
    for (int k = 0; k < K; k++) {
      const size_t i0 = (size_t)k * per;
      const size_t cnt = i0 >= n ? 0 : ((n - i0 < per) ? n - i0 : per);
      if (cnt) {
        CK(cudaMemcpyAsync(d_s + 32 * i0, scalars + 32 * i0, cnt * 32, cudaMemcpyHostToDevice, ctx->copy_stream));
        CK(cudaMemcpyAsync(d_p + (size_t)CV::IN_BYTES * i0, points + (size_t)CV::IN_BYTES * i0, cnt * (size_t)CV::IN_BYTES, cudaMemcpyHostToDevice, ctx->copy_stream));
      }
      CK(cudaEventRecord(ctx->gev[1 + k], ctx->copy_stream));
    }
    ctx->h2d_chunks = K;
  } else {
    CK(cudaMemcpyAsync(d_s, scalars, n * 32, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_p, points, n * (size_t)CV::IN_BYTES, cudaMemcpyHostToDevice, ctx->stream));
  }
  rc = msm_enqueue<CV>(ctx, n, pl, d_s, d_p, d_o, affine_out);
  ctx->h2d_chunks = 0;
  if (rc) return rc;
  CK(cudaMemcpyAsync(out, d_o, affine_out ? CV::IN_BYTES : CV::OUT_BYTES, cudaMemcpyDeviceToHost, ctx->stream));
  if (!wait) { CK(cudaMemcpyAsync(ctx->h_flags, ctx->d_flags, 4, cudaMemcpyDeviceToHost, ctx->stream)); return B2K_OK; }   // b2k_wait fetches + clears
  return status_finish(ctx);
}

// Also the status query of the *_dev entry points, which only enqueue: the device status word (scalar range, malformed
// point) is sticky across them, fetched and cleared here.
inline int msm_wait(b2k_ctx* ctx) {
  if (!ctx) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  CK(cudaMemcpyAsync(ctx->h_flags, ctx->d_flags, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemsetAsync(ctx->d_flags, 0, 4, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return check_flags(ctx);
}

template <class CV, bool AFF>
int mul_batch_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points, void* d_out) {
  if (!ctx || !d_scalars || !d_points || !d_out || n == 0) {
    if (ctx) ctx->err = "bad argument";
    return B2K_ERR_ARG;
  }
  CK(cudaSetDevice(ctx->device));
  const unsigned grid = (unsigned)((n + 127) / 128);
  // (the 3- and 4-blocks-per-SM variants of the G1 kernel measured slower than the compiler's own register allocation,
  //  and tripled the build time of this translation unit: removed; b2k_set_mul_occupancy
  //  is accepted and ignored)
  k_mul_batch<CV, AFF><<<grid, 128, 0, ctx->stream>>>(
      n, (const uint8_t*)d_scalars, (const uint8_t*)d_points, (uint8_t*)d_out, ctx->d_flags, ctx->use_glv);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return B2K_OK;
}

template <class CV, bool AFF>
int mul_batch_host(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out) {
  if (!ctx || !scalars || !points || !out || n == 0) {
    if (ctx) ctx->err = "bad argument";
    return B2K_ERR_ARG;
  }
  CK(cudaSetDevice(ctx->device));
  const size_t ob = AFF ? (size_t)CV::IN_BYTES : (size_t)CV::OUT_BYTES;
  size_t bytes = pad256(n * 32) + pad256(n * (size_t)CV::IN_BYTES) + pad256(n * ob) + 1024;
  int rc = arena_reserve(ctx, bytes);
  if (rc) return rc;
  auto* d_s = arena_take<uint8_t>(ctx, n * 32);
  auto* d_p = arena_take<uint8_t>(ctx, n * (size_t)CV::IN_BYTES);
  auto* d_o = arena_take<uint8_t>(ctx, n * ob);
  CK(cudaMemsetAsync(ctx->d_flags, 0, 4, ctx->stream));
  CK(cudaMemcpyAsync(d_s, scalars, n * 32, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(d_p, points, n * (size_t)CV::IN_BYTES, cudaMemcpyHostToDevice, ctx->stream));
  rc = mul_batch_dev<CV, AFF>(ctx, n, d_s, d_p, d_o);
  if (rc) return rc;
  CK(cudaMemcpyAsync(out, d_o, n * ob, cudaMemcpyDeviceToHost, ctx->stream));
  return status_finish(ctx);
}


}  // namespace b2k_host
