// msm_host.cuh -- host-side launch templates shared by the translation units of libb2kyber.so
// (plan selection, scratch layout, stage timing, enqueue of the MSM pipeline and of mul_batch).
#pragma once
#include "host_call.cuh"
#include "kernels.cuh"

namespace b2k_host {
using namespace b2k;
constexpr int N_EV = B2K_N_EV;

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

// scratch of the bucket reduction of w_cnt windows: tp chunk partials per window, the level-1 run sums, the window-sum sub-blocks
template <class X>
struct TailBufs {
  X* partials = nullptr;
  X* runs = nullptr;
  X* wpart = nullptr;
  void carve(Carve& c, size_t w_cnt, size_t tp, const ReducePlan& rp) {
    partials = c.take<X>(w_cnt * tp);
    runs = c.take<X>(w_cnt * (size_t)rp.T1);
    wpart = c.take<X>(w_cnt * 128);
  }
};

// reduction plan of the w_cnt windows one rank owns after a bucket exchange: the single-level chunk keeps >= 16k reduction
// threads for these few windows (b2k_set_msm_chunk still forces it)
inline ReducePlan owned_reduce_plan(const b2k_ctx* ctx, int nb, int w_cnt) {
  int m = 1;
  while (m < 64 && m * 2 <= nb && ((size_t)w_cnt * nb) / (size_t)(m * 2) >= 16384) m *= 2;
  if (ctx->force_m > 0 && ctx->force_m <= nb && (ctx->force_m & (ctx->force_m - 1)) == 0) m = ctx->force_m;
  return reduce_plan(ctx, nb, m);
}

// The bucket-reduction tail of w_cnt windows of nb buckets into wsum: level 1, level 2 if rp has two levels, then the window
// sums in one pass or as S sub-blocks and their sum.  The callers reduce different bucket sources (local buckets, received
// parts, peer memory), so level1(grid) launches level 1 itself: one thread per level-1 chunk, 128 per block, on ctx->stream.
// levels_done, if given, is recorded between the levels and the window sum.
template <class CV, class Level1>
int reduce_windows(b2k_ctx* ctx, int nb, int w_cnt, const ReducePlan& rp, const TailBufs<Xyzz<typename CV::F>>& t,
                   Xyzz<typename CV::F>* wsum, Level1&& level1, cudaEvent_t levels_done = nullptr) {
  cudaStream_t st = ctx->stream;
  level1((unsigned)(((size_t)w_cnt * rp.T1 + 127) / 128));
  if (rp.levels == 2) {
    const size_t n2 = (size_t)w_cnt * (rp.T1 / rp.m2);
    k_msm_reduce_l2<CV><<<(unsigned)((n2 + 127) / 128), 128, 0, st>>>(nb, rp.m1, rp.m2, rp.log2_m1, w_cnt, t.runs, t.partials);
  }
  if (levels_done) CK(cudaEventRecord(levels_done, st));
  const int S = window_sum_split(rp.TP);
  if (S > 1) {
    k_msm_window_sum<CV><<<w_cnt * S, 128, 0, st>>>(rp.TP / S, t.partials, t.wpart);      // (w, s) -> wpart[w S + s]
    k_msm_window_sum<CV><<<w_cnt, 128, 0, st>>>(S, t.wpart, wsum);
  } else {
    k_msm_window_sum<CV><<<w_cnt, 128, 0, st>>>(rp.TP, t.partials, wsum);
  }
  ctx->launches += rp.levels + (S > 1 ? 2 : 1);
  return B2K_OK;
}

// ---- one MSM call: plan, the sizes derived from it, and its scratch ---------------------------------------------------------
template <class CV>
struct MsmLayout {
  using F = typename CV::F;
  using X = Xyzz<F>;
  MsmPlan pl;
  bool glv = false;
  size_t n_in = 0, n = 0;        // pairs of the call; pairs the digit / sort / accumulate stages see (msm_virtual_n)
  size_t total = 0;              // W x buckets per window
  ReducePlan rp;
  AffinePlan ap;
  uint32_t L = 0, smax = 0;      // slice length and slice count of the pairs
  uint32_t La = 0, sa = 0;       // the same after the affine rounds (La = L without rounds)
  bool split = false;            // affine rounds as three kernels (b2k_set_msm_affine_split)

  Affine<F>* pts = nullptr;
  int16_t* digits = nullptr;     // digit columns, window-major
  uint32_t *counts = nullptr, *offs = nullptr, *cursor = nullptr;
  SortRec* recs = nullptr;       // coarse-partitioned (entry, bucket) records of the bucket sort
  uint32_t* entries = nullptr;
  X* buckets = nullptr;
  TailBufs<X> tail;
  X* wsum = nullptr;
  X* spart = nullptr;            // slice partials
  uint32_t* big_list = nullptr;
  uint32_t* bsum = nullptr;      // block sums of the scan, 1024 words per scanned column
  uint32_t* offs_rt = nullptr;   // bucket offsets after round r + 1: offs_rt + r (total + 1), written by the scan (columns 1..R)
  Affine<F>* aff_rt[2] = {nullptr, nullptr};
  F* pt_pre = nullptr;           // split rounds: prefix products and per-thread accumulators
  F* pt_accs = nullptr;

  void carve(Carve& c) {
    pts = c.take<Affine<F>>(n);
    digits = c.take<int16_t>(n * (size_t)pl.W);
    counts = c.take<uint32_t>(total + 1);
    offs = c.take<uint32_t>(total + 1);
    cursor = c.take<uint32_t>(total + 1);
    recs = c.take<SortRec>(n * (size_t)pl.W);
    entries = c.take<uint32_t>(n * (size_t)pl.W);
    buckets = c.take<X>(total);
    const size_t T = pl.nb / pl.m;         // the grouped tail reduces single-level chunks whatever rp says
    tail.carve(c, pl.W, rp.TP > T ? rp.TP : T, rp);
    wsum = c.take<X>(pl.W);
    spart = c.take<X>(2 * (size_t)(sa > smax ? sa : smax));
    big_list = c.take<uint32_t>(total + 1);
    bsum = c.take<uint32_t>(1024 * (size_t)(1 + ap.R));
    if (ap.R > 0) {
      offs_rt = c.take<uint32_t>((size_t)ap.R * (total + 1));
      aff_rt[0] = c.take<Affine<F>>(ap.bound[1]);
      if (ap.R > 1) aff_rt[1] = c.take<Affine<F>>(ap.bound[2]);
      if (split) {
        pt_pre = c.take<F>(ap.pre_elems);
        pt_accs = c.take<F>(ap.max_T);
      }
    }
  }
};

template <class CV>
MsmLayout<CV> msm_layout(const b2k_ctx* ctx, size_t n_in) {
  MsmLayout<CV> s;
  s.pl = msm_plan<CV>(ctx, n_in);
  s.glv = msm_uses_glv<CV>(ctx, n_in);
  s.n_in = n_in;
  s.n = msm_virtual_n<CV>(ctx, n_in);
  s.total = (size_t)s.pl.W * s.pl.nb;
  s.rp = reduce_plan(ctx, s.pl.nb, s.pl.m);
  s.ap = affine_plan<CV>(ctx, s.n, s.pl);
  s.split = ctx->affine_split != 0;
  s.L = slice_len(s.n, s.pl, ctx->force_L);
  s.smax = (uint32_t)((s.n * (size_t)s.pl.W + s.L - 1) / s.L) + 1;
  s.La = s.ap.R > 0 ? slice_len_entries(s.ap.bound[s.ap.R], ctx->force_L) : s.L;
  s.sa = s.ap.R > 0 ? (uint32_t)((s.ap.bound[s.ap.R] + s.La - 1) / s.La) + 1 : 0;
  return s;
}

// The prologue of every MSM entry point: argument and size checks, device, plan, and one reservation of the arena for the
// call's staged inputs (stage(Carve&) takes them, in front of the scratch) and the pipeline's scratch.  args_ok: the caller's
// pointer arguments are usable.
template <class CV, class Stage>
int msm_begin(b2k_ctx* ctx, size_t n, bool args_ok, MsmLayout<CV>& s, Stage&& stage) {
  if (!ctx || !args_ok || n == 0 || n >= (size_t(1) << 31)) {
    if (ctx) ctx->err = "bad argument";
    return B2K_ERR_ARG;
  }
  CK(cudaSetDevice(ctx->device));
  s = msm_layout<CV>(ctx, n);
  // sorted-entry positions are 32-bit (offs[], cursor, entries, slice bounds): a problem whose pairs x windows reach 2^32 is refused
  if ((unsigned long long)s.n * (unsigned long long)s.pl.W >= (1ull << 32)) {
    ctx->err = "MSM too large for one call: pairs x windows must stay below 2^32 (split the batch or use the sharded entry points)";
    return B2K_ERR_ARG;
  }
  if (s.total > 1024u * 1024u || (s.pl.nb >> sort_shift(s.pl.c)) > PART_BPW) { ctx->err = "too many buckets"; return B2K_ERR_ARG; }
  return arena_carve(ctx, [&](Carve& c) {
    stage(c);
    s.carve(c);
  });
}

// ---- stages of the pipeline -----------------------------------------------------------------------------------------------
// front end: load (digits and bucket histogram), scan of the bucket offsets, partition and bin sort of the entries
template <class CV>
int msm_front(b2k_ctx* ctx, const MsmLayout<CV>& s, const uint8_t* d_scalars_in, const uint8_t* d_points) {
  cudaStream_t st = ctx->stream;
  const MsmPlan& pl = s.pl;
  const size_t n = s.n, n_in = s.n_in, total = s.total;
  const unsigned sblocks = (unsigned)((total + 1023) / 1024);
  CK(cudaEventRecord(ctx->ev[0], st));
  CK(cudaMemsetAsync(s.counts, 0, (total + 1) * 4, st));
  if (ctx->h2d_chunks > 1 && !s.glv) CK(cudaStreamWaitEvent(st, ctx->gev[ctx->h2d_chunks], 0));   // (not reached: msm_host chunks GLV calls only)
  if (!s.glv) {
    k_msm_load<CV><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, d_scalars_in, d_points, s.pts, pl, s.digits, s.counts, ctx->d_flags);
  } else if constexpr (GlvTraits<CV>::enabled) {
    // host-buffer call with h2d_chunks > 1: the inputs arrive in chunks on the copy stream (msm_host); every chunk is prepared as
    // soon as it has landed, so that only the last chunk's front-end work is left when the copy ends
    const int K = ctx->h2d_chunks > 1 ? ctx->h2d_chunks : 1;
    const size_t per = (n_in + K - 1) / K;
    for (int k = 0; k < K; k++) {
      const size_t i0 = (size_t)k * per;
      if (i0 >= n_in) break;
      const size_t cnt = (n_in - i0 < per) ? n_in - i0 : per;
      if (K > 1) CK(cudaStreamWaitEvent(st, ctx->gev[1 + k], 0));
      k_glv_prepare_bls381<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(n_in, i0, cnt, d_scalars_in, d_points, s.pts, pl, s.digits, s.counts, ctx->d_flags);
    }
  }
  CK(cudaEventRecord(ctx->ev[1], st));             // the digits and the histogram come out of the load pass: ev[1..2] is empty
  CK(cudaEventRecord(ctx->ev[2], st));
  const dim3 cols(sblocks, 1 + s.ap.R), tops(1, 1 + s.ap.R);     // the histogram + the bucket sizes after each affine round
  k_scan_blocks<<<cols, 1024, 0, st>>>((uint32_t)total, s.counts, s.offs, s.offs_rt, s.bsum);
  k_scan_tops<<<tops, 1024, 0, st>>>(sblocks, (uint32_t)total, s.bsum, s.offs, s.offs_rt);
  k_scan_finish<<<cols, 1024, 0, st>>>((uint32_t)total, s.bsum, s.offs, s.offs_rt, s.cursor);
  CK(cudaEventRecord(ctx->ev[3], st));
  const int S = sort_shift(pl.c);
  const size_t nrec = n * (size_t)pl.W;
  k_msm_partition<<<(unsigned)((n + PART_TILE - 1) / PART_TILE), PART_T, 0, st>>>((uint32_t)n, pl, S, s.digits, s.cursor, s.recs);
  k_msm_bin_sort<<<(unsigned)((nrec + BSORT_TILE - 1) / BSORT_TILE), BSORT_T, 0, st>>>((uint32_t)total, S, s.recs, s.offs, s.counts, s.entries);
  ctx->launches += 6;                              // load (the chunked prepare counts once), three scan passes, partition, bin sort
  return B2K_OK;
}

// one affine pair-tree round: the operands of every bucket (offsets offs_cur) are added in pairs into out (offsets offs_nxt);
// round 0 (FIRST) gathers its operands through the sorted entries
template <class CV, bool FIRST>
int affine_round(b2k_ctx* ctx, const MsmLayout<CV>& s, int r, const Affine<typename CV::F>* in, const uint32_t* offs_cur,
                 const uint32_t* offs_nxt, Affine<typename CV::F>* out) {
  using F = typename CV::F;
  cudaStream_t st = ctx->stream;
  const uint32_t B = s.ap.B[r], total = (uint32_t)s.total;
  const unsigned grid = s.ap.T[r] / 128;
  const uint32_t* entries = FIRST ? s.entries : nullptr;
  ctx->launches += s.split ? 3 : 1;
  if (!s.split) {
    k_msm_pairtree_round<CV, FIRST><<<grid, 128, 0, st>>>(B, total, in, entries, offs_cur, offs_nxt, out);
    return B2K_OK;
  }
  constexpr size_t fstage_bytes = 128 * 4 * sizeof(F);              // two 2-coordinate buffers per thread (24 KB for G1)
  if (fstage_bytes <= 48 * 1024 && ((ctx->pt_stage >> (FIRST ? 2 : 3)) & 1))
    k_pt_forward_staged<CV, FIRST><<<grid, 128, fstage_bytes, st>>>(B, total, in, entries, offs_cur, offs_nxt, s.pt_pre, s.pt_accs);
  else
    k_pt_forward<CV, FIRST><<<grid, 128, 0, st>>>(B, total, in, entries, offs_cur, offs_nxt, s.pt_pre, s.pt_accs);
  if (ctx->acc_minb == 5) k_pt_invert<F, 5><<<grid, 128, 0, st>>>(B, total, offs_nxt, s.pt_accs);
  else k_pt_invert<F, 4><<<grid, 128, 0, st>>>(B, total, offs_nxt, s.pt_accs);
  constexpr size_t stage_bytes = 128 * (4 * sizeof(Affine<F>) + sizeof(F));   // per thread two 2-point buffers + one prefix product (54 KB for G1)
  if (stage_bytes <= 56 * 1024 && ((ctx->pt_stage >> (FIRST ? 0 : 1)) & 1)) {
    if (!ctx->pt_stage_opted) {                     // more than 48 KB of dynamic shared memory needs the opt-in (per device: kept per context)
      CK(cudaFuncSetAttribute(k_pt_backward_staged<CV, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)stage_bytes));
      CK(cudaFuncSetAttribute(k_pt_backward_staged<CV, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)stage_bytes));
      ctx->pt_stage_opted = true;
    }
    k_pt_backward_staged<CV, FIRST><<<grid, 128, stage_bytes, st>>>(B, total, in, entries, offs_cur, offs_nxt, s.pt_pre, s.pt_accs, out);
  } else {
    k_pt_backward<CV, FIRST><<<grid, 128, 0, st>>>(B, total, in, entries, offs_cur, offs_nxt, s.pt_pre, s.pt_accs, out);
  }
  return B2K_OK;
}

// accumulate into buckets: one thread per bucket (b2k_set_msm_variant), or the slices (after the affine rounds if the plan has
// them) and the fix-up of the buckets they cut
template <class CV>
int msm_accumulate(b2k_ctx* ctx, const MsmLayout<CV>& s, Xyzz<typename CV::F>* buckets) {
  cudaStream_t st = ctx->stream;
  const uint32_t total = (uint32_t)s.total;
  if (ctx->use_v1) {
    CK(cudaEventRecord(ctx->ev[4], st));
    CK(cudaEventRecord(ctx->ev[10], st));
    k_msm_accumulate<CV><<<(total + 127) / 128, 128, 0, st>>>(s.total, s.pts, s.offs, s.entries, buckets);
    ctx->launches += 1;
    CK(cudaEventRecord(ctx->ev[9], st));
    return B2K_OK;
  }
  uint32_t* big_count = s.bsum + 1023;      // last word of the block-sum page is never a block sum (<= 1023 blocks used)
  CK(cudaMemsetAsync(buckets, 0, s.total * sizeof(Xyzz<typename CV::F>), st));
  CK(cudaMemsetAsync(big_count, 0, 4, st));
  CK(cudaEventRecord(ctx->ev[4], st));
  const uint32_t* offs = s.offs;             // bucket offsets of what the slices add up
  if (s.ap.R > 0) {
    if constexpr (AffineTraits<CV>::enabled) {
      // affine pair-tree rounds: operands of every bucket halve per round; the slices below finish the rest
      const Affine<typename CV::F>* in = s.pts;
      for (int r = 0; r < s.ap.R; r++) {
        const uint32_t* offs_nxt = s.offs_rt + (size_t)r * (s.total + 1);
        auto* out = s.aff_rt[r & 1];
        int rc = r == 0 ? affine_round<CV, true>(ctx, s, r, in, offs, offs_nxt, out) : affine_round<CV, false>(ctx, s, r, in, offs, offs_nxt, out);
        if (rc) return rc;
        offs = offs_nxt;
        in = out;
      }
      CK(cudaEventRecord(ctx->ev[10], st));        // end of the rounds
      k_msm_accumulate_slices_direct<CV, slice_minb<CV>()><<<(s.sa + 127) / 128, 128, 0, st>>>(s.sa, s.La, total, in, offs, buckets, s.spart);
    }
  } else {
    CK(cudaEventRecord(ctx->ev[10], st));
    // slice_minb resident blocks per SM (above); b2k_set_msm_occupancy is ignored.
    k_msm_accumulate_slices<CV, slice_minb<CV>()><<<(s.smax + 127) / 128, 128, 0, st>>>(s.smax, s.L, total, s.pts, s.offs, s.entries, buckets, s.spart);
  }
  CK(cudaEventRecord(ctx->ev[9], st));
  k_msm_fixup<CV><<<(total + 127) / 128, 128, 0, st>>>(total, s.La, offs, buckets, s.spart, big_count, s.big_list);
  k_msm_fixup_big<CV><<<256, 128, 0, st>>>(s.La, offs, buckets, s.spart, big_count, s.big_list);
  ctx->launches += 3;                        // the slices and the two fix-ups
  return B2K_OK;
}

// overlapped tail (b2k_set_msm_groups): groups of windows, top group first; reduction of group g on stream2 while the main
// stream accumulates group g-1.  ms[4] = all accumulate launches, ms[5] = what is left after them.
template <class CV>
int msm_grouped(b2k_ctx* ctx, const MsmLayout<CV>& s, int G, uint8_t* d_out, int affine_out) {
  cudaStream_t st = ctx->stream, s2 = ctx->stream2;
  const MsmPlan& pl = s.pl;
  const int T = pl.nb / pl.m;
  uint32_t* ranges = s.bsum + 900;                 // G+1 words
  uint32_t* bigc = s.bsum + 920;                   // one counter per group
  CK(cudaMemsetAsync(s.buckets, 0, s.total * sizeof(Xyzz<typename CV::F>), st));
  CK(cudaMemsetAsync(bigc, 0, 64, st));
  k_msm_group_ranges<<<1, 32, 0, st>>>(G, pl.W, pl.nb, s.L, (uint32_t)s.total, s.offs, ranges);
  ctx->launches += 1;
  CK(cudaEventRecord(ctx->ev[4], st));
  CK(cudaEventRecord(ctx->ev[10], st));
  for (int g = G - 1; g >= 0; g--) {
    const int w_lo = g * pl.W / G, w_hi = (g + 1) * pl.W / G, w_cnt = w_hi - w_lo;
    k_msm_accumulate_slices_range<CV><<<(s.smax + 127) / 128, 128, 0, st>>>(ranges, g, s.L, (uint32_t)s.total, s.pts, s.offs, s.entries, s.buckets, s.spart);
    CK(cudaEventRecord(ctx->gev[g], st));
    CK(cudaStreamWaitEvent(s2, ctx->gev[g], 0));
    const uint32_t gid_lo = (uint32_t)((size_t)w_lo * pl.nb), gid_hi = (uint32_t)((size_t)w_hi * pl.nb);
    k_msm_fixup_range<CV><<<(gid_hi - gid_lo + 127) / 128, 128, 0, s2>>>(gid_lo, gid_hi, s.L, s.offs, s.buckets, s.spart, bigc + g, s.big_list + gid_lo);
    k_msm_fixup_big<CV><<<64, 128, 0, s2>>>(s.L, s.offs, s.buckets, s.spart, bigc + g, s.big_list + gid_lo);
    size_t nch = (size_t)w_cnt * T;
    k_msm_reduce_chunks_range<CV><<<(unsigned)((nch + 127) / 128), 128, 0, s2>>>(pl, w_lo, w_cnt, s.buckets, s.tail.partials);
    k_msm_window_sum<CV><<<w_cnt, 128, 0, s2>>>(T, s.tail.partials, s.wsum, w_lo);
    ctx->launches += 5;
  }
  CK(cudaEventRecord(ctx->ev[9], st));           // end of the accumulate launches
  CK(cudaEventRecord(ctx->gev[G], s2));
  CK(cudaStreamWaitEvent(st, ctx->gev[G], 0));
  for (int e = 5; e <= 7; e++) CK(cudaEventRecord(ctx->ev[e], st));
  k_msm_final<CV><<<1, 128, 0, st>>>(pl, s.wsum, d_out, affine_out);
  ctx->launches += 1;
  CK(cudaEventRecord(ctx->ev[8], st));
  return B2K_OK;
}

// Enqueue the whole MSM on ctx->stream into the scratch msm_begin carved. d_scalars/d_points/d_out are device pointers.
// ext_buckets (bucket exchange, multi-GPU shape 1): the pipeline stops after the fix-up and leaves the W x 2^(c-1) buckets there.
template <class CV>
int msm_enqueue(b2k_ctx* ctx, const MsmLayout<CV>& s, const uint8_t* d_scalars, const uint8_t* d_points, uint8_t* d_out,
                int affine_out = 0, Xyzz<typename CV::F>* ext_buckets = nullptr) {
  cudaStream_t st = ctx->stream;
  const MsmPlan& pl = s.pl;
  auto* buckets = ext_buckets ? ext_buckets : s.buckets;
  int* lp = ctx->last_plan;                // what b2k_last_msm_plan reports
  lp[LP_C] = pl.c; lp[LP_W] = pl.W; lp[LP_NB] = pl.nb; lp[LP_M] = pl.m;
  lp[LP_SLICE] = (int)s.La;
  lp[LP_ROUNDS] = s.ap.R;
  for (int r = 0; r < PT_MAX_ROUNDS; r++) lp[LP_BATCH + r] = r < s.ap.R ? (int)s.ap.B[r] : 0;
  lp[LP_GLV] = s.glv ? 1 : 0;
  lp[LP_SPLIT] = (s.ap.R > 0 && s.split) ? 1 : 0;
  lp[LP_LEVELS] = s.rp.levels; lp[LP_M1] = s.rp.m1; lp[LP_M2] = s.rp.levels == 2 ? s.rp.m2 : 0;
  int rc = msm_front<CV>(ctx, s, d_scalars, d_points);
  if (rc) return rc;
  const int G = (!ext_buckets && !ctx->use_v1 && ctx->msm_groups > 1 && pl.W >= 2 * ctx->msm_groups && ctx->stream2) ? ctx->msm_groups : 1;
  if (G > 1) {
    rc = msm_grouped<CV>(ctx, s, G, d_out, affine_out);
    if (rc) return rc;
  } else {
    rc = msm_accumulate<CV>(ctx, s, buckets);
    if (rc) return rc;
    CK(cudaEventRecord(ctx->ev[5], st));
    if (ext_buckets) {                       // the tail runs after the exchange (msm_reduce_windows_dev / msm_finish_dev)
      for (int e = 6; e <= 8; e++) CK(cudaEventRecord(ctx->ev[e], st));
    } else {
      const ReducePlan& rp = s.rp;
      const auto& t = s.tail;
      rc = reduce_windows<CV>(ctx, pl.nb, pl.W, rp, t, s.wsum, [&](unsigned grid) {
        if (rp.levels == 2) k_msm_reduce_l1<CV><<<grid, 128, 0, st>>>(pl.nb, rp.m1, rp.m2, pl.W, 1, buckets, t.partials, t.runs);
        else k_msm_reduce_chunks<CV><<<grid, 128, 0, st>>>(pl, buckets, t.partials);
      }, ctx->ev[6]);
      if (rc) return rc;
      CK(cudaEventRecord(ctx->ev[7], st));
      k_msm_final<CV><<<1, 128, 0, st>>>(pl, s.wsum, d_out, affine_out);
      ctx->launches += 1;
      CK(cudaEventRecord(ctx->ev[8], st));
    }
  }
  CK(cudaGetLastError());
  ctx->timings_valid = true;
  return B2K_OK;
}

template <class CV>
int msm_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points, void* d_out, int affine_out = 0) {
  MsmLayout<CV> s;
  int rc = msm_begin<CV>(ctx, n, d_scalars && d_points && d_out, s, [](Carve&) {});
  if (rc) return rc;
  return msm_enqueue<CV>(ctx, s, (const uint8_t*)d_scalars, (const uint8_t*)d_points, (uint8_t*)d_out, affine_out);
}

// ---- multi-GPU bucket exchange (SURVEY 8e shape 1) ---------------------------------------------------------------------
// Three device-side steps around the two collectives the host issues (kyber_b200/multi.py: msm_bucket_exchange):
//   msm_buckets            pairs of this rank -> its W x 2^(c-1) partial buckets (raw Xyzz limbs, Montgomery form)
//   [ncclAllToAll]         rank g receives windows [g W/G, (g+1) W/G) of every rank
//   msm_reduce_windows_dev sum of the G partials fused into the chunk reduction, then the window sums of these windows
//   [ncclAllGather]        W window sums (W x sizeof(Xyzz)) on every rank
//   msm_finish_dev         Horner over the windows, affine, wire bytes
// plan_out = {c, W, buckets per window, bytes per bucket}; every rank must run the same plan (same n class, same switches).
// host = false: scalars / points are device pointers.  host = true: they are HOST buffers (page-locked for the copies to
// overlap other contexts' kernels), staged in the context's arena, and the whole sequence is only enqueued (the sharded entry
// points of b2k_multi.cu).
template <class CV>
int msm_buckets(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, bool host, void* d_buckets, size_t cap_bytes,
                int* plan_out) {
  using X = Xyzz<typename CV::F>;
  MsmLayout<CV> s;
  uint8_t *d_s = nullptr, *d_p = nullptr;        // host: the staged copies
  int rc = msm_begin<CV>(ctx, n, scalars && points && d_buckets, s, [&](Carve& c) {
    if (!host) return;
    d_s = c.take<uint8_t>(n * 32);
    d_p = c.take<uint8_t>(n * (size_t)CV::IN_BYTES);
  });
  if (rc) return rc;
  const MsmPlan& pl = s.pl;
  if (plan_out) { plan_out[0] = pl.c; plan_out[1] = pl.W; plan_out[2] = pl.nb; plan_out[3] = (int)sizeof(X); }
  if (cap_bytes < (size_t)pl.W * pl.nb * sizeof(X) || (reinterpret_cast<uintptr_t>(d_buckets) & 15)) {
    ctx->err = "bucket buffer too small or not 16-byte aligned";
    return B2K_ERR_ARG;
  }
  if (host) {
    CK(cudaMemcpyAsync(d_s, scalars, n * 32, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_p, points, n * (size_t)CV::IN_BYTES, cudaMemcpyHostToDevice, ctx->stream));
    scalars = d_s;
    points = d_p;
  }
  return msm_enqueue<CV>(ctx, s, scalars, points, nullptr, 0, reinterpret_cast<X*>(d_buckets));
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
  const ReducePlan rp = owned_reduce_plan(ctx, nb, w_cnt);
  TailBufs<X> t;
  int rc = arena_carve(ctx, [&](Carve& cv) { t.carve(cv, w_cnt, rp.TP, rp); });
  if (rc) return rc;
  const X* recv = reinterpret_cast<const X*>(d_recv);
  rc = reduce_windows<CV>(ctx, nb, w_cnt, rp, t, reinterpret_cast<X*>(d_wsum), [&](unsigned grid) {
    if (rp.levels == 2) k_msm_reduce_l1<CV><<<grid, 128, 0, st>>>(nb, rp.m1, rp.m2, w_cnt, parts, recv, t.partials, t.runs);
    else k_msm_reduce_chunks_parts<CV><<<grid, 128, 0, st>>>(nb, rp.m1, w_cnt, parts, recv, t.partials);
  });
  if (rc) return rc;
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
  MsmLayout<CV> s;
  uint8_t *d_s = nullptr, *d_p = nullptr, *d_o = nullptr;
  int rc = msm_begin<CV>(ctx, n, scalars && points && out, s, [&](Carve& c) {
    d_s = c.take<uint8_t>(n * 32);
    d_p = c.take<uint8_t>(n * (size_t)CV::IN_BYTES);
    d_o = c.take<uint8_t>(256);
  });
  if (rc) return rc;
  CK(cudaMemsetAsync(ctx->d_flags, 0, 4, ctx->stream));
  // Large G1 batches: the H2D copy goes in 8 chunks on its own stream and the front end (k_glv_prepare: range and curve checks, the
  // endomorphism split, 8 field products per pair) runs chunk by chunk under it -- a blocking call no longer holds every kernel back until the
  // last byte has arrived (VERDICT r1 weak 6).  gev[0] orders the copies behind whatever still reads the arena, gev[1..8] hand the chunks over.
  const bool chunked = s.glv && ctx->msm_groups <= 1 && n >= (size_t(1) << 18) && copy_stream(ctx);
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
  rc = msm_enqueue<CV>(ctx, s, d_s, d_p, d_o, affine_out);
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
