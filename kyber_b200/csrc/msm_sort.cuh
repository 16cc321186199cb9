// msm_sort.cuh -- the MSM's bucket sort: (point index | sign) entries grouped by bucket, from the window-major int16 digit
// columns that the point-load pass writes (kernels.cuh: k_glv_prepare_bls381, k_msm_load) and the offsets of the histogram scan.
//
// Two passes, neither with one global atomic per entry, and both staging their output in shared memory so that every store of a
// warp lands in one contiguous run (a store of 32 scattered words costs 32 L2 sectors; measured, the unstaged passes spent most of
// their time there):
//   partition : a block takes a tile of pairs and goes through their windows one by one.  Per window it counts the tile's entries
//               over the window's COARSE bins (2^S consecutive buckets), reserves one run per non-empty bin with one atomic on
//               cursor[bin << S] (the scan sets it to the bin's first offset), groups the (entry, bucket) records by bin in shared
//               memory and copies them out.  recs[] is then grouped by coarse bin, every bin inside its final range
//               [offs[bin << S], offs[(bin + 1) << S]) of entries[].
//   bin sort  : a block takes a fixed range of recs[]; its buckets lie within SORT_SLOTS of the first record's coarse bin, so it
//               ranks them on shared-memory counters, scans the counters into tile offsets, reserves one run per bucket by an
//               atomicSub on counts[bucket] (the histogram, no longer needed after the scan: it ends at zero), groups the entries
//               by bucket in shared memory and copies them out.  Any bucket past the slots (tiles that cross many sparse bins,
//               small problems) reserves and stores per entry, from the same counter.
// The order of entries inside a bucket is not fixed (a bucket sum is a group element); the set is.  Both kernels take their
// shared-memory counters through smem_inc: the lanes of a warp that hit one counter (skewed scalars put whole warps on one
// bucket) share one atomic.  The per-thread bodies are phases between block barriers, so that tests/host_emul runs them block
// by block on the CPU.
#pragma once
#include "msm.cuh"

namespace b2k {

constexpr int SORT_SLOTS = 2048;                // bucket counters of the bin sort
constexpr int PART_T = 512, PART_P = 8;         // partition: threads, pairs per thread (tile = 4096 pairs)
constexpr int PART_TILE = PART_T * PART_P;
constexpr int PART_BPW = 32;                    // most coarse bins per window (c = 16: 2^15 >> 10)
constexpr int BSORT_T = 512, BSORT_I = 8;       // bin sort: threads, records per thread (tile = 4096 records)
constexpr int BSORT_TILE = BSORT_T * BSORT_I;
constexpr int BSORT_SPT = SORT_SLOTS / BSORT_T; // slots per thread in the tile scan

// coarse bin = bucket >> S, S <= c - 1 so that a bin never crosses a window.  2^(S+1) <= SORT_SLOTS: a bin-sort tile that spans
// two bins still ranks on shared counters.  At C2 (c = 16) that is 32 bins of 1024 buckets per window.
constexpr int sort_shift(int c) { return c - 1 < 10 ? c - 1 : 10; }

struct alignas(8) SortRec { uint32_t word, bucket; };     // word = point index | sign << 31, bucket = w nb + |d| - 1

B2K_D uint32_t sort_word(uint32_t i, int d) { return i | (d < 0 ? 0x80000000u : 0u); }
B2K_D uint32_t sort_bucket(const MsmPlan& pl, int w, int d) { return (uint32_t)w * (uint32_t)pl.nb + (uint32_t)(d < 0 ? -d : d) - 1u; }

#ifdef B2K_HOST_EMUL
B2K_D uint32_t smem_inc(uint32_t* s, uint32_t key, bool on) { return on ? s[key]++ : 0u; }
B2K_D uint32_t glob_add(uint32_t* p, uint32_t v) { uint32_t o = *p; *p = o + v; return o; }
B2K_D uint32_t glob_sub(uint32_t* p, uint32_t v) { uint32_t o = *p; *p = o - v; return o; }
#else
// s[key] += 1 for every lane with on, returning the lane's old value as if the lanes had gone one by one.  All 32 lanes of the
// warp must call it together.
B2K_D uint32_t smem_inc(uint32_t* s, uint32_t key, bool on) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t peers = __match_any_sync(0xffffffffu, on ? key : 0xffffffffu);
  const int leader = __ffs(peers) - 1;
  uint32_t base = 0;
  if (on && lane == (uint32_t)leader) base = atomicAdd(&s[key], (uint32_t)__popc(peers));
  base = __shfl_sync(0xffffffffu, base, leader);
  return base + (uint32_t)__popc(peers & ((1u << lane) - 1u));
}
B2K_D uint32_t glob_add(uint32_t* p, uint32_t v) { return atomicAdd(p, v); }
B2K_D uint32_t glob_sub(uint32_t* p, uint32_t v) { return atomicSub(p, v); }
#endif

// ---- digit columns + histogram (the point-load pass: kernels.cuh k_msm_load, k_glv_prepare_bls381) ----------------------------
// window-major signed digits of pair i: digits[w n + i] (0 = no entry; |d| <= 2^(c-1) <= 2^15 fits int16), counts[bucket] += 1
B2K_D void msm_digits_store(const Scalar256& s, const MsmPlan& pl, size_t n, size_t i, int16_t* __restrict__ digits,
                            uint32_t* __restrict__ counts) {
  uint32_t sp[9];
  msm_recode(sp, s, pl.K);
  for (int w = 0; w < pl.W; w++) {
    const int d = msm_digit(sp, pl.c, w);
    digits[(size_t)w * n + i] = (int16_t)d;
    if (d) glob_add(&counts[sort_bucket(pl, w, d)], 1u);
  }
}

// ---- partition: one window of one tile per round of five phases --------------------------------------------------------------
// shared state of a round: hist[b] = entries of the tile in bin b of the window (zero at the start of a round), loff[b] = their
// first position in the staging array stage[], delta[b] = recs[] position of the run minus loff[b], ntile = entries of the round
struct PartShared {
  uint32_t hist[PART_BPW], loff[PART_BPW], delta[PART_BPW], ntile;
  SortRec stage[PART_TILE];
};
struct PartItems { int d[PART_P]; uint32_t rank[PART_P]; };
B2K_D uint32_t part_pair(uint32_t tid, uint32_t blk, int k) { return blk * (uint32_t)PART_TILE + (uint32_t)(k * PART_T) + tid; }
// 1: digits of the tile in window w, ranks within their bins
B2K_D void sort_part_rank(uint32_t tid, uint32_t blk, uint32_t n, const MsmPlan& pl, int S, int w, const int16_t* digits,
                          PartShared& sh, PartItems& it) {
  const int16_t* col = digits + (size_t)w * n;
#pragma unroll
  for (int k = 0; k < PART_P; k++) {
    const uint32_t i = part_pair(tid, blk, k);
    const int d = i < n ? (int)col[i] : 0;
    it.d[k] = d;
    const uint32_t b = d ? (uint32_t)((d < 0 ? -d : d) - 1) >> S : 0u;
    it.rank[k] = smem_inc(sh.hist, b, d != 0);
  }
}
// 2: tile offsets of the bins (bpw <= PART_BPW, one thread)
B2K_D void sort_part_scan(uint32_t tid, uint32_t bpw, PartShared& sh) {
  if (tid) return;
  uint32_t run = 0;
  for (uint32_t b = 0; b < bpw; b++) { sh.loff[b] = run; run += sh.hist[b]; }
  sh.ntile = run;
}
// 3: one run per non-empty bin (and the histogram back to zero), then the records into the staging array
B2K_D void sort_part_reserve_stage(uint32_t tid, uint32_t blk, uint32_t n, const MsmPlan& pl, int S, int w, uint32_t bpw,
                                   uint32_t* cursor, PartShared& sh, const PartItems& it) {
  if (tid < bpw) {
    const uint32_t c = sh.hist[tid];
    sh.hist[tid] = 0;
    if (c) sh.delta[tid] = glob_add(&cursor[(size_t)(w * bpw + tid) << S], c) - sh.loff[tid];
  }
#pragma unroll
  for (int k = 0; k < PART_P; k++) {
    const int d = it.d[k];
    if (!d) continue;
    const uint32_t b = (uint32_t)((d < 0 ? -d : d) - 1) >> S;
    sh.stage[sh.loff[b] + it.rank[k]] = SortRec{sort_word(part_pair(tid, blk, k), d), sort_bucket(pl, w, d)};
  }
}
// 4: the staged records out, runs of consecutive positions
B2K_D void sort_part_flush(uint32_t tid, const MsmPlan& pl, int S, int w, uint32_t bpw, const PartShared& sh, SortRec* recs) {
  for (uint32_t j = tid; j < sh.ntile; j += PART_T) {
    const SortRec r = sh.stage[j];
    const uint32_t b = (r.bucket - (uint32_t)w * (uint32_t)pl.nb) >> S;
    recs[sh.delta[b] + j] = r;
  }
}

// ---- bin sort -----------------------------------------------------------------------------------------------------------------
struct BinShared {
  uint32_t slot[SORT_SLOTS];       // tile counts per bucket, then (entries position of the run - tile offset)
  uint32_t loff[SORT_SLOTS];       // tile offset of the bucket's entries in stage[]
  uint32_t tsum[BSORT_T];          // scan: per-thread sums of BSORT_SPT slots, then their exclusive prefix within a group of 32
  uint32_t gsum[BSORT_T / 32];     // scan: group totals, then their exclusive prefix
  uint32_t nstage;
  uint32_t word[BSORT_TILE];
  uint16_t key[BSORT_TILE];
};
struct BinSortItems { SortRec r[BSORT_I]; uint32_t rank[BSORT_I]; };
// first bucket of the coarse bin of the tile's first record: no bucket of the tile is below it
B2K_D uint32_t sort_tile_base(uint32_t blk, int S, const SortRec* recs) { return (recs[(size_t)blk * BSORT_TILE].bucket >> S) << S; }
B2K_D size_t bin_rec(uint32_t tid, uint32_t blk, int k) { return (size_t)blk * BSORT_TILE + (size_t)(k * BSORT_T) + tid; }   // 64-bit: nrec may come within a tile of 2^32
// 1: ranks within the tile on slot[bucket - base]
B2K_D void sort_bin_rank(uint32_t tid, uint32_t blk, uint32_t nrec, uint32_t base, const SortRec* recs, BinShared& sh, BinSortItems& it) {
#pragma unroll
  for (int k = 0; k < BSORT_I; k++) {
    const size_t r = bin_rec(tid, blk, k);
    const bool on = r < nrec;
    it.r[k] = on ? recs[r] : SortRec{0u, base};
    const uint32_t key = it.r[k].bucket - base;
    it.rank[k] = smem_inc(sh.slot, key, on && key < (uint32_t)SORT_SLOTS);
  }
}
// 2-4: exclusive scan of the slots into loff (per thread, per group of 32 threads, over the groups)
B2K_D void sort_bin_scan1(uint32_t tid, BinShared& sh) {
  uint32_t s = 0;
  for (int j = 0; j < BSORT_SPT; j++) s += sh.slot[tid * BSORT_SPT + j];
  sh.tsum[tid] = s;
}
B2K_D void sort_bin_scan2(uint32_t tid, BinShared& sh) {
  if (tid >= (uint32_t)(BSORT_T / 32)) return;
  uint32_t run = 0;
  for (uint32_t j = 32 * tid; j < 32 * tid + 32; j++) { const uint32_t v = sh.tsum[j]; sh.tsum[j] = run; run += v; }
  sh.gsum[tid] = run;
}
B2K_D void sort_bin_scan3(uint32_t tid, BinShared& sh) {
  if (tid) return;
  uint32_t run = 0;
  for (int g = 0; g < BSORT_T / 32; g++) { const uint32_t v = sh.gsum[g]; sh.gsum[g] = run; run += v; }
  sh.nstage = run;
}
// 5: tile offsets, and one run per bucket of the tile: counts[g] holds how many entries of bucket g are still unplaced; its runs
// fill from the top
B2K_D void sort_bin_reserve(uint32_t tid, uint32_t base, const uint32_t* offs, uint32_t* counts, BinShared& sh) {
  uint32_t run = sh.gsum[tid / 32] + sh.tsum[tid];
  for (int j = 0; j < BSORT_SPT; j++) {
    const uint32_t s = tid * BSORT_SPT + j, c = sh.slot[s];
    sh.loff[s] = run;
    if (c) { const uint32_t g = base + s; sh.slot[s] = offs[g] + glob_sub(&counts[g], c) - c - run; }
    run += c;
  }
}
// 6: entries into the staging array; a bucket past the slots reserves and stores each entry on its own
B2K_D void sort_bin_stage(uint32_t tid, uint32_t blk, uint32_t nrec, uint32_t base, const BinSortItems& it, const uint32_t* offs,
                          uint32_t* counts, uint32_t* entries, BinShared& sh) {
#pragma unroll
  for (int k = 0; k < BSORT_I; k++) {
    if (bin_rec(tid, blk, k) >= nrec) continue;
    const uint32_t g = it.r[k].bucket, key = g - base;
    if (key < (uint32_t)SORT_SLOTS) {
      const uint32_t p = sh.loff[key] + it.rank[k];
      sh.word[p] = it.r[k].word;
      sh.key[p] = (uint16_t)key;
    } else {
      entries[offs[g] + glob_sub(&counts[g], 1u) - 1u] = it.r[k].word;
    }
  }
}
// 7: the staged entries out, runs of consecutive positions
B2K_D void sort_bin_flush(uint32_t tid, const BinShared& sh, uint32_t* entries) {
  for (uint32_t j = tid; j < sh.nstage; j += BSORT_T) entries[sh.slot[sh.key[j]] + j] = sh.word[j];
}

#ifdef __CUDACC__
// coarse partition of the entries of a tile of 4096 pairs into recs[] (grouped by coarse bin, each bin in its final range)
static __global__ void __launch_bounds__(PART_T) k_msm_partition(uint32_t n, MsmPlan pl, int S, const int16_t* __restrict__ digits,
                                                                 uint32_t* __restrict__ cursor, SortRec* __restrict__ recs) {
  __shared__ PartShared sh;
  const uint32_t tid = threadIdx.x, bpw = (uint32_t)pl.nb >> S;
  if (tid < PART_BPW) sh.hist[tid] = 0;
  __syncthreads();
  for (int w = 0; w < pl.W; w++) {
    PartItems it;
    sort_part_rank(tid, blockIdx.x, n, pl, S, w, digits, sh, it);
    __syncthreads();
    sort_part_scan(tid, bpw, sh);
    __syncthreads();
    sort_part_reserve_stage(tid, blockIdx.x, n, pl, S, w, bpw, cursor, sh, it);
    __syncthreads();
    sort_part_flush(tid, pl, S, w, bpw, sh, recs);
    __syncthreads();
  }
}
// records -> entries[] in bucket order, a tile of 4096 records per block; the entry count is offs[total]
static __global__ void __launch_bounds__(BSORT_T) k_msm_bin_sort(uint32_t total, int S, const SortRec* __restrict__ recs,
                                                                 const uint32_t* __restrict__ offs, uint32_t* __restrict__ counts,
                                                                 uint32_t* __restrict__ entries) {
  __shared__ BinShared sh;
  const uint32_t tid = threadIdx.x, nrec = offs[total];
  if ((size_t)blockIdx.x * BSORT_TILE >= nrec) return;
  const uint32_t base = sort_tile_base(blockIdx.x, S, recs);
  for (uint32_t s = tid; s < (uint32_t)SORT_SLOTS; s += BSORT_T) sh.slot[s] = 0;
  __syncthreads();
  BinSortItems it;
  sort_bin_rank(tid, blockIdx.x, nrec, base, recs, sh, it);
  __syncthreads();
  sort_bin_scan1(tid, sh);
  __syncthreads();
  sort_bin_scan2(tid, sh);
  __syncthreads();
  sort_bin_scan3(tid, sh);
  __syncthreads();
  sort_bin_reserve(tid, base, offs, counts, sh);
  __syncthreads();
  sort_bin_stage(tid, blockIdx.x, nrec, base, it, offs, counts, entries, sh);
  __syncthreads();
  sort_bin_flush(tid, sh, entries);
}
#endif

}  // namespace b2k
