// Host emulation of the MSM's bucket sort (msm_sort.cuh): digit columns + histogram as the point-load pass writes them, the scan,
// then k_msm_partition and k_msm_bin_sort block by block, every phase between two block barriers run for all threads of the block
// before the next one.  Compared with the plain counting sort (one cursor per bucket, one entry at a time).
// Test infrastructure only; never loaded by the product.
#include "../../kyber_b200/csrc/constants.cuh"
#include "../../kyber_b200/csrc/fp.cuh"
#include "../../kyber_b200/csrc/msm.cuh"
#include "../../kyber_b200/csrc/msm_sort.cuh"
#include <algorithm>
#include <cstring>
#include <vector>
using namespace b2k;

// the device plan (msm_host.cuh: make_plan) for window c over scalars of `bits` bits
static MsmPlan plan_of(int c, int bits) {
  MsmPlan pl; pl.c = c; pl.W = (bits + c) / c; pl.nb = 1 << (c - 1); pl.m = 1;
  memset(pl.K, 0, sizeof pl.K);
  for (int w = 0; w < pl.W; w++) { int bit = c * w + c - 1; pl.K[bit >> 5] |= 1u << (bit & 31); }
  return pl;
}

static void scan(const std::vector<uint32_t>& counts, uint32_t total, std::vector<uint32_t>& offs) {
  offs.assign(total + 1, 0);
  uint32_t run = 0;
  for (uint32_t g = 0; g < total; g++) { offs[g] = run; run += counts[g]; }
  offs[total] = run;
}

extern "C" {
// n 32-byte big-endian scalars, window c, scalar bits.  Returns 0 when the two sorts agree: same offsets, the same multiset of
// (index | sign) in every bucket, every histogram counter back at zero and every coarse cursor at the end of its bin.
// stats[0] = entries, stats[1] = largest coarse bin, stats[2] = mean entries per non-empty coarse bin, stats[3] = entries that
// reserved past the bin sort's shared slots.
int emul_msm_sort_check(size_t n, const uint8_t* scalars, int c, int bits, uint64_t* stats) {
  const MsmPlan pl = plan_of(c, bits);
  const uint32_t total = (uint32_t)pl.W * pl.nb;
  const int S = sort_shift(c);
  const uint32_t nbins = total >> S, bpw = (uint32_t)pl.nb >> S;
  if (bpw > (uint32_t)PART_BPW) return -1;

  // reference: histogram, scan, scatter with one cursor per bucket
  std::vector<uint32_t> ref_counts(total, 0);
  std::vector<std::vector<int>> dig(n);
  for (size_t i = 0; i < n; i++) {
    Scalar256 s; scalar_load_be(s, scalars + 32 * i);
    uint32_t sp[9]; msm_recode(sp, s, pl.K);
    for (int w = 0; w < pl.W; w++) { int d = msm_digit(sp, c, w); dig[i].push_back(d); if (d) ref_counts[(size_t)w * pl.nb + (d < 0 ? -d : d) - 1]++; }
  }
  std::vector<uint32_t> ref_offs;
  scan(ref_counts, total, ref_offs);
  std::vector<uint32_t> cur(ref_offs.begin(), ref_offs.end() - 1), ref_entries(ref_offs[total]);
  for (size_t i = 0; i < n; i++)
    for (int w = 0; w < pl.W; w++) { int d = dig[i][w]; if (d) { size_t g = (size_t)w * pl.nb + (d < 0 ? -d : d) - 1; ref_entries[cur[g]++] = (uint32_t)i | (d < 0 ? 0x80000000u : 0u); } }

  // the device path: digit columns + histogram, scan, partition, bin sort
  std::vector<int16_t> digits(n * (size_t)pl.W);
  std::vector<uint32_t> counts(total + 1, 0);
  for (size_t i = 0; i < n; i++) { Scalar256 s; scalar_load_be(s, scalars + 32 * i); msm_digits_store(s, pl, n, i, digits.data(), counts.data()); }
  std::vector<uint32_t> offs;
  scan(std::vector<uint32_t>(counts.begin(), counts.end() - 1), total, offs);
  if (offs != ref_offs) return 1;
  const uint32_t nrec = offs[total];
  std::vector<uint32_t> cursor(offs);                      // k_scan_finish: cursor = column 0
  std::vector<SortRec> recs((size_t)nrec + 1);
  static PartShared psh;
  std::vector<PartItems> pit(PART_T);
  const uint32_t pblocks = (uint32_t)((n + PART_TILE - 1) / PART_TILE);
  for (uint32_t b = 0; b < pblocks; b++) {
    for (uint32_t t = 0; t < PART_BPW; t++) psh.hist[t] = 0;
    for (int w = 0; w < pl.W; w++) {
      for (uint32_t t = 0; t < PART_T; t++) sort_part_rank(t, b, (uint32_t)n, pl, S, w, digits.data(), psh, pit[t]);
      for (uint32_t t = 0; t < PART_T; t++) sort_part_scan(t, bpw, psh);
      for (uint32_t t = 0; t < PART_T; t++) sort_part_reserve_stage(t, b, (uint32_t)n, pl, S, w, bpw, cursor.data(), psh, pit[t]);
      for (uint32_t t = 0; t < PART_T; t++) sort_part_flush(t, pl, S, w, bpw, psh, recs.data());
    }
  }
  uint64_t big = 0, nonempty = 0;
  for (uint32_t cb = 0; cb < nbins; cb++) {
    const uint32_t lo = offs[(size_t)cb << S], hi = offs[(size_t)(cb + 1) << S];
    if (cursor[(size_t)cb << S] != hi) return 2;           // every coarse run reserved exactly once
    for (uint32_t p = lo; p < hi; p++) if ((recs[p].bucket >> S) != cb) return 3;
    big = std::max<uint64_t>(big, hi - lo);
    nonempty += hi > lo;
  }
  std::vector<uint32_t> entries(nrec, 0xFFFFFFFFu);
  static BinShared bsh;
  std::vector<BinSortItems> items(BSORT_T);
  uint64_t spill = 0;
  const uint32_t bblocks = (uint32_t)(((size_t)n * pl.W + BSORT_TILE - 1) / BSORT_TILE);
  for (uint32_t b = 0; b < bblocks; b++) {
    if ((size_t)b * BSORT_TILE >= nrec) continue;
    const uint32_t base = sort_tile_base(b, S, recs.data());
    memset(&bsh, 0xEE, sizeof bsh);                          // shared memory starts undefined
    for (uint32_t s = 0; s < (uint32_t)SORT_SLOTS; s++) bsh.slot[s] = 0;
    for (uint32_t t = 0; t < BSORT_T; t++) sort_bin_rank(t, b, nrec, base, recs.data(), bsh, items[t]);
    for (uint32_t t = 0; t < BSORT_T; t++) sort_bin_scan1(t, bsh);
    for (uint32_t t = 0; t < BSORT_T; t++) sort_bin_scan2(t, bsh);
    for (uint32_t t = 0; t < BSORT_T; t++) sort_bin_scan3(t, bsh);
    for (uint32_t t = 0; t < BSORT_T; t++) sort_bin_reserve(t, base, offs.data(), counts.data(), bsh);
    for (uint32_t t = 0; t < BSORT_T; t++) {
      for (int k = 0; k < BSORT_I; k++) {
        const size_t r = bin_rec(t, b, k);
        if (r < nrec && items[t].r[k].bucket - base >= (uint32_t)SORT_SLOTS) spill++;
      }
      sort_bin_stage(t, b, nrec, base, items[t], offs.data(), counts.data(), entries.data(), bsh);
    }
    for (uint32_t t = 0; t < BSORT_T; t++) sort_bin_flush(t, bsh, entries.data());
  }
  for (uint32_t g = 0; g < total; g++) if (counts[g] != 0) return 4;
  for (uint32_t g = 0; g < total; g++) {
    std::vector<uint32_t> a(entries.begin() + offs[g], entries.begin() + offs[g + 1]);
    std::vector<uint32_t> e(ref_entries.begin() + offs[g], ref_entries.begin() + offs[g + 1]);
    std::sort(a.begin(), a.end());
    std::sort(e.begin(), e.end());
    if (a != e) return 5;
  }
  stats[0] = nrec; stats[1] = big; stats[2] = nonempty ? nrec / nonempty : 0; stats[3] = spill;
  return 0;
}
}
