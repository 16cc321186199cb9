// Host emulation of the MSM's affine pair-tree rounds with every round's bucket offsets taken from the histogram scan up front
// (kernels.cuh: k_scan_blocks / k_scan_tops / k_scan_finish, column y = ceil(counts / 2^y)), as msm_host.cuh enqueues them.
// Test infrastructure only; never loaded by the product.
#include "../../kyber_b200/csrc/constants.cuh"
#include "../../kyber_b200/csrc/fp.cuh"
#include "../../kyber_b200/csrc/msm.cuh"
#include "../../kyber_b200/csrc/msm_affine.cuh"
#include <cstring>
#include <vector>
using namespace b2k;

// the three scan passes over columns 0..R, block by block (1024 counters per block), into the device layout:
// column 0 -> offs[0 .. total], column y >= 1 -> offs_rounds[(y - 1) (total + 1) ..]
static void scan_columns(const uint32_t* counts, uint32_t total, int R, uint32_t* offs, uint32_t* offs_rounds) {
  const uint32_t nblocks = (total + 1023) / 1024;
  for (int y = 0; y <= R; y++) {
    uint32_t* col = y == 0 ? offs : offs_rounds + (size_t)(y - 1) * (total + 1);
    std::vector<uint32_t> bsum(nblocks);
    for (uint32_t b = 0; b < nblocks; b++) {                 // pass A: per-block exclusive scan + block totals
      uint32_t run = 0;
      for (uint32_t i = b * 1024; i < total && i < (b + 1) * 1024; i++) { col[i] = run; run += pt_round_count(counts[i], (uint32_t)y); }
      bsum[b] = run;
    }
    uint32_t run = 0;                                        // pass B: scan of the block totals, grand total
    for (uint32_t b = 0; b < nblocks; b++) { const uint32_t v = bsum[b]; bsum[b] = run; run += v; }
    col[total] = run;
    for (uint32_t i = 0; i < total; i++) col[i] += bsum[i / 1024];   // pass C
  }
}

static MsmPlan plan_of(int c, int m) {
  MsmPlan pl; pl.c = c; pl.W = (256 + c - 1) / c; pl.nb = 1 << (c - 1); pl.m = m;
  uint32_t K[9] = {0};
  for (int w = 0; w < pl.W; w++) { int bit = c * w + c - 1; if (bit < 288) K[bit >> 5] |= 1u << (bit & 31); }
  memcpy(pl.K, K, sizeof K);
  return pl;
}

// digits, counting sort, R split rounds on the precomputed offsets (forward / invert / backward; `staged`: the cp.async-staged
// forward and backward variants), balanced slices, fix-up, chunk reduction, Horner
template <class CV>
static int msm_onescan(size_t n, const uint8_t* scalars, const uint8_t* pts, int c, int m, int L, int rounds, int PB, bool staged, uint8_t* out) {
  using F = typename CV::F;
  const MsmPlan pl = plan_of(c, m);
  std::vector<Affine<F>> P(n);
  for (size_t i = 0; i < n; i++) CV::load(P[i], pts + CV::IN_BYTES * i);
  const uint32_t total = (uint32_t)pl.W * pl.nb;
  std::vector<uint32_t> counts(total + 1, 0);
  for (size_t i = 0; i < n; i++) {
    Scalar256 s; scalar_load_be(s, scalars + 32 * i);
    if (!scalar_in_range<typename CV::ScalarField>(s)) return -3;
    uint32_t sp[9]; msm_recode(sp, s, pl.K);
    for (int w = 0; w < pl.W; w++) { int d = msm_digit(sp, c, w); if (d) counts[(size_t)w * pl.nb + (d < 0 ? -d : d) - 1]++; }
  }
  std::vector<uint32_t> offs(total + 1), offs_rt((size_t)(rounds > 0 ? rounds : 1) * (total + 1));
  scan_columns(counts.data(), total, rounds, offs.data(), offs_rt.data());
  std::vector<uint32_t> cursor(offs.begin(), offs.end()), entries(offs[total] + 1);
  for (size_t i = 0; i < n; i++) {
    Scalar256 s; scalar_load_be(s, scalars + 32 * i);
    uint32_t sp[9]; msm_recode(sp, s, pl.K);
    for (int w = 0; w < pl.W; w++) { int d = msm_digit(sp, c, w); if (d) { size_t g = (size_t)w * pl.nb + (d < 0 ? -d : d) - 1; entries[cursor[g]++] = (uint32_t)i | (d < 0 ? 0x80000000u : 0); } }
  }
  const uint32_t* offs_cur = offs.data();
  std::vector<Affine<F>> cur;
  for (int r = 0; r < rounds; r++) {
    const uint32_t* no = offs_rt.data() + (size_t)r * (total + 1);
    std::vector<Affine<F>> nxt(no[total] + 1);
    const uint32_t T = (no[total] + PB - 1) / PB + 1;      // one thread past the end: must be a no-op
    const Affine<F>* in = r == 0 ? P.data() : cur.data();
    std::vector<F> pre((size_t)T * PB), accs(T);
    for (uint32_t t = 0; t < T; t++) {
      if (staged) {
        alignas(16) unsigned char slots[4 * sizeof(F)];
        memset(slots, 0xEE, sizeof slots);
        if (r == 0) msm_pairtree_forward_staged<CV, true>(t, (uint32_t)PB, T, total, in, entries.data(), offs_cur, no, pre.data(), accs.data(), slots, 0);
        else msm_pairtree_forward_staged<CV, false>(t, (uint32_t)PB, T, total, in, nullptr, offs_cur, no, pre.data(), accs.data(), slots, 0);
      } else if (r == 0) msm_pairtree_forward<CV, true>(t, (uint32_t)PB, T, total, in, entries.data(), offs_cur, no, pre.data(), accs.data());
      else msm_pairtree_forward<CV, false>(t, (uint32_t)PB, T, total, in, nullptr, offs_cur, no, pre.data(), accs.data());
    }
    for (uint32_t t = 0; t < T; t++) msm_pairtree_invert<F>(t, (uint32_t)PB, total, no, accs.data());
    for (uint32_t t = 0; t < T; t++) {
      if (staged) {
        alignas(16) unsigned char slots[4 * sizeof(Affine<F>) + sizeof(F)];
        memset(slots, 0xEE, sizeof slots);
        if (r == 0) msm_pairtree_backward_staged<CV, true>(t, (uint32_t)PB, T, total, in, entries.data(), offs_cur, no, pre.data(), accs.data(), nxt.data(), slots, 0);
        else msm_pairtree_backward_staged<CV, false>(t, (uint32_t)PB, T, total, in, nullptr, offs_cur, no, pre.data(), accs.data(), nxt.data(), slots, 0);
      } else if (r == 0) msm_pairtree_backward<CV, true>(t, (uint32_t)PB, T, total, in, entries.data(), offs_cur, no, pre.data(), accs.data(), nxt.data());
      else msm_pairtree_backward<CV, false>(t, (uint32_t)PB, T, total, in, nullptr, offs_cur, no, pre.data(), accs.data(), nxt.data());
    }
    cur.swap(nxt);
    offs_cur = no;
  }
  std::vector<Xyzz<F>> B(total);
  memset((void*)B.data(), 0, total * sizeof(Xyzz<F>));
  const uint32_t E = offs_cur[total], S = (E + L - 1) / L;
  std::vector<Xyzz<F>> spart(2 * (size_t)S + 2);
  for (uint32_t j = 0; j < S; j++) {
    if (rounds) msm_accumulate_slice<CV, true>(j, (uint32_t)L, total, cur.data(), offs_cur, nullptr, B.data(), spart.data());
    else msm_accumulate_slice<CV>(j, (uint32_t)L, total, P.data(), offs_cur, entries.data(), B.data(), spart.data());
  }
  for (uint32_t g = 0; g < total; g++) {
    if (msm_fixup_bucket<CV, 3>(g, (uint32_t)L, offs_cur, B.data(), spart.data())) {   // the block-parallel path, serially
      const uint32_t j0 = offs_cur[g] / L, j1 = (offs_cur[g + 1] - 1) / L;
      Xyzz<F> a = spart[2 * (size_t)j0 + 1];
      for (uint32_t j = j0 + 1; j <= j1; j++) xyzz_add(a, a, spart[2 * (size_t)j]);
      B[g] = a;
    }
  }
  const int T = pl.nb / m;
  std::vector<Xyzz<F>> wsum(pl.W);
  for (int w = 0; w < pl.W; w++) {
    Xyzz<F> a; xyzz_set_inf(a);
    for (int t = 0; t < T; t++) { Xyzz<F> part; msm_reduce_chunk<CV>(part, &B[(size_t)w * pl.nb], t, m); xyzz_add(a, a, part); }
    wsum[w] = a;
  }
  Xyzz<F> r; msm_horner<CV>(r, wsum.data(), pl.W, c);
  Affine<F> a; xyzz_to_affine(a, r);
  CV::store(out, a);
  return 0;
}

extern "C" {
// columns 0..R of the multi-column scan, (R + 1) (total + 1) words: column 0 then the R round columns
void emul_scan_columns(const uint32_t* counts, uint32_t total, int R, uint32_t* out) {
  scan_columns(counts, total, R, out, out + (total + 1));
}
int emul_bls12381_g1_msm_affine_onescan(size_t n, const uint8_t* s, const uint8_t* p, int c, int m, int L, int rounds, int PB, int staged, uint8_t* o) {
  return msm_onescan<Bls381G1>(n, s, p, c, m, L, rounds, PB, staged != 0, o);
}
}
