// Host emulation of the edwards25519 MSM and share/poly device code (test infrastructure only): the per-thread bodies of
// ed_msm.cuh and lagrange.cuh, driven in the order the kernels of b2k_ed25519_msm.cu run them.
#include <vector>
#include "../../kyber_b200/csrc/ed_msm.cuh"
#include "../../kyber_b200/csrc/lagrange.cuh"
using namespace b2k;

static void store_le(uint8_t* out, const EFp& a) {
  EFp c;
  fp_from_mont(c, a);
  for (int j = 0; j < 32; j++) out[j] = (uint8_t)(c.v[j >> 2] >> (8 * (j & 3)));
}

// the plan make_plan (msm_host.cuh) builds for 256-bit scalars, window c and chunk m
static MsmPlan plan(int c, int m) {
  MsmPlan pl;
  pl.c = c; pl.W = (256 + c) / c; pl.nb = 1 << (c - 1); pl.m = m;
  for (int j = 0; j < 9; j++) pl.K[j] = 0;
  for (int w = 0; w < pl.W; w++) { const int bit = c * w + c - 1; pl.K[bit >> 5] |= 1u << (bit & 31); }
  return pl;
}

// the block-wide sums of k_ed_msm_fixup_big / k_ed_msm_window_sum: 128 strided partial sums, then the same tree
static EdExt block_tree(std::vector<EdExt>& sm) {
  for (int h = 64; h > 0; h >>= 1)
    for (int tid = 0; tid < h; tid++) ed_add(sm[tid], sm[tid], sm[tid + h]);
  return sm[0];
}

extern "C" {
// the load pass for one pair: Niels form (3 x 32 canonical little-endian bytes), the W digits of the ruled scalar; returns
// whether the point decoded
int emul_ed_load(const uint8_t* scalar, const uint8_t* point, int c, int16_t* digits, uint8_t* niels) {
  const MsmPlan pl = plan(c, 1);
  std::vector<uint32_t> counts((size_t)pl.W * pl.nb + 1, 0);
  EdNiels q;
  const bool ok = ed_msm_load(1, 0, scalar, point, &q, pl, digits, counts.data());
  store_le(niels, q.ypx); store_le(niels + 32, q.ymx); store_le(niels + 64, q.t2d);
  return ok ? 1 : 0;
}

void emul_ed_scalar_rule(const uint8_t* k_in, uint8_t* k_out) {
  uint32_t k[8];
  sc_load_le(k, k_in);
  ed_scalar_rule(k);
  for (int j = 0; j < 32; j++) k_out[j] = (uint8_t)(k[j >> 2] >> (8 * (j & 3)));
}

// The whole MSM with window c, chunk m, slice length L; buckets with more than serial_max partials (2 or 64) take the
// block-parallel fix-up.  Returns the number of points that did not decode; stats = {cut buckets, block-parallel buckets}.
int emul_ed_msm(uint32_t n, const uint8_t* scalars, const uint8_t* points, int c, int m, uint32_t L, int serial_max, uint8_t* out,
                uint32_t* stats) {
  const MsmPlan pl = plan(c, m);
  const uint32_t total = (uint32_t)pl.W * pl.nb;
  std::vector<EdNiels> pts(n);
  std::vector<int16_t> digits((size_t)n * pl.W);
  std::vector<uint32_t> counts(total + 1, 0), offs(total + 1, 0), cur(total + 1);
  int bad = 0;
  for (uint32_t i = 0; i < n; i++) bad += !ed_msm_load(n, i, scalars, points, pts.data(), pl, digits.data(), counts.data());
  for (uint32_t g = 0; g < total; g++) offs[g + 1] = offs[g] + counts[g];
  cur = offs;
  const uint32_t E = offs[total];
  std::vector<uint32_t> entries(E > 0 ? E : 1);
  for (int w = 0; w < pl.W; w++)
    for (uint32_t i = 0; i < n; i++) {
      const int d = digits[(size_t)w * n + i];
      if (d) entries[cur[sort_bucket(pl, w, d)]++] = sort_word(i, d);
    }
  const uint32_t smax = (uint32_t)(((size_t)n * pl.W + L - 1) / L) + 1;
  std::vector<EdExt> buckets(total), spart(2 * (size_t)smax);
  for (uint32_t j = 0; j < smax; j++) ed_accumulate_slice(j, L, total, pts.data(), offs.data(), entries.data(), buckets.data(), spart.data());
  stats[0] = stats[1] = 0;
  for (uint32_t g = 0; g < total; g++) {
    const uint32_t s = offs[g], t = offs[g + 1];
    if (t > s && s / L != (t - 1) / L) stats[0]++;
    const bool big = serial_max == 2 ? ed_fixup_bucket<2>(g, L, offs.data(), buckets.data(), spart.data())
                                     : ed_fixup_bucket<64>(g, L, offs.data(), buckets.data(), spart.data());
    if (!big) continue;
    stats[1]++;
    std::vector<EdExt> sm(128);
    for (uint32_t tid = 0; tid < 128; tid++) ed_fixup_strided(sm[tid], tid, 128, s / L, (t - 1) / L, spart.data());
    buckets[g] = block_tree(sm);
  }
  const int T = pl.nb / pl.m;
  std::vector<EdExt> partials((size_t)pl.W * T), wsum(pl.W);
  for (size_t id = 0; id < (size_t)pl.W * T; id++) ed_reduce_chunk(partials[id], buckets.data() + (id / T) * pl.nb, (int)(id % T), pl.m);
  for (int w = 0; w < pl.W; w++) {
    std::vector<EdExt> sm(128);
    for (int tid = 0; tid < 128; tid++) {
      ed_set_identity(sm[tid]);
      for (int t = tid; t < T; t += 128) ed_add(sm[tid], sm[tid], partials[(size_t)w * T + t]);
    }
    wsum[w] = block_tree(sm);
  }
  EdExt r;
  ed_msm_horner(r, wsum.data(), pl.W, pl.c);
  ed_encode(out, r);
  return bad;
}

// lambda_i mod l for every i, 32-byte little-endian; returns 0 when two indices are equal
int emul_ed_lagrange(uint32_t t, const uint32_t* idx, uint8_t* out) {
  int ok = 1;
  for (uint32_t i = 0; i < t; i++) ok &= lagrange_at_zero<Ed25519Fr, true>(i, t, idx, out + 32 * (size_t)i) ? 1 : 0;
  return ok;
}

// PubPoly.Eval at one index (commits [t][32]); returns the number of commitments that did not decode
int emul_ed_pubpoly_eval(uint32_t t, const uint8_t* commits, uint32_t index, uint8_t* out) {
  std::vector<EdNiels> cm(t);
  int bad = 0;
  for (uint32_t j = 0; j < t; j++) bad += !ed_load_niels(cm[j], commits + 32 * (size_t)j);
  EdExt v;
  ed_pubpoly_horner(v, cm.data(), t, (uint64_t)index + 1u);
  ed_encode(out, v);
  return bad;
}

// PubPoly.Check of one share (32 bytes little-endian) against commits [t][32]
int emul_ed_pubpoly_check(uint32_t t, const uint8_t* commits, uint32_t index, const uint8_t* share) {
  std::vector<EdNiels> cm(t);
  for (uint32_t j = 0; j < t; j++) ed_load_niels(cm[j], commits + 32 * (size_t)j);
  EdNiels btab[8];
  ed_load_base_table(btab);
  return ed_pubpoly_check_one(cm.data(), t, index, share, btab) ? 1 : 0;
}

// s B by the geScalarMult schedule (the base-point half of the check), encoded
void emul_ed_ge_scalar_mult_base(const uint8_t* k_le, uint8_t* out) {
  EdNiels btab[8];
  ed_load_base_table(btab);
  uint32_t k[8];
  sc_load_le(k, k_le);
  EdExt r;
  ed_ge_scalar_mult_base(r, k, btab);
  ed_encode(out, r);
}
}
