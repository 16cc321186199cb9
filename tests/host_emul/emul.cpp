// Host emulation of the device limb code (test infrastructure only; never loaded by the product).
#include "../../kyber_b200/csrc/constants.cuh"
#include "../../kyber_b200/csrc/fp.cuh"
#include "../../kyber_b200/csrc/tower.cuh"
using namespace b2k;
extern "C" {
#define FIELD_API(name, C)                                                                        \
  void emul_##name##_mul(const uint32_t* a, const uint32_t* b, uint32_t* r) {                      \
    Fp<C> x, y, z; for (int i = 0; i < C::N; i++) { x.v[i] = a[i]; y.v[i] = b[i]; }                \
    fp_mul(z, x, y); for (int i = 0; i < C::N; i++) r[i] = z.v[i]; }                               \
  void emul_##name##_add(const uint32_t* a, const uint32_t* b, uint32_t* r) {                      \
    Fp<C> x, y, z; for (int i = 0; i < C::N; i++) { x.v[i] = a[i]; y.v[i] = b[i]; }                \
    fp_add(z, x, y); for (int i = 0; i < C::N; i++) r[i] = z.v[i]; }                               \
  void emul_##name##_sub(const uint32_t* a, const uint32_t* b, uint32_t* r) {                      \
    Fp<C> x, y, z; for (int i = 0; i < C::N; i++) { x.v[i] = a[i]; y.v[i] = b[i]; }                \
    fp_sub(z, x, y); for (int i = 0; i < C::N; i++) r[i] = z.v[i]; }                               \
  void emul_##name##_addsub(const uint32_t* a, const uint32_t* b, int minus, uint32_t* r) {        \
    Fp<C> x, y, z; for (int i = 0; i < C::N; i++) { x.v[i] = a[i]; y.v[i] = b[i]; }                \
    fp_addsub(z, x, y, minus != 0); for (int i = 0; i < C::N; i++) r[i] = z.v[i]; }                \
  void emul_##name##_sqr(const uint32_t* a, uint32_t* r) {                                         \
    Fp<C> x, z; for (int i = 0; i < C::N; i++) x.v[i] = a[i];                                      \
    fp_sqr(z, x); for (int i = 0; i < C::N; i++) r[i] = z.v[i]; }                                  \
  void emul_##name##_wide_mul(const uint32_t* a, const uint32_t* b, uint32_t* t) {                 \
    detail::wide_mul<C::N>(t, a, b); }                                                             \
  void emul_##name##_wide_sqr(const uint32_t* a, uint32_t* t) { detail::wide_sqr<C::N>(t, a); }    \
  void emul_##name##_redc(const uint32_t* t, uint32_t* r) {                                        \
    detail::redc_wide<C>(r, t); fp_reduce_once<C>(r); }                                            \
  void emul_##name##_neg(const uint32_t* a, uint32_t* r) {                                         \
    Fp<C> x, z; for (int i = 0; i < C::N; i++) x.v[i] = a[i];                                      \
    fp_neg(z, x); for (int i = 0; i < C::N; i++) r[i] = z.v[i]; }                                  \
  void emul_##name##_inv(const uint32_t* a, uint32_t* r) {                                         \
    Fp<C> x, z; for (int i = 0; i < C::N; i++) x.v[i] = a[i];                                      \
    fp_inv(z, x); for (int i = 0; i < C::N; i++) r[i] = z.v[i]; }                                  \
  void emul_##name##_inv_fermat(const uint32_t* a, uint32_t* r) {                                  \
    Fp<C> x, z; for (int i = 0; i < C::N; i++) x.v[i] = a[i];                                      \
    fp_inv_fermat(z, x); for (int i = 0; i < C::N; i++) r[i] = z.v[i]; }                           \
  void emul_##name##_to_mont(const uint32_t* a, uint32_t* r) {                                     \
    Fp<C> x, z; for (int i = 0; i < C::N; i++) x.v[i] = a[i];                                      \
    fp_to_mont(z, x); for (int i = 0; i < C::N; i++) r[i] = z.v[i]; }                              \
  void emul_##name##_from_mont(const uint32_t* a, uint32_t* r) {                                   \
    Fp<C> x, z; for (int i = 0; i < C::N; i++) x.v[i] = a[i];                                      \
    fp_from_mont(z, x); for (int i = 0; i < C::N; i++) r[i] = z.v[i]; }
#define FP2_LAZY_API(name, C)                                                                      \
  void emul_##name##_fp2_mul_pair(const uint32_t* a, const uint32_t* b, uint32_t* r, uint32_t* rl) { \
    Fp2<C> x, y, z, zl;                                                                            \
    for (int i = 0; i < C::N; i++) { x.c0.v[i] = a[i]; x.c1.v[i] = a[C::N + i]; y.c0.v[i] = b[i]; y.c1.v[i] = b[C::N + i]; } \
    fp2_mul(z, x, y); fp2_mul_lazy(zl, x, y);                                                      \
    for (int i = 0; i < C::N; i++) { r[i] = z.c0.v[i]; r[C::N + i] = z.c1.v[i]; rl[i] = zl.c0.v[i]; rl[C::N + i] = zl.c1.v[i]; } }
FP2_LAZY_API(fp381, Bls381Fp)
FP2_LAZY_API(fp254, Bn254Fp)
FP2_LAZY_API(fp256, Bn256Fp)
FIELD_API(fp381, Bls381Fp)
FIELD_API(fr381, Bls381Fr)
FIELD_API(fp254, Bn254Fp)
FIELD_API(fp256, Bn256Fp)
FIELD_API(fp25519, Ed25519Fp)
}

// ------------------------------------------------------------------------------------------------
// curve-level emulation: run the per-thread kernel bodies in plain loops
#include "../../kyber_b200/csrc/msm.cuh"
#include "../../kyber_b200/csrc/msm_affine.cuh"
#include <vector>
#include <cstring>

template <class CV>
static void emul_mul_batch(size_t n, const uint8_t* scalars, const uint8_t* pts, uint8_t* out) {
  for (size_t i = 0; i < n; i++) {
    Scalar256 k; scalar_load_be(k, scalars + 32 * i);
    Affine<typename CV::F> p; CV::load(p, pts + CV::IN_BYTES * i);
    Jac<typename CV::F> r; scalar_mul<CV>(r, k, p);
    Affine<typename CV::F> a; jac_to_affine(a, r);
    CV::store(out + CV::OUT_BYTES * i, a);
  }
}

struct EmulInv { template <class F> void operator()(F& r, const F& a) const { f_inv_bg(r, a); } };
static void emul_mul_batch_glv(size_t n, const uint8_t* scalars, const uint8_t* pts, uint8_t* out) {
  using CV = Bls381G1;
  for (size_t i = 0; i < n; i++) {
    Scalar256 k; scalar_load_be(k, scalars + 32 * i);
    Affine<CV::F> p; CV::load(p, pts + CV::IN_BYTES * i);
    Jac<CV::F> r; scalar_mul_glv_bls381(r, k, p, EmulInv{});
    Affine<CV::F> a; jac_to_affine(a, r);
    CV::store(out + CV::OUT_BYTES * i, a);
  }
}

template <class CV>
static void emul_mul_batch_w4(size_t n, const uint8_t* scalars, const uint8_t* pts, uint8_t* out) {
  for (size_t i = 0; i < n; i++) {
    Scalar256 k; scalar_load_be(k, scalars + 32 * i);
    Affine<typename CV::F> p; CV::load(p, pts + CV::IN_BYTES * i);
    Jac<typename CV::F> r; scalar_mul_w4<CV>(r, k, p, EmulInv{});
    Affine<typename CV::F> a; jac_to_affine(a, r);
    CV::store(out + CV::OUT_BYTES * i, a);
  }
}

// the device's plan (msm_host.cuh: make_plan): signed-digit recoding needs windows for scalar_bits + 1 bits
static MsmPlan emul_plan(int c, int m, int scalar_bits) {
  MsmPlan pl; pl.c = c; pl.W = (scalar_bits + c) / c; pl.nb = 1 << (c - 1); pl.m = m;
  // K = sum_w 2^(c-1) 2^(cw)
  uint32_t K[9] = {0};
  for (int w = 0; w < pl.W; w++) { int bit = c * w + c - 1; if (bit < 288) K[bit >> 5] |= 1u << (bit & 31); }
  memcpy(pl.K, K, sizeof K);
  return pl;
}

static int g_pt_stage = 0;        // emul_set_pt_stage: run the backward pass of the split rounds through the cp.async-staged variant
// digits, counting sort, (affine rounds,) accumulate, fix-up: the W x 2^(c-1) buckets of these pairs
template <class CV>
static int emul_msm_buckets(size_t n, const uint8_t* scalars, const uint8_t* pts, const MsmPlan& pl, std::vector<Xyzz<typename CV::F>>& B,
                            int L = 0, int rounds = 0, int PB = 8, bool split = false) {
  using F = typename CV::F;
  const int c = pl.c;
  std::vector<Affine<F>> P(n);
  for (size_t i = 0; i < n; i++) CV::load(P[i], pts + CV::IN_BYTES * i);
  size_t total = (size_t)pl.W * pl.nb;
  std::vector<uint32_t> counts(total + 1, 0), offs(total + 1, 0);
  for (size_t i = 0; i < n; i++) {
    Scalar256 s; scalar_load_be(s, scalars + 32 * i);
    if (!scalar_in_range<typename CV::ScalarField>(s)) return -3;
    uint32_t sp[9]; msm_recode(sp, s, pl.K);
    for (int w = 0; w < pl.W; w++) { int d = msm_digit(sp, c, w); if (d) counts[(size_t)w * pl.nb + (d < 0 ? -d : d) - 1]++; }
  }
  for (size_t g = 0; g < total; g++) offs[g + 1] = offs[g] + counts[g];
  std::vector<uint32_t> cursor(offs.begin(), offs.end()), entries(offs[total]);
  for (size_t i = 0; i < n; i++) {
    Scalar256 s; scalar_load_be(s, scalars + 32 * i);
    uint32_t sp[9]; msm_recode(sp, s, pl.K);
    for (int w = 0; w < pl.W; w++) { int d = msm_digit(sp, c, w); if (d) { size_t g = (size_t)w * pl.nb + (d < 0 ? -d : d) - 1; entries[cursor[g]++] = (uint32_t)i | (d < 0 ? 0x80000000u : 0); } }
  }
  B.assign(total, Xyzz<F>());
  if (L == 0) {
    for (size_t g = 0; g < total; g++) msm_accumulate_bucket<CV>(B[g], P.data(), entries.data(), offs[g], offs[g + 1]);
  } else {   // v2: fixed-length slices + fix-up (buckets start as all-zero = infinity, like cudaMemset)
    memset((void*)B.data(), 0, total * sizeof(Xyzz<F>));
    // affine pair-tree rounds (msm_affine.cuh): every round halves the operand list of every bucket
    std::vector<Affine<F>> cur;
    for (int r = 0; r < rounds; r++) {
      std::vector<uint32_t> no(total + 1, 0);
      for (size_t g = 0; g < total; g++) no[g + 1] = no[g] + ((offs[g + 1] - offs[g] + 1) >> 1);
      std::vector<Affine<F>> nxt(no[total] + 1);
      uint32_t T = (no[total] + PB - 1) / PB + 1;      // one thread past the end: must be a no-op
      if (split) {                                     // three kernels per round: forward / invert / backward
        std::vector<F> pre((size_t)T * PB), accs(T);
        for (uint32_t t = 0; t < T; t++) {
          if (g_pt_stage) {
            alignas(16) unsigned char slots[4 * sizeof(F)];
            memset(slots, 0xEE, sizeof slots);
            if (r == 0) msm_pairtree_forward_staged<CV, true>(t, (uint32_t)PB, T, (uint32_t)total, P.data(), entries.data(), offs.data(), no.data(), pre.data(), accs.data(), slots, 0);
            else msm_pairtree_forward_staged<CV, false>(t, (uint32_t)PB, T, (uint32_t)total, cur.data(), nullptr, offs.data(), no.data(), pre.data(), accs.data(), slots, 0);
            continue;
          }
          if (r == 0) msm_pairtree_forward<CV, true>(t, (uint32_t)PB, T, (uint32_t)total, P.data(), entries.data(), offs.data(), no.data(), pre.data(), accs.data());
          else msm_pairtree_forward<CV, false>(t, (uint32_t)PB, T, (uint32_t)total, cur.data(), nullptr, offs.data(), no.data(), pre.data(), accs.data());
        }
        for (uint32_t t = 0; t < T; t++) msm_pairtree_invert<F>(t, (uint32_t)PB, (uint32_t)total, no.data(), accs.data());
        for (uint32_t t = 0; t < T; t++) {
          if (g_pt_stage) {                            // operands staged by (emulated, deferred) cp.async: k_pt_backward_staged
            alignas(16) unsigned char slots[4 * sizeof(Affine<F>) + sizeof(F)];
            memset(slots, 0xEE, sizeof slots);
            if (r == 0) msm_pairtree_backward_staged<CV, true>(t, (uint32_t)PB, T, (uint32_t)total, P.data(), entries.data(), offs.data(), no.data(), pre.data(), accs.data(), nxt.data(), slots, 0);
            else msm_pairtree_backward_staged<CV, false>(t, (uint32_t)PB, T, (uint32_t)total, cur.data(), nullptr, offs.data(), no.data(), pre.data(), accs.data(), nxt.data(), slots, 0);
            continue;
          }
          if (r == 0) msm_pairtree_backward<CV, true>(t, (uint32_t)PB, T, (uint32_t)total, P.data(), entries.data(), offs.data(), no.data(), pre.data(), accs.data(), nxt.data());
          else msm_pairtree_backward<CV, false>(t, (uint32_t)PB, T, (uint32_t)total, cur.data(), nullptr, offs.data(), no.data(), pre.data(), accs.data(), nxt.data());
        }
      } else
      for (uint32_t t = 0; t < T; t++) {
        if (r == 0) msm_pairtree_round<CV, true>(t, (uint32_t)PB, (uint32_t)total, P.data(), entries.data(), offs.data(), no.data(), nxt.data());
        else msm_pairtree_round<CV, false>(t, (uint32_t)PB, (uint32_t)total, cur.data(), nullptr, offs.data(), no.data(), nxt.data());
      }
      cur.swap(nxt);
      offs.swap(no);
    }
    uint32_t E = offs[total];
    uint32_t S = (E + L - 1) / L;
    std::vector<Xyzz<F>> spart(2 * (size_t)S + 2);
    for (uint32_t j = 0; j < S; j++) {
      if (rounds) msm_accumulate_slice<CV, true>(j, (uint32_t)L, (uint32_t)total, cur.data(), offs.data(), nullptr, B.data(), spart.data());
      else msm_accumulate_slice<CV>(j, (uint32_t)L, (uint32_t)total, P.data(), offs.data(), entries.data(), B.data(), spart.data());
    }
    for (size_t g = 0; g < total; g++) {
      bool big = msm_fixup_bucket<CV, 3>((uint32_t)g, (uint32_t)L, offs.data(), B.data(), spart.data());
      if (big) {   // emulate the block-parallel path serially
        uint32_t s0 = offs[g], t0 = offs[g + 1], j0 = s0 / L, j1 = (t0 - 1) / L;
        Xyzz<F> a = spart[2 * (size_t)j0 + 1];
        for (uint32_t j = j0 + 1; j <= j1; j++) xyzz_add(a, a, spart[2 * (size_t)j]);
        B[g] = a;
      }
    }
  }
  return 0;
}

template <class CV>
static int emul_msm(size_t n, const uint8_t* scalars, const uint8_t* pts, int c, int m, uint8_t* out, int L = 0, int rounds = 0, int PB = 8, bool split = false) {
  using F = typename CV::F;
  MsmPlan pl = emul_plan(c, m, CV::SCALAR_BITS);
  std::vector<Xyzz<F>> B;
  int rc = emul_msm_buckets<CV>(n, scalars, pts, pl, B, L, rounds, PB, split);
  if (rc) return rc;
  int T = pl.nb / m;
  std::vector<Xyzz<F>> part((size_t)pl.W * T), wsum(pl.W);
  for (int w = 0; w < pl.W; w++) for (int t = 0; t < T; t++) msm_reduce_chunk<CV>(part[(size_t)w * T + t], &B[(size_t)w * pl.nb], t, m);
  for (int w = 0; w < pl.W; w++) { Xyzz<F> a; xyzz_set_inf(a); for (int t = 0; t < T; t++) xyzz_add(a, a, part[(size_t)w * T + t]); wsum[w] = a; }
  Xyzz<F> r; msm_horner<CV>(r, wsum.data(), pl.W, c);
  Affine<F> a; xyzz_to_affine(a, r);
  CV::store(out, a);
  return 0;
}

// Multi-GPU bucket exchange (msm_host.cuh: msm_buckets_dev / msm_reduce_windows_dev / msm_finish_dev) with `world`
// virtual ranks: contiguous shards of the pairs -> partial buckets per rank -> "all-to-all" (rank g gets windows
// [g wc, (g+1) wc) of every rank, layout [part][wc][nb]) -> msm_reduce_chunk_parts + window sums -> "all-gather" -> Horner.
template <class CV>
static int emul_msm_exchange(size_t n, const uint8_t* scalars, const uint8_t* pts, int c, int m, int L, int rounds, int PB, int world, uint8_t* out, int m2 = 0) {
  using F = typename CV::F;
  using X = Xyzz<F>;
  MsmPlan pl = emul_plan(c, m, CV::SCALAR_BITS);
  if (world < 1 || pl.W % world) return -2;
  const int wc = pl.W / world;
  std::vector<std::vector<X>> Bs(world);
  for (int r = 0; r < world; r++) {
    size_t lo = n * r / world, hi = n * (r + 1) / world;
    if (hi > lo) {
      int rc = emul_msm_buckets<CV>(hi - lo, scalars + 32 * lo, pts + CV::IN_BYTES * lo, pl, Bs[r], L, rounds, PB, true);
      if (rc) return rc;
    } else {
      Bs[r].resize((size_t)pl.W * pl.nb);
      memset((void*)Bs[r].data(), 0, Bs[r].size() * sizeof(X));
    }
  }
  std::vector<X> wsum(pl.W);
  const int T = pl.nb / m;
  for (int g = 0; g < world; g++) {
    std::vector<X> recv((size_t)world * wc * pl.nb);
    for (int p = 0; p < world; p++) memcpy((void*)&recv[(size_t)p * wc * pl.nb], (const void*)&Bs[p][(size_t)g * wc * pl.nb], (size_t)wc * pl.nb * sizeof(X));
    for (int w = 0; w < wc; w++) {
      X a; xyzz_set_inf(a);
      if (m2 > 0) {     // two-level reduction (msm_reduce_l1 / msm_reduce_l2): the window sum is the sum of all T + T/m2 partials
        if (T % m2) return -2;
        int lg = 0; while ((1 << lg) < m) lg++;
        std::vector<X> runs(T);
        for (int t = 0; t < T; t++) {
          X part;
          msm_reduce_l1<CV>(part, runs[t], &recv[(size_t)w * pl.nb], world, (size_t)wc * pl.nb, t, m);
          xyzz_add(a, a, part);
        }
        for (int u = 0; u < T / m2; u++) {
          X part;
          msm_reduce_l2<CV>(part, runs.data(), u, m2, lg);
          xyzz_add(a, a, part);
        }
      } else
      for (int t = 0; t < T; t++) {
        X part;
        msm_reduce_chunk_parts<CV>(part, &recv[(size_t)w * pl.nb], world, (size_t)wc * pl.nb, t, m);
        xyzz_add(a, a, part);
      }
      wsum[g * wc + w] = a;
    }
  }
  X r; msm_horner<CV>(r, wsum.data(), pl.W, c);
  Affine<F> a; xyzz_to_affine(a, r);
  CV::store(out, a);
  return 0;
}

extern "C" {
// two-level bucket reduction (m1, m2), single rank or `world` virtual ranks
int emul_bls12381_g1_msm_reduce2(size_t n, const uint8_t* s, const uint8_t* p, int c, int m1, int m2, int L, int world, uint8_t* o) {
  return emul_msm_exchange<Bls381G1>(n, s, p, c, m1, L, 0, 1, world, o, m2);
}
int emul_bn254_g1_msm_reduce2(size_t n, const uint8_t* s, const uint8_t* p, int c, int m1, int m2, int L, uint8_t* o) {
  return emul_msm_exchange<Bn254G1>(n, s, p, c, m1, L, 0, 1, 1, o, m2);
}
int emul_bls12381_g1_msm_exchange(size_t n, const uint8_t* s, const uint8_t* p, int c, int m, int L, int rounds, int PB, int world, uint8_t* o) {
  return emul_msm_exchange<Bls381G1>(n, s, p, c, m, L, rounds, PB, world, o);
}
void emul_bls12381_g1_mul_batch_w4(size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { emul_mul_batch_w4<Bls381G1>(n, s, p, o); }
void emul_bn254_g1_mul_batch_w4(size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { emul_mul_batch_w4<Bn254G1>(n, s, p, o); }
void emul_bls12381_g1_mul_batch_glv(size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { emul_mul_batch_glv(n, s, p, o); }
void emul_bls12381_g1_mul_batch(size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { emul_mul_batch<Bls381G1>(n, s, p, o); }
int emul_bls12381_g1_msm(size_t n, const uint8_t* s, const uint8_t* p, int c, int m, uint8_t* o) { return emul_msm<Bls381G1>(n, s, p, c, m, o); }
// GLV front end + the same pipeline over the 2n split pairs
int emul_bls12381_g1_msm_glv(size_t n, const uint8_t* s, const uint8_t* p, int c, int m, int L, uint8_t* o) {
  std::vector<uint8_t> vs(64 * n), vp(192 * n);
  for (size_t i = 0; i < n; i++) {
    Scalar256 k; scalar_load_be(k, s + 32 * i);
    if (!scalar_in_range<Bls381Fr>(k)) return -3;
    GlvSplit sp; glv_split_bls381(sp, k);
    Affine<Fp<Bls381Fp>> p0, p1, p2;
    Bls381G1::load(p0, p + 96 * i);
    glv_points_bls381(p1, p2, p0, sp);
    Bls381G1::store_affine(&vp[96 * i], p1); Bls381G1::store_affine(&vp[96 * (n + i)], p2);
    for (int j = 0; j < 8; j++) for (int b = 0; b < 4; b++) {
      vs[32 * i + 4 * j + b] = (uint8_t)(sp.k1.v[7 - j] >> (24 - 8 * b));
      vs[32 * (n + i) + 4 * j + b] = (uint8_t)(sp.k2.v[7 - j] >> (24 - 8 * b));
    }
  }
  return emul_msm<Bls381G1>(2 * n, vs.data(), vp.data(), c, m, o, L);
}
// k -> k1 (32 B BE), k2 (32 B BE), flags bit0 = neg1, bit1 = neg2
int emul_glv_split_bls381(const uint8_t* k32, uint8_t* k1, uint8_t* k2) {
  Scalar256 k; scalar_load_be(k, k32);
  GlvSplit sp; glv_split_bls381(sp, k);
  for (int j = 0; j < 8; j++) for (int b = 0; b < 4; b++) { k1[4 * j + b] = (uint8_t)(sp.k1.v[7 - j] >> (24 - 8 * b)); k2[4 * j + b] = (uint8_t)(sp.k2.v[7 - j] >> (24 - 8 * b)); }
  return (sp.neg1 ? 1 : 0) | (sp.neg2 ? 2 : 0);
}
// balanced slices after `rounds` affine pair-tree rounds with PB outputs per thread
int emul_bls12381_g1_msm_affine(size_t n, const uint8_t* s, const uint8_t* p, int c, int m, int L, int rounds, int PB, uint8_t* o) { return emul_msm<Bls381G1>(n, s, p, c, m, o, L, rounds, PB); }
int emul_bls12381_g1_msm_affine_split(size_t n, const uint8_t* s, const uint8_t* p, int c, int m, int L, int rounds, int PB, uint8_t* o) { return emul_msm<Bls381G1>(n, s, p, c, m, o, L, rounds, PB, true); }
int emul_bn254_g1_msm_affine(size_t n, const uint8_t* s, const uint8_t* p, int c, int m, int L, int rounds, int PB, uint8_t* o) { return emul_msm<Bn254G1>(n, s, p, c, m, o, L, rounds, PB); }
int emul_bls12381_g1_msm_v2(size_t n, const uint8_t* s, const uint8_t* p, int c, int m, int L, uint8_t* o) { return emul_msm<Bls381G1>(n, s, p, c, m, o, L); }
void emul_bn254_g1_mul_batch(size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { emul_mul_batch<Bn254G1>(n, s, p, o); }
int emul_bn254_g1_msm(size_t n, const uint8_t* s, const uint8_t* p, int c, int m, uint8_t* o) { return emul_msm<Bn254G1>(n, s, p, c, m, o); }
}

// ------------------------------------------------------------------------------------------------
#include "../../kyber_b200/csrc/pairing.cuh"
extern "C" {
void emul_bls12381_pair(const uint8_t* g1, const uint8_t* g2, uint8_t* gt576) {
  Affine<BFp> P; Affine<BFp2> Q;
  Bls381G1::load(P, g1); g2_load(Q, g2);
  BFp12 f, e;
  miller_loop<1>(f, &P, &Q);
  final_exponentiation(e, f);
  gt_store(gt576, e);
}
// final_exponentiation (exponent 3(p^12-1)/r) == final_exponentiation_exact cubed, on a Miller-loop output
int emul_bls12381_final_exp_is_exact_cubed(const uint8_t* g1, const uint8_t* g2) {
  Affine<BFp> P; Affine<BFp2> Q;
  Bls381G1::load(P, g1); g2_load(Q, g2);
  BFp12 f, e, x, x3;
  miller_loop<1>(f, &P, &Q);
  final_exponentiation(e, f);
  final_exponentiation_exact(x, f);
  fp12_sqr(x3, x); fp12_mul(x3, x3, x);
  uint8_t a[576], b[576];
  gt_store(a, e); gt_store(b, x3);
  for (int i = 0; i < 576; i++) if (a[i] != b[i]) return 0;
  return 1;
}
// e(a1,a2) == e(b1,b2)
int emul_bls12381_pairing_check(const uint8_t* a1, const uint8_t* a2, const uint8_t* b1, const uint8_t* b2) {
  Affine<BFp> P[2]; Affine<BFp2> Q[2];
  Bls381G1::load(P[0], a1); g2_load(Q[0], a2);
  Bls381G1::load(P[1], b1); g2_load(Q[1], b2);
  fp_neg(P[1].y, P[1].y);
  BFp12 f, e;
  miller_loop<2>(f, P, Q);
  final_exponentiation(e, f);
  return fp12_is_one(e) ? 1 : 0;
}
}

// ------------------------------------------------------------------------------------------------
#include "../../kyber_b200/csrc/codec.cuh"
extern "C" {
int emul_bls12381_g1_decompress(const uint8_t* in48, uint8_t* out96) {
  Affine<BFp> a;
  bool ok = g1_decompress(a, in48, true);
  if (ok) Bls381G1::store_affine(out96, a);
  return ok ? 1 : 0;
}
int emul_bls12381_g2_decompress(const uint8_t* in96, uint8_t* out192) {
  Affine<BFp2> a;
  bool ok = g2_decompress(a, in96, true);
  if (ok) Bls381G2::store_affine(out192, a);
  return ok ? 1 : 0;
}
void emul_bls12381_g2_mul_batch_w4(size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { emul_mul_batch_w4<Bls381G2>(n, s, p, o); }
void emul_bls12381_g2_mul_batch(size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { emul_mul_batch<Bls381G2>(n, s, p, o); }
int emul_bls12381_g2_msm(size_t n, const uint8_t* s, const uint8_t* p, int c, int m, int L, uint8_t* o) { return emul_msm<Bls381G2>(n, s, p, c, m, o, L); }
}

// ------------------------------------------------------------------------------------------------
// the MSM template over the other groups: bn254 G2 (Fp2, 8 limbs), bn256 G1 (10 limbs) and bn256 G2 (Fp2, 10 limbs)
#include "../../kyber_b200/csrc/bn_pairing.cuh"
#include "../../kyber_b200/csrc/bn256.cuh"
extern "C" {
int emul_bn254_g2_msm(size_t n, const uint8_t* s, const uint8_t* p, int c, int m, int L, uint8_t* o) { return emul_msm<Bn254G2>(n, s, p, c, m, o, L); }
int emul_bn256_g1_msm(size_t n, const uint8_t* s, const uint8_t* p, int c, int m, int L, uint8_t* o) { return emul_msm<Bn256G1>(n, s, p, c, m, o, L); }
int emul_bn256_g2_msm(size_t n, const uint8_t* s, const uint8_t* p, int c, int m, int L, uint8_t* o) { return emul_msm<Bn256G2>(n, s, p, c, m, o, L); }
}
extern "C" void emul_set_pt_stage(int on) { g_pt_stage = on; }
