// msm.cuh -- per-thread bodies of the batched scalar-multiplication and Pippenger MSM kernels.
//
// Replaces (reference call sites; the reference has no batched entry point, only Go loops):
//   kilic.G1Elt.Mul                    pairing/bls12381/kilic/g1.go:110-116   (one s*P per call)
//   bn254 curvePoint.Mul               pairing/bn254/curve.go:196-218
//   the loops  Tmp.Mul(l_i, y_i); Acc.Add(Acc, Tmp)   share/poly.go:461-473 (RecoverCommit)
//              sig.Mul(coef, sig); agg.Add(...)       sign/bdn/bdn.go:126-161 (AggregateSignatures)
//
// MSM pipeline (window c bits, W = ceil(256/c) windows, signed digits -> 2^(c-1) buckets/window):
//   digits+count  : s' = s + K (K = sum of 2^(c-1) at every window) so that window digits of s' minus
//                   2^(c-1) are the signed digits; histogram of (window, |digit|) by atomics (in the pass that loads the
//                   points, into window-major int16 digit columns: msm_sort.cuh)
//   scan          : exclusive prefix sum of the histogram -> bucket start offsets
//   scatter       : counting sort of (point index | sign) by bucket, coarse partition + bin sort (msm_sort.cuh)
//   accumulate    : one thread per bucket, XYZZ += +-P (mixed add 8M+2S), points gathered by index
//   reduce        : per (window, chunk of m buckets): running sums  A = sum (k-k0) B_k,  S = sum B_k,
//                   partial = A + k0*S ; then per-window tree sum of the partials
//   final         : Horner over windows (c doublings per window), to affine, to wire bytes
// The per-thread bodies below are plain functions of explicit indices so that tests/host_emul can run
// them on the CPU; the __global__ wrappers live in kernels.cu.
#pragma once
#include <stddef.h>
#include "curves.cuh"

namespace b2k {

struct MsmPlan {
  int c;           // window bits, 2..16
  int W;           // windows
  int nb;          // buckets per window = 2^(c-1)
  int m;           // reduction chunk (power of two, divides nb)
  uint32_t K[9];   // recoding offset, little-endian limbs
};

// signed digit of window w of s' (s' given as 9 limbs):  returns d in [-2^(c-1), 2^(c-1)-1]
B2K_D int msm_digit(const uint32_t* sp, int c, int w) {
  int bit = c * w;
  int limb = bit >> 5, sh = bit & 31;
  uint64_t two = (uint64_t)sp[limb] | ((uint64_t)(limb + 1 < 9 ? sp[limb + 1] : 0u) << 32);
  uint32_t e = (uint32_t)(two >> sh) & ((1u << c) - 1u);
  return (int)e - (1 << (c - 1));
}

// s' = s + K  (9 limbs)
B2K_D void msm_recode(uint32_t* sp, const Scalar256& s, const uint32_t* K) {
  sp[0] = ptx::add_cc(s.v[0], K[0]);
#pragma unroll
  for (int j = 1; j < 8; j++) sp[j] = ptx::addc_cc(s.v[j], K[j]);
  sp[8] = ptx::addc(0, K[8]);
}

// ---- accumulate: one bucket -----------------------------------------------------------------
// entries[start..end) hold (point index | sign << 31)
template <class CV>
B2K_D void msm_accumulate_bucket(Xyzz<typename CV::F>& acc, const Affine<typename CV::F>* pts,
                                 const uint32_t* entries, uint32_t start, uint32_t end) {
  xyzz_set_inf(acc);
  for (uint32_t e = start; e < end; e++) {
    uint32_t v = entries[e];
    Affine<typename CV::F> q = pts[v & 0x7fffffffu];
    xyzz_madd(acc, acc, q, (v >> 31) != 0);
  }
}

// ---- reduce: one chunk of m consecutive buckets ------------------------------------------------
// buckets of this window: B[0..nb) where B[k] holds digit magnitude k+1.  Chunk t covers k in
// [t*m, (t+1)*m).  partial = sum_{k} (k+1) * B[k].
template <class CV>
B2K_D void msm_reduce_chunk(Xyzz<typename CV::F>& out, const Xyzz<typename CV::F>* B, int t, int m) {
  using X = Xyzz<typename CV::F>;
  X run, acc;
  xyzz_set_inf(run);
  xyzz_set_inf(acc);
  for (int k = m - 1; k >= 0; k--) {
    X b = B[t * m + k];
    xyzz_add(run, run, b);
    xyzz_add(acc, acc, run);      // after the loop: acc = sum (k+1) B[t*m+k], run = sum B
  }
  if (t != 0) {
    X off;
    xyzz_mul_small(off, run, (uint32_t)(t * m));
    xyzz_add(acc, acc, off);
  }
  out = acc;
}

// Multi-GPU bucket exchange (SURVEY 8e shape 1): the buckets of a window arrive as `parts` partial arrays, one per
// rank, laid out [part][stride]; the bucket-wise EC addition of the partials is fused into the chunk reduction, which
// reads the receive buffer of the all-to-all directly.  B points at bucket 0 of the window inside part 0.
template <class CV>
B2K_D void msm_reduce_chunk_parts(Xyzz<typename CV::F>& out, const Xyzz<typename CV::F>* B, int parts, size_t stride, int t, int m) {
  using X = Xyzz<typename CV::F>;
  X run, acc;
  xyzz_set_inf(run);
  xyzz_set_inf(acc);
  for (int k = m - 1; k >= 0; k--) {
    X b = B[t * m + k];
    for (int p = 1; p < parts; p++) {
      X q = B[(size_t)p * stride + (size_t)(t * m + k)];
      xyzz_add(b, b, q);
    }
    xyzz_add(run, run, b);
    xyzz_add(acc, acc, run);
  }
  if (t != 0) {
    X off;
    xyzz_mul_small(off, run, (uint32_t)(t * m));
    xyzz_add(acc, acc, off);
  }
  out = acc;
}

// ---- two-level bucket reduction ---------------------------------------------------------------------------------------
// The chunk offset (t m) * run of msm_reduce_chunk is a ~13-bit double-and-add PER CHUNK: half of the single-level
// reduction's field products, and divergent inside a warp.  Two levels move it to where there are m1 times fewer operands:
//   level 1, chunk t of m1 buckets:   acc_t = sum_j (j+1) B[t m1 + j],   run_t = sum_j B[t m1 + j]          (no scalar mul)
//   window sum = sum_t acc_t + m1 * sum_t t * run_t
//   level 2, chunk u of m2 runs:      m1 * sum_v (u m2 + v) run_{u m2 + v}     (running sums + ONE small scalar mul per m1 m2 buckets)
// Both outputs go into one partials array ([T1 level-1 sums][T1/m2 level-2 sums] per window) that k_msm_window_sum adds up.
// `parts`/`stride`: the bucket is the sum of `parts` partial arrays (multi-GPU bucket exchange), 1/0 otherwise.
// Units in the by-reference Fp2 layout (tower.cuh: B2K_FP2_BYREF): the three Fp2 points live across an addition would leave the
// field products underneath too few registers, so there the additions are out of line and the points stay in memory.
template <class F>
B2K_NI void xyzz_add_ool(Xyzz<F>& r, const Xyzz<F>& p, const Xyzz<F>& q) { xyzz_add(r, p, q); }
template <class F>
B2K_D void xyzz_add_reduce(Xyzz<F>& r, const Xyzz<F>& p, const Xyzz<F>& q) {
#ifdef B2K_FP2_BYREF
  if constexpr (sizeof(F) > 48) { xyzz_add_ool(r, p, q); return; }
#endif
  xyzz_add(r, p, q);
}
template <class CV>
B2K_D void msm_reduce_l1(Xyzz<typename CV::F>& acc_out, Xyzz<typename CV::F>& run_out, const Xyzz<typename CV::F>* B,
                         int parts, size_t stride, int t, int m1) {
  using X = Xyzz<typename CV::F>;
  X run, acc;
  xyzz_set_inf(run);
  xyzz_set_inf(acc);
  for (int k = m1 - 1; k >= 0; k--) {
    X b = B[t * m1 + k];
    for (int p = 1; p < parts; p++) {
      X q = B[(size_t)p * stride + (size_t)(t * m1 + k)];
      xyzz_add_reduce(b, b, q);
    }
    xyzz_add_reduce(run, run, b);
    xyzz_add_reduce(acc, acc, run);
  }
  acc_out = acc;
  run_out = run;
}
// R = the T1 level-1 run sums of one window; out = m1 * sum_{v < m2} (u m2 + v) R[u m2 + v],  m1 = 2^log2_m1
template <class CV>
B2K_D void msm_reduce_l2(Xyzz<typename CV::F>& out, const Xyzz<typename CV::F>* R, int u, int m2, int log2_m1) {
  using X = Xyzz<typename CV::F>;
  X run, acc;
  xyzz_set_inf(run);
  xyzz_set_inf(acc);
  for (int v = m2 - 1; v >= 1; v--) {
    X b = R[u * m2 + v];
    xyzz_add(run, run, b);
    xyzz_add(acc, acc, run);      // after the loop: acc = sum v R[u m2 + v]
  }
  if (u != 0) {
    X b = R[u * m2];
    xyzz_add(run, run, b);        // run = sum R
    X off;
    xyzz_mul_small(off, run, (uint32_t)(u * m2));
    xyzz_add(acc, acc, off);
  }
  for (int i = 0; i < log2_m1; i++) xyzz_dbl(acc, acc);
  out = acc;
}

// ---- final: Horner over window sums --------------------------------------------------------------
template <class CV>
B2K_D void msm_horner(Xyzz<typename CV::F>& out, const Xyzz<typename CV::F>* wsum, int W, int c) {
  using X = Xyzz<typename CV::F>;
  X acc = wsum[W - 1];
  for (int w = W - 2; w >= 0; w--) {
    for (int i = 0; i < c; i++) xyzz_dbl(acc, acc);
    X t = wsum[w];
    xyzz_add(acc, acc, t);
  }
  out = acc;
}

// ---- GLV split for BLS12-381 G1 ---------------------------------------------------------------------
// phi(x, y) = (beta x, y) acts on G1 as multiplication by lambda = -x^2 (x the curve parameter, r = x^4 - x^2 + 1), so with
// k (or r - k, whichever is smaller) = q X2 +- rem,  X2 = x^2,  |rem| <= X2/2:
//      k P = s ( +-rem P + q (-phi(P)) ),     rem, q < 2^127.
// The MSM then runs over 2n points and 127-bit scalars: half the windows to reduce and half the doublings in the final
// Horner chain for the same number of bucket additions.  (The reference's bn254 Mul uses the same idea on one point,
// pairing/bn254/curve.go:196-218 with lattice.go:47-108; here the split is exact division by x^2.)
struct GlvSplit { Scalar256 k1, k2; bool neg1, neg2; };

constexpr int GLV_BITS_BLS381 = 127;

// out[0..NA+NB) = a * b   (32-bit limbs, plain C: runs unchanged in the host emulation; sizes are compile-time so that
// everything unrolls into registers)
template <int NA, int NB>
B2K_D void limbs_mul(uint32_t* out, const uint32_t* a, const uint32_t* b) {
#pragma unroll
  for (int i = 0; i < NA + NB; i++) out[i] = 0;
#pragma unroll
  for (int i = 0; i < NA; i++) {
    uint64_t carry = 0;
#pragma unroll
    for (int j = 0; j < NB; j++) {
      uint64_t t = (uint64_t)a[i] * b[j] + out[i + j] + carry;
      out[i + j] = (uint32_t)t;
      carry = t >> 32;
    }
    out[i + NB] = (uint32_t)carry;
  }
}
// a -= b over N limbs, returns the borrow
template <int N>
B2K_D uint32_t limbs_sub(uint32_t* a, const uint32_t* b) {
  uint64_t br = 0;
#pragma unroll
  for (int i = 0; i < N; i++) {
    uint64_t d = (uint64_t)a[i] - b[i] - br;
    a[i] = (uint32_t)d;
    br = (d >> 32) & 1u;
  }
  return (uint32_t)br;
}
// a >= b  <=>  a - b does not borrow
template <int N>
B2K_D bool limbs_geq(const uint32_t* a, const uint32_t* b) {
  uint64_t br = 0;
#pragma unroll
  for (int i = 0; i < N; i++) br = (((uint64_t)a[i] - b[i] - br) >> 32) & 1u;
  return br == 0;
}
template <int N>
B2K_D void limbs_inc(uint32_t* a) {
  uint32_t c = 1;
#pragma unroll
  for (int j = 0; j < N; j++) { a[j] += c; c = (c && a[j] == 0) ? 1u : 0u; }
}

B2K_D void glv_split_bls381(GlvSplit& out, const Scalar256& k) {
  // x^2 = 0xac45a401 0001a402 00000001 00000000 (128 bits), mu = floor(2^256 / x^2) (129 bits)
  const uint32_t XX[5] = {0x00000000u, 0x00000001u, 0x0001a402u, 0xac45a401u, 0u};
  const uint32_t MU[5] = {0xf6cfee2eu, 0x63f6e522u, 0xe01faaddu, 0x7c6becf1u, 0x1u};
  uint32_t kk[8], t[8];
  bool neg = false;
#pragma unroll
  for (int j = 0; j < 8; j++) { kk[j] = k.v[j]; t[j] = Bls381Fr::mod(j); }
  limbs_sub<8>(t, kk);                              // r - k  (k < r is checked by the caller)
  if (!limbs_geq<8>(t, kk)) {
#pragma unroll
    for (int j = 0; j < 8; j++) kk[j] = t[j];
    neg = true;
  }
  uint32_t prod[13], q[5], qx[10], rem[5];
  limbs_mul<8, 5>(prod, kk, MU);
#pragma unroll
  for (int j = 0; j < 5; j++) q[j] = prod[8 + j];   // floor(kk mu / 2^256) in {Q-1, Q}
  limbs_mul<5, 5>(qx, q, XX);
#pragma unroll
  for (int j = 0; j < 5; j++) rem[j] = kk[j];
  limbs_sub<5>(rem, qx);                            // kk - q x^2 < 2 x^2 < 2^129: 160 bits are enough
  if (limbs_geq<5>(rem, XX)) {
    limbs_sub<5>(rem, XX);
    limbs_inc<5>(q);
  }
  // balance: 2 rem > x^2  ->  rem = x^2 - rem, q += 1, sign flipped
  uint32_t dbl[5];
#pragma unroll
  for (int j = 4; j > 0; j--) dbl[j] = (rem[j] << 1) | (rem[j - 1] >> 31);
  dbl[0] = rem[0] << 1;
  bool negr = false;
  if (!limbs_geq<5>(XX, dbl)) {
    uint32_t x2[5];
#pragma unroll
    for (int j = 0; j < 5; j++) x2[j] = XX[j];
    limbs_sub<5>(x2, rem);
#pragma unroll
    for (int j = 0; j < 5; j++) rem[j] = x2[j];
    limbs_inc<5>(q);
    negr = true;
  }
#pragma unroll
  for (int j = 0; j < 8; j++) { out.k1.v[j] = j < 4 ? rem[j] : 0u; out.k2.v[j] = j < 4 ? q[j] : 0u; }
  out.neg1 = neg != negr;
  out.neg2 = neg;
}

// the two points of the split: p1 = +-P, p2 = +-(-phi(P)) = (beta x, -+y); infinity (0,0) maps to itself
B2K_D void glv_points_bls381(Affine<Fp<Bls381Fp>>& p1, Affine<Fp<Bls381Fp>>& p2, const Affine<Fp<Bls381Fp>>& p, const GlvSplit& sp) {
  Fp<Bls381Fp> beta;
#pragma unroll
  for (int j = 0; j < 12; j++) beta.v[j] = Bls381Fp::beta(j);
  fp_mul(p2.x, p.x, beta);
  p2.y = p.y;
  if (!sp.neg2) fp_neg(p2.y, p2.y);
  p1 = p;
  if (sp.neg1) fp_neg(p1.y, p1.y);
}

// ---- independent scalar multiplication -----------------------------------------------------------
// k*P, MSB-first double-and-add over the 256-bit scalar (Jacobian, mixed additions).
template <class CV>
B2K_D void scalar_mul(Jac<typename CV::F>& r, const Scalar256& k, const Affine<typename CV::F>& p) {
  Jac<typename CV::F> acc;
  jac_set_inf(acc);
  bool started = false;
  for (int i = 255; i >= 0; i--) {
    if (started) jac_dbl(acc, acc);
    if ((k.v[i >> 5] >> (i & 31)) & 1u) {
      jac_madd(acc, acc, p);
      started = true;
    }
  }
  r = acc;
}

// ---- independent scalar multiplication, fixed signed windows (every curve) ---------------------------------------------
// k P over signed radix-16 digits of the full 256-bit scalar and one affine table {P .. 8P}: 65 x (4 doublings + 1 mixed
// addition), the same instruction stream in every lane (scalar_mul above pays an addition per bit as soon as ONE lane of
// the warp has that bit set).  Valid for any k < 2^256 and any point of the curve: a table entry j P (j <= 8) that is
// infinity -- BLS12-381 G1 has points of order 3, such as (0, +-2); the G2 twists and the bn254 / bn256 curves have no points of
// order <= 8 -- is left out of the batched inversion and stored as the affine infinity (0, 0), which jac_madd adds as a no-op.
template <class CV, class INV>
B2K_D void scalar_mul_w4(Jac<typename CV::F>& r, const Scalar256& k, const Affine<typename CV::F>& p, INV inv_fn) {
  using F = typename CV::F;
  if (aff_is_inf(p)) { jac_set_inf(r); return; }
  Affine<F> tab[8];
  tab[0] = p;
  {
    Jac<F> tj[8];
    jac_from_affine(tj[0], p);
    jac_dbl(tj[1], tj[0]);
    for (int j = 2; j < 8; j++) jac_madd(tj[j], tj[j - 1], p);
    F pre[8], acc, zi, zi2;
    f_set_one(acc);
    for (int j = 1; j < 8; j++) {
      pre[j] = acc;
      if (!jac_is_inf(tj[j])) f_mul(acc, acc, tj[j].Z);
    }
    inv_fn(acc, acc);
    for (int j = 7; j >= 1; j--) {
      if (jac_is_inf(tj[j])) { aff_set_inf(tab[j]); continue; }
      f_mul(zi, acc, pre[j]);
      f_mul(acc, acc, tj[j].Z);
      f_sqr(zi2, zi);
      f_mul(tab[j].x, tj[j].X, zi2);
      f_mul(zi2, zi2, zi);
      f_mul(tab[j].y, tj[j].Y, zi2);
    }
  }
  // s' = s + 0x888..8 (65 nibbles = 260 bits), top-aligned in 9 limbs; nibble_i(s') - 8 is the signed digit
  uint32_t d[9];
  {
    uint32_t a[9];
    uint64_t c = 0;
    for (int j = 0; j < 9; j++) {
      uint64_t t = (uint64_t)(j < 8 ? k.v[j] : 0u) + (j < 8 ? 0x88888888u : 0x8u) + c;
      a[j] = (uint32_t)t; c = t >> 32;
    }
    for (int j = 8; j > 0; j--) d[j] = (a[j] << 28) | (a[j - 1] >> 4);
    d[0] = a[0] << 28;
  }
  Jac<F> acc;
  jac_set_inf(acc);
  for (int i = 64; i >= 0; i--) {
    if (i != 64) { jac_dbl(acc, acc); jac_dbl(acc, acc); jac_dbl(acc, acc); jac_dbl(acc, acc); }
    const int e = (int)(d[8] >> 28) - 8;
    for (int j = 8; j > 0; j--) d[j] = (d[j] << 4) | (d[j - 1] >> 28);
    d[0] <<= 4;
    if (e) {
      Affine<F> q = tab[(e < 0 ? -e : e) - 1];
      if (e < 0) f_neg(q.y, q.y);
      jac_madd(acc, acc, q);
    }
  }
  r = acc;
}

// ---- independent scalar multiplication on BLS12-381 G1 with the endomorphism -----------------------------------------
// k P = +-k1 P + k2 (-phi P) with 127-bit k1, k2 (glv_split_bls381), both walked together in signed radix-16 digits over
// ONE affine table {P, 2P .. 8P} (phi maps the table: x -> beta x): 33 x (4 doublings + 2 mixed additions) instead of
// 255 doublings + ~128 additions, and every lane of a warp does the same work in every step (a double-and-add loop pays
// the addition whenever ANY lane has a set bit).  The table is normalised with one batched inversion.
// Requires P in the order-r subgroup (operands are what UnmarshalBinary accepted, kilic/g1.go:127-131), like the MSM's
// front end; the reference's bn254 Mul uses the same decomposition (pairing/bn254/curve.go:196-218).
template <class F, class INV>
B2K_D void scalar_mul_glv_bls381(Jac<F>& r, const Scalar256& k, const Affine<F>& p, INV inv_fn) {
  if (aff_is_inf(p)) { jac_set_inf(r); return; }
  GlvSplit sp;
  glv_split_bls381(sp, k);
  // table j P, j = 1..8: Jacobian chain, then to affine with one inversion (Z_1 = 1)
  Jac<F> tj[8];
  jac_from_affine(tj[0], p);
  jac_dbl(tj[1], tj[0]);
  for (int j = 2; j < 8; j++) jac_madd(tj[j], tj[j - 1], p);
  Affine<F> tab[8];
  tab[0] = p;
  {
    F pre[8], acc, zi, zi2;
    f_set_one(acc);
    for (int j = 1; j < 8; j++) { pre[j] = acc; f_mul(acc, acc, tj[j].Z); }     // j P is never infinity for j < r
    inv_fn(acc, acc);
    for (int j = 7; j >= 1; j--) {
      f_mul(zi, acc, pre[j]);
      f_mul(acc, acc, tj[j].Z);
      f_sqr(zi2, zi);
      f_mul(tab[j].x, tj[j].X, zi2);
      f_mul(zi2, zi2, zi);
      f_mul(tab[j].y, tj[j].Y, zi2);
    }
  }
  // s' = s + 0x888..8 (33 nibbles): nibble_i(s') - 8 is the signed digit; kept top-aligned in 5 limbs (160 bits >= 132 + 28)
  uint32_t d1[5], d2[5];
  {
    const uint32_t KK[5] = {0x88888888u, 0x88888888u, 0x88888888u, 0x88888888u, 0x8u};
    uint64_t c1 = 0, c2 = 0;
    uint32_t a1[5], a2[5];
    for (int j = 0; j < 5; j++) {
      uint64_t t1 = (uint64_t)(j < 4 ? sp.k1.v[j] : 0u) + KK[j] + c1; a1[j] = (uint32_t)t1; c1 = t1 >> 32;
      uint64_t t2 = (uint64_t)(j < 4 ? sp.k2.v[j] : 0u) + KK[j] + c2; a2[j] = (uint32_t)t2; c2 = t2 >> 32;
    }
    for (int j = 4; j > 0; j--) { d1[j] = (a1[j] << 28) | (a1[j - 1] >> 4); d2[j] = (a2[j] << 28) | (a2[j - 1] >> 4); }
    d1[0] = a1[0] << 28; d2[0] = a2[0] << 28;
  }
  F beta;
  for (int j = 0; j < F::N; j++) beta.v[j] = Bls381Fp::beta(j);
  Jac<F> acc;
  jac_set_inf(acc);
  for (int i = 32; i >= 0; i--) {
    if (i != 32) { jac_dbl(acc, acc); jac_dbl(acc, acc); jac_dbl(acc, acc); jac_dbl(acc, acc); }
    const int e1 = (int)(d1[4] >> 28) - 8, e2 = (int)(d2[4] >> 28) - 8;
    for (int j = 4; j > 0; j--) { d1[j] = (d1[j] << 4) | (d1[j - 1] >> 28); d2[j] = (d2[j] << 4) | (d2[j - 1] >> 28); }
    d1[0] <<= 4; d2[0] <<= 4;
    if (e1) {                                       // +-|e1| P, sign = neg1 xor (e1 < 0)
      Affine<F> q = tab[(e1 < 0 ? -e1 : e1) - 1];
      if (sp.neg1 != (e1 < 0)) f_neg(q.y, q.y);
      jac_madd(acc, acc, q);
    }
    if (e2) {                                       // +-|e2| (-phi P) = (beta x, -+y): y keeps its sign iff neg2 xor (e2 < 0)
      Affine<F> q = tab[(e2 < 0 ? -e2 : e2) - 1];
      f_mul(q.x, q.x, beta);
      if (sp.neg2 == (e2 < 0)) f_neg(q.y, q.y);
      jac_madd(acc, acc, q);
    }
  }
  r = acc;
}

}  // namespace b2k

// =================================================================================================
// v2 accumulate: fixed-length slices of the sorted entry list (perfectly balanced, skew-proof)
// =================================================================================================
// The sorted entries are cut into slices of L consecutive entries regardless of bucket boundaries;
// one thread per slice performs exactly L mixed additions.  A bucket that lies entirely inside a
// slice is written straight to buckets[]; a bucket cut by a slice boundary gets one partial sum per
// slice it touches (spart[2*j+0] if it started before slice j, spart[2*j+1] if it starts inside slice
// j and runs past its end) and msm_fixup_bucket() adds the partials.  Work per thread is independent
// of the scalar distribution (all-equal scalars, 128-bit BDN coefficients, short top windows ...).
namespace b2k {

// largest g in [0,total) with offs[g] <= pos   (offs non-decreasing, offs[0] = 0, offs[total] > pos)
B2K_D uint32_t msm_find_bucket(const uint32_t* offs, uint32_t total, uint32_t pos) {
  uint32_t lo = 0, hi = total;
  while (hi - lo > 1) {
    uint32_t mid = lo + ((hi - lo) >> 1);
    if (offs[mid] <= pos) lo = mid; else hi = mid;
  }
  return lo;
}

template <class CV>
B2K_D void msm_slice_flush(const Xyzz<typename CV::F>& acc, uint32_t g, uint32_t s, uint32_t t, uint32_t j,
                           uint32_t b, uint32_t e, Xyzz<typename CV::F>* buckets, Xyzz<typename CV::F>* spart) {
  if (s >= b && t <= e) buckets[g] = acc;
  else spart[2 * (size_t)j + (s < b ? 0 : 1)] = acc;
}

// DIRECT: the sorted operands themselves are in pts[] (output of the affine pair-tree rounds, msm_affine.cuh), no entries
template <class CV, bool DIRECT = false>
B2K_D void msm_accumulate_slice(uint32_t j, uint32_t L, uint32_t total, const Affine<typename CV::F>* pts,
                                const uint32_t* offs, const uint32_t* entries,
                                Xyzz<typename CV::F>* buckets, Xyzz<typename CV::F>* spart) {
  const uint32_t E = offs[total];
  const uint32_t b = j * L;
  if (b >= E) return;
  const uint32_t e = (E - b < L) ? E : b + L;
  uint32_t g = msm_find_bucket(offs, total, b);
  uint32_t gs = offs[g], ge = offs[g + 1];
  Xyzz<typename CV::F> acc;
  xyzz_set_inf(acc);
  for (uint32_t pos = b; pos < e; pos++) {
    if (pos == ge) {                       // crossed into a later bucket
      msm_slice_flush<CV>(acc, g, gs, ge, j, b, e, buckets, spart);
      xyzz_set_inf(acc);
      do { g++; gs = ge; ge = offs[g + 1]; } while (ge <= pos);
    }
    if (DIRECT) {
      Affine<typename CV::F> q = pts[pos];
      xyzz_madd(acc, acc, q, false);
    } else {
      uint32_t v = entries[pos];
      Affine<typename CV::F> q = pts[v & 0x7fffffffu];
      xyzz_madd(acc, acc, q, (v >> 31) != 0);
    }
  }
  msm_slice_flush<CV>(acc, g, gs, ge, j, b, e, buckets, spart);
}

// Combine the partials of a bucket that was cut by slice boundaries.  Returns true when the bucket has
// more than SERIAL_MAX partials (left to the block-parallel path), false when done / nothing to do.
template <class CV, int SERIAL_MAX>
B2K_D bool msm_fixup_bucket(uint32_t g, uint32_t L, const uint32_t* offs, Xyzz<typename CV::F>* buckets,
                            const Xyzz<typename CV::F>* spart) {
  uint32_t s = offs[g], t = offs[g + 1];
  if (t == s) return false;
  uint32_t j0 = s / L, j1 = (t - 1) / L;
  if (j0 == j1) return false;
  if (j1 - j0 + 1 > (uint32_t)SERIAL_MAX) return true;
  Xyzz<typename CV::F> acc = spart[2 * (size_t)j0 + 1];
  for (uint32_t j = j0 + 1; j <= j1; j++) {
    Xyzz<typename CV::F> p = spart[2 * (size_t)j];
    xyzz_add(acc, acc, p);
  }
  buckets[g] = acc;
  return false;
}

}  // namespace b2k
