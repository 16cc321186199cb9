// ed_msm.cuh -- per-thread bodies of the edwards25519 Pippenger MSM and of the share/poly kernels built on it.
//
// Replaces (reference, group/edwards25519 and share/poly.go):
//   the loops  Tmp.Mul(l_i, y_i); Acc.Add(Acc, Tmp)    share/poly.go:461-473 (RecoverCommit)    -> MSM
//   PubPoly.Eval                                     share/poly.go:340-357                     -> ed_pubpoly_horner
//   PubPoly.Check = Eval + Mul(s, b) + Equal         share/poly.go:405-409                     -> ed_pubpoly_check_one
//
// The MSM runs the pipeline of msm.cuh with the Edwards group law: the point-agnostic stages (plan, digit columns and histogram,
// scan, partition and bin sort: msm_host.cuh, msm_sort.cuh) are shared, the point stages are written here:
//   load       : decode (FromBytes, ge.go:110-150) into Niels form (y + x, y - x, 2 d x y), Montgomery, once per point; the scalar
//                rule below; signed digits of 256-bit scalars (W = ceil(257 / c) windows) and the histogram
//   accumulate : balanced slices of L sorted entries into extended (X:Y:Z:T) buckets by the mixed addition (7M, ed25519.cuh:
//                ed_madd); -P swaps y + x with y - x and negates 2 d x y.  The addition law is complete, so identity,
//                doubling, negation and torsion operands take no branch, and the slices are skew-proof like the Weierstrass ones
//   fix-up     : buckets cut by slice boundaries add their partials (ed_add); empty buckets are set to the identity here
//   reduce     : one level of chunked running sums, a small multiple per chunk, a block-wide sum per window, Horner, encode
//
// Scalars are read the way the reference's Point.Mul (geScalarMult, ge.go:443-502, varTime off) reads them: the plain
// little-endian integer k, except that its signed-nibble recoding can leave a top digit e63 above 8, for which selectCached
// (ge.go:419-433) selects nothing.  The product is then (k - e63 2^252) P, and the load pass multiplies by that integer instead
// (ed_scalar_rule, ed_scalar.cuh).  There is no reduction mod l: the points may have a torsion part.
#pragma once
#include "ed25519.cuh"
#include "msm_sort.cuh"

namespace b2k {

// ---- load pass: point i to Niels form, scalar rule, digit columns and histogram (msm_digits_store) -------------------------------
B2K_D bool ed_msm_load(size_t n, size_t i, const uint8_t* scalars, const uint8_t* wire, EdNiels* pts, const MsmPlan& pl,
                       int16_t* digits, uint32_t* counts) {
  EdNiels q;
  const bool ok = ed_load_niels(q, wire + 32 * i);
  pts[i] = q;
  Scalar256 s;
  sc_load_le(s.v, scalars + 32 * i);
  ed_scalar_rule(s.v);
  msm_digits_store(s, pl, n, i, digits, counts);
  return ok;
}

// ---- balanced slices (msm.cuh: msm_accumulate_slice, with the same partial layout) ---------------------------------------------
B2K_D void ed_slice_flush(const EdExt& acc, uint32_t g, uint32_t s, uint32_t t, uint32_t j, uint32_t b, uint32_t e,
                          EdExt* buckets, EdExt* spart) {
  if (s >= b && t <= e) buckets[g] = acc;
  else spart[2 * (size_t)j + (s < b ? 0 : 1)] = acc;
}

B2K_D void ed_accumulate_slice(uint32_t j, uint32_t L, uint32_t total, const EdNiels* pts, const uint32_t* offs,
                               const uint32_t* entries, EdExt* buckets, EdExt* spart) {
  const uint32_t E = offs[total];
  const uint32_t b = j * L;
  if (b >= E) return;
  const uint32_t e = (E - b < L) ? E : b + L;
  uint32_t g = msm_find_bucket(offs, total, b);
  uint32_t gs = offs[g], ge = offs[g + 1];
  EdExt acc;
  ed_set_identity(acc);
  for (uint32_t pos = b; pos < e; pos++) {
    if (pos == ge) {                       // crossed into a later bucket
      ed_slice_flush(acc, g, gs, ge, j, b, e, buckets, spart);
      ed_set_identity(acc);
      do { g++; gs = ge; ge = offs[g + 1]; } while (ge <= pos);
    }
    const uint32_t v = entries[pos];
    const EdNiels q = pts[v & 0x7fffffffu];
    ed_madd(acc, q, (v >> 31) != 0);
  }
  ed_slice_flush(acc, g, gs, ge, j, b, e, buckets, spart);
}

// Bucket g after the slices: the identity if it is empty, the sum of its partials if slice boundaries cut it.  Returns true when
// it has more than SERIAL_MAX partials (left to the block-parallel path, ed_fixup_strided).
template <int SERIAL_MAX>
B2K_D bool ed_fixup_bucket(uint32_t g, uint32_t L, const uint32_t* offs, EdExt* buckets, const EdExt* spart) {
  const uint32_t s = offs[g], t = offs[g + 1];
  if (t == s) {
    EdExt z;
    ed_set_identity(z);
    buckets[g] = z;
    return false;
  }
  const uint32_t j0 = s / L, j1 = (t - 1) / L;
  if (j0 == j1) return false;
  if (j1 - j0 + 1 > (uint32_t)SERIAL_MAX) return true;
  EdExt acc = spart[2 * (size_t)j0 + 1];
  for (uint32_t j = j0 + 1; j <= j1; j++) {
    const EdExt p = spart[2 * (size_t)j];
    ed_add(acc, acc, p);
  }
  buckets[g] = acc;
  return false;
}

// thread tid of nt of the block-parallel fix-up: the sum of partials j0 + tid, j0 + tid + nt, ... of a bucket spanning slices j0..j1
B2K_D void ed_fixup_strided(EdExt& acc, uint32_t tid, uint32_t nt, uint32_t j0, uint32_t j1, const EdExt* spart) {
  ed_set_identity(acc);
  for (uint32_t j = j0 + tid; j <= j1; j += nt) {
    const EdExt p = spart[2 * (size_t)j + (j == j0 ? 1 : 0)];
    ed_add(acc, acc, p);
  }
}

// ---- reduction ------------------------------------------------------------------------------------------------------------
// chunk t of m consecutive buckets of one window (B[k] holds digit magnitude k + 1): out = sum_k (k + 1) B[t m + k]
B2K_D void ed_reduce_chunk(EdExt& out, const EdExt* B, int t, int m) {
  EdExt run, acc;
  ed_set_identity(run);
  ed_set_identity(acc);
  for (int k = m - 1; k >= 0; k--) {
    const EdExt b = B[t * m + k];
    ed_add(run, run, b);
    ed_add(acc, acc, run);                 // after the loop: acc = sum (k + 1) B[t m + k], run = sum B
  }
  if (t != 0) {
    EdExt off;
    ed_mul_small(off, run, (uint32_t)(t * m));
    ed_add(acc, acc, off);
  }
  out = acc;
}

// Horner over the window sums: c doublings per window (the first c - 1 without T)
B2K_D void ed_msm_horner(EdExt& out, const EdExt* wsum, int W, int c) {
  EdExt acc = wsum[W - 1];
  for (int w = W - 2; w >= 0; w--) {
    for (int i = 0; i < c - 1; i++) ed_dbl_xyz(acc, acc);
    ed_dbl(acc, acc);
    const EdExt t = wsum[w];
    ed_add(acc, acc, t);
  }
  out = acc;
}

// ---- share/poly -----------------------------------------------------------------------------------------------------------
// r = k B by geScalarMult's schedule (ed_mul_digits) over btab = 1..8 B (ed_load_base_table)
B2K_D void ed_ge_scalar_mult_base(EdExt& r, const uint32_t* k, const EdNiels* btab) { ed_mul_digits(r, k, btab); }

// PubPoly.Check of one private share (index, 32-byte little-endian value) against t commitments in Niels form: the Horner value
// and share B compared projectively
B2K_D bool ed_pubpoly_check_one(const EdNiels* cm, uint32_t t, uint32_t index, const uint8_t* share, const EdNiels* btab) {
  EdExt v, w;
  ed_pubpoly_horner(v, cm, t, (uint64_t)index + 1u);
  uint32_t k[8];
  sc_load_le(k, share);
  ed_ge_scalar_mult_base(w, k, btab);
  return ed_eq(v, w);
}

}  // namespace b2k
