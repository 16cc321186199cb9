// bdn.cuh -- sign/bdn on the device: AggregatePublicKeys for many participation masks over one roster.
//
// Replaces: bdn.AggregatePublicKeys   sign/bdn/bdn.go:166-181
//   With the terms of NewMask (mask.go:34-64, publicTerms[i] = (c_i + 1) PK_i) cached per roster, the aggregate key of a mask
//   is the plain sum of the enabled terms: bit i of byte i/8, little-endian within the byte (mask.go:88-97), for i < n.
// The bodies below are written once over the group law of ec.cuh, so one code path serves G1 (Fp) and G2 (Fp2) of BLS12-381
// and bn256; the kernels of b2k_bdn.cu drive them, tests/host_emul/emul_bdn.cpp runs them on the host.
//   work split: one warp per (mask, slice of BDN_SLICE roster members); lane l owns mask word l of the slice and walks its
//               set bits with mixed XYZZ additions; the lanes' sums meet in a warp reduction, the slices' sums per mask.
//   complement: a mask with more than n/2 bits set sums its DISABLED terms instead and finishes with S - partial, where S is
//               the roster total (the same masked sum over the all-ones mask).  Same point, about half the additions at worst.
#pragma once
#include "curves.cuh"

namespace b2k {

constexpr uint32_t BDN_SLICE = 1024;   // roster members per warp: 32 lanes x one 32-bit mask word each

B2K_D uint32_t bdn_popc(uint32_t x) {
#if defined(__CUDACC__)
  return (uint32_t)__popc(x);
#else
  return (uint32_t)__builtin_popcount(x);
#endif
}
B2K_D int bdn_ffs(uint32_t x) {        // 1 + index of the lowest set bit (x != 0)
#if defined(__CUDACC__)
  return __ffs(x);
#else
  return __builtin_ffs((int)x);
#endif
}

// bits of roster members [32 w, 32 w + 32) in a mask row of `stride` bytes; row == nullptr is the all-ones mask.
// Positions >= n are cleared, as the reference's loop over i < n ignores them.
B2K_D uint32_t bdn_mask_word(const uint8_t* row, size_t stride, uint32_t n, uint32_t w) {
  if ((size_t)w * 32 >= n) return 0;
  const uint32_t left = n - 32 * w;
  const uint32_t valid = left >= 32 ? 0xFFFFFFFFu : ((1u << left) - 1u);
  if (!row) return valid;
  uint32_t v = 0;
  for (int b = 0; b < 4; b++) {
    const size_t at = 4 * (size_t)w + b;
    if (at < stride) v |= (uint32_t)row[at] << (8 * b);
  }
  return v & valid;
}

// the word a lane sums: the enabled terms, or the disabled ones when the mask takes the complement
B2K_D uint32_t bdn_lane_bits(const uint8_t* row, size_t stride, uint32_t n, uint32_t w, bool comp) {
  const uint32_t v = bdn_mask_word(row, stride, n, w);
  return comp ? (~v & bdn_mask_word(nullptr, stride, n, w)) : v;
}

// more than half of the n bits set: the mask is summed through its complement
B2K_D bool bdn_complement(const uint8_t* row, size_t stride, uint32_t n) {
  uint32_t pop = 0;
  for (uint32_t w = 0; (size_t)w * 32 < n; w++) pop += bdn_popc(bdn_mask_word(row, stride, n, w));
  return 2 * pop > n;
}

// The group law on XYZZ points, out of line and by reference over Fp2 in the by-reference Fp2 layout (tower.cuh: B2K_FP2_BYREF),
// as xyzz_add_reduce (msm.cuh) does: an Fp2 point held by value across an addition leaves the field products underneath too few
// registers, and every product then pays callee-save spills.  The points stay in memory instead.
template <class F>
B2K_NI void bdn_add_ool(Xyzz<F>& r, const Xyzz<F>& p, const Xyzz<F>& q) { xyzz_add(r, p, q); }
template <class F>
B2K_NI void bdn_madd_ool(Xyzz<F>& r, const Affine<F>& q) { xyzz_madd(r, r, q, false); }
template <class F>
B2K_D void bdn_add(Xyzz<F>& r, const Xyzz<F>& p, const Xyzz<F>& q) {
#ifdef B2K_FP2_BYREF
  if constexpr (sizeof(F) > 48) { bdn_add_ool(r, p, q); return; }
#endif
  xyzz_add(r, p, q);
}
template <class F>
B2K_D void bdn_madd(Xyzz<F>& acc, const Affine<F>& q) {
#ifdef B2K_FP2_BYREF
  if constexpr (sizeof(F) > 48) { bdn_madd_ool(acc, q); return; }
#endif
  xyzz_madd(acc, acc, q, false);
}

// acc += terms[base + b] for every set bit b of bits (duplicates, negations and infinity terms are xyzz_madd's cases)
template <class F>
B2K_D void bdn_walk(Xyzz<F>& acc, uint32_t bits, const Affine<F>* terms, uint32_t base) {
  while (bits) {
    const int b = bdn_ffs(bits) - 1;
    bits &= bits - 1;
    bdn_madd(acc, terms[base + b]);
  }
}

// the sum of a mask's slice partials
template <class F>
B2K_D void bdn_combine(Xyzz<F>& r, const Xyzz<F>* part, uint32_t nslices) {
  r = part[0];
  for (uint32_t s = 1; s < nslices; s++) bdn_add(r, r, part[s]);
}

// S - partial for a complemented mask, in place
template <class F>
B2K_D void bdn_apply_complement(Xyzz<F>& acc, const Xyzz<F>& total) {
  f_neg(acc.Y, acc.Y);
  bdn_add(acc, total, acc);
}

// a mask's aggregate key: its slices combined, S - partial for a complemented mask, one inversion to affine
template <class F>
B2K_D void bdn_finish(Affine<F>& r, const Xyzz<F>* part, uint32_t nslices, bool comp, const Xyzz<F>& total) {
  Xyzz<F> acc;
  bdn_combine(acc, part, nslices);
  if (comp) bdn_apply_complement(acc, total);
  xyzz_to_affine(r, acc);
}

}  // namespace b2k

#if defined(__CUDACC__)
// ---- host side, shared by the translation units that aggregate (b2k_bdn.cu) and verify (b2k_h2c.cu, b2k_bn256.cu) ----------
#include "host_call.cuh"

namespace b2k_host {

enum BdnGroup { BDN_BLS_G2 = 0, BDN_BLS_G1 = 1, BDN_BN256_G2 = 2 };

// scratch of one aggregation: the terms in Montgomery affine form, the complement flags, the (mask, slice) partials, and the
// roster total's slice partials followed by the total itself
struct BdnScratch {
  void* terms = nullptr;
  uint8_t* comp = nullptr;
  void* part = nullptr;
  void* total = nullptr;
  size_t nslices = 0;
};

int bdn_args(b2k_ctx* ctx, size_t n, size_t m);                 // n, m within 1..the documented caps
void bdn_layout(Carve& c, BdnScratch& s, BdnGroup g, size_t n, size_t m);
// out + k out_stride = operand bytes of mask k's aggregate key (all zeros for infinity); every pointer on the device
int bdn_aggregate_enqueue(b2k_ctx* ctx, BdnGroup g, const BdnScratch& s, size_t n, const uint8_t* d_terms, size_t m,
                          const uint8_t* d_masks, uint8_t* d_out, size_t out_stride);
// status[k] = B2K_BDN_SIG when the signature did not decode, else B2K_BDN_OK / B2K_BDN_INVALID from the pairing check
int bdn_status_enqueue(b2k_ctx* ctx, size_t m, const uint8_t* d_sig_ok, const uint8_t* d_pair_ok, uint8_t* d_status);

}  // namespace b2k_host
#endif
