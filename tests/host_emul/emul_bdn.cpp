// Host emulation of the sign/bdn masked sums (test infrastructure only): the bodies of bdn.cuh on BLS12-381 G1, driven in the
// order the kernels of b2k_bdn.cu run them -- load, the roster total over the all-ones mask, the complement choice, one warp's
// 32 lanes per (mask, slice) with the warp reduction's pairing order, and the finish.
#include <vector>
#include "../../kyber_b200/csrc/bdn.cuh"
using namespace b2k;
using F = Fp<Bls381Fp>;
using X = Xyzz<F>;

// what one warp of k_bdn_masked_sum writes for (row, slice s): lanes' walks, then the shuffle-down tree
static X warp_sum(const uint8_t* row, size_t stride, uint32_t n, uint32_t s, bool comp, const Affine<F>* terms) {
  X lane[32];
  for (uint32_t l = 0; l < 32; l++) {
    const uint32_t w = s * 32 + l;
    xyzz_set_inf(lane[l]);
    bdn_walk(lane[l], bdn_lane_bits(row, stride, n, w, comp), terms, 32 * w);
  }
  for (int d = 16; d > 0; d >>= 1) {
    X next[32];
    for (int l = 0; l < 32; l++) xyzz_add(next[l], lane[l], lane[l + d < 32 ? l + d : l]);
    for (int l = 0; l < 32; l++) lane[l] = next[l];
  }
  return lane[0];
}

extern "C" {
// out[k] = operand bytes of mask k's aggregate over terms[n][96]; comp_out[k] = whether it was summed through its complement;
// returns 0, or -1 when a term is malformed
int emul_bdn_aggregate(uint32_t n, const uint8_t* terms_wire, uint32_t m, const uint8_t* masks, uint8_t* out, uint8_t* comp_out) {
  const size_t stride = (n + 7) / 8;
  const uint32_t ns = (n + BDN_SLICE - 1) / BDN_SLICE;
  std::vector<Affine<F>> terms(n);
  bool good = true;
  for (uint32_t i = 0; i < n; i++) good = load_checked<Bls381G1>(terms[i], terms_wire + 96 * i) && good;
  if (!good) return -1;
  std::vector<X> total(ns + 1);
  for (uint32_t s = 0; s < ns; s++) total[s] = warp_sum(nullptr, stride, n, s, false, terms.data());
  bdn_combine(total[ns], total.data(), ns);
  std::vector<X> part(ns);
  for (uint32_t k = 0; k < m; k++) {
    const uint8_t* row = masks + k * stride;
    const bool comp = bdn_complement(row, stride, n);
    comp_out[k] = comp ? 1 : 0;
    for (uint32_t s = 0; s < ns; s++) part[s] = warp_sum(row, stride, n, s, comp, terms.data());
    Affine<F> r;
    bdn_finish(r, part.data(), ns, comp, total[ns]);
    Bls381G1::store_affine(out + 96 * k, r);
  }
  return 0;
}
}
