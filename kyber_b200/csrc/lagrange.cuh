// lagrange.cuh -- the Lagrange weights at zero of share.RecoverCommit (share/poly.go:459-471: num *= x_j, den *= x_j - x_i,
// num / den), one weight per thread.  Shared by the RecoverCommit entry points of every group (b2k_share.cu, b2k_ed25519_msm.cu).
#pragma once
#include "fp.cuh"

namespace b2k {

// lambda_i = prod_{j != i} x_j / (x_j - x_i)  mod the order of FR, x = index + 1 (index 0xffffffff gives 2^32), written as a
// 32-byte scalar: big-endian (the pairing groups' scalar encoding) or little-endian (LE: edwards25519's).  Returns false
// when another index equals index i (the denominator would be zero).
template <class FR, bool LE>
B2K_D bool lagrange_at_zero(uint32_t i, uint32_t t, const uint32_t* __restrict__ idx, uint8_t* __restrict__ out) {
  using S = Fp<FR>;
  S num, den, xi, xj, d;
  bool ok = true;
  fp_set_one(num);
  fp_set_one(den);
  fp_set_zero(xi);
  const uint32_t ii = idx[i];
  xi.v[0] = ii + 1u; xi.v[1] = (ii == 0xffffffffu) ? 1u : 0u;
  fp_to_mont(xi, xi);
  for (uint32_t j = 0; j < t; j++) {
    if (j == i) continue;
    const uint32_t jj = idx[j];
    if (jj == ii) ok = false;
    fp_set_zero(xj);
    xj.v[0] = jj + 1u; xj.v[1] = (jj == 0xffffffffu) ? 1u : 0u;
    fp_to_mont(xj, xj);
    fp_mul(num, num, xj);
    fp_sub(d, xj, xi);
    fp_mul(den, den, d);
  }
  fp_inv(den, den);
  fp_mul(num, num, den);
  fp_from_mont(num, num);
#pragma unroll
  for (int k = 0; k < 8; k++) {
    if (LE) {
      uint8_t* q = out + 4 * k;
      q[0] = (uint8_t)num.v[k]; q[1] = (uint8_t)(num.v[k] >> 8); q[2] = (uint8_t)(num.v[k] >> 16); q[3] = (uint8_t)(num.v[k] >> 24);
    } else {
      uint8_t* q = out + 4 * (7 - k);
      q[0] = (uint8_t)(num.v[k] >> 24); q[1] = (uint8_t)(num.v[k] >> 16); q[2] = (uint8_t)(num.v[k] >> 8); q[3] = (uint8_t)num.v[k];
    }
  }
  return ok;
}

#ifdef __CUDACC__
// scalars[i] = lambda_i; a duplicate index sets bit 4 of the status word (reported as B2K_ERR_ARG)
template <class FR, bool LE = false>
__global__ void __launch_bounds__(128) k_lagrange_at_zero(uint32_t t, const uint32_t* __restrict__ idx,
                                                          uint8_t* __restrict__ scalars, uint32_t* flags) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= t) return;
  if (!lagrange_at_zero<FR, LE>(i, t, idx, scalars + 32 * (size_t)i)) atomicOr(flags, FLAG_DUP_INDEX);
}
#endif

}  // namespace b2k
