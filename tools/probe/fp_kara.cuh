// fp_kara.cuh -- PROBE: the one-level Karatsuba wide product of fp.cuh (detail::kara_term) used for a whole Montgomery product,
// timed against the CIOS fp_mul by fpmul_probe.cu and checked under host emulation (tests/test_fp_kara_emulation.py).  Not used
// by the library: on an H100 the product was no faster than fp_mul (DESIGN.md section 4); only the sum of two products
// (fp_mul_sum2) gained, and that one is in fp.cuh.
#pragma once
#include "../../kyber_b200/csrc/fp.cuh"

namespace b2k {
namespace detail {

// t[0..2N) = a * b, exact for any N-limb operands (the contract of wide_mul)
template <int N>
B2K_D void wide_mul_kara(uint32_t* t, const uint32_t* a, const uint32_t* b) {
  if constexpr (N % 4 != 0) {
    wide_mul<N>(t, a, b);
  } else {
    uint32_t mid[N + 1];
    kara_term<N, true>(t, mid, a, b);
    kara_finish<N>(t, mid);
  }
}

}  // namespace detail

// a b R^-1 through the Karatsuba wide product: 3/4 N^2 + N^2 multiply-adds instead of 2 N^2 (BLS12-381: 252 instead of 288)
template <class C>
B2K_D void fp_mul_k_inl(Fp<C>& r, const Fp<C>& a, const Fp<C>& b) {
  constexpr int N = C::N;
  uint32_t t[2 * N], u[N];
  detail::wide_mul_kara<N>(t, a.v, b.v);
  detail::redc_wide<C>(u, t);
  fp_reduce_once<C>(u);
#pragma unroll
  for (int j = 0; j < N; j++) r.v[j] = u[j];
}

}  // namespace b2k
