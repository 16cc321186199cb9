// tower.cuh -- Fp2 / Fp6 / Fp12 extension towers over fp.cuh, all limbs in registers / local arrays.
//
//   Fp2  = Fp[u]/(u^2+1)                      (both BLS12-381 and bn254: i^2 = -1,
//                                              reference bn254: pairing/bn254/gfp2.go:82-157)
//   Fp6  = Fp2[v]/(v^3 - xi)                  xi = 1+u (BLS12-381), 9+u (bn254 gfp2.go:104-126)
//   Fp12 = Fp6[w]/(w^2 - v)                   (bn254: pairing/bn254/gfp6.go, gfp12.go)
// A tower config T supplies  typename T::Base (the Fp config) and  mul_xi(Fp2&).
#pragma once
#include "constants.cuh"
#include "fp.cuh"

namespace b2k {

template <class C>
struct Fp2 {
  Fp<C> c0, c1;  // c0 + c1*u
};

template <class C> B2K_D void fp2_add(Fp2<C>& r, const Fp2<C>& a, const Fp2<C>& b) { fp_add(r.c0, a.c0, b.c0); fp_add(r.c1, a.c1, b.c1); }
template <class C> B2K_D void fp2_sub(Fp2<C>& r, const Fp2<C>& a, const Fp2<C>& b) { fp_sub(r.c0, a.c0, b.c0); fp_sub(r.c1, a.c1, b.c1); }
template <class C> B2K_D void fp2_neg(Fp2<C>& r, const Fp2<C>& a) { fp_neg(r.c0, a.c0); fp_neg(r.c1, a.c1); }
template <class C> B2K_D void fp2_conj(Fp2<C>& r, const Fp2<C>& a) { r.c0 = a.c0; fp_neg(r.c1, a.c1); }
template <class C> B2K_D void fp2_dbl(Fp2<C>& r, const Fp2<C>& a) { fp_add(r.c0, a.c0, a.c0); fp_add(r.c1, a.c1, a.c1); }
template <class C> B2K_D bool fp2_is_zero(const Fp2<C>& a) { return fp_is_zero(a.c0) && fp_is_zero(a.c1); }
template <class C> B2K_D bool fp2_eq(const Fp2<C>& a, const Fp2<C>& b) { return fp_eq(a.c0, b.c0) && fp_eq(a.c1, b.c1); }
template <class C> B2K_D void fp2_set_zero(Fp2<C>& r) { fp_set_zero(r.c0); fp_set_zero(r.c1); }
template <class C> B2K_D void fp2_set_one(Fp2<C>& r) { fp_set_one(r.c0); fp_set_zero(r.c1); }

// Karatsuba: 3 base multiplications.  Out of line, but the three products are inlined so that the six
// input limbs-vectors are loaded once and every intermediate stays in registers (one 24-word store per
// Fp2 product instead of three round trips through local memory).
// B2K_COMPACT_FIELD: one by-value body (operands and result in registers through the ABI) whose three products are calls
// to the single out-of-line Fp product (fp.cuh) -- ~1 KB of code instead of 16 KB.
// B2K_FP2_BYREF (set by a translation unit in front of its includes) keeps the by-reference Fp2 product below with the
// out-of-line Fp product underneath: kernels that hold whole Fp2 points by value (the G2 MSM: a 96-word XYZZ accumulator plus
// temporaries) otherwise leave the register allocator so little room that the Fp product itself is compiled with 100-470 extra
// instructions (tools/codegen_check.py: 470-853 instead of 385 in b2k_g2.o); the pairing kernels are the opposite case
// (by value measured faster than by reference at 65 536 checks).
#if defined(B2K_COMPACT_FIELD) && !defined(B2K_FP2_BYREF)
template <class C>
B2K_NI Fp2<C> fp2_mul_v(Fp2<C> a, Fp2<C> b) {
  Fp<C> t0, t1, s0, s1;
  Fp2<C> r;
  fp_mul(t0, a.c0, b.c0);
  fp_mul(t1, a.c1, b.c1);
  fp_add(s0, a.c0, a.c1);
  fp_add(s1, b.c0, b.c1);
  fp_mul(s0, s0, s1);
  fp_sub(s0, s0, t0);
  fp_sub(r.c1, s0, t1);
  fp_sub(r.c0, t0, t1);
  return r;
}
template <class C> B2K_D void fp2_mul(Fp2<C>& r, const Fp2<C>& a, const Fp2<C>& b) { r = fp2_mul_v<C>(a, b); }
#else
template <class C>
B2K_NI void fp2_mul(Fp2<C>& r, const Fp2<C>& a, const Fp2<C>& b) {
  const Fp<C> a0 = a.c0, a1 = a.c1, b0 = b.c0, b1 = b.c1;
  Fp<C> t0, t1, s0, s1;
  fp_mul(t0, a0, b0);
  fp_mul(t1, a1, b1);
  fp_add(s0, a0, a1);
  fp_add(s1, b0, b1);
  fp_mul(s0, s0, s1);
  fp_sub(s0, s0, t0);
  fp_sub(s0, s0, t1);
  fp_sub(t0, t0, t1);
  r.c1 = s0;
  r.c0 = t0;
}
#endif

// Karatsuba with lazy reduction: three WIDE products (fp.cuh: detail::wide_mul, N^2 multiply-adds each) and only two
// Montgomery reductions -- 5 N^2 multiply-adds instead of the 6 N^2 of three reduced products.
//   c1 = (a0 + a1)(b0 + b1) - a0 b0 - a1 b1   (>= 0 as integers; the sums are left unreduced: 2p < 2^(32N), 4p^2 < p 2^(32N))
//   c0 = a0 b0 - a1 b1                        (+ p 2^(32N) when negative: adds p to the upper half)
// Out of line; the products are inlined so that the operands are loaded once and every intermediate stays in registers.
// The one-thread-per-pairing kernel is LATENCY-bound (2 warps per scheduler), where trading one reduction for ~100 add/sub
// instructions measured slower; kept for throughput-bound callers and tested in the emulation.
template <class C>
B2K_NI void fp2_mul_lazy(Fp2<C>& r, const Fp2<C>& a, const Fp2<C>& b) {
  constexpr int N = C::N;
  uint32_t t0[2 * N], t1[2 * N], s[2 * N], sa[N], sb[N];
  detail::wide_mul<N>(t0, a.c0.v, b.c0.v);
  detail::wide_mul<N>(t1, a.c1.v, b.c1.v);
  sa[0] = ptx::add_cc(a.c0.v[0], a.c1.v[0]);
#pragma unroll
  for (int j = 1; j < N - 1; j++) sa[j] = ptx::addc_cc(a.c0.v[j], a.c1.v[j]);
  sa[N - 1] = ptx::addc(a.c0.v[N - 1], a.c1.v[N - 1]);
  sb[0] = ptx::add_cc(b.c0.v[0], b.c1.v[0]);
#pragma unroll
  for (int j = 1; j < N - 1; j++) sb[j] = ptx::addc_cc(b.c0.v[j], b.c1.v[j]);
  sb[N - 1] = ptx::addc(b.c0.v[N - 1], b.c1.v[N - 1]);
  detail::wide_mul<N>(s, sa, sb);
  s[0] = ptx::sub_cc(s[0], t0[0]);
#pragma unroll
  for (int j = 1; j < 2 * N - 1; j++) s[j] = ptx::subc_cc(s[j], t0[j]);
  s[2 * N - 1] = ptx::subc(s[2 * N - 1], t0[2 * N - 1]);
  s[0] = ptx::sub_cc(s[0], t1[0]);
#pragma unroll
  for (int j = 1; j < 2 * N - 1; j++) s[j] = ptx::subc_cc(s[j], t1[j]);
  s[2 * N - 1] = ptx::subc(s[2 * N - 1], t1[2 * N - 1]);
  t0[0] = ptx::sub_cc(t0[0], t1[0]);
#pragma unroll
  for (int j = 1; j < 2 * N; j++) t0[j] = ptx::subc_cc(t0[j], t1[j]);
  const uint32_t borrow = ptx::subc(0, 0);                  // all-ones if a0 b0 < a1 b1
  t0[N] = ptx::add_cc(t0[N], C::mod(0) & borrow);
#pragma unroll
  for (int j = 1; j < N - 1; j++) t0[N + j] = ptx::addc_cc(t0[N + j], C::mod(j) & borrow);
  t0[2 * N - 1] = ptx::addc(t0[2 * N - 1], C::mod(N - 1) & borrow);
  uint32_t u[N];
  detail::redc_wide<C>(u, s);
  fp_reduce_once<C>(u);
#pragma unroll
  for (int j = 0; j < N; j++) r.c1.v[j] = u[j];
  detail::redc_wide<C>(u, t0);
  fp_reduce_once<C>(u);
#pragma unroll
  for (int j = 0; j < N; j++) r.c0.v[j] = u[j];
}

// complex squaring: 2 base multiplications (same register-resident structure)
#if defined(B2K_COMPACT_FIELD) && !defined(B2K_FP2_BYREF)
template <class C>
B2K_NI Fp2<C> fp2_sqr_v(Fp2<C> a) {
  Fp<C> s, d, m;
  Fp2<C> r;
  fp_add(s, a.c0, a.c1);
  fp_sub(d, a.c0, a.c1);
  fp_mul(m, a.c0, a.c1);
  fp_mul(r.c0, s, d);
  fp_add(r.c1, m, m);
  return r;
}
template <class C> B2K_D void fp2_sqr(Fp2<C>& r, const Fp2<C>& a) { r = fp2_sqr_v<C>(a); }
#else
template <class C>
B2K_NI void fp2_sqr(Fp2<C>& r, const Fp2<C>& a) {
  const Fp<C> a0 = a.c0, a1 = a.c1;
  Fp<C> s, d, m;
  fp_add(s, a0, a1);
  fp_sub(d, a0, a1);
  fp_mul(m, a0, a1);
  fp_mul(s, s, d);
  fp_add(m, m, m);
  r.c0 = s;
  r.c1 = m;
}
#endif

template <class C>
B2K_D void fp2_mul_fp(Fp2<C>& r, const Fp2<C>& a, const Fp<C>& k) { fp_mul_c(r.c0, a.c0, k); fp_mul_c(r.c1, a.c1, k); }

template <class C>
B2K_NI void fp2_inv(Fp2<C>& r, const Fp2<C>& a) {
  Fp<C> n, t;
  fp_sqr_c(n, a.c0);
  fp_sqr_c(t, a.c1);
  fp_add(n, n, t);
  fp_inv(n, n);
  fp_mul_c(r.c0, a.c0, n);
  fp_mul_c(t, a.c1, n);
  fp_neg(r.c1, t);
}

// ---- uniform "field" vocabulary so curve code is written once for Fp and Fp2 -------------------
template <class C> B2K_D void f_add(Fp<C>& r, const Fp<C>& a, const Fp<C>& b) { fp_add(r, a, b); }
template <class C> B2K_D void f_sub(Fp<C>& r, const Fp<C>& a, const Fp<C>& b) { fp_sub(r, a, b); }
template <class C> B2K_D void f_mul(Fp<C>& r, const Fp<C>& a, const Fp<C>& b) { fp_mul(r, a, b); }
template <class C> B2K_D void f_sqr(Fp<C>& r, const Fp<C>& a) { fp_sqr(r, a); }
template <class C> B2K_D void f_neg(Fp<C>& r, const Fp<C>& a) { fp_neg(r, a); }
template <class C> B2K_D void f_dbl(Fp<C>& r, const Fp<C>& a) { fp_add(r, a, a); }
template <class C> B2K_D void f_inv(Fp<C>& r, const Fp<C>& a) { fp_inv(r, a); }
template <class C> B2K_D bool f_is_zero(const Fp<C>& a) { return fp_is_zero(a); }
template <class C> B2K_D bool f_eq(const Fp<C>& a, const Fp<C>& b) { return fp_eq(a, b); }
template <class C> B2K_D void f_set_zero(Fp<C>& r) { fp_set_zero(r); }
template <class C> B2K_D void f_set_one(Fp<C>& r) { fp_set_one(r); }

template <class C> B2K_D void f_mul_i(Fp<C>& r, const Fp<C>& a, const Fp<C>& b) { fp_mul_i(r, a, b); }
template <class C> B2K_D void f_sqr_i(Fp<C>& r, const Fp<C>& a) { fp_sqr_i(r, a); }
template <class C> B2K_D void f_mul_i(Fp2<C>& r, const Fp2<C>& a, const Fp2<C>& b) { fp2_mul(r, a, b); }
template <class C> B2K_D void f_sqr_i(Fp2<C>& r, const Fp2<C>& a) { fp2_sqr(r, a); }
// r = a b - c d for the Y3 of the XYZZ additions over Fp (ec.cuh): one reduction for both products, (a b + (p - c) d) R^-1
// (fp.cuh, fp_mul_sum2); t is scratch.  Fp2 (G2) and the probe fields keep two products and a subtraction (f_is_base).
template <class F> inline constexpr bool f_is_base = false;
template <class C> inline constexpr bool f_is_base<Fp<C>> = true;
template <class C>
B2K_D void f_mul_sub(Fp<C>& r, const Fp<C>& a, const Fp<C>& b, const Fp<C>& c, const Fp<C>& d, Fp<C>& t) {
  fp_neg(t, c);
  fp_mul_sum2(r, a, b, t, d);
}
template <class C> B2K_D void f_add(Fp2<C>& r, const Fp2<C>& a, const Fp2<C>& b) { fp2_add(r, a, b); }
template <class C> B2K_D void f_sub(Fp2<C>& r, const Fp2<C>& a, const Fp2<C>& b) { fp2_sub(r, a, b); }
template <class C> B2K_D void f_mul(Fp2<C>& r, const Fp2<C>& a, const Fp2<C>& b) { fp2_mul(r, a, b); }
template <class C> B2K_D void f_sqr(Fp2<C>& r, const Fp2<C>& a) { fp2_sqr(r, a); }
template <class C> B2K_D void f_neg(Fp2<C>& r, const Fp2<C>& a) { fp2_neg(r, a); }
template <class C> B2K_D void f_dbl(Fp2<C>& r, const Fp2<C>& a) { fp2_dbl(r, a); }
template <class C> B2K_D void f_inv(Fp2<C>& r, const Fp2<C>& a) { fp2_inv(r, a); }
template <class C> B2K_D bool f_is_zero(const Fp2<C>& a) { return fp2_is_zero(a); }
template <class C> B2K_D bool f_eq(const Fp2<C>& a, const Fp2<C>& b) { return fp2_eq(a, b); }
template <class C> B2K_D void f_set_zero(Fp2<C>& r) { fp2_set_zero(r); }
template <class C> B2K_D void f_set_one(Fp2<C>& r) { fp2_set_one(r); }

// ---- tower configs ------------------------------------------------------------------------------
struct Bls381Tower {
  using Base = Bls381Fp;
  // xi = 1 + u:  (a0 + a1 u)(1 + u) = (a0 - a1) + (a0 + a1) u
  B2K_D static void mul_xi(Fp2<Base>& r, const Fp2<Base>& a) {
    Fp<Base> t;
    fp_sub(t, a.c0, a.c1);
    fp_add(r.c1, a.c0, a.c1);
    r.c0 = t;
  }
};

struct Bn254Tower {
  using Base = Bn254Fp;
  // xi = 9 + u (pairing/bn254/gfp2.go:104-126):  (9 a0 - a1) + (9 a1 + a0) u
  B2K_D static void mul_xi(Fp2<Base>& r, const Fp2<Base>& a) {
    Fp<Base> t0, t1, n0, n1;
    fp_add(t0, a.c0, a.c0); fp_add(t0, t0, t0); fp_add(t0, t0, t0); fp_add(t0, t0, a.c0);  // 9 a0
    fp_add(t1, a.c1, a.c1); fp_add(t1, t1, t1); fp_add(t1, t1, t1); fp_add(t1, t1, a.c1);  // 9 a1
    fp_sub(n0, t0, a.c1);
    fp_add(n1, t1, a.c0);
    r.c0 = n0; r.c1 = n1;
  }
};

// ---- Fp6 ----------------------------------------------------------------------------------------
template <class T>
struct Fp6 {
  Fp2<typename T::Base> c0, c1, c2;  // c0 + c1 v + c2 v^2
};

template <class T> B2K_D void fp6_add(Fp6<T>& r, const Fp6<T>& a, const Fp6<T>& b) { fp2_add(r.c0, a.c0, b.c0); fp2_add(r.c1, a.c1, b.c1); fp2_add(r.c2, a.c2, b.c2); }
template <class T> B2K_D void fp6_sub(Fp6<T>& r, const Fp6<T>& a, const Fp6<T>& b) { fp2_sub(r.c0, a.c0, b.c0); fp2_sub(r.c1, a.c1, b.c1); fp2_sub(r.c2, a.c2, b.c2); }
template <class T> B2K_D void fp6_neg(Fp6<T>& r, const Fp6<T>& a) { fp2_neg(r.c0, a.c0); fp2_neg(r.c1, a.c1); fp2_neg(r.c2, a.c2); }
template <class T> B2K_D void fp6_set_zero(Fp6<T>& r) { fp2_set_zero(r.c0); fp2_set_zero(r.c1); fp2_set_zero(r.c2); }
template <class T> B2K_D void fp6_set_one(Fp6<T>& r) { fp2_set_one(r.c0); fp2_set_zero(r.c1); fp2_set_zero(r.c2); }
template <class T> B2K_D bool fp6_eq(const Fp6<T>& a, const Fp6<T>& b) { return fp2_eq(a.c0, b.c0) && fp2_eq(a.c1, b.c1) && fp2_eq(a.c2, b.c2); }

// multiply by v: (c0,c1,c2) -> (xi*c2, c0, c1)
template <class T>
B2K_D void fp6_mul_v(Fp6<T>& r, const Fp6<T>& a) {
  Fp2<typename T::Base> t;
  T::mul_xi(t, a.c2);
  r.c2 = a.c1;
  r.c1 = a.c0;
  r.c0 = t;
}

// Karatsuba/Toom-style: 6 Fp2 multiplications
template <class T>
B2K_NI void fp6_mul(Fp6<T>& r, const Fp6<T>& a, const Fp6<T>& b) {
  using F2 = Fp2<typename T::Base>;
  F2 v0, v1, v2, t0, t1, t2, s;
  fp2_mul(v0, a.c0, b.c0);
  fp2_mul(v1, a.c1, b.c1);
  fp2_mul(v2, a.c2, b.c2);
  // c0 = v0 + xi((a1+a2)(b1+b2) - v1 - v2)
  fp2_add(t0, a.c1, a.c2); fp2_add(s, b.c1, b.c2); fp2_mul(t0, t0, s);
  fp2_sub(t0, t0, v1); fp2_sub(t0, t0, v2); T::mul_xi(t0, t0); fp2_add(t0, t0, v0);
  // c1 = (a0+a1)(b0+b1) - v0 - v1 + xi v2
  fp2_add(t1, a.c0, a.c1); fp2_add(s, b.c0, b.c1); fp2_mul(t1, t1, s);
  fp2_sub(t1, t1, v0); fp2_sub(t1, t1, v1); T::mul_xi(s, v2); fp2_add(t1, t1, s);
  // c2 = (a0+a2)(b0+b2) - v0 - v2 + v1
  fp2_add(t2, a.c0, a.c2); fp2_add(s, b.c0, b.c2); fp2_mul(t2, t2, s);
  fp2_sub(t2, t2, v0); fp2_sub(t2, t2, v2); fp2_add(t2, t2, v1);
  r.c0 = t0; r.c1 = t1; r.c2 = t2;
}

template <class T>
B2K_D void fp6_sqr(Fp6<T>& r, const Fp6<T>& a) { fp6_mul(r, a, a); }

// multiply by a sparse element (b0, b1, 0): 5 Fp2 multiplications
template <class T>
B2K_NI void fp6_mul_by_01(Fp6<T>& r, const Fp6<T>& a, const Fp2<typename T::Base>& b0, const Fp2<typename T::Base>& b1) {
  using F2 = Fp2<typename T::Base>;
  F2 v0, v1, t0, t1, t2, s;
  fp2_mul(v0, a.c0, b0);
  fp2_mul(v1, a.c1, b1);
  // c0 = v0 + xi((a1+a2) b1 - v1)
  fp2_add(t0, a.c1, a.c2); fp2_mul(t0, t0, b1); fp2_sub(t0, t0, v1); T::mul_xi(t0, t0); fp2_add(t0, t0, v0);
  // c1 = (a0+a1)(b0+b1) - v0 - v1
  fp2_add(t1, a.c0, a.c1); fp2_add(s, b0, b1); fp2_mul(t1, t1, s); fp2_sub(t1, t1, v0); fp2_sub(t1, t1, v1);
  // c2 = a2 b0 + v1        ( (a0+a2) b0 - v0 + v1 )
  fp2_mul(t2, a.c2, b0); fp2_add(t2, t2, v1);
  r.c0 = t0; r.c1 = t1; r.c2 = t2;
}

// multiply by a sparse element (0, b1, 0): 3 Fp2 multiplications
template <class T>
B2K_NI void fp6_mul_by_1(Fp6<T>& r, const Fp6<T>& a, const Fp2<typename T::Base>& b1) {
  using F2 = Fp2<typename T::Base>;
  F2 t0, t1, t2;
  fp2_mul(t0, a.c2, b1); T::mul_xi(t0, t0);
  fp2_mul(t1, a.c0, b1);
  fp2_mul(t2, a.c1, b1);
  r.c0 = t0; r.c1 = t1; r.c2 = t2;
}

template <class T>
B2K_D void fp6_mul_fp2(Fp6<T>& r, const Fp6<T>& a, const Fp2<typename T::Base>& k) {
  fp2_mul(r.c0, a.c0, k); fp2_mul(r.c1, a.c1, k); fp2_mul(r.c2, a.c2, k);
}

template <class T>
B2K_NI void fp6_inv(Fp6<T>& r, const Fp6<T>& a) {
  using F2 = Fp2<typename T::Base>;
  F2 t0, t1, t2, s, d;
  // t0 = a0^2 - xi a1 a2 ; t1 = xi a2^2 - a0 a1 ; t2 = a1^2 - a0 a2
  fp2_sqr(t0, a.c0); fp2_mul(s, a.c1, a.c2); T::mul_xi(s, s); fp2_sub(t0, t0, s);
  fp2_sqr(t1, a.c2); T::mul_xi(t1, t1); fp2_mul(s, a.c0, a.c1); fp2_sub(t1, t1, s);
  fp2_sqr(t2, a.c1); fp2_mul(s, a.c0, a.c2); fp2_sub(t2, t2, s);
  // d = a0 t0 + xi (a2 t1 + a1 t2)
  fp2_mul(d, a.c2, t1); fp2_mul(s, a.c1, t2); fp2_add(d, d, s); T::mul_xi(d, d);
  fp2_mul(s, a.c0, t0); fp2_add(d, d, s);
  fp2_inv(d, d);
  fp2_mul(r.c0, t0, d); fp2_mul(r.c1, t1, d); fp2_mul(r.c2, t2, d);
}

// ---- Fp12 ---------------------------------------------------------------------------------------
template <class T>
struct Fp12 {
  Fp6<T> c0, c1;  // c0 + c1 w
};

template <class T> B2K_D void fp12_set_one(Fp12<T>& r) { fp6_set_one(r.c0); fp6_set_zero(r.c1); }
template <class T> B2K_D bool fp12_eq(const Fp12<T>& a, const Fp12<T>& b) { return fp6_eq(a.c0, b.c0) && fp6_eq(a.c1, b.c1); }
template <class T> B2K_D void fp12_conj(Fp12<T>& r, const Fp12<T>& a) { r.c0 = a.c0; fp6_neg(r.c1, a.c1); }
template <class T>
B2K_D bool fp12_is_one(const Fp12<T>& a) {
  Fp12<T> one;
  fp12_set_one(one);
  return fp12_eq(a, one);
}

template <class T>
B2K_NI void fp12_mul(Fp12<T>& r, const Fp12<T>& a, const Fp12<T>& b) {
  Fp6<T> t0, t1, s0, s1;
  fp6_mul(t0, a.c0, b.c0);
  fp6_mul(t1, a.c1, b.c1);
  fp6_add(s0, a.c0, a.c1);
  fp6_add(s1, b.c0, b.c1);
  fp6_mul(s0, s0, s1);
  fp6_sub(s0, s0, t0);
  fp6_sub(r.c1, s0, t1);
  fp6_mul_v(t1, t1);
  fp6_add(r.c0, t0, t1);
}

// complex squaring: 2 Fp6 multiplications
template <class T>
B2K_NI void fp12_sqr(Fp12<T>& r, const Fp12<T>& a) {
  Fp6<T> ab, s, t;
  fp6_mul(ab, a.c0, a.c1);
  fp6_add(s, a.c0, a.c1);
  fp6_mul_v(t, a.c1);
  fp6_add(t, t, a.c0);
  fp6_mul(s, s, t);        // (a0+a1)(a0+v a1) = a0^2 + v a1^2 + (1+v) a0 a1
  fp6_sub(s, s, ab);
  fp6_mul_v(t, ab);
  fp6_sub(r.c0, s, t);
  fp6_add(r.c1, ab, ab);
}

template <class T>
B2K_NI void fp12_inv(Fp12<T>& r, const Fp12<T>& a) {
  Fp6<T> d, t;
  fp6_sqr(d, a.c0);
  fp6_sqr(t, a.c1);
  fp6_mul_v(t, t);
  fp6_sub(d, d, t);
  fp6_inv(d, d);
  fp6_mul(r.c0, a.c0, d);
  fp6_mul(t, a.c1, d);
  fp6_neg(r.c1, t);
}

// ---- squaring in the cyclotomic subgroup (Granger-Scott): 3 Fp4 squarings = 9 Fp2 squarings ------------------------------------
// Valid only for elements of order dividing p^4 - p^2 + 1, i.e. after the easy part of a final exponentiation; checked against
// the generic fp12_sqr in the tests.  Slots: z0 = c0.c0, z4 = c0.c1, z3 = c0.c2, z2 = c1.c0, z1 = c1.c1, z5 = c1.c2; every
// output slot depends on its own input slot and one Fp4 square, so r may alias f.
// Everything here is out of line and BY REFERENCE on purpose: every live Fp2 of a caller is 2 N registers that the interprocedural
// register allocation takes away from the field products underneath.  With the ten Fp2 values of the textbook formulation held by
// value in one function, ptxas compiled EVERY fp_mul of the pairing kernels with ~120 extra moves and a callee-save spill
// (500 instead of 385 instructions, in the function that is 72 % of the run time); tools/codegen_check.py keeps watch.
template <class T>
B2K_NI void fp4_sqr(Fp2<typename T::Base>& c0, Fp2<typename T::Base>& c1, const Fp2<typename T::Base>& a, const Fp2<typename T::Base>& b) {
  Fp2<typename T::Base> t0, t1, t2;
  fp2_sqr(t0, a);
  fp2_sqr(t1, b);
  T::mul_xi(t2, t1);
  fp2_add(c0, t2, t0);
  fp2_add(t2, a, b);
  fp2_sqr(t2, t2);
  fp2_sub(t2, t2, t0);
  fp2_sub(c1, t2, t1);
}
// r = 3 t + 2 z (SIGN = +1) or 3 t - 2 z (SIGN = -1); r may alias z
template <int SIGN, class C>
B2K_NI void cyclotomic_fix(Fp2<C>& r, const Fp2<C>& t, const Fp2<C>& z) {
  Fp2<C> u;
  if (SIGN > 0) fp2_add(u, t, z); else fp2_sub(u, t, z);
  fp2_dbl(u, u);
  fp2_add(r, u, t);
}
template <class T>
B2K_NI void fp12_cyclotomic_sqr(Fp12<T>& r, const Fp12<T>& f) {
  Fp2<typename T::Base> t0, t1, t2, t3, t4, t5;
  fp4_sqr<T>(t0, t1, f.c0.c0, f.c1.c1);          // (z0, z1)
  fp4_sqr<T>(t2, t3, f.c1.c0, f.c0.c2);          // (z2, z3)
  fp4_sqr<T>(t4, t5, f.c0.c1, f.c1.c2);          // (z4, z5)
  T::mul_xi(t5, t5);
  cyclotomic_fix<-1>(r.c0.c0, t0, f.c0.c0);      // z0 = 3 t0 - 2 z0
  cyclotomic_fix<+1>(r.c1.c1, t1, f.c1.c1);      // z1 = 3 t1 + 2 z1
  cyclotomic_fix<-1>(r.c0.c1, t2, f.c0.c1);      // z4 = 3 t2 - 2 z4
  cyclotomic_fix<+1>(r.c1.c2, t3, f.c1.c2);      // z5 = 3 t3 + 2 z5
  cyclotomic_fix<+1>(r.c1.c0, t5, f.c1.c0);      // z2 = 3 xi t5 + 2 z2
  cyclotomic_fix<-1>(r.c0.c2, t4, f.c0.c2);      // z3 = 3 t4 - 2 z3
}

}  // namespace b2k
