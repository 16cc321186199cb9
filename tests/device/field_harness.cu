// field_harness.cu -- test-only entry points into the field and tower arithmetic (fp.cuh, fp_inv.cuh, tower.cuh, pairing.cuh,
// bn_pairing.cuh, codec.cuh), one case per thread on RAW MONTGOMERY LIMBS, so that a test picks the limb patterns itself.
// Not a library unit.  Built three times by __graft_entry__.build() with the library's NVCC_FLAGS:
//   libfield_harness_compact.so   -DB2K_COMPACT_FIELD=1 (the library's default layout: out-of-line by-value products)
//   libfield_harness_byref.so     -DB2K_COMPACT_FIELD=1 -DB2K_FP2_BYREF (the by-reference Fp2 product of b2k_g2.cu)
//   libfield_harness_inlined.so   without B2K_COMPACT_FIELD (the layout of the *_inlined.cu units)
// and by g++ with -DB2K_HOST_EMUL (tests/test_field_arith_emulation.py), where every carry-chain instruction of ptx.cuh is
// emulated in C: the same case list on both tells the code generation of the device apart from the limb algorithm.
//
// Entry points (all return a cudaError_t, 0 on the host):
//   fh_fp_<field>(op, alias, n, in, out)     in: n x 4 operands (a, b, c, d) of N words; out: n x N words
//   fh_tw_<tower>(op, alias, n, in, out)     in: n x 2 Fp12 (a, b) of 12 N words; out: n x (12 N + 1) words, the last one a flag
// An Fp12 travels as its 12 Fp coefficients in tower order c0.c0.c0, c0.c0.c1, c0.c1.c0, ..., c1.c2.c1; an Fp2 or Fp6 operand is
// the leading 2 or 6 of them.  alias selects how the result and the operands share storage: 0 none, 1 op(x, x, y) (the result
// overwrites the first operand), 2 op(y, x, y) (the result overwrites the second), 3 op(x, x, x) (every operand is the first).
#include "../../kyber_b200/csrc/constants.cuh"
#include "../../kyber_b200/csrc/codec.cuh"
#include "../../kyber_b200/csrc/bn_pairing.cuh"
#include <stddef.h>
#include <type_traits>
#ifdef __CUDACC__
#include <cuda_runtime.h>
#endif

using namespace b2k;

namespace {

enum FpOp {
  FP_ADD, FP_SUB, FP_NEG, FP_DBL, FP_ADDSUB_PLUS, FP_ADDSUB_MINUS, FP_MUL, FP_SQR, FP_MUL_I, FP_MUL_SUM2, FP_TO_MONT, FP_FROM_MONT,
  FP_INV, FP_INV_FERMAT, FP_INV_VARTIME, FP_POW_SQRT, FP_POW_LEGENDRE, FP_POW_P58, FP_GT_HALF, FP_LT_MOD, FP_STORE_BE, FP_LOAD_BE
};
enum TwOp {
  F2_MUL, F2_SQR, F2_INV, F2_MUL_LAZY, F2_MUL_XI, F6_MUL, F6_SQR, F6_INV, F6_MUL_BY_01, F6_MUL_BY_1,
  F12_MUL, F12_SQR, F12_INV, F12_CONJ, F12_CYCLOTOMIC_SQR, F12_FROB1, F12_FROB2, F12_FROB3, BLS_FP_SQRT, BLS_FP2_SQRT
};

// the exponents a field configuration carries (constants.cuh): ExpSqrt, ExpLegendre, ExpP58
template <class C, class = void> struct HasSqrt : std::false_type {};
template <class C> struct HasSqrt<C, std::void_t<typename C::ExpSqrt>> : std::true_type {};
template <class C, class = void> struct HasLegendre : std::false_type {};
template <class C> struct HasLegendre<C, std::void_t<typename C::ExpLegendre>> : std::true_type {};
template <class C, class = void> struct HasP58 : std::false_type {};
template <class C> struct HasP58<C, std::void_t<typename C::ExpP58>> : std::true_type {};

template <class C> B2K_D void ld(Fp<C>& r, const uint32_t* p) {
  for (int j = 0; j < C::N; j++) r.v[j] = p[j];
}
template <class C> B2K_D void st(uint32_t* p, const Fp<C>& a) {
  for (int j = 0; j < C::N; j++) p[j] = a.v[j];
}
template <class C> B2K_D void set_flag(Fp<C>& r, bool f) {
  fp_set_zero(r);
  r.v[0] = f ? 1u : 0u;
}

// r = op(a, b, c, d); r may be the same object as any operand (the caller picks the aliasing)
template <class C>
B2K_D void fp_apply(int op, Fp<C>& r, const Fp<C>& a, const Fp<C>& b, const Fp<C>& c, const Fp<C>& d) {
  switch (op) {
    case FP_ADD: fp_add(r, a, b); break;
    case FP_SUB: fp_sub(r, a, b); break;
    case FP_NEG: fp_neg(r, a); break;
    case FP_DBL: fp_dbl(r, a); break;
    case FP_ADDSUB_PLUS: fp_addsub(r, a, b, false); break;
    case FP_ADDSUB_MINUS: fp_addsub(r, a, b, true); break;
    case FP_MUL: fp_mul(r, a, b); break;
    case FP_SQR: fp_sqr(r, a); break;
    case FP_MUL_I: fp_mul_i(r, a, b); break;
    case FP_MUL_SUM2: fp_mul_sum2(r, a, b, c, d); break;
    case FP_TO_MONT: fp_to_mont(r, a); break;
    case FP_FROM_MONT: fp_from_mont(r, a); break;
    case FP_INV: fp_inv(r, a); break;
    case FP_INV_FERMAT: fp_inv_fermat(r, a); break;
    case FP_INV_VARTIME: fp_inv_vartime(r, a); break;
    case FP_POW_SQRT:
      if constexpr (HasSqrt<C>::value) fp_pow_const<C, typename C::ExpSqrt>(r, a); else fp_set_zero(r);
      break;
    case FP_POW_LEGENDRE:
      if constexpr (HasLegendre<C>::value) fp_pow_const<C, typename C::ExpLegendre>(r, a); else fp_set_zero(r);
      break;
    case FP_POW_P58:
      if constexpr (HasP58<C>::value) fp_pow_const<C, typename C::ExpP58>(r, a); else fp_set_zero(r);
      break;
    case FP_GT_HALF: set_flag(r, fp_canon_gt_half(a)); break;
    case FP_LT_MOD: set_flag(r, fp_canon_lt_mod(a)); break;
    case FP_STORE_BE: {                       // the 4 N big-endian bytes, read back as little-endian words
      uint8_t buf[4 * C::N];
      fp_store_be(buf, a);
      for (int j = 0; j < C::N; j++)
        r.v[j] = buf[4 * j] | ((uint32_t)buf[4 * j + 1] << 8) | ((uint32_t)buf[4 * j + 2] << 16) | ((uint32_t)buf[4 * j + 3] << 24);
      break;
    }
    case FP_LOAD_BE: {                        // the words of a as little-endian bytes, parsed as a big-endian number
      uint8_t buf[4 * C::N];
      for (int j = 0; j < C::N; j++) {
        buf[4 * j] = (uint8_t)a.v[j]; buf[4 * j + 1] = (uint8_t)(a.v[j] >> 8);
        buf[4 * j + 2] = (uint8_t)(a.v[j] >> 16); buf[4 * j + 3] = (uint8_t)(a.v[j] >> 24);
      }
      fp_load_be(r, buf);
      break;
    }
    default: fp_set_zero(r);
  }
}

template <class C>
B2K_D void fp_case(int op, int alias, const uint32_t* in, uint32_t* out) {
  constexpr int N = C::N;
  Fp<C> a, b, c, d, r;
  ld(a, in); ld(b, in + N); ld(c, in + 2 * N); ld(d, in + 3 * N);
  switch (alias) {
    case 1: fp_apply(op, a, a, b, c, d); r = a; break;
    case 2: fp_apply(op, b, a, b, c, d); r = b; break;
    case 3: fp_apply(op, a, a, a, a, a); r = a; break;
    default: fp_apply(op, r, a, b, c, d);
  }
  st(out, r);
}

// ---- towers: the Fp12 in / out helpers and the Frobenius map of each configuration ----------------------------------------
template <class T> using TFp = Fp<typename T::Base>;
template <class T> using TFp2 = Fp2<typename T::Base>;

template <class T> B2K_D void ld12(Fp12<T>& r, const uint32_t* p) {
  constexpr int N = T::Base::N;
  Fp6<T>* h[2] = {&r.c0, &r.c1};
  for (int i = 0; i < 2; i++) {
    TFp2<T>* q[3] = {&h[i]->c0, &h[i]->c1, &h[i]->c2};
    for (int k = 0; k < 3; k++) { ld(q[k]->c0, p + (6 * i + 2 * k) * N); ld(q[k]->c1, p + (6 * i + 2 * k + 1) * N); }
  }
}
template <class T> B2K_D void st12(uint32_t* p, const Fp12<T>& a) {
  constexpr int N = T::Base::N;
  const Fp6<T>* h[2] = {&a.c0, &a.c1};
  for (int i = 0; i < 2; i++) {
    const TFp2<T>* q[3] = {&h[i]->c0, &h[i]->c1, &h[i]->c2};
    for (int k = 0; k < 3; k++) { st(p + (6 * i + 2 * k) * N, q[k]->c0); st(p + (6 * i + 2 * k + 1) * N, q[k]->c1); }
  }
}

struct BlsH {
  using T = Bls381Tower;
  static constexpr bool IS_BLS = true;
  template <int J> B2K_D static void frob(Fp12<T>& r, const Fp12<T>& a) { fp12_frobenius<J>(r, a); }
};
template <class PC> struct BnH {
  using T = typename PC::T;
  static constexpr bool IS_BLS = false;
  template <int J> B2K_D static void frob(Fp12<T>& r, const Fp12<T>& a) { bn_frobenius<PC, J>(r, a); }
};

// r = op(a, b) on the level of the operation (Fp2: a.c0.c0, Fp6: a.c0, Fp12: a); flag = the boolean result of a square root
template <class H>
B2K_D void tw_apply(int op, Fp12<typename H::T>& r, const Fp12<typename H::T>& a, const Fp12<typename H::T>& b, bool& flag) {
  using T = typename H::T;
  switch (op) {
    case F2_MUL: fp2_mul(r.c0.c0, a.c0.c0, b.c0.c0); break;
    case F2_SQR: fp2_sqr(r.c0.c0, a.c0.c0); break;
    case F2_INV: fp2_inv(r.c0.c0, a.c0.c0); break;
    case F2_MUL_LAZY: fp2_mul_lazy(r.c0.c0, a.c0.c0, b.c0.c0); break;
    case F2_MUL_XI: T::mul_xi(r.c0.c0, a.c0.c0); break;
    case F6_MUL: fp6_mul(r.c0, a.c0, b.c0); break;
    case F6_SQR: fp6_sqr(r.c0, a.c0); break;
    case F6_INV: fp6_inv(r.c0, a.c0); break;
    case F6_MUL_BY_01: fp6_mul_by_01(r.c0, a.c0, b.c0.c0, b.c0.c1); break;
    case F6_MUL_BY_1: fp6_mul_by_1(r.c0, a.c0, b.c0.c0); break;
    case F12_MUL: fp12_mul(r, a, b); break;
    case F12_SQR: fp12_sqr(r, a); break;
    case F12_INV: fp12_inv(r, a); break;
    case F12_CONJ: fp12_conj(r, a); break;
    case F12_CYCLOTOMIC_SQR: fp12_cyclotomic_sqr(r, a); break;
    case F12_FROB1: H::template frob<1>(r, a); break;
    case F12_FROB2: H::template frob<2>(r, a); break;
    case F12_FROB3: H::template frob<3>(r, a); break;
    case BLS_FP_SQRT:
      if constexpr (H::IS_BLS) flag = fp_sqrt(r.c0.c0.c0, a.c0.c0.c0);
      break;
    case BLS_FP2_SQRT:
      if constexpr (H::IS_BLS) flag = fp2_sqrt(r.c0.c0, a.c0.c0);
      break;
    default: break;
  }
}

template <class H>
B2K_D void tw_case(int op, int alias, const uint32_t* in, uint32_t* out) {
  using T = typename H::T;
  constexpr int N = T::Base::N;
  Fp12<T> a, b, r;
  ld12(a, in); ld12(b, in + 12 * N);
  bool flag = false;
  // unused result coefficients come back as zero (the operations below write only their own level)
  fp6_set_zero(r.c0); fp6_set_zero(r.c1);
  switch (alias) {
    case 1: tw_apply<H>(op, a, a, b, flag); r = a; break;
    case 2: tw_apply<H>(op, b, a, b, flag); r = b; break;
    case 3: tw_apply<H>(op, a, a, a, flag); r = a; break;
    default: tw_apply<H>(op, r, a, b, flag);
  }
  st12(out, r);
  out[12 * N] = flag ? 1u : 0u;
}

#ifdef __CUDACC__
template <class C>
__global__ void k_fp(int op, int alias, int n, const uint32_t* in, uint32_t* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  fp_case<C>(op, alias, in + (size_t)i * 4 * C::N, out + (size_t)i * C::N);
}
template <class H>
__global__ void k_tw(int op, int alias, int n, const uint32_t* in, uint32_t* out) {
  constexpr int N = H::T::Base::N;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  tw_case<H>(op, alias, in + (size_t)i * 24 * N, out + (size_t)i * (12 * N + 1));
}

// H2D, one launch, D2H; every step's status is returned (the first failure wins)
template <class K>
int run(K kernel, int op, int alias, int n, const uint32_t* in, size_t in_words, uint32_t* out, size_t out_words) {
  if (n <= 0) return 0;
  uint32_t *d_in = nullptr, *d_out = nullptr;
  cudaError_t e = cudaMalloc(&d_in, in_words * n * 4);
  if (e == cudaSuccess) e = cudaMalloc(&d_out, out_words * n * 4);
  if (e == cudaSuccess) e = cudaMemcpy(d_in, in, in_words * n * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    kernel<<<(n + 127) / 128, 128>>>(op, alias, n, d_in, d_out);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpy(out, d_out, out_words * n * 4, cudaMemcpyDeviceToHost);
  cudaFree(d_in);
  cudaFree(d_out);
  return (int)e;
}
template <class C> int run_fp(int op, int alias, int n, const uint32_t* in, uint32_t* out) {
  return run(k_fp<C>, op, alias, n, in, 4 * C::N, out, C::N);
}
template <class H> int run_tw(int op, int alias, int n, const uint32_t* in, uint32_t* out) {
  constexpr int N = H::T::Base::N;
  return run(k_tw<H>, op, alias, n, in, 24 * N, out, 12 * N + 1);
}
#else
template <class C> int run_fp(int op, int alias, int n, const uint32_t* in, uint32_t* out) {
  for (int i = 0; i < n; i++) fp_case<C>(op, alias, in + (size_t)i * 4 * C::N, out + (size_t)i * C::N);
  return 0;
}
template <class H> int run_tw(int op, int alias, int n, const uint32_t* in, uint32_t* out) {
  constexpr int N = H::T::Base::N;
  for (int i = 0; i < n; i++) tw_case<H>(op, alias, in + (size_t)i * 24 * N, out + (size_t)i * (12 * N + 1));
  return 0;
}
#endif

}  // namespace

extern "C" {
#define FH_FP(name, C) \
  int fh_fp_##name(int op, int alias, int n, const uint32_t* in, uint32_t* out) { return run_fp<C>(op, alias, n, in, out); }
#define FH_TW(name, H) \
  int fh_tw_##name(int op, int alias, int n, const uint32_t* in, uint32_t* out) { return run_tw<H>(op, alias, n, in, out); }
FH_FP(bls381_fp, Bls381Fp)
FH_FP(bls381_fr, Bls381Fr)
FH_FP(bn254_fp, Bn254Fp)
FH_FP(bn254_fr, Bn254Fr)
FH_FP(bn256_fp, Bn256Fp)
FH_FP(ed25519_fp, Ed25519Fp)
FH_FP(ed25519_fr, Ed25519Fr)
FH_TW(bls381, BlsH)
FH_TW(bn254, BnH<Bn254Pair>)
FH_TW(bn256, BnH<Bn256Pair>)
}
