// b2k_bn_codec.cu -- batched UnmarshalBinary validation for the BN curves (SURVEY 8f row 2: wire-format checks on device).
//
// What the reference's UnmarshalBinary accepts, per point of a batch (ok[i] = 1 when the Go call would return nil):
//   bn254 G1  pairing/bn254/point.go:146-185   every coordinate below p (gfP.Unmarshal, gfp.go:101-119), then on the curve
//                                               y^2 = x^3 + 3; 64 zero bytes = infinity
//   bn254 G2  pairing/bn254/point.go:473-523   coordinates below p, on the twist y^2 = x^3 + 3/(9+i) AND killed by the group
//                                               order (twistPoint.IsOnCurve, twist.go:50-66: cneg.Mul(c, Order) must be infinity)
//   bn256 G1  pairing/bn256/point.go:206-238   NO range check (gfP.Unmarshal, gfp.go:115-122, montEncode reduces), on the curve
//   bn256 G2  pairing/bn256/point.go:469-506   no range check, on the twist y^2 = x^3 + 3/(3+i); no order check
//                                               (twist.go:50-61)
// The engine's Mul/MSM/pairing entry points take operands that passed these checks (what a Go adapter holds after
// UnmarshalBinary); these kernels are that gate for whole batches.
#include "msm_host.cuh"
#include "bn256.cuh"
#include "bn_pairing.cuh"
using namespace b2k_host;

namespace b2k {

template <class C> B2K_D void bn_raw32(Fp<C>& r, const uint8_t* p) {      // 32 bytes big-endian -> plain limbs (upper limbs zero)
#pragma unroll
  for (int j = 0; j < C::N; j++) r.v[j] = 0;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const uint8_t* q = p + 4 * (7 - j);
    r.v[j] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
  }
}

template <class C> B2K_D void bn_curve_b(Fp<C>& b) {
#pragma unroll
  for (int j = 0; j < C::N; j++) b.v[j] = C::curve_b(j);
}
template <class C> B2K_D void bn_curve_b(Fp2<C>& b) {
#pragma unroll
  for (int j = 0; j < C::N; j++) { b.c0.v[j] = C::twist_b_c0(j); b.c1.v[j] = C::twist_b_c1(j); }
}

// NC = base-field coordinates per point (2 for G1, 4 for G2, in wire order)
template <class CV, int NC, bool RANGE_CHECK, bool ORDER_CHECK>
__global__ void __launch_bounds__(128) k_bn_unmarshal_check(size_t n, const uint8_t* __restrict__ in, uint8_t* __restrict__ ok) {
  using F = typename CV::F;
  using FC = typename CV::FC;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* w = in + (size_t)CV::IN_BYTES * i;
  if (RANGE_CHECK) {
    for (int c = 0; c < NC; c++) {
      Fp<FC> t;
      bn_raw32(t, w + 32 * c);
      if (!fp_canon_lt_mod(t)) { ok[i] = 0; return; }
    }
  }
  Affine<F> p;
  CV::load(p, w);
  if (aff_is_inf(p)) { ok[i] = 1; return; }
  F y2, x3, b;
  f_sqr(y2, p.y);
  f_sqr(x3, p.x); f_mul(x3, x3, p.x);
  bn_curve_b(b);
  f_add(x3, x3, b);
  bool good = f_eq(y2, x3);
  if (ORDER_CHECK && good) {
    Scalar256 ord;
#pragma unroll
    for (int j = 0; j < 8; j++) ord.v[j] = CV::ScalarField::mod(j);
    Jac<F> r;
    scalar_mul<CV>(r, ord, p);
    good = jac_is_inf(r);
  }
  ok[i] = good ? 1 : 0;
}

}  // namespace b2k

template <class CV, int NC, bool RANGE_CHECK, bool ORDER_CHECK>
static int bn_unmarshal_check(b2k_ctx* ctx, size_t n, const uint8_t* in, uint8_t* ok) {
  if (!ctx || !in || !ok || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  uint8_t *d_in = nullptr, *d_ok = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_in = c.in(in, n, CV::IN_BYTES);
    d_ok = c.out(ok, n);
  }, [&]() -> int {
    k_bn_unmarshal_check<CV, NC, RANGE_CHECK, ORDER_CHECK><<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(n, d_in, d_ok);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  });
}

extern "C" {
int b2k_bn254_g1_unmarshal_check(b2k_ctx* c, size_t n, const uint8_t* in, uint8_t* ok) { return bn_unmarshal_check<Bn254G1, 2, true, false>(c, n, in, ok); }
int b2k_bn254_g2_unmarshal_check(b2k_ctx* c, size_t n, const uint8_t* in, uint8_t* ok) { return bn_unmarshal_check<Bn254G2, 4, true, true>(c, n, in, ok); }
int b2k_bn256_g1_unmarshal_check(b2k_ctx* c, size_t n, const uint8_t* in, uint8_t* ok) { return bn_unmarshal_check<Bn256G1, 2, false, false>(c, n, in, ok); }
int b2k_bn256_g2_unmarshal_check(b2k_ctx* c, size_t n, const uint8_t* in, uint8_t* ok) { return bn_unmarshal_check<Bn256G2, 4, false, false>(c, n, in, ok); }
}  // extern "C"
