// b2k_bn256.cu -- C ABI entry points for bn256: G1/G2 Point.Mul batches, MSM and pairings.
#include "msm_host.cuh"
#include "bn256.cuh"
#include "bn_pairing.cuh"
#define B2K_COOP_BN256 1
#include "coop_pairing.cuh"          // small batches: one warp per pairing
using namespace b2k_host;

namespace b2k {
using PC6 = Bn256Pair;
using Coop256 = coop::Curve<Bn256G1, Bn256G2, Bn256Fp, PFp12<Bn256Pair>, coop::BN256_P1, coop::BN256_P2>;

// pairing/bn256/suite.go:99-105 Pair -> optimalAte (optate.go:266-274): identity when an operand is infinity
__global__ void __launch_bounds__(64, 4) k_bn256_pair(size_t n, const uint8_t* __restrict__ g1, const uint8_t* __restrict__ g2,
                                                      uint8_t* __restrict__ gt, uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<PFp<PC6>> P;
  Affine<PFp2<PC6>> Q;
  bool good = load_checked<Bn256G1>(P, g1 + 64 * i);
  good = load_checked<Bn256G2>(Q, g2 + 128 * i) && good;
  if (!good) atomicOr(flags, FLAG_POINT);
  PFp12<PC6> f, e;
  bn_miller_loop<PC6, 1>(f, &P, &Q);
  bn_final_exponentiation<PC6>(e, f);
  if (aff_is_inf(P) || aff_is_inf(Q)) fp12_set_one(e);
  bn_gt_store<PC6>(gt + 384 * i, e);
}

// ok[i] = e(a1,a2) == e(b1,b2)   (bn256 ValidatePairing = two pairings + Equal, suite.go:107-109)
__global__ void __launch_bounds__(64, 4) k_bn256_pairing_check(size_t n, const uint8_t* __restrict__ a1,
                                                               const uint8_t* __restrict__ a2, const uint8_t* __restrict__ b1,
                                                               const uint8_t* __restrict__ b2, uint8_t* __restrict__ ok, uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<PFp<PC6>> P[2];
  Affine<PFp2<PC6>> Q[2];
  bool good = load_checked<Bn256G1>(P[0], a1 + 64 * i);
  good = load_checked<Bn256G2>(Q[0], a2 + 128 * i) && good;
  good = load_checked<Bn256G1>(P[1], b1 + 64 * i) && good;
  good = load_checked<Bn256G2>(Q[1], b2 + 128 * i) && good;
  if (!good) { atomicOr(flags, FLAG_POINT); ok[i] = 0; return; }
  fp_neg(P[1].y, P[1].y);
  PFp12<PC6> f, e;
  bn_miller_loop<PC6, 2>(f, P, Q);
  bn_final_exponentiation<PC6>(e, f);
  ok[i] = fp12_is_one(e) ? 1 : 0;
}
}  // namespace b2k

extern "C" {
int b2k_bn256_g1_mul_batch(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return mul_batch_host<Bn256G1, false>(c, n, s, p, o); }
int b2k_bn256_g1_msm(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return msm_host<Bn256G1>(c, n, s, p, o); }
int b2k_bn256_g2_mul_batch(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return mul_batch_host<Bn256G2, false>(c, n, s, p, o); }
int b2k_bn256_g2_msm(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return msm_host<Bn256G2>(c, n, s, p, o); }

int b2k_bn256_pair(b2k_ctx* ctx, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* gt) {
  if (!ctx || !g1 || !g2 || !gt || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  uint8_t *d1 = nullptr, *d2 = nullptr, *dg = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d1 = c.in(g1, n, 64);
    d2 = c.in(g2, n, 128);
    dg = c.out(gt, n, 384);
  }, [&]() -> int {
    cudaStream_t st = ctx->stream;
    if (ctx->coop_max_n > 0 && n <= (size_t)(ctx->coop_max_n < 8192 ? ctx->coop_max_n : 8192))   // break-even measured near 8 192 on this curve
      coop::k_coop_bn_pair<Coop256, PC6><<<(unsigned)n, 32, Coop256::L::BYTES, st>>>(n, d1, d2, dg, ctx->d_flags);
    else
      k_bn256_pair<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(n, d1, d2, dg, ctx->d_flags);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  });
}

int b2k_bn256_pairing_check(b2k_ctx* ctx, size_t n, const uint8_t* a1, const uint8_t* a2, const uint8_t* b1,
                            const uint8_t* b2, uint8_t* ok) {
  if (!ctx || !a1 || !a2 || !b1 || !b2 || !ok || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  uint8_t *da1 = nullptr, *da2 = nullptr, *db1 = nullptr, *db2 = nullptr, *dok = nullptr;
  const int rc = host_call(ctx, [&](Carve& c) {
    da1 = c.in(a1, n, 64);
    da2 = c.in(a2, n, 128);
    db1 = c.in(b1, n, 64);
    db2 = c.in(b2, n, 128);
    dok = c.out(ok, n);
  }, [&]() -> int {
    cudaStream_t st = ctx->stream;
    if (ctx->coop_max_n > 0 && n <= (size_t)(ctx->coop_max_n < 8192 ? ctx->coop_max_n : 8192))   // break-even measured near 8 192 on this curve
      coop::k_coop_bn_pairing_check<Coop256><<<(unsigned)n, 32, Coop256::L::BYTES, st>>>(n, da1, da2, db1, db2, dok, ctx->d_flags);
    else
      k_bn256_pairing_check<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(n, da1, da2, db1, db2, dok, ctx->d_flags);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  });
  return rc == B2K_ERR_POINT ? B2K_OK : rc;   // a malformed operand already failed its own check
}
}  // extern "C"
