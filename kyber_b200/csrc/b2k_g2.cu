// b2k_g2.cu -- C ABI entry points for BLS12-381 G2 (Point.Mul batches, MSM) and for batched ZCash
// decompression + subgroup checks of G1/G2 (UnmarshalBinary, kilic/g1.go:127-131, g2.go:126-130).
#define B2K_FP2_BYREF 1   // Fp2 products out of line BY REFERENCE (tower.cuh): the G2 MSM / Point.Mul kernels of this unit hold whole Fp2 points by value
#include "msm_host.cuh"
#include "codec.cuh"
using namespace b2k_host;

namespace b2k {
// out[i] = operand-form point, ok[i] = 1 for a valid encoding of a subgroup point, else 0 (out zeroed)
__global__ void __launch_bounds__(128) k_g1_decompress(size_t n, const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                                                       uint8_t* __restrict__ ok, int check_subgroup) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<BFp> a;
  bool good = g1_decompress(a, in + 48 * i, check_subgroup != 0);
  if (!good) aff_set_inf(a);
  Bls381G1::store_affine(out + 96 * i, a);
  ok[i] = good ? 1 : 0;
}
__global__ void __launch_bounds__(64) k_g2_decompress(size_t n, const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                                                      uint8_t* __restrict__ ok, int check_subgroup) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<BFp2> a;
  bool good = g2_decompress(a, in + 96 * i, check_subgroup != 0);
  if (!good) aff_set_inf(a);
  Bls381G2::store_affine(out + 192 * i, a);
  ok[i] = good ? 1 : 0;
}
}  // namespace b2k

// stage the wire bytes, then the *_dev entry point
template <class Dev>
static int decompress_host(b2k_ctx* ctx, size_t n, const uint8_t* in, uint8_t* out, uint8_t* ok, size_t in_bytes, size_t out_bytes, Dev dev) {
  if (!ctx || !in || !out || !ok || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  uint8_t *di = nullptr, *dout = nullptr, *dk = nullptr;
  return host_call(ctx, [&](Carve& c) {
    di = c.in(in, n, in_bytes);
    dout = c.out(out, n, out_bytes);
    dk = c.out(ok, n);
  }, [&] { return dev(ctx, n, di, dout, dk); });
}

extern "C" {
int b2k_bls12381_g1_decompress_dev(b2k_ctx* ctx, size_t n, const void* in, void* out, void* ok) {
  if (!ctx || !in || !out || !ok || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  k_g1_decompress<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(n, (const uint8_t*)in, (uint8_t*)out, (uint8_t*)ok, 1);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return B2K_OK;
}
int b2k_bls12381_g2_decompress_dev(b2k_ctx* ctx, size_t n, const void* in, void* out, void* ok) {
  if (!ctx || !in || !out || !ok || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  k_g2_decompress<<<(unsigned)((n + 63) / 64), 64, 0, ctx->stream>>>(n, (const uint8_t*)in, (uint8_t*)out, (uint8_t*)ok, 1);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return B2K_OK;
}
int b2k_bls12381_g1_decompress(b2k_ctx* ctx, size_t n, const uint8_t* in, uint8_t* out, uint8_t* ok) {
  return decompress_host(ctx, n, in, out, ok, 48, 96, b2k_bls12381_g1_decompress_dev);
}
int b2k_bls12381_g2_decompress(b2k_ctx* ctx, size_t n, const uint8_t* in, uint8_t* out, uint8_t* ok) {
  return decompress_host(ctx, n, in, out, ok, 96, 192, b2k_bls12381_g2_decompress_dev);
}
int b2k_bls12381_g2_mul_batch(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return mul_batch_host<Bls381G2, false>(c, n, s, p, o); }
int b2k_bls12381_g2_mul_batch_affine(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return mul_batch_host<Bls381G2, true>(c, n, s, p, o); }
int b2k_bls12381_g2_mul_batch_affine_dev(b2k_ctx* c, size_t n, const void* s, const void* p, void* o) { return mul_batch_dev<Bls381G2, true>(c, n, s, p, o); }
int b2k_bls12381_g2_msm(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return msm_host<Bls381G2>(c, n, s, p, o); }
int b2k_bls12381_g2_msm_affine(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return msm_host<Bls381G2>(c, n, s, p, o, 1); }
int b2k_bls12381_g2_msm_dev(b2k_ctx* c, size_t n, const void* s, const void* p, void* o) { return msm_dev<Bls381G2>(c, n, s, p, o); }
}  // extern "C"
