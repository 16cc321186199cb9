// b2k_ed25519.cu -- C ABI entry point for batched edwards25519 Point.Mul
// (group/edwards25519/point.go:235-258 called in a loop, e.g. util/test/group.go:118-122).
#include "host_call.cuh"
#include "ed25519.cuh"
using namespace b2k_host;

namespace b2k {
__global__ void __launch_bounds__(128) k_ed25519_mul_batch(size_t n, const uint8_t* __restrict__ scalars,
                                                           const uint8_t* __restrict__ pts, uint8_t* __restrict__ out,
                                                           uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  EdExt p, r;
  if (!ed_decode(p, pts + 32 * i)) {
    atomicOr(flags, FLAG_POINT);
    for (int j = 0; j < 32; j++) out[32 * i + j] = 0;
    return;
  }
  ed_scalar_mul(r, scalars + 32 * i, p);               // geScalarMult: a top digit above 8 selects nothing
  ed_encode(out + 32 * i, r);
}
}  // namespace b2k

extern "C" {
int b2k_ed25519_mul_batch_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points, void* d_out) {
  if (!ctx || !d_scalars || !d_points || !d_out || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  k_ed25519_mul_batch<<<blocks_of(n, 128), 128, 0, ctx->stream>>>(n, (const uint8_t*)d_scalars, (const uint8_t*)d_points,
                                                                  (uint8_t*)d_out, ctx->d_flags);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return B2K_OK;
}
int b2k_ed25519_mul_batch(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out) {
  if (!ctx || !scalars || !points || !out || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  uint8_t *ds = nullptr, *dp = nullptr, *dout = nullptr;
  int rc = arena_carve(ctx, [&](Carve& c) {
    ds = c.take<uint8_t>(n * 32);
    dp = c.take<uint8_t>(n * 32);
    dout = c.take<uint8_t>(n * 32);
  });
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  if ((rc = status_begin(ctx))) return rc;
  CK(cudaMemcpyAsync(ds, scalars, n * 32, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(dp, points, n * 32, cudaMemcpyHostToDevice, st));
  rc = b2k_ed25519_mul_batch_dev(ctx, n, ds, dp, dout);
  if (rc) return rc;
  CK(cudaMemcpyAsync(out, dout, n * 32, cudaMemcpyDeviceToHost, st));
  return status_finish(ctx);
}
}  // extern "C"
