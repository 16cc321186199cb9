// b2k_pairing.cu -- C ABI entry points for batched BLS12-381 pairings (separate translation unit so the
// two large kernel families compile in parallel).
#include <cuda_runtime.h>
#include <string>
#include "../../include/b2kyber.h"
#include "b2k_ctx.h"
#include "pairing_kernels.cuh"
#define B2K_COOP_BLS 1
#include "coop_pairing.cuh"
#include "msm_host.cuh"

using namespace b2k;


extern "C" {

// Miller values of the split kernels: one grow-only buffer per context (nullptr when the allocation fails: the caller falls back to the fused kernel)
static BFp12* pair_scratch(const b2k_ctx* cctx, size_t n) {
  b2k_ctx* ctx = const_cast<b2k_ctx*>(cctx);
  const size_t need = n * sizeof(BFp12);
  if (need > ctx->pair_scratch_cap) {
    cudaStreamSynchronize(ctx->stream);                       // nothing in flight may still read the old buffer
    if (ctx->pair_scratch) cudaFree(ctx->pair_scratch);
    ctx->pair_scratch = nullptr; ctx->pair_scratch_cap = 0;
    void* p = nullptr;
    if (cudaMalloc(&p, need) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    ctx->pair_scratch = p; ctx->pair_scratch_cap = need;
  }
  return reinterpret_cast<BFp12*>(ctx->pair_scratch);
}

void b2k_internal_launch_pair(const b2k_ctx* ctx, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* gt) {
  if (ctx->coop_max_n > 0 && n <= (size_t)ctx->coop_max_n) {       // small batch: one WARP per pairing (coop_pairing.cuh)
    coop::k_coop_pair<<<(unsigned)n, 32, coop::SMEM_BYTES, ctx->stream>>>(n, g1, g2, gt, ctx->d_flags);
    return;
  }
  int v = ctx->pair_variant;
  if (v >= 16) {
    if (BFp12* f = pair_scratch(ctx, n)) { launch_pair_split(ctx, v - 16, n, g1, g2, gt, f); return; }
    v = 0;
  }
  const int layout = v / 4, shape = v % 4;
  if (layout == 1) b2k_internal_launch_pair_inlined(ctx, shape, n, g1, g2, gt);
  else launch_pair_v(ctx, shape, n, g1, g2, gt);
}
void b2k_internal_launch_pairing_check(const b2k_ctx* ctx, size_t n, const uint8_t* a1, const uint8_t* a2, const uint8_t* b1,
                                       const uint8_t* b2, uint8_t* ok, int b2_broadcast, const uint8_t* pre_ok) {
  if (ctx->coop_max_n > 0 && n <= (size_t)ctx->coop_max_n) {
    coop::k_coop_pairing_check<<<(unsigned)n, 32, coop::SMEM_BYTES, ctx->stream>>>(n, a1, a2, b1, b2, ok, b2_broadcast, pre_ok, ctx->d_flags);
    return;
  }
  int v = ctx->pair_variant;
  if (v >= 16) {
    if (BFp12* f = pair_scratch(ctx, n)) { launch_pairing_check_split(ctx, v - 16, n, a1, a2, b1, b2, ok, b2_broadcast, pre_ok, f); return; }
    v = 0;
  }
  const int layout = v / 4, shape = v % 4;
  if (layout == 1) b2k_internal_launch_pairing_check_inlined(ctx, shape, n, a1, a2, b1, b2, ok, b2_broadcast, pre_ok);
  else launch_pairing_check_v(ctx, shape, n, a1, a2, b1, b2, ok, b2_broadcast, pre_ok);
}

int b2k_bls12381_pair_dev(b2k_ctx* ctx, size_t n, const void* d_g1, const void* d_g2, void* d_gt) {
  if (!ctx || !d_g1 || !d_g2 || !d_gt || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  b2k_internal_launch_pair(ctx, n, (const uint8_t*)d_g1, (const uint8_t*)d_g2, (uint8_t*)d_gt);
  CK(cudaGetLastError());
  ctx->launches += (ctx->pair_variant >= 16 && !(ctx->coop_max_n > 0 && n <= (size_t)ctx->coop_max_n)) ? 2 : 1;
  return B2K_OK;
}

int b2k_bls12381_pair(b2k_ctx* ctx, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* gt) {
  if (!ctx || !g1 || !g2 || !gt || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  uint8_t *d1 = nullptr, *d2 = nullptr, *dg = nullptr;
  return b2k_host::host_call(ctx, [&](b2k_host::Carve& c) {
    d1 = c.in(g1, n, 96);
    d2 = c.in(g2, n, 192);
    dg = c.out(gt, n, 576);
  }, [&] { return b2k_bls12381_pair_dev(ctx, n, d1, d2, dg); });
}

int b2k_bls12381_pairing_check_dev(b2k_ctx* ctx, size_t n, const void* a1, const void* a2, const void* b1,
                                   const void* b2, void* d_ok) {
  if (!ctx || !a1 || !a2 || !b1 || !b2 || !d_ok || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  b2k_internal_launch_pairing_check(ctx, n, (const uint8_t*)a1, (const uint8_t*)a2, (const uint8_t*)b1, (const uint8_t*)b2, (uint8_t*)d_ok, 0, nullptr);
  CK(cudaGetLastError());
  ctx->launches += (ctx->pair_variant >= 16 && !(ctx->coop_max_n > 0 && n <= (size_t)ctx->coop_max_n)) ? 2 : 1;
  return B2K_OK;
}

int b2k_bls12381_pairing_check(b2k_ctx* ctx, size_t n, const uint8_t* a1, const uint8_t* a2, const uint8_t* b1,
                               const uint8_t* b2, uint8_t* ok) {
  if (!ctx || !a1 || !a2 || !b1 || !b2 || !ok || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  uint8_t *da1 = nullptr, *da2 = nullptr, *db1 = nullptr, *db2 = nullptr, *dok = nullptr;
  const int rc = b2k_host::host_call(ctx, [&](b2k_host::Carve& c) {
    da1 = c.in(a1, n, 96);
    da2 = c.in(a2, n, 192);
    db1 = c.in(b1, n, 96);
    db2 = c.in(b2, n, 192);
    dok = c.out(ok, n);
  }, [&] { return b2k_bls12381_pairing_check_dev(ctx, n, da1, da2, db1, db2, dok); });
  // a malformed operand already made its own check fail (ok[i] = 0): like the reference's ValidatePairing, the call itself
  // reports per-element booleans, not an error
  return rc == B2K_ERR_POINT ? B2K_OK : rc;
}

int b2k_set_pairing_coop(b2k_ctx* ctx, int max_n) {
  if (!ctx || max_n < 0) return B2K_ERR_ARG;
  ctx->coop_max_n = max_n;
  return B2K_OK;
}

int b2k_set_pairing_variant(b2k_ctx* ctx, int v) {
  if (!ctx || v < 0 || (v < 16 && (v > 7 || (v % 4) == 3)) || v >= 16 + 4) return B2K_ERR_ARG;
  ctx->pair_variant = v;
  return B2K_OK;
}

}  // extern "C"
