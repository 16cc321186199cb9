// b2k_bn_hash.cu -- C ABI entry points for batched hash-to-G1 on the in-tree BN curves (bn254: Keccak-256 XMD + SvdW,
// pairing/bn254/point.go:208-285; bn256: SHA-256 try-and-increment, pairing/bn256/point.go:261-312).
#include "msm_host.cuh"
#include "bn_hash.cuh"
using namespace b2k_host;

namespace b2k {

__global__ void __launch_bounds__(128) k_bn254_hash_to_g1(size_t n, const uint8_t* __restrict__ msgs, const uint32_t* __restrict__ offs,
                                                          const uint8_t* __restrict__ dst, uint32_t dst_len, uint8_t* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<NFp254> a;
  bn254_hash_to_g1(a, msgs + offs[i], (offs[i + 1] >= offs[i] ? offs[i + 1] - offs[i] : 0u), dst, dst_len);
  Bn254G1::store(out + 64 * i, a);
}

__global__ void __launch_bounds__(128) k_bn256_hash_to_g1(size_t n, const uint8_t* __restrict__ msgs, const uint32_t* __restrict__ offs,
                                                          uint8_t* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<B256Fp> a;
  bn256_hash_to_g1(a, msgs + offs[i], (offs[i + 1] >= offs[i] ? offs[i + 1] - offs[i] : 0u));
  Bn256G1::store(out + 64 * i, a);
}

// bn256 HashG1 (pairing/bn256/hash.go:10-12): dst may be empty (the reference's tests pass nil)
__global__ void __launch_bounds__(128) k_bn256_hash_g1(size_t n, const uint8_t* __restrict__ msgs, const uint32_t* __restrict__ offs,
                                                       const uint8_t* __restrict__ dst, uint32_t dst_len, uint8_t* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<B256Fp> a;
  bn256_hash_g1(a, msgs + offs[i], (offs[i + 1] >= offs[i] ? offs[i + 1] - offs[i] : 0u), dst, dst_len);
  Bn256G1::store(out + 64 * i, a);
}

}  // namespace b2k

using namespace b2k;

// which: 0 = bn254 (dst used), 1 = bn256 try-and-increment (dst ignored), 2 = bn256 HashG1 (dst optional)
static int hash_dev(b2k_ctx* ctx, int which, size_t n, const void* d_msgs, const void* d_offsets, const void* d_dst, uint32_t dst_len,
                    void* d_out) {
  if (!ctx || !d_msgs || !d_offsets || !d_out || n == 0) return B2K_ERR_ARG;
  if (which == 0 && (!d_dst || dst_len == 0 || dst_len > 255)) return B2K_ERR_ARG;
  if (which == 2 && (dst_len > 255 || (dst_len && !d_dst))) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  const unsigned grid = (unsigned)((n + 127) / 128);
  if (which == 2)
    k_bn256_hash_g1<<<grid, 128, 0, ctx->stream>>>(n, (const uint8_t*)d_msgs, (const uint32_t*)d_offsets, (const uint8_t*)d_dst,
                                                  dst_len, (uint8_t*)d_out);
  else if (which == 0)
    k_bn254_hash_to_g1<<<grid, 128, 0, ctx->stream>>>(n, (const uint8_t*)d_msgs, (const uint32_t*)d_offsets, (const uint8_t*)d_dst,
                                                     dst_len, (uint8_t*)d_out);
  else
    k_bn256_hash_to_g1<<<grid, 128, 0, ctx->stream>>>(n, (const uint8_t*)d_msgs, (const uint32_t*)d_offsets, (uint8_t*)d_out);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return B2K_OK;
}

static int hash_host(b2k_ctx* ctx, int which, size_t n, const uint8_t* msgs, const uint32_t* offsets, const uint8_t* dst, uint32_t dst_len,
                     uint8_t* out) {
  if (!ctx || !msgs || !offsets || !out || n == 0) return B2K_ERR_ARG;
  if (which == 0 && (!dst || dst_len == 0 || dst_len > 255)) return B2K_ERR_ARG;
  if (which == 2 && (dst_len > 255 || (dst_len && !dst))) return B2K_ERR_ARG;
  if (check_offsets(ctx, n, offsets)) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  uint8_t *dm = nullptr, *dd = nullptr, *dout = nullptr;
  uint32_t* doff = nullptr;
  return host_call(ctx, [&](Carve& c) {
    dm = c.in(msgs, offsets[n]);
    doff = c.in(offsets, n + 1);
    dd = c.in(dst, dst_len);
    dout = c.out(out, n, 64);
  }, [&] { return hash_dev(ctx, which, n, dm, doff, dd, dst_len, dout); });
}

extern "C" {

int b2k_bn254_hash_to_g1_dev(b2k_ctx* ctx, size_t n, const void* d_msgs, const void* d_offsets, const void* d_dst, uint32_t dst_len,
                             void* d_out) {
  return hash_dev(ctx, 0, n, d_msgs, d_offsets, d_dst, dst_len, d_out);
}
int b2k_bn254_hash_to_g1(b2k_ctx* ctx, size_t n, const uint8_t* msgs, const uint32_t* offsets, const uint8_t* dst, uint32_t dst_len,
                         uint8_t* out) {
  return hash_host(ctx, 0, n, msgs, offsets, dst, dst_len, out);
}
int b2k_bn256_hash_to_g1_dev(b2k_ctx* ctx, size_t n, const void* d_msgs, const void* d_offsets, void* d_out) {
  return hash_dev(ctx, 1, n, d_msgs, d_offsets, nullptr, 0, d_out);
}
int b2k_bn256_hash_to_g1(b2k_ctx* ctx, size_t n, const uint8_t* msgs, const uint32_t* offsets, uint8_t* out) {
  return hash_host(ctx, 1, n, msgs, offsets, nullptr, 0, out);
}
int b2k_bn256_hash_g1_dev(b2k_ctx* ctx, size_t n, const void* d_msgs, const void* d_offsets, const void* d_dst, uint32_t dst_len, void* d_out) {
  return hash_dev(ctx, 2, n, d_msgs, d_offsets, d_dst, dst_len, d_out);
}
int b2k_bn256_hash_g1(b2k_ctx* ctx, size_t n, const uint8_t* msgs, const uint32_t* offsets, const uint8_t* dst, uint32_t dst_len, uint8_t* out) {
  return hash_host(ctx, 2, n, msgs, offsets, dst, dst_len, out);
}

}  // extern "C"
