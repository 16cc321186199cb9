// b2k_eddsa.cu -- C ABI entry points for batched Ed25519 signature verification: eddsa.VerifyWithChecks
// (sign/eddsa/eddsa.go:149-229) for n signatures per call, one thread each (eddsa.cuh).
#include "host_call.cuh"
#include "eddsa.cuh"
using namespace b2k_host;

namespace b2k {

__global__ void __launch_bounds__(128) k_ed25519_verify(size_t n, const uint8_t* __restrict__ pks, const uint8_t* __restrict__ msgs,
                                                        const uint32_t* __restrict__ offs, const uint8_t* __restrict__ sigs,
                                                        uint8_t* __restrict__ status) {
  __shared__ EdNiels btab[8];                           // 1..8 B, 768 bytes, read by every thread of the block
  if (threadIdx.x == 0) ed_load_base_table(btab);
  __syncthreads();
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t o0 = offs[i], o1 = offs[i + 1];
  status[i] = (uint8_t)ed_verify(pks + 32 * i, msgs + o0, o1 >= o0 ? o1 - o0 : 0u, sigs + 64 * i, btab);
}

}  // namespace b2k

extern "C" {

int b2k_ed25519_verify_dev(b2k_ctx* ctx, size_t n, const void* d_pks, const void* d_msgs, const void* d_offsets,
                           const void* d_sigs, void* d_status) {
  if (!ctx || !d_pks || !d_msgs || !d_offsets || !d_sigs || !d_status || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  k_ed25519_verify<<<blocks_of(n, 128), 128, 0, ctx->stream>>>(n, (const uint8_t*)d_pks, (const uint8_t*)d_msgs,
                                                                       (const uint32_t*)d_offsets, (const uint8_t*)d_sigs,
                                                                       (uint8_t*)d_status);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return B2K_OK;
}

int b2k_ed25519_verify(b2k_ctx* ctx, size_t n, const uint8_t* pks, const uint8_t* msgs, const uint32_t* offsets,
                       const uint8_t* sigs, uint8_t* status) {
  if (!ctx || !pks || !msgs || !offsets || !sigs || !status || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  if (check_offsets(ctx, n, offsets)) return B2K_ERR_ARG;
  uint8_t *d_pk = nullptr, *d_sig = nullptr, *d_msg = nullptr, *d_st = nullptr;
  uint32_t* d_off = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_pk = c.in(pks, n, 32);
    d_sig = c.in(sigs, n, 64);
    d_msg = c.in(msgs, offsets[n]);
    d_off = c.in(offsets, n + 1);
    d_st = c.out(status, n);
  }, [&] { return b2k_ed25519_verify_dev(ctx, n, d_pk, d_msg, d_off, d_sig, d_st); });
}

}  // extern "C"
