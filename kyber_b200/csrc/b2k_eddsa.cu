// b2k_eddsa.cu -- C ABI entry points for batched Ed25519 signature verification: eddsa.VerifyWithChecks
// (sign/eddsa/eddsa.go:149-229) for n signatures per call, one thread each (eddsa.cuh).
#include "msm_host.cuh"
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
  k_ed25519_verify<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(n, (const uint8_t*)d_pks, (const uint8_t*)d_msgs,
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
  const size_t mbytes = offsets[n];
  const size_t o_pk = 0, o_sig = o_pk + n * 32, o_msg = o_sig + n * 64, o_off = (o_msg + mbytes + 15) & ~size_t(15),
               o_st = o_off + (n + 1) * 4, total = o_st + n;
  uint8_t* blob = (uint8_t*)b2k_arena_in(ctx, total);  // the context's input arena: one allocation, reused across calls
  if (!blob) { ctx->err = "out of device memory"; return B2K_ERR_CUDA; }
  cudaStream_t st = ctx->stream;
  int rc = B2K_OK;
  do {
    if (cudaMemcpyAsync(blob + o_pk, pks, n * 32, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(blob + o_sig, sigs, n * 64, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        (mbytes && cudaMemcpyAsync(blob + o_msg, msgs, mbytes, cudaMemcpyHostToDevice, st) != cudaSuccess) ||
        cudaMemcpyAsync(blob + o_off, offsets, (n + 1) * 4, cudaMemcpyHostToDevice, st) != cudaSuccess) { rc = B2K_ERR_CUDA; break; }
    rc = b2k_ed25519_verify_dev(ctx, n, blob + o_pk, blob + o_msg, blob + o_off, blob + o_sig, blob + o_st);
    if (rc) break;
    if (cudaMemcpyAsync(status, blob + o_st, n, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) rc = B2K_ERR_CUDA;
  } while (0);
  cudaStreamSynchronize(st);
  if (rc == B2K_ERR_CUDA) ctx->err = "CUDA failure in ed25519_verify";
  return rc;
}

}  // extern "C"
