// b2k_schnorr.cu -- C ABI entry points for batched sign/schnorr verification over BLS12-381 keys on G1 or on G2:
// schnorr.VerifyWithChecks (sign/schnorr/schnorr.go:89-183) for n signatures per call, one thread each (schnorr.cuh).
#include "host_call.cuh"
#include "msm_affine.cuh"
#include "schnorr.cuh"
using namespace b2k_host;

namespace b2k {

struct SchnorrInv { template <class F> B2K_D void operator()(F& r, const F& a) const { f_inv_bg(r, a); } };

template <class CV>
__global__ void __launch_bounds__(128) k_schnorr_verify(size_t n, const uint8_t* __restrict__ pks, const uint8_t* __restrict__ msgs,
                                                        const uint32_t* __restrict__ offs, const uint8_t* __restrict__ sigs,
                                                        uint8_t* __restrict__ status) {
  using F = typename CV::F;
  constexpr int PL = CV::OUT_BYTES;
  __shared__ Affine<F> btab[8];                         // 1..8 B: 768 bytes on G1, 1536 on G2, read by every thread of the block
  if (threadIdx.x == 0) schnorr_base_table<CV>(btab, SchnorrInv{});
  __syncthreads();
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t o0 = offs[i], o1 = offs[i + 1];
  status[i] = (uint8_t)schnorr_verify<CV>(pks + PL * i, msgs + o0, o1 >= o0 ? o1 - o0 : 0u, sigs + (PL + 32) * i, btab, SchnorrInv{});
}

template <class CV>
int schnorr_verify_dev(b2k_ctx* ctx, size_t n, const void* d_pks, const void* d_msgs, const void* d_offsets, const void* d_sigs,
                       void* d_status) {
  if (!ctx || !d_pks || !d_msgs || !d_offsets || !d_sigs || !d_status || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  k_schnorr_verify<CV><<<blocks_of(n, 128), 128, 0, ctx->stream>>>(n, (const uint8_t*)d_pks, (const uint8_t*)d_msgs,
                                                                  (const uint32_t*)d_offsets, (const uint8_t*)d_sigs,
                                                                  (uint8_t*)d_status);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return B2K_OK;
}

template <class CV>
int schnorr_verify_host(b2k_ctx* ctx, size_t n, const uint8_t* pks, const uint8_t* msgs, const uint32_t* offsets,
                        const uint8_t* sigs, uint8_t* status) {
  constexpr int PL = CV::OUT_BYTES;
  if (!ctx || !pks || !msgs || !offsets || !sigs || !status || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  if (check_offsets(ctx, n, offsets)) return B2K_ERR_ARG;
  uint8_t *d_pk = nullptr, *d_sig = nullptr, *d_msg = nullptr, *d_st = nullptr;
  uint32_t* d_off = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_pk = c.in(pks, n, PL);
    d_sig = c.in(sigs, n, PL + 32);
    d_msg = c.in(msgs, offsets[n]);
    d_off = c.in(offsets, n + 1);
    d_st = c.out(status, n);
  }, [&] { return schnorr_verify_dev<CV>(ctx, n, d_pk, d_msg, d_off, d_sig, d_st); });
}

}  // namespace b2k

extern "C" {

int b2k_bls12381_g1_schnorr_verify(b2k_ctx* c, size_t n, const uint8_t* pks, const uint8_t* msgs, const uint32_t* offsets,
                                   const uint8_t* sigs, uint8_t* status) {
  return schnorr_verify_host<Bls381G1>(c, n, pks, msgs, offsets, sigs, status);
}
int b2k_bls12381_g1_schnorr_verify_dev(b2k_ctx* c, size_t n, const void* pks, const void* msgs, const void* offsets, const void* sigs,
                                       void* status) {
  return schnorr_verify_dev<Bls381G1>(c, n, pks, msgs, offsets, sigs, status);
}
int b2k_bls12381_g2_schnorr_verify(b2k_ctx* c, size_t n, const uint8_t* pks, const uint8_t* msgs, const uint32_t* offsets,
                                   const uint8_t* sigs, uint8_t* status) {
  return schnorr_verify_host<Bls381G2>(c, n, pks, msgs, offsets, sigs, status);
}
int b2k_bls12381_g2_schnorr_verify_dev(b2k_ctx* c, size_t n, const void* pks, const void* msgs, const void* offsets, const void* sigs,
                                       void* status) {
  return schnorr_verify_dev<Bls381G2>(c, n, pks, msgs, offsets, sigs, status);
}
}  // extern "C"
