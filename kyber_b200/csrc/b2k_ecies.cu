// b2k_ecies.cu -- C ABI entry points for ECIES on edwards25519 (ecies.cuh), one thread per ciphertext:
//   b2k_ed25519_ecies_decrypt   ecies.Decrypt(edwards25519, priv, ctxt_i, sha256.New) for n ciphertexts under one key
//   b2k_ed25519_ecies_encrypt   ecies.Encrypt(edwards25519, pub_i, msg_i, sha256.New) with the caller's ephemeral r_i
// Both calls stage their inputs in the context's arena, and clear the staged bytes (keys, r, plaintexts, ciphertexts) before
// they return, so that no secret outlives the call in device memory the context keeps.
#include "host_call.cuh"
#include "ecies.cuh"
using namespace b2k_host;

namespace b2k {

constexpr int ECIES_BS = 128;

// one block recodes the key once into shared memory; each thread decrypts one ciphertext
__global__ void __launch_bounds__(ECIES_BS) k_ecies_decrypt(size_t n, uint32_t clen, const uint8_t* __restrict__ priv,
                                                            const uint8_t* __restrict__ ct, uint8_t* __restrict__ msg,
                                                            uint8_t* __restrict__ status) {
  __shared__ int8_t e[64];
  if (threadIdx.x == 0) {
    uint32_t k[8];
    sc_load_le(k, priv);
    sc_recode4(e, k);
  }
  __syncthreads();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  status[i] = (uint8_t)ecies_decrypt_one(e, ct + (size_t)(32 + clen) * i, clen, msg + (size_t)(clen - 16) * i);
}

// the comb of B is copied once per block into shared memory (24 KiB); each thread encrypts one message
__global__ void __launch_bounds__(ECIES_BS) k_ecies_encrypt(size_t n, uint32_t len, const uint8_t* __restrict__ pubs,
                                                            const uint8_t* __restrict__ rs, const uint8_t* __restrict__ msgs,
                                                            uint8_t* __restrict__ out, uint8_t* __restrict__ status) {
  __shared__ uint32_t btab[ECIES_TAB_WORDS];
  for (uint32_t w = threadIdx.x; w < ECIES_TAB_WORDS; w += blockDim.x) btab[w] = ecies_base_comb[w];
  __syncthreads();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  status[i] = (uint8_t)ecies_encrypt_one(pubs + 32 * i, rs + 32 * i, btab, msgs + (size_t)len * i, len,
                                         out + (size_t)(len + 48) * i);
}

}  // namespace b2k

extern "C" {

int b2k_ed25519_ecies_decrypt(b2k_ctx* ctx, const uint8_t* priv, size_t n, size_t len, const uint8_t* ctxt, uint8_t* msg,
                              uint8_t* status) {
  if (!ctx || !priv || !ctxt || !msg || !status || n == 0) return bad_arg(ctx, "bad argument");
  if (len < 16 || len > B2K_ECIES_MAX_LEN + 16) return bad_arg(ctx, "ciphertext length out of range");
  CK(cudaSetDevice(ctx->device));
  uint8_t *d_priv = nullptr, *d_ct = nullptr, *d_msg = nullptr, *d_st = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_priv = c.in(priv, 32);
    d_ct = c.in(ctxt, n, 32 + len);
    d_msg = c.out(msg, n, len - 16);
    d_st = c.out(status, n);
  }, [&]() -> int {
    b2k::k_ecies_decrypt<<<blocks_of(n, b2k::ECIES_BS), b2k::ECIES_BS, 0, ctx->stream>>>(n, (uint32_t)len, d_priv, d_ct, d_msg, d_st);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  }, true);
}

int b2k_ed25519_ecies_encrypt(b2k_ctx* ctx, size_t n, const uint8_t* pubs, const uint8_t* r, size_t len, const uint8_t* msg,
                              uint8_t* ctxt, uint8_t* status) {
  if (!ctx || !pubs || !r || !msg || !ctxt || !status || n == 0) return bad_arg(ctx, "bad argument");
  if (len > B2K_ECIES_MAX_LEN) return bad_arg(ctx, "message length out of range");
  CK(cudaSetDevice(ctx->device));
  uint8_t *d_pub = nullptr, *d_r = nullptr, *d_msg = nullptr, *d_ct = nullptr, *d_st = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_pub = c.in(pubs, n, 32);
    d_r = c.in(r, n, 32);
    d_msg = c.in(msg, n, len);
    d_ct = c.out(ctxt, n, len + 48);
    d_st = c.out(status, n);
  }, [&]() -> int {
    b2k::k_ecies_encrypt<<<blocks_of(n, b2k::ECIES_BS), b2k::ECIES_BS, 0, ctx->stream>>>(n, (uint32_t)len, d_pub, d_r, d_msg, d_ct,
                                                                                         d_st);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  }, true);
}

}  // extern "C"
