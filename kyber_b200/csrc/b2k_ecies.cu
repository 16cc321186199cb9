// b2k_ecies.cu -- C ABI entry points for ECIES on edwards25519 (ecies.cuh), one thread per ciphertext:
//   b2k_ed25519_ecies_decrypt   ecies.Decrypt(edwards25519, priv, ctxt_i, sha256.New) for n ciphertexts under one key
//   b2k_ed25519_ecies_encrypt   ecies.Encrypt(edwards25519, pub_i, msg_i, sha256.New) with the caller's ephemeral r_i
// Both calls stage their inputs in the context's input arena, and clear the staged bytes (keys, r, plaintexts, ciphertexts)
// before they return, so that no secret outlives the call in device memory the context keeps.
#include "msm_host.cuh"
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

namespace {

unsigned blocks_of(size_t n, unsigned bs) { return (unsigned)((n + bs - 1) / bs); }

int bad_arg(b2k_ctx* ctx, const char* why) {
  if (ctx) ctx->err = why;
  return B2K_ERR_ARG;
}

size_t up256(size_t v) { return (v + 255) & ~size_t(255); }

// n records of `per` bytes each fit in size_t with room for the padding between the staged arrays
bool sizes_fit(size_t n, size_t per) { return per == 0 || n <= (SIZE_MAX / 4) / per; }

// the staged bytes are cleared and the stream drained whatever happened before
int finish(b2k_ctx* ctx, uint8_t* blob, size_t total, int rc, const char* what) {
  cudaMemsetAsync(blob, 0, total, ctx->stream);
  if (cudaStreamSynchronize(ctx->stream) != cudaSuccess && rc == B2K_OK) rc = B2K_ERR_CUDA;
  if (rc == B2K_ERR_CUDA) ctx->err = what;
  return rc;
}

}  // namespace

extern "C" {

int b2k_ed25519_ecies_decrypt(b2k_ctx* ctx, const uint8_t* priv, size_t n, size_t len, const uint8_t* ctxt, uint8_t* msg,
                              uint8_t* status) {
  if (!ctx || !priv || !ctxt || !msg || !status || n == 0) return bad_arg(ctx, "bad argument");
  if (len < 16 || len > B2K_ECIES_MAX_LEN + 16) return bad_arg(ctx, "ciphertext length out of range");
  if (!sizes_fit(n, 32 + len + len)) return bad_arg(ctx, "batch too large");
  CK(cudaSetDevice(ctx->device));
  const size_t o_ct = 256, o_msg = up256(o_ct + n * (32 + len)), o_st = up256(o_msg + n * (len - 16)), total = o_st + n;
  uint8_t* blob = (uint8_t*)b2k_arena_in(ctx, total);
  if (!blob) { ctx->err = "out of device memory"; return B2K_ERR_CUDA; }
  cudaStream_t st = ctx->stream;
  int rc = B2K_OK;
  do {
    if (cudaMemcpyAsync(blob, priv, 32, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(blob + o_ct, ctxt, n * (32 + len), cudaMemcpyHostToDevice, st) != cudaSuccess) { rc = B2K_ERR_CUDA; break; }
    b2k::k_ecies_decrypt<<<blocks_of(n, b2k::ECIES_BS), b2k::ECIES_BS, 0, st>>>(n, (uint32_t)len, blob, blob + o_ct,
                                                                                  blob + o_msg, blob + o_st);
    if (cudaGetLastError() != cudaSuccess) { rc = B2K_ERR_CUDA; break; }
    ctx->launches += 1;
    if ((len > 16 && cudaMemcpyAsync(msg, blob + o_msg, n * (len - 16), cudaMemcpyDeviceToHost, st) != cudaSuccess) ||
        cudaMemcpyAsync(status, blob + o_st, n, cudaMemcpyDeviceToHost, st) != cudaSuccess) rc = B2K_ERR_CUDA;
  } while (0);
  return finish(ctx, blob, total, rc, "CUDA failure in ed25519_ecies_decrypt");
}

int b2k_ed25519_ecies_encrypt(b2k_ctx* ctx, size_t n, const uint8_t* pubs, const uint8_t* r, size_t len, const uint8_t* msg,
                              uint8_t* ctxt, uint8_t* status) {
  if (!ctx || !pubs || !r || !msg || !ctxt || !status || n == 0) return bad_arg(ctx, "bad argument");
  if (len > B2K_ECIES_MAX_LEN) return bad_arg(ctx, "message length out of range");
  if (!sizes_fit(n, 64 + len + len + 48)) return bad_arg(ctx, "batch too large");
  CK(cudaSetDevice(ctx->device));
  const size_t o_r = up256(32 * n), o_msg = up256(o_r + 32 * n), o_ct = up256(o_msg + n * len),
               o_st = up256(o_ct + n * (len + 48)), total = o_st + n;
  uint8_t* blob = (uint8_t*)b2k_arena_in(ctx, total);
  if (!blob) { ctx->err = "out of device memory"; return B2K_ERR_CUDA; }
  cudaStream_t st = ctx->stream;
  int rc = B2K_OK;
  do {
    if (cudaMemcpyAsync(blob, pubs, 32 * n, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(blob + o_r, r, 32 * n, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        (len && cudaMemcpyAsync(blob + o_msg, msg, n * len, cudaMemcpyHostToDevice, st) != cudaSuccess)) { rc = B2K_ERR_CUDA; break; }
    b2k::k_ecies_encrypt<<<blocks_of(n, b2k::ECIES_BS), b2k::ECIES_BS, 0, st>>>(n, (uint32_t)len, blob, blob + o_r,
                                                                                  blob + o_msg, blob + o_ct, blob + o_st);
    if (cudaGetLastError() != cudaSuccess) { rc = B2K_ERR_CUDA; break; }
    ctx->launches += 1;
    if (cudaMemcpyAsync(ctxt, blob + o_ct, n * (len + 48), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(status, blob + o_st, n, cudaMemcpyDeviceToHost, st) != cudaSuccess) rc = B2K_ERR_CUDA;
  } while (0);
  return finish(ctx, blob, total, rc, "CUDA failure in ed25519_ecies_encrypt");
}

}  // extern "C"
