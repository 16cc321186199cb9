// b2k_ecies_bls.cu -- C ABI entry points for ECIES on BLS12-381 with keys on G1 or on G2 (ecies_bls.cuh), one thread per
// ciphertext:
//   b2k_bls12381_g{1,2}_ecies_decrypt   ecies.Decrypt(G1 or G2, priv, ctxt_i, sha256.New) for n ciphertexts under one key
//   b2k_bls12381_g{1,2}_ecies_encrypt   ecies.Encrypt(G1 or G2, pub_i, msg_i, sha256.New) with the caller's ephemeral r_i
// Both calls check every scalar against r on the host without an early exit, stage their inputs in the context's arena, and
// clear the staged bytes (keys, r, plaintexts, ciphertexts) before they return, so that no secret outlives the call in device
// memory the context keeps.
#include "host_call.cuh"
#include "ecies_bls.cuh"
using namespace b2k_host;

namespace b2k {

constexpr int ECIES_BLS_BS = 128;

// one block recodes the key once into shared memory, where every thread reads the same digit at the same step; each thread
// decrypts one ciphertext
template <class CV>
__global__ void __launch_bounds__(ECIES_BLS_BS) k_ecies_bls_decrypt(size_t n, uint32_t clen, const uint8_t* __restrict__ priv,
                                                                    const uint8_t* __restrict__ ct, uint8_t* __restrict__ msg,
                                                                    uint8_t* __restrict__ status) {
  constexpr int PL = CV::OUT_BYTES;
  __shared__ int8_t e[ECIES_BLS_DIGITS];
  if (threadIdx.x == 0) ct_recode(e, priv);
  __syncthreads();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  status[i] = (uint8_t)ecies_bls_decrypt_one<CV>(e, ct + (size_t)(PL + clen) * i, clen, msg + (size_t)(clen - 16) * i);
}

// 1..8 G is built once per block into shared memory (1152 bytes on G1, 2304 on G2); each thread encrypts one message
template <class CV>
__global__ void __launch_bounds__(ECIES_BLS_BS) k_ecies_bls_encrypt(size_t n, uint32_t len, const uint8_t* __restrict__ pubs,
                                                                    const uint8_t* __restrict__ rs, const uint8_t* __restrict__ msgs,
                                                                    uint8_t* __restrict__ out, uint8_t* __restrict__ status) {
  constexpr int PL = CV::OUT_BYTES;
  __shared__ Proj<typename CV::F> btab[8];
  if (threadIdx.x == 0) ecies_bls_base_table<CV>(btab);
  __syncthreads();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  status[i] = (uint8_t)ecies_bls_encrypt_one<CV>(pubs + (size_t)PL * i, rs + 32 * i, btab, msgs + (size_t)len * i, len,
                                                 out + (size_t)(PL + len + 16) * i);
}

}  // namespace b2k

namespace {

// r, 32 bytes big-endian (kilic/scalar.go:11-12)
constexpr uint8_t BLS_R_BE[32] = {0x73, 0xed, 0xa7, 0x53, 0x29, 0x9d, 0x7d, 0x48, 0x33, 0x39, 0xd8, 0x08, 0x09, 0xa1, 0xd8, 0x05,
                                  0x53, 0xbd, 0xa4, 0x02, 0xff, 0xfe, 0x5b, 0xfe, 0xff, 0xff, 0xff, 0xff, 0x00, 0x00, 0x00, 0x01};

// 1 unless every one of the n 32-byte big-endian scalars is below r: s - r over all 32 bytes, its final borrow is s < r; the
// outcomes are ANDed over every scalar, so the time depends on n only, never on a scalar's bytes
uint32_t any_scalar_out_of_range(const uint8_t* s, size_t n) {
  uint32_t all_below = 1;
  for (size_t i = 0; i < n; i++) {
    uint32_t borrow = 0;
    for (int j = 31; j >= 0; j--) borrow = ((uint32_t)s[32 * i + j] - BLS_R_BE[j] - borrow) >> 31;
    all_below &= borrow;
  }
  return all_below ^ 1u;
}

template <class CV>
int ecies_bls_decrypt(b2k_ctx* ctx, const uint8_t* priv, size_t n, size_t len, const uint8_t* ctxt, uint8_t* msg, uint8_t* status) {
  constexpr size_t PL = CV::OUT_BYTES;
  if (!ctx || !priv || !ctxt || !msg || !status || n == 0) return bad_arg(ctx, "bad argument");
  if (len < 16 || len > B2K_ECIES_MAX_LEN + 16) return bad_arg(ctx, "ciphertext length out of range");
  if (any_scalar_out_of_range(priv, 1)) {
    ctx->err = "private key not below r";
    return B2K_ERR_SCALAR_RANGE;
  }
  CK(cudaSetDevice(ctx->device));
  uint8_t *d_priv = nullptr, *d_ct = nullptr, *d_msg = nullptr, *d_st = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_priv = c.in(priv, 32);
    d_ct = c.in(ctxt, n, PL + len);
    d_msg = c.out(msg, n, len - 16);
    d_st = c.out(status, n);
  }, [&]() -> int {
    b2k::k_ecies_bls_decrypt<CV><<<blocks_of(n, b2k::ECIES_BLS_BS), b2k::ECIES_BLS_BS, 0, ctx->stream>>>(n, (uint32_t)len, d_priv,
                                                                                                         d_ct, d_msg, d_st);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  }, true);
}

template <class CV>
int ecies_bls_encrypt(b2k_ctx* ctx, size_t n, const uint8_t* pubs, const uint8_t* r, size_t len, const uint8_t* msg,
                      uint8_t* ctxt, uint8_t* status) {
  constexpr size_t PL = CV::OUT_BYTES;
  if (!ctx || !pubs || !r || !msg || !ctxt || !status || n == 0) return bad_arg(ctx, "bad argument");
  if (len > B2K_ECIES_MAX_LEN) return bad_arg(ctx, "message length out of range");
  size_t bytes;
  if (__builtin_mul_overflow(n, PL + len + 16, &bytes)) return bad_arg(ctx, "batch too large");   // before r is read
  if (any_scalar_out_of_range(r, n)) {
    ctx->err = "ephemeral scalar not below r";
    return B2K_ERR_SCALAR_RANGE;
  }
  CK(cudaSetDevice(ctx->device));
  uint8_t *d_pub = nullptr, *d_r = nullptr, *d_msg = nullptr, *d_ct = nullptr, *d_st = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_pub = c.in(pubs, n, PL);
    d_r = c.in(r, n, 32);
    d_msg = c.in(msg, n, len);
    d_ct = c.out(ctxt, n, PL + len + 16);
    d_st = c.out(status, n);
  }, [&]() -> int {
    b2k::k_ecies_bls_encrypt<CV><<<blocks_of(n, b2k::ECIES_BLS_BS), b2k::ECIES_BLS_BS, 0, ctx->stream>>>(n, (uint32_t)len, d_pub,
                                                                                                         d_r, d_msg, d_ct, d_st);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  }, true);
}

}  // namespace

extern "C" {

int b2k_bls12381_g1_ecies_decrypt(b2k_ctx* ctx, const uint8_t* priv, size_t n, size_t len, const uint8_t* ctxt, uint8_t* msg,
                                  uint8_t* status) {
  return ecies_bls_decrypt<Bls381G1>(ctx, priv, n, len, ctxt, msg, status);
}
int b2k_bls12381_g2_ecies_decrypt(b2k_ctx* ctx, const uint8_t* priv, size_t n, size_t len, const uint8_t* ctxt, uint8_t* msg,
                                  uint8_t* status) {
  return ecies_bls_decrypt<Bls381G2>(ctx, priv, n, len, ctxt, msg, status);
}
int b2k_bls12381_g1_ecies_encrypt(b2k_ctx* ctx, size_t n, const uint8_t* pubs, const uint8_t* r, size_t len, const uint8_t* msg,
                                  uint8_t* ctxt, uint8_t* status) {
  return ecies_bls_encrypt<Bls381G1>(ctx, n, pubs, r, len, msg, ctxt, status);
}
int b2k_bls12381_g2_ecies_encrypt(b2k_ctx* ctx, size_t n, const uint8_t* pubs, const uint8_t* r, size_t len, const uint8_t* msg,
                                  uint8_t* ctxt, uint8_t* status) {
  return ecies_bls_encrypt<Bls381G2>(ctx, n, pubs, r, len, msg, ctxt, status);
}

}  // extern "C"
