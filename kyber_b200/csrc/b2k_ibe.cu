// b2k_ibe.cu -- Boneh-Franklin IBE (CCA) on BLS12-381: n ciphertexts under one private key, or n messages to one identity, per call.
//
// Replaces n x DecryptCCAonG1 / DecryptCCAonG2 / EncryptCCAonG1 / EncryptCCAonG2 (encrypt/ibe/ibe.go:51-231).  The case this serves:
// when a round's key is published, every ciphertext locked to that round (drand timelock) decrypts with the same G2 point.
//
// Decrypt: decode U (per-element flag) -> pairing with the key -> one thread per ciphertext for H2, the xors, H4, H3, r Base == U.
//   The pairing: the existing launcher (one warp per pairing up to coop_max_n), except for U on G1 above that size, where every
//   pairing shares its G2 argument and the Miller loop runs against a table of that point's lines (k_ibe_pair_fixed_q).
// Encrypt: Q_id = hash of the identity and Gid = e(master, Q_id) once; one thread per message for r, U and W; Gid^r through the
//   GT exponentiation of b2k_bls12381_gt_exp; V = sigma xor H2(Gid^r).
#include "msm_host.cuh"
#include "pairing_kernels.cuh"
#include "ibe.cuh"
using namespace b2k_host;

extern "C" void b2k_internal_launch_bls12381_gt_exp(const b2k_ctx* c, size_t n, const uint8_t* ds, const uint8_t* da, uint8_t* dout);

namespace b2k {

template <class CV> struct IbeCodec;
template <> struct IbeCodec<Bls381G1> {
  B2K_D static bool decompress(Affine<BFp>& a, const uint8_t* in) { return g1_decompress(a, in, true); }
};
template <> struct IbeCodec<Bls381G2> {
  B2K_D static bool decompress(Affine<BFp2>& a, const uint8_t* in) { return g2_decompress(a, in, true); }
};

// compressed wire -> operand bytes (infinity, and what does not decode, as all-zero operands) and a per-element flag
template <class CV>
__global__ void __launch_bounds__(64) k_ibe_decode(size_t n, const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                                                   uint8_t* __restrict__ ok) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<typename CV::F> a;
  const bool good = IbeCodec<CV>::decompress(a, in + (size_t)CV::OUT_BYTES * i);
  if (!good) aff_set_inf(a);
  CV::store_affine(out + (size_t)CV::IN_BYTES * i, a);
  ok[i] = good ? 1 : 0;
}

// the key (or master) point: decoded once, FLAG_POINT when it does not decode, written `copies` times in operand form
template <class CV>
__global__ void k_ibe_key(const uint8_t* __restrict__ in, size_t copies, uint8_t* __restrict__ out, uint32_t* flags) {
  __shared__ uint8_t op[CV::IN_BYTES];
  if (threadIdx.x == 0) {
    Affine<typename CV::F> a;
    if (!IbeCodec<CV>::decompress(a, in)) { aff_set_inf(a); if (blockIdx.x == 0) atomicOr(flags, FLAG_POINT); }
    CV::store_affine(op, a);
  }
  __syncthreads();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < copies * CV::IN_BYTES; i += (size_t)gridDim.x * blockDim.x)
    out[i] = op[i % CV::IN_BYTES];
}

// the line table of one G2 point (operand form); live = 0 for the point at infinity (every pairing is then 1)
__global__ void k_ibe_line_table(const uint8_t* __restrict__ q, BlsLineCoef* __restrict__ tab, uint32_t* __restrict__ live, uint32_t* flags) {
  if (threadIdx.x || blockIdx.x) return;
  Affine<BFp2> Q;
  if (!load_checked<Bls381G2>(Q, q)) atomicOr(flags, FLAG_POINT);   // a malformed operand counts as infinity, as in k_bls_pair
  *live = aff_is_inf(Q) ? 0u : 1u;
  miller_fixed_q_table(tab, Q);
}

// gt[i] = e(g1[i], Q) for the Q of the table: the table in shared memory, per step f^2 and one sparse product
__global__ void __launch_bounds__(64, 4) k_ibe_pair_fixed_q(size_t n, const uint8_t* __restrict__ g1, const BlsLineCoef* __restrict__ tab,
                                                             const uint32_t* __restrict__ live, uint8_t* __restrict__ gt, uint32_t* flags) {
  __shared__ BlsLineCoef sm[BLS_MILLER_STEPS];
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(tab);
    uint32_t* dst = reinterpret_cast<uint32_t*>(sm);
    for (uint32_t k = threadIdx.x; k < sizeof(sm) / 4; k += blockDim.x) dst[k] = src[k];
  }
  __syncthreads();
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<BFp> P;
  if (!load_checked<Bls381G1>(P, g1 + 96 * i)) atomicOr(flags, FLAG_POINT);
  BFp12 f, e;
  if (*live) miller_fixed_q(f, P, sm);
  else fp12_set_one(f);
  final_exponentiation(e, f);
  gt_store(gt + 576 * i, e);
}

template <class CV>
__global__ void __launch_bounds__(64) k_ibe_decrypt_finish(size_t n, uint32_t len, const uint8_t* __restrict__ gt, const uint8_t* __restrict__ u,
                                                           const uint8_t* __restrict__ u_ok, const uint8_t* __restrict__ v,
                                                           const uint8_t* __restrict__ w, uint8_t* __restrict__ msg, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<typename CV::F> U;
  CV::load(U, u + (size_t)CV::IN_BYTES * i);
  status[i] = ibe_decrypt_finish<CV>(msg + (size_t)len * i, gt + 576 * i, U, u_ok[i] != 0, v + (size_t)len * i, w + (size_t)len * i, len,
                                     InvBingcd{});
}

// r, U, W per message, and Gid copied next to each exponent (the GT exponentiation takes one base per element)
template <class CV>
__global__ void __launch_bounds__(64) k_ibe_encrypt(size_t n, uint32_t len, const uint8_t* __restrict__ msgs, const uint8_t* __restrict__ sigmas,
                                                    const uint8_t* __restrict__ gid, uint8_t* __restrict__ u, uint8_t* __restrict__ r,
                                                    uint8_t* __restrict__ w, uint8_t* __restrict__ gidn, uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (!ibe_encrypt_body<CV>(u + (size_t)CV::OUT_BYTES * i, r + 32 * i, w + (size_t)len * i, msgs + (size_t)len * i, sigmas + (size_t)len * i,
                            len, InvBingcd{}))
    atomicOr(flags, FLAG_IBE_H3);
  for (int k = 0; k < 576; k++) gidn[576 * i + k] = gid[k];
}

__global__ void __launch_bounds__(128) k_ibe_encrypt_v(size_t n, uint32_t len, const uint8_t* __restrict__ gtr, const uint8_t* __restrict__ sigmas,
                                                       uint8_t* __restrict__ v) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t h[32];
  ibe_h2(h, gtr + 576 * i);
  for (uint32_t k = 0; k < len; k++) v[(size_t)len * i + k] = sigmas[(size_t)len * i + k] ^ h[k];
}

}  // namespace b2k

using namespace b2k;

namespace {

constexpr uint8_t DST_G1[] = "BLS_SIG_BLS12381G1_XMD:SHA-256_SSWU_RO_NUL_";
constexpr uint8_t DST_G2[] = "BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_NUL_";

// gt[i] = e(g1[i], q) for one G2 point q (operand form) through the line table
void fixed_q_layout(Carve& c, BlsLineCoef*& tab, uint32_t*& live) {
  tab = c.take<BlsLineCoef>(BLS_MILLER_STEPS);
  live = c.take<uint32_t>(1);
}
int pair_fixed_q(b2k_ctx* ctx, size_t n, const uint8_t* d_g1, const uint8_t* d_q, BlsLineCoef* tab, uint32_t* live, uint8_t* d_gt) {
  k_ibe_line_table<<<1, 32, 0, ctx->stream>>>(d_q, tab, live, ctx->d_flags);
  k_ibe_pair_fixed_q<<<blocks_of(n, 64), 64, 0, ctx->stream>>>(n, d_g1, tab, live, d_gt, ctx->d_flags);
  CK(cudaGetLastError());
  ctx->launches += 2;
  return B2K_OK;
}

// DecryptCCAonG1 (KEY = G2, U on G1) / DecryptCCAonG2 (KEY = G1, U on G2)
template <class UG, class KG>
int ibe_decrypt(b2k_ctx* ctx, const uint8_t* priv, size_t n, const uint8_t* u, size_t len, const uint8_t* v, const uint8_t* w, uint8_t* msg,
                uint8_t* status) {
  if (!ctx) return B2K_ERR_ARG;
  if (!priv || !u || !status || n == 0 || n >= (size_t(1) << 31) || len > IBE_MAX_LEN || (len && (!v || !w || !msg)))
    return bad_arg(ctx, "bad argument (n >= 1, len <= 32)");
  CK(cudaSetDevice(ctx->device));
  constexpr bool u_on_g1 = UG::OUT_BYTES == 48;
  const bool fixed_q = u_on_g1 && !(ctx->coop_max_n > 0 && n <= (size_t)ctx->coop_max_n);
  const size_t copies = fixed_q ? 1 : n;
  uint8_t *d_key = nullptr, *d_uw = nullptr, *d_v = nullptr, *d_w = nullptr, *d_u = nullptr, *d_ok = nullptr, *d_keys = nullptr,
          *d_gt = nullptr, *d_m = nullptr, *d_st = nullptr;
  BlsLineCoef* tab = nullptr;
  uint32_t* live = nullptr;
  const int rc = host_call(ctx, [&](Carve& c) {
    d_key = c.in(priv, KG::OUT_BYTES);
    d_uw = c.in(u, n, UG::OUT_BYTES);
    d_v = c.in(v, n, len);
    d_w = c.in(w, n, len);
    d_u = c.take<uint8_t>(n, UG::IN_BYTES);
    d_ok = c.take<uint8_t>(n);
    d_keys = c.take<uint8_t>(copies, KG::IN_BYTES);
    d_gt = c.take<uint8_t>(n, 576);
    fixed_q_layout(c, tab, live);
    d_m = c.out(msg, n, len);
    d_st = c.out(status, n);
  }, [&]() -> int {
    cudaStream_t st = ctx->stream;
    const unsigned kb = blocks_of(copies * KG::IN_BYTES, 256);
    k_ibe_key<KG><<<kb < 1024 ? kb : 1024, 256, 0, st>>>(d_key, copies, d_keys, ctx->d_flags);
    k_ibe_decode<UG><<<blocks_of(n, 64), 64, 0, st>>>(n, d_uw, d_u, d_ok);
    CK(cudaGetLastError());
    ctx->launches += 2;
    if (fixed_q) {
      if (int rc = pair_fixed_q(ctx, n, d_u, d_keys, tab, live, d_gt)) return rc;
    } else {
      if (u_on_g1) b2k_internal_launch_pair(ctx, n, d_u, d_keys, d_gt);     // e(U, private)
      else b2k_internal_launch_pair(ctx, n, d_keys, d_u, d_gt);             // e(private, U)
      CK(cudaGetLastError());
      ctx->launches += (ctx->pair_variant >= 16 && !(ctx->coop_max_n > 0 && n <= (size_t)ctx->coop_max_n)) ? 2 : 1;
    }
    k_ibe_decrypt_finish<UG><<<blocks_of(n, 64), 64, 0, st>>>(n, (uint32_t)len, d_gt, d_u, d_ok, d_v, d_w, d_m, d_st);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  });
  if (rc == B2K_ERR_POINT) ctx->err = "the private key does not decode";
  return rc;
}

// EncryptCCAonG1 (MG = G1 master, Q_id on G2, U on G1) / EncryptCCAonG2 (MG = G2 master, Q_id on G1, U on G2)
template <class MG, class QG>
int ibe_encrypt(b2k_ctx* ctx, const uint8_t* master, const uint8_t* id, size_t id_len, const uint8_t* dst, size_t dst_len, size_t n,
                size_t len, const uint8_t* msgs, const uint8_t* sigmas, uint8_t* u, uint8_t* v, uint8_t* w) {
  if (!ctx) return B2K_ERR_ARG;
  if (!dst) { dst = MG::OUT_BYTES == 48 ? DST_G2 : DST_G1; dst_len = sizeof(DST_G1) - 1; }
  if (!master || (!id && id_len) || id_len >= (size_t(1) << 31) || dst_len == 0 || dst_len > 255 || !u || n == 0 || n >= (size_t(1) << 31) ||
      len > IBE_MAX_LEN || (len && (!msgs || !sigmas || !v || !w)))
    return bad_arg(ctx, "bad argument (n >= 1, len <= 32, 1 <= dst_len <= 255)");
  CK(cudaSetDevice(ctx->device));
  using UG = MG;
  const uint32_t off[2] = {0, (uint32_t)id_len};
  uint8_t *d_mw = nullptr, *d_id = nullptr, *d_dst = nullptr, *d_msg = nullptr, *d_sig = nullptr, *d_master = nullptr, *d_q = nullptr,
          *d_gid = nullptr, *d_r = nullptr, *d_gidn = nullptr, *d_gtr = nullptr, *d_u = nullptr, *d_v = nullptr, *d_w = nullptr;
  uint32_t* d_off = nullptr;
  const int rc = host_call(ctx, [&](Carve& c) {
    d_mw = c.in(master, MG::OUT_BYTES);
    d_id = c.in(id, id_len);
    d_off = c.in(off, 2);
    d_dst = c.in(dst, dst_len);
    d_msg = c.in(msgs, n, len);
    d_sig = c.in(sigmas, n, len);
    d_master = c.take<uint8_t>(MG::IN_BYTES);
    d_q = c.take<uint8_t>(QG::IN_BYTES);
    d_gid = c.take<uint8_t>(576);
    d_r = c.take<uint8_t>(n, 32);
    d_gidn = c.take<uint8_t>(n, 576);
    d_gtr = c.take<uint8_t>(n, 576);
    d_u = c.out(u, n, UG::OUT_BYTES);
    d_v = c.out(v, n, len);
    d_w = c.out(w, n, len);
  }, [&]() -> int {
    cudaStream_t st = ctx->stream;
    k_ibe_key<MG><<<1, 64, 0, st>>>(d_mw, 1, d_master, ctx->d_flags);
    CK(cudaGetLastError());
    ctx->launches += 1;
    int rc = QG::OUT_BYTES == 96 ? b2k_bls12381_hash_to_g2_dev(ctx, 1, d_id, d_off, d_dst, (uint32_t)dst_len, d_q)
                                 : b2k_bls12381_hash_to_g1_dev(ctx, 1, d_id, d_off, d_dst, (uint32_t)dst_len, d_q);
    if (rc) return rc;
    if (MG::OUT_BYTES == 48) b2k_internal_launch_pair(ctx, 1, d_master, d_q, d_gid);     // Gid = e(master, Q_id)
    else b2k_internal_launch_pair(ctx, 1, d_q, d_master, d_gid);                         // Gid = e(Q_id, master)
    k_ibe_encrypt<UG><<<blocks_of(n, 64), 64, 0, st>>>(n, (uint32_t)len, d_msg, d_sig, d_gid, d_u, d_r, d_w, d_gidn, ctx->d_flags);
    CK(cudaGetLastError());
    b2k_internal_launch_bls12381_gt_exp(ctx, n, d_r, d_gidn, d_gtr);
    k_ibe_encrypt_v<<<blocks_of(n, 128), 128, 0, st>>>(n, (uint32_t)len, d_gtr, d_sig, d_v);
    CK(cudaGetLastError());
    ctx->launches += 4;
    return B2K_OK;
  });
  if (rc == B2K_ERR_POINT) ctx->err = "the master key does not decode";
  return rc;
}

}  // namespace

extern "C" {

int b2k_bls12381_ibe_decrypt_cca_g1(b2k_ctx* ctx, const uint8_t* priv, size_t n, const uint8_t* u, size_t len, const uint8_t* v,
                                    const uint8_t* w, uint8_t* msg, uint8_t* status) {
  return ibe_decrypt<Bls381G1, Bls381G2>(ctx, priv, n, u, len, v, w, msg, status);
}
int b2k_bls12381_ibe_decrypt_cca_g2(b2k_ctx* ctx, const uint8_t* priv, size_t n, const uint8_t* u, size_t len, const uint8_t* v,
                                    const uint8_t* w, uint8_t* msg, uint8_t* status) {
  return ibe_decrypt<Bls381G2, Bls381G1>(ctx, priv, n, u, len, v, w, msg, status);
}
int b2k_bls12381_ibe_encrypt_cca_g1(b2k_ctx* ctx, const uint8_t* master, const uint8_t* id, size_t id_len, const uint8_t* dst, size_t dst_len,
                                    size_t n, size_t len, const uint8_t* msgs, const uint8_t* sigmas, uint8_t* u, uint8_t* v, uint8_t* w) {
  return ibe_encrypt<Bls381G1, Bls381G2>(ctx, master, id, id_len, dst, dst_len, n, len, msgs, sigmas, u, v, w);
}
int b2k_bls12381_ibe_encrypt_cca_g2(b2k_ctx* ctx, const uint8_t* master, const uint8_t* id, size_t id_len, const uint8_t* dst, size_t dst_len,
                                    size_t n, size_t len, const uint8_t* msgs, const uint8_t* sigmas, uint8_t* u, uint8_t* v, uint8_t* w) {
  return ibe_encrypt<Bls381G2, Bls381G1>(ctx, master, id, id_len, dst, dst_len, n, len, msgs, sigmas, u, v, w);
}

int b2k_bls12381_pair_fixed_g2(b2k_ctx* ctx, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* gt) {
  if (!ctx || !g1 || !g2 || !gt || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  uint8_t *d1 = nullptr, *d2 = nullptr, *dg = nullptr;
  BlsLineCoef* tab = nullptr;
  uint32_t* live = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d1 = c.in(g1, n, 96);
    d2 = c.in(g2, 192);
    dg = c.out(gt, n, 576);
    fixed_q_layout(c, tab, live);
  }, [&] { return pair_fixed_q(ctx, n, d1, d2, tab, live, dg); });
}

}  // extern "C"
