// b2k_pvss.cu -- C ABI entry points for DLEQ proof verification and the PVSS share checks on edwards25519 (pvss.cuh):
//   b2k_ed25519_dleq_verify / _dev         dleq.Proof.Verify, proof/dleq/dleq.go:161-172, for n proofs
//   b2k_ed25519_pvss_verify_enc_shares     pvss.VerifyEncShareBatch, share/pvss/pvss.go:168-194, for m deals in one call
//   b2k_ed25519_pvss_verify_dec_shares     pvss.VerifyDecShareBatch, pvss.go:281-299
#include "host_call.cuh"
#include "pvss.cuh"
using namespace b2k_host;

namespace b2k {

__global__ void __launch_bounds__(128) k_ed_dleq_verify(size_t n, const uint8_t* __restrict__ g, const uint8_t* __restrict__ h,
                                                        const uint8_t* __restrict__ xg, const uint8_t* __restrict__ xh,
                                                        const uint8_t* __restrict__ proofs, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  status[i] = (uint8_t)dleq_verify_one(g + 32 * i, h + 32 * i, xg + 32 * i, xh + 32 * i, proofs + 128 * i);
}

// commitments of every deal into Niels form; one that does not decode marks its deal
__global__ void __launch_bounds__(256) k_pvss_load_commits(size_t mt, uint32_t t, const uint8_t* __restrict__ commits,
                                                           EdNiels* __restrict__ cm, uint32_t* __restrict__ bad) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= mt) return;
  EdNiels q;
  if (!ed_load_niels(q, commits + 32 * i)) bad[i / t] = 1;
  cm[i] = q;
}

// hashed[d][0..3][i] = coms[i], V[i], VG[i], VH[i] of deal d, canonical (the order computeGlobalChallenge hashes them in)
__global__ void __launch_bounds__(128) k_pvss_hashed_points(uint32_t m, uint32_t t, uint32_t n, const EdNiels* __restrict__ cm,
                                                            const uint8_t* __restrict__ v, const uint8_t* __restrict__ proofs,
                                                            uint8_t* __restrict__ hashed, uint32_t* __restrict__ bad) {
  size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (size_t)m * n) return;
  const uint32_t d = (uint32_t)(id / n), i = (uint32_t)(id % n);
  if (!pvss_hashed_points(hashed + (size_t)d * 128 * n + 32 * (size_t)i, 32 * (size_t)n, cm + (size_t)d * t, t, i, v + 32 * id,
                          proofs + 128 * id))
    bad[d] = 1;
}

// one thread per deal: H decodes, then the deal's challenge Pick(XOF(SHA-256 over its 4 n hashed points))
__global__ void __launch_bounds__(128) k_pvss_deal_challenge(uint32_t m, uint32_t n, const uint8_t* __restrict__ h,
                                                             const uint8_t* __restrict__ hashed, uint32_t* __restrict__ bad,
                                                             uint32_t* __restrict__ chal) {
  uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= m) return;
  EdExt H;
  if (!ed_decode(H, h + 32 * (size_t)d)) bad[d] = 1;
  if (bad[d]) return;
  uint8_t dig[32];
  sha256_blocks(dig, hashed + (size_t)d * 128 * n, 2 * (size_t)n);
  sc_pick(chal + 8 * (size_t)d, dig, 32);
}

__global__ void __launch_bounds__(128) k_pvss_enc_verify(uint32_t m, uint32_t n, const uint8_t* __restrict__ h,
                                                         const uint8_t* __restrict__ x, const uint8_t* __restrict__ sh,
                                                         const uint8_t* __restrict__ v, const uint8_t* __restrict__ proofs,
                                                         const uint32_t* __restrict__ bad, const uint32_t* __restrict__ chal,
                                                         uint8_t* __restrict__ status) {
  size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (size_t)m * n) return;
  const uint32_t d = (uint32_t)(id / n);
  status[id] = bad[d] ? (uint8_t)DLEQ_POINT
                      : (uint8_t)pvss_enc_share(h + 32 * (size_t)d, x + 32 * id, sh + 32 * id, v + 32 * id, proofs + 128 * id,
                                                chal + 8 * (size_t)d);
}

__global__ void __launch_bounds__(128) k_pvss_dec_verify(size_t n, const uint8_t* __restrict__ g, const uint8_t* __restrict__ x,
                                                         const uint8_t* __restrict__ enc_v, const uint8_t* __restrict__ dec_v,
                                                         const uint8_t* __restrict__ proofs, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  status[i] = (uint8_t)pvss_dec_share(g, x + 32 * i, enc_v + 32 * i, dec_v + 32 * i, proofs + 128 * i);
}

}  // namespace b2k

namespace {

int dleq_enqueue(b2k_ctx* ctx, size_t n, const uint8_t* g, const uint8_t* h, const uint8_t* xg, const uint8_t* xh,
                 const uint8_t* proofs, uint8_t* status) {
  k_ed_dleq_verify<<<blocks_of(n, 128), 128, 0, ctx->stream>>>(n, g, h, xg, xh, proofs, status);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return B2K_OK;
}

}  // namespace

extern "C" {

int b2k_ed25519_dleq_verify_dev(b2k_ctx* ctx, size_t n, const void* d_g, const void* d_h, const void* d_xg, const void* d_xh,
                                const void* d_proofs, void* d_status) {
  if (!ctx || !d_g || !d_h || !d_xg || !d_xh || !d_proofs || !d_status || n == 0) return bad_arg(ctx, "bad argument");
  CK(cudaSetDevice(ctx->device));
  return dleq_enqueue(ctx, n, (const uint8_t*)d_g, (const uint8_t*)d_h, (const uint8_t*)d_xg, (const uint8_t*)d_xh,
                      (const uint8_t*)d_proofs, (uint8_t*)d_status);
}

int b2k_ed25519_dleq_verify(b2k_ctx* ctx, size_t n, const uint8_t* g, const uint8_t* h, const uint8_t* xg, const uint8_t* xh,
                            const uint8_t* proofs, uint8_t* status) {
  if (!ctx || !g || !h || !xg || !xh || !proofs || !status || n == 0) return bad_arg(ctx, "bad argument");
  CK(cudaSetDevice(ctx->device));
  uint8_t *d_g = nullptr, *d_h = nullptr, *d_xg = nullptr, *d_xh = nullptr, *d_p = nullptr, *d_st = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_g = c.in(g, n, 32);
    d_h = c.in(h, n, 32);
    d_xg = c.in(xg, n, 32);
    d_xh = c.in(xh, n, 32);
    d_p = c.in(proofs, n, 128);
    d_st = c.out(status, n);
  }, [&] { return dleq_enqueue(ctx, n, d_g, d_h, d_xg, d_xh, d_p, d_st); });
}

int b2k_ed25519_pvss_verify_enc_shares(b2k_ctx* ctx, size_t m, size_t t, size_t n, const uint8_t* h, const uint8_t* commits,
                                       const uint8_t* x, const uint8_t* sh, const uint8_t* v, const uint8_t* proofs,
                                       uint8_t* status) {
  if (!ctx || !h || !commits || !x || !sh || !v || !proofs || !status || m == 0 || t == 0 || n == 0 ||
      m * t >= (size_t(1) << 31) || m * n >= (size_t(1) << 31))
    return bad_arg(ctx, "bad argument");
  CK(cudaSetDevice(ctx->device));
  const size_t mt = m * t, mn = m * n;
  uint8_t *d_h = nullptr, *d_c = nullptr, *d_x = nullptr, *d_sh = nullptr, *d_v = nullptr, *d_p = nullptr, *d_hashed = nullptr,
          *d_st = nullptr;
  EdNiels* d_cm = nullptr;
  uint32_t *d_bad = nullptr, *d_chal = nullptr;
  cudaStream_t st = ctx->stream;
  // stages, one kernel each (tools/perf_pvss.py times them by name): commitments, coms (Horner) and canonical points,
  // per-deal hash and Pick, per-share verify
  return host_call(ctx, [&](Carve& c) {
    d_h = c.in(h, m, 32);
    d_c = c.in(commits, mt, 32);
    d_x = c.in(x, mn, 32);
    d_sh = c.in(sh, mn, 32);
    d_v = c.in(v, mn, 32);
    d_p = c.in(proofs, mn, 128);
    d_cm = c.take<EdNiels>(mt);
    d_hashed = c.take<uint8_t>(mn, 128);
    d_bad = c.take<uint32_t>(m);
    d_chal = c.take<uint32_t>(m, 8);
    d_st = c.out(status, mn);
  }, [&]() -> int {
    CK(cudaMemsetAsync(d_bad, 0, m * 4, st));
    k_pvss_load_commits<<<blocks_of(mt, 256), 256, 0, st>>>(mt, (uint32_t)t, d_c, d_cm, d_bad);
    k_pvss_hashed_points<<<blocks_of(mn, 128), 128, 0, st>>>((uint32_t)m, (uint32_t)t, (uint32_t)n, d_cm, d_v, d_p, d_hashed, d_bad);
    k_pvss_deal_challenge<<<blocks_of(m, 128), 128, 0, st>>>((uint32_t)m, (uint32_t)n, d_h, d_hashed, d_bad, d_chal);
    k_pvss_enc_verify<<<blocks_of(mn, 128), 128, 0, st>>>((uint32_t)m, (uint32_t)n, d_h, d_x, d_sh, d_v, d_p, d_bad, d_chal, d_st);
    CK(cudaGetLastError());
    ctx->launches += 4;
    return B2K_OK;
  });
}

int b2k_ed25519_pvss_verify_dec_shares(b2k_ctx* ctx, size_t n, const uint8_t* g, const uint8_t* x, const uint8_t* enc_v,
                                       const uint8_t* dec_v, const uint8_t* proofs, uint8_t* status) {
  if (!ctx || !g || !x || !enc_v || !dec_v || !proofs || !status || n == 0) return bad_arg(ctx, "bad argument");
  CK(cudaSetDevice(ctx->device));
  uint8_t *d_g = nullptr, *d_x = nullptr, *d_e = nullptr, *d_d = nullptr, *d_p = nullptr, *d_st = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_g = c.in(g, 32);
    d_x = c.in(x, n, 32);
    d_e = c.in(enc_v, n, 32);
    d_d = c.in(dec_v, n, 32);
    d_p = c.in(proofs, n, 128);
    d_st = c.out(status, n);
  }, [&]() -> int {
    k_pvss_dec_verify<<<blocks_of(n, 128), 128, 0, ctx->stream>>>(n, d_g, d_x, d_e, d_d, d_p, d_st);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  });
}

}  // extern "C"
