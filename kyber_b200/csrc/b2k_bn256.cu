// b2k_bn256.cu -- C ABI entry points for bn256: G1/G2 Point.Mul batches, MSM, pairings and the BDN batch verification.
#include "msm_host.cuh"
#include "bn256.cuh"
#include "bn_pairing.cuh"
#define B2K_COOP_BN256 1
#include "coop_pairing.cuh"          // small batches: one warp per pairing
#include "bdn.cuh"
using namespace b2k_host;

namespace b2k {
using PC6 = Bn256Pair;
using Coop256 = coop::Curve<Bn256G1, Bn256G2, Bn256Fp, PFp12<Bn256Pair>, coop::BN256_P1, coop::BN256_P2>;

// pairing/bn256/suite.go:99-105 Pair -> optimalAte (optate.go:266-274): identity when an operand is infinity
__global__ void __launch_bounds__(64, 4) k_bn256_pair(size_t n, const uint8_t* __restrict__ g1, const uint8_t* __restrict__ g2,
                                                      uint8_t* __restrict__ gt, uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<PFp<PC6>> P;
  Affine<PFp2<PC6>> Q;
  bool good = load_checked<Bn256G1>(P, g1 + 64 * i);
  good = load_checked<Bn256G2>(Q, g2 + 128 * i) && good;
  if (!good) atomicOr(flags, FLAG_POINT);
  PFp12<PC6> f, e;
  bn_miller_loop<PC6, 1>(f, &P, &Q);
  bn_final_exponentiation<PC6>(e, f);
  if (aff_is_inf(P) || aff_is_inf(Q)) fp12_set_one(e);
  bn_gt_store<PC6>(gt + 384 * i, e);
}

// ok[i] = e(a1,a2) == e(b1,b2)   (bn256 ValidatePairing = two pairings + Equal, suite.go:107-109)
__global__ void __launch_bounds__(64, 4) k_bn256_pairing_check(size_t n, const uint8_t* __restrict__ a1,
                                                               const uint8_t* __restrict__ a2, const uint8_t* __restrict__ b1,
                                                               const uint8_t* __restrict__ b2, uint8_t* __restrict__ ok, uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<PFp<PC6>> P[2];
  Affine<PFp2<PC6>> Q[2];
  bool good = load_checked<Bn256G1>(P[0], a1 + 64 * i);
  good = load_checked<Bn256G2>(Q[0], a2 + 128 * i) && good;
  good = load_checked<Bn256G1>(P[1], b1 + 64 * i) && good;
  good = load_checked<Bn256G2>(Q[1], b2 + 128 * i) && good;
  if (!good) { atomicOr(flags, FLAG_POINT); ok[i] = 0; return; }
  fp_neg(P[1].y, P[1].y);
  PFp12<PC6> f, e;
  bn_miller_loop<PC6, 2>(f, P, Q);
  bn_final_exponentiation<PC6>(e, f);
  ok[i] = fp12_is_one(e) ? 1 : 0;
}

// bls.Verify's UnmarshalBinary of a bn256 signature (pairing/bn256/point.go:206-238: reduced coordinates, on the curve):
// out[i] = the decoded point (infinity when it does not decode), ok[i] = 1 when it decodes
__global__ void __launch_bounds__(128) k_bn256_g1_decode(size_t n, const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                                                         uint8_t* __restrict__ ok) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<PFp<PC6>> p;
  ok[i] = load_checked<Bn256G1>(p, in + 64 * i) ? 1 : 0;
  Bn256G1::store(out + 64 * i, p);
}

// slots 1 .. n-1 of buf[n][128] = slot 0: the pairing check's per-element G2 base, filled on the device from one copy
__global__ void k_bn256_repeat128(size_t n, uint8_t* buf) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;      // one 32-bit word per thread
  uint32_t* w = reinterpret_cast<uint32_t*>(buf);
  if (t >= 32 && t < 32 * n) w[t] = w[t % 32];
}
}  // namespace b2k

namespace {
// ok[i] = e(a1,a2) == e(b1,b2), every buffer on the device: the enqueue of b2k_bn256_pairing_check and of the BDN batch
int bn256_pairing_check_enqueue(b2k_ctx* ctx, size_t n, const uint8_t* da1, const uint8_t* da2, const uint8_t* db1, const uint8_t* db2,
                                uint8_t* dok) {
  cudaStream_t st = ctx->stream;
  if (ctx->coop_max_n > 0 && n <= (size_t)(ctx->coop_max_n < 8192 ? ctx->coop_max_n : 8192))   // break-even measured near 8 192 on this curve
    coop::k_coop_bn_pairing_check<Coop256><<<(unsigned)n, 32, Coop256::L::BYTES, st>>>(n, da1, da2, db1, db2, dok, ctx->d_flags);
  else
    k_bn256_pairing_check<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(n, da1, da2, db1, db2, dok, ctx->d_flags);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return B2K_OK;
}

// the G2 base point of bn256 (pairing/bn256/twist.go twistGen) in the 128-byte wire form
constexpr uint8_t BN256_G2_BASE[128] = {
    0x2e, 0xcc, 0xa4, 0x46, 0xff, 0x6f, 0x3d, 0x4d, 0x03, 0xc7, 0x6e, 0x9b, 0x5c, 0x75, 0x2f, 0x28, 0xbc, 0x37, 0xb3, 0x64, 0xcb, 0x05,
    0xac, 0x4a, 0x37, 0xeb, 0x32, 0xe1, 0xc3, 0x24, 0x59, 0x70, 0x8f, 0x25, 0x38, 0x6f, 0x72, 0xc9, 0x46, 0x2b, 0x81, 0x59, 0x7d, 0x65,
    0xae, 0x20, 0x92, 0xc4, 0xb9, 0x77, 0x92, 0x15, 0x5d, 0xcd, 0xaa, 0xd3, 0x2b, 0x8a, 0x6d, 0xd4, 0x17, 0x92, 0x53, 0x4c, 0x2d, 0xb1,
    0x0e, 0xf5, 0x23, 0x3b, 0x0f, 0xe3, 0x96, 0x2b, 0x9e, 0xe6, 0xa4, 0xbb, 0xc2, 0xb5, 0xbd, 0xe0, 0x1a, 0x54, 0xf3, 0x51, 0x3d, 0x42,
    0xdf, 0x97, 0x2e, 0x12, 0x8f, 0x31, 0xbf, 0x12, 0x27, 0x4e, 0x57, 0x47, 0xe8, 0xca, 0xfa, 0xcc, 0x37, 0x16, 0xcc, 0x86, 0x99, 0xdb,
    0x79, 0xb2, 0x2f, 0x0e, 0x4f, 0xf3, 0xc2, 0x3e, 0x89, 0x8f, 0x69, 0x44, 0x20, 0xa3, 0xbe, 0x30, 0x87, 0xa5};
}  // namespace

extern "C" {
int b2k_bn256_g1_mul_batch(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return mul_batch_host<Bn256G1, false>(c, n, s, p, o); }
int b2k_bn256_g1_msm(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return msm_host<Bn256G1>(c, n, s, p, o); }
int b2k_bn256_g2_mul_batch(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return mul_batch_host<Bn256G2, false>(c, n, s, p, o); }
int b2k_bn256_g2_msm(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return msm_host<Bn256G2>(c, n, s, p, o); }

int b2k_bn256_pair(b2k_ctx* ctx, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* gt) {
  if (!ctx || !g1 || !g2 || !gt || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  uint8_t *d1 = nullptr, *d2 = nullptr, *dg = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d1 = c.in(g1, n, 64);
    d2 = c.in(g2, n, 128);
    dg = c.out(gt, n, 384);
  }, [&]() -> int {
    cudaStream_t st = ctx->stream;
    if (ctx->coop_max_n > 0 && n <= (size_t)(ctx->coop_max_n < 8192 ? ctx->coop_max_n : 8192))   // break-even measured near 8 192 on this curve
      coop::k_coop_bn_pair<Coop256, PC6><<<(unsigned)n, 32, Coop256::L::BYTES, st>>>(n, d1, d2, dg, ctx->d_flags);
    else
      k_bn256_pair<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(n, d1, d2, dg, ctx->d_flags);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  });
}

int b2k_bn256_pairing_check(b2k_ctx* ctx, size_t n, const uint8_t* a1, const uint8_t* a2, const uint8_t* b1,
                            const uint8_t* b2, uint8_t* ok) {
  if (!ctx || !a1 || !a2 || !b1 || !b2 || !ok || n == 0) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  uint8_t *da1 = nullptr, *da2 = nullptr, *db1 = nullptr, *db2 = nullptr, *dok = nullptr;
  const int rc = host_call(ctx, [&](Carve& c) {
    da1 = c.in(a1, n, 64);
    da2 = c.in(a2, n, 128);
    db1 = c.in(b1, n, 64);
    db2 = c.in(b2, n, 128);
    dok = c.out(ok, n);
  }, [&] { return bn256_pairing_check_enqueue(ctx, n, da1, da2, db1, db2, dok); });
  return rc == B2K_ERR_POINT ? B2K_OK : rc;   // a malformed operand already failed its own check
}

// sign/bdn on bn256 (NewSchemeOnG1(bn256.NewSuite())): bls.Verify under each mask's aggregate key, e(H(m), X) == e(sig, G2 base),
// H = the try-and-increment hash of b2k_bn256_hash_to_g1.  B2K_ERR_POINT comes only from a malformed term.
int b2k_bn256_bdn_verify_g1sig(b2k_ctx* ctx, size_t n, const uint8_t* terms, size_t m, const uint8_t* masks, const uint8_t* msgs,
                               const uint32_t* offsets, const uint8_t* sigs, uint8_t* status) {
  if (!ctx || !terms || !masks || !msgs || !offsets || !sigs || !status) return B2K_ERR_ARG;
  if (int rc = bdn_args(ctx, n, m)) return rc;
  CK(cudaSetDevice(ctx->device));
  if (check_offsets(ctx, m, offsets)) return B2K_ERR_ARG;
  BdnScratch a;
  uint8_t *d_terms = nullptr, *d_masks = nullptr, *d_msg = nullptr, *d_sig = nullptr, *d_base = nullptr, *d_status = nullptr;
  uint8_t *keys = nullptr, *hm = nullptr, *sg = nullptr, *sig_ok = nullptr, *pair_ok = nullptr;
  uint32_t* d_off = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_terms = c.in(terms, n, 128);
    d_masks = c.in(masks, m, (n + 7) / 8);
    d_msg = c.in(msgs, offsets[m]);
    d_off = c.in(offsets, m + 1);
    d_sig = c.in(sigs, m, 64);
    d_base = c.take<uint8_t>(m, 128);
    c.copy_in(d_base, BN256_G2_BASE, 128);            // one copy of the base; k_bn256_repeat128 fills the other slots
    d_status = c.out(status, m);
    bdn_layout(c, a, BDN_BN256_G2, n, m);
    keys = c.take<uint8_t>(m, 128);
    hm = c.take<uint8_t>(m, 64);
    sg = c.take<uint8_t>(m, 64);
    sig_ok = c.take<uint8_t>(m);
    pair_ok = c.take<uint8_t>(m);
  }, [&]() -> int {
    if (int rc = bdn_aggregate_enqueue(ctx, BDN_BN256_G2, a, n, d_terms, m, d_masks, keys, 128)) return rc;
    k_bn256_repeat128<<<blocks_of(32 * m, 256), 256, 0, ctx->stream>>>(m, d_base);
    k_bn256_g1_decode<<<blocks_of(m, 128), 128, 0, ctx->stream>>>(m, d_sig, sg, sig_ok);
    CK(cudaGetLastError());
    ctx->launches += 2;
    if (int rc = b2k_bn256_hash_to_g1_dev(ctx, m, d_msg, d_off, hm)) return rc;
    if (int rc = bn256_pairing_check_enqueue(ctx, m, hm, keys, sg, d_base, pair_ok)) return rc;
    return bdn_status_enqueue(ctx, m, sig_ok, pair_ok, d_status);
  });
}
}  // extern "C"
