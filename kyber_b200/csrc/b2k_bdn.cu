// b2k_bdn.cu -- the host-side half of sign/bdn: the rogue-key coefficients.
//
// Replaces: bdn.hashPointToR   sign/bdn/bdn.go:29-63
//   blake2s.NewXOF(OutputLengthUnknown, nil) absorbs every public key's MarshalBinary in roster order, 16 bytes are
//   squeezed per key, reversed when the scalar type is big-endian (mod.Int: every pairing suite of the reference) and
//   SetBytes'd -- i.e. the 16 bytes are read LITTLE-endian.  Aggregation uses c_i + 1 (bdn.go:150-154, mask.go:58-61).
// The absorb phase is one sequential hash chain over n * pub_len bytes: inherently serial, it stays on the host here as
// in the reference (it is <1% of the curve work it feeds: the MSM over (c_i + 1, S_i) / (c_i + 1, PK_i) on the device).
// The squeeze phase (BLAKE2X: one independent compression per 32 output bytes) is spread over host threads.
// The coefficients need no device work and no context.
//
// The device half (bdn.cuh drives the bodies): the roster's terms (NewMask, mask.go:34-64) through the existing decoders and
// Point.Mul batches, and AggregatePublicKeys (bdn.go:166-181) for many masks at once as masked sums of those terms.
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

#include "../../include/b2kyber.h"
#define B2K_FP2_BYREF 1   // Fp2 products out of line by reference (tower.cuh), as in the G2 MSM of b2k_g2.cu: the G2 bodies hold whole XYZZ points
#include "codec.cuh"
#include "bn256.cuh"
#include "bdn.cuh"

namespace {

constexpr uint32_t IV[8] = {0x6A09E667u, 0xBB67AE85u, 0x3C6EF372u, 0xA54FF53Au, 0x510E527Fu, 0x9B05688Cu, 0x1F83D9ABu, 0x5BE0CD19u};
constexpr uint8_t SIGMA[10][16] = {
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
    {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
    {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
    {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
    {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0}};

inline uint32_t rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
inline uint32_t le32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

// BLAKE2s (RFC 7693) with an explicit 32-byte parameter block, streaming
struct Blake2s {
  uint32_t h[8];
  uint64_t t = 0;
  uint8_t buf[64];
  size_t fill = 0;

  explicit Blake2s(const uint8_t param[32]) {
    for (int i = 0; i < 8; i++) h[i] = IV[i] ^ le32(param + 4 * i);
  }
  void compress(const uint8_t* blk, bool last) {
    uint32_t m[16], v[16];
    for (int i = 0; i < 16; i++) m[i] = le32(blk + 4 * i);
    for (int i = 0; i < 8; i++) { v[i] = h[i]; v[8 + i] = IV[i]; }
    v[12] ^= (uint32_t)t;
    v[13] ^= (uint32_t)(t >> 32);
    if (last) v[14] = ~v[14];
    auto G = [&](int a, int b, int c, int d, uint32_t x, uint32_t y) {
      v[a] = v[a] + v[b] + x; v[d] = rotr(v[d] ^ v[a], 16);
      v[c] = v[c] + v[d];     v[b] = rotr(v[b] ^ v[c], 12);
      v[a] = v[a] + v[b] + y; v[d] = rotr(v[d] ^ v[a], 8);
      v[c] = v[c] + v[d];     v[b] = rotr(v[b] ^ v[c], 7);
    };
    for (int r = 0; r < 10; r++) {
      const uint8_t* s = SIGMA[r];
      G(0, 4, 8, 12, m[s[0]], m[s[1]]);   G(1, 5, 9, 13, m[s[2]], m[s[3]]);
      G(2, 6, 10, 14, m[s[4]], m[s[5]]);  G(3, 7, 11, 15, m[s[6]], m[s[7]]);
      G(0, 5, 10, 15, m[s[8]], m[s[9]]);  G(1, 6, 11, 12, m[s[10]], m[s[11]]);
      G(2, 7, 8, 13, m[s[12]], m[s[13]]); G(3, 4, 9, 14, m[s[14]], m[s[15]]);
    }
    for (int i = 0; i < 8; i++) h[i] ^= v[i] ^ v[8 + i];
  }
  void update(const uint8_t* p, size_t n) {
    while (n > 0) {
      if (fill == 64) { t += 64; compress(buf, false); fill = 0; }   // a full buffer is only flushed when more follows
      size_t k = 64 - fill;
      if (k > n) k = n;
      std::memcpy(buf + fill, p, k);
      fill += k; p += k; n -= k;
    }
  }
  void final(uint8_t out[32]) {
    t += fill;
    std::memset(buf + fill, 0, 64 - fill);
    compress(buf, true);
    for (int i = 0; i < 8; i++) { out[4 * i] = (uint8_t)h[i]; out[4 * i + 1] = (uint8_t)(h[i] >> 8); out[4 * i + 2] = (uint8_t)(h[i] >> 16); out[4 * i + 3] = (uint8_t)(h[i] >> 24); }
  }
};

// parameter block: digest_len, key_len, fanout, depth, leaf_len(4), node_offset(4), xof_len(2), node_depth, inner_len, salt(8), personal(8)
void param_block(uint8_t p[32], uint8_t digest, uint8_t fanout, uint8_t depth, uint32_t leaf, uint32_t node_offset, uint16_t xof_len,
                 uint8_t node_depth, uint8_t inner) {
  std::memset(p, 0, 32);
  p[0] = digest; p[2] = fanout; p[3] = depth;
  p[4] = (uint8_t)leaf; p[5] = (uint8_t)(leaf >> 8); p[6] = (uint8_t)(leaf >> 16); p[7] = (uint8_t)(leaf >> 24);
  p[8] = (uint8_t)node_offset; p[9] = (uint8_t)(node_offset >> 8); p[10] = (uint8_t)(node_offset >> 16); p[11] = (uint8_t)(node_offset >> 24);
  p[12] = (uint8_t)xof_len; p[13] = (uint8_t)(xof_len >> 8);
  p[14] = node_depth; p[15] = inner;
}

}  // namespace

extern "C" int b2k_bdn_coefficients(size_t n, const uint8_t* pubs, size_t pub_len, int add_one, uint8_t* out32n) {
  if ((n > 0 && (!pubs || !out32n)) || pub_len == 0) return B2K_ERR_ARG;
  if (n > (size_t)1 << 32) return B2K_ERR_ARG;           // BLAKE2Xs stream limit (2^32 blocks of 32 bytes) is far above
  uint8_t p[32], h0[32];
  param_block(p, 32, 1, 1, 0, 0, 0xFFFF, 0, 0);           // root: XOF length "unknown"
  Blake2s root(p);
  root.update(pubs, n * pub_len);
  root.final(h0);
  const size_t nblocks = (16 * n + 31) / 32;
  auto squeeze = [&](size_t lo, size_t hi) {
    for (size_t b = lo; b < hi; b++) {
      uint8_t pp[32], o[32];
      param_block(pp, 32, 0, 0, 32, (uint32_t)b, 0xFFFF, 0, 32);
      Blake2s node(pp);
      node.update(h0, 32);
      node.final(o);
      for (int half = 0; half < 2; half++) {
        const size_t i = 2 * b + half;
        if (i >= n) break;
        // 16 stream bytes, little-endian value c < 2^128; scalar wire format is 32 bytes big-endian
        uint8_t* dst = out32n + 32 * i;
        std::memset(dst, 0, 16);
        for (int k = 0; k < 16; k++) dst[31 - k] = o[16 * half + k];
        if (add_one) {
          for (int k = 31; k >= 0; k--) { if (++dst[k] != 0) break; }
        }
      }
    }
  };
  unsigned nt = std::thread::hardware_concurrency();
  if (nt > 16) nt = 16;
  if (nt < 1 || nblocks < 4096) nt = 1;
  if (nt == 1) {
    squeeze(0, nblocks);
  } else {
    std::vector<std::thread> th;
    const size_t per = (nblocks + nt - 1) / nt;
    for (unsigned k = 0; k < nt; k++) {
      const size_t lo = k * per, hi = lo + per < nblocks ? lo + per : nblocks;
      if (lo < hi) th.emplace_back(squeeze, lo, hi);
    }
    for (auto& x : th) x.join();
  }
  return B2K_OK;
}

// ---- the device half ------------------------------------------------------------------------------------------------------
namespace b2k {

constexpr unsigned BDN_BLOCK = 64;   // two warps per block in the masked sum

// operand bytes -> Montgomery affine in scratch, re-validated like every operand (FLAG_POINT, the term counts as infinity)
template <class CV>
__global__ void __launch_bounds__(128) k_bdn_load(size_t n, const uint8_t* __restrict__ wire, Affine<typename CV::F>* __restrict__ terms,
                                                  uint32_t* flags) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<typename CV::F> a;
  if (!load_checked<CV>(a, wire + (size_t)CV::IN_BYTES * i)) atomicOr(flags, FLAG_POINT);
  terms[i] = a;
}

__global__ void __launch_bounds__(128) k_bdn_complement(size_t m, uint32_t n, const uint8_t* __restrict__ masks, size_t stride,
                                                        uint8_t* __restrict__ comp) {
  const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) comp[k] = bdn_complement(masks + k * stride, stride, n) ? 1 : 0;
}

// part[k nslices + s] = the masked sum of slice s of mask k: one warp per (mask, slice), lane l walks mask word 32 s + l, then the
// lanes' sums meet in a tree through shared memory (the points stay in memory: see bdn_add).
// masks == nullptr: the all-ones mask (m = 1), i.e. the slices of the roster total.
template <class CV>
__global__ void __launch_bounds__(BDN_BLOCK) k_bdn_masked_sum(size_t m, uint32_t n, uint32_t nslices, const uint8_t* __restrict__ masks,
                                                              size_t stride, const uint8_t* __restrict__ comp,
                                                              const Affine<typename CV::F>* __restrict__ terms, Xyzz<typename CV::F>* __restrict__ part) {
  using X = Xyzz<typename CV::F>;
  __shared__ X lane_sum[BDN_BLOCK];
  const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (warp >= m * nslices) return;                     // whole warps only: blockDim is a multiple of 32
  const size_t k = warp / nslices;
  const uint32_t w = (uint32_t)(warp % nslices) * 32 + lane;
  const uint32_t bits = bdn_lane_bits(masks ? masks + k * stride : nullptr, stride, n, w, comp && comp[k]);
  X& acc = lane_sum[threadIdx.x];
  xyzz_set_inf(acc);
  bdn_walk(acc, bits, terms, 32 * w);
  __syncwarp();
#pragma unroll 1
  for (uint32_t d = 16; d > 0; d >>= 1) {
    if (lane < d) bdn_add(acc, acc, lane_sum[threadIdx.x + d]);
    __syncwarp();
  }
  if (lane == 0) part[warp] = acc;
}

// total[nslices] = the roster total from its slice partials total[0 .. nslices)
template <class CV>
__global__ void k_bdn_total(uint32_t nslices, Xyzz<typename CV::F>* total) {
  if (threadIdx.x || blockIdx.x) return;
  Xyzz<typename CV::F> r;
  bdn_combine(r, total, nslices);
  total[nslices] = r;
}

// out + k out_stride = mask k's aggregate key in operand form
template <class CV>
__global__ void __launch_bounds__(64) k_bdn_finish(size_t m, uint32_t nslices, const Xyzz<typename CV::F>* __restrict__ part,
                                                   const uint8_t* __restrict__ comp, const Xyzz<typename CV::F>* __restrict__ total,
                                                   uint8_t* __restrict__ out, size_t out_stride) {
  const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= m) return;
  Affine<typename CV::F> r;
  bdn_finish(r, part + k * nslices, nslices, comp[k] != 0, *total);
  CV::store_affine(out + k * out_stride, r);
}

// FLAG_POINT when a roster key did not decode (NewMask only ever sees decoded points)
__global__ void k_bdn_require(size_t n, const uint8_t* __restrict__ ok, uint32_t* flags) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !ok[i]) atomicOr(flags, FLAG_POINT);
}

__global__ void k_bdn_status(size_t m, const uint8_t* __restrict__ sig_ok, const uint8_t* __restrict__ pair_ok,
                             uint8_t* __restrict__ status) {
  const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) status[k] = !sig_ok[k] ? B2K_BDN_SIG : (pair_ok[k] ? B2K_BDN_OK : B2K_BDN_INVALID);
}

}  // namespace b2k

namespace b2k_host {

int bdn_args(b2k_ctx* ctx, size_t n, size_t m) {
  if (n == 0 || m == 0 || n > B2K_BDN_MAX_N || m > B2K_BDN_MAX_M) return bad_arg(ctx, "bdn: n and m must be in 1..2^20");
  return B2K_OK;
}

namespace {

template <class CV>
void layout_of(Carve& c, BdnScratch& s, size_t n, size_t m) {
  using F = typename CV::F;
  s.nslices = (n + BDN_SLICE - 1) / BDN_SLICE;
  s.terms = c.take<Affine<F>>(n);
  s.comp = c.take<uint8_t>(m);
  s.part = c.take<Xyzz<F>>(m, s.nslices);
  s.total = c.take<Xyzz<F>>(s.nslices + 1);
}

template <class CV>
int aggregate_enqueue(b2k_ctx* ctx, const BdnScratch& s, size_t n, const uint8_t* d_terms, size_t m, const uint8_t* d_masks,
                      uint8_t* d_out, size_t out_stride) {
  using F = typename CV::F;
  cudaStream_t st = ctx->stream;
  const size_t stride = (n + 7) / 8;
  const uint32_t ns = (uint32_t)s.nslices;
  auto* terms = static_cast<Affine<F>*>(s.terms);
  auto* part = static_cast<Xyzz<F>*>(s.part);
  auto* total = static_cast<Xyzz<F>*>(s.total);
  k_bdn_load<CV><<<blocks_of(n, 128), 128, 0, st>>>(n, d_terms, terms, ctx->d_flags);
  k_bdn_masked_sum<CV><<<blocks_of(32 * (size_t)ns, BDN_BLOCK), BDN_BLOCK, 0, st>>>(1, (uint32_t)n, ns, nullptr, stride, nullptr, terms, total);
  k_bdn_total<CV><<<1, 32, 0, st>>>(ns, total);
  k_bdn_complement<<<blocks_of(m, 128), 128, 0, st>>>(m, (uint32_t)n, d_masks, stride, s.comp);
  k_bdn_masked_sum<CV><<<blocks_of(32 * m * ns, BDN_BLOCK), BDN_BLOCK, 0, st>>>(m, (uint32_t)n, ns, d_masks, stride, s.comp, terms, part);
  k_bdn_finish<CV><<<blocks_of(m, 64), 64, 0, st>>>(m, ns, part, s.comp, total + ns, d_out, out_stride);
  CK(cudaGetLastError());
  ctx->launches += 6;
  return B2K_OK;
}

}  // namespace

void bdn_layout(Carve& c, BdnScratch& s, BdnGroup g, size_t n, size_t m) {
  if (g == BDN_BLS_G2) layout_of<Bls381G2>(c, s, n, m);
  else if (g == BDN_BLS_G1) layout_of<Bls381G1>(c, s, n, m);
  else layout_of<Bn256G2>(c, s, n, m);
}

int bdn_aggregate_enqueue(b2k_ctx* ctx, BdnGroup g, const BdnScratch& s, size_t n, const uint8_t* d_terms, size_t m,
                          const uint8_t* d_masks, uint8_t* d_out, size_t out_stride) {
  if (g == BDN_BLS_G2) return aggregate_enqueue<Bls381G2>(ctx, s, n, d_terms, m, d_masks, d_out, out_stride);
  if (g == BDN_BLS_G1) return aggregate_enqueue<Bls381G1>(ctx, s, n, d_terms, m, d_masks, d_out, out_stride);
  return aggregate_enqueue<Bn256G2>(ctx, s, n, d_terms, m, d_masks, d_out, out_stride);
}

int bdn_status_enqueue(b2k_ctx* ctx, size_t m, const uint8_t* d_sig_ok, const uint8_t* d_pair_ok, uint8_t* d_status) {
  k_bdn_status<<<blocks_of(m, 256), 256, 0, ctx->stream>>>(m, d_sig_ok, d_pair_ok, d_status);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return B2K_OK;
}

}  // namespace b2k_host

namespace {
using namespace b2k_host;

constexpr size_t operand_bytes(BdnGroup g) { return g == BDN_BLS_G2 ? 192 : g == BDN_BLS_G1 ? 96 : 128; }

int aggregate_host(b2k_ctx* ctx, BdnGroup g, size_t n, const uint8_t* terms, size_t m, const uint8_t* masks, uint8_t* out) {
  if (!ctx || !terms || !masks || !out) return B2K_ERR_ARG;
  if (int rc = bdn_args(ctx, n, m)) return rc;
  CK(cudaSetDevice(ctx->device));
  const size_t ob = operand_bytes(g);
  BdnScratch s;
  uint8_t *d_terms = nullptr, *d_masks = nullptr, *d_out = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_terms = c.in(terms, n, ob);
    d_masks = c.in(masks, m, (n + 7) / 8);
    d_out = c.out(out, m, ob);
    bdn_layout(c, s, g, n, m);
  }, [&] { return bdn_aggregate_enqueue(ctx, g, s, n, d_terms, m, d_masks, d_out, ob); });
}

int aggregate_dev(b2k_ctx* ctx, BdnGroup g, size_t n, const void* d_terms, size_t m, const void* d_masks, void* d_out) {
  if (!ctx || !d_terms || !d_masks || !d_out) return B2K_ERR_ARG;
  if (int rc = bdn_args(ctx, n, m)) return rc;
  CK(cudaSetDevice(ctx->device));
  BdnScratch s;
  if (int rc = arena_carve(ctx, [&](Carve& c) { bdn_layout(c, s, g, n, m); })) return rc;
  return bdn_aggregate_enqueue(ctx, g, s, n, (const uint8_t*)d_terms, m, (const uint8_t*)d_masks, (uint8_t*)d_out, operand_bytes(g));
}

// BLS12-381 terms: coefficients over the input (= MarshalBinary) bytes on the host, then UnmarshalBinary and Point.Mul on the device
using DevCall = int (*)(b2k_ctx*, size_t, const void*, const void*, void*);
int bls_terms(b2k_ctx* ctx, size_t n, const uint8_t* pubs, uint8_t* terms, size_t wire, size_t operand,
              int (*decompress)(b2k_ctx*, size_t, const void*, void*, void*), DevCall mul) {
  if (!ctx || !pubs || !terms) return B2K_ERR_ARG;
  if (int rc = bdn_args(ctx, n, 1)) return rc;
  CK(cudaSetDevice(ctx->device));
  std::vector<uint8_t> fac(32 * n);
  if (int rc = b2k_bdn_coefficients(n, pubs, wire, 1, fac.data())) return rc;
  uint8_t *d_pub = nullptr, *d_fac = nullptr, *d_dec = nullptr, *d_ok = nullptr, *d_out = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_pub = c.in(pubs, n, wire);
    d_fac = c.in(fac.data(), n, 32);
    d_dec = c.take<uint8_t>(n, operand);
    d_ok = c.take<uint8_t>(n);
    d_out = c.out(terms, n, operand);
  }, [&]() -> int {
    if (int rc = decompress(ctx, n, d_pub, d_dec, d_ok)) return rc;
    k_bdn_require<<<blocks_of(n, 256), 256, 0, ctx->stream>>>(n, d_ok, ctx->d_flags);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return mul(ctx, n, d_fac, d_dec, d_out);
  });
}

// bn256 p, big-endian: Unmarshal reduces every coordinate below 2^256 < 2p by at most one subtraction (gfp.go:115-122)
constexpr uint8_t BN256_P[32] = {0x8f, 0xb5, 0x01, 0xe3, 0x4a, 0xa3, 0x87, 0xf9, 0xaa, 0x6f, 0xec, 0xb8, 0x61, 0x84, 0xdc, 0x21,
                                 0xee, 0x5b, 0x88, 0xd1, 0x20, 0xb5, 0xb5, 0x9e, 0x18, 0x5c, 0xac, 0x6c, 0x5e, 0x08, 0x96, 0x67};
void bn256_reduce32(uint8_t* v) {
  if (std::memcmp(v, BN256_P, 32) < 0) return;      // big-endian bytes compare as numbers
  int borrow = 0;
  for (int k = 31; k >= 0; k--) {
    const int d = (int)v[k] - BN256_P[k] - borrow;
    borrow = d < 0;
    v[k] = (uint8_t)(d + (borrow ? 256 : 0));
  }
}

}  // namespace

extern "C" {

int b2k_bls12381_g2_bdn_terms(b2k_ctx* ctx, size_t n, const uint8_t* pubs, uint8_t* terms) {
  return bls_terms(ctx, n, pubs, terms, 96, 192, b2k_bls12381_g2_decompress_dev, b2k_bls12381_g2_mul_batch_affine_dev);
}
int b2k_bls12381_g1_bdn_terms(b2k_ctx* ctx, size_t n, const uint8_t* pubs, uint8_t* terms) {
  return bls_terms(ctx, n, pubs, terms, 48, 96, b2k_bls12381_g1_decompress_dev, b2k_bls12381_g1_mul_batch_affine_dev);
}
// bn256: the coefficients hash the canonical re-encoding (MarshalBinary of the decoded key); the Point.Mul batch re-checks the
// twist equation, which is all bn256's Unmarshal checks (pairing/bn256/point.go:469-506)
int b2k_bn256_g2_bdn_terms(b2k_ctx* ctx, size_t n, const uint8_t* pubs, uint8_t* terms) {
  if (!ctx || !pubs || !terms) return B2K_ERR_ARG;
  if (int rc = bdn_args(ctx, n, 1)) return rc;
  std::vector<uint8_t> canon(pubs, pubs + 128 * n), fac(32 * n);
  for (size_t i = 0; i < 4 * n; i++) bn256_reduce32(canon.data() + 32 * i);
  if (int rc = b2k_bdn_coefficients(n, canon.data(), 128, 1, fac.data())) return rc;
  return b2k_bn256_g2_mul_batch(ctx, n, fac.data(), canon.data(), terms);
}

int b2k_bls12381_g2_bdn_aggregate_keys(b2k_ctx* ctx, size_t n, const uint8_t* terms, size_t m, const uint8_t* masks, uint8_t* out) {
  return aggregate_host(ctx, BDN_BLS_G2, n, terms, m, masks, out);
}
int b2k_bls12381_g2_bdn_aggregate_keys_dev(b2k_ctx* ctx, size_t n, const void* d_terms, size_t m, const void* d_masks, void* d_out) {
  return aggregate_dev(ctx, BDN_BLS_G2, n, d_terms, m, d_masks, d_out);
}
int b2k_bls12381_g1_bdn_aggregate_keys(b2k_ctx* ctx, size_t n, const uint8_t* terms, size_t m, const uint8_t* masks, uint8_t* out) {
  return aggregate_host(ctx, BDN_BLS_G1, n, terms, m, masks, out);
}
int b2k_bls12381_g1_bdn_aggregate_keys_dev(b2k_ctx* ctx, size_t n, const void* d_terms, size_t m, const void* d_masks, void* d_out) {
  return aggregate_dev(ctx, BDN_BLS_G1, n, d_terms, m, d_masks, d_out);
}
int b2k_bn256_g2_bdn_aggregate_keys(b2k_ctx* ctx, size_t n, const uint8_t* terms, size_t m, const uint8_t* masks, uint8_t* out) {
  return aggregate_host(ctx, BDN_BN256_G2, n, terms, m, masks, out);
}

}  // extern "C"
