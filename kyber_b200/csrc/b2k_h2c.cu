// b2k_h2c.cu -- C ABI entry points for batched hash-to-G1 and batched BLS signature verification
// (signatures on G1, public keys on G2): the per-signature work of bls.Verify, sign/bls/bls.go:82-96.
#include "msm_host.cuh"
#include "h2c_g2.cuh"
#include "pairing_kernels.cuh"
#include "bdn.cuh"
using namespace b2k_host;

namespace b2k {

__global__ void __launch_bounds__(128) k_hash_to_g1(size_t n, const uint8_t* __restrict__ msgs,
                                                    const uint32_t* __restrict__ offs, const uint8_t* __restrict__ dst,
                                                    uint32_t dst_len, uint8_t* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<BFp> a;
  hash_to_g1(a, msgs + offs[i], (offs[i + 1] >= offs[i] ? offs[i + 1] - offs[i] : 0u), dst, dst_len);
  Bls381G1::store_affine(out + 96 * i, a);
}

__global__ void __launch_bounds__(64) k_hash_to_g2(size_t n, const uint8_t* __restrict__ msgs,
                                                   const uint32_t* __restrict__ offs, const uint8_t* __restrict__ dst,
                                                   uint32_t dst_len, uint8_t* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<BFp2> a;
  hash_to_g2(a, msgs + offs[i], (offs[i + 1] >= offs[i] ? offs[i + 1] - offs[i] : 0u), dst, dst_len);
  Bls381G2::store_affine(out + 192 * i, a);
}

__global__ void k_write_g1_generator(uint8_t* out96) {
  if (threadIdx.x || blockIdx.x) return;
  Affine<BFp> g;
  Bls381G1::generator(g);
  Bls381G1::store_affine(out96, g);
}

__global__ void k_write_g2_generator(uint8_t* out192) {
  if (threadIdx.x || blockIdx.x) return;
  Affine<BFp2> g;
  for (int j = 0; j < 12; j++) {
    g.x.c0.v[j] = Bls381Fp::g2x0(j); g.x.c1.v[j] = Bls381Fp::g2x1(j);
    g.y.c0.v[j] = Bls381Fp::g2y0(j); g.y.c1.v[j] = Bls381Fp::g2y1(j);
  }
  Bls381G2::store_affine(out192, g);
}

__global__ void k_and_flags(size_t n, const uint8_t* a, const uint8_t* b, uint8_t* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i] & b[i];
}

// the decompression kernels of b2k_g2.cu, built here without B2K_FP2_BYREF: that build of the G2 kernel takes a 2608-byte stack
// frame against 2112 bytes here, and a one-signature verify_g1sig through it measured ~1 % slower (H100 80GB HBM3, 700 W)
__global__ void __launch_bounds__(128) k_g1_decompress_v(size_t n, const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                                                         uint8_t* __restrict__ ok) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<BFp> a;
  bool good = g1_decompress(a, in + 48 * i, true);
  if (!good) aff_set_inf(a);
  Bls381G1::store_affine(out + 96 * i, a);
  ok[i] = good ? 1 : 0;
}
__global__ void __launch_bounds__(64) k_g2_decompress_v(size_t n, const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                                                        uint8_t* __restrict__ ok) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<BFp2> a;
  bool good = g2_decompress(a, in + 96 * i, true);
  if (!good) aff_set_inf(a);
  Bls381G2::store_affine(out + 192 * i, a);
  ok[i] = good ? 1 : 0;
}

}  // namespace b2k

namespace {

// hash_to_g1/g2 from host buffers: out_bytes per point, dev = the *_dev entry point
template <class Dev>
int hash_host(b2k_ctx* ctx, size_t n, const uint8_t* msgs, const uint32_t* offsets, const uint8_t* dst, uint32_t dst_len, uint8_t* out,
              size_t out_bytes, Dev dev) {
  if (!ctx || !msgs || !offsets || !dst || !out || n == 0 || dst_len == 0 || dst_len > 255) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  if (check_offsets(ctx, n, offsets)) return B2K_ERR_ARG;
  uint8_t *dm = nullptr, *dd = nullptr, *dout = nullptr;
  uint32_t* doff = nullptr;
  return host_call(ctx, [&](Carve& c) {
    dm = c.in(msgs, offsets[n]);
    doff = c.in(offsets, n + 1);
    dd = c.in(dst, dst_len);
    dout = c.out(out, n, out_bytes);
  }, [&] { return dev(ctx, n, dm, doff, dd, dst_len, dout); });
}

// scratch of bls.Verify for n signatures: decompressed keys and signatures, H(m) (in the signature's group), the decode flags
// and the generator (in the key's group)
struct VerifyScratch {
  uint8_t *pk, *sg, *hm, *ok1, *ok2, *okc, *gen;
};
void verify_layout(Carve& c, VerifyScratch& s, size_t n, bool sig_g1) {
  const size_t pk_bytes = sig_g1 ? 192 : 96, sig_bytes = sig_g1 ? 96 : 192;
  s.pk = c.take<uint8_t>(n, pk_bytes);
  s.sg = c.take<uint8_t>(n, sig_bytes);
  s.hm = c.take<uint8_t>(n, sig_bytes);
  s.ok1 = c.take<uint8_t>(n);
  s.ok2 = c.take<uint8_t>(n);
  s.okc = c.take<uint8_t>(n);
  s.gen = c.take<uint8_t>(pk_bytes);
}

// bls.Verify's key-independent tail, every buffer on the device: the generator (in the key's group), UnmarshalBinary of the
// signatures (ok2), H(msg), and the pairing check of s.pk (decoded by the caller, with its flags in ok1) against them:
//   sig_g1: e(H(m), pk) == e(sig, G2 generator)
//   else (bls.NewSchemeOnG2, sign/bls/bls.go:48-59): pk in G1, sig in G2, H(msg) in G2, e(pk, H(m)) == e(G1 base, sig)
// Shared by bls.Verify (verify_enqueue) and the BDN batch, whose keys are aggregates (bdn_verify_enqueue).
int verify_tail(b2k_ctx* ctx, bool sig_g1, const VerifyScratch& s, size_t n, const void* msgs, const void* offsets, const void* dst,
                uint32_t dst_len, const void* sigs, void* ok) {
  cudaStream_t st = ctx->stream;
  const uint8_t *m = (const uint8_t*)msgs, *d = (const uint8_t*)dst, *g = (const uint8_t*)sigs;
  const uint32_t* o = (const uint32_t*)offsets;
  if (sig_g1) {
    k_write_g2_generator<<<1, 32, 0, st>>>(s.gen);
    k_g1_decompress_v<<<blocks_of(n, 128), 128, 0, st>>>(n, g, s.sg, s.ok2);
  } else {
    k_write_g1_generator<<<1, 32, 0, st>>>(s.gen);
    k_g2_decompress_v<<<blocks_of(n, 64), 64, 0, st>>>(n, g, s.sg, s.ok2);
  }
  k_and_flags<<<blocks_of(n, 256), 256, 0, st>>>(n, s.ok1, s.ok2, s.okc);
  if (sig_g1) {
    k_hash_to_g1<<<blocks_of(n, 128), 128, 0, st>>>(n, m, o, d, dst_len, s.hm);
    b2k_internal_launch_pairing_check(ctx, n, s.hm, s.pk, s.sg, s.gen, (uint8_t*)ok, 1, s.okc);
  } else {
    k_hash_to_g2<<<blocks_of(n, 64), 64, 0, st>>>(n, m, o, d, dst_len, s.hm);
    b2k_internal_launch_pairing_check(ctx, n, s.pk, s.hm, s.gen, s.sg, (uint8_t*)ok, 2, s.okc);   // b = (base [shared], sig)
  }
  CK(cudaGetLastError());
  ctx->launches += 5;
  return B2K_OK;
}

// ok[i] = bls.Verify(pk_i, msg_i, sig_i), every buffer on the device: UnmarshalBinary of the keys, then the shared tail
int verify_enqueue(b2k_ctx* ctx, bool sig_g1, const VerifyScratch& s, size_t n, const void* pks, const void* msgs, const void* offsets,
                   const void* dst, uint32_t dst_len, const void* sigs, void* ok) {
  const uint8_t* p = (const uint8_t*)pks;
  if (sig_g1) k_g2_decompress_v<<<blocks_of(n, 64), 64, 0, ctx->stream>>>(n, p, s.pk, s.ok1);
  else k_g1_decompress_v<<<blocks_of(n, 128), 128, 0, ctx->stream>>>(n, p, s.pk, s.ok1);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return verify_tail(ctx, sig_g1, s, n, msgs, offsets, dst, dst_len, sigs, ok);
}

// BDN: bls.Verify under each mask's aggregate key (written straight into the key slots of the tail's scratch), then statuses
struct BdnVerifyScratch {
  VerifyScratch v;
  BdnScratch a;
  uint8_t* pair_ok;
};
void bdn_verify_layout(Carve& c, BdnVerifyScratch& s, size_t n, size_t m, bool sig_g1) {
  verify_layout(c, s.v, m, sig_g1);
  bdn_layout(c, s.a, sig_g1 ? BDN_BLS_G2 : BDN_BLS_G1, n, m);
  s.pair_ok = c.take<uint8_t>(m);
}
int bdn_verify_enqueue(b2k_ctx* ctx, bool sig_g1, const BdnVerifyScratch& s, size_t n, const void* terms, size_t m, const void* masks,
                       const void* msgs, const void* offsets, const void* dst, uint32_t dst_len, const void* sigs, void* status) {
  int rc = bdn_aggregate_enqueue(ctx, sig_g1 ? BDN_BLS_G2 : BDN_BLS_G1, s.a, n, (const uint8_t*)terms, m, (const uint8_t*)masks,
                                 s.v.pk, sig_g1 ? 192 : 96);
  if (rc) return rc;
  CK(cudaMemsetAsync(s.v.ok1, 1, m, ctx->stream));      // an aggregate key is a point by construction
  rc = verify_tail(ctx, sig_g1, s.v, m, msgs, offsets, dst, dst_len, sigs, s.pair_ok);
  if (rc) return rc;
  return bdn_status_enqueue(ctx, m, s.v.ok2, s.pair_ok, (uint8_t*)status);
}

int bdn_verify_dev(b2k_ctx* ctx, bool sig_g1, size_t n, const void* d_terms, size_t m, const void* d_masks, const void* d_msgs,
                   const void* d_offsets, const void* d_dst, uint32_t dst_len, const void* d_sigs, void* d_status) {
  if (!ctx || !d_terms || !d_masks || !d_msgs || !d_offsets || !d_dst || !d_sigs || !d_status || dst_len == 0 || dst_len > 255)
    return B2K_ERR_ARG;
  if (int rc = bdn_args(ctx, n, m)) return rc;
  CK(cudaSetDevice(ctx->device));
  BdnVerifyScratch s;
  if (int rc = arena_carve(ctx, [&](Carve& c) { bdn_verify_layout(c, s, n, m, sig_g1); })) return rc;
  return bdn_verify_enqueue(ctx, sig_g1, s, n, d_terms, m, d_masks, d_msgs, d_offsets, d_dst, dst_len, d_sigs, d_status);
}

// bad signature data is a status; B2K_ERR_POINT comes only from a malformed term and stays a call error
int bdn_verify_host(b2k_ctx* ctx, bool sig_g1, size_t n, const uint8_t* terms, size_t m, const uint8_t* masks, const uint8_t* msgs,
                    const uint32_t* offsets, const uint8_t* dst, uint32_t dst_len, const uint8_t* sigs, uint8_t* status) {
  if (!ctx || !terms || !masks || !msgs || !offsets || !dst || !sigs || !status || dst_len == 0 || dst_len > 255) return B2K_ERR_ARG;
  if (int rc = bdn_args(ctx, n, m)) return rc;
  CK(cudaSetDevice(ctx->device));
  if (check_offsets(ctx, m, offsets)) return B2K_ERR_ARG;
  BdnVerifyScratch s;
  uint8_t *d_terms = nullptr, *d_masks = nullptr, *d_sig = nullptr, *d_msg = nullptr, *d_dst = nullptr, *d_status = nullptr;
  uint32_t* d_off = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_terms = c.in(terms, n, sig_g1 ? 192 : 96);
    d_masks = c.in(masks, m, (n + 7) / 8);
    d_sig = c.in(sigs, m, sig_g1 ? 48 : 96);
    d_msg = c.in(msgs, offsets[m]);
    d_off = c.in(offsets, m + 1);
    d_dst = c.in(dst, dst_len);
    d_status = c.out(status, m);
    bdn_verify_layout(c, s, n, m, sig_g1);
  }, [&] { return bdn_verify_enqueue(ctx, sig_g1, s, n, d_terms, m, d_masks, d_msg, d_off, d_dst, dst_len, d_sig, d_status); });
}

int verify_dev(b2k_ctx* ctx, bool sig_g1, size_t n, const void* d_pks, const void* d_msgs, const void* d_offsets, const void* d_dst,
               uint32_t dst_len, const void* d_sigs, void* d_ok) {
  if (!ctx || !d_pks || !d_msgs || !d_offsets || !d_dst || !d_sigs || !d_ok || n == 0 || dst_len == 0 || dst_len > 255)
    return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  VerifyScratch s;
  int rc = arena_carve(ctx, [&](Carve& c) { verify_layout(c, s, n, sig_g1); });
  if (rc) return rc;
  return verify_enqueue(ctx, sig_g1, s, n, d_pks, d_msgs, d_offsets, d_dst, dst_len, d_sigs, d_ok);
}

int verify_host(b2k_ctx* ctx, bool sig_g1, size_t n, const uint8_t* pks, const uint8_t* msgs, const uint32_t* offsets, const uint8_t* dst,
                uint32_t dst_len, const uint8_t* sigs, uint8_t* ok) {
  if (!ctx || !pks || !msgs || !offsets || !dst || !sigs || !ok || n == 0 || dst_len == 0 || dst_len > 255) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  if (check_offsets(ctx, n, offsets)) return B2K_ERR_ARG;
  VerifyScratch s;
  uint8_t *d_pk = nullptr, *d_sig = nullptr, *d_msg = nullptr, *d_dst = nullptr, *d_ok = nullptr;
  uint32_t* d_off = nullptr;
  const int rc = host_call(ctx, [&](Carve& c) {
    d_pk = c.in(pks, n, sig_g1 ? 96 : 48);
    d_sig = c.in(sigs, n, sig_g1 ? 48 : 96);
    d_msg = c.in(msgs, offsets[n]);
    d_off = c.in(offsets, n + 1);
    d_dst = c.in(dst, dst_len);
    d_ok = c.out(ok, n);
    verify_layout(c, s, n, sig_g1);
  }, [&] { return verify_enqueue(ctx, sig_g1, s, n, d_pk, d_msg, d_off, d_dst, dst_len, d_sig, d_ok); });
  return rc == B2K_ERR_POINT ? B2K_OK : rc;   // a malformed operand already failed its own check: per-element booleans
}

}  // namespace

extern "C" {

int b2k_bls12381_hash_to_g1_dev(b2k_ctx* ctx, size_t n, const void* d_msgs, const void* d_offsets, const void* d_dst,
                                uint32_t dst_len, void* d_out) {
  if (!ctx || !d_msgs || !d_offsets || !d_dst || !d_out || n == 0 || dst_len == 0 || dst_len > 255) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  k_hash_to_g1<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(n, (const uint8_t*)d_msgs, (const uint32_t*)d_offsets,
                                                                    (const uint8_t*)d_dst, dst_len, (uint8_t*)d_out);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return B2K_OK;
}

int b2k_bls12381_hash_to_g1(b2k_ctx* ctx, size_t n, const uint8_t* msgs, const uint32_t* offsets, const uint8_t* dst,
                            uint32_t dst_len, uint8_t* out) {
  return hash_host(ctx, n, msgs, offsets, dst, dst_len, out, 96, b2k_bls12381_hash_to_g1_dev);
}

int b2k_bls12381_hash_to_g2_dev(b2k_ctx* ctx, size_t n, const void* d_msgs, const void* d_offsets, const void* d_dst,
                                uint32_t dst_len, void* d_out) {
  if (!ctx || !d_msgs || !d_offsets || !d_dst || !d_out || n == 0 || dst_len == 0 || dst_len > 255) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  k_hash_to_g2<<<(unsigned)((n + 63) / 64), 64, 0, ctx->stream>>>(n, (const uint8_t*)d_msgs, (const uint32_t*)d_offsets,
                                                                  (const uint8_t*)d_dst, dst_len, (uint8_t*)d_out);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return B2K_OK;
}

int b2k_bls12381_hash_to_g2(b2k_ctx* ctx, size_t n, const uint8_t* msgs, const uint32_t* offsets, const uint8_t* dst,
                            uint32_t dst_len, uint8_t* out) {
  return hash_host(ctx, n, msgs, offsets, dst, dst_len, out, 192, b2k_bls12381_hash_to_g2_dev);
}

// bls.Verify, sign/bls/bls.go:82-96, for signatures on G1 / keys on G2 (g1sig) and signatures on G2 / keys on G1 (g2sig).
// The *_dev forms take device buffers; scratch comes from the context arena.
int b2k_bls12381_verify_g1sig_dev(b2k_ctx* ctx, size_t n, const void* d_pks96, const void* d_msgs, const void* d_offsets,
                                  const void* d_dst, uint32_t dst_len, const void* d_sigs48, void* d_ok) {
  return verify_dev(ctx, true, n, d_pks96, d_msgs, d_offsets, d_dst, dst_len, d_sigs48, d_ok);
}
int b2k_bls12381_verify_g2sig_dev(b2k_ctx* ctx, size_t n, const void* d_pks48, const void* d_msgs, const void* d_offsets,
                                  const void* d_dst, uint32_t dst_len, const void* d_sigs96, void* d_ok) {
  return verify_dev(ctx, false, n, d_pks48, d_msgs, d_offsets, d_dst, dst_len, d_sigs96, d_ok);
}
int b2k_bls12381_verify_g1sig(b2k_ctx* ctx, size_t n, const uint8_t* pks96, const uint8_t* msgs, const uint32_t* offsets,
                              const uint8_t* dst, uint32_t dst_len, const uint8_t* sigs48, uint8_t* ok) {
  return verify_host(ctx, true, n, pks96, msgs, offsets, dst, dst_len, sigs48, ok);
}
int b2k_bls12381_verify_g2sig(b2k_ctx* ctx, size_t n, const uint8_t* pks48, const uint8_t* msgs, const uint32_t* offsets,
                              const uint8_t* dst, uint32_t dst_len, const uint8_t* sigs96, uint8_t* ok) {
  return verify_host(ctx, false, n, pks48, msgs, offsets, dst, dst_len, sigs96, ok);
}

// sign/bdn: bls.Verify under the aggregate key of each mask over one roster's terms (b2k_bdn.cu aggregates)
int b2k_bls12381_bdn_verify_g1sig(b2k_ctx* ctx, size_t n, const uint8_t* terms, size_t m, const uint8_t* masks, const uint8_t* msgs,
                                  const uint32_t* offsets, const uint8_t* dst, uint32_t dst_len, const uint8_t* sigs, uint8_t* status) {
  return bdn_verify_host(ctx, true, n, terms, m, masks, msgs, offsets, dst, dst_len, sigs, status);
}
int b2k_bls12381_bdn_verify_g1sig_dev(b2k_ctx* ctx, size_t n, const void* d_terms, size_t m, const void* d_masks, const void* d_msgs,
                                      const void* d_offsets, const void* d_dst, uint32_t dst_len, const void* d_sigs, void* d_status) {
  return bdn_verify_dev(ctx, true, n, d_terms, m, d_masks, d_msgs, d_offsets, d_dst, dst_len, d_sigs, d_status);
}
int b2k_bls12381_bdn_verify_g2sig(b2k_ctx* ctx, size_t n, const uint8_t* terms, size_t m, const uint8_t* masks, const uint8_t* msgs,
                                  const uint32_t* offsets, const uint8_t* dst, uint32_t dst_len, const uint8_t* sigs, uint8_t* status) {
  return bdn_verify_host(ctx, false, n, terms, m, masks, msgs, offsets, dst, dst_len, sigs, status);
}
int b2k_bls12381_bdn_verify_g2sig_dev(b2k_ctx* ctx, size_t n, const void* d_terms, size_t m, const void* d_masks, const void* d_msgs,
                                      const void* d_offsets, const void* d_dst, uint32_t dst_len, const void* d_sigs, void* d_status) {
  return bdn_verify_dev(ctx, false, n, d_terms, m, d_masks, d_msgs, d_offsets, d_dst, dst_len, d_sigs, d_status);
}

}  // extern "C"
