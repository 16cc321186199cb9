// b2k_h2c.cu -- C ABI entry points for batched hash-to-G1 and batched BLS signature verification
// (signatures on G1, public keys on G2): the per-signature work of bls.Verify, sign/bls/bls.go:82-96.
#include "msm_host.cuh"
#include "h2c_g2.cuh"
#include "pairing_kernels.cuh"
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

// same kernels as b2k_g2.cu, local to this translation unit
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
  if (!ctx || !msgs || !offsets || !dst || !out || n == 0 || dst_len == 0 || dst_len > 255) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  if (check_offsets(ctx, n, offsets)) return B2K_ERR_ARG;
  size_t mbytes = offsets[n];
  int rc = arena_reserve(ctx, mbytes + (n + 1) * 4 + 256 + n * 96 + 4096);
  if (rc) return rc;
  uint8_t* dm = arena_take<uint8_t>(ctx, mbytes + 1);
  uint32_t* doff = arena_take<uint32_t>(ctx, n + 1);
  uint8_t* dd = arena_take<uint8_t>(ctx, 256);
  uint8_t* dout = arena_take<uint8_t>(ctx, n * 96);
  if (mbytes) CK(cudaMemcpyAsync(dm, msgs, mbytes, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(doff, offsets, (n + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(dd, dst, dst_len, cudaMemcpyHostToDevice, ctx->stream));
  rc = b2k_bls12381_hash_to_g1_dev(ctx, n, dm, doff, dd, dst_len, dout);
  if (rc) return rc;
  CK(cudaMemcpyAsync(out, dout, n * 96, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return B2K_OK;
}

// ok[i] = bls.Verify(pk_i, msg_i, sig_i) for signatures on G1 / keys on G2:
//   UnmarshalBinary(pk) , UnmarshalBinary(sig) , H(msg) , e(H(m), pk) == e(sig, G2 generator)
// All buffers are DEVICE pointers; scratch comes from the context arena.
int b2k_bls12381_verify_g1sig_dev(b2k_ctx* ctx, size_t n, const void* d_pks96, const void* d_msgs, const void* d_offsets,
                                  const void* d_dst, uint32_t dst_len, const void* d_sigs48, void* d_ok) {
  if (!ctx || !d_pks96 || !d_msgs || !d_offsets || !d_dst || !d_sigs48 || !d_ok || n == 0 || dst_len == 0 || dst_len > 255)
    return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  int rc = arena_reserve(ctx, n * (192 + 96 + 96 + 3) + 8192);
  if (rc) return rc;
  uint8_t* pk = arena_take<uint8_t>(ctx, n * 192);
  uint8_t* sg = arena_take<uint8_t>(ctx, n * 96);
  uint8_t* hm = arena_take<uint8_t>(ctx, n * 96);
  uint8_t* ok1 = arena_take<uint8_t>(ctx, n);
  uint8_t* ok2 = arena_take<uint8_t>(ctx, n);
  uint8_t* okc = arena_take<uint8_t>(ctx, n);
  uint8_t* gen = arena_take<uint8_t>(ctx, 192);
  cudaStream_t st = ctx->stream;
  k_write_g2_generator<<<1, 32, 0, st>>>(gen);
  k_g2_decompress_v<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(n, (const uint8_t*)d_pks96, pk, ok1);
  k_g1_decompress_v<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(n, (const uint8_t*)d_sigs48, sg, ok2);
  k_and_flags<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, ok1, ok2, okc);
  k_hash_to_g1<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(n, (const uint8_t*)d_msgs, (const uint32_t*)d_offsets,
                                                          (const uint8_t*)d_dst, dst_len, hm);
  b2k_internal_launch_pairing_check(ctx, n, hm, pk, sg, gen, (uint8_t*)d_ok, 1, okc);
  CK(cudaGetLastError());
  ctx->launches += 6;
  return B2K_OK;
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
  if (!ctx || !msgs || !offsets || !dst || !out || n == 0 || dst_len == 0 || dst_len > 255) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  if (check_offsets(ctx, n, offsets)) return B2K_ERR_ARG;
  size_t mbytes = offsets[n];
  int rc = arena_reserve(ctx, mbytes + (n + 1) * 4 + 256 + n * 192 + 4096);
  if (rc) return rc;
  uint8_t* dm = arena_take<uint8_t>(ctx, mbytes + 1);
  uint32_t* doff = arena_take<uint32_t>(ctx, n + 1);
  uint8_t* dd = arena_take<uint8_t>(ctx, 256);
  uint8_t* dout = arena_take<uint8_t>(ctx, n * 192);
  if (mbytes) CK(cudaMemcpyAsync(dm, msgs, mbytes, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(doff, offsets, (n + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(dd, dst, dst_len, cudaMemcpyHostToDevice, ctx->stream));
  rc = b2k_bls12381_hash_to_g2_dev(ctx, n, dm, doff, dd, dst_len, dout);
  if (rc) return rc;
  CK(cudaMemcpyAsync(out, dout, n * 192, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return B2K_OK;
}

// ok[i] = bls.Verify for the scheme with signatures on G2 / keys on G1 (bls.NewSchemeOnG2, sign/bls/bls.go:48-59):
//   UnmarshalBinary(pk in G1), UnmarshalBinary(sig in G2), H(msg) in G2, e(G1 base, sig) == e(pk, H(m))
int b2k_bls12381_verify_g2sig_dev(b2k_ctx* ctx, size_t n, const void* d_pks48, const void* d_msgs, const void* d_offsets,
                                  const void* d_dst, uint32_t dst_len, const void* d_sigs96, void* d_ok) {
  if (!ctx || !d_pks48 || !d_msgs || !d_offsets || !d_dst || !d_sigs96 || !d_ok || n == 0 || dst_len == 0 || dst_len > 255)
    return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  int rc = arena_reserve(ctx, n * (96 + 192 + 192 + 3) + 8192);
  if (rc) return rc;
  uint8_t* pk = arena_take<uint8_t>(ctx, n * 96);
  uint8_t* sg = arena_take<uint8_t>(ctx, n * 192);
  uint8_t* hm = arena_take<uint8_t>(ctx, n * 192);
  uint8_t* ok1 = arena_take<uint8_t>(ctx, n);
  uint8_t* ok2 = arena_take<uint8_t>(ctx, n);
  uint8_t* okc = arena_take<uint8_t>(ctx, n);
  uint8_t* gen = arena_take<uint8_t>(ctx, 96);
  cudaStream_t st = ctx->stream;
  k_write_g1_generator<<<1, 32, 0, st>>>(gen);
  k_g1_decompress_v<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(n, (const uint8_t*)d_pks48, pk, ok1);
  k_g2_decompress_v<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(n, (const uint8_t*)d_sigs96, sg, ok2);
  k_and_flags<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, ok1, ok2, okc);
  k_hash_to_g2<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(n, (const uint8_t*)d_msgs, (const uint32_t*)d_offsets,
                                                        (const uint8_t*)d_dst, dst_len, hm);
  // e(pk, H(m)) == e(base, sig): a = (pk, hm), b = (base [shared], sig)
  b2k_internal_launch_pairing_check(ctx, n, pk, hm, gen, sg, (uint8_t*)d_ok, 2, okc);
  CK(cudaGetLastError());
  ctx->launches += 6;
  return B2K_OK;
}

int b2k_bls12381_verify_g2sig(b2k_ctx* ctx, size_t n, const uint8_t* pks48, const uint8_t* msgs, const uint32_t* offsets,
                              const uint8_t* dst, uint32_t dst_len, const uint8_t* sigs96, uint8_t* ok) {
  if (!ctx || !pks48 || !msgs || !offsets || !dst || !sigs96 || !ok || n == 0 || dst_len == 0 || dst_len > 255) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  size_t mbytes = offsets[n];
  uint8_t* blob = nullptr;
  size_t o_pk = 0, o_sig = o_pk + n * 48, o_msg = o_sig + n * 96, o_off = (o_msg + mbytes + 15) & ~size_t(15),
         o_dst = o_off + (n + 1) * 4, o_ok = o_dst + 256, total = o_ok + n;
  if (check_offsets(ctx, n, offsets)) return B2K_ERR_ARG;
  blob = (uint8_t*)b2k_arena_in(ctx, total);        // the context's input arena (no cudaMalloc / cudaFree per call: both synchronise the device)
  if (!blob) { ctx->err = "out of device memory"; return B2K_ERR_CUDA; }
  cudaStream_t st = ctx->stream;
  int rc = B2K_OK;
  do {
    if (cudaMemcpyAsync(blob + o_pk, pks48, n * 48, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(blob + o_sig, sigs96, n * 96, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        (mbytes && cudaMemcpyAsync(blob + o_msg, msgs, mbytes, cudaMemcpyHostToDevice, st) != cudaSuccess) ||
        cudaMemcpyAsync(blob + o_off, offsets, (n + 1) * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(blob + o_dst, dst, dst_len, cudaMemcpyHostToDevice, st) != cudaSuccess) { rc = B2K_ERR_CUDA; break; }
    rc = b2k_bls12381_verify_g2sig_dev(ctx, n, blob + o_pk, blob + o_msg, blob + o_off, blob + o_dst, dst_len,
                                       blob + o_sig, blob + o_ok);
    if (rc) break;
    if (cudaMemcpyAsync(ok, blob + o_ok, n, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) rc = B2K_ERR_CUDA;
  } while (0);
  cudaStreamSynchronize(st);
  if (rc == B2K_ERR_CUDA) ctx->err = "CUDA failure in verify_g2sig";
  return rc;
}

int b2k_bls12381_verify_g1sig(b2k_ctx* ctx, size_t n, const uint8_t* pks96, const uint8_t* msgs, const uint32_t* offsets,
                              const uint8_t* dst, uint32_t dst_len, const uint8_t* sigs48, uint8_t* ok) {
  if (!ctx || !pks96 || !msgs || !offsets || !dst || !sigs48 || !ok || n == 0 || dst_len == 0 || dst_len > 255) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  size_t mbytes = offsets[n];
  // inputs live in a separate allocation because verify_dev re-reserves the arena
  uint8_t* blob = nullptr;
  size_t o_pk = 0, o_sig = o_pk + n * 96, o_msg = o_sig + n * 48, o_off = (o_msg + mbytes + 15) & ~size_t(15),
         o_dst = o_off + (n + 1) * 4, o_ok = o_dst + 256, total = o_ok + n;
  if (check_offsets(ctx, n, offsets)) return B2K_ERR_ARG;
  blob = (uint8_t*)b2k_arena_in(ctx, total);        // the context's input arena (no cudaMalloc / cudaFree per call: both synchronise the device)
  if (!blob) { ctx->err = "out of device memory"; return B2K_ERR_CUDA; }
  cudaStream_t st = ctx->stream;
  int rc = B2K_OK;
  do {
    if (cudaMemcpyAsync(blob + o_pk, pks96, n * 96, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(blob + o_sig, sigs48, n * 48, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        (mbytes && cudaMemcpyAsync(blob + o_msg, msgs, mbytes, cudaMemcpyHostToDevice, st) != cudaSuccess) ||
        cudaMemcpyAsync(blob + o_off, offsets, (n + 1) * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(blob + o_dst, dst, dst_len, cudaMemcpyHostToDevice, st) != cudaSuccess) { rc = B2K_ERR_CUDA; break; }
    rc = b2k_bls12381_verify_g1sig_dev(ctx, n, blob + o_pk, blob + o_msg, blob + o_off, blob + o_dst, dst_len,
                                       blob + o_sig, blob + o_ok);
    if (rc) break;
    if (cudaMemcpyAsync(ok, blob + o_ok, n, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) rc = B2K_ERR_CUDA;
  } while (0);
  cudaStreamSynchronize(st);
  if (rc == B2K_ERR_CUDA) ctx->err = "CUDA failure in verify_g1sig";
  return rc;
}

}  // extern "C"
