// b2k_shuffle.cu -- C ABI entry points for Neff's shuffle verifier on edwards25519 (shuffle.cuh, shuffle_transcript.h):
//   b2k_ed25519_shuffle_verify                proof.HashVerify(suite, proto, shuffle.Verifier(...), proof) for m shuffles
//                                             (proof/hash.go:168-175, shuffle/pair.go:239-312, shuffle/simple.go:186-254)
//   b2k_ed25519_shuffle_sequence_verifiable   shuffle.GetSequenceVerifiable, shuffle/sequences.go:155-190
// Stages of the verifier, one kernel each (tools/perf_shuffle.py times them by name): decode every point once; U, W per shuffle;
// one thread per thver; one thread per i for (33) and the Phi terms with a per-block sum; per shuffle the sum of the block
// partials, (34), (35) and the status.  The transcript runs on host threads while the decode runs on the device.
#include "host_call.cuh"
#include "shuffle_transcript.h"
using namespace b2k_host;

namespace b2k {

constexpr int SHUF_BS = 128;                                // threads per block of the per-i kernels

// every point of the batch, decoded once: proof items pp[m][12k + 3] (scalar items untouched), inputs ip[4][m][k] (X, Y, Xbar,
// Ybar), bases gh[2][m] (G, H; g or h null = the base point).  A point that does not decode flags its shuffle.
__global__ void __launch_bounds__(256) k_shuffle_decode(uint32_t m, uint32_t k, const uint8_t* __restrict__ proofs,
                                                        const uint8_t* __restrict__ in4, const uint8_t* __restrict__ g,
                                                        const uint8_t* __restrict__ h, EdAff* __restrict__ pp,
                                                        EdAff* __restrict__ ip, EdAff* __restrict__ gh, uint8_t* __restrict__ flags) {
  const uint64_t id = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t nitem = ShufItems::total(k), np = (uint64_t)m * nitem, ni = 4ull * m * k;
  uint32_t s;
  bool ok;
  if (id < np) {
    s = (uint32_t)(id / nitem);
    if (!ShufItems::is_point(k, id % nitem)) return;
    ok = ed_decode_aff(pp[id], proofs + 32 * id);
  } else if (id < np + ni) {
    const uint64_t j = id - np;
    s = (uint32_t)((j % ((uint64_t)m * k)) / k);
    ok = ed_decode_aff(ip[j], in4 + 32 * j);
  } else if (id < np + ni + 2ull * m) {
    const uint32_t j = (uint32_t)(id - np - ni), which = j / m;
    s = j % m;
    const uint8_t* src = which ? h : g;
    uint8_t base[32];
    if (!src) ed_base_bytes(base);
    ok = ed_decode_aff(gh[j], src ? src + 32 * (size_t)s : base);
  } else {
    return;
  }
  if (!ok) flags[4 * (size_t)s + SHUF_F_POINT] = 1;
}

// uw[s] = -t G, uw[m + s] = -t Gamma (SimpleShuffle.Verify step 5)
__global__ void __launch_bounds__(SHUF_BS) k_shuffle_uw(uint32_t m, uint32_t k, const EdAff* __restrict__ pp,
                                                        const EdAff* __restrict__ gh, const uint8_t* __restrict__ tc,
                                                        EdExt* __restrict__ uw) {
  const uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= 2 * m) return;
  const uint32_t s = id % m;
  uint32_t t[8], nt[8];
  sc_load_le(t, tc + 64 * (size_t)s);
  sc_neg_mod_l(nt, t);
  EdExt B;
  ed_from_aff(B, id < m ? gh[s] : pp[(size_t)s * ShufItems::total(k)]);
  ed_mul_var(uw[id], nt, B);
}

// one thread per thver: 2k per shuffle
__global__ void __launch_bounds__(SHUF_BS) k_shuffle_thver(uint32_t m, uint32_t k, const uint8_t* __restrict__ proofs,
                                                           const EdAff* __restrict__ pp, const EdAff* __restrict__ gh,
                                                           const EdExt* __restrict__ uw, const uint8_t* __restrict__ tc,
                                                           uint8_t* __restrict__ flags) {
  const uint64_t id = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= 2ull * m * k) return;
  const uint32_t s = (uint32_t)(id / (2ull * k)), i = (uint32_t)(id % (2ull * k));
  if (flags[4 * (size_t)s + SHUF_F_POINT]) return;
  const uint64_t nitem = ShufItems::total(k);
  uint32_t c[8];
  sc_load_le(c, tc + 64 * (size_t)s + 32);
  if (!shuffle_thver_i(k, i, pp + s * nitem, proofs + 32 * s * nitem, uw[s], uw[m + s], gh[s], c))
    flags[4 * (size_t)s + SHUF_F_SIMPLE] = 1;
}

// the sum of the block's points v[0..blockDim) (shared memory), left in v[0]
__device__ void ed_block_sum(EdExt* v) {
  for (unsigned w = blockDim.x / 2; w > 0; w >>= 1) {
    __syncthreads();
    if (threadIdx.x < w) ed_add(v[threadIdx.x], v[threadIdx.x], v[threadIdx.x + w]);
  }
  __syncthreads();
}

// block b covers i in [SHUF_BS c, SHUF_BS (c + 1)) of shuffle s = b / nchunk, c = b % nchunk: check (33) for each i, and the
// block's sums of the Phi1 / Phi2 terms into part[s][0 / 1][c]
__global__ void __launch_bounds__(SHUF_BS) k_shuffle_pair_terms(uint32_t m, uint32_t k, uint32_t nchunk,
                                                                const uint8_t* __restrict__ proofs, const EdAff* __restrict__ pp,
                                                                const EdAff* __restrict__ ip, const uint8_t* __restrict__ zrho,
                                                                uint8_t* __restrict__ flags, EdExt* __restrict__ part) {
  __shared__ EdExt sum[SHUF_BS];
  const uint32_t s = blockIdx.x / nchunk, c = blockIdx.x % nchunk, i = c * SHUF_BS + threadIdx.x;
  const uint64_t nitem = ShufItems::total(k), mk = (uint64_t)m * k, si = (uint64_t)s * k + i;
  EdExt t1, t2;
  ed_set_identity(t1);
  ed_set_identity(t2);
  if (i < k && !flags[4 * (size_t)s + SHUF_F_POINT]) {
    const EdAff* p = pp + s * nitem;
    const uint8_t* proof = proofs + 32 * s * nitem;
    if (!shuffle_check33(k, i, p, proof)) flags[4 * (size_t)s + SHUF_F_PAIR] = 1;
    uint32_t zs[8], zr[8];
    sc_load_le(zs, proof + 32 * ShufItems::zsigma(k, i));
    sc_load_le(zr, zrho + 32 * si);
    shuffle_phi_terms(t1, t2, zs, zr, ip[si], ip[mk + si], ip[2 * mk + si], ip[3 * mk + si]);
  }
  for (int which = 0; which < 2; which++) {
    sum[threadIdx.x] = which ? t2 : t1;
    ed_block_sum(sum);
    if (threadIdx.x == 0) part[(2 * (size_t)s + which) * nchunk + c] = sum[0];
    __syncthreads();
  }
}

// one block per shuffle: Phi1, Phi2 from the block partials, (34) and (35), then the status (POINT > SIMPLE > PAIR)
__global__ void __launch_bounds__(SHUF_BS) k_shuffle_resolve(uint32_t m, uint32_t k, uint32_t nchunk,
                                                             const uint8_t* __restrict__ proofs, const EdAff* __restrict__ pp,
                                                             const EdAff* __restrict__ gh, const EdExt* __restrict__ part,
                                                             uint8_t* __restrict__ flags, uint8_t* __restrict__ status) {
  __shared__ EdExt sum[SHUF_BS];
  __shared__ EdExt phi[2];
  const uint32_t s = blockIdx.x;
  for (int which = 0; which < 2; which++) {
    EdExt acc;
    ed_set_identity(acc);
    for (uint32_t c = threadIdx.x; c < nchunk; c += blockDim.x) ed_add(acc, acc, part[(2 * (size_t)s + which) * nchunk + c]);
    sum[threadIdx.x] = acc;
    ed_block_sum(sum);
    if (threadIdx.x == 0) phi[which] = sum[0];
    __syncthreads();
  }
  uint8_t* f = flags + 4 * (size_t)s;
  if (threadIdx.x < 2 && !f[SHUF_F_POINT]) {                // thread 0: (34) over G, thread 1: (35) over H
    const uint64_t nitem = ShufItems::total(k);
    const EdAff* p = pp + s * nitem;
    uint32_t ztau[8];
    sc_load_le(ztau, proofs + 32 * (s * nitem + ShufItems::ztau(k)));
    const int w = threadIdx.x;
    if (!shuffle_check34(p[w ? ShufItems::lambda2(k) : ShufItems::lambda1(k)], ztau, gh[w * m + s], phi[w])) f[SHUF_F_PAIR] = 1;
  }
  __syncthreads();
  if (threadIdx.x == 0) status[s] = shuffle_status(f);
}

// GetSequenceVerifiable: decode the [4][nq][k] points; bad -> FLAG_POINT
__global__ void __launch_bounds__(256) k_shuffle_seq_decode(uint64_t n, const uint8_t* __restrict__ in4, EdAff* __restrict__ pts,
                                                            uint32_t* flags) {
  const uint64_t id = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n) return;
  if (!ed_decode_aff(pts[id], in4 + 32 * id)) atomicOr(flags, FLAG_POINT);
}

// one thread per (output o, i): out[o][i] = sum_j e[j] pts[o][j][i], canonical encoding
__global__ void __launch_bounds__(SHUF_BS) k_shuffle_seq_terms(uint32_t nq, uint32_t k, const EdAff* __restrict__ pts,
                                                               const uint8_t* __restrict__ e, uint8_t* __restrict__ out) {
  const uint64_t id = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= 4ull * k) return;
  const uint64_t o = id / k, i = id % k;
  EdExt acc;
  shuffle_sequence_term(acc, nq, pts + o * nq * k + i, k, e);
  ed_encode(out + 32 * id, acc);
}

}  // namespace b2k

namespace {

unsigned host_threads() {
  unsigned nt = std::thread::hardware_concurrency();
  return nt < 1 ? 1 : nt > 32 ? 32 : nt;
}

}  // namespace

extern "C" {

int b2k_ed25519_shuffle_verify(b2k_ctx* ctx, size_t m, size_t k, const uint8_t* g, const uint8_t* h, const uint8_t* x,
                               const uint8_t* y, const uint8_t* xbar, const uint8_t* ybar, const uint8_t* proofs,
                               const uint8_t* proto, uint32_t proto_len, uint8_t* status) {
  if (!ctx || !x || !y || !xbar || !ybar || !proofs || !status || (proto_len && !proto) || m == 0 || k < 2 ||
      m > B2K_SHUFFLE_MAX_PAIRS || k > B2K_SHUFFLE_MAX_PAIRS || m * k > B2K_SHUFFLE_MAX_PAIRS)
    return bad_arg(ctx, "bad argument");
  CK(cudaSetDevice(ctx->device));
  const size_t nitem = 12 * k + 3, mk = m * k, nchunk = (k + SHUF_BS - 1) / SHUF_BS;
  uint8_t *d_p = nullptr, *d_in = nullptr, *d_g = nullptr, *d_h = nullptr, *d_zrho = nullptr, *d_tc = nullptr, *d_fl = nullptr,
          *d_st = nullptr;
  EdAff *d_pp = nullptr, *d_ip = nullptr, *d_gh = nullptr;
  EdExt *d_uw = nullptr, *d_part = nullptr;
  int rc = arena_carve(ctx, [&](Carve& c) {
    d_p = c.take<uint8_t>(m * nitem * 32);
    d_in = c.take<uint8_t>(4 * mk * 32);
    if (g) d_g = c.take<uint8_t>(m * 32);
    if (h) d_h = c.take<uint8_t>(m * 32);
    d_zrho = c.take<uint8_t>(mk * 32);
    d_tc = c.take<uint8_t>(m * 64);
    d_fl = c.take<uint8_t>(m * 4);
    d_st = c.take<uint8_t>(m);
    d_pp = c.take<EdAff>(m * nitem);
    d_ip = c.take<EdAff>(4 * mk);
    d_gh = c.take<EdAff>(2 * m);
    d_uw = c.take<EdExt>(2 * m);
    d_part = c.take<EdExt>(2 * m * nchunk);
  });
  if (rc) return rc;
  // the transcript (host threads) runs while the inputs are staged and decoded on the device
  std::vector<uint8_t> zrho(mk * 32), tc(m * 64);
  std::thread fs([&] { b2k::shuffle_host::transcripts(m, k, proofs, proto, proto_len, zrho.data(), tc.data(), host_threads()); });
  cudaStream_t st = ctx->stream;
  auto stage = [&]() -> int {
    CK(cudaMemsetAsync(d_fl, 0, m * 4, st));
    CK(cudaMemcpyAsync(d_p, proofs, m * nitem * 32, cudaMemcpyHostToDevice, st));
    const uint8_t* in[4] = {x, y, xbar, ybar};
    for (int q = 0; q < 4; q++) CK(cudaMemcpyAsync(d_in + q * mk * 32, in[q], mk * 32, cudaMemcpyHostToDevice, st));
    if (g) CK(cudaMemcpyAsync(d_g, g, m * 32, cudaMemcpyHostToDevice, st));
    if (h) CK(cudaMemcpyAsync(d_h, h, m * 32, cudaMemcpyHostToDevice, st));
    k_shuffle_decode<<<blocks_of(m * nitem + 4 * mk + 2 * m, 256), 256, 0, st>>>((uint32_t)m, (uint32_t)k, d_p, d_in, d_g, d_h,
                                                                                 d_pp, d_ip, d_gh, d_fl);
    CK(cudaGetLastError());
    return B2K_OK;
  };
  rc = stage();
  fs.join();
  if (rc) return rc;
  CK(cudaMemcpyAsync(d_zrho, zrho.data(), mk * 32, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_tc, tc.data(), m * 64, cudaMemcpyHostToDevice, st));
  k_shuffle_uw<<<blocks_of(2 * m, SHUF_BS), SHUF_BS, 0, st>>>((uint32_t)m, (uint32_t)k, d_pp, d_gh, d_tc, d_uw);
  k_shuffle_thver<<<blocks_of(2 * mk, SHUF_BS), SHUF_BS, 0, st>>>((uint32_t)m, (uint32_t)k, d_p, d_pp, d_gh, d_uw, d_tc, d_fl);
  k_shuffle_pair_terms<<<(unsigned)(m * nchunk), SHUF_BS, 0, st>>>((uint32_t)m, (uint32_t)k, (uint32_t)nchunk, d_p, d_pp, d_ip,
                                                                    d_zrho, d_fl, d_part);
  k_shuffle_resolve<<<(unsigned)m, SHUF_BS, 0, st>>>((uint32_t)m, (uint32_t)k, (uint32_t)nchunk, d_p, d_pp, d_gh, d_part, d_fl,
                                                     d_st);
  CK(cudaGetLastError());
  ctx->launches += 5;
  CK(cudaMemcpyAsync(status, d_st, m, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return B2K_OK;
}

int b2k_ed25519_shuffle_sequence_verifiable(b2k_ctx* ctx, size_t nq, size_t k, const uint8_t* x, const uint8_t* y,
                                            const uint8_t* xbar, const uint8_t* ybar, const uint8_t* e, uint8_t* x_up,
                                            uint8_t* y_up, uint8_t* x_down, uint8_t* y_down) {
  if (!ctx || !x || !y || !xbar || !ybar || !e || !x_up || !y_up || !x_down || !y_down || nq == 0 || k == 0 ||
      nq > B2K_SHUFFLE_MAX_PAIRS || k > B2K_SHUFFLE_MAX_PAIRS || nq * k > B2K_SHUFFLE_MAX_PAIRS)
    return bad_arg(ctx, "bad argument");
  CK(cudaSetDevice(ctx->device));
  const size_t n = nq * k;
  uint8_t *d_in = nullptr, *d_e = nullptr, *d_out = nullptr;
  EdAff* d_pts = nullptr;
  int rc = arena_carve(ctx, [&](Carve& c) {
    d_in = c.take<uint8_t>(4 * n * 32);
    d_e = c.take<uint8_t>(nq * 32);
    d_out = c.take<uint8_t>(4 * k * 32);
    d_pts = c.take<EdAff>(4 * n);
  });
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  if ((rc = status_begin(ctx))) return rc;
  const uint8_t* in[4] = {x, y, xbar, ybar};
  for (int q = 0; q < 4; q++) CK(cudaMemcpyAsync(d_in + q * n * 32, in[q], n * 32, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_e, e, nq * 32, cudaMemcpyHostToDevice, st));
  k_shuffle_seq_decode<<<blocks_of(4 * n, 256), 256, 0, st>>>(4 * n, d_in, d_pts, ctx->d_flags);
  k_shuffle_seq_terms<<<blocks_of(4 * k, SHUF_BS), SHUF_BS, 0, st>>>((uint32_t)nq, (uint32_t)k, d_pts, d_e, d_out);
  CK(cudaGetLastError());
  ctx->launches += 2;
  uint8_t* outs[4] = {x_up, y_up, x_down, y_down};
  for (int q = 0; q < 4; q++) CK(cudaMemcpyAsync(outs[q], d_out + q * k * 32, k * 32, cudaMemcpyDeviceToHost, st));
  return status_finish(ctx);
}

}  // extern "C"
