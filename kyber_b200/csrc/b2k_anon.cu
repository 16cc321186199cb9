// b2k_anon.cu -- C ABI entry point for ring signature verification on edwards25519 (anon.cuh):
//   b2k_ed25519_anon_verify   anon.Verify(suite, msg_j, ring, scope, sig_j) for m signatures over one ring and one scope
//                             (sign/anon/sig.go:192-248)
// Stages, one kernel each (tools/perf_anon.py times them by name): per signature the Tag and the H1pre midstate; the link base
// (linkable only, one thread); the comb tables of B and H; then per chunk of ANON_CHUNK ring positions the tables of the chunk's
// keys and one thread per signature walking the chunk; last the comparison with C0.  Every signature visits the ring positions
// in the same order, so all threads of a step read the same key's table.
#include "host_call.cuh"
#include "anon.cuh"
using namespace b2k_host;

namespace b2k {

constexpr int ANON_BS = 128;                                // threads per block of the per-signature kernels
constexpr uint32_t ANON_CHUNK = 128;                        // ring positions per step launch: 4 MiB of key tables

// per signature: status POINT if the Tag does not decode, else the H1pre midstate, c = C0 and (linkable) the decoded Tag and its
// canonical encoding
__global__ void __launch_bounds__(ANON_BS) k_anon_setup(uint32_t m, uint32_t n, int linkable, const uint8_t* __restrict__ msgs,
                                                        const uint32_t* __restrict__ offs, const uint8_t* __restrict__ sigs,
                                                        size_t siglen, const uint8_t* __restrict__ scope, uint32_t slen,
                                                        Blake2bMid* __restrict__ mid, uint32_t* __restrict__ cs,
                                                        EdAff* __restrict__ tag_aff, uint8_t* __restrict__ tag_bytes,
                                                        uint8_t* __restrict__ status) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const uint8_t* sig = sigs + siglen * j;
  uint8_t* tb = tag_bytes + 32 * (size_t)j;
  if (linkable) {
    EdExt T;
    if (!ed_decode(T, sig + 32 * ((size_t)n + 1))) { status[j] = ANON_POINT; return; }
    ed_encode_z1(tb, T);
    tag_aff[j].x = T.X;
    tag_aff[j].y = T.Y;
  }
  status[j] = ANON_OK;
  const uint32_t o0 = offs[j], o1 = offs[j + 1];
  Blake2bMid s;
  anon_h1pre(s, msgs + o0, o1 - o0, scope, slen, linkable ? tb : nullptr);
  mid[j] = s;
  sc_load_le(cs + 8 * (size_t)j, sig);
}

// bases[1] = the link base Point.Pick(blake2xb.New(scope)); one thread
__global__ void k_anon_link_base(const uint8_t* __restrict__ scope, uint32_t slen, uint8_t* __restrict__ bases, uint32_t* flags) {
  if (!anon_link_base(bases + 32, scope, slen)) atomicOr(flags, FLAG_POINT);   // no point in 256 tries: probability ~2^-256
}

// the comb tables of nb bases (tab[b][32][8]), one thread per (base, k); a base that does not decode flags the call
__global__ void __launch_bounds__(ANON_BS) k_anon_tables(uint32_t nb, const uint8_t* __restrict__ keys, EdCached* __restrict__ tab,
                                                         uint32_t* flags) {
  const uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= 8 * nb) return;
  const uint32_t b = id >> 3, k = (id & 7) + 1;
  EdExt P;
  if (!ed_decode(P, keys + 32 * (size_t)b)) {
    if (k == 1) atomicOr(flags, FLAG_POINT);
    return;
  }
  ed_comb_table_column(tab + (size_t)b * 8 * ANON_ROWS, k, P);
}

// ring positions [i0, i0 + cnt) of every signature: c <- H1(s_i B + c L_i [, s_i H + c Tag])
__global__ void __launch_bounds__(ANON_BS) k_anon_ring_step(uint32_t m, uint32_t i0, uint32_t cnt, int linkable,
                                                            const uint8_t* __restrict__ sigs, size_t siglen,
                                                            const EdCached* __restrict__ fixed_tab,
                                                            const EdCached* __restrict__ key_tab, const Blake2bMid* __restrict__ mid,
                                                            uint32_t* __restrict__ cs, const EdAff* __restrict__ tag_aff,
                                                            const uint8_t* __restrict__ status) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m || status[j] != ANON_OK) return;
  const Blake2bMid pre = mid[j];
  EdCached tagtab[8];
  if (linkable) {
    EdExt T;
    ed_from_aff(T, tag_aff[j]);
    ed_cached_table(tagtab, T);
  }
  uint32_t c[8];
#pragma unroll
  for (int q = 0; q < 8; q++) c[q] = cs[8 * (size_t)j + q];
  const uint8_t* sig = sigs + siglen * j;
  const EdCached* th = linkable ? fixed_tab + 8 * ANON_ROWS : nullptr;
  for (uint32_t i = 0; i < cnt; i++) {
    uint32_t s[8];
    sc_load_le(s, sig + 32 * ((size_t)i0 + i + 1));
    anon_ring_step(c, s, fixed_tab, key_tab + (size_t)i * 8 * ANON_ROWS, th, tagtab, pre);
  }
#pragma unroll
  for (int q = 0; q < 8; q++) cs[8 * (size_t)j + q] = c[q];
}

// the status (OK iff c == C0 as raw bytes) and the tag of every OK linkable signature (zero otherwise)
__global__ void __launch_bounds__(ANON_BS) k_anon_finish(uint32_t m, int linkable, const uint8_t* __restrict__ sigs, size_t siglen,
                                                         const uint32_t* __restrict__ cs, const uint8_t* __restrict__ tag_bytes,
                                                         uint8_t* __restrict__ status, uint8_t* __restrict__ tags) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  uint8_t st = status[j];
  if (st == ANON_OK && !pvss_challenge_is(sigs + siglen * j, cs + 8 * (size_t)j)) st = ANON_INVALID;
  status[j] = st;
  for (int q = 0; q < 32; q++) tags[32 * (size_t)j + q] = st == ANON_OK && linkable ? tag_bytes[32 * (size_t)j + q] : 0;
}

}  // namespace b2k

extern "C" {

int b2k_ed25519_anon_verify(b2k_ctx* ctx, size_t n, const uint8_t* ring, int linkable, const uint8_t* scope, size_t scope_len,
                            size_t m, const uint8_t* msgs, const uint32_t* offsets, const uint8_t* sigs, uint8_t* status,
                            uint8_t* tags) {
  if (!ctx || (n && !ring) || !msgs || !offsets || !sigs || !status || (linkable && scope_len && !scope) || m == 0)
    return bad_arg(ctx, "bad argument");
  if (m > B2K_ANON_MAX || n > B2K_ANON_MAX || m * (n + 2) > B2K_ANON_MAX || scope_len > B2K_ANON_MAX)
    return bad_arg(ctx, "batch too large");
  CK(cudaSetDevice(ctx->device));
  if (check_offsets(ctx, m, offsets)) return B2K_ERR_ARG;
  linkable = linkable ? 1 : 0;
  const size_t slen = linkable ? scope_len : 0, siglen = 32 * (n + 1 + linkable), mbytes = offsets[m];
  const size_t nfix = 1 + linkable, kmax = n < ANON_CHUNK ? n : ANON_CHUNK;
  uint8_t *d_sig = nullptr, *d_msg = nullptr, *d_scope = nullptr, *d_ring = nullptr, *d_fix = nullptr, *d_tagb = nullptr,
          *d_st = nullptr, *d_tags = nullptr;
  uint32_t *d_off = nullptr, *d_c = nullptr;
  Blake2bMid* d_mid = nullptr;
  EdAff* d_taga = nullptr;
  EdCached *d_ftab = nullptr, *d_ktab = nullptr;
  uint8_t base[32];
  ed_base_bytes(base);
  return host_call(ctx, [&](Carve& c) {
    d_sig = c.in(sigs, m, siglen);
    d_msg = c.in(msgs, mbytes);
    d_off = c.in(offsets, m + 1);
    d_scope = c.in(scope, slen);
    d_ring = c.in(ring, n, 32);
    d_fix = c.take<uint8_t>(64);
    c.copy_in(d_fix, base, 32);
    d_tagb = c.take<uint8_t>(m, 32);
    d_st = c.out(status, m);
    d_tags = c.take<uint8_t>(m, 32);
    if (tags) c.copy_out(tags, d_tags, 32 * m);
    d_c = c.take<uint32_t>(m, 8);
    d_mid = c.take<Blake2bMid>(m);
    d_taga = c.take<EdAff>(m);
    d_ftab = c.take<EdCached>(nfix * 8 * ANON_ROWS);
    d_ktab = c.take<EdCached>((kmax ? kmax : 1) * 8 * ANON_ROWS);
  }, [&]() -> int {
    cudaStream_t st = ctx->stream;
    const unsigned gm = blocks_of(m, ANON_BS);
    k_anon_setup<<<gm, ANON_BS, 0, st>>>((uint32_t)m, (uint32_t)n, linkable, d_msg, d_off, d_sig, siglen, d_scope, (uint32_t)slen,
                                         d_mid, d_c, d_taga, d_tagb, d_st);
    int launches = 2;
    if (n) {
      if (linkable) { k_anon_link_base<<<1, 1, 0, st>>>(d_scope, (uint32_t)slen, d_fix, ctx->d_flags); launches++; }
      k_anon_tables<<<blocks_of(8 * nfix, ANON_BS), ANON_BS, 0, st>>>((uint32_t)nfix, d_fix, d_ftab, ctx->d_flags);
      launches++;
      for (size_t i0 = 0; i0 < n; i0 += ANON_CHUNK) {
        const uint32_t cnt = (uint32_t)(n - i0 < ANON_CHUNK ? n - i0 : ANON_CHUNK);
        k_anon_tables<<<blocks_of(8 * cnt, ANON_BS), ANON_BS, 0, st>>>(cnt, d_ring + 32 * i0, d_ktab, ctx->d_flags);
        k_anon_ring_step<<<gm, ANON_BS, 0, st>>>((uint32_t)m, (uint32_t)i0, cnt, linkable, d_sig, siglen, d_ftab, d_ktab, d_mid, d_c,
                                                 d_taga, d_st);
        launches += 2;
      }
    }
    k_anon_finish<<<gm, ANON_BS, 0, st>>>((uint32_t)m, linkable, d_sig, siglen, d_c, d_tagb, d_st, d_tags);
    CK(cudaGetLastError());
    ctx->launches += launches;
    return B2K_OK;
  });
}

}  // extern "C"
