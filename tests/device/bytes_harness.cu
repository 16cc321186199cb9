// bytes_harness.cu -- test-only entry points into the byte and scalar code every edwards25519 protocol reads through (sha256.cuh,
// sha512.cuh, blake2b.cuh, ed_scalar.cuh, ecies.cuh), one case per thread, 128 threads per block.  Not a library unit: the
// library headers are included unchanged.  Built by __graft_entry__.build() with the library's NVCC_FLAGS
// (libbytes_harness.so) and by g++ with -DB2K_HOST_EMUL (tests/test_bytes_emulation.py); tests/bytes_cases.py holds the case
// list and the expected values of both.
//
// Entry point (returns a cudaError_t, 0 on the host):
//   bh_run(op, n, hdr, pool, pool_len, out, out_len)
//     hdr:  n x 16 words: off[4], len[4] (four byte fragments of pool), arg[4], out_off, out_len, 0, 0
//     pool: the input bytes of every case;  out: the output bytes of every case, pre-filled by the caller (copied in and back)
// A fragment of length 0 may have any offset.  The operations and what they read and write are listed at Op below.
#include "../../kyber_b200/csrc/ecies.cuh"
#include "../../kyber_b200/csrc/sha512.cuh"
#include "../../kyber_b200/csrc/blake2b.cuh"
#include <stddef.h>
#include <utility>
#ifdef __CUDACC__
#include <cuda_runtime.h>
#endif

using namespace b2k;

namespace {

// f0..f3: the fragments, a0..a3: the arguments; every output is written to the case's output bytes in the order given
enum Op {
  SHA256_UPDATE,     // init, update(f0), update(f1), update(f2), final -> 32
  SHA256_ZERO,       // init, update_zero(a0), update(f0), update(f1), update(f2), final -> 32 (expand_message_xmd's Z_pad)
  SHA256_BLOCKS,     // sha256_blocks(f0, len0 / 64) -> 32
  HMAC_SHA256,       // hmac_sha256(key f0, f1, f2, f3) -> 32
  ECIES_KDF,         // ecies_kdf(f0[32]) -> 44
  SHA512_3,          // sha512_3(f0, f1, f2) -> the 64 digest bytes
  SHA512_CHALLENGE,  // sha512_3 -> sha512_digest_le -> sc_reduce512 -> 32 (little-endian)
  BLAKE2B,           // BLAKE2b-512 midstate: f0..f3 absorbed in order, each in chunks of a0 bytes (0: whole) -> 64
  XB_ROOT,           // blake2xb_root(f0) -> 64; blake2xb_begin(f0), blake2b_absorb(f1), blake2b_finish -> 64
  XB_BLOCK,          // blake2xb_block(root f0[64], a0) -> 64
  SC_PICK,           // sc_pick(f0) -> 32; sc_pick_root(blake2xb_root(f0)) -> 32
  SC_CANONICAL,      // sc_is_canonical(f0[32]) -> 1
  SC_REDUCE512,      // sc_reduce512(f0[64]) -> 32
  SC_NEG,            // sc_neg_mod_l(f0[32]) -> 32
  SC_RECODE4,        // sc_recode4(f0[32]) -> 64 signed digits
  SC_RULE,           // ed_scalar_rule(f0[32]) in place -> 32
  CHALLENGE_IS,      // pvss_challenge_is(f0[32], limbs of f1[32]) -> 1
  AES_SUBBYTES,      // aes_subbytes32(f0[32]) -> 32
  AES_EXPAND,        // aes256_expand(f0[32]) -> 240
  AES_ENCRYPT2,      // aes256_encrypt2(f1[32], round keys of f0[32]) -> 32
  GHASH,             // H = f0[16]: ghash_bytes(f1), then the length block of gcm_tag -> X, 16
  GCM_SEAL,          // gcm_seal(k44 f0[44], f1) -> len1 + 16
  GCM_OPEN,          // gcm_open(k44 f0[44], f1) -> the plaintext (len1 - 16), then the flag (1)
  SELECT_CACHED,     // ed_select_cached(tab = 1..8 P, P = f0 decoded, d = (int)a0) added to the identity -> 32 (ed_encode_ct)
  SELECT_NIELS,      // ed_select_niels(row a1 of ecies_base_comb, d = (int)a0) added to the identity -> 32 (ed_encode_ct)
  MUL_VAR,           // ecies_mul_var(sc_recode4(f0[32]), 1..8 P, P = f1 decoded) -> 32 (ed_encode_ct)
  MUL_BASE,          // ecies_mul_base(sc_recode4(f0[32]), ecies_base_comb) -> 32 (ed_encode_ct)
  NOPS
};
constexpr int HDR = 16;

struct Case {
  const uint8_t* f[4];
  uint32_t n[4], a[4];
  uint8_t* out;
};

B2K_D void limbs_in(uint32_t* s, const uint8_t* b, int nl) {
  for (int j = 0; j < nl; j++)
    s[j] = (uint32_t)b[4 * j] | ((uint32_t)b[4 * j + 1] << 8) | ((uint32_t)b[4 * j + 2] << 16) | ((uint32_t)b[4 * j + 3] << 24);
}
B2K_D void limbs_out(uint8_t* o, const uint32_t* s, int nl) {
  for (int i = 0; i < 4 * nl; i++) o[i] = (uint8_t)(s[i >> 2] >> (8 * (i & 3)));
}
B2K_D void words_le_out(uint8_t* o, const uint64_t* w, int nw) {
  for (int i = 0; i < 8 * nw; i++) o[i] = (uint8_t)(w[i >> 3] >> (8 * (i & 7)));
}
B2K_D void copy(uint8_t* d, const uint8_t* s, uint32_t n) {
  for (uint32_t i = 0; i < n; i++) d[i] = s[i];
}

template <int op>
B2K_D void run_case(const Case& c) {
  uint8_t* o = c.out;
  if constexpr (op == SHA256_UPDATE || op == SHA256_ZERO) {
    Sha256 s;
    sha256_init(s);
    if (op == SHA256_ZERO) sha256_update_zero(s, c.a[0]);
    sha256_update(s, c.f[0], c.n[0]);
    sha256_update(s, c.f[1], c.n[1]);
    sha256_update(s, c.f[2], c.n[2]);
    uint8_t d[32];
    sha256_final(s, d);
    copy(o, d, 32);
  } else if constexpr (op == SHA256_BLOCKS) {
    uint8_t d[32];
    sha256_blocks(d, c.f[0], c.n[0] / 64);
    copy(o, d, 32);
  } else if constexpr (op == HMAC_SHA256) {
    uint8_t d[32];
    hmac_sha256(d, c.f[0], c.n[0], c.f[1], c.n[1], c.f[2], c.n[2], c.f[3], c.n[3]);
    copy(o, d, 32);
  } else if constexpr (op == ECIES_KDF) {
    uint8_t dh[32], k44[44];
    copy(dh, c.f[0], 32);
    ecies_kdf(k44, dh);
    copy(o, k44, 44);
  } else if constexpr (op == SHA512_3 || op == SHA512_CHALLENGE) {
    uint64_t h[8];
    sha512_3(h, c.f[0], c.n[0], c.f[1], c.n[1], c.f[2], c.n[2]);
    if (op == SHA512_3) {
      for (int i = 0; i < 64; i++) o[i] = (uint8_t)(h[i >> 3] >> (56 - 8 * (i & 7)));
    } else {
      uint32_t x[16], r[8];
      sha512_digest_le(x, h);
      sc_reduce512(r, x);
      limbs_out(o, r, 8);
    }
  } else if constexpr (op == BLAKE2B) {
    Blake2bMid s;
    blake2b_init(s.h, 0x01010040u, 0, 0);                // digest 64, no key, fanout 1, depth 1
    s.t = 0;
    s.n = 0;
    for (int i = 0; i < 16; i++) s.m[i] = 0;
    for (int k = 0; k < 4; k++) {
      const uint32_t step = c.a[0] ? c.a[0] : c.n[k];
      for (uint32_t p = 0; p < c.n[k]; p += step) blake2b_absorb(s, c.f[k] + p, c.n[k] - p < step ? c.n[k] - p : step);
    }
    uint64_t d[8];
    blake2b_finish(d, s);
    words_le_out(o, d, 8);
  } else if constexpr (op == XB_ROOT) {
    uint64_t h0[8], d[8];
    blake2xb_root(h0, c.f[0], c.n[0]);
    words_le_out(o, h0, 8);
    Blake2bMid s;
    blake2xb_begin(s, c.f[0], c.n[0]);
    blake2b_absorb(s, c.f[1], c.n[1]);
    blake2b_finish(d, s);
    words_le_out(o + 64, d, 8);
  } else if constexpr (op == XB_BLOCK) {
    uint64_t h0[8], d[8];
    for (int j = 0; j < 8; j++) {
      uint64_t w = 0;
      for (int q = 7; q >= 0; q--) w = (w << 8) | c.f[0][8 * j + q];
      h0[j] = w;
    }
    blake2xb_block(d, h0, c.a[0]);
    words_le_out(o, d, 8);
  } else if constexpr (op == SC_PICK) {
    uint32_t s[8], t[8];
    uint64_t h0[8];
    sc_pick(s, c.f[0], c.n[0]);
    blake2xb_root(h0, c.f[0], c.n[0]);
    sc_pick_root(t, h0);
    limbs_out(o, s, 8);
    limbs_out(o + 32, t, 8);
  } else if constexpr (op == SC_CANONICAL) {
    uint32_t s[8];
    limbs_in(s, c.f[0], 8);
    o[0] = sc_is_canonical(s) ? 1 : 0;
  } else if constexpr (op == SC_REDUCE512) {
    uint32_t x[16], r[8];
    limbs_in(x, c.f[0], 16);
    sc_reduce512(r, x);
    limbs_out(o, r, 8);
  } else if constexpr (op == SC_NEG) {
    uint32_t s[8], r[8];
    limbs_in(s, c.f[0], 8);
    sc_neg_mod_l(r, s);
    limbs_out(o, r, 8);
  } else if constexpr (op == SC_RECODE4) {
    uint32_t s[8];
    int8_t e[64];
    limbs_in(s, c.f[0], 8);
    sc_recode4(e, s);
    for (int i = 0; i < 64; i++) o[i] = (uint8_t)e[i];
  } else if constexpr (op == SC_RULE) {
    uint32_t s[8];
    limbs_in(s, c.f[0], 8);
    ed_scalar_rule(s);
    limbs_out(o, s, 8);
  } else if constexpr (op == CHALLENGE_IS) {
    uint32_t want[8];
    limbs_in(want, c.f[1], 8);
    o[0] = pvss_challenge_is(c.f[0], want) ? 1 : 0;
  } else if constexpr (op == AES_SUBBYTES) {
    uint8_t b[32];
    copy(b, c.f[0], 32);
    aes_subbytes32(b);
    copy(o, b, 32);
  } else if constexpr (op == AES_EXPAND || op == AES_ENCRYPT2) {
    uint8_t key[32], rk[240];
    copy(key, c.f[0], 32);
    aes256_expand(rk, key);
    if (op == AES_EXPAND) {
      copy(o, rk, 240);
    } else {
      uint8_t b[32];
      copy(b, c.f[1], 32);
      aes256_encrypt2(b, rk);
      copy(o, b, 32);
    }
  } else if constexpr (op == GHASH) {
    Ghash g;
    g.hh = load_be64(c.f[0]); g.hl = load_be64(c.f[0] + 8); g.xh = 0; g.xl = 0;
    ghash_bytes(g, c.f[1], c.n[1]);
    uint8_t lb[16];
    store_be64(lb, 0);
    store_be64(lb + 8, (uint64_t)c.n[1] * 8);
    ghash_block(g, lb);
    store_be64(o, g.xh); store_be64(o + 8, g.xl);
  } else if constexpr (op == GCM_SEAL || op == GCM_OPEN) {
    uint8_t k44[44];
    copy(k44, c.f[0], 44);
    if (op == GCM_SEAL) gcm_seal(k44, c.f[1], c.n[1], o);
    else o[c.n[1] - 16] = gcm_open(k44, c.f[1], c.n[1], o) ? 1 : 0;
  } else if constexpr (op == SELECT_CACHED || op == SELECT_NIELS) {
    EdExt Q;
    ed_set_identity(Q);
    if (op == SELECT_CACHED) {
      EdExt P;
      ed_decode(P, c.f[0]);
      EdCached tab[8], s;
      ed_cached_table(tab, P);
      ed_select_cached(s, tab, (int)c.a[0]);
      ed_add_cached(Q, Q, s.ypx, s.ymx, &s.z2, s.t2d, false);
    } else {
      EdNiels s;
      ed_select_niels(s, ecies_base_comb + 8 * 24 * c.a[1], (int)c.a[0]);
      ed_add_cached(Q, Q, s.ypx, s.ymx, nullptr, s.t2d, false);
    }
    ed_encode_ct(o, Q);
  } else if constexpr (op == MUL_VAR || op == MUL_BASE) {
    uint32_t k[8];
    int8_t e[64];
    limbs_in(k, c.f[0], 8);
    sc_recode4(e, k);
    EdExt Q;
    if (op == MUL_VAR) {
      EdExt P;
      ed_decode(P, c.f[1]);
      EdCached tab[8];
      ed_cached_table(tab, P);
      ecies_mul_var(Q, e, tab);
    } else {
      ecies_mul_base(Q, e, ecies_base_comb);
    }
    ed_encode_ct(o, Q);
  }
}

B2K_D Case case_of(const uint32_t* h, const uint8_t* pool, uint8_t* out) {
  Case c;
  for (int k = 0; k < 4; k++) { c.f[k] = pool + h[k]; c.n[k] = h[4 + k]; c.a[k] = h[8 + k]; }
  c.out = out + h[12];
  return c;
}

#ifdef __CUDACC__
template <int op>
__global__ void __launch_bounds__(128) k_case(int n, const uint32_t* hdr, const uint8_t* pool, uint8_t* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  run_case<op>(case_of(hdr + (size_t)HDR * i, pool, out));
}

// H2D, one launch, D2H; every step's status is returned (the first failure wins)
template <int op>
int run_op(int n, const uint32_t* hdr, const uint8_t* pool, uint64_t pool_len, uint8_t* out, uint64_t out_len) {
  if (n <= 0) return 0;
  uint32_t* d_hdr = nullptr;
  uint8_t *d_pool = nullptr, *d_out = nullptr;
  cudaError_t e = cudaMalloc(&d_hdr, (size_t)HDR * n * 4);
  if (e == cudaSuccess) e = cudaMalloc(&d_pool, pool_len ? pool_len : 1);
  if (e == cudaSuccess) e = cudaMalloc(&d_out, out_len ? out_len : 1);
  if (e == cudaSuccess) e = cudaMemcpy(d_hdr, hdr, (size_t)HDR * n * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && pool_len) e = cudaMemcpy(d_pool, pool, pool_len, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && out_len) e = cudaMemcpy(d_out, out, out_len, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    k_case<op><<<(n + 127) / 128, 128>>>(n, d_hdr, d_pool, d_out);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e == cudaSuccess && out_len) e = cudaMemcpy(out, d_out, out_len, cudaMemcpyDeviceToHost);
  cudaFree(d_hdr);
  cudaFree(d_pool);
  cudaFree(d_out);
  return (int)e;
}
#else
template <int op>
int run_op(int n, const uint32_t* hdr, const uint8_t* pool, uint64_t, uint8_t* out, uint64_t) {
  for (int i = 0; i < n; i++) run_case<op>(case_of(hdr + (size_t)HDR * i, pool, out));
  return 0;
}
#endif

// the run-time operation code -> its instantiation; an unknown code is an error (cudaErrorInvalidValue = 1)
template <int... OPS>
int dispatch(int op, int n, const uint32_t* hdr, const uint8_t* pool, uint64_t pool_len, uint8_t* out, uint64_t out_len,
             std::integer_sequence<int, OPS...>) {
  using Fn = int (*)(int, const uint32_t*, const uint8_t*, uint64_t, uint8_t*, uint64_t);
  static constexpr Fn table[] = {run_op<OPS>...};
  if (op < 0 || op >= (int)sizeof...(OPS)) return 1;
  return table[op](n, hdr, pool, pool_len, out, out_len);
}

}  // namespace

extern "C" int bh_run(int op, int n, const uint32_t* hdr, const uint8_t* pool, uint64_t pool_len, uint8_t* out, uint64_t out_len) {
  return dispatch(op, n, hdr, pool, pool_len, out, out_len, std::make_integer_sequence<int, NOPS>{});
}
