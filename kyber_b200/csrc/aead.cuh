// aead.cuh -- the symmetric half of ECIES (encrypt/ecies/ecies.go:114-131 and the AEAD it opens), per thread, in constant time:
// HKDF-SHA256 to 44 bytes (key || nonce), AES-256 without tables, and GCM with a mask-only GHASH.  Shared by ECIES on
// edwards25519 (ecies.cuh) and on BLS12-381 (ecies_bls.cuh); it includes no curve code.
//
// Replaces (reference):
//   deriveKey                 ecies.go:114-131 (hkdf.New(sha256, dh.MarshalBinary(), nil, nil), 44 bytes) -> hkdf_sha256_44
//   crypto/aes + cipher.NewGCM (AES-256, 12-byte nonce, 16-byte tag, no AAD)                -> aes256_*, gcm_*
//
// Secret here: the ikm (the encoded DH point), the HKDF output, the AES round keys and state, the GHASH key H and the
// plaintext.  No branch and no memory address depends on them:
//   - AES: no tables.  SubBytes is a bitsliced circuit over eight 32-bit bit planes holding two blocks: the inversion in
//     GF(2^8) as x^254 (11 products of bit planes), then the affine map.  The key schedule's SubWord runs through the same circuit.
//   - GHASH: a carry-less product with masks, 128 steps whatever the operands.  The tag comparison ORs the XORs of all 16 bytes
//     and the outcome masks the plaintext.
// What does branch is public: lengths and loop counts.
#pragma once
#include "sha256.cuh"

#ifdef B2K_ECIES_COUNT
// host emulation only: how many times each constant-time helper ran (tests/test_ecies_emulation.py,
// tests/test_ecies_bls12381_emulation.py: the counts must not depend on the key, r, the point or the message bytes).  The
// array is defined by the emulation, with as many slots as the counters its curve uses (ECIES_CNT_* here and in ecies_bls.cuh).
extern uint64_t ecies_counts[];
#define ECIES_TICK(k) (ecies_counts[k]++)
#else
#define ECIES_TICK(k) ((void)0)
#endif

namespace b2k {

enum { ECIES_OK = 0, ECIES_POINT = 1, ECIES_AUTH = 2 };   // B2K_ECIES_* of include/b2kyber.h
enum { ECIES_CNT_SELECT = 0, ECIES_CNT_WINDOW = 1, ECIES_CNT_SBOX = 2, ECIES_CNT_GHASH = 3 };

// ---- masks -------------------------------------------------------------------------------------------------------------------
B2K_D uint32_t ct_eq_mask(uint32_t a, uint32_t b) {       // ~0 if a == b else 0
  const uint32_t x = a ^ b;
  return ((x | (0u - x)) >> 31) - 1u;
}

// ---- HKDF-SHA256 (RFC 5869), salt nil, info nil, 44 bytes ------------------------------------------------------------------
// k44 = HKDF(ikm[0:ikm_len]) [0:44]: 32 bytes of edwards25519 dh, 48 of BLS12-381 G1, 96 of G2
B2K_NI void hkdf_sha256_44(uint8_t* k44, const uint8_t* ikm, uint32_t ikm_len) {
  uint8_t prk[32], t1[32], t2[32];
  const uint8_t zeros[32] = {}, one = 1, two = 2;
  hmac_sha256(prk, zeros, 32, ikm, ikm_len, nullptr, 0, nullptr, 0);  // Extract: salt nil = 32 zero bytes
  hmac_sha256(t1, prk, 32, &one, 1, nullptr, 0, nullptr, 0);          // T1 = HMAC(PRK, 0x01)
  hmac_sha256(t2, prk, 32, t1, 32, &two, 1, nullptr, 0);              // T2 = HMAC(PRK, T1 || 0x02)
  for (int i = 0; i < 32; i++) k44[i] = t1[i];
  for (int i = 0; i < 12; i++) k44[32 + i] = t2[i];
}

// the edwards25519 form: a 32-byte dh
B2K_D void ecies_kdf(uint8_t* k44, const uint8_t* dh) { hkdf_sha256_44(k44, dh, 32); }

// ---- AES-256 (FIPS-197) -------------------------------------------------------------------------------------------------------
// r = a b in GF(2^8) = GF(2)[x] / (x^8 + x^4 + x^3 + x + 1), on bit planes (plane i = bit i of 32 bytes)
B2K_D void gf8_mul_planes(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  uint32_t c[15];
#pragma unroll
  for (int k = 0; k < 15; k++) c[k] = 0;
#pragma unroll
  for (int i = 0; i < 8; i++)
#pragma unroll
    for (int j = 0; j < 8; j++) c[i + j] ^= a[i] & b[j];
#pragma unroll
  for (int k = 14; k >= 8; k--) { c[k - 4] ^= c[k]; c[k - 5] ^= c[k]; c[k - 7] ^= c[k]; c[k - 8] ^= c[k]; }
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = c[i];
}

// the S-box on 32 bytes at once: x^254 (0 -> 0) as x^2, x^3, x^6, x^12, x^15, x^240, x^252, x^254, then the affine map
B2K_NI void aes_sbox_planes(uint32_t* s) {
  ECIES_TICK(ECIES_CNT_SBOX);
  uint32_t x2[8], x3[8], x12[8], x15[8], t[8];
  gf8_mul_planes(x2, s, s);
  gf8_mul_planes(x3, x2, s);
  gf8_mul_planes(t, x3, x3);                                   // x^6
  gf8_mul_planes(x12, t, t);
  gf8_mul_planes(x15, x12, x3);
  gf8_mul_planes(t, x15, x15);                                 // x^30
  gf8_mul_planes(t, t, t);                                     // x^60
  gf8_mul_planes(t, t, t);                                     // x^120
  gf8_mul_planes(t, t, t);                                     // x^240
  gf8_mul_planes(t, t, x12);                                   // x^252
  gf8_mul_planes(t, t, x2);                                    // x^254
#pragma unroll
  for (int i = 0; i < 8; i++)
    s[i] = t[i] ^ t[(i + 4) & 7] ^ t[(i + 5) & 7] ^ t[(i + 6) & 7] ^ t[(i + 7) & 7] ^ (((0x63u >> i) & 1u) ? 0xffffffffu : 0u);
}

// SubBytes of 32 bytes (two blocks): transpose to bit planes, the circuit, transpose back
B2K_NI void aes_subbytes32(uint8_t* b) {
  uint32_t pl[8];
#pragma unroll
  for (int i = 0; i < 8; i++) {
    uint32_t w = 0;
#pragma unroll
    for (int k = 0; k < 32; k++) w |= (uint32_t)((b[k] >> i) & 1) << k;
    pl[i] = w;
  }
  aes_sbox_planes(pl);
#pragma unroll
  for (int k = 0; k < 32; k++) {
    uint32_t v = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) v |= ((pl[i] >> k) & 1u) << i;
    b[k] = (uint8_t)v;
  }
}

// the 15 round keys (240 bytes) of a 32-byte key
B2K_NI void aes256_expand(uint8_t* rk, const uint8_t* key) {
  for (int i = 0; i < 32; i++) rk[i] = key[i];
  uint8_t rcon = 1;
  for (int i = 8; i < 60; i++) {
    uint8_t t[32] = {};
    for (int q = 0; q < 4; q++) t[q] = rk[4 * (i - 1) + q];
    if ((i & 7) == 0) {
      const uint8_t t0 = t[0];
      t[0] = t[1]; t[1] = t[2]; t[2] = t[3]; t[3] = t0;      // RotWord
      aes_subbytes32(t);
      t[0] ^= rcon;
      rcon = (uint8_t)(rcon << 1);
    } else if ((i & 7) == 4) {
      aes_subbytes32(t);
    }
    for (int q = 0; q < 4; q++) rk[4 * i + q] = rk[4 * (i - 8) + q] ^ t[q];
  }
}

B2K_D uint8_t aes_xtime(uint8_t b) { return (uint8_t)((b << 1) ^ (0x1b & (0u - (uint32_t)(b >> 7)))); }

// two blocks (b[0..15], b[16..31]) encrypted in place
B2K_NI void aes256_encrypt2(uint8_t* b, const uint8_t* rk) {
#pragma unroll
  for (int i = 0; i < 32; i++) b[i] ^= rk[i & 15];
  for (int r = 1; r <= 14; r++) {
    aes_subbytes32(b);
#pragma unroll
    for (int h = 0; h < 32; h += 16) {
      uint8_t s[16];
#pragma unroll
      for (int c = 0; c < 4; c++)
#pragma unroll
        for (int q = 0; q < 4; q++) s[q + 4 * c] = b[h + q + 4 * ((c + q) & 3)];      // ShiftRows
      if (r != 14) {
#pragma unroll
        for (int c = 0; c < 4; c++) {                                                  // MixColumns
          const uint8_t a0 = s[4 * c], a1 = s[4 * c + 1], a2 = s[4 * c + 2], a3 = s[4 * c + 3], x = a0 ^ a1 ^ a2 ^ a3;
          s[4 * c] = a0 ^ x ^ aes_xtime(a0 ^ a1);
          s[4 * c + 1] = a1 ^ x ^ aes_xtime(a1 ^ a2);
          s[4 * c + 2] = a2 ^ x ^ aes_xtime(a2 ^ a3);
          s[4 * c + 3] = a3 ^ x ^ aes_xtime(a3 ^ a0);
        }
      }
#pragma unroll
      for (int i = 0; i < 16; i++) b[h + i] = s[i] ^ rk[16 * r + i];
    }
  }
}

// ---- GCM (SP 800-38D) -----------------------------------------------------------------------------------------------------
struct Ghash { uint64_t hh, hl, xh, xl; };                  // H and the running X, as big-endian 128-bit halves

B2K_D uint64_t load_be64(const uint8_t* p) {
  uint64_t v = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) v = (v << 8) | p[i];
  return v;
}

B2K_D void store_be64(uint8_t* p, uint64_t v) {
#pragma unroll
  for (int i = 0; i < 8; i++) p[i] = (uint8_t)(v >> (56 - 8 * i));
}

// X = (X ^ blk) H: the bit-serial product of SP 800-38D Algorithm 1 with masks in place of both conditions
B2K_NI void ghash_block(Ghash& g, const uint8_t* blk) {
  ECIES_TICK(ECIES_CNT_GHASH);
  const uint64_t xh = g.xh ^ load_be64(blk), xl = g.xl ^ load_be64(blk + 8);
  uint64_t zh = 0, zl = 0, vh = g.hh, vl = g.hl;
  for (int i = 0; i < 128; i++) {
    const uint64_t bit = i < 64 ? (xh >> (63 - i)) & 1 : (xl >> (127 - i)) & 1, m = 0 - bit;
    zh ^= vh & m; zl ^= vl & m;
    const uint64_t lsb = 0 - (vl & 1);
    vl = (vl >> 1) | (vh << 63);
    vh = (vh >> 1) ^ (0xe100000000000000ull & lsb);
  }
  g.xh = zh; g.xl = zl;
}

// GHASH over len bytes, the last partial block zero-padded
B2K_D void ghash_bytes(Ghash& g, const uint8_t* p, uint32_t len) {
  for (uint32_t o = 0; o < len; o += 16) {
    uint8_t blk[16];
    for (int i = 0; i < 16; i++) blk[i] = o + i < len ? p[o + i] : 0;
    ghash_block(g, blk);
  }
}

// out[i] = (in[i] ^ keystream[i]) & mask, keystream = E(nonce || ctr) for ctr = 2, 3, ... (inc32 of J0), two blocks per call
B2K_D void gcm_ctr(const uint8_t* rk, const uint8_t* nonce, const uint8_t* in, uint8_t* out, uint32_t len, uint8_t mask) {
  for (uint32_t o = 0; o < len; o += 32) {
    uint8_t ks[32];
    const uint32_t ctr = 2 + o / 16;
    for (int h = 0; h < 2; h++) {
      for (int i = 0; i < 12; i++) ks[16 * h + i] = nonce[i];
      const uint32_t c = ctr + h;
      ks[16 * h + 12] = (uint8_t)(c >> 24); ks[16 * h + 13] = (uint8_t)(c >> 16);
      ks[16 * h + 14] = (uint8_t)(c >> 8); ks[16 * h + 15] = (uint8_t)c;
    }
    aes256_encrypt2(ks, rk);
    for (uint32_t i = 0; i < 32 && o + i < len; i++) out[o + i] = (uint8_t)((in[o + i] ^ ks[i]) & mask);
  }
}

// the round keys of k44[0:32], H = E(0^128) and E(J0), J0 = k44[32:44] || 0^31 || 1
B2K_D void gcm_setup(uint8_t* rk, Ghash& g, uint8_t* ej0, const uint8_t* k44) {
  aes256_expand(rk, k44);
  uint8_t b[32] = {};
  for (int i = 0; i < 12; i++) b[16 + i] = k44[32 + i];
  b[31] = 1;
  aes256_encrypt2(b, rk);
  g.hh = load_be64(b); g.hl = load_be64(b + 8); g.xh = 0; g.xl = 0;
  for (int i = 0; i < 16; i++) ej0[i] = b[16 + i];
}

// tag = E(J0) ^ GHASH(C || len block), no AAD
B2K_D void gcm_tag(uint8_t* tag, Ghash& g, const uint8_t* ej0, const uint8_t* c, uint32_t len) {
  ghash_bytes(g, c, len);
  uint8_t lb[16];
  store_be64(lb, 0);
  store_be64(lb + 8, (uint64_t)len * 8);
  ghash_block(g, lb);
  uint8_t s[16];
  store_be64(s, g.xh); store_be64(s + 8, g.xl);
  for (int i = 0; i < 16; i++) tag[i] = s[i] ^ ej0[i];
}

// Seal: out = C || tag (len + 16 bytes)
B2K_NI void gcm_seal(const uint8_t* k44, const uint8_t* msg, uint32_t len, uint8_t* out) {
  uint8_t rk[240], ej0[16];
  Ghash g;
  gcm_setup(rk, g, ej0, k44);
  gcm_ctr(rk, k44 + 32, msg, out, len, 0xff);
  gcm_tag(out + len, g, ej0, out, len);
}

// Open of ct = C || tag (clen >= 16 bytes): msg = the plaintext if the tag matches, zeros otherwise; true iff it matched
B2K_NI bool gcm_open(const uint8_t* k44, const uint8_t* ct, uint32_t clen, uint8_t* msg) {
  uint8_t rk[240], ej0[16], tag[16];
  Ghash g;
  const uint32_t len = clen - 16;
  gcm_setup(rk, g, ej0, k44);
  gcm_tag(tag, g, ej0, ct, len);
  uint32_t diff = 0;
  for (int i = 0; i < 16; i++) diff |= (uint32_t)(tag[i] ^ ct[len + i]);
  const uint32_t ok = ct_eq_mask(diff, 0);
  gcm_ctr(rk, k44 + 32, ct, msg, len, (uint8_t)ok);
  return ok != 0;
}

}  // namespace b2k
