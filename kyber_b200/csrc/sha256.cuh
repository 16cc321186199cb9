// sha256.cuh -- SHA-256 (FIPS 180-4), streaming over byte fragments, per thread, and HMAC-SHA256 on it.  Used by hash-to-curve
// (h2c.cuh, bn_hash.cuh), by the PVSS challenges (pvss.cuh, sha256_blocks) and by ECIES's HKDF (ecies.cuh); kept apart so that the edwards25519 units do not pull in BLS12-381 code.
#pragma once
#include <stddef.h>
#include "ptx.cuh"

namespace b2k {

struct Sha256 {
  uint32_t h[8];
  uint8_t buf[64];
  uint32_t fill;
  uint64_t total;
};

B2K_D uint32_t sha_rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }

B2K_NI void sha256_compress(uint32_t* h, const uint8_t* blk) {
  const uint32_t K[64] = {
      0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01,
      0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc,
      0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147,
      0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
      0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08,
      0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
      0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
  uint32_t w[64];
  for (int i = 0; i < 16; i++)
    w[i] = ((uint32_t)blk[4 * i] << 24) | ((uint32_t)blk[4 * i + 1] << 16) | ((uint32_t)blk[4 * i + 2] << 8) | blk[4 * i + 3];
  for (int i = 16; i < 64; i++) {
    uint32_t s0 = sha_rotr(w[i - 15], 7) ^ sha_rotr(w[i - 15], 18) ^ (w[i - 15] >> 3);
    uint32_t s1 = sha_rotr(w[i - 2], 17) ^ sha_rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
    w[i] = w[i - 16] + s0 + w[i - 7] + s1;
  }
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
  for (int i = 0; i < 64; i++) {
    uint32_t S1 = sha_rotr(e, 6) ^ sha_rotr(e, 11) ^ sha_rotr(e, 25);
    uint32_t ch = (e & f) ^ (~e & g);
    uint32_t t1 = hh + S1 + ch + K[i] + w[i];
    uint32_t S0 = sha_rotr(a, 2) ^ sha_rotr(a, 13) ^ sha_rotr(a, 22);
    uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
    uint32_t t2 = S0 + mj;
    hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

B2K_D void sha256_init(Sha256& s) {
  const uint32_t iv[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
  for (int i = 0; i < 8; i++) s.h[i] = iv[i];
  s.fill = 0;
  s.total = 0;
}

B2K_D void sha256_update(Sha256& s, const uint8_t* p, uint32_t n) {
  for (uint32_t i = 0; i < n; i++) {
    s.buf[s.fill++] = p[i];
    if (s.fill == 64) { sha256_compress(s.h, s.buf); s.fill = 0; }
  }
  s.total += n;
}

B2K_D void sha256_update_zero(Sha256& s, uint32_t n) {
  for (uint32_t i = 0; i < n; i++) {
    s.buf[s.fill++] = 0;
    if (s.fill == 64) { sha256_compress(s.h, s.buf); s.fill = 0; }
  }
  s.total += n;
}

B2K_D void sha256_final(Sha256& s, uint8_t* out32) {
  uint64_t bits = s.total * 8;
  s.buf[s.fill++] = 0x80;
  if (s.fill > 56) {
    while (s.fill < 64) s.buf[s.fill++] = 0;
    sha256_compress(s.h, s.buf);
    s.fill = 0;
  }
  while (s.fill < 56) s.buf[s.fill++] = 0;
  for (int i = 0; i < 8; i++) s.buf[56 + i] = (uint8_t)(bits >> (56 - 8 * i));
  sha256_compress(s.h, s.buf);
  for (int i = 0; i < 8; i++) {
    out32[4 * i] = (uint8_t)(s.h[i] >> 24); out32[4 * i + 1] = (uint8_t)(s.h[i] >> 16);
    out32[4 * i + 2] = (uint8_t)(s.h[i] >> 8); out32[4 * i + 3] = (uint8_t)s.h[i];
  }
}

// SHA-256 of nblk whole 64-byte blocks at p; digest (big-endian bytes) in out
B2K_D void sha256_blocks(uint8_t* out, const uint8_t* p, size_t nblk) {
  Sha256 s;
  sha256_init(s);
  for (size_t k = 0; k < nblk; k++) sha256_compress(s.h, p + 64 * k);
  s.total = 64 * nblk;
  sha256_final(s, out);
}

// HMAC-SHA256 with a key of at most 64 bytes (longer keys are hashed first, RFC 2104), message given as three fragments
B2K_NI void hmac_sha256(uint8_t* out32, const uint8_t* key, uint32_t key_len, const uint8_t* m1, uint32_t n1, const uint8_t* m2,
                        uint32_t n2, const uint8_t* m3, uint32_t n3) {
  uint8_t k[64], kh[32], inner[32];
  Sha256 s;
  if (key_len > 64) {
    sha256_init(s); sha256_update(s, key, key_len); sha256_final(s, kh);
    key = kh; key_len = 32;
  }
  for (uint32_t i = 0; i < 64; i++) k[i] = (i < key_len ? key[i] : 0) ^ 0x36;
  sha256_init(s);
  sha256_update(s, k, 64);
  if (n1) sha256_update(s, m1, n1);
  if (n2) sha256_update(s, m2, n2);
  if (n3) sha256_update(s, m3, n3);
  sha256_final(s, inner);
  for (uint32_t i = 0; i < 64; i++) k[i] ^= 0x36 ^ 0x5c;
  sha256_init(s);
  sha256_update(s, k, 64);
  sha256_update(s, inner, 32);
  sha256_final(s, out32);
}

}  // namespace b2k
