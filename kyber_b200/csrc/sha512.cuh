// sha512.cuh -- SHA-512 (FIPS 180-4) per thread, over the concatenation of three byte strings streamed from memory: the hash of
// Ed25519 (eddsa.cuh).  sha_rotr on 64-bit words is host-callable: BLAKE2b (blake2b.cuh) uses it too.
#pragma once
#include "constants.cuh"

namespace b2k {

B2K_HD uint64_t sha_rotr(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }

// one compression of the 16 big-endian message words w (overwritten by the schedule)
B2K_D void sha512_compress(uint64_t* h, uint64_t* w) {
  uint64_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], k = h[7];
#pragma unroll
  for (int t = 0; t < 80; t++) {
    if (t >= 16) {
      const uint64_t w15 = w[(t - 15) & 15], w2 = w[(t - 2) & 15];
      w[t & 15] += (sha_rotr(w15, 1) ^ sha_rotr(w15, 8) ^ (w15 >> 7)) + w[(t - 7) & 15] +
                   (sha_rotr(w2, 19) ^ sha_rotr(w2, 61) ^ (w2 >> 6));
    }
    const uint64_t t1 = k + (sha_rotr(e, 14) ^ sha_rotr(e, 18) ^ sha_rotr(e, 41)) + ((e & f) ^ (~e & g)) + Sha512K::k(t) + w[t & 15];
    const uint64_t t2 = (sha_rotr(a, 28) ^ sha_rotr(a, 34) ^ sha_rotr(a, 39)) + ((a & b) ^ (a & c) ^ (b & c));
    k = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += k;
}

// h = SHA-512(a[0..na) || b[0..nb) || c[0..nc)) as the eight state words (the digest is their big-endian bytes).  Blocks that
// lie inside c read it directly; the others (the prefix, the tail and the padding) go through the byte selector.
B2K_D void sha512_3(uint64_t* h, const uint8_t* a, uint32_t na, const uint8_t* b, uint32_t nb, const uint8_t* c, uint32_t nc) {
#pragma unroll
  for (int j = 0; j < 8; j++) h[j] = Sha512K::iv(j);
  const uint64_t len = (uint64_t)na + nb + nc, pre = (uint64_t)na + nb;
  const uint64_t blocks = (len + 16) / 128 + 1;
  uint64_t w[16];
  for (uint64_t blk = 0; blk < blocks; blk++) {
    const uint64_t base = blk * 128;
    if (base >= pre && base + 128 <= len) {
      const uint8_t* p = c + (base - pre);
      for (int i = 0; i < 16; i++) {
        uint64_t v = 0;
        for (int j = 0; j < 8; j++) v = (v << 8) | p[8 * i + j];
        w[i] = v;
      }
    } else {
      for (int i = 0; i < 16; i++) {
        uint64_t v = 0;
        for (int j = 0; j < 8; j++) {
          const uint64_t pos = base + 8 * i + j;
          uint8_t byte;
          if (pos < na) byte = a[pos];
          else if (pos < pre) byte = b[pos - na];
          else if (pos < len) byte = c[pos - pre];
          else if (pos == len) byte = 0x80;
          else byte = 0;
          v = (v << 8) | byte;
        }
        w[i] = v;
      }
      if (blk == blocks - 1) w[15] = len << 3;          // the bit length, 128-bit big-endian (the upper word stays 0)
    }
    sha512_compress(h, w);
  }
}

// the digest read as a 512-bit little-endian integer (mod.NewIntBytes with the scalar's little-endian order): 16 limbs
B2K_D void sha512_digest_le(uint32_t* x, const uint64_t* h) {
#pragma unroll
  for (int i = 0; i < 16; i++) {
    const uint32_t w = (i & 1) ? (uint32_t)h[i >> 1] : (uint32_t)(h[i >> 1] >> 32);   // bytes 4i..4i+3 of the digest
    x[i] = (w >> 24) | ((w >> 8) & 0xff00u) | ((w << 8) & 0xff0000u) | (w << 24);
  }
}

}  // namespace b2k
