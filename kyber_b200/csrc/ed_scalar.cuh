// ed_scalar.cuh -- edwards25519 scalars as 8 little-endian 32-bit limbs: the arithmetic mod l and the signed-nibble recoding
// that every variable-time multiplication (ed25519.cuh) and the constant-time ones (ecies.cuh) read scalars through.
//
// Replaces (reference):
//   scalar.IsCanonical          group/edwards25519/scalar.go:2299-2333   -> sc_is_canonical
//   scalar.SetBytes / Neg       scalar.go:187-189, :119-128 (mod l)       -> sc_reduce512, sc_neg_mod_l
//   Scalar.Equal of a challenge                                         -> pvss_challenge_is
//   the recoding of geScalarMult ge.go:443-466                           -> sc_recode4, ed_scalar_rule
#pragma once
#include "constants.cuh"

namespace b2k {

B2K_D void sc_load_le(uint32_t* s, const uint8_t* b) {
#pragma unroll
  for (int j = 0; j < 8; j++) s[j] = (uint32_t)b[4 * j] | ((uint32_t)b[4 * j + 1] << 8) | ((uint32_t)b[4 * j + 2] << 16) | ((uint32_t)b[4 * j + 3] << 24);
}

// scalar.IsCanonical: s < l as a 256-bit little-endian integer
B2K_D bool sc_is_canonical(const uint32_t* s) {
  for (int j = 7; j >= 0; j--) {
    if (s[j] != Ed25519Verify::ell(j)) return s[j] < Ed25519Verify::ell(j);
  }
  return false;
}

// Scalar.Equal(C, Pick(...)), the challenge check of PVSS and of the ring signatures: the raw 32 bytes of C against the limbs of
// the picked scalar want
B2K_D bool pvss_challenge_is(const uint8_t* c_bytes, const uint32_t* want) {
  uint32_t c[8], o = 0;
  sc_load_le(c, c_bytes);
#pragma unroll
  for (int j = 0; j < 8; j++) o |= c[j] ^ want[j];
  return o == 0;
}

// r = x mod l for a 512-bit x (16 limbs), Barrett with b = 2^32, k = 8 (HAC 14.42): q = floor(floor(x / b^7) mu / b^9),
// r = (x - q l) mod b^9, then at most two subtractions of l.
B2K_D void sc_reduce512(uint32_t* r, const uint32_t* x) {
  uint32_t q2[18];
  for (int j = 0; j < 18; j++) q2[j] = 0;
  for (int i = 0; i < 9; i++) {                         // q1 = x[7..15], q2 = q1 * mu
    uint64_t carry = 0;
    for (int j = 0; j < 9; j++) {
      const uint64_t t = (uint64_t)x[7 + i] * Ed25519Verify::mu(j) + q2[i + j] + carry;
      q2[i + j] = (uint32_t)t;
      carry = t >> 32;
    }
    q2[i + 9] = (uint32_t)carry;
  }
  uint32_t ql[9];                                       // (q3 * l) mod b^9, q3 = q2[9..17]
  for (int j = 0; j < 9; j++) ql[j] = 0;
  for (int i = 0; i < 9; i++) {
    uint64_t carry = 0;
    for (int j = 0; i + j < 9 && j < 8; j++) {
      const uint64_t t = (uint64_t)q2[9 + i] * Ed25519Verify::ell(j) + ql[i + j] + carry;
      ql[i + j] = (uint32_t)t;
      carry = t >> 32;
    }
    if (i + 8 < 9) ql[i + 8] += (uint32_t)carry;
  }
  uint32_t t[9];
  uint64_t borrow = 0;
  for (int j = 0; j < 9; j++) {                         // (x mod b^9) - (q3 l mod b^9), mod b^9
    const uint64_t d = (uint64_t)x[j] - ql[j] - borrow;
    t[j] = (uint32_t)d;
    borrow = (d >> 63) & 1;
  }
  for (int pass = 0; pass < 3; pass++) {                // t < 3 l
    bool ge = t[8] != 0;
    if (!ge) {
      ge = true;
      for (int j = 7; j >= 0; j--)
        if (t[j] != Ed25519Verify::ell(j)) { ge = t[j] > Ed25519Verify::ell(j); break; }
    }
    if (!ge) break;
    borrow = 0;
    for (int j = 0; j < 9; j++) {
      const uint64_t d = (uint64_t)t[j] - (j < 8 ? Ed25519Verify::ell(j) : 0u) - borrow;
      t[j] = (uint32_t)d;
      borrow = (d >> 63) & 1;
    }
  }
  for (int j = 0; j < 8; j++) r[j] = t[j];
}

// r = (-b) mod l, canonical, for any 256-bit b (Scalar.Neg)
B2K_D void sc_neg_mod_l(uint32_t* r, const uint32_t* b) {
  uint32_t x[16];
#pragma unroll
  for (int j = 0; j < 8; j++) { x[j] = b[j]; x[j + 8] = 0; }
  sc_reduce512(r, x);
  uint32_t o = 0;
#pragma unroll
  for (int j = 0; j < 8; j++) o |= r[j];
  if (!o) return;
  uint64_t borrow = 0;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const uint64_t d = (uint64_t)Ed25519Verify::ell(j) - r[j] - borrow;
    r[j] = (uint32_t)d;
    borrow = (d >> 63) & 1;
  }
}

// k as 64 signed base-16 digits: e[0..62] in [-8, 8), e[63] in [0, 16], k = sum e[i] 16^i.  geScalarMult adds nothing for a
// top digit above 8 (selectCached, ge.go:419-433): the multiplications apply that rule at each digit (ed_digit_add).
B2K_D void sc_recode4(int8_t* e, const uint32_t* k) {
  int carry = 0;
  for (int i = 0; i < 63; i++) {
    const int v = (int)((k[i >> 3] >> (4 * (i & 7))) & 15u) + carry;
    carry = (v + 8) >> 4;
    e[i] = (int8_t)(v - (carry << 4));
  }
  e[63] = (int8_t)((k[7] >> 28) + carry);
}

// k -> the integer geScalarMult multiplies by, modulo the group exponent 8 l.  With low = k mod 2^252 and carry the carry the
// recoding of the 63 lower nibbles leaves for the top one, e63 = (k >> 252) + carry.  Up to e63 = 8 that is k itself; above,
// the top digit is dropped and the product is (low - carry 2^252) P, replaced here by low + carry (8 l - 2^252) < 2^256, which is
// the same multiple of every point of the curve (8 l is the order of the whole group).
B2K_D void ed_scalar_rule(uint32_t* k) {
  int carry = 0;
  for (int i = 0; i < 63; i++) {
    const int v = (int)((k[i >> 3] >> (4 * (i & 7))) & 15u) + carry;
    carry = (v + 8) >> 4;
  }
  if ((int)(k[7] >> 28) + carry <= 8) return;
  k[7] &= 0x0fffffffu;
  if (!carry) return;
  uint32_t c[8];                                       // 8 l - 2^252 (l < 2^253: the shift stays in 256 bits)
#pragma unroll
  for (int j = 0; j < 8; j++) c[j] = (Ed25519Verify::ell(j) << 3) | (j ? Ed25519Verify::ell(j - 1) >> 29 : 0u);
  c[7] -= 0x10000000u;
  uint64_t s = 0;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    s += (uint64_t)k[j] + c[j];
    k[j] = (uint32_t)s;
    s >>= 32;
  }
}

}  // namespace b2k
