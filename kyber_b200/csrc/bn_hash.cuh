// bn_hash.cuh -- hash-to-G1 of the two in-tree BN curves, one message per thread.
//
// bn254 (replaces pointG1.Hash -> hashToPoint, pairing/bn254/point.go:208-218):
//   hashToField      point.go:220-232   expand_message_xmd with legacy Keccak-256 (rate 136), 96 bytes, 2 x (48 bytes mod p)
//   mapToPoint       point.go:234-285   Shallue-van de Woestijne map, Z = 1, constants constants.go:71-80 (derived in
//                                       tools/gen_constants.py), legendre = e^((p-1)/2), sqrt = e^((p+1)/4), sgn0 = parity
//   p0 + p1, no cofactor (h = 1).  Default DST "BN254G1_XMD:KECCAK-256_SVDW_RO_" (suite.go:43).
//   This is the per-message step of bls.Sign / bls.Verify on bn254 (sign/bls/bls.go:67-96).
// bn256 (replaces pointG1.Hash -> hashToPoint, pairing/bn256/point.go:261-312):
//   x = SHA-256(m) mod p, then try-and-increment: the first x' >= x with x'^3 + 3 a square; y = (x'^3+3)^((p+1)/4)
//   (what big.Int.ModSqrt returns for p = 3 mod 4), no sign adjustment.  Used by sign/bls and sign/bdn on bn256: the
//   byte-exact BDN fixtures of the reference hash their message with it.
// bn256 HashG1 (replaces HashG1, pairing/bn256/hash.go:10-110; base-field hash gfp.go:46-67):
//   t = HKDF-SHA256(secret = msg, salt = dst, info = "H2C" 0 1)[0:48] mod p, then the Shallue-van de Woestijne map of
//   hash.go:14-110 statement by statement (s = sqrt(-3) the reference's root; legendre = e^((p-1)/2); sqrt = e^((p+1)/4);
//   sign0 = "canonical value >= (p-1)/2", gfp.go:137-148).  Pinned by the reference's 11 KATs (hash_test.go:11-57).
#pragma once
#include "h2c.cuh"
#include "bn256.cuh"

namespace b2k {

// ---- legacy Keccak-256 (pad 0x01 ... 0x80), streaming ------------------------------------------------------------
struct Keccak256 {
  uint64_t a[25];          // lane (x, y) at a[x + 5 y]
  uint32_t fill;           // bytes absorbed into the current rate block
};

B2K_D uint64_t k_rol(uint64_t v, int n) { return (v << n) | (v >> (64 - n)); }

B2K_NI void keccak_f1600(uint64_t* a) {
  const uint64_t RC[24] = {
      0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808AULL, 0x8000000080008000ULL, 0x000000000000808BULL,
      0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL, 0x000000000000008AULL, 0x0000000000000088ULL,
      0x0000000080008009ULL, 0x000000008000000AULL, 0x000000008000808BULL, 0x800000000000008BULL, 0x8000000000008089ULL,
      0x8000000000008003ULL, 0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800AULL, 0x800000008000000AULL,
      0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};
  // rho offsets by lane index x + 5y, and the pi destination of each lane
  const int ROT[25] = {0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14};
  for (int r = 0; r < 24; r++) {
    uint64_t c[5], d[5], b[25];
    for (int x = 0; x < 5; x++) c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
    for (int x = 0; x < 5; x++) d[x] = c[(x + 4) % 5] ^ k_rol(c[(x + 1) % 5], 1);
    for (int y = 0; y < 5; y++)
      for (int x = 0; x < 5; x++) {
        const uint64_t v = a[x + 5 * y] ^ d[x];
        const int rot = ROT[x + 5 * y];
        b[y + 5 * ((2 * x + 3 * y) % 5)] = rot ? k_rol(v, rot) : v;
      }
    for (int y = 0; y < 5; y++)
      for (int x = 0; x < 5; x++) a[x + 5 * y] = b[x + 5 * y] ^ (~b[(x + 1) % 5 + 5 * y] & b[(x + 2) % 5 + 5 * y]);
    a[0] ^= RC[r];
  }
}

B2K_D void keccak_init(Keccak256& k) {
  for (int i = 0; i < 25; i++) k.a[i] = 0;
  k.fill = 0;
}
B2K_D void keccak_absorb_byte(Keccak256& k, uint8_t v) {
  k.a[k.fill >> 3] ^= (uint64_t)v << (8 * (k.fill & 7));
  if (++k.fill == 136) { keccak_f1600(k.a); k.fill = 0; }
}
B2K_D void keccak_update(Keccak256& k, const uint8_t* p, uint32_t n) {
  for (uint32_t i = 0; i < n; i++) keccak_absorb_byte(k, p[i]);
}
B2K_D void keccak_final(Keccak256& k, uint8_t* out32) {
  k.a[k.fill >> 3] ^= (uint64_t)0x01 << (8 * (k.fill & 7));
  k.a[16] ^= 0x8000000000000000ULL;                       // last byte of the 136-byte rate block
  keccak_f1600(k.a);
  for (int i = 0; i < 32; i++) out32[i] = (uint8_t)(k.a[i >> 3] >> (8 * (i & 7)));
}

// expand_message_xmd (RFC 9380 5.3.1) with Keccak-256, 96 output bytes (ell = 3)
B2K_NI void expand_message_xmd_keccak_96(uint8_t* out96, const uint8_t* msg, uint32_t msg_len, const uint8_t* dst, uint32_t dst_len) {
  Keccak256 k;
  uint8_t b0[32], bi[32];
  const uint8_t dl = (uint8_t)dst_len;
  keccak_init(k);
  keccak_f1600(k.a);                                      // Z_pad: one all-zero rate block
  keccak_update(k, msg, msg_len);
  keccak_absorb_byte(k, 0); keccak_absorb_byte(k, 96);    // I2OSP(96, 2)
  keccak_absorb_byte(k, 0);                               // I2OSP(0, 1)
  keccak_update(k, dst, dst_len);
  keccak_absorb_byte(k, dl);
  keccak_final(k, b0);
  for (int i = 1; i <= 3; i++) {
    keccak_init(k);
    for (int j = 0; j < 32; j++) keccak_absorb_byte(k, i == 1 ? b0[j] : (uint8_t)(b0[j] ^ bi[j]));
    keccak_absorb_byte(k, (uint8_t)i);
    keccak_update(k, dst, dst_len);
    keccak_absorb_byte(k, dl);
    keccak_final(k, bi);
    for (int j = 0; j < 32; j++) out96[32 * (i - 1) + j] = bi[j];
  }
}

using NFp254 = Fp<Bn254Fp>;

// 48 big-endian bytes -> element mod p in Montgomery form: (hi 2^256 + lo) R = M(M(hi, R^2), R^2) + M(lo mod p, R^2).
// lo < 2^256 < 6p is brought below p first (5 conditional subtractions): the Montgomery product keeps its running sum
// below a + p, which must fit the 8 limbs.
B2K_D void bn254_fp_from_48_bytes(NFp254& r, const uint8_t* p) {
  NFp254 hi, lo, r2, m;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const uint8_t* q = p + 16 + 4 * (7 - j);
    lo.v[j] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
    r2.v[j] = Bn254Fp::r2(j);
    m.v[j] = Bn254Fp::mod(j);
  }
  for (int k = 0; k < 5; k++) fp_sub(lo, lo, m);          // a - p, plus p back when it borrows
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const uint8_t* q = p + 4 * (3 - j);
    hi.v[j] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
    hi.v[4 + j] = 0;
  }
  fp_mul_c(hi, hi, r2);
  fp_mul_c(hi, hi, r2);
  fp_mul_c(lo, lo, r2);
  fp_add(r, hi, lo);
}

B2K_D void bn254_g(NFp254& r, const NFp254& x) {            // x^3 + 3
  NFp254 b;
#pragma unroll
  for (int j = 0; j < 8; j++) b.v[j] = Bn254Fp::curve_b(j);
  fp_sqr_c(r, x); fp_mul_c(r, r, x); fp_add(r, r, b);
}

B2K_D bool bn254_is_square_nonzero(const NFp254& a) {       // legendre(a) == 1
  NFp254 f, one;
  fp_pow_const<Bn254Fp, Bn254Fp::ExpLegendre>(f, a);
  fp_set_one(one);
  return fp_eq(f, one);
}

B2K_D uint32_t bn254_sgn0(const NFp254& a_mont) {
  NFp254 c;
  fp_from_mont(c, a_mont);
  return c.v[0] & 1u;
}

B2K_NI void bn254_map_to_point(Affine<NFp254>& out, const NFp254& u) {
  NFp254 c1, c2, c3, c4, one, tv1, tv2, tv3, tv5, tv8, x1, x2, x3, gx;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    c1.v[j] = Bn254Fp::svdw_c1(j); c2.v[j] = Bn254Fp::svdw_c2(j);
    c3.v[j] = Bn254Fp::svdw_c3(j); c4.v[j] = Bn254Fp::svdw_c4(j);
  }
  fp_set_one(one);
  fp_sqr_c(tv1, u); fp_mul_c(tv1, tv1, c1);                 // u^2 g(Z)
  fp_add(tv2, one, tv1);
  fp_sub(tv1, one, tv1);
  fp_mul_c(tv3, tv1, tv2); fp_inv(tv3, tv3);                // inv0
  fp_mul_c(tv5, u, tv1); fp_mul_c(tv5, tv5, tv3); fp_mul_c(tv5, tv5, c3);
  fp_sub(x1, c2, tv5);
  fp_add(x2, c2, tv5);
  fp_sqr_c(tv8, tv2); fp_mul_c(tv8, tv8, tv3);
  fp_sqr_c(x3, tv8); fp_mul_c(x3, c4, x3); fp_add(x3, one, x3);
  NFp254 x;
  bn254_g(gx, x1);
  if (bn254_is_square_nonzero(gx)) {
    x = x1;
  } else {
    bn254_g(gx, x2);
    if (bn254_is_square_nonzero(gx)) x = x2;
    else { x = x3; bn254_g(gx, x3); }
  }
  NFp254 y;
  fp_pow_const<Bn254Fp, Bn254Fp::ExpSqrt>(y, gx);
  if (bn254_sgn0(u) != bn254_sgn0(y)) fp_neg(y, y);
  out.x = x; out.y = y;
}

B2K_D void bn254_hash_to_g1(Affine<NFp254>& out, const uint8_t* msg, uint32_t msg_len, const uint8_t* dst, uint32_t dst_len) {
  uint8_t uni[96];
  expand_message_xmd_keccak_96(uni, msg, msg_len, dst, dst_len);
  NFp254 u0, u1;
  bn254_fp_from_48_bytes(u0, uni);
  bn254_fp_from_48_bytes(u1, uni + 48);
  Affine<NFp254> p0, p1;
  bn254_map_to_point(p0, u0);
  bn254_map_to_point(p1, u1);
  Jac<NFp254> a, b;
  jac_from_affine(a, p0);
  jac_from_affine(b, p1);
  jac_add(a, a, b);
  jac_to_affine(out, a);
}

// ---- bn256: SHA-256, reduce, try-and-increment -------------------------------------------------------------------
B2K_D void bn256_hash_to_g1(Affine<B256Fp>& out, const uint8_t* msg, uint32_t msg_len) {
  Sha256 s;
  uint8_t dg[32];
  sha256_init(s);
  sha256_update(s, msg, msg_len);
  sha256_final(s, dg);
  B256Fp x, one, b, t, y, y2;
  bn256_load32(x, dg);            // to_mont multiplies by R^2 and reduces: any 256-bit value is accepted (value mod p)
  fp_set_one(one);
#pragma unroll
  for (int j = 0; j < 10; j++) b.v[j] = Bn256Fp::curve_b(j);
  for (;;) {
    fp_sqr_c(t, x); fp_mul_c(t, t, x); fp_add(t, t, b);
    fp_pow_const<Bn256Fp, Bn256Fp::ExpSqrt>(y, t);
    fp_sqr_c(y2, y);
    if (fp_eq(y2, t)) break;
    fp_add(x, x, one);
  }
  out.x = x; out.y = y;
}

// ---- bn256 HashG1: HKDF-SHA256 + Shallue-van de Woestijne ------------------------------------------------------------
// gfp.go:137-148 sign0: +1 when the canonical value is >= (p-1)/2, else -1
B2K_D int bn256_sign0(const B256Fp& a_mont) {
  B256Fp x;
  fp_from_mont(x, a_mont);
  ptx::sub_cc(x.v[0], Bn256Fp::half(0));                       // x - (p-1)/2 borrows  <=>  x < (p-1)/2
#pragma unroll
  for (int j = 1; j < 10; j++) ptx::subc_cc(x.v[j], Bn256Fp::half(j));
  return ptx::subc(0, 0) != 0 ? -1 : 1;
}
// gfp.go:150-162 legendre: e^((p-1)/2) as 0 / +1 / -1
B2K_D int bn256_legendre(const B256Fp& a) {
  B256Fp f, one;
  fp_pow_const<Bn256Fp, Bn256Fp::ExpLegendre>(f, a);
  if (fp_is_zero(f)) return 0;
  fp_set_one(one);
  return fp_eq(f, one) ? 1 : -1;
}
B2K_D void bn256_g(B256Fp& r, const B256Fp& x) {                // x^3 + 3
  B256Fp b;
#pragma unroll
  for (int j = 0; j < 10; j++) b.v[j] = Bn256Fp::curve_b(j);
  fp_sqr_c(r, x); fp_mul_c(r, r, x); fp_add(r, r, b);
}

B2K_NI void bn256_map_to_curve(Affine<B256Fp>& out, const B256Fp& t) {
  B256Fp one, b, s, smh, a, t2, st, w0, w, tw, x, y;
  fp_set_one(one);
#pragma unroll
  for (int j = 0; j < 10; j++) { b.v[j] = Bn256Fp::curve_b(j); s.v[j] = Bn256Fp::svdw_s(j); smh.v[j] = Bn256Fp::svdw_s_m1_half(j); }
  fp_sqr_c(t2, t); fp_add(a, b, t2); fp_add(a, a, one);          // a = 1 + B + t^2
  fp_mul_c(st, s, t);
  fp_mul_c(w0, st, a);
  fp_inv_fermat(w0, w0);                                         // gfP.Invert: e^(p-2), 0 -> 0
  fp_sqr_c(w, st); fp_mul_c(w, w, w0);                           // w = (s t)^2 / (s t a)
  const int e = bn256_sign0(t);
  fp_mul_c(tw, t, w);
  fp_sub(x, smh, tw);                                            // x1 = (s - 1)/2 - t w
  bn256_g(y, x);
  if (bn256_legendre(y) != 1) {
    B256Fp m1;
    fp_neg(m1, one);
    fp_sub(x, m1, x);                                            // x2 = -1 - x1
    bn256_g(y, x);
    if (bn256_legendre(y) != 1) {
      fp_sqr_c(x, a); fp_sqr_c(x, x); fp_mul_c(x, x, w0); fp_mul_c(x, x, w0); fp_add(x, x, one);   // x3 = 1 + a^4 w0^2
      bn256_g(y, x);
    }
  }
  B256Fp r;
  fp_pow_const<Bn256Fp, Bn256Fp::ExpSqrt>(r, y);
  if (e != bn256_sign0(r)) fp_neg(r, r);
  out.x = x; out.y = r;
}

B2K_D void bn256_hash_g1(Affine<B256Fp>& out, const uint8_t* msg, uint32_t msg_len, const uint8_t* dst, uint32_t dst_len) {
  uint8_t zeros[32], prk[32], t1[32], t2[32];
  const uint8_t info1[6] = {'H', '2', 'C', 0, 1, 1}, info2[6] = {'H', '2', 'C', 0, 1, 2};
  for (int i = 0; i < 32; i++) zeros[i] = 0;
  if (dst_len == 0) hmac_sha256(prk, zeros, 32, msg, msg_len, nullptr, 0, nullptr, 0);      // HKDF-Extract, nil salt = 32 zero bytes
  else hmac_sha256(prk, dst, dst_len, msg, msg_len, nullptr, 0, nullptr, 0);
  hmac_sha256(t1, prk, 32, info1, 6, nullptr, 0, nullptr, 0);                               // HKDF-Expand, 48 bytes = T1 || T2[0:16]
  hmac_sha256(t2, prk, 32, t1, 32, info2, 6, nullptr, 0);
  // 48 bytes big-endian mod p: hi (16 bytes) * 2^256 + lo (32 bytes), both through the Montgomery conversion (which reduces)
  uint8_t hi32[32], lo32[32];
  for (int i = 0; i < 16; i++) { hi32[i] = 0; hi32[16 + i] = t1[i]; lo32[i] = t1[16 + i]; lo32[16 + i] = t2[i]; }
  B256Fp hi, lo, two256, c;
  bn256_load32(hi, hi32);
  bn256_load32(lo, lo32);
#pragma unroll
  for (int j = 0; j < 10; j++) two256.v[j] = (j == 8) ? 1u : 0u;
  fp_to_mont(c, two256);
  fp_mul_c(hi, hi, c);
  fp_add(lo, lo, hi);
  bn256_map_to_curve(out, lo);
}

}  // namespace b2k
