// h2c.cuh -- RFC 9380 hash_to_curve for BLS12-381 G1 (suite BLS12381G1_XMD:SHA-256_SSWU_RO_), per thread.
//
// Replaces: kilic.G1Elt.Hash -> third-party HashToCurve(msg, dst)   pairing/bls12381/kilic/g1.go:161-170
// (default DST "BLS_SIG_BLS12381G1_XMD:SHA-256_SSWU_RO_NUL_", g1.go:17; per-suite override suite.go:32-46),
// the per-message step of bls.Sign/Verify (sign/bls/bls.go:67-96).
// Pipeline: expand_message_xmd(SHA-256) -> 2 field elements -> simplified SWU on E' -> derived 11-isogeny
// (tools/derive_isogeny.py) evaluated projectively -> add -> clear cofactor by h_eff = 1 - x.
// Pinned end-to-end by the reference's signature KATs (tests/test_gpu_bls12381_h2c.py).
#pragma once
#include "codec.cuh"
#include "iso_g1_constants.cuh"
#include "sha256.cuh"

namespace b2k {

// ---- expand_message_xmd, 128 output bytes (two field elements of L = 64 bytes) ----------------------------
// dst must be <= 255 bytes (longer DSTs are pre-hashed by the caller, RFC 9380 5.3.3)
B2K_NI void expand_message_xmd_128(uint8_t* out128, const uint8_t* msg, uint32_t msg_len, const uint8_t* dst, uint32_t dst_len) {
  Sha256 s;
  uint8_t b0[32], bi[32], t[32];
  const uint8_t dl = (uint8_t)dst_len;
  const uint8_t lib[3] = {0, 128, 0};               // I2OSP(128, 2) || I2OSP(0, 1)
  sha256_init(s);
  sha256_update_zero(s, 64);
  sha256_update(s, msg, msg_len);
  sha256_update(s, lib, 3);
  sha256_update(s, dst, dst_len);
  sha256_update(s, &dl, 1);
  sha256_final(s, b0);
  for (int i = 1; i <= 4; i++) {
    const uint8_t idx = (uint8_t)i;
    if (i == 1) { for (int k = 0; k < 32; k++) t[k] = b0[k]; }
    else { for (int k = 0; k < 32; k++) t[k] = b0[k] ^ bi[k]; }
    sha256_init(s);
    sha256_update(s, t, 32);
    sha256_update(s, &idx, 1);
    sha256_update(s, dst, dst_len);
    sha256_update(s, &dl, 1);
    sha256_final(s, bi);
    for (int k = 0; k < 32; k++) out128[32 * (i - 1) + k] = bi[k];
  }
}

B2K_D void fp_load_table(BFp& r, const uint32_t* t) {
#pragma unroll
  for (int j = 0; j < 12; j++) r.v[j] = t[j];
}

// 64 big-endian bytes -> value mod p, Montgomery form:  hi * 2^256 + lo
B2K_D void fp_from_64_bytes(BFp& r, const uint8_t* b) {
  BFp hi, lo, c;
  fp_set_zero(hi); fp_set_zero(lo);
  for (int j = 0; j < 8; j++) {
    const uint8_t* q = b + 4 * (7 - j);
    hi.v[j] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
    q = b + 32 + 4 * (7 - j);
    lo.v[j] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
  }
  fp_to_mont(hi, hi);
  fp_to_mont(lo, lo);
  fp_load_table(c, TWO_POW_256);
  fp_mul_c(hi, hi, c);
  fp_add(r, hi, lo);
}

B2K_D uint32_t fp_sgn0(const BFp& a_mont) {
  BFp c;
  fp_from_mont(c, a_mont);
  return c.v[0] & 1u;
}

// simplified SWU map onto E': y^2 = x^3 + A'x + B'  (RFC 9380 6.6.2, straight-line version with one inversion)
B2K_NI void map_to_curve_sswu(BFp& x, BFp& y, const BFp& u) {
  BFp A, B, Zc, t, tv1, x1, gx, u2, c;
  fp_load_table(A, SSWU_A); fp_load_table(B, SSWU_B); fp_load_table(Zc, SSWU_Z);
  fp_sqr_c(u2, u);
  fp_mul_c(t, Zc, u2);                  // Z u^2
  fp_sqr_c(tv1, t); fp_add(tv1, tv1, t);   // Z^2 u^4 + Z u^2
  if (fp_is_zero(tv1)) {
    fp_load_table(x1, SSWU_B_OVER_ZA);
  } else {
    fp_inv(tv1, tv1);
    fp_set_one(c); fp_add(tv1, tv1, c);
    fp_load_table(c, SSWU_NEG_B_OVER_A);
    fp_mul_c(x1, c, tv1);
  }
  fp_sqr_c(gx, x1); fp_add(gx, gx, A); fp_mul_c(gx, gx, x1); fp_add(gx, gx, B);   // x1^3 + A x1 + B
  BFp yy;
  if (fp_sqrt(yy, gx)) {
    x = x1;
  } else {
    fp_mul_c(x, t, x1);                 // x2 = Z u^2 x1
    fp_sqr_c(gx, x); fp_add(gx, gx, A); fp_mul_c(gx, gx, x); fp_add(gx, gx, B);
    fp_sqrt(yy, gx);                    // always a square when gx1 is not
  }
  if (fp_sgn0(u) != fp_sgn0(yy)) fp_neg(yy, yy);
  y = yy;
}

B2K_D void horner(BFp& r, const uint32_t (*coef)[12], int n, const BFp& x) {
  BFp acc, c;
  fp_load_table(acc, coef[n - 1]);
  for (int k = n - 2; k >= 0; k--) {
    fp_mul_c(acc, acc, x);
    fp_load_table(c, coef[k]);
    fp_add(acc, acc, c);
  }
  r = acc;
}

// iso_map(x', y') = (xn/xd, y' yn/yd) returned as a Jacobian point (Z = xd yd), no inversion
B2K_NI void iso_map_g1(Jac<BFp>& r, const BFp& x, const BFp& y) {
  BFp xn, xd, yn, yd, t;
  horner(xn, ISO_G1_XNUM, 12, x);
  horner(xd, ISO_G1_XDEN, 11, x);
  horner(yn, ISO_G1_YNUM, 16, x);
  horner(yd, ISO_G1_YDEN, 16, x);
  fp_mul_c(r.Z, xd, yd);
  if (fp_is_zero(r.Z)) { jac_set_inf(r); return; }      // kernel of the isogeny
  fp_sqr_c(t, yd);                                      // yd^2
  fp_mul_c(r.X, xn, xd); fp_mul_c(r.X, r.X, t);         // xn xd yd^2
  fp_mul_c(r.Y, y, yn); fp_mul_c(r.Y, r.Y, t);          // y yn yd^2
  fp_sqr_c(t, xd); fp_mul_c(t, t, xd);                  // xd^3
  fp_mul_c(r.Y, r.Y, t);
}

// full hash_to_curve: result affine (Montgomery) in G1
B2K_D void hash_to_g1(Affine<BFp>& out, const uint8_t* msg, uint32_t msg_len, const uint8_t* dst, uint32_t dst_len) {
  uint8_t uni[128];
  expand_message_xmd_128(uni, msg, msg_len, dst, dst_len);
  BFp u0, u1, x, y;
  fp_from_64_bytes(u0, uni);
  fp_from_64_bytes(u1, uni + 64);
  Jac<BFp> q0, q1, acc;
  map_to_curve_sswu(x, y, u0); iso_map_g1(q0, x, y);
  map_to_curve_sswu(x, y, u1); iso_map_g1(q1, x, y);
  jac_add(q0, q0, q1);
  // clear cofactor: [h_eff] R, h_eff = |x| + 1 = 0xd201000000010001
  acc = q0;
  for (int b = 62; b >= 0; b--) {
    jac_dbl(acc, acc);
    if ((BLS_X_ABS >> b) & 1) jac_add(acc, acc, q0);
  }
  jac_add(acc, acc, q0);
  jac_to_affine(out, acc);
}

}  // namespace b2k
