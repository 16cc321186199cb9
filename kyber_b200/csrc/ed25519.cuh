// ed25519.cuh -- edwards25519 batch Point.Mul: -x^2 + y^2 = 1 + d x^2 y^2 over 2^255 - 19.
//
// Replaces (reference, in-tree ref10 port):
//   point.Mul                 group/edwards25519/point.go:235-258
//   geScalarMult / Vartime    group/edwards25519/ge.go:443-502, ge_mult_vartime.go:11-73
//   FromBytes / ToBytes       group/edwards25519/ge.go:110-150, :99-107
// Semantics kept: the scalar is the raw 256-bit little-endian integer (no reduction mod l,
// scalar.go:226-233), non-canonical y is accepted on decode, the result is the canonical 32-byte
// encoding.  Field: same Montgomery template as the pairing curves (8 x 32-bit limbs), extended
// coordinates (X:Y:Z:T), complete unified addition (a = -1, d non-square) and dedicated doubling.
#pragma once
#include "constants.cuh"
#include "fp.cuh"

namespace b2k {

using EFp = Fp<Ed25519Fp>;
struct EdExt { EFp X, Y, Z, T; };

B2K_D void ed_load_const(EFp& r, uint32_t (*f)(int)) {
#pragma unroll
  for (int j = 0; j < 8; j++) r.v[j] = f(j);
}

B2K_D void ed_set_identity(EdExt& p) { fp_set_zero(p.X); fp_set_one(p.Y); fp_set_one(p.Z); fp_set_zero(p.T); }

// add-2008-hwcd-3 (a = -1), complete: 8M + 1 multiplication by 2d
B2K_D void ed_add(EdExt& r, const EdExt& p, const EdExt& q) {
  EFp A, B, C, Dd, E, F, G, H, t, d2;
  fp_sub(A, p.Y, p.X); fp_sub(t, q.Y, q.X); fp_mul(A, A, t);
  fp_add(B, p.Y, p.X); fp_add(t, q.Y, q.X); fp_mul(B, B, t);
  ed_load_const(d2, Ed25519Fp::ed_2d);
  fp_mul(C, p.T, q.T); fp_mul(C, C, d2);
  fp_mul(Dd, p.Z, q.Z); fp_add(Dd, Dd, Dd);
  fp_sub(E, B, A); fp_sub(F, Dd, C); fp_add(G, Dd, C); fp_add(H, B, A);
  fp_mul(r.X, E, F); fp_mul(r.Y, G, H); fp_mul(r.T, E, H); fp_mul(r.Z, F, G);
}

// dbl-2008-hwcd (a = -1): 4M + 4S
B2K_D void ed_dbl(EdExt& r, const EdExt& p) {
  EFp A, B, C, Dd, E, F, G, H, t;
  fp_sqr(A, p.X); fp_sqr(B, p.Y);
  fp_sqr(C, p.Z); fp_add(C, C, C);
  fp_neg(Dd, A);                                    // a A, a = -1
  fp_add(t, p.X, p.Y); fp_sqr(E, t); fp_sub(E, E, A); fp_sub(E, E, B);
  fp_add(G, Dd, B); fp_sub(F, G, C); fp_sub(H, Dd, B);
  fp_mul(r.X, E, F); fp_mul(r.Y, G, H); fp_mul(r.T, E, H); fp_mul(r.Z, F, G);
}

// FromBytes (ge.go:110-150): returns false when no x exists for this y
B2K_D bool ed_decode(EdExt& r, const uint8_t* b) {
  EFp y, u, v, v3, x, t, one, d;
#pragma unroll
  for (int j = 0; j < 8; j++) y.v[j] = (uint32_t)b[4 * j] | ((uint32_t)b[4 * j + 1] << 8) | ((uint32_t)b[4 * j + 2] << 16) | ((uint32_t)b[4 * j + 3] << 24);
  const uint32_t sign = y.v[7] >> 31;
  y.v[7] &= 0x7fffffffu;
  fp_to_mont(y, y);                                 // values >= p are reduced by the multiplication
  fp_reduce_once<Ed25519Fp>(y.v);
  fp_set_one(one);
  ed_load_const(d, Ed25519Fp::ed_d);
  fp_sqr(u, y); fp_mul(v, u, d); fp_sub(u, u, one); fp_add(v, v, one);     // u = y^2 - 1, v = d y^2 + 1
  fp_sqr(v3, v); fp_mul(v3, v3, v);                 // v^3
  fp_sqr(t, v3); fp_mul(t, t, v); fp_mul(t, t, u);  // u v^7
  fp_pow_const<Ed25519Fp, Ed25519Fp::ExpP58>(x, t);
  fp_mul(x, x, v3); fp_mul(x, x, u);                // x = u v^3 (u v^7)^((p-5)/8)
  fp_sqr(t, x); fp_mul(t, t, v);                    // v x^2
  if (!fp_eq(t, u)) {
    EFp nu;
    fp_neg(nu, u);
    if (!fp_eq(t, nu)) return false;
    EFp s;
    ed_load_const(s, Ed25519Fp::sqrt_m1);
    fp_mul(x, x, s);
  }
  EFp xc;
  fp_from_mont(xc, x);
  if ((xc.v[0] & 1u) != sign) fp_neg(x, x);
  r.X = x; r.Y = y; fp_set_one(r.Z); fp_mul(r.T, x, y);
  return true;
}

// ToBytes of a point with Z = 1 (as ed_decode leaves it): the canonical encoding, no inversion
B2K_D void ed_encode_z1(uint8_t* out, const EdExt& p) {
  EFp x, y;
  fp_from_mont(x, p.X); fp_from_mont(y, p.Y);
  y.v[7] |= (x.v[0] & 1u) << 31;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    out[4 * j] = (uint8_t)y.v[j]; out[4 * j + 1] = (uint8_t)(y.v[j] >> 8);
    out[4 * j + 2] = (uint8_t)(y.v[j] >> 16); out[4 * j + 3] = (uint8_t)(y.v[j] >> 24);
  }
}

// ToBytes (ge.go:99-107)
B2K_D void ed_encode(uint8_t* out, const EdExt& p) {
  EFp zi;
  EdExt a;
  fp_inv(zi, p.Z);
  fp_mul(a.X, p.X, zi); fp_mul(a.Y, p.Y, zi);
  ed_encode_z1(out, a);
}

// out = k * P, k the raw little-endian 256-bit integer
B2K_D void ed_scalar_mul(EdExt& r, const uint8_t* k_le, const EdExt& p) {
  EdExt acc;
  ed_set_identity(acc);
  for (int i = 255; i >= 0; i--) {
    ed_dbl(acc, acc);
    if ((k_le[i >> 3] >> (i & 7)) & 1) ed_add(acc, acc, p);
  }
  r = acc;
}

}  // namespace b2k
