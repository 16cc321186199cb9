// ed25519.cuh -- the edwards25519 point layer: -x^2 + y^2 = 1 + d x^2 y^2 over 2^255 - 19.  The types, the group law, the codecs
// and checks, and the variable-time scalar multiplications that every edwards25519 protocol header builds on.
//
// Replaces (reference, in-tree ref10 port):
//   point.Mul                 group/edwards25519/point.go:235-258
//   geScalarMult / Vartime    group/edwards25519/ge.go:443-502, ge_mult_vartime.go:11-73   -> ed_mul_digits
//   FromBytes / ToBytes       group/edwards25519/ge.go:110-150, :99-107
//   point.IsCanonical         group/edwards25519/point.go:296-323      -> ed_bytes_canonical
//   point.HasSmallOrder       group/edwards25519/point.go:260-294      -> ed_has_small_order
// Semantics kept: a scalar is the raw 256-bit little-endian integer (no reduction mod l, scalar.go:226-233) read through
// geScalarMult's signed nibbles, whose top digit is dropped when it exceeds 8; non-canonical y is accepted on decode; results
// are the canonical 32-byte encoding.  Field: same Montgomery template as the pairing curves (8 x 32-bit limbs), extended
// coordinates (X:Y:Z:T), complete unified addition (a = -1, d non-square) and dedicated doubling.
#pragma once
#include "constants.cuh"
#include "fp.cuh"
#include "ed_scalar.cuh"

namespace b2k {

using EFp = Fp<Ed25519Fp>;
struct EdExt { EFp X, Y, Z, T; };
struct EdCached { EFp ypx, ymx, z2, t2d; };             // (Y + X, Y - X, 2 Z, 2 d T)
struct EdNiels { EFp ypx, ymx, t2d; };                   // (y + x, y - x, 2 d x y), Z = 1
// a decoded point (Z = 1); an operand that does not decode is stored as the identity
struct EdAff { EFp x, y; };

B2K_D void ed_load_const(EFp& r, uint32_t (*f)(int)) {
#pragma unroll
  for (int j = 0; j < 8; j++) r.v[j] = f(j);
}

B2K_D void ed_set_identity(EdExt& p) { fp_set_zero(p.X); fp_set_one(p.Y); fp_set_one(p.Z); fp_set_zero(p.T); }

// ---- the group law ---------------------------------------------------------------------------------------------------
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

// dbl-2008-hwcd without the T output (3M + 4S): for the doublings that another doubling follows
B2K_D void ed_dbl_xyz(EdExt& r, const EdExt& p) {
  EFp A, B, C, Dd, E, F, G, H, t;
  fp_sqr(A, p.X); fp_sqr(B, p.Y);
  fp_sqr(C, p.Z); fp_add(C, C, C);
  fp_neg(Dd, A);
  fp_add(t, p.X, p.Y); fp_sqr(E, t); fp_sub(E, E, A); fp_sub(E, E, B);
  fp_add(G, Dd, B); fp_sub(F, G, C); fp_sub(H, Dd, B);
  fp_mul(r.X, E, F); fp_mul(r.Y, G, H); fp_mul(r.Z, F, G);
}

// r = p + q or p - q (neg): add-2008-hwcd-3 on a cached operand, 8M; -q swaps Y + X with Y - X and negates 2 d T
B2K_D void ed_add_cached(EdExt& r, const EdExt& p, const EFp& ypx, const EFp& ymx, const EFp* z2, const EFp& t2d, bool neg) {
  EFp A, B, C, Dd, E, F, G, H, t;
  fp_sub(t, p.Y, p.X); fp_mul(A, t, neg ? ypx : ymx);
  fp_add(t, p.Y, p.X); fp_mul(B, t, neg ? ymx : ypx);
  fp_mul(C, p.T, t2d);
  if (neg) fp_neg(C, C);
  if (z2) fp_mul(Dd, p.Z, *z2);
  else fp_add(Dd, p.Z, p.Z);                            // Z = 1 (mixed addition, 7M)
  fp_sub(E, B, A); fp_sub(F, Dd, C); fp_add(G, Dd, C); fp_add(H, B, A);
  fp_mul(r.X, E, F); fp_mul(r.Y, G, H); fp_mul(r.T, E, H); fp_mul(r.Z, F, G);
}

// acc += q or acc -= q (mixed addition, 7M)
B2K_D void ed_madd(EdExt& acc, const EdNiels& q, bool neg) { ed_add_cached(acc, acc, q.ypx, q.ymx, nullptr, q.t2d, neg); }

B2K_D void ed_neg(EdExt& p) { fp_neg(p.X, p.X); fp_neg(p.T, p.T); }

// ---- codecs and checks -----------------------------------------------------------------------------------------------
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

// the encoding of the base point B (y = 4/5, x positive); host-callable too
B2K_HD void ed_base_bytes(uint8_t* b) {
  b[0] = 0x58;
  for (int j = 1; j < 32; j++) b[j] = 0x66;
}

// point.IsCanonical on the raw bytes: rejects exactly y in [p, 2^255), bit 255 (the sign of x) ignored
B2K_D bool ed_bytes_canonical(const uint8_t* b) {
  if ((b[31] & 0x7f) != 0x7f) return true;
  for (int i = 30; i > 0; i--)
    if (b[i] != 0xff) return true;
  return b[0] < 0xed;
}

// point.HasSmallOrder: the canonical y of the point (its encoding without the sign bit) is that of a point of order 1, 2,
// 4 or 8 (0, 1, p - 1 and the two order-8 y values).  p comes from ed_decode, so Z = 1.
B2K_D bool ed_has_small_order(const EdExt& p) {
  EFp y;
  fp_from_mont(y, p.Y);
  for (int k = 0; k < 5; k++) {
    uint32_t o = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) o |= y.v[j] ^ Ed25519Verify::small_y(8 * k + j);
    if (o == 0) return true;
  }
  return false;
}

// exact equality of two projective points: X1 Z2 = X2 Z1 and Y1 Z2 = Y2 Z1
B2K_D bool ed_eq(const EdExt& p, const EdExt& q) {
  EFp a, b;
  fp_mul(a, p.X, q.Z); fp_mul(b, q.X, p.Z);
  if (!fp_eq(a, b)) return false;
  fp_mul(a, p.Y, q.Z); fp_mul(b, q.Y, p.Z);
  return fp_eq(a, b);
}

// p == Q for a decoded p (Z = 1): X_p Z_Q = X_Q and Y_p Z_Q = Y_Q
B2K_D bool ed_eq_z1(const EdExt& p, const EdExt& Q) {
  EFp t;
  fp_mul(t, p.X, Q.Z);
  if (!fp_eq(t, Q.X)) return false;
  fp_mul(t, p.Y, Q.Z);
  return fp_eq(t, Q.Y);
}

B2K_D bool ed_eq_aff(const EdAff& a, const EdExt& Q) {
  EdExt p;
  p.X = a.x; p.Y = a.y;
  return ed_eq_z1(p, Q);
}

// ---- the forms ---------------------------------------------------------------------------------------------------------
B2K_D void ed_to_cached(EdCached& c, const EdExt& p) {
  EFp d2;
  ed_load_const(d2, Ed25519Fp::ed_2d);
  fp_add(c.ypx, p.Y, p.X); fp_sub(c.ymx, p.Y, p.X); fp_add(c.z2, p.Z, p.Z); fp_mul(c.t2d, p.T, d2);
}

// t[k - 1] = k A in cached form, k = 1..8
B2K_D void ed_cached_table(EdCached* t, const EdExt& A) {
  EdExt P;
  ed_to_cached(t[0], A);
  ed_dbl(P, A);
  ed_to_cached(t[1], P);
  for (int k = 2; k < 8; k++) {
    ed_add_cached(P, P, t[0].ypx, t[0].ymx, &t[0].z2, t[0].t2d, false);
    ed_to_cached(t[k], P);
  }
}

B2K_D void ed_niels_identity(EdNiels& q) { fp_set_one(q.ypx); fp_set_one(q.ymx); fp_set_zero(q.t2d); }

// FromBytes into Niels form; a point that does not decode becomes the identity and the call returns false
B2K_D bool ed_load_niels(EdNiels& q, const uint8_t* b) {
  EdExt p;
  if (!ed_decode(p, b)) { ed_niels_identity(q); return false; }
  EFp d2;
  ed_load_const(d2, Ed25519Fp::ed_2d);
  fp_add(q.ypx, p.Y, p.X); fp_sub(q.ymx, p.Y, p.X); fp_mul(q.t2d, p.T, d2);
  return true;
}

// the generated table k B, k = 1..8 (constants.cuh, Ed25519Verify::base_tab)
B2K_D void ed_load_base_table(EdNiels* t) {
#pragma unroll
  for (int k = 0; k < 8; k++) {
#pragma unroll
    for (int j = 0; j < 8; j++) {
      t[k].ypx.v[j] = Ed25519Verify::base_tab(24 * k + j);
      t[k].ymx.v[j] = Ed25519Verify::base_tab(24 * k + 8 + j);
      t[k].t2d.v[j] = Ed25519Verify::base_tab(24 * k + 16 + j);
    }
  }
}

B2K_D void ed_from_aff(EdExt& p, const EdAff& a) { p.X = a.x; p.Y = a.y; fp_set_one(p.Z); fp_mul(p.T, a.x, a.y); }

B2K_D bool ed_decode_aff(EdAff& a, const uint8_t* b) {
  EdExt p;
  const bool ok = ed_decode(p, b);
  if (!ok) ed_set_identity(p);
  a.x = p.X; a.y = p.Y;
  return ok;
}

// ---- variable-time multiplications -------------------------------------------------------------------------------------
B2K_D void ed_add_entry(EdExt& Q, const EdCached& t, bool neg) { ed_add_cached(Q, Q, t.ypx, t.ymx, &t.z2, t.t2d, neg); }
B2K_D void ed_add_entry(EdExt& Q, const EdNiels& t, bool neg) { ed_madd(Q, t, neg); }

// The digit step of geScalarMult: Q += d T for a digit d of sc_recode4, tab[k - 1] = k T (k = 1..8, cached or Niels).  A
// digit above 8 (only a top one can be) selects nothing, as selectCached (ge.go:419-433) does.
template <class E>
B2K_D void ed_digit_add(EdExt& Q, const E* tab, int d) {
  if (d != 0 && d <= 8) ed_add_entry(Q, tab[(d < 0 ? -d : d) - 1], d < 0);
}

// Q = geScalarMult(a, A) + geScalarMult(b, B) (Straus): one joint pass over the 64 signed nibbles of a and b, four doublings
// between digits, ta = 1..8 A and tb = 1..8 B.  tb null: Q = geScalarMult(a, A) alone (b is not read).
template <class TA, class TB>
B2K_D void ed_mul_digits(EdExt& Q, const uint32_t* a, const TA* ta, const uint32_t* b, const TB* tb) {
  int8_t ea[64], eb[64];
  sc_recode4(ea, a);
  if (tb) sc_recode4(eb, b);
  ed_set_identity(Q);
  for (int i = 63; i >= 0; i--) {
    if (i != 63) { ed_dbl_xyz(Q, Q); ed_dbl_xyz(Q, Q); ed_dbl_xyz(Q, Q); ed_dbl(Q, Q); }
    const int da = ea[i], db = tb ? eb[i] : 0;
    ed_digit_add(Q, ta, da);
    if (tb) ed_digit_add(Q, tb, db);
  }
}

template <class T>
B2K_D void ed_mul_digits(EdExt& Q, const uint32_t* a, const T* ta) { ed_mul_digits<T, T>(Q, a, ta, nullptr, nullptr); }

// Q = geScalarMult(r, P) for a raw 256-bit r, over a per-thread cached table (indexed at run time: local memory)
B2K_D void ed_mul_var(EdExt& Q, const uint32_t* r, const EdExt& P) {
  EdCached tp[8];
  ed_cached_table(tp, P);
  ed_mul_digits(Q, r, tp);
}

// out = Point.Mul(k, P) for the raw 32 little-endian bytes k (geScalarMult, ed_mul_var)
B2K_D void ed_scalar_mul(EdExt& out, const uint8_t* k_le, const EdExt& P) {
  uint32_t k[8];
  sc_load_le(k, k_le);
  ed_mul_var(out, k, P);
}

// Q = geScalarMult(r, P) + geScalarMult(c, P2) for raw 256-bit r and c, over two per-thread cached tables
B2K_D void ed_double_mul_var(EdExt& Q, const uint32_t* r, const EdExt& P, const uint32_t* c, const EdExt& P2) {
  EdCached tp[8], tq[8];
  ed_cached_table(tp, P);
  ed_cached_table(tq, P2);
  ed_mul_digits(Q, r, tp, c, tq);
}

// r = k p for a small k, double-and-add from the top bit
B2K_D void ed_mul_small(EdExt& r, const EdExt& p, uint32_t k) {
  if (!k) { ed_set_identity(r); return; }
  int top = 31;
  while (!((k >> top) & 1u)) top--;
  EdExt acc = p;
  for (int b = top - 1; b >= 0; b--) {
    ed_dbl(acc, acc);
    if ((k >> b) & 1u) ed_add(acc, acc, p);
  }
  r = acc;
}

// v = sum_j x^j C_j (Horner, share/poly.go:343-346), x v by double-and-add over the bits of x below its top bit (x >= 1)
B2K_D void ed_pubpoly_horner(EdExt& v, const EdNiels* cm, uint32_t t, uint64_t x) {
  int top = 63;
  while (top > 0 && !((x >> top) & 1u)) top--;
  ed_set_identity(v);
  for (int j = (int)t - 1; j >= 0; j--) {
    EdExt acc = v;
    for (int b = top - 1; b >= 0; b--) {
      ed_dbl(acc, acc);
      if ((x >> b) & 1u) ed_add(acc, acc, v);
    }
    const EdNiels c = cm[j];
    ed_add_cached(v, acc, c.ypx, c.ymx, nullptr, c.t2d, false);
  }
}

}  // namespace b2k
