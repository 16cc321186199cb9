// ec.cuh -- short-Weierstrass group law for a = 0 curves (y^2 = x^3 + b), written once over the
// field vocabulary f_* of tower.cuh, so the same code serves
//   G1 of BLS12-381 / bn254 / bn256  (F = Fp<...>)   and   G2 (F = Fp2<...>).
//
// Reference behaviour being replaced (formulas are standard EFD ones, not transcribed):
//   bn254 curvePoint.Add / Double      pairing/bn254/curve.go:76-161, 163-194 (Jacobian, a = 0)
//   bn254 twistPoint.Add / Double      pairing/bn254/twist.go:73-165
//   kilic G1/G2 Add/Double (third-party) via pairing/bls12381/kilic/g1.go:92-108
// Every exceptional case of the group law is handled (P+inf, P+P, P+(-P)), because Pippenger buckets
// do hit them; the reference's formulas branch on the same cases (bn254/curve.go:77-84,128-131).
//
// Coordinates:
//   Affine<F>  (x, y), infinity encoded as (0, 0)   [never on the curve since b != 0]
//   Jac<F>     x = X/Z^2, y = Y/Z^3, infinity Z = 0         -- scalar multiplication (cheap doubling)
//   Xyzz<F>    x = X/ZZ,  y = Y/ZZZ, infinity ZZ = 0        -- bucket accumulation (cheap mixed add)
#pragma once
#include "tower.cuh"

namespace b2k {

template <class F> struct Affine { F x, y; };
template <class F> struct Jac { F X, Y, Z; };
template <class F> struct Xyzz { F X, Y, ZZ, ZZZ; };

template <class F> B2K_D bool aff_is_inf(const Affine<F>& p) { return f_is_zero(p.x) && f_is_zero(p.y); }
template <class F> B2K_D void aff_set_inf(Affine<F>& p) { f_set_zero(p.x); f_set_zero(p.y); }
template <class F> B2K_D bool jac_is_inf(const Jac<F>& p) { return f_is_zero(p.Z); }
template <class F> B2K_D void jac_set_inf(Jac<F>& p) { f_set_one(p.X); f_set_one(p.Y); f_set_zero(p.Z); }
template <class F> B2K_D bool xyzz_is_inf(const Xyzz<F>& p) { return f_is_zero(p.ZZ); }
template <class F> B2K_D void xyzz_set_inf(Xyzz<F>& p) { f_set_one(p.X); f_set_one(p.Y); f_set_zero(p.ZZ); f_set_zero(p.ZZZ); }

template <class F>
B2K_D void jac_from_affine(Jac<F>& r, const Affine<F>& p) {
  if (aff_is_inf(p)) { jac_set_inf(r); return; }
  r.X = p.x; r.Y = p.y; f_set_one(r.Z);
}

template <class F>
B2K_D void xyzz_from_affine(Xyzz<F>& r, const Affine<F>& p) {
  if (aff_is_inf(p)) { xyzz_set_inf(r); return; }
  r.X = p.x; r.Y = p.y; f_set_one(r.ZZ); f_set_one(r.ZZZ);
}

// ---- Jacobian ---------------------------------------------------------------------------------
// dbl-2009-l (a = 0): 2M + 5S
template <class F>
B2K_D void jac_dbl(Jac<F>& r, const Jac<F>& p) {
  F A, B, C, D, E, T;
  f_sqr(A, p.X);
  f_sqr(B, p.Y);
  f_sqr(C, B);
  f_add(D, p.X, B); f_sqr(D, D); f_sub(D, D, A); f_sub(D, D, C); f_dbl(D, D);
  f_dbl(E, A); f_add(E, E, A);
  f_mul(T, p.Y, p.Z);                 // before X/Y are overwritten (r may alias p)
  f_sqr(A, E);                        // F
  f_sub(A, A, D); f_sub(A, A, D);     // X3
  f_dbl(C, C); f_dbl(C, C); f_dbl(C, C);
  f_sub(D, D, A); f_mul(D, E, D); f_sub(r.Y, D, C);
  r.X = A;
  f_dbl(r.Z, T);                      // Y = 0 never happens on a prime-order a=0 curve; Z=0 stays 0
}

template <class F>
B2K_NI void jac_dbl_rare(Jac<F>& r, const Jac<F>& p) { jac_dbl(r, p); }

// madd-2007-bl: 7M + 4S, with all exceptional cases
template <class F>
B2K_D void jac_madd(Jac<F>& r, const Jac<F>& p, const Affine<F>& q) {
  if (aff_is_inf(q)) { r = p; return; }
  if (jac_is_inf(p)) { r.X = q.x; r.Y = q.y; f_set_one(r.Z); return; }
  F Z1Z1, U2, S2, H, HH, I, J, rr, V, T;
  f_sqr(Z1Z1, p.Z);
  f_mul(U2, q.x, Z1Z1);
  f_mul(S2, q.y, p.Z); f_mul(S2, S2, Z1Z1);
  f_sub(H, U2, p.X);
  f_sub(rr, S2, p.Y);
  if (f_is_zero(H)) {
    if (f_is_zero(rr)) { jac_dbl_rare(r, p); return; }
    jac_set_inf(r); return;
  }
  f_dbl(rr, rr);
  f_sqr(HH, H);
  f_dbl(I, HH); f_dbl(I, I);
  f_mul(J, H, I);
  f_mul(V, p.X, I);
  f_add(T, p.Z, H); f_sqr(T, T); f_sub(T, T, Z1Z1); f_sub(T, T, HH);   // Z3
  f_sqr(U2, rr); f_sub(U2, U2, J); f_sub(U2, U2, V); f_sub(U2, U2, V);  // X3
  f_sub(V, V, U2); f_mul(V, rr, V);
  f_mul(J, p.Y, J); f_dbl(J, J);
  f_sub(r.Y, V, J);
  r.X = U2;
  r.Z = T;
}

// add-2007-bl: 11M + 5S, with all exceptional cases
template <class F>
B2K_D void jac_add(Jac<F>& r, const Jac<F>& p, const Jac<F>& q) {
  if (jac_is_inf(q)) { r = p; return; }
  if (jac_is_inf(p)) { r = q; return; }
  F Z1Z1, Z2Z2, U1, U2, S1, S2, H, I, J, rr, V, T;
  f_sqr(Z1Z1, p.Z);
  f_sqr(Z2Z2, q.Z);
  f_mul(U1, p.X, Z2Z2);
  f_mul(U2, q.X, Z1Z1);
  f_mul(S1, p.Y, q.Z); f_mul(S1, S1, Z2Z2);
  f_mul(S2, q.Y, p.Z); f_mul(S2, S2, Z1Z1);
  f_sub(H, U2, U1);
  f_sub(rr, S2, S1);
  if (f_is_zero(H)) {
    if (f_is_zero(rr)) { jac_dbl_rare(r, p); return; }
    jac_set_inf(r); return;
  }
  f_dbl(rr, rr);
  f_dbl(I, H); f_sqr(I, I);
  f_mul(J, H, I);
  f_mul(V, U1, I);
  f_add(T, p.Z, q.Z); f_sqr(T, T); f_sub(T, T, Z1Z1); f_sub(T, T, Z2Z2); f_mul(T, T, H);  // Z3
  f_sqr(U2, rr); f_sub(U2, U2, J); f_sub(U2, U2, V); f_sub(U2, U2, V);                    // X3
  f_sub(V, V, U2); f_mul(V, rr, V);
  f_mul(S1, S1, J); f_dbl(S1, S1);
  f_sub(r.Y, V, S1);
  r.X = U2;
  r.Z = T;
}

template <class F>
B2K_D void jac_neg(Jac<F>& r, const Jac<F>& p) { r.X = p.X; f_neg(r.Y, p.Y); r.Z = p.Z; }

// one field inversion
template <class F>
B2K_D void jac_to_affine(Affine<F>& r, const Jac<F>& p) {
  if (jac_is_inf(p)) { aff_set_inf(r); return; }
  F zi, zi2;
  f_inv(zi, p.Z);
  f_sqr(zi2, zi);
  f_mul(r.x, p.X, zi2);
  f_mul(zi2, zi2, zi);
  f_mul(r.y, p.Y, zi2);
}

// ---- XYZZ -------------------------------------------------------------------------------------
// dbl-2008-s-1 (a = 0): 6M + 4S ... used only outside the hot loop
template <class F>
B2K_D void xyzz_dbl(Xyzz<F>& r, const Xyzz<F>& p) {
  if (xyzz_is_inf(p)) { r = p; return; }
  F U, V, W, S, M, T;
  f_dbl(U, p.Y);
  f_sqr(V, U);
  f_mul(W, U, V);
  f_mul(S, p.X, V);
  f_sqr(M, p.X); f_dbl(T, M); f_add(M, M, T);
  f_mul(T, W, p.Y);                       // W*Y1 (before Y is overwritten)
  f_mul(r.ZZ, V, p.ZZ);
  f_mul(r.ZZZ, W, p.ZZZ);
  f_sqr(U, M); f_sub(U, U, S); f_sub(U, U, S);   // X3
  f_sub(S, S, U); f_mul(S, M, S); f_sub(r.Y, S, T);
  r.X = U;
}

template <class F>
B2K_NI void xyzz_dbl_rare(Xyzz<F>& r, const Xyzz<F>& p) { xyzz_dbl(r, p); }

// madd-2008-s: 8M + 2S; q given affine, optionally negated (signed-digit buckets).  Over Fp, Y3 = R (Q - X3) - Y1 PPP is one
// sum of two products (f_mul_sub); Fp2 keeps two products: that form of Y3 tripped an illegal access in the G2 MSM on sm_90a
template <class F>
B2K_D void xyzz_madd(Xyzz<F>& r, const Xyzz<F>& p, const Affine<F>& q, bool negate) {
  if (aff_is_inf(q)) { r = p; return; }
  F qy;
  if (negate) f_neg(qy, q.y); else qy = q.y;
  if (xyzz_is_inf(p)) { r.X = q.x; r.Y = qy; f_set_one(r.ZZ); f_set_one(r.ZZZ); return; }
  F U2, S2, P, R, PP, PPP, Q;
  f_mul(U2, q.x, p.ZZ);
  f_mul(S2, qy, p.ZZZ);
  f_sub(P, U2, p.X);
  f_sub(R, S2, p.Y);
  if (f_is_zero(P)) {
    if (f_is_zero(R)) {                   // same point: double the affine operand
      Xyzz<F> t; t.X = q.x; t.Y = qy; f_set_one(t.ZZ); f_set_one(t.ZZZ);
      xyzz_dbl_rare(r, t); return;
    }
    xyzz_set_inf(r); return;
  }
  f_sqr(PP, P);
  f_mul(PPP, P, PP);
  f_mul(Q, p.X, PP);
  f_sqr(U2, R); f_sub(U2, U2, PPP); f_sub(U2, U2, Q); f_sub(U2, U2, Q);   // X3
  f_sub(Q, Q, U2);
  if constexpr (f_is_base<F>) {
    f_mul_sub(r.Y, R, Q, p.Y, PPP, S2);                                    // R (Q - X3) - Y1 PPP
  } else {
    f_mul(Q, R, Q);
    f_mul(S2, p.Y, PPP);
    f_sub(r.Y, Q, S2);
  }
  r.X = U2;
  f_mul(r.ZZ, p.ZZ, PP);
  f_mul(r.ZZZ, p.ZZZ, PPP);
}

// add-2008-s: 12M + 2S (Y3 likewise over Fp)
template <class F>
B2K_D void xyzz_add(Xyzz<F>& r, const Xyzz<F>& p, const Xyzz<F>& q) {
  if (xyzz_is_inf(q)) { r = p; return; }
  if (xyzz_is_inf(p)) { r = q; return; }
  F U1, U2, S1, S2, P, R, PP, PPP, Q;
  f_mul(U1, p.X, q.ZZ);
  f_mul(U2, q.X, p.ZZ);
  f_mul(S1, p.Y, q.ZZZ);
  f_mul(S2, q.Y, p.ZZZ);
  f_sub(P, U2, U1);
  f_sub(R, S2, S1);
  if (f_is_zero(P)) {
    if (f_is_zero(R)) { xyzz_dbl_rare(r, p); return; }
    xyzz_set_inf(r); return;
  }
  f_sqr(PP, P);
  f_mul(PPP, P, PP);
  f_mul(Q, U1, PP);
  f_sqr(U2, R); f_sub(U2, U2, PPP); f_sub(U2, U2, Q); f_sub(U2, U2, Q);   // X3
  if constexpr (f_is_base<F>) {
    f_sub(Q, Q, U2);
    f_mul(U1, p.ZZ, q.ZZ);
    f_mul(S2, p.ZZZ, q.ZZZ);
    f_mul_sub(r.Y, R, Q, S1, PPP, S1);                                     // R (Q - X3) - S1 PPP
  } else {
    f_sub(Q, Q, U2); f_mul(Q, R, Q);
    f_mul(S1, S1, PPP);
    f_mul(U1, p.ZZ, q.ZZ);
    f_mul(S2, p.ZZZ, q.ZZZ);
    f_sub(r.Y, Q, S1);
  }
  r.X = U2;
  f_mul(r.ZZ, U1, PP);
  f_mul(r.ZZZ, S2, PPP);
}

template <class F>
B2K_D void xyzz_to_affine(Affine<F>& r, const Xyzz<F>& p) {
  if (xyzz_is_inf(p)) { aff_set_inf(r); return; }
  // 1/ZZZ, then 1/ZZ = ZZZ^-2 * ZZ^2 ... keep it simple: one inversion of ZZ*ZZZ
  F t, ti, a;
  f_mul(t, p.ZZ, p.ZZZ);
  f_inv(ti, t);
  f_mul(a, ti, p.ZZZ);          // 1/ZZ
  f_mul(r.x, p.X, a);
  f_mul(a, ti, p.ZZ);           // 1/ZZZ
  f_mul(r.y, p.Y, a);
}

// XYZZ -> Jacobian without inversion:  (X*ZZ... ) choose Z = ZZZ/ZZ is not available; instead use
// Z := ZZZ*ZZ ... we avoid the conversion entirely: scalar multiplication of XYZZ points uses xyzz_dbl.

// k * P for a small public-size integer k (bucket-reduction chunk offsets): plain double-and-add.
template <class F>
B2K_D void xyzz_mul_small(Xyzz<F>& r, const Xyzz<F>& p, uint32_t k) {
  Xyzz<F> acc;
  xyzz_set_inf(acc);
  for (int i = 31; i >= 0; i--) {
    xyzz_dbl(acc, acc);
    if ((k >> i) & 1) xyzz_add(acc, acc, p);
  }
  r = acc;
}

}  // namespace b2k
