// ecies_bls.cuh -- ECIES on BLS12-381 with keys on G1 or on G2, HKDF-SHA256 and AES-256-GCM, one ciphertext per thread, in
// constant time.  The group arithmetic is written once over the f_* vocabulary of tower.cuh (F = Fp for G1, Fp2 for G2).
//
// Replaces (reference):
//   ecies.Encrypt / Decrypt   encrypt/ecies/ecies.go:23-112 (group = the suite's G1 or G2, hash sha256.New)
//   Point.Mul (secret scalar) kilic G1/G2 Mul                                  -> ct_mul (no GLV, no wNAF)
//   Point.MarshalBinary       kilic/g1.go:119-124, g2.go:118-123 (ZCash compressed) -> ct_compress
//   Point.UnmarshalBinary     kilic/g1.go:127-131, g2.go:126-130              -> g1_decompress / g2_decompress (codec.cuh)
//   deriveKey, AES-GCM        ecies.go:114-131                                -> hkdf_sha256_44, gcm_* (aead.cuh)
//
// Secret here: the private key, r, dh, R before it is published, the HKDF output, the AES state and the plaintext.  No branch
// and no memory address depends on them:
//   - points are homogeneous projective (X : Y : Z), x = X/Z, y = Y/Z, with the exception-free formulas of Renes, Costello and
//     Batina 2016 for a = 0 (Algorithm 7: complete addition, Algorithm 9: doubling; b3 = 3b = 12 on G1, 12 (1 + u) on G2, a
//     product by additions only).  The identity (0 : 1 : 0), P = Q and P = -Q go through the same instructions.
//   - the table 1..8 P is built with the same formulas (one doubling, six additions), without inversion.
//   - scalars (< r < 2^255) are recoded into 65 signed radix-16 digits in [-8, 7] (SignedW4<8>, schnorr.cuh: a fixed carry
//     chain, no data-dependent branch).  Every digit reads all 8 table entries and keeps one with masks (ct_select), negates
//     Y under a mask, and adds it with the complete addition, 4 doublings between digits: the same sequence for every scalar.
//     The private key is recoded once per block into shared memory, where every thread reads the same digit at the same step.
//   - r G runs the same walk over 1..8 G, built once per block in shared memory and read by every thread at the same index.
//   - dh and R are compressed with the Fermat inversion (fp_inv_fermat, a fixed chain of products; on G2 of the norm
//     c0^2 + c1^2, times the conjugate), the sign flag comes from a borrow chain against (p - 1)/2 (on G2 chosen between c1
//     and c0 by a mask on c1 == 0), and the infinity encoding 0xC0 || 0... by a mask on Z == 0.
//   - the symmetric half is aead.cuh's.
// What does branch is public: the decoding of R or of the public key (its failure is the status), lengths, and loop counts.
#pragma once
#include "aead.cuh"
#include "codec.cuh"
#include "schnorr.cuh"

namespace b2k {

// operation counters beyond aead.cuh's (host emulation, B2K_ECIES_COUNT)
enum { ECIES_CNT_ADD = 4, ECIES_CNT_DBL = 5, ECIES_CNT_INV = 6, ECIES_CNT_BLS = 7 };
constexpr int ECIES_BLS_DIGITS = 65;                         // signed radix-16 digits of a scalar below r

template <class F> struct Proj { F X, Y, Z; };

// ---- masks -------------------------------------------------------------------------------------------------------------------
template <class C>
B2K_D void f_cmov(Fp<C>& r, const Fp<C>& a, uint32_t m) {
#pragma unroll
  for (int j = 0; j < C::N; j++) r.v[j] = (r.v[j] & ~m) | (a.v[j] & m);
}
template <class C>
B2K_D void f_cmov(Fp2<C>& r, const Fp2<C>& a, uint32_t m) { f_cmov(r.c0, a.c0, m); f_cmov(r.c1, a.c1, m); }

template <class C>
B2K_D uint32_t f_zero_mask(const Fp<C>& a) {                 // ~0 if a == 0 else 0
  uint32_t o = 0;
#pragma unroll
  for (int j = 0; j < C::N; j++) o |= a.v[j];
  return ct_eq_mask(o, 0);
}
template <class C>
B2K_D uint32_t f_zero_mask(const Fp2<C>& a) { return f_zero_mask(a.c0) & f_zero_mask(a.c1); }

// r = 3 b a: 12 a on G1, 12 (1 + u) a on G2
B2K_D void f_mul_b3(BFp& r, const BFp& a) {
  BFp t4, t8;
  fp_add(t4, a, a); fp_add(t4, t4, t4); fp_add(t8, t4, t4); fp_add(r, t8, t4);
}
B2K_D void f_mul_b3(BFp2& r, const BFp2& a) {
  BFp2 t4, t8;
  fp2_add(t4, a, a); fp2_add(t4, t4, t4); fp2_add(t8, t4, t4); fp2_add(t8, t8, t4);
  Bls381Tower::mul_xi(r, t8);
}

// ---- the group law (Renes-Costello-Batina 2016, a = 0) -------------------------------------------------------------------------
template <class F>
B2K_D void proj_set_identity(Proj<F>& p) { f_set_zero(p.X); f_set_one(p.Y); f_set_zero(p.Z); }

// (x : y : 1), or (0 : 1 : 0) for infinity's (0, 0), by masks
template <class F>
B2K_D void proj_from_affine(Proj<F>& r, const Affine<F>& p) {
  const uint32_t inf = f_zero_mask(p.x) & f_zero_mask(p.y);
  F one;
  f_set_one(one);
  r.X = p.x; r.Y = p.y; f_cmov(r.Y, one, inf);
  r.Z = one; f_set_zero(one); f_cmov(r.Z, one, inf);
}

// r = p + q, complete (Algorithm 7): 12 products, 2 products by 3b; r may alias p or q
template <class F>
B2K_NI void ct_add(Proj<F>& r, const Proj<F>& p, const Proj<F>& q) {
  ECIES_TICK(ECIES_CNT_ADD);
  F t0, t1, t2, t3, t4, x3, y3, z3;
  f_mul(t0, p.X, q.X); f_mul(t1, p.Y, q.Y); f_mul(t2, p.Z, q.Z);
  f_add(t3, p.X, p.Y); f_add(t4, q.X, q.Y); f_mul(t3, t3, t4);
  f_add(t4, t0, t1); f_sub(t3, t3, t4); f_add(t4, p.Y, p.Z);
  f_add(x3, q.Y, q.Z); f_mul(t4, t4, x3); f_add(x3, t1, t2);
  f_sub(t4, t4, x3); f_add(x3, p.X, p.Z); f_add(y3, q.X, q.Z);
  f_mul(x3, x3, y3); f_add(y3, t0, t2); f_sub(y3, x3, y3);
  f_add(x3, t0, t0); f_add(t0, x3, t0); f_mul_b3(t2, t2);
  f_add(z3, t1, t2); f_sub(t1, t1, t2); f_mul_b3(y3, y3);
  f_mul(x3, t4, y3); f_mul(t2, t3, t1); f_sub(x3, t2, x3);
  f_mul(y3, y3, t0); f_mul(t1, t1, z3); f_add(y3, t1, y3);
  f_mul(t0, t0, t3); f_mul(z3, z3, t4); f_add(z3, z3, t0);
  r.X = x3; r.Y = y3; r.Z = z3;
}

// r = 2 p (Algorithm 9): 6 products, 2 squarings, 1 product by 3b; the identity stays the identity; r may alias p
template <class F>
B2K_NI void ct_dbl(Proj<F>& r, const Proj<F>& p) {
  ECIES_TICK(ECIES_CNT_DBL);
  F t0, t1, t2, x3, y3, z3;
  f_sqr(t0, p.Y); f_add(z3, t0, t0); f_add(z3, z3, z3);
  f_add(z3, z3, z3); f_mul(t1, p.Y, p.Z); f_sqr(t2, p.Z);
  f_mul_b3(t2, t2); f_mul(x3, t2, z3); f_add(y3, t0, t2);
  f_mul(z3, t1, z3); f_add(t1, t2, t2); f_add(t2, t1, t2);
  f_sub(t0, t0, t2); f_mul(y3, t0, y3); f_add(y3, x3, y3);
  f_mul(t1, p.X, p.Y); f_mul(x3, t0, t1); f_add(x3, x3, x3);
  r.X = x3; r.Y = y3; r.Z = z3;
}

// tab[k - 1] = k P, k = 1..8
template <class F>
B2K_D void ct_table(Proj<F>* tab, const Affine<F>& p) {
  proj_from_affine(tab[0], p);
  ct_dbl(tab[1], tab[0]);
  for (int k = 2; k < 8; k++) ct_add(tab[k], tab[k - 1], tab[0]);
}

// c = d T for d in [-8, 7] (tab[k - 1] = k T): all 8 entries are read, one is kept with masks, Y is negated under a mask
template <class F>
B2K_D void ct_select(Proj<F>& c, const Proj<F>* tab, int d) {
  ECIES_TICK(ECIES_CNT_SELECT);
  const uint32_t neg = (uint32_t)(d >> 31), a = ((uint32_t)d ^ neg) - neg;
  proj_set_identity(c);
  for (int k = 0; k < 8; k++) {
    const uint32_t m = ct_eq_mask(a, (uint32_t)k + 1);
    f_cmov(c.X, tab[k].X, m); f_cmov(c.Y, tab[k].Y, m); f_cmov(c.Z, tab[k].Z, m);
  }
  F ny;
  f_neg(ny, c.Y);
  f_cmov(c.Y, ny, neg);
}

// the 65 digits of k < r, most significant first
B2K_D void ct_recode(int8_t* e, const uint8_t* k_be) {
  Scalar256 k;
  scalar_load_be(k, k_be);
  SignedW4<8> w;
  w.init(k.v);
  for (int i = 0; i < ECIES_BLS_DIGITS; i++) e[i] = (int8_t)w.next();
}

// Q = k P for the digits e of k (ct_recode) and tab = 1..8 P (ct_table): 64 windows of 4 doublings, 65 selections and 65
// complete additions, for every scalar
template <class F>
B2K_NI void ct_mul(Proj<F>& Q, const int8_t* e, const Proj<F>* tab) {
  proj_set_identity(Q);
  for (int i = 0; i < ECIES_BLS_DIGITS; i++) {
    if (i != 0) {
      ECIES_TICK(ECIES_CNT_WINDOW);
      ct_dbl(Q, Q); ct_dbl(Q, Q); ct_dbl(Q, Q); ct_dbl(Q, Q);
    }
    Proj<F> c;
    ct_select(c, tab, e[i]);
    ct_add(Q, Q, c);
  }
}

// ---- compression (MarshalBinary) ---------------------------------------------------------------------------------------------
// 1 / z by Fermat (0 -> 0); on Fp2 through the norm: (c0 - c1 u) / (c0^2 + c1^2)
B2K_D void ct_inv(BFp& r, const BFp& a) {
  ECIES_TICK(ECIES_CNT_INV);
  fp_inv_fermat(r, a);
}
B2K_D void ct_inv(BFp2& r, const BFp2& a) {
  ECIES_TICK(ECIES_CNT_INV);
  BFp n, t;
  fp_sqr_c(n, a.c0); fp_sqr_c(t, a.c1); fp_add(n, n, t);
  fp_inv_fermat(n, n);
  fp_mul_c(r.c0, a.c0, n);
  fp_mul_c(t, a.c1, n);
  fp_neg(r.c1, t);
}

// the sign flag (0x20 or 0) of y in Montgomery form: y > (p - 1)/2 on G1; lexicographically largest on G2 (c1, or c0 when
// c1 = 0), as Bls381G1::store / Bls381G2::store decide it
B2K_D uint32_t ct_sign_flag(const BFp& y) {
  BFp c;
  fp_from_mont(c, y);
  return (0u - (uint32_t)fp_canon_gt_half<Bls381Fp>(c)) & 0x20u;
}
B2K_D uint32_t ct_sign_flag(const BFp2& y) {
  BFp c0, c1;
  fp_from_mont(c0, y.c0);
  fp_from_mont(c1, y.c1);
  const uint32_t z1 = f_zero_mask(c1);
  const uint32_t g0 = 0u - (uint32_t)fp_canon_gt_half<Bls381Fp>(c0), g1 = 0u - (uint32_t)fp_canon_gt_half<Bls381Fp>(c1);
  return ((g1 & ~z1) | (g0 & z1)) & 0x20u;
}

B2K_D void ct_store_x(uint8_t* out, const BFp& x) {
  BFp t;
  fp_from_mont(t, x); fp_store_be(out, t);
}
B2K_D void ct_store_x(uint8_t* out, const BFp2& x) {        // x.c1 || x.c0
  BFp t;
  fp_from_mont(t, x.c1); fp_store_be(out, t);
  fp_from_mont(t, x.c0); fp_store_be(out + 48, t);
}

// MarshalBinary of p: ZCash compressed, PL = 48 (G1) or 96 (G2) bytes; the identity is 0xC0 || 0...
template <class F, int PL>
B2K_NI void ct_compress(uint8_t* out, const Proj<F>& p) {
  F zi, x, y;
  ct_inv(zi, p.Z);
  f_mul(x, p.X, zi);
  f_mul(y, p.Y, zi);
  ct_store_x(out, x);
  const uint32_t inf = f_zero_mask(p.Z);                      // then zi = 0, x = 0
  out[0] = (uint8_t)((((uint32_t)out[0] | 0x80u | ct_sign_flag(y)) & ~inf) | (0xC0u & inf));
}

// ---- one ciphertext ---------------------------------------------------------------------------------------------------------
template <class CV>
B2K_D bool ecies_bls_decode(Affine<typename CV::F>& p, const uint8_t* in) {
  if constexpr (CV::OUT_BYTES == 48) return g1_decompress(p, in, true);
  else return g2_decompress(p, in, true);
}

// 1..8 G of the group's generator
template <class CV>
B2K_D void ecies_bls_base_table(Proj<typename CV::F>* tab) {
  Affine<typename CV::F> g;
  CV::generator(g);
  ct_table(tab, g);
}

// Decrypt of ct = R || C || tag (PL + clen bytes) under the key recoded in e (shared by the block): msg (clen - 16 bytes) and
// the status; msg is zero unless ECIES_OK
template <class CV>
B2K_D int ecies_bls_decrypt_one(const int8_t* e, const uint8_t* ct, uint32_t clen, uint8_t* msg) {
  using F = typename CV::F;
  constexpr int PL = CV::OUT_BYTES;
  Affine<F> R;
  if (!ecies_bls_decode<CV>(R, ct)) {
    for (uint32_t i = 0; i + 16 < clen; i++) msg[i] = 0;
    return ECIES_POINT;
  }
  Proj<F> tab[8], dh;
  ct_table(tab, R);
  ct_mul(dh, e, tab);
  uint8_t dhb[PL], k44[44];
  ct_compress<F, PL>(dhb, dh);
  hkdf_sha256_44(k44, dhb, PL);
  return gcm_open(k44, ct + PL, clen, msg) ? ECIES_OK : ECIES_AUTH;
}

// Encrypt of msg (len bytes) to pub with the ephemeral r (32 bytes big-endian, below r): out = R || C || tag (PL + len + 16
// bytes), zero unless ECIES_OK; btab = 1..8 G (ecies_bls_base_table)
template <class CV>
B2K_D int ecies_bls_encrypt_one(const uint8_t* pub, const uint8_t* r, const Proj<typename CV::F>* btab, const uint8_t* msg,
                                uint32_t len, uint8_t* out) {
  using F = typename CV::F;
  constexpr int PL = CV::OUT_BYTES;
  Affine<F> P;
  if (!ecies_bls_decode<CV>(P, pub)) {
    for (uint32_t i = 0; i < PL + len + 16; i++) out[i] = 0;
    return ECIES_POINT;
  }
  int8_t e[ECIES_BLS_DIGITS];
  ct_recode(e, r);
  Proj<F> Q, tab[8];
  ct_mul(Q, e, btab);
  ct_compress<F, PL>(out, Q);
  ct_table(tab, P);
  ct_mul(Q, e, tab);
  uint8_t dhb[PL], k44[44];
  ct_compress<F, PL>(dhb, Q);
  hkdf_sha256_44(k44, dhb, PL);
  gcm_seal(k44, msg, len, out + PL);
  return ECIES_OK;
}

}  // namespace b2k
