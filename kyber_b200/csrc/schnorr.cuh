// schnorr.cuh -- sign/schnorr VerifyWithChecks over BLS12-381 keys on G1 or on G2, one signature per thread.
//
// Replaces (reference):
//   schnorr.VerifyWithChecks    sign/schnorr/schnorr.go:89-183 (called per packet by dkg.VerifyPacketSignature through
//                               schnorr.Verify, share/dkg/pedersen/structs.go:293-348; by share/vss and share/dkg/rabin)
//   R, public.UnmarshalBinary   kilic G1Elt / G2Elt FromCompressed with the subgroup check -> g1_decompress / g2_decompress
//   s.UnmarshalBinary           mod.Int, rejects s >= r (group/mod/int.go:359-372) -> scalar_in_range
//   h = SetBytes(SHA-512(...))  mod.Int.SetBytes: the 64-byte digest read big-endian, mod r (int.go:404-411) -> fr_from_be512
//   s B == R + h public         -> schnorr_equation + jac_eq_affine
// Every input is public, so the code runs in variable time.  The checks run in the reference's order and the first one that
// fails gives the status (SCHNORR_* below, the values of B2K_SCHNORR_* in include/b2kyber.h).  Of the reference's checks, the
// point and scalar types of this suite have neither IsCanonical nor HasSmallOrder, and "point not in correct group" cannot fail:
// UnmarshalBinary already refused every point outside the order-r subgroup.
//
// The digest is over R.MarshalTo || public.MarshalTo || msg.  Hashing the input bytes instead is exact, because the decoders
// accept only encodings that are their own re-encoding: the compression flag set, the sign flag consistent with y, every
// coordinate below p, and infinity only as 0xC0 followed by zeros (sign flag clear, x = 0).  An encoding that decodes is
// therefore the MarshalBinary of the point it decodes to.
//
// Infinity is a valid R and a valid key, as in the reference: with public = O the signature is valid iff s B = R, and
// (R, s, public) = (O, 0, O) is accepted.
//
// The equation is evaluated as Q = s B + h (-public) in one signed radix-16 walk that shares the doublings (Straus), then
// compared with R in Jacobian form (no inversion).  The tables 1..8 B are staged in shared memory once per block
// (schnorr_base_table); 1..8 (-public) are built per thread and normalised with one inversion.
//   G1: both scalars are split with glv_split_bls381 (valid: B and the decoded key lie in the subgroup, where phi acts as
//       -x^2): four 127-bit digit streams over 33 steps, the phi images read from the same tables (x -> beta x).
//   G2: two 255-bit scalars over 65 steps.
// jac_madd handles the doubling and the inverse cases, which a key such as +-B or a small multiple of B reaches.
#pragma once
#include "codec.cuh"
#include "msm.cuh"
#include "sha512.cuh"

namespace b2k {

enum { SCHNORR_OK = 0, SCHNORR_R = 1, SCHNORR_S = 2, SCHNORR_PK = 3, SCHNORR_INVALID = 4 };

// h = (w[0] || ... || w[7]) mod r for the 512-bit big-endian integer of eight 64-bit words (the SHA-512 state is that digest):
// with hi, lo the two 256-bit halves, each brought below r by at most two subtractions (2^256 < 3 r), h = hi 2^256 + lo =
// mont(hi, R^2) + lo, R = 2^256 the Montgomery radix of Bls381Fr.
B2K_D void fr_from_be512(Scalar256& h, const uint64_t* w) {
  using Fr = Fp<Bls381Fr>;
  Fr hi, lo, r2;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    hi.v[2 * j] = (uint32_t)w[3 - j]; hi.v[2 * j + 1] = (uint32_t)(w[3 - j] >> 32);
    lo.v[2 * j] = (uint32_t)w[7 - j]; lo.v[2 * j + 1] = (uint32_t)(w[7 - j] >> 32);
  }
  uint32_t m[8];
#pragma unroll
  for (int j = 0; j < 8; j++) { m[j] = Bls381Fr::mod(j); r2.v[j] = Bls381Fr::r2(j); }
  for (int k = 0; k < 2; k++) {
    if (limbs_geq<8>(hi.v, m)) limbs_sub<8>(hi.v, m);
    if (limbs_geq<8>(lo.v, m)) limbs_sub<8>(lo.v, m);
  }
  fp_mul(hi, hi, r2);
  fp_add(hi, hi, lo);
#pragma unroll
  for (int j = 0; j < 8; j++) h.v[j] = hi.v[j];
}

// tab[j - 1] = j P, j = 1..8, affine, normalised with one inversion; P must have order > 8 or be infinity (all entries
// infinity).  Points of G1 and G2 have order r.
template <class F, class INV>
B2K_D void schnorr_table8(Affine<F>* tab, const Affine<F>& p, INV inv_fn) {
  if (aff_is_inf(p)) {
    for (int j = 0; j < 8; j++) aff_set_inf(tab[j]);
    return;
  }
  Jac<F> tj[8];
  jac_from_affine(tj[0], p);
  jac_dbl(tj[1], tj[0]);
  for (int j = 2; j < 8; j++) jac_madd(tj[j], tj[j - 1], p);
  tab[0] = p;
  F pre[8], acc, zi, zi2;
  f_set_one(acc);
  for (int j = 1; j < 8; j++) { pre[j] = acc; f_mul(acc, acc, tj[j].Z); }
  inv_fn(acc, acc);
  for (int j = 7; j >= 1; j--) {
    f_mul(zi, acc, pre[j]);
    f_mul(acc, acc, tj[j].Z);
    f_sqr(zi2, zi);
    f_mul(tab[j].x, tj[j].X, zi2);
    f_mul(zi2, zi2, zi);
    f_mul(tab[j].y, tj[j].Y, zi2);
  }
}

// 1..8 B for the group's generator
template <class CV, class INV>
B2K_D void schnorr_base_table(Affine<typename CV::F>* tab, INV inv_fn) {
  Affine<typename CV::F> g;
  CV::generator(g);
  schnorr_table8(tab, g, inv_fn);
}

// signed radix-16 digits of k < 2^(32 NL - 4): k + 0x88..8 top-aligned in NL + 1 limbs; each step takes the top nibble minus 8
template <int NL>
struct SignedW4 {
  uint32_t d[NL + 1];
  B2K_D void init(const uint32_t* k) {
    uint32_t a[NL + 1];
    uint64_t c = 0;
    for (int j = 0; j <= NL; j++) {
      const uint64_t t = (uint64_t)(j < NL ? k[j] : 0u) + (j < NL ? 0x88888888u : 0x8u) + c;
      a[j] = (uint32_t)t; c = t >> 32;
    }
    for (int j = NL; j > 0; j--) d[j] = (a[j] << 28) | (a[j - 1] >> 4);
    d[0] = a[0] << 28;
  }
  B2K_D int next() {
    const int e = (int)(d[NL] >> 28) - 8;
    for (int j = NL; j > 0; j--) d[j] = (d[j] << 4) | (d[j - 1] >> 28);
    d[0] <<= 4;
    return e;
  }
};

// acc += e T (T = 1..8 P), with the result's y negated when flip; phi: x -> beta x (G1 only)
template <class F>
B2K_D void schnorr_add_digit(Jac<F>& acc, const Affine<F>* tab, int e, bool flip, const F* beta) {
  if (!e) return;
  Affine<F> q = tab[(e < 0 ? -e : e) - 1];
  if (beta) f_mul(q.x, q.x, *beta);
  if (flip != (e < 0)) f_neg(q.y, q.y);
  jac_madd(acc, acc, q);
}

// Q = s B + h N for s, h < r; btab = 1..8 B, ntab = 1..8 N (N = -public)
template <class CV>
B2K_D void schnorr_equation(Jac<typename CV::F>& Q, const Scalar256& s, const Scalar256& h, const Affine<typename CV::F>* btab,
                            const Affine<typename CV::F>* ntab) {
  using F = typename CV::F;
  jac_set_inf(Q);
  if constexpr (CV::OUT_BYTES == 48) {
    // k P = +-k1 P + k2 (-phi P): the second stream adds (beta x, -+y) of the table entry, as scalar_mul_glv_bls381
    GlvSplit gs, gh;
    glv_split_bls381(gs, s);
    glv_split_bls381(gh, h);
    SignedW4<4> s1, s2, h1, h2;
    s1.init(gs.k1.v); s2.init(gs.k2.v); h1.init(gh.k1.v); h2.init(gh.k2.v);
    F beta;
    for (int j = 0; j < F::N; j++) beta.v[j] = Bls381Fp::beta(j);
    for (int i = 32; i >= 0; i--) {
      if (i != 32) { jac_dbl(Q, Q); jac_dbl(Q, Q); jac_dbl(Q, Q); jac_dbl(Q, Q); }
      schnorr_add_digit(Q, btab, s1.next(), gs.neg1, (const F*)nullptr);
      schnorr_add_digit(Q, btab, s2.next(), !gs.neg2, &beta);
      schnorr_add_digit(Q, ntab, h1.next(), gh.neg1, (const F*)nullptr);
      schnorr_add_digit(Q, ntab, h2.next(), !gh.neg2, &beta);
    }
  } else {
    SignedW4<8> ds, dh;
    ds.init(s.v); dh.init(h.v);
    for (int i = 64; i >= 0; i--) {
      if (i != 64) { jac_dbl(Q, Q); jac_dbl(Q, Q); jac_dbl(Q, Q); jac_dbl(Q, Q); }
      schnorr_add_digit(Q, btab, ds.next(), false, (const F*)nullptr);
      schnorr_add_digit(Q, ntab, dh.next(), false, (const F*)nullptr);
    }
  }
}

// VerifyWithChecks(g, pk, msg, sig) for one signature of CV::OUT_BYTES + 32 bytes (R || s): SCHNORR_OK or the first failing
// check; btab = 1..8 B (schnorr_base_table)
template <class CV, class INV>
B2K_D int schnorr_verify(const uint8_t* pk, const uint8_t* msg, uint32_t mlen, const uint8_t* sig, const Affine<typename CV::F>* btab,
                         INV inv_fn) {
  using F = typename CV::F;
  constexpr int PL = CV::OUT_BYTES;
  Affine<F> R, A;
  bool ok;
  if constexpr (PL == 48) ok = g1_decompress(R, sig, true);
  else ok = g2_decompress(R, sig, true);
  if (!ok) return SCHNORR_R;
  Scalar256 s, h;
  scalar_load_be(s, sig + PL);
  if (!scalar_in_range<Bls381Fr>(s)) return SCHNORR_S;
  if constexpr (PL == 48) ok = g1_decompress(A, pk, true);
  else ok = g2_decompress(A, pk, true);
  if (!ok) return SCHNORR_PK;
  uint64_t hs[8];
  sha512_3(hs, sig, PL, pk, PL, msg, mlen);             // SHA-512(R || public || msg), schnorr.go:163-178
  fr_from_be512(h, hs);
  Affine<F> ntab[8];                                   // k (-public), k = 1..8: indexed at run time (local memory)
  f_neg(A.y, A.y);                                      // -O = O: (0, 0) stays (0, 0)
  schnorr_table8(ntab, A, inv_fn);
  Jac<F> Q;
  schnorr_equation<CV>(Q, s, h, btab, ntab);
  return jac_eq_affine(Q, R) ? SCHNORR_OK : SCHNORR_INVALID;
}

}  // namespace b2k
