// anon.cuh -- ring signature verification (sign/anon) on edwards25519: the per-thread bodies of the verifier.
//
// Replaces (reference):
//   anon.Verify               sign/anon/sig.go:192-248                                         -> the kernels of b2k_anon.cu
//   signH1pre / signH1        sig.go:24-46 (blake2xb.New(message), Write(scope), Write(tag); Clone, Write(PG [, PH]), Pick)
//                                                                                              -> anon_h1pre, anon_h1
//   Point.Pick = Embed(nil)   group/edwards25519/point.go:132-182                              -> anon_link_base
//   geScalarMultBase          group/edwards25519/ge.go:373-417 (over a table of any base)     -> ed_comb_table_column, ed_comb
// Scalars (C0, S_i) are read raw, as UnmarshalBinary leaves them: every multiplication keeps geScalarMult's top-digit rule (a
// top signed nibble above 8 selects nothing).  The ring's fixed bases (B, the link base H and the ring keys) are multiplied by
// geScalarMultBase's own schedule over a 32-row table per base: row j holds k 256^j P (k = 1..8) in cached form; the odd digits
// are added first, then 4 doublings, then the even digits.  That is the same group sum as geScalarMult's, torsion included.
// The challenge comparison is Scalar.Equal (pvss_challenge_is): the raw bytes of C0 against the final c.  What is hashed is
// the canonical encoding of every point, the tag included.
#pragma once
#include "ed25519.cuh"
#include "blake2b.cuh"

namespace b2k {

enum { ANON_OK = 0, ANON_INVALID = 1, ANON_POINT = 2 };
constexpr int ANON_ROWS = 32;                               // table rows per base; a table is 32 x 8 EdCached = 32 KiB
constexpr int ANON_LINK_TRIES = 256;                        // 32-byte chunks tried for the link base (each is a point w.p. ~1/2)

// ---- the comb over a fixed base ---------------------------------------------------------------------------------------------
// column k of P's table (k = 1..8, one thread per k): tab[8 j + k - 1] = cached(k 256^j P) for j = 0..31
B2K_D void ed_comb_table_column(EdCached* tab, uint32_t k, const EdExt& P) {
  EdExt Q = P;
  for (uint32_t i = 1; i < k; i++) ed_add(Q, Q, P);
  for (int j = 0; j < ANON_ROWS; j++) {
    ed_to_cached(tab[8 * j + k - 1], Q);
    if (j + 1 < ANON_ROWS) {
      for (int d = 0; d < 7; d++) ed_dbl_xyz(Q, Q);
      ed_dbl(Q, Q);
    }
  }
}

// Q = geScalarMultBase(a) over table ta + the same over table tb for b (tb may be null): one joint pass, at most 128 table
// additions and 4 doublings
B2K_D void ed_comb(EdExt& Q, const uint32_t* a, const EdCached* ta, const uint32_t* b, const EdCached* tb) {
  int8_t ea[64], eb[64];
  sc_recode4(ea, a);
  if (tb) sc_recode4(eb, b);
  ed_set_identity(Q);
  for (int i = 1; i < 64; i += 2) {
    ed_digit_add(Q, ta + 8 * (i >> 1), ea[i]);
    if (tb) ed_digit_add(Q, tb + 8 * (i >> 1), eb[i]);
  }
  ed_dbl_xyz(Q, Q); ed_dbl_xyz(Q, Q); ed_dbl_xyz(Q, Q); ed_dbl(Q, Q);
  for (int i = 0; i < 64; i += 2) {
    ed_digit_add(Q, ta + 8 * (i >> 1), ea[i]);
    if (tb) ed_digit_add(Q, tb + 8 * (i >> 1), eb[i]);
  }
}

// ---- hashing ----------------------------------------------------------------------------------------------------------------
// H1pre = blake2xb.New(message), then Write(scope) and Write(tag) when linkable (tag: canonical, or null)
B2K_D void anon_h1pre(Blake2bMid& s, const uint8_t* msg, uint32_t mlen, const uint8_t* scope, uint32_t slen, const uint8_t* tag) {
  blake2xb_begin(s, msg, mlen);
  if (tag) {
    blake2b_absorb(s, scope, slen);
    blake2b_absorb(s, tag, 32);
  }
}

// c = Pick(H1pre.Clone() || pg [|| ph]) (ph null when unlinkable)
B2K_D void anon_h1(uint32_t* c, const Blake2bMid& pre, const uint8_t* pg, const uint8_t* ph) {
  Blake2bMid s = pre;
  blake2b_absorb(s, pg, 32);
  if (ph) blake2b_absorb(s, ph, 32);
  uint64_t h0[8];
  blake2b_finish(h0, s);
  sc_pick_root(c, h0);
}

// Point.Pick(blake2xb.New(scope)): consecutive 32-byte chunks of the stream; a chunk that does not decode is skipped, the point
// is multiplied by the cofactor (geScalarMult(8): three doublings) and a product equal to the identity is skipped too.  Returns
// false if none of ANON_LINK_TRIES chunks gives a point (probability about 2^-256).
B2K_D bool anon_link_base(uint8_t* out, const uint8_t* scope, uint32_t slen) {
  uint64_t h0[8], blk[8];
  blake2xb_root(h0, scope, slen);
  for (int i = 0; i < ANON_LINK_TRIES / 2; i++) {
    blake2xb_block(blk, h0, (uint32_t)i);
    for (int half = 0; half < 2; half++) {
      uint8_t b[32];
      for (int j = 0; j < 32; j++) b[j] = (uint8_t)(blk[4 * half + (j >> 3)] >> (8 * (j & 7)));
      EdExt P;
      if (!ed_decode(P, b)) continue;
      ed_dbl(P, P); ed_dbl(P, P); ed_dbl(P, P);
      EFp zero;
      fp_set_zero(zero);
      if (fp_eq(P.X, zero) && fp_eq(P.Y, P.Z)) continue;
      ed_encode(out, P);
      return true;
    }
  }
  return false;
}

// ---- one ring position ------------------------------------------------------------------------------------------------------
// c <- H1(s B + c L [, s H + c Tag]): tb, tl, th the tables of B, L_i and H (th null when unlinkable), tagtab 1..8 Tag
B2K_D void anon_ring_step(uint32_t* c, const uint32_t* s, const EdCached* tb, const EdCached* tl, const EdCached* th,
                          const EdCached* tagtab, const Blake2bMid& pre) {
  EdExt PG, PH;
  ed_comb(PG, s, tb, c, tl);
  uint8_t pg[32], ph[32];
  if (th) {
    EdExt T;
    ed_comb(PH, s, th, nullptr, nullptr);
    ed_mul_digits(T, c, tagtab);
    ed_add(PH, PH, T);
    EFp zi, zg, zh;                                         // one inversion for both (Montgomery's trick)
    fp_mul(zi, PG.Z, PH.Z);
    fp_inv(zi, zi);
    fp_mul(zg, zi, PH.Z);
    fp_mul(zh, zi, PG.Z);
    EdExt a;
    fp_mul(a.X, PG.X, zg); fp_mul(a.Y, PG.Y, zg);
    ed_encode_z1(pg, a);
    fp_mul(a.X, PH.X, zh); fp_mul(a.Y, PH.Y, zh);
    ed_encode_z1(ph, a);
  } else {
    ed_encode(pg, PG);
  }
  anon_h1(c, pre, pg, th ? ph : nullptr);
}

}  // namespace b2k
