// pvss.cuh -- DLEQ proof verification and the PVSS share checks on edwards25519, one proof per thread.
//
// Replaces (reference):
//   dleq.Proof.Verify            proof/dleq/dleq.go:161-172                                       -> dleq_holds
//   blake2xb.New(seed)           xof/blake2xb/blake.go:19-41 (blake2b.NewXOF(unknown, seed[:64]) + Write(seed[64:]))
//                                                                                                 -> blake2xb_root, blake2xb_block
//   Scalar.Pick                  group/edwards25519/scalar.go:180-185 -> random.Int(l), util/random/rand.go:19-46 -> sc_pick
//   computeGlobalChallenge       share/pvss/pvss.go:116-149 (coms by ed_pubpoly_horner at the position i + 1)
//   VerifyEncShare               pvss.go:154-163                                                  -> pvss_enc_share
//   VerifyDecShare               pvss.go:248-277                                                  -> pvss_dec_share
//
// Scalars C and R are read raw, as Point.Mul reads them (geScalarMult, no reduction mod l; a top signed nibble above 8 selects
// nothing), so the points' torsion parts count exactly as in the reference.  The challenge comparison is Scalar.Equal: the raw
// 32 bytes of C against the little-endian bytes of the picked scalar.  What is hashed is MarshalTo of the DECODED points, i.e.
// their canonical encodings, never the input bytes.  Points are compared projectively against the decoded (Z = 1) commitments.
// Statuses (DLEQ_*, the values of B2K_DLEQ_* in include/b2kyber.h) follow the reference's order: an operand that does not decode
// first, then the challenge, then the two equations.
#pragma once
#include "ed_msm.cuh"
#include "sha256.cuh"

namespace b2k {

enum { DLEQ_OK = 0, DLEQ_CHALLENGE = 1, DLEQ_INVALID = 2, DLEQ_POINT = 3 };

// ---- BLAKE2b (RFC 7693) and BLAKE2Xb ------------------------------------------------------------------------------------
// host-callable too (B2K_HD): the shuffle verifier runs its Fiat-Shamir transcript on host threads with this same code
struct Blake2bSigma {
  B2K_HD static int s(int r, int i) {
    constexpr uint8_t t[10][16] = {{0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
                                   {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
                                   {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
                                   {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
                                   {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0}};
    return t[r % 10][i];
  }
  B2K_HD static uint64_t iv(int j) {                    // BLAKE2b's IV is SHA-512's
    constexpr uint64_t t[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                               0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
    return t[j];
  }
};

B2K_HD void blake2b_g(uint64_t* v, int a, int b, int c, int d, uint64_t x, uint64_t y) {
  v[a] = v[a] + v[b] + x; v[d] = sha_rotr(v[d] ^ v[a], 32);
  v[c] = v[c] + v[d]; v[b] = sha_rotr(v[b] ^ v[c], 24);
  v[a] = v[a] + v[b] + y; v[d] = sha_rotr(v[d] ^ v[a], 16);
  v[c] = v[c] + v[d]; v[b] = sha_rotr(v[b] ^ v[c], 63);
}

// one compression of the 16 little-endian message words m; t = bytes hashed so far including this block (< 2^64 here)
B2K_HNI void blake2b_compress(uint64_t* h, const uint64_t* m, uint64_t t, bool last) {
  uint64_t v[16];
#pragma unroll
  for (int i = 0; i < 8; i++) { v[i] = h[i]; v[i + 8] = Blake2bSigma::iv(i); }
  v[12] ^= t;
  if (last) v[14] = ~v[14];
#pragma unroll
  for (int r = 0; r < 12; r++) {
    blake2b_g(v, 0, 4, 8, 12, m[Blake2bSigma::s(r, 0)], m[Blake2bSigma::s(r, 1)]);
    blake2b_g(v, 1, 5, 9, 13, m[Blake2bSigma::s(r, 2)], m[Blake2bSigma::s(r, 3)]);
    blake2b_g(v, 2, 6, 10, 14, m[Blake2bSigma::s(r, 4)], m[Blake2bSigma::s(r, 5)]);
    blake2b_g(v, 3, 7, 11, 15, m[Blake2bSigma::s(r, 6)], m[Blake2bSigma::s(r, 7)]);
    blake2b_g(v, 0, 5, 10, 15, m[Blake2bSigma::s(r, 8)], m[Blake2bSigma::s(r, 9)]);
    blake2b_g(v, 1, 6, 11, 12, m[Blake2bSigma::s(r, 10)], m[Blake2bSigma::s(r, 11)]);
    blake2b_g(v, 2, 7, 8, 13, m[Blake2bSigma::s(r, 12)], m[Blake2bSigma::s(r, 13)]);
    blake2b_g(v, 3, 4, 9, 14, m[Blake2bSigma::s(r, 14)], m[Blake2bSigma::s(r, 15)]);
  }
#pragma unroll
  for (int i = 0; i < 8; i++) h[i] ^= v[i] ^ v[i + 8];
}

// h = IV xor the parameter block, whose words 0..2 are given (the rest is zero in every use here)
B2K_HD void blake2b_init(uint64_t* h, uint64_t p0, uint64_t p1, uint64_t p2) {
#pragma unroll
  for (int i = 0; i < 8; i++) h[i] = Blake2bSigma::iv(i);
  h[0] ^= p0; h[1] ^= p1; h[2] ^= p2;
}

// A BLAKE2b midstate: the chaining value h, the bytes compressed so far t, and the pending block m of n <= 128 bytes (little-
// endian words).  A full block is compressed only when more input arrives, so the last block can still take the final flag.
struct Blake2bMid { uint64_t h[8]; uint64_t t; uint64_t m[16]; uint32_t n; };

B2K_HD void blake2b_absorb(Blake2bMid& s, const uint8_t* p, uint32_t len) {
  for (uint32_t k = 0; k < len; k++) {
    if (s.n == 128) {
      s.t += 128;
      blake2b_compress(s.h, s.m, s.t, false);
      for (int i = 0; i < 16; i++) s.m[i] = 0;
      s.n = 0;
    }
    s.m[s.n >> 3] |= (uint64_t)p[k] << (8 * (s.n & 7));
    s.n++;
  }
}

// the 64-byte digest (8 little-endian words) of everything absorbed: the pending block compressed as the last one
B2K_HD void blake2b_finish(uint64_t* out, const Blake2bMid& s) {
  uint64_t m[16];
  for (int i = 0; i < 16; i++) m[i] = s.m[i];
  for (int i = 0; i < 8; i++) out[i] = s.h[i];
  blake2b_compress(out, m, s.t + s.n, true);
}

// blake2xb.New(seed) as a midstate, to which XOF.Write appends (the same stream blake2xb_root hashes in one go)
B2K_HD void blake2xb_begin(Blake2bMid& s, const uint8_t* seed, uint32_t len) {
  const uint32_t klen = len < 64 ? len : 64;
  blake2b_init(s.h, 64u | (klen << 8) | (1u << 16) | (1u << 24), 0xffffffffull << 32, 0);
  s.t = 0;
  s.n = 0;
  for (int i = 0; i < 16; i++) s.m[i] = 0;
  blake2b_absorb(s, seed, klen);
  if (klen) s.n = 128;
  blake2b_absorb(s, seed + klen, len - klen);
}

// The root hash of blake2xb.New(seed): BLAKE2b-512 KEYED with seed[0, min(len, 64)) over the message seed[64, len), with
// fanout 1, depth 1 and the XOF length 2^32 - 1 (unknown) in the parameter block.  A key is hashed as a zero-padded first block.
B2K_D void blake2xb_root(uint64_t* h0, const uint8_t* seed, uint32_t len) {
  const uint32_t klen = len < 64 ? len : 64, mlen = len - klen;
  blake2b_init(h0, 64u | (klen << 8) | (1u << 16) | (1u << 24), 0xffffffffull << 32, 0);
  const uint32_t slen = klen ? 128 + mlen : 0;          // the stream hashed: the padded key block, then the message
  const uint32_t nblk = slen ? (slen + 127) / 128 : 1;
  for (uint32_t b = 0; b < nblk; b++) {
    uint64_t m[16];
    for (int i = 0; i < 16; i++) {
      uint64_t w = 0;
      for (int j = 7; j >= 0; j--) {
        const uint32_t pos = 128 * b + 8 * i + j;
        uint8_t byte = 0;
        if (pos < 128) { if (pos < klen) byte = seed[pos]; }
        else if (pos - 128 < mlen) byte = seed[64 + pos - 128];
        w = (w << 8) | byte;
      }
      m[i] = w;
    }
    blake2b_compress(h0, m, 128 * (b + 1) < slen ? 128 * (b + 1) : slen, b == nblk - 1);
  }
}

// output block i of the XOF (64 bytes as 8 little-endian words): unkeyed BLAKE2b-512 of the 64-byte root hash with the BLAKE2X
// node parameters: leaf length 64, node offset i, XOF length 2^32 - 1, inner length 64
B2K_HD void blake2xb_block(uint64_t* out, const uint64_t* h0, uint32_t i) {
  blake2b_init(out, 64ull | (64ull << 32), (uint64_t)i | (0xffffffffull << 32), 64ull << 8);
  uint64_t m[16];
#pragma unroll
  for (int j = 0; j < 8; j++) { m[j] = h0[j]; m[j + 8] = 0; }
  blake2b_compress(out, m, 64, true);
}

// Scalar.Pick of the XOF whose root hash is h0, as 8 little-endian limbs: random.Int(l) draws 32 stream bytes, clears the top 3
// bits of the first (l has 253 bits), reads them big-endian and draws again while the value is >= l.  An output block holds two
// draws.
B2K_D void sc_pick_root(uint32_t* s, const uint64_t* h0) {
  uint64_t blk[8];
  for (uint32_t i = 0;; i++) {
    blake2xb_block(blk, h0, i);
    for (int half = 0; half < 2; half++) {
#pragma unroll
      for (int j = 0; j < 8; j++) {                     // limb j holds draw bytes 31 - 4 j - q (q = 0..3) at bits 8 q
        uint32_t v = 0;
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const int p = 32 * half + 31 - 4 * j - q;
          v |= (uint32_t)((blk[p >> 3] >> (8 * (p & 7))) & 0xff) << (8 * q);
        }
        s[j] = v;
      }
      s[7] &= 0x1fffffffu;
      if (sc_is_canonical(s)) return;
    }
  }
}

// Scalar.Pick(blake2xb.New(seed)): the same draws from the root of the seed.  It keeps its own copy of the loop: written as
// blake2xb_root + sc_pick_root, the PVSS challenge kernels compiled for sm_90a (CUDA 12.9) produced different challenges on
// an H100, while the host build and a standalone kernel of the same code agreed with the reference.
B2K_D void sc_pick(uint32_t* s, const uint8_t* seed, uint32_t len) {
  uint64_t h0[8], blk[8];
  blake2xb_root(h0, seed, len);
  for (uint32_t i = 0;; i++) {
    blake2xb_block(blk, h0, i);
    for (int half = 0; half < 2; half++) {
#pragma unroll
      for (int j = 0; j < 8; j++) {
        uint32_t v = 0;
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const int p = 32 * half + 31 - 4 * j - q;
          v |= (uint32_t)((blk[p >> 3] >> (8 * (p & 7))) & 0xff) << (8 * q);
        }
        s[j] = v;
      }
      s[7] &= 0x1fffffffu;
      if (sc_is_canonical(s)) return;
    }
  }
}

// SHA-256 of nblk whole 64-byte blocks at p; digest (big-endian bytes) in out
B2K_D void sha256_blocks(uint8_t* out, const uint8_t* p, size_t nblk) {
  Sha256 s;
  sha256_init(s);
  for (size_t k = 0; k < nblk; k++) sha256_compress(s.h, p + 64 * k);
  s.total = 64 * nblk;
  sha256_final(s, out);
}

// Scalar.Equal(C, Pick(XOF(digest))): the raw bytes of C against the picked scalar
B2K_D bool pvss_challenge_is(const uint8_t* c_bytes, const uint32_t* want) {
  uint32_t c[8], o = 0;
  sc_load_le(c, c_bytes);
#pragma unroll
  for (int j = 0; j < 8; j++) o |= c[j] ^ want[j];
  return o == 0;
}

// ---- the joint multiplication over two variable bases ----------------------------------------------------------------------
// Q = geScalarMult(r, P) + geScalarMult(c, P2) for raw 256-bit r and c: one joint signed-4-bit double-and-add over the
// per-thread cached tables 1..8 P and 1..8 P2 (indexed at run time: local memory).  A digit above 8 (only the top one, e63, can
// be) selects nothing, as selectCached (ge.go:419-433) does, so the sum is exactly that of the two reference multiplications.
B2K_D void ed_double_mul_var(EdExt& Q, const uint32_t* r, const EdExt& P, const uint32_t* c, const EdExt& P2) {
  EdCached tp[8], tq[8];
  ed_cached_table(tp, P);
  ed_cached_table(tq, P2);
  int8_t er[64], ec[64];
  sc_recode4(er, r);
  sc_recode4(ec, c);
  ed_set_identity(Q);
  for (int i = 63; i >= 0; i--) {
    if (i != 63) { ed_dbl_xyz(Q, Q); ed_dbl_xyz(Q, Q); ed_dbl_xyz(Q, Q); ed_dbl(Q, Q); }
    const int dr = er[i], dc = ec[i];
    if (dr != 0 && dr <= 8) {
      const EdCached& t = tp[(dr < 0 ? -dr : dr) - 1];
      ed_add_cached(Q, Q, t.ypx, t.ymx, &t.z2, t.t2d, dr < 0);
    }
    if (dc != 0 && dc <= 8) {
      const EdCached& t = tq[(dc < 0 ? -dc : dc) - 1];
      ed_add_cached(Q, Q, t.ypx, t.ymx, &t.z2, t.t2d, dc < 0);
    }
  }
}

// ---- proofs ----------------------------------------------------------------------------------------------------------------
// the operands of dleq.Proof.Verify(G, H, xG, xH) and the proof's VG, VH, decoded (Z = 1)
struct DleqPoints { EdExt G, H, xG, xH, VG, VH; };

// p == Q for a decoded p (Z = 1): X_p Z_Q = X_Q and Y_p Z_Q = Y_Q
B2K_D bool ed_eq_z1(const EdExt& p, const EdExt& Q) {
  EFp t;
  fp_mul(t, p.X, Q.Z);
  if (!fp_eq(t, Q.X)) return false;
  fp_mul(t, p.Y, Q.Z);
  return fp_eq(t, Q.Y);
}

B2K_D bool dleq_decode_proof(DleqPoints& d, const uint8_t* proof) { return ed_decode(d.VG, proof + 64) && ed_decode(d.VH, proof + 96); }

// VG == R G + C xG and VH == R H + C xH (dleq.go:161-172); proof = C || R || VG || VH
B2K_D bool dleq_holds(const DleqPoints& d, const uint8_t* proof) {
  uint32_t c[8], r[8];
  sc_load_le(c, proof);
  sc_load_le(r, proof + 32);
  EdExt Q;
  ed_double_mul_var(Q, r, d.G, c, d.xG);
  if (!ed_eq_z1(d.VG, Q)) return false;
  ed_double_mul_var(Q, r, d.H, c, d.xH);
  return ed_eq_z1(d.VH, Q);
}

// dleq.Proof.Verify of one proof: DLEQ_POINT, DLEQ_INVALID or DLEQ_OK
B2K_D int dleq_verify_one(const uint8_t* g, const uint8_t* h, const uint8_t* xg, const uint8_t* xh, const uint8_t* proof) {
  DleqPoints d;
  if (!ed_decode(d.G, g) || !ed_decode(d.H, h) || !ed_decode(d.xG, xg) || !ed_decode(d.xH, xh) || !dleq_decode_proof(d, proof))
    return DLEQ_POINT;
  return dleq_holds(d, proof) ? DLEQ_OK : DLEQ_INVALID;
}

// The hashed points of share i of a deal (computeGlobalChallenge): slot 0 = coms[i] = sum_j (i + 1)^j C_j (computeCommitments,
// pvss.go:94-114: the POSITION i, not the share's index), slots 1..3 = V, VG, VH, each canonical, at out + k stride.  Returns
// false when V, VG or VH does not decode.
B2K_D bool pvss_hashed_points(uint8_t* out, size_t stride, const EdNiels* cm, uint32_t t, uint32_t i, const uint8_t* v,
                              const uint8_t* proof) {
  EdExt p;
  ed_pubpoly_horner(p, cm, t, (uint64_t)i + 1u);
  ed_encode(out, p);
  for (int k = 1; k < 4; k++) {
    if (!ed_decode(p, k == 1 ? v : proof + 32 * k)) return false;
    ed_encode_z1(out + k * stride, p);
  }
  return true;
}

// VerifyEncShare (pvss.go:154-163) of one share of a deal whose hashed points and H decoded: C against the deal's challenge,
// then Verify(H, X, sH, V)
B2K_D int pvss_enc_share(const uint8_t* h, const uint8_t* x, const uint8_t* sh, const uint8_t* v, const uint8_t* proof,
                         const uint32_t* chal) {
  DleqPoints d;                                         // G = H, H = X, xG = sH, xH = V
  if (!ed_decode(d.G, h) || !ed_decode(d.H, x) || !ed_decode(d.xG, sh) || !ed_decode(d.xH, v) || !dleq_decode_proof(d, proof))
    return DLEQ_POINT;
  if (!pvss_challenge_is(proof, chal)) return DLEQ_CHALLENGE;
  return dleq_holds(d, proof) ? DLEQ_OK : DLEQ_INVALID;
}

// VerifyDecShare (pvss.go:248-277) of one share: C against Pick(XOF(SHA-256(X || encV || VG || VH))), then
// Verify(G, decV, X, encV)
B2K_D int pvss_dec_share(const uint8_t* g, const uint8_t* x, const uint8_t* enc_v, const uint8_t* dec_v, const uint8_t* proof) {
  DleqPoints d;                                         // G = G, H = decV, xG = X, xH = encV
  if (!ed_decode(d.G, g) || !ed_decode(d.H, dec_v) || !ed_decode(d.xG, x) || !ed_decode(d.xH, enc_v) || !dleq_decode_proof(d, proof))
    return DLEQ_POINT;
  uint8_t buf[128], dig[32];
  ed_encode_z1(buf, d.xG); ed_encode_z1(buf + 32, d.xH); ed_encode_z1(buf + 64, d.VG); ed_encode_z1(buf + 96, d.VH);
  sha256_blocks(dig, buf, 2);
  uint32_t want[8];
  sc_pick(want, dig, 32);
  if (!pvss_challenge_is(proof, want)) return DLEQ_CHALLENGE;
  return dleq_holds(d, proof) ? DLEQ_OK : DLEQ_INVALID;
}

}  // namespace b2k
