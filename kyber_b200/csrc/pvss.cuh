// pvss.cuh -- DLEQ proof verification and the PVSS share checks on edwards25519, one proof per thread.
//
// Replaces (reference):
//   dleq.Proof.Verify            proof/dleq/dleq.go:161-172                                       -> dleq_holds
//   Scalar.Pick(blake2xb.New(seed))                                                               -> sc_pick (blake2b.cuh)
//   computeGlobalChallenge       share/pvss/pvss.go:116-149 (coms by ed_pubpoly_horner at the position i + 1)
//   VerifyEncShare               pvss.go:154-163                                                  -> pvss_enc_share
//   VerifyDecShare               pvss.go:248-277                                                  -> pvss_dec_share
//
// Scalars C and R are read raw, as Point.Mul reads them (geScalarMult, no reduction mod l; a top signed nibble above 8 selects
// nothing: ed_double_mul_var), so the points' torsion parts count exactly as in the reference.  The challenge comparison is
// Scalar.Equal (pvss_challenge_is): the raw 32 bytes of C against the little-endian bytes of the picked scalar.  What is hashed is
// MarshalTo of the DECODED points, i.e. their canonical encodings, never the input bytes.  Points are compared projectively
// against the decoded (Z = 1) commitments.
// Statuses (DLEQ_*, the values of B2K_DLEQ_* in include/b2kyber.h) follow the reference's order: an operand that does not decode
// first, then the challenge, then the two equations.
#pragma once
#include "ed25519.cuh"
#include "blake2b.cuh"
#include "sha256.cuh"

namespace b2k {

enum { DLEQ_OK = 0, DLEQ_CHALLENGE = 1, DLEQ_INVALID = 2, DLEQ_POINT = 3 };

// ---- proofs ----------------------------------------------------------------------------------------------------------------
// the operands of dleq.Proof.Verify(G, H, xG, xH) and the proof's VG, VH, decoded (Z = 1)
struct DleqPoints { EdExt G, H, xG, xH, VG, VH; };

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
