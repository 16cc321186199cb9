// shuffle.cuh -- Neff's verifiable shuffle of ElGamal pairs on edwards25519: the per-thread bodies of the verifier.
//
// Replaces (reference):
//   PairShuffle.Verify        shuffle/pair.go:239-312 (step 7: Phi1, Phi2 and the checks (33), (34), (35))
//   SimpleShuffle.Verify      shuffle/simple.go:186-254 (U, W, Xhat, Yhat and the 2k thver checks)
//   thver                     simple.go:178-183                                             -> shuffle_thver
//   GetSequenceVerifiable     shuffle/sequences.go:155-190                                  -> shuffle_sequence_term
// The Fiat-Shamir transcript (proof.HashVerify, proof/hash.go:92-175) runs on the host (b2k_shuffle.cu); the device gets t, c and
// Zrho as canonical little-endian scalars.  Scalars read from the proof (Zsigma, Ztau, Zalpha) are raw 256-bit integers, as
// UnmarshalBinary leaves them (scalar.go:226-232): every multiplication by them keeps geScalarMult's top-digit rule
// (ed_double_mul_var, ed_mul_var).  thver negates its scalar b mod l (Neg = scSub(0, b), scalar.go:119-128); Phi's Sub negates the
// POINT (point.go:209-221), which differs from negating the scalar when X has a torsion part.  Equality is exact point equality.
// G or H absent means the base point: geScalarMultBase drops a top digit above 8 exactly as geScalarMult does, so the base is
// just another variable base here.
#pragma once
#include "ed25519.cuh"

namespace b2k {

enum { SHUF_OK = 0, SHUF_SIMPLE = 1, SHUF_PAIR = 2, SHUF_POINT = 3 };
enum { SHUF_F_POINT = 0, SHUF_F_SIMPLE = 1, SHUF_F_PAIR = 2 };   // per-shuffle flag bytes flags[4 s + f]

// ---- the proof: fixbuf encodings of ega1, ega3, ega5, ssa0, ssa2, ssa4 in that order, 32-byte items ----------------------
//   ega1  Gamma, A[k], C[k], U[k], W[k], Lambda1, Lambda2       items [0, 4k + 3)
//   ega3  D[k]                                                  [4k + 3, 5k + 3)
//   ega5  Zsigma[k], Ztau                                       [5k + 3, 6k + 4)
//   ssa0  X[k], Y[k]                                            [6k + 4, 8k + 4)
//   ssa2  Theta[2k]                                             [8k + 4, 10k + 4)
//   ssa4  Zalpha[2k - 1]                                        [10k + 4, 12k + 3)
struct ShufItems {
  B2K_HD static uint64_t total(uint64_t k) { return 12 * k + 3; }
  B2K_HD static uint64_t w(uint64_t k, uint64_t i) { return 3 * k + 1 + i; }
  B2K_HD static uint64_t lambda1(uint64_t k) { return 4 * k + 1; }
  B2K_HD static uint64_t lambda2(uint64_t k) { return 4 * k + 2; }
  B2K_HD static uint64_t d(uint64_t k, uint64_t i) { return 4 * k + 3 + i; }
  B2K_HD static uint64_t zsigma(uint64_t k, uint64_t i) { return 5 * k + 3 + i; }
  B2K_HD static uint64_t ztau(uint64_t k) { return 6 * k + 3; }
  B2K_HD static uint64_t x(uint64_t k, uint64_t i) { return 6 * k + 4 + i; }
  B2K_HD static uint64_t y(uint64_t k, uint64_t i) { return 7 * k + 4 + i; }
  B2K_HD static uint64_t theta(uint64_t k, uint64_t i) { return 8 * k + 4 + i; }
  B2K_HD static uint64_t zalpha(uint64_t k, uint64_t i) { return 10 * k + 4 + i; }
  B2K_HD static bool is_point(uint64_t k, uint64_t j) { return !(j >= 5 * k + 3 && j < 6 * k + 4) && j < 10 * k + 4; }
};

// thver(A, B, T, a, b): a A + Neg(b) B == T, a raw, b negated mod l, T decoded
B2K_D bool shuffle_thver(const EdExt& A, const EdExt& B, const EdAff& T, const uint32_t* a, const uint32_t* b) {
  uint32_t nb[8];
  sc_neg_mod_l(nb, b);
  EdExt Q;
  ed_double_mul_var(Q, a, A, nb, B);
  return ed_eq_aff(T, Q);
}

// thver number i (0 <= i < 2k) of SimpleShuffle.Verify: (Xhat_i, Yhat_i) for i < k, else (Gamma, G); a = c for i = 0, else
// Zalpha[i - 1]; b = c for i = 2k - 1, else Zalpha[i].  pp: the shuffle's decoded proof items, proof: its bytes, U = -t G,
// W = -t Gamma, c: the challenge (8 limbs)
B2K_D bool shuffle_thver_i(uint32_t k, uint32_t i, const EdAff* pp, const uint8_t* proof, const EdExt& U, const EdExt& W,
                           const EdAff& G, const uint32_t* c) {
  EdExt A, B;
  if (i < k) {
    ed_from_aff(A, pp[ShufItems::x(k, i)]); ed_add(A, A, U);
    ed_from_aff(B, pp[ShufItems::y(k, i)]); ed_add(B, B, W);
  } else {
    ed_from_aff(A, pp[0]);
    ed_from_aff(B, G);
  }
  uint32_t a[8], b[8];
  if (i == 0) {
#pragma unroll
    for (int j = 0; j < 8; j++) a[j] = c[j];
  } else {
    sc_load_le(a, proof + 32 * ShufItems::zalpha(k, i - 1));
  }
  if (i == 2 * k - 1) {
#pragma unroll
    for (int j = 0; j < 8; j++) b[j] = c[j];
  } else {
    sc_load_le(b, proof + 32 * ShufItems::zalpha(k, i));
  }
  return shuffle_thver(A, B, pp[ShufItems::theta(k, i)], a, b);
}

// (33): Zsigma_i Gamma == W_i + D_i, evaluated as Zsigma_i Gamma + (-D_i) == W_i (the same group equation)
B2K_D bool shuffle_check33(uint32_t k, uint32_t i, const EdAff* pp, const uint8_t* proof) {
  uint32_t zs[8];
  sc_load_le(zs, proof + 32 * ShufItems::zsigma(k, i));
  EdExt Gm, Q, D;
  ed_from_aff(Gm, pp[0]);
  ed_mul_var(Q, zs, Gm);
  ed_from_aff(D, pp[ShufItems::d(k, i)]);
  ed_neg(D);
  ed_add(Q, Q, D);
  return ed_eq_aff(pp[ShufItems::w(k, i)], Q);
}

// the i-th terms of (31) and (32): Zsigma_i Xbar_i - Zrho_i X_i and Zsigma_i Ybar_i - Zrho_i Y_i, as Zsigma_i Xbar_i +
// Zrho_i (-X_i) (Sub negates the point)
B2K_D void shuffle_phi_terms(EdExt& t1, EdExt& t2, const uint32_t* zsigma, const uint32_t* zrho, const EdAff& x, const EdAff& y,
                             const EdAff& xbar, const EdAff& ybar) {
  EdExt P, N;
  ed_from_aff(P, xbar); ed_from_aff(N, x); ed_neg(N);
  ed_double_mul_var(t1, zsigma, P, zrho, N);
  ed_from_aff(P, ybar); ed_from_aff(N, y); ed_neg(N);
  ed_double_mul_var(t2, zsigma, P, zrho, N);
}

// (34) / (35): Lambda + Ztau G == Phi
B2K_D bool shuffle_check34(const EdAff& lambda, const uint32_t* ztau, const EdAff& G, const EdExt& phi) {
  EdExt Q, L, B;
  ed_from_aff(B, G);
  ed_mul_var(Q, ztau, B);
  ed_from_aff(L, lambda);
  ed_add(Q, Q, L);
  return ed_eq(Q, phi);
}

B2K_D uint8_t shuffle_status(const uint8_t* f) {
  return f[SHUF_F_POINT] ? (uint8_t)SHUF_POINT : f[SHUF_F_SIMPLE] ? (uint8_t)SHUF_SIMPLE : f[SHUF_F_PAIR] ? (uint8_t)SHUF_PAIR
                                                                                                           : (uint8_t)SHUF_OK;
}

// GetSequenceVerifiable, one output point: sum_j e[j] P[j] over the nq rows (P[j] = pts[j * stride]), two rows per joint
// multiplication
B2K_D void shuffle_sequence_term(EdExt& acc, uint32_t nq, const EdAff* pts, size_t stride, const uint8_t* e) {
  ed_set_identity(acc);
  uint32_t j = 0;
  for (; j + 1 < nq; j += 2) {
    uint32_t e0[8], e1[8];
    sc_load_le(e0, e + 32 * (size_t)j);
    sc_load_le(e1, e + 32 * (size_t)(j + 1));
    EdExt P0, P1, Q;
    ed_from_aff(P0, pts[j * stride]);
    ed_from_aff(P1, pts[(j + 1) * stride]);
    ed_double_mul_var(Q, e0, P0, e1, P1);
    ed_add(acc, acc, Q);
  }
  if (j < nq) {
    uint32_t e0[8];
    sc_load_le(e0, e + 32 * (size_t)j);
    EdExt P0, Q;
    ed_from_aff(P0, pts[j * stride]);
    ed_mul_var(Q, e0, P0);
    ed_add(acc, acc, Q);
  }
}

}  // namespace b2k
