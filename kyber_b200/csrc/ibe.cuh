// ibe.cuh -- per-thread bodies of Boneh-Franklin IBE (CCA) on BLS12-381, and the Miller loop against one fixed G2 point.
//
// Replaces (reference call sites):
//   EncryptCCAonG1 / DecryptCCAonG1     encrypt/ibe/ibe.go:51-134   (U on G1, identities and private keys on G2)
//   EncryptCCAonG2 / DecryptCCAonG2     encrypt/ibe/ibe.go:148-231  (U on G2, identities and private keys on G1)
//   h3 / h4 / gtToHash                  encrypt/ibe/ibe.go:234-309
// With Hash = SHA-256 (the suite's s.Hash()):
//   H2(gt)          = SHA256("IBE-H2" || GT.MarshalBinary)[:len]            (gt_store, 576 B)
//   H4(sigma)       = SHA256("IBE-H4" || sigma)[:len]
//   H3(sigma, msg)  : buf = SHA256("IBE-H3" || sigma || msg); for i = 1 .. 65534: h = SHA256(LE16(i) || buf), h[0] >>= 1,
//                     the first h below r (big-endian) is the scalar.  The shift is 256 - 255 bits; both BLS12-381 back-ends of
//                     the reference read scalars big-endian.
#pragma once
#include "codec.cuh"
#include "msm.cuh"
#include "sha256.cuh"

namespace b2k {

constexpr uint32_t IBE_MAX_LEN = 32;                       // s.Hash().Size()
enum : uint8_t { IBE_OK = 0, IBE_PROOF = 1, IBE_POINT = 2 };  // B2K_IBE_* of include/b2kyber.h

B2K_D void ibe_tagged_hash(uint8_t out[32], char tag_digit, const uint8_t* a, uint32_t alen, const uint8_t* b, uint32_t blen) {
  const uint8_t tag[6] = {'I', 'B', 'E', '-', 'H', (uint8_t)tag_digit};
  Sha256 s;
  sha256_init(s);
  sha256_update(s, tag, 6);
  sha256_update(s, a, alen);
  sha256_update(s, b, blen);
  sha256_final(s, out);
}
B2K_D void ibe_h2(uint8_t out[32], const uint8_t* gt576) { ibe_tagged_hash(out, '2', gt576, 576, nullptr, 0); }
B2K_D void ibe_h4(uint8_t out[32], const uint8_t* sigma, uint32_t len) { ibe_tagged_hash(out, '4', sigma, len, nullptr, 0); }

// r = H3(sigma, msg); false when all 65534 candidates are >= r (the reference's "rejection sampling failure")
B2K_D bool ibe_h3(Scalar256& r, const uint8_t* sigma, const uint8_t* msg, uint32_t len) {
  uint8_t buf[32], h[32];
  ibe_tagged_hash(buf, '3', sigma, len, msg, len);
  for (uint32_t i = 1; i < 65535u; i++) {
    const uint8_t it[2] = {(uint8_t)i, (uint8_t)(i >> 8)};
    Sha256 s;
    sha256_init(s);
    sha256_update(s, it, 2);
    sha256_update(s, buf, 32);
    sha256_final(s, h);
    h[0] >>= 1;
    scalar_load_be(r, h);
    if (scalar_in_range<Bls381Fr>(r)) return true;
  }
  return false;
}

// r Base with the device code of PriPoly.Commit's batch (k_commit_batch, b2k_share2.cu): GLV on G1, signed windows on G2
template <class CV, class INV>
B2K_D void ibe_base_mul(Jac<typename CV::F>& r, const Scalar256& k, INV inv_fn) {
  Affine<typename CV::F> g;
  CV::generator(g);
  if constexpr (CV::OUT_BYTES == 48) scalar_mul_glv_bls381(r, k, g, inv_fn);
  else scalar_mul_w4<CV>(r, k, g, inv_fn);
}

// DecryptCCAonG1/G2 steps 1-3 for one ciphertext, after the pairing: gt = e(U, private) (or e(private, U)) as 576 bytes, U the
// decoded point (u_ok false: it did not decode).  Writes msg (zeroed unless OK) and returns the IBE_* status.
template <class CV, class INV>
B2K_D uint8_t ibe_decrypt_finish(uint8_t* msg_out, const uint8_t* gt, const Affine<typename CV::F>& U, bool u_ok, const uint8_t* v,
                                 const uint8_t* w, uint32_t len, INV inv_fn) {
  uint8_t sigma[IBE_MAX_LEN], m[IBE_MAX_LEN], h[32];
  uint8_t st = IBE_POINT;
  if (u_ok) {
    ibe_h2(h, gt);
    for (uint32_t i = 0; i < len; i++) sigma[i] = v[i] ^ h[i];
    ibe_h4(h, sigma, len);
    for (uint32_t i = 0; i < len; i++) m[i] = w[i] ^ h[i];
    Scalar256 r;
    st = IBE_PROOF;
    if (ibe_h3(r, sigma, m, len)) {
      Jac<typename CV::F> rp;
      ibe_base_mul<CV>(rp, r, inv_fn);
      if (jac_eq_affine(rp, U)) st = IBE_OK;
    }
  }
  for (uint32_t i = 0; i < len; i++) msg_out[i] = st == IBE_OK ? m[i] : 0;
  return st;
}

// EncryptCCAonG1/G2 steps 3, 4 and 6 for one message: r = H3(sigma, msg) (32 B big-endian, the exponent of Gid), U = r Base
// (compressed), W = msg xor H4(sigma).  False when H3 finds no scalar.
template <class CV, class INV>
B2K_D bool ibe_encrypt_body(uint8_t* u_out, uint8_t* r_out, uint8_t* w_out, const uint8_t* msg, const uint8_t* sigma, uint32_t len,
                            INV inv_fn) {
  using F = typename CV::F;
  Scalar256 r;
  const bool ok = ibe_h3(r, sigma, msg, len);
  if (!ok) for (int j = 0; j < 8; j++) r.v[j] = 0;
  Jac<F> rp;
  ibe_base_mul<CV>(rp, r, inv_fn);
  Affine<F> a;
  if (jac_is_inf(rp)) aff_set_inf(a);
  else {
    F zi, zi2;
    inv_fn(zi, rp.Z);
    f_sqr(zi2, zi);
    f_mul(a.x, rp.X, zi2);
    f_mul(zi2, zi2, zi);
    f_mul(a.y, rp.Y, zi2);
  }
  CV::store(u_out, a);
  for (int j = 0; j < 8; j++) {
    const uint32_t x = r.v[7 - j];
    r_out[4 * j] = (uint8_t)(x >> 24); r_out[4 * j + 1] = (uint8_t)(x >> 16); r_out[4 * j + 2] = (uint8_t)(x >> 8); r_out[4 * j + 3] = (uint8_t)x;
  }
  uint8_t h[32];
  ibe_h4(h, sigma, len);
  for (uint32_t i = 0; i < len; i++) w_out[i] = msg[i] ^ h[i];
  return ok;
}

// ---- Miller loop against a fixed G2 point ----------------------------------------------------------------------------------
// In the lines of pairing.cuh only l2 and l3 depend on P, each as (a G2 quantity) x (a coordinate of P): l2 = c2 xP, l3 = c3 yP.
// With Q fixed, T's doublings and additions and (l0, c2, c3) are the same for every P: walked once (miller_fixed_q_table, by the
// unchanged step functions evaluated at xP = yP = 1), each P then pays only f^2 and the sparse product per step.
struct BlsLineCoef { BFp2 l0, c2, c3; };
constexpr int BLS_MILLER_STEPS = 68;                        // 63 doublings + 5 additions (the set bits of |x| below the top one)

B2K_D void miller_fixed_q_table(BlsLineCoef* tab, const Affine<BFp2>& Q) {
  Affine<BFp> one;
  fp_set_one(one.x); fp_set_one(one.y);
  Jac<BFp2> T;
  T.X = Q.x; T.Y = Q.y; fp2_set_one(T.Z);
  BlsLine l;
  int s = 0;
  for (int b = 62; b >= 0; b--) {
    miller_double_step(l, T, one);
    tab[s].l0 = l.l0; tab[s].c2 = l.l2; tab[s].c3 = l.l3; s++;
    if ((BLS_X_ABS >> b) & 1) {
      miller_add_step(l, T, Q, one);
      tab[s].l0 = l.l0; tab[s].c2 = l.l2; tab[s].c3 = l.l3; s++;
    }
  }
}

// f = f_{|x|,Q}(P) conjugated, as miller_loop<1>, for the Q of the table (a P at infinity contributes 1; the caller handles a Q
// at infinity)
B2K_D void miller_fixed_q(BFp12& f, const Affine<BFp>& P, const BlsLineCoef* tab) {
  fp12_set_one(f);
  if (aff_is_inf(P)) return;
  BlsLine l;
  int s = 0;
  for (int b = 62; b >= 0; b--) {
    fp12_sqr(f, f);
    l.l0 = tab[s].l0; fp2_mul_fp(l.l2, tab[s].c2, P.x); fp2_mul_fp(l.l3, tab[s].c3, P.y); s++;
    fp12_mul_line(f, l);
    if ((BLS_X_ABS >> b) & 1) {
      l.l0 = tab[s].l0; fp2_mul_fp(l.l2, tab[s].c2, P.x); fp2_mul_fp(l.l3, tab[s].c3, P.y); s++;
      fp12_mul_line(f, l);
    }
  }
  fp12_conj(f, f);
}

}  // namespace b2k
