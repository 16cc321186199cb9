// Host emulation of ECIES on BLS12-381 (test infrastructure only): the per-thread bodies of ecies_bls.cuh for keys on G1 and
// on G2, built with the operation counters (B2K_ECIES_COUNT) that tests/test_ecies_bls12381_emulation.py compares across keys,
// points and messages.  g2 = 0: G1 (points of 48 bytes), 1: G2 (96 bytes).
#define B2K_ECIES_COUNT 1
#include <cstring>
#include "../../kyber_b200/csrc/ecies_bls.cuh"
using namespace b2k;

uint64_t ecies_counts[ECIES_CNT_BLS];

template <class CV>
static int mul(const uint8_t* k, const uint8_t* p, uint8_t* out) {
  using F = typename CV::F;
  Proj<F> tab[8], Q;
  if (p) {
    Affine<F> P;
    if (!ecies_bls_decode<CV>(P, p)) return -1;
    ct_table(tab, P);
  } else {
    ecies_bls_base_table<CV>(tab);
  }
  int8_t e[ECIES_BLS_DIGITS];
  ct_recode(e, k);
  ct_mul(Q, e, tab);
  ct_compress<F, CV::OUT_BYTES>(out, Q);
  return 0;
}

// compression of the affine point in uncompressed bytes (x || y, zero = infinity), scaled by z (32 bytes BE, as a field
// element of Fp, z != 0), so that Z != 1
template <class CV>
static void compress(const uint8_t* xy, const uint8_t* z, uint8_t* out) {
  using F = typename CV::F;
  Affine<F> a;
  CV::load(a, xy);
  Proj<F> p;
  proj_from_affine(p, a);
  BFp zz, zb;
  fp_load_be(zb, z);
  fp_to_mont(zz, zb);
  if constexpr (CV::OUT_BYTES == 48) {
    fp_mul(p.X, p.X, zz); fp_mul(p.Y, p.Y, zz); fp_mul(p.Z, p.Z, zz);
  } else {
    F s;
    s.c0 = zz; s.c1 = zz;                                   // z (1 + u)
    f_mul(p.X, p.X, s); f_mul(p.Y, p.Y, s); f_mul(p.Z, p.Z, s);
  }
  ct_compress<F, CV::OUT_BYTES>(out, p);
}

template <class CV>
static void decrypt(const uint8_t* priv, size_t n, uint32_t clen, const uint8_t* ct, uint8_t* msg, uint8_t* status) {
  int8_t e[ECIES_BLS_DIGITS];
  ct_recode(e, priv);
  constexpr int PL = CV::OUT_BYTES;
  for (size_t i = 0; i < n; i++) status[i] = (uint8_t)ecies_bls_decrypt_one<CV>(e, ct + (PL + clen) * i, clen, msg + (clen - 16) * i);
}

template <class CV>
static void encrypt(size_t n, const uint8_t* pubs, const uint8_t* rs, uint32_t len, const uint8_t* msgs, uint8_t* out,
                    uint8_t* status) {
  constexpr int PL = CV::OUT_BYTES;
  Proj<typename CV::F> btab[8];
  ecies_bls_base_table<CV>(btab);
  for (size_t i = 0; i < n; i++)
    status[i] = (uint8_t)ecies_bls_encrypt_one<CV>(pubs + PL * i, rs + 32 * i, btab, msgs + (size_t)len * i, len,
                                                   out + (size_t)(PL + len + 16) * i);
}

extern "C" {
void emul_counts(uint64_t* out, int reset) {
  for (int i = 0; i < ECIES_CNT_BLS; i++) out[i] = ecies_counts[i];
  if (reset) memset(ecies_counts, 0, sizeof(ecies_counts));
}

// k P (p compressed, or null for the generator) through the constant-time table, walk and compression; -1 if P does not decode
int emul_mul(int g2, const uint8_t* k, const uint8_t* p, uint8_t* out) {
  return g2 ? mul<Bls381G2>(k, p, out) : mul<Bls381G1>(k, p, out);
}

void emul_compress(int g2, const uint8_t* xy, const uint8_t* z, uint8_t* out) {
  if (g2) compress<Bls381G2>(xy, z, out);
  else compress<Bls381G1>(xy, z, out);
}

void emul_decrypt(int g2, const uint8_t* priv, size_t n, uint32_t clen, const uint8_t* ct, uint8_t* msg, uint8_t* status) {
  if (g2) decrypt<Bls381G2>(priv, n, clen, ct, msg, status);
  else decrypt<Bls381G1>(priv, n, clen, ct, msg, status);
}

void emul_encrypt(int g2, size_t n, const uint8_t* pubs, const uint8_t* rs, uint32_t len, const uint8_t* msgs, uint8_t* out,
                  uint8_t* status) {
  if (g2) encrypt<Bls381G2>(n, pubs, rs, len, msgs, out, status);
  else encrypt<Bls381G1>(n, pubs, rs, len, msgs, out, status);
}
}
