// Host emulation of ECIES on edwards25519 (test infrastructure only): the per-thread bodies of ecies.cuh, built with the
// operation counters (B2K_ECIES_COUNT) that tests/test_ecies_emulation.py compares across keys, points and messages.
#define B2K_ECIES_COUNT 1
#include <cstring>
#include "../../kyber_b200/csrc/ecies.cuh"
using namespace b2k;

uint64_t ecies_counts[4];

static void recode(int8_t* e, const uint8_t* s) {
  uint32_t k[8];
  sc_load_le(k, s);
  sc_recode4(e, k);
}

extern "C" {
void emul_counts(uint64_t* out, int reset) {
  for (int i = 0; i < 4; i++) out[i] = ecies_counts[i];
  if (reset) memset(ecies_counts, 0, sizeof(ecies_counts));
}

// geScalarMult(s, P) through the constant-time table and selection; -1 if P does not decode
int emul_mul_var(const uint8_t* s, const uint8_t* p, uint8_t* out) {
  EdExt P, Q;
  if (!ed_decode(P, p)) return -1;
  EdCached tab[8];
  ed_cached_table(tab, P);
  int8_t e[64];
  recode(e, s);
  ecies_mul_var(Q, e, tab);
  ed_encode_ct(out, Q);
  return 0;
}

// geScalarMultBase(s) over the comb
void emul_mul_base(const uint8_t* s, uint8_t* out) {
  int8_t e[64];
  recode(e, s);
  EdExt Q;
  ecies_mul_base(Q, e, ecies_base_comb);
  ed_encode_ct(out, Q);
}

// n ciphertexts of 32 + clen bytes under one key, as k_ecies_decrypt runs them
void emul_decrypt(const uint8_t* priv, size_t n, uint32_t clen, const uint8_t* ct, uint8_t* msg, uint8_t* status) {
  int8_t e[64];
  recode(e, priv);
  for (size_t i = 0; i < n; i++) status[i] = (uint8_t)ecies_decrypt_one(e, ct + (32 + clen) * i, clen, msg + (clen - 16) * i);
}

void emul_encrypt(size_t n, const uint8_t* pubs, const uint8_t* rs, uint32_t len, const uint8_t* msgs, uint8_t* out,
                  uint8_t* status) {
  for (size_t i = 0; i < n; i++)
    status[i] = (uint8_t)ecies_encrypt_one(pubs + 32 * i, rs + 32 * i, ecies_base_comb, msgs + (size_t)len * i, len,
                                           out + (size_t)(len + 48) * i);
}
}
