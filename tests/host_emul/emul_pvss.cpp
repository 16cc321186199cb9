// Host emulation of the DLEQ / PVSS device code (test infrastructure only): the per-thread bodies of pvss.cuh, driven in the
// order the kernels of b2k_pvss.cu run them.
#include <vector>
#include "../../kyber_b200/csrc/pvss.cuh"
using namespace b2k;

static void limbs_to_le(uint8_t* out, const uint32_t* s) {
  for (int j = 0; j < 32; j++) out[j] = (uint8_t)(s[j >> 2] >> (8 * (j & 3)));
}

extern "C" {
// BLAKE2b-512 of msg with the given parameter words 0..2 (RFC 7693 with an explicit parameter block; no key)
void emul_blake2b(const uint8_t* msg, uint32_t len, uint64_t p0, uint64_t p1, uint64_t p2, uint8_t* out) {
  uint64_t h[8];
  blake2b_init(h, p0, p1, p2);
  const uint32_t nblk = len ? (len + 127) / 128 : 1;
  for (uint32_t b = 0; b < nblk; b++) {
    uint64_t m[16];
    for (int i = 0; i < 16; i++) {
      uint64_t w = 0;
      for (int j = 7; j >= 0; j--) {
        const uint32_t pos = 128 * b + 8 * i + j;
        w = (w << 8) | (pos < len ? msg[pos] : 0);
      }
      m[i] = w;
    }
    blake2b_compress(h, m, 128 * (b + 1) < len ? 128 * (b + 1) : len, b == nblk - 1);
  }
  for (int i = 0; i < 64; i++) out[i] = (uint8_t)(h[i >> 3] >> (8 * (i & 7)));
}

// the root hash and output blocks 0..nblk-1 of blake2xb.New(seed)
void emul_blake2xb(const uint8_t* seed, uint32_t len, uint32_t nblk, uint8_t* root, uint8_t* out) {
  uint64_t h0[8], b[8];
  blake2xb_root(h0, seed, len);
  for (int i = 0; i < 64; i++) root[i] = (uint8_t)(h0[i >> 3] >> (8 * (i & 7)));
  for (uint32_t k = 0; k < nblk; k++) {
    blake2xb_block(b, h0, k);
    for (int i = 0; i < 64; i++) out[64 * k + i] = (uint8_t)(b[i >> 3] >> (8 * (i & 7)));
  }
}

void emul_sc_pick(const uint8_t* seed, uint32_t len, uint8_t* out) {
  uint32_t s[8];
  sc_pick(s, seed, len);
  limbs_to_le(out, s);
}

// geScalarMult(r, P) + geScalarMult(c, P2), encoded; false if a point does not decode
int emul_double_mul_var(const uint8_t* r, const uint8_t* p, const uint8_t* c, const uint8_t* p2, uint8_t* out) {
  EdExt P, P2, Q;
  if (!ed_decode(P, p) || !ed_decode(P2, p2)) return 0;
  uint32_t rl[8], cl[8];
  sc_load_le(rl, r);
  sc_load_le(cl, c);
  ed_double_mul_var(Q, rl, P, cl, P2);
  ed_encode(out, Q);
  return 1;
}

int emul_dleq_verify(const uint8_t* g, const uint8_t* h, const uint8_t* xg, const uint8_t* xh, const uint8_t* proof) {
  return dleq_verify_one(g, h, xg, xh, proof);
}

int emul_dec_share(const uint8_t* g, const uint8_t* x, const uint8_t* enc_v, const uint8_t* dec_v, const uint8_t* proof) {
  return pvss_dec_share(g, x, enc_v, dec_v, proof);
}

// one deal of k_pvss_load_commits, k_pvss_hashed_points, k_pvss_deal_challenge and k_pvss_enc_verify; chal_out = the
// deal's challenge (zero if the deal is marked)
void emul_enc_shares(uint32_t t, uint32_t n, const uint8_t* h, const uint8_t* commits, const uint8_t* x, const uint8_t* sh,
                     const uint8_t* v, const uint8_t* proofs, uint8_t* status, uint8_t* chal_out) {
  std::vector<EdNiels> cm(t);
  std::vector<uint8_t> hashed(128 * (size_t)n);
  uint32_t bad = 0, chal[8] = {0};
  for (uint32_t j = 0; j < t; j++)
    if (!ed_load_niels(cm[j], commits + 32 * j)) bad = 1;
  for (uint32_t i = 0; i < n; i++)
    if (!pvss_hashed_points(hashed.data() + 32 * (size_t)i, 32 * (size_t)n, cm.data(), t, i, v + 32 * i, proofs + 128 * i)) bad = 1;
  EdExt H;
  if (!ed_decode(H, h)) bad = 1;
  if (!bad) {
    uint8_t dig[32];
    sha256_blocks(dig, hashed.data(), 2 * (size_t)n);
    sc_pick(chal, dig, 32);
  }
  limbs_to_le(chal_out, chal);
  for (uint32_t i = 0; i < n; i++)
    status[i] = bad ? (uint8_t)DLEQ_POINT : (uint8_t)pvss_enc_share(h, x + 32 * i, sh + 32 * i, v + 32 * i, proofs + 128 * i, chal);
}
}
