// Host emulation of the Ed25519 verification device code (test infrastructure only).
#include "../../kyber_b200/csrc/eddsa.cuh"
using namespace b2k;

static void store_le(uint8_t* out, const EFp& a) {
  EFp c;
  fp_from_mont(c, a);
  for (int j = 0; j < 32; j++) out[j] = (uint8_t)(c.v[j >> 2] >> (8 * (j & 3)));
}

extern "C" {
// SHA-512(a[0..na) || b[0..nb) || c[0..nc)) -> 64 digest bytes
void emul_sha512_3(const uint8_t* a, uint32_t na, const uint8_t* b, uint32_t nb, const uint8_t* c, uint32_t nc, uint8_t* out) {
  uint64_t h[8];
  sha512_3(h, a, na, b, nb, c, nc);
  for (int i = 0; i < 64; i++) out[i] = (uint8_t)(h[i >> 3] >> (56 - 8 * (i & 7)));
}

// 64 little-endian bytes -> their value mod l, 32 little-endian bytes
void emul_reduce512(const uint8_t* in, uint8_t* out) {
  uint32_t x[16], r[8];
  for (int i = 0; i < 16; i++) x[i] = (uint32_t)in[4 * i] | ((uint32_t)in[4 * i + 1] << 8) | ((uint32_t)in[4 * i + 2] << 16) | ((uint32_t)in[4 * i + 3] << 24);
  sc_reduce512(r, x);
  for (int j = 0; j < 32; j++) out[j] = (uint8_t)(r[j >> 2] >> (8 * (j & 3)));
}

// the staged base table: k B for k = 1..8 as (y + x, y - x, 2 d x y), canonical little-endian, 8 x 96 bytes
void emul_base_table(uint8_t* out) {
  EdNiels t[8];
  ed_load_base_table(t);
  for (int k = 0; k < 8; k++) {
    store_le(out + 96 * k, t[k].ypx); store_le(out + 96 * k + 32, t[k].ymx); store_le(out + 96 * k + 64, t[k].t2d);
  }
}

int emul_ed25519_verify(const uint8_t* pk, const uint8_t* msg, uint32_t mlen, const uint8_t* sig) {
  EdNiels t[8];
  ed_load_base_table(t);
  return ed_verify(pk, msg, mlen, sig, t);
}
}
