// Host emulation of the Ed25519 verification device code (test infrastructure only).
#include "../../kyber_b200/csrc/eddsa.cuh"
using namespace b2k;

static void store_le(uint8_t* out, const EFp& a) {
  EFp c;
  fp_from_mont(c, a);
  for (int j = 0; j < 32; j++) out[j] = (uint8_t)(c.v[j >> 2] >> (8 * (j & 3)));
}

extern "C" {
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
