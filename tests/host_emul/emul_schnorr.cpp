// Host emulation of the sign/schnorr verification device code (test infrastructure only): the reduction of a 512-bit
// big-endian digest mod r, and the per-signature body of k_schnorr_verify for keys on G1 and on G2.
#include "../../kyber_b200/csrc/msm_affine.cuh"
#include "../../kyber_b200/csrc/schnorr.cuh"
using namespace b2k;

struct EmulInv { template <class F> void operator()(F& r, const F& a) const { f_inv_bg(r, a); } };

extern "C" {
// out = (in[0..64) read big-endian) mod r, 32 bytes big-endian
void emul_fr_from_be512(const uint8_t* in, uint8_t* out) {
  uint64_t w[8];
  for (int i = 0; i < 8; i++) {
    w[i] = 0;
    for (int j = 0; j < 8; j++) w[i] = (w[i] << 8) | in[8 * i + j];
  }
  Scalar256 h;
  fr_from_be512(h, w);
  for (int j = 0; j < 8; j++) {
    const uint32_t x = h.v[7 - j];
    out[4 * j] = (uint8_t)(x >> 24); out[4 * j + 1] = (uint8_t)(x >> 16); out[4 * j + 2] = (uint8_t)(x >> 8); out[4 * j + 3] = (uint8_t)x;
  }
}

// schnorr_verify for one signature; g2 = 0: keys on G1 (pk [48], sig [80]), 1: keys on G2 (pk [96], sig [128])
int emul_schnorr_verify(int g2, const uint8_t* pk, const uint8_t* msg, uint32_t mlen, const uint8_t* sig) {
  if (g2) {
    static Affine<BFp2> t[8];
    static bool init = false;
    if (!init) { schnorr_base_table<Bls381G2>(t, EmulInv{}); init = true; }
    return schnorr_verify<Bls381G2>(pk, msg, mlen, sig, t, EmulInv{});
  }
  static Affine<BFp> t[8];
  static bool init = false;
  if (!init) { schnorr_base_table<Bls381G1>(t, EmulInv{}); init = true; }
  return schnorr_verify<Bls381G1>(pk, msg, mlen, sig, t, EmulInv{});
}
}
