// Host emulation of the IBE device code (test infrastructure only): the fixed-G2 Miller loop against miller_loop<1>, and the
// per-thread bodies of the decrypt-finish and encrypt kernels of b2k_ibe.cu.
#include "../../kyber_b200/csrc/ibe.cuh"
#include "../../kyber_b200/csrc/msm_affine.cuh"
using namespace b2k;

struct EmulInv { template <class F> void operator()(F& r, const F& a) const { f_inv_bg(r, a); } };

extern "C" {
// gt = final_exponentiation(miller) for P (operand [96]) and Q (operand [192]); fixed = 1 through the line table
void emul_ibe_pair(const uint8_t* p96, const uint8_t* q192, int fixed, uint8_t* gt576) {
  Affine<BFp> P;
  Affine<BFp2> Q;
  Bls381G1::load(P, p96);
  Bls381G2::load(Q, q192);
  BFp12 f, e;
  if (fixed) {
    static BlsLineCoef tab[BLS_MILLER_STEPS];
    miller_fixed_q_table(tab, Q);
    if (aff_is_inf(Q)) fp12_set_one(f);
    else miller_fixed_q(f, P, tab);
  } else {
    miller_loop<1>(f, &P, &Q);
  }
  final_exponentiation(e, f);
  gt_store(gt576, e);
}

// ibe_decrypt_finish for U compressed (group 1: [48], 2: [96]); returns the status
int emul_ibe_decrypt_finish(int group, const uint8_t* gt, const uint8_t* u, const uint8_t* v, const uint8_t* w, uint32_t len, uint8_t* msg) {
  if (group == 1) {
    Affine<BFp> U;
    const bool ok = g1_decompress(U, u, true);
    if (!ok) aff_set_inf(U);
    return ibe_decrypt_finish<Bls381G1>(msg, gt, U, ok, v, w, len, EmulInv{});
  }
  Affine<BFp2> U;
  const bool ok = g2_decompress(U, u, true);
  if (!ok) aff_set_inf(U);
  return ibe_decrypt_finish<Bls381G2>(msg, gt, U, ok, v, w, len, EmulInv{});
}

// ibe_encrypt_body: U compressed, r [32] big-endian, W; returns 1 when H3 found a scalar
int emul_ibe_encrypt_body(int group, const uint8_t* msg, const uint8_t* sigma, uint32_t len, uint8_t* u, uint8_t* r, uint8_t* w) {
  return group == 1 ? ibe_encrypt_body<Bls381G1>(u, r, w, msg, sigma, len, EmulInv{})
                    : ibe_encrypt_body<Bls381G2>(u, r, w, msg, sigma, len, EmulInv{});
}

// compression round trip: compressed -> decode -> Bls381G*::store
int emul_ibe_recompress(int group, const uint8_t* in, uint8_t* out) {
  if (group == 1) {
    Affine<BFp> a;
    if (!g1_decompress(a, in, true)) return 0;
    Bls381G1::store(out, a);
    return 1;
  }
  Affine<BFp2> a;
  if (!g2_decompress(a, in, true)) return 0;
  Bls381G2::store(out, a);
  return 1;
}
}
