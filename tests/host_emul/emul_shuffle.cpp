// Host emulation of the shuffle verifier (test infrastructure only): the per-thread bodies of shuffle.cuh and the host
// transcript of shuffle_transcript.h, driven in the order the kernels of b2k_shuffle.cu run them.
#include <vector>
#include "../../kyber_b200/csrc/shuffle_transcript.h"
using namespace b2k;

static bool load(EdExt& p, const uint8_t* b) {
  EdAff a;
  const bool ok = ed_decode_aff(a, b);
  ed_from_aff(p, a);
  return ok;
}

extern "C" {
// the transcript of one shuffle: zrho[k][32], t[32], c[32]
void emul_transcript(size_t k, const uint8_t* proof, const uint8_t* proto, uint32_t plen, uint8_t* zrho, uint8_t* t, uint8_t* c,
                     unsigned nt) {
  shuffle_host::transcript(k, proof, proto, plen, zrho, t, c, nt);
}

// n picks from blake2xb.New(seed) with nt threads; returns the stream position after them (in 32-byte draws)
uint64_t emul_pick_many(const uint8_t* seed, uint32_t len, size_t n, uint8_t* out, unsigned nt) {
  shuffle_host::Pubrand pr;
  pr.seed(seed, len, nullptr, 0);
  shuffle_host::pick_many(pr, n, out, nt);
  return pr.pos;
}

// thver(A, B, T, a, b) on encodings; -1 if a point does not decode
int emul_thver(const uint8_t* A, const uint8_t* B, const uint8_t* T, const uint8_t* a, const uint8_t* b) {
  EdExt pa, pb;
  EdAff t;
  if (!load(pa, A) || !load(pb, B) || !ed_decode_aff(t, T)) return -1;
  uint32_t al[8], bl[8];
  sc_load_le(al, a);
  sc_load_le(bl, b);
  return shuffle_thver(pa, pb, t, al, bl) ? 1 : 0;
}

// Zsigma P + Zrho (-Q), encoded (the Phi term); Zsigma P (ed_mul_var), encoded
int emul_phi_term(const uint8_t* zs, const uint8_t* p, const uint8_t* zr, const uint8_t* q, uint8_t* out, uint8_t* out_mul) {
  EdAff P, Q;
  if (!ed_decode_aff(P, p) || !ed_decode_aff(Q, q)) return 0;
  uint32_t a[8], b[8];
  sc_load_le(a, zs);
  sc_load_le(b, zr);
  EdExt t1, t2, m, pp;
  shuffle_phi_terms(t1, t2, a, b, Q, Q, P, P);
  ed_encode(out, t1);
  ed_from_aff(pp, P);
  ed_mul_var(m, a, pp);
  ed_encode(out_mul, m);
  return 1;
}

void emul_neg_mod_l(const uint8_t* b, uint8_t* out) {
  uint32_t s[8], r[8];
  sc_load_le(s, b);
  sc_neg_mod_l(r, s);
  for (int j = 0; j < 32; j++) out[j] = (uint8_t)(r[j >> 2] >> (8 * (j & 3)));
}

// GetSequenceVerifiable of one output point over nq rows pts[nq][32], e[nq][32]; 0 if a point does not decode
int emul_sequence_term(uint32_t nq, const uint8_t* pts, const uint8_t* e, uint8_t* out) {
  std::vector<EdAff> a(nq);
  for (uint32_t j = 0; j < nq; j++)
    if (!ed_decode_aff(a[j], pts + 32 * j)) return 0;
  EdExt acc;
  shuffle_sequence_term(acc, nq, a.data(), 1, e);
  ed_encode(out, acc);
  return 1;
}

// b2k_ed25519_shuffle_verify for m shuffles, every kernel body in order on the host; the block sums of k_shuffle_pair_terms
// and k_shuffle_resolve are replayed in chunks of 128 with the same grouping
void emul_shuffle_verify(size_t m, size_t k, const uint8_t* g, const uint8_t* h, const uint8_t* x, const uint8_t* y,
                         const uint8_t* xbar, const uint8_t* ybar, const uint8_t* proofs, const uint8_t* proto, uint32_t plen,
                         uint8_t* status) {
  const size_t nitem = ShufItems::total(k), mk = m * k, bs = 128, nchunk = (k + bs - 1) / bs;
  std::vector<uint8_t> zrho(mk * 32), tc(m * 64), flags(4 * m, 0);
  shuffle_host::transcripts(m, k, proofs, proto, plen, zrho.data(), tc.data(), 2);
  std::vector<EdAff> pp(m * nitem), ip(4 * mk), gh(2 * m);
  // k_shuffle_decode
  for (size_t s = 0; s < m; s++) {
    for (size_t j = 0; j < nitem; j++)
      if (ShufItems::is_point(k, j) && !ed_decode_aff(pp[s * nitem + j], proofs + 32 * (s * nitem + j))) flags[4 * s] = 1;
    const uint8_t* in[4] = {x, y, xbar, ybar};
    for (int q = 0; q < 4; q++)
      for (size_t i = 0; i < k; i++)
        if (!ed_decode_aff(ip[q * mk + s * k + i], in[q] + 32 * (s * k + i))) flags[4 * s] = 1;
    uint8_t base[32];
    ed_base_bytes(base);
    if (!ed_decode_aff(gh[s], g ? g + 32 * s : base)) flags[4 * s] = 1;
    if (!ed_decode_aff(gh[m + s], h ? h + 32 * s : base)) flags[4 * s] = 1;
  }
  for (size_t s = 0; s < m; s++) {
    uint8_t* f = flags.data() + 4 * s;
    const EdAff* p = pp.data() + s * nitem;
    const uint8_t* proof = proofs + 32 * s * nitem;
    // k_shuffle_uw
    uint32_t t[8], nt[8], c[8];
    sc_load_le(t, tc.data() + 64 * s);
    sc_load_le(c, tc.data() + 64 * s + 32);
    sc_neg_mod_l(nt, t);
    EdExt B, U, W;
    ed_from_aff(B, gh[s]); ed_mul_var(U, nt, B);
    ed_from_aff(B, p[0]); ed_mul_var(W, nt, B);
    if (f[SHUF_F_POINT]) { status[s] = shuffle_status(f); continue; }
    // k_shuffle_thver
    for (uint32_t i = 0; i < 2 * k; i++)
      if (!shuffle_thver_i((uint32_t)k, i, p, proof, U, W, gh[s], c)) f[SHUF_F_SIMPLE] = 1;
    // k_shuffle_pair_terms, then k_shuffle_resolve
    EdExt phi[2];
    ed_set_identity(phi[0]);
    ed_set_identity(phi[1]);
    for (size_t ch = 0; ch < nchunk; ch++) {
      EdExt part[2];
      ed_set_identity(part[0]);
      ed_set_identity(part[1]);
      for (size_t i = ch * bs; i < (ch + 1) * bs && i < k; i++) {
        if (!shuffle_check33((uint32_t)k, (uint32_t)i, p, proof)) f[SHUF_F_PAIR] = 1;
        uint32_t zs[8], zr[8];
        sc_load_le(zs, proof + 32 * ShufItems::zsigma(k, i));
        sc_load_le(zr, zrho.data() + 32 * (s * k + i));
        const size_t si = s * k + i;
        EdExt t1, t2;
        shuffle_phi_terms(t1, t2, zs, zr, ip[si], ip[mk + si], ip[2 * mk + si], ip[3 * mk + si]);
        ed_add(part[0], part[0], t1);
        ed_add(part[1], part[1], t2);
      }
      ed_add(phi[0], phi[0], part[0]);
      ed_add(phi[1], phi[1], part[1]);
    }
    uint32_t ztau[8];
    sc_load_le(ztau, proof + 32 * ShufItems::ztau(k));
    if (!shuffle_check34(p[ShufItems::lambda1(k)], ztau, gh[s], phi[0]) ||
        !shuffle_check34(p[ShufItems::lambda2(k)], ztau, gh[m + s], phi[1]))
      f[SHUF_F_PAIR] = 1;
    status[s] = shuffle_status(f);
  }
}
}
