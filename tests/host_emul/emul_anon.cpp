// Host emulation of the ring signature verifier (test infrastructure only): the per-thread bodies of anon.cuh, driven in the
// order the kernels of b2k_anon.cu run them.
#include <vector>
#include "../../kyber_b200/csrc/anon.cuh"
using namespace b2k;

static void limbs_to_le(uint8_t* out, const uint32_t* s) {
  for (int j = 0; j < 32; j++) out[j] = (uint8_t)(s[j >> 2] >> (8 * (j & 3)));
}

// the table of a base encoding (k_anon_tables: one call per column k); false if it does not decode
static bool table(std::vector<EdCached>& tab, const uint8_t* p) {
  EdExt P;
  if (!ed_decode(P, p)) return false;
  tab.resize(8 * ANON_ROWS);
  for (uint32_t k = 1; k <= 8; k++) ed_comb_table_column(tab.data(), k, P);
  return true;
}

extern "C" {
// c = H1(H1pre(msg, scope, tag), pg [, ph]) as 32 little-endian bytes; tag null = unlinkable (no scope, no ph)
void emul_h1(const uint8_t* msg, uint32_t mlen, const uint8_t* scope, uint32_t slen, const uint8_t* tag, const uint8_t* pg,
             const uint8_t* ph, uint8_t* out) {
  Blake2bMid pre;
  anon_h1pre(pre, msg, mlen, scope, slen, tag);
  uint32_t c[8];
  anon_h1(c, pre, pg, tag ? ph : nullptr);
  limbs_to_le(out, c);
}

int emul_link_base(const uint8_t* scope, uint32_t slen, uint8_t* out) { return anon_link_base(out, scope, slen) ? 1 : 0; }

// geScalarMultBase's schedule over the tables of P (a) and Q (b; Q null = none), encoded; -1 if a point does not decode
int emul_comb(const uint8_t* a, const uint8_t* P, const uint8_t* b, const uint8_t* Q, uint8_t* out) {
  std::vector<EdCached> ta, tb;
  if (!table(ta, P) || (Q && !table(tb, Q))) return -1;
  uint32_t al[8], bl[8];
  sc_load_le(al, a);
  if (Q) sc_load_le(bl, b);
  EdExt R;
  ed_comb(R, al, ta.data(), Q ? bl : nullptr, Q ? tb.data() : nullptr);
  ed_encode(out, R);
  return 0;
}

// anon.Verify of m signatures through every body in order (setup, link base, the fixed tables, chunks of `chunk` positions,
// finish); returns -1 if a ring key does not decode, else 0 with status[m] and tags[m][32]
int emul_anon_verify(size_t n, const uint8_t* ring, int linkable, const uint8_t* scope, uint32_t slen, size_t m,
                     const uint8_t* msgs, const uint32_t* offs, const uint8_t* sigs, uint32_t chunk, uint8_t* status,
                     uint8_t* tags) {
  const size_t siglen = 32 * (n + 1 + linkable);
  std::vector<Blake2bMid> mid(m);
  std::vector<uint32_t> cs(8 * m);
  std::vector<EdAff> tag_aff(m);
  std::vector<uint8_t> tag_bytes(32 * m);
  for (size_t j = 0; j < m; j++) {                          // k_anon_setup
    const uint8_t* sig = sigs + siglen * j;
    status[j] = ANON_OK;
    if (linkable) {
      EdExt T;
      if (!ed_decode(T, sig + 32 * (n + 1))) { status[j] = ANON_POINT; continue; }
      ed_encode_z1(&tag_bytes[32 * j], T);
      tag_aff[j].x = T.X;
      tag_aff[j].y = T.Y;
    }
    anon_h1pre(mid[j], msgs + offs[j], offs[j + 1] - offs[j], scope, linkable ? slen : 0, linkable ? &tag_bytes[32 * j] : nullptr);
    sc_load_le(&cs[8 * j], sig);
  }
  if (n) {
    uint8_t fix[64];
    ed_base_bytes(fix);
    if (linkable && !anon_link_base(fix + 32, scope, slen)) return -2;     // k_anon_link_base
    std::vector<EdCached> tb, th;                           // k_anon_tables of the fixed bases
    table(tb, fix);
    if (linkable) table(th, fix + 32);
    for (size_t i0 = 0; i0 < n; i0 += chunk) {
      const size_t cnt = n - i0 < chunk ? n - i0 : chunk;
      std::vector<std::vector<EdCached>> tl(cnt);           // k_anon_tables of the chunk's keys
      for (size_t i = 0; i < cnt; i++)
        if (!table(tl[i], ring + 32 * (i0 + i))) return -1;
      for (size_t j = 0; j < m; j++) {                      // k_anon_ring_step
        if (status[j] != ANON_OK) continue;
        EdCached tagtab[8];
        if (linkable) {
          EdExt T;
          ed_from_aff(T, tag_aff[j]);
          ed_cached_table(tagtab, T);
        }
        for (size_t i = 0; i < cnt; i++) {
          uint32_t s[8];
          sc_load_le(s, sigs + siglen * j + 32 * (i0 + i + 1));
          anon_ring_step(&cs[8 * j], s, tb.data(), tl[i].data(), linkable ? th.data() : nullptr, tagtab, mid[j]);
        }
      }
    }
  }
  for (size_t j = 0; j < m; j++) {                          // k_anon_finish
    if (status[j] == ANON_OK && !pvss_challenge_is(sigs + siglen * j, &cs[8 * j])) status[j] = ANON_INVALID;
    for (int q = 0; q < 32; q++) tags[32 * j + q] = status[j] == ANON_OK && linkable ? tag_bytes[32 * j + q] : 0;
  }
  return 0;
}
}
