// shuffle_transcript.h -- host code: the Fiat-Shamir transcript of proof.HashVerify around shuffle.Verifier, on host threads.
//
// Replaces (reference):
//   hashVerifier.consumeMsg / PubRand   proof/hash.go:111-142: Reseed, then Write of the RAW proof bytes read since the last PubRand
//   xof.Reseed                          xof/blake2xb/blake.go:55-75: 128 stream bytes -> New(them): key = the first 64, message =
//                                       the last 64
//   ScalarUnmarshalFrom on the XOF      group/internal/marshalling/marshal.go:53-63 -> Scalar.Pick (32-byte draws, top 3 bits
//                                       cleared, big-endian, drawn again while >= l)
// The verifier's PubRand calls (shuffle/pair.go:239-312, simple.go:186-254): absorb ega1, pick k Zrho; absorb ega3, pick Zlambda
// (unused, but it consumes stream); absorb ega5 || ssa0 in one write, pick t; absorb ssa2, pick c.  ssa4 is never absorbed.
// Each absorb is one sequential BLAKE2b chain (hash.go keeps it so); the Zrho squeeze is spread over threads: every BLAKE2X
// output block is independent, so blocks are hashed in parallel and a scan over the accept flags gives the positions.
// BLAKE2b itself is blake2b.cuh's (host-callable).
#pragma once
#include <cmath>
#include <cstring>
#include <thread>
#include <vector>

#include "blake2b.cuh"
#include "shuffle.cuh"

namespace b2k {
namespace shuffle_host {

// l, little-endian bytes
constexpr uint8_t kL[32] = {0xed, 0xd3, 0xf5, 0x5c, 0x1a, 0x63, 0x12, 0x58, 0xd6, 0x9c, 0xf7, 0xa2, 0xde, 0xf9, 0xde, 0x14,
                            0,    0,    0,    0,    0,    0,    0,    0,    0,    0,    0,    0,    0,    0,    0,    0x10};

// BLAKE2b-512 streamed from memory (the compression of blake2b.cuh)
struct Blake2bStream {
  uint64_t* h;
  uint64_t t = 0;
  uint8_t buf[128];
  size_t fill = 0;

  void block(const uint8_t* p, bool last) {
    uint64_t m[16];
    std::memcpy(m, p, 128);                             // little-endian words (x86-64 and aarch64 hosts)
    blake2b_compress(h, m, t, last);
  }
  void update(const uint8_t* p, size_t n) {
    while (n > 0) {
      if (fill == 128) { t += 128; block(buf, false); fill = 0; }   // a full block is compressed only once more follows
      if (fill == 0 && n > 128) { t += 128; block(p, false); p += 128; n -= 128; continue; }
      size_t c = 128 - fill < n ? 128 - fill : n;
      std::memcpy(buf + fill, p, c);
      fill += c; p += c; n -= c;
    }
  }
  void final() {
    t += fill;
    std::memset(buf + fill, 0, 128 - fill);
    block(buf, true);
  }
};

// The XOF: the root hash of blake2xb.New(seed) followed by Write(msg), and the read position in 32-byte draws
struct Pubrand {
  uint64_t h0[8];
  uint64_t pos = 0;

  // blake2xb.New(key) + Write(msg): BLAKE2b-512 keyed with key[0, min(klen, 64)) over key[64, klen) || msg, XOF parameters
  void seed(const uint8_t* key, size_t klen, const uint8_t* msg, size_t mlen) {
    const size_t kb = klen < 64 ? klen : 64;
    blake2b_init(h0, 64u | ((uint64_t)kb << 8) | (1u << 16) | (1u << 24), 0xffffffffull << 32, 0);
    Blake2bStream s{h0};
    if (kb) {
      uint8_t kblk[128] = {0};
      std::memcpy(kblk, key, kb);
      s.update(kblk, 128);
    }
    if (klen > 64) s.update(key + 64, klen - 64);
    if (mlen) s.update(msg, mlen);
    s.final();
    pos = 0;
  }
  // draw u (32 bytes) of the stream
  void draw(uint8_t* out, uint64_t u) const {
    uint64_t b[8];
    blake2xb_block(b, h0, (uint32_t)(u >> 1));
    std::memcpy(out, (const uint8_t*)b + 32 * (u & 1), 32);
  }
  // consumeMsg: Reseed, then Write(msg)
  void absorb(const uint8_t* msg, size_t len) {
    uint8_t key[128];
    for (int q = 0; q < 4; q++) draw(key + 32 * q, pos + q);
    seed(key, 128, msg, len);
  }
};

// one draw of random.Int(l): clears the top 3 bits of the first byte, reads big-endian; out = the little-endian bytes; false
// when the value is >= l (the draw is rejected)
inline bool pick_accept(uint8_t* out, const uint8_t* draw) {
  for (int j = 0; j < 32; j++) out[j] = draw[31 - j];
  out[31] &= 0x1f;
  for (int j = 31; j >= 0; j--)
    if (out[j] != kL[j]) return out[j] < kL[j];
  return false;
}

inline void pick(Pubrand& pr, uint8_t* out) {
  uint8_t d[32];
  do pr.draw(d, pr.pos++);
  while (!pick_accept(out, d));
}

// n picks into out[n][32] with nt threads: draws are hashed in parallel batches, then taken in stream order
inline void pick_many(Pubrand& pr, size_t n, uint8_t* out, unsigned nt) {
  if (nt <= 1 || n < 1024) {
    for (size_t i = 0; i < n; i++) pick(pr, out + 32 * i);
    return;
  }
  size_t got = 0;
  std::vector<uint8_t> val;
  std::vector<uint8_t> ok;
  while (got < n) {
    const size_t need = n - got, batch = 2 * need + 64 + (size_t)(8.0 * std::sqrt((double)need));   // accept rate ~1/2
    val.resize(32 * batch);
    ok.resize(batch);
    const uint64_t base = pr.pos;
    auto work = [&](size_t lo, size_t hi) {
      uint64_t b[8];
      uint64_t cur = ~0ull;
      for (size_t u = lo; u < hi; u++) {
        const uint64_t a = base + u;
        if ((a >> 1) != cur) { cur = a >> 1; blake2xb_block(b, pr.h0, (uint32_t)cur); }
        ok[u] = pick_accept(&val[32 * u], (const uint8_t*)b + 32 * (a & 1));
      }
    };
    std::vector<std::thread> th;
    const size_t per = (batch + nt - 1) / nt;
    for (unsigned q = 0; q < nt; q++) {
      const size_t lo = q * per, hi = lo + per < batch ? lo + per : batch;
      if (lo < hi) th.emplace_back(work, lo, hi);
    }
    for (auto& x : th) x.join();
    size_t u = 0;
    for (; u < batch && got < n; u++)
      if (ok[u]) std::memcpy(out + 32 * got++, &val[32 * u], 32);
    pr.pos = base + u;
  }
}

// The verifier's side of proof.HashVerify(suite, proto, shuffle.Verifier(...), proof) for one shuffle of k pairs: zrho[k][32],
// t[32], c[32] (canonical little-endian)
inline void transcript(size_t k, const uint8_t* proof, const uint8_t* proto, size_t proto_len, uint8_t* zrho, uint8_t* t,
                       uint8_t* c, unsigned nt) {
  Pubrand pr;
  pr.seed(proto, proto_len, nullptr, 0);
  uint8_t zl[32];
  pr.absorb(proof, 32 * (4 * k + 3));                  // ega1
  pick_many(pr, k, zrho, nt);
  pr.absorb(proof + 32 * (4 * k + 3), 32 * k);         // ega3
  pick(pr, zl);                                         // Zlambda
  pr.absorb(proof + 32 * (5 * k + 3), 32 * (3 * k + 1));   // ega5 || ssa0
  pick(pr, t);
  pr.absorb(proof + 32 * (8 * k + 4), 32 * (2 * k));   // ssa2
  pick(pr, c);
}

// m transcripts on up to nt threads (one shuffle per thread; the spare threads of a small batch squeeze Zrho)
inline void transcripts(size_t m, size_t k, const uint8_t* proofs, const uint8_t* proto, size_t proto_len, uint8_t* zrho,
                        uint8_t* tc, unsigned nt) {
  const size_t plen = 32 * ShufItems::total(k);
  const unsigned outer = m < nt ? (unsigned)m : nt, inner = nt / (outer ? outer : 1);
  auto run = [&](unsigned q) {
    for (size_t s = q; s < m; s += outer)
      transcript(k, proofs + plen * s, proto, proto_len, zrho + 32 * k * s, tc + 64 * s, tc + 64 * s + 32, inner);
  };
  if (outer <= 1) { run(0); return; }
  std::vector<std::thread> th;
  for (unsigned q = 0; q < outer; q++) th.emplace_back(run, q);
  for (auto& x : th) x.join();
}

}  // namespace shuffle_host
}  // namespace b2k
