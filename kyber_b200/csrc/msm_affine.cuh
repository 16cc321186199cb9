// msm_affine.cuh -- affine pair-tree rounds of the MSM's bucket accumulation.
//
// The bucket sums of the Pippenger pipeline (msm.cuh; reference loops share/poly.go:461-473, sign/bdn/bdn.go:126-161)
// are bound by the integer multiply pipe, not by HBM (DESIGN.md section 4): a mixed XYZZ addition costs 10 field
// products.  An AFFINE addition costs 1 inversion + 3 products, and inversions batch (Montgomery's trick: 3 products per
// element + one shared inversion), i.e. 6 products per addition -- if independent additions are available.  The serial
// "acc += P" of a bucket is not; a pair tree is: one ROUND replaces the k sorted operands of every bucket by the
// ceil(k/2) sums of neighbouring pairs (an odd last operand is carried over), and the rounds' outputs are again affine
// points grouped by bucket.  R rounds shrink the entry list 2^R-fold, for 40 % fewer products but extra HBM traffic: each
// round writes its outputs and a prefix-product array and reads them back.  On H100 (3.35 TB/s) that traffic costs about
// what the saved products gain (DESIGN.md section 4), so the automatic plan runs no rounds there (msm_host.cuh: affine_plan);
// the XYZZ slices of msm.cuh finish what the rounds leave.  A bucket of k operands holds ceil(k / 2^r) after r rounds, so the
// bucket offsets of every round follow from the main histogram (pt_round_count; one multi-column scan, kernels.cuh).
//
// One thread owns B consecutive OUTPUT positions of a round:
//   forward : fetch the two operands, classify, d_j = x2 - x1 (2 y1 for a doubling, 1 when nothing is to invert),
//             pre[j] = d_0 ... d_{j-1}                                                    1 product
//   invert  : the running product, once per thread (branch-free binary GCD, fp_inv.cuh)
//   backward: 1/d_j = inv pre[j], inv *= d_j, lambda = (y2 - y1)/d_j, x3 = lambda^2 - x1 - x2,
//             y3 = lambda (x1 - x3) - y1                                                   5 products
// Every exceptional case of the group law is handled (operand at infinity, P + P, P + (-P)): skewed scalar sets put equal
// points into one bucket.
#pragma once
#include "msm.cuh"
#include "fp_inv.cuh"
#ifdef B2K_HOST_EMUL
#include <cstring>
#include <vector>
#endif

namespace b2k {

template <class C> B2K_D void f_inv_bg(Fp<C>& r, const Fp<C>& a) { fp_inv_bingcd(r, a); }
template <class C> B2K_D void f_inv_bg(Fp2<C>& r, const Fp2<C>& a) {
  Fp<C> n, t;
  fp_sqr_c(n, a.c0); fp_sqr_c(t, a.c1); fp_add(n, n, t);
  fp_inv_bingcd(n, n);
  fp_mul_c(r.c0, a.c0, n); fp_mul_c(t, a.c1, n); fp_neg(r.c1, t);
}

// (Round 2 tried software prefetch here -- `prefetch.global.L1` of the next output's operands and prefix product one iteration
//  ahead, because ncu shows `long_scoreboard` stalls in the round-1 kernels: measured SLOWER; the extra address arithmetic and
//  the L1 traffic cost more than the latency they hide.  Removed.)

constexpr int PT_MAXB = 64;     // outputs per thread (length of the prefix-product array in local memory)
enum : int { PT_COPY1 = 0, PT_COPY2 = 1, PT_ADD = 2, PT_DBL = 3, PT_INF = 4 };

// operands of a bucket of k after r rounds: ceil(k / 2^r) (= r halvings with the odd operand carried over)
B2K_D uint32_t pt_round_count(uint32_t k, uint32_t r) { return (k >> r) + ((k & ((1u << r) - 1u)) != 0u); }

// operands of the output at input position a (pairs start at even offsets of the bucket's run [.., end))
template <class CV, bool FIRST>
B2K_D bool pt_fetch(Affine<typename CV::F>& p1, Affine<typename CV::F>& p2, const Affine<typename CV::F>* in,
                    const uint32_t* entries, uint32_t a, uint32_t end) {
  const bool pair = a + 1 < end;
  if (FIRST) {                                        // round 0 gathers by the sorted (index | sign) entries
    uint32_t v = entries[a];
    p1 = in[v & 0x7fffffffu];
    if (v >> 31) f_neg(p1.y, p1.y);
    if (pair) {
      v = entries[a + 1];
      p2 = in[v & 0x7fffffffu];
      if (v >> 31) f_neg(p2.y, p2.y);
    } else p2 = p1;
  } else {
    p1 = in[a];
    p2 = pair ? in[a + 1] : p1;
  }
  return pair;
}

// what the output is and the denominator d its slope needs (1 when none)
template <class F>
B2K_D int pt_classify(F& d, const Affine<F>& p1, const Affine<F>& p2, bool pair) {
  f_set_one(d);
  if (!pair || aff_is_inf(p2)) return PT_COPY1;
  if (aff_is_inf(p1)) return PT_COPY2;
  F dx;
  f_sub(dx, p2.x, p1.x);
  if (!f_is_zero(dx)) { d = dx; return PT_ADD; }
  if (f_eq(p1.y, p2.y) && !f_is_zero(p1.y)) { f_dbl(d, p1.y); return PT_DBL; }
  return PT_INF;                                      // P + (-P), or a 2-torsion point doubled
}

// thread t of a round: outputs [t B, min((t+1) B, offs_out[total]))
template <class CV, bool FIRST>
B2K_D void msm_pairtree_round(uint32_t t, uint32_t B, uint32_t total, const Affine<typename CV::F>* in,
                              const uint32_t* entries, const uint32_t* offs_in, const uint32_t* offs_out,
                              Affine<typename CV::F>* out) {
  using F = typename CV::F;
  const uint32_t nout = offs_out[total];
  const uint32_t q0 = t * B;
  if (q0 >= nout) return;
  const uint32_t q1 = (nout - q0 < B) ? nout : q0 + B;
  F pre[PT_MAXB];
  uint32_t g = msm_find_bucket(offs_out, total, q0);
  uint32_t os = offs_out[g], oe = offs_out[g + 1], is = offs_in[g], ie = offs_in[g + 1];
  F acc;
  f_set_one(acc);
  for (uint32_t q = q0; q < q1; q++) {
    while (q >= oe) { g++; os = oe; oe = offs_out[g + 1]; is = ie; ie = offs_in[g + 1]; }
    Affine<F> p1, p2;
    F d;
    const bool pair = pt_fetch<CV, FIRST>(p1, p2, in, entries, is + 2 * (q - os), ie);
    pt_classify(d, p1, p2, pair);
    pre[q - q0] = acc;
    f_mul(acc, acc, d);
  }
  F inv;
  f_inv_bg(inv, acc);                                 // every d is non-zero, so is their product
  for (uint32_t q = q1; q-- > q0;) {
    while (q < os) { g--; oe = os; os = offs_out[g]; ie = is; is = offs_in[g]; }
    Affine<F> p1, p2, r;
    F d, dinv, lam, tt;
    const bool pair = pt_fetch<CV, FIRST>(p1, p2, in, entries, is + 2 * (q - os), ie);
    const int kind = pt_classify(d, p1, p2, pair);
    f_mul(dinv, inv, pre[q - q0]);
    if (q > q0) f_mul(inv, inv, d);
    if (kind == PT_DBL) { f_sqr(tt, p1.x); f_dbl(lam, tt); f_add(tt, lam, tt); }   // 3 x^2 (rare)
    else f_sub(tt, p2.y, p1.y);
    f_mul(lam, tt, dinv);
    f_sqr(r.x, lam); f_sub(r.x, r.x, p1.x); f_sub(r.x, r.x, p2.x);
    f_sub(tt, p1.x, r.x); f_mul(r.y, lam, tt); f_sub(r.y, r.y, p1.y);
    if (kind == PT_COPY1) r = p1;
    else if (kind == PT_COPY2) r = p2;
    else if (kind == PT_INF) aff_set_inf(r);
    out[q] = r;
  }
}

// ---- the same round as three kernels (forward products / inversions / backward additions) ------------------------------
// One fused kernel keeps three very different code regions (one inlined product; the 2 000-instruction inversion; five
// inlined products) resident at once and runs them all at the register budget of the widest; split, every phase has
// compact code and its own occupancy, the prefix products travel through a coalesced global array pre[j * T + t] and the
// running product / its inverse through accs[t].  The forward pass reads only the x coordinates (dx is all it needs;
// x = 0 or dx = 0 fall back to the full classification).  (Inverting at the end of the forward kernel instead was measured
// on H100: the one-wave forward grid reaches its inversions together, so they stay a tail, and the forward loop compiles
// worse next to them -- slower than the separate pass.)
template <class CV, bool FIRST>
B2K_D void pt_denominator(typename CV::F& d, const Affine<typename CV::F>* in, const uint32_t* entries, uint32_t a, uint32_t end) {
  using F = typename CV::F;
  f_set_one(d);
  if (a + 1 >= end) return;                           // single operand: carried over
  F x1, x2, dx;
  if (FIRST) { x1 = in[entries[a] & 0x7fffffffu].x; x2 = in[entries[a + 1] & 0x7fffffffu].x; }
  else { x1 = in[a].x; x2 = in[a + 1].x; }
  f_sub(dx, x2, x1);
  if (!f_is_zero(x1) && !f_is_zero(x2) && !f_is_zero(dx)) { d = dx; return; }
  Affine<F> p1, p2;                                   // rare: possible infinity / doubling / cancellation
  const bool pair = pt_fetch<CV, FIRST>(p1, p2, in, entries, a, end);
  pt_classify(d, p1, p2, pair);
}

// forward: T = number of threads of the round (stride of pre[]); thread t leaves its running product in accs[t]
template <class CV, bool FIRST>
B2K_D void msm_pairtree_forward(uint32_t t, uint32_t B, uint32_t T, uint32_t total, const Affine<typename CV::F>* in,
                                const uint32_t* entries, const uint32_t* offs_in, const uint32_t* offs_out,
                                typename CV::F* pre, typename CV::F* accs) {
  using F = typename CV::F;
  const uint32_t nout = offs_out[total];
  const uint32_t q0 = t * B;
  if (q0 >= nout) return;
  const uint32_t q1 = (nout - q0 < B) ? nout : q0 + B;
  uint32_t g = msm_find_bucket(offs_out, total, q0);
  uint32_t os = offs_out[g], oe = offs_out[g + 1], is = offs_in[g], ie = offs_in[g + 1];
  F acc;
  f_set_one(acc);
  for (uint32_t q = q0; q < q1; q++) {
    while (q >= oe) { g++; os = oe; oe = offs_out[g + 1]; is = ie; ie = offs_in[g + 1]; }
    F d;
    pt_denominator<CV, FIRST>(d, in, entries, is + 2 * (q - os), ie);
    pre[(size_t)(q - q0) * T + t] = acc;
    f_mul_i(acc, acc, d);
  }
  accs[t] = acc;
}

// inversions: one per thread that has outputs
template <class F>
B2K_D void msm_pairtree_invert(uint32_t t, uint32_t B, uint32_t total, const uint32_t* offs_out, F* accs) {
  if ((uint64_t)t * B >= offs_out[total]) return;
  F v = accs[t], r;
  f_inv_bg(r, v);
  accs[t] = r;
}

// backward: the additions themselves
template <class CV, bool FIRST>
B2K_D void msm_pairtree_backward(uint32_t t, uint32_t B, uint32_t T, uint32_t total, const Affine<typename CV::F>* in,
                                 const uint32_t* entries, const uint32_t* offs_in, const uint32_t* offs_out,
                                 const typename CV::F* pre, const typename CV::F* accs, Affine<typename CV::F>* out) {
  using F = typename CV::F;
  const uint32_t nout = offs_out[total];
  const uint32_t q0 = t * B;
  if (q0 >= nout) return;
  const uint32_t q1 = (nout - q0 < B) ? nout : q0 + B;
  uint32_t g = msm_find_bucket(offs_out, total, q1 - 1);
  uint32_t os = offs_out[g], oe = offs_out[g + 1], is = offs_in[g], ie = offs_in[g + 1];
  (void)oe;
  F inv = accs[t];
  for (uint32_t q = q1; q-- > q0;) {
    while (q < os) { g--; os = offs_out[g]; ie = is; is = offs_in[g]; }
    Affine<F> p1, p2, r;
    F d, dinv, lam, tt;
    const bool pair = pt_fetch<CV, FIRST>(p1, p2, in, entries, is + 2 * (q - os), ie);
    const int kind = pt_classify(d, p1, p2, pair);
    F pj = pre[(size_t)(q - q0) * T + t];
    f_mul_i(dinv, inv, pj);
    if (q > q0) f_mul_i(inv, inv, d);
    if (kind == PT_DBL) { f_sqr(tt, p1.x); f_dbl(lam, tt); f_add(tt, lam, tt); }   // (rare: stays a call in the compact layout)
    else f_sub(tt, p2.y, p1.y);
    f_mul_i(lam, tt, dinv);
    f_sqr_i(r.x, lam); f_sub(r.x, r.x, p1.x); f_sub(r.x, r.x, p2.x);
    f_sub(tt, p1.x, r.x); f_mul_i(r.y, lam, tt); f_sub(r.y, r.y, p1.y);
    if (kind == PT_COPY1) r = p1;
    else if (kind == PT_COPY2) r = p2;
    else if (kind == PT_INF) aff_set_inf(r);
    out[q] = r;
  }
}

// ---- backward pass with asynchronously staged operands ---------------------------------------------------------------------
// ncu on the split rounds: the backward kernels spend a sizeable share of their cycles per
// issued instruction waiting for the two operand points of the output they are about to compute (`long_scoreboard`; round 0 gathers
// them through the sorted entries, a DRAM round trip), with the multiply pipe busy most of the time.  Prefetching them into registers costs the
// 48 registers the kernel does not have (128 = 4 blocks per SM), and `prefetch.global.L1` measured slower.  Here the operands of
// output q-1 travel global -> shared memory with cp.async (LDGSTS, 16 bytes each, no register staging) while output q is computed:
// per thread two 2-point buffers and one slot for the prefix product (4 x 96 + 48 B; 54 KB per block of 128 threads, four blocks per SM as before).  Round 0 also loads
// the two sorted entries of output q-2, so that the gather addresses of q-1 are in registers when its copies are issued.
namespace stage {
#ifndef B2K_HOST_EMUL
using addr_t = uint32_t;                                     // shared-window address
B2K_D addr_t addr(void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
B2K_D void cp16(addr_t dst, const void* src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory"); }
B2K_D void commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> B2K_D void wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
#else
// host emulation (tests/host_emul): copies really are deferred -- they land when a wait retires their group, oldest first -- so a
// schedule that reads a buffer too early or overwrites one too soon fails the emulation tests, not only the GPU run
using addr_t = unsigned char*;
struct Piece { unsigned char* dst; const unsigned char* src; };
inline std::vector<std::vector<Piece>>& groups() { static thread_local std::vector<std::vector<Piece>> g(1); return g; }
inline addr_t addr(void* p) { return reinterpret_cast<unsigned char*>(p); }
inline void cp16(addr_t dst, const void* src) { groups().back().push_back({dst, reinterpret_cast<const unsigned char*>(src)}); }
inline void commit() { groups().emplace_back(); }
template <int N> inline void wait() {
  auto& g = groups();                                        // g.back() is the open (uncommitted) group
  while (g.size() > (size_t)N + 1) {
    for (const Piece& c : g.front()) memcpy(c.dst, c.src, 16);
    g.erase(g.begin());
  }
}
#endif
template <int BYTES> B2K_D void copy(addr_t dst, const void* src) {
  static_assert(BYTES % 16 == 0, "16-byte pieces");
#pragma unroll
  for (int i = 0; i < BYTES / 16; i++) cp16(dst + 16 * i, reinterpret_cast<const unsigned char*>(src) + 16 * i);
}
}  // namespace stage

// where the operands of one output live: input position a of a run ending at `end`; round 0: the two sorted entries at a, a + 1
struct PtLook { uint32_t a, end, v0, v1; };

template <class CV, bool FIRST>
B2K_D void msm_pairtree_backward_staged(uint32_t t, uint32_t B, uint32_t T, uint32_t total, const Affine<typename CV::F>* in,
                                        const uint32_t* entries, const uint32_t* offs_in, const uint32_t* offs_out,
                                        const typename CV::F* pre, const typename CV::F* accs, Affine<typename CV::F>* out,
                                        unsigned char* smem, uint32_t lane) {
  using F = typename CV::F;
  using A = Affine<F>;
  static_assert(sizeof(A) % 16 == 0, "cp.async moves 16-byte pieces");
  const uint32_t nout = offs_out[total];
  const uint32_t q0 = t * B;
  if (q0 >= nout) return;                                    // (no block-wide barrier below: every thread waits for its own copies only)
  const uint32_t q1 = (nout - q0 < B) ? nout : q0 + B;
  // per thread: [2 buffers][2 operand points] + [1 prefix product]  (PT_STAGE_BYTES<F> below)
  unsigned char* mine = smem + (size_t)lane * (4 * sizeof(A) + sizeof(F));
  A* slot = reinterpret_cast<A*>(mine);
  F* pslot = reinterpret_cast<F*>(mine + 4 * sizeof(A));
  const stage::addr_t sbase = stage::addr(slot), spre = stage::addr(pslot);
  uint32_t g = msm_find_bucket(offs_out, total, q1 - 1);
  uint32_t os = offs_out[g], is = offs_in[g], ie = offs_in[g + 1];
  // the bucket cursor only moves backwards; look(q) must be called with decreasing q
  auto look = [&](uint32_t q) {
    while (q < os) { g--; os = offs_out[g]; ie = is; is = offs_in[g]; }
    PtLook L;
    L.a = is + 2 * (q - os); L.end = ie; L.v0 = 0; L.v1 = 0;
    if (FIRST) { L.v0 = entries[L.a]; L.v1 = (L.a + 1 < L.end) ? entries[L.a + 1] : L.v0; }
    return L;
  };
  auto issue = [&](const PtLook& L, int buf, uint32_t q) {   // the two operands of output q into buffer `buf`, its prefix product into the one slot
    const stage::addr_t dst = sbase + (uint32_t)(2 * buf * sizeof(A));
    if (FIRST) {
      stage::copy<sizeof(A)>(dst, in + (L.v0 & 0x7fffffffu));
      if (L.a + 1 < L.end) stage::copy<sizeof(A)>(dst + (uint32_t)sizeof(A), in + (L.v1 & 0x7fffffffu));
    } else {
      stage::copy<sizeof(A)>(dst, in + L.a);
      if (L.a + 1 < L.end) stage::copy<sizeof(A)>(dst + (uint32_t)sizeof(A), in + L.a + 1);
    }
    stage::copy<sizeof(F)>(spre, pre + (size_t)(q - q0) * T + t);
  };
  PtLook cur = look(q1 - 1), nxt = cur;
  issue(cur, 0, q1 - 1);
  stage::commit();
  bool have_nxt = q1 - 1 > q0;
  if (have_nxt) nxt = look(q1 - 2);
  F inv = accs[t];
  int k = 0;
  for (uint32_t q = q1 - 1;; q--, k ^= 1) {
    stage::wait<0>();                                        // the one group in flight: operands + prefix product of output q
    const bool pair = cur.a + 1 < cur.end;
    Affine<F> p1 = slot[2 * k], p2, r;
    if (pair) p2 = slot[2 * k + 1]; else p2 = p1;
    F pj = *pslot;
    if (FIRST) {
      if (cur.v0 >> 31) f_neg(p1.y, p1.y);
      if (pair) { if (cur.v1 >> 31) f_neg(p2.y, p2.y); } else p2.y = p1.y;
    }
    F d, dinv, lam, tt;
    const int kind = pt_classify(d, p1, p2, pair);
    f_mul_i(dinv, inv, pj);                                  // consumes pj: its shared-memory read is complete, the slot may be refilled
    PtLook aft = nxt;
    bool have_aft = false;
    if (have_nxt) {
      issue(nxt, k ^ 1, q - 1);                              // output q-1 (round 0: its entries were loaded during the previous iteration)
      if (q - 1 > q0) { aft = look(q - 2); have_aft = true; }
    }
    stage::commit();
    if (q > q0) f_mul_i(inv, inv, d);
    if (kind == PT_DBL) { f_sqr(tt, p1.x); f_dbl(lam, tt); f_add(tt, lam, tt); }
    else f_sub(tt, p2.y, p1.y);
    f_mul_i(lam, tt, dinv);
    f_sqr_i(r.x, lam); f_sub(r.x, r.x, p1.x); f_sub(r.x, r.x, p2.x);
    f_sub(tt, p1.x, r.x); f_mul_i(r.y, lam, tt); f_sub(r.y, r.y, p1.y);
    if (kind == PT_COPY1) r = p1;
    else if (kind == PT_COPY2) r = p2;
    else if (kind == PT_INF) aff_set_inf(r);
    out[q] = r;
    if (q == q0) break;
    cur = nxt; nxt = aft; have_nxt = have_aft;
  }
  stage::wait<0>();
}

// forward pass, staged the same way: only the two x coordinates of an output travel (48 bytes each; the rare x = 0 / equal-x
// cases re-read the full points).  ncu: this pass waits 6-9 of its 15 cycles per issued instruction for them.
template <class CV, bool FIRST>
B2K_D void msm_pairtree_forward_staged(uint32_t t, uint32_t B, uint32_t T, uint32_t total, const Affine<typename CV::F>* in,
                                       const uint32_t* entries, const uint32_t* offs_in, const uint32_t* offs_out,
                                       typename CV::F* pre, typename CV::F* accs, unsigned char* smem, uint32_t lane) {
  using F = typename CV::F;
  static_assert(sizeof(F) % 16 == 0, "cp.async moves 16-byte pieces");
  const uint32_t nout = offs_out[total];
  const uint32_t q0 = t * B;
  if (q0 >= nout) return;
  const uint32_t q1 = (nout - q0 < B) ? nout : q0 + B;
  F* slot = reinterpret_cast<F*>(smem) + 4 * lane;           // [buffer][x1, x2]
  const stage::addr_t sbase = stage::addr(slot);
  uint32_t g = msm_find_bucket(offs_out, total, q0);
  uint32_t os = offs_out[g], oe = offs_out[g + 1], is = offs_in[g], ie = offs_in[g + 1];
  auto look = [&](uint32_t q) {                              // increasing q only
    while (q >= oe) { g++; os = oe; oe = offs_out[g + 1]; is = ie; ie = offs_in[g + 1]; }
    PtLook L;
    L.a = is + 2 * (q - os); L.end = ie; L.v0 = 0; L.v1 = 0;
    if (FIRST && L.a + 1 < L.end) { L.v0 = entries[L.a]; L.v1 = entries[L.a + 1]; }
    return L;
  };
  auto issue = [&](const PtLook& L, int buf) {
    if (L.a + 1 >= L.end) return;                            // single operand: carried over, nothing to invert
    const stage::addr_t dst = sbase + (uint32_t)(2 * buf * sizeof(F));
    const Affine<F>* s1 = FIRST ? in + (L.v0 & 0x7fffffffu) : in + L.a;
    const Affine<F>* s2 = FIRST ? in + (L.v1 & 0x7fffffffu) : in + L.a + 1;
    stage::copy<sizeof(F)>(dst, &s1->x);
    stage::copy<sizeof(F)>(dst + (uint32_t)sizeof(F), &s2->x);
  };
  PtLook cur = look(q0), nxt = cur;
  issue(cur, 0);
  stage::commit();
  bool have_nxt = q0 + 1 < q1;
  if (have_nxt) nxt = look(q0 + 1);
  F acc;
  f_set_one(acc);
  int k = 0;
  for (uint32_t q = q0;; q++, k ^= 1) {
    PtLook aft = nxt;
    bool have_aft = false;
    if (have_nxt) {
      issue(nxt, k ^ 1);
      if (q + 2 < q1) { aft = look(q + 2); have_aft = true; }
    }
    stage::commit();
    stage::wait<1>();
    F d;
    f_set_one(d);
    if (cur.a + 1 < cur.end) {
      F x1 = slot[2 * k], x2 = slot[2 * k + 1], dx;
      f_sub(dx, x2, x1);
      if (!f_is_zero(x1) && !f_is_zero(x2) && !f_is_zero(dx)) d = dx;
      else {                                                 // rare: possible infinity / doubling / cancellation
        Affine<F> p1, p2;
        const bool pair = pt_fetch<CV, FIRST>(p1, p2, in, entries, cur.a, cur.end);
        pt_classify(d, p1, p2, pair);
      }
    }
    pre[(size_t)(q - q0) * T + t] = acc;
    f_mul_i(acc, acc, d);
    if (q + 1 == q1) break;
    cur = nxt; nxt = aft; have_nxt = have_aft;
  }
  stage::wait<0>();
  accs[t] = acc;
}

}  // namespace b2k
