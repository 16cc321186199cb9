// fp.cuh -- prime-field arithmetic in Montgomery form, 32-bit limbs held in registers.
//
// One template serves every base field on the hot path:
//   Bls381Fp (N=12 limbs)  -- replaces the third-party 6x64-bit Go/asm field under
//                             pairing/bls12381/kilic (reference call sites kilic/g1.go:110-116)
//   Bn254Fp  (N=8 limbs)   -- replaces gfpMul/gfpAdd/gfpSub/gfpNeg, pairing/bn254/gfp_amd64.s:39-129,
//                             gfp_generic.go:26-173 (256-bit CIOS Montgomery, R = 2^256)
// A config class C supplies N, M0 = -p^-1 mod 2^32 and mod(j)/r1(j)/r2(j) limb accessors that are
// compile-time constants after unrolling (they become IMAD immediates, no constant-bank traffic).
//
// Montgomery product layout ("even/odd wide rows"): the running sum T is kept as two interleaved
// accumulators whose 64-bit slots are aligned to even resp. odd limb positions, so that every
// a[j]*b[i] product is ONE 64-bit multiply-add into one slot, carries rippling slot to slot along a
// row (IMAD.WIDE.U32 + .X in SASS).  After the reduction row the sum is divided by 2^32, which swaps
// the roles of the two accumulators; the single stray limb that changes parity is fed into the next
// row as its carry-in.  Cost per product: 2*N*N/2 + N*N ... = 2*N^2 32x32->64 multiply-adds + O(N).
#pragma once
#include "ptx.cuh"

namespace b2k {

template <class C>
struct alignas(16) Fp {
  static constexpr int N = C::N;
  uint32_t v[N];
};

namespace detail {

// acc[j..j+1] = a[j]*b   (j even, j < N)
template <int N>
B2K_D void row_mul(uint32_t* acc, const uint32_t* a, uint32_t b) {
#pragma unroll
  for (int j = 0; j < N; j += 2) {
    acc[j] = ptx::mul_lo(a[j], b);
    acc[j + 1] = ptx::mul_hi(a[j], b);
  }
}

// acc[j..j+1] += a[j]*b  with the carry rippling upward; leaves the row's carry-out in CC.
template <int N>
B2K_D void row_mad(uint32_t* acc, const uint32_t* a, uint32_t b) {
  acc[0] = ptx::mad_lo_cc(a[0], b, acc[0]);
  acc[1] = ptx::madc_hi_cc(a[0], b, acc[1]);
#pragma unroll
  for (int j = 2; j < N; j += 2) {
    acc[j] = ptx::madc_lo_cc(a[j], b, acc[j]);
    acc[j + 1] = ptx::madc_hi_cc(a[j], b, acc[j + 1]);
  }
}

// Same with carry-IN from CC, reading the accumulator two limbs higher (the /2^32 role swap):
// acc[j..j+1] = a[j]*b + acc[j+2..j+3];  the top slot gets a[N-2]*b + 0.  No carry-out by bound.
template <int N>
B2K_D void row_madc_shift(uint32_t* acc, const uint32_t* a, uint32_t b) {
#pragma unroll
  for (int j = 0; j < N - 2; j += 2) {
    acc[j] = ptx::madc_lo_cc(a[j], b, acc[j + 2]);
    acc[j + 1] = ptx::madc_hi_cc(a[j], b, acc[j + 3]);
  }
  acc[N - 2] = ptx::madc_lo_cc(a[N - 2], b, 0);
  acc[N - 1] = ptx::madc_hi(a[N - 2], b, 0);
}

// acc += m * MOD[OFF], MOD[OFF+2], ...  (modulus limbs are immediates)
template <class C, int OFF>
B2K_D void row_mad_mod(uint32_t* acc, uint32_t m) {
  acc[0] = ptx::mad_lo_cc(C::mod(OFF), m, acc[0]);
  acc[1] = ptx::madc_hi_cc(C::mod(OFF), m, acc[1]);
#pragma unroll
  for (int j = 2; j < C::N; j += 2) {
    acc[j] = ptx::madc_lo_cc(C::mod(OFF + j), m, acc[j]);
    acc[j + 1] = ptx::madc_hi_cc(C::mod(OFF + j), m, acc[j + 1]);
  }
}

// One "multiply row by b, reduce one limb" step.  lo = accumulator whose slot 0 is limb position 0.
template <class C, bool FIRST>
B2K_D void mont_step(uint32_t* lo, uint32_t* hi, const uint32_t* a, uint32_t b) {
  constexpr int N = C::N;
  if (FIRST) {
    row_mul<N>(hi, a + 1, b);
    row_mul<N>(lo, a, b);
  } else {
    lo[0] = ptx::add_cc(lo[0], hi[1]);      // the stray limb (position 0 after the shift)
    row_madc_shift<N>(hi, a + 1, b);        // odd limbs of a, old hi read two limbs up
    row_mad<N>(lo, a, b);                   // even limbs of a
    hi[N - 1] = ptx::addc(hi[N - 1], 0);
  }
  uint32_t m = lo[0] * C::M0;
  row_mad_mod<C, 1>(hi, m);
  row_mad_mod<C, 0>(lo, m);
  hi[N - 1] = ptx::addc(hi[N - 1], 0);
}

// ---- wide (unreduced) products and the stand-alone Montgomery reduction ---------------------------------------------
// Used by fp_sqr (N(N+1)/2 products instead of N^2 before the reduction) and by the lazily reduced Fp2 product of
// tower.cuh (three wide products, two reductions).  Same even/odd idea as above without the sliding: E[k] sits at limb k,
// O[k] at limb k + 1, 64-bit slots start at even indices of either array, so every 32x32 product is one multiply-add into
// one slot and a row is two carry chains.  Rows are issued in an order in which the limb right above a chain's last slot
// has only ever received carries (chain ends never move down), so one add absorbs the chain's carry-out.

// acc[s + 2t .. s + 2t + 1] += a[j0 + 2t] * b for t < CNT as one carry chain; carry-out into acc[s + 2 CNT] if that is < LIM
template <int CNT, int LIM>
B2K_D void chain_mad(uint32_t* acc, int s, const uint32_t* a, int j0, uint32_t b) {
  if (CNT <= 0) return;
  acc[s] = ptx::mad_lo_cc(a[j0], b, acc[s]);
  acc[s + 1] = ptx::madc_hi_cc(a[j0], b, acc[s + 1]);
#pragma unroll
  for (int t = 1; t < CNT; t++) {
    acc[s + 2 * t] = ptx::madc_lo_cc(a[j0 + 2 * t], b, acc[s + 2 * t]);
    acc[s + 2 * t + 1] = ptx::madc_hi_cc(a[j0 + 2 * t], b, acc[s + 2 * t + 1]);
  }
  if (s + 2 * CNT < LIM) acc[s + 2 * CNT] = ptx::addc(acc[s + 2 * CNT], 0);
  else ptx::addc(0, 0);                      // (no carry by bound; consumes CC so that nothing stale is left behind)
}

// t[0..2N) = E + (O << 32)
template <int N>
B2K_D void wide_merge(uint32_t* t, const uint32_t* E, const uint32_t* O) {
  t[0] = E[0];
  t[1] = ptx::add_cc(E[1], O[0]);
#pragma unroll
  for (int k = 2; k < 2 * N - 1; k++) t[k] = ptx::addc_cc(E[k], O[k - 1]);
  t[2 * N - 1] = ptx::addc(E[2 * N - 1], O[2 * N - 2]);
}

// t[0..2N) = a * b   (N^2 multiply-adds)
template <int N>
B2K_D void wide_mul(uint32_t* t, const uint32_t* a, const uint32_t* b) {
  uint32_t E[2 * N], O[2 * N];
#pragma unroll
  for (int k = 0; k < 2 * N; k++) { E[k] = 0; O[k] = 0; }
#pragma unroll
  for (int i = 0; i < N; i += 2) {
    chain_mad<N / 2, 2 * N>(E, i, a, 0, b[i]);          // a_even * b_i   at limbs i + j
    chain_mad<N / 2, 2 * N>(O, i, a, 1, b[i]);          // a_odd  * b_i   at limbs i + j = (i + j - 1) + 1
    chain_mad<N / 2, 2 * N>(O, i, a, 0, b[i + 1]);      // a_even * b_i+1 at limbs i + 1 + j
    chain_mad<N / 2, 2 * N>(E, i + 2, a, 1, b[i + 1]);  // a_odd  * b_i+1 at limbs i + 1 + j (even)
  }
  wide_merge<N>(t, E, O);
}

// rows I and I + 1 of the off-diagonal triangle: row r = a_r * a_j, j = r+1, r+3, ... lands on odd limbs r + j -> O[r + j - 1],
// j = r+2, r+4, ... on even limbs -> E[r + j]   (template recursion: the chain lengths are compile-time)
template <int N, int I>
B2K_D void wide_sqr_rows(uint32_t* E, uint32_t* O, const uint32_t* a) {
  if constexpr (I + 1 < N) {
    chain_mad<(N - I) / 2, 2 * N>(O, 2 * I, a, I + 1, a[I]);
    chain_mad<(N - 1 - I) / 2, 2 * N>(E, 2 * I + 2, a, I + 2, a[I]);
    chain_mad<(N - 1 - I) / 2, 2 * N>(O, 2 * I + 2, a, I + 2, a[I + 1]);
    chain_mad<(N - 2 - I) / 2, 2 * N>(E, 2 * I + 4, a, I + 3, a[I + 1]);
    wide_sqr_rows<N, I + 2>(E, O, a);
  }
}

// t[0..2N) = a^2   (N(N-1)/2 off-diagonal multiply-adds, doubled by a one-bit shift, + N diagonal ones)
template <int N>
B2K_D void wide_sqr(uint32_t* t, const uint32_t* a) {
  uint32_t E[2 * N], O[2 * N], m[2 * N];
#pragma unroll
  for (int k = 0; k < 2 * N; k++) { E[k] = 0; O[k] = 0; }
  wide_sqr_rows<N, 0>(E, O, a);
  wide_merge<N>(m, E, O);
  // t = 2 m + sum_i a_i^2 2^(64 i)
  t[0] = ptx::mad_lo_cc(a[0], a[0], 0);
  t[1] = ptx::madc_hi_cc(a[0], a[0], m[1] << 1);      // m[0] = 0 (no product lands on limb 0)
#pragma unroll
  for (int i = 1; i < N; i++) {
    t[2 * i] = ptx::madc_lo_cc(a[i], a[i], (m[2 * i] << 1) | (m[2 * i - 1] >> 31));
    t[2 * i + 1] = ptx::madc_hi_cc(a[i], a[i], (m[2 * i + 1] << 1) | (m[2 * i] >> 31));
  }
  ptx::addc(0, 0);
}

// hi[j..j+1] = MOD[1 + j] * m + hi[j+2..j+3] with carry-in from CC (the /2^32 role swap fused into the odd modulus row)
template <class C>
B2K_D void row_madc_shift_mod(uint32_t* acc, uint32_t m) {
  constexpr int N = C::N;
#pragma unroll
  for (int j = 0; j < N - 2; j += 2) {
    acc[j] = ptx::madc_lo_cc(C::mod(1 + j), m, acc[j + 2]);
    acc[j + 1] = ptx::madc_hi_cc(C::mod(1 + j), m, acc[j + 3]);
  }
  acc[N - 2] = ptx::madc_lo_cc(C::mod(N - 1), m, 0);
  acc[N - 1] = ptx::madc_hi(C::mod(N - 1), m, 0);
}

template <class C, bool FIRST>
B2K_D void redc_step(uint32_t* lo, uint32_t* hi) {
  constexpr int N = C::N;
  if (FIRST) {
    const uint32_t m = lo[0] * C::M0;
#pragma unroll
    for (int j = 0; j < N; j += 2) { hi[j] = ptx::mul_lo(C::mod(1 + j), m); hi[j + 1] = ptx::mul_hi(C::mod(1 + j), m); }
    row_mad_mod<C, 0>(lo, m);
  } else {
    lo[0] = ptx::add_cc(lo[0], hi[1]);      // the stray limb; its carry enters the odd row below
    const uint32_t m = lo[0] * C::M0;
    row_madc_shift_mod<C>(hi, m);
    row_mad_mod<C, 0>(lo, m);
  }
  hi[N - 1] = ptx::addc(hi[N - 1], 0);
}

// r[0..N) = t / 2^(32N) mod p, in [0, 2p) for t < p 2^(32N)   (N^2 multiply-adds; caller finishes with fp_reduce_once)
template <class C>
B2K_D void redc_wide(uint32_t* r, const uint32_t* t) {
  constexpr int N = C::N;
  uint32_t ev[N], od[N];
#pragma unroll
  for (int j = 0; j < N; j++) ev[j] = t[j];
#pragma unroll
  for (int i = 0; i < N; i += 2) {
    if (i == 0) redc_step<C, true>(ev, od);
    else redc_step<C, false>(ev, od);
    redc_step<C, false>(od, ev);
  }
  ev[0] = ptx::add_cc(ev[0], od[1]);        // REDC(t mod 2^(32N)) <= p ...
#pragma unroll
  for (int j = 1; j < N - 1; j++) ev[j] = ptx::addc_cc(ev[j], od[j + 1]);
  ev[N - 1] = ptx::addc(ev[N - 1], 0);
  r[0] = ptx::add_cc(ev[0], t[N]);          // ... + floor(t / 2^(32N))
#pragma unroll
  for (int j = 1; j < N - 1; j++) r[j] = ptx::addc_cc(ev[j], t[N + j]);
  r[N - 1] = ptx::addc(ev[N - 1], t[2 * N - 1]);
}

// ---- one-level subtractive Karatsuba wide products (the sum of two products of the XYZZ formulas, ec.cuh) -------------------
// With H = N/2, B = 2^(32H), a = a0 + a1 B, b = b0 + b1 B, z0 = a0 b0, z2 = a1 b1:
//   a b = z0 + (z0 + z2 - (a0 - a1)(b0 - b1)) B + z2 B^2,
// where (a0 - a1)(b0 - b1) = +-|a0 - a1| |b0 - b1| by the signs of the two differences.  3 H^2 = 3/4 N^2 multiply-adds
// instead of N^2, for ~110 additions and selects that run on the integer ALU, which the FMA-heavy pipe leaves idle.  The
// halves go through wide_mul<H>, whose rows pair limbs, so H must be even: N = 12 and 8.  N = 10 (bn256) keeps the
// schoolbook wide_mul.

// d = |x0 - x1| for the two H-limb halves of x; returns all-ones if x0 < x1, else 0 (also when x0 = x1: d = 0)
template <int H>
B2K_D uint32_t half_absdiff(uint32_t* d, const uint32_t* x) {
  d[0] = ptx::sub_cc(x[0], x[H]);
#pragma unroll
  for (int j = 1; j < H; j++) d[j] = ptx::subc_cc(x[j], x[H + j]);
  const uint32_t neg = ptx::subc(0, 0);
  d[0] = ptx::add_cc(d[0] ^ neg, neg & 1u);          // two's complement negation when negative: (d ^ ~0) + 1
#pragma unroll
  for (int j = 1; j < H - 1; j++) d[j] = ptx::addc_cc(d[j] ^ neg, 0);
  d[H - 1] = ptx::addc(d[H - 1] ^ neg, 0);
  return neg;
}

// One Karatsuba term a b into (t, mid), with H even.  FIRST: t = z0 + z2 B^2 and mid = z0 + z2 -+ |a0 - a1| |b0 - b1|; later terms
// add to both, z2 before z0, so that every partial sum stays below the final one and the carry out of the top limb is 0.
// mid holds N + 1 limbs modulo 2^(32(N+1)): it starts from the signed |..||..|, so only one half-product and the half-operand
// pair it needs are live at a time; a term's middle part lies in [0, 2^(64H+1)), two of them below 2^(32(N+1)).
template <int N, bool FIRST>
B2K_D void kara_term(uint32_t* t, uint32_t* mid, const uint32_t* a, const uint32_t* b) {
  constexpr int H = N / 2;
  uint32_t z[N], da[H], db[H];
  const uint32_t sa = half_absdiff<H>(da, a), sb = half_absdiff<H>(db, b);
  wide_mul<H>(z, da, db);
  const uint32_t m = ~(sa ^ sb);                      // all-ones: (a0 - a1)(b0 - b1) >= 0, so the middle part subtracts it
  ptx::add_cc(m, m & 1u);                             // carry-in 1 for the two's complement (~0 + 1 carries, 0 + 0 does not)
#pragma unroll
  for (int j = 0; j < N; j++) mid[j] = ptx::addc_cc(FIRST ? 0 : mid[j], z[j] ^ m);
  mid[N] = ptx::addc(FIRST ? 0 : mid[N], m);
  wide_mul<H>(z, a + H, b + H);                       // z2
  if (FIRST) {
#pragma unroll
    for (int j = 0; j < N; j++) t[N + j] = z[j];
  } else {
    t[N] = ptx::add_cc(t[N], z[0]);
#pragma unroll
    for (int j = 1; j < N - 1; j++) t[N + j] = ptx::addc_cc(t[N + j], z[j]);
    t[2 * N - 1] = ptx::addc(t[2 * N - 1], z[N - 1]);
  }
  mid[0] = ptx::add_cc(mid[0], z[0]);
#pragma unroll
  for (int j = 1; j < N; j++) mid[j] = ptx::addc_cc(mid[j], z[j]);
  mid[N] = ptx::addc(mid[N], 0);
  wide_mul<H>(z, a, b);                               // z0
  if (FIRST) {
#pragma unroll
    for (int j = 0; j < N; j++) t[j] = z[j];
  } else {
    t[0] = ptx::add_cc(t[0], z[0]);
#pragma unroll
    for (int j = 1; j < N; j++) t[j] = ptx::addc_cc(t[j], z[j]);
#pragma unroll
    for (int j = N; j < 2 * N - 1; j++) t[j] = ptx::addc_cc(t[j], 0);
    t[2 * N - 1] = ptx::addc(t[2 * N - 1], 0);
  }
  mid[0] = ptx::add_cc(mid[0], z[0]);
#pragma unroll
  for (int j = 1; j < N; j++) mid[j] = ptx::addc_cc(mid[j], z[j]);
  mid[N] = ptx::addc(mid[N], 0);
}

// t += mid B
template <int N>
B2K_D void kara_finish(uint32_t* t, const uint32_t* mid) {
  constexpr int H = N / 2;
  t[H] = ptx::add_cc(t[H], mid[0]);
#pragma unroll
  for (int j = 1; j <= N; j++) t[H + j] = ptx::addc_cc(t[H + j], mid[j]);
#pragma unroll
  for (int k = H + N + 1; k < 2 * N - 1; k++) t[k] = ptx::addc_cc(t[k], 0);
  t[2 * N - 1] = ptx::addc(t[2 * N - 1], 0);
}

// t[0..2N) = a * b + c * d for a sum below 2^(64N); the two middle parts share one mid and one shifted addition
template <int N>
B2K_D void wide_mul_kara_sum2(uint32_t* t, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d) {
  static_assert(N % 4 == 0, "Karatsuba halves of an even limb count");
  uint32_t mid[N + 1];
  kara_term<N, true>(t, mid, a, b);
  kara_term<N, false>(t, mid, c, d);
  kara_finish<N>(t, mid);
}

}  // namespace detail

// ---- comparison / conditional subtraction ---------------------------------------------------
// r = a - MOD if a >= MOD else a          (a < 2*MOD)
template <class C>
B2K_D void fp_reduce_once(uint32_t* a) {
  constexpr int N = C::N;
  uint32_t t[N];
  t[0] = ptx::sub_cc(a[0], C::mod(0));
#pragma unroll
  for (int j = 1; j < N; j++) t[j] = ptx::subc_cc(a[j], C::mod(j));
  uint32_t borrow = ptx::subc(0, 0);  // 0xffffffff if a < MOD
#pragma unroll
  for (int j = 0; j < N; j++) a[j] = borrow ? a[j] : t[j];
}

template <class C>
B2K_D void fp_mul_inl(Fp<C>& r, const Fp<C>& a, const Fp<C>& b) {
  constexpr int N = C::N;
  static_assert(N % 2 == 0, "even limb count");
  static_assert(C::BITS <= 32 * C::N - 1, "p < 2^(32N-1): the merged rows and fp_reduce_once carry nothing out of the top limb");
  uint32_t ev[N], od[N];
#pragma unroll
  for (int i = 0; i < N; i += 2) {
    if (i == 0)
      detail::mont_step<C, true>(ev, od, a.v, b.v[0]);
    else
      detail::mont_step<C, false>(ev, od, a.v, b.v[i]);
    detail::mont_step<C, false>(od, ev, a.v, b.v[i + 1]);
  }
  // merge: ev[0] is limb 0; od[k] sits at limb k-1 (its slot 0 was the stray limb)
  ev[0] = ptx::add_cc(ev[0], od[1]);
#pragma unroll
  for (int j = 1; j < N - 1; j++) ev[j] = ptx::addc_cc(ev[j], od[j + 1]);
  ev[N - 1] = ptx::addc(ev[N - 1], 0);
  fp_reduce_once<C>(ev);
#pragma unroll
  for (int j = 0; j < N; j++) r.v[j] = ev[j];
}

// a^2: N(N+1)/2 + N^2 multiply-adds instead of 2 N^2 (BLS12-381: 222 instead of 288)
template <class C>
B2K_D void fp_sqr_inl(Fp<C>& r, const Fp<C>& a) {
  constexpr int N = C::N;
  uint32_t t[2 * N], u[N];
  detail::wide_sqr<N>(t, a.v);
  detail::redc_wide<C>(u, t);
  fp_reduce_once<C>(u);
#pragma unroll
  for (int j = 0; j < N; j++) r.v[j] = u[j];
}


// (a b + c d) R^-1 with ONE reduction: both products accumulate into one wide buffer, a b + c d < 2 p^2 < p 2^(32N) for
// operands below p (2 p < 2^(32N) for every field here), which is what redc_wide needs.  N = 10 (bn256), whose halves would
// have an odd limb count, adds two CIOS products instead.
template <class C>
B2K_D void fp_mul_sum2_inl(Fp<C>& r, const Fp<C>& a, const Fp<C>& b, const Fp<C>& c, const Fp<C>& d) {
  constexpr int N = C::N;
  if constexpr (N % 4 != 0) {
    Fp<C> ab, cd;
    fp_mul_inl(ab, a, b);
    fp_mul_inl(cd, c, d);
    fp_add(r, ab, cd);
  } else {
    uint32_t t[2 * N], u[N];
    detail::wide_mul_kara_sum2<N>(t, a.v, b.v, c.v, d.v);
    detail::redc_wide<C>(u, t);
    fp_reduce_once<C>(u);
#pragma unroll
    for (int j = 0; j < N; j++) r.v[j] = u[j];
  }
}

// ---- code layout of the two products ----------------------------------------------------------------------------------------
// Default: fully inlined at every use (a 381-bit product is ~330 instructions = 5.3 KB of SASS).  A translation unit compiled
// with B2K_COMPACT_FIELD gets ONE out-of-line copy of each product instead, called BY VALUE: nvcc passes the 2 x N operand
// words and the N result words in registers (no local-memory round trip; verified in SASS: no LDL/STL around the CALL), at
// the price of ~3 N register moves per call.  Why it matters: the instruction caches are small (L0 ~6 KB, L1.5 32 KB per SM,
// then L2): ncu shows the pairing kernel stalled 35 % of its cycles on instruction fetch (`no_instruction`) with 530 KB of
// code, and the XYZZ bucket kernel 22 % with 53 KB per loop iteration.
// always inlined, whatever the layout of the translation unit (the affine pair-tree rounds measured faster that way)
template <class C> B2K_D void fp_mul_i(Fp<C>& r, const Fp<C>& a, const Fp<C>& b) { fp_mul_inl(r, a, b); }
template <class C> B2K_D void fp_sqr_i(Fp<C>& r, const Fp<C>& a) { fp_sqr_inl(r, a); }
#ifdef B2K_COMPACT_FIELD
template <class C> B2K_NI Fp<C> fp_mul_v(Fp<C> a, Fp<C> b) { Fp<C> r; fp_mul_inl(r, a, b); return r; }
template <class C> B2K_NI Fp<C> fp_sqr_v(Fp<C> a) { Fp<C> r; fp_sqr_inl(r, a); return r; }
template <class C> B2K_D void fp_mul(Fp<C>& r, const Fp<C>& a, const Fp<C>& b) { r = fp_mul_v<C>(a, b); }
template <class C> B2K_D void fp_sqr(Fp<C>& r, const Fp<C>& a) { r = fp_sqr_v<C>(a); }
#else
template <class C> B2K_D void fp_mul(Fp<C>& r, const Fp<C>& a, const Fp<C>& b) { fp_mul_inl(r, a, b); }
template <class C> B2K_D void fp_sqr(Fp<C>& r, const Fp<C>& a) { fp_sqr_inl(r, a); }
#endif

// the sum of two products (fp_mul_sum2_inl), same layout rule; operands and result by value in the compact layout
#ifdef B2K_COMPACT_FIELD
template <class C> B2K_NI Fp<C> fp_mul_sum2_v(Fp<C> a, Fp<C> b, Fp<C> c, Fp<C> d) { Fp<C> r; fp_mul_sum2_inl(r, a, b, c, d); return r; }
template <class C>
B2K_D void fp_mul_sum2(Fp<C>& r, const Fp<C>& a, const Fp<C>& b, const Fp<C>& c, const Fp<C>& d) { r = fp_mul_sum2_v<C>(a, b, c, d); }
#else
template <class C>
B2K_D void fp_mul_sum2(Fp<C>& r, const Fp<C>& a, const Fp<C>& b, const Fp<C>& c, const Fp<C>& d) { fp_mul_sum2_inl(r, a, b, c, d); }
#endif

// out-of-line copies for code that is too large to inline a 300-instruction product at every use
// (towers, exponentiations); operands then travel through local memory.
#ifdef B2K_COMPACT_FIELD
template <class C> B2K_D void fp_mul_c(Fp<C>& r, const Fp<C>& a, const Fp<C>& b) { fp_mul(r, a, b); }
template <class C> B2K_D void fp_sqr_c(Fp<C>& r, const Fp<C>& a) { fp_sqr(r, a); }
#else
template <class C>
B2K_NI void fp_mul_c(Fp<C>& r, const Fp<C>& a, const Fp<C>& b) { fp_mul(r, a, b); }
template <class C>
B2K_NI void fp_sqr_c(Fp<C>& r, const Fp<C>& a) { fp_sqr(r, a); }
#endif

template <class C>
B2K_D void fp_add(Fp<C>& r, const Fp<C>& a, const Fp<C>& b) {
  constexpr int N = C::N;
  static_assert(C::BITS <= 32 * C::N - 1, "p < 2^(32N-1): the sum of two operands below p has no carry out of the top limb");
  uint32_t t[N];
  t[0] = ptx::add_cc(a.v[0], b.v[0]);
#pragma unroll
  for (int j = 1; j < N - 1; j++) t[j] = ptx::addc_cc(a.v[j], b.v[j]);
  t[N - 1] = ptx::addc(a.v[N - 1], b.v[N - 1]);  // p < 2^(32N-1): no carry out
  fp_reduce_once<C>(t);
#pragma unroll
  for (int j = 0; j < N; j++) r.v[j] = t[j];
}

template <class C>
B2K_D void fp_sub(Fp<C>& r, const Fp<C>& a, const Fp<C>& b) {
  constexpr int N = C::N;
  uint32_t t[N];
  t[0] = ptx::sub_cc(a.v[0], b.v[0]);
#pragma unroll
  for (int j = 1; j < N; j++) t[j] = ptx::subc_cc(a.v[j], b.v[j]);
  uint32_t borrow = ptx::subc(0, 0);  // all-ones if a < b
  t[0] = ptx::add_cc(t[0], C::mod(0) & borrow);
#pragma unroll
  for (int j = 1; j < N - 1; j++) t[j] = ptx::addc_cc(t[j], C::mod(j) & borrow);
  t[N - 1] = ptx::addc(t[N - 1], C::mod(N - 1) & borrow);
#pragma unroll
  for (int j = 0; j < N; j++) r.v[j] = t[j];
}

template <class C>
B2K_D bool fp_is_zero(const Fp<C>& a) {
  uint32_t o = 0;
#pragma unroll
  for (int j = 0; j < C::N; j++) o |= a.v[j];
  return o == 0;
}

template <class C>
B2K_D bool fp_eq(const Fp<C>& a, const Fp<C>& b) {
  uint32_t o = 0;
#pragma unroll
  for (int j = 0; j < C::N; j++) o |= a.v[j] ^ b.v[j];
  return o == 0;
}

// r = a + b or a - b mod p in ONE instruction stream (callers whose lanes mix additions and subtractions: coop_pairing.cuh):
//   s = a + (b ^ m) + (m & 1), m = 0 / ~0 (a - b as a + ~b + 1; its carry-out is "no borrow");
//   t = s - p for an addition, s + p for a subtraction; r = t where the addition reached p / the subtraction borrowed, else s.
template <class C>
B2K_D void fp_addsub(Fp<C>& r, const Fp<C>& a, const Fp<C>& b, bool minus) {
  constexpr int N = C::N;
  const uint32_t m = minus ? 0xffffffffu : 0u, nm = ~m;
  uint32_t s[N], t[N];
  ptx::add_cc(m, m & 1u);                                    // carry-in = 1 for the two's complement (~0 + 1 carries, 0 + 0 does not)
#pragma unroll
  for (int j = 0; j < N; j++) s[j] = ptx::addc_cc(a.v[j], b.v[j] ^ m);
  const uint32_t carry = ptx::addc(0, 0);                    // subtraction: 1 = no borrow; addition: the sum's bit 32 N
  ptx::add_cc(nm, nm & 1u);
#pragma unroll
  for (int j = 0; j < N; j++) t[j] = ptx::addc_cc(s[j], C::mod(j) ^ nm);
  const uint32_t c2 = ptx::addc(0, 0);                       // addition: 1 = s - p did not borrow
  const bool take = minus ? (carry == 0) : ((carry | c2) != 0);
#pragma unroll
  for (int j = 0; j < N; j++) r.v[j] = take ? t[j] : s[j];
}

template <class C>
B2K_D void fp_neg(Fp<C>& r, const Fp<C>& a) {
  constexpr int N = C::N;
  uint32_t nz = 0;
#pragma unroll
  for (int j = 0; j < N; j++) nz |= a.v[j];
  uint32_t mask = nz ? 0xffffffffu : 0u;  // -0 = 0
  uint32_t t[N];
  t[0] = ptx::sub_cc(C::mod(0) & mask, a.v[0]);
#pragma unroll
  for (int j = 1; j < N - 1; j++) t[j] = ptx::subc_cc(C::mod(j) & mask, a.v[j]);
  t[N - 1] = ptx::subc(C::mod(N - 1) & mask, a.v[N - 1]);
#pragma unroll
  for (int j = 0; j < N; j++) r.v[j] = t[j];
}

template <class C>
B2K_D void fp_dbl(Fp<C>& r, const Fp<C>& a) { fp_add(r, a, a); }

template <class C>
B2K_D void fp_set_zero(Fp<C>& r) {
#pragma unroll
  for (int j = 0; j < C::N; j++) r.v[j] = 0;
}

template <class C>
B2K_D void fp_set_one(Fp<C>& r) {  // Montgomery one = R mod p
#pragma unroll
  for (int j = 0; j < C::N; j++) r.v[j] = C::r1(j);
}

// plain integer -> Montgomery form:  a * R^2 * R^-1
template <class C>
B2K_D void fp_to_mont(Fp<C>& r, const Fp<C>& a) {
  Fp<C> r2;
#pragma unroll
  for (int j = 0; j < C::N; j++) r2.v[j] = C::r2(j);
  fp_mul(r, a, r2);
}

// Montgomery form -> canonical integer in [0,p):  a * 1 * R^-1
template <class C>
B2K_D void fp_from_mont(Fp<C>& r, const Fp<C>& a) {
  Fp<C> one;
#pragma unroll
  for (int j = 0; j < C::N; j++) one.v[j] = (j == 0);
  fp_mul(r, a, one);
}

// a^e for a public exponent given as NE 32-bit little-endian limbs (plain square-and-multiply with a
// 4-bit fixed window; exponents on this path are field constants: p-2, (p+1)/4, (p-1)/2 ...).
template <class C, class E>
B2K_NI void fp_pow_const(Fp<C>& r, const Fp<C>& a) {
  Fp<C> tbl[16];
  fp_set_one(tbl[0]);
  tbl[1] = a;
  for (int i = 2; i < 16; i++) fp_mul_c(tbl[i], tbl[i - 1], a);
  Fp<C> acc;
  fp_set_one(acc);
  bool started = false;
  for (int i = E::NE * 8 - 1; i >= 0; i--) {
    uint32_t nib = (E::limb(i >> 3) >> ((i & 7) * 4)) & 15u;
    if (started) {
      fp_sqr_c(acc, acc); fp_sqr_c(acc, acc); fp_sqr_c(acc, acc); fp_sqr_c(acc, acc);
    }
    if (nib) {
      if (started) fp_mul_c(acc, acc, tbl[nib]);
      else acc = tbl[nib];
      started = true;
    }
  }
  r = acc;
}

// Fermat inverse a^(p-2); inverse of 0 is 0.  Kept as the independent cross-check of fp_inv (tests/host_emul).
template <class C>
B2K_D void fp_inv_fermat(Fp<C>& r, const Fp<C>& a) { fp_pow_const<C, typename C::ExpPm2>(r, a); }

// The inversion every kernel uses: branch-free binary GCD on 64-bit approximations (fp_inv.cuh, included at the end of
// this file) -- about a tenth of the Fermat ladder's multiply-pipe time, most of it on the otherwise idle integer ALU.
// Same contract: Montgomery in, Montgomery out, inverse of 0 is 0.
template <class C> B2K_NI void fp_inv_bingcd(Fp<C>& out, const Fp<C>& x);
template <class C>
B2K_D void fp_inv(Fp<C>& r, const Fp<C>& a) { fp_inv_bingcd(r, a); }

// canonical comparison helper: is (canonical, non-Montgomery) a > (p-1)/2 ?
template <class C>
B2K_D bool fp_canon_gt_half(const Fp<C>& a) {
  // a > h  <=>  h - a borrows
  ptx::sub_cc(C::half(0), a.v[0]);
#pragma unroll
  for (int j = 1; j < C::N; j++) ptx::subc_cc(C::half(j), a.v[j]);
  return ptx::subc(0, 0) != 0;
}

// canonical comparison helper: plain integer a < p ?
template <class C>
B2K_D bool fp_canon_lt_mod(const Fp<C>& a) {
  ptx::sub_cc(a.v[0], C::mod(0));
#pragma unroll
  for (int j = 1; j < C::N; j++) ptx::subc_cc(a.v[j], C::mod(j));
  return ptx::subc(0, 0) != 0;
}

// ---- byte codecs (big-endian wire <-> little-endian limbs) -------------------------------------
template <class C>
B2K_D void fp_load_be(Fp<C>& r, const uint8_t* p) {  // 4*N bytes big-endian
#pragma unroll
  for (int j = 0; j < C::N; j++) {
    const uint8_t* q = p + 4 * (C::N - 1 - j);
    r.v[j] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
  }
}

template <class C>
B2K_D void fp_store_be(uint8_t* p, const Fp<C>& a) {
#pragma unroll
  for (int j = 0; j < C::N; j++) {
    uint8_t* q = p + 4 * (C::N - 1 - j);
    q[0] = (uint8_t)(a.v[j] >> 24); q[1] = (uint8_t)(a.v[j] >> 16);
    q[2] = (uint8_t)(a.v[j] >> 8); q[3] = (uint8_t)a.v[j];
  }
}

}  // namespace b2k

#include "fp_inv.cuh"
