// Host emulation of the Karatsuba products (fp.cuh: the sum of two products; tools/probe/fp_kara.cuh: the single product) and of
// the XYZZ additions that use the sum of two (ec.cuh), next to those formulas written with the CIOS product alone (test
// infrastructure only).
#include "../../kyber_b200/csrc/constants.cuh"
#include "../../kyber_b200/csrc/ec.cuh"
#include "../../tools/probe/fp_kara.cuh"
using namespace b2k;

namespace {
template <class C> Fp<C> load(const uint32_t* a) { Fp<C> x; for (int i = 0; i < C::N; i++) x.v[i] = a[i]; return x; }
template <class C> void store(uint32_t* r, const Fp<C>& x) { for (int i = 0; i < C::N; i++) r[i] = x.v[i]; }

template <class F> Xyzz<F> load_xyzz(const uint32_t* p) {
  constexpr int N = sizeof(F) / 4;
  Xyzz<F> r;
  for (int i = 0; i < N; i++) { r.X.v[i] = p[i]; r.Y.v[i] = p[N + i]; r.ZZ.v[i] = p[2 * N + i]; r.ZZZ.v[i] = p[3 * N + i]; }
  return r;
}
template <class F> void store_xyzz(uint32_t* r, const Xyzz<F>& p) {
  constexpr int N = sizeof(F) / 4;
  for (int i = 0; i < N; i++) { r[i] = p.X.v[i]; r[N + i] = p.Y.v[i]; r[2 * N + i] = p.ZZ.v[i]; r[3 * N + i] = p.ZZZ.v[i]; }
}

// madd-2008-s and add-2008-s with eight and twelve CIOS products, Y3 as two products and a subtraction
template <class F>
void old_madd(Xyzz<F>& r, const Xyzz<F>& p, const Affine<F>& q, bool negate) {
  if (aff_is_inf(q)) { r = p; return; }
  F qy;
  if (negate) f_neg(qy, q.y); else qy = q.y;
  if (xyzz_is_inf(p)) { r.X = q.x; r.Y = qy; f_set_one(r.ZZ); f_set_one(r.ZZZ); return; }
  F U2, S2, P, R, PP, PPP, Q;
  f_mul(U2, q.x, p.ZZ); f_mul(S2, qy, p.ZZZ); f_sub(P, U2, p.X); f_sub(R, S2, p.Y);
  if (f_is_zero(P)) {
    if (f_is_zero(R)) { Xyzz<F> t; t.X = q.x; t.Y = qy; f_set_one(t.ZZ); f_set_one(t.ZZZ); xyzz_dbl(r, t); return; }
    xyzz_set_inf(r); return;
  }
  f_sqr(PP, P); f_mul(PPP, P, PP); f_mul(Q, p.X, PP);
  f_sqr(U2, R); f_sub(U2, U2, PPP); f_sub(U2, U2, Q); f_sub(U2, U2, Q);
  f_sub(Q, Q, U2); f_mul(Q, R, Q); f_mul(S2, p.Y, PPP); f_sub(r.Y, Q, S2);
  r.X = U2; f_mul(r.ZZ, p.ZZ, PP); f_mul(r.ZZZ, p.ZZZ, PPP);
}
template <class F>
void old_add(Xyzz<F>& r, const Xyzz<F>& p, const Xyzz<F>& q) {
  if (xyzz_is_inf(q)) { r = p; return; }
  if (xyzz_is_inf(p)) { r = q; return; }
  F U1, U2, S1, S2, P, R, PP, PPP, Q;
  f_mul(U1, p.X, q.ZZ); f_mul(U2, q.X, p.ZZ); f_mul(S1, p.Y, q.ZZZ); f_mul(S2, q.Y, p.ZZZ);
  f_sub(P, U2, U1); f_sub(R, S2, S1);
  if (f_is_zero(P)) {
    if (f_is_zero(R)) { xyzz_dbl(r, p); return; }
    xyzz_set_inf(r); return;
  }
  f_sqr(PP, P); f_mul(PPP, P, PP); f_mul(Q, U1, PP);
  f_sqr(U2, R); f_sub(U2, U2, PPP); f_sub(U2, U2, Q); f_sub(U2, U2, Q);
  f_sub(Q, Q, U2); f_mul(Q, R, Q); f_mul(S1, S1, PPP);
  f_mul(U1, p.ZZ, q.ZZ); f_mul(S2, p.ZZZ, q.ZZZ);
  f_sub(r.Y, Q, S1); r.X = U2; f_mul(r.ZZ, U1, PP); f_mul(r.ZZZ, S2, PPP);
}
}  // namespace

extern "C" {
#define KARA_FIELD_API(name, C)                                                                    \
  void emul_##name##_wide_mul_kara(const uint32_t* a, const uint32_t* b, uint32_t* t) {           \
    detail::wide_mul_kara<C::N>(t, a, b); }                                                        \
  void emul_##name##_mul_k(const uint32_t* a, const uint32_t* b, uint32_t* r) {                   \
    Fp<C> z; fp_mul_k_inl(z, load<C>(a), load<C>(b)); store(r, z); }                               \
  void emul_##name##_mul_sum2(const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d, uint32_t* r) { \
    Fp<C> z; fp_mul_sum2_inl(z, load<C>(a), load<C>(b), load<C>(c), load<C>(d)); store(r, z); }
#define KARA_SUM2_API(name, C)                                                                     \
  void emul_##name##_wide_mul_kara_sum2(const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d, uint32_t* t) { \
    detail::wide_mul_kara_sum2<C::N>(t, a, b, c, d); }
KARA_FIELD_API(fp381, Bls381Fp)
KARA_FIELD_API(fp254, Bn254Fp)
KARA_FIELD_API(fp256, Bn256Fp)
KARA_SUM2_API(fp381, Bls381Fp)
KARA_SUM2_API(fp254, Bn254Fp)

// BLS12-381 G1, Montgomery limbs: p = X|Y|ZZ|ZZZ (4 x 12 words), q = x|y (2 x 12); old != 0 runs the CIOS-only formulas.
// The formulas run in place (r aliasing p), as the bucket kernels call them.
using F381 = Fp<Bls381Fp>;
void emul_xyzz381_madd(const uint32_t* p, const uint32_t* q, int negate, int old, uint32_t* r) {
  Xyzz<F381> a = load_xyzz<F381>(p);
  Affine<F381> b{load<Bls381Fp>(q), load<Bls381Fp>(q + 12)};
  if (old) old_madd(a, a, b, negate != 0); else xyzz_madd(a, a, b, negate != 0);
  store_xyzz(r, a);
}
void emul_xyzz381_add(const uint32_t* p, const uint32_t* q, int old, uint32_t* r) {
  Xyzz<F381> a = load_xyzz<F381>(p), b = load_xyzz<F381>(q);
  if (old) old_add(a, a, b); else xyzz_add(a, a, b);
  store_xyzz(r, a);
}
}
