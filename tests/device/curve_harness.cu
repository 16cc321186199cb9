// curve_harness.cu -- test-only entry points into the per-thread curve code (ec.cuh, curves.cuh, codec.cuh, msm.cuh, h2c.cuh,
// h2c_g2.cuh, ed25519.cuh), one case per thread on RAW MONTGOMERY LIMBS, so that a test picks
// the coordinates, the projective scale and the exceptional operands itself.  Not a library unit: the library headers are
// included unchanged.  Built three times by __graft_entry__.build() with the library's NVCC_FLAGS, like field_harness.cu:
//   libcurve_harness_compact.so   -DB2K_COMPACT_FIELD=1
//   libcurve_harness_byref.so     -DB2K_COMPACT_FIELD=1 -DB2K_FP2_BYREF (the layout b2k_g2.cu builds the G2 formulas in)
//   libcurve_harness_inlined.so   without B2K_COMPACT_FIELD (the BLS12-381 G1 family only, see the entry points below)
// and by g++ with -DB2K_HOST_EMUL (tests/test_curve_arith_emulation.py); the two bodies that live in kernels.cuh, which only
// nvcc compiles, are device-only (W_JAC_TO_AFFINE_BG, W_XYZZ_TO_AFFINE_VT leave the output zero on the host).
//
// Entry points (all return a cudaError_t, 0 on the host):
//   ch_w_<group>(op, alias, n, in, out)   a short-Weierstrass group with E words per coordinate (N for G1, 2 N for G2, c0 first)
//       in:  n x (A[4 E], B[4 E], k[8], w)     A, B: (X, Y, Z | ZZ, ZZZ) or (x, y); k: a 256-bit scalar, little-endian words;
//                                               w: a small argument (negate, check_subgroup)
//       out: n x (R[4 E], flag)
//   ch_xmd(op, alias, n, in, out)         in: n x (msg_len, dst_len, msg[64], dst[64]) (bytes little-endian in the words);
//                                         out: n x 64 words (128 or 256 bytes)
//   ch_ed(op, alias, n, in, out)          in: n x (P[32], Q[32], bytes[8], k[8], w); out: n x (R[32], bytes[8], flag)
// alias selects how the result and the operands share storage: 0 none, 1 r = p, 2 r = q, 3 r = p = q.
#include "../../kyber_b200/csrc/constants.cuh"
#include "../../kyber_b200/csrc/h2c_g2.cuh"
#include "../../kyber_b200/csrc/bn256.cuh"
#include "../../kyber_b200/csrc/bn_pairing.cuh"
#include "../../kyber_b200/csrc/msm.cuh"
#include "../../kyber_b200/csrc/msm_affine.cuh"
#include "../../kyber_b200/csrc/ed25519.cuh"
#include <stddef.h>
#include <utility>
#ifdef __CUDACC__
#include "../../kyber_b200/csrc/kernels.cuh"
#include <cuda_runtime.h>
#endif

using namespace b2k;

namespace {

enum WOp {
  W_JAC_DBL, W_JAC_ADD, W_JAC_MADD, W_JAC_NEG, W_JAC_TO_AFFINE, W_JAC_TO_AFFINE_BG,
  W_XYZZ_DBL, W_XYZZ_ADD, W_XYZZ_ADD_REDUCE, W_XYZZ_MADD, W_XYZZ_TO_AFFINE, W_XYZZ_TO_AFFINE_VT, W_XYZZ_MUL_SMALL,
  W_AFF_ON_CURVE, W_JAC_EQ_AFFINE, W_SCALAR_MUL, W_SCALAR_MUL_W4,
  // BLS12-381 only (G1: the first group, G2: the second)
  W_JAC_MUL_XABS, W_JAC_MUL_XABS_JAC, W_IN_SUBGROUP, W_DECOMPRESS, W_MAP_SSWU, W_ISO_MAP, W_SGN0,
  W_GLV_SPLIT, W_SCALAR_MUL_GLV, W_FP_FROM_64_BYTES,          // G1
  W_JAC_PSI, W_CLEAR_COFACTOR                                 // G2
};
enum EdOp {
  ED_ADD, ED_DBL, ED_DBL_XYZ, ED_ADD_CACHED, ED_MADD, ED_DECODE, ED_DECODE_AFF, ED_ENCODE, ED_ENCODE_Z1, ED_BYTES_CANONICAL,
  ED_HAS_SMALL_ORDER, ED_EQ, ED_SCALAR_MUL, ED_MUL_VAR
};

// the batched inversion of the scalar-multiplication tables (the library's kernels pass the binary-GCD one, kernels.cuh)
struct InvBg { template <class F> B2K_D void operator()(F& r, const F& a) const { f_inv_bg(r, a); } };

template <class C> B2K_D void ld(Fp<C>& r, const uint32_t* p) {
  for (int j = 0; j < C::N; j++) r.v[j] = p[j];
}
template <class C> B2K_D void ld(Fp2<C>& r, const uint32_t* p) { ld(r.c0, p); ld(r.c1, p + C::N); }
template <class C> B2K_D void st(uint32_t* p, const Fp<C>& a) {
  for (int j = 0; j < C::N; j++) p[j] = a.v[j];
}
template <class C> B2K_D void st(uint32_t* p, const Fp2<C>& a) { st(p, a.c0); st(p + C::N, a.c1); }
B2K_D void ld_bytes(uint8_t* b, const uint32_t* w, int len) {
  for (int i = 0; i < len; i++) b[i] = (uint8_t)(w[i >> 2] >> (8 * (i & 3)));
}
B2K_D void st_bytes(uint32_t* w, const uint8_t* b, int len) {
  for (int i = 0; i < len; i += 4) w[i >> 2] = b[i] | ((uint32_t)b[i + 1] << 8) | ((uint32_t)b[i + 2] << 16) | ((uint32_t)b[i + 3] << 24);
}

// the groups: curve configuration, coordinate field, words per coordinate, and which BLS12-381 group it is (0: none, 1: G1, 2: G2)
template <class F> struct Words;
template <class C> struct Words<Fp<C>> { static constexpr int n = C::N; };
template <class C> struct Words<Fp2<C>> { static constexpr int n = 2 * C::N; };
template <class CV_, int BLS_> struct Grp {
  using CV = CV_;
  using F = typename CV::F;
  static constexpr int E = Words<F>::n;       // not sizeof(F) / 4: Fp is 16-byte aligned
  static constexpr int BLS = BLS_;
};

template <class F> B2K_D Jac<F> jac_of(const F* a) { Jac<F> p; p.X = a[0]; p.Y = a[1]; p.Z = a[2]; return p; }
template <class F> B2K_D Xyzz<F> xyzz_of(const F* a) { Xyzz<F> p; p.X = a[0]; p.Y = a[1]; p.ZZ = a[2]; p.ZZZ = a[3]; return p; }
template <class F> B2K_D Affine<F> aff_of(const F* a) { Affine<F> p; p.x = a[0]; p.y = a[1]; return p; }
template <class F> B2K_D void put(F* r, const Jac<F>& p) { r[0] = p.X; r[1] = p.Y; r[2] = p.Z; }
template <class F> B2K_D void put(F* r, const Xyzz<F>& p) { r[0] = p.X; r[1] = p.Y; r[2] = p.ZZ; r[3] = p.ZZZ; }
template <class F> B2K_D void put(F* r, const Affine<F>& p) { r[0] = p.x; r[1] = p.y; }

// r = op(p, q) with the aliasing of the case: 0 op(r, p, q), 1 op(p, p, q), 2 op(q, p, q), 3 op(p, p, p)
#define CH_BINARY(T, fn, A, B)            \
  {                                       \
    T p = A, q = B, r;                    \
    switch (alias) {                      \
      case 1: fn(p, p, q); r = p; break;  \
      case 2: fn(q, p, q); r = q; break;  \
      case 3: fn(p, p, p); r = p; break;  \
      default: fn(r, p, q);               \
    }                                     \
    put(R, r);                            \
  }
#define CH_UNARY(T, fn, A)                \
  {                                       \
    T p = A, r;                           \
    if (alias == 1) { fn(p, p); r = p; }  \
    else fn(r, p);                        \
    put(R, r);                            \
  }

template <class G, int op>
B2K_D void w_case(int alias, const uint32_t* in, uint32_t* out) {
  using F = typename G::F;
  using CV = typename G::CV;
  constexpr int E = G::E;
  F a[4], b[4], R[4];
  for (int i = 0; i < 4; i++) { ld(a[i], in + i * E); ld(b[i], in + (4 + i) * E); f_set_zero(R[i]); }
  Scalar256 k;
  for (int j = 0; j < 8; j++) k.v[j] = in[8 * E + j];
  const uint32_t w = in[8 * E + 8];
  uint32_t flag = 0;
  switch (op) {
    case W_JAC_DBL: CH_UNARY(Jac<F>, jac_dbl, jac_of(a)) break;
    case W_JAC_ADD: CH_BINARY(Jac<F>, jac_add, jac_of(a), jac_of(b)) break;
    case W_JAC_MADD: {
      Jac<F> p = jac_of(a), r;
      const Affine<F> q = aff_of(b);
      if (alias == 1) { jac_madd(p, p, q); r = p; } else jac_madd(r, p, q);
      put(R, r);
      break;
    }
    case W_JAC_NEG: CH_UNARY(Jac<F>, jac_neg, jac_of(a)) break;
    case W_JAC_TO_AFFINE: { Affine<F> r; jac_to_affine(r, jac_of(a)); put(R, r); break; }
    case W_XYZZ_DBL: CH_UNARY(Xyzz<F>, xyzz_dbl, xyzz_of(a)) break;
    case W_XYZZ_ADD: CH_BINARY(Xyzz<F>, xyzz_add, xyzz_of(a), xyzz_of(b)) break;
    case W_XYZZ_ADD_REDUCE: CH_BINARY(Xyzz<F>, xyzz_add_reduce, xyzz_of(a), xyzz_of(b)) break;
    case W_XYZZ_MADD: {
      Xyzz<F> p = xyzz_of(a), r;
      const Affine<F> q = aff_of(b);
      if (alias == 1) { xyzz_madd(p, p, q, w != 0); r = p; } else xyzz_madd(r, p, q, w != 0);
      put(R, r);
      break;
    }
    case W_XYZZ_TO_AFFINE: { Affine<F> r; xyzz_to_affine(r, xyzz_of(a)); put(R, r); break; }
#ifdef __CUDACC__
    case W_JAC_TO_AFFINE_BG: { Affine<F> r; jac_to_affine_bg(r, jac_of(a)); put(R, r); break; }
    case W_XYZZ_TO_AFFINE_VT: { Affine<F> r; xyzz_to_affine_vt(r, xyzz_of(a)); put(R, r); break; }
#endif
    case W_XYZZ_MUL_SMALL: {
      Xyzz<F> p = xyzz_of(a), r;
      if (alias == 1) { xyzz_mul_small(p, p, k.v[0]); r = p; } else xyzz_mul_small(r, p, k.v[0]);
      put(R, r);
      break;
    }
    case W_AFF_ON_CURVE: flag = aff_on_curve<CV>(aff_of(a)); break;
    case W_JAC_EQ_AFFINE: flag = jac_eq_affine(jac_of(a), aff_of(b)); break;
    case W_SCALAR_MUL: { Jac<F> r; scalar_mul<CV>(r, k, aff_of(a)); put(R, r); break; }
    case W_SCALAR_MUL_W4: { Jac<F> r; scalar_mul_w4<CV>(r, k, aff_of(a), InvBg{}); put(R, r); break; }
    default: break;
  }
  if constexpr (G::BLS != 0) {
    switch (op) {
      case W_JAC_MUL_XABS: { Jac<F> r; jac_mul_xabs(r, aff_of(a)); put(R, r); break; }
      case W_JAC_MUL_XABS_JAC: CH_UNARY(Jac<F>, jac_mul_xabs_jac, jac_of(a)) break;
      default: break;
    }
  }
  if constexpr (G::BLS == 1) {
    switch (op) {
      case W_IN_SUBGROUP: flag = g1_in_subgroup(aff_of(a)); break;
      case W_DECOMPRESS: {
        uint8_t buf[48];
        ld_bytes(buf, in, 48);
        Affine<F> r;
        aff_set_inf(r);
        flag = g1_decompress(r, buf, w != 0);
        put(R, r);
        break;
      }
      case W_MAP_SSWU: { Affine<F> r; map_to_curve_sswu(r.x, r.y, a[0]); put(R, r); break; }
      case W_ISO_MAP: { Jac<F> r; iso_map_g1(r, a[0], a[1]); put(R, r); break; }
      case W_SGN0: flag = fp_sgn0(a[0]); break;
      case W_GLV_SPLIT: {
        GlvSplit sp;
        glv_split_bls381(sp, k);
        uint32_t* o = out;
        for (int j = 0; j < 8; j++) { o[j] = sp.k1.v[j]; o[8 + j] = sp.k2.v[j]; }
        o[16] = sp.neg1; o[17] = sp.neg2;
        for (int j = 18; j <= 4 * E; j++) o[j] = 0;
        return;
      }
      case W_SCALAR_MUL_GLV: { Jac<F> r; scalar_mul_glv_bls381(r, k, aff_of(a), InvBg{}); put(R, r); break; }
      case W_FP_FROM_64_BYTES: {
        uint8_t buf[64];
        ld_bytes(buf, in, 64);
        fp_from_64_bytes(R[0], buf);
        break;
      }
      default: break;
    }
  }
  if constexpr (G::BLS == 2) {
    switch (op) {
      case W_IN_SUBGROUP: flag = g2_in_subgroup(aff_of(a)); break;
      case W_DECOMPRESS: {
        uint8_t buf[96];
        ld_bytes(buf, in, 96);
        Affine<F> r;
        aff_set_inf(r);
        flag = g2_decompress(r, buf, w != 0);
        put(R, r);
        break;
      }
      case W_MAP_SSWU: { Affine<F> r; map_to_curve_sswu_g2(r.x, r.y, a[0]); put(R, r); break; }
      case W_ISO_MAP: { Jac<F> r; iso_map_g2(r, a[0], a[1]); put(R, r); break; }
      case W_SGN0: flag = fp2_sgn0(a[0]); break;
      case W_JAC_PSI: CH_UNARY(Jac<F>, jac_psi, jac_of(a)) break;
      case W_CLEAR_COFACTOR: CH_UNARY(Jac<F>, g2_clear_cofactor, jac_of(a)) break;
      default: break;
    }
  }
  for (int i = 0; i < 4; i++) st(out + i * E, R[i]);
  out[4 * E] = flag;
}

// ---- expand_message_xmd ----------------------------------------------------------------------------------------------------
constexpr int XMD_IN = 2 + 64 + 64, XMD_OUT = 64;
template <int op>
B2K_D void xmd_case(int, const uint32_t* in, uint32_t* out) {
  uint8_t msg[256], dst[256], o[256];
  const uint32_t ml = in[0] < 256 ? in[0] : 256, dl = in[1] < 256 ? in[1] : 255;
  ld_bytes(msg, in + 2, 256);
  ld_bytes(dst, in + 66, 256);
  for (int i = 0; i < 256; i++) o[i] = 0;
  if constexpr (op == 0) expand_message_xmd_128(o, msg, ml, dst, dl);
  else expand_message_xmd_256(o, msg, ml, dst, dl);
  st_bytes(out, o, 256);
}

// ---- edwards25519 ------------------------------------------------------------------------------------------------------------
constexpr int ED_IN = 32 + 32 + 8 + 8 + 1, ED_OUT = 32 + 8 + 1;
B2K_D EdExt ed_of(const uint32_t* p) { EdExt e; ld(e.X, p); ld(e.Y, p + 8); ld(e.Z, p + 16); ld(e.T, p + 24); return e; }
B2K_D void ed_put(uint32_t* p, const EdExt& e) { st(p, e.X); st(p + 8, e.Y); st(p + 16, e.Z); st(p + 24, e.T); }
B2K_D void ed_cached_add(EdExt& r, const EdExt& p, const EdCached& c, uint32_t w) {
  ed_add_cached(r, p, c.ypx, c.ymx, (w & 1) ? &c.z2 : nullptr, c.t2d, (w & 2) != 0);
}

template <int op>
B2K_D void ed_case(int alias, const uint32_t* in, uint32_t* out) {
  const EdExt a = ed_of(in), b = ed_of(in + 32);
  uint8_t bytes[32], ob[32];
  ld_bytes(bytes, in + 64, 32);
  const uint32_t* k = in + 72;
  const uint32_t w = in[80];
  EdExt R;
  fp_set_zero(R.X); fp_set_zero(R.Y); fp_set_zero(R.Z); fp_set_zero(R.T);
  for (int i = 0; i < 32; i++) ob[i] = 0;
  uint32_t flag = 0;
  switch (op) {
    case ED_ADD: {
      EdExt p = a, q = b;
      switch (alias) {
        case 1: ed_add(p, p, q); R = p; break;
        case 2: ed_add(q, p, q); R = q; break;
        case 3: ed_add(p, p, p); R = p; break;
        default: ed_add(R, p, q);
      }
      break;
    }
    case ED_DBL: { EdExt p = a; if (alias == 1) { ed_dbl(p, p); R = p; } else ed_dbl(R, p); break; }
    case ED_DBL_XYZ: { EdExt p = a; if (alias == 1) { ed_dbl_xyz(p, p); R = p; } else ed_dbl_xyz(R, p); break; }
    case ED_ADD_CACHED: {                      // w bit 0: pass 2 Z (else Z = 1 is assumed), bit 1: subtract
      EdCached c;
      ed_to_cached(c, b);
      EdExt p = a;
      if (alias == 1) { ed_cached_add(p, p, c, w); R = p; } else ed_cached_add(R, p, c, w);
      break;
    }
    case ED_MADD: {                            // q with Z = 1 as a Niels point, added in place (w: subtract)
      EdCached c;
      ed_to_cached(c, b);
      EdNiels nq;
      nq.ypx = c.ypx; nq.ymx = c.ymx; nq.t2d = c.t2d;
      R = a;
      ed_madd(R, nq, w != 0);
      break;
    }
    case ED_DECODE: flag = ed_decode(R, bytes); break;
    case ED_DECODE_AFF: {
      EdAff e;
      flag = ed_decode_aff(e, bytes);
      R.X = e.x; R.Y = e.y;
      break;
    }
    case ED_ENCODE: ed_encode(ob, a); break;
    case ED_ENCODE_Z1: ed_encode_z1(ob, a); break;
    case ED_BYTES_CANONICAL: flag = ed_bytes_canonical(bytes); break;
    case ED_HAS_SMALL_ORDER: flag = ed_has_small_order(a); break;
    case ED_EQ: flag = ed_eq(a, b); break;
    case ED_SCALAR_MUL: {
      uint8_t kb[32];
      ld_bytes(kb, k, 32);
      ed_scalar_mul(R, kb, a);
      break;
    }
    case ED_MUL_VAR: ed_mul_var(R, k, a); break;
    default: break;
  }
  ed_put(out, R);
  st_bytes(out + 32, ob, 32);
  out[40] = flag;
}

using GBls1 = Grp<Bls381G1, 1>;
using GBls2 = Grp<Bls381G2, 2>;
using GBn254_1 = Grp<Bn254G1, 0>;
using GBn254_2 = Grp<Bn254G2, 0>;
using GBn256_1 = Grp<Bn256G1, 0>;
using GBn256_2 = Grp<Bn256G2, 0>;

// one kernel per (family, operation): the operation is a template argument, so that every kernel holds only its own body (one
// kernel with every body of a group behind a switch costs the optimiser and the register allocator minutes per layout)
template <class G> struct WCase {
  static constexpr int IN = 8 * G::E + 9, OUT = 4 * G::E + 1, NOPS = W_CLEAR_COFACTOR + 1;
  template <int op> B2K_D static void run(int alias, const uint32_t* in, uint32_t* out) { w_case<G, op>(alias, in, out); }
};
struct XmdCase {
  static constexpr int IN = XMD_IN, OUT = XMD_OUT, NOPS = 2;
  template <int op> B2K_D static void run(int alias, const uint32_t* in, uint32_t* out) { xmd_case<op>(alias, in, out); }
};
struct EdCase {
  static constexpr int IN = ED_IN, OUT = ED_OUT, NOPS = ED_MUL_VAR + 1;
  template <int op> B2K_D static void run(int alias, const uint32_t* in, uint32_t* out) { ed_case<op>(alias, in, out); }
};

#ifdef __CUDACC__
template <class K, int op>
__global__ void k_case(int alias, int n, const uint32_t* in, uint32_t* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  K::template run<op>(alias, in + (size_t)i * K::IN, out + (size_t)i * K::OUT);
}

// H2D, one launch, D2H; every step's status is returned (the first failure wins)
template <class K, int op>
int run_op(int alias, int n, const uint32_t* in, uint32_t* out) {
  if (n <= 0) return 0;
  uint32_t *d_in = nullptr, *d_out = nullptr;
  cudaError_t e = cudaMalloc(&d_in, (size_t)K::IN * n * 4);
  if (e == cudaSuccess) e = cudaMalloc(&d_out, (size_t)K::OUT * n * 4);
  if (e == cudaSuccess) e = cudaMemcpy(d_in, in, (size_t)K::IN * n * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    k_case<K, op><<<(n + 63) / 64, 64>>>(alias, n, d_in, d_out);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpy(out, d_out, (size_t)K::OUT * n * 4, cudaMemcpyDeviceToHost);
  cudaFree(d_in);
  cudaFree(d_out);
  return (int)e;
}
#else
template <class K, int op>
int run_op(int alias, int n, const uint32_t* in, uint32_t* out) {
  for (int i = 0; i < n; i++) K::template run<op>(alias, in + (size_t)i * K::IN, out + (size_t)i * K::OUT);
  return 0;
}
#endif

// the run-time operation code -> its instantiation; an unknown code is an error (cudaErrorInvalidValue = 1)
template <class K, int... OPS>
int dispatch(int op, int alias, int n, const uint32_t* in, uint32_t* out, std::integer_sequence<int, OPS...>) {
  using Fn = int (*)(int, int, const uint32_t*, uint32_t*);
  static constexpr Fn table[] = {run_op<K, OPS>...};
  if (op < 0 || op >= (int)sizeof...(OPS)) return 1;
  return table[op](alias, n, in, out);
}
template <class K> int run(int op, int alias, int n, const uint32_t* in, uint32_t* out) {
  return dispatch<K>(op, alias, n, in, out, std::make_integer_sequence<int, K::NOPS>{});
}

}  // namespace

// The inlined layout exports the BLS12-381 G1 family only.  That is the group whose curve arithmetic the library compiles in that
// layout (b2k_msm_inlined.cu: the G1 MSM and Point.Mul batch; b2k_pairing_inlined.cu adds only the operand check aff_on_curve of
// G1 and G2); with every family, nvcc spent more than five minutes on the inlined layout, against under four on the others.
extern "C" {
#define CH_W(name, G) \
  int ch_w_##name(int op, int alias, int n, const uint32_t* in, uint32_t* out) { return run<WCase<G>>(op, alias, n, in, out); }
CH_W(bls381_g1, GBls1)
#if defined(B2K_COMPACT_FIELD) || !defined(__CUDACC__)
CH_W(bls381_g2, GBls2)
CH_W(bn254_g1, GBn254_1)
CH_W(bn254_g2, GBn254_2)
CH_W(bn256_g1, GBn256_1)
CH_W(bn256_g2, GBn256_2)
int ch_xmd(int op, int alias, int n, const uint32_t* in, uint32_t* out) { return run<XmdCase>(op, alias, n, in, out); }
int ch_ed(int op, int alias, int n, const uint32_t* in, uint32_t* out) { return run<EdCase>(op, alias, n, in, out); }
#endif
}
