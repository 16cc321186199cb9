// b2k_gt.cu -- the target group as a kyber.Group, the Miller / Finalize split and n-pair product checks (batched).
//
// Replaces (reference call sites):
//   GT as an additively written group: Add = Fp12 product, Neg = inverse, Mul = exponentiation, Null = 1
//       pairing/bls12381/kilic/gt.go:33-83 (third-party arithmetic behind it), pairing/bn254/point.go:560-623
//   pointGT.Miller / pointGT.Finalize          pairing/bn254/point.go:768-786  (exported so that callers can multiply several
//       Miller outputs and pay ONE final exponentiation), bn256 twins pairing/bn256/point.go
//   product-of-pairings checks  prod_i e(P_i, Q_i) == 1   (SURVEY.md 8e: "multiply Miller outputs, one final exponentiation");
//       the 2-pair special case is Suite.ValidatePairing (kilic/suite.go:57-68, pairing/bn254/suite.go:138-144)
//   G1 / G2 Point.Add, Sub, Neg as batches     kilic/g1.go:92-108, g2.go:91-107 (single operations in the reference)
// One thread per element / per pair; the product check runs the Miller kernel, multiplies the values of a block in shared
// memory (one Fp12 per block), a last block multiplies those, and ONE final exponentiation follows.
#include <cuda_runtime.h>
#include <string>
#include "../../include/b2kyber.h"
#include "msm_host.cuh"
#include "pairing.cuh"
#include "codec.cuh"
#include "bn256.cuh"
#include "bn_pairing.cuh"
#define B2K_COOP_GT 1
#include "coop_pairing.cuh"          // small batches of GT.Mul: one warp per element

using namespace b2k;
using namespace b2k_host;

namespace b2k {

// ---- per-curve pairing configurations ------------------------------------------------------------------------------------
B2K_D void gt_load(BFp12& f, const uint8_t* in) {               // inverse of gt_store (pairing.cuh): 576 B, highest coefficient first
  BFp2* order[6] = {&f.c1.c2, &f.c1.c1, &f.c1.c0, &f.c0.c2, &f.c0.c1, &f.c0.c0};
  for (int i = 0; i < 6; i++) {
    BFp t;
    fp_load_be(t, in + 96 * i); fp_to_mont(order[i]->c1, t);
    fp_load_be(t, in + 96 * i + 48); fp_to_mont(order[i]->c0, t);
  }
}
B2K_D bool gt_wire_canonical(const uint8_t* in) { return wire_coords_canonical<Bls381Fp, 12>(in); }

template <class PC>
B2K_D void bn_gt_load(PFp12<PC>& f, const uint8_t* in) {        // inverse of bn_gt_store: 384 B
  PFp2<PC>* order[6] = {&f.c1.c2, &f.c1.c1, &f.c1.c0, &f.c0.c2, &f.c0.c1, &f.c0.c0};
  for (int i = 0; i < 6; i++) { PC::load32(order[i]->c1, in + 64 * i); PC::load32(order[i]->c0, in + 64 * i + 32); }
}

struct BlsPairing {
  using F12 = BFp12;
  using FC = Bls381Fp;
  using CoopSqr = coop::BLS_SQR;
  using CoopMul = coop::BLS_MUL;
  using G1 = Bls381G1;
  using G2 = Bls381G2;
  using Fr = Bls381Fr;
  static constexpr int GT_BYTES = 576;
  B2K_D static void load(F12& f, const uint8_t* p) { gt_load(f, p); }
  B2K_D static void store(uint8_t* p, const F12& f) { gt_store(p, f); }
  B2K_D static bool canonical(const uint8_t* p) { return gt_wire_canonical(p); }
  B2K_D static void miller(F12& f, const Affine<G1::F>& P, const Affine<G2::F>& Q) { miller_loop<1>(f, &P, &Q); }
  B2K_D static void final_exp(F12& r, const F12& f) { final_exponentiation(r, f); }
};
template <class PC, class G1T, class G2T, class FrT, bool RANGE>
struct BnPairing {
  using F12 = PFp12<PC>;
  using FC = typename PC::FC;
  using CoopSqr = coop::BN254_SQR;                            // (only bn254 has GT.Mul in the ABI; bn256 never instantiates the exponentiation)
  using CoopMul = coop::BN254_MUL;
  using G1 = G1T;
  using G2 = G2T;
  using Fr = FrT;
  static constexpr int GT_BYTES = 384;
  B2K_D static void load(F12& f, const uint8_t* p) { bn_gt_load<PC>(f, p); }
  B2K_D static void store(uint8_t* p, const F12& f) { bn_gt_store<PC>(p, f); }
  B2K_D static bool canonical(const uint8_t* p) { return !RANGE || wire_coords_canonical<typename PC::FC, 12>(p); }
  B2K_D static void miller(F12& f, const Affine<typename G1::F>& P, const Affine<typename G2::F>& Q) {
    if (aff_is_inf(P) || aff_is_inf(Q)) { fp12_set_one(f); return; }     // optate.go:267-269
    bn_miller_loop<PC, 1>(f, &P, &Q);
  }
  B2K_D static void final_exp(F12& r, const F12& f) { bn_final_exponentiation<PC>(r, f); }
};
using Bn254Pairing = BnPairing<Bn254Pair, Bn254G1, Bn254G2, Bn254Fr, true>;
using Bn256Pairing = BnPairing<Bn256Pair, Bn256G1, Bn256G2, Bn256Fr, false>;

// ---- GT group operations -------------------------------------------------------------------------------------------------
template <class P>
__global__ void __launch_bounds__(64, 4) k_gt_mul(size_t n, const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, uint8_t* __restrict__ out,
                                                  uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (!P::canonical(a + (size_t)P::GT_BYTES * i) || !P::canonical(b + (size_t)P::GT_BYTES * i)) atomicOr(flags, FLAG_POINT);
  typename P::F12 x, y;
  P::load(x, a + (size_t)P::GT_BYTES * i);
  P::load(y, b + (size_t)P::GT_BYTES * i);
  fp12_mul(x, x, y);
  P::store(out + (size_t)P::GT_BYTES * i, x);
}
template <class P>
__global__ void __launch_bounds__(64, 4) k_gt_inv(size_t n, const uint8_t* __restrict__ a, uint8_t* __restrict__ out, uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (!P::canonical(a + (size_t)P::GT_BYTES * i)) atomicOr(flags, FLAG_POINT);
  typename P::F12 x, y;
  P::load(x, a + (size_t)P::GT_BYTES * i);
  fp12_inv(y, x);
  P::store(out + (size_t)P::GT_BYTES * i, y);
}
// out = a^s: plain square-and-multiply over the 256-bit scalar (valid for ANY Fp12 element, like the generic Exp of the back-ends)
template <class P>
__global__ void __launch_bounds__(64, 4) k_gt_exp(size_t n, const uint8_t* __restrict__ scalars, const uint8_t* __restrict__ a,
                                                  uint8_t* __restrict__ out, uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Scalar256 k;
  scalar_load_be(k, scalars + 32 * i);
  if (!scalar_in_range<typename P::Fr>(k)) atomicOr(flags, FLAG_SCALAR_RANGE);
  if (!P::canonical(a + (size_t)P::GT_BYTES * i)) atomicOr(flags, FLAG_POINT);
  typename P::F12 x, acc;
  P::load(x, a + (size_t)P::GT_BYTES * i);
  fp12_set_one(acc);
  bool started = false;
  for (int b = 255; b >= 0; b--) {
    if (started) fp12_sqr(acc, acc);
    if ((k.v[b >> 5] >> (b & 31)) & 1u) {
      if (started) fp12_mul(acc, acc, x);
      else { acc = x; started = true; }
    }
  }
  P::store(out + (size_t)P::GT_BYTES * i, acc);
}

// The same exponentiation for SMALL batches, one WARP per element (coop_pairing.cuh): GT.Mul is called one element at a time by the
// reference's IBE (encrypt/ibe: Gid^r), and one thread needs ~15 ms for its 255 Fp12 squarings and ~128 products.  The two steps are
// programs of the cooperative interpreter (19 and 15 rounds on BLS12-381: the 36 / 54 Fp products of a step run in two rounds); the
// accumulator lives in the programs' first 12 input slots, the base beside the slot array.
template <class P, class C, class SQR, class MUL>
__global__ void __launch_bounds__(32, 16) k_coop_gt_exp(size_t n, const uint8_t* __restrict__ scalars, const uint8_t* __restrict__ a,
                                                        uint8_t* __restrict__ out, uint32_t* flags) {
  constexpr int NS = (SQR::SLOTS > MUL::SLOTS ? SQR::SLOTS : MUL::SLOTS) | 1;
  constexpr int N = C::N;
  extern __shared__ __align__(16) uint32_t gt_sm[];
  uint32_t* S = gt_sm;                                       // slots, limb-major
  uint32_t* base = gt_sm + (size_t)N * NS;                   // the element a: 12 coefficients, limb-major with stride 12
  const int lane = threadIdx.x;
  const size_t i = blockIdx.x;
  if (i >= n) return;
  Scalar256 k;
  scalar_load_be(k, scalars + 32 * i);                       // every lane: the loop below is warp-uniform
  if (lane == 0) {
    if (!scalar_in_range<typename P::Fr>(k)) atomicOr(flags, FLAG_SCALAR_RANGE);
    if (!P::canonical(a + (size_t)P::GT_BYTES * i)) atomicOr(flags, FLAG_POINT);
    typename P::F12 x;
    P::load(x, a + (size_t)P::GT_BYTES * i);
    const Fp<C>* c = reinterpret_cast<const Fp<C>*>(&x);
    for (int q = 0; q < 12; q++)
      for (int j = 0; j < N; j++) base[j * 12 + q] = c[q].v[j];
  }
  __syncwarp();
  auto put = [&](int slot0, const uint32_t* src, int stride, const uint16_t* idx) {   // 12 values into slots slot0 .. slot0 + 11
    uint32_t v[N];
    if (lane < 12) {
#pragma unroll
      for (int j = 0; j < N; j++) v[j] = idx ? src[j * stride + idx[lane]] : src[j * stride + lane];
    }
    __syncwarp();
    if (lane < 12) {
#pragma unroll
      for (int j = 0; j < N; j++) S[j * NS + slot0 + lane] = v[j];
    }
    __syncwarp();
  };
  auto consts = [&](int one, int zero) {
    if (lane < N) { S[lane * NS + one] = C::r1(lane); S[lane * NS + zero] = 0u; }
    __syncwarp();
  };
  bool started = false;
  for (int b = 255; b >= 0; b--) {
    if (started) {
      consts(SQR::ONE, SQR::ZERO);
      coop::run<SQR, NS, C>(S, lane);
      put(0, S, NS, SQR::out());                             // acc = acc^2
    }
    if ((k.v[b >> 5] >> (b & 31)) & 1u) {
      if (started) {
        put(12, base, 12, nullptr);                          // second operand = a
        consts(MUL::ONE, MUL::ZERO);
        coop::run<MUL, NS, C>(S, lane);
        put(0, S, NS, MUL::out());                           // acc = acc * a
      } else {
        put(0, base, 12, nullptr);                           // acc = a
        started = true;
      }
    }
  }
  if (lane == 0) {
    typename P::F12 r;
    if (started) {
      Fp<C>* c = reinterpret_cast<Fp<C>*>(&r);
      for (int q = 0; q < 12; q++)
        for (int j = 0; j < N; j++) c[q].v[j] = S[j * NS + q];
    } else fp12_set_one(r);                                  // a^0
    P::store(out + (size_t)P::GT_BYTES * i, r);
  }
}

// ---- Miller / Finalize -----------------------------------------------------------------------------------------------------
template <class P>
__global__ void __launch_bounds__(64, 4) k_miller(size_t n, const uint8_t* __restrict__ g1, const uint8_t* __restrict__ g2, uint8_t* __restrict__ out,
                                                  uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<typename P::G1::F> A;
  Affine<typename P::G2::F> B;
  bool good = load_checked<typename P::G1>(A, g1 + (size_t)P::G1::IN_BYTES * i);
  good = load_checked<typename P::G2>(B, g2 + (size_t)P::G2::IN_BYTES * i) && good;
  if (!good) atomicOr(flags, FLAG_POINT);
  typename P::F12 f;
  P::miller(f, A, B);
  P::store(out + (size_t)P::GT_BYTES * i, f);
}
template <class P>
__global__ void __launch_bounds__(64, 4) k_final_exp(size_t n, const uint8_t* __restrict__ in, uint8_t* __restrict__ out, uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (!P::canonical(in + (size_t)P::GT_BYTES * i)) atomicOr(flags, FLAG_POINT);
  typename P::F12 f, e;
  P::load(f, in + (size_t)P::GT_BYTES * i);
  P::final_exp(e, f);
  P::store(out + (size_t)P::GT_BYTES * i, e);
}

// ---- prod_i e(P_i, Q_i) == 1 with ONE final exponentiation -------------------------------------------------------------------
constexpr int PROD_BLOCK = 32;
template <class F12>
B2K_D void block_product(F12* sm, F12& v) {                       // v of thread 0 = product over the block
  const int tid = threadIdx.x;
  sm[tid] = v;
  __syncthreads();
  for (int h = PROD_BLOCK / 2; h > 0; h >>= 1) {
    if (tid < h) {
      F12 a = sm[tid], b = sm[tid + h];
      fp12_mul(a, a, b);
      sm[tid] = a;
    }
    __syncthreads();
  }
  v = sm[0];
}
// partial[block] = product of the block's share of n Miller values (wire form, as k_miller wrote them).  The Miller loops run in
// k_miller, the kernel Miller()/Pair() use: a variant that ran the loop inside this kernel (under `if (i < n)`, then the block
// product) returned wrong products for bn254 only on the device -- bn256, BLS12-381 and the host emulation were right, and so was every
// piece in isolation (tools/debug/tree_debug.cu, tools/debug_bn_product.py); unexplained, so the composition that is tested
// piece by piece is the one that ships.  Cost: 384 / 576 bytes written and read per pair, nothing next to a Miller loop.
template <class P>
__global__ void __launch_bounds__(PROD_BLOCK) k_gt_block_product(size_t n, const uint8_t* __restrict__ millers, typename P::F12* __restrict__ partial) {
  extern __shared__ __align__(16) unsigned char smraw[];
  auto* sm = reinterpret_cast<typename P::F12*>(smraw);
  typename P::F12 f;
  fp12_set_one(f);
  for (size_t i = (size_t)blockIdx.x * PROD_BLOCK + threadIdx.x; i < n; i += (size_t)gridDim.x * PROD_BLOCK) {
    typename P::F12 m;
    P::load(m, millers + (size_t)P::GT_BYTES * i);
    fp12_mul(f, f, m);
  }
  block_product(sm, f);
  if (threadIdx.x == 0) partial[blockIdx.x] = f;
}
// product of the per-block partials -> ONE Fp12 (the product of all Miller values), written in wire form; the single final
// exponentiation is then the ordinary k_final_exp launch over that one element
template <class P>
__global__ void __launch_bounds__(PROD_BLOCK) k_product_tree(size_t nparts, const typename P::F12* __restrict__ partial, uint8_t* __restrict__ f_out) {
  extern __shared__ __align__(16) unsigned char smraw[];
  auto* sm = reinterpret_cast<typename P::F12*>(smraw);
  typename P::F12 f;
  fp12_set_one(f);
  for (size_t j = threadIdx.x; j < nparts; j += PROD_BLOCK) {
    typename P::F12 p = partial[j];
    fp12_mul(f, f, p);
  }
  block_product(sm, f);
  if (threadIdx.x == 0) P::store(f_out, f);
}

// ---- G1 / G2 group operations on operand-form points ---------------------------------------------------------------------------
template <class CV>
__global__ void __launch_bounds__(128) k_add_batch(size_t n, const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, int negate_b,
                                                   uint8_t* __restrict__ out, uint32_t* flags) {
  using F = typename CV::F;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<F> p, q, r;
  bool good = load_checked<CV>(p, a + (size_t)CV::IN_BYTES * i);
  good = load_checked<CV>(q, b + (size_t)CV::IN_BYTES * i) && good;
  if (!good) atomicOr(flags, FLAG_POINT);
  if (negate_b) f_neg(q.y, q.y);
  Jac<F> j;
  jac_from_affine(j, p);
  jac_madd(j, j, q);                            // handles P + P, P - P, infinities
  jac_to_affine_bg(r, j);
  CV::store_affine(out + (size_t)CV::IN_BYTES * i, r);
}

}  // namespace b2k

// ================================================================================================
namespace {

// out[i] = a[i]^scalars[i] on device buffers: one warp per element for small batches, one thread per element above
template <class P>
void launch_gt_exp(const b2k_ctx* ctx, size_t n, const uint8_t* ds, const uint8_t* da, uint8_t* dout) {
  if (ctx->coop_max_n > 0 && n <= (size_t)(ctx->coop_max_n < 4096 ? ctx->coop_max_n : 4096)) {
    using SQR = typename P::CoopSqr;
    using MUL = typename P::CoopMul;
    using C = typename P::FC;
    constexpr int NS = (SQR::SLOTS > MUL::SLOTS ? SQR::SLOTS : MUL::SLOTS) | 1;
    k_coop_gt_exp<P, C, SQR, MUL><<<(unsigned)n, 32, (size_t)C::N * (NS + 12) * 4, ctx->stream>>>(n, ds, da, dout, ctx->d_flags);
  } else
    k_gt_exp<P><<<(unsigned)((n + 63) / 64), 64, 0, ctx->stream>>>(n, ds, da, dout, ctx->d_flags);
}

template <class P>
int gt_binary(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* a, const uint8_t* b, uint8_t* out, int op) {
  if (!ctx || !a || !out || n == 0 || (op == 0 && !b) || (op == 2 && !scalars)) return bad_arg(ctx, "bad argument");
  CK(cudaSetDevice(ctx->device));
  const size_t gb = (size_t)P::GT_BYTES;
  uint8_t *da = nullptr, *db = nullptr, *ds = nullptr, *dout = nullptr;
  return host_call(ctx, [&](Carve& c) {
    da = c.in(a, n, gb);
    db = c.in(b, op == 0 ? n : 0, gb);
    ds = c.in(scalars, op == 2 ? n : 0, 32);
    dout = c.out(out, n, gb);
  }, [&]() -> int {
    const unsigned grid = (unsigned)((n + 63) / 64);
    if (op == 0) k_gt_mul<P><<<grid, 64, 0, ctx->stream>>>(n, da, db, dout, ctx->d_flags);
    else if (op == 1) k_gt_inv<P><<<grid, 64, 0, ctx->stream>>>(n, da, dout, ctx->d_flags);
    else launch_gt_exp<P>(ctx, n, ds, da, dout);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  });
}

template <class P>
int miller_host(b2k_ctx* ctx, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* out) {
  if (!ctx || !g1 || !g2 || !out || n == 0) return bad_arg(ctx, "bad argument");
  CK(cudaSetDevice(ctx->device));
  uint8_t *d1 = nullptr, *d2 = nullptr, *dg = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d1 = c.in(g1, n, P::G1::IN_BYTES);
    d2 = c.in(g2, n, P::G2::IN_BYTES);
    dg = c.out(out, n, P::GT_BYTES);
  }, [&]() -> int {
    k_miller<P><<<(unsigned)((n + 63) / 64), 64, 0, ctx->stream>>>(n, d1, d2, dg, ctx->d_flags);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  });
}

template <class P>
int final_exp_host(b2k_ctx* ctx, size_t n, const uint8_t* in, uint8_t* out) {
  if (!ctx || !in || !out || n == 0) return bad_arg(ctx, "bad argument");
  CK(cudaSetDevice(ctx->device));
  uint8_t *di = nullptr, *dout = nullptr;
  return host_call(ctx, [&](Carve& c) {
    di = c.in(in, n, P::GT_BYTES);
    dout = c.out(out, n, P::GT_BYTES);
  }, [&]() -> int {
    k_final_exp<P><<<(unsigned)((n + 63) / 64), 64, 0, ctx->stream>>>(n, di, dout, ctx->d_flags);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  });
}

// ok[0] = (prod_i e(g1_i, g2_i) == 1); gt (optional) = the product's bytes
template <class P>
int product_check_host(b2k_ctx* ctx, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* ok, uint8_t* gt) {
  using F12 = typename P::F12;
  if (!ctx || !g1 || !g2 || (!ok && !gt) || n == 0 || n >= (size_t(1) << 31)) return bad_arg(ctx, "bad argument");
  CK(cudaSetDevice(ctx->device));
  const size_t gb = (size_t)P::GT_BYTES;
  size_t nblk = (n + b2k::PROD_BLOCK - 1) / b2k::PROD_BLOCK;
  if (nblk > 4096) nblk = 4096;                                              // beyond that a thread multiplies several values
  uint8_t hgt[576];
  uint8_t *d1 = nullptr, *d2 = nullptr, *dm = nullptr, *df = nullptr, *dgt = nullptr;
  F12* parts = nullptr;
  const int rc = host_call(ctx, [&](Carve& c) {
    d1 = c.in(g1, n, P::G1::IN_BYTES);
    d2 = c.in(g2, n, P::G2::IN_BYTES);
    dm = c.take<uint8_t>(n, gb);
    parts = c.take<F12>(nblk);
    df = c.take<uint8_t>(gb);
    dgt = c.out(gt ? gt : hgt, gb);
  }, [&]() -> int {
    cudaStream_t st = ctx->stream;
    const size_t smem = b2k::PROD_BLOCK * sizeof(F12);
    k_miller<P><<<(unsigned)((n + 63) / 64), 64, 0, st>>>(n, d1, d2, dm, ctx->d_flags);
    k_gt_block_product<P><<<(unsigned)nblk, b2k::PROD_BLOCK, smem, st>>>(n, dm, parts);
    k_product_tree<P><<<1, b2k::PROD_BLOCK, smem, st>>>(nblk, parts, df);
    k_final_exp<P><<<1, 64, 0, st>>>(1, df, dgt, ctx->d_flags);               // ONE final exponentiation
    CK(cudaGetLastError());
    ctx->launches += 4;
    return B2K_OK;
  });
  if (rc) return rc;
  if (ok) {
    const uint8_t* e = gt ? gt : hgt;                                      // GT one = 0 ... 0 1 (only the last coefficient, c0.c0.c0)
    bool one = e[gb - 1] == 1;
    for (size_t i = 0; one && i + 1 < gb; i++) one = e[i] == 0;
    ok[0] = one ? 1 : 0;
  }
  return B2K_OK;
}

template <class CV>
int add_batch_host(b2k_ctx* ctx, size_t n, const uint8_t* a, const uint8_t* b, int negate_b, uint8_t* out) {
  if (!ctx || !a || !b || !out || n == 0) return bad_arg(ctx, "bad argument");
  CK(cudaSetDevice(ctx->device));
  uint8_t *da = nullptr, *db = nullptr, *dout = nullptr;
  return host_call(ctx, [&](Carve& c) {
    da = c.in(a, n, CV::IN_BYTES);
    db = c.in(b, n, CV::IN_BYTES);
    dout = c.out(out, n, CV::IN_BYTES);
  }, [&]() -> int {
    k_add_batch<CV><<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(n, da, db, negate_b, dout, ctx->d_flags);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  });
}

}  // namespace

extern "C" {

int b2k_bls12381_gt_mul(b2k_ctx* c, size_t n, const uint8_t* a, const uint8_t* b, uint8_t* o) { return gt_binary<BlsPairing>(c, n, nullptr, a, b, o, 0); }
int b2k_bls12381_gt_inv(b2k_ctx* c, size_t n, const uint8_t* a, uint8_t* o) { return gt_binary<BlsPairing>(c, n, nullptr, a, nullptr, o, 1); }
int b2k_bls12381_gt_exp(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* a, uint8_t* o) { return gt_binary<BlsPairing>(c, n, s, a, nullptr, o, 2); }
int b2k_bn254_gt_mul(b2k_ctx* c, size_t n, const uint8_t* a, const uint8_t* b, uint8_t* o) { return gt_binary<Bn254Pairing>(c, n, nullptr, a, b, o, 0); }
int b2k_bn254_gt_inv(b2k_ctx* c, size_t n, const uint8_t* a, uint8_t* o) { return gt_binary<Bn254Pairing>(c, n, nullptr, a, nullptr, o, 1); }
int b2k_bn254_gt_exp(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* a, uint8_t* o) { return gt_binary<Bn254Pairing>(c, n, s, a, nullptr, o, 2); }

int b2k_bls12381_miller(b2k_ctx* c, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* o) { return miller_host<BlsPairing>(c, n, g1, g2, o); }
int b2k_bls12381_final_exp(b2k_ctx* c, size_t n, const uint8_t* in, uint8_t* o) { return final_exp_host<BlsPairing>(c, n, in, o); }
int b2k_bls12381_pairing_product_check(b2k_ctx* c, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* ok) { return product_check_host<BlsPairing>(c, n, g1, g2, ok, nullptr); }
int b2k_bls12381_pairing_product(b2k_ctx* c, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* gt) { return product_check_host<BlsPairing>(c, n, g1, g2, nullptr, gt); }

int b2k_bn254_miller(b2k_ctx* c, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* o) { return miller_host<Bn254Pairing>(c, n, g1, g2, o); }
int b2k_bn254_finalize(b2k_ctx* c, size_t n, const uint8_t* in, uint8_t* o) { return final_exp_host<Bn254Pairing>(c, n, in, o); }
int b2k_bn254_pairing_product_check(b2k_ctx* c, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* ok) { return product_check_host<Bn254Pairing>(c, n, g1, g2, ok, nullptr); }
int b2k_bn256_miller(b2k_ctx* c, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* o) { return miller_host<Bn256Pairing>(c, n, g1, g2, o); }
int b2k_bn256_finalize(b2k_ctx* c, size_t n, const uint8_t* in, uint8_t* o) { return final_exp_host<Bn256Pairing>(c, n, in, o); }
int b2k_bn256_pairing_product_check(b2k_ctx* c, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* ok) { return product_check_host<Bn256Pairing>(c, n, g1, g2, ok, nullptr); }

int b2k_bls12381_g1_add_batch(b2k_ctx* c, size_t n, const uint8_t* a, const uint8_t* b, int neg, uint8_t* o) { return add_batch_host<Bls381G1>(c, n, a, b, neg, o); }
int b2k_bls12381_g2_add_batch(b2k_ctx* c, size_t n, const uint8_t* a, const uint8_t* b, int neg, uint8_t* o) { return add_batch_host<Bls381G2>(c, n, a, b, neg, o); }

// the exponentiation dispatch of b2k_bls12381_gt_exp on device buffers (the IBE encryption's Gid^r, b2k_ibe.cu); enqueue only
void b2k_internal_launch_bls12381_gt_exp(const b2k_ctx* c, size_t n, const uint8_t* ds, const uint8_t* da, uint8_t* dout) {
  launch_gt_exp<BlsPairing>(c, n, ds, da, dout);
}

}  // extern "C"
