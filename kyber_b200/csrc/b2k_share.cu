// b2k_share.cu -- share.RecoverCommit and share.PubPoly.Eval on the device.
//
// RecoverCommit (reference share/poly.go:449-476): the O(t^2) mod.Int products (num *= x_j, den *= x_j - x_i,
// :464-470), the t modular inversions (num.Div, :471) and the t Point.Mul + Add (:471-472) -> Lagrange kernel + MSM.
// The caller (Go: xyCommit, poly.go:418-445) still sorts the shares by index and passes the first t
// (index, point) pairs; x_i = index_i + 1.
// PubPoly.Eval / Shares (poly.go:340-357): v = sum_j x^j C_j by Horner, one thread per evaluation index; this is the
// per-partial-signature cost of tbls.Recover (sign/tbls/tbls.go:118-151: public.Eval(idx) for every share).
#define B2K_FP2_BYREF 1   // Fp2 products out of line BY REFERENCE (tower.cuh): instantiates the G2 MSM kernels (RecoverCommit on G2): same layout as b2k_g2.cu, or the weak host stubs of the two units would name different device code
#include "msm_host.cuh"
#include "codec.cuh"
#include "lagrange.cuh"
using namespace b2k_host;

namespace b2k {

// v = sum_j x^j C_j  (Horner: v = x v + C_j, poly.go:343-346), x * v by double-and-add over the bits of x (top bit consumed).
// Out of line: inlined into k_pubpoly_check next to its scalar multiplication, sm_90a code gave wrong G2 points for t >= 2.
template <class CV>
__device__ __noinline__ void pubpoly_horner(Jac<typename CV::F>& v, const Affine<typename CV::F>* __restrict__ cm, uint32_t t, uint64_t x) {
  using F = typename CV::F;
  int top = 63;
  while (top > 0 && !((x >> top) & 1)) top--;
  jac_set_inf(v);
  for (int j = (int)t - 1; j >= 0; j--) {
    Jac<F> acc = v;
    for (int b = top - 1; b >= 0; b--) {
      jac_dbl(acc, acc);
      if ((x >> b) & 1) jac_add(acc, acc, v);
    }
    Affine<F> c = cm[j];
    jac_madd(v, acc, c);
  }
}

// out[i] = sum_j (idx_i + 1)^j C_j, operand form
template <class CV>
__global__ void __launch_bounds__(128) k_pubpoly_eval(uint32_t t, const Affine<typename CV::F>* __restrict__ commits, uint32_t n,
                                                      const uint32_t* __restrict__ idx, uint8_t* __restrict__ out) {
  using F = typename CV::F;
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Jac<F> v;
  pubpoly_horner<CV>(v, commits, t, (uint64_t)idx[i] + 1u);
  Affine<F> a;
  jac_to_affine(a, v);
  CV::store_affine(out + (size_t)CV::IN_BYTES * i, a);
}

// PubPoly.Check for a batch of dealers (share/poly.go:405-409 as run once per received deal by
// share/vss/pedersen/vss.go:636-645 and share/dkg/pedersen/dkg.go:489-494, 826-834): thread (d, k) evaluates dealer d's
// commitment polynomial at idx[d][k] + 1 by Horner, multiplies the base point by the private share and compares the two
// results projectively (no inversion).  A share that is not below the group order fails its check (the reference drops
// such a deal when UnmarshalBinary errors, dkg.go:484-487).
template <class CV>
__global__ void __launch_bounds__(128) k_pubpoly_check(uint32_t m, uint32_t t, const Affine<typename CV::F>* __restrict__ commits,
                                                       uint32_t n, const uint32_t* __restrict__ idx,
                                                       const uint8_t* __restrict__ shares, uint8_t* __restrict__ ok, int use_glv) {
  using F = typename CV::F;
  size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (size_t)m * n) return;
  const uint32_t d = (uint32_t)(id / n);
  Jac<F> v;
  pubpoly_horner<CV>(v, commits + (size_t)d * t, t, (uint64_t)idx[id] + 1u);
  Scalar256 k;
  scalar_load_be(k, shares + 32 * id);
  if (!scalar_in_range<typename CV::ScalarField>(k)) { ok[id] = 0; return; }
  Affine<F> g;
  CV::generator(g);
  Jac<F> w;
  if constexpr (MulGlv<CV>::enabled) {
    if (use_glv) scalar_mul_glv_bls381(w, k, g, InvBingcd{});
    else scalar_mul<CV>(w, k, g);
  } else {
    scalar_mul<CV>(w, k, g);
  }
  // v == w  <=>  both infinite, or X_v Z_w^2 == X_w Z_v^2 and Y_v Z_w^3 == Y_w Z_v^3
  bool same;
  if (jac_is_inf(v) || jac_is_inf(w)) same = jac_is_inf(v) && jac_is_inf(w);
  else {
    F zv2, zw2, a, b;
    f_sqr(zv2, v.Z); f_sqr(zw2, w.Z);
    f_mul(a, v.X, zw2); f_mul(b, w.X, zv2);
    same = f_eq(a, b);
    f_mul(zv2, zv2, v.Z); f_mul(zw2, zw2, w.Z);
    f_mul(a, v.Y, zw2); f_mul(b, w.Y, zv2);
    same = same && f_eq(a, b);
  }
  ok[id] = same ? 1 : 0;
}

}  // namespace b2k

template <class CV, class FR>
static int recover_commit(b2k_ctx* ctx, size_t t, const uint32_t* indices, const uint8_t* points, uint8_t* out) {
  MsmLayout<CV> s;
  uint32_t* d_idx = nullptr;
  uint8_t *d_s = nullptr, *d_p = nullptr, *d_o = nullptr;
  int rc = msm_begin<CV>(ctx, t, indices && points && out, s, [&](Carve& c) {
    d_idx = c.take<uint32_t>(t);
    d_s = c.take<uint8_t>(t * 32);
    d_p = c.take<uint8_t>(t * (size_t)CV::IN_BYTES);
    d_o = c.take<uint8_t>(256);
  });
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  if ((rc = status_begin(ctx))) return rc;
  CK(cudaMemcpyAsync(d_idx, indices, t * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_p, points, t * (size_t)CV::IN_BYTES, cudaMemcpyHostToDevice, st));
  k_lagrange_at_zero<FR><<<(unsigned)((t + 127) / 128), 128, 0, st>>>((uint32_t)t, d_idx, d_s, ctx->d_flags);
  ctx->launches += 1;
  rc = msm_enqueue<CV>(ctx, s, d_s, d_p, d_o);
  if (rc) return rc;
  CK(cudaMemcpyAsync(out, d_o, CV::OUT_BYTES, cudaMemcpyDeviceToHost, st));
  return status_finish(ctx);
}

template <class CV>
static int pubpoly_eval(b2k_ctx* ctx, size_t t, const uint8_t* commits, size_t n, const uint32_t* indices, uint8_t* out) {
  using F = typename CV::F;
  if (!ctx || !commits || !indices || !out || t == 0 || n == 0 || t >= (size_t(1) << 31) || n >= (size_t(1) << 31)) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  uint8_t *d_c = nullptr, *d_o = nullptr;
  uint32_t* d_idx = nullptr;
  Affine<F>* d_cm = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_c = c.in(commits, t, CV::IN_BYTES);
    d_idx = c.in(indices, n);
    d_cm = c.take<Affine<F>>(t);
    d_o = c.out(out, n, CV::IN_BYTES);
  }, [&]() -> int {
    cudaStream_t st = ctx->stream;
    k_load_points<CV><<<(unsigned)((t + 255) / 256), 256, 0, st>>>(t, d_c, d_cm, ctx->d_flags);
    k_pubpoly_eval<CV><<<(unsigned)((n + 127) / 128), 128, 0, st>>>((uint32_t)t, d_cm, (uint32_t)n, d_idx, d_o);
    CK(cudaGetLastError());
    ctx->launches += 2;
    return B2K_OK;
  });
}

template <class CV>
static int pubpoly_check(b2k_ctx* ctx, size_t m, size_t t, const uint8_t* commits, size_t n, const uint32_t* indices,
                         const uint8_t* shares, uint8_t* ok) {
  using F = typename CV::F;
  if (!ctx || !commits || !indices || !shares || !ok || m == 0 || t == 0 || n == 0 || m * t >= (size_t(1) << 31) ||
      m * n >= (size_t(1) << 31)) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  const size_t mt = m * t, mn = m * n;
  uint8_t *d_c = nullptr, *d_s = nullptr, *d_ok = nullptr;
  uint32_t* d_idx = nullptr;
  Affine<F>* d_cm = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_c = c.in(commits, mt, CV::IN_BYTES);
    d_idx = c.in(indices, mn);
    d_s = c.in(shares, mn, 32);
    d_cm = c.take<Affine<F>>(mt);
    d_ok = c.out(ok, mn);
  }, [&]() -> int {
    cudaStream_t st = ctx->stream;
    k_load_points<CV><<<(unsigned)((mt + 255) / 256), 256, 0, st>>>(mt, d_c, d_cm, ctx->d_flags);
    k_pubpoly_check<CV><<<(unsigned)((mn + 127) / 128), 128, 0, st>>>((uint32_t)m, (uint32_t)t, d_cm, (uint32_t)n, d_idx, d_s, d_ok, ctx->use_glv);
    CK(cudaGetLastError());
    ctx->launches += 2;
    return B2K_OK;
  });
}

extern "C" {

int b2k_bls12381_g1_pubpoly_check(b2k_ctx* c, size_t m, size_t t, const uint8_t* commits, size_t n, const uint32_t* idx, const uint8_t* shares, uint8_t* ok) { return pubpoly_check<Bls381G1>(c, m, t, commits, n, idx, shares, ok); }
int b2k_bls12381_g2_pubpoly_check(b2k_ctx* c, size_t m, size_t t, const uint8_t* commits, size_t n, const uint32_t* idx, const uint8_t* shares, uint8_t* ok) { return pubpoly_check<Bls381G2>(c, m, t, commits, n, idx, shares, ok); }
int b2k_bn254_pubpoly_check(b2k_ctx* c, size_t m, size_t t, const uint8_t* commits, size_t n, const uint32_t* idx, const uint8_t* shares, uint8_t* ok) { return pubpoly_check<Bn254G1>(c, m, t, commits, n, idx, shares, ok); }
int b2k_bn254_recover_commit(b2k_ctx* c, size_t t, const uint32_t* idx, const uint8_t* pts, uint8_t* out) { return recover_commit<Bn254G1, Bn254Fr>(c, t, idx, pts, out); }
int b2k_bls12381_g1_recover_commit(b2k_ctx* c, size_t t, const uint32_t* idx, const uint8_t* pts, uint8_t* out) { return recover_commit<Bls381G1, Bls381Fr>(c, t, idx, pts, out); }
int b2k_bls12381_g2_recover_commit(b2k_ctx* c, size_t t, const uint32_t* idx, const uint8_t* pts, uint8_t* out) { return recover_commit<Bls381G2, Bls381Fr>(c, t, idx, pts, out); }
int b2k_bls12381_g1_pubpoly_eval(b2k_ctx* c, size_t t, const uint8_t* commits, size_t n, const uint32_t* idx, uint8_t* out) { return pubpoly_eval<Bls381G1>(c, t, commits, n, idx, out); }
int b2k_bls12381_g2_pubpoly_eval(b2k_ctx* c, size_t t, const uint8_t* commits, size_t n, const uint32_t* idx, uint8_t* out) { return pubpoly_eval<Bls381G2>(c, t, commits, n, idx, out); }

}  // extern "C"
