// b2k_share2.cu -- share.RecoverPubPoly and PriPoly.Commit on the device (split from b2k_share.cu: the two halves compile in parallel).
//
// RecoverPubPoly (poly.go:480-508): the whole public polynomial from t shares, commits[k] = sum_j L_j[k] y_j with L_j the
// Lagrange basis polynomials (lagrangeBasis, poly.go:513-545): master polynomial M(x) = prod (x - x_m) built by one block in t
// steps, L_j = M / (x - x_j) / M'(x_j) by synthetic division (one thread per j, O(t) each instead of the reference's O(t^2)
// polynomial products per j), then t^2 scalar multiplications and t column sums.
// PriPoly.Commit (poly.go:143-149): commits[i] = coeffs[i] * B for one base point B -- a fixed-base batch.
#define B2K_FP2_BYREF 1   // Fp2 products out of line BY REFERENCE (tower.cuh): G2 RecoverPubPoly / Commit batches: same layout as b2k_g2.cu
#include "msm_host.cuh"
#include "codec.cuh"
using namespace b2k_host;

namespace b2k {

// ---- RecoverPubPoly ---------------------------------------------------------------------------------------------------------
template <class FR>
B2K_D void fr_from_index(Fp<FR>& x, uint32_t idx) {                 // x = idx + 1 in Montgomery form (poly.go:440)
  fp_set_zero(x);
  x.v[0] = idx + 1u; x.v[1] = (idx == 0xffffffffu) ? 1u : 0u;
  fp_to_mont(x, x);
}
// M(x) = prod_m (x - x_m), coefficients c[0..t] (Montgomery), built in t steps by ONE block: c'[i] = c[i-1] - x_k c[i]
template <class FR>
__global__ void __launch_bounds__(1024) k_master_poly(uint32_t t, const uint32_t* __restrict__ idx, Fp<FR>* __restrict__ ca, Fp<FR>* __restrict__ cb) {
  using S = Fp<FR>;
  S* cur = ca;
  S* nxt = cb;
  for (uint32_t i = threadIdx.x; i <= t; i += blockDim.x) { S v; if (i == 0) fp_set_one(v); else fp_set_zero(v); cur[i] = v; }
  __syncthreads();
  for (uint32_t k = 0; k < t; k++) {
    S xk;
    fr_from_index<FR>(xk, idx[k]);
    for (uint32_t i = threadIdx.x; i <= k + 1; i += blockDim.x) {
      S lo, hi, r;
      if (i > 0) lo = cur[i - 1]; else fp_set_zero(lo);
      if (i <= k) { hi = cur[i]; fp_mul(hi, hi, xk); } else fp_set_zero(hi);
      fp_sub(r, lo, hi);
      nxt[i] = r;
    }
    __syncthreads();
    S* tmp = cur; cur = nxt; nxt = tmp;
  }
  if (cur != ca) {                                                  // result always in ca
    for (uint32_t i = threadIdx.x; i <= t; i += blockDim.x) ca[i] = cur[i];
  }
}
// thread j: q = M / (x - x_j) (synthetic division, top down), d = q(x_j) = prod_{m != j} (x_j - x_m), row j of the basis matrix
// = q / d, written as big-endian scalars in COLUMN-major order: scal[k][j] = L_j[k]  (so that the terms of commit k are contiguous)
template <class FR>
__global__ void __launch_bounds__(128) k_lagrange_basis(uint32_t t, const uint32_t* __restrict__ idx, const Fp<FR>* __restrict__ c,
                                                        Fp<FR>* __restrict__ rows, uint8_t* __restrict__ scal, uint32_t* flags) {
  using S = Fp<FR>;
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= t) return;
  S xj, q, acc;
  fr_from_index<FR>(xj, idx[j]);
  fp_set_one(q);                                                    // q_{t-1} = c_t = 1
  acc = q;
  rows[(size_t)j * t + (t - 1)] = q;
  for (uint32_t i = t - 1; i >= 1; i--) {                          // q_{i-1} = c_i + x_j q_i
    S ci = c[i];
    fp_mul(q, q, xj);
    fp_add(q, q, ci);
    rows[(size_t)j * t + (i - 1)] = q;
    fp_mul(acc, acc, xj);
    fp_add(acc, acc, q);
  }
  if (fp_is_zero(acc)) atomicOr(flags, FLAG_DUP_INDEX);                         // x_j is a double root: duplicate index
  S inv;
  fp_inv(inv, acc);
  for (uint32_t k = 0; k < t; k++) {
    S v = rows[(size_t)j * t + k];
    fp_mul(v, v, inv);
    fp_from_mont(v, v);
    uint8_t* out = scal + 32 * ((size_t)k * t + j);
#pragma unroll
    for (int w = 0; w < 8; w++) {
      uint8_t* o = out + 4 * (7 - w);
      o[0] = (uint8_t)(v.v[w] >> 24); o[1] = (uint8_t)(v.v[w] >> 16); o[2] = (uint8_t)(v.v[w] >> 8); o[3] = (uint8_t)v.v[w];
    }
  }
}
// terms[k t + j] = scal[k][j] * y_j, normalised to affine by the same batched-per-thread pattern as k_mul_batch
template <class CV>
__global__ void __launch_bounds__(128) k_scale_points(size_t n, uint32_t t, const uint8_t* __restrict__ scal, const Affine<typename CV::F>* __restrict__ pts,
                                                      Affine<typename CV::F>* __restrict__ terms, uint32_t* flags, int use_glv) {
  size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n) return;
  Scalar256 k;
  scalar_load_be(k, scal + 32 * id);
  if (!scalar_in_range<typename CV::ScalarField>(k)) { atomicOr(flags, FLAG_SCALAR_RANGE); for (int w = 0; w < 8; w++) k.v[w] = 0; }
  Affine<typename CV::F> p = pts[id % t];
  Jac<typename CV::F> r;
  if constexpr (MulGlv<CV>::enabled) {
    if (use_glv) scalar_mul_glv_bls381(r, k, p, InvBingcd{});
    else scalar_mul_w4<CV>(r, k, p, InvBingcd{});
  } else {
    scalar_mul_w4<CV>(r, k, p, InvBingcd{});
  }
  Affine<typename CV::F> a;
  jac_to_affine_bg(a, r);
  terms[id] = a;
}
// sums[k] = sum_j terms[k t + j] (Jacobian): one block per k, mixed additions into per-thread sums, then a shared-memory tree
template <class CV>
__global__ void __launch_bounds__(64) k_column_sum(uint32_t t, const Affine<typename CV::F>* __restrict__ terms, Jac<typename CV::F>* __restrict__ sums) {
  using J = Jac<typename CV::F>;
  __shared__ J sm[64];
  const int tid = threadIdx.x;
  const size_t k = blockIdx.x;
  J acc;
  jac_set_inf(acc);
  for (uint32_t j = tid; j < t; j += 64) {
    Affine<typename CV::F> v = terms[k * t + j];
    jac_madd(acc, acc, v);
  }
  sm[tid] = acc;
  __syncthreads();
  for (int h = 32; h > 0; h >>= 1) {
    if (tid < h) {
      J a = sm[tid], b = sm[tid + h];
      jac_add(a, a, b);
      sm[tid] = a;
    }
    __syncthreads();
  }
  if (tid == 0) sums[k] = sm[0];
}
// out[k] = sums[k] in operand form (one thread per commitment)
template <class CV>
__global__ void __launch_bounds__(128) k_sums_to_affine(uint32_t t, const Jac<typename CV::F>* __restrict__ sums, uint8_t* __restrict__ out) {
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= t) return;
  Jac<typename CV::F> s = sums[k];
  Affine<typename CV::F> a;
  jac_to_affine_bg(a, s);
  CV::store_affine(out + (size_t)CV::IN_BYTES * k, a);
}
// out[i] = scalars[i] * B (operand form): PriPoly.Commit's loop (poly.go:145-147) over one base point
template <class CV>
__global__ void __launch_bounds__(128) k_commit_batch(size_t n, const uint8_t* __restrict__ scal, const uint8_t* __restrict__ base_wire,
                                                      uint8_t* __restrict__ out, uint32_t* flags, int use_glv) {
  size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n) return;
  Scalar256 k;
  scalar_load_be(k, scal + 32 * id);
  if (!scalar_in_range<typename CV::ScalarField>(k)) { atomicOr(flags, FLAG_SCALAR_RANGE); for (int w = 0; w < 8; w++) k.v[w] = 0; }
  Affine<typename CV::F> p;
  if (base_wire) { if (!load_checked<CV>(p, base_wire)) atomicOr(flags, FLAG_POINT); }
  else CV::generator(p);
  Jac<typename CV::F> r;
  if constexpr (MulGlv<CV>::enabled) {
    if (use_glv) scalar_mul_glv_bls381(r, k, p, InvBingcd{});
    else scalar_mul_w4<CV>(r, k, p, InvBingcd{});
  } else {
    scalar_mul_w4<CV>(r, k, p, InvBingcd{});
  }
  Affine<typename CV::F> a;
  jac_to_affine_bg(a, r);
  CV::store_affine(out + (size_t)CV::IN_BYTES * id, a);
}

}  // namespace b2k

using namespace b2k;

// share.RecoverPubPoly (poly.go:480-508): commits_out[k] (operand form), k = 0..t-1
template <class CV, class FR>
static int recover_pubpoly(b2k_ctx* ctx, size_t t, const uint32_t* indices, const uint8_t* points, uint8_t* commits_out) {
  using F = typename CV::F;
  using S = Fp<FR>;
  if (!ctx || !indices || !points || !commits_out || t == 0 || t > 4096) return bad_arg(ctx, "bad argument (1 <= t <= 4096)");
  CK(cudaSetDevice(ctx->device));
  const size_t tt = t * t;
  uint32_t* d_idx = nullptr;
  uint8_t *d_p = nullptr, *scal = nullptr, *d_o = nullptr;
  Affine<F> *d_pm = nullptr, *terms = nullptr;
  S *ca = nullptr, *cb = nullptr, *rows = nullptr;
  Jac<F>* sums = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_idx = c.in(indices, t);
    d_p = c.in(points, t, CV::IN_BYTES);
    d_pm = c.take<Affine<F>>(t);
    ca = c.take<S>(t + 1);
    cb = c.take<S>(t + 1);
    rows = c.take<S>(tt);
    scal = c.take<uint8_t>(tt, 32);
    terms = c.take<Affine<F>>(tt);
    sums = c.take<Jac<F>>(t);
    d_o = c.out(commits_out, t, CV::IN_BYTES);
  }, [&]() -> int {
    cudaStream_t st = ctx->stream;
    k_load_points<CV><<<(unsigned)((t + 255) / 256), 256, 0, st>>>(t, d_p, d_pm, ctx->d_flags);
    k_master_poly<FR><<<1, 1024, 0, st>>>((uint32_t)t, d_idx, ca, cb);
    k_lagrange_basis<FR><<<(unsigned)((t + 127) / 128), 128, 0, st>>>((uint32_t)t, d_idx, ca, rows, scal, ctx->d_flags);
    k_scale_points<CV><<<(unsigned)((tt + 127) / 128), 128, 0, st>>>(tt, (uint32_t)t, scal, d_pm, terms, ctx->d_flags, ctx->use_glv);
    k_column_sum<CV><<<(unsigned)t, 64, 0, st>>>((uint32_t)t, terms, sums);
    k_sums_to_affine<CV><<<(unsigned)((t + 127) / 128), 128, 0, st>>>((uint32_t)t, sums, d_o);
    CK(cudaGetLastError());
    ctx->launches += 6;
    return B2K_OK;
  });
}

// PriPoly.Commit (poly.go:143-149): out[i] = scalars[i] * base (base == NULL: the group's generator), operand form
template <class CV>
static int commit_batch(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* base, uint8_t* out) {
  if (!ctx || !scalars || !out || n == 0) return bad_arg(ctx, "bad argument");
  CK(cudaSetDevice(ctx->device));
  uint8_t *d_s = nullptr, *d_b = nullptr, *d_o = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_s = c.in(scalars, n, 32);
    d_b = c.in(base, base ? CV::IN_BYTES : 0);
    d_o = c.out(out, n, CV::IN_BYTES);
  }, [&]() -> int {
    k_commit_batch<CV><<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(n, d_s, base ? d_b : nullptr, d_o, ctx->d_flags, ctx->use_glv);
    CK(cudaGetLastError());
    ctx->launches += 1;
    return B2K_OK;
  });
}

extern "C" {

int b2k_bls12381_g1_recover_pubpoly(b2k_ctx* c, size_t t, const uint32_t* idx, const uint8_t* pts, uint8_t* out) { return recover_pubpoly<Bls381G1, Bls381Fr>(c, t, idx, pts, out); }
int b2k_bls12381_g2_recover_pubpoly(b2k_ctx* c, size_t t, const uint32_t* idx, const uint8_t* pts, uint8_t* out) { return recover_pubpoly<Bls381G2, Bls381Fr>(c, t, idx, pts, out); }
int b2k_bn254_recover_pubpoly(b2k_ctx* c, size_t t, const uint32_t* idx, const uint8_t* pts, uint8_t* out) { return recover_pubpoly<Bn254G1, Bn254Fr>(c, t, idx, pts, out); }
int b2k_bls12381_g1_commit_batch(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* base, uint8_t* out) { return commit_batch<Bls381G1>(c, n, s, base, out); }
int b2k_bls12381_g2_commit_batch(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* base, uint8_t* out) { return commit_batch<Bls381G2>(c, n, s, base, out); }
int b2k_bn254_commit_batch(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* base, uint8_t* out) { return commit_batch<Bn254G1>(c, n, s, base, out); }

}  // extern "C"
