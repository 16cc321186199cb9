// kernels.cuh -- __global__ wrappers around the per-thread bodies of msm.cuh (sm_90a).
#pragma once
#include "msm.cuh"
#include "fp_inv.cuh"
#include "msm_affine.cuh"
#include "msm_sort.cuh"

namespace b2k {

// error flag bits written by kernels
enum : uint32_t { FLAG_SCALAR_RANGE = 1u, FLAG_POINT = 2u, FLAG_COMM_TIMEOUT = 32u };   // (4u: duplicate share index, b2k_share.cu)

// ---- operand conversion: wire bytes -> Montgomery affine (AoS, one point = 2*N limbs) -----------
template <class CV>
__global__ void __launch_bounds__(256) k_load_points(size_t n, const uint8_t* __restrict__ wire,
                                                     Affine<typename CV::F>* __restrict__ pts, uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<typename CV::F> p;
  if (!load_checked<CV>(p, wire + (size_t)CV::IN_BYTES * i)) atomicOr(flags, FLAG_POINT);
  pts[i] = p;
}

// ---- MSM front end: digit columns + histogram from the pass that loads the points ------------------------------------------
// Digit columns and histogram: msm_digits_store (msm_sort.cuh).
//
// groups without GLV: operand conversion, scalar range check and digits of pair i
template <class CV>
__global__ void __launch_bounds__(256) k_msm_load(size_t n, const uint8_t* __restrict__ scalars, const uint8_t* __restrict__ wire,
                                                  Affine<typename CV::F>* __restrict__ pts, MsmPlan pl, int16_t* __restrict__ digits,
                                                  uint32_t* __restrict__ counts, uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<typename CV::F> p;
  if (!load_checked<CV>(p, wire + (size_t)CV::IN_BYTES * i)) atomicOr(flags, FLAG_POINT);
  pts[i] = p;
  Scalar256 s;
  scalar_load_be(s, scalars + 32 * i);
  if (!scalar_in_range<typename CV::ScalarField>(s)) atomicOr(flags, FLAG_SCALAR_RANGE);
  msm_digits_store(s, pl, n, i, digits, counts);
}

// ---- GLV front end (BLS12-381 G1): operand conversion + scalar split + digits in one pass -------------------------------------
// pts[i] = +-P_i, pts[n+i] = +-(-phi(P_i)) = (beta x, -+y); the digits of the two 127-bit magnitudes go to rows i and n + i of the
// digit columns (2n rows), so that the sort and accumulate stages run unchanged over 2n (scalar, point) pairs.
// The launch covers pairs [i0, i0 + cnt) of the n of the call: the host-buffer MSM launches it once per chunk of its input copy.
static __global__ void __launch_bounds__(256) k_glv_prepare_bls381(size_t n, size_t i0, size_t cnt, const uint8_t* __restrict__ scalars,
                                                                   const uint8_t* __restrict__ wire,
                                                                   Affine<Fp<Bls381Fp>>* __restrict__ pts, MsmPlan pl,
                                                                   int16_t* __restrict__ digits, uint32_t* __restrict__ counts,
                                                                   uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cnt) return;
  i += i0;
  using F = Fp<Bls381Fp>;
  Scalar256 k;
  scalar_load_be(k, scalars + 32 * i);
  if (!scalar_in_range<Bls381Fr>(k)) {
    atomicOr(flags, FLAG_SCALAR_RANGE);
    for (int j = 0; j < 8; j++) k.v[j] = 0;
  }
  GlvSplit sp;
  glv_split_bls381(sp, k);
  Affine<F> p0, p, e;
  if (!load_checked<Bls381G1>(p0, wire + (size_t)Bls381G1::IN_BYTES * i)) atomicOr(flags, FLAG_POINT);
  glv_points_bls381(p, e, p0, sp);
  pts[i] = p;
  pts[n + i] = e;
  msm_digits_store(sp.k1, pl, 2 * n, i, digits, counts);
  msm_digits_store(sp.k2, pl, 2 * n, n + i, digits, counts);
}

// ---- independent scalar multiplications ----------------------------------------------------------
// warp-wide inversions go through the branch-free binary GCD (fp_inv.cuh): every lane inverts at the same time
struct InvBingcd { template <class F> B2K_D void operator()(F& r, const F& a) const { f_inv_bg(r, a); } };
template <class F>
B2K_D void jac_to_affine_bg(Affine<F>& r, const Jac<F>& p) {
  if (jac_is_inf(p)) { aff_set_inf(r); return; }
  F zi, zi2;
  f_inv_bg(zi, p.Z);
  f_sqr(zi2, zi);
  f_mul(r.x, p.X, zi2);
  f_mul(zi2, zi2, zi);
  f_mul(r.y, p.Y, zi2);
}
template <class CV> struct MulGlv { static constexpr bool enabled = false; };
template <> struct MulGlv<Bls381G1> { static constexpr bool enabled = true; };

template <class CV, bool AFFINE_OUT, int MINB = 1>
__global__ void __launch_bounds__(128, MINB) k_mul_batch(size_t n, const uint8_t* __restrict__ scalars,
                                                   const uint8_t* __restrict__ wire, uint8_t* __restrict__ out,
                                                   uint32_t* flags, int use_glv) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Scalar256 k;
  scalar_load_be(k, scalars + 32 * i);
  if (!scalar_in_range<typename CV::ScalarField>(k)) {
    atomicOr(flags, FLAG_SCALAR_RANGE);
    for (int j = 0; j < 8; j++) k.v[j] = 0;
  }
  Affine<typename CV::F> p;
  if (!load_checked<CV>(p, wire + (size_t)CV::IN_BYTES * i)) atomicOr(flags, FLAG_POINT);
  Jac<typename CV::F> r;
  if constexpr (MulGlv<CV>::enabled) {
    if (use_glv) scalar_mul_glv_bls381(r, k, p, InvBingcd{});
    else scalar_mul_w4<CV>(r, k, p, InvBingcd{});
  } else {
    scalar_mul_w4<CV>(r, k, p, InvBingcd{});
  }
  Affine<typename CV::F> a;
  jac_to_affine_bg(a, r);
  if (AFFINE_OUT) CV::store_affine(out + (size_t)CV::IN_BYTES * i, a);
  else CV::store(out + (size_t)CV::OUT_BYTES * i, a);
}

// ---- MSM stage 2: exclusive scan of the histogram (3 small kernels, 1024 elements per block) -------
// Column y = blockIdx.y scans the bucket sizes after y affine pair-tree rounds, ceil(counts / 2^y) (msm_affine.cuh); column 0
// (the histogram itself) goes to offs, column y >= 1 to offs_rounds + (y - 1) (total + 1).  Block totals: bsum + 1024 y.
B2K_D uint32_t* scan_column(uint32_t total, uint32_t* offs, uint32_t* offs_rounds, uint32_t y) {
  return y == 0 ? offs : offs_rounds + (size_t)(y - 1) * (total + 1);
}
// pass A: per-block exclusive scan + block totals
static __global__ void __launch_bounds__(1024) k_scan_blocks(uint32_t total, const uint32_t* __restrict__ counts,
                                                      uint32_t* __restrict__ offs, uint32_t* __restrict__ offs_rounds,
                                                      uint32_t* __restrict__ bsum) {
  __shared__ uint32_t wsum[32];
  const uint32_t y = blockIdx.y;
  offs = scan_column(total, offs, offs_rounds, y);
  bsum += 1024u * y;
  uint32_t i = blockIdx.x * 1024u + threadIdx.x;
  uint32_t v = (i < total) ? pt_round_count(counts[i], y) : 0u;
  uint32_t x = v;
  int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) wsum[warp] = x;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = wsum[lane], z = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      uint32_t y = __shfl_up_sync(0xffffffffu, z, d);
      if (lane >= d) z += y;
    }
    wsum[lane] = z - w;                       // exclusive prefix of warp totals
    if (lane == 31) bsum[blockIdx.x] = z;     // block total
  }
  __syncthreads();
  if (i < total) offs[i] = x - v + wsum[warp];
}
// pass B: exclusive scan of the block totals (<= 1024 blocks), grand total to offs[total]
static __global__ void __launch_bounds__(1024) k_scan_tops(uint32_t nblocks, uint32_t total, uint32_t* __restrict__ bsum,
                                                    uint32_t* __restrict__ offs, uint32_t* __restrict__ offs_rounds) {
  __shared__ uint32_t sm[1024];
  offs = scan_column(total, offs, offs_rounds, blockIdx.y);
  bsum += 1024u * blockIdx.y;
  int tid = threadIdx.x;
  uint32_t v = ((uint32_t)tid < nblocks) ? bsum[tid] : 0u;
  sm[tid] = v;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {
    uint32_t y = (tid >= d) ? sm[tid - d] : 0u;
    __syncthreads();
    sm[tid] += y;
    __syncthreads();
  }
  if ((uint32_t)tid < nblocks) bsum[tid] = sm[tid] - v;
  if (tid == 1023) offs[total] = sm[1023];
}
// pass C: add block offsets, duplicate column 0 into the scatter cursor
static __global__ void __launch_bounds__(1024) k_scan_finish(uint32_t total, const uint32_t* __restrict__ bsum,
                                                      uint32_t* __restrict__ offs, uint32_t* __restrict__ offs_rounds,
                                                      uint32_t* __restrict__ cursor) {
  const uint32_t y = blockIdx.y;
  offs = scan_column(total, offs, offs_rounds, y);
  uint32_t i = blockIdx.x * 1024u + threadIdx.x;
  if (i >= total) return;
  uint32_t o = offs[i] + bsum[1024u * y + blockIdx.x];
  offs[i] = o;
  if (y == 0) cursor[i] = o;
}

// ---- MSM stage 3: bucket sort in two passes: k_msm_partition, k_msm_bin_sort (msm_sort.cuh) --------------------------------

// ---- MSM stage 4: bucket accumulate (THE hot kernel) ---------------------------------------------
template <class CV>
__global__ void __launch_bounds__(128) k_msm_accumulate(size_t total, const Affine<typename CV::F>* __restrict__ pts,
                                                        const uint32_t* __restrict__ offs,
                                                        const uint32_t* __restrict__ entries,
                                                        Xyzz<typename CV::F>* __restrict__ buckets) {
  size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= total) return;
  Xyzz<typename CV::F> acc;
  msm_accumulate_bucket<CV>(acc, pts, entries, offs[g], offs[g + 1]);
  buckets[g] = acc;
}

// ---- MSM stage 4 (v2): fixed-length slices of the sorted entries (balanced, skew-proof) ------------
template <class CV, int MINB>
__global__ void __launch_bounds__(128, MINB) k_msm_accumulate_slices(uint32_t nslices, uint32_t L, uint32_t total,
                                                               const Affine<typename CV::F>* __restrict__ pts,
                                                               const uint32_t* __restrict__ offs,
                                                               const uint32_t* __restrict__ entries,
                                                               Xyzz<typename CV::F>* __restrict__ buckets,
                                                               Xyzz<typename CV::F>* __restrict__ spart) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nslices) return;
  msm_accumulate_slice<CV>(j, L, total, pts, offs, entries, buckets, spart);
}

// same over the output of the affine pair-tree rounds (the operands themselves, already sorted by bucket)
template <class CV, int MINB>
__global__ void __launch_bounds__(128, MINB) k_msm_accumulate_slices_direct(uint32_t nslices, uint32_t L, uint32_t total,
                                                                      const Affine<typename CV::F>* __restrict__ pts,
                                                                      const uint32_t* __restrict__ offs,
                                                                      Xyzz<typename CV::F>* __restrict__ buckets,
                                                                      Xyzz<typename CV::F>* __restrict__ spart) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nslices) return;
  msm_accumulate_slice<CV, true>(j, L, total, pts, offs, nullptr, buckets, spart);
}

// ---- MSM stage 4a: affine pair-tree rounds (msm_affine.cuh; bucket offsets of every round from the stage-2 scan) -------
// one thread = B consecutive outputs: B batched affine additions around one inversion
template <class CV, bool FIRST>
__global__ void __launch_bounds__(128, 4) k_msm_pairtree_round(uint32_t B, uint32_t total,
                                                               const Affine<typename CV::F>* __restrict__ in,
                                                               const uint32_t* __restrict__ entries,
                                                               const uint32_t* __restrict__ offs_in,
                                                               const uint32_t* __restrict__ offs_out,
                                                               Affine<typename CV::F>* __restrict__ out) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  msm_pairtree_round<CV, FIRST>(t, B, total, in, entries, offs_in, offs_out, out);
}

// the same round split by phase (msm_affine.cuh): T = threads of the launch = stride of pre[]
template <class CV, bool FIRST>
__global__ void __launch_bounds__(128, 5) k_pt_forward(uint32_t B, uint32_t total, const Affine<typename CV::F>* __restrict__ in,
                                                       const uint32_t* __restrict__ entries, const uint32_t* __restrict__ offs_in,
                                                       const uint32_t* __restrict__ offs_out, typename CV::F* __restrict__ pre,
                                                       typename CV::F* __restrict__ accs) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  msm_pairtree_forward<CV, FIRST>(t, B, gridDim.x * blockDim.x, total, in, entries, offs_in, offs_out, pre, accs);
}
// MINB = 5 caps the kernel at 96 registers: its one wave of 4 blocks per SM then leaves exactly one 128-register block slot,
// so a product kernel of ANOTHER MSM in flight (another context) can run under this latency-bound inversion pass.
// Measured with 4 MSMs in flight: no gain either way, off by default.
template <class F, int MINB = 4>
__global__ void __launch_bounds__(128, MINB) k_pt_invert(uint32_t B, uint32_t total, const uint32_t* __restrict__ offs_out, F* __restrict__ accs) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  msm_pairtree_invert<F>(t, B, total, offs_out, accs);
}
template <class CV, bool FIRST>
__global__ void __launch_bounds__(128, 4) k_pt_backward(uint32_t B, uint32_t total, const Affine<typename CV::F>* __restrict__ in,
                                                        const uint32_t* __restrict__ entries, const uint32_t* __restrict__ offs_in,
                                                        const uint32_t* __restrict__ offs_out, const typename CV::F* __restrict__ pre,
                                                        const typename CV::F* __restrict__ accs, Affine<typename CV::F>* __restrict__ out) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  msm_pairtree_backward<CV, FIRST>(t, B, gridDim.x * blockDim.x, total, in, entries, offs_in, offs_out, pre, accs, out);
}

// forward pass with the x coordinates of the next output staged by cp.async; dynamic shared memory: blockDim.x * 4 * sizeof(F)
template <class CV, bool FIRST>
__global__ void __launch_bounds__(128, 5) k_pt_forward_staged(uint32_t B, uint32_t total, const Affine<typename CV::F>* __restrict__ in,
                                                              const uint32_t* __restrict__ entries, const uint32_t* __restrict__ offs_in,
                                                              const uint32_t* __restrict__ offs_out, typename CV::F* __restrict__ pre,
                                                              typename CV::F* __restrict__ accs) {
  extern __shared__ __align__(16) unsigned char pt_smem[];
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  msm_pairtree_forward_staged<CV, FIRST>(t, B, gridDim.x * blockDim.x, total, in, entries, offs_in, offs_out, pre, accs, pt_smem, threadIdx.x);
}
// backward pass with the operands of the next output staged global -> shared by cp.async (msm_affine.cuh); dynamic shared memory:
// blockDim.x * (4 * sizeof(Affine) + sizeof(F))
template <class CV, bool FIRST>
__global__ void __launch_bounds__(128, 4) k_pt_backward_staged(uint32_t B, uint32_t total, const Affine<typename CV::F>* __restrict__ in,
                                                               const uint32_t* __restrict__ entries, const uint32_t* __restrict__ offs_in,
                                                               const uint32_t* __restrict__ offs_out, const typename CV::F* __restrict__ pre,
                                                               const typename CV::F* __restrict__ accs, Affine<typename CV::F>* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char pt_smem[];
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  msm_pairtree_backward_staged<CV, FIRST>(t, B, gridDim.x * blockDim.x, total, in, entries, offs_in, offs_out, pre, accs, out, pt_smem, threadIdx.x);
}

// buckets cut by slice boundaries: add their partials (<= 64 serially, larger ones go to a work list)
template <class CV>
__global__ void __launch_bounds__(128) k_msm_fixup(uint32_t total, uint32_t L, const uint32_t* __restrict__ offs,
                                                   Xyzz<typename CV::F>* __restrict__ buckets,
                                                   const Xyzz<typename CV::F>* __restrict__ spart,
                                                   uint32_t* __restrict__ big_count, uint32_t* __restrict__ big_list) {
  uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= total) return;
  if (msm_fixup_bucket<CV, 64>(g, L, offs, buckets, spart)) big_list[atomicAdd(big_count, 1u)] = g;
}

// heavily populated buckets (skewed scalars): one block per listed bucket, strided sums + smem tree
template <class CV>
__global__ void __launch_bounds__(128) k_msm_fixup_big(uint32_t L, const uint32_t* __restrict__ offs,
                                                       Xyzz<typename CV::F>* __restrict__ buckets,
                                                       const Xyzz<typename CV::F>* __restrict__ spart,
                                                       const uint32_t* __restrict__ big_count,
                                                       const uint32_t* __restrict__ big_list) {
  using X = Xyzz<typename CV::F>;
  __shared__ X sm[128];
  const int tid = threadIdx.x;
  const uint32_t nbig = *big_count;
  for (uint32_t k = blockIdx.x; k < nbig; k += gridDim.x) {
    uint32_t g = big_list[k];
    uint32_t s = offs[g], t = offs[g + 1];
    uint32_t j0 = s / L, j1 = (t - 1) / L;
    X acc;
    xyzz_set_inf(acc);
    for (uint32_t j = j0 + tid; j <= j1; j += 128) {
      X p = spart[2 * (size_t)j + (j == j0 ? 1 : 0)];
      xyzz_add(acc, acc, p);
    }
    sm[tid] = acc;
    __syncthreads();
    for (int h = 64; h > 0; h >>= 1) {
      if (tid < h) {
        X a = sm[tid], b = sm[tid + h];
        xyzz_add(a, a, b);
        sm[tid] = a;
      }
      __syncthreads();
    }
    if (tid == 0) buckets[g] = sm[0];
    __syncthreads();
  }
}

// ---- grouped variants: the windows are processed in G groups (top group first) so that the bucket
// reduction of one group (second stream) overlaps the accumulate pass of the next (main stream) -------------
// ranges[g] = first slice of group g (the slice holding the first sorted entry of its lowest window),
// ranges[G] = number of slices.  A slice shared by two groups belongs to the upper one, which runs first.
static __global__ void k_msm_group_ranges(int G, int W, int nb, uint32_t L, uint32_t total,
                                          const uint32_t* __restrict__ offs, uint32_t* __restrict__ ranges) {
  if (threadIdx.x || blockIdx.x) return;
  for (int g = 0; g < G; g++) ranges[g] = offs[(size_t)(g * W / G) * nb] / L;
  ranges[G] = (offs[total] + L - 1) / L;
}

template <class CV>
__global__ void __launch_bounds__(128) k_msm_accumulate_slices_range(const uint32_t* __restrict__ ranges, int g, uint32_t L,
                                                                     uint32_t total,
                                                                     const Affine<typename CV::F>* __restrict__ pts,
                                                                     const uint32_t* __restrict__ offs,
                                                                     const uint32_t* __restrict__ entries,
                                                                     Xyzz<typename CV::F>* __restrict__ buckets,
                                                                     Xyzz<typename CV::F>* __restrict__ spart) {
  uint32_t j = ranges[g] + blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= ranges[g + 1]) return;
  msm_accumulate_slice<CV>(j, L, total, pts, offs, entries, buckets, spart);
}

template <class CV>
__global__ void __launch_bounds__(128) k_msm_fixup_range(uint32_t gid_lo, uint32_t gid_hi, uint32_t L,
                                                         const uint32_t* __restrict__ offs,
                                                         Xyzz<typename CV::F>* __restrict__ buckets,
                                                         const Xyzz<typename CV::F>* __restrict__ spart,
                                                         uint32_t* __restrict__ big_count, uint32_t* __restrict__ big_list) {
  uint32_t g = gid_lo + blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= gid_hi) return;
  if (msm_fixup_bucket<CV, 64>(g, L, offs, buckets, spart)) big_list[atomicAdd(big_count, 1u)] = g;
}

template <class CV>
__global__ void __launch_bounds__(128) k_msm_reduce_chunks_range(MsmPlan pl, int w_lo, int w_cnt,
                                                                 const Xyzz<typename CV::F>* __restrict__ buckets,
                                                                 Xyzz<typename CV::F>* __restrict__ partials) {
  int T = pl.nb / pl.m;
  size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (size_t)w_cnt * T) return;
  int w = w_lo + (int)(id / T), t = (int)(id % T);
  Xyzz<typename CV::F> out;
  msm_reduce_chunk<CV>(out, buckets + (size_t)w * pl.nb, t, pl.m);
  partials[(size_t)w * T + t] = out;
}

// ---- MSM stage 5: per-chunk running sums ---------------------------------------------------------
template <class CV>
__global__ void __launch_bounds__(128) k_msm_reduce_chunks(MsmPlan pl, const Xyzz<typename CV::F>* __restrict__ buckets,
                                                           Xyzz<typename CV::F>* __restrict__ partials) {
  int T = pl.nb / pl.m;
  size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (size_t)pl.W * T) return;
  int w = (int)(id / T), t = (int)(id % T);
  Xyzz<typename CV::F> out;
  msm_reduce_chunk<CV>(out, buckets + (size_t)w * pl.nb, t, pl.m);
  partials[id] = out;
}

// bucket exchange: chunk reduction of w_cnt windows whose buckets are the sum of `parts` received partial arrays,
// recv layout [part][w_cnt][nb] (what ncclAllToAll leaves on the rank owning these windows)
template <class CV>
__global__ void __launch_bounds__(128) k_msm_reduce_chunks_parts(int nb, int m, int w_cnt, int parts,
                                                                 const Xyzz<typename CV::F>* __restrict__ recv,
                                                                 Xyzz<typename CV::F>* __restrict__ partials) {
  int T = nb / m;
  size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (size_t)w_cnt * T) return;
  int w = (int)(id / T), t = (int)(id % T);
  Xyzz<typename CV::F> out;
  msm_reduce_chunk_parts<CV>(out, recv + (size_t)w * nb, parts, (size_t)w_cnt * nb, t, m);
  partials[id] = out;
}

// ---- two-level bucket reduction (msm.cuh: msm_reduce_l1 / msm_reduce_l2) ---------------------------------------------------
// partials layout per window: [T1 = nb/m1 level-1 sums][T2 = T1/m2 level-2 sums], TP = T1 + T2; runs: [w_cnt][T1]
template <class CV>
__global__ void __launch_bounds__(128) k_msm_reduce_l1(int nb, int m1, int m2, int w_cnt, int parts,
                                                       const Xyzz<typename CV::F>* __restrict__ buckets,
                                                       Xyzz<typename CV::F>* __restrict__ partials,
                                                       Xyzz<typename CV::F>* __restrict__ runs) {
  const int T1 = nb / m1, TP = T1 + T1 / m2;
  size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (size_t)w_cnt * T1) return;
  int w = (int)(id / T1), t = (int)(id % T1);
  Xyzz<typename CV::F> acc, run;
  msm_reduce_l1<CV>(acc, run, buckets + (size_t)w * nb, parts, (size_t)w_cnt * nb, t, m1);
  partials[(size_t)w * TP + t] = acc;
  runs[id] = run;
}
template <class CV>
__global__ void __launch_bounds__(128) k_msm_reduce_l2(int nb, int m1, int m2, int log2_m1, int w_cnt,
                                                       const Xyzz<typename CV::F>* __restrict__ runs,
                                                       Xyzz<typename CV::F>* __restrict__ partials) {
  const int T1 = nb / m1, T2 = T1 / m2, TP = T1 + T2;
  size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (size_t)w_cnt * T2) return;
  int w = (int)(id / T2), u = (int)(id % T2);
  Xyzz<typename CV::F> out;
  msm_reduce_l2<CV>(out, runs + (size_t)w * T1, u, m2, log2_m1);
  partials[(size_t)w * TP + T1 + u] = out;
}

// ---- MSM stage 6: per-window sum of the partials (one block per window) --------------------------
template <class CV>
__global__ void __launch_bounds__(128) k_msm_window_sum(int T, const Xyzz<typename CV::F>* __restrict__ partials,
                                                        Xyzz<typename CV::F>* __restrict__ wsum, int w_lo = 0) {
  using X = Xyzz<typename CV::F>;
  __shared__ X sm[128];
  int tid = threadIdx.x, w = w_lo + blockIdx.x;
  X acc;
  xyzz_set_inf(acc);
  for (int t = tid; t < T; t += 128) {
    X p = partials[(size_t)w * T + t];
    xyzz_add(acc, acc, p);
  }
  sm[tid] = acc;
  __syncthreads();
  for (int s = 64; s > 0; s >>= 1) {
    if (tid < s) {
      X a = sm[tid], b = sm[tid + s];
      xyzz_add(a, a, b);
      sm[tid] = a;
    }
    __syncthreads();
  }
  if (tid == 0) wsum[w] = sm[0];
}

// single-thread inversions of the serial tail use the binary extended Euclid (fp_inv.cuh)
template <class C> B2K_D void f_inv_vt(Fp<C>& r, const Fp<C>& a) { fp_inv_vartime(r, a); }
template <class C> B2K_D void f_inv_vt(Fp2<C>& r, const Fp2<C>& a) {
  Fp<C> n, t;
  fp_sqr_c(n, a.c0); fp_sqr_c(t, a.c1); fp_add(n, n, t);
  fp_inv_vartime(n, n);
  fp_mul_c(r.c0, a.c0, n); fp_mul_c(t, a.c1, n); fp_neg(r.c1, t);
}
template <class F>
B2K_D void xyzz_to_affine_vt(Affine<F>& r, const Xyzz<F>& p) {
  if (xyzz_is_inf(p)) { aff_set_inf(r); return; }
  F t, ti, a;
  f_mul(t, p.ZZ, p.ZZZ);
  f_inv_vt(ti, t);
  f_mul(a, ti, p.ZZZ); f_mul(r.x, p.X, a);      // X / ZZ
  f_mul(a, ti, p.ZZ);  f_mul(r.y, p.Y, a);      // Y / ZZZ
}

// ---- MSM stage 7: Horner over windows, affine, wire bytes ------------------------------------------
// The 240 doublings of the Horner recombination are a serial chain; a lone thread needs ~1.2 us per
// field multiplication.  Four warps (one active lane each, so that they issue on different SM
// sub-partitions) split the independent multiplications of every XYZZ doubling into 3 stages.
template <class CV>
__global__ void __launch_bounds__(128) k_msm_final(MsmPlan pl, const Xyzz<typename CV::F>* __restrict__ wsum,
                                                   uint8_t* __restrict__ out, int affine_out) {
  using F = typename CV::F;
  __shared__ Xyzz<F> acc;
  __shared__ F U, V, Wt, S, M, T, MM, Yt;
  const int warp = threadIdx.x >> 5;
  const bool lead = (threadIdx.x & 31) == 0;
  if (threadIdx.x == 0) acc = wsum[pl.W - 1];
  __syncthreads();
  for (int w = pl.W - 2; w >= 0; w--) {
    for (int i = 0; i < pl.c; i++) {
      const bool inf = xyzz_is_inf(acc);     // same value in every thread
      if (!inf) {
        if (lead) {                          // stage 1:  V = (2Y)^2   |  M = 3 X^2
          if (warp == 0) { f_dbl(U, acc.Y); f_sqr(V, U); }
          else if (warp == 1) { F t; f_sqr(t, acc.X); f_dbl(M, t); f_add(M, M, t); }
        }
        __syncthreads();
        if (lead) {                          // stage 2:  W = U V | S = X V | ZZ *= V | MM = M^2
          if (warp == 0) f_mul(Wt, U, V);
          else if (warp == 1) f_mul(S, acc.X, V);
          else if (warp == 2) { F t; f_mul(t, V, acc.ZZ); acc.ZZ = t; }
          else f_sqr(MM, M);
        }
        __syncthreads();
        if (lead) {                          // stage 3:  T = W Y | ZZZ *= W | X3, M (S - X3)
          if (warp == 0) f_mul(T, Wt, acc.Y);
          else if (warp == 1) { F t; f_mul(t, Wt, acc.ZZZ); acc.ZZZ = t; }
          else if (warp == 2) {
            F x3, t;
            f_sub(x3, MM, S); f_sub(x3, x3, S);
            f_sub(t, S, x3); f_mul(t, M, t);
            acc.X = x3; Yt = t;
          }
        }
        __syncthreads();
        if (threadIdx.x == 0) f_sub(acc.Y, Yt, T);
        __syncthreads();
      }
    }
    if (threadIdx.x == 0) {
      Xyzz<F> t = wsum[w], a = acc;
      xyzz_add(a, a, t);
      acc = a;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    Xyzz<F> r = acc;
    Affine<F> a;
    xyzz_to_affine_vt(a, r);
    if (affine_out) CV::store_affine(out, a);
    else CV::store(out, a);
  }
}

}  // namespace b2k
