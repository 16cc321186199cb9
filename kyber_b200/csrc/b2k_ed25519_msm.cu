// b2k_ed25519_msm.cu -- edwards25519 Pippenger MSM and the share/poly entry points on it (ed_msm.cuh):
//   b2k_ed25519_msm / _dev         sum_i k_i P_i with Point.Mul's scalar reading       (share/poly.go:461-473, the Mul + Add loops)
//   b2k_ed25519_recover_commit     share.RecoverCommit, share/poly.go:449-476 (pvss.RecoverSecret pvss.go:322, DKG resharing dkg.go:965)
//   b2k_ed25519_pubpoly_eval       share.PubPoly.Eval, share/poly.go:340-357
//   b2k_ed25519_pubpoly_check      share.PubPoly.Check, share/poly.go:405-409, per deal in vss.go:636-645 and dkg.go:489-494, 826-834
#include "msm_host.cuh"
#include "ed_msm.cuh"
#include "lagrange.cuh"
using namespace b2k_host;

namespace b2k {

// ---- MSM kernels --------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_ed_msm_load(size_t n, const uint8_t* __restrict__ scalars, const uint8_t* __restrict__ wire,
                                                     EdNiels* __restrict__ pts, MsmPlan pl, int16_t* __restrict__ digits,
                                                     uint32_t* __restrict__ counts, uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (!ed_msm_load(n, i, scalars, wire, pts, pl, digits, counts)) atomicOr(flags, FLAG_POINT);
}

__global__ void __launch_bounds__(128) k_ed_msm_slices(uint32_t nslices, uint32_t L, uint32_t total, const EdNiels* __restrict__ pts,
                                                       const uint32_t* __restrict__ offs, const uint32_t* __restrict__ entries,
                                                       EdExt* __restrict__ buckets, EdExt* __restrict__ spart) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nslices) return;
  ed_accumulate_slice(j, L, total, pts, offs, entries, buckets, spart);
}

__global__ void __launch_bounds__(128) k_ed_msm_fixup(uint32_t total, uint32_t L, const uint32_t* __restrict__ offs,
                                                      EdExt* __restrict__ buckets, const EdExt* __restrict__ spart,
                                                      uint32_t* __restrict__ big_count, uint32_t* __restrict__ big_list) {
  uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= total) return;
  if (ed_fixup_bucket<64>(g, L, offs, buckets, spart)) big_list[atomicAdd(big_count, 1u)] = g;
}

// buckets with more than 64 partials (skewed scalars): one block per listed bucket, strided sums and a shared-memory tree
__global__ void __launch_bounds__(128) k_ed_msm_fixup_big(uint32_t L, const uint32_t* __restrict__ offs, EdExt* __restrict__ buckets,
                                                          const EdExt* __restrict__ spart, const uint32_t* __restrict__ big_count,
                                                          const uint32_t* __restrict__ big_list) {
  __shared__ EdExt sm[128];
  const int tid = threadIdx.x;
  const uint32_t nbig = *big_count;
  for (uint32_t k = blockIdx.x; k < nbig; k += gridDim.x) {
    const uint32_t g = big_list[k];
    const uint32_t s = offs[g], t = offs[g + 1];
    EdExt acc;
    ed_fixup_strided(acc, tid, 128, s / L, (t - 1) / L, spart);
    sm[tid] = acc;
    __syncthreads();
    for (int h = 64; h > 0; h >>= 1) {
      if (tid < h) {
        EdExt a = sm[tid], b = sm[tid + h];
        ed_add(a, a, b);
        sm[tid] = a;
      }
      __syncthreads();
    }
    if (tid == 0) buckets[g] = sm[0];
    __syncthreads();
  }
}

__global__ void __launch_bounds__(128) k_ed_msm_reduce_chunks(MsmPlan pl, const EdExt* __restrict__ buckets, EdExt* __restrict__ partials) {
  const int T = pl.nb / pl.m;
  size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (size_t)pl.W * T) return;
  const int w = (int)(id / T), t = (int)(id % T);
  EdExt out;
  ed_reduce_chunk(out, buckets + (size_t)w * pl.nb, t, pl.m);
  partials[id] = out;
}

// one block per window: wsum[w] = sum of the window's T chunk partials
__global__ void __launch_bounds__(128) k_ed_msm_window_sum(int T, const EdExt* __restrict__ partials, EdExt* __restrict__ wsum) {
  __shared__ EdExt sm[128];
  const int tid = threadIdx.x, w = blockIdx.x;
  EdExt acc;
  ed_set_identity(acc);
  for (int t = tid; t < T; t += 128) {
    const EdExt p = partials[(size_t)w * T + t];
    ed_add(acc, acc, p);
  }
  sm[tid] = acc;
  __syncthreads();
  for (int h = 64; h > 0; h >>= 1) {
    if (tid < h) {
      EdExt a = sm[tid], b = sm[tid + h];
      ed_add(a, a, b);
      sm[tid] = a;
    }
    __syncthreads();
  }
  if (tid == 0) wsum[w] = sm[0];
}

// Horner over the windows and the encoding, one thread
__global__ void k_ed_msm_final(MsmPlan pl, const EdExt* __restrict__ wsum, uint8_t* __restrict__ out) {
  if (threadIdx.x || blockIdx.x) return;
  EdExt r;
  ed_msm_horner(r, wsum, pl.W, pl.c);
  ed_encode(out, r);
}

// ---- share/poly kernels ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_ed_load_niels(size_t n, const uint8_t* __restrict__ wire, EdNiels* __restrict__ out, uint32_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  EdNiels q;
  if (!ed_load_niels(q, wire + 32 * i)) atomicOr(flags, FLAG_POINT);
  out[i] = q;
}

// out[i] = encode(sum_j (idx_i + 1)^j C_j)
__global__ void __launch_bounds__(128) k_ed_pubpoly_eval(uint32_t t, const EdNiels* __restrict__ commits, uint32_t n,
                                                         const uint32_t* __restrict__ idx, uint8_t* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  EdExt v;
  ed_pubpoly_horner(v, commits, t, (uint64_t)idx[i] + 1u);
  ed_encode(out + 32 * (size_t)i, v);
}

// ok[d n + k] = PubPoly.Check of dealer d's share k; 1..8 B staged in shared memory as in k_ed25519_verify
__global__ void __launch_bounds__(128) k_ed_pubpoly_check(uint32_t m, uint32_t t, const EdNiels* __restrict__ commits, uint32_t n,
                                                          const uint32_t* __restrict__ idx, const uint8_t* __restrict__ shares,
                                                          uint8_t* __restrict__ ok) {
  __shared__ EdNiels btab[8];
  if (threadIdx.x == 0) ed_load_base_table(btab);
  __syncthreads();
  size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (size_t)m * n) return;
  const uint32_t d = (uint32_t)(id / n);
  ok[id] = ed_pubpoly_check_one(commits + (size_t)d * t, t, idx[id], shares + 32 * id, btab) ? 1 : 0;
}

}  // namespace b2k

namespace {

constexpr int ED_SCALAR_BITS = 256;      // Point.Mul reads the whole 256-bit integer (no reduction mod l)

// one edwards25519 MSM call: plan, sizes and scratch (the Edwards counterpart of MsmLayout)
struct EdMsmLayout {
  MsmPlan pl;
  size_t n = 0, total = 0;
  uint32_t L = 0, smax = 0;
  EdNiels* pts = nullptr;
  int16_t* digits = nullptr;
  uint32_t *counts = nullptr, *offs = nullptr, *cursor = nullptr;
  SortRec* recs = nullptr;
  uint32_t* entries = nullptr;
  EdExt* buckets = nullptr;
  EdExt* spart = nullptr;        // slice partials, two per slice
  uint32_t* big_list = nullptr;  // buckets for the block-parallel fix-up, and their count
  uint32_t* big_count = nullptr;
  uint32_t* bsum = nullptr;      // block sums of the scan
  EdExt* partials = nullptr;     // chunk partials, W x (nb / m)
  EdExt* wsum = nullptr;

  void carve(Carve& c) {
    pts = c.take<EdNiels>(n);
    digits = c.take<int16_t>(n * (size_t)pl.W);
    counts = c.take<uint32_t>(total + 1);
    offs = c.take<uint32_t>(total + 1);
    cursor = c.take<uint32_t>(total + 1);
    recs = c.take<SortRec>(n * (size_t)pl.W);
    entries = c.take<uint32_t>(n * (size_t)pl.W);
    buckets = c.take<EdExt>(total);
    spart = c.take<EdExt>(2 * (size_t)smax);
    big_list = c.take<uint32_t>(total + 1);
    big_count = c.take<uint32_t>(1);
    bsum = c.take<uint32_t>(1024);
    partials = c.take<EdExt>((size_t)pl.W * (pl.nb / pl.m));
    wsum = c.take<EdExt>(pl.W);
  }
};

// the prologue of every edwards25519 MSM entry point (msm_begin's checks with the Edwards layout)
template <class Stage>
int ed_msm_begin(b2k_ctx* ctx, size_t n, bool args_ok, EdMsmLayout& s, Stage&& stage) {
  if (!ctx || !args_ok || n == 0 || n >= (size_t(1) << 31)) {
    if (ctx) ctx->err = "bad argument";
    return B2K_ERR_ARG;
  }
  CK(cudaSetDevice(ctx->device));
  s = EdMsmLayout{};
  s.pl = make_plan(n, ctx->force_c, ED_SCALAR_BITS, ctx->force_m);
  s.n = n;
  s.total = (size_t)s.pl.W * s.pl.nb;
  s.L = slice_len(n, s.pl, ctx->force_L);
  s.smax = (uint32_t)((n * (size_t)s.pl.W + s.L - 1) / s.L) + 1;
  if ((unsigned long long)n * (unsigned long long)s.pl.W >= (1ull << 32)) {
    ctx->err = "MSM too large for one call: pairs x windows must stay below 2^32 (split the batch)";
    return B2K_ERR_ARG;
  }
  if (s.total > 1024u * 1024u || (s.pl.nb >> sort_shift(s.pl.c)) > PART_BPW) { ctx->err = "too many buckets"; return B2K_ERR_ARG; }
  return arena_carve(ctx, [&](Carve& c) {
    stage(c);
    s.carve(c);
  });
}

// Enqueue the whole MSM on ctx->stream into the scratch ed_msm_begin carved; device pointers.  The stage events keep the
// meaning b2k_last_timings documents: [0] load (decoding included, the digits come out of it: [1] = 0), [2] scan, [3] sort,
// [4] slices, [9] fix-up, [5] chunk reduction, [6] window sums, [7] Horner and encoding; no affine rounds ([10] = 0).
int ed_msm_enqueue(b2k_ctx* ctx, const EdMsmLayout& s, const uint8_t* d_scalars, const uint8_t* d_points, uint8_t* d_out) {
  cudaStream_t st = ctx->stream;
  const MsmPlan& pl = s.pl;
  const size_t n = s.n, total = s.total;
  int* lp = ctx->last_plan;
  for (int i = 0; i < LP_SLOTS; i++) lp[i] = 0;
  lp[LP_C] = pl.c; lp[LP_W] = pl.W; lp[LP_NB] = pl.nb; lp[LP_M] = pl.m;
  lp[LP_SLICE] = (int)s.L;
  lp[LP_LEVELS] = 1; lp[LP_M1] = pl.m;
  const unsigned sblocks = (unsigned)((total + 1023) / 1024);
  CK(cudaEventRecord(ctx->ev[0], st));
  CK(cudaMemsetAsync(s.counts, 0, (total + 1) * 4, st));
  k_ed_msm_load<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, d_scalars, d_points, s.pts, pl, s.digits, s.counts, ctx->d_flags);
  CK(cudaEventRecord(ctx->ev[1], st));
  CK(cudaEventRecord(ctx->ev[2], st));
  k_scan_blocks<<<sblocks, 1024, 0, st>>>((uint32_t)total, s.counts, s.offs, nullptr, s.bsum);
  k_scan_tops<<<1, 1024, 0, st>>>(sblocks, (uint32_t)total, s.bsum, s.offs, nullptr);
  k_scan_finish<<<sblocks, 1024, 0, st>>>((uint32_t)total, s.bsum, s.offs, nullptr, s.cursor);
  CK(cudaEventRecord(ctx->ev[3], st));
  const int S = sort_shift(pl.c);
  const size_t nrec = n * (size_t)pl.W;
  k_msm_partition<<<(unsigned)((n + PART_TILE - 1) / PART_TILE), PART_T, 0, st>>>((uint32_t)n, pl, S, s.digits, s.cursor, s.recs);
  k_msm_bin_sort<<<(unsigned)((nrec + BSORT_TILE - 1) / BSORT_TILE), BSORT_T, 0, st>>>((uint32_t)total, S, s.recs, s.offs, s.counts, s.entries);
  CK(cudaMemsetAsync(s.big_count, 0, 4, st));
  CK(cudaEventRecord(ctx->ev[4], st));
  CK(cudaEventRecord(ctx->ev[10], st));
  k_ed_msm_slices<<<(s.smax + 127) / 128, 128, 0, st>>>(s.smax, s.L, (uint32_t)total, s.pts, s.offs, s.entries, s.buckets, s.spart);
  CK(cudaEventRecord(ctx->ev[9], st));
  k_ed_msm_fixup<<<(unsigned)((total + 127) / 128), 128, 0, st>>>((uint32_t)total, s.L, s.offs, s.buckets, s.spart, s.big_count, s.big_list);
  k_ed_msm_fixup_big<<<256, 128, 0, st>>>(s.L, s.offs, s.buckets, s.spart, s.big_count, s.big_list);
  CK(cudaEventRecord(ctx->ev[5], st));
  const int T = pl.nb / pl.m;
  k_ed_msm_reduce_chunks<<<(unsigned)(((size_t)pl.W * T + 127) / 128), 128, 0, st>>>(pl, s.buckets, s.partials);
  CK(cudaEventRecord(ctx->ev[6], st));
  k_ed_msm_window_sum<<<pl.W, 128, 0, st>>>(T, s.partials, s.wsum);
  CK(cudaEventRecord(ctx->ev[7], st));
  k_ed_msm_final<<<1, 32, 0, st>>>(pl, s.wsum, d_out);
  CK(cudaEventRecord(ctx->ev[8], st));
  ctx->launches += 12;                  // load, three scan passes, partition, bin sort, slices, two fix-ups, chunks, window sums, final
  CK(cudaGetLastError());
  ctx->timings_valid = true;
  return B2K_OK;
}

int ed_msm_host(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out) {
  EdMsmLayout s;
  uint8_t *d_s = nullptr, *d_p = nullptr, *d_o = nullptr;
  int rc = ed_msm_begin(ctx, n, scalars && points && out, s, [&](Carve& c) {
    d_s = c.take<uint8_t>(n * 32);
    d_p = c.take<uint8_t>(n * 32);
    d_o = c.take<uint8_t>(256);
  });
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  if ((rc = status_begin(ctx))) return rc;
  CK(cudaMemcpyAsync(d_s, scalars, n * 32, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_p, points, n * 32, cudaMemcpyHostToDevice, st));
  if ((rc = ed_msm_enqueue(ctx, s, d_s, d_p, d_o))) return rc;
  CK(cudaMemcpyAsync(out, d_o, 32, cudaMemcpyDeviceToHost, st));
  return status_finish(ctx);
}

int ed_recover_commit(b2k_ctx* ctx, size_t t, const uint32_t* indices, const uint8_t* points, uint8_t* out) {
  EdMsmLayout s;
  uint32_t* d_idx = nullptr;
  uint8_t *d_s = nullptr, *d_p = nullptr, *d_o = nullptr;
  int rc = ed_msm_begin(ctx, t, indices && points && out, s, [&](Carve& c) {
    d_idx = c.take<uint32_t>(t);
    d_s = c.take<uint8_t>(t * 32);
    d_p = c.take<uint8_t>(t * 32);
    d_o = c.take<uint8_t>(256);
  });
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  if ((rc = status_begin(ctx))) return rc;
  CK(cudaMemcpyAsync(d_idx, indices, t * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_p, points, t * 32, cudaMemcpyHostToDevice, st));
  k_lagrange_at_zero<Ed25519Fr, true><<<(unsigned)((t + 127) / 128), 128, 0, st>>>((uint32_t)t, d_idx, d_s, ctx->d_flags);
  ctx->launches += 1;
  if ((rc = ed_msm_enqueue(ctx, s, d_s, d_p, d_o))) return rc;
  CK(cudaMemcpyAsync(out, d_o, 32, cudaMemcpyDeviceToHost, st));
  return status_finish(ctx);
}

int ed_pubpoly_eval(b2k_ctx* ctx, size_t t, const uint8_t* commits, size_t n, const uint32_t* indices, uint8_t* out) {
  if (!ctx || !commits || !indices || !out || t == 0 || n == 0 || t >= (size_t(1) << 31) || n >= (size_t(1) << 31))
    return bad_arg(ctx, "bad argument");
  CK(cudaSetDevice(ctx->device));
  uint8_t *d_c = nullptr, *d_o = nullptr;
  EdNiels* d_cm = nullptr;
  uint32_t* d_idx = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_c = c.in(commits, t, 32);
    d_idx = c.in(indices, n);
    d_cm = c.take<EdNiels>(t);
    d_o = c.out(out, n, 32);
  }, [&]() -> int {
    cudaStream_t st = ctx->stream;
    k_ed_load_niels<<<(unsigned)((t + 255) / 256), 256, 0, st>>>(t, d_c, d_cm, ctx->d_flags);
    k_ed_pubpoly_eval<<<(unsigned)((n + 127) / 128), 128, 0, st>>>((uint32_t)t, d_cm, (uint32_t)n, d_idx, d_o);
    CK(cudaGetLastError());
    ctx->launches += 2;
    return B2K_OK;
  });
}

int ed_pubpoly_check(b2k_ctx* ctx, size_t m, size_t t, const uint8_t* commits, size_t n, const uint32_t* indices,
                     const uint8_t* shares, uint8_t* ok) {
  if (!ctx || !commits || !indices || !shares || !ok || m == 0 || t == 0 || n == 0 || m * t >= (size_t(1) << 31) ||
      m * n >= (size_t(1) << 31))
    return bad_arg(ctx, "bad argument");
  CK(cudaSetDevice(ctx->device));
  const size_t mt = m * t, mn = m * n;
  uint8_t *d_c = nullptr, *d_s = nullptr, *d_ok = nullptr;
  EdNiels* d_cm = nullptr;
  uint32_t* d_idx = nullptr;
  return host_call(ctx, [&](Carve& c) {
    d_c = c.in(commits, mt, 32);
    d_idx = c.in(indices, mn);
    d_s = c.in(shares, mn, 32);
    d_cm = c.take<EdNiels>(mt);
    d_ok = c.out(ok, mn);
  }, [&]() -> int {
    cudaStream_t st = ctx->stream;
    k_ed_load_niels<<<(unsigned)((mt + 255) / 256), 256, 0, st>>>(mt, d_c, d_cm, ctx->d_flags);
    k_ed_pubpoly_check<<<(unsigned)((mn + 127) / 128), 128, 0, st>>>((uint32_t)m, (uint32_t)t, d_cm, (uint32_t)n, d_idx, d_s, d_ok);
    CK(cudaGetLastError());
    ctx->launches += 2;
    return B2K_OK;
  });
}

}  // namespace

extern "C" {

int b2k_ed25519_msm(b2k_ctx* ctx, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out) {
  return ed_msm_host(ctx, n, scalars, points, out);
}
int b2k_ed25519_msm_dev(b2k_ctx* ctx, size_t n, const void* d_scalars, const void* d_points, void* d_out) {
  EdMsmLayout s;
  int rc = ed_msm_begin(ctx, n, d_scalars && d_points && d_out, s, [](Carve&) {});
  if (rc) return rc;
  return ed_msm_enqueue(ctx, s, (const uint8_t*)d_scalars, (const uint8_t*)d_points, (uint8_t*)d_out);
}
int b2k_ed25519_recover_commit(b2k_ctx* ctx, size_t t, const uint32_t* indices, const uint8_t* points, uint8_t* out) {
  return ed_recover_commit(ctx, t, indices, points, out);
}
int b2k_ed25519_pubpoly_eval(b2k_ctx* ctx, size_t t, const uint8_t* commits, size_t n, const uint32_t* indices, uint8_t* out) {
  return ed_pubpoly_eval(ctx, t, commits, n, indices, out);
}
int b2k_ed25519_pubpoly_check(b2k_ctx* ctx, size_t m, size_t t, const uint8_t* commits, size_t n, const uint32_t* indices,
                              const uint8_t* shares, uint8_t* ok) {
  return ed_pubpoly_check(ctx, m, t, commits, n, indices, shares, ok);
}

}  // extern "C"
