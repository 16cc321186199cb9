// b2k_multi.cu -- the sharded (multi-GPU) BLS12-381 G1 MSM inside the library (SURVEY.md 8b `b2k_msm_multi_gpu`, 8e).
//
// Replaces, for terms that live on several GPUs, the same Mul+Add loops as b2k_bls12381_g1_msm
// (share/poly.go:461-473, sign/bdn/bdn.go:126-161).  The pairs are partitioned by rank; the one exchange step is the
// "all-reduce of partial bucket sums" BASELINE.json names, written as what it is for curve points (NCCL cannot add them):
//
//   every rank   pairs -> W x 2^(c-1) partial buckets in its EXCHANGE SLAB (stable cudaMalloc, mapped by every peer:
//                cudaDeviceEnablePeerAccess inside one process, CUDA IPC across processes)
//   signal       release-store of the step number into every peer's flag word          (k_comm_signal)
//   wait         spin on the own flag words until every peer has published this step   (k_comm_wait)
//   ONE kernel   rank g pulls windows [g W/G, (g+1) W/G) of EVERY rank straight out of the peers' slabs over NVLink
//                (plain loads through the mapped pointers) and fuses the G-way bucket-wise EC addition into the
//                running-sum reduction of those windows                                 (k_msm_reduce_l1_peers)
//   push         the w_cnt window sums go to every peer's slab + signal; Horner over all W windows on every rank.
//
// No NCCL kernel has to become co-resident with the product kernels of the other steps in flight, and the transfer
// overlaps the arithmetic load by load.  The same slabs also carry the cheap shape 2 (each rank finishes its own MSM,
// 96-byte results are pushed, every rank adds them).  An NCCL transport of the same exchange (grouped ncclSend/ncclRecv =
// all-to-all, then ncclAllGather; libnccl.so.2 resolved at run time) is kept beside it for A/B measurements and for
// ranks that cannot map each other's memory.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <unistd.h>
#include <cstdio>
#include <cstring>
#include <new>
#include <string>

#include "../../include/b2kyber.h"
#include "msm_host.cuh"

using namespace b2k;
using namespace b2k_host;

namespace {

using CV = Bls381G1;
using X = Xyzz<CV::F>;
constexpr int MAXR = B2K_MAX_RANKS;

// slab layout (identical on every rank, so peers address each other's regions by offset)
constexpr size_t SLAB_BUCKETS = (size_t)16 * 32768 * sizeof(X);          // up to W = 16 windows of 2^15 buckets (c = 16, no split)
constexpr size_t SLAB_WSUM = (size_t)64 * sizeof(X);                      // all W window sums
constexpr size_t SLAB_RES = (size_t)MAXR * 96;                            // shape 2: one operand-form point per rank
constexpr size_t SLAB_FLAGS = 4 * MAXR * sizeof(uint32_t);                // ready / done / wsum-ready / result-ready, one word per peer
constexpr size_t OFF_WSUM = SLAB_BUCKETS;
constexpr size_t OFF_RES = OFF_WSUM + SLAB_WSUM;
constexpr size_t OFF_FLAGS = (OFF_RES + SLAB_RES + 255) & ~size_t(255);
constexpr size_t OFF_ONES = OFF_FLAGS + ((SLAB_FLAGS + 255) & ~size_t(255));   // MAXR unit scalars (shape 2's final sum)
constexpr size_t OFF_OUT = OFF_ONES + MAXR * 32;                               // result bytes of the host-buffer calls
constexpr size_t SLAB_BYTES = OFF_OUT + 256;
enum { F_READY = 0, F_DONE = 1, F_WSUM = 2, F_RES = 3 };

struct Blob {                      // what b2k_comm_export hands to the other ranks (<= B2K_COMM_BLOB_BYTES)
  cudaIpcMemHandle_t handle;
  uint64_t pid;
  uint64_t ptr;                    // valid inside process `pid`
  int32_t rank, device;
  uint64_t bytes;
};
static_assert(sizeof(Blob) <= B2K_COMM_BLOB_BYTES, "blob size");

// ---- NCCL, resolved at run time (no link-time dependency: a process that already loaded torch's libnccl.so.2 gets that one)
struct Id128 { char b[128]; };        // ncclUniqueId (passed by value)
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, Id128, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  int (*Send)(const void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*Recv)(void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
NcclApi g_nccl;
bool nccl_load(std::string& err) {
  if (g_nccl.lib) return true;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) { err = std::string("dlopen libnccl.so.2: ") + dlerror(); return false; }
  auto sym = [&](const char* n) { return dlsym(h, n); };
  g_nccl.GetUniqueId = (int (*)(void*))sym("ncclGetUniqueId");
  g_nccl.CommInitRank = (int (*)(void**, int, Id128, int))sym("ncclCommInitRank");
  g_nccl.CommDestroy = (int (*)(void*))sym("ncclCommDestroy");
  g_nccl.GroupStart = (int (*)())sym("ncclGroupStart");
  g_nccl.GroupEnd = (int (*)())sym("ncclGroupEnd");
  g_nccl.Send = (int (*)(const void*, size_t, int, int, void*, cudaStream_t))sym("ncclSend");
  g_nccl.Recv = (int (*)(void*, size_t, int, int, void*, cudaStream_t))sym("ncclRecv");
  g_nccl.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))sym("ncclAllGather");
  g_nccl.GetErrorString = (const char* (*)(int))sym("ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.CommDestroy || !g_nccl.GroupStart || !g_nccl.GroupEnd || !g_nccl.Send ||
      !g_nccl.Recv || !g_nccl.AllGather) { err = "libnccl.so.2 lacks a required symbol"; return false; }
  g_nccl.lib = h;
  return true;
}
constexpr int NCCL_UINT8 = 1;     // ncclUint8 (nccl.h)

}  // namespace

struct b2k_comm {
  b2k_ctx* ctx = nullptr;
  int nranks = 1, rank = 0;
  char* slab = nullptr;
  char* peer[MAXR] = {};           // every rank's slab as seen from this device (peer[rank] == slab)
  bool ipc_open[MAXR] = {};
  bool connected = false;
  uint32_t step = 0;
  uint8_t* h_out = nullptr;        // page-locked result buffer of b2k_bls12381_g1_msm_multi_gpu (a D2H copy into pageable memory
                                   // would block the enqueueing host thread until the peers arrive -- which it enqueues next)
  void* nccl = nullptr;            // ncclComm_t when the NCCL transport is selected
  char* recv = nullptr;            // NCCL transport: receive buffer of the all-to-all
  int last_plan[4] = {};
};

namespace {

struct PeerPtrs { char* p[MAXR]; };

// thread p < nranks: release-store `value` into flag word [which][rank] of peer p's slab
__global__ void k_comm_signal(PeerPtrs pp, int nranks, int rank, int which, uint32_t value) {
  const int p = threadIdx.x;
  if (p >= nranks) return;
  __threadfence_system();                                   // everything this stream wrote before is visible system-wide first
  uint32_t* f = reinterpret_cast<uint32_t*>(pp.p[p] + OFF_FLAGS) + which * MAXR + rank;
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(f), "r"(value) : "memory");
}

// thread p < nranks: spin until flag word [which][p] of the OWN slab reaches `value` (written by peer p).  A peer that never
// arrives (crashed process, mismatched call sequence) raises FLAG_COMM_TIMEOUT after ~10 s instead of hanging the device.
__global__ void k_comm_wait(char* slab, int nranks, int which, uint32_t value, uint32_t* status) {
  const int p = threadIdx.x;
  if (p >= nranks) return;
  const uint32_t* f = reinterpret_cast<const uint32_t*>(slab + OFF_FLAGS) + which * MAXR + p;
  unsigned long long t0, t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  for (;;) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
    if ((int32_t)(v - value) >= 0) break;
    __nanosleep(200);
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    if (t - t0 > 10000000000ull) { atomicOr(status, FLAG_COMM_TIMEOUT); break; }
  }
}

// level 1 of the bucket reduction (msm.cuh: msm_reduce_l1) for the windows [w_lo, w_lo + w_cnt) this rank owns, every bucket
// being the sum of `parts` partials fetched from the peers' slabs (rotated start: rank g begins with its own slab, then g+1 ...,
// so that the G ranks do not all pull from the same peer at once).  levels == 1: the chunk's offset multiple is added here.
__global__ void __launch_bounds__(128) k_msm_reduce_l1_peers(int nb, int m1, int m2, int levels, int w_lo, int w_cnt, int parts, int rank,
                                                             PeerPtrs pp, X* __restrict__ partials, X* __restrict__ runs) {
  const int T1 = nb / m1, TP = levels == 2 ? T1 + T1 / m2 : T1;
  const size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (size_t)w_cnt * T1) return;
  const int w = (int)(id / T1), t = (int)(id % T1);
  const size_t base = (size_t)(w_lo + w) * nb + (size_t)t * m1;
  X run, acc;
  xyzz_set_inf(run);
  xyzz_set_inf(acc);
  for (int k = m1 - 1; k >= 0; k--) {
    X b = reinterpret_cast<const X*>(pp.p[rank])[base + k];
    for (int i = 1; i < parts; i++) {
      int p = rank + i; if (p >= parts) p -= parts;
      X q = reinterpret_cast<const X*>(pp.p[p])[base + k];
      xyzz_add(b, b, q);
    }
    xyzz_add(run, run, b);
    xyzz_add(acc, acc, run);
  }
  if (levels == 2) {
    runs[id] = run;
  } else if (t != 0) {
    X off;
    xyzz_mul_small(off, run, (uint32_t)(t * m1));
    xyzz_add(acc, acc, off);
  }
  partials[(size_t)w * TP + t] = acc;
}

// copy `words` 32-bit words from src to offset `off` of EVERY peer's slab, then publish `value` in flag [which][rank] of each
__global__ void __launch_bounds__(256) k_comm_push(PeerPtrs pp, int nranks, int rank, size_t off, const uint32_t* __restrict__ src, int words,
                                                   int which, uint32_t value) {
  for (int i = threadIdx.x; i < nranks * words; i += blockDim.x) {
    const int p = i / words, j = i % words;
    reinterpret_cast<uint32_t*>(pp.p[p] + off)[j] = src[j];
  }
  __threadfence_system();
  __syncthreads();
  if ((int)threadIdx.x < nranks) {
    uint32_t* f = reinterpret_cast<uint32_t*>(pp.p[threadIdx.x] + OFF_FLAGS) + which * MAXR + rank;
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(f), "r"(value) : "memory");
  }
}

PeerPtrs peer_ptrs(const b2k_comm* cm) {
  PeerPtrs pp;
  for (int i = 0; i < MAXR; i++) pp.p[i] = i < cm->nranks ? cm->peer[i] : nullptr;
  return pp;
}

#define CKN(call)                                                                                          \
  do {                                                                                                     \
    int r_ = (call);                                                                                       \
    if (r_ != 0) {                                                                                         \
      ctx->err = std::string(#call) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r_) : "NCCL error"); \
      return B2K_ERR_CUDA;                                                                                 \
    }                                                                                                      \
  } while (0)

// windows of this rank reduced from `parts` sources into cm's slab region wsum[w_lo .. w_lo + w_cnt)
int reduce_owned_windows(b2k_comm* cm, int c, int w_lo, int w_cnt, bool from_peers) {
  b2k_ctx* ctx = cm->ctx;
  cudaStream_t st = ctx->stream;
  const int nb = 1 << (c - 1);
  const ReducePlan rp = owned_reduce_plan(ctx, nb, w_cnt);
  TailBufs<X> t;
  X* mine = nullptr;
  int rc = arena_carve(ctx, [&](Carve& cv) {
    t.carve(cv, w_cnt, rp.TP, rp);
    mine = cv.take<X>(w_cnt);
  });
  if (rc) return rc;
  const X* recv = reinterpret_cast<const X*>(cm->recv);   // NCCL transport: recv = [parts][w_cnt][nb]
  rc = reduce_windows<CV>(ctx, nb, w_cnt, rp, t, mine, [&](unsigned grid) {
    if (from_peers)
      k_msm_reduce_l1_peers<<<grid, 128, 0, st>>>(nb, rp.m1, rp.m2, rp.levels, w_lo, w_cnt, cm->nranks, cm->rank, peer_ptrs(cm), t.partials, t.runs);
    else if (rp.levels == 2) k_msm_reduce_l1<CV><<<grid, 128, 0, st>>>(nb, rp.m1, rp.m2, w_cnt, cm->nranks, recv, t.partials, t.runs);
    else k_msm_reduce_chunks_parts<CV><<<grid, 128, 0, st>>>(nb, rp.m1, w_cnt, cm->nranks, recv, t.partials);
  });
  if (rc) return rc;
  CK(cudaGetLastError());
  // the window sums of this rank go to every rank (own slab included)
  if (cm->nccl) {
    CKN(g_nccl.AllGather(mine, cm->slab + OFF_WSUM, (size_t)w_cnt * sizeof(X), NCCL_UINT8, cm->nccl, st));
  } else {
    k_comm_push<<<1, 256, 0, st>>>(peer_ptrs(cm), cm->nranks, cm->rank, OFF_WSUM + (size_t)w_lo * sizeof(X),
                                   reinterpret_cast<const uint32_t*>(mine), (int)(w_cnt * sizeof(X) / 4), F_WSUM, cm->step);
    k_comm_wait<<<1, 32, 0, st>>>(cm->slab, cm->nranks, F_WSUM, cm->step, ctx->d_flags);
    ctx->launches += 2;
  }
  return B2K_OK;
}

// everything after the rank's partial buckets are in its slab (stream-ordered): exchange, owned windows, all window sums, Horner
int exchange_and_finish(b2k_comm* cm, const int* plan, void* d_out) {
  b2k_ctx* ctx = cm->ctx;
  cudaStream_t st = ctx->stream;
  const int c = plan[0], W = plan[1], nb = plan[2];
  if (W % cm->nranks) { ctx->err = "bucket exchange needs the window count to be a multiple of the rank count"; return B2K_ERR_ARG; }
  const int w_cnt = W / cm->nranks, w_lo = cm->rank * w_cnt;
  if (cm->nccl) {
    const size_t chunk = (size_t)w_cnt * nb * sizeof(X);      // windows of rank p are contiguous in the window-major bucket array
    CKN(g_nccl.GroupStart());
    for (int p = 0; p < cm->nranks; p++) {
      CKN(g_nccl.Send(cm->slab + (size_t)p * chunk, chunk, NCCL_UINT8, p, cm->nccl, st));
      CKN(g_nccl.Recv(cm->recv + (size_t)p * chunk, chunk, NCCL_UINT8, p, cm->nccl, st));
    }
    CKN(g_nccl.GroupEnd());
    int rc = reduce_owned_windows(cm, c, w_lo, w_cnt, false);
    if (rc) return rc;
  } else {
    k_comm_signal<<<1, 32, 0, st>>>(peer_ptrs(cm), cm->nranks, cm->rank, F_READY, cm->step);
    k_comm_wait<<<1, 32, 0, st>>>(cm->slab, cm->nranks, F_READY, cm->step, ctx->d_flags);
    ctx->launches += 2;
    int rc = reduce_owned_windows(cm, c, w_lo, w_cnt, true);
    if (rc) return rc;
    // the peers may overwrite their buckets once every reader is done: publish "done reading step s" (k_comm_push already
    // follows the reduction kernels in stream order, a separate flag keeps the two meanings apart)
    k_comm_signal<<<1, 32, 0, st>>>(peer_ptrs(cm), cm->nranks, cm->rank, F_DONE, cm->step);
    ctx->launches += 1;
  }
  CK(cudaGetLastError());
  return b2k_bls12381_g1_msm_finish_dev(ctx, c, W, cm->slab + OFF_WSUM, d_out, 0);
}

int begin_step(b2k_comm* cm) {
  b2k_ctx* ctx = cm->ctx;
  if (!cm->connected) { ctx->err = "communicator not connected (b2k_comm_connect)"; return B2K_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  cm->step++;
  if (!cm->nccl && cm->step > 1) {            // nobody may still be reading the buckets / results of the previous step
    k_comm_wait<<<1, 32, 0, ctx->stream>>>(cm->slab, cm->nranks, F_DONE, cm->step - 1, ctx->d_flags);
    ctx->launches += 1;
  }
  return B2K_OK;
}

int sharded_any(b2k_comm* cm, size_t n, const void* scalars, const void* points, bool host, void* d_out, int shape) {
  if (!cm || !cm->ctx) return B2K_ERR_ARG;
  b2k_ctx* ctx = cm->ctx;
  if (!scalars || !points || !d_out || n == 0 || (shape != 0 && shape != 1)) { ctx->err = "bad argument"; return B2K_ERR_ARG; }
  int rc = begin_step(cm);
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  if (shape == 0) {
    int plan[4];
    rc = host ? b2k_internal_bls12381_g1_msm_buckets_host(ctx, n, (const uint8_t*)scalars, (const uint8_t*)points, cm->slab, SLAB_BUCKETS, plan)
              : b2k_bls12381_g1_msm_buckets_dev(ctx, n, scalars, points, cm->slab, SLAB_BUCKETS, plan);
    if (rc) return rc;
    memcpy(cm->last_plan, plan, sizeof plan);
    return exchange_and_finish(cm, plan, d_out);
  }
  // shape 2: every rank finishes its own MSM (operand form, 96 B), the results travel, every rank adds them
  if (cm->nccl) { ctx->err = "result exchange over NCCL: use the peer transport"; return B2K_ERR_ARG; }
  if (host) { ctx->err = "result exchange takes device buffers"; return B2K_ERR_ARG; }
  uint8_t* mine = reinterpret_cast<uint8_t*>(cm->slab + OFF_OUT) + 128;       // staging for the push (own slab, private region)
  rc = b2k_bls12381_g1_msm_affine_dev(ctx, n, scalars, points, mine);
  if (rc) return rc;
  k_comm_push<<<1, 256, 0, st>>>(peer_ptrs(cm), cm->nranks, cm->rank, OFF_RES + (size_t)cm->rank * 96, reinterpret_cast<const uint32_t*>(mine), 24,
                                 F_RES, cm->step);
  k_comm_wait<<<1, 32, 0, st>>>(cm->slab, cm->nranks, F_RES, cm->step, ctx->d_flags);
  ctx->launches += 2;
  rc = b2k_bls12381_g1_msm_dev(ctx, (size_t)cm->nranks, cm->slab + OFF_ONES, cm->slab + OFF_RES, d_out);
  if (rc) return rc;
  k_comm_signal<<<1, 32, 0, st>>>(peer_ptrs(cm), cm->nranks, cm->rank, F_DONE, cm->step);
  ctx->launches += 1;
  CK(cudaGetLastError());
  return B2K_OK;
}

}  // namespace

// ================================================================================================
extern "C" {

int b2k_comm_create(b2k_ctx* ctx, int nranks, int rank, b2k_comm** out) {
  if (!ctx || !out || nranks < 1 || nranks > MAXR || rank < 0 || rank >= nranks) { if (ctx) ctx->err = "bad argument"; return B2K_ERR_ARG; }
  *out = nullptr;
  CK(cudaSetDevice(ctx->device));
  b2k_comm* cm = new (std::nothrow) b2k_comm();
  if (!cm) return B2K_ERR_ARG;
  cm->ctx = ctx; cm->nranks = nranks; cm->rank = rank;
  if (cudaMalloc(&cm->slab, SLAB_BYTES) != cudaSuccess) { ctx->err = "cudaMalloc of the exchange slab failed"; delete cm; return B2K_ERR_CUDA; }
  if (cudaMemset(cm->slab + OFF_WSUM, 0, SLAB_BYTES - OFF_WSUM) != cudaSuccess) { cudaFree(cm->slab); delete cm; return B2K_ERR_CUDA; }
  uint8_t ones[MAXR * 32];
  memset(ones, 0, sizeof ones);
  for (int i = 0; i < MAXR; i++) ones[32 * i + 31] = 1;
  if (cudaMemcpy(cm->slab + OFF_ONES, ones, sizeof ones, cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(cm->slab); delete cm; return B2K_ERR_CUDA; }
  if (cudaMallocHost(&cm->h_out, 64) != cudaSuccess) { cudaFree(cm->slab); delete cm; return B2K_ERR_CUDA; }
  cm->peer[rank] = cm->slab;
  cm->connected = nranks == 1;
  *out = cm;
  return B2K_OK;
}

int b2k_comm_export(b2k_comm* cm, uint8_t* blob) {
  if (!cm || !blob) return B2K_ERR_ARG;
  b2k_ctx* ctx = cm->ctx;
  CK(cudaSetDevice(ctx->device));
  Blob b;
  memset(&b, 0, sizeof b);
  CK(cudaIpcGetMemHandle(&b.handle, cm->slab));
  b.pid = (uint64_t)getpid();
  b.ptr = (uint64_t)reinterpret_cast<uintptr_t>(cm->slab);
  b.rank = cm->rank; b.device = ctx->device; b.bytes = SLAB_BYTES;
  memset(blob, 0, B2K_COMM_BLOB_BYTES);
  memcpy(blob, &b, sizeof b);
  return B2K_OK;
}

int b2k_comm_connect(b2k_comm* cm, const uint8_t* blobs) {
  if (!cm || !blobs) return B2K_ERR_ARG;
  b2k_ctx* ctx = cm->ctx;
  CK(cudaSetDevice(ctx->device));
  for (int p = 0; p < cm->nranks; p++) {
    Blob b;
    memcpy(&b, blobs + (size_t)p * B2K_COMM_BLOB_BYTES, sizeof b);
    if (b.rank != p || b.bytes != SLAB_BYTES) { ctx->err = "communicator blobs out of order or from another library build"; return B2K_ERR_ARG; }
    if (p == cm->rank) continue;
    if (b.pid == (uint64_t)getpid()) {                         // same process: map the peer device directly
      if (b.device != ctx->device) {
        int can = 0;
        CK(cudaDeviceCanAccessPeer(&can, ctx->device, b.device));
        if (!can) { ctx->err = "peer access between the two devices is not possible"; return B2K_ERR_CUDA; }
        cudaError_t e = cudaDeviceEnablePeerAccess(b.device, 0);
        if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
        else if (e != cudaSuccess) { ctx->err = std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e); return B2K_ERR_CUDA; }
      }
      cm->peer[p] = reinterpret_cast<char*>((uintptr_t)b.ptr);
    } else {
      void* m = nullptr;
      CK(cudaIpcOpenMemHandle(&m, b.handle, cudaIpcMemLazyEnablePeerAccess));
      cm->peer[p] = (char*)m;
      cm->ipc_open[p] = true;
    }
  }
  cm->connected = true;
  return B2K_OK;
}

int b2k_comm_connect_local(b2k_comm** comms, int nranks) {
  if (!comms || nranks < 1 || nranks > MAXR) return B2K_ERR_ARG;
  uint8_t blobs[MAXR * B2K_COMM_BLOB_BYTES];
  for (int p = 0; p < nranks; p++) {
    if (!comms[p] || comms[p]->nranks != nranks || comms[p]->rank != p) return B2K_ERR_ARG;
    int rc = b2k_comm_export(comms[p], blobs + (size_t)p * B2K_COMM_BLOB_BYTES);
    if (rc) return rc;
  }
  for (int p = 0; p < nranks; p++) {
    int rc = b2k_comm_connect(comms[p], blobs);
    if (rc) return rc;
  }
  return B2K_OK;
}

int b2k_nccl_unique_id(uint8_t* id) {
  std::string err;
  if (!id || !nccl_load(err)) return B2K_ERR_CUDA;
  return g_nccl.GetUniqueId(id) == 0 ? B2K_OK : B2K_ERR_CUDA;
}

int b2k_comm_use_nccl(b2k_comm* cm, const uint8_t* id) {
  if (!cm || !id) return B2K_ERR_ARG;
  b2k_ctx* ctx = cm->ctx;
  if (!nccl_load(ctx->err)) return B2K_ERR_CUDA;
  CK(cudaSetDevice(ctx->device));
  Id128 u;
  memcpy(u.b, id, 128);
  CKN(g_nccl.CommInitRank(&cm->nccl, cm->nranks, u, cm->rank));
  if (!cm->recv) CK(cudaMalloc(&cm->recv, SLAB_BUCKETS));
  cm->connected = true;
  return B2K_OK;
}

void b2k_comm_destroy(b2k_comm* cm) {
  if (!cm) return;
  cudaSetDevice(cm->ctx->device);
  cudaStreamSynchronize(cm->ctx->stream);
  if (cm->nccl && g_nccl.CommDestroy) g_nccl.CommDestroy(cm->nccl);
  for (int p = 0; p < cm->nranks; p++)
    if (cm->ipc_open[p]) cudaIpcCloseMemHandle(cm->peer[p]);
  if (cm->recv) cudaFree(cm->recv);
  if (cm->h_out) cudaFreeHost(cm->h_out);
  if (cm->slab) cudaFree(cm->slab);
  delete cm;
}

int b2k_comm_last_plan(const b2k_comm* cm, int* plan) {
  if (!cm || !plan) return B2K_ERR_ARG;
  memcpy(plan, cm->last_plan, sizeof cm->last_plan);
  return B2K_OK;
}

int b2k_bls12381_g1_msm_sharded_dev(b2k_comm* cm, size_t n, const void* d_scalars, const void* d_points, void* d_out, int shape) {
  return sharded_any(cm, n, d_scalars, d_points, false, d_out, shape);
}

int b2k_bls12381_g1_msm_sharded_async(b2k_comm* cm, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out) {
  if (!cm || !cm->ctx || !out) return B2K_ERR_ARG;
  b2k_ctx* ctx = cm->ctx;
  CK(cudaSetDevice(ctx->device));
  CK(cudaMemsetAsync(ctx->d_flags, 0, 4, ctx->stream));
  int rc = sharded_any(cm, n, scalars, points, true, cm->slab + OFF_OUT, 0);
  if (rc) return rc;
  CK(cudaMemcpyAsync(out, cm->slab + OFF_OUT, 48, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(ctx->h_flags, ctx->d_flags, 4, cudaMemcpyDeviceToHost, ctx->stream));
  return B2K_OK;
}

// Single process, ngpu contexts (the cgo adapter's shape: one Go process drives the whole box).  Pairs are partitioned
// contiguously; every device's work is only enqueued (the exchange waits are device-side), then all are collected.
int b2k_bls12381_g1_msm_multi_gpu(b2k_comm** comms, int ngpu, size_t n, const uint8_t* scalars, const uint8_t* points, uint8_t* out) {
  if (!comms || ngpu < 1 || ngpu > MAXR || !scalars || !points || !out || n < (size_t)ngpu) return B2K_ERR_ARG;
  uint8_t res[MAXR][64];
  const size_t base = n / ngpu, rem = n % ngpu;
  for (int g = 0; g < ngpu; g++)
    if (!comms[g] || !comms[g]->ctx || comms[g]->nranks != ngpu || comms[g]->rank != g) return B2K_ERR_ARG;
  int plan[4];                              // every rank must run ONE plan: the window width of the largest shard, pinned for all
  int rc0 = b2k_bls12381_g1_msm_bucket_plan(comms[0]->ctx, base + (rem ? 1 : 0), plan);
  if (rc0) return rc0;
  size_t lo = 0;
  for (int g = 0; g < ngpu; g++) {
    const size_t cnt = base + ((size_t)g < rem ? 1 : 0);
    b2k_ctx* ctx = comms[g]->ctx;
    const int keep = ctx->force_c;
    if (!keep) ctx->force_c = plan[0];
    // (pageable inputs: the H2D copies stage through the driver and return; the result goes to the communicator's pinned buffer)
    int rc = b2k_bls12381_g1_msm_sharded_async(comms[g], cnt, scalars + 32 * lo, points + 96 * lo, comms[g]->h_out);
    ctx->force_c = keep;
    if (rc) return rc;                      // (peers already enqueued time out on the device and report it from b2k_wait)
    lo += cnt;
  }
  int first = B2K_OK;
  for (int g = 0; g < ngpu; g++) {
    int rc = b2k_wait(comms[g]->ctx);
    if (rc && !first) first = rc;
  }
  if (first) return first;
  for (int g = 0; g < ngpu; g++) memcpy(res[g], comms[g]->h_out, 48);
  for (int g = 1; g < ngpu; g++)
    if (memcmp(res[g], res[0], 48)) { comms[0]->ctx->err = "ranks disagree on the sharded MSM result"; return B2K_ERR_CUDA; }
  memcpy(out, res[0], 48);
  return B2K_OK;
}

}  // extern "C"
