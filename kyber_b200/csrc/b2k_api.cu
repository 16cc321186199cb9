// b2k_api.cu -- the C ABI of include/b2kyber.h: context, scratch arena, stage timing, launches.
// Host side is plumbing only; every arithmetic step runs in the sm_90a kernels of kernels.cuh.
#include <cuda_runtime.h>
#include <cstdio>
#include <cstring>
#include <string>
#include <new>

#include "../../include/b2kyber.h"
#include "msm_host.cuh"

using namespace b2k;

#include "b2k_ctx.h"

using Arena = b2k_arena;


namespace {

int arena_reserve_impl(b2k_ctx* ctx, size_t bytes) {
  Arena& a = ctx->arena;
  a.used = 0;
  if (bytes <= a.cap) return B2K_OK;
  if (a.base) {
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaFree(a.base));
    a.base = nullptr;
    a.cap = 0;
  }
  size_t want = bytes + (bytes >> 3);
  CK(cudaMalloc(&a.base, want));
  a.cap = want;
  return B2K_OK;
}

template <class T>
T* arena_take_impl(b2k_ctx* ctx, size_t count) {
  Arena& a = ctx->arena;
  size_t off = (a.used + 255) & ~size_t(255);
  size_t bytes = count * sizeof(T);
  if (off + bytes > a.cap) return nullptr;
  a.used = off + bytes;
  return reinterpret_cast<T*>(a.base + off);
}

}  // namespace

int b2k_arena_reserve(b2k_ctx* ctx, size_t bytes) { return arena_reserve_impl(ctx, bytes); }
void* b2k_arena_take(b2k_ctx* ctx, size_t bytes) { return arena_take_impl<char>(ctx, bytes); }

using namespace b2k_host;

// ================================================================================================
extern "C" {

const char* b2k_version(void) { return "b2kyber 0.1 (sm_90a)"; }

int b2k_create(int device, b2k_ctx** out) {
  if (!out) return B2K_ERR_ARG;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0 || device < 0 || device >= count) return B2K_ERR_NO_DEVICE;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return B2K_ERR_NO_DEVICE;
  if (prop.major != 9 || prop.minor != 0) return B2K_ERR_NO_DEVICE;   // sm_90a code only; no fallback
  b2k_ctx* ctx = new (std::nothrow) b2k_ctx();
  if (!ctx) return B2K_ERR_ARG;
  ctx->device = device;
  ctx->sm_count = prop.multiProcessorCount;
  bool ok = cudaSetDevice(device) == cudaSuccess &&
            cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) == cudaSuccess &&
            cudaMalloc(&ctx->d_flags, 256) == cudaSuccess &&
            cudaMallocHost(&ctx->h_flags, 256) == cudaSuccess &&
            cudaMemset(ctx->d_flags, 0, 256) == cudaSuccess;
  for (int i = 0; ok && i < N_EV; i++) ok = cudaEventCreate(&ctx->ev[i]) == cudaSuccess;
  for (int i = 0; ok && i < 10; i++) ok = cudaEventCreateWithFlags(&ctx->gev[i], cudaEventDisableTiming) == cudaSuccess;
  // (the high-priority side stream of the grouped-tail experiment is created on demand by b2k_set_msm_groups: an idle stream
  //  still occupies one of the device's hardware queues, and the spin-waits of b2k_multi.cu want those for themselves)
  if (!ok) { delete ctx; return B2K_ERR_CUDA; }
  ctx->own_stream = true;
  *ctx->h_flags = 0;
  *out = ctx;
  return B2K_OK;
}

void b2k_destroy(b2k_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->arena.base) cudaFree(ctx->arena.base);
  if (ctx->pair_scratch) cudaFree(ctx->pair_scratch);
  if (ctx->d_flags) cudaFree(ctx->d_flags);
  if (ctx->h_flags) cudaFreeHost(ctx->h_flags);
  for (int i = 0; i < N_EV; i++) cudaEventDestroy(ctx->ev[i]);
  for (int i = 0; i < 10; i++) cudaEventDestroy(ctx->gev[i]);
  if (ctx->stream2) { cudaStreamSynchronize(ctx->stream2); cudaStreamDestroy(ctx->stream2); }
  if (ctx->copy_stream) { cudaStreamSynchronize(ctx->copy_stream); cudaStreamDestroy(ctx->copy_stream); }
  if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

const char* b2k_last_error(const b2k_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int b2k_set_stream(b2k_ctx* ctx, void* cuda_stream) {
  if (!ctx) return B2K_ERR_ARG;
  CK(cudaStreamSynchronize(ctx->stream));
  if (ctx->own_stream) { cudaStreamDestroy(ctx->stream); ctx->own_stream = false; }
  ctx->stream = (cudaStream_t)cuda_stream;
  return B2K_OK;
}

int b2k_synchronize(b2k_ctx* ctx) {
  if (!ctx) return B2K_ERR_ARG;
  CK(cudaStreamSynchronize(ctx->stream));
  return B2K_OK;
}

int b2k_last_timings(b2k_ctx* ctx, float* ms, int max) {
  if (!ctx || !ms || max <= 0) return B2K_ERR_ARG;
  if (!ctx->timings_valid) return 0;
  CK(cudaStreamSynchronize(ctx->stream));
  int n = 0;
  for (int i = 0; i < 8 && n < max; i++, n++) {
    if (i == 4) CK(cudaEventElapsedTime(&ms[i], ctx->ev[4], ctx->ev[9]));
    else CK(cudaEventElapsedTime(&ms[i], ctx->ev[i], ctx->ev[i + 1]));
  }
  if (n < max) { CK(cudaEventElapsedTime(&ms[8], ctx->ev[0], ctx->ev[8])); n++; }
  if (n < max) { CK(cudaEventElapsedTime(&ms[9], ctx->ev[9], ctx->ev[5])); n++; }
  if (n < max) { CK(cudaEventElapsedTime(&ms[10], ctx->ev[4], ctx->ev[10])); n++; }
  return n;
}

int b2k_last_msm_plan(const b2k_ctx* ctx, int* out, int max) {
  if (!ctx || !out || max <= 0) return B2K_ERR_ARG;
  int n = max < LP_SLOTS ? max : LP_SLOTS;
  for (int i = 0; i < n; i++) out[i] = ctx->last_plan[i];
  return n;
}

int b2k_set_msm_affine(b2k_ctx* ctx, int rounds, int batch) {
  if (!ctx || rounds < -1 || rounds > 8 || batch < 0 || batch > 1024) return B2K_ERR_ARG;
  ctx->affine_rounds = rounds;
  ctx->affine_batch = batch;
  return B2K_OK;
}

int b2k_set_msm_affine_split(b2k_ctx* ctx, int split) {
  if (!ctx || (split != 0 && split != 1)) return B2K_ERR_ARG;
  ctx->affine_split = split;
  return B2K_OK;
}

int b2k_set_msm_staging(b2k_ctx* ctx, int mask) {
  if (!ctx || mask < 0 || mask > 15) return B2K_ERR_ARG;
  ctx->pt_stage = mask;
  return B2K_OK;
}

int b2k_set_msm_window(b2k_ctx* ctx, int c) {
  if (!ctx || (c != 0 && (c < 4 || c > 16))) return B2K_ERR_ARG;
  ctx->force_c = c;
  return B2K_OK;
}

uint64_t b2k_launch_count(const b2k_ctx* ctx) { return ctx ? ctx->launches : 0; }

int b2k_set_msm_slice(b2k_ctx* ctx, int L) {
  if (!ctx || L < 0 || L > 4096) return B2K_ERR_ARG;
  ctx->force_L = L;
  return B2K_OK;
}

int b2k_set_msm_chunk(b2k_ctx* ctx, int m) {
  if (!ctx || m < 0 || m > 32768) return B2K_ERR_ARG;
  ctx->force_m = m;
  return B2K_OK;
}

int b2k_set_msm_reduce(b2k_ctx* ctx, int levels, int m1, int m2) {
  auto pow2 = [](int v) { return v > 0 && (v & (v - 1)) == 0; };
  if (!ctx || levels < 0 || levels > 2 || (m1 != 0 && (!pow2(m1) || m1 > 64)) || (m2 != 0 && (!pow2(m2) || m2 > 64))) return B2K_ERR_ARG;
  ctx->reduce_levels = levels;
  ctx->reduce_m1 = m1;
  ctx->reduce_m2 = m2;
  return B2K_OK;
}

int b2k_set_msm_occupancy(b2k_ctx* ctx, int blocks_per_sm) {
  if (!ctx || blocks_per_sm < 4 || blocks_per_sm > 6) return B2K_ERR_ARG;
  ctx->acc_minb = blocks_per_sm;
  return B2K_OK;
}

int b2k_set_mul_occupancy(b2k_ctx* ctx, int blocks_per_sm) {
  if (!ctx || (blocks_per_sm != 0 && blocks_per_sm != 3 && blocks_per_sm != 4)) return B2K_ERR_ARG;
  ctx->mul_minb = blocks_per_sm;
  return B2K_OK;
}

int b2k_set_msm_glv(b2k_ctx* ctx, int on) {
  if (!ctx) return B2K_ERR_ARG;
  ctx->use_glv = on ? 1 : 0;
  return B2K_OK;
}

int b2k_set_msm_groups(b2k_ctx* ctx, int groups) {
  if (!ctx || groups < 1 || groups > 8) return B2K_ERR_ARG;
  if (groups > 1 && !ctx->stream2) {
    CK(cudaSetDevice(ctx->device));
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);      // hi = greatest priority (numerically lowest)
    CK(cudaStreamCreateWithPriority(&ctx->stream2, cudaStreamNonBlocking, hi));
  }
  ctx->msm_groups = groups;
  return B2K_OK;
}

int b2k_set_msm_variant(b2k_ctx* ctx, int v1) {
  if (!ctx) return B2K_ERR_ARG;
  ctx->use_v1 = v1 ? 1 : 0;
  return B2K_OK;
}

int b2k_bls12381_g1_msm(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return msm_host<Bls381G1>(c, n, s, p, o); }
int b2k_bls12381_g1_msm_affine(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return msm_host<Bls381G1>(c, n, s, p, o, 1); }
int b2k_bls12381_g1_msm_async(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, uint8_t* o) { return msm_host<Bls381G1>(c, n, s, p, o, 0, false); }
// also the status query of the *_dev entry points, which only enqueue: the device status word is sticky across them
int b2k_wait(b2k_ctx* ctx) {
  if (!ctx) return B2K_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  return status_finish(ctx);
}
int b2k_bls12381_g1_msm_dev(b2k_ctx* c, size_t n, const void* s, const void* p, void* o) {
  if (c && c->msm_layout == 1) return b2k_internal_bls12381_g1_msm_dev_inlined(c, n, s, p, o, 0);
  return msm_dev<Bls381G1>(c, n, s, p, o);
}
int b2k_set_msm_layout(b2k_ctx* ctx, int layout) {
  if (!ctx || layout < 0 || layout > 1) return B2K_ERR_ARG;
  ctx->msm_layout = layout;
  return B2K_OK;
}
int b2k_bls12381_g1_msm_affine_dev(b2k_ctx* c, size_t n, const void* s, const void* p, void* o) { return msm_dev<Bls381G1>(c, n, s, p, o, 1); }

int b2k_bls12381_g1_msm_bucket_plan(b2k_ctx* c, size_t n, int* plan) { return msm_bucket_plan<Bls381G1>(c, n, plan); }
int b2k_bls12381_g1_msm_buckets_dev(b2k_ctx* c, size_t n, const void* s, const void* p, void* b, size_t cap, int* plan) { return msm_buckets<Bls381G1>(c, n, (const uint8_t*)s, (const uint8_t*)p, false, b, cap, plan); }
// internal (b2k_ctx.h): host-staged bucket pass for the sharded entry points of b2k_multi.cu
int b2k_internal_bls12381_g1_msm_buckets_host(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, void* b, size_t cap, int* plan) { return msm_buckets<Bls381G1>(c, n, s, p, true, b, cap, plan); }
int b2k_bls12381_g1_msm_reduce_windows_dev(b2k_ctx* c, int cbits, int w_cnt, int parts, const void* recv, void* wsum) { return msm_reduce_windows_dev<Bls381G1>(c, cbits, w_cnt, parts, recv, wsum); }
int b2k_bls12381_g1_msm_finish_dev(b2k_ctx* c, int cbits, int W, const void* wsum, void* out, int affine_out) { return msm_finish_dev<Bls381G1>(c, cbits, W, wsum, out, affine_out); }


}  // extern "C"
