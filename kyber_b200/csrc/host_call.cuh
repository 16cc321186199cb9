// host_call.cuh -- what every C ABI entry point of libb2kyber.so does around its kernels: error checks, the scratch arena,
// the device status word and launch sizes.  The MSM's launch templates (msm_host.cuh) build on it.
#pragma once
#include <cuda_runtime.h>
#include <cstring>
#include <string>
#include "../../include/b2kyber.h"
#include "b2k_ctx.h"

namespace b2k {
// error flag bits written by kernels into the device status word
enum : uint32_t { FLAG_SCALAR_RANGE = 1u, FLAG_POINT = 2u, FLAG_COMM_TIMEOUT = 32u };   // (4u: duplicate share index, b2k_share.cu)
}  // namespace b2k

namespace b2k_host {
using namespace b2k;

#define CK(call)                                                                       \
  do {                                                                                 \
    cudaError_t e_ = (call);                                                           \
    if (e_ != cudaSuccess) {                                                           \
      ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_);                   \
      return B2K_ERR_CUDA;                                                             \
    }                                                                                  \
  } while (0)

inline int bad_arg(b2k_ctx* ctx, const char* why) {
  if (ctx) ctx->err = why;
  return B2K_ERR_ARG;
}

inline unsigned blocks_of(size_t n, unsigned bs) { return (unsigned)((n + bs - 1) / bs); }

inline int arena_reserve(b2k_ctx* ctx, size_t bytes) { return b2k_arena_reserve(ctx, bytes); }
template <class T>
T* arena_take(b2k_ctx* ctx, size_t count) { return reinterpret_cast<T*>(b2k_arena_take(ctx, count * sizeof(T))); }
inline size_t pad256(size_t b) { return (b + 255) & ~size_t(255); }

// ---- scratch carving ------------------------------------------------------------------------------------------------------
// Sub-buffers of the context's arena, 256-byte aligned as b2k_arena_take hands them out.  Every layout is written once, as a
// function of a Carve, and run twice: without an arena it only counts the bytes, with one it takes them (ok turns false if the
// arena runs out), so the bytes reserved are exactly the bytes taken.
struct Carve {
  b2k_ctx* arena = nullptr;
  size_t bytes = 0;
  bool ok = true;
  template <class T>
  T* take(size_t count) {
    bytes = pad256(bytes) + count * sizeof(T);
    if (!arena) return nullptr;
    T* p = arena_take<T>(arena, count);
    ok = ok && p;
    return p;
  }
};
// reserve the arena for what carve(Carve&) takes, then take it
template <class Fn>
int arena_carve(b2k_ctx* ctx, Fn&& carve) {
  Carve count;
  carve(count);
  int rc = arena_reserve(ctx, count.bytes);
  if (rc) return rc;
  Carve take{ctx};
  carve(take);
  if (!take.ok) { ctx->err = "scratch arena too small"; return B2K_ERR_ARG; }
  return B2K_OK;
}

// ---- the status word ------------------------------------------------------------------------------------------------------
inline int check_flags(b2k_ctx* ctx) {
  uint32_t f = *ctx->h_flags;
  if (f & FLAG_SCALAR_RANGE) { ctx->err = "scalar not below the group order"; return B2K_ERR_SCALAR_RANGE; }
  if (f & FLAG_POINT) { ctx->err = "malformed operand point"; return B2K_ERR_POINT; }
  if (f & FLAG_COMM_TIMEOUT) { ctx->err = "multi-GPU exchange: a peer rank did not arrive within 10 s"; return B2K_ERR_COMM; }
  return B2K_OK;
}

// message offsets of the host entry points: non-decreasing (ADVICE r1: a decreasing pair would make a kernel read ~4 GiB)
inline int check_offsets(b2k_ctx* ctx, size_t n, const uint32_t* offsets) {
  for (size_t i = 0; i < n; i++)
    if (offsets[i + 1] < offsets[i]) { ctx->err = "message offsets must be non-decreasing"; return B2K_ERR_ARG; }
  return B2K_OK;
}

// host-buffer entry points: the device status word is cleared in front of the call's work, fetched AND cleared behind it
// (a failed call must not leave a stale bit for a later *_dev sequence + b2k_wait)
inline int status_begin(b2k_ctx* ctx) {
  CK(cudaMemsetAsync(ctx->d_flags, 0, 4, ctx->stream));
  return B2K_OK;
}
inline int status_fetch_async(b2k_ctx* ctx) {
  CK(cudaMemcpyAsync(ctx->h_flags, ctx->d_flags, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemsetAsync(ctx->d_flags, 0, 4, ctx->stream));
  return B2K_OK;
}
inline int status_finish(b2k_ctx* ctx) {
  int rc = status_fetch_async(ctx);
  if (rc) return rc;
  CK(cudaStreamSynchronize(ctx->stream));
  return check_flags(ctx);
}

}  // namespace b2k_host
