// host_call.cuh -- what every C ABI entry point of libb2kyber.so does around its kernels: error checks, the scratch arena,
// the device status word and launch sizes.  The MSM's launch templates (msm_host.cuh) build on it.
#pragma once
#include <cuda_runtime.h>
#include <cstring>
#include <string>
#include <vector>
#include "../../include/b2kyber.h"
#include "b2k_ctx.h"

namespace b2k {
// error flag bits written by kernels into the device status word
enum : uint32_t {
  FLAG_SCALAR_RANGE = 1u,
  FLAG_POINT = 2u,
  FLAG_DUP_INDEX = 4u,      // two shares with the same index (Lagrange interpolation)
  FLAG_COMM_TIMEOUT = 32u,
  FLAG_IBE_H3 = 64u,        // IBE's H3 found no scalar below r (rejection sampling failure)
};
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

// ---- scratch carving and staging -----------------------------------------------------------------------------------------
// Sub-buffers of the context's arena, 256-byte aligned as b2k_arena_take hands them out.  Every layout is written once, as a
// function of a Carve, and run twice: without an arena it only counts the bytes (ok turns false if the count overflows size_t),
// with one it takes them (ok turns false if the arena runs out), so the bytes reserved are exactly the bytes taken.  The take
// pass also records the copies of staged inputs (in) and results (out), which host_call enqueues around the kernels.
struct Carve {
  struct Copy {
    void* dst;
    const void* src;
    size_t bytes;
  };
  b2k_ctx* arena = nullptr;
  size_t bytes = 0;
  bool ok = true;
  std::vector<Copy> ins, outs;   // take pass only, in declaration order; copies of 0 bytes are left out

  // scratch: count x width elements of T
  template <class T>
  T* take(size_t count, size_t width = 1) {
    size_t b = 0, at = bytes + 255;
    if (!ok || __builtin_mul_overflow(count, width, &count) || __builtin_mul_overflow(count, sizeof(T), &b) || at < bytes ||
        __builtin_add_overflow(at & ~size_t(255), b, &bytes)) {
      ok = false;
      return nullptr;
    }
    if (!arena) return nullptr;
    T* p = arena_take<T>(arena, count);
    ok = ok && p;
    return p;
  }
  // a staged input, copied from the host in front of the kernels; the pointer is valid at count 0 too
  template <class T>
  T* in(const T* host, size_t count, size_t width = 1) {
    T* d = take<T>(count, width);
    copy_in(d, host, count * width);
    return d;
  }
  // a result, copied to the host behind the kernels
  template <class T>
  T* out(T* host, size_t count, size_t width = 1) {
    T* d = take<T>(count, width);
    copy_out(host, d, count * width);
    return d;
  }
  // the same copies into or out of part of a buffer already taken
  template <class T>
  void copy_in(T* dev, const T* host, size_t count) {
    if (arena && ok && count) ins.push_back({dev, host, count * sizeof(T)});
  }
  template <class T>
  void copy_out(T* host, const T* dev, size_t count) {
    if (arena && ok && count) outs.push_back({host, dev, count * sizeof(T)});
  }
};

// reserve the arena for what layout(Carve&) takes, then take it into `take`
template <class Fn>
int arena_carve(b2k_ctx* ctx, Fn&& layout, Carve& take) {
  Carve count;
  layout(count);
  if (!count.ok) return bad_arg(ctx, "batch too large");
  int rc = arena_reserve(ctx, count.bytes);
  if (rc) return rc;
  take.arena = ctx;
  layout(take);
  if (!take.ok) { ctx->err = "scratch arena too small"; return B2K_ERR_ARG; }
  return B2K_OK;
}
template <class Fn>
int arena_carve(b2k_ctx* ctx, Fn&& layout) {
  Carve take;
  return arena_carve(ctx, layout, take);
}

// ---- the status word ------------------------------------------------------------------------------------------------------
// Only calls whose kernels set FLAG_DUP_INDEX or FLAG_IBE_H3 can see them; they are reported before the other bits.
inline int check_flags(b2k_ctx* ctx) {
  uint32_t f = *ctx->h_flags;
  if (f & FLAG_DUP_INDEX) { ctx->err = "duplicate share index"; return B2K_ERR_ARG; }
  if (f & FLAG_IBE_H3) { ctx->err = "rejection sampling failure"; return B2K_ERR_ARG; }
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

// ---- one host-buffer call -------------------------------------------------------------------------------------------------
// Carves layout(Carve&) out of one reservation of the arena, clears the status word, copies the staged inputs in, runs
// enqueue(), copies the results out, fetches and clears the status word and drains the stream, on every path.  With wipe the
// carved bytes are zeroed before the drain, so that no staged secret outlives the call in device memory the context keeps.
template <class Layout, class Enqueue>
int host_call(b2k_ctx* ctx, Layout&& layout, Enqueue&& enqueue, bool wipe = false) {
  Carve c;
  int rc = arena_carve(ctx, layout, c);
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  rc = [&]() -> int {
    CK(cudaMemsetAsync(ctx->d_flags, 0, 4, st));
    for (const Carve::Copy& x : c.ins) CK(cudaMemcpyAsync(x.dst, x.src, x.bytes, cudaMemcpyHostToDevice, st));
    if (int e = enqueue()) return e;
    for (const Carve::Copy& x : c.outs) CK(cudaMemcpyAsync(x.dst, x.src, x.bytes, cudaMemcpyDeviceToHost, st));
    return status_fetch_async(ctx);
  }();
  if (rc) cudaMemsetAsync(ctx->d_flags, 0, 4, st);   // a failed call leaves no stale bit either
  if (wipe && cudaMemsetAsync(ctx->arena.base, 0, c.bytes, st) != cudaSuccess && !rc) {
    ctx->err = "clearing the staged bytes failed";
    rc = B2K_ERR_CUDA;
  }
  const cudaError_t e = cudaStreamSynchronize(st);
  if (rc) return rc;
  if (e != cudaSuccess) { ctx->err = std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e); return B2K_ERR_CUDA; }
  return check_flags(ctx);
}

}  // namespace b2k_host
