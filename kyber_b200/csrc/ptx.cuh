// ptx.cuh -- carry-chain integer primitives for sm_90a.
//
// On the device every primitive is ONE PTX instruction (add.cc / addc / mad.lo.cc / madc.hi.cc ...);
// ptxas pairs a (mad.lo.cc, madc.hi.cc) couple on the same operands into one IMAD.WIDE.U32 with
// carry-in/out, which is what the Montgomery kernels in fp.cuh are laid out for.
//
// When compiled by a host compiler (B2K_HOST_EMUL, used ONLY by tests/host_emul to check the limb
// logic on a machine without a GPU) the same names are emulated with an explicit carry flag.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B2K_D __device__ __forceinline__
#define B2K_NI static __device__ __noinline__
#define B2K_HD __host__ __device__ __forceinline__        // also called by host code of a .cu unit (the shuffle transcript)
#define B2K_HNI static __host__ __device__ __noinline__
#else
#define B2K_D inline
#define B2K_NI inline
#define B2K_HD inline
#define B2K_HNI inline
#ifndef B2K_HOST_EMUL
#define B2K_HOST_EMUL 1
#endif
#endif

namespace b2k {
namespace ptx {

#if defined(__CUDACC__)

B2K_D uint32_t add_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2K_D uint32_t addc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2K_D uint32_t addc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2K_D uint32_t sub_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2K_D uint32_t subc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2K_D uint32_t subc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2K_D uint32_t mul_lo(uint32_t a, uint32_t b) { uint32_t r; asm volatile("mul.lo.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2K_D uint32_t mul_hi(uint32_t a, uint32_t b) { uint32_t r; asm volatile("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2K_D uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B2K_D uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B2K_D uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B2K_D uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }

#else  // host emulation ------------------------------------------------------------------------

static thread_local uint32_t g_cc = 0;
inline uint32_t add_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b; g_cc = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t addc_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b + g_cc; g_cc = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t addc(uint32_t a, uint32_t b) { return a + b + g_cc; }
inline uint32_t sub_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b; g_cc = (uint32_t)(t >> 63); return (uint32_t)t; }
inline uint32_t subc_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b - g_cc; g_cc = (uint32_t)(t >> 63); return (uint32_t)t; }
inline uint32_t subc(uint32_t a, uint32_t b) { return a - b - g_cc; }
inline uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }
inline uint32_t mul_hi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
inline uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (uint64_t)(uint32_t)(a * b) + c; g_cc = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (uint64_t)(uint32_t)(a * b) + c + g_cc; g_cc = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (((uint64_t)a * b) >> 32) + c + g_cc; g_cc = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { return (uint32_t)(((uint64_t)a * b) >> 32) + c + g_cc; }

#endif

}  // namespace ptx
}  // namespace b2k
