// Carry-chain primitives: PTX mad.lo.cc / madc.hi.cc / add.cc / sub.cc on sm_90a,
// with a bit-exact host emulation (explicit carry flag) so that the SAME field /
// curve templates can be unit-tested on a CPU-only box (tests/, -m "not gpu").
// The host path is test scaffolding for the arithmetic templates, not a product
// fallback: every product entry point in capi.cu requires a CUDA device.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define HD __host__ __device__ __forceinline__
#define HDNI __host__ __device__ __noinline__
#define DEV __device__ __forceinline__
#else
#define HD inline
#define HDNI
#define DEV inline
#endif

namespace gb200 {
namespace ptx {

#ifndef __CUDA_ARCH__
// host emulation state: the PTX condition-code carry flag
struct HostCC { static uint32_t& cf() { static thread_local uint32_t v = 0; return v; } };
#endif

// r = a + b, CF = carry
HD uint32_t add_cc(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
  uint32_t r; asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r;
#else
  uint64_t t = (uint64_t)a + b; HostCC::cf() = (uint32_t)(t >> 32); return (uint32_t)t;
#endif
}
// r = a + b + CF, CF = carry
HD uint32_t addc_cc(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
  uint32_t r; asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r;
#else
  uint64_t t = (uint64_t)a + b + HostCC::cf(); HostCC::cf() = (uint32_t)(t >> 32); return (uint32_t)t;
#endif
}
// r = a + b + CF (CF unchanged / don't care)
HD uint32_t addc(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
  uint32_t r; asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r;
#else
  return a + b + HostCC::cf();
#endif
}
// r = a - b, CF = borrow
HD uint32_t sub_cc(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
  uint32_t r; asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r;
#else
  uint64_t t = (uint64_t)a - b; HostCC::cf() = (uint32_t)(t >> 63); return (uint32_t)t;
#endif
}
HD uint32_t subc_cc(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
  uint32_t r; asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r;
#else
  uint64_t t = (uint64_t)a - b - HostCC::cf(); HostCC::cf() = (uint32_t)(t >> 63); return (uint32_t)t;
#endif
}
// r = a - b - CF  (all-ones when 0 - 0 - borrow)
HD uint32_t subc(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
  uint32_t r; asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r;
#else
  return a - b - HostCC::cf();
#endif
}
// r = lo(a*b) + c, CF = carry
HD uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) {
#ifdef __CUDA_ARCH__
  uint32_t r; asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r;
#else
  uint64_t t = (uint64_t)(uint32_t)((uint64_t)a * b) + c; HostCC::cf() = (uint32_t)(t >> 32); return (uint32_t)t;
#endif
}
HD uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) {
#ifdef __CUDA_ARCH__
  uint32_t r; asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r;
#else
  uint64_t t = (uint64_t)(uint32_t)((uint64_t)a * b) + c + HostCC::cf(); HostCC::cf() = (uint32_t)(t >> 32); return (uint32_t)t;
#endif
}
HD uint32_t mad_hi_cc(uint32_t a, uint32_t b, uint32_t c) {
#ifdef __CUDA_ARCH__
  uint32_t r; asm volatile("mad.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r;
#else
  uint64_t t = (((uint64_t)a * b) >> 32) + c; HostCC::cf() = (uint32_t)(t >> 32); return (uint32_t)t;
#endif
}
HD uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) {
#ifdef __CUDA_ARCH__
  uint32_t r; asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r;
#else
  uint64_t t = (((uint64_t)a * b) >> 32) + c + HostCC::cf(); HostCC::cf() = (uint32_t)(t >> 32); return (uint32_t)t;
#endif
}
HD uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }

// L2 prefetch of the line holding p (no register destination, no fault on a bad address); no-op on the host
HD void prefetch_l2(const void* p) {
#ifdef __CUDA_ARCH__
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
#else
  (void)p;
#endif
}

}  // namespace ptx
}  // namespace gb200
