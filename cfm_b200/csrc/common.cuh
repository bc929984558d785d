// cfm_b200 -- shared device/host helpers for the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/cfm_b200.h"

namespace cfm {

// ---- error plumbing (thread-local last-error string; see api.cu) -------------
void set_error(const char* fmt, ...);

#define CFM_CUDA_OK(expr)                                                         \
  do {                                                                            \
    cudaError_t _e = (expr);                                                      \
    if (_e != cudaSuccess) {                                                      \
      ::cfm::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,              \
                       cudaGetErrorString(_e));                                   \
      return CFM_ERR_CUDA;                                                        \
    }                                                                             \
  } while (0)

#define CFM_REQUIRE(cond, ...)                                                    \
  do {                                                                            \
    if (!(cond)) {                                                                \
      ::cfm::set_error(__VA_ARGS__);                                              \
      return CFM_ERR_ARG;                                                         \
    }                                                                             \
  } while (0)

void note_launches(int n);  // bumps the process-wide kernel-launch counter (cfm_launch_count)
int sm_count();             // cached cudaDevAttrMultiProcessorCount of the current device
int cc_major_minor();       // major*10+minor of the current device
size_t l2_bytes();          // cached cudaDevAttrL2CacheSize of the current device

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---- device helpers ------------------------------------------------------------
#ifdef __CUDACC__
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
constexpr double kLn2d = 0.69314718055994530942;
constexpr double kLog2ed = 1.44269504088896340736;
constexpr float kNegBig = -1.0e30f;  // finite stand-in for -inf in running maxima

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float lg2f(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// log2 with ~2^-22 ABSOLUTE error for any positive normal x: lg2.approx is only relatively accurate, so
// it is applied to the mantissa in [1, 2) and the exponent is added exactly
__device__ __forceinline__ float lg2_abs(float x) {
  const int b = __float_as_int(x);
  const float e = (float)((b >> 23) - 127);
  const float m = __int_as_float((b & 0x007fffff) | 0x3f800000);
  return e + lg2f(m);
}
// streaming 128-bit load: no L1 allocation (data is touched once per sweep from this SM)
__device__ __forceinline__ float4 ldg_stream4(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// atomic max for non-negative floats (bit pattern order == value order)
__device__ __forceinline__ void atomic_max_nonneg(float* addr, float v) {
  atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
}
#endif  // __CUDACC__

}  // namespace cfm
