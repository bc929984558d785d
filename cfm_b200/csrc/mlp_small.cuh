// Device pieces shared by the kernels that keep a SMALL MLP (w = 32 * U) in shared memory and give one warp two rows:
// ode_small.cu (sampling) and train_small.cu (the training loss and its parameter gradients).  Lane l owns hidden
// units U*l .. U*l+U-1 and reads its weights of one input with one conflict-free shared-memory access.
#pragma once
#include "mlp_common.cuh"

namespace cfm {

constexpr int RB = 2;  // rows evaluated together by one warp

// the U consecutive floats a lane owns, as one 4*U-byte shared-memory access (p is 4*U-byte aligned)
template <int U>
__device__ __forceinline__ void lds_units(const float* p, float (&v)[U]) {
  if constexpr (U == 1) { v[0] = *p; }
  else if constexpr (U == 2) { const float2 t = *reinterpret_cast<const float2*>(p); v[0] = t.x; v[1] = t.y; }
  else { const float4 t = *reinterpret_cast<const float4*>(p); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
}
template <int U>
__device__ __forceinline__ void sts_units(float* p, const float (&v)[U]) {
  if constexpr (U == 1) { *p = v[0]; }
  else if constexpr (U == 2) { *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]); }
  else { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
}

// d act / dx at the pre-activation x, from the same ex2 approximation act_apply_fast uses
__device__ __forceinline__ float act_deriv_fast(float x, int act) {
  if (act == CFM_ACT_SELU) {
    const float scale = 1.0507009873554804934193349852946f;
    const float negcoef = (float)(1.6732632423543772848170429916717 * 1.0507009873554804934193349852946);
    return x > 0.f ? scale : ex2f(x * kLog2e) * negcoef;
  }
  const float s = __fdividef(1.f, 1.f + ex2f(-x * kLog2e));  // SiLU' = s + x s (1 - s), s = sigmoid(x)
  return fmaf(x * s, 1.f - s, s);
}

// d^2 act / dx^2 at the pre-activation x, from the same ex2 approximation: SELU'' = lambda alpha e^x for x <= 0 and 0
// for x > 0; SiLU'' = s (1 - s) (2 + x (1 - 2 s))
__device__ __forceinline__ float act_deriv2_fast(float x, int act) {
  if (act == CFM_ACT_SELU) {
    const float negcoef = (float)(1.6732632423543772848170429916717 * 1.0507009873554804934193349852946);
    return x > 0.f ? 0.f : ex2f(x * kLog2e) * negcoef;
  }
  const float s = __fdividef(1.f, 1.f + ex2f(-x * kLog2e));
  return s * (1.f - s) * fmaf(x, fmaf(-2.f, s, 1.f), 2.f);
}

// acc[r][q] += sum_i m[i][u0 + q] * v[r][i] for the RB rows of v ([RB][W] in shared memory): m is [W][W] with the
// lane's U columns contiguous, v is read as float4 broadcasts (the loop of mlp_eval's layers 1 and 2)
template <int U>
__device__ __forceinline__ void rb_matvec(const float* m, const float* v, float (&acc)[RB][U], int u0) {
  constexpr int W = 32 * U;
  float wv[U];
#pragma unroll 2
  for (int i = 0; i < W; i += 4) {
    const float4 va = *reinterpret_cast<const float4*>(v + i);
    const float4 vb = *reinterpret_cast<const float4*>(v + W + i);
    const float vs[RB][4] = {{va.x, va.y, va.z, va.w}, {vb.x, vb.y, vb.z, vb.w}};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      lds_units<U>(m + (size_t)(i + c) * W + u0, wv);
#pragma unroll
      for (int q = 0; q < U; ++q) {
        acc[0][q] = fmaf(wv[q], vs[0][c], acc[0][q]);
        acc[1][q] = fmaf(wv[q], vs[1][c], acc[1][q]);
      }
    }
  }
}

}  // namespace cfm
