// Brownian increments of the SDE samplers (sde_small_kernel in ode_small.cu, sde_tc.cu) and the Hutchinson probes of
// cnf_tc.cu: one standard normal (or Rademacher sign) per
// (seed, step n, row r, column c), so a given draw is the same in both kernel classes, at any batch size and launch
// shape.  One Philox4x32-10 block (counter (c / 4, r lo, r hi, n), key (seed lo, seed hi)) serves 4 columns; 24-bit
// uniforms in (0, 1); Box-Muller on (u0, u1) for columns 4q, 4q + 1 and on (u2, u3) for 4q + 2, 4q + 3.
// Also the step state the Euler drivers of sde_tc.cu and cnf_tc.cu share (cfm_sde_state, cfm_cnf_tc_state).
#pragma once
#include <curand_philox4x32_x.h>
#include <stdint.h>

#include "common.cuh"

namespace cfm {

__device__ __forceinline__ uint4 sde_philox(uint64_t seed, int n, int64_t r, int q) {
  return curand_Philox4x32_10(make_uint4((unsigned)q, (unsigned)(uint64_t)r, (unsigned)((uint64_t)r >> 32), (unsigned)n),
                              make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
}

// exact: 24-bit integer * 2^-24 + 2^-25
__device__ __forceinline__ float sde_uniform(unsigned x) { return __fmaf_rn((float)(x >> 8), 0x1p-24f, 0x1p-25f); }

// Standard normal of (step n, row r, column c).  Depends on nothing else.
__device__ __forceinline__ float sde_normal(uint64_t seed, int n, int64_t r, int c) {
  const uint4 x = sde_philox(seed, n, r, c >> 2);
  const bool hi = c & 2;
  const unsigned xa = hi ? x.z : x.x, xb = hi ? x.w : x.y;
  const float ua = sde_uniform(xa);
  const float ub = sde_uniform(xb);
  float s, co;
  sincospif(2.f * ub, &s, &co);
  return sqrtf(-2.f * logf(ua)) * ((c & 1) ? s : co);
}

// The normals of columns 4q .. 4q + 3 from one Philox block: component i equals sde_normal(seed, n, r, 4q + i) bit
// for bit (the same operations on the same uniforms).
__device__ __forceinline__ float4 sde_normal4(uint64_t seed, int n, int64_t r, int q) {
  const uint4 x = sde_philox(seed, n, r, q);
  float s0, c0, s1, c1;
  sincospif(2.f * sde_uniform(x.y), &s0, &c0);
  sincospif(2.f * sde_uniform(x.w), &s1, &c1);
  const float r0 = sqrtf(-2.f * logf(sde_uniform(x.x))), r1 = sqrtf(-2.f * logf(sde_uniform(x.z)));
  return make_float4(r0 * c0, r0 * s0, r1 * c1, r1 * s1);
}

// Rademacher signs of columns 4q .. 4q + 3 from the same Philox block: column 4q + i is -1 where the top bit of word i
// is set and +1 otherwise (the Hutchinson probes of csrc/cnf_tc.cu).
__device__ __forceinline__ float4 sde_rademacher4(uint64_t seed, int n, int64_t r, int q) {
  const uint4 x = sde_philox(seed, n, r, q);
  auto sgn = [](unsigned v) { return (v >> 31) ? -1.f : 1.f; };
  return make_float4(sgn(x.x), sgn(x.y), sgn(x.z), sgn(x.w));
}

// ---- step state of the tensor-core Euler drivers ------------------------------------------------------------------
// The state side of the tensor-core class (mlp_tc_supported(batch, dim, w, dim) without w): CFM_OK, or CFM_ERR_ARG
// with the error naming the entry point `what`.
inline int tc_state_shape(const char* what, int batch, int dim) {
  CFM_REQUIRE(batch >= 128 && dim >= 32 && dim % 8 == 0,
              "%s: unsupported shape B=%d dim=%d (B >= 128, dim >= 32, dim %% 8 == 0)", what, batch, dim);
  return CFM_OK;
}

// End of a step kernel that ran step n: the CTA that finishes last moves the state on to step n + 1 at time t_next.
// Every CTA must have read st->n before it gets here.  State: a struct with int n, float t and unsigned ticket.
template <class State>
__device__ __forceinline__ void step_advance(State* st, int n, float t_next) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&st->ticket, 1u) == gridDim.x - 1) {
      st->n = n + 1;
      st->t = t_next;
      st->ticket = 0u;
    }
  }
}

}  // namespace cfm
