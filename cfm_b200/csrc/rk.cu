// Dormand-Prince 5(4) lock-step driver pieces (torchdyn NeuralODE(solver="dopri5") semantics;
// call sites in the reference: examples/2D_tutorials/tutorial_training_8_gaussians_to_moons.ipynb
// :332-338; torchdyn itself is un-vendored -- SURVEY.md Appendix B).
//
// The whole batch advances with ONE scalar step size (global RMS error norm), so the step
// controller is a handful of scalars.  They live in a device struct (cfm_rk_state): every kernel
// of a step reads t/dt from it, the error norm is accumulated into it, and a one-thread control
// kernel does accept/reject, checkpoint clipping and step-size adaptation in fp32 exactly in the
// order torchdyn's _adaptive_odeint does (rk_control.cuh, shared with ode_small.cu).  A full step (6 stage-input kernels + 6 MLP forwards +
// error norm + control + commit) is therefore enqueued without any host round trip.
//
// Buffers (fp32, numel = B*D each): x, xnew, xs (stage input), k[0..6] contiguous (k1..k7).
// All elementwise kernels are HBM-bound: float4 accesses, grid = 4 CTAs/SM, grid-stride loops.
#include "gemm_h3.cuh"  // pack4h
#include "rk_control.cuh"
#include "rk_tableau.h"

namespace cfm {

// fp16x3 operand split (gemm_h3.cuh): hi = fp16(v), lo = fp16((v - hi) * 2^11), saturating.  Not split_h3_sat: the
// clamp before __float2half_rn turns a NaN into -65504, where cvt.rn.satfinite keeps it NaN, so the two differ on a
// NaN state.
__device__ __forceinline__ void rk_split_h3(float v, __half& hi, __half& lo) {
  const float c = fminf(fmaxf(v, -65504.f), 65504.f);
  hi = __float2half_rn(c);
  const float r = (v - __half2float(hi)) * 2048.f;
  lo = __float2half_rn(fminf(fmaxf(r, -65504.f), 65504.f));
}


__constant__ float kC[7] = CFM_RK_C_INIT;
__constant__ float kA[7][6] = CFM_RK_A_INIT;
// b5 - b4 (embedded error weights), k1..k7
__constant__ float kE[7] = CFM_RK_E_INIT;

// L2 policies for the stage-input reads: a dopri5 step re-reads x and k1 in every one of its six stage inputs while
// ~1 GB of other traffic (2.5x the L2) passes in between; loading them evict_last keeps them resident.  k2..k6 are
// loaded evict_first.
__device__ __forceinline__ uint64_t rk_policy(bool last) {
  uint64_t p;
  if (last) asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  else asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ float4 rk_ld_pol(const float4* ptr, uint64_t pol) {
  float4 v;
  asm("ld.global.nc.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"  // (not volatile: schedulable like a plain load)
      : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(ptr), "l"(pol));
  return v;
}

static inline int rk_ew_grid(int64_t numel) {
  int64_t blocks = (numel / 4 + 255) / 256 + 1;
  const int64_t cap = (int64_t)sm_count() * 8;
  return (int)(blocks < cap ? blocks : cap);
}

static inline int rk_stage_grid(int64_t numel) {  // at most 8 CTAs per SM
  int64_t blocks = (numel / 8 + 255) / 256 + 1;
  const int64_t cap = (int64_t)sm_count() * 8;
  return (int)(blocks < cap ? blocks : cap);
}

__device__ __forceinline__ double block_sum_to(double v, double* smem32) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) smem32[warp] = v;
  __syncthreads();
  double t = 0.0;
  if (warp == 0) {
    t = lane < (blockDim.x >> 5) ? smem32[lane] : 0.0;
    t = warp_sum(t);
  }
  return t;  // valid in warp 0 lane 0
}

// host/device compile-time copies of the tableau (same initialisers as the __constant__ arrays: identical fp32 values)
__host__ __device__ constexpr float rk_a(int s, int j) { constexpr float t[7][6] = CFM_RK_A_INIT; return t[s][j]; }
__host__ __device__ constexpr float rk_e(int j) { constexpr float t[7] = CFM_RK_E_INIT; return t[j]; }

// xs (stage 1..5) or xnew (stage 6) = x + dt * sum_j a[stage][j] * k_j ; also t_stage = t + c*dt.
// STAGE is a template parameter so that the loads of a thread -- x and the stage's derivative arrays, for U float4
// positions -- are straight-line code issued back to back (up to 12 independent 128-bit loads in flight per thread);
// L2 policies: see rk_policy above.
template <int STAGE>
__global__ void __launch_bounds__(256)
rk_stage_input_kernel(const cfm_rk_state* __restrict__ st, const float* __restrict__ x,
                      const float* __restrict__ k, float* __restrict__ out,
                      __half* __restrict__ out_hi, __half* __restrict__ out_lo,
                      float* __restrict__ t_stage, float* __restrict__ err_partial, int64_t numel) {
  if (st->done) return;
  constexpr int stage = STAGE;
  constexpr int U = 2;
  const float dt = st->dt;
  const uint64_t pol_last = rk_policy(true), pol_first = rk_policy(false);
  if (blockIdx.x == 0 && threadIdx.x == 0 && t_stage) *t_stage = fmaf(kC[stage], dt, st->t);
  float a[6];
#pragma unroll
  for (int j = 0; j < 6; ++j) a[j] = dt * rk_a(stage, j);
  const int64_t n4 = (numel & 3) ? 0 : (numel >> 2);  // k_j bases stay 16B-aligned only then
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < n4; i0 += U * stride) {
    float4 v[U], kk[U][6];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * stride < n4 ? i0 + u * stride : i0;  // (a clamped duplicate instead of a branch)
      v[u] = rk_ld_pol(reinterpret_cast<const float4*>(x) + i, pol_last);
#pragma unroll
      for (int j = 0; j < 6; ++j)
        if (j < stage && rk_a(stage, j) != 0.f) {
          const float4* kp = reinterpret_cast<const float4*>(k + (int64_t)j * numel) + i;
          kk[u][j] = rk_ld_pol(kp, j == 0 ? pol_last : pol_first);
        }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * stride;
      if (i >= n4) break;
      float4 e6 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int j = 0; j < 6; ++j)
        if (j < stage && rk_a(stage, j) != 0.f) {
          v[u].x = fmaf(a[j], kk[u][j].x, v[u].x); v[u].y = fmaf(a[j], kk[u][j].y, v[u].y);
          v[u].z = fmaf(a[j], kk[u][j].z, v[u].z); v[u].w = fmaf(a[j], kk[u][j].w, v[u].w);
          if (stage == 6) {  // stage 6 reads k1..k6 anyway: hand the error estimate's first six terms to the norm kernel
            e6.x = fmaf(rk_e(j), kk[u][j].x, e6.x); e6.y = fmaf(rk_e(j), kk[u][j].y, e6.y);
            e6.z = fmaf(rk_e(j), kk[u][j].z, e6.z); e6.w = fmaf(rk_e(j), kk[u][j].w, e6.w);
          }
        }
      if (stage == 6 && err_partial) reinterpret_cast<float4*>(err_partial)[i] = e6;
      if (out) reinterpret_cast<float4*>(out)[i] = v[u];
      if (out_hi) {  // operand pair for the tensor-core MLP: the fp32 stage input is never re-read
        __half h[4], l[4];
        rk_split_h3(v[u].x, h[0], l[0]); rk_split_h3(v[u].y, h[1], l[1]);
        rk_split_h3(v[u].z, h[2], l[2]); rk_split_h3(v[u].w, h[3], l[3]);
        reinterpret_cast<uint2*>(out_hi)[i] = pack4h(h);
        reinterpret_cast<uint2*>(out_lo)[i] = pack4h(l);
      }
    }
  }
  for (int64_t i = (n4 << 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += stride) {
    float v = x[i], e6 = 0.f;
    for (int j = 0; j < stage; ++j) {
      v = fmaf(a[j], k[(int64_t)j * numel + i], v);
      if (kA[stage][j] != 0.f) e6 = fmaf(kE[j], k[(int64_t)j * numel + i], e6);
    }
    if (err_partial) err_partial[i] = e6;
    if (out) out[i] = v;
    if (out_hi) { __half h, l; rk_split_h3(v, h, l); out_hi[i] = h; out_lo[i] = l; }
  }
}

// err_acc += sum( (dt * sum_j e_j k_j / (atol + rtol * max(|x|, |xnew|)))^2 )
__global__ void rk_error_norm_kernel(cfm_rk_state* st, const float* __restrict__ x,
                                     const float* __restrict__ xnew, const float* __restrict__ k,
                                     const float* __restrict__ err_partial, int64_t numel) {
  __shared__ double red[32];
  if (st->done) return;
  const float dt = st->dt, atol = st->atol, rtol = st->rtol;
  double acc = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += stride) {
    float e = 0.f;
    if (err_partial) {  // sum_{j<=6} e_j k_j was accumulated by the stage-6 kernel (same order of operations)
      e = fmaf(kE[6], k[6 * numel + i], err_partial[i]);
    } else {
#pragma unroll
      for (int j = 0; j < 7; ++j)
        if (kE[j] != 0.f) e = fmaf(kE[j], k[(int64_t)j * numel + i], e);
    }
    e *= dt;
    const float r = e / rk_err_tol(x[i], xnew[i], atol, rtol);
    acc += (double)r * (double)r;
  }
  const double t = block_sum_to(acc, red);
  if (threadIdx.x == 0) atomicAdd(&st->err_acc, t);
}

__global__ void rk_control_kernel(cfm_rk_state* st, const float* __restrict__ t_span, int64_t numel) {
  if (st->done) { st->commit = 0; return; }  // a step enqueued past the end of the interval is a no-op
  const float ratio = (float)sqrt(st->err_acc / (double)numel);
  st->err_acc = 0.0;
  st->commit = rk_control(*st, ratio, t_span) ? 1 : 0;
}

// accepted: x <- xnew, k1 <- k7 (FSAL), optional checkpoint copy
__global__ void rk_commit_kernel(const cfm_rk_state* __restrict__ st, float* __restrict__ x,
                                 const float* __restrict__ xnew, float* __restrict__ k,
                                 float* __restrict__ traj, int64_t numel) {
  if (!st->commit) return;
  const int slot = st->save_slot;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const float* k7 = k + 6 * numel;
  const int64_t n4 = (numel & 3) ? 0 : (numel >> 2);  // k_j bases stay 16B-aligned only then
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = reinterpret_cast<const float4*>(xnew)[i];
    reinterpret_cast<float4*>(x)[i] = v;
    reinterpret_cast<float4*>(k)[i] = reinterpret_cast<const float4*>(k7)[i];
    if (slot >= 0) reinterpret_cast<float4*>(traj + (int64_t)slot * numel)[i] = v;
  }
  for (int64_t i = (n4 << 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += stride) {
    x[i] = xnew[i];
    k[i] = k7[i];
    if (slot >= 0) traj[(int64_t)slot * numel + i] = xnew[i];
  }
}

// ---- Hairer initial step (torchdyn init_step) -------------------------------------------------
// scratch[0] = sum (x/scale)^2, scratch[1] = sum (f0/scale)^2, scratch[2] = sum ((f1-f0)/scale)^2
__global__ void rk_init_reduce_a(const cfm_rk_state* __restrict__ st, const float* __restrict__ x,
                                 const float* __restrict__ f0, double* scratch, int64_t numel) {
  __shared__ double red[32];
  const float atol = st->atol, rtol = st->rtol;
  double a0 = 0.0, a1 = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t n4 = ((numel & 3) == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(f0)) & 15) == 0)
                         ? (numel >> 2) : 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {  // 128-bit loads
    const float4 xv = reinterpret_cast<const float4*>(x)[i], fv = reinterpret_cast<const float4*>(f0)[i];
    const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, fs[4] = {fv.x, fv.y, fv.z, fv.w};
    float s0 = 0.f, s1 = 0.f;  // four squares per partial: fp32 is ample, the long sums are float64
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float sc = rk_init_scale(xs[c], atol, rtol);
      const float p = xs[c] / sc, q = fs[c] / sc;
      s0 = fmaf(p, p, s0);
      s1 = fmaf(q, q, s1);
    }
    a0 += (double)s0;
    a1 += (double)s1;
  }
  for (int64_t i = (n4 << 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += stride) {
    const float sc = rk_init_scale(x[i], atol, rtol);
    const float p = x[i] / sc, q = f0[i] / sc;
    a0 += (double)p * p;
    a1 += (double)q * q;
  }
  double t = block_sum_to(a0, red);
  if (threadIdx.x == 0) atomicAdd(&scratch[0], t);
  __syncthreads();
  t = block_sum_to(a1, red);
  if (threadIdx.x == 0) atomicAdd(&scratch[1], t);
}
__global__ void rk_init_probe(const cfm_rk_state* st, const float* __restrict__ x, const float* __restrict__ f0,
                              float* __restrict__ x_probe, float* __restrict__ t_stage,
                              const double* __restrict__ scratch, int64_t numel, int64_t numel_global) {
  const float h0 = rk_h0(scratch[0], scratch[1], (double)numel_global);
  if (blockIdx.x == 0 && threadIdx.x == 0 && t_stage) *t_stage = st->t + h0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += stride)
    x_probe[i] = fmaf(h0, f0[i], x[i]);
}
__global__ void rk_init_reduce_b(const cfm_rk_state* __restrict__ st, const float* __restrict__ x,
                                 const float* __restrict__ f0, const float* __restrict__ f1,
                                 double* scratch, int64_t numel) {
  __shared__ double red[32];
  const float atol = st->atol, rtol = st->rtol;
  double a = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += stride) {
    const float sc = rk_init_scale(x[i], atol, rtol);
    const float q = (f1[i] - f0[i]) / sc;
    a += (double)q * q;
  }
  const double t = block_sum_to(a, red);
  if (threadIdx.x == 0) atomicAdd(&scratch[2], t);
}
__global__ void rk_init_finish(cfm_rk_state* st, const float* __restrict__ t_span,
                               const double* __restrict__ scratch, int64_t numel) {
  const double n = (double)numel;
  rk_init_step(*st, rk_h0(scratch[0], scratch[1], n), scratch[1], scratch[2], n, t_span);
}

__global__ void axpy_kernel(const float* __restrict__ x, const float* __restrict__ k, float h,
                            float* __restrict__ out, int64_t numel) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += stride)
    out[i] = fmaf(h, k[i], x[i]);
}

}  // namespace cfm

using namespace cfm;

#define RK_CHECK(cond) CFM_REQUIRE(cond, "%s: bad argument (" #cond ")", __func__)

extern "C" int cfm_rk_stage_input(const cfm_rk_state* st, const float* x, const float* k, float* out,
                                  void* out_hi, void* out_lo, float* t_stage, float* err_partial, int64_t numel,
                                  int stage, void* stream) {
  RK_CHECK(st && x && k && (out || out_hi) && numel > 0 && stage >= 1 && stage <= 6);
  RK_CHECK((out_hi == nullptr) == (out_lo == nullptr));
  RK_CHECK(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(out) |
             reinterpret_cast<uintptr_t>(out_hi) | reinterpret_cast<uintptr_t>(out_lo)) & 15) == 0);
  RK_CHECK(err_partial == nullptr || stage == 6);
  using Kern = void (*)(const cfm_rk_state*, const float*, const float*, float*, __half*, __half*, float*, float*, int64_t);
  static const Kern table[6] = {rk_stage_input_kernel<1>, rk_stage_input_kernel<2>, rk_stage_input_kernel<3>,
                                rk_stage_input_kernel<4>, rk_stage_input_kernel<5>, rk_stage_input_kernel<6>};
  const Kern kern = table[stage - 1];
  kern<<<rk_stage_grid(numel), 256, 0, (cudaStream_t)stream>>>(
      st, x, k, out, reinterpret_cast<__half*>(out_hi), reinterpret_cast<__half*>(out_lo), t_stage, err_partial, numel);
  ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
extern "C" int cfm_rk_error_norm(cfm_rk_state* st, const float* x, const float* xnew, const float* k,
                                 const float* err_partial, int64_t numel, void* stream) {
  RK_CHECK(st && x && xnew && k && numel > 0);
  rk_error_norm_kernel<<<rk_ew_grid(numel), 256, 0, (cudaStream_t)stream>>>(st, x, xnew, k, err_partial, numel); ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
extern "C" int cfm_rk_control(cfm_rk_state* st, const float* t_span, int64_t numel, void* stream) {
  RK_CHECK(st && t_span && numel > 0);
  rk_control_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(st, t_span, numel); ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
extern "C" int cfm_rk_commit(const cfm_rk_state* st, float* x, const float* xnew, float* k, float* traj,
                             int64_t numel, void* stream) {
  RK_CHECK(st && x && xnew && k && traj && numel > 0);
  rk_commit_kernel<<<rk_ew_grid(numel), 256, 0, (cudaStream_t)stream>>>(st, x, xnew, k, traj, numel); ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
// The Hairer initial step in four calls (sums phase 0, probe, sums phase 1, finish), so that a sharded (lock-step)
// driver can all-reduce the partial sums in `scratch` between them and pass the GLOBAL element count to the steps
// that turn sums into norms
extern "C" int cfm_rk_init_sums(const cfm_rk_state* st, const float* x, const float* f0, const float* f1,
                                double* scratch, int64_t numel, int phase, void* stream) {
  RK_CHECK(st && x && f0 && scratch && numel > 0 && (phase == 0 || (phase == 1 && f1)));
  cudaStream_t s = (cudaStream_t)stream;
  if (phase == 0) {
    CFM_CUDA_OK(cudaMemsetAsync(scratch, 0, 4 * sizeof(double), s));
    rk_init_reduce_a<<<rk_ew_grid(numel), 256, 0, s>>>(st, x, f0, scratch, numel); ::cfm::note_launches(1);
  } else {
    rk_init_reduce_b<<<rk_ew_grid(numel), 256, 0, s>>>(st, x, f0, f1, scratch, numel); ::cfm::note_launches(1);
  }
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
extern "C" int cfm_rk_init_probe(cfm_rk_state* st, const float* x, const float* f0, float* x_probe,
                                 float* t_stage, const double* scratch, int64_t numel, int64_t numel_global,
                                 void* stream) {
  RK_CHECK(st && x && f0 && x_probe && scratch && numel > 0 && numel_global >= numel);
  rk_init_probe<<<rk_ew_grid(numel), 256, 0, (cudaStream_t)stream>>>(st, x, f0, x_probe, t_stage, scratch, numel,
                                                                 numel_global); ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
extern "C" int cfm_rk_init_finish(cfm_rk_state* st, const float* t_span, const double* scratch,
                                  int64_t numel_global, void* stream) {
  RK_CHECK(st && t_span && scratch && numel_global > 0);
  rk_init_finish<<<1, 1, 0, (cudaStream_t)stream>>>(st, t_span, scratch, numel_global); ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
extern "C" int cfm_axpy_f32(const float* x, const float* k, float h, float* x_out, int64_t numel,
                            void* stream) {
  RK_CHECK(x && k && x_out && numel > 0);
  axpy_kernel<<<rk_ew_grid(numel), 256, 0, (cudaStream_t)stream>>>(x, k, h, x_out, numel); ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
