// torchdyn's dopri5 step controller (_adaptive_odeint, init_step, adapt_step, hairer_norm), one definition for both
// ODE drivers: the one-thread control kernels of the multi-kernel driver (rk.cu, state in device memory) and the
// controller that every thread of the one-launch kernel replicates (ode_small.cu, state in registers).  Scalar fp32
// in torchdyn's order of operations; the drivers only turn their sums of squares into norms differently.
// t_span is read-only for the whole run.
#pragma once
#include "common.cuh"

namespace cfm {

// per-element scale of the Hairer initial step: atol + |x| rtol
__device__ __forceinline__ float rk_init_scale(float x, float atol, float rtol) { return atol + fabsf(x) * rtol; }

// per-element tolerance of the error norm: atol + rtol max(|x|, |xnew|)
__device__ __forceinline__ float rk_err_tol(float x, float xnew, float atol, float rtol) {
  return atol + rtol * fmaxf(fabsf(x), fabsf(xnew));
}

// top of torchdyn's while-loop for the NEXT step: clip to t_end, clip to the next checkpoint
__device__ __forceinline__ void rk_prestep(cfm_rk_state& s, const float* t_span) {
  if (!(s.t < s.t_end)) { s.done = 1; return; }
  if (s.t + s.dt > s.t_end) s.dt = s.t_end - s.t;
  if (s.ckpt < s.n_span && s.t + s.dt > __ldg(t_span + s.ckpt)) {
    s.dt_old = s.dt;
    s.ckpt_flag = 1;
    s.dt = __ldg(t_span + s.ckpt) - s.t;
  }
}

// Hairer's first guess from sum (x/scale)^2 and sum (f0/scale)^2 over numel elements
__device__ __forceinline__ float rk_h0(double sum_x2, double sum_f02, double numel) {
  const float d0 = (float)sqrt(sum_x2 / numel), d1 = (float)sqrt(sum_f02 / numel);
  return (d0 < 1e-5f || d1 < 1e-5f) ? 1e-6f : 0.01f * d0 / d1;
}

// the rest of the initial step once f1 = f(t0 + h0, x + h0 f0) is known (sum_df2 = sum ((f1 - f0)/scale)^2), then
// the pre-step of the first step
__device__ __forceinline__ void rk_init_step(cfm_rk_state& s, float h0, double sum_f02, double sum_df2, double numel,
                                             const float* t_span) {
  const float d1 = (float)sqrt(sum_f02 / numel);
  const float d2 = (float)sqrt(sum_df2 / numel) / h0;
  float h1;
  if (d1 <= 1e-15f && d2 <= 1e-15f) h1 = fmaxf(1e-6f, h0 * 1e-3f);
  else h1 = powf(0.01f / fmaxf(d1, d2), 1.f / 6.f);
  s.dt = fminf(100.f * h0, h1);
  s.dt_old = h0;
  s.nfe += 2;
  s.ckpt = 1;
  s.ckpt_flag = 0;
  s.done = 0;
  rk_prestep(s, t_span);
}

// After a step attempt with error norm `ratio`: accept/reject, checkpoint bookkeeping (save_slot >= 0: the new state
// is t_span[save_slot]'s record), adapt_step(safety .9, min .2, max 10, order 5) and the pre-step of the next step.
// Returns whether the step was accepted.
__device__ __forceinline__ bool rk_control(cfm_rk_state& s, float ratio, const float* t_span) {
  s.ratio = ratio;
  s.nfe += 6;
  const bool accept = ratio <= 1.f;
  s.save_slot = -1;
  if (accept) {
    float tn = s.t + s.dt;
    // torchdyn records a checkpoint when t + dt == t_span[ckpt]; a step that was clipped to land
    // on the checkpoint is snapped onto it so fp32 rounding of t + (t_ckpt - t) cannot miss it
    if (s.ckpt < s.n_span && (tn == __ldg(t_span + s.ckpt) || s.ckpt_flag)) {
      tn = __ldg(t_span + s.ckpt);
      s.save_slot = s.ckpt;
      s.ckpt++;
    }
    s.t = tn;
    s.accepted++;
  } else {
    s.rejected++;
  }
  float dt = s.dt;
  if (s.ckpt_flag) { dt = s.dt_old - dt; s.ckpt_flag = 0; }
  if (ratio == 0.f) {
    dt = dt * 10.f;
  } else {
    const float min_factor = ratio < 1.f ? 1.f : 0.2f;
    const float factor = fminf(10.f, fmaxf(0.9f / powf(ratio, 0.2f), min_factor));
    dt = dt * factor;
  }
  s.dt = dt;
  rk_prestep(s, t_span);
  return accept;
}

}  // namespace cfm
