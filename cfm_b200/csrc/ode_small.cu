// Whole-trajectory ODE sampling for SMALL vector-field MLPs in ONE cooperative launch (SURVEY.md 8 f-2).
//
// Reference call sites: examples/2D_tutorials/tutorial_training_8_gaussians_to_moons.ipynb:332-338
// (NeuralODE(torch_wrapper(MLP(dim=2, w=64, time_varying=True)), solver="dopri5", atol=rtol=1e-4)
// .trajectory(x, linspace(0, 1, 100)) on 1024 samples) and runner/src/models/components/solver.py:184-199.
// At that size one MLP forward is a microsecond of arithmetic, so the multi-kernel driver (ode.py +
// rk.cu: ~15 launches per step) is launch-latency-bound (~15 launch latencies per step).  Here
// the whole integration -- Hairer initial step, every dopri5 stage, the 6 MLP evaluations per step,
// the global error norm, the step controller, FSAL and the checkpoint writes -- runs in one
// persistent kernel:
//
//   * weights (<= ~100 KB) are staged once in shared memory, transposed so that lane l owns hidden
//     units U*l .. U*l+U-1 (w = 32*U) and reads its weights with one conflict-free LDS per input;
//   * one warp integrates TWO sample rows at a time (register blocking: every weight read from shared
//     memory feeds two FMAs -- with one row per warp the kernel was bound by shared-memory bandwidth,
//     every warp streaming the full 32 KB of hidden weights per evaluation); a warp owns
//     rows_per_warp rows, whose x, k1..k7 and xnew live in shared memory for the whole trajectory --
//     HBM is touched only for x0 and for the recorded t_span points;
//   * the controller is replicated: every thread evaluates the same scalar accept/reject logic
//     (torchdyn's, rk_control.cuh, shared with rk.cu) from the same grid-wide error sum, so the only grid-level
//     communication is ONE deterministic all-reduce (per-CTA partials -> grid barrier -> every CTA
//     folds the partials in the same order) per step;
//   * solver = euler needs no barrier at all.
//
// Tried and dropped (no faster per C1 trajectory, so the simpler form stays): one row per warp with twice
// the warps (shared-memory bandwidth-bound: every warp streams all 32 KB of hidden weights per evaluation), and
// a K-split variant in which four warps share a row pair (a quarter of every layer's inputs each, partial sums
// met behind 128-thread named barriers: 5x fewer instructions per warp, but four barriers per evaluation and the
// Runge-Kutta arithmetic of a 2-D state serialised in one warp ate the gain).
//
// CNF variant (CNF = true; the exact-likelihood field of cnf_wrapper, DESIGN.md section 3.8): the state row is
// [x, ll] (dim + 1 floats) and the field is [f(t, x), tr(df/dx)].  mlp_eval carries dim forward-mode tangents
// T_k = dh/dx_k next to the activations: registers for the lane's own units, the per-warp hidden buffers for
// layer inputs (hbuf grows by 1 + dim).  The f part runs exactly the instructions of the plain variant, so the
// x columns are bit-identical to it; the trace costs about dim more forwards per evaluation.
#include <cooperative_groups.h>
#include <curand_philox4x32_x.h>

#include "mlp_common.cuh"
#include "rk_control.cuh"
#include "rk_tableau.h"

namespace cg = cooperative_groups;

namespace cfm {

namespace {

__constant__ float kC[7] = CFM_RK_C_INIT;
__constant__ float kA[7][6] = CFM_RK_A_INIT;
__constant__ float kE[7] = CFM_RK_E_INIT;

struct OdeSmallParams {
  const float *W0, *b0, *W1, *b1, *W2, *b2, *W3, *b3;  // torch Linear layout [out][in]
  int dim, w, tv, act;
  const float* x0;
  int64_t B;
  const float* t_span;
  int n_span;
  float atol, rtol;
  int solver;  // 0 dopri5, 1 euler
  float* traj;  // [n_span][B][dim] ([n_span][B][dim + 1] for the CNF variant; so is x0)
  cfm_rk_state* st;
  double* partials;  // [2][3][gridDim.x]
  int rows_per_warp;
  int max_steps;
};

constexpr int kSlots = 9;  // x, k1..k7, xnew
constexpr int RB = 2;      // rows evaluated together by one warp

struct SmemPlan {
  int dimp;
  size_t wt0, wtime, b0, wt1, b1, wt2, b2, wt3, b3, hbuf, xin, state, red, total;  // float offsets / bytes
};
// cnf: the state row has dim + 1 columns and each hidden buffer row carries dim tangent rows after it
__host__ __device__ inline SmemPlan ode_small_plan(int dim, int w, int nwarps, int rpw, bool cnf = false) {
  SmemPlan s;
  s.dimp = (dim + (cnf ? 1 : 0) + 3) / 4 * 4;
  size_t o = 0;
  auto take = [&](size_t n) { size_t r = o; o += (n + 3) / 4 * 4; return r; };
  s.wt0 = take((size_t)dim * w);
  s.wtime = take(w);
  s.b0 = take(w);
  s.wt1 = take((size_t)w * w);
  s.b1 = take(w);
  s.wt2 = take((size_t)w * w);
  s.b2 = take(w);
  s.wt3 = take((size_t)w * dim);
  s.b3 = take(dim);
  s.hbuf = take((size_t)nwarps * RB * 2 * w * (cnf ? 1 + dim : 1));
  s.xin = take((size_t)nwarps * RB * s.dimp);
  s.state = take((size_t)nwarps * rpw * kSlots * s.dimp);
  s.red = take(2 * 3 * 32 + 8);  // doubles: 3 x 32 per-warp partials + 3 totals
  s.total = o * sizeof(float);
  return s;
}

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

// One MLP evaluation f(t, x) for RB rows at once: x_r = xin0 / xin1 -> out0 / out1 (shared memory, dim
// floats each).  hA, hB: per-warp hidden buffers, [RB][W] each.
// CNF: out_r also receives div_r = tr(df/dx) at [dim]; hA, hB are [RB][W] activations followed by [RB][dim][W]
// tangents, and dim <= 8 (the layer-3 branch that ends in a warp reduction).
// Deliberately NOT inlined and with rolled loops: the kernel runs 1-2 warps per scheduler, and
// straight-line code of a few thousand instructions would not stay in the instruction cache.
// Copy: the SDE kernel calls its own instantiation (Copy = 1, same source).  With one instantiation shared between
// both kernels ptxas compiled the ODE kernels' call sites differently; with two, their code is exactly what it was.
template <int U, bool CNF, int Copy = 0>
__device__ __noinline__ void mlp_eval(const float* __restrict__ sm, const SmemPlan& pl, int dim, int tv, int act,
                                      const float* xin0, const float* xin1, float t, float* hA, float* hB,
                                      float* out0, float* out1, int lane) {
  constexpr int W = 32 * U;
  const int u0 = U * lane;
  float acc[RB][U], wv[U];
  [[maybe_unused]] float dact[RB][U];        // CNF: act'(pre-activation) of this lane's units
  [[maybe_unused]] float dv[RB] = {0.f, 0.f};  // CNF: this lane's share of the divergence
  // layer 0: dim (+ time) -> W
  lds_units<U>(sm + pl.b0 + u0, acc[0]);
  if (tv) {
    lds_units<U>(sm + pl.wtime + u0, wv);
#pragma unroll
    for (int q = 0; q < U; ++q) acc[0][q] = fmaf(t, wv[q], acc[0][q]);
  }
#pragma unroll
  for (int q = 0; q < U; ++q) acc[1][q] = acc[0][q];
#pragma unroll 2
  for (int i = 0; i < dim; ++i) {
    const float xa = xin0[i], xb = xin1[i];
    lds_units<U>(sm + pl.wt0 + (size_t)i * W + u0, wv);
#pragma unroll
    for (int q = 0; q < U; ++q) {
      acc[0][q] = fmaf(wv[q], xa, acc[0][q]);
      acc[1][q] = fmaf(wv[q], xb, acc[1][q]);
    }
  }
#pragma unroll
  for (int r = 0; r < RB; ++r) {
    if constexpr (CNF) {
#pragma unroll
      for (int q = 0; q < U; ++q) dact[r][q] = act_deriv_fast(acc[r][q], act);
    }
#pragma unroll
    for (int q = 0; q < U; ++q) acc[r][q] = act_apply_fast(acc[r][q], act);
    sts_units<U>(hA + r * W + u0, acc[r]);
  }
  if constexpr (CNF) {
    // layer-0 tangents: T_k = act'(pre0) * W0x[:, k] (the time column does not depend on x)
    for (int k = 0; k < dim; ++k) {
      lds_units<U>(sm + pl.wt0 + (size_t)k * W + u0, wv);
#pragma unroll
      for (int r = 0; r < RB; ++r) {
        float tk[U];
#pragma unroll
        for (int q = 0; q < U; ++q) tk[q] = dact[r][q] * wv[q];
        sts_units<U>(hA + (RB + r * dim + k) * W + u0, tk);
      }
    }
  }
  __syncwarp();
  // layers 1, 2: W -> W
#pragma unroll 1
  for (int layer = 0; layer < 2; ++layer) {
    const float* wt = sm + (layer == 0 ? pl.wt1 : pl.wt2);
    const float* bb = sm + (layer == 0 ? pl.b1 : pl.b2);
    const float* hin = layer == 0 ? hA : hB;
    float* hout = layer == 0 ? hB : hA;
    lds_units<U>(bb + u0, acc[0]);
#pragma unroll
    for (int q = 0; q < U; ++q) acc[1][q] = acc[0][q];
#pragma unroll 2
    for (int i = 0; i < W; i += 4) {
      const float4 ha = *reinterpret_cast<const float4*>(hin + i);
      const float4 hb = *reinterpret_cast<const float4*>(hin + W + i);
      const float hs[RB][4] = {{ha.x, ha.y, ha.z, ha.w}, {hb.x, hb.y, hb.z, hb.w}};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        lds_units<U>(wt + (size_t)(i + c) * W + u0, wv);
#pragma unroll
        for (int q = 0; q < U; ++q) {
          acc[0][q] = fmaf(wv[q], hs[0][c], acc[0][q]);
          acc[1][q] = fmaf(wv[q], hs[1][c], acc[1][q]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      if constexpr (CNF) {
#pragma unroll
        for (int q = 0; q < U; ++q) dact[r][q] = act_deriv_fast(acc[r][q], act);
      }
#pragma unroll
      for (int q = 0; q < U; ++q) acc[r][q] = act_apply_fast(acc[r][q], act);
      sts_units<U>(hout + r * W + u0, acc[r]);
    }
    if constexpr (CNF) {
      // tangents: T_k <- act'(pre) * (W T_k), one weight pass per input direction k
      for (int k = 0; k < dim; ++k) {
        const float* ta = hin + (RB + k) * W;
        const float* tb = hin + (RB + dim + k) * W;
        float tk[RB][U];
#pragma unroll
        for (int r = 0; r < RB; ++r)
#pragma unroll
          for (int q = 0; q < U; ++q) tk[r][q] = 0.f;
#pragma unroll 2
        for (int i = 0; i < W; i += 4) {
          const float4 va = *reinterpret_cast<const float4*>(ta + i);
          const float4 vb = *reinterpret_cast<const float4*>(tb + i);
          const float ts[RB][4] = {{va.x, va.y, va.z, va.w}, {vb.x, vb.y, vb.z, vb.w}};
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            lds_units<U>(wt + (size_t)(i + c) * W + u0, wv);
#pragma unroll
            for (int q = 0; q < U; ++q) {
              tk[0][q] = fmaf(wv[q], ts[0][c], tk[0][q]);
              tk[1][q] = fmaf(wv[q], ts[1][c], tk[1][q]);
            }
          }
        }
#pragma unroll
        for (int r = 0; r < RB; ++r)
#pragma unroll
          for (int q = 0; q < U; ++q) tk[r][q] *= dact[r][q];
        if (layer == 0) {
#pragma unroll
          for (int r = 0; r < RB; ++r) sts_units<U>(hout + (RB + r * dim + k) * W + u0, tk[r]);
        } else {
          // last hidden layer: only (W3 T_k)_k enters the trace, so fold row k of W3 in here
#pragma unroll
          for (int q = 0; q < U; ++q) {
            const float w3 = sm[pl.wt3 + (size_t)(u0 + q) * dim + k];
            dv[0] = fmaf(w3, tk[0][q], dv[0]);
            dv[1] = fmaf(w3, tk[1][q], dv[1]);
          }
        }
      }
    }
    __syncwarp();
  }
  // layer 3: W -> dim (h2 is in hA; this lane's own units are still in acc)
  if (dim <= 8) {
    for (int e = 0; e < dim; ++e) {
      float pa = 0.f, pb = 0.f;
#pragma unroll
      for (int q = 0; q < U; ++q) {
        const float w3 = sm[pl.wt3 + (size_t)(u0 + q) * dim + e];
        pa = fmaf(w3, acc[0][q], pa);
        pb = fmaf(w3, acc[1][q], pb);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {  // two interleaved butterfly reductions
        pa += __shfl_xor_sync(0xffffffffu, pa, o);
        pb += __shfl_xor_sync(0xffffffffu, pb, o);
      }
      if (lane == 0) {
        const float b3 = sm[pl.b3 + e];
        out0[e] = pa + b3;
        out1[e] = pb + b3;
      }
    }
    if constexpr (CNF) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        dv[0] += __shfl_xor_sync(0xffffffffu, dv[0], o);
        dv[1] += __shfl_xor_sync(0xffffffffu, dv[1], o);
      }
      if (lane == 0) {
        out0[dim] = dv[0];
        out1[dim] = dv[1];
      }
    }
  } else {
    for (int e = lane; e < dim; e += 32) {
      float a0 = sm[pl.b3 + e], a1 = a0;
#pragma unroll 2
      for (int i = 0; i < W; i += 4) {
        const float4 ha = *reinterpret_cast<const float4*>(hA + i);
        const float4 hb = *reinterpret_cast<const float4*>(hA + W + i);
        const float w0 = sm[pl.wt3 + (size_t)i * dim + e], w1 = sm[pl.wt3 + (size_t)(i + 1) * dim + e];
        const float w2 = sm[pl.wt3 + (size_t)(i + 2) * dim + e], w3 = sm[pl.wt3 + (size_t)(i + 3) * dim + e];
        a0 = fmaf(w0, ha.x, a0); a1 = fmaf(w0, hb.x, a1);
        a0 = fmaf(w1, ha.y, a0); a1 = fmaf(w1, hb.y, a1);
        a0 = fmaf(w2, ha.z, a0); a1 = fmaf(w2, hb.z, a1);
        a0 = fmaf(w3, ha.w, a0); a1 = fmaf(w3, hb.w, a1);
      }
      out0[e] = a0;
      out1[e] = a1;
    }
  }
  __syncwarp();
}

// Deterministic grid-wide sum of NV doubles: every thread of every CTA returns the same bits.
template <int NV>
__device__ __noinline__ void grid_sum(cg::grid_group& grid, double (&v)[NV], double* partials, int buf, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int G = gridDim.x;
#pragma unroll
  for (int q = 0; q < NV; ++q) {
    const double s = warp_sum(v[q]);
    if (lane == 0) red[q * 32 + warp] = s;
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int q = 0; q < NV; ++q) {
      double s = lane < nwarps ? red[q * 32 + lane] : 0.0;
      s = warp_sum(s);
      if (lane == 0) partials[((size_t)buf * 3 + q) * G + blockIdx.x] = s;
    }
  }
  __threadfence();
  grid.sync();
  if (warp == 0) {
#pragma unroll
    for (int q = 0; q < NV; ++q) {
      double s = 0.0;
      for (int c = lane; c < G; c += 32) s += __ldcg(partials + ((size_t)buf * 3 + q) * G + c);
      s = warp_sum(s);
      if (lane == 0) red[96 + q] = s;
    }
  }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < NV; ++q) v[q] = red[96 + q];
  __syncthreads();  // red is reused by the next call
}

template <int U, int MAXT, bool CNF>
__global__ void __launch_bounds__(MAXT, 1) ode_small_kernel(const OdeSmallParams p) {
  constexpr int W = 32 * U;
  extern __shared__ __align__(16) float sm[];
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int dim = p.dim, tv = p.tv, act = p.act, rpw = p.rows_per_warp;
  const int sw = CNF ? dim + 1 : dim;  // state columns: x (and the log-density column ll)
  const SmemPlan pl = ode_small_plan(dim, W, nwarps, rpw, CNF);
  const int dimp = pl.dimp;
  const int in0 = dim + tv;

  // ---- stage the weights (transposed: [in][out]) ----
  for (int idx = tid; idx < W * dim; idx += blockDim.x) {
    const int u = idx / dim, i = idx % dim;
    sm[pl.wt0 + (size_t)i * W + u] = p.W0[(size_t)u * in0 + i];
  }
  for (int u = tid; u < W; u += blockDim.x) {
    sm[pl.wtime + u] = tv ? p.W0[(size_t)u * in0 + dim] : 0.f;
    sm[pl.b0 + u] = p.b0[u];
    sm[pl.b1 + u] = p.b1[u];
    sm[pl.b2 + u] = p.b2[u];
  }
  for (int idx = tid; idx < W * W; idx += blockDim.x) {
    const int u = idx / W, i = idx % W;
    sm[pl.wt1 + (size_t)i * W + u] = p.W1[idx];
    sm[pl.wt2 + (size_t)i * W + u] = p.W2[idx];
  }
  for (int idx = tid; idx < dim * W; idx += blockDim.x) {
    const int e = idx / W, i = idx % W;
    sm[pl.wt3 + (size_t)i * dim + e] = p.W3[idx];
  }
  for (int e = tid; e < dim; e += blockDim.x) sm[pl.b3 + e] = p.b3[e];

  const int hsz = CNF ? RB * W * (1 + dim) : RB * W;     // one hidden buffer: [RB][W] (+ [RB][dim][W] tangents)
  float* hA = sm + pl.hbuf + (size_t)warp * 2 * hsz;
  float* hB = hA + hsz;
  float* xin = sm + pl.xin + (size_t)warp * RB * dimp;    // [RB][dimp]
  double* red = reinterpret_cast<double*>(sm + pl.red);
  const int64_t gwarp = (int64_t)blockIdx.x * nwarps + warp, wstride = (int64_t)gridDim.x * nwarps;
  // local row j (group j / RB, member j % RB): the RB rows of a group are neighbours in the batch
  auto row_of = [&](int j) -> int64_t { return (gwarp + (int64_t)(j / RB) * wstride) * RB + (j % RB); };
  auto slot = [&](int j, int s) -> float* { return sm + pl.state + (((size_t)warp * rpw + j) * kSlots + s) * dimp; };
  const int64_t B = p.B;
  const double numel = (double)B * (double)sw;

  // ---- x0 -> state (rows past the batch: zeros, integrated along but never stored or counted), traj[0] ----
  for (int j = 0; j < rpw; ++j) {
    const int64_t r = row_of(j);
    for (int e = lane; e < sw; e += 32) {
      const float v = r < B ? p.x0[r * sw + e] : 0.f;
      slot(j, 0)[e] = v;
      if (r < B) p.traj[r * sw + e] = v;
    }
  }
  __syncthreads();

  const int n_span = p.n_span;
  if (p.solver == 1) {
    // ---- euler (torchdyn fixed-step: one step per t_span interval) ----
    for (int n = 0; n + 1 < n_span; ++n) {
      const float t = __ldg(p.t_span + n), h = __ldg(p.t_span + n + 1) - t;
      for (int g = 0; g < rpw; g += RB) {
        if (row_of(g) >= B) break;
        mlp_eval<U, CNF>(sm, pl, dim, tv, act, slot(g, 0), slot(g + 1, 0), t, hA, hB, slot(g, 1), slot(g + 1, 1), lane);
#pragma unroll
        for (int m = 0; m < RB; ++m) {
          const int64_t r = row_of(g + m);
          float* x = slot(g + m, 0);
          const float* k = slot(g + m, 1);
          for (int e = lane; e < sw; e += 32) {
            const float v = fmaf(h, k[e], x[e]);
            x[e] = v;
            if (r < B) p.traj[((int64_t)(n + 1) * B + r) * sw + e] = v;
          }
        }
        __syncwarp();
      }
    }
    if (blockIdx.x == 0 && tid == 0) {
      cfm_rk_state* st = p.st;
      st->t = __ldg(p.t_span + n_span - 1);
      st->done = 1;
      st->nfe = n_span - 1;
      st->accepted = n_span - 1;
      st->rejected = 0;
    }
    return;
  }

  // ---- dopri5 (torchdyn _adaptive_odeint semantics; rk_control.cuh's controller, replicated in every thread) ----
  cfm_rk_state s = {};
  s.atol = p.atol;
  s.rtol = p.rtol;
  s.t = __ldg(p.t_span);
  s.t_end = __ldg(p.t_span + n_span - 1);
  s.n_span = n_span;
  int pbuf = 0;

  {
    // k1 = f(t0, x); Hairer's initial step: d0 = |x/sc|, d1 = |f0/sc|
    double s2[2] = {0.0, 0.0};
    for (int g = 0; g < rpw; g += RB) {
      if (row_of(g) >= B) break;
      mlp_eval<U, CNF>(sm, pl, dim, tv, act, slot(g, 0), slot(g + 1, 0), s.t, hA, hB, slot(g, 1), slot(g + 1, 1),
                       lane);
#pragma unroll
      for (int m = 0; m < RB; ++m) {
        if (row_of(g + m) >= B) continue;
        for (int e = lane; e < sw; e += 32) {
          const float xv = slot(g + m, 0)[e], f0 = slot(g + m, 1)[e];
          const float sc = rk_init_scale(xv, s.atol, s.rtol);
          const float a = xv / sc, b = f0 / sc;
          s2[0] += (double)a * a;
          s2[1] += (double)b * b;
        }
      }
    }
    grid_sum<2>(grid, s2, p.partials, pbuf, red);
    pbuf ^= 1;
    const float h0 = rk_h0(s2[0], s2[1], numel);
    double s1[1] = {0.0};
    for (int g = 0; g < rpw; g += RB) {
      if (row_of(g) >= B) break;
#pragma unroll
      for (int m = 0; m < RB; ++m)
        for (int e = lane; e < sw; e += 32) xin[m * dimp + e] = fmaf(h0, slot(g + m, 1)[e], slot(g + m, 0)[e]);
      __syncwarp();
      mlp_eval<U, CNF>(sm, pl, dim, tv, act, xin, xin + dimp, s.t + h0, hA, hB, slot(g, 2), slot(g + 1, 2), lane);
#pragma unroll
      for (int m = 0; m < RB; ++m) {
        if (row_of(g + m) >= B) continue;
        for (int e = lane; e < sw; e += 32) {
          const float sc = rk_init_scale(slot(g + m, 0)[e], s.atol, s.rtol);
          const float q = (slot(g + m, 2)[e] - slot(g + m, 1)[e]) / sc;
          s1[0] += (double)q * q;
        }
      }
    }
    grid_sum<1>(grid, s1, p.partials, pbuf, red);
    pbuf ^= 1;
    rk_init_step(s, h0, s2[1], s1[0], numel, p.t_span);
  }

  int steps = 0;
  while (!s.done && steps < p.max_steps) {
    ++steps;
    double es[1] = {0.0};
    for (int g = 0; g < rpw; g += RB) {
      if (row_of(g) >= B) break;
#pragma unroll 1
      for (int stage = 1; stage <= 6; ++stage) {
        float a[6];
#pragma unroll
        for (int q = 0; q < 6; ++q) a[q] = s.dt * kA[stage][q];
        float* d0p = stage < 6 ? xin : slot(g, 8);
        float* d1p = stage < 6 ? xin + dimp : slot(g + 1, 8);
#pragma unroll
        for (int m = 0; m < RB; ++m) {
          float* dst = m == 0 ? d0p : d1p;
          const float* x = slot(g + m, 0);
          for (int e = lane; e < sw; e += 32) {
            float v = x[e];
#pragma unroll
            for (int q = 0; q < 6; ++q)
              if (q < stage && kA[stage][q] != 0.f) v = fmaf(a[q], slot(g + m, 1 + q)[e], v);
            dst[e] = v;
          }
        }
        __syncwarp();
        mlp_eval<U, CNF>(sm, pl, dim, tv, act, d0p, d1p, s.t + kC[stage] * s.dt, hA, hB, slot(g, 1 + stage),
                    slot(g + 1, 1 + stage), lane);
      }
#pragma unroll
      for (int m = 0; m < RB; ++m) {
        if (row_of(g + m) >= B) continue;
        const float* x = slot(g + m, 0);
        for (int e = lane; e < sw; e += 32) {
          float er = 0.f;
#pragma unroll
          for (int q = 0; q < 7; ++q)
            if (kE[q] != 0.f) er = fmaf(kE[q], slot(g + m, 1 + q)[e], er);
          er *= s.dt;
          const float rr = er / rk_err_tol(x[e], slot(g + m, 8)[e], s.atol, s.rtol);
          es[0] += (double)rr * (double)rr;
        }
      }
    }
    grid_sum<1>(grid, es, p.partials, pbuf, red);
    pbuf ^= 1;
    const bool accept = rk_control(s, (float)sqrt(es[0] / numel), p.t_span);
    // ---- commit: x <- xnew, k1 <- k7 (FSAL), checkpoint ----
    if (accept) {
      for (int j = 0; j < rpw; ++j) {
        const int64_t r = row_of(j);
        if (r >= B) break;
        for (int e = lane; e < sw; e += 32) {
          const float v = slot(j, 8)[e];
          slot(j, 0)[e] = v;
          slot(j, 1)[e] = slot(j, 7)[e];
          if (s.save_slot >= 0) p.traj[((int64_t)s.save_slot * B + r) * sw + e] = v;
        }
      }
      __syncwarp();
    }
  }
  if (blockIdx.x == 0 && tid == 0) {
    s.save_slot = -1;  // every checkpoint is already in traj
    *p.st = s;
  }
}

struct Launch {
  int grid, nwarps, rpw;
  size_t smem;
};

// CNF: at most this many warps per CTA.  With the tangent loops the kernel spills at the 128 registers per thread
// that 512-thread launch bounds leave, and not at 256 threads (ptxas -v).
constexpr int kCnfMaxWarps = 8;

template <int U>
int plan_launch(int64_t B, int dim, bool cnf, Launch* out) {
  const int sms = sm_count();
  const int64_t groups = (B + RB - 1) / RB;  // a warp integrates RB rows at a time
  const int max_warps = cnf ? kCnfMaxWarps : 32;
  int64_t grid = 0, gpw = 0;
  auto shape = [&](int nwarps) {
    grid = (groups + nwarps - 1) / nwarps;
    if (grid > sms) grid = sms;
    const int64_t per = grid * nwarps;
    gpw = (groups + per - 1) / per;  // groups per warp
  };
  int nwarps = 4;
  for (;; nwarps *= 2) {  // prefer more warps per CTA over several groups per warp
    shape(nwarps);
    if (gpw == 1 || nwarps == max_warps) break;
  }
  for (;;) {
    if (gpw > (1 << 19)) return 0;
    const SmemPlan pl = ode_small_plan(dim, 32 * U, nwarps, (int)gpw * RB, cnf);
    if (pl.total <= 200 * 1024) {
      out->grid = (int)grid; out->nwarps = nwarps; out->rpw = (int)gpw * RB; out->smem = pl.total;
      return 1;
    }
    // CNF: the tangent buffers grow with the warps per CTA while the per-CTA row state does not, so fewer warps
    // with more row groups each may still fit -- down to one warp, which w = 128 with dim 7 or 8 needs at any batch
    if (!cnf || nwarps == 1) return 0;
    nwarps /= 2;
    shape(nwarps);
  }
}

int plan_any(int64_t B, int dim, int w, Launch* out, bool cnf = false) {
  if (B <= 0 || dim <= 0 || dim > 1024) return 0;
  if (cnf && dim > 8) return 0;  // the exact trace takes the layer-3 branch that ends in a warp reduction
  if (w == 32) return plan_launch<1>(B, dim, cnf, out);
  if (w == 64) return plan_launch<2>(B, dim, cnf, out);
  if (w == 128) return plan_launch<4>(B, dim, cnf, out);
  return 0;
}

template <int U, int MAXT, bool CNF>
int launch_t(const OdeSmallParams& p, const Launch& L, cudaStream_t s) {
  const void* kern = (const void*)ode_small_kernel<U, MAXT, CNF>;
  CFM_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.smem));
  int per_sm = 0;
  CFM_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, L.nwarps * 32, L.smem));
  CFM_REQUIRE(per_sm >= 1 && L.grid <= per_sm * sm_count(), "ode_small: the grid is not co-resident");
  void* args[] = {const_cast<OdeSmallParams*>(&p)};
  CFM_CUDA_OK(cudaLaunchCooperativeKernel(kern, dim3(L.grid), dim3(L.nwarps * 32), args, L.smem, s));
  note_launches(1);
  return CFM_OK;
}
// No 1024-thread instantiation for w = 128: at 32 warps W1, W2 (128 KB) and the hidden buffers (64 KB) plus the row
// state exceed the planner's 200 KB, so plan_launch never returns such a launch.
template <int U>
int launch(const OdeSmallParams& p, const Launch& L, cudaStream_t s) {
  if (L.nwarps <= 8) return launch_t<U, 256, false>(p, L, s);
  if (L.nwarps <= 16) return launch_t<U, 512, false>(p, L, s);
  if constexpr (U < 4) {
    return launch_t<U, 1024, false>(p, L, s);
  } else {
    CFM_REQUIRE(false, "ode_small: %d warps per CTA at w = 128 (the planner gives at most 16)", L.nwarps);
  }
}
template <int U>
int launch_cnf(const OdeSmallParams& p, const Launch& L, cudaStream_t s) {
  static_assert(kCnfMaxWarps <= 8, "the CNF variant is instantiated for 256-thread CTAs only");
  return launch_t<U, 256, true>(p, L, s);
}

int trajectory(bool cnf, const char* what, const float* W0, const float* b0, const float* W1, const float* b1,
               const float* W2, const float* b2, const float* W3, const float* b3, int dim, int w, int time_varying,
               int act, const float* x0, int64_t batch, const float* t_span, int n_span, float atol, float rtol,
               int solver, float* traj, cfm_rk_state* state_out, void* workspace, size_t workspace_bytes,
               void* stream) {
  CFM_REQUIRE(W0 && b0 && W1 && b1 && W2 && b2 && W3 && b3 && x0 && t_span && traj && state_out && workspace,
              "%s: null pointer", what);
  CFM_REQUIRE(n_span >= 2 && (solver == 0 || solver == 1) && (act == CFM_ACT_SELU || act == CFM_ACT_SILU),
              "%s: bad argument", what);
  CFM_REQUIRE(workspace_bytes >= cfm_ode_small_workspace_bytes(batch, dim, w), "%s: workspace too small", what);
  Launch L;
  CFM_REQUIRE(plan_any(batch, dim, w, &L, cnf), "%s: unsupported shape B=%lld dim=%d w=%d", what, (long long)batch,
              dim, w);
  OdeSmallParams p;
  p.W0 = W0; p.b0 = b0; p.W1 = W1; p.b1 = b1; p.W2 = W2; p.b2 = b2; p.W3 = W3; p.b3 = b3;
  p.dim = dim; p.w = w; p.tv = time_varying ? 1 : 0; p.act = act;
  p.x0 = x0; p.B = batch; p.t_span = t_span; p.n_span = n_span; p.atol = atol; p.rtol = rtol;
  p.solver = solver; p.traj = traj; p.st = state_out; p.partials = reinterpret_cast<double*>(workspace);
  p.rows_per_warp = L.rpw; p.max_steps = 1000000;
  cudaStream_t s = (cudaStream_t)stream;
  CFM_CUDA_OK(cudaMemsetAsync(state_out, 0, sizeof(cfm_rk_state), s));
  if (cnf) {
    if (w == 32) return launch_cnf<1>(p, L, s);
    if (w == 64) return launch_cnf<2>(p, L, s);
    return launch_cnf<4>(p, L, s);
  }
  if (w == 32) return launch<1>(p, L, s);
  if (w == 64) return launch<2>(p, L, s);
  return launch<4>(p, L, s);
}

// ==== Schrodinger-bridge SDE sampling: fixed-step Euler-Maruyama, dy = [drift(t, y) + score(t, y)] dt + sigma dW ====
// Two MLPs (drift, score) of the same shape, evaluated by mlp_eval<U, false> one after the other from two weight sets
// staged side by side in shared memory.  The step grid is the same scalar sequence in every thread and rows are
// independent, so there is no grid barrier and the launch is an ordinary one.  Outputs are linear interpolations
// between the states before and after the step that brackets them (torchsde's linear_interp); the host tabulates,
// per step, which outputs it brackets and their two weights.

struct SdeSmallParams {
  const float *W0[2], *b0[2], *W1[2], *b1[2], *W2[2], *b2[2], *W3[2], *b3[2];  // [0] drift, [1] score; [out][in]
  int dim, act;
  float sigma;
  const float* x0;
  int64_t B;
  const float* grid;       // [n_steps + 1] step times
  int n_steps;
  const int* out_begin;    // [n_steps + 1]: step n brackets outputs out_begin[n] .. out_begin[n + 1] - 1 (all >= 1)
  const float* out_a;      // [n_out] weight of the state before the bracketing step
  const float* out_b;      // [n_out] weight of the state after it
  uint64_t seed;
  const float* dw;         // nullable: [n_steps][B][dim] Brownian increments instead of the device stream
  float* traj;             // [n_out][B][dim]
  int rows_per_warp;
};

constexpr int kSdeSlots = 4;  // y, y before the last step, drift(t, y), score(t, y)

struct SdePlan {
  SmemPlan net;  // offsets of ONE weight set (net.dimp: padded row length); the score set starts `set2` floats later
  size_t set2, hbuf, state, total;
};
__host__ __device__ inline SdePlan sde_small_plan(int dim, int w, int nwarps, int rpw) {
  SdePlan s;
  s.net = ode_small_plan(dim, w, 0, 0);  // with no warps nothing is laid out after b3: hbuf = one weight set's floats
  s.set2 = s.net.hbuf;
  size_t o = 2 * s.set2;
  s.hbuf = o;
  o += (size_t)nwarps * RB * 2 * w;
  s.state = o;
  o += (size_t)nwarps * rpw * kSdeSlots * s.net.dimp;
  s.total = o * sizeof(float);
  return s;
}

// Standard normal of (step n, row r, column c): one Philox4x32-10 block per 4 columns, 24-bit uniforms in (0, 1),
// Box-Muller on (u0, u1) for columns 4q, 4q + 1 and on (u2, u3) for 4q + 2, 4q + 3.  Depends on nothing else.
__device__ __forceinline__ float sde_normal(uint64_t seed, int n, int64_t r, int c) {
  const uint4 x = curand_Philox4x32_10(
      make_uint4((unsigned)(c >> 2), (unsigned)(uint64_t)r, (unsigned)((uint64_t)r >> 32), (unsigned)n),
      make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
  const bool hi = c & 2;
  const unsigned xa = hi ? x.z : x.x, xb = hi ? x.w : x.y;
  const float ua = __fmaf_rn((float)(xa >> 8), 0x1p-24f, 0x1p-25f);  // exact: 24-bit integer * 2^-24 + 2^-25
  const float ub = __fmaf_rn((float)(xb >> 8), 0x1p-24f, 0x1p-25f);
  float s, co;
  sincospif(2.f * ub, &s, &co);
  return sqrtf(-2.f * logf(ua)) * ((c & 1) ? s : co);
}

template <int U, int MAXT>
__global__ void __launch_bounds__(MAXT, 1) sde_small_kernel(const SdeSmallParams p) {
  constexpr int W = 32 * U;
  extern __shared__ __align__(16) float sm[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int dim = p.dim, act = p.act, rpw = p.rows_per_warp, in0 = dim + 1;
  const SdePlan pl = sde_small_plan(dim, W, nwarps, rpw);
  const SmemPlan& np = pl.net;
  const int dimp = np.dimp;

  // ---- stage both weight sets (transposed, as ode_small_kernel does); the time column is always present ----
#pragma unroll 1
  for (int q = 0; q < 2; ++q) {
    float* ws = sm + q * pl.set2;
    for (int idx = tid; idx < W * dim; idx += blockDim.x) {
      const int u = idx / dim, i = idx % dim;
      ws[np.wt0 + (size_t)i * W + u] = p.W0[q][(size_t)u * in0 + i];
    }
    for (int u = tid; u < W; u += blockDim.x) {
      ws[np.wtime + u] = p.W0[q][(size_t)u * in0 + dim];
      ws[np.b0 + u] = p.b0[q][u];
      ws[np.b1 + u] = p.b1[q][u];
      ws[np.b2 + u] = p.b2[q][u];
    }
    for (int idx = tid; idx < W * W; idx += blockDim.x) {
      const int u = idx / W, i = idx % W;
      ws[np.wt1 + (size_t)i * W + u] = p.W1[q][idx];
      ws[np.wt2 + (size_t)i * W + u] = p.W2[q][idx];
    }
    for (int idx = tid; idx < dim * W; idx += blockDim.x) {
      const int e = idx / W, i = idx % W;
      ws[np.wt3 + (size_t)i * dim + e] = p.W3[q][idx];
    }
    for (int e = tid; e < dim; e += blockDim.x) ws[np.b3 + e] = p.b3[q][e];
  }

  float* hA = sm + pl.hbuf + (size_t)warp * 2 * RB * W;
  float* hB = hA + RB * W;
  const int64_t gwarp = (int64_t)blockIdx.x * nwarps + warp, wstride = (int64_t)gridDim.x * nwarps;
  auto row_of = [&](int j) -> int64_t { return (gwarp + (int64_t)(j / RB) * wstride) * RB + (j % RB); };
  auto slot = [&](int j, int s) -> float* {
    return sm + pl.state + (((size_t)warp * rpw + j) * kSdeSlots + s) * dimp;
  };
  const int64_t B = p.B;

  // ---- y0 -> state (rows past the batch: zeros, integrated along but never stored), traj[0] ----
  for (int j = 0; j < rpw; ++j) {
    const int64_t r = row_of(j);
    for (int e = lane; e < dim; e += 32) {
      const float v = r < B ? p.x0[r * dim + e] : 0.f;
      slot(j, 0)[e] = v;
      if (r < B) p.traj[r * dim + e] = v;
    }
  }
  __syncthreads();

  const float sigma = p.sigma;
  for (int n = 0; n < p.n_steps; ++n) {
    const float t = __ldg(p.grid + n), h = __ldg(p.grid + n + 1) - t;
    const float sh = sqrtf(h);
    const int k0 = __ldg(p.out_begin + n), k1 = __ldg(p.out_begin + n + 1);
    for (int g = 0; g < rpw; g += RB) {
      if (row_of(g) >= B) break;
      mlp_eval<U, false, 1>(sm, np, dim, 1, act, slot(g, 0), slot(g + 1, 0), t, hA, hB, slot(g, 2), slot(g + 1, 2),
                            lane);
      mlp_eval<U, false, 1>(sm + pl.set2, np, dim, 1, act, slot(g, 0), slot(g + 1, 0), t, hA, hB, slot(g, 3),
                         slot(g + 1, 3), lane);
#pragma unroll
      for (int m = 0; m < RB; ++m) {
        const int64_t r = row_of(g + m);
        float* y = slot(g + m, 0);
        float* yp = slot(g + m, 1);
        const float* d = slot(g + m, 2);
        const float* s = slot(g + m, 3);
        for (int e = lane; e < dim; e += 32) {
          float dW = 0.f;
          if (r < B)
            dW = p.dw ? __ldg(p.dw + ((int64_t)n * B + r) * dim + e) : __fmul_rn(sh, sde_normal(p.seed, n, r, e));
          const float y0 = y[e];
          const float y1 = __fadd_rn(fmaf(h, __fadd_rn(d[e], s[e]), y0), __fmul_rn(sigma, dW));
          yp[e] = y0;
          y[e] = y1;
          if (r < B)
            for (int k = k0; k < k1; ++k)
              p.traj[((int64_t)k * B + r) * dim + e] =
                  __fadd_rn(__fmul_rn(__ldg(p.out_a + k), y0), __fmul_rn(__ldg(p.out_b + k), y1));
        }
      }
      __syncwarp();
    }
  }
}

// SDE: at most this many warps per CTA.  At the 64 registers per thread of a 1024-thread launch bound the kernel spills
// (ptxas -v: 36 / 68 bytes at w = 32 / 64), at 512 threads it does not.
constexpr int kSdeMaxWarps = 16;

template <int U>
int plan_sde(int64_t B, int dim, Launch* out) {
  const int sms = sm_count();
  const int64_t groups = (B + RB - 1) / RB;
  int64_t grid = 0, gpw = 0;
  int nwarps = 4;
  for (;; nwarps *= 2) {  // prefer more warps per CTA over several groups per warp, as plan_launch does
    grid = (groups + nwarps - 1) / nwarps;
    if (grid > sms) grid = sms;
    gpw = (groups + grid * nwarps - 1) / (grid * nwarps);
    if (gpw == 1 || nwarps == kSdeMaxWarps) break;
  }
  if (gpw > (1 << 19)) return 0;
  const SdePlan pl = sde_small_plan(dim, 32 * U, nwarps, (int)gpw * RB);
  if (pl.total > 200 * 1024) return 0;
  out->grid = (int)grid; out->nwarps = nwarps; out->rpw = (int)gpw * RB; out->smem = pl.total;
  return 1;
}

int plan_sde_any(int64_t B, int dim, int w, Launch* out) {
  if (B <= 0 || dim <= 0 || dim > 1024) return 0;
  if (w == 32) return plan_sde<1>(B, dim, out);
  if (w == 64) return plan_sde<2>(B, dim, out);
  return 0;  // w = 128: the two W1/W2 pairs alone take 256 KB
}

template <int U, int MAXT>
int launch_sde_t(const SdeSmallParams& p, const Launch& L, cudaStream_t s) {
  const void* kern = (const void*)sde_small_kernel<U, MAXT>;
  CFM_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.smem));
  sde_small_kernel<U, MAXT><<<L.grid, L.nwarps * 32, L.smem, s>>>(p);
  CFM_CUDA_OK(cudaGetLastError());
  note_launches(1);
  return CFM_OK;
}
template <int U>
int launch_sde(const SdeSmallParams& p, const Launch& L, cudaStream_t s) {
  static_assert(kSdeMaxWarps <= 16, "the SDE kernel is instantiated for 256- and 512-thread CTAs only");
  if (L.nwarps <= 8) return launch_sde_t<U, 256>(p, L, s);
  return launch_sde_t<U, 512>(p, L, s);
}

}  // namespace

}  // namespace cfm

using namespace cfm;

extern "C" int cfm_ode_small_supported(int64_t batch, int dim, int w, int out_dim) {
  Launch L;
  return (out_dim == dim) && plan_any(batch, dim, w, &L);
}

extern "C" int cfm_ode_small_cnf_supported(int64_t batch, int dim, int w) {
  Launch L;
  return plan_any(batch, dim, w, &L, true);
}

extern "C" size_t cfm_ode_small_workspace_bytes(int64_t batch, int dim, int w) {
  (void)batch; (void)dim; (void)w;
  return align_up((size_t)2 * 3 * (size_t)sm_count() * sizeof(double), 256);
}

extern "C" int cfm_ode_small_trajectory_f32(const float* W0, const float* b0, const float* W1, const float* b1,
                                            const float* W2, const float* b2, const float* W3, const float* b3,
                                            int dim, int w, int time_varying, int act, const float* x0, int64_t batch,
                                            const float* t_span, int n_span, float atol, float rtol, int solver,
                                            float* traj, cfm_rk_state* state_out, void* workspace,
                                            size_t workspace_bytes, void* stream) {
  return trajectory(false, "cfm_ode_small_trajectory_f32", W0, b0, W1, b1, W2, b2, W3, b3, dim, w, time_varying,
                    act, x0, batch, t_span, n_span, atol, rtol, solver, traj, state_out, workspace, workspace_bytes,
                    stream);
}

extern "C" int cfm_ode_small_cnf_trajectory_f32(const float* W0, const float* b0, const float* W1, const float* b1,
                                                const float* W2, const float* b2, const float* W3, const float* b3,
                                                int dim, int w, int time_varying, int act, const float* x0,
                                                int64_t batch, const float* t_span, int n_span, float atol,
                                                float rtol, int solver, float* traj, cfm_rk_state* state_out,
                                                void* workspace, size_t workspace_bytes, void* stream) {
  return trajectory(true, "cfm_ode_small_cnf_trajectory_f32", W0, b0, W1, b1, W2, b2, W3, b3, dim, w,
                    time_varying, act, x0, batch, t_span, n_span, atol, rtol, solver, traj, state_out, workspace,
                    workspace_bytes, stream);
}

extern "C" int cfm_sde_small_supported(int64_t batch, int dim, int w) {
  Launch L;
  return plan_sde_any(batch, dim, w, &L);
}

extern "C" int cfm_sde_small_euler_f32(const float* const* drift_host, const float* const* score_host, int dim,
                                       int w, int act, float sigma, const float* x0, int64_t batch, const float* grid,
                                       int n_steps, const int* out_begin, const float* out_a, const float* out_b, int n_out,
                                       uint64_t seed, const float* increments, float* traj, void* stream) {
  const char* what = "cfm_sde_small_euler_f32";
  CFM_REQUIRE(drift_host && score_host && x0 && grid && out_begin && out_a && out_b && traj, "%s: null pointer", what);
  for (int i = 0; i < 8; ++i) CFM_REQUIRE(drift_host[i] && score_host[i], "%s: null weight pointer", what);
  CFM_REQUIRE(n_steps >= 1 && n_out >= 2 && (act == CFM_ACT_SELU || act == CFM_ACT_SILU), "%s: bad argument", what);
  Launch L;
  CFM_REQUIRE(plan_sde_any(batch, dim, w, &L), "%s: unsupported shape B=%lld dim=%d w=%d", what, (long long)batch,
              dim, w);
  SdeSmallParams p;
  for (int q = 0; q < 2; ++q) {
    const float* const* n = q == 0 ? drift_host : score_host;
    p.W0[q] = n[0]; p.b0[q] = n[1]; p.W1[q] = n[2]; p.b1[q] = n[3];
    p.W2[q] = n[4]; p.b2[q] = n[5]; p.W3[q] = n[6]; p.b3[q] = n[7];
  }
  p.dim = dim; p.act = act; p.sigma = sigma; p.x0 = x0; p.B = batch;
  p.grid = grid; p.n_steps = n_steps; p.out_begin = out_begin; p.out_a = out_a; p.out_b = out_b;
  p.seed = seed; p.dw = increments; p.traj = traj; p.rows_per_warp = L.rpw;
  cudaStream_t s = (cudaStream_t)stream;
  if (w == 32) return launch_sde<1>(p, L, s);
  return launch_sde<2>(p, L, s);
}
