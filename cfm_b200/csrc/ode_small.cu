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
//     (torchdyn's, as restated in rk.cu) from the same grid-wide error sum, so the only grid-level
//     communication is ONE deterministic all-reduce (per-CTA partials -> grid barrier -> every CTA
//     folds the partials in the same order) per step;
//   * solver = euler needs no barrier at all.
//
// Tried and dropped (no faster per C1 trajectory, so the simpler form stays): one row per warp with twice
// the warps (shared-memory bandwidth-bound: every warp streams all 32 KB of hidden weights per evaluation), and
// a K-split variant in which four warps share a row pair (a quarter of every layer's inputs each, partial sums
// met behind 128-thread named barriers: 5x fewer instructions per warp, but four barriers per evaluation and the
// Runge-Kutta arithmetic of a 2-D state serialised in one warp ate the gain).
#include <cooperative_groups.h>

#include "mlp_common.cuh"

namespace cg = cooperative_groups;

namespace cfm {

namespace {

__constant__ float oC[7] = {0.f, 1.f / 5, 3.f / 10, 4.f / 5, 8.f / 9, 1.f, 1.f};
__constant__ float oA[7][6] = {
    {0, 0, 0, 0, 0, 0},
    {1.f / 5, 0, 0, 0, 0, 0},
    {3.f / 40, 9.f / 40, 0, 0, 0, 0},
    {44.f / 45, -56.f / 15, 32.f / 9, 0, 0, 0},
    {19372.f / 6561, -25360.f / 2187, 64448.f / 6561, -212.f / 729, 0, 0},
    {9017.f / 3168, -355.f / 33, 46732.f / 5247, 49.f / 176, -5103.f / 18656, 0},
    {35.f / 384, 0.f, 500.f / 1113, 125.f / 192, -2187.f / 6784, 11.f / 84}};
__constant__ float oE[7] = {(float)(35.0 / 384 - 1951.0 / 21600), 0.f,
                            (float)(500.0 / 1113 - 22642.0 / 50085),
                            (float)(125.0 / 192 - 451.0 / 720),
                            (float)(-2187.0 / 6784 + 12231.0 / 42400),
                            (float)(11.0 / 84 - 649.0 / 6300), (float)(-1.0 / 60)};

struct OdeSmallParams {
  const float *W0, *b0, *W1, *b1, *W2, *b2, *W3, *b3;  // torch Linear layout [out][in]
  int dim, w, tv, act;
  const float* x0;
  int64_t B;
  const float* t_span;
  int n_span;
  float atol, rtol;
  int solver;  // 0 dopri5, 1 euler
  float* traj;  // [n_span][B][dim]
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
__host__ __device__ inline SmemPlan ode_small_plan(int dim, int w, int nwarps, int rpw) {
  SmemPlan s;
  s.dimp = (dim + 3) / 4 * 4;
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
  s.hbuf = take((size_t)nwarps * RB * 2 * w);
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

// One MLP evaluation f(t, x) for RB rows at once: x_r = xin0 / xin1 -> out0 / out1 (shared memory, dim
// floats each).  hA, hB: per-warp hidden buffers, [RB][W] each.
// Deliberately NOT inlined and with rolled loops: the kernel runs 1-2 warps per scheduler, and
// straight-line code of a few thousand instructions would not stay in the instruction cache.
template <int U>
__device__ __noinline__ void mlp_eval(const float* __restrict__ sm, const SmemPlan& pl, int dim, int tv, int act,
                                      const float* xin0, const float* xin1, float t, float* hA, float* hB,
                                      float* out0, float* out1, int lane) {
  constexpr int W = 32 * U;
  const int u0 = U * lane;
  float acc[RB][U], wv[U];
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
#pragma unroll
    for (int q = 0; q < U; ++q) acc[r][q] = act_apply_fast(acc[r][q], act);
    sts_units<U>(hA + r * W + u0, acc[r]);
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
#pragma unroll
      for (int q = 0; q < U; ++q) acc[r][q] = act_apply_fast(acc[r][q], act);
      sts_units<U>(hout + r * W + u0, acc[r]);
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

template <int U, int MAXT>
__global__ void __launch_bounds__(MAXT, 1) ode_small_kernel(const OdeSmallParams p) {
  constexpr int W = 32 * U;
  extern __shared__ __align__(16) float sm[];
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int dim = p.dim, tv = p.tv, act = p.act, rpw = p.rows_per_warp;
  const SmemPlan pl = ode_small_plan(dim, W, nwarps, rpw);
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

  float* hA = sm + pl.hbuf + (size_t)warp * RB * 2 * W;  // [RB][W]
  float* hB = hA + RB * W;                                // [RB][W]
  float* xin = sm + pl.xin + (size_t)warp * RB * dimp;    // [RB][dimp]
  double* red = reinterpret_cast<double*>(sm + pl.red);
  const int64_t gwarp = (int64_t)blockIdx.x * nwarps + warp, wstride = (int64_t)gridDim.x * nwarps;
  // local row j (group j / RB, member j % RB): the RB rows of a group are neighbours in the batch
  auto row_of = [&](int j) -> int64_t { return (gwarp + (int64_t)(j / RB) * wstride) * RB + (j % RB); };
  auto slot = [&](int j, int s) -> float* { return sm + pl.state + (((size_t)warp * rpw + j) * kSlots + s) * dimp; };
  const int64_t B = p.B;
  const double numel = (double)B * (double)dim;

  // ---- x0 -> state (rows past the batch: zeros, integrated along but never stored or counted), traj[0] ----
  for (int j = 0; j < rpw; ++j) {
    const int64_t r = row_of(j);
    for (int e = lane; e < dim; e += 32) {
      const float v = r < B ? p.x0[r * dim + e] : 0.f;
      slot(j, 0)[e] = v;
      if (r < B) p.traj[r * dim + e] = v;
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
        mlp_eval<U>(sm, pl, dim, tv, act, slot(g, 0), slot(g + 1, 0), t, hA, hB, slot(g, 1), slot(g + 1, 1), lane);
#pragma unroll
        for (int m = 0; m < RB; ++m) {
          const int64_t r = row_of(g + m);
          float* x = slot(g + m, 0);
          const float* k = slot(g + m, 1);
          for (int e = lane; e < dim; e += 32) {
            const float v = fmaf(h, k[e], x[e]);
            x[e] = v;
            if (r < B) p.traj[((int64_t)(n + 1) * B + r) * dim + e] = v;
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

  // ---- dopri5 (torchdyn _adaptive_odeint semantics; scalar controller replicated in every thread) ----
  const float atol = p.atol, rtol = p.rtol;
  float t = __ldg(p.t_span), dt = 0.f, dt_old = 0.f, ratio = 0.f;
  const float t_end = __ldg(p.t_span + n_span - 1);
  int ckpt = 1, ckpt_flag = 0, done = 0, accepted = 0, rejected = 0, nfe = 0, pbuf = 0;

  auto prestep = [&]() {
    if (!(t < t_end)) { done = 1; return; }
    if (t + dt > t_end) dt = t_end - t;
    if (ckpt < n_span && t + dt > __ldg(p.t_span + ckpt)) {
      dt_old = dt;
      ckpt_flag = 1;
      dt = __ldg(p.t_span + ckpt) - t;
    }
  };

  {
    // k1 = f(t0, x); Hairer's initial step: d0 = |x/sc|, d1 = |f0/sc|
    double s2[2] = {0.0, 0.0};
    for (int g = 0; g < rpw; g += RB) {
      if (row_of(g) >= B) break;
      mlp_eval<U>(sm, pl, dim, tv, act, slot(g, 0), slot(g + 1, 0), t, hA, hB, slot(g, 1), slot(g + 1, 1), lane);
#pragma unroll
      for (int m = 0; m < RB; ++m) {
        if (row_of(g + m) >= B) continue;
        for (int e = lane; e < dim; e += 32) {
          const float xv = slot(g + m, 0)[e], f0 = slot(g + m, 1)[e];
          const float sc = atol + fabsf(xv) * rtol;
          const float a = xv / sc, b = f0 / sc;
          s2[0] += (double)a * a;
          s2[1] += (double)b * b;
        }
      }
    }
    grid_sum<2>(grid, s2, p.partials, pbuf, red);
    pbuf ^= 1;
    const float d0 = (float)sqrt(s2[0] / numel), d1 = (float)sqrt(s2[1] / numel);
    const float h0 = (d0 < 1e-5f || d1 < 1e-5f) ? 1e-6f : 0.01f * d0 / d1;
    double s1[1] = {0.0};
    for (int g = 0; g < rpw; g += RB) {
      if (row_of(g) >= B) break;
#pragma unroll
      for (int m = 0; m < RB; ++m)
        for (int e = lane; e < dim; e += 32) xin[m * dimp + e] = fmaf(h0, slot(g + m, 1)[e], slot(g + m, 0)[e]);
      __syncwarp();
      mlp_eval<U>(sm, pl, dim, tv, act, xin, xin + dimp, t + h0, hA, hB, slot(g, 2), slot(g + 1, 2), lane);
#pragma unroll
      for (int m = 0; m < RB; ++m) {
        if (row_of(g + m) >= B) continue;
        for (int e = lane; e < dim; e += 32) {
          const float sc = atol + fabsf(slot(g + m, 0)[e]) * rtol;
          const float q = (slot(g + m, 2)[e] - slot(g + m, 1)[e]) / sc;
          s1[0] += (double)q * q;
        }
      }
    }
    grid_sum<1>(grid, s1, p.partials, pbuf, red);
    pbuf ^= 1;
    const float d2 = (float)sqrt(s1[0] / numel) / h0;
    float h1;
    if (d1 <= 1e-15f && d2 <= 1e-15f) h1 = fmaxf(1e-6f, h0 * 1e-3f);
    else h1 = powf(0.01f / fmaxf(d1, d2), 1.f / 6.f);
    dt = fminf(100.f * h0, h1);
    dt_old = h0;
    nfe = 2;
    prestep();
  }

  int steps = 0;
  while (!done && steps < p.max_steps) {
    ++steps;
    double es[1] = {0.0};
    for (int g = 0; g < rpw; g += RB) {
      if (row_of(g) >= B) break;
#pragma unroll 1
      for (int stage = 1; stage <= 6; ++stage) {
        float a[6];
#pragma unroll
        for (int q = 0; q < 6; ++q) a[q] = dt * oA[stage][q];
        float* d0p = stage < 6 ? xin : slot(g, 8);
        float* d1p = stage < 6 ? xin + dimp : slot(g + 1, 8);
#pragma unroll
        for (int m = 0; m < RB; ++m) {
          float* dst = m == 0 ? d0p : d1p;
          const float* x = slot(g + m, 0);
          for (int e = lane; e < dim; e += 32) {
            float v = x[e];
#pragma unroll
            for (int q = 0; q < 6; ++q)
              if (q < stage && oA[stage][q] != 0.f) v = fmaf(a[q], slot(g + m, 1 + q)[e], v);
            dst[e] = v;
          }
        }
        __syncwarp();
        mlp_eval<U>(sm, pl, dim, tv, act, d0p, d1p, t + oC[stage] * dt, hA, hB, slot(g, 1 + stage),
                    slot(g + 1, 1 + stage), lane);
      }
#pragma unroll
      for (int m = 0; m < RB; ++m) {
        if (row_of(g + m) >= B) continue;
        const float* x = slot(g + m, 0);
        for (int e = lane; e < dim; e += 32) {
          float er = 0.f;
#pragma unroll
          for (int q = 0; q < 7; ++q)
            if (oE[q] != 0.f) er = fmaf(oE[q], slot(g + m, 1 + q)[e], er);
          er *= dt;
          const float tol = atol + rtol * fmaxf(fabsf(x[e]), fabsf(slot(g + m, 8)[e]));
          const float rr = er / tol;
          es[0] += (double)rr * (double)rr;
        }
      }
    }
    grid_sum<1>(grid, es, p.partials, pbuf, red);
    pbuf ^= 1;
    // ---- controller (rk.cu rk_control_kernel, torchdyn order) ----
    ratio = (float)sqrt(es[0] / numel);
    nfe += 6;
    const bool accept = ratio <= 1.f;
    int save_slot = -1;
    if (accept) {
      float tn = t + dt;
      if (ckpt < n_span && (tn == __ldg(p.t_span + ckpt) || ckpt_flag)) {
        tn = __ldg(p.t_span + ckpt);
        save_slot = ckpt;
        ckpt++;
      }
      t = tn;
      accepted++;
    } else {
      rejected++;
    }
    float ndt = dt;
    if (ckpt_flag) { ndt = dt_old - dt; ckpt_flag = 0; }
    if (ratio == 0.f) {
      ndt = ndt * 10.f;
    } else {
      const float min_factor = ratio < 1.f ? 1.f : 0.2f;
      const float factor = fminf(10.f, fmaxf(0.9f / powf(ratio, 0.2f), min_factor));
      ndt = ndt * factor;
    }
    dt = ndt;
    prestep();
    // ---- commit: x <- xnew, k1 <- k7 (FSAL), checkpoint ----
    if (accept) {
      for (int j = 0; j < rpw; ++j) {
        const int64_t r = row_of(j);
        if (r >= B) break;
        for (int e = lane; e < dim; e += 32) {
          const float v = slot(j, 8)[e];
          slot(j, 0)[e] = v;
          slot(j, 1)[e] = slot(j, 7)[e];
          if (save_slot >= 0) p.traj[((int64_t)save_slot * B + r) * dim + e] = v;
        }
      }
      __syncwarp();
    }
  }
  if (blockIdx.x == 0 && tid == 0) {
    cfm_rk_state* st = p.st;
    st->t = t; st->dt = dt; st->t_end = t_end; st->atol = atol; st->rtol = rtol;
    st->dt_old = dt_old; st->ratio = ratio; st->ckpt_flag = ckpt_flag; st->ckpt = ckpt;
    st->n_span = n_span; st->commit = 0; st->done = done; st->save_slot = -1;
    st->accepted = accepted; st->rejected = rejected; st->nfe = nfe; st->err_acc = 0.0;
  }
}

struct Launch {
  int grid, nwarps, rpw;
  size_t smem;
};

template <int U>
int plan_launch(int64_t B, int dim, Launch* out) {
  const int sms = sm_count();
  const int64_t groups = (B + RB - 1) / RB;  // a warp integrates RB rows at a time
  for (int nwarps = 4; nwarps <= 32; nwarps *= 2) {
    int64_t grid = (groups + nwarps - 1) / nwarps;
    if (grid > sms) grid = sms;
    const int64_t per = grid * nwarps;
    const int64_t gpw = (groups + per - 1) / per;  // groups per warp
    if (gpw > 1 && nwarps < 32) continue;  // prefer more warps per CTA over several groups per warp
    if (gpw > (1 << 19)) return 0;
    const SmemPlan pl = ode_small_plan(dim, 32 * U, nwarps, (int)gpw * RB);
    if (pl.total > 200 * 1024) return 0;
    out->grid = (int)grid; out->nwarps = nwarps; out->rpw = (int)gpw * RB; out->smem = pl.total;
    return 1;
  }
  return 0;
}

int plan_any(int64_t B, int dim, int w, Launch* out) {
  if (B <= 0 || dim <= 0 || dim > 1024) return 0;
  if (w == 32) return plan_launch<1>(B, dim, out);
  if (w == 64) return plan_launch<2>(B, dim, out);
  if (w == 128) return plan_launch<4>(B, dim, out);
  return 0;
}

template <int U, int MAXT>
int launch_t(const OdeSmallParams& p, const Launch& L, cudaStream_t s) {
  const void* kern = (const void*)ode_small_kernel<U, MAXT>;
  CFM_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.smem));
  int per_sm = 0;
  CFM_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, L.nwarps * 32, L.smem));
  CFM_REQUIRE(per_sm >= 1 && L.grid <= per_sm * sm_count(), "ode_small: the grid is not co-resident");
  void* args[] = {const_cast<OdeSmallParams*>(&p)};
  CFM_CUDA_OK(cudaLaunchCooperativeKernel(kern, dim3(L.grid), dim3(L.nwarps * 32), args, L.smem, s));
  note_launches(1);
  return CFM_OK;
}
template <int U>
int launch(const OdeSmallParams& p, const Launch& L, cudaStream_t s) {
  if (L.nwarps <= 8) return launch_t<U, 256>(p, L, s);
  if (L.nwarps <= 16) return launch_t<U, 512>(p, L, s);
  return launch_t<U, 1024>(p, L, s);
}

}  // namespace

}  // namespace cfm

using namespace cfm;

extern "C" int cfm_ode_small_supported(int64_t batch, int dim, int w, int out_dim) {
  Launch L;
  return (out_dim == dim) && plan_any(batch, dim, w, &L);
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
  CFM_REQUIRE(W0 && b0 && W1 && b1 && W2 && b2 && W3 && b3 && x0 && t_span && traj && state_out && workspace,
              "cfm_ode_small_trajectory_f32: null pointer");
  CFM_REQUIRE(n_span >= 2 && (solver == 0 || solver == 1) && (act == CFM_ACT_SELU || act == CFM_ACT_SILU),
              "cfm_ode_small_trajectory_f32: bad argument");
  CFM_REQUIRE(workspace_bytes >= cfm_ode_small_workspace_bytes(batch, dim, w),
              "cfm_ode_small_trajectory_f32: workspace too small");
  Launch L;
  CFM_REQUIRE(plan_any(batch, dim, w, &L), "cfm_ode_small_trajectory_f32: unsupported shape B=%lld dim=%d w=%d",
              (long long)batch, dim, w);
  OdeSmallParams p;
  p.W0 = W0; p.b0 = b0; p.W1 = W1; p.b1 = b1; p.W2 = W2; p.b2 = b2; p.W3 = W3; p.b3 = b3;
  p.dim = dim; p.w = w; p.tv = time_varying ? 1 : 0; p.act = act;
  p.x0 = x0; p.B = batch; p.t_span = t_span; p.n_span = n_span; p.atol = atol; p.rtol = rtol;
  p.solver = solver; p.traj = traj; p.st = state_out; p.partials = reinterpret_cast<double*>(workspace);
  p.rows_per_warp = L.rpw; p.max_steps = 1000000;
  cudaStream_t s = (cudaStream_t)stream;
  CFM_CUDA_OK(cudaMemsetAsync(state_out, 0, sizeof(cfm_rk_state), s));
  if (w == 32) return launch<1>(p, L, s);
  if (w == 64) return launch<2>(p, L, s);
  return launch<4>(p, L, s);
}
