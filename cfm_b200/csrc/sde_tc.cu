// Euler-Maruyama steps of Schrodinger-bridge SDEs with WIDE drift and score MLPs (the tensor-core class of the fp16x3
// forward, e.g. MLP(784, w=256)): torchsde.sdeint(SDE(drift, score, sigma), y0, ts, method="euler", dt) as
// cfm_b200/sde.py drives it.  A step is two launches: the pair forward (mlp_h3.cu: both nets on the state's fp16x3
// operand pair, one launch) and the elementwise step kernel below, which
//   * draws dW (device stream: sde_common.cuh, the draws of sde_small_kernel) or reads the caller's increment,
//   * y1 = fmaf(h, drift + score, y0) + sigma dW, the small kernel's expression,
//   * writes the outputs interpolated on the step, y1 and y1's (hi, lo) split for the next forward,
//   * advances the step index and the time the next forward reads.
// Everything a step needs from one call to the next -- step index, time, seed, trajectory and increment pointers --
// lives in a device struct (cfm_sde_state) written by the init kernel, so one captured step replays for the whole
// trajectory with no host round trip and no per-call pointer in the graph.  Shared with cnf_tc.cu: the operand split
// (split4_store, gemm_h3.cuh), the state's shape rule and step advance (sde_common.cuh) and the launch grid
// (common.cuh).
#include "gemm_h3.cuh"
#include "mlp_common.cuh"
#include "sde_common.cuh"

namespace cfm {

// state <- (seed, step 0, t = grid[0], traj, increments); y = traj[0] = y0 and y0's operand split
__global__ void sde_tc_init_kernel(cfm_sde_state* __restrict__ st, const float4* __restrict__ y0, float4* __restrict__ y,
                                   __half* __restrict__ hi, __half* __restrict__ lo, float* traj, const float* inc,
                                   uint64_t seed, const float* __restrict__ grid, int n_steps, int64_t n4) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    st->seed = seed; st->traj = traj; st->increments = inc;
    st->n = 0; st->n_steps = n_steps; st->t = grid[0]; st->ticket = 0u;
  }
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = y0[i];
    y[i] = v;
    reinterpret_cast<float4*>(traj)[i] = v;
    split4_store(v, hi, lo, i);
  }
}

// One Euler-Maruyama step n = st->n over all B * D elements, 4 columns of one row per thread and iteration (D % 8 == 0);
// the CTA that finishes last advances the state.  A step enqueued past n_steps does nothing.
__global__ void __launch_bounds__(256)
sde_tc_step_kernel(cfm_sde_state* st, float4* __restrict__ y, const float4* __restrict__ d,
                   const float4* __restrict__ s, __half* __restrict__ hi, __half* __restrict__ lo,
                   const float* __restrict__ grid, const int* __restrict__ out_begin, const float* __restrict__ out_a,
                   const float* __restrict__ out_b, float sigma, int dim4, int64_t n4) {
  const int n = st->n;
  if (n >= st->n_steps) return;
  const uint64_t seed = st->seed;
  const float4* inc = reinterpret_cast<const float4*>(st->increments);
  float4* traj = reinterpret_cast<float4*>(st->traj);
  const float t = grid[n], h = grid[n + 1] - t;
  const float sh = sqrtf(h);
  const int k0 = out_begin[n], k1 = out_begin[n + 1];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 y0 = y[i], dd = d[i], ss = s[i];
    float4 dw;
    if (inc != nullptr) {
      dw = inc[(int64_t)n * n4 + i];
    } else {
      const int64_t r = i / dim4;
      const float4 z = sde_normal4(seed, n, r, (int)(i - r * dim4));
      dw = make_float4(__fmul_rn(sh, z.x), __fmul_rn(sh, z.y), __fmul_rn(sh, z.z), __fmul_rn(sh, z.w));
    }
    float4 y1;
    y1.x = __fadd_rn(fmaf(h, __fadd_rn(dd.x, ss.x), y0.x), __fmul_rn(sigma, dw.x));
    y1.y = __fadd_rn(fmaf(h, __fadd_rn(dd.y, ss.y), y0.y), __fmul_rn(sigma, dw.y));
    y1.z = __fadd_rn(fmaf(h, __fadd_rn(dd.z, ss.z), y0.z), __fmul_rn(sigma, dw.z));
    y1.w = __fadd_rn(fmaf(h, __fadd_rn(dd.w, ss.w), y0.w), __fmul_rn(sigma, dw.w));
    for (int k = k0; k < k1; ++k) {
      const float a = __ldg(out_a + k), b = __ldg(out_b + k);
      traj[(int64_t)k * n4 + i] = make_float4(__fadd_rn(__fmul_rn(a, y0.x), __fmul_rn(b, y1.x)),
                                              __fadd_rn(__fmul_rn(a, y0.y), __fmul_rn(b, y1.y)),
                                              __fadd_rn(__fmul_rn(a, y0.z), __fmul_rn(b, y1.z)),
                                              __fadd_rn(__fmul_rn(a, y0.w), __fmul_rn(b, y1.w)));
    }
    y[i] = y1;
    split4_store(y1, hi, lo, i);
  }
  step_advance(st, n, grid[n + 1]);
}

}  // namespace cfm

using namespace cfm;

extern "C" int cfm_sde_tc_supported(int batch, int dim, int w) { return mlp_tc_supported(batch, dim, w, dim); }

extern "C" int cfm_sde_tc_init(cfm_sde_state* state, const float* y0, float* y, void* y_hi, void* y_lo, float* traj,
                               const float* increments, uint64_t seed, const float* grid, int n_steps, int batch,
                               int dim, void* stream) {
  const char* what = "cfm_sde_tc_init";
  CFM_REQUIRE(state && y0 && y && y_hi && y_lo && traj && grid, "%s: null pointer", what);
  CFM_REQUIRE(n_steps >= 1, "%s: n_steps must be >= 1 (got %d)", what, n_steps);
  if (const int rc = tc_state_shape(what, batch, dim)) return rc;
  CFM_REQUIRE(aligned16(y0) && aligned16(y) && aligned16(y_hi) && aligned16(y_lo) && aligned16(traj) &&
                  aligned16(increments) && (reinterpret_cast<uintptr_t>(state) & 7) == 0,
              "%s: y0, y, y_hi, y_lo, traj and increments must be 16-byte aligned, the state 8-byte aligned", what);
  const int64_t n4 = (int64_t)batch * dim / 4;
  sde_tc_init_kernel<<<ew_grid(n4), 256, 0, (cudaStream_t)stream>>>(
      state, reinterpret_cast<const float4*>(y0), reinterpret_cast<float4*>(y), reinterpret_cast<__half*>(y_hi),
      reinterpret_cast<__half*>(y_lo), traj, increments, seed, grid, n_steps, n4);
  note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}

extern "C" int cfm_sde_tc_euler_step(cfm_sde_state* state, float* y, const float* drift, const float* score,
                                     void* y_hi, void* y_lo, const float* grid, const int* out_begin,
                                     const float* out_a, const float* out_b, float sigma, int batch, int dim,
                                     void* stream) {
  const char* what = "cfm_sde_tc_euler_step";
  CFM_REQUIRE(state && y && drift && score && y_hi && y_lo && grid && out_begin && out_a && out_b, "%s: null pointer",
              what);
  if (const int rc = tc_state_shape(what, batch, dim)) return rc;
  CFM_REQUIRE(aligned16(y) && aligned16(drift) && aligned16(score) && aligned16(y_hi) && aligned16(y_lo) &&
                  (reinterpret_cast<uintptr_t>(state) & 7) == 0,
              "%s: y, drift, score, y_hi and y_lo must be 16-byte aligned, the state 8-byte aligned", what);
  const int64_t n4 = (int64_t)batch * dim / 4;
  sde_tc_step_kernel<<<ew_grid(n4), 256, 0, (cudaStream_t)stream>>>(
      state, reinterpret_cast<float4*>(y), reinterpret_cast<const float4*>(drift),
      reinterpret_cast<const float4*>(score), reinterpret_cast<__half*>(y_hi), reinterpret_cast<__half*>(y_lo), grid,
      out_begin, out_a, out_b, sigma, dim / 4, n4);
  note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
