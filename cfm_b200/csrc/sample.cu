// Pair sampling from a coupling:  (i, j) ~ pi   (reference: torchcfm/optimal_transport.py:116-121)
//
// The reference flattens the float64 plan, normalises it, and calls np.random.choice, i.e.
//   cdf = cumsum(p) / cumsum(p)[-1];  k = searchsorted(cdf, uniform, side='right');  (i, j) = divmod(k, n1)
// Here the N^2 plan is never materialised.  The inverse CDF is evaluated hierarchically:
//   1. row masses r_i = sum_j pi_ij (one warp per row, float64 accumulation, one pass over M),
//   2. an in-block float64 scan of r -> row cdf (n0 entries),
//   3. per draw (one warp each): binary-search the row, then a warp-scan along that row of pi
//      entries recomputed from (M, log_u, log_v) to find the column where the cdf crosses.
// This equals the flat searchsorted up to float64 rounding of the cumulative sums.  The uniforms
// come from the host's np.random stream so the reference's RNG contract is kept.
#include "sinkhorn_common.cuh"

namespace cfm {

struct PotEntry {  // pi_ij = exp(-M_ij/reg + lu_i + lv_j), NumPy's fp32 rounding of -M/reg
  const float* M;
  int64_t ldm;
  float reg;
  const float* cost_max;  // device scalar, read when normalize != 0
  int normalize;
  const double* lu;
  const double* lv;
  __device__ __forceinline__ double operator()(int i, int j) const {
    float m = __ldg(M + (int64_t)i * ldm + j);
    if (normalize) m = __fdiv_rn(m, __ldg(cost_max));
    const double e = (double)(-__fdiv_rn(m, reg)) + lu[i] + lv[j];
    return (double)expf((float)e);
  }
};
struct DenseEntry {
  const double* P;
  int64_t ld;
  __device__ __forceinline__ double operator()(int i, int j) const { return P[(int64_t)i * ld + j]; }
};

template <class E>
__global__ void row_mass_kernel(E ent, int n0, int n1, double* __restrict__ rowmass, int32_t* status) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= n0) return;
  double s = 0.0;
  for (int j = lane; j < n1; j += 32) s += ent(warp, j);
  s = warp_sum(s);
  if (lane == 0) {
    rowmass[warp] = s;
    if (!isfinite(s) && status) atomicOr(status, CFM_FLAG_NONFINITE);
  }
}

// <P, M> = sum_ij pi_ij * M_ij  (pot.sinkhorn2, torchcfm/optimal_transport.py:288,300)
__global__ void plan_dot_cost_kernel(PotEntry ent, int n0, int n1, double* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= n0) return;
  const float cm = ent.normalize ? __ldg(ent.cost_max) : 1.f;
  double s = 0.0;
  for (int j = lane; j < n1; j += 32) {
    float m = __ldg(ent.M + (int64_t)warp * ent.ldm + j);
    if (ent.normalize) m = __fdiv_rn(m, cm);
    s += ent(warp, j) * (double)m;
  }
  s = warp_sum(s);
  if (lane == 0 && s != 0.0) atomicAdd(out, s);
}

// single CTA: inclusive float64 scan of rowmass[0..n) -> rowcdf; rowcdf[n] = total
__global__ void __launch_bounds__(1024) row_cdf_kernel(const double* __restrict__ rowmass, int n,
                                                       double* __restrict__ rowcdf, int32_t* status) {
  __shared__ double wsum[32];
  __shared__ double carry_s;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int per = (n + 1023) / 1024;
  const int beg = min(n, tid * per), end = min(n, beg + per);
  double local = 0.0;
  for (int i = beg; i < end; ++i) local += rowmass[i];
  // block exclusive scan of `local`
  double incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    double w = wsum[lane];
    double wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double t = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += t;
    }
    wsum[lane] = wi - w;  // exclusive prefix of warp sums
    if (lane == 31) carry_s = wi;
  }
  __syncthreads();
  double run = wsum[warp] + (incl - local);
  for (int i = beg; i < end; ++i) {
    run += rowmass[i];
    rowcdf[i] = run;
  }
  if (tid == 0) {
    rowcdf[n] = carry_s;
    if (status && fabs(carry_s) < 1e-8) atomicOr(status, CFM_FLAG_ZERO_MASS);
  }
}

template <class E>
__global__ void draw_kernel(E ent, int n0, int n1, const double* __restrict__ rowcdf,
                            const double* __restrict__ uniforms, int n_draws,
                            int64_t* __restrict__ i_out, int64_t* __restrict__ j_out) {
  const int draw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (draw >= n_draws) return;
  const double total = rowcdf[n0];
  const double u = uniforms[draw];
  if (!(fabs(total) >= 1e-8)) {
    // optimal_transport.py:93-96: uniform plan
    if (lane == 0) {
      const int64_t size = (int64_t)n0 * n1;
      int64_t k = (int64_t)(u * (double)size);
      if (k >= size) k = size - 1;
      i_out[draw] = k / n1;
      j_out[draw] = k % n1;
    }
    return;
  }
  const double target = u * total;
  // first row with rowcdf[i] > target
  int lo = 0, hi = n0 - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (rowcdf[mid] > target) hi = mid; else lo = mid + 1;
  }
  const int i = lo;
  double run = i > 0 ? rowcdf[i - 1] : 0.0;
  int jsel = -1, jlast_pos = -1;
  for (int j0 = 0; j0 < n1 && jsel < 0; j0 += 32) {
    const int j = j0 + lane;
    const double v = j < n1 ? ent(i, j) : 0.0;
    double incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    const bool hit = (j < n1) && (run + incl > target);
    const unsigned ballot = __ballot_sync(0xffffffffu, hit);
    const unsigned pos = __ballot_sync(0xffffffffu, (j < n1) && v > 0.0);
    if (pos) jlast_pos = j0 + 31 - __clz(pos);
    if (ballot) jsel = j0 + __ffs(ballot) - 1;
    run += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (jsel < 0) jsel = jlast_pos >= 0 ? jlast_pos : n1 - 1;  // rounding at the row's end
  if (lane == 0) {
    if (i_out) i_out[draw] = i;
    j_out[draw] = jsel;
  }
}


// ---- fast draw for Sinkhorn potentials whose last update was the row update ---------------------
// Row masses are then exactly a_i = 1/n0 by construction (u_i = log a_i - LSE_j(...)), so the row is
// i = floor(u * n0) and only the within-row inversion needs the plan.  The weights are the plan entries
// themselves,  w_j = pi_ij = exp(-M_ij/reg + lu_i + lv_j)  (<= a_i, and their row sum is a_i): every
// exponent is <= 0 and the largest one is >= -log(n0 n1), so a row can neither overflow nor underflow
// whatever |M/reg| is (the first version normalised by lv_0 only; its exponent  -M_ij/reg + lv_j - lv_0
// = log pi_ij - (lu_i + lv_0)  is O(M/reg) and under/overflowed fp32 whole rows for M/reg >~ 100).
// Two exponent flavours, selected on the device by the same rule as the solver (|M/reg| <= 64: fp32):
//   fast     x = M*c2 + (lv2_j + lu2_i) in fp32 log2 units (all terms <~ 100)
//   precise  x = (double)(-(M / cmax) / reg) + lu_i + lv_j with NumPy's fp32 roundings of the quotients and
//            float64 adds (terms are ~1e4 and cancel to ~ -10), then one fp32 ex2
// When no log_u is available (row-conditional draws of an arbitrary potential pair) a first pass takes
// the row maximum of -M_ij/reg + lv_j instead.  One warp per draw, coalesced float4 passes over the row
// (after the first they hit L1/L2): pass A totals the row, pass B walks 1024-column blocks to the one
// holding the target and resolves it with a warp scan.
template <bool F64>
struct RowWeight {
  const float* row;
  const double* lv;
  float c2, reg, cmax;
  int normalize;
  float shift32;    // fast: lu2_i (or -rowmax) in log2 units
  double shift64;   // precise: lu_i (or -rowmax) in natural-log units
  __device__ __forceinline__ float expo(float m, int j) const {  // log2 of the (shifted) weight
    if (F64) {
      const float mn = normalize ? __fdiv_rn(m, cmax) : m;
      return (float)(((double)(-__fdiv_rn(mn, reg)) + shift64 + lv[j]) * kLog2ed);
    }
    return fmaf(m, c2, (float)(lv[j] * kLog2ed) + shift32);
  }
  __device__ __forceinline__ float one(int j) const { return ex2f(expo(__ldg(row + j), j)); }
  __device__ __forceinline__ float4 four(int j) const {
    const float4 m = *reinterpret_cast<const float4*>(row + j);
    return make_float4(ex2f(expo(m.x, j)), ex2f(expo(m.y, j + 1)), ex2f(expo(m.z, j + 2)), ex2f(expo(m.w, j + 3)));
  }
};

// Last column of [b0, bend) whose weight is positive, or -1.  Only the rare walks that reach the end of a block or of
// the row without crossing their target call it.
template <bool F64>
__device__ __forceinline__ int last_positive(const RowWeight<F64>& W, int b0, int bend, bool vec, int lane) {
  int jl = -1;
  if (vec) {
    for (int j = b0 + lane * 4; j < bend; j += 128) {
      const float4 w = W.four(j);
      jl = w.w > 0.f ? j + 3 : w.z > 0.f ? j + 2 : w.y > 0.f ? j + 1 : w.x > 0.f ? j : jl;
    }
  } else {
    for (int j = b0 + lane; j < bend; j += 32) if (W.one(j) > 0.f) jl = j;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) jl = max(jl, __shfl_xor_sync(0xffffffffu, jl, o));
  return jl;
}

// pass B: coarse blocks of 1024 columns, then a fine scan inside the block whose sum crosses `target`.  Returns the
// column, or -1 when the row ends without crossing; `run` is then the sum of all the row's weights.
template <bool F64>
__device__ __forceinline__ int walk_row(const RowWeight<F64>& W, int n1, bool vec, double target, int lane,
                                        double& run) {
  run = 0.0;
  for (int b0 = 0; b0 < n1; b0 += 1024) {
    const int bend = min(n1, b0 + 1024);
    double bp = 0.0;
    if (vec) {
      for (int j = b0 + lane * 4; j < bend; j += 128) { const float4 w = W.four(j); bp += (double)((w.x + w.y) + (w.z + w.w)); }
    } else {
      for (int j = b0 + lane; j < bend; j += 32) bp += (double)W.one(j);
    }
    const double bsum = warp_sum(bp);
    if (!(run + bsum > target)) { run += bsum; continue; }
    // fine scan: 128 (vec) or 32 (scalar) columns per step, in natural column order
    const int step = vec ? 128 : 32;
    for (int j0 = b0; j0 < bend; j0 += step) {
      float w[4] = {0.f, 0.f, 0.f, 0.f};
      const int j = j0 + (vec ? lane * 4 : lane);
      if (j < bend) {
        if (vec) { const float4 q = W.four(j); w[0] = q.x; w[1] = q.y; w[2] = q.z; w[3] = q.w; }
        else w[0] = W.one(j);
      }
      const double mine = (double)((w[0] + w[1]) + (w[2] + w[3]));
      double incl = mine;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const double t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      const bool hit = (j < bend) && (run + incl > target);
      const unsigned ballot = __ballot_sync(0xffffffffu, hit);
      if (ballot) {
        const int src = __ffs(ballot) - 1;
        // the winning lane resolves the element inside its float4; if the element-wise float64 sum ends a rounding
        // short of the fp32 group sum, the group's last element of positive weight is the draw
        int jj = -1;
        if (lane == src) {
          double r2 = run + incl - mine;
          const int cnt = vec ? 4 : 1;
          for (int c = 0; c < cnt; ++c) {
            if (w[c] > 0.f) jj = j + c;
            r2 += (double)w[c];
            if (r2 > target) { jj = j + c; break; }
          }
        }
        return __shfl_sync(0xffffffffu, jj, src);
      }
      run += __shfl_sync(0xffffffffu, incl, 31);
    }
    // the block's sum crossed the target but the in-order scan, summed in another order, ended a rounding short:
    // the target sits at the block's end, whose last weighted column is the draw (never a column of weight 0)
    const int jl = last_positive(W, b0, bend, vec, lane);
    return jl >= 0 ? jl : bend - 1;
  }
  return -1;
}

// known_total > 0: the row's mass is known analytically (1/n0: the weights are the plan entries and the potentials'
// last update was the row update), so the totalling pass over the row is skipped -- one pass less over 32 KB per draw.
// The weights' own sum differs from it by their rounding (~1e-6 relative): a walk that runs off the row's end is
// repeated against the sum it measured, so the draw never lands on a column of weight 0.
template <bool F64>
__device__ __forceinline__ int draw_in_row(RowWeight<F64>& W, bool have_shift, int n1, bool vec, double frac,
                                           int lane, int32_t* status, double known_total) {
  if (!have_shift) {  // pass 0: row maximum of the exponent, so that the largest weight is 1
    W.shift32 = 0.f; W.shift64 = 0.0;
    float mx = -3.0e38f;
    for (int j = lane; j < n1; j += 32) mx = fmaxf(mx, W.expo(__ldg(W.row + j), j));
    mx = warp_max(mx);
    W.shift32 = -mx;
    W.shift64 = -(double)mx * kLn2d;
  }
  // pass A: row total (unless known)
  double total = known_total;
  if (!(known_total > 0.0)) {
    double part = 0.0;  // float64 partial sums: keeps the cdf within ~1e-8 of the float64 reference
    if (vec) {
      for (int j = lane * 4; j < n1; j += 128) { const float4 w = W.four(j); part += (double)((w.x + w.y) + (w.z + w.w)); }
    } else {
      for (int j = lane; j < n1; j += 32) part += (double)W.one(j);
    }
    total = warp_sum(part);
  }
  if (!(total > 0.0) || !isfinite(total)) {
    if (lane == 0 && status) atomicOr(status, CFM_FLAG_NONFINITE);
    return min(n1 - 1, (int)(frac * (double)n1));
  }
  double run;
  int jsel = walk_row(W, n1, vec, frac * total, lane, run);
  // no crossing: the weights sum to less than the total the target was taken from.  Invert against their own sum,
  // which the second walk adds up in the same order (it crosses unless frac rounds to 1)
  if (jsel < 0 && run > 0.0) jsel = walk_row(W, n1, vec, frac * run, lane, run);
  if (jsel < 0) {  // frac == 1, or NaN weights, which never cross the target
    if (!(run == run) && lane == 0 && status) atomicOr(status, CFM_FLAG_NONFINITE);
    jsel = last_positive(W, 0, n1, vec, lane);
    if (jsel < 0) jsel = n1 - 1;
  }
  return jsel;
}

__global__ void draw_uniform_rows_kernel(const float* __restrict__ M, int n0, int n1, int64_t ldm,
                                         float reg, const float* __restrict__ cost_max, int normalize,
                                         const double* __restrict__ lu, const double* __restrict__ lv,
                                         const double* __restrict__ uniforms,
                                         const int64_t* __restrict__ rows, int n_draws,
                                         int64_t* __restrict__ i_out, int64_t* __restrict__ j_out,
                                         int32_t* status) {
  const int draw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (draw >= n_draws) return;
  const double u = uniforms[draw];
  int i;
  double frac;
  if (rows != nullptr) {  // row-conditional draw  j ~ pi[i, :] / sum(pi[i, :])  (sample_trajectory, :239-248)
    i = (int)rows[draw];
    i = min(max(i, 0), n0 - 1);
    frac = u;
  } else {
    i = (int)(u * (double)n0);
    if (i >= n0) i = n0 - 1;
    frac = u * (double)n0 - (double)i;  // position inside row i's cdf cell, in [0, 1)
  }
  const float cmax = cost_max ? __ldg(cost_max) : 1.f;
  const float scale = normalize ? cmax : 1.f;
  const float c2 = -kLog2e / (reg * scale);
  const float* row = M + (int64_t)i * ldm;
  const bool vec = ((ldm & 3) == 0) && ((n1 & 3) == 0) && ((reinterpret_cast<uintptr_t>(M) & 15) == 0);
  // the solver's auto-mode rule: beyond |M/reg| ~ 64 the exponent needs float64 adds
  const bool precise = cost_max ? sk_needs_f64(cmax, normalize, reg) : true;
  int jsel;
  // with log_u the weights are pi_ij and their row sum is a_i = 1/n0 (row update last): no totalling pass.  A
  // potential pair that is not finite (NaN costs) falls back to the measured total, which flags it.  So does a solve
  // in fp32 arithmetic (status[2] == 0, precision="fp32") at |M/reg| > 64: its fp32 exponents of magnitude up to
  // |M/reg| move the row masses of the precise weights further from 1/n0 than their own rounding does.
  const double lui = lu ? lu[i] : 0.0;
  const bool fp32_solve_precise_draw = precise && status != nullptr && status[2] == 0;
  const double known = (lu != nullptr && lui == lui && fabs(lui) < 1.0e300 && !fp32_solve_precise_draw)
                           ? 1.0 / (double)n0 : -1.0;
  if (precise) {
    RowWeight<true> W{row, lv, c2, reg, cmax, normalize, 0.f, lui};
    jsel = draw_in_row<true>(W, lu != nullptr, n1, vec, frac, lane, status, known);
  } else {
    RowWeight<false> W{row, lv, c2, reg, cmax, normalize, lu ? (float)(lui * kLog2ed) : 0.f, 0.0};
    jsel = draw_in_row<false>(W, lu != nullptr, n1, vec, frac, lane, status, known);
  }
  if (lane == 0) {
    if (i_out) i_out[draw] = i;
    j_out[draw] = jsel;
  }
}

__global__ void perm_draw_kernel(const int32_t* __restrict__ sigma, const double* __restrict__ stairs,
                                 int n, const double* __restrict__ uniforms, int n_draws,
                                 int64_t* __restrict__ i_out, int64_t* __restrict__ j_out) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= n_draws) return;
  const double u = uniforms[d];
  int lo = 0, hi = n - 1;  // first k with stairs[k] > u  (searchsorted side='right')
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (stairs[mid] > u) hi = mid; else lo = mid + 1;
  }
  i_out[d] = lo;
  const int j = sigma[lo];
  j_out[d] = (j >= 0 && j < n) ? j : lo;  // an infeasible solve leaves rows unassigned (status says so): stay in range
}

template <class E>
static int sample_common(E ent, int n0, int n1, const double* uniforms, int n_draws, int64_t* i_out,
                         int64_t* j_out, int32_t* status, void* ws, size_t ws_bytes, cudaStream_t s) {
  CFM_REQUIRE(ws && ws_bytes >= cfm_plan_sample_workspace_bytes(n0), "plan sample: workspace too small");
  double* rowmass = reinterpret_cast<double*>(ws);
  double* rowcdf = rowmass + n0;
  row_mass_kernel<E><<<(n0 + 7) / 8, 256, 0, s>>>(ent, n0, n1, rowmass, status); ::cfm::note_launches(1);
  row_cdf_kernel<<<1, 1024, 0, s>>>(rowmass, n0, rowcdf, status); ::cfm::note_launches(1);
  if (n_draws > 0)
    draw_kernel<E><<<(n_draws + 7) / 8, 256, 0, s>>>(ent, n0, n1, rowcdf, uniforms, n_draws, i_out, j_out); ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}

}  // namespace cfm

using namespace cfm;

extern "C" size_t cfm_plan_sample_workspace_bytes(int n0) { return ((size_t)2 * n0 + 2) * sizeof(double); }

extern "C" int cfm_plan_sample(const float* M, int n0, int n1, int64_t ldm, float reg,
                               const float* cost_max, int normalize, const double* log_u,
                               const double* log_v, int uniform_rows, const double* uniforms,
                               int n_draws, int64_t* i_out, int64_t* j_out, int32_t* status,
                               void* workspace, size_t workspace_bytes, void* stream) {
  CFM_REQUIRE(M && log_u && log_v && (n_draws == 0 || (uniforms && i_out && j_out)),
              "cfm_plan_sample: null pointer");
  CFM_REQUIRE(n0 > 0 && n1 > 0 && ldm >= n1 && n_draws >= 0, "cfm_plan_sample: bad shape");
  CFM_REQUIRE(!(normalize && !cost_max), "cfm_plan_sample: normalize needs cost_max");
  if (uniform_rows) {
    if (n_draws == 0) return CFM_OK;
    draw_uniform_rows_kernel<<<(n_draws + 7) / 8, 256, 0, (cudaStream_t)stream>>>(
        M, n0, n1, ldm, reg, cost_max, normalize, log_u, log_v, uniforms, nullptr, n_draws, i_out, j_out, status); ::cfm::note_launches(1);
    CFM_CUDA_OK(cudaGetLastError());
    return CFM_OK;
  }
  PotEntry ent{M, ldm, reg, cost_max, normalize, log_u, log_v};
  return sample_common(ent, n0, n1, uniforms, n_draws, i_out, j_out, status, workspace,
                       workspace_bytes, (cudaStream_t)stream);
}

extern "C" int cfm_plan_sample_rows(const float* M, int n0, int n1, int64_t ldm, float reg,
                                    const float* cost_max, int normalize, const double* log_u,
                                    const double* log_v, const int64_t* rows, const double* uniforms,
                                    int n_draws, int64_t* j_out, int32_t* status, void* stream) {
  CFM_REQUIRE(M && log_v && (n_draws == 0 || (rows && uniforms && j_out)), "cfm_plan_sample_rows: null pointer");
  CFM_REQUIRE(n0 > 0 && n1 > 0 && ldm >= n1 && n_draws >= 0, "cfm_plan_sample_rows: bad shape");
  CFM_REQUIRE(!(normalize && !cost_max), "cfm_plan_sample_rows: normalize needs cost_max");
  if (n_draws == 0) return CFM_OK;
  draw_uniform_rows_kernel<<<(n_draws + 7) / 8, 256, 0, (cudaStream_t)stream>>>(
      M, n0, n1, ldm, reg, cost_max, normalize, log_u, log_v, uniforms, rows, n_draws, nullptr, j_out, status); ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}

extern "C" int cfm_dense_plan_sample_f64(const double* plan, int n0, int n1, const double* uniforms,
                                         int n_draws, int64_t* i_out, int64_t* j_out,
                                         void* workspace, size_t workspace_bytes, void* stream) {
  CFM_REQUIRE(plan && uniforms && i_out && j_out, "cfm_dense_plan_sample_f64: null pointer");
  CFM_REQUIRE(n0 > 0 && n1 > 0 && n_draws >= 0, "cfm_dense_plan_sample_f64: bad shape");
  DenseEntry ent{plan, (int64_t)n1};
  return sample_common(ent, n0, n1, uniforms, n_draws, i_out, j_out, nullptr, workspace,
                       workspace_bytes, (cudaStream_t)stream);
}

extern "C" int cfm_perm_plan_sample(const int32_t* sigma, const double* stairs, int n,
                                    const double* uniforms, int n_draws, int64_t* i_out,
                                    int64_t* j_out, void* stream) {
  CFM_REQUIRE(sigma && stairs && uniforms && i_out && j_out, "cfm_perm_plan_sample: null pointer");
  CFM_REQUIRE(n > 0 && n_draws >= 0, "cfm_perm_plan_sample: bad shape");
  if (n_draws == 0) return CFM_OK;
  perm_draw_kernel<<<(n_draws + 255) / 256, 256, 0, (cudaStream_t)stream>>>(sigma, stairs, n, uniforms,
                                                                          n_draws, i_out, j_out); ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}

extern "C" int cfm_plan_dot_cost(const float* M, int n0, int n1, int64_t ldm, float reg,
                                 const float* cost_max, int normalize, const double* log_u,
                                 const double* log_v, double* out, void* stream) {
  CFM_REQUIRE(M && log_u && log_v && out, "cfm_plan_dot_cost: null pointer");
  CFM_REQUIRE(n0 > 0 && n1 > 0 && ldm >= n1, "cfm_plan_dot_cost: bad shape");
  CFM_REQUIRE(!(normalize && !cost_max), "cfm_plan_dot_cost: normalize needs cost_max");
  cudaStream_t s = (cudaStream_t)stream;
  CFM_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(double), s));
  PotEntry ent{M, ldm, reg, cost_max, normalize, log_u, log_v};
  plan_dot_cost_kernel<<<(n0 + 7) / 8, 256, 0, s>>>(ent, n0, n1, out); ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
