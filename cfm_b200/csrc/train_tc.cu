// The flow-matching regression loss of a WIDE vector-field MLP and all its parameter gradients on the tensor cores
// (DESIGN.md section 3.15): the class the fp16x3 forward samples (mlp_tc_supported's shapes, e.g. BASELINE config 3,
// 785 -> 256 -> 256 -> 256 -> 784), any batch >= 1.  Same loss, gradient layout and with_grad contract as
// cfm_mlp_small_mse_grad_f32 (train_small.cu):
//     loss = mean((s_r * MLP([x_r, t_r]) - target_r)^2),  d loss / d (W0, b0, W1, b1, W2, b2, W3, b3).
//
// Every GEMM is a launch_gemm_h3 call (fp16x3 wgmma, fp32-grade) with an epilogue of this file.  With L = 2 / (B out):
//   forward   layer l: the epilogue keeps the fp32 pre-activation (for act'), the (hi, lo) split of the activation
//             row-major (the next layer's A operand) and a transposed (hi, lo) copy [unit][batch] (the K-major operand of
//             the weight gradient) whose last row is ones (the bias gradient); layer 0 adds t_r * W0[:, dim] per row.
//             Layer 3 forms d = s y - target, the float64 loss partials and r = s d.
//   deltas    e_3 = r, e_{l-1} = act'(pre_{l-1}) * (e_l W_l) for l = 3, 2, 1; the true delta is L e.  Every e is split
//             with ONE power of two from its max |e| (split_pair_kernel, the rule of prep_rows_h3's uniform_absmax): the
//             raw delta L s d is ~3e-7 |d| at B = 8192, out = 784, below fp16's normal range.  The scale must be uniform
//             because the weight gradient contracts over the batch.  Epilogues undo it exactly and apply L in fp32.
//   dW_l      = L e_l^T [a_{l-1}; 1] with K = batch: split-K (gemm_tc.cuh), fp32 partials folded in slice order by
//             tc_fold_kernel, which also folds the loss partials in a fixed order.  dW0's second operand is
//             [x; t; 1]^T, so the time column and b0 come out of the same GEMM.
// Launches per call (cfm_launch_count): with_grad != 0: 19 -- x split, weight max, weight split, 4 forward GEMMs,
// 4 delta splits, 3 delta GEMMs, 4 weight-gradient GEMMs, the fold; with_grad == 0: 8 (the first seven and the fold,
// which then folds the loss only; same instructions up to the loss, so the same loss bits).  No floating-point atomics
// touch a sum: the same call gives the same bits.  The weights are split anew on every call.
#include <algorithm>

#include "gemm_h3.cuh"
#include "mlp_small.cuh"  // act_deriv_fast

namespace cfm {

namespace {

constexpr int64_t kTcMaxBatch = (int64_t)1 << 30;  // int row and K indices of the GEMM core
// Split-K slice rule of the weight-gradient GEMMs (K = batch, in chunks of kHK = 64):
//   accuracy   a slice holds at most kSliceMaxChunks chunks (512 of K, 32 wgmma k-steps per accumulator chain, fewer
//              than the 49 of the K = 784 GEMM whose error DESIGN 3.1 measured);
//   occupancy  at least kSliceTargetItems / tiles slices, so that tiles x slices fills an H100's 132 SMs.
// The rule depends on the shape alone (not on the device), so the bits do not either.
constexpr int kSliceMaxChunks = 8;
constexpr int kSliceTargetItems = 132;

struct Slicing { int slices, chunks, bound; };  // bound: >= slices, non-decreasing in the batch (workspace size)
Slicing slicing(int64_t batch, int n0, int n1) {
  const int nk = (int)((batch + kHK - 1) / kHK);
  const int tiles = ((n0 + kTM - 1) / kTM) * ((n1 + kTN - 1) / kTN);
  int s = (nk + kSliceMaxChunks - 1) / kSliceMaxChunks;
  const int occ = (kSliceTargetItems + tiles - 1) / tiles;
  s = std::max(s, std::min(nk, occ));
  const int chunks = (nk + s - 1) / s;
  return {(nk + chunks - 1) / chunks, chunks, s};
}

// ---- workspace -------------------------------------------------------------------------------------------------
struct TcPlan {
  int64_t ldb;      // row stride of the transposed [.][batch] operands (batch rounded up to 8 halves)
  int64_t ldo8;     // out_dim rounded up to 8
  size_t am;        // 8 floats: max |W_l| (l = 0..3), max |e_3|, |e_2|, |e_1|, |e_0|
  size_t wh[4], wl[4], wth[4], wtl[4];  // weights row-major [out][in] and transposed [in][out] (l = 1..3)
  size_t xh, xl, xth, xtl;              // x [B][dim]; [x, t, 1]^T [dim + 2][ldb]
  size_t pre[3], ah[3], al[3], ath[3], atl[3];  // per hidden layer: fp32 pre [B][w], a (hi, lo), [a; 1]^T (hi, lo)
  size_t e[4], eh[4], el[4], eth[4], etl[4];    // e_l, l = 0..3 (index l): fp32 [B][n], (hi, lo), transposed
  size_t loss;      // float64 loss partials, one per 32 x 32 output chunk of layer 3
  int64_t n_loss;
  size_t part[4];   // split-K partials of dW_l: [slices][n0][ldp]
  Slicing sl[4];
  int gn0[4], gn1[4];
  int64_t ldp[4];
  size_t total;
};

TcPlan tc_plan(int64_t B, int dim, int w, int out_dim) {
  TcPlan p;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes, 1024); return r; };
  p.ldb = (B + 7) / 8 * 8;
  p.ldo8 = (out_dim + 7) / 8 * 8;
  const int rows[4] = {w, w, w, out_dim}, cols[4] = {dim, w, w, w};
  const int64_t tld[4] = {0, w, w, p.ldo8};
  p.am = take(8 * sizeof(float));
  for (int l = 0; l < 4; ++l) {
    p.wh[l] = take((size_t)rows[l] * cols[l] * 2);
    p.wl[l] = take((size_t)rows[l] * cols[l] * 2);
    p.wth[l] = l ? take((size_t)cols[l] * tld[l] * 2) : 0;
    p.wtl[l] = l ? take((size_t)cols[l] * tld[l] * 2) : 0;
  }
  p.xh = take((size_t)B * dim * 2);
  p.xl = take((size_t)B * dim * 2);
  p.xth = take((size_t)(dim + 2) * p.ldb * 2);
  p.xtl = take((size_t)(dim + 2) * p.ldb * 2);
  for (int l = 0; l < 3; ++l) {
    p.pre[l] = take((size_t)B * w * 4);
    p.ah[l] = take((size_t)B * w * 2);
    p.al[l] = take((size_t)B * w * 2);
    p.ath[l] = take((size_t)(w + 1) * p.ldb * 2);
    p.atl[l] = take((size_t)(w + 1) * p.ldb * 2);
  }
  for (int l = 0; l < 4; ++l) {
    const int n = l == 3 ? out_dim : w;
    const int64_t ld = l == 3 ? p.ldo8 : w;
    p.e[l] = take((size_t)B * n * 4);
    p.eh[l] = l ? take((size_t)B * ld * 2) : 0;  // e_0 only enters dW0, transposed
    p.el[l] = l ? take((size_t)B * ld * 2) : 0;
    p.eth[l] = take((size_t)n * p.ldb * 2);
    p.etl[l] = take((size_t)n * p.ldb * 2);
  }
  p.n_loss = ((B + 31) / 32) * ((out_dim + 31) / 32);
  p.loss = take((size_t)p.n_loss * sizeof(double));
  for (int l = 0; l < 4; ++l) {
    p.gn0[l] = rows[l];
    p.gn1[l] = cols[l] + (l == 0 ? 2 : 1);  // + the time column (layer 0) + the bias
    p.ldp[l] = (p.gn1[l] + 31) / 32 * 32;   // whole 32-column chunks
    p.sl[l] = slicing(B, p.gn0[l], p.gn1[l]);
    p.part[l] = take((size_t)p.sl[l].bound * p.gn0[l] * p.ldp[l] * 4);
  }
  p.total = o;
  return p;
}

// ---- (hi, lo) splits in both layouts ---------------------------------------------------------------------------
struct SplitJob {
  const float* src;  // [rows][lds], columns [0, cols) read
  int64_t lds;
  int rows, cols;
  const float* tcol;  // nullable: one more column, tcol[row] (the row times)
  int ones;           // one more column of ones
  const float* am;    // nullable: scale by h3_pow2_scale(*am); else unscaled (saturating)
  __half *hi, *lo;    // nullable: row-major [rows][ld], columns [0, cols)
  int64_t ld;
  __half *hiT, *loT;  // nullable: transposed [all columns][ldT], columns [0, rows)
  int64_t ldT;
};
struct SplitJobs { SplitJob j[4]; };

// one 32 x 32 tile of job blockIdx.z per CTA: coalesced reads, coalesced writes in both layouts
__global__ void __launch_bounds__(256) split_pair_kernel(const SplitJobs jobs) {
  __shared__ float tile[32][33];
  const SplitJob& J = jobs.j[blockIdx.z];
  const int ncols = J.cols + (J.tcol ? 1 : 0) + J.ones;
  const int64_t r0 = (int64_t)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  if (r0 >= J.rows || c0 >= ncols) return;  // CTA-uniform
  const float sc = J.am ? h3_pow2_scale(__ldg(J.am)) : 1.f;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = ty + 8 * i, c = c0 + tx;
    const int64_t row = r0 + r;
    float v = 0.f;
    if (row < J.rows) {
      if (c < J.cols) v = J.src[row * J.lds + c] * sc;
      else if (c == J.cols && J.tcol) v = J.tcol[row];
      else if (c < ncols) v = 1.f;
    }
    tile[r][tx] = v;
    if (J.hi && row < J.rows && c < J.cols) {
      __half h, l;
      split_h3_sat(v, h, l);
      J.hi[row * J.ld + c] = h;
      J.lo[row * J.ld + c] = l;
    }
  }
  if (J.hiT == nullptr) return;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + 8 * i;
    const int64_t row = r0 + tx;
    if (c < ncols && row < J.rows) {
      __half h, l;
      split_h3_sat(tile[tx][ty + 8 * i], h, l);
      J.hiT[c * J.ldT + row] = h;
      J.loT[c * J.ldT + row] = l;
    }
  }
}

int launch_split(const SplitJobs& jobs, int njobs, cudaStream_t s) {
  int64_t rt = 0, ct = 0;
  for (int k = 0; k < njobs; ++k) {
    const SplitJob& J = jobs.j[k];
    rt = std::max<int64_t>(rt, (J.rows + 31) / 32);
    ct = std::max<int64_t>(ct, (J.cols + (J.tcol ? 1 : 0) + J.ones + 31) / 32);
  }
  split_pair_kernel<<<dim3((unsigned)rt, (unsigned)ct, njobs), 256, 0, s>>>(jobs);
  note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}

// max |W_l| over the columns the GEMMs read (finite entries only), l = blockIdx.y
struct AbsJobs {
  const float* src[4];
  int64_t lds[4];
  int rows[4], cols[4];
  float* out;  // [4], zeroed before
};
__global__ void __launch_bounds__(256) weight_absmax_kernel(const AbsJobs J) {
  const int l = blockIdx.y;
  const int64_t n = (int64_t)J.rows[l] * J.cols[l];
  float am = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = fabsf(__ldg(J.src[l] + (i / J.cols[l]) * J.lds[l] + i % J.cols[l]));
    am = (v <= 3.0e38f) ? fmaxf(am, v) : am;
  }
  am = warp_max(am);
  if ((threadIdx.x & 31) == 0) atomic_max_nonneg(J.out + l, am);
}

// ---- GEMM epilogues (interface: gemm_tc.cuh) -------------------------------------------------------------------
__device__ __forceinline__ float inv_pow2_scale(const float* am) { return 1.f / h3_pow2_scale(__ldg(am)); }

// hidden layer: pre = acc / s_W + b (+ t_r W0[:, dim]); writes pre, a = act(pre) split row-major and transposed
struct TcHiddenEpi {
  static constexpr bool kSplitK = false;
  const float* bias;
  const float* am_w;
  const float* tcol;  // nullable (layer 0): W0[:, dim], stride tstride
  int64_t tstride;
  const float* t;
  int act;
  float* pre;
  __half *hi, *lo, *hiT, *loT;
  int64_t ld, ldT;
  float trow, inv_s;
  __device__ __forceinline__ void begin_row(int row, bool ok) {
    inv_s = inv_pow2_scale(am_w);
    trow = (tcol && ok) ? __ldg(t + row) : 0.f;
  }
  __device__ __forceinline__ void store32(int row0, int lane, int col0, const float (&r)[32], int n0, int n1,
                                          float* tile) {
    const int row = row0 + lane;
    const bool ok = row < n0, full = col0 + 32 <= n1;
    float o[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      float v = 0.f;
      if (col0 + c < n1) {
        v = fmaf(r[c], inv_s, __ldg(bias + col0 + c));
        if (tcol) v = fmaf(trow, __ldg(tcol + (col0 + c) * tstride), v);
      }
      o[c] = v;
    }
    if (full) tc_store_chunk32(tile, o, pre + (int64_t)row0 * ld + col0, ld, n0 - row0, lane);
    else if (ok)
#pragma unroll
      for (int c = 0; c < 32; ++c)
        if (col0 + c < n1) pre[(int64_t)row * ld + col0 + c] = o[c];
    if (!ok) return;
#pragma unroll
    for (int c = 0; c < 32; ++c) o[c] = act_apply_fast(o[c], act);
    __half* ph = hi + (int64_t)row * ld + col0;
    __half* pl = lo + (int64_t)row * ld + col0;
    if (full) {
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        __half hh[8], ll[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) split_h3_sat(o[8 * g + c], hh[c], ll[c]);
        *reinterpret_cast<uint4*>(ph + 8 * g) = pack8h(hh);
        *reinterpret_cast<uint4*>(pl + 8 * g) = pack8h(ll);
      }
    }
#pragma unroll
    for (int c = 0; c < 32; ++c)
      if (col0 + c < n1) {  // lane = row: 64 contiguous bytes per column and array
        __half h, l;
        split_h3_sat(o[c], h, l);
        if (!full) { ph[c] = h; pl[c] = l; }
        hiT[(int64_t)(col0 + c) * ldT + row] = h;
        loT[(int64_t)(col0 + c) * ldT + row] = l;
      }
    if (col0 + 32 >= n1) {  // the chunk that ends the row writes its ones entry
      hiT[(int64_t)n1 * ldT + row] = __float2half_rn(1.f);
      loT[(int64_t)n1 * ldT + row] = __float2half_rn(0.f);
    }
  }
  __device__ __forceinline__ void finish(int) {}
};

// layer 3: y = acc / s_W + b, d = s y - target; loss partial sum d^2 per 32 x 32 chunk (float64), e_3 = r = s d
struct TcOutEpi {
  static constexpr bool kSplitK = false;
  const float* bias;
  const float* am_w;
  const float* row_scale;  // nullable
  const float* target;     // [B][out_dim]
  float* r;                // [B][out_dim]
  double* loss_parts;
  int ncol32;
  float* am_r;
  float s, inv_s, amax;
  __device__ __forceinline__ void begin_row(int row, bool ok) {
    inv_s = inv_pow2_scale(am_w);
    s = ok ? (row_scale ? __ldg(row_scale + row) : 1.f) : 0.f;
  }
  __device__ __forceinline__ void store32(int row0, int lane, int col0, const float (&acc)[32], int n0, int n1,
                                          float* tile) {
    const int row = row0 + lane;
    const bool ok = row < n0;
    float o[32];
    double part = 0.0;
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      float v = 0.f;
      if (ok && col0 + c < n1) {
        const float y = fmaf(acc[c], inv_s, __ldg(bias + col0 + c));
        const float d = fmaf(s, y, -__ldg(target + (int64_t)row * n1 + col0 + c));
        part += (double)d * (double)d;
        v = s * d;
        const float a = fabsf(v);
        amax = (a <= 3.0e38f) ? fmaxf(amax, a) : amax;
      }
      o[c] = v;
    }
    if (col0 + 32 <= n1) tc_store_chunk32(tile, o, r + (int64_t)row0 * n1 + col0, n1, n0 - row0, lane);
    else if (ok)
#pragma unroll
      for (int c = 0; c < 32; ++c)
        if (col0 + c < n1) r[(int64_t)row * n1 + col0 + c] = o[c];
    part = warp_sum(part);
    if (lane == 0) loss_parts[(int64_t)(row0 >> 5) * ncol32 + (col0 >> 5)] = part;
  }
  __device__ __forceinline__ void finish(int lane) {
    const float m = warp_max(amax);
    if (lane == 0) atomic_max_nonneg(am_r, m);
  }
};

// delta GEMM: e_{l-1} = act'(pre_{l-1}) * (acc / (s_e s_W)), written fp32 [B][w] with its max |.|
struct TcDeltaEpi {
  static constexpr bool kSplitK = false;
  const float* am_e;
  const float* am_w;
  const float* pre;
  int act;
  float* e;
  int64_t ld;
  float* am_out;
  float inv_e, inv_w, amax;
  __device__ __forceinline__ void begin_row(int, bool) {
    inv_e = inv_pow2_scale(am_e);
    inv_w = inv_pow2_scale(am_w);
  }
  __device__ __forceinline__ void store32(int row0, int lane, int col0, const float (&acc)[32], int n0, int n1,
                                          float* tile) {
    const int row = row0 + lane;
    const bool ok = row < n0, full = col0 + 32 <= n1;
    const float* pr = pre + (int64_t)row * ld + col0;
    float pv[32];
    if (ok && full) {
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(pr) + g);
        pv[4 * g] = q.x; pv[4 * g + 1] = q.y; pv[4 * g + 2] = q.z; pv[4 * g + 3] = q.w;
      }
    } else {
#pragma unroll
      for (int c = 0; c < 32; ++c) pv[c] = (ok && col0 + c < n1) ? __ldg(pr + c) : 0.f;
    }
    float o[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      float v = 0.f;
      if (ok && col0 + c < n1) {
        v = act_deriv_fast(pv[c], act) * ((acc[c] * inv_e) * inv_w);
        const float a = fabsf(v);
        amax = (a <= 3.0e38f) ? fmaxf(amax, a) : amax;
      }
      o[c] = v;
    }
    if (full) tc_store_chunk32(tile, o, e + (int64_t)row0 * ld + col0, ld, n0 - row0, lane);
    else if (ok)
#pragma unroll
      for (int c = 0; c < 32; ++c)
        if (col0 + c < n1) e[(int64_t)row * ld + col0 + c] = o[c];
  }
  __device__ __forceinline__ void finish(int lane) {
    const float m = warp_max(amax);
    if (lane == 0) atomic_max_nonneg(am_out, m);
  }
};

// weight gradient, split-K: the raw fp32 partial of slice s goes to part[s][n0][ldp] (whole 32-column chunks)
struct TcGradEpi {
  static constexpr bool kSplitK = true;
  int k_slices, k_chunks;
  float* part;
  int64_t ldp, slice_stride;
  float* cur;
  __device__ __forceinline__ void begin_slice(int s) { cur = part + (int64_t)s * slice_stride; }
  __device__ __forceinline__ void begin_row(int, bool) {}
  __device__ __forceinline__ void store32(int row0, int lane, int col0, const float (&acc)[32], int n0, int,
                                          float* tile) {
    tc_store_chunk32(tile, acc, cur + (int64_t)row0 * ldp + col0, ldp, n0 - row0, lane);
  }
  __device__ __forceinline__ void finish(int) {}
};

// ---- the fold: dW_l = L / s_e * sum over slices (in slice order) into the flat gradients; the loss ------------
struct FoldJob {
  const float* part;
  int slices, n0, n1;
  int64_t ldp;
  const float* am_e;
  int w_off, b_off;  // column c < n1 - 1 -> grads[w_off + u (n1 - 1) + c]; the last column -> grads[b_off + u]
};
struct FoldParams {
  FoldJob j[4];
  int njobs;
  float L;
  float* grads;
  const double* loss_parts;
  int64_t n_loss;
  double count;  // B out_dim
  float* loss;
};
__global__ void __launch_bounds__(256) tc_fold_kernel(const FoldParams p) {
  if (blockIdx.x == 0) {
    __shared__ double red[8];
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < p.n_loss; i += 256) s += p.loss_parts[i];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      double tot = 0.0;
      for (int k = 0; k < 8; ++k) tot += red[k];
      *p.loss = (float)(tot / p.count);
    }
  }
  int64_t total = 0;
  for (int k = 0; k < p.njobs; ++k) total += (int64_t)p.j[k].n0 * p.j[k].n1;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    int k = 0;
    int64_t i = idx;
    while (i >= (int64_t)p.j[k].n0 * p.j[k].n1) { i -= (int64_t)p.j[k].n0 * p.j[k].n1; ++k; }
    const FoldJob& J = p.j[k];
    const int u = (int)(i / J.n1), c = (int)(i % J.n1);
    const float* q = J.part + (int64_t)u * J.ldp + c;
    const int64_t stride = (int64_t)J.n0 * J.ldp;
    float s = 0.f;
    for (int sl = 0; sl < J.slices; ++sl) s += __ldcg(q + sl * stride);
    const float g = (s * inv_pow2_scale(J.am_e)) * p.L;
    p.grads[c < J.n1 - 1 ? J.w_off + (int64_t)u * (J.n1 - 1) + c : J.b_off + u] = g;
  }
}

}  // namespace

}  // namespace cfm

using namespace cfm;

extern "C" int cfm_mlp_tc_train_supported(int64_t batch, int dim, int w, int out_dim) {
  // the tensor-core forward's shape rule (mlp_h3.cu) without its batch floor: rows of any batch are GEMM rows or K
  return batch >= 1 && batch <= kTcMaxBatch && mlp_tc_supported(128, dim, w, out_dim);
}

extern "C" size_t cfm_mlp_tc_train_workspace_bytes(int64_t batch, int dim, int w, int out_dim) {
  if (!cfm_mlp_tc_train_supported(batch, dim, w, out_dim)) return 0;
  return tc_plan(batch, dim, w, out_dim).total;
}

extern "C" int cfm_mlp_tc_mse_grad_f32(const float* W0, const float* b0, const float* W1, const float* b1,
                                       const float* W2, const float* b2, const float* W3, const float* b3, int dim,
                                       int w, int out_dim, int act, const float* x, const float* t,
                                       const float* target, const float* row_scale, int64_t batch, int with_grad,
                                       float* loss, float* grads, void* workspace, size_t workspace_bytes,
                                       void* stream) {
  const char* what = "cfm_mlp_tc_mse_grad_f32";
  CFM_REQUIRE(W0 && b0 && W1 && b1 && W2 && b2 && W3 && b3 && x && t && target && loss && workspace,
              "%s: null pointer", what);
  CFM_REQUIRE(grads || !with_grad, "%s: with_grad needs a grads buffer", what);
  CFM_REQUIRE(act == CFM_ACT_SELU || act == CFM_ACT_SILU, "%s: unknown activation %d", what, act);
  CFM_REQUIRE(cfm_mlp_tc_train_supported(batch, dim, w, out_dim),
              "%s: unsupported shape B=%lld dim=%d w=%d out_dim=%d (dim >= 32, dim %% 8 == 0, w >= 32, w %% 8 == 0, "
              "out_dim %% 4 == 0, 1 <= B <= 2^30)", what, (long long)batch, dim, w, out_dim);
  CFM_REQUIRE(workspace_bytes >= cfm_mlp_tc_train_workspace_bytes(batch, dim, w, out_dim), "%s: workspace too small",
              what);
  CFM_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 15) == 0, "%s: the workspace must be 16-byte aligned", what);
  cudaStream_t s = (cudaStream_t)stream;
  const int B = (int)batch;
  const TcPlan P = tc_plan(batch, dim, w, out_dim);
  char* ws = reinterpret_cast<char*>(workspace);
  auto F = [&](size_t off) { return reinterpret_cast<float*>(ws + off); };
  auto H = [&](size_t off) { return reinterpret_cast<__half*>(ws + off); };
  float* am = F(P.am);
  const float* Ws[4] = {W0, W1, W2, W3};
  const float* bs[4] = {b0, b1, b2, b3};
  const int rows[4] = {w, w, w, out_dim}, cols[4] = {dim, w, w, w};
  const int64_t lds[4] = {dim + 1, w, w, w}, tld[4] = {0, w, w, P.ldo8};
  int rc;

  CFM_CUDA_OK(cudaMemsetAsync(am, 0, 8 * sizeof(float), s));
  // x -> (hi, lo) [B][dim] and [x, t, 1]^T
  {
    SplitJobs J = {};
    J.j[0] = SplitJob{x, dim, B, dim, t, 1, nullptr, H(P.xh), H(P.xl), dim,
                      with_grad ? H(P.xth) : nullptr, H(P.xtl), P.ldb};
    if ((rc = launch_split(J, 1, s)) != CFM_OK) return rc;
  }
  // weights: one power of two per layer from max |W_l|, row-major and (for the deltas) transposed
  {
    AbsJobs A;
    for (int l = 0; l < 4; ++l) { A.src[l] = Ws[l]; A.lds[l] = lds[l]; A.rows[l] = rows[l]; A.cols[l] = cols[l]; }
    A.out = am;
    int blocks = (int)std::min<int64_t>(((int64_t)w * std::max(dim, w) + 255) / 256, 256);
    weight_absmax_kernel<<<dim3(blocks, 4), 256, 0, s>>>(A);
    note_launches(1);
    CFM_CUDA_OK(cudaGetLastError());
    SplitJobs J = {};
    for (int l = 0; l < 4; ++l)
      J.j[l] = SplitJob{Ws[l], lds[l], rows[l], cols[l], nullptr, 0, am + l, H(P.wh[l]), H(P.wl[l]), cols[l],
                        (l && with_grad) ? H(P.wth[l]) : nullptr, l ? H(P.wtl[l]) : nullptr, tld[l]};
    if ((rc = launch_split(J, 4, s)) != CFM_OK) return rc;
  }
  // forward
  const __half* inh = H(P.xh);
  const __half* inl = H(P.xl);
  for (int l = 0; l < 3; ++l) {
    TcHiddenEpi e{bs[l], am + l, l == 0 ? W0 + dim : nullptr, dim + 1, t, act, F(P.pre[l]), H(P.ah[l]), H(P.al[l]),
                  H(P.ath[l]), H(P.atl[l]), w, P.ldb, 0.f, 0.f};
    if ((rc = launch_gemm_h3(inh, inl, B, cols[l], H(P.wh[l]), H(P.wl[l]), w, cols[l], cols[l], e, s)) != CFM_OK)
      return rc;
    inh = H(P.ah[l]); inl = H(P.al[l]);
  }
  {
    TcOutEpi e{b3, am + 3, row_scale, target, F(P.e[3]), reinterpret_cast<double*>(ws + P.loss),
               (out_dim + 31) / 32, am + 4, 0.f, 0.f, 0.f};
    if ((rc = launch_gemm_h3(inh, inl, B, w, H(P.wh[3]), H(P.wl[3]), out_dim, w, w, e, s)) != CFM_OK) return rc;
  }
  FoldParams fp = {};
  fp.L = (float)(2.0 / ((double)batch * (double)out_dim));
  fp.grads = grads;
  fp.loss_parts = reinterpret_cast<const double*>(ws + P.loss);
  fp.n_loss = P.n_loss;
  fp.count = (double)batch * (double)out_dim;
  fp.loss = loss;
  if (with_grad) {
    // deltas: split e_l (both layouts), then e_{l-1} = act'(pre_{l-1}) (e_l W_l)
    for (int l = 3; l >= 0; --l) {
      const int n = l == 3 ? out_dim : w;
      const int64_t ld = l == 3 ? P.ldo8 : w;
      SplitJobs J = {};
      J.j[0] = SplitJob{F(P.e[l]), n, B, n, nullptr, 0, am + 4 + (3 - l), l ? H(P.eh[l]) : nullptr,
                        l ? H(P.el[l]) : nullptr, ld, H(P.eth[l]), H(P.etl[l]), P.ldb};
      if ((rc = launch_split(J, 1, s)) != CFM_OK) return rc;
      if (l == 0) break;
      TcDeltaEpi e{am + 4 + (3 - l), am + l, F(P.pre[l - 1]), act, F(P.e[l - 1]), w, am + 4 + (4 - l), 0.f, 0.f, 0.f};
      if ((rc = launch_gemm_h3(H(P.eh[l]), H(P.el[l]), B, ld, H(P.wth[l]), H(P.wtl[l]), w, ld, n, e, s)) != CFM_OK)
        return rc;
    }
    // dW_l = e_l^T [a_{l-1}; 1] (dW0: [x; t; 1]), split-K
    const int w_off[4] = {0, w * (dim + 1) + w, w * (dim + 1) + w + (w * w + w), w * (dim + 1) + w + 2 * (w * w + w)};
    for (int l = 0; l < 4; ++l) {
      const __half* bh = l ? H(P.ath[l - 1]) : H(P.xth);
      const __half* bl = l ? H(P.atl[l - 1]) : H(P.xtl);
      const int64_t stride = (int64_t)P.gn0[l] * P.ldp[l];
      TcGradEpi e{P.sl[l].slices, P.sl[l].chunks, F(P.part[l]), P.ldp[l], stride, nullptr};
      if ((rc = launch_gemm_h3(H(P.eth[l]), H(P.etl[l]), P.gn0[l], P.ldb, bh, bl, P.gn1[l], P.ldb, B, e, s)) != CFM_OK)
        return rc;
      fp.j[l] = FoldJob{F(P.part[l]), P.sl[l].slices, P.gn0[l], P.gn1[l], P.ldp[l], am + 4 + (3 - l), w_off[l],
                        w_off[l] + rows[l] * (P.gn1[l] - 1)};
    }
    fp.njobs = 4;
  }
  int64_t total = 0;
  for (int k = 0; k < fp.njobs; ++k) total += (int64_t)fp.j[k].n0 * fp.j[k].n1;
  tc_fold_kernel<<<ew_grid(total), 256, 0, s>>>(fp);
  note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
