// The flow-matching regression loss of a SMALL vector-field MLP and all its parameter gradients in ONE cooperative
// launch (DESIGN.md section 3.12).
//
// Reference call sites: the training cells of examples/2D_tutorials/tutorial_training_8_gaussians_to_moons.ipynb
// (raw lines 166-186, 310-330, 458-479, 602-623), Flow_matching_tutorial.ipynb and SF2M_tutorial.ipynb:
//     vt = model(torch.cat([xt, t[:, None]], dim=-1)); loss = torch.mean((vt - ut) ** 2); loss.backward()
// For MLP(dim=2, w=64, time_varying=True) at batch 256 that is about 30 stock-PyTorch launches of a microsecond of
// arithmetic each.  Here one kernel computes
//     loss = mean((s_r * MLP([x_r, t_r]) - target_r)^2)   (s = row_scale, or 1)
// and d loss / d (W0, b0, W1, b1, W2, b2, W3, b3):
//
//   * the weights are staged once per CTA in shared memory in the two layouts of ode_small.cu's gradient variant:
//     transposed ([in][out], lane l owns hidden units U*l .. U*l+U-1) for the forward, torch's [out][in] for the
//     reverse products W^T delta; W3 serves both directions from one [w][out_dim] copy;
//   * rows stream from HBM in tiles of kTile = 16 (8 warps x 2 rows per warp, the blocking of mlp_eval): no per-row
//     state stays resident, so any batch >= 1 is supported.  Every row carries its own time as the last input column;
//   * per row pair a warp runs the forward keeping act'(pre_l) of its own units, forms the residual
//     r = 2 s (s y - target) / (B out_dim), adds (s y - target)^2 to a float64 loss partial, and runs the reverse pass
//     delta_3 = r, delta_2, delta_1, delta_0 (no input gradient).  a_{l-1} and delta_l of the tile go to shared memory;
//   * after a CTA barrier all 256 threads add the tile's outer products dW_l += delta_l (x) a_{l-1} into registers:
//     every thread owns a fixed (2U x 2U) block of dW1 and of dW2 and a few entries of dW0, dW3 and the biases, for
//     the whole kernel, rows in batch order, fp32 FMA;
//   * each CTA writes its partial gradients and its loss partial to the workspace; after ONE grid barrier the CTAs
//     fold the partials entry by entry in CTA order.  No floating-point atomics: with the same batch on the same
//     card the result is the same bits every run.
//
// with_grad = 0 stops each row after the loss and folds only the loss; the forward instructions are the same, so the
// loss has the bits of the with-gradient call.
#include "train_small.cuh"

namespace cg = cooperative_groups;

namespace cfm {

namespace {

constexpr int kOutP = 8;  // floats per stashed delta_3 row

struct TrainParams {
  const float *W0, *b0, *W1, *b1, *W2, *b2, *W3, *b3;  // torch Linear layout [out][in]; time = last column of W0
  int dim, out_dim, act, with_grad;
  const float *x, *t, *target, *row_scale;  // [B][dim], [B], [B][out_dim], [B] or null
  int64_t B;
  float* loss;          // [1]
  float* grads;         // W0, b0, W1, b1, W2, b2, W3, b3 flat
  double* loss_parts;   // [gridDim.x]
  float* grad_parts;    // [gridDim.x][n_params]
};

struct TrainPlan {
  size_t wt0, wtime, b0, b1, b2, wt1, wt2, wu1, wu2, wt3, b3;  // weights (float offsets)
  size_t in, a0, a1, a2, d0, d1, d2, d3, red;                  // the tile's stash; red: kWarps doubles
  size_t total;                                                // bytes
};
__host__ __device__ inline TrainPlan train_plan(int dim, int w, int out_dim) {
  TrainPlan s;
  size_t o = 0;
  auto take = [&](size_t n) { size_t r = o; o += (n + 3) / 4 * 4; return r; };
  s.wt0 = take((size_t)dim * w);
  s.wtime = take(w);
  s.b0 = take(w);
  s.b1 = take(w);
  s.b2 = take(w);
  s.wt1 = take((size_t)w * w);
  s.wt2 = take((size_t)w * w);
  s.wu1 = take((size_t)w * w);
  s.wu2 = take((size_t)w * w);
  s.wt3 = take((size_t)w * out_dim);
  s.b3 = take(out_dim);
  s.in = take((size_t)kTile * kInP);
  s.a0 = take((size_t)kTile * w);
  s.a1 = take((size_t)kTile * w);
  s.a2 = take((size_t)kTile * w);
  s.d0 = take((size_t)kTile * w);
  s.d1 = take((size_t)kTile * w);
  s.d2 = take((size_t)kTile * w);
  s.d3 = take((size_t)kTile * kOutP);
  s.red = take(2 * kWarps);
  s.total = o * sizeof(float);
  return s;
}

template <int U>
__global__ void __launch_bounds__(kThreads, 1) mlp_train_kernel(const TrainParams p) {
  constexpr int W = 32 * U;
  constexpr int BS = 2 * U;                             // a thread's block of dW1 / dW2 is BS x BS
  constexpr int NG = kThreads / W;                      // thread groups that share a hidden unit in dW0 / dW3
  constexpr int NI0 = (kMaxDim + 1 + NG - 1) / NG;      // dW0 entries per thread
  constexpr int NE3 = (kMaxDim + NG - 1) / NG;          // dW3 entries per thread
  static_assert((NI0 - 1) * NG + NG <= kInP && (NE3 - 1) * NG + NG <= kOutP, "stash rows are read past their data");
  extern __shared__ __align__(16) float sm[];
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int dim = p.dim, out_dim = p.out_dim, act = p.act, in0 = dim + 1;
  const bool with_grad = p.with_grad != 0;
  const TrainPlan pl = train_plan(dim, W, out_dim);

  // ---- stage the weights; zero the stash rows whose padding is read but never written ----
  for (int idx = tid; idx < W * dim; idx += kThreads) {
    const int u = idx / dim, i = idx % dim;
    sm[pl.wt0 + (size_t)i * W + u] = p.W0[(size_t)u * in0 + i];
  }
  for (int u = tid; u < W; u += kThreads) {
    sm[pl.wtime + u] = p.W0[(size_t)u * in0 + dim];
    sm[pl.b0 + u] = p.b0[u];
    sm[pl.b1 + u] = p.b1[u];
    sm[pl.b2 + u] = p.b2[u];
  }
  for (int idx = tid; idx < W * W; idx += kThreads) {
    const int u = idx / W, i = idx % W;
    const float w1 = p.W1[idx], w2 = p.W2[idx];
    sm[pl.wt1 + (size_t)i * W + u] = w1;
    sm[pl.wt2 + (size_t)i * W + u] = w2;
    sm[pl.wu1 + idx] = w1;
    sm[pl.wu2 + idx] = w2;
  }
  for (int idx = tid; idx < out_dim * W; idx += kThreads) {
    const int e = idx / W, i = idx % W;
    sm[pl.wt3 + (size_t)i * out_dim + e] = p.W3[idx];
  }
  for (int e = tid; e < out_dim; e += kThreads) sm[pl.b3 + e] = p.b3[e];
  for (int idx = tid; idx < kTile * kInP; idx += kThreads) sm[pl.in + idx] = 0.f;
  for (int idx = tid; idx < kTile * kOutP; idx += kThreads) sm[pl.d3 + idx] = 0.f;
  __syncthreads();

  const int u0 = U * lane;
  const int lr = warp * RB;  // the warp's first row within the tile
  float* in_s = sm + pl.in;
  float* a0_s = sm + pl.a0;
  float* a1_s = sm + pl.a1;
  float* a2_s = sm + pl.a2;
  float* d0_s = sm + pl.d0;
  float* d1_s = sm + pl.d1;
  float* d2_s = sm + pl.d2;
  float* d3_s = sm + pl.d3;
  const int64_t B = p.B;
  const int64_t ntiles = (B + kTile - 1) / kTile;
  const float rscale = 2.f / ((float)B * (float)out_dim);

  // this thread's gradient entries, summed over every tile the CTA takes
  const int oy = (tid / 16) * BS, ix = (tid % 16) * BS;  // dW1, dW2: outputs oy .., inputs ix ..
  const int ou = tid % W, grp = tid / W;                 // dW0[ou][grp + k NG], dW3[grp + k NG][ou]
  float gW1[BS][BS], gW2[BS][BS], gb1[BS], gb2[BS], gW0[NI0], gW3[NE3], gb0 = 0.f, gb3 = 0.f;
#pragma unroll
  for (int j = 0; j < BS; ++j) {
    gb1[j] = gb2[j] = 0.f;
#pragma unroll
    for (int k = 0; k < BS; ++k) gW1[j][k] = gW2[j][k] = 0.f;
  }
#pragma unroll
  for (int k = 0; k < NI0; ++k) gW0[k] = 0.f;
#pragma unroll
  for (int k = 0; k < NE3; ++k) gW3[k] = 0.f;
  double lsum = 0.0;  // every lane of a warp holds the same value

#pragma unroll 1
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t base = tile * kTile;
    const int nrows = (int)(B - base < kTile ? B - base : kTile);
    if (lr < nrows) {
      // ---- the warp's two rows (the second may lie past the batch: zeros in, nothing counted) ----
      bool valid[RB];
      float sc[RB], tt[RB];
#pragma unroll
      for (int m = 0; m < RB; ++m) {
        const int64_t row = base + lr + m;
        valid[m] = row < B;
        sc[m] = valid[m] ? (p.row_scale ? __ldg(p.row_scale + row) : 1.f) : 0.f;
        tt[m] = valid[m] ? __ldg(p.t + row) : 0.f;
        if (lane < dim) in_s[(lr + m) * kInP + lane] = valid[m] ? __ldg(p.x + row * dim + lane) : 0.f;
        if (lane == dim) in_s[(lr + m) * kInP + lane] = tt[m];
      }
      __syncwarp();
      float acc[RB][U], wv[U], dact[3][RB][U];
      // layer 0: [x, t] -> W, the row's own t entering as the last input column
      lds_units<U>(sm + pl.b0 + u0, acc[0]);
      lds_units<U>(sm + pl.wtime + u0, wv);
#pragma unroll
      for (int q = 0; q < U; ++q) {
        acc[1][q] = fmaf(tt[1], wv[q], acc[0][q]);
        acc[0][q] = fmaf(tt[0], wv[q], acc[0][q]);
      }
#pragma unroll 2
      for (int i = 0; i < dim; ++i) {
        const float xa = in_s[lr * kInP + i], xb = in_s[(lr + 1) * kInP + i];
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
        for (int q = 0; q < U; ++q) {
          dact[0][r][q] = act_deriv_fast(acc[r][q], act);
          acc[r][q] = act_apply_fast(acc[r][q], act);
        }
        sts_units<U>(a0_s + (lr + r) * W + u0, acc[r]);
      }
      __syncwarp();
      // layers 1, 2
#pragma unroll
      for (int layer = 1; layer <= 2; ++layer) {
        lds_units<U>(sm + (layer == 1 ? pl.b1 : pl.b2) + u0, acc[0]);
#pragma unroll
        for (int q = 0; q < U; ++q) acc[1][q] = acc[0][q];
        rb_matvec<U>(sm + (layer == 1 ? pl.wt1 : pl.wt2), (layer == 1 ? a0_s : a1_s) + lr * W, acc, u0);
#pragma unroll
        for (int r = 0; r < RB; ++r) {
#pragma unroll
          for (int q = 0; q < U; ++q) {
            dact[layer][r][q] = act_deriv_fast(acc[r][q], act);
            acc[r][q] = act_apply_fast(acc[r][q], act);
          }
          sts_units<U>((layer == 1 ? a1_s : a2_s) + (lr + r) * W + u0, acc[r]);
        }
        __syncwarp();
      }
      // layer 3 (this lane's units of h2 are still in acc), the residual, the loss and W3^T r
      float g[RB][U];
#pragma unroll
      for (int r = 0; r < RB; ++r)
#pragma unroll
        for (int q = 0; q < U; ++q) g[r][q] = 0.f;
      for (int e = 0; e < out_dim; ++e) {
        float w3[U], y[RB] = {0.f, 0.f};
#pragma unroll
        for (int q = 0; q < U; ++q) {
          w3[q] = sm[pl.wt3 + (size_t)(u0 + q) * out_dim + e];
          y[0] = fmaf(w3[q], acc[0][q], y[0]);
          y[1] = fmaf(w3[q], acc[1][q], y[1]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {  // two interleaved butterflies: every lane ends with the sums
          y[0] += __shfl_xor_sync(0xffffffffu, y[0], o);
          y[1] += __shfl_xor_sync(0xffffffffu, y[1], o);
        }
        const float b3 = sm[pl.b3 + e];
#pragma unroll
        for (int m = 0; m < RB; ++m) {
          float d = 0.f;
          if (valid[m]) d = fmaf(sc[m], y[m] + b3, -__ldg(p.target + (base + lr + m) * out_dim + e));
          lsum += (double)d * (double)d;
          const float res = sc[m] * d * rscale;
          if (lane == 0) d3_s[(lr + m) * kOutP + e] = res;
#pragma unroll
          for (int q = 0; q < U; ++q) g[m][q] = fmaf(w3[q], res, g[m][q]);
        }
      }
      if (with_grad) {
        // delta_2 = act'(pre2) * (W3^T r)
#pragma unroll
        for (int r = 0; r < RB; ++r) {
#pragma unroll
          for (int q = 0; q < U; ++q) acc[r][q] = g[r][q] * dact[2][r][q];
          sts_units<U>(d2_s + (lr + r) * W + u0, acc[r]);
        }
        __syncwarp();
        // delta_1 = act'(pre1) * (W2^T delta_2), delta_0 = act'(pre0) * (W1^T delta_1)
#pragma unroll
        for (int layer = 1; layer >= 0; --layer) {
#pragma unroll
          for (int r = 0; r < RB; ++r)
#pragma unroll
            for (int q = 0; q < U; ++q) acc[r][q] = 0.f;
          rb_matvec<U>(sm + (layer == 1 ? pl.wu2 : pl.wu1), (layer == 1 ? d2_s : d1_s) + lr * W, acc, u0);
#pragma unroll
          for (int r = 0; r < RB; ++r) {
#pragma unroll
            for (int q = 0; q < U; ++q) acc[r][q] *= dact[layer][r][q];
            sts_units<U>((layer == 1 ? d1_s : d0_s) + (lr + r) * W + u0, acc[r]);
          }
          __syncwarp();
        }
      }
    }
    if (with_grad) {
      __syncthreads();
      // ---- dW_l += delta_l (x) a_{l-1} over the tile's rows, in row order ----
#pragma unroll 2
      for (int r = 0; r < nrows; ++r) {
        float dl[BS], al[BS];
        lds_units<BS>(d1_s + r * W + oy, dl);
        lds_units<BS>(a0_s + r * W + ix, al);
#pragma unroll
        for (int j = 0; j < BS; ++j) {
          gb1[j] += dl[j];
#pragma unroll
          for (int k = 0; k < BS; ++k) gW1[j][k] = fmaf(dl[j], al[k], gW1[j][k]);
        }
        lds_units<BS>(d2_s + r * W + oy, dl);
        lds_units<BS>(a1_s + r * W + ix, al);
#pragma unroll
        for (int j = 0; j < BS; ++j) {
          gb2[j] += dl[j];
#pragma unroll
          for (int k = 0; k < BS; ++k) gW2[j][k] = fmaf(dl[j], al[k], gW2[j][k]);
        }
        const float d0 = d0_s[r * W + ou], h2 = a2_s[r * W + ou];
        gb0 += d0;
#pragma unroll
        for (int k = 0; k < NI0; ++k) gW0[k] = fmaf(d0, in_s[r * kInP + grp + k * NG], gW0[k]);
#pragma unroll
        for (int k = 0; k < NE3; ++k) gW3[k] = fmaf(d3_s[r * kOutP + grp + k * NG], h2, gW3[k]);
        if (tid < kOutP) gb3 += d3_s[r * kOutP + tid];
      }
      __syncthreads();  // the next tile overwrites the stash
    }
  }

  // ---- this CTA's partials ----
  const ParamOffsets po = param_offsets(dim, W, out_dim);
  double* red = reinterpret_cast<double*>(sm + pl.red);
  if (lane == 0) red[warp] = lsum;
  __syncthreads();
  if (tid == 0) {
    double s = 0.0;
    for (int k = 0; k < kWarps; ++k) s += red[k];
    p.loss_parts[blockIdx.x] = s;
  }
  if (with_grad) {
    float* part = p.grad_parts + (size_t)blockIdx.x * po.total;
#pragma unroll
    for (int j = 0; j < BS; ++j) {
#pragma unroll
      for (int k = 0; k < BS; ++k) {
        part[po.W1 + (oy + j) * W + ix + k] = gW1[j][k];
        part[po.W2 + (oy + j) * W + ix + k] = gW2[j][k];
      }
      if (ix == 0) {
        part[po.b1 + oy + j] = gb1[j];
        part[po.b2 + oy + j] = gb2[j];
      }
    }
#pragma unroll
    for (int k = 0; k < NI0; ++k)
      if (grp + k * NG < in0) part[po.W0 + ou * in0 + grp + k * NG] = gW0[k];
#pragma unroll
    for (int k = 0; k < NE3; ++k)
      if (grp + k * NG < out_dim) part[po.W3 + (grp + k * NG) * W + ou] = gW3[k];
    if (grp == 0) part[po.b0 + ou] = gb0;
    if (tid < out_dim) part[po.b3 + tid] = gb3;
  }
  __threadfence();
  grid.sync();

  // ---- fold the partials in CTA order: the same bits whatever the timing ----
  const int G = gridDim.x;
  if (with_grad) {
    for (int idx = blockIdx.x * kThreads + tid; idx < po.total; idx += G * kThreads) {
      float s = 0.f;
      for (int c = 0; c < G; ++c) s += __ldcg(p.grad_parts + (size_t)c * po.total + idx);
      p.grads[idx] = s;
    }
  }
  if (blockIdx.x == 0 && warp == 0) {
    double s = 0.0;
    for (int c = lane; c < G; c += 32) s += __ldcg(p.loss_parts + c);
    s = warp_sum(s);
    if (lane == 0) *p.loss = (float)(s / ((double)B * (double)out_dim));
  }
}

bool class_supported(int dim, int w, int out_dim) {
  return (w == 32 || w == 64) && dim >= 1 && dim <= kMaxDim && out_dim >= 1 && out_dim <= kMaxDim;
}

template <int U>
int launch_train(TrainParams& p, int grid, char* ws, cudaStream_t s) {
  return launch_folded("cfm_mlp_small_mse_grad_f32", (const void*)mlp_train_kernel<U>,
                       train_plan(p.dim, 32 * U, p.out_dim).total, p, grid, ws, s);
}

}  // namespace

}  // namespace cfm

using namespace cfm;

extern "C" int cfm_mlp_small_train_supported(int64_t batch, int dim, int w, int out_dim) {
  return batch >= 1 && class_supported(dim, w, out_dim);
}

extern "C" size_t cfm_mlp_small_train_workspace_bytes(int64_t batch, int dim, int w, int out_dim) {
  if (!cfm_mlp_small_train_supported(batch, dim, w, out_dim)) return 0;
  const size_t g = (size_t)ctas_for(batch);
  return align_up(g * sizeof(double), 256) +
         align_up(g * (size_t)param_offsets(dim, w, out_dim).total * sizeof(float), 256);
}

extern "C" int cfm_mlp_small_mse_grad_f32(const float* W0, const float* b0, const float* W1, const float* b1,
                                          const float* W2, const float* b2, const float* W3, const float* b3,
                                          int dim, int w, int out_dim, int act, const float* x, const float* t,
                                          const float* target, const float* row_scale, int64_t batch, int with_grad,
                                          float* loss, float* grads, void* workspace, size_t workspace_bytes,
                                          void* stream) {
  const char* what = "cfm_mlp_small_mse_grad_f32";
  CFM_REQUIRE(W0 && b0 && W1 && b1 && W2 && b2 && W3 && b3 && x && t && target && loss && workspace,
              "%s: null pointer", what);
  CFM_REQUIRE(grads || !with_grad, "%s: with_grad needs a grads buffer", what);
  CFM_REQUIRE(act == CFM_ACT_SELU || act == CFM_ACT_SILU, "%s: unknown activation %d", what, act);
  CFM_REQUIRE(cfm_mlp_small_train_supported(batch, dim, w, out_dim),
              "%s: unsupported shape B=%lld dim=%d w=%d out_dim=%d (w in {32, 64}, dim <= 8, out_dim <= 8, B >= 1)",
              what, (long long)batch, dim, w, out_dim);
  CFM_REQUIRE(workspace_bytes >= cfm_mlp_small_train_workspace_bytes(batch, dim, w, out_dim),
              "%s: workspace too small", what);
  TrainParams p;
  p.W0 = W0; p.b0 = b0; p.W1 = W1; p.b1 = b1; p.W2 = W2; p.b2 = b2; p.W3 = W3; p.b3 = b3;
  p.dim = dim; p.out_dim = out_dim; p.act = act; p.with_grad = with_grad ? 1 : 0;
  p.x = x; p.t = t; p.target = target; p.row_scale = row_scale; p.B = batch;
  p.loss = loss; p.grads = grads;
  const int grid = ctas_for(batch);
  cudaStream_t s = (cudaStream_t)stream;
  if (w == 32) return launch_train<1>(p, grid, (char*)workspace, s);
  return launch_train<2>(p, grid, (char*)workspace, s);
}
