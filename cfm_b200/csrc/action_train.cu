// The action-matching loss of a SMALL scalar-action MLP and all its parameter gradients in ONE cooperative launch
// (DESIGN.md section 3.13).  It lives in its own translation unit: in one module with mlp_train_kernel, ptxas
// compiled that kernel's unchanged PTX to different SASS.
//
// The action-matching cell of tutorial_training_8_gaussians_to_moons.ipynb trains a scalar action s = MLP(dim,
// out_dim=1, time_varying=True) on
//     loss = mean_r [ s(x0_r, 0) - s(x1_r, 1) + 1/2 |d s / d x (xt_r, t_r)|^2 + d s / d t (xt_r, t_r) ]
// with a double backward.  mlp_action_train_kernel computes the loss and its gradients for all eight parameters in
// the layout of mlp_train_kernel.  Per batch row:
//   * the endpoints z0 = [x0, 0] and z1 = [x1, 1]: forward, then the plain reverse pass with cotangent +1/B, -1/B;
//   * the middle point z = [xt, t]: forward keeping act' and act'' of the lane's units; the reverse pass for the input
//     gradient g = grad_z s (g_2 = act'(pre2) W3^T, g_l = act'(pre_l) m_l with m_l = W_{l+1}^T g_{l+1}, grad_z s =
//     W0^T g_0: one butterfly per input column); the loss term 1/2 |g_x|^2 + g_t.  With c = [g_x, 1] held fixed the
//     parameter gradient of that term is the one of s' = D_c s(z): the tangent forward p'_0 = W0 c, h'_l =
//     act'(pre_l) p'_l, p'_{l+1} = W_{l+1} h'_l, and its reverse pass, whose tangent adjoints are g_l / B again and
//     whose primal adjoints are Q_2 = act''(pre2) p'_2 W3^T / B, Q_l = act'(pre_l) W_{l+1}^T Q_{l+1} +
//     act''(pre_l) p'_l m_l / B.
// Every batch row so gives four (delta, a) pairs per layer, stashed as four virtual rows of the tile (slot-major, so
// a warp's two rows of one slot stay adjacent for rb_matvec): end 0 (delta_l, h_l(z0)), end 1 (delta_l, h_l(z1)), the
// middle's primal pair (Q_l, h_l(z)) and its tangent pair (g_l / B, h'_l); the inputs of layer 0 are z0, z1, z and c.
// The tangent pair has no bias term.  dW3 = sum_r (h_2(z0) - h_2(z1) + h'_2(z)) / B.  b3 cancels in s(z0) - s(z1) and
// does not enter grad s, so its gradient is written as exactly 0 (Adam would turn rounding noise there into
// full-size steps).
#include "train_small.cuh"

namespace cg = cooperative_groups;

namespace cfm {

namespace {

constexpr int kSlots = 4;
constexpr int kEnd0 = 0, kEnd1 = 1, kMid = 2, kTan = 3;

struct ActionParams {
  const float *W0, *W1, *W2, *W3, *b0, *b1, *b2;  // torch Linear layout [out][in]; time = last column of W0
  int dim, act, with_grad;
  const float *xt, *t, *x0, *x1;  // [B][dim], [B], [B][dim], [B][dim]
  int64_t B;
  float* loss;          // [1]
  float* grads;         // W0, b0, W1, b1, W2, b2, W3, b3 flat
  double* loss_parts;   // [gridDim.x]
  float* grad_parts;    // [gridDim.x][n_params]
};

struct ActionPlan {
  size_t wt0, b0, b1, b2, wt1, wt2, wu1, wu2, w3;  // weights (float offsets); wt0 is [dim + 1][w], time last
  size_t in, a0, a1, a2, d0, d1, d2, red;          // the tile's stash, kSlots * kTile virtual rows; red: kWarps doubles
  size_t total;                                    // bytes
};
__host__ __device__ inline ActionPlan action_plan(int dim, int w) {
  ActionPlan s;
  size_t o = 0;
  auto take = [&](size_t n) { size_t r = o; o += (n + 3) / 4 * 4; return r; };
  const size_t rows = (size_t)kSlots * kTile;
  s.wt0 = take((size_t)(dim + 1) * w);
  s.b0 = take(w);
  s.b1 = take(w);
  s.b2 = take(w);
  s.wt1 = take((size_t)w * w);
  s.wt2 = take((size_t)w * w);
  s.wu1 = take((size_t)w * w);
  s.wu2 = take((size_t)w * w);
  s.w3 = take(w);
  s.in = take(rows * kInP);
  s.a0 = take(rows * w);
  s.a1 = take(rows * w);
  s.a2 = take(rows * w);
  s.d0 = take(rows * w);
  s.d1 = take(rows * w);
  s.d2 = take(rows * w);
  s.red = take(2 * kWarps);
  s.total = o * sizeof(float);
  return s;
}

// acc[r][q] += sum_{i < n} m[i][u0 + q] * v[r][i] for the RB input rows of v ([RB][kInP] in shared memory)
template <int U>
__device__ __forceinline__ void rb_matvec_in(const float* m, const float* v, int n, float (&acc)[RB][U], int u0) {
  constexpr int W = 32 * U;
  float wv[U];
#pragma unroll 2
  for (int i = 0; i < n; ++i) {
    const float xa = v[i], xb = v[kInP + i];
    lds_units<U>(m + (size_t)i * W + u0, wv);
#pragma unroll
    for (int q = 0; q < U; ++q) {
      acc[0][q] = fmaf(wv[q], xa, acc[0][q]);
      acc[1][q] = fmaf(wv[q], xb, acc[1][q]);
    }
  }
}

// layers 0-2 of the warp's two stash rows vr, vr + 1: h_l to the a_l stash, act'(pre_l) (and act''(pre_l) with D2) of
// the lane's units to registers; h_2 stays in acc
template <int U, bool D2>
__device__ __forceinline__ void action_forward(float* sm, const ActionPlan& pl, int in0, int act, int vr, int u0,
                                               float (&acc)[RB][U], float (&dact)[3][RB][U],
                                               float (&ddact)[3][RB][U]) {
  constexpr int W = 32 * U;
#pragma unroll
  for (int layer = 0; layer <= 2; ++layer) {
    lds_units<U>(sm + (layer == 0 ? pl.b0 : layer == 1 ? pl.b1 : pl.b2) + u0, acc[0]);
#pragma unroll
    for (int q = 0; q < U; ++q) acc[1][q] = acc[0][q];
    if (layer == 0) rb_matvec_in<U>(sm + pl.wt0, sm + pl.in + (size_t)vr * kInP, in0, acc, u0);
    else rb_matvec<U>(sm + (layer == 1 ? pl.wt1 : pl.wt2), sm + (layer == 1 ? pl.a0 : pl.a1) + (size_t)vr * W, acc, u0);
#pragma unroll
    for (int r = 0; r < RB; ++r) {
#pragma unroll
      for (int q = 0; q < U; ++q) {
        dact[layer][r][q] = act_deriv_fast(acc[r][q], act);
        if (D2) ddact[layer][r][q] = act_deriv2_fast(acc[r][q], act);
        acc[r][q] = act_apply_fast(acc[r][q], act);
      }
      sts_units<U>(sm + (layer == 0 ? pl.a0 : layer == 1 ? pl.a1 : pl.a2) + (size_t)(vr + r) * W + u0, acc[r]);
    }
    __syncwarp();
  }
}

template <int U>
__global__ void __launch_bounds__(kThreads, 1) mlp_action_train_kernel(const ActionParams p) {
  constexpr int W = 32 * U;
  constexpr int BS = 2 * U;                         // a thread's block of dW1 / dW2 is BS x BS
  constexpr int NG = kThreads / W;                  // thread groups that share a hidden unit in dW0
  constexpr int NI0 = (kMaxDim + 1 + NG - 1) / NG;  // dW0 entries per thread
  static_assert((NI0 - 1) * NG + NG <= kInP, "stash rows are read past their data");
  extern __shared__ __align__(16) float sm[];
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int dim = p.dim, act = p.act, in0 = dim + 1;
  const bool with_grad = p.with_grad != 0;
  const ActionPlan pl = action_plan(dim, W);

  // ---- stage the weights; zero the input rows, whose padding is read but never written ----
  for (int idx = tid; idx < W * in0; idx += kThreads) {
    const int u = idx / in0, i = idx % in0;
    sm[pl.wt0 + (size_t)i * W + u] = p.W0[idx];
  }
  for (int u = tid; u < W; u += kThreads) {
    sm[pl.b0 + u] = p.b0[u];
    sm[pl.b1 + u] = p.b1[u];
    sm[pl.b2 + u] = p.b2[u];
    sm[pl.w3 + u] = p.W3[u];
  }
  for (int idx = tid; idx < W * W; idx += kThreads) {
    const int u = idx / W, i = idx % W;
    const float w1 = p.W1[idx], w2 = p.W2[idx];
    sm[pl.wt1 + (size_t)i * W + u] = w1;
    sm[pl.wt2 + (size_t)i * W + u] = w2;
    sm[pl.wu1 + idx] = w1;
    sm[pl.wu2 + idx] = w2;
  }
  for (int idx = tid; idx < kSlots * kTile * kInP; idx += kThreads) sm[pl.in + idx] = 0.f;
  __syncthreads();

  const int u0 = U * lane;
  const int lr = warp * RB;  // the warp's first row within a slot of the tile
  float* in_s = sm + pl.in;
  float* a_s[3] = {sm + pl.a0, sm + pl.a1, sm + pl.a2};
  float* d_s[3] = {sm + pl.d0, sm + pl.d1, sm + pl.d2};
  const float* wu_s[3] = {nullptr, sm + pl.wu1, sm + pl.wu2};  // wu_s[l] = W_l in [out][in]: W_l^T delta_l
  const float* wt_s[3] = {sm + pl.wt0, sm + pl.wt1, sm + pl.wt2};
  const int64_t B = p.B;
  const int64_t ntiles = (B + kTile - 1) / kTile;
  const float invB = 1.f / (float)B;
  float w3[U];
  lds_units<U>(sm + pl.w3 + u0, w3);

  // this thread's gradient entries, summed over every tile the CTA takes
  const int oy = (tid / 16) * BS, ix = (tid % 16) * BS;  // dW1, dW2: outputs oy .., inputs ix ..
  const int ou = tid % W, grp = tid / W;                 // dW0[ou][grp + k NG], dW3[0][ou]
  float gW1[BS][BS], gW2[BS][BS], gb1[BS], gb2[BS], gW0[NI0], gb0 = 0.f, gW3 = 0.f;
#pragma unroll
  for (int j = 0; j < BS; ++j) {
    gb1[j] = gb2[j] = 0.f;
#pragma unroll
    for (int k = 0; k < BS; ++k) gW1[j][k] = gW2[j][k] = 0.f;
  }
#pragma unroll
  for (int k = 0; k < NI0; ++k) gW0[k] = 0.f;
  double lsum = 0.0;  // every lane of a warp holds the same value

#pragma unroll 1
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t base = tile * kTile;
    const int nrows = (int)(B - base < kTile ? B - base : kTile);
    if (lr < nrows) {
      // ---- the warp's two rows at three points (the second row may lie past the batch: zeros in, nothing counted)
      bool valid[RB];
#pragma unroll
      for (int m = 0; m < RB; ++m) {
        const int64_t row = base + lr + m;
        valid[m] = row < B;
        float* z0 = in_s + (size_t)(kEnd0 * kTile + lr + m) * kInP;
        float* z1 = in_s + (size_t)(kEnd1 * kTile + lr + m) * kInP;
        float* z = in_s + (size_t)(kMid * kTile + lr + m) * kInP;
        if (lane < dim) {
          z0[lane] = valid[m] ? __ldg(p.x0 + row * dim + lane) : 0.f;
          z1[lane] = valid[m] ? __ldg(p.x1 + row * dim + lane) : 0.f;
          z[lane] = valid[m] ? __ldg(p.xt + row * dim + lane) : 0.f;
        }
        if (lane == dim) {
          z0[lane] = 0.f;
          z1[lane] = 1.f;
          z[lane] = valid[m] ? __ldg(p.t + row) : 0.f;
        }
      }
      __syncwarp();
      float acc[RB][U], dact[3][RB][U], ddact[3][RB][U];
      double lrow[RB] = {0.0, 0.0};

      // the endpoints: s(z0) - s(z1) without b3, which cancels; the reverse pass with cotangent +-1/B
#pragma unroll 1
      for (int e = kEnd0; e <= kEnd1; ++e) {
        const int vr = e * kTile + lr;
        action_forward<U, false>(sm, pl, in0, act, vr, u0, acc, dact, ddact);
        float y[RB] = {0.f, 0.f};
#pragma unroll
        for (int q = 0; q < U; ++q) {
          y[0] = fmaf(w3[q], acc[0][q], y[0]);
          y[1] = fmaf(w3[q], acc[1][q], y[1]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {  // two interleaved butterflies: every lane ends with the sums
          y[0] += __shfl_xor_sync(0xffffffffu, y[0], o);
          y[1] += __shfl_xor_sync(0xffffffffu, y[1], o);
        }
#pragma unroll
        for (int m = 0; m < RB; ++m) lrow[m] += e == kEnd0 ? (double)y[m] : -(double)y[m];
        if (with_grad) {
          const float cot = e == kEnd0 ? invB : -invB;
#pragma unroll
          for (int r = 0; r < RB; ++r) {
#pragma unroll
            for (int q = 0; q < U; ++q) acc[r][q] = w3[q] * cot * dact[2][r][q];
            sts_units<U>(d_s[2] + (size_t)(vr + r) * W + u0, acc[r]);
          }
          __syncwarp();
#pragma unroll
          for (int layer = 1; layer >= 0; --layer) {
#pragma unroll
            for (int r = 0; r < RB; ++r)
#pragma unroll
              for (int q = 0; q < U; ++q) acc[r][q] = 0.f;
            rb_matvec<U>(wu_s[layer + 1], d_s[layer + 1] + (size_t)vr * W, acc, u0);
#pragma unroll
            for (int r = 0; r < RB; ++r) {
#pragma unroll
              for (int q = 0; q < U; ++q) acc[r][q] *= dact[layer][r][q];
              sts_units<U>(d_s[layer] + (size_t)(vr + r) * W + u0, acc[r]);
            }
            __syncwarp();
          }
        }
      }

      // the middle point: g = grad_z s by the reverse pass; g_l (scaled by 1/B at the end) is the tangent pair's delta
      const int vm = kMid * kTile + lr, vt = kTan * kTile + lr;
      action_forward<U, true>(sm, pl, in0, act, vm, u0, acc, dact, ddact);
#pragma unroll
      for (int r = 0; r < RB; ++r) {
#pragma unroll
        for (int q = 0; q < U; ++q) acc[r][q] = w3[q] * dact[2][r][q];
        sts_units<U>(d_s[2] + (size_t)(vt + r) * W + u0, acc[r]);
      }
      __syncwarp();
      float mv[2][RB][U];  // m_l = W_{l+1}^T g_{l+1}
#pragma unroll
      for (int layer = 1; layer >= 0; --layer) {
#pragma unroll
        for (int r = 0; r < RB; ++r)
#pragma unroll
          for (int q = 0; q < U; ++q) mv[layer][r][q] = 0.f;
        rb_matvec<U>(wu_s[layer + 1], d_s[layer + 1] + (size_t)vt * W, mv[layer], u0);
#pragma unroll
        for (int r = 0; r < RB; ++r) {
#pragma unroll
          for (int q = 0; q < U; ++q) acc[r][q] = mv[layer][r][q] * dact[layer][r][q];
          sts_units<U>(d_s[layer] + (size_t)(vt + r) * W + u0, acc[r]);
        }
        __syncwarp();
      }
      // grad_z s = W0^T g_0, one butterfly per input column; c = [g_x, 1] becomes the tangent slot's input row
#pragma unroll 1
      for (int i = 0; i < in0; ++i) {
        float wv[U], gz[RB] = {0.f, 0.f};
        lds_units<U>(sm + pl.wt0 + (size_t)i * W + u0, wv);
#pragma unroll
        for (int q = 0; q < U; ++q) {
          gz[0] = fmaf(wv[q], acc[0][q], gz[0]);
          gz[1] = fmaf(wv[q], acc[1][q], gz[1]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          gz[0] += __shfl_xor_sync(0xffffffffu, gz[0], o);
          gz[1] += __shfl_xor_sync(0xffffffffu, gz[1], o);
        }
#pragma unroll
        for (int m = 0; m < RB; ++m) {
          lrow[m] += i < dim ? 0.5 * (double)gz[m] * (double)gz[m] : (double)gz[m];
          if (lane == i) in_s[(size_t)(vt + m) * kInP + i] = i < dim ? gz[m] : 1.f;
        }
      }
#pragma unroll
      for (int m = 0; m < RB; ++m)
        if (valid[m]) lsum += lrow[m];

      if (with_grad) {
        __syncwarp();
        // the tangent forward p'_l, h'_l = act'(pre_l) p'_l, and the terms rq_l = act''(pre_l) p'_l m_l / B of Q_l
        float rq[3][RB][U];
#pragma unroll
        for (int layer = 0; layer <= 2; ++layer) {
#pragma unroll
          for (int r = 0; r < RB; ++r)
#pragma unroll
            for (int q = 0; q < U; ++q) acc[r][q] = 0.f;
          if (layer == 0) rb_matvec_in<U>(wt_s[0], in_s + (size_t)vt * kInP, in0, acc, u0);
          else rb_matvec<U>(wt_s[layer], a_s[layer - 1] + (size_t)vt * W, acc, u0);
#pragma unroll
          for (int r = 0; r < RB; ++r) {
#pragma unroll
            for (int q = 0; q < U; ++q) {
              const float mq = layer == 2 ? w3[q] : mv[layer][r][q];
              rq[layer][r][q] = ddact[layer][r][q] * acc[r][q] * mq * invB;
              acc[r][q] *= dact[layer][r][q];
            }
            sts_units<U>(a_s[layer] + (size_t)(vt + r) * W + u0, acc[r]);
          }
          __syncwarp();
        }
        // Q_2 = rq_2, Q_l = act'(pre_l) W_{l+1}^T Q_{l+1} + rq_l: the primal pair's deltas
#pragma unroll
        for (int r = 0; r < RB; ++r) sts_units<U>(d_s[2] + (size_t)(vm + r) * W + u0, rq[2][r]);
        __syncwarp();
#pragma unroll
        for (int layer = 1; layer >= 0; --layer) {
#pragma unroll
          for (int r = 0; r < RB; ++r)
#pragma unroll
            for (int q = 0; q < U; ++q) acc[r][q] = 0.f;
          rb_matvec<U>(wu_s[layer + 1], d_s[layer + 1] + (size_t)vm * W, acc, u0);
#pragma unroll
          for (int r = 0; r < RB; ++r) {
#pragma unroll
            for (int q = 0; q < U; ++q) acc[r][q] = fmaf(acc[r][q], dact[layer][r][q], rq[layer][r][q]);
            sts_units<U>(d_s[layer] + (size_t)(vm + r) * W + u0, acc[r]);
          }
          __syncwarp();
        }
        // the tangent pair's deltas are g_l / B (each lane rescales its own units; every product reading them is done)
#pragma unroll
        for (int layer = 0; layer <= 2; ++layer) {
#pragma unroll
          for (int r = 0; r < RB; ++r) {
            float* dp = d_s[layer] + (size_t)(vt + r) * W + u0;
            lds_units<U>(dp, acc[r]);
#pragma unroll
            for (int q = 0; q < U; ++q) acc[r][q] *= invB;
            sts_units<U>(dp, acc[r]);
          }
        }
      }
    }
    if (with_grad) {
      __syncthreads();
      // ---- dW_l += delta_l (x) a_{l-1} over the tile's rows in row order, four virtual rows each ----
#pragma unroll 1
      for (int r = 0; r < nrows; ++r) {
#pragma unroll
        for (int k = 0; k < kSlots; ++k) {
          const int vr = k * kTile + r;
          float dl[BS], al[BS];
          lds_units<BS>(d_s[1] + vr * W + oy, dl);
          lds_units<BS>(a_s[0] + vr * W + ix, al);
#pragma unroll
          for (int j = 0; j < BS; ++j) {
            if (k != kTan) gb1[j] += dl[j];
#pragma unroll
            for (int c = 0; c < BS; ++c) gW1[j][c] = fmaf(dl[j], al[c], gW1[j][c]);
          }
          lds_units<BS>(d_s[2] + vr * W + oy, dl);
          lds_units<BS>(a_s[1] + vr * W + ix, al);
#pragma unroll
          for (int j = 0; j < BS; ++j) {
            if (k != kTan) gb2[j] += dl[j];
#pragma unroll
            for (int c = 0; c < BS; ++c) gW2[j][c] = fmaf(dl[j], al[c], gW2[j][c]);
          }
          const float d0 = d_s[0][vr * W + ou];
          if (k != kTan) gb0 += d0;
#pragma unroll
          for (int c = 0; c < NI0; ++c) gW0[c] = fmaf(d0, in_s[vr * kInP + grp + c * NG], gW0[c]);
        }
        gW3 = fmaf(invB, a_s[2][(kEnd0 * kTile + r) * W + ou], gW3);
        gW3 = fmaf(-invB, a_s[2][(kEnd1 * kTile + r) * W + ou], gW3);
        gW3 = fmaf(invB, a_s[2][(kTan * kTile + r) * W + ou], gW3);
      }
      __syncthreads();  // the next tile overwrites the stash
    }
  }

  // ---- this CTA's partials ----
  const ParamOffsets po = param_offsets(dim, W, 1);
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
    if (grp == 0) {
      part[po.b0 + ou] = gb0;
      part[po.W3 + ou] = gW3;
    }
    if (tid == 0) part[po.b3] = 0.f;
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
    if (lane == 0) *p.loss = (float)(s / (double)B);
  }
}

template <int U>
int launch_action(ActionParams& p, int grid, char* ws, cudaStream_t s) {
  return launch_folded("cfm_mlp_small_action_grad_f32", (const void*)mlp_action_train_kernel<U>,
                       action_plan(p.dim, 32 * U).total, p, grid, ws, s);
}

}  // namespace

}  // namespace cfm

using namespace cfm;

extern "C" int cfm_mlp_small_action_grad_f32(const float* W0, const float* b0, const float* W1, const float* b1,
                                             const float* W2, const float* b2, const float* W3, const float* b3,
                                             int dim, int w, int act, const float* xt, const float* t,
                                             const float* x0, const float* x1, int64_t batch, int with_grad,
                                             float* loss, float* grads, void* workspace, size_t workspace_bytes,
                                             void* stream) {
  const char* what = "cfm_mlp_small_action_grad_f32";
  CFM_REQUIRE(W0 && b0 && W1 && b1 && W2 && b2 && W3 && b3 && xt && t && x0 && x1 && loss && workspace,
              "%s: null pointer", what);
  CFM_REQUIRE(grads || !with_grad, "%s: with_grad needs a grads buffer", what);
  CFM_REQUIRE(act == CFM_ACT_SELU || act == CFM_ACT_SILU, "%s: unknown activation %d", what, act);
  CFM_REQUIRE(cfm_mlp_small_train_supported(batch, dim, w, 1),
              "%s: unsupported shape B=%lld dim=%d w=%d (w in {32, 64}, dim <= 8, B >= 1)", what, (long long)batch,
              dim, w);
  CFM_REQUIRE(workspace_bytes >= cfm_mlp_small_train_workspace_bytes(batch, dim, w, 1), "%s: workspace too small",
              what);
  ActionParams p;
  p.W0 = W0; p.b0 = b0; p.W1 = W1; p.b1 = b1; p.W2 = W2; p.b2 = b2; p.W3 = W3;
  p.dim = dim; p.act = act; p.with_grad = with_grad ? 1 : 0;
  p.xt = xt; p.t = t; p.x0 = x0; p.x1 = x1; p.B = batch;
  p.loss = loss; p.grads = grads;
  const int grid = ctas_for(batch);
  cudaStream_t s = (cudaStream_t)stream;
  if (w == 32) return launch_action<1>(p, grid, (char*)workspace, s);
  return launch_action<2>(p, grid, (char*)workspace, s);
}
