// Gradients through the exact-likelihood Euler trajectory of cnf_wrapper (DESIGN.md section 3.14): one cooperative
// launch computes the gradient of L(traj) for all eight parameters of a SMALL MLP and for the initial state, given
// the trajectory the forward kernel (ode_small.cu, CNF variant, solver = euler) stored and dL/dtraj.  It lives in its
// own translation unit for the reason action_train.cu does: sharing a module changed the SASS ptxas made for the
// kernels already in it.
//
// The forward takes one Euler step per t_span interval on the state [x, l]:
//     h_n = t_{n+1} - t_n (fp32, as the forward forms it),  f_n = f(t_n, x_n),  d_n = tr df/dx (t_n, x_n),
//     x_{n+1} = x_n + h_n f_n,  l_{n+1} = l_n + h_n d_n.
// Every x_n is in the stored trajectory, so the discrete adjoint needs no recomputation of states.  With G_n =
// dL/dtraj[n] and a_N = G_N, for n = N-1 .. 0 and the scalar phi_n(x, theta) = a_{x,n+1} . f(t_n, x) +
// a_{l,n+1} d(t_n, x):
//     a_{x,n} = G_{x,n} + a_{x,n+1} + h_n grad_x phi_n,   a_{l,n} = G_{l,n} + a_{l,n+1},   theta_bar += h_n grad_theta phi_n
// and the input gradient is a_0.  The kernel folds h_n into the cotangents: a' = h_n a_{x,n+1}, c' = h_n a_{l,n+1}.
//
// phi for one row.  Forward: pre_l, h_l = act(pre_l); the dim tangent chains of section 3.8 on pre-activations,
// p_{0,k} = W0[:, k], T_{l,k} = act'(pre_l) p_{l,k}, p_{l+1,k} = W_{l+1} T_{l,k}; f = W3 h_2 + b3, d = sum_k W3[k, :]
// . T_{2,k}.  Reverse, from the tangent adjoints tau_{2,k} = c' W3[k, :] and tau_{l,k} = W_{l+1}^T e_{l+1,k}:
//     e_{l,k} = act'(pre_l) tau_{l,k}                                                  (adjoint of p_{l,k})
//     delta_2 = act'(pre_2) W3^T a' + act''(pre_2) sum_k tau_{2,k} p_{2,k}
//     delta_l = act'(pre_l) W_{l+1}^T delta_{l+1} + act''(pre_l) sum_k tau_{l,k} p_{l,k}      (l = 1, 0)
//     h_n grad_x phi = W0x^T delta_0
// and every hidden layer receives one primal outer product and dim tangent ones per (row, step):
//     dW_l += delta_l (x) h_{l-1} + sum_k e_{l,k} (x) T_{l-1,k},  db_l += delta_l   (h_{-1} = [x, t], T_{-1,k} = unit k)
//     dW3 += a' (x) h_2 + c' sum_k unit_k (x) T_{2,k},  db3 += a'.
//
// Layout (one phase).  A CTA takes a tile of R rows (one row pair per warp, R <= 16: fewer for batches that would
// leave SMs idle, and when the stash does not fit in shared memory) and walks the steps n = N-1 .. 0 for them.  At
// every step each warp reads x_n of its two rows, runs the forward and the tangents, then the reverse pass, and
// stashes 1 + dim (delta, input) pairs per layer and row (slot-major virtual rows: slot 0 the primal pair, slot k + 1
// tangent k); after a CTA barrier all 256 threads add the tile's outer products into per-thread registers in row
// order, as mlp_train_kernel does.  The per-CTA partials are
// folded in CTA order after one grid barrier (train_small.cuh): no floating-point atomics, the same bits on every call.
#include "train_small.cuh"

namespace cg = cooperative_groups;

namespace cfm {

namespace {

struct CnfBackParams {
  const float *W0, *W1, *W2, *W3, *b0, *b1, *b2;  // torch Linear layout [out][in]; time = last column of W0
  int dim, act, rows;                             // rows: R, the rows of one tile
  const float* traj;                              // [n_span][B][dim + 1]
  const float* t_span;                            // [n_span]
  int n_span;
  const float* gout;    // [n_span][B][dim + 1]
  float* grad_z;        // [B][dim + 1] or null
  int64_t B;
  float* grads;         // W0, b0, W1, b1, W2, b2, W3, b3 flat
  double* loss_parts;   // the fold's layout (train_small.cuh); this kernel has no loss
  float* grad_parts;    // [gridDim.x][n_params]
};

struct CnfBackPlan {
  size_t wt0, b0, b1, b2, wt1, wt2, wu1, wu2, w3;  // weights (float offsets); wt0 is [dim + 1][w], w3 is W3 [dim][w]
  size_t in, a0, a1, a2, d0, d1, d2;               // the tile's stash, (1 + dim) * R virtual rows
  size_t adj, cot;                                 // per row: a_{n} (being formed) and h_n a_{n+1}, kInP floats each
  size_t total;                                    // bytes
};
__host__ __device__ inline CnfBackPlan cnf_back_plan(int dim, int w, int rows) {
  CnfBackPlan s;
  size_t o = 0;
  auto take = [&](size_t n) { size_t r = o; o += (n + 3) / 4 * 4; return r; };
  const size_t vrows = (size_t)(1 + dim) * rows;
  s.wt0 = take((size_t)(dim + 1) * w);
  s.b0 = take(w);
  s.b1 = take(w);
  s.b2 = take(w);
  s.wt1 = take((size_t)w * w);
  s.wt2 = take((size_t)w * w);
  s.wu1 = take((size_t)w * w);
  s.wu2 = take((size_t)w * w);
  s.w3 = take((size_t)dim * w);
  s.in = take(vrows * kInP);
  s.a0 = take(vrows * w);
  s.a1 = take(vrows * w);
  s.a2 = take(vrows * w);
  s.d0 = take(vrows * w);
  s.d1 = take(vrows * w);
  s.d2 = take(vrows * w);
  s.adj = take((size_t)rows * kInP);
  s.cot = take((size_t)rows * kInP);
  s.total = o * sizeof(float);
  return s;
}

constexpr size_t kSmemBudget = 227 * 1024;  // the opt-in shared memory of one H100 CTA

// Rows per tile: the fewest that still give every one of kMaxCtas CTAs a tile (a step's outer products take time in
// proportion to the tile's rows, the row pairs' chains do not), up to kTile, then halved until the stash fits (dim = 8
// at w = 64 takes at most 8)
inline int cnf_back_rows(int64_t batch, int dim, int w) {
  int r = RB;
  while (r < kTile && (int64_t)r * kMaxCtas < batch) r *= 2;
  for (; r >= RB; r /= 2)
    if (cnf_back_plan(dim, w, r).total <= kSmemBudget) return r;
  return 0;
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

template <int U>
__device__ __forceinline__ void zero(float (&acc)[RB][U]) {
#pragma unroll
  for (int r = 0; r < RB; ++r)
#pragma unroll
    for (int q = 0; q < U; ++q) acc[r][q] = 0.f;
}

// The forward, the tangents and the reverse pass of phi for the warp's two rows (slot-0 virtual rows lr, lr + 1).
// Leaves the stash filled: a_l = h_l / T_{l,k}, d_l = delta_l / e_{l,k}; returns delta_0 of the lane's units in acc.
// Not inlined, for the reason mlp_eval is not (ode_small.cu).
template <int U>
__device__ __noinline__ void row_pair_phi(float* sm, const CnfBackPlan& pl, int dim, int act, int R, int lr,
                                          float (&acc)[RB][U]) {
  constexpr int W = 32 * U;
  const int lane = threadIdx.x & 31, u0 = U * lane;
  float* a_s[3] = {sm + pl.a0, sm + pl.a1, sm + pl.a2};
  float* d_s[3] = {sm + pl.d0, sm + pl.d1, sm + pl.d2};
  const float* wt_s[3] = {sm + pl.wt0, sm + pl.wt1, sm + pl.wt2};
  const float* wu_s[3] = {nullptr, sm + pl.wu1, sm + pl.wu2};  // W_l in [out][in]: W_l^T v is rb_matvec over it
  const float* cot = sm + pl.cot + (size_t)lr * kInP;
  float d1[3][RB][U], d2[3][RB][U];  // act', act'' of the lane's units at every layer
  float wv[U];

  // ---- forward: h_l -> a_l slot 0; p_{l,k} -> d_l slot k + 1 (l >= 1), T_{l,k} -> a_l slot k + 1 ----
#pragma unroll
  for (int layer = 0; layer <= 2; ++layer) {
    lds_units<U>(sm + (layer == 0 ? pl.b0 : layer == 1 ? pl.b1 : pl.b2) + u0, acc[0]);
#pragma unroll
    for (int q = 0; q < U; ++q) acc[1][q] = acc[0][q];
    if (layer == 0) rb_matvec_in<U>(wt_s[0], sm + pl.in + (size_t)lr * kInP, dim + 1, acc, u0);
    else rb_matvec<U>(wt_s[layer], a_s[layer - 1] + (size_t)lr * W, acc, u0);
#pragma unroll
    for (int r = 0; r < RB; ++r) {
#pragma unroll
      for (int q = 0; q < U; ++q) {
        d1[layer][r][q] = act_deriv_fast(acc[r][q], act);
        d2[layer][r][q] = act_deriv2_fast(acc[r][q], act);
        acc[r][q] = act_apply_fast(acc[r][q], act);
      }
      sts_units<U>(a_s[layer] + (size_t)(lr + r) * W + u0, acc[r]);
    }
#pragma unroll 1
    for (int k = 0; k < dim; ++k) {
      const size_t vk = (size_t)(k + 1) * R + lr;
      if (layer == 0) {
        lds_units<U>(wt_s[0] + (size_t)k * W + u0, wv);
#pragma unroll
        for (int r = 0; r < RB; ++r)
#pragma unroll
          for (int q = 0; q < U; ++q) acc[r][q] = wv[q];
      } else {
        zero<U>(acc);
        rb_matvec<U>(wt_s[layer], a_s[layer - 1] + vk * W, acc, u0);
      }
#pragma unroll
      for (int r = 0; r < RB; ++r) {
        if (layer > 0) sts_units<U>(d_s[layer] + (vk + r) * W + u0, acc[r]);
#pragma unroll
        for (int q = 0; q < U; ++q) acc[r][q] *= d1[layer][r][q];
        sts_units<U>(a_s[layer] + (vk + r) * W + u0, acc[r]);
      }
    }
    __syncwarp();
  }

  // ---- reverse.  Layer 2: delta_2 from W3^T a' and the tangent adjoints tau_{2,k} = c' W3[k, :] ----
  float rq[RB][U];
  zero<U>(acc);
  zero<U>(rq);
#pragma unroll 1
  for (int k = 0; k < dim; ++k) {
    const size_t vk = (size_t)(k + 1) * R + lr;
    lds_units<U>(sm + pl.w3 + (size_t)k * W + u0, wv);
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      const float a = cot[r * kInP + k], c = cot[r * kInP + dim];
      float p[U], e[U];
      lds_units<U>(d_s[2] + (vk + r) * W + u0, p);
#pragma unroll
      for (int q = 0; q < U; ++q) {
        acc[r][q] = fmaf(wv[q], a, acc[r][q]);
        const float tau = c * wv[q];
        rq[r][q] = fmaf(tau, p[q], rq[r][q]);
        e[q] = tau * d1[2][r][q];
      }
      sts_units<U>(d_s[2] + (vk + r) * W + u0, e);
    }
  }
#pragma unroll
  for (int r = 0; r < RB; ++r) {
#pragma unroll
    for (int q = 0; q < U; ++q) acc[r][q] = fmaf(d1[2][r][q], acc[r][q], d2[2][r][q] * rq[r][q]);
    sts_units<U>(d_s[2] + (size_t)(lr + r) * W + u0, acc[r]);
  }
  __syncwarp();

  // ---- layers 1, 0: tau_{l,k} = W_{l+1}^T e_{l+1,k}, delta_l = act' W_{l+1}^T delta_{l+1} + act'' sum_k tau p ----
#pragma unroll
  for (int layer = 1; layer >= 0; --layer) {
    zero<U>(rq);
#pragma unroll 1
    for (int k = 0; k < dim; ++k) {
      const size_t vk = (size_t)(k + 1) * R + lr;
      zero<U>(acc);
      rb_matvec<U>(wu_s[layer + 1], d_s[layer + 1] + vk * W, acc, u0);
      float p[RB][U];
      if (layer == 0) {
        lds_units<U>(wt_s[0] + (size_t)k * W + u0, p[0]);
#pragma unroll
        for (int q = 0; q < U; ++q) p[1][q] = p[0][q];
      } else {
#pragma unroll
        for (int r = 0; r < RB; ++r) lds_units<U>(d_s[layer] + (vk + r) * W + u0, p[r]);
      }
#pragma unroll
      for (int r = 0; r < RB; ++r) {
#pragma unroll
        for (int q = 0; q < U; ++q) {
          rq[r][q] = fmaf(acc[r][q], p[r][q], rq[r][q]);
          acc[r][q] *= d1[layer][r][q];
        }
        sts_units<U>(d_s[layer] + (vk + r) * W + u0, acc[r]);
      }
    }
    zero<U>(acc);
    rb_matvec<U>(wu_s[layer + 1], d_s[layer + 1] + (size_t)lr * W, acc, u0);
#pragma unroll
    for (int r = 0; r < RB; ++r) {
#pragma unroll
      for (int q = 0; q < U; ++q) acc[r][q] = fmaf(d1[layer][r][q], acc[r][q], d2[layer][r][q] * rq[r][q]);
      sts_units<U>(d_s[layer] + (size_t)(lr + r) * W + u0, acc[r]);
    }
    __syncwarp();
  }
}

template <int U>
__global__ void __launch_bounds__(kThreads, 1) cnf_euler_backward_kernel(const CnfBackParams p) {
  constexpr int W = 32 * U;
  constexpr int BS = 2 * U;                                 // a thread's block of dW1 / dW2 is BS x BS
  constexpr int NG = kThreads / W;                          // thread groups that share a hidden unit in dW0
  constexpr int NI0 = (kMaxDim + 1 + NG - 1) / NG;          // dW0 entries per thread
  constexpr int NW3 = (kMaxDim * W + kThreads - 1) / kThreads;  // dW3 entries per thread
  static_assert((NI0 - 1) * NG + NG <= kInP, "stash rows are read past their data");
  extern __shared__ __align__(16) float sm[];
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int dim = p.dim, act = p.act, in0 = dim + 1, sw = dim + 1, R = p.rows;
  const CnfBackPlan pl = cnf_back_plan(dim, W, R);
  const int vrows = (1 + dim) * R;

  // ---- stage the weights; input rows: zeros, and unit k in the rows of tangent slot k + 1 ----
  for (int idx = tid; idx < W * in0; idx += kThreads) {
    const int u = idx / in0, i = idx % in0;
    sm[pl.wt0 + (size_t)i * W + u] = p.W0[idx];
  }
  for (int u = tid; u < W; u += kThreads) {
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
  for (int idx = tid; idx < dim * W; idx += kThreads) sm[pl.w3 + idx] = p.W3[idx];
  for (int idx = tid; idx < vrows * kInP; idx += kThreads) {
    const int vr = idx / kInP, i = idx % kInP;
    sm[pl.in + idx] = (vr >= R && i == vr / R - 1) ? 1.f : 0.f;
  }
  __syncthreads();

  const int u0 = U * lane;
  const int lr = warp * RB;  // the warp's first row within the tile
  float* in_s = sm + pl.in;
  const float* a_s[3] = {sm + pl.a0, sm + pl.a1, sm + pl.a2};
  const float* d_s[3] = {sm + pl.d0, sm + pl.d1, sm + pl.d2};
  float* adj = sm + pl.adj;
  float* cot = sm + pl.cot;
  const int64_t B = p.B;
  const int N = p.n_span - 1;  // steps
  const int64_t ntiles = (B + R - 1) / R;

  // this thread's gradient entries, summed over every (row, step) the CTA takes
  const int oy = (tid / 16) * BS, ix = (tid % 16) * BS;  // dW1, dW2: outputs oy .., inputs ix ..
  const int ou = tid % W, grp = tid / W;                 // dW0[ou][grp + k NG]
  float gW1[BS][BS], gW2[BS][BS], gb1[BS], gb2[BS], gW0[NI0], gW3[NW3], gb0 = 0.f, gb3 = 0.f;
#pragma unroll
  for (int j = 0; j < BS; ++j) {
    gb1[j] = gb2[j] = 0.f;
#pragma unroll
    for (int k = 0; k < BS; ++k) gW1[j][k] = gW2[j][k] = 0.f;
  }
#pragma unroll
  for (int k = 0; k < NI0; ++k) gW0[k] = 0.f;
#pragma unroll
  for (int k = 0; k < NW3; ++k) gW3[k] = 0.f;

#pragma unroll 1
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t base = tile * R;
    const int nrows = (int)(B - base < R ? B - base : R);
    const bool active = lr < nrows;  // warp-uniform; the pair's second row may lie past the batch (zeros throughout)
    if (active && lane < sw) {
#pragma unroll
      for (int m = 0; m < RB; ++m) {
        const int64_t row = base + lr + m;
        adj[(lr + m) * kInP + lane] = row < B ? __ldg(p.gout + ((int64_t)N * B + row) * sw + lane) : 0.f;  // a_N
      }
    }
#pragma unroll 1
    for (int n = N - 1; n >= 0; --n) {
      if (active) {
        const float t = __ldg(p.t_span + n), h = __ldg(p.t_span + n + 1) - t;
        if (lane < sw) {
#pragma unroll
          for (int m = 0; m < RB; ++m) {
            const int64_t row = base + lr + m;
            const int j = (lr + m) * kInP + lane;
            in_s[j] = lane < dim ? (row < B ? __ldg(p.traj + ((int64_t)n * B + row) * sw + lane) : 0.f) : t;
            cot[j] = h * adj[j];
          }
        }
        __syncwarp();
        float acc[RB][U];
        row_pair_phi<U>(sm, pl, dim, act, R, lr, acc);
        // h_n grad_x phi = W0x^T delta_0: one butterfly per column; lane i keeps column i
        float gx[RB] = {0.f, 0.f};
#pragma unroll 1
        for (int i = 0; i < dim; ++i) {
          float wv[U], g[RB] = {0.f, 0.f};
          lds_units<U>(sm + pl.wt0 + (size_t)i * W + u0, wv);
#pragma unroll
          for (int q = 0; q < U; ++q) {
            g[0] = fmaf(wv[q], acc[0][q], g[0]);
            g[1] = fmaf(wv[q], acc[1][q], g[1]);
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            g[0] += __shfl_xor_sync(0xffffffffu, g[0], o);
            g[1] += __shfl_xor_sync(0xffffffffu, g[1], o);
          }
          if (lane == i) {
            gx[0] = g[0];
            gx[1] = g[1];
          }
        }
        if (lane < sw) {  // a_n = G_n + a_{n+1} + h_n grad_x phi (gx = 0 in the log-density column)
#pragma unroll
          for (int m = 0; m < RB; ++m) {
            const int64_t row = base + lr + m;
            const int j = (lr + m) * kInP + lane;
            const float g = row < B ? __ldg(p.gout + ((int64_t)n * B + row) * sw + lane) : 0.f;
            adj[j] = g + (adj[j] + gx[m]);
          }
        }
      }
      __syncthreads();
      // ---- the step's outer products over the tile's rows in row order, 1 + dim virtual rows each ----
#pragma unroll 1
      for (int r = 0; r < nrows; ++r) {
#pragma unroll 1
        for (int k = 0; k <= dim; ++k) {
          const int vr = k * R + r;
          float dl[BS], al[BS];
          lds_units<BS>(d_s[1] + vr * W + oy, dl);
          lds_units<BS>(a_s[0] + vr * W + ix, al);
#pragma unroll
          for (int j = 0; j < BS; ++j) {
            if (k == 0) gb1[j] += dl[j];
#pragma unroll
            for (int c = 0; c < BS; ++c) gW1[j][c] = fmaf(dl[j], al[c], gW1[j][c]);
          }
          lds_units<BS>(d_s[2] + vr * W + oy, dl);
          lds_units<BS>(a_s[1] + vr * W + ix, al);
#pragma unroll
          for (int j = 0; j < BS; ++j) {
            if (k == 0) gb2[j] += dl[j];
#pragma unroll
            for (int c = 0; c < BS; ++c) gW2[j][c] = fmaf(dl[j], al[c], gW2[j][c]);
          }
          const float d0 = d_s[0][vr * W + ou];
          if (k == 0) gb0 += d0;
#pragma unroll
          for (int c = 0; c < NI0; ++c) gW0[c] = fmaf(d0, in_s[vr * kInP + grp + c * NG], gW0[c]);
        }
        const float c = cot[r * kInP + dim];
#pragma unroll
        for (int j = 0; j < NW3; ++j) {
          const int idx = tid + j * kThreads;
          if (idx < dim * W) {
            const int e = idx / W, u = idx % W;
            gW3[j] = fmaf(cot[r * kInP + e], a_s[2][r * W + u], gW3[j]);
            gW3[j] = fmaf(c, a_s[2][((e + 1) * R + r) * W + u], gW3[j]);
          }
        }
        if (tid < dim) gb3 += cot[r * kInP + tid];
      }
      __syncthreads();  // the next step overwrites the stash
    }
    if (active && lane < sw && p.grad_z) {
#pragma unroll
      for (int m = 0; m < RB; ++m) {
        const int64_t row = base + lr + m;
        if (row < B) p.grad_z[row * sw + lane] = adj[(lr + m) * kInP + lane];
      }
    }
  }

  // ---- this CTA's partials ----
  const ParamOffsets po = param_offsets(dim, W, dim);
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
  if (grp == 0) part[po.b0 + ou] = gb0;
#pragma unroll
  for (int j = 0; j < NW3; ++j) {
    const int idx = tid + j * kThreads;
    if (idx < dim * W) part[po.W3 + idx] = gW3[j];
  }
  if (tid < dim) part[po.b3 + tid] = gb3;
  __threadfence();
  grid.sync();

  // ---- fold the partials in CTA order: the same bits whatever the timing ----
  const int G = gridDim.x;
  for (int idx = blockIdx.x * kThreads + tid; idx < po.total; idx += G * kThreads) {
    float s = 0.f;
    for (int c = 0; c < G; ++c) s += __ldcg(p.grad_parts + (size_t)c * po.total + idx);
    p.grads[idx] = s;
  }
}

// CTAs a batch can use: one per tile of R rows, up to kMaxCtas
inline int back_ctas(int64_t batch, int R) {
  const int64_t tiles = (batch + R - 1) / R;
  return (int)(tiles < kMaxCtas ? tiles : kMaxCtas);
}

template <int U>
int launch_back(CnfBackParams& p, char* ws, cudaStream_t s) {
  return launch_folded("cfm_ode_small_cnf_euler_backward_f32", (const void*)cnf_euler_backward_kernel<U>,
                       cnf_back_plan(p.dim, 32 * U, p.rows).total, p, back_ctas(p.B, p.rows), ws, s);
}

}  // namespace

}  // namespace cfm

using namespace cfm;

extern "C" int cfm_ode_small_cnf_backward_supported(int64_t batch, int dim, int w) {
  return (w == 32 || w == 64) && dim >= 1 && dim <= kMaxDim && batch >= 1 && cnf_back_rows(batch, dim, w) > 0 &&
         cfm_ode_small_cnf_supported(batch, dim, w);
}

extern "C" size_t cfm_ode_small_cnf_backward_workspace_bytes(int64_t batch, int n_span, int dim, int w) {
  (void)batch; (void)n_span;  // one phase: the adjoint state lives in shared memory, only the fold's partials here
  const int n = param_offsets(dim, w, dim).total;
  return align_up((size_t)kMaxCtas * sizeof(double), 256) + (size_t)kMaxCtas * n * sizeof(float);
}

extern "C" int cfm_ode_small_cnf_euler_backward_f32(const float* W0, const float* b0, const float* W1,
                                                    const float* b1, const float* W2, const float* b2,
                                                    const float* W3, const float* b3, int dim, int w, int act,
                                                    const float* traj, int64_t batch, const float* t_span, int n_span,
                                                    const float* grad_traj, float* grad_z, float* grads,
                                                    void* workspace, size_t workspace_bytes, void* stream) {
  const char* what = "cfm_ode_small_cnf_euler_backward_f32";
  CFM_REQUIRE(W0 && b0 && W1 && b1 && W2 && b2 && W3 && b3 && traj && t_span && grad_traj && grads && workspace,
              "%s: null pointer", what);
  CFM_REQUIRE(act == CFM_ACT_SELU || act == CFM_ACT_SILU, "%s: unknown activation %d", what, act);
  CFM_REQUIRE(n_span >= 2, "%s: n_span = %d (the span needs at least two points)", what, n_span);
  CFM_REQUIRE(cfm_ode_small_cnf_backward_supported(batch, dim, w),
              "%s: unsupported shape B=%lld dim=%d w=%d (w in {32, 64}, dim <= 8 and a batch the forward plans)", what,
              (long long)batch, dim, w);
  CFM_REQUIRE(workspace_bytes >= cfm_ode_small_cnf_backward_workspace_bytes(batch, n_span, dim, w),
              "%s: workspace too small", what);
  CnfBackParams p;
  p.W0 = W0; p.b0 = b0; p.W1 = W1; p.b1 = b1; p.W2 = W2; p.b2 = b2; p.W3 = W3;
  p.dim = dim; p.act = act; p.rows = cnf_back_rows(batch, dim, w);
  p.traj = traj; p.t_span = t_span; p.n_span = n_span; p.gout = grad_traj; p.grad_z = grad_z; p.B = batch;
  p.grads = grads;
  cudaStream_t s = (cudaStream_t)stream;
  if (w == 32) return launch_back<1>(p, (char*)workspace, s);
  return launch_back<2>(p, (char*)workspace, s);
}
