// The action-matching gradient field of WIDE scalar actions on the tensor cores (DESIGN.md section 3.18): the field of
// torch_wrapper(GradModel(MLP(dim, out_dim=1, w, time_varying=True))) for actions in the tensor-core class
// (B >= 128, dim >= 32, dim and w multiples of 8, w >= 32; e.g. the MNIST shape 785 -> 256 -> 256 -> 256 -> 1), as
// cfm_b200/ode.py drives it with Euler or dopri5:
//     v(t, x) = grad_x s(t, x) = W0x^T (D0 * W1^T (D1 * W2^T (D2 * w3))),   D_l = act'(pre_l),  W0x = W0[:, :dim].
// In batch-row form g2 = D2 * w3, g1 = D1 * (g2 W2), g0 = D0 * (g1 W1), v = g0 W0x: a forward pass to layer 2 and a
// reverse pass of three GEMMs.  s itself, b3 and layer 2's activation are never formed.  One evaluation is six launches
// (seven when x comes as fp32 and is split first), all on the fp16x3 core of gemm_h3.cuh under this file's entry:
//   layers 0, 1   primal GEMMs on the forward blob's weight pairs, launched by cnf_tc.cu on its own primal GEMM (the
//                 same instantiation the Hutchinson field runs): bias, t W0[:, dim] at layer 0, activation, saturating
//                 (hi, lo) split, and D0, D1 in fp32 (two buffers: the reverse pass reads both);
//   layer 2       primal GEMM whose epilogue writes only the split of g2 * 2^k (GradSeedEpi);
//   reverse       e W^T on the prepared K-major transposed pairs W2^T, W1^T ([w][w]) and W0x^T ([dim][w]): the first
//                 two multiply by D and split (GradReverseEpi), the last writes v = acc 2^-k in fp32, row stride dim,
//                 any 4-byte alignment: dopri5's stage slots are misaligned for odd B (GradOutEpi).
// Scale of the reverse chain: the chain is linear in w3, so g2 carries ONE power of two 2^k, fixed when the blob is
// prepared and undone exactly by the last epilogue: the largest with max|W3| 2^k < 2^7 (from the forward blob's layer-3
// scale; a small trained W3 then keeps the splits in fp16's normal range) whose bound of every split of the chain,
// max|act'| max|W3| 2^k max(1, max|act'| C2, max|act'|^2 C2 C1) with C_l W_l's largest column abs-sum, stays at or
// below fp16's 65504, so no saturating split clamps for any input (DESIGN 3.18).  Scaling W3 by a power of two scales v
// by the same power, bit for bit.
// No floating-point atomics: the same call gives the same bits.  The Euler driver's init and step kernels work like
// cnf_tc.cu's: step index, time and the trajectory and span pointers live in a device struct, and a captured step
// replays for the whole trajectory.
#include <algorithm>

#include "gemm_h3.cuh"
#include "mlp_small.cuh"  // act_deriv_fast
#include "sde_common.cuh"

namespace cfm {

int cnf_tc_primal_hidden(const __half* ah, const __half* al, int batch, int K, const void* wh, const void* wl,
                         int64_t ldw, int w, const float* bias, const float* inv_ws, const float* tcol,
                         const float* t_dev, int act, float* dact, __half* out_hi, __half* out_lo,
                         cudaStream_t s);  // cnf_tc.cu

namespace {

bool grad_tc_shape(int batch, int dim, int w) { return mlp_tc_supported(batch, dim, w, dim) != 0; }

// the prepared blob: the chain's two scale factors {2^k, 2^-k / s_0}, then the K-major transposed (hi, lo) pairs of W0x
// ([dim][w]), W1 and W2 ([w][w]), row stride w, each layer scaled by the forward blob's power of two s_l for that layer
struct GradBlob {
  size_t sc, wth[3], wtl[3], total;
};
GradBlob grad_blob(int dim, int w) {
  GradBlob b;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes, 1024); return r; };
  b.sc = take(2 * sizeof(float));
  for (int l = 0; l < 3; ++l) {
    const size_t rows = l == 0 ? dim : w;
    b.wth[l] = take(rows * w * 2);
    b.wtl[l] = take(rows * w * 2);
  }
  b.total = o;
  return b;
}

struct GradWs {
  size_t xh, xl, ah, al, bh, bl, d0, d1, total;
};
GradWs grad_ws(int batch, int dim, int w) {
  GradWs p;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes, 1024); return r; };
  const size_t bd = (size_t)batch * dim, bw = (size_t)batch * w;
  p.xh = take(bd * 2); p.xl = take(bd * 2);
  p.ah = take(bw * 2); p.al = take(bw * 2); p.bh = take(bw * 2); p.bl = take(bw * 2);  // ping-pong operands
  p.d0 = take(bw * 4); p.d1 = take(bw * 4);
  p.total = o;
  return p;
}

// ---- prepare: W_l [w][cols] (stride lds, fp32, in the forward blob) -> (W_l s_l)^T split, [cols][w] -------------------
struct TransposeJob {
  const float* src;
  int64_t lds;
  int cols;
  const float* inv_ws;  // the forward blob's 1 / s_l (one power of two per layer)
  __half *hi, *lo;
};
struct TransposeJobs {
  TransposeJob j[3];
  const float* w3;       // the forward blob's W3 [w], fp32
  const float* inv_ws3;  // the forward blob's 1 / s_3
  float* sc;             // out: {2^k, 2^-k / s_0}
};

// max|act'| over the activations the field takes: SELU's lambda alpha = 1.75809934..., rounded up (SiLU's is 1.0998)
constexpr float kActPrimeMax = 1.7581f;
constexpr int kTransposeThreads = 256;

// The chain factors {2^k, 2^-k / s_0}, by one CTA of 256 threads.  The forward blob's layer-3 scale s_3 puts
// max|W3| s_3 in [2^13, 2^14), so s_3 2^-7 is the largest 2^k with max|W3| 2^k < 2^7.  Each reverse layer l multiplies
// |g| by at most max|act'| C_l, C_l = max_i sum_j |W_l[j, i]|, so every split sees at most
//     max|act'| max|W3| 2^k max(1, max|act'| C2, max|act'|^2 C2 C1);
// 2^k is lowered to the largest power of two that keeps this at or below 65504.  One thread per column adds its rows in
// order and the maxima are exact, so the factors do not depend on the schedule.  Both rules scale with max|W3| by
// exact powers of two, so W3 2^p still gives 2^-p 2^k.
__device__ __forceinline__ void grad_chain_scale(const TransposeJobs& jobs, int w) {
  __shared__ float red[3][kTransposeThreads / 32];
  float c1 = 0.f, c2 = 0.f, m3 = 0.f;
  for (int i = threadIdx.x; i < w; i += kTransposeThreads) {
    float s1 = 0.f, s2 = 0.f;
    for (int j = 0; j < w; ++j) {
      s1 += fabsf(__ldg(jobs.j[1].src + (int64_t)j * jobs.j[1].lds + i));
      s2 += fabsf(__ldg(jobs.j[2].src + (int64_t)j * jobs.j[2].lds + i));
    }
    c1 = fmaxf(c1, s1); c2 = fmaxf(c2, s2); m3 = fmaxf(m3, fabsf(__ldg(jobs.w3 + i)));
  }
  c1 = warp_max(c1); c2 = warp_max(c2); m3 = warp_max(m3);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { red[0][wid] = c1; red[1][wid] = c2; red[2][wid] = m3; }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int i = 1; i < kTransposeThreads / 32; ++i) {
    c1 = fmaxf(c1, red[0][i]); c2 = fmaxf(c2, red[1][i]); m3 = fmaxf(m3, red[2][i]);
  }
  float k = 0x1p-7f / __ldg(jobs.inv_ws3);
  const float b2 = kActPrimeMax * m3;            // |g2| / 2^k
  const float b1 = b2 * (kActPrimeMax * c2);     // |g1| / 2^k
  const float b0 = b1 * (kActPrimeMax * c1);     // |g0| / 2^k
  const float peak = fmaxf(b2, fmaxf(b1, b0));
  // the largest power of two <= 65504 / peak: the quotient's exponent bits (it is normal, or inf for a tiny peak)
  if (peak > 0.f && peak <= 3.0e38f) k = fminf(k, __int_as_float(__float_as_int(65504.f / peak) & 0x7f800000));
  jobs.sc[0] = k;
  jobs.sc[1] = __ldg(jobs.j[0].inv_ws) / k;
}

// one 32 x 32 tile of layer blockIdx.z < 3 per CTA: coalesced reads along the inputs, coalesced writes along the units;
// CTA (0, 0, 3) forms the chain factors (it reads only the forward blob, so it runs beside the tiles)
__global__ void __launch_bounds__(kTransposeThreads) grad_transpose_split_kernel(const TransposeJobs jobs, int w) {
  if (blockIdx.z == 3) {  // CTA-uniform
    if ((blockIdx.x | blockIdx.y) == 0) grad_chain_scale(jobs, w);
    return;
  }
  __shared__ float tile[32][33];
  const TransposeJob& J = jobs.j[blockIdx.z];
  const int u0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  if (c0 >= J.cols) return;  // CTA-uniform
  const float sc = 1.f / __ldg(J.inv_ws);  // exact: a power of two
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int u = u0 + ty + 8 * i, c = c0 + tx;
    tile[ty + 8 * i][tx] = (u < w && c < J.cols) ? J.src[(int64_t)u * J.lds + c] * sc : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + 8 * i, u = u0 + tx;
    if (c < J.cols && u < w) {
      __half h, l;
      split_h3(tile[tx][ty + 8 * i], h, l);
      J.hi[(int64_t)c * w + u] = h;
      J.lo[(int64_t)c * w + u] = l;
    }
  }
}

// ---- the field -----------------------------------------------------------------------------------------------------
// one row's 32 values -> their saturating (hi, lo) split at hi/lo + [0, n); n is a multiple of 4 (N = w or dim, both
// multiples of 8), so a partial chunk is whole quads too
__device__ __forceinline__ void split_row(const float (&v)[32], __half* hi, __half* lo, int n) {
#pragma unroll
  for (int g = 0; g < 8; ++g)
    if (4 * g < n) split4_store(make_float4(v[4 * g], v[4 * g + 1], v[4 * g + 2], v[4 * g + 3]), hi, lo, g);
}

// fp32 x -> its saturating (hi, lo) split, one thread per 4 columns
__global__ void __launch_bounds__(256) grad_split_kernel(const float4* __restrict__ x, __half* __restrict__ hi,
                                                         __half* __restrict__ lo, int64_t n4) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) split4_store(x[i], hi, lo, i);
}

// layer 2: pre = acc / s_2 + b2; g2 2^k = act'(pre) (w3 2^k), split
struct GradSeedEpi {
  const float* bias;
  const float* inv_ws;
  const float* w3;       // [w] fp32
  const float* sk;       // the prepared blob's 2^k
  int act;
  __half* out_hi;        // [B][ldo]
  __half* out_lo;
  int64_t ldo;
  __device__ __forceinline__ void begin_row(int, bool) {}
  __device__ __forceinline__ void store32(int row0, int lane, int col0, const float (&r)[32], int n0, int n1,
                                          float*) {
    const int row = row0 + lane;
    if (row >= n0) return;  // no warp-collective operation follows
    const float k = __ldg(sk);
    float g[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      g[c] = 0.f;
      if (col0 + c < n1) {
        const float p = fmaf(r[c], __ldg(inv_ws + col0 + c), __ldg(bias + col0 + c));
        g[c] = act_deriv_fast(p, act) * (__ldg(w3 + col0 + c) * k);
      }
    }
    split_row(g, out_hi + (int64_t)row * ldo + col0, out_lo + (int64_t)row * ldo + col0, n1 - col0);
  }
  __device__ __forceinline__ void finish(int) {}
};

// reverse GEMM of layer l = 2, 1: g_{l-1} = D_{l-1} (acc / s_l), split
struct GradReverseEpi {
  const float* inv_ws;   // the forward blob's 1 / s_l (uniform over the layer's rows)
  const float* dact;     // D_{l-1} [B][ldo]
  __half* out_hi;        // [B][ldo]
  __half* out_lo;
  int64_t ldo;
  __device__ __forceinline__ void begin_row(int, bool) {}
  __device__ __forceinline__ void store32(int row0, int lane, int col0, const float (&r)[32], int n0, int n1,
                                          float*) {
    const int row = row0 + lane;
    if (row >= n0) return;  // no warp-collective operation follows
    const bool full = col0 + 32 <= n1;
    const float* dr = dact + (int64_t)row * ldo + col0;  // 16-byte aligned when full (ldo % 8 == 0)
    float e[32];
    if (full) {
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(dr) + g);
        e[4 * g] = q.x; e[4 * g + 1] = q.y; e[4 * g + 2] = q.z; e[4 * g + 3] = q.w;
      }
    } else {
#pragma unroll
      for (int c = 0; c < 32; ++c) e[c] = col0 + c < n1 ? __ldg(dr + c) : 0.f;
    }
    const float s = __ldg(inv_ws);
#pragma unroll
    for (int c = 0; c < 32; ++c) e[c] *= r[c] * s;
    split_row(e, out_hi + (int64_t)row * ldo + col0, out_lo + (int64_t)row * ldo + col0, n1 - col0);
  }
  __device__ __forceinline__ void finish(int) {}
};

// reverse GEMM of layer 0: v = acc 2^-k / s_0, fp32
struct GradOutEpi {
  const float* scale;    // the prepared blob's 2^-k / s_0
  float* v;              // [B][ldo], any 4-byte alignment
  int64_t ldo;
  __device__ __forceinline__ void begin_row(int, bool) {}
  __device__ __forceinline__ void store32(int row0, int lane, int col0, const float (&r)[32], int n0, int n1,
                                          float* tile) {
    const int row = row0 + lane;
    const float s = __ldg(scale);
    float e[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) e[c] = r[c] * s;
    float* base = v + (int64_t)row0 * ldo + col0;
    if (col0 + 32 <= n1 && (ldo & 3) == 0 && aligned16(base)) {
      tc_store_chunk32(tile, e, base, ldo, n0 - row0, lane);
    } else if (row < n0) {
#pragma unroll
      for (int c = 0; c < 32; ++c)
        if (col0 + c < n1) v[(int64_t)row * ldo + col0 + c] = e[c];
    }
  }
  __device__ __forceinline__ void finish(int) {}
};

// The GEMMs of this file: the persistent fp16x3 core of gemm_tc.cuh under an entry of their own, so that the
// instantiations other files' tests pin stay as they are; tests/test_grad_tc_host.py pins these three.
template <class Epi>
__global__ void __launch_bounds__(kWgThreads, 1)
grad_gemm_kernel(const __grid_constant__ CUtensorMap map_ah, const __grid_constant__ CUtensorMap map_al,
                 const __grid_constant__ CUtensorMap map_bh, const __grid_constant__ CUtensorMap map_bl,
                 const TcShape p, Epi epi) {
  gemm_wg_body<H3Scheme, Epi, false>(map_ah, map_al, map_bh, map_bl, p, epi);
}

// ---- Euler driver -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
grad_euler_init_kernel(cfm_grad_tc_state* __restrict__ st, const float4* __restrict__ x0, float4* __restrict__ x,
                       __half* __restrict__ hi, __half* __restrict__ lo, float4* traj, const float* t_span,
                       int n_steps, int64_t n4) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    st->traj = reinterpret_cast<float*>(traj); st->t_span = t_span;
    st->n = 0; st->n_steps = n_steps; st->t = t_span[0]; st->ticket = 0u;
  }
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = x0[i];
    x[i] = v;
    traj[i] = v;
    split4_store(v, hi, lo, i);
  }
}

// step n = st->n: x <- fmaf(h, v, x), traj[n + 1], the split of x; the CTA that finishes last advances the state.  A
// step enqueued past n_steps does nothing.
__global__ void __launch_bounds__(256)
grad_euler_step_kernel(cfm_grad_tc_state* st, float4* __restrict__ x, const float4* __restrict__ v,
                       __half* __restrict__ hi, __half* __restrict__ lo, int64_t n4) {
  const int n = st->n;
  if (n >= st->n_steps) return;
  const float* ts = st->t_span;
  const float t0 = ts[n], t1 = ts[n + 1];
  const float h = (float)((double)t1 - (double)t0);  // the plain Euler driver's step: float(ts[n + 1] - ts[n])
  float4* out = reinterpret_cast<float4*>(st->traj) + (int64_t)(n + 1) * n4;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 a = x[i], k = v[i];
    const float4 r = make_float4(fmaf(h, k.x, a.x), fmaf(h, k.y, a.y), fmaf(h, k.z, a.z), fmaf(h, k.w, a.w));
    x[i] = r;
    out[i] = r;
    split4_store(r, hi, lo, i);
  }
  step_advance(st, n, t1);
}

}  // namespace

}  // namespace cfm

using namespace cfm;

extern "C" int cfm_grad_tc_supported(int batch, int dim, int w) { return grad_tc_shape(batch, dim, w) ? 1 : 0; }

extern "C" size_t cfm_grad_tc_prepared_bytes(int dim, int w) {
  return grad_tc_shape(128, dim, w) ? grad_blob(dim, w).total : 0;
}

extern "C" int cfm_grad_tc_prepare(const void* mlp_prepared, int dim, int w, void* prepared, size_t prepared_bytes,
                                   void* stream) {
  const char* what = "cfm_grad_tc_prepare";
  CFM_REQUIRE(mlp_prepared && prepared, "%s: null pointer", what);
  CFM_REQUIRE(grad_tc_shape(128, dim, w),
              "%s: unsupported shape dim=%d w=%d (dim >= 32, dim and w multiples of 8, w >= 32)", what, dim, w);
  const GradBlob G = grad_blob(dim, w);
  CFM_REQUIRE(prepared_bytes >= G.total, "%s: blob too small (%zu < %zu)", what, prepared_bytes, G.total);
  CFM_REQUIRE(aligned16(mlp_prepared) && aligned16(prepared), "%s: both blobs must be 16-byte aligned", what);
  const MlpBlobHeader h = mlp_layout(dim, w, 1, 1);
  const MlpTcWeights W = mlp_tc_weights(h, mlp_prepared);
  const char* src = reinterpret_cast<const char*>(mlp_prepared);
  char* dst = reinterpret_cast<char*>(prepared);
  const int64_t off[3] = {h.off_w0x, h.off_w1, h.off_w2}, lds[3] = {h.dimp, w, w};
  TransposeJobs J;
  J.w3 = reinterpret_cast<const float*>(src + h.off_w3);
  J.inv_ws3 = W.inv_ws[3];
  J.sc = reinterpret_cast<float*>(dst + G.sc);
  for (int l = 0; l < 3; ++l)
    J.j[l] = TransposeJob{reinterpret_cast<const float*>(src + off[l]), lds[l], l ? w : dim, W.inv_ws[l],
                          reinterpret_cast<__half*>(dst + G.wth[l]), reinterpret_cast<__half*>(dst + G.wtl[l])};
  const dim3 grid((w + 31) / 32, (std::max(dim, w) + 31) / 32, 4);  // z = 3: the chain factors' CTA
  grad_transpose_split_kernel<<<grid, kTransposeThreads, 0, (cudaStream_t)stream>>>(J, w);
  note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}

extern "C" size_t cfm_grad_tc_workspace_bytes(int batch, int dim, int w) {
  return grad_tc_shape(batch, dim, w) ? grad_ws(batch, dim, w).total : 0;
}

extern "C" int cfm_grad_tc_field_f32(const void* mlp_prepared, const void* grad_prepared, const float* x,
                                     const void* x_hi, const void* x_lo, int batch, int dim, int w, int act,
                                     const float* t_dev, float* v, void* workspace, size_t workspace_bytes,
                                     void* stream) {
  const char* what = "cfm_grad_tc_field_f32";
  CFM_REQUIRE(mlp_prepared && grad_prepared && v && workspace && t_dev, "%s: null pointer", what);
  CFM_REQUIRE((x != nullptr) != (x_hi != nullptr) && (x_hi == nullptr) == (x_lo == nullptr),
              "%s: pass either x or the pair (x_hi, x_lo)", what);
  CFM_REQUIRE(act == CFM_ACT_SELU || act == CFM_ACT_SILU, "%s: unknown activation %d", what, act);
  CFM_REQUIRE(grad_tc_shape(batch, dim, w),
              "%s: unsupported shape B=%d dim=%d w=%d (B >= 128, dim >= 32, dim and w multiples of 8, w >= 32)", what,
              batch, dim, w);
  const GradWs P = grad_ws(batch, dim, w);
  CFM_REQUIRE(workspace_bytes >= P.total, "%s: workspace too small (%zu < %zu)", what, workspace_bytes, P.total);
  CFM_REQUIRE(aligned16(x) && aligned16(x_hi) && aligned16(x_lo) && aligned16(workspace) && aligned16(mlp_prepared) &&
                  aligned16(grad_prepared),
              "%s: x, x_hi, x_lo, the blobs and the workspace must be 16-byte aligned", what);
  CFM_REQUIRE((reinterpret_cast<uintptr_t>(v) & 3) == 0, "%s: v must be 4-byte aligned", what);
  cudaStream_t s = (cudaStream_t)stream;
  const MlpBlobHeader h = mlp_layout(dim, w, 1, 1);
  const MlpTcWeights W = mlp_tc_weights(h, mlp_prepared);
  const GradBlob G = grad_blob(dim, w);
  const char* blob = reinterpret_cast<const char*>(mlp_prepared);
  const char* gblob = reinterpret_cast<const char*>(grad_prepared);
  char* ws = reinterpret_cast<char*>(workspace);
  auto H = [&](size_t off) { return reinterpret_cast<__half*>(ws + off); };
  auto F = [&](int64_t off) { return reinterpret_cast<const float*>(blob + off); };
  auto GH = [&](size_t off) { return reinterpret_cast<const __half*>(gblob + off); };
  float* d[2] = {reinterpret_cast<float*>(ws + P.d0), reinterpret_cast<float*>(ws + P.d1)};
  int rc;

  const __half* ph = reinterpret_cast<const __half*>(x_hi);
  const __half* pl = reinterpret_cast<const __half*>(x_lo);
  if (x != nullptr) {
    const int64_t n4 = (int64_t)batch * dim / 4;
    grad_split_kernel<<<ew_grid(n4), 256, 0, s>>>(reinterpret_cast<const float4*>(x), H(P.xh), H(P.xl), n4);
    note_launches(1);
    CFM_CUDA_OK(cudaGetLastError());
    ph = H(P.xh); pl = H(P.xl);
  }
  // forward: layers 0, 1 -> a (split) and D; layer 2 -> g2 2^k (split)
  const int64_t boff[3] = {h.off_b0, h.off_b1, h.off_b2};
  for (int l = 0; l < 2; ++l) {
    const int K = l ? w : dim;
    __half* oh = H(l ? P.bh : P.ah);
    __half* ol = H(l ? P.bl : P.al);
    rc = cnf_tc_primal_hidden(ph, pl, batch, K, W.wh[l], W.wl[l], W.ld[l], w, F(boff[l]), W.inv_ws[l],
                              l == 0 ? F(h.off_w0t) : nullptr, t_dev, act, d[l], oh, ol, s);
    if (rc != CFM_OK) return rc;
    ph = oh; pl = ol;
  }
  const float* sc = reinterpret_cast<const float*>(gblob + G.sc);
  GradSeedEpi se{F(boff[2]), W.inv_ws[2], F(h.off_w3), sc, act, H(P.ah), H(P.al), w};
  rc = launch_gemm_h3<GradSeedEpi, grad_gemm_kernel<GradSeedEpi>>(
      ph, pl, batch, w, reinterpret_cast<const __half*>(W.wh[2]), reinterpret_cast<const __half*>(W.wl[2]), w, W.ld[2],
      w, se, s);
  if (rc != CFM_OK) return rc;
  // reverse: g1 = D1 (g2 W2) into b, g0 = D0 (g1 W1) into a, v = g0 W0x
  GradReverseEpi r2{W.inv_ws[2], d[1], H(P.bh), H(P.bl), w};
  rc = launch_gemm_h3<GradReverseEpi, grad_gemm_kernel<GradReverseEpi>>(H(P.ah), H(P.al), batch, w, GH(G.wth[2]),
                                                                         GH(G.wtl[2]), w, w, w, r2, s);
  if (rc != CFM_OK) return rc;
  GradReverseEpi r1{W.inv_ws[1], d[0], H(P.ah), H(P.al), w};
  rc = launch_gemm_h3<GradReverseEpi, grad_gemm_kernel<GradReverseEpi>>(H(P.bh), H(P.bl), batch, w, GH(G.wth[1]),
                                                                         GH(G.wtl[1]), w, w, w, r1, s);
  if (rc != CFM_OK) return rc;
  GradOutEpi r0{sc + 1, v, dim};
  rc = launch_gemm_h3<GradOutEpi, grad_gemm_kernel<GradOutEpi>>(H(P.ah), H(P.al), batch, w, GH(G.wth[0]),
                                                                 GH(G.wtl[0]), dim, w, w, r0, s);
  if (rc != CFM_OK) return rc;
  return CFM_OK;
}

extern "C" int cfm_grad_tc_euler_init(cfm_grad_tc_state* state, const float* x0, float* x, void* x_hi, void* x_lo,
                                      float* traj, const float* t_span, int n_span, int batch, int dim,
                                      void* stream) {
  const char* what = "cfm_grad_tc_euler_init";
  CFM_REQUIRE(state && x0 && x && x_hi && x_lo && traj && t_span, "%s: null pointer", what);
  CFM_REQUIRE(n_span >= 2, "%s: n_span must be >= 2 (got %d)", what, n_span);
  if (const int rc = tc_state_shape(what, batch, dim)) return rc;
  CFM_REQUIRE(aligned16(x0) && aligned16(x) && aligned16(x_hi) && aligned16(x_lo) && aligned16(traj) &&
                  (reinterpret_cast<uintptr_t>(state) & 7) == 0,
              "%s: x0, x, x_hi, x_lo and traj must be 16-byte aligned, the state 8-byte aligned", what);
  const int64_t n4 = (int64_t)batch * dim / 4;
  grad_euler_init_kernel<<<ew_grid(n4), 256, 0, (cudaStream_t)stream>>>(
      state, reinterpret_cast<const float4*>(x0), reinterpret_cast<float4*>(x), reinterpret_cast<__half*>(x_hi),
      reinterpret_cast<__half*>(x_lo), reinterpret_cast<float4*>(traj), t_span, n_span - 1, n4);
  note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}

extern "C" int cfm_grad_tc_euler_step(cfm_grad_tc_state* state, float* x, const float* v, void* x_hi, void* x_lo,
                                      int batch, int dim, void* stream) {
  const char* what = "cfm_grad_tc_euler_step";
  CFM_REQUIRE(state && x && v && x_hi && x_lo, "%s: null pointer", what);
  if (const int rc = tc_state_shape(what, batch, dim)) return rc;
  CFM_REQUIRE(aligned16(x) && aligned16(v) && aligned16(x_hi) && aligned16(x_lo) &&
                  (reinterpret_cast<uintptr_t>(state) & 7) == 0,
              "%s: x, v, x_hi and x_lo must be 16-byte aligned, the state 8-byte aligned", what);
  const int64_t n4 = (int64_t)batch * dim / 4;
  grad_euler_step_kernel<<<ew_grid(n4), 256, 0, (cudaStream_t)stream>>>(
      state, reinterpret_cast<float4*>(x), reinterpret_cast<const float4*>(v), reinterpret_cast<__half*>(x_hi),
      reinterpret_cast<__half*>(x_lo), n4);
  note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
