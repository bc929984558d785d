// Shared between mlp.cu (SIMT path, prepare/forward entry points) and mlp_h3.cu (tensor-core paths).
#pragma once
#include "common.cuh"

namespace cfm {

struct MlpBlobHeader {
  int32_t magic, dim, w, out_dim, time_varying, dimp;  // dimp = dim rounded up to 4
  int64_t off_w0x, off_w0t, off_b0, off_w1, off_b1, off_w2, off_b2, off_w3, off_b3, off_tc, total;
};
constexpr int32_t kMlpMagic = 0x4d4c5031;  // "MLP1"

size_t mlp_tc_blob_bytes(int dim, int w, int out_dim);  // mlp_h3.cu
int mlp_tc_prepare(const MlpBlobHeader& h, void* blob, cudaStream_t s);
int mlp_tc_supported(int batch, int dim, int w, int out_dim);
size_t mlp_tc_workspace_bytes(int batch, int dim, int w, int out_dim);
int mlp_tc_forward(const MlpBlobHeader& h, const void* blob, const float* x, const void* x_hi,
                   const void* x_lo, int batch, const float* t_dev, float t_host, int act, float* y, void* ws,
                   size_t ws_bytes, const int32_t* skip, cudaStream_t s);
// two weight blobs of one shape on the same (x_hi, x_lo): y_a = net_a(x), y_b = net_b(x); ws holds two
// mlp_tc_workspace_bytes halves
int mlp_tc_pair_forward(const MlpBlobHeader& h, const void* blob_a, const void* blob_b, const void* x_hi,
                        const void* x_lo, int batch, const float* t_dev, float t_host, int act, float* y_a,
                        float* y_b, void* ws, size_t ws_bytes, cudaStream_t s);
// the tensor-core section of a prepared blob, layer l = 0..3: fp16 weight pair (hi, lo) [rows][ld[l]] (rows scaled by
// one power of two per layer) and the per-row inverse scale; ld[0] covers W0's x columns only (cnf_tc.cu)
struct MlpTcWeights {
  const void* wh[4];
  const void* wl[4];
  const float* inv_ws[4];
  int64_t ld[4];
};
MlpTcWeights mlp_tc_weights(const MlpBlobHeader& h, const void* blob);

static inline MlpBlobHeader mlp_layout(int dim, int w, int out_dim, int tv) {
  MlpBlobHeader h;
  memset(&h, 0, sizeof(h));
  h.magic = kMlpMagic; h.dim = dim; h.w = w; h.out_dim = out_dim; h.time_varying = tv;
  h.dimp = (dim + 3) / 4 * 4;
  size_t o = align_up(sizeof(MlpBlobHeader), 256);
  auto take = [&](size_t floats) { size_t r = o; o += align_up(floats * 4, 256); return (int64_t)r; };
  h.off_w0x = take((size_t)w * h.dimp);
  h.off_w0t = take(w);
  h.off_b0 = take(w);
  h.off_w1 = take((size_t)w * w);
  h.off_b1 = take(w);
  h.off_w2 = take((size_t)w * w);
  h.off_b2 = take(w);
  h.off_w3 = take((size_t)out_dim * w);
  h.off_b3 = take(out_dim);
  h.off_tc = (int64_t)o;
  o += mlp_tc_blob_bytes(dim, w, out_dim);
  h.total = (int64_t)o;
  return h;
}

__device__ __forceinline__ float act_apply(float x, int act) {
  if (act == CFM_ACT_SELU) {
    const float scale = 1.0507009873554804934193349852946f;
    const float negcoef = (float)(1.6732632423543772848170429916717 * 1.0507009873554804934193349852946);
    return x > 0.f ? x * scale : expm1f(x) * negcoef;
  }
  return x / (1.f + __expf(-x));  // SiLU
}

// branch-free variant for the tensor-core epilogues (issue-bound: every instruction per element counts).
// SELU negative branch: expm1(x) = ex2(x log2e) - 1.  Near zero the subtraction cancels, so the RELATIVE
// error of the result grows, but its ABSOLUTE error stays at ~1.5e-7 (ex2.approx is good to 2^-22 of a value
// <= 1), which is what the max-norm gate of the MLP (1e-5 of max|y|) sees; the SIMT path keeps expm1f.
// SiLU through one ex2 and one fast reciprocal.
template <int ACT>
__device__ __forceinline__ float act_fast(float x) {
  if (ACT == CFM_ACT_SELU) {
    const float scale = 1.0507009873554804934193349852946f;
    const float negcoef = (float)(1.6732632423543772848170429916717 * 1.0507009873554804934193349852946);
    // e overflows to +inf for large positive x; the select discards that branch (NaN still propagates: NaN > 0 is false)
    const float e = ex2f(x * kLog2e);
    const float neg = fmaf(e, negcoef, -negcoef);
    return x > 0.f ? x * scale : neg;
  }
  return __fdividef(x, 1.f + ex2f(-x * kLog2e));
}
__device__ __forceinline__ float act_apply_fast(float x, int act) {
  return act == CFM_ACT_SELU ? act_fast<CFM_ACT_SELU>(x) : act_fast<CFM_ACT_SILU>(x);
}

}  // namespace cfm
