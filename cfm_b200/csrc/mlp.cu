// MLP vector field  y = net(cat([x, t], 1))
// (reference: torchcfm/models/models.py:4-21 composed with torchcfm/utils.py:51-52).
//
// Layout: x (B, dim) fp32 row-major; weights in nn.Linear layout (out, in).  cfm_mlp_prepare
// builds, once per weight set, a device blob with
//   * the first-layer weight split into its x-part (w, dim) -- rows padded to a multiple of 4
//     floats so every row is 16-byte aligned -- and its t-column (w): since t is one scalar for
//     the whole batch (utils.py:52), cat([x, t]) @ W0^T == x @ W0x^T + t * w0t, so the
//     (B, dim+1) concatenation is never materialised and t folds into the bias;
//   * the remaining weights / biases copied contiguously;
//   * (algo 2) row-scaled fp16 (hi, lo) splits of all weights for the tensor-core paths (mlp_h3.cu).
// algo 1 (this file): four SIMT fp32 GEMMs with fused bias + activation epilogues (true fp32
// FMA, the numerics of the reference's cuBLAS sgemm with TF32 off).
#include "gemm_simt.cuh"
#include "mlp_common.cuh"

namespace cfm {

__global__ void mlp_split_w0_kernel(const float* __restrict__ W0, int w, int dim, int in0, int dimp,
                                    float* __restrict__ w0x, float* __restrict__ w0t) {
  const int n = blockIdx.x;
  for (int k = threadIdx.x; k < dimp; k += blockDim.x)
    w0x[(int64_t)n * dimp + k] = k < dim ? W0[(int64_t)n * in0 + k] : 0.f;
  if (threadIdx.x == 0) w0t[n] = in0 > dim ? W0[(int64_t)n * in0 + dim] : 0.f;
}

// the blob header travels as a kernel argument (by value): no host buffer has to outlive the call, no sync
__global__ void mlp_write_header_kernel(const MlpBlobHeader h, MlpBlobHeader* dst) { *dst = h; }

struct BiasActEpilogue {
  const float* bias;   // (N)
  const float* tcol;   // (N) or null: + t * tcol[n]
  const float* t_dev;  // device scalar or null
  float t_host;
  int act;             // -1: none
  float* out;
  int64_t ldo;
  __device__ __forceinline__ void operator()(int m, int n, float4 acc, int valid) {
    const float t = tcol ? (t_dev ? __ldg(t_dev) : t_host) : 0.f;
    float o[4] = {acc.x, acc.y, acc.z, acc.w};
    float* dst = out + (int64_t)m * ldo + n;
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (c < valid) {
        float v = o[c] + bias[n + c];
        if (tcol) v = fmaf(t, tcol[n + c], v);
        o[c] = act >= 0 ? act_apply(v, act) : v;
      }
    if (valid == 4 && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
      *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
    } else {
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (c < valid) dst[c] = o[c];
    }
  }
  __device__ __forceinline__ void finish() {}
};

}  // namespace cfm

using namespace cfm;

extern "C" size_t cfm_mlp_prepared_bytes(int dim, int w, int out_dim, int time_varying) {
  return (size_t)mlp_layout(dim, w, out_dim, time_varying).total;
}

extern "C" int cfm_mlp_prepare(const float* W0, const float* b0, const float* W1, const float* b1,
                               const float* W2, const float* b2, const float* W3, const float* b3,
                               int dim, int w, int out_dim, int time_varying, void* prepared,
                               size_t prepared_bytes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  CFM_REQUIRE(W0 && b0 && W1 && b1 && W2 && b2 && W3 && b3 && prepared, "cfm_mlp_prepare: null pointer");
  CFM_REQUIRE(dim > 0 && w > 0 && out_dim > 0, "cfm_mlp_prepare: bad dims");
  const MlpBlobHeader h = mlp_layout(dim, w, out_dim, time_varying ? 1 : 0);
  CFM_REQUIRE(prepared_bytes >= (size_t)h.total, "cfm_mlp_prepare: blob too small (%zu < %lld)",
              prepared_bytes, (long long)h.total);
  char* B = reinterpret_cast<char*>(prepared);
  mlp_write_header_kernel<<<1, 1, 0, s>>>(h, reinterpret_cast<MlpBlobHeader*>(B)); ::cfm::note_launches(1);
  const int in0 = dim + (time_varying ? 1 : 0);
  mlp_split_w0_kernel<<<w, 256, 0, s>>>(W0, w, dim, in0, h.dimp, reinterpret_cast<float*>(B + h.off_w0x),
                                        reinterpret_cast<float*>(B + h.off_w0t)); ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  auto cp = [&](int64_t off, const float* src, size_t n) {
    return cudaMemcpyAsync(B + off, src, n * 4, cudaMemcpyDeviceToDevice, s);
  };
  CFM_CUDA_OK(cp(h.off_b0, b0, w));
  CFM_CUDA_OK(cp(h.off_w1, W1, (size_t)w * w));
  CFM_CUDA_OK(cp(h.off_b1, b1, w));
  CFM_CUDA_OK(cp(h.off_w2, W2, (size_t)w * w));
  CFM_CUDA_OK(cp(h.off_b2, b2, w));
  CFM_CUDA_OK(cp(h.off_w3, W3, (size_t)out_dim * w));
  CFM_CUDA_OK(cp(h.off_b3, b3, out_dim));
  return mlp_tc_prepare(h, prepared, s);
}

extern "C" size_t cfm_mlp_workspace_bytes(int batch, int dim, int w, int out_dim, int algo) {
  size_t b = 2 * align_up((size_t)batch * w * 4, 256);
  if (algo != 1) {
    const size_t t = mlp_tc_workspace_bytes(batch, dim, w, out_dim);
    if (t > b) b = t;
  }
  return b;
}

extern "C" int cfm_mlp_forward_f32(const void* prepared, const float* x, int batch, int dim, int w,
                                   int out_dim, int time_varying, const float* t_dev, float t_host,
                                   int act, float* y, int algo, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  CFM_REQUIRE(prepared && x && y && workspace, "cfm_mlp_forward_f32: null pointer");
  CFM_REQUIRE(batch > 0, "cfm_mlp_forward_f32: batch must be > 0");
  CFM_REQUIRE(act == CFM_ACT_SELU || act == CFM_ACT_SILU, "cfm_mlp_forward_f32: unknown activation %d", act);
  CFM_REQUIRE(algo >= 0 && algo <= 2, "cfm_mlp_forward_f32: unknown algo %d", algo);
  const MlpBlobHeader h = mlp_layout(dim, w, out_dim, time_varying ? 1 : 0);
  const bool tc_ok = mlp_tc_supported(batch, dim, w, out_dim) != 0;
  if (algo == 2) CFM_REQUIRE(tc_ok, "cfm_mlp_forward_f32: tensor-core path unsupported for this shape");
  const bool use_tc = algo == 2 || (algo == 0 && tc_ok);
  CFM_REQUIRE(workspace_bytes >= cfm_mlp_workspace_bytes(batch, dim, w, out_dim, use_tc ? 2 : 1),
              "cfm_mlp_forward_f32: workspace too small");
  const char* B = reinterpret_cast<const char*>(prepared);
  if (use_tc)
    return mlp_tc_forward(h, prepared, x, nullptr, nullptr, batch, t_dev, t_host, act, y, workspace,
                          workspace_bytes, nullptr, s);
  auto P = [&](int64_t off) { return reinterpret_cast<const float*>(B + off); };
  float* hA = reinterpret_cast<float*>(workspace);
  float* hB = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + align_up((size_t)batch * w * 4, 256));
  BiasActEpilogue e0{P(h.off_b0), time_varying ? P(h.off_w0t) : nullptr, t_dev, t_host, act, hA, (int64_t)w};
  CFM_CUDA_OK(launch_gemm_nt_simt(x, (int64_t)dim, P(h.off_w0x), (int64_t)h.dimp, batch, w, dim, e0, s));
  BiasActEpilogue e1{P(h.off_b1), nullptr, nullptr, 0.f, act, hB, (int64_t)w};
  CFM_CUDA_OK(launch_gemm_nt_simt(hA, (int64_t)w, P(h.off_w1), (int64_t)w, batch, w, w, e1, s));
  BiasActEpilogue e2{P(h.off_b2), nullptr, nullptr, 0.f, act, hA, (int64_t)w};
  CFM_CUDA_OK(launch_gemm_nt_simt(hB, (int64_t)w, P(h.off_w2), (int64_t)w, batch, w, w, e2, s));
  BiasActEpilogue e3{P(h.off_b3), nullptr, nullptr, 0.f, -1, y, (int64_t)out_dim};
  CFM_CUDA_OK(launch_gemm_nt_simt(hA, (int64_t)w, P(h.off_w3), (int64_t)w, batch, out_dim, w, e3, s));
  return CFM_OK;
}

extern "C" int cfm_mlp_tc_supported(int batch, int dim, int w, int out_dim) {
  return mlp_tc_supported(batch, dim, w, out_dim);
}

extern "C" int cfm_mlp_forward_split_gated_f32(const void* prepared, const void* x_hi, const void* x_lo, int batch,
                                               int dim, int w, int out_dim, int time_varying, const float* t_dev,
                                               float t_host, int act, float* y, const int32_t* skip_if_nonzero,
                                               void* workspace, size_t workspace_bytes, void* stream) {
  CFM_REQUIRE(prepared && x_hi && x_lo && y && workspace, "cfm_mlp_forward_split_gated_f32: null pointer");
  CFM_REQUIRE(act == CFM_ACT_SELU || act == CFM_ACT_SILU,
              "cfm_mlp_forward_split_gated_f32: unknown activation %d", act);
  CFM_REQUIRE(mlp_tc_supported(batch, dim, w, out_dim) != 0,
              "cfm_mlp_forward_split_gated_f32: shape not supported by the tensor-core path");
  const MlpBlobHeader h = mlp_layout(dim, w, out_dim, time_varying ? 1 : 0);
  return mlp_tc_forward(h, prepared, nullptr, x_hi, x_lo, batch, t_dev, t_host, act, y, workspace,
                        workspace_bytes, skip_if_nonzero, (cudaStream_t)stream);
}
