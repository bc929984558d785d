// Cost matrix  M = torch.cdist(x0, x1) ** 2   (reference: torchcfm/optimal_transport.py:84)
//
// HBM layout: x0 (n0,d), x1 (n1,d) fp32 row-major; M (n0,n1) fp32 row-major, row stride ldm.
// Two code paths behind cfm_sqdist_f32 (algo 0 = auto picks one of them; 2, a retired 3xTF32 path, is refused):
//   algo 1  SIMT fp32 FMA GEMM (gemm_simt.cuh)      -- any shape / alignment
//   algo 3  wgmma fp16x3 GEMM (sqdist_h3.cu)        -- d % 4 == 0, 16B-aligned rows
// Both apply the epilogue
//   M_ij = (sqrt(max(|x0_i|^2 + |x1_j|^2 - 2 <x0_i, x1_j>, 0)))^2
// which follows ATen's _euclidean_dist (clamp_min(0).sqrt()) and the reference's `** 2`.
#include "gemm_simt.cuh"

namespace cfm {

// one warp per row: |x_r|^2 in fp32
__global__ void row_sqnorm_kernel(const float* __restrict__ X, int rows, int d,
                                  float* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const float* p = X + (int64_t)warp * d;
  float s = 0.f;
  for (int k = lane; k < d; k += 32) s = fmaf(p[k], p[k], s);
  s = warp_sum(s);
  if (lane == 0) out[warp] = s;
}

struct SqDistEpilogue {
  const float* nx;  // |x0_i|^2
  const float* ny;  // |x1_j|^2
  float* M;
  int64_t ldm;
  float* cost_max;  // nullable
  int squared;
  float tmax;

  __device__ __forceinline__ float one(float dot, float a, float b) {
    const float d2 = (a + b) - 2.f * dot;
    float v = d2 < 0.f ? 0.f : d2;  // clamp_min(0) that lets NaN through, like ATen's (fmaxf would swallow it)
    float r = __fsqrt_rn(v);
    return squared ? r * r : r;
  }
  __device__ __forceinline__ void operator()(int m, int n, float4 acc, int valid) {
    const float a = nx[m];
    float* dst = M + (int64_t)m * ldm + n;
    float o[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (c < valid) {
        o[c] = one(o[c], a, ny[n + c]);
        tmax = fmaxf(tmax, o[c]);
      }
    if (valid == 4 && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
      *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
    } else {
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (c < valid) dst[c] = o[c];
    }
  }
  __device__ __forceinline__ void finish() {
    if (cost_max == nullptr) return;
    float m = warp_max(tmax);
    if ((threadIdx.x & 31) == 0) atomic_max_nonneg(cost_max, m);
  }
};

// shapes the tensor-core path takes: whole 16-byte units per row, 16-byte aligned operands
static bool tc_supported(int d, const float* x0, const float* x1, const float* M, int64_t ldm) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(x0) | reinterpret_cast<uintptr_t>(x1) | reinterpret_cast<uintptr_t>(M);
  return (d % 4 == 0) && (a % 16 == 0) && (ldm % 4 == 0);
}

// implemented in sqdist_h3.cu (fp16x3 scheme; the pre-pass also writes the row norms)
size_t sqdist_h3_workspace_bytes(int n0, int n1, int d);
int sqdist_h3_launch(const float* x0, const float* x1, float* M, int n0, int n1, int d, int64_t ldm, int squared,
                     float* cost_max, float* nx, float* ny, void* ws, size_t ws_bytes, cudaStream_t s);

static size_t norms_bytes(int n0, int n1) {
  return align_up((size_t)n0 * 4, 256) + align_up((size_t)n1 * 4, 256);
}

}  // namespace cfm

using namespace cfm;

extern "C" size_t cfm_sqdist_workspace_bytes(int n0, int n1, int d, int algo) {
  size_t b = norms_bytes(n0, n1);
  if (algo != 1) b += sqdist_h3_workspace_bytes(n0, n1, d);  // auto / 3
  return b;
}

extern "C" int cfm_sqdist_f32(const float* x0, const float* x1, float* M, int n0, int n1, int d,
                              int64_t ldm, int squared, float* cost_max, int algo,
                              void* workspace, size_t workspace_bytes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  CFM_REQUIRE(x0 && x1 && M, "cfm_sqdist_f32: null pointer");
  CFM_REQUIRE(n0 > 0 && n1 > 0 && d > 0 && ldm >= n1, "cfm_sqdist_f32: bad shape n0=%d n1=%d d=%d ldm=%lld",
              n0, n1, d, (long long)ldm);
  CFM_REQUIRE(algo == 0 || algo == 1 || algo == 3, "cfm_sqdist_f32: unknown algo %d", algo);
  const bool tc_ok = tc_supported(d, x0, x1, M, ldm);
  if (algo == 3) CFM_REQUIRE(tc_ok, "cfm_sqdist_f32: tensor-core path needs d %% 4 == 0, 16B-aligned x0/x1/M and ldm %% 4 == 0");
  const bool use_h3 = (algo == 3) || (algo == 0 && tc_ok && (int64_t)n0 * n1 >= 256 * 256 && d >= 32);
  const size_t need = norms_bytes(n0, n1) + (use_h3 ? sqdist_h3_workspace_bytes(n0, n1, d) : 0);
  CFM_REQUIRE(workspace && workspace_bytes >= need, "cfm_sqdist_f32: workspace too small (%zu < %zu)",
              workspace_bytes, need);
  float* nx = reinterpret_cast<float*>(workspace);
  float* ny = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + align_up((size_t)n0 * 4, 256));
  void* tcws = reinterpret_cast<char*>(workspace) + norms_bytes(n0, n1);

  if (cost_max) CFM_CUDA_OK(cudaMemsetAsync(cost_max, 0, sizeof(float), s));
  if (use_h3)  // norms, row scales and the fp16 operand split come from one fused pre-pass per input
    return sqdist_h3_launch(x0, x1, M, n0, n1, d, ldm, squared, cost_max, nx, ny, tcws,
                            workspace_bytes - norms_bytes(n0, n1), s);
  row_sqnorm_kernel<<<(n0 + 7) / 8, 256, 0, s>>>(x0, n0, d, nx); ::cfm::note_launches(1);
  row_sqnorm_kernel<<<(n1 + 7) / 8, 256, 0, s>>>(x1, n1, d, ny); ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  SqDistEpilogue epi{nx, ny, M, ldm, cost_max, squared, 0.f};
  CFM_CUDA_OK(launch_gemm_nt_simt(x0, (int64_t)d, x1, (int64_t)d, n0, n1, d, epi, s));
  return CFM_OK;
}
