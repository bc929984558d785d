// Pieces shared by the training kernels of small MLPs: mlp_train_kernel (train_small.cu, the flow-matching loss) and
// mlp_action_train_kernel (action_train.cu, the action-matching loss).  Both stream rows in tiles of kTile, add outer
// products into per-thread registers and fold per-CTA partials in CTA order after one grid barrier; they share the
// workspace layout [grid] float64 loss partials, then [grid][n_params] floats, which
// cfm_mlp_small_train_workspace_bytes sizes.
#pragma once
#include <cooperative_groups.h>

#include "mlp_small.cuh"

namespace cfm {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kTile = kWarps * RB;  // rows per CTA pass
constexpr int kMaxDim = 8;          // dim and out_dim: layer 3 and the residual end in warp reductions
constexpr int kInP = 16;            // floats per stashed input row: x, t, zero padding
// Most CTAs a launch uses and the workspace is sized for: one per SM of an H100 SXM (the launch also stays within the
// device's own SMs).  Each CTA stages all weights and adds one partial-gradient vector to the fold, but on an H100
// more CTAs were never slower, up to one per SM at every batch measured (DESIGN.md section 3.12).
constexpr int kMaxCtas = 132;

// parameters() order: W0 [w][dim + 1], b0, W1 [w][w], b1, W2, b2, W3 [out_dim][w], b3
struct ParamOffsets {
  int W0, b0, W1, b1, W2, b2, W3, b3, total;
};
__host__ __device__ inline ParamOffsets param_offsets(int dim, int w, int out_dim) {
  ParamOffsets p;
  p.W0 = 0;
  p.b0 = p.W0 + w * (dim + 1);
  p.W1 = p.b0 + w;
  p.b1 = p.W1 + w * w;
  p.W2 = p.b1 + w;
  p.b2 = p.W2 + w * w;
  p.W3 = p.b2 + w;
  p.b3 = p.W3 + out_dim * w;
  p.total = p.b3 + out_dim;
  return p;
}

// CTAs a batch can use: one per tile of rows, up to kMaxCtas (the launch also stays within the device's SMs)
inline int ctas_for(int64_t batch) {
  const int64_t tiles = (batch + kTile - 1) / kTile;
  return (int)(tiles < kMaxCtas ? tiles : kMaxCtas);
}

// one cooperative launch of kThreads-thread CTAs; p.loss_parts and p.grad_parts point into the workspace
template <typename Params>
int launch_folded(const char* what, const void* kern, size_t smem, Params& p, int grid, char* ws, cudaStream_t s) {
  CFM_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  CFM_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, smem));
  CFM_REQUIRE(per_sm >= 1, "%s: the kernel does not fit on this device", what);
  if (grid > per_sm * sm_count()) grid = per_sm * sm_count();  // a cooperative grid must be co-resident
  p.loss_parts = reinterpret_cast<double*>(ws);
  p.grad_parts = reinterpret_cast<float*>(ws + align_up((size_t)grid * sizeof(double), 256));
  void* args[] = {&p};
  CFM_CUDA_OK(cudaLaunchCooperativeKernel(kern, dim3(grid), dim3(kThreads), args, smem, s));
  note_launches(1);
  return CFM_OK;
}

}  // namespace cfm
