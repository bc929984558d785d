// SIMT fp32 "NT" GEMM core:  acc[m,n] = sum_k A[m,k] * B[n,k]  (both row-major),
// true fp32 FMA accumulation (the numerics of cuBLAS sgemm with TF32 off, which is
// what torch.cdist / nn.Linear use in the reference).  128x128x16 tiles, 256 threads,
// 8x8 register micro-tiles, register-prefetch double buffering.  The epilogue functor
// sees one float4 of a row at a time:  epi(m, n, acc4, valid_cols).
//
// Used by: sqdist.cu (cost matrix, small/unaligned shapes and as the cross-check for
// the tensor-core paths) and mlp.cu (layer GEMMs with bias+activation epilogue).
#pragma once
#include "common.cuh"

namespace cfm {

constexpr int kGemmBM = 128, kGemmBN = 128, kGemmBK = 16, kGemmThreads = 256;

// Loads 4 consecutive k-elements of row `r` (or zeros outside the matrix).
__device__ __forceinline__ float4 gemm_load4(const float* __restrict__ P, int64_t ld, int rows,
                                             int K, int r, int k, bool vec_ok) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (r < rows) {
    const float* p = P + (int64_t)r * ld + k;
    if (vec_ok && k + 3 < K) {
      v = *reinterpret_cast<const float4*>(p);
    } else {
      if (k + 0 < K) v.x = p[0];
      if (k + 1 < K) v.y = p[1];
      if (k + 2 < K) v.z = p[2];
      if (k + 3 < K) v.w = p[3];
    }
  }
  return v;
}

template <class Epi>
__global__ void __launch_bounds__(kGemmThreads, 2)
gemm_nt_simt_kernel(const float* __restrict__ A, int64_t lda, const float* __restrict__ B,
                    int64_t ldb, int M, int N, int K, int m_base, Epi epi) {
  __shared__ __align__(16) float As[2][kGemmBK][kGemmBM];
  __shared__ __align__(16) float Bs[2][kGemmBK][kGemmBN];

  const int tid = threadIdx.x;
  const int m0 = m_base + blockIdx.y * kGemmBM;
  const int n0 = blockIdx.x * kGemmBN;
  const bool a_vec = ((lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
  const bool b_vec = ((ldb & 3) == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0);

  // loader mapping: 128 rows x 16 k = 512 float4; thread -> rows {lr, lr+64}, k-quad lk
  const int lr = tid >> 2;
  const int lk = (tid & 3) * 4;
  // compute mapping
  const int ty = tid >> 4;  // 0..15 -> rows ty*4 and 64+ty*4
  const int tx = tid & 15;  // 0..15 -> cols tx*4 and 64+tx*4

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 pa0, pa1, pb0, pb1;
  auto gload = [&](int k0) {
    pa0 = gemm_load4(A, lda, M, K, m0 + lr, k0 + lk, a_vec);
    pa1 = gemm_load4(A, lda, M, K, m0 + lr + 64, k0 + lk, a_vec);
    pb0 = gemm_load4(B, ldb, N, K, n0 + lr, k0 + lk, b_vec);
    pb1 = gemm_load4(B, ldb, N, K, n0 + lr + 64, k0 + lk, b_vec);
  };
  auto sstore = [&](int buf) {
    As[buf][lk + 0][lr] = pa0.x; As[buf][lk + 1][lr] = pa0.y;
    As[buf][lk + 2][lr] = pa0.z; As[buf][lk + 3][lr] = pa0.w;
    As[buf][lk + 0][lr + 64] = pa1.x; As[buf][lk + 1][lr + 64] = pa1.y;
    As[buf][lk + 2][lr + 64] = pa1.z; As[buf][lk + 3][lr + 64] = pa1.w;
    Bs[buf][lk + 0][lr] = pb0.x; Bs[buf][lk + 1][lr] = pb0.y;
    Bs[buf][lk + 2][lr] = pb0.z; Bs[buf][lk + 3][lr] = pb0.w;
    Bs[buf][lk + 0][lr + 64] = pb1.x; Bs[buf][lk + 1][lr + 64] = pb1.y;
    Bs[buf][lk + 2][lr + 64] = pb1.z; Bs[buf][lk + 3][lr + 64] = pb1.w;
  };

  const int nk = (K + kGemmBK - 1) / kGemmBK;
  gload(0);
  sstore(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) gload((kt + 1) * kGemmBK);
#pragma unroll
    for (int k = 0; k < kGemmBK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      sstore(buf ^ 1);
      __syncthreads();
    }
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= M) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = n0 + h * 64 + tx * 4;
      if (n >= N) continue;
      const float4 v = make_float4(acc[i][h * 4 + 0], acc[i][h * 4 + 1], acc[i][h * 4 + 2],
                                   acc[i][h * 4 + 3]);
      epi(m, n, v, min(4, N - n));
    }
  }
  epi.finish();
}

template <class Epi>
inline cudaError_t launch_gemm_nt_simt(const float* A, int64_t lda, const float* B, int64_t ldb,
                                       int M, int N, int K, Epi epi, cudaStream_t s) {
  // gridDim.y holds at most 65535 tile rows: a larger M takes one launch per 65535 tile rows, each starting at row
  // m_base, so every tile is computed exactly as in a single launch
  const int mtiles = (int)(((int64_t)M + kGemmBM - 1) / kGemmBM);
  const unsigned ntiles = (unsigned)(((int64_t)N + kGemmBN - 1) / kGemmBN);
  for (int mt = 0; mt < mtiles; mt += 65535) {
    const dim3 grid(ntiles, mtiles - mt < 65535 ? mtiles - mt : 65535);
    gemm_nt_simt_kernel<Epi><<<grid, kGemmThreads, 0, s>>>(A, lda, B, ldb, M, N, K, mt * kGemmBM, epi);
    ::cfm::note_launches(1);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace cfm
