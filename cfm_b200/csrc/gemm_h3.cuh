// Hopper tensor-core GEMM, fp16x3 scheme:  D[m, n] = sum_k A[m, k] * B[n, k]  at fp32-grade accuracy on the
// fp16 wgmma path (twice the tf32 rate, half the operand bytes).
//
// Every fp32 operand x is carried as two fp16 arrays,  hi = fp16(x)  and  lo = fp16((x - hi) * 2^11)
// (round to nearest: |x - hi| <= 2^-11 |x|, so the scaled residual has hi's magnitude and never goes
// subnormal before x itself is ~1e-8; x = hi + lo * 2^-11 to 2^-22 relative).  Products of fp16 numbers
// are exact in fp32, so
//     acc0 += A_hi . B_hi                     (register accumulator 0)
//     acc1 += A_hi . B_lo + A_lo . B_hi       (register accumulator 1, carries the common factor 2^11)
//     D     = acc0 + acc1 * 2^-11             (epilogue)
// drops only the lo.lo term (2^-22 relative): the NumPy emulation of the representation
// (tests/test_host.py::test_fp16x3_operand_split_emulation) gives 1.5e-8 of sum|a||b| at d = 784,
// 3xTF32 with truncating splits 7e-8.  Range: fp16 tops out at 65504, so producers scale rows by a power of
// two where the data is unbounded (cost matrix: per-row scales, exact) and saturate otherwise.
//
// Runs on the persistent GEMM core of gemm_tc.cuh (TMA producer warpgroup, two consumer warpgroups issuing
// wgmma m64n128k16, 3-stage ring), with a K-chunk of 64 fp16 (= the 128-byte swizzle atom), 4 k-steps of K = 16
// per chunk and 3 MMAs per k-step into the two accumulators (2 x 64 registers per thread: the 128 x 128 tile is
// the largest whose two fp32 accumulators fit the register file).
#pragma once
#include <cuda_fp16.h>

#include "gemm_tc.cuh"

namespace cfm {

constexpr int kHK = 64;                    // K-chunk in fp16 elements
constexpr int kHABytes = kTM * kHK * 2;    // 16 KB: one A (hi or lo) tile
constexpr float kH3Scale = 2048.f;         // 2^11: scale of the lo parts
constexpr float kH3InvScale = 1.f / 2048.f;

struct H3Scheme {
  static constexpr int kElem = 2, kKChunk = kHK, kKStep = 16, kNAcc = 2;
  __device__ static __forceinline__ void mma(float (&d0)[64], float (&d1)[64], uint64_t ah, uint64_t al, uint64_t bh,
                                             uint64_t bl, uint32_t first) {
    wg_mma_f16_n128(d1, ah, bl, first);
    wg_mma_f16_n128(d1, al, bh, 1u);
    wg_mma_f16_n128(d0, ah, bh, first);
  }
  __device__ static __forceinline__ float combine(float a0, float a1) { return fmaf(a1, kH3InvScale, a0); }
};

// fp32 -> (hi, lo) of the fp16x3 scheme; v must already carry the producer's range scale
__device__ __forceinline__ void split_h3(float v, __half& hi, __half& lo) {
  hi = __float2half_rn(v);
  lo = __float2half_rn((v - __half2float(hi)) * kH3Scale);
}
// saturating variant for unscaled producers (activations): |v| > 65504 clamps instead of becoming inf
// (cvt.rn.satfinite: one instruction per conversion)
__device__ __forceinline__ __half f2h_satfinite(float v) {
  unsigned short r;
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(r) : "f"(v));
  return __ushort_as_half(r);
}
__device__ __forceinline__ void split_h3_sat(float v, __half& hi, __half& lo) {
  hi = f2h_satfinite(v);
  lo = f2h_satfinite((v - __half2float(hi)) * kH3Scale);
}

// two values at once: packed (hi0 | hi1 << 16) and (lo0 | lo1 << 16) via cvt.rn.satfinite.f16x2.f32
__device__ __forceinline__ void split_h3_sat_x2(float v0, float v1, uint32_t& hi2, uint32_t& lo2) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi2) : "f"(v1), "f"(v0));  // first source -> upper half
  const __half2 h = *reinterpret_cast<const __half2*>(&hi2);
  const float r0 = (v0 - __low2float(h)) * kH3Scale, r1 = (v1 - __high2float(h)) * kH3Scale;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo2) : "f"(r1), "f"(r0));
}

// ---- host side -------------------------------------------------------------------------------------
// (rows, d) fp16 row-major (row stride ld halves, ld % 8 == 0) -> box of (box_rows x 64 halves), 128B swizzle,
// zero fill outside [0, d) x [0, rows).  Descriptors are cached by (base, shape): see sqdist_h3.cu.
int tc_make_map_f16(CUtensorMap* m, const __half* base, int rows, int d, int64_t ld, int box_rows);

// Epilogue functor interface: see gemm_tc.cuh (acc = acc0 + acc1 * 2^-11)
template <class Epi>
inline int launch_gemm_h3(const __half* ah, const __half* al, int n0, int64_t lda, const __half* bh,
                          const __half* bl, int n1, int64_t ldb, int d, Epi epi, cudaStream_t s) {
  CUtensorMap mah, mal, mbh, mbl;
  int rc;
  if ((rc = tc_make_map_f16(&mah, ah, n0, d, lda, kTM)) != CFM_OK) return rc;
  if ((rc = tc_make_map_f16(&mal, al, n0, d, lda, kTM)) != CFM_OK) return rc;
  if ((rc = tc_make_map_f16(&mbh, bh, n1, d, ldb, kTN)) != CFM_OK) return rc;
  if ((rc = tc_make_map_f16(&mbl, bl, n1, d, ldb, kTN)) != CFM_OK) return rc;
  return launch_gemm_wg<H3Scheme>(mah, mal, mbh, mbl, n0, n1, d, epi, s);
}

}  // namespace cfm
