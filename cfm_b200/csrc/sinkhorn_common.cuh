// Shared pieces of the two Sinkhorn kernels (sinkhorn.cu: generic fused sweep through L2;
// sinkhorn_v2.cu: smem-staged sweep fed by bulk async copies).
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace cfm {

constexpr int kSkThreads = 512;
constexpr int kSkWarps = kSkThreads / 32;
constexpr int kSkChunk = kSkWarps;  // rows per chunk: one warp per row in the row phase
constexpr int kSkMaxKG = 4;         // column groups (float4) per thread per panel
constexpr int kPanelCols = kSkThreads * 4 * kSkMaxKG;  // 8192

struct SkParams {
  const float* M;
  int n0, n1;
  int64_t ldm;
  float reg;
  const float* cost_max;
  int normalize;
  int max_iters;
  double stop_thr;
  int check_every;
  int precise;      // 0 fast, 1 precise, -1 auto
  double stall_tol; // <=0: off.  else stop when a check improves err by less than this fraction
  double* log_u;
  double* log_v;
  int32_t* status;
  double* err_out;
  // workspace
  void* u_work;     // n0  pot_t
  void* v_work[2];  // n1p pot_t each
  void* part_m;     // grid * n1p pot_t
  void* part_s;     // grid * n1p sum_t
  double* err_ring; // 4
  int n1p;          // n1 rounded up to a multiple of 4
  int vec;          // float4 path usable
  int v_in_smem;
  float l2_resident_frac;  // sinkhorn_v2: share of each slab loaded with L2 evict_last (0: default policy)
  unsigned char* mq;  // sinkhorn_v2: 3-byte fixed-point copy of M (n0 rows of ldc bytes; null: fp32 sweeps only)
  int64_t ldc;        //              its row pitch in bytes, align16(3 * n1)
  int run_if;       // 0 always; 1 only when auto-mode resolves to fast; 2 only when it resolves to precise
  int timeline;     // seeded solver: globaltimer marks of one iteration (CFM_SK_TL; debug aid)
  int screen;       // mixed mode: fp32 screening of negligible terms (0 only for precise = 4, the unscreened reference)
  int mixed;        // precise mode only: float64 potentials and exponent ARGUMENTS, fp32 exponentials (see expd)
};

template <bool P> struct Tr;
template <> struct Tr<false> {
  using pot_t = float;  // potentials / running maxima
  using sum_t = float;  // sums of exponentials
  __device__ static __forceinline__ float init() { return -1.0e30f; }
};
template <> struct Tr<true> {
  using pot_t = double;
  using sum_t = double;  // float64 exp + sums: POT's stopThr=1e-9 needs marginals resolved to ~1e-12
  __device__ static __forceinline__ double init() { return -1.0e300; }
};

// exponent of one plan entry given the cost entry and the opposite-side potential
template <bool P> struct Xf;
template <> struct Xf<false> {  // log2 units: x = M * (-log2e/(reg*scale)) + p2
  float c2;
  __device__ __forceinline__ float operator()(float m, float p) const { return fmaf(m, c2, p); }
};
template <> struct Xf<true> {  // natural-log units, NumPy's fp32 rounding of -M/reg, f64 add
  float reg, cmax;
  int norm;
  __device__ __forceinline__ double operator()(float m, double p) const {
    const float mn = norm ? __fdiv_rn(m, cmax) : m;
    return (double)(-__fdiv_rn(mn, reg)) + p;
  }
};
__device__ __forceinline__ float expdiff(float x, float m) { return ex2f(x - m); }
__device__ __forceinline__ double expdiff(double x, double m) { return exp(x - m); }
// exp(x - m) for the log-sum-exp recurrences.  MIX (float64 mode only): the difference is formed in float64 --
// that is where |M/reg| ~ 1e4 needs the bits -- and only then rounded to fp32 and exponentiated with ex2:
// relative error ~1e-7 per term instead of 1e-16, at a fifth of the float64-pipe instructions (a float64 exp is
// ~30 of them).
template <bool MIX> __device__ __forceinline__ float expd(float x, float m) { return ex2f(x - m); }
template <bool MIX> __device__ __forceinline__ double expd(double x, double m) {
  if (MIX) return (double)ex2f((float)(x - m) * kLog2e);
  return exp(x - m);
}
__device__ __forceinline__ float lse_fin(float m, float s) { return m + log2f(s); }
__device__ __forceinline__ double lse_fin(double m, double s) { return m + log(s); }
__device__ __forceinline__ float vmax(float a, float b) { return fmaxf(a, b); }
__device__ __forceinline__ double vmax(double a, double b) { return fmax(a, b); }

// load 4 consecutive cost entries of a row starting at column j (pad +inf => zero weight)
template <bool VEC>
__device__ __forceinline__ float4 load_cost4(const float* __restrict__ row, int j, int n1) {
  if (VEC) return ldg_stream4(row + j);
  float4 r;
  const float inf = __int_as_float(0x7f800000);
  r.x = (j + 0 < n1) ? __ldg(row + j + 0) : inf;
  r.y = (j + 1 < n1) ? __ldg(row + j + 1) : inf;
  r.z = (j + 2 < n1) ? __ldg(row + j + 2) : inf;
  r.w = (j + 3 < n1) ? __ldg(row + j + 3) : inf;
  return r;
}

template <class T> struct Vec4 { T x, y, z, w; };

// potentials are rewritten during the kernel by other CTAs: read them either from the smem
// stage (SM) or through ld.global.cg (L2, coherent), never through L1 / the .nc path.
template <bool SM, class T>
__device__ __forceinline__ Vec4<T> load_pot4(const T* p, int j) {  // p padded to n1p
  Vec4<T> r;
  if (SM) { r.x = p[j]; r.y = p[j + 1]; r.z = p[j + 2]; r.w = p[j + 3]; }
  else { r.x = __ldcg(p + j); r.y = __ldcg(p + j + 1); r.z = __ldcg(p + j + 2); r.w = __ldcg(p + j + 3); }
  return r;
}

}  // namespace cfm
