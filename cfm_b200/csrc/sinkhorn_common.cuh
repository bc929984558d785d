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
  // workspace (sinkhorn.cu sk_layout); the control region at its start holds the timeline marks, the error ring and
  // the seeded solver's per-CTA minima
  unsigned long long* tl;  // 32 %globaltimer marks (CFM_SK_TL; debug aid)
  double* err_ring;        // 4 marginal-error sums, slot it % 4 for iteration it
  float* dmin_u;           // kSkMaxGrid per-CTA minima of (u_new - u_old) (seeded solver)
  float* dmin_v;           // kSkMaxGrid per-CTA minima of (v_new - v_old) (seeded solver)
  void* u_work;     // n0  pot_t
  void* v_work[2];  // n1p pot_t each
  void* part_m;     // grid * n1p pot_t
  void* part_s;     // grid * n1p sum_t
  int n1p;          // n1 rounded up to a multiple of 4
  int vec;          // float4 path usable
  int v_in_smem;
  float l2_resident_frac;  // sinkhorn_v2: share of each slab loaded with L2 evict_last (0: default policy)
  unsigned char* mq;  // sinkhorn_v2: 3-byte fixed-point copy of M (n0 rows of ldc bytes; null: fp32 sweeps only)
  int64_t ldc;        //              its row pitch in bytes, align16(3 * n1)
  int ldn;            //              bytes of a row whose chunk takes 22-bit entries (0: every chunk keeps 3 bytes)
  int* n_narrow;      //              control region: chunks of the copy the last solve wrote at 22 bits
  int fp32_by_v2;   // auto mode: sinkhorn_v2_kernel solves the fp32 case, the generic kernel only the float64 one
  int timeline;     // CFM_SK_TL: globaltimer marks of one iteration (debug aid)
  int screen;       // mixed mode: fp32 screening of negligible terms (0 only for precise = 4, the unscreened reference)
  int mixed;        // precise mode only: float64 potentials and exponent ARGUMENTS, fp32 exponentials (see expd)
};
constexpr int kSkMaxGrid = 512;  // CTAs the per-CTA minima have room for

// Beyond |M/reg| = 64 the fp32 log2-domain exponent loses the answer and the solve needs float64 potentials.  The
// auto mode of both solver kernels and the pair draw (sample.cu) decide by this one rule.
__device__ __forceinline__ bool sk_needs_f64(float cmax, int normalize, float reg) {
  return !((normalize ? 1.f : cmax) / reg <= 64.f);
}

// rows [begin, end) of CTA b: n0 / nblk each, the first n0 % nblk CTAs one more
struct SkSlab { int begin, end; };
__device__ __forceinline__ SkSlab sk_slab(int n0, int nblk, int b) {
  const int base = n0 / nblk, rem = n0 % nblk;
  const int begin = b * base + min(b, rem);
  return {begin, begin + base + (b < rem ? 1 : 0)};
}

// ---- the iteration loop shared by the solvers ----
// Iteration it sweeps rows (new u) and, unless it is the last and no check, column partials (the next v).  A check
// iteration sums the column-marginal error of (u, v_cur) into slot it % 4 of the error ring.
struct SkStep { bool last, check, do_col; };
__device__ __forceinline__ SkStep sk_step(const SkParams& p, int it) {
  const bool last = it == p.max_iters - 1, check = it % p.check_every == 0;
  return {last, check, !last || check};
}
struct SkLoop {
  double err = 1.0, prev_check_err = -1.0;
  bool converged = false;
  int iters = 0;
};
// prologue: clear the error ring and the count of 22-bit chunks (every solver, so a solve that writes no copy leaves
// 0 there; sinkhorn_v2's CTAs add their counts after the grid barrier that follows this)
__device__ __forceinline__ void sk_ring_init(const SkParams& p) {
  if (blockIdx.x == 0 && threadIdx.x < 4) p.err_ring[threadIdx.x] = 0.0;
  if (blockIdx.x == 0 && threadIdx.x == 0 && p.n_narrow != nullptr) *p.n_narrow = 0;
}
// the error slot of iteration it (between the grid barriers around the combine).  It clears slot it + 2 for later:
// that slot's last reader, the check of iteration it - 2, is two grid barriers back.
__device__ __forceinline__ double* sk_err_slot(const SkParams& p, int it) {
  if (blockIdx.x == 0 && threadIdx.x == 0) p.err_ring[(it + 2) & 3] = 0.0;
  return p.err_ring + (it & 3);
}
// add this thread's share of the squared marginal error to *slot (every thread of the CTA calls; two block barriers)
__device__ __forceinline__ void sk_err_add(double err_local, double* slot, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  err_local = warp_sum(err_local);
  if (lane == 0) red[warp] = err_local;
  __syncthreads();
  if (warp == 0) {
    double t = lane < kSkWarps ? red[lane] : 0.0;
    t = warp_sum(t);
    if (lane == 0) atomicAdd(slot, t);
  }
  __syncthreads();
}
// the check after the grid barrier that completed iteration it's error sum: true when the solve stops.  POT's rule
// err < stop_thr, or (stall_tol > 0) a check that improved err by less than that fraction once the RMS relative
// column error is below 1e-5
__device__ __forceinline__ bool sk_check_stops(SkLoop& L, const SkParams& p, int it) {
  L.err = sqrt(__ldcg(p.err_ring + (it & 3)));
  if (L.err < p.stop_thr) { L.converged = true; return true; }
  if (p.stall_tol > 0.0 && L.prev_check_err >= 0.0 && L.err > (1.0 - p.stall_tol) * L.prev_check_err &&
      L.err * sqrt((double)p.n1) < 1e-5) { L.converged = true; return true; }
  L.prev_check_err = L.err;
  return false;
}
// outputs: log_v in natural-log units (to_ln: the working units' scale) and the status word
// {flags, iterations, arithmetic (0 fp32, 1 float64, 2 float64 arguments + fp32 exponentials), kernel variant}
template <class T>
__device__ __forceinline__ void sk_finish(const SkParams& p, const SkLoop& L, const T* v, double to_ln, int arith,
                                          int variant) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < p.n1; j += gridDim.x * blockDim.x)
    p.log_v[j] = (double)__ldcg(v + j) * to_ln;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    int flags = 0;
    if (!L.converged) flags |= CFM_FLAG_NOT_CONVERGED;
    if (!(L.err == L.err)) flags |= CFM_FLAG_NONFINITE;
    p.status[0] = flags;
    p.status[1] = L.iters;
    p.status[2] = arith;
    p.status[3] = variant;
    *p.err_out = L.err;
  }
}

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
