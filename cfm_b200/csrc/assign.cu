// Exact optimal assignment for uniform equal-size marginals.
//
// Replaces pot.emd(a, b, M) (torchcfm/optimal_transport.py:49, called at :87) and
// scipy.optimize.linear_sum_assignment (:179).  With a = b = 1/n the LP optimum is P_sigma / n,
// so the solver only has to return sigma.  The reference solves in float64 on the fp32 costs
// (POT casts M to float64); so does this kernel.
//
// Algorithm: shortest augmenting paths with dual variables (Jonker-Volgenant / Crouse form).
//   init   u_i = min_j c_ij, greedy matching on the argmin columns (keeps complementary slackness;
//          assign_fast_kernel adds a column reduction and a second claim, see there)
//   then for every still-free row: Dijkstra over columns on reduced costs c_ij - u_i - v_j,
//   dual update, augmentation.  The optimum is unique almost surely for continuous data, so the
//   result equals the reference's sigma bit for bit; ties are broken deterministically
//   (free column first, then lowest index).
//
// GPU mapping: the problem at the reference's sizes (n = 128..256, BASELINE config 1) is a
// 256 KB latency-bound graph search, not a bandwidth problem.  One CTA runs the whole solve; each
// Dijkstra step is one coalesced row read of M + one block-wide argmin (warp shuffles + one smem
// hop).  No host round trips: sigma stays on the device for the sampling kernel.
// cfm_assign_exact_f32 picks the code path from n alone:
//   n <= 4096          assign_fast_kernel<KCB>, nt = max(64, round32(n)) <= 1024 threads, KCB = 1, 2 or 4
//                      columns per thread (n = 2049..3072: column slot 3 is padding on every thread),
//                      per-column state in registers, and the first cache_rows rows of M staged in shared
//                      memory (every row up to n = 222, 4 rows at n = 4096)
//   4097 <= n <= 5534  assign_kernel with u and every per-column array (v, shortest, path, row4col, srlist,
//                      scanned flags) in shared memory: 37 n + 16 bytes <= 200 KB
//   n >= 5535          assign_kernel with all of them in the global workspace
#include <float.h>

#include "common.cuh"

namespace cfm {

constexpr int kAsgMaxThreads = 1024;

struct AsgParams {
  const float* M;
  int n;
  int64_t ldm;
  const float* cost_max;
  int normalize;
  int32_t* sigma;      // col4row (output)
  double* total_cost;
  int32_t* status;     // {flags, augmentations}
  // global-memory backing when the per-column arrays do not fit in shared memory
  double* g_u;         // n (always global)
  double* g_v;         // n
  double* g_short;     // n
  int32_t* g_path;     // n
  int32_t* g_row4col;  // n
  int32_t* g_srlist;   // n
  unsigned char* g_sc; // n
  int use_smem;
  int cache_rows;      // assign_fast_kernel: the first cache_rows rows of M are staged in shared memory
};

struct MinKey {
  double val;
  int free_col;  // 1 when the column is unassigned (preferred on ties)
  int j;
};
__device__ __forceinline__ bool key_less(const MinKey& a, const MinKey& b) {
  if (a.val != b.val) return a.val < b.val;
  if (a.free_col != b.free_col) return a.free_col > b.free_col;
  return a.j < b.j;
}
__device__ __forceinline__ MinKey key_shfl_xor(const MinKey& k, int o) {
  MinKey r;
  r.val = __shfl_xor_sync(0xffffffffu, k.val, o);
  r.free_col = __shfl_xor_sync(0xffffffffu, k.free_col, o);
  r.j = __shfl_xor_sync(0xffffffffu, k.j, o);
  return r;
}
__device__ __forceinline__ MinKey warp_argmin(MinKey k) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const MinKey t = key_shfl_xor(k, o);
    if (key_less(t, k)) k = t;
  }
  return k;
}

__global__ void __launch_bounds__(kAsgMaxThreads, 1) assign_kernel(const AsgParams p) {
  extern __shared__ __align__(16) unsigned char asg_smem[];
  const int n = p.n, tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
  const int nwarps = nt >> 5;

  double* v; double* shortest; int32_t* path; int32_t* row4col; int32_t* srlist; unsigned char* sc;
  if (p.use_smem) {
    unsigned char* q = asg_smem;
    v = reinterpret_cast<double*>(q); q += (size_t)n * 8;
    shortest = reinterpret_cast<double*>(q); q += (size_t)n * 8;
    path = reinterpret_cast<int32_t*>(q); q += (size_t)n * 4;
    row4col = reinterpret_cast<int32_t*>(q); q += (size_t)n * 4;
    srlist = reinterpret_cast<int32_t*>(q); q += (size_t)n * 4;
    sc = q;
  } else {
    v = p.g_v; shortest = p.g_short; path = p.g_path; row4col = p.g_row4col; srlist = p.g_srlist;
    sc = p.g_sc;
  }
  // row duals: shared memory too when everything fits (one L2 round trip less per Dijkstra step)
  double* u = p.use_smem ? reinterpret_cast<double*>(asg_smem + ((size_t)n * 29 + 7) / 8 * 8) : p.g_u;
  int32_t* col4row = p.sigma;

  __shared__ MinKey wkey[2][32];  // per-warp candidates, double-buffered by step parity
  __shared__ int s_naug, s_bad, s_steps;

  const float cmax = (p.normalize && p.cost_max) ? __ldg(p.cost_max) : 1.f;
  auto cost = [&](int i, int j) -> double {
    float m = __ldg(p.M + (int64_t)i * p.ldm + j);
    if (p.normalize) m = __fdiv_rn(m, cmax);
    return (double)m;
  };

  // ---- init: v = 0, nothing assigned ----
  for (int j = tid; j < n; j += nt) { v[j] = 0.0; row4col[j] = -1; col4row[j] = -1; }
  if (tid == 0) { s_naug = 0; s_bad = 0; s_steps = 0; }
  __syncthreads();
  // u_i = min_j c_ij ; claim argmin column for the lowest-index row that wants it
  for (int i = warp; i < n; i += nwarps) {
    MinKey k{DBL_MAX, 0, 0x7fffffff};
    for (int j = lane; j < n; j += 32) {
      const double c = cost(i, j);
      MinKey t{c, 0, j};
      if (key_less(t, k)) k = t;
    }
    k = warp_argmin(k);
    if (lane == 0) {
      u[i] = k.val;
      path[i] = k.j;  // scratch: preferred column of row i
    }
  }
  __syncthreads();
  if (tid == 0) {
    // sequential greedy (n steps, trivial): first come first served keeps it deterministic
    for (int i = 0; i < n; ++i) {
      const int j = path[i];
      if (j >= 0 && j < n && row4col[j] < 0 && isfinite(u[i])) { row4col[j] = i; col4row[i] = j; }
    }
  }
  __syncthreads();

  // ---- augment every free row ----
  // Every thread tracks (i, minval, sink) redundantly: after ONE block barrier per Dijkstra step each
  // thread folds the per-warp candidates itself, so no second exchange is needed.  Per-column state
  // (shortest, path, scanned flag) is owned by the thread that scans the column.
  int steps_total = 0;
  for (int cur = 0; cur < n; ++cur) {
    if (col4row[cur] >= 0) continue;  // uniform: col4row is only written before a barrier
    for (int j = tid; j < n; j += nt) { shortest[j] = DBL_MAX; sc[j] = 0; }
    int i = cur, sink = -1, nsr = 0, par = 0;
    double minval = 0.0;
    bool bad = false;
    while (sink < 0) {
      if (tid == 0) srlist[nsr] = i;
      ++nsr;
      const double ui = u[i];
      MinKey k{DBL_MAX, 0, 0x7fffffff};
      for (int j = tid; j < n; j += nt) {
        if (sc[j]) continue;
        const double r = minval + cost(i, j) - ui - v[j];
        double sj = shortest[j];
        if (r < sj) { sj = r; shortest[j] = r; path[j] = i; }
        MinKey t{sj, row4col[j] < 0 ? 1 : 0, j};
        if (key_less(t, k)) k = t;
      }
      k = warp_argmin(k);
      if (lane == 0) wkey[par][warp] = k;
      __syncthreads();
      // every warp folds the <= 32 per-warp candidates with its own shuffle tree (no second barrier)
      MinKey best = lane < nwarps ? wkey[par][lane] : MinKey{DBL_MAX, 0, 0x7fffffff};
      best = warp_argmin(best);
      par ^= 1;
      ++steps_total;
      if (!(best.val < DBL_MAX) || best.j >= n) { bad = true; break; }  // infeasible (inf / nan costs)
      minval = best.val;
      if ((best.j % nt) == tid) sc[best.j] = 1;  // the owner of that column marks it scanned
      const int r4c = row4col[best.j];
      if (r4c < 0) sink = best.j; else i = r4c;
    }
    if (bad) { if (tid == 0) s_bad = 1; break; }
    __syncthreads();  // all scans finished: shortest / sc / srlist are final
    // dual updates (Crouse eq. for u over scanned rows, v over scanned columns)
    for (int q = tid; q < nsr; q += nt) {
      const int ii = srlist[q];
      if (ii == cur) u[ii] += minval; else u[ii] += minval - shortest[col4row[ii]];
    }
    for (int j = tid; j < n; j += nt)
      if (sc[j]) v[j] -= minval - shortest[j];
    __syncthreads();
    if (tid == 0) {
      int j = sink;
      while (true) {  // walk the alternating path back to `cur`
        const int ii = path[j];
        row4col[j] = ii;
        const int jprev = col4row[ii];
        col4row[ii] = j;
        j = jprev;
        if (ii == cur) break;
      }
      s_naug++;
    }
    __syncthreads();
  }
  if (tid == 0) s_steps = steps_total;
  __syncthreads();

  // ---- outputs ----
  double part = 0.0;
  if (!s_bad)
    for (int i = tid; i < n; i += nt) part += cost(i, col4row[i]);
  part = warp_sum(part);
  __shared__ double wsum[32];
  if (lane == 0) wsum[warp] = part;
  __syncthreads();
  if (warp == 0) {
    double t = lane < nwarps ? wsum[lane] : 0.0;
    t = warp_sum(t);
    if (lane == 0) {
      *p.total_cost = t;
      // NaN costs do not stop the search (every comparison with them is false) but poison the objective
      p.status[0] = (s_bad ? CFM_FLAG_INFEASIBLE : 0) | ((t == t && fabs(t) < 1.0e300) ? 0 : CFM_FLAG_NONFINITE);
      p.status[1] = s_naug;
      p.status[2] = s_steps;
    }
  }
}


// float64 <-> unsigned 64-bit image with the same ordering (total order, -0 < +0, NaNs at the ends)
__device__ __forceinline__ unsigned long long dkey(double x) {
  const long long b = __double_as_longlong(x);
  return (unsigned long long)b ^ ((unsigned long long)(b >> 63) | 0x8000000000000000ull);
}
__device__ __forceinline__ double dkey_inv(unsigned long long k) {
  const unsigned long long b = (k & 0x8000000000000000ull) ? (k ^ 0x8000000000000000ull) : ~k;
  return __longlong_as_double((long long)b);
}
struct IKey {
  unsigned long long k;  // dkey(shortest): smaller is better
  unsigned sec;          // (assigned column ? 1 << 24 : 0) | column: free columns first, then lowest index
};
__device__ __forceinline__ IKey ikey_min(const IKey& a, const IKey& b) {
  const bool lt = (b.k < a.k) || (b.k == a.k && b.sec < a.sec);
  IKey r;
  r.k = lt ? b.k : a.k;
  r.sec = lt ? b.sec : a.sec;
  return r;
}

// ---- the general fast path (n <= 4096): whole CTA, thread t owns columns t, t + nt, ... (KCB of them) ------
// The same shortest augmenting paths and Dijkstra tie-breaking as assign_kernel, with a stronger greedy start (the
// row reduction, then a column reduction and a second claim per free column) and reduced costs evaluated as
// (minval - u_i) + (c_ij - v_j).  So the two kernels return the same sigma only where the optimum is unique (almost
// surely for continuous costs).  Reformulated so that every warp executes as few instructions per Dijkstra step as
// possible -- a lone warp retires one dependent
// instruction every few cycles, so the step time IS the per-warp instruction count.  Per-column state (dual v, shortest label, predecessor, scanned / free bits)
// lives in registers; labels are kept as integer-orderable images of the float64 values (dkey) so that the hot
// loop is branch-free integer selects -- lanes disagree on every predicate, and divergent float64 compares were
// the bulk of the old step time; r = (minval - u_i) + (c_ij - v_j) costs two float64 adds per column.
// per step one cost load + one relaxation per owned column, a three-REDUX warp argmin, ONE block barrier
// (per-warp candidates are double-buffered by step parity), a second three-REDUX fold that every warp does
// for itself, and one shared-memory lookup of the matched row.
template <int KCB>
__global__ void __launch_bounds__(1024, 1) assign_fast_kernel(const AsgParams p) {
  extern __shared__ __align__(16) unsigned char asg_smem[];
  const int n = p.n, tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
  double* u = reinterpret_cast<double*>(asg_smem);          // n
  double* sh_s = u + n;                                    // n
  int32_t* path_s = reinterpret_cast<int32_t*>(sh_s + n);  // n
  int32_t* c4r = path_s + n;                               // n   col4row
  int32_t* srlist = c4r + n;                               // n
  int32_t* r4c_s = srlist + n;                             // n   row4col
  // The cost row of the current search row is THE long-latency operation of a Dijkstra step (ncu: the first use
  // of the loaded cost is the top stall; M no longer fits the L1 next to everything else at n = 256).  The rows
  // that fit are staged in shared memory once; the search reads them with LDS latency.
  const float* mcache = reinterpret_cast<const float*>(r4c_s + n);
  const int ncache = p.cache_rows;
  {
    float* mc = const_cast<float*>(mcache);
    for (int idx = tid; idx < ncache * n; idx += nt) {
      const int r = idx / n, j = idx - r * n;
      mc[idx] = __ldg(p.M + (int64_t)r * p.ldm + j);
    }
  }
  __shared__ unsigned long long wk[2][32];
  __shared__ unsigned wsec[2][32];
  __shared__ double wsum[32];
  const float cmax = (p.normalize && p.cost_max) ? __ldg(p.cost_max) : 1.f;
  auto cost = [&](int i, int j) -> double {
    float m = __ldg(p.M + (int64_t)i * p.ldm + j);
    if (p.normalize) m = __fdiv_rn(m, cmax);
    return (double)m;
  };
  for (int j = tid; j < n; j += nt) { r4c_s[j] = -1; c4r[j] = -1; }
  __syncthreads();
  for (int i = warp; i < n; i += nwarps) {  // u_i = min_j c_ij, preferred column (same keys as assign_kernel)
    MinKey k{DBL_MAX, 0, 0x7fffffff};
    for (int j = lane; j < n; j += 32) {
      MinKey t{cost(i, j), 0, j};
      if (key_less(t, k)) k = t;
    }
    k = warp_argmin(k);
    if (lane == 0) { u[i] = k.val; path_s[i] = k.j; }
  }
  __syncthreads();
  // column reduction on top of the row reduction: v_j = min_i (c_ij - u_i) >= 0 keeps the duals feasible and makes
  // one more edge per column tight, so the greedy start matches more rows and the searches that remain are
  // shorter (simulated on the test shapes: 10 % fewer Dijkstra steps at n = 256, d = 2; 50-70 % fewer for d >= 8)
  double v[KCB];
  unsigned long long shk[KCB];
  int pth[KCB];
  unsigned padmask = 0, freemask = 0;
  {
    unsigned long long vk[KCB];
    int arow[KCB];
#pragma unroll
    for (int k = 0; k < KCB; ++k) { vk[k] = ~0ull; arow[k] = -1; if (tid + nt * k >= n) padmask |= 1u << k; }
    for (int i = 0; i < n; ++i) {
      const double ui = u[i];
      const float* mrow = p.M + (int64_t)i * p.ldm + tid;
#pragma unroll
      for (int k = 0; k < KCB; ++k) {
        if ((padmask >> k) & 1u) continue;
        float m = __ldg(mrow + nt * k);
        if (p.normalize) m = __fdiv_rn(m, cmax);
        const double r = (double)m - ui;
        const unsigned long long rk = (r == r) ? dkey(r) : ~0ull;
        const bool lt = rk < vk[k];
        vk[k] = lt ? rk : vk[k];
        arow[k] = lt ? i : arow[k];
      }
    }
#pragma unroll
    for (int k = 0; k < KCB; ++k) {
      const int j = tid + nt * k;
      const double vj = (vk[k] != ~0ull) ? dkey_inv(vk[k]) : 0.0;
      v[k] = isfinite(vj) ? vj : 0.0;  // a column of +inf costs: leave its dual at 0, the search reports infeasible
      pth[k] = -1;
      if (j < n) srlist[j] = isfinite(vj) ? arow[k] : -1;  // scratch: the row that makes column j tight
    }
  }
  __syncthreads();
  if (tid == 0) {
    // sequential greedy start (2n trivial steps, deterministic): every row claims its row-minimum column, then
    // every column still free claims the row of its column minimum if that row is still free
    for (int i = 0; i < n; ++i) {
      const int j = path_s[i];
      if (j >= 0 && j < n && r4c_s[j] < 0 && isfinite(u[i])) { r4c_s[j] = i; c4r[i] = j; }
    }
    for (int j = 0; j < n; ++j) {
      const int i = srlist[j];
      if (i >= 0 && r4c_s[j] < 0 && c4r[i] < 0) { r4c_s[j] = i; c4r[i] = j; }
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < KCB; ++k) {
    const int j = tid + nt * k;
    if (j < n && r4c_s[j] < 0) freemask |= 1u << k;
  }
  const unsigned long long kmax = dkey(DBL_MAX);
  int naug = 0, steps_total = 0, par = 0;
  bool bad = false;
  for (int cur = 0; cur < n && !bad; ++cur) {
    if (c4r[cur] >= 0) continue;  // uniform: c4r changes only between barriers
    unsigned scmask = padmask;
#pragma unroll
    for (int k = 0; k < KCB; ++k) shk[k] = kmax;
    int i = cur, sink = -1, nsr = 0;
    double minval = 0.0;
    while (sink < 0) {
      if (tid == 0) srlist[nsr] = i;
      ++nsr;
      const double base = minval - u[i];
      float c[KCB];
      if (i < ncache) {
        const float* mrow = mcache + (size_t)i * n + tid;
#pragma unroll
        for (int k = 0; k < KCB; ++k) c[k] = (padmask >> k) & 1u ? 0.f : mrow[nt * k];
      } else {
        const float* mrow = p.M + (int64_t)i * p.ldm + tid;
#pragma unroll
        for (int k = 0; k < KCB; ++k) c[k] = (padmask >> k) & 1u ? 0.f : __ldg(mrow + nt * k);
      }
      IKey best{~0ull, 0xffffffffu};
#pragma unroll
      for (int k = 0; k < KCB; ++k) {
        const bool open = !((scmask >> k) & 1u);
        float m = c[k];
        if (p.normalize) m = __fdiv_rn(m, cmax);
        const double r = base + ((double)m - v[k]);
        const unsigned long long rk = (r == r) ? dkey(r) : ~0ull;
        const bool upd = open && (rk < shk[k]);
        shk[k] = upd ? rk : shk[k];
        pth[k] = upd ? i : pth[k];
        IKey t;
        t.k = open ? shk[k] : ~0ull;
        t.sec = ((freemask >> k) & 1u ? 0u : (1u << 24)) | (unsigned)(tid + nt * k);
        best = KCB == 1 ? t : ikey_min(best, t);
      }
      {
        const unsigned hi = (unsigned)(best.k >> 32), lo = (unsigned)best.k;
        const unsigned mh = __reduce_min_sync(0xffffffffu, hi);
        const unsigned ml = __reduce_min_sync(0xffffffffu, hi == mh ? lo : 0xffffffffu);
        const unsigned ms = __reduce_min_sync(0xffffffffu, (hi == mh && lo == ml) ? best.sec : 0xffffffffu);
        if (lane == 0) { wk[par][warp] = ((unsigned long long)mh << 32) | ml; wsec[par][warp] = ms; }
      }
      __syncthreads();
      {
        const unsigned long long ck = lane < nwarps ? wk[par][lane] : ~0ull;
        const unsigned cs = lane < nwarps ? wsec[par][lane] : 0xffffffffu;
        const unsigned hi = (unsigned)(ck >> 32), lo = (unsigned)ck;
        const unsigned mh = __reduce_min_sync(0xffffffffu, hi);
        const unsigned ml = __reduce_min_sync(0xffffffffu, hi == mh ? lo : 0xffffffffu);
        const unsigned ms = __reduce_min_sync(0xffffffffu, (hi == mh && lo == ml) ? cs : 0xffffffffu);
        best.k = ((unsigned long long)mh << 32) | ml;
        best.sec = ms;
      }
      par ^= 1;
      ++steps_total;
      const int bj = (int)(best.sec & 0xffffffu);
      if (best.k >= kmax || bj >= n) { bad = true; break; }
      minval = dkey_inv(best.k);
      if (KCB == 1) { if (tid == bj) scmask |= 1u; }
      else if (tid == bj % nt) scmask |= 1u << (bj / nt);
      if (best.sec >> 24) i = r4c_s[bj]; else sink = bj;
    }
    if (bad) break;
#pragma unroll
    for (int k = 0; k < KCB; ++k) {
      const int j = tid + nt * k;
      if (j < n) { sh_s[j] = dkey_inv(shk[k]); path_s[j] = pth[k]; }
    }
    __syncthreads();
    for (int q = tid; q < nsr; q += nt) {
      const int ii = srlist[q];
      if (ii == cur) u[ii] += minval; else u[ii] += minval - sh_s[c4r[ii]];
    }
#pragma unroll
    for (int k = 0; k < KCB; ++k)
      if (((scmask & ~padmask) >> k) & 1u) v[k] -= minval - dkey_inv(shk[k]);
    if (tid == sink % nt) freemask &= ~(1u << (sink / nt));
    __syncthreads();
    if (tid == 0) {
      int j = sink;
      while (true) {
        const int ii = path_s[j];
        r4c_s[j] = ii;
        const int jprev = c4r[ii];
        c4r[ii] = j;
        j = jprev;
        if (ii == cur) break;
      }
    }
    ++naug;
    __syncthreads();
  }
  __syncthreads();
  double part = 0.0;
  if (!bad)
    for (int i = tid; i < n; i += nt) part += cost(i, c4r[i]);
  part = warp_sum(part);
  if (lane == 0) wsum[warp] = part;
  for (int i = tid; i < n; i += nt) p.sigma[i] = c4r[i];
  __syncthreads();
  if (warp == 0) {
    double t = lane < nwarps ? wsum[lane] : 0.0;
    t = warp_sum(t);
    if (lane == 0) {
      *p.total_cost = t;
      p.status[0] = (bad ? CFM_FLAG_INFEASIBLE : 0) | ((t == t && fabs(t) < 1.0e300) ? 0 : CFM_FLAG_NONFINITE);
      p.status[1] = naug;
      p.status[2] = steps_total;
    }
  }
}

static size_t asg_fast_smem_bytes(int n) { return (size_t)n * (8 + 8 + 4 * 4) + 16; }

static size_t asg_smem_bytes(int n) { return ((size_t)n * 29 + 7) / 8 * 8 + (size_t)n * 8 + 16; }

}  // namespace cfm

using namespace cfm;

extern "C" size_t cfm_assign_workspace_bytes(int n) {
  // u (always) + global backing for everything else
  return align_up((size_t)n * 8, 256) * 3 + align_up((size_t)n * 4, 256) * 3 + align_up((size_t)n, 256);
}

extern "C" int cfm_assign_exact_f32(const float* M, int n, int64_t ldm, const float* cost_max,
                                    int normalize, int32_t* sigma, double* total_cost,
                                    int32_t* status, void* workspace, size_t workspace_bytes,
                                    void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  CFM_REQUIRE(M && sigma && total_cost && status && workspace, "cfm_assign_exact_f32: null pointer");
  CFM_REQUIRE(n > 0 && ldm >= n, "cfm_assign_exact_f32: bad shape n=%d ldm=%lld", n, (long long)ldm);
  CFM_REQUIRE(!(normalize && !cost_max), "cfm_assign_exact_f32: normalize needs cost_max");
  CFM_REQUIRE(workspace_bytes >= cfm_assign_workspace_bytes(n), "cfm_assign_exact_f32: workspace too small");
  AsgParams p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.n = n; p.ldm = ldm; p.cost_max = cost_max; p.normalize = normalize;
  p.sigma = sigma; p.total_cost = total_cost; p.status = status;
  char* w = reinterpret_cast<char*>(workspace);
  const size_t a8 = align_up((size_t)n * 8, 256), a4 = align_up((size_t)n * 4, 256);
  p.g_u = reinterpret_cast<double*>(w); w += a8;
  p.g_v = reinterpret_cast<double*>(w); w += a8;
  p.g_short = reinterpret_cast<double*>(w); w += a8;
  p.g_path = reinterpret_cast<int32_t*>(w); w += a4;
  p.g_row4col = reinterpret_cast<int32_t*>(w); w += a4;
  p.g_srlist = reinterpret_cast<int32_t*>(w); w += a4;
  p.g_sc = reinterpret_cast<unsigned char*>(w);
  if (n <= 4096) {
    size_t sb = asg_fast_smem_bytes(n);
    {
      const size_t room = (size_t)200 * 1024 > sb ? (size_t)200 * 1024 - sb : 0;
      size_t rows = room / ((size_t)n * 4);
      if (rows > (size_t)n) rows = n;
      p.cache_rows = (int)rows;
      sb += rows * (size_t)n * 4;
    }
    int nt = ((n + 31) / 32) * 32;
    if (nt < 64) nt = 64;
    if (nt > 1024) nt = 1024;
    const int kcb = (n + nt - 1) / nt;
    if (kcb == 1) {
      CFM_CUDA_OK(cudaFuncSetAttribute(assign_fast_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sb));
      assign_fast_kernel<1><<<1, nt, sb, s>>>(p);
    } else if (kcb == 2) {
      CFM_CUDA_OK(cudaFuncSetAttribute(assign_fast_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sb));
      assign_fast_kernel<2><<<1, nt, sb, s>>>(p);
    } else {
      CFM_CUDA_OK(cudaFuncSetAttribute(assign_fast_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sb));
      assign_fast_kernel<4><<<1, nt, sb, s>>>(p);
    }
    ::cfm::note_launches(1);
    CFM_CUDA_OK(cudaGetLastError());
    return CFM_OK;
  }
  const size_t smem = asg_smem_bytes(n);
  p.use_smem = smem <= 200 * 1024;
  const size_t dyn = p.use_smem ? smem : 0;
  CFM_CUDA_OK(cudaFuncSetAttribute(assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
  int threads = ((n + 31) / 32) * 32;
  if (threads < 64) threads = 64;
  if (threads > kAsgMaxThreads) threads = kAsgMaxThreads;
  assign_kernel<<<1, threads, dyn, s>>>(p); ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
