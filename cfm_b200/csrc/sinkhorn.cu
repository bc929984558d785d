// Persistent log-domain Sinkhorn on uniform marginals.
//
// Replaces pot.sinkhorn(a, b, M, reg) as called at torchcfm/optimal_transport.py:87 (bound at
// :51) with POT's sinkhorn_log algorithm (ot/bregman/_sinkhorn.py): per iteration
//     v = logb - LSE_i(Mr_ij + u_i)      (column pass)
//     u = loga - LSE_j(Mr_ij + v_j)      (row pass),        Mr = -M/reg
// with the column-marginal L2 error tested every `check_every` iterations.
//
// Design (one cooperative launch for the whole solve, grid = resident CTAs):
//   * CTA b owns a contiguous slab of rows.  One *fused sweep* per iteration: for each chunk of
//     16 rows the CTA first computes the row LSEs (u update, one warp per row, streaming M from
//     HBM), then immediately re-reads the same 16 rows -- now L2 hits -- to add them, with the
//     fresh u, to per-thread running (max, sum) accumulators of the columns it owns.  M therefore
//     crosses HBM ONCE per iteration, not twice (algorithmic bytes 2*N^2*4 per iteration; DRAM
//     traffic ~ half of that).
//   * per-CTA column partials (max, sum) go to a [cta][n1] workspace; after a grid barrier each
//     CTA combines a slice of columns (8 lanes per column), writes the new v and the marginal
//     error, and a second barrier publishes them.
//   * the opposite potential v is staged in shared memory once per sweep (the row phase reads
//     it 16x per chunk); potentials written during the kernel are only ever read through
//     ld.global.cg or smem, never through the non-coherent path.
//   * two arithmetic modes chosen on the device: fast (fp32 log2-domain, one FFMA + one ex2 per
//     element) and precise (float64 potentials, IEEE fp32 division forming -M/reg exactly as
//     NumPy does, for |M/reg| >> 64 where fp32 exponents lose the answer; SURVEY.md 11(ii)).
//   * precise mode with fp32 exponentials ("mixed", the default of the precise regime) runs in
//     sinkhorn_run_seeded: every term is screened in fp32 against a threshold derived from the
//     previous iteration's log-sum-exp, only the plan's support takes the float64 path (BASELINE
//     config 4; see the comment above sinkhorn_run_seeded).
#include <stdlib.h>

#include "sinkhorn_common.cuh"

namespace cfm {

// ---- row phase: one warp computes LSE_j(x(M_rj, v_j)) for one row ---------------------------
template <bool P, bool VEC, bool SM, bool MIX>
__device__ __forceinline__ typename Tr<P>::pot_t row_lse(const float* __restrict__ row,
                                                         const typename Tr<P>::pot_t* vsrc,
                                                         int n1, int ng,
                                                         const Xf<P>& xf, int lane) {
  using pot_t = typename Tr<P>::pot_t;
  using sum_t = typename Tr<P>::sum_t;
  pot_t m = Tr<P>::init();
  sum_t s = 0;
  constexpr int U = P ? 4 : 8;
  for (int g0 = 0; g0 < ng; g0 += 32 * U) {
    float4 c[U];
    Vec4<pot_t> pv[U];
#pragma unroll
    for (int q = 0; q < U; ++q) {
      const int g = g0 + q * 32 + lane;
      if (g < ng) {
        c[q] = load_cost4<VEC>(row, g * 4, n1);
        pv[q] = load_pot4<SM, pot_t>(vsrc, g * 4);
      } else {
        const float inf = __int_as_float(0x7f800000);
        c[q] = make_float4(inf, inf, inf, inf);
        pv[q].x = pv[q].y = pv[q].z = pv[q].w = (pot_t)0;
      }
    }
    pot_t x[U][4];
    pot_t bm = m;
#pragma unroll
    for (int q = 0; q < U; ++q) {
      x[q][0] = xf(c[q].x, pv[q].x); x[q][1] = xf(c[q].y, pv[q].y);
      x[q][2] = xf(c[q].z, pv[q].z); x[q][3] = xf(c[q].w, pv[q].w);
      bm = vmax(bm, vmax(vmax(x[q][0], x[q][1]), vmax(x[q][2], x[q][3])));
    }
    sum_t acc = s * expd<MIX>(m, bm);
#pragma unroll
    for (int q = 0; q < U; ++q)
      acc += (expd<MIX>(x[q][0], bm) + expd<MIX>(x[q][1], bm)) +
             (expd<MIX>(x[q][2], bm) + expd<MIX>(x[q][3], bm));
    s = acc;
    m = bm;
  }
  // warp combine of (m, s)
  pot_t wm = warp_max(m);
  sum_t ws = warp_sum(s * expd<MIX>(m, wm));
  return lse_fin(wm, ws);
}


// ---- float64-potential mode with fp32 exponentials ("mixed"), screened -------------------------------------
// Where this mode is needed (|M/reg| ~ 1e4, SB-CFM with small sigma) the plan is extremely sparse: all but a few
// percent of the terms of a log-sum-exp lie more than 30 units below its maximum (e^-30 ~ 1e-13 each) and only cost
// XU-pipe conversions (ncu on BASELINE config 4: XU 56 %, 42 instructions per element visit: two IEEE divisions, three
// fp32<->fp64 conversions and one ex2 per element).  Every element is therefore first SCREENED in fp32 -- one FFMA
// t = M * (-1/(reg scale)) + fp32(potential), good to ~1e-3 absolute, against thr = running maximum - 32 -- and only
// the survivors (collected in a per-lane bit mask, then processed one per lane per trip so that a warp does not
// walk the full element loop for one hit) take the exact path, which is unchanged: NumPy's fp32 quotient, float64
// add, float64 difference to the running maximum, fp32 ex2.  Terms dropped are < e^-30 of a maximum that is itself
// <= the final one: < n * 1e-13 relative.  NaN costs fail `t <= thr` and are therefore never dropped.
constexpr float kScreenGap = 34.f;  // fp32 screening error ~1e-3 at |M/reg| ~ 1e4: dropped terms are < e^-33 of the maximum

__device__ __forceinline__ void lse_take(double x, double& m, double& s) {
  if (x > m) {
    s = s * expd<true>(m, x) + 1.0;
    m = x;
  } else {  // (also taken by NaN)
    s += expd<true>(x, m);
  }
}

template <bool VEC>
__device__ __forceinline__ double row_lse_screened(const float* __restrict__ row, const double* v_s,
                                                   const float* vh_s, int n1, int ng, const Xf<true>& xf, float nr,
                                                   int lane) {
  constexpr int U = 4;
  // pass 1: fp32 maximum of the row's exponents (fmaxf drops NaN operands; a NaN cost is caught in pass 2)
  float tmax = -3.0e38f;
  for (int g0 = 0; g0 < ng; g0 += 32 * U) {
#pragma unroll
    for (int q = 0; q < U; ++q) {
      const int g = g0 + q * 32 + lane;
      if (g < ng) {
        const float4 c = load_cost4<VEC>(row, g * 4, n1);
        const float4 vh = *reinterpret_cast<const float4*>(vh_s + g * 4);
        tmax = fmaxf(fmaxf(tmax, fmaxf(fmaf(c.x, nr, vh.x), fmaf(c.y, nr, vh.y))),
                     fmaxf(fmaf(c.z, nr, vh.z), fmaf(c.w, nr, vh.w)));
      }
    }
  }
  const float thr = warp_max(tmax) - kScreenGap;
  // pass 2: the terms within kScreenGap of it (typically one to three per row) take the exact path
  double m = Tr<true>::init(), s = 0.0;
  for (int g0 = 0; g0 < ng; g0 += 32 * U) {
    unsigned mask = 0;
#pragma unroll
    for (int q = 0; q < U; ++q) {
      const int g = g0 + q * 32 + lane;
      if (g < ng) {
        const float4 c = load_cost4<VEC>(row, g * 4, n1);
        const float4 vh = *reinterpret_cast<const float4*>(vh_s + g * 4);
        mask |= (!(fmaf(c.x, nr, vh.x) <= thr) ? 1u : 0u) << (4 * q);
        mask |= (!(fmaf(c.y, nr, vh.y) <= thr) ? 1u : 0u) << (4 * q + 1);
        mask |= (!(fmaf(c.z, nr, vh.z) <= thr) ? 1u : 0u) << (4 * q + 2);
        mask |= (!(fmaf(c.w, nr, vh.w) <= thr) ? 1u : 0u) << (4 * q + 3);
      }
    }
    while (__any_sync(0xffffffffu, mask != 0u)) {
      if (mask != 0u) {
        const int e = __ffs((int)mask) - 1;
        mask &= mask - 1u;
        const int col = (g0 + (e >> 2) * 32 + lane) * 4 + (e & 3);
        if (col < n1) lse_take(xf(__ldg(row + col), v_s[col]), m, s);
      }
    }
  }
  const double wm = warp_max(m);
  const double ws = warp_sum(s * expd<true>(m, wm));
  return lse_fin(wm, ws);
}


// ---- the solver body ---------------------------------------------------------------------------
template <bool P, bool VEC, int KG, bool MIX>
__device__ void sinkhorn_run(const SkParams& p, unsigned char* smem_raw) {
  using pot_t = typename Tr<P>::pot_t;
  using sum_t = typename Tr<P>::sum_t;
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nblk = gridDim.x, b = blockIdx.x;
  const int n0 = p.n0, n1 = p.n1, n1p = p.n1p, ng = n1p / 4;

  __shared__ pot_t u_chunk[kSkChunk];
  __shared__ float uh_chunk[kSkChunk];              // screened mode: fp32 copies of u_chunk
  __shared__ double red[kSkWarps];
  pot_t* v_s = reinterpret_cast<pot_t*>(smem_raw);  // n1p entries when p.v_in_smem
  float* vh_s = reinterpret_cast<float*>(smem_raw + (size_t)p.n1p * sizeof(pot_t));  // screened mode: fp32 copies
  constexpr bool kScreen = P && MIX;
  const bool screen = kScreen && p.v_in_smem && p.screen;
  if (tid < kSkChunk) { u_chunk[tid] = (pot_t)0; uh_chunk[tid] = 0.f; }  // padding rows must never see NaN bits
  __syncthreads();

  pot_t* u_work = reinterpret_cast<pot_t*>(p.u_work);
  pot_t* v_work[2] = {reinterpret_cast<pot_t*>(p.v_work[0]), reinterpret_cast<pot_t*>(p.v_work[1])};
  pot_t* part_m = reinterpret_cast<pot_t*>(p.part_m);
  sum_t* part_s = reinterpret_cast<sum_t*>(p.part_s);

  // element transform and the log-marginals in this mode's units
  Xf<P> xf;
  pot_t loga, logb;
  const float cmax = p.cost_max ? __ldg(p.cost_max) : 1.f;
  if constexpr (P) {
    xf.reg = p.reg; xf.cmax = cmax; xf.norm = p.normalize;
    loga = -log((double)n0); logb = -log((double)n1);
  } else {
    const float scale = p.normalize ? cmax : 1.f;
    xf.c2 = -kLog2e / (p.reg * scale);
    loga = -log2f((float)n0); logb = -log2f((float)n1);
  }
  const double to_ln = P ? 1.0 : kLn2d;  // working units -> natural log
  const float nr = -1.f / (p.reg * (p.normalize ? cmax : 1.f));  // screening only: t ~ -M/(reg scale) + potential

  // slab of rows owned by this CTA (first `rem` CTAs get one extra row)
  const int base = n0 / nblk, rem = n0 % nblk;
  const int r_begin = b * base + min(b, rem);
  const int r_end = r_begin + base + (b < rem ? 1 : 0);
  const int npanel = (n1p + kPanelCols - 1) / kPanelCols;

  // one sweep: (optional) row phase -> u ; (optional) column partials with that u
  auto sweep = [&](bool do_row, bool do_col, const pot_t* v_cur) {
    if (do_row && p.v_in_smem) {
      for (int j = tid; j < n1p; j += kSkThreads) {
        const pot_t vj = (j < n1) ? __ldcg(v_cur + j) : (pot_t)0;
        v_s[j] = vj;
        if (screen) vh_s[j] = (float)vj;
      }
      __syncthreads();
    }
    const pot_t* vsrc = p.v_in_smem ? v_s : v_cur;
    for (int panel = 0; panel < npanel; ++panel) {
      pot_t cm[KG][4];
      sum_t cs[KG][4];
      float cthr[kScreen ? KG : 1][4];  // screened mode: fp32 threshold = running column maximum - kScreenGap
#pragma unroll
      for (int k = 0; k < KG; ++k)
#pragma unroll
        for (int c = 0; c < 4; ++c) { cm[k][c] = Tr<P>::init(); cs[k][c] = 0; if (kScreen) cthr[k][c] = -3.0e38f; }
      const int gpan = panel * (kPanelCols / 4);

      for (int r0 = r_begin; r0 < r_end; r0 += kSkChunk) {
        const int R = min(kSkChunk, r_end - r0);
        // -- row phase (first panel only; later panels re-use u from global) --
        if (panel == 0) {
          if (warp < R) {
            pot_t uval = (pot_t)0;
            if (do_row) {
              const float* row = p.M + (int64_t)(r0 + warp) * p.ldm;
              pot_t lse;
              if constexpr (kScreen) {
                if (screen) lse = row_lse_screened<VEC>(row, v_s, vh_s, n1, ng, xf, nr, lane);
                else if (p.v_in_smem) lse = row_lse<P, VEC, true, MIX>(row, vsrc, n1, ng, xf, lane);
                else lse = row_lse<P, VEC, false, MIX>(row, vsrc, n1, ng, xf, lane);
              } else if (p.v_in_smem) lse = row_lse<P, VEC, true, MIX>(row, vsrc, n1, ng, xf, lane);
              else lse = row_lse<P, VEC, false, MIX>(row, vsrc, n1, ng, xf, lane);
              uval = loga - lse;
              if (lane == 0) {
                u_work[r0 + warp] = uval;
                p.log_u[r0 + warp] = (double)uval * to_ln;
              }
            }
            if (lane == 0) { u_chunk[warp] = uval; uh_chunk[warp] = (float)uval; }
          }
        } else if (warp < R && lane == 0) {
          const pot_t uval = do_row ? u_work[r0 + warp] : (pot_t)0;
          u_chunk[warp] = uval; uh_chunk[warp] = (float)uval;
        }
        if (!do_col) continue;
        __syncthreads();
        // -- column phase: thread owns float4 groups g = gpan + tid + 512*k --
        if constexpr (kScreen) {
          if (screen) {
            // screened: every thread of the CTA takes part in the warp votes (no early `continue`)
#pragma unroll
            for (int k = 0; k < KG; ++k) {
              const int g = gpan + tid + kSkThreads * k;
              const bool gv = g < ng;
              for (int rb = 0; rb < R; rb += 8) {
                float4 c[8];
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                  if (gv && rb + q < R) {
                    c[q] = load_cost4<VEC>(p.M + (int64_t)(r0 + rb + q) * p.ldm, g * 4, n1);
                  } else {
                    const float inf = __int_as_float(0x7f800000);
                    c[q] = make_float4(inf, inf, inf, inf);
                  }
                }
                float uh[8];
#pragma unroll
                for (int q = 0; q < 8; ++q) uh[q] = uh_chunk[(rb + q) & (kSkChunk - 1)];
#pragma unroll
                for (int cc = 0; cc < 4; ++cc) {
                  // pass 1: fp32 maximum of the block's eight terms; threshold relative to max(running, block)
                  float t[8];
                  float bm = -3.0e38f;
#pragma unroll
                  for (int q = 0; q < 8; ++q) {
                    const float cv = cc == 0 ? c[q].x : cc == 1 ? c[q].y : cc == 2 ? c[q].z : c[q].w;
                    t[q] = fmaf(cv, nr, uh[q]);
                    bm = fmaxf(bm, t[q]);
                  }
                  cthr[k][cc] = fmaxf(cthr[k][cc], bm - kScreenGap);
                  unsigned mask = 0;
#pragma unroll
                  for (int q = 0; q < 8; ++q) mask |= (!(t[q] <= cthr[k][cc]) ? 1u : 0u) << q;
                  // pass 2: survivors (typically none or one) take the exact path, one per lane per trip
                  while (__any_sync(0xffffffffu, mask != 0u)) {
                    if (mask != 0u) {
                      const int e = __ffs((int)mask) - 1;
                      mask &= mask - 1u;
                      // the cost entry of row e out of registers (three levels of selects, no reload)
                      const float4 c01 = (e & 1) ? ((e & 2) ? c[3] : c[1]) : ((e & 2) ? c[2] : c[0]);
                      const float4 c45 = (e & 1) ? ((e & 2) ? c[7] : c[5]) : ((e & 2) ? c[6] : c[4]);
                      const float4 ce = (e & 4) ? c45 : c01;
                      const float cv = cc == 0 ? ce.x : cc == 1 ? ce.y : cc == 2 ? ce.z : ce.w;
                      lse_take(xf(cv, u_chunk[(rb + e) & (kSkChunk - 1)]), cm[k][cc], cs[k][cc]);
                    }
                  }
                }
              }
            }
            __syncthreads();  // u_chunk is rewritten by the next chunk's row phase
            continue;
          }
        }
#pragma unroll
        for (int k = 0; k < KG; ++k) {
          const int g = gpan + tid + kSkThreads * k;
          if (g >= ng) continue;
          for (int rb = 0; rb < R; rb += 8) {
            float4 c[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) {
              if (rb + q < R) {
                c[q] = load_cost4<VEC>(p.M + (int64_t)(r0 + rb + q) * p.ldm, g * 4, n1);
              } else {
                const float inf = __int_as_float(0x7f800000);
                c[q] = make_float4(inf, inf, inf, inf);
              }
            }
#pragma unroll
            for (int cc = 0; cc < 4; ++cc) {
              pot_t x[8];
              pot_t bm = cm[k][cc];
#pragma unroll
              for (int q = 0; q < 8; ++q) {
                const float cv = cc == 0 ? c[q].x : cc == 1 ? c[q].y : cc == 2 ? c[q].z : c[q].w;
                x[q] = xf(cv, u_chunk[(rb + q) & (kSkChunk - 1)]);
                bm = vmax(bm, x[q]);
              }
              sum_t acc = cs[k][cc] * expd<MIX>(cm[k][cc], bm);
#pragma unroll
              for (int q = 0; q < 8; ++q) acc += expd<MIX>(x[q], bm);
              cs[k][cc] = acc;
              cm[k][cc] = bm;
            }
          }
        }
        __syncthreads();  // u_chunk is rewritten by the next chunk's row phase
      }
      if (do_col) {
#pragma unroll
        for (int k = 0; k < KG; ++k) {
          const int g = gpan + tid + kSkThreads * k;
          if (g >= ng) continue;
          pot_t* pm = part_m + (int64_t)b * n1p + g * 4;
          sum_t* ps = part_s + (int64_t)b * n1p + g * 4;
#pragma unroll
          for (int c = 0; c < 4; ++c) { pm[c] = cm[k][c]; ps[c] = cs[k][c]; }
        }
      }
    }
  };

  // combine the per-CTA column partials of a slice of columns -> v_new, marginal error
  auto combine = [&](const pot_t* v_cur, pot_t* v_new, bool have_cur, double* err_slot) {
    const int cpc = (n1 + nblk - 1) / nblk;
    const int c_begin = b * cpc, c_end = min(n1, c_begin + cpc);
    double err_local = 0.0;
    const int sub = tid & 7;
    for (int j0 = c_begin; j0 < c_end; j0 += (kSkThreads >> 3)) {
      // every thread takes the same trip count (shuffles below); idle columns contribute nothing
      const int j = j0 + (tid >> 3);
      const bool act = j < c_end;
      pot_t m = Tr<P>::init();
      sum_t s = 0;
      if (act) {
        for (int c0 = sub; c0 < nblk; c0 += 8 * 4) {
          pot_t mm[4];
          sum_t ss[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int c = c0 + q * 8;
            if (c < nblk) {
              mm[q] = __ldcg(part_m + (int64_t)c * n1p + j);
              ss[q] = __ldcg(part_s + (int64_t)c * n1p + j);
            } else { mm[q] = Tr<P>::init(); ss[q] = 0; }
          }
          pot_t bm = vmax(vmax(mm[0], mm[1]), vmax(mm[2], mm[3]));
          bm = vmax(bm, m);
          sum_t acc = s * expd<MIX>(m, bm);
#pragma unroll
          for (int q = 0; q < 4; ++q) acc += ss[q] * expd<MIX>(mm[q], bm);
          s = acc; m = bm;
        }
      }
      // reduce over the 8 lanes of this column
      pot_t gm = m;
#pragma unroll
      for (int o = 4; o > 0; o >>= 1) gm = vmax(gm, __shfl_xor_sync(0xffffffffu, gm, o));
      sum_t gs = s * expd<MIX>(m, gm);
#pragma unroll
      for (int o = 4; o > 0; o >>= 1) gs += __shfl_xor_sync(0xffffffffu, gs, o);
      if (act && sub == 0) {
        const pot_t lse = lse_fin(gm, gs);
        const pot_t vn = logb - lse;
        v_new[j] = vn;
        if (have_cur) {
          // column marginal of (u, v_cur): exp(v_cur + lse); POT: err = ||colsum - b||_2
          const double d = ((double)__ldcg(v_cur + j) - (double)vn) * to_ln;
          const double e = expm1(d) / (double)n1;
          err_local += e * e;
        }
      }
    }
    if (err_slot != nullptr) {
      err_local = warp_sum(err_local);
      if (lane == 0) red[warp] = err_local;
      __syncthreads();
      if (warp == 0) {
        double t = lane < kSkWarps ? red[lane] : 0.0;
        t = warp_sum(t);
        if (lane == 0) atomicAdd(err_slot, t);
      }
      __syncthreads();
    }
  };

  // ---- prologue: v^0 = logb - LSE_i(Mr_ij + 0) ----
  if (b == 0 && tid < 4) p.err_ring[tid] = 0.0;
  sweep(false, true, nullptr);
  grid.sync();
  combine(nullptr, v_work[0], false, nullptr);
  grid.sync();

  int cur = 0, iters = 0;
  bool converged = false;
  double err = 1.0, prev_check_err = -1.0;
  for (int it = 0; it < p.max_iters; ++it) {
    const bool last = (it == p.max_iters - 1);
    const bool check = (it % p.check_every) == 0;
    const bool do_col = !last || check;
    sweep(true, do_col, v_work[cur]);
    iters = it + 1;
    if (!do_col) break;
    grid.sync();
    if (b == 0 && tid == 0) p.err_ring[(it + 2) & 3] = 0.0;
    combine(v_work[cur], v_work[cur ^ 1], true, &p.err_ring[it & 3]);
    grid.sync();
    if (check) {
      err = sqrt(__ldcg(&p.err_ring[it & 3]));
      if (err < p.stop_thr) { converged = true; break; }
      if (p.stall_tol > 0.0 && prev_check_err >= 0.0 &&
          err > (1.0 - p.stall_tol) * prev_check_err &&
          err * sqrt((double)n1) < 1e-5) { converged = true; break; }
      prev_check_err = err;
    }
    if (last) break;
    cur ^= 1;
  }

  // ---- outputs ----
  for (int j = b * kSkThreads + tid; j < n1; j += nblk * kSkThreads)
    p.log_v[j] = (double)__ldcg(v_work[cur] + j) * to_ln;
  if (b == 0 && tid == 0) {
    int flags = 0;
    if (!converged) flags |= CFM_FLAG_NOT_CONVERGED;
    if (!(err == err)) flags |= CFM_FLAG_NONFINITE;
    p.status[0] = flags;
    p.status[1] = iters;
    p.status[2] = P ? (MIX ? 2 : 1) : 0;  // 0 fp32, 1 float64, 2 float64 arguments + fp32 exponentials
    p.status[3] = 0;
    *p.err_out = err;
  }
}


// ---- float64-potential mode, seeded screening (BASELINE config 4 regime) -------------------------------------
// The potentials of consecutive Sinkhorn iterations do not DROP by more than a few units (config 4: min du, min dv > -5
// from the first iteration on; scripts/sim/sinkhorn_screening.py), and every log-sum-exp of this iteration is bounded below by the one the previous
// iteration computed for the same row / column:
//     LSE_i(Mr_i. + v_new) >= LSE_i(Mr_i. + v_old) + min_j (v_new_j - v_old_j),      (rows; columns alike with u)
// because every term grows by at least that minimum.  So the threshold below which a term is negligible is known
// BEFORE the pass: thr = previous LSE + (global minimum change of the other potential) - 34, one fp32 number per row /
// column.  The pass is then one FFMA and one compare per element; the ~0.05 % of the elements above the threshold
// (the plan's support: a couple per row / column over the WHOLE matrix) take the exact float64 path.  Nothing is
// assumed: if the potentials moved a lot the thresholds merely drop and more terms take the exact path.
// Per iteration: row pass over the CTA's slab -> grid barrier (global min of du) -> column pass -> barrier ->
// combine (v_new, min of dv, marginal error) -> barrier.
// candidates of the float4 groups [g_begin, g_end) of one row -> warp-reduced (maximum, sum relative to it)
template <bool VEC, int U, bool L1>
__device__ __forceinline__ void row_range_seeded(const float* __restrict__ row, const double* v_s, const float* vh_s,
                                                 int n1, int g_begin, int g_end, const Xf<true>& xf, float nr, float thr,
                                                 int lane, double& wm, double& ws) {
  double m = Tr<true>::init(), s = 0.0;
  for (int g0 = g_begin; g0 < g_end; g0 += 32 * U) {
    unsigned gm = 0;  // bit q: float4 group q of this lane holds a candidate
    float4 c[U];
#pragma unroll
    for (int q = 0; q < U; ++q) {  // all loads of the block first: U independent 128-bit loads in flight per lane
      const int g = g0 + q * 32 + lane;
      if (g < g_end) c[q] = (VEC && L1) ? __ldg(reinterpret_cast<const float4*>(row + g * 4)) : load_cost4<VEC>(row, g * 4, n1);
    }
#pragma unroll
    for (int q = 0; q < U; ++q) {
      const int g = g0 + q * 32 + lane;
      if (g < g_end) {
        const float4 vh = *reinterpret_cast<const float4*>(vh_s + g * 4);
        // (NaN fails `<=`: a NaN cost or potential is a candidate, never dropped)
        const bool le = (fmaf(c[q].x, nr, vh.x) <= thr) & (fmaf(c[q].y, nr, vh.y) <= thr) &
                        (fmaf(c[q].z, nr, vh.z) <= thr) & (fmaf(c[q].w, nr, vh.w) <= thr);
        gm |= (le ? 0u : 1u) << q;
      }
    }
    while (__any_sync(0xffffffffu, gm != 0u)) {
      if (gm != 0u) {
        const int q = __ffs((int)gm) - 1;
        gm &= gm - 1u;
        const int col0 = (g0 + q * 32 + lane) * 4;
        const float4 cq = (VEC && L1) ? __ldg(reinterpret_cast<const float4*>(row + col0)) : load_cost4<VEC>(row, col0, n1);
        const float ce[4] = {cq.x, cq.y, cq.z, cq.w};
#pragma unroll
        for (int e = 0; e < 4; ++e)  // only the elements of the group that are candidates themselves
          if (col0 + e < n1 && !(fmaf(ce[e], nr, vh_s[col0 + e]) <= thr)) lse_take(xf(ce[e], v_s[col0 + e]), m, s);
      }
    }
  }
  wm = warp_max(m);
  ws = warp_sum(s * expd<true>(m, wm));
}

template <bool VEC>
__device__ __forceinline__ double row_lse_seeded(const float* __restrict__ row, const double* v_s,
                                                 const float* vh_s, int n1, int ng, const Xf<true>& xf, float nr,
                                                 float thr, int lane, bool& empty) {
  double wm, ws;
  row_range_seeded<VEC, 4, false>(row, v_s, vh_s, n1, 0, ng, xf, nr, thr, lane, wm, ws);
  empty = !(ws > 0.0);  // (cannot happen with a valid bound; the caller then repeats the row unseeded)
  return lse_fin(wm, ws);
}

__device__ __forceinline__ float block_min_f(float v, float* red32, int tid) {
  v = -warp_max(-v);
  if ((tid & 31) == 0) red32[tid >> 5] = v;
  __syncthreads();
  float r = red32[0];
#pragma unroll
  for (int w = 1; w < kSkWarps; ++w) r = fminf(r, red32[w]);
  __syncthreads();
  return r;
}

template <bool VEC, int KG>
__device__ void sinkhorn_run_seeded(const SkParams& p, unsigned char* smem_raw) {
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nblk = gridDim.x, b = blockIdx.x;
  const int n0 = p.n0, n1 = p.n1, n1p = p.n1p, ng = n1p / 4;

  __shared__ double u_chunk[kSkChunk];
  __shared__ float uh_chunk[kSkChunk];
  __shared__ double red[kSkWarps];
  __shared__ float redf[kSkWarps];
  double* v_s = reinterpret_cast<double*>(smem_raw);
  float* vh_s = reinterpret_cast<float*>(smem_raw + (size_t)n1p * sizeof(double));
  if (tid < kSkChunk) { u_chunk[tid] = 0.0; uh_chunk[tid] = 0.f; }
  __syncthreads();

  double* u_work = reinterpret_cast<double*>(p.u_work);
  double* v_work[2] = {reinterpret_cast<double*>(p.v_work[0]), reinterpret_cast<double*>(p.v_work[1])};
  double* part_m = reinterpret_cast<double*>(p.part_m);
  double* part_s = reinterpret_cast<double*>(p.part_s);
  float* dmin_u = reinterpret_cast<float*>(p.err_ring + 8);  // [nblk] per-CTA min of (u_new - u_old)
  float* dmin_v = dmin_u + 512;                                // [nblk] per-CTA min of (v_new - v_old)

  Xf<true> xf;
  const float cmax = p.cost_max ? __ldg(p.cost_max) : 1.f;
  xf.reg = p.reg; xf.cmax = cmax; xf.norm = p.normalize;
  const double loga = -log((double)n0), logb = -log((double)n1);
  const float nr = -1.f / (p.reg * (p.normalize ? cmax : 1.f));
  const float kBig = 3.0e38f;

  const int base = n0 / nblk, rem = n0 % nblk;
  const int r_begin = b * base + min(b, rem);
  const int r_end = r_begin + base + (b < rem ? 1 : 0);

  auto stage_v = [&](const double* v_cur) {
    for (int j = tid; j < n1p; j += kSkThreads) {
      const double vj = (j < n1) ? __ldcg(v_cur + j) : 0.0;
      v_s[j] = vj;
      vh_s[j] = (float)vj;
    }
    __syncthreads();
  };
  auto global_min = [&](const float* slots) -> float {  // min over the per-CTA slots (after a grid barrier)
    float v = kBig;
    for (int c = tid; c < nblk; c += kSkThreads) v = fminf(v, __ldcg(slots + c));
    return block_min_f(v, redf, tid);
  };

  // rows of the slab: u_new = loga - LSE_j(Mr_ij + v_j); seeded with the previous pass's LSE when there is one
  auto row_phase = [&](bool seeded, float dv_min) {
    float dmin = kBig;
    for (int r0 = r_begin + warp; r0 < r_end; r0 += kSkWarps) {
      const float* row = p.M + (int64_t)r0 * p.ldm;
      const double u_old = seeded ? u_work[r0] : 0.0;
      double lse;
      bool empty = true;
      if (seeded) {
        const float thr = __double2float_rd(loga - u_old + (double)dv_min) - kScreenGap;
        lse = row_lse_seeded<VEC>(row, v_s, vh_s, n1, ng, xf, nr, thr, lane, empty);
      }
      if (empty) lse = row_lse_screened<VEC>(row, v_s, vh_s, n1, ng, xf, nr, lane);  // (warp-uniform)
      const double uval = loga - lse;
      if (lane == 0) {
        u_work[r0] = uval;
        p.log_u[r0] = uval;
        dmin = fminf(dmin, __double2float_rd(uval - u_old));
      }
    }
    dmin = block_min_f(lane == 0 ? dmin : kBig, redf, tid);
    if (tid == 0) dmin_u[b] = dmin;
  };

  // column partials over the slab with the u of u_work (use_u) or u = 0; seeded: thr_j = LSE_prev_j + du_min - gap
  auto col_phase = [&](bool use_u, bool seeded, float du_min) {
    double cm[KG][4], cs[KG][4];
    float cthr[KG][4];
#pragma unroll
    for (int k = 0; k < KG; ++k)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        cm[k][c] = Tr<true>::init(); cs[k][c] = 0.0;
        const int col = (tid + kSkThreads * k) * 4 + c;
        cthr[k][c] = seeded ? (col < n1 ? __double2float_rd(logb - v_s[col] + (double)du_min) - kScreenGap : kBig) : -kBig;
      }
    for (int r0 = r_begin; r0 < r_end; r0 += kSkChunk) {
      const int R = min(kSkChunk, r_end - r0);
      if (tid < kSkChunk) {
        const double uv = (use_u && tid < R) ? u_work[r0 + tid] : 0.0;
        u_chunk[tid] = uv; uh_chunk[tid] = (float)uv;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < KG; ++k) {
        const int g = tid + kSkThreads * k;
        const bool gv = g < ng;
        for (int rb = 0; rb < R; rb += 8) {
          float4 c[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            if (gv && rb + q < R) {
              c[q] = load_cost4<VEC>(p.M + (int64_t)(r0 + rb + q) * p.ldm, g * 4, n1);
            } else {
              const float inf = __int_as_float(0x7f800000);
              c[q] = make_float4(inf, inf, inf, inf);
            }
          }
          float uh[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) uh[q] = uh_chunk[rb + q];
          if (!seeded) {  // no previous LSE (the very first column pass): thresholds from the block maxima
#pragma unroll
            for (int q = 0; q < 8; ++q) {
              cthr[k][0] = fmaxf(cthr[k][0], fmaf(c[q].x, nr, uh[q]) - kScreenGap);
              cthr[k][1] = fmaxf(cthr[k][1], fmaf(c[q].y, nr, uh[q]) - kScreenGap);
              cthr[k][2] = fmaxf(cthr[k][2], fmaf(c[q].z, nr, uh[q]) - kScreenGap);
              cthr[k][3] = fmaxf(cthr[k][3], fmaf(c[q].w, nr, uh[q]) - kScreenGap);
            }
          }
          unsigned hm = 0;  // bit q: row q of the block holds a candidate in one of the four columns
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const bool le = (fmaf(c[q].x, nr, uh[q]) <= cthr[k][0]) & (fmaf(c[q].y, nr, uh[q]) <= cthr[k][1]) &
                            (fmaf(c[q].z, nr, uh[q]) <= cthr[k][2]) & (fmaf(c[q].w, nr, uh[q]) <= cthr[k][3]);
            hm |= (le ? 0u : 1u) << q;
          }
          while (__any_sync(0xffffffffu, hm != 0u)) {
            if (hm != 0u) {
              const int e = __ffs((int)hm) - 1;
              hm &= hm - 1u;
              const float4 c01 = (e & 1) ? ((e & 2) ? c[3] : c[1]) : ((e & 2) ? c[2] : c[0]);
              const float4 c45 = (e & 1) ? ((e & 2) ? c[7] : c[5]) : ((e & 2) ? c[6] : c[4]);
              const float4 ce = (e & 4) ? c45 : c01;
              const float ue = uh_chunk[rb + e];
              const double ud = u_chunk[rb + e];
              if (!(fmaf(ce.x, nr, ue) <= cthr[k][0])) lse_take(xf(ce.x, ud), cm[k][0], cs[k][0]);
              if (!(fmaf(ce.y, nr, ue) <= cthr[k][1])) lse_take(xf(ce.y, ud), cm[k][1], cs[k][1]);
              if (!(fmaf(ce.z, nr, ue) <= cthr[k][2])) lse_take(xf(ce.z, ud), cm[k][2], cs[k][2]);
              if (!(fmaf(ce.w, nr, ue) <= cthr[k][3])) lse_take(xf(ce.w, ud), cm[k][3], cs[k][3]);
            }
          }
        }
      }
      __syncthreads();  // u_chunk is restaged for the next chunk
    }
#pragma unroll
    for (int k = 0; k < KG; ++k) {
      const int g = tid + kSkThreads * k;
      if (g >= ng) continue;
      double* pm = part_m + (int64_t)b * n1p + g * 4;
      double* ps = part_s + (int64_t)b * n1p + g * 4;
#pragma unroll
      for (int c = 0; c < 4; ++c) { pm[c] = cm[k][c]; ps[c] = cs[k][c]; }
    }
  };


  // Fused sweep (iterations >= 1): per chunk of 8 rows the row LSEs (two warps per row, half a row each) and, with the
  // fresh u, the column candidates of the same rows -- the chunk (8 x 16 KB at n1 = 4096) is still in L1, so M crosses
  // the L2 -> SM path once per iteration and no grid barrier separates the two phases.  The column thresholds need the
  // global minimum of this iteration's u changes, which is not known yet: an ASSUMED value is used (the previous
  // iteration's minimum - 8) and verified after the barrier; the caller repeats the column pass in the rare case it
  // was too optimistic.
  __shared__ double half_m[2][8], half_s[2][8];
  auto fused_phase = [&](float dv_min, float du_assumed) {
    double cm[KG][4], cs[KG][4];
    float cthr[KG][4];
#pragma unroll
    for (int k = 0; k < KG; ++k)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        cm[k][c] = Tr<true>::init(); cs[k][c] = 0.0;
        const int col = (tid + kSkThreads * k) * 4 + c;
        cthr[k][c] = col < n1 ? __double2float_rd(logb - v_s[col] + (double)du_assumed) - kScreenGap : kBig;
      }
    const int ngh = ((ng + 1) / 2 + 31) / 32 * 32;  // float4 groups of the first half-row
    const int rr = warp & 7, half = warp >> 3;
    float dmin = kBig;
    unsigned long long* ctl = reinterpret_cast<unsigned long long*>(reinterpret_cast<char*>(p.err_ring) + 4608) + (b == 0 ? 0 : 16);
    const bool ctl_on = p.timeline == 2 && (b == 0 || b == nblk - 1) && (tid == 0 || tid == 511);
#define SK_TLC(slot) do { if (ctl_on && r0 == r_begin + 8) { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); ctl[(slot) + (tid == 0 ? 0 : 5)] = t_; } } while (0)
    for (int r0 = r_begin; r0 < r_end; r0 += 8) {
      const int R = min(8, r_end - r0);
      SK_TLC(0);
      if (rr < R) {
        const float* row = p.M + (int64_t)(r0 + rr) * p.ldm;
        const float thr = __double2float_rd(loga - u_work[r0 + rr] + (double)dv_min) - kScreenGap;
        double wm, ws;
        row_range_seeded<VEC, 8, true>(row, v_s, vh_s, n1, half ? ngh : 0, half ? ng : min(ngh, ng), xf, nr, thr, lane, wm, ws);
        if (lane == 0) { half_m[half][rr] = wm; half_s[half][rr] = ws; }
      }
      SK_TLC(1);
      __syncthreads();
      SK_TLC(2);
      if (warp < R) {  // warp w finishes row r0 + w
        const double m0 = half_m[0][warp], m1 = half_m[1][warp];
        const double mm = vmax(m0, m1);
        const double ss = half_s[0][warp] * expd<true>(m0, mm) + half_s[1][warp] * expd<true>(m1, mm);
        double lse = lse_fin(mm, ss);
        const float* row = p.M + (int64_t)(r0 + warp) * p.ldm;
        if (!(ss > 0.0)) lse = row_lse_screened<VEC>(row, v_s, vh_s, n1, ng, xf, nr, lane);  // (warp-uniform; never with a valid bound)
        const double uval = loga - lse;
        if (lane == 0) {
          dmin = fminf(dmin, __double2float_rd(uval - u_work[r0 + warp]));
          u_work[r0 + warp] = uval;
          p.log_u[r0 + warp] = uval;
          u_chunk[warp] = uval; uh_chunk[warp] = (float)uval;
        }
      } else if (warp < 8 && lane == 0) {
        u_chunk[warp] = 0.0; uh_chunk[warp] = 0.f;
      }
      __syncthreads();
      SK_TLC(3);
#pragma unroll
      for (int k = 0; k < KG; ++k) {
        const int g = tid + kSkThreads * k;
        const bool gv = g < ng;
        float4 c[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          if (gv && q < R) {
            c[q] = VEC ? __ldg(reinterpret_cast<const float4*>(p.M + (int64_t)(r0 + q) * p.ldm + g * 4))
                       : load_cost4<VEC>(p.M + (int64_t)(r0 + q) * p.ldm, g * 4, n1);
          } else {
            const float inf = __int_as_float(0x7f800000);
            c[q] = make_float4(inf, inf, inf, inf);
          }
        }
        float uh[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) uh[q] = uh_chunk[q];
        unsigned hm = 0;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const bool le = (fmaf(c[q].x, nr, uh[q]) <= cthr[k][0]) & (fmaf(c[q].y, nr, uh[q]) <= cthr[k][1]) &
                          (fmaf(c[q].z, nr, uh[q]) <= cthr[k][2]) & (fmaf(c[q].w, nr, uh[q]) <= cthr[k][3]);
          hm |= (le ? 0u : 1u) << q;
        }
        while (__any_sync(0xffffffffu, hm != 0u)) {
          if (hm != 0u) {
            const int e = __ffs((int)hm) - 1;
            hm &= hm - 1u;
            const float4 c01 = (e & 1) ? ((e & 2) ? c[3] : c[1]) : ((e & 2) ? c[2] : c[0]);
            const float4 c45 = (e & 1) ? ((e & 2) ? c[7] : c[5]) : ((e & 2) ? c[6] : c[4]);
            const float4 ce = (e & 4) ? c45 : c01;
            const float ue = uh_chunk[e];
            const double ud = u_chunk[e];
            if (!(fmaf(ce.x, nr, ue) <= cthr[k][0])) lse_take(xf(ce.x, ud), cm[k][0], cs[k][0]);
            if (!(fmaf(ce.y, nr, ue) <= cthr[k][1])) lse_take(xf(ce.y, ud), cm[k][1], cs[k][1]);
            if (!(fmaf(ce.z, nr, ue) <= cthr[k][2])) lse_take(xf(ce.z, ud), cm[k][2], cs[k][2]);
            if (!(fmaf(ce.w, nr, ue) <= cthr[k][3])) lse_take(xf(ce.w, ud), cm[k][3], cs[k][3]);
          }
        }
      }
      SK_TLC(4);
      // (no third barrier: u_chunk / half_* are rewritten only behind the next chunk's first barrier)
    }
#pragma unroll
    for (int k = 0; k < KG; ++k) {
      const int g = tid + kSkThreads * k;
      if (g >= ng) continue;
      double* pm = part_m + (int64_t)b * n1p + g * 4;
      double* ps = part_s + (int64_t)b * n1p + g * 4;
#pragma unroll
      for (int c = 0; c < 4; ++c) { pm[c] = cm[k][c]; ps[c] = cs[k][c]; }
    }
    dmin = block_min_f(lane == 0 ? dmin : kBig, redf, tid);
    if (tid == 0) dmin_u[b] = dmin;
  };

  // combine the per-CTA column partials of a slice of columns -> v_new, marginal error, min of (v_new - v_cur)
  auto combine = [&](const double* v_cur, double* v_new, bool have_cur, double* err_slot) {
    const int cpc = (n1 + nblk - 1) / nblk;
    const int c_begin = b * cpc, c_end = min(n1, c_begin + cpc);
    double err_local = 0.0;
    float dmin = kBig;
    const int sub = tid & 7;
    for (int j0 = c_begin; j0 < c_end; j0 += (kSkThreads >> 3)) {
      const int j = j0 + (tid >> 3);
      const bool act = j < c_end;
      double m = Tr<true>::init(), s = 0.0;
      if (act) {
        for (int c0 = sub; c0 < nblk; c0 += 8 * 4) {
          double mm[4], ss[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int c = c0 + q * 8;
            if (c < nblk) {
              mm[q] = __ldcg(part_m + (int64_t)c * n1p + j);
              ss[q] = __ldcg(part_s + (int64_t)c * n1p + j);
            } else { mm[q] = Tr<true>::init(); ss[q] = 0.0; }
          }
          double bm = vmax(vmax(mm[0], mm[1]), vmax(mm[2], mm[3]));
          bm = vmax(bm, m);
          double acc = s * expd<true>(m, bm);
#pragma unroll
          for (int q = 0; q < 4; ++q) acc += ss[q] * expd<true>(mm[q], bm);
          s = acc; m = bm;
        }
      }
      double gm = m;
#pragma unroll
      for (int o = 4; o > 0; o >>= 1) gm = vmax(gm, __shfl_xor_sync(0xffffffffu, gm, o));
      double gs = s * expd<true>(m, gm);
#pragma unroll
      for (int o = 4; o > 0; o >>= 1) gs += __shfl_xor_sync(0xffffffffu, gs, o);
      if (act && sub == 0) {
        const double vn = logb - lse_fin(gm, gs);
        v_new[j] = vn;
        if (have_cur) {
          const double vc = __ldcg(v_cur + j);
          dmin = fminf(dmin, __double2float_rd(vn - vc));
          const double e = expm1(vc - vn) / (double)n1;  // column marginal of (u, v_cur) minus 1/n1
          err_local += e * e;
        }
      }
    }
    dmin = block_min_f(dmin, redf, tid);
    if (tid == 0) dmin_v[b] = dmin;
    if (err_slot != nullptr) {
      err_local = warp_sum(err_local);
      if (lane == 0) red[warp] = err_local;
      __syncthreads();
      if (warp == 0) {
        double t = lane < kSkWarps ? red[lane] : 0.0;
        t = warp_sum(t);
        if (lane == 0) atomicAdd(err_slot, t);
      }
      __syncthreads();
    }
  };

  // ---- prologue: v^0 = logb - LSE_i(Mr_ij + 0) ----
  if (b == 0 && tid < 4) p.err_ring[tid] = 0.0;
  col_phase(false, false, 0.f);
  grid.sync();
  combine(nullptr, v_work[0], false, nullptr);
  grid.sync();

  int cur = 0, iters = 0;
  bool converged = false;
  double err = 1.0, prev_check_err = -1.0;
  float du_prev = 0.f;  // global minimum of the u changes of the previous iteration
  // CFM_SK_TL=1: %globaltimer marks of iteration 50 for the first and the last CTA (scripts/c4_timeline.py)
  unsigned long long* tl = reinterpret_cast<unsigned long long*>(reinterpret_cast<char*>(p.err_ring) + 4608) + (b == 0 ? 0 : 16);
  const bool tl_on = p.timeline && (b == 0 || b == nblk - 1) && tid == 0;
#define SK_TL(slot) do { if (tl_on && it == 50) { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); tl[slot] = t_; } } while (0)
  for (int it = 0; it < p.max_iters; ++it) {
    const bool last = (it == p.max_iters - 1);
    const bool check = (it % p.check_every) == 0;
    const bool do_col = !last || check;
    SK_TL(0);
    stage_v(v_work[cur]);
    SK_TL(1);
    const float dv_min = it > 0 ? global_min(dmin_v) : 0.f;
    SK_TL(2);
    const bool fused = it > 0 && do_col;
    if (!fused) {
      row_phase(it > 0, dv_min);
      SK_TL(3);
      iters = it + 1;
      if (!do_col) break;
      grid.sync();
      SK_TL(4);
      du_prev = global_min(dmin_u);
      col_phase(true, true, du_prev);
      SK_TL(5);
      grid.sync();
      SK_TL(6);
    } else {
      const float du_assumed = du_prev - 8.f;
      fused_phase(dv_min, du_assumed);
      SK_TL(5);
      iters = it + 1;
      grid.sync();
      SK_TL(6);
      du_prev = global_min(dmin_u);   // the true minimum: every CTA reads the same slots and takes the same branch
      if (!(du_prev >= du_assumed)) {  // the assumption was too optimistic (or NaN): column pass again, exact bound
        col_phase(true, true, du_prev);
        grid.sync();
      }
    }
    SK_TL(7);
    if (b == 0 && tid == 0) p.err_ring[(it + 2) & 3] = 0.0;
    combine(v_work[cur], v_work[cur ^ 1], true, &p.err_ring[it & 3]);
    SK_TL(8);
    grid.sync();
    SK_TL(9);
    if (check) {
      err = sqrt(__ldcg(&p.err_ring[it & 3]));
      if (err < p.stop_thr) { converged = true; break; }
      if (p.stall_tol > 0.0 && prev_check_err >= 0.0 &&
          err > (1.0 - p.stall_tol) * prev_check_err &&
          err * sqrt((double)n1) < 1e-5) { converged = true; break; }
      prev_check_err = err;
    }
    if (last) break;
    cur ^= 1;
  }
#undef SK_TL

  for (int j = b * kSkThreads + tid; j < n1; j += nblk * kSkThreads) p.log_v[j] = __ldcg(v_work[cur] + j);
  if (b == 0 && tid == 0) {
    int flags = 0;
    if (!converged) flags |= CFM_FLAG_NOT_CONVERGED;
    if (!(err == err)) flags |= CFM_FLAG_NONFINITE;
    p.status[0] = flags;
    p.status[1] = iters;
    p.status[2] = 2;
    p.status[3] = 1;  // kernel variant: seeded screening
    *p.err_out = err;
  }
}

template <bool VEC, int KG>
__global__ void __launch_bounds__(kSkThreads, 1) sinkhorn_kernel(const SkParams p) {
  extern __shared__ __align__(16) unsigned char sk_smem[];
  bool precise = p.precise == 1;
  if (p.precise < 0) {
    const float cmax = p.cost_max ? __ldg(p.cost_max) : 0.f;
    const float span = (p.normalize ? 1.f : cmax) / p.reg;
    precise = !(span <= 64.f);
  }
  if (p.run_if == 2 && !precise) return;  // the fast case was taken by sinkhorn_v2_kernel
  if (precise) {
    // mixed arithmetic on one column panel with v staged in shared memory: the seeded-screening solver
    if (p.mixed && p.screen == 1 && p.v_in_smem && p.n1p <= kSkThreads * 4 * KG) sinkhorn_run_seeded<VEC, KG>(p, sk_smem);
    else if (p.mixed) sinkhorn_run<true, VEC, KG, true>(p, sk_smem);
    else sinkhorn_run<true, VEC, KG, false>(p, sk_smem);
  } else {
    sinkhorn_run<false, VEC, KG, false>(p, sk_smem);
  }
}

// ---- plan materialisation: plan_ij = exp(-M_ij/reg + log_u_i + log_v_j) in float64 ----------
__global__ void plan_materialize_kernel(const float* __restrict__ M, int n0, int n1, int64_t ldm,
                                        float reg, const float* cost_max, int normalize,
                                        const double* __restrict__ lu, const double* __restrict__ lv,
                                        double* __restrict__ plan, double* mass, int32_t* status) {
  const float cmax = (normalize && cost_max) ? __ldg(cost_max) : 1.f;
  const int i = blockIdx.y;
  const double ui = lu[i];
  double local = 0.0;
  bool bad = false;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n1; j += gridDim.x * blockDim.x) {
    float m = M[(int64_t)i * ldm + j];
    if (normalize) m = __fdiv_rn(m, cmax);
    const double v = exp((double)(-__fdiv_rn(m, reg)) + ui + lv[j]);
    plan[(int64_t)i * n1 + j] = v;
    local += v;
    bad |= !isfinite(v);
  }
  local = warp_sum(local);
  if ((threadIdx.x & 31) == 0 && local != 0.0) atomicAdd(mass, local);
  if (bad) atomicOr(status, CFM_FLAG_NONFINITE);
}

size_t sinkhorn_v2_compact_pitch(int n0, int n1);  // sinkhorn_v2.cu

struct SkLayout {
  size_t u, v0, v1, pm, ps, ring, mq, mq_bytes, total;
};
static SkLayout sk_layout(int n0, int n1, int grid) {
  const size_t n1p = (size_t)(n1 + 3) / 4 * 4;
  SkLayout L;
  size_t o = 0;
  L.u = o; o += align_up((size_t)n0 * 8, 256);
  L.v0 = o; o += align_up(n1p * 8, 256);
  L.v1 = o; o += align_up(n1p * 8, 256);
  L.pm = o; o += align_up((size_t)grid * n1p * 8, 256);
  L.ps = o; o += align_up((size_t)grid * n1p * 8, 256);
  L.ring = o; o += 8192;  // err ring (4 doubles) + per-CTA minima of the potential changes (2 x 512 floats)
  L.mq_bytes = (size_t)n0 * sinkhorn_v2_compact_pitch(n0, n1);  // 3-byte cost copy (shapes whose fp32 M streams)
  L.mq = o; o += align_up(L.mq_bytes, 256);
  L.total = o;
  return L;
}
static int sk_grid_upper() { return sm_count() * 2; }
int sinkhorn_v2_launch(SkParams& p, cudaStream_t s);  // sinkhorn_v2.cu

}  // namespace cfm

using namespace cfm;

extern "C" size_t cfm_sinkhorn_workspace_bytes(int n0, int n1) {
  return sk_layout(n0, n1, sk_grid_upper()).total;
}

template <bool VEC, int KG>
static int sk_launch(SkParams& p, size_t smem, void* workspace, cudaStream_t s) {
  auto kern = sinkhorn_kernel<VEC, KG>;
  CFM_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  CFM_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kSkThreads, smem));
  CFM_REQUIRE(per_sm >= 1, "cfm_sinkhorn_log_f32: kernel does not fit on an SM (smem %zu)", smem);
  int grid = sm_count() * (per_sm > 2 ? 2 : per_sm);
  if (grid > p.n0) grid = p.n0;  // at least one row per CTA
  if (grid > sk_grid_upper()) grid = sk_grid_upper();
  const SkLayout L = sk_layout(p.n0, p.n1, sk_grid_upper());
  char* w = reinterpret_cast<char*>(workspace);
  p.u_work = w + L.u;
  p.v_work[0] = w + L.v0;
  p.v_work[1] = w + L.v1;
  p.part_m = w + L.pm;
  p.part_s = w + L.ps;
  p.err_ring = reinterpret_cast<double*>(w + L.ring);
  void* args[] = {(void*)&p};
  CFM_CUDA_OK(cudaLaunchCooperativeKernel((void*)kern, dim3(grid), dim3(kSkThreads), args, smem, s));
  note_launches(1);
  return CFM_OK;
}

extern "C" int cfm_sinkhorn_log_f32(const float* M, int n0, int n1, int64_t ldm, float reg,
                                       const float* cost_max, int normalize, int max_iters,
                                       double stop_thr, int check_every, int precise,
                                       double stall_tol, double* log_u, double* log_v,
                                       int32_t* status, double* err, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  CFM_REQUIRE(M && log_u && log_v && status && err && workspace, "cfm_sinkhorn_log_f32: null pointer");
  CFM_REQUIRE(n0 > 0 && n1 > 0 && ldm >= n1, "cfm_sinkhorn_log_f32: bad shape n0=%d n1=%d ldm=%lld", n0,
              n1, (long long)ldm);
  CFM_REQUIRE(reg > 0.f, "cfm_sinkhorn_log_f32: reg must be > 0 (got %g)", (double)reg);
  CFM_REQUIRE(max_iters >= 1 && check_every >= 1, "cfm_sinkhorn_log_f32: max_iters/check_every must be >= 1");
  CFM_REQUIRE(!(normalize && !cost_max), "cfm_sinkhorn_log_f32: normalize needs cost_max");
  CFM_REQUIRE(!(precise < 0 && !cost_max), "cfm_sinkhorn_log_f32: precise=-1 (auto) needs cost_max");
  CFM_REQUIRE(workspace_bytes >= cfm_sinkhorn_workspace_bytes(n0, n1),
              "cfm_sinkhorn_log_f32: workspace too small (%zu < %zu)", workspace_bytes,
              cfm_sinkhorn_workspace_bytes(n0, n1));
  SkParams p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.n0 = n0; p.n1 = n1; p.ldm = ldm; p.reg = reg; p.cost_max = cost_max;
  p.normalize = normalize; p.max_iters = max_iters; p.stop_thr = stop_thr;
  p.check_every = check_every; p.precise = precise; p.stall_tol = stall_tol;
  p.log_u = log_u; p.log_v = log_v; p.status = status; p.err_out = err;
  p.n1p = (n1 + 3) / 4 * 4;
  p.vec = ((n1 & 3) == 0) && ((ldm & 3) == 0) && ((reinterpret_cast<uintptr_t>(M) & 15) == 0);
  const SkLayout L = sk_layout(n0, n1, sk_grid_upper());
  {
    char* w = reinterpret_cast<char*>(workspace);
    p.u_work = w + L.u; p.v_work[0] = w + L.v0; p.v_work[1] = w + L.v1;
    p.part_m = w + L.pm; p.part_s = w + L.ps; p.err_ring = reinterpret_cast<double*>(w + L.ring);
    p.mq = L.mq_bytes ? reinterpret_cast<unsigned char*>(w + L.mq) : nullptr;
  }
  // CFM_SK_TL: timeline marks, read by both kernels (so set before the smem-staged launch)
  static int tl = -1;
  if (tl < 0) { const char* e = getenv("CFM_SK_TL"); tl = e ? atoi(e) : 0; }
  p.timeline = tl;
  // precise: -1 auto, 0 fp32, 1 float64, 2 fp32 on the generic kernel, 3 float64 with fp32 exponentials ("mixed"),
  // 4 = 3 without the screening of negligible terms
  p.screen = 1;
  if (precise == 4) { precise = 3; p.screen = 0; }  // mixed without the fp32 screening (cross-checks)
  if (precise == 3) { precise = 1; p.precise = 1; p.mixed = 1; }
  else if (precise < 0) p.mixed = 1;  // auto mode needing float64 potentials: "mixed" (fp32 exponentials of float64 differences)
  // fast fp32 mode on aligned n1 <= 8192: smem-staged kernel (sinkhorn_v2.cu)
  if (precise == 2) { precise = 0; p.precise = 0; }  // fast arithmetic, generic kernel (cross-checks)
  else if (precise != 1) {
    p.run_if = precise < 0 ? 1 : 0;
    const int rc = sinkhorn_v2_launch(p, s);
    if (rc < 0) return rc;
    if (rc == CFM_OK) {
      if (precise == 0) return CFM_OK;
      p.run_if = 2;  // auto: the generic kernel below only runs when float64 potentials are needed
    } else {
      p.run_if = 0;
    }
  }
  const size_t vbytes = (size_t)p.n1p * 12;  // float64 stage + its fp32 copy (screened mixed mode)
  p.v_in_smem = vbytes <= 160 * 1024;
  const size_t smem = p.v_in_smem ? vbytes : 0;
  const int ng = p.n1p / 4;
  const int kg_need = (ng + kSkThreads - 1) / kSkThreads;
  if (p.vec) {
    if (kg_need <= 1) return sk_launch<true, 1>(p, smem, workspace, s);
    if (kg_need <= 2) return sk_launch<true, 2>(p, smem, workspace, s);
    return sk_launch<true, 4>(p, smem, workspace, s);  // n1 > 8192: several column panels
  }
  if (kg_need <= 1) return sk_launch<false, 1>(p, smem, workspace, s);
  if (kg_need <= 2) return sk_launch<false, 2>(p, smem, workspace, s);
  return sk_launch<false, 4>(p, smem, workspace, s);
}

extern "C" int cfm_plan_materialize_f64(const float* M, int n0, int n1, int64_t ldm, float reg,
                                        const float* cost_max, int normalize, const double* log_u,
                                        const double* log_v, double* plan, double* mass,
                                        int32_t* status, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  CFM_REQUIRE(M && log_u && log_v && plan && mass && status, "cfm_plan_materialize_f64: null pointer");
  CFM_REQUIRE(n0 > 0 && n1 > 0 && ldm >= n1, "cfm_plan_materialize_f64: bad shape");
  CFM_REQUIRE(!(normalize && !cost_max), "cfm_plan_materialize_f64: normalize needs cost_max");
  CFM_CUDA_OK(cudaMemsetAsync(mass, 0, sizeof(double), s));
  dim3 grid((n1 + 1023) / 1024 > 8 ? 8 : (n1 + 1023) / 1024, n0);
  plan_materialize_kernel<<<grid, 256, 0, s>>>(M, n0, n1, ldm, reg, cost_max, normalize, log_u, log_v,
                                              plan, mass, status); ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
