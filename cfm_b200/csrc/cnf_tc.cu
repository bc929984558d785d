// Hutchinson's log-likelihood field of WIDE MLP flows on the tensor cores (DESIGN.md section 3.17): the field of
// cnf_wrapper(MLP(dim, w, time_varying=True), likelihood_estimator="hutch_gaussian" / "hutch_rademacher") for models
// in the tensor-core class (mlp_tc_supported(B, dim, w, dim), e.g. BASELINE config 3, 785 -> 256 -> 256 -> 256 -> 784),
// as cfm_b200/ode.py drives it with Euler or dopri5:
//     d/dt [x, ll] = [f(t, x), eps . (J eps)],   J = df/dx at (t, x),   one fresh probe eps per field evaluation.
// eps^T J eps is eps . (J eps), a forward-mode tangent: one more pass through the same four GEMMs with act'(pre) in
// place of act.  One evaluation is ten launches:
//   probe     eps (Gaussian: sde_normal4; Rademacher: sde_rademacher4) of ordinal *ordinal_dev + offset, kept in fp32
//             for the contraction and split (hi, lo) as the tangent's layer-0 operand; an fp32 x is split here too;
//   layer l   primal GEMM (the fp16x3 core of gemm_h3.cuh on the prepared blob's weight pair): the epilogue of
//             mlp_h3.cu's per-layer path (bias, t W0[:, dim] at layer 0, activation, saturating (hi, lo) split), which also stores act'(pre)
//             in fp32; then the tangent GEMM on the same weights: u_{l+1} = act'(pre_l) * (W_l u_l), no bias, no time
//             column, saturating (hi, lo) split.  The primal of layer l + 1 overwrites act'(pre_l) only after the tangent
//             of layer l has read it (stream order), so one buffer serves all three hidden layers;
//   layer 3   the primal writes f; the tangent writes one float64 partial sum_c eps[r, c] (W3 u_3)[r, c] per row and
//             32-column chunk;
//   fold      div_r = sum of row r's partials in chunk order.
// No floating-point atomics touch a sum: the same call gives the same bits.  The Euler driver's init and step kernels
// work like sde_tc.cu's: the step index (= the probe ordinal), time, seed and trajectory pointer live in a device
// struct, so a captured step replays for the whole trajectory.  Shared with sde_tc.cu: the operand split and packing
// (gemm_h3.cuh), the state's shape rule and step advance (sde_common.cuh) and the launch grid (common.cuh); the GEMMs
// go through launch_gemm_h3 with this file's kernel entry.
#include "gemm_h3.cuh"
#include "mlp_small.cuh"  // act_deriv_fast
#include "sde_common.cuh"

namespace cfm {

namespace {

struct CnfWs {
  size_t xh, xl, eps, uh, ul, ah, al, bh, bl, th, tl, sh, sl, dact, parts, total;
  int nchunk;
};
CnfWs cnf_ws(int batch, int dim, int w) {
  CnfWs p;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes, 1024); return r; };
  const size_t bd = (size_t)batch * dim, bw = (size_t)batch * w;
  p.nchunk = (dim + 31) / 32;
  p.xh = take(bd * 2); p.xl = take(bd * 2);
  p.eps = take(bd * 4);
  p.uh = take(bd * 2); p.ul = take(bd * 2);
  p.ah = take(bw * 2); p.al = take(bw * 2); p.bh = take(bw * 2); p.bl = take(bw * 2);  // primal ping-pong
  p.th = take(bw * 2); p.tl = take(bw * 2); p.sh = take(bw * 2); p.sl = take(bw * 2);  // tangent ping-pong
  p.dact = take(bw * 4);
  p.parts = take((size_t)batch * p.nchunk * sizeof(double));
  p.total = o;
  return p;
}

bool cnf_tc_shape(int batch, int dim, int w) { return mlp_tc_supported(batch, dim, w, dim) != 0; }

// one row's 32 values -> (hi, lo) at hi/lo + [0, 32) (16-byte aligned) or, for a partial chunk, [0, n)
__device__ __forceinline__ void split_row32(const float (&v)[32], __half* hi, __half* lo, bool full, int n) {
  if (full) {
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      __half hh[8], ll[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) split_h3_sat(v[8 * g + c], hh[c], ll[c]);
      *reinterpret_cast<uint4*>(hi + 8 * g) = pack8h(hh);
      *reinterpret_cast<uint4*>(lo + 8 * g) = pack8h(ll);
    }
  } else {
#pragma unroll
    for (int c = 0; c < 32; ++c)
      if (c < n) { __half h, l; split_h3_sat(v[c], h, l); hi[c] = h; lo[c] = l; }
  }
}

// eps of probe ordinal *ord + ord_off, fp32 and split; x (nullable) split.  One thread per 4 columns of a row.
__global__ void __launch_bounds__(256)
cnf_probe_kernel(const float4* __restrict__ x, __half* __restrict__ xh, __half* __restrict__ xl,
                 float4* __restrict__ eps, __half* __restrict__ uh, __half* __restrict__ ul,
                 const uint64_t* __restrict__ seed_dev, const int32_t* __restrict__ ord, int ord_off, int estimator,
                 int dim4, int64_t n4) {
  const uint64_t seed = *seed_dev;
  const int n = *ord + ord_off;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const int64_t r = i / dim4;
    const int q = (int)(i - r * dim4);
    const float4 z = estimator == CFM_HUTCH_GAUSSIAN ? sde_normal4(seed, n, r, q) : sde_rademacher4(seed, n, r, q);
    eps[i] = z;
    split4_store(z, uh, ul, i);
    if (x != nullptr) split4_store(x[i], xh, xl, i);
  }
}

// primal layer: pre = acc / s_W + b (+ t W0[:, dim]); hidden: act'(pre) fp32 and act(pre) split, output layer: f.
// The value expressions are MlpH3Epilogue's (mlp_h3.cu), so f has the bits of the per-layer forward.
struct CnfPrimalEpi {
  const float* bias;
  const float* inv_ws;
  const float* tcol;   // layer 0: W0[:, dim]
  const float* t_dev;
  int act;             // -1: output layer
  float* dact;         // hidden: [B][ldo]
  __half* out_hi;      // hidden: [B][ldo]
  __half* out_lo;
  float* f;            // output layer: [B][ldo], any 4-byte alignment
  int64_t ldo;
  float t;
  __device__ __forceinline__ void begin_row(int, bool) { t = tcol ? __ldg(t_dev) : 0.f; }
  __device__ __forceinline__ void store32(int row0, int lane, int col0, const float (&r)[32], int n0, int n1,
                                          float* tile) {
    const int row = row0 + lane;
    const bool full = col0 + 32 <= n1;
    float v[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      float p = 0.f;
      if (col0 + c < n1) {
        p = fmaf(r[c], __ldg(inv_ws + col0 + c), __ldg(bias + col0 + c));
        if (tcol) p = fmaf(t, __ldg(tcol + col0 + c), p);
      }
      v[c] = p;
    }
    if (act < 0) {
      float* base = f + (int64_t)row0 * ldo + col0;
      if (full && (ldo & 3) == 0 && aligned16(base)) {
        tc_store_chunk32(tile, v, base, ldo, n0 - row0, lane);
      } else if (row < n0) {
#pragma unroll
        for (int c = 0; c < 32; ++c)
          if (col0 + c < n1) f[(int64_t)row * ldo + col0 + c] = v[c];
      }
      return;
    }
    if (row >= n0) return;  // no warp-collective operation follows
    // act'(pre) four columns at a time, straight from the row layout (a 32-value array would spill next to the
    // accumulators)
    float* dr = dact + (int64_t)row * ldo + col0;
    if (full) {
#pragma unroll
      for (int g = 0; g < 8; ++g)
        reinterpret_cast<float4*>(dr)[g] =
            make_float4(act_deriv_fast(v[4 * g], act), act_deriv_fast(v[4 * g + 1], act),
                        act_deriv_fast(v[4 * g + 2], act), act_deriv_fast(v[4 * g + 3], act));
    } else {
#pragma unroll
      for (int c = 0; c < 32; ++c)
        if (col0 + c < n1) dr[c] = act_deriv_fast(v[c], act);
    }
#pragma unroll
    for (int c = 0; c < 32; ++c) v[c] = act_apply_fast(v[c], act);
    split_row32(v, out_hi + (int64_t)row * ldo + col0, out_lo + (int64_t)row * ldo + col0, full, n1 - col0);
  }
  __device__ __forceinline__ void finish(int) {}
};

// tangent layer: J_l u = acc / s_W; hidden: u' = act'(pre) * J_l u, split; output layer: float64 partial of
// sum_c eps[r, c] (J_3 u)[r, c] over the chunk's columns
struct CnfTangentEpi {
  const float* inv_ws;
  const float* dact;   // hidden: [B][ldo]
  __half* out_hi;      // hidden: [B][ldo]
  __half* out_lo;
  int64_t ldo;
  const float* eps;    // output layer: [B][ldo]; null on hidden layers
  double* parts;       // output layer: [B][nchunk]
  int nchunk;
  __device__ __forceinline__ void begin_row(int, bool) {}
  __device__ __forceinline__ void store32(int row0, int lane, int col0, const float (&r)[32], int n0, int n1,
                                          float*) {
    const int row = row0 + lane;
    if (row >= n0) return;  // no warp-collective operation follows
    const bool full = col0 + 32 <= n1;
    const float* src = (eps ? eps : dact) + (int64_t)row * ldo + col0;  // 16-byte aligned when full (ldo % 8 == 0)
    float m[32];
    if (full) {
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(src) + g);
        m[4 * g] = q.x; m[4 * g + 1] = q.y; m[4 * g + 2] = q.z; m[4 * g + 3] = q.w;
      }
    } else {
#pragma unroll
      for (int c = 0; c < 32; ++c) m[c] = col0 + c < n1 ? __ldg(src + c) : 0.f;
    }
    float jv[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) jv[c] = col0 + c < n1 ? r[c] * __ldg(inv_ws + col0 + c) : 0.f;
    if (eps) {
      double part = 0.0;
#pragma unroll
      for (int c = 0; c < 32; ++c) part = fma((double)m[c], (double)jv[c], part);
      parts[(int64_t)row * nchunk + (col0 >> 5)] = part;
      return;
    }
#pragma unroll
    for (int c = 0; c < 32; ++c) jv[c] *= m[c];
    split_row32(jv, out_hi + (int64_t)row * ldo + col0, out_lo + (int64_t)row * ldo + col0, full, n1 - col0);
  }
  __device__ __forceinline__ void finish(int) {}
};

// The GEMMs of this file: the persistent fp16x3 core of gemm_tc.cuh (gemm_wg_body, no split-K) under an entry of their
// own, so that the instantiations of gemm_wg_kernel (cost matrix, per-layer MLP) and of gemm_wg_splitk_kernel (training)
// stay the ones their tests pin; tests/test_cnf_tc_host.py pins these two.
template <class Epi>
__global__ void __launch_bounds__(kWgThreads, 1)
cnf_gemm_kernel(const __grid_constant__ CUtensorMap map_ah, const __grid_constant__ CUtensorMap map_al,
                const __grid_constant__ CUtensorMap map_bh, const __grid_constant__ CUtensorMap map_bl, const TcShape p,
                Epi epi) {
  gemm_wg_body<H3Scheme, Epi, false>(map_ah, map_al, map_bh, map_bl, p, epi);
}

// div_r = sum over chunks k of parts[r][k], in k order
__global__ void __launch_bounds__(256) cnf_fold_kernel(const double* __restrict__ parts, int nchunk,
                                                       float* __restrict__ div, int batch) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= batch) return;
  double s = 0.0;
  for (int k = 0; k < nchunk; ++k) s += parts[(int64_t)r * nchunk + k];
  div[r] = (float)s;
}

// ---- Euler driver -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
cnf_euler_init_kernel(cfm_cnf_tc_state* __restrict__ st, const float* __restrict__ z0, float4* __restrict__ x,
                      float* __restrict__ ll, __half* __restrict__ hi, __half* __restrict__ lo, float* traj,
                      const float* t_span, int n_steps, uint64_t seed, int dim4, int64_t n4, int batch) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    st->seed = seed; st->traj = traj; st->t_span = t_span;
    st->n = 0; st->n_steps = n_steps; st->t = t_span[0]; st->ticket = 0u;
  }
  const int64_t ld = 4 * dim4 + 1;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int64_t i = tid; i < n4; i += stride) {
    const int64_t r = i / dim4;
    const float* zr = z0 + r * ld + 4 * (i - r * dim4);
    const float4 v = make_float4(zr[0], zr[1], zr[2], zr[3]);
    x[i] = v;
    split4_store(v, hi, lo, i);
  }
  for (int64_t r = tid; r < batch; r += stride) ll[r] = z0[r * ld + ld - 1];
  for (int64_t i = tid; i < (int64_t)batch * ld; i += stride) traj[i] = z0[i];
}

// step n = st->n: x <- fmaf(h, f, x), ll <- fmaf(h, div, ll), traj[n + 1], the split of x; the CTA that finishes last
// advances the state.  A step enqueued past n_steps does nothing.
__global__ void __launch_bounds__(256)
cnf_euler_step_kernel(cfm_cnf_tc_state* st, float4* __restrict__ x, float* __restrict__ ll,
                      const float4* __restrict__ f, const float* __restrict__ div, __half* __restrict__ hi,
                      __half* __restrict__ lo, int dim4, int64_t n4, int batch) {
  const int n = st->n;
  if (n >= st->n_steps) return;
  const float* ts = st->t_span;
  const float t0 = ts[n], t1 = ts[n + 1];
  const float h = (float)((double)t1 - (double)t0);  // the plain Euler driver's step: float(ts[n + 1] - ts[n])
  const int64_t ld = 4 * dim4 + 1;
  float* out = st->traj + (int64_t)(n + 1) * batch * ld;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int64_t i = tid; i < n4; i += stride) {
    const float4 a = x[i], k = f[i];
    const float4 v = make_float4(fmaf(h, k.x, a.x), fmaf(h, k.y, a.y), fmaf(h, k.z, a.z), fmaf(h, k.w, a.w));
    x[i] = v;
    split4_store(v, hi, lo, i);
    const int64_t r = i / dim4;
    float* o = out + r * ld + 4 * (i - r * dim4);
    o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
  }
  for (int64_t r = tid; r < batch; r += stride) {
    const float v = fmaf(h, div[r], ll[r]);
    ll[r] = v;
    out[r * ld + ld - 1] = v;
  }
  step_advance(st, n, t1);
}

}  // namespace

// One hidden primal layer on its own: the split of act(pre) to (out_hi, out_lo) and act'(pre) to dact, all [B][w].
// The gradient field of grad_tc.cu runs its layers 0 and 1 through this, on the same kernel instantiation.
int cnf_tc_primal_hidden(const __half* ah, const __half* al, int batch, int K, const void* wh, const void* wl,
                         int64_t ldw, int w, const float* bias, const float* inv_ws, const float* tcol,
                         const float* t_dev, int act, float* dact, __half* out_hi, __half* out_lo, cudaStream_t s) {
  CnfPrimalEpi pe;
  pe.bias = bias; pe.inv_ws = inv_ws; pe.tcol = tcol; pe.t_dev = t_dev; pe.act = act; pe.dact = dact;
  pe.out_hi = out_hi; pe.out_lo = out_lo; pe.f = nullptr; pe.ldo = w; pe.t = 0.f;
  return launch_gemm_h3<CnfPrimalEpi, cnf_gemm_kernel<CnfPrimalEpi>>(ah, al, batch, K, reinterpret_cast<const __half*>(wh),
                                                                     reinterpret_cast<const __half*>(wl), w, ldw, K, pe,
                                                                     s);
}

}  // namespace cfm

using namespace cfm;

extern "C" int cfm_cnf_tc_supported(int batch, int dim, int w) { return cnf_tc_shape(batch, dim, w) ? 1 : 0; }

extern "C" size_t cfm_cnf_tc_workspace_bytes(int batch, int dim, int w) {
  return cnf_tc_shape(batch, dim, w) ? cnf_ws(batch, dim, w).total : 0;
}

extern "C" int cfm_cnf_tc_field_f32(const void* prepared, const float* x, const void* x_hi, const void* x_lo,
                                    int batch, int dim, int w, int act, int estimator, const float* t_dev,
                                    const uint64_t* seed_dev, const int32_t* ordinal_dev, int ordinal_offset,
                                    float* f, float* div, void* workspace, size_t workspace_bytes, void* stream) {
  const char* what = "cfm_cnf_tc_field_f32";
  CFM_REQUIRE(prepared && f && div && workspace && t_dev && seed_dev && ordinal_dev, "%s: null pointer", what);
  CFM_REQUIRE((x != nullptr) != (x_hi != nullptr) && (x_hi == nullptr) == (x_lo == nullptr),
              "%s: pass either x or the pair (x_hi, x_lo)", what);
  CFM_REQUIRE(act == CFM_ACT_SELU || act == CFM_ACT_SILU, "%s: unknown activation %d", what, act);
  CFM_REQUIRE(estimator == CFM_HUTCH_GAUSSIAN || estimator == CFM_HUTCH_RADEMACHER, "%s: unknown estimator %d", what,
              estimator);
  CFM_REQUIRE(cnf_tc_shape(batch, dim, w),
              "%s: unsupported shape B=%d dim=%d w=%d (B >= 128, dim >= 32, dim and w multiples of 8, w >= 32)", what,
              batch, dim, w);
  const CnfWs P = cnf_ws(batch, dim, w);
  CFM_REQUIRE(workspace_bytes >= P.total, "%s: workspace too small (%zu < %zu)", what, workspace_bytes, P.total);
  CFM_REQUIRE(aligned16(x) && aligned16(x_hi) && aligned16(x_lo) && aligned16(workspace),
              "%s: x, x_hi, x_lo and the workspace must be 16-byte aligned", what);
  CFM_REQUIRE(((reinterpret_cast<uintptr_t>(f) | reinterpret_cast<uintptr_t>(div)) & 3) == 0,
              "%s: f and div must be 4-byte aligned", what);
  cudaStream_t s = (cudaStream_t)stream;
  const MlpBlobHeader h = mlp_layout(dim, w, dim, 1);
  const MlpTcWeights W = mlp_tc_weights(h, prepared);
  const char* blob = reinterpret_cast<const char*>(prepared);
  char* ws = reinterpret_cast<char*>(workspace);
  auto H = [&](size_t off) { return reinterpret_cast<__half*>(ws + off); };
  auto F = [&](int64_t off) { return reinterpret_cast<const float*>(blob + off); };

  const int64_t n4 = (int64_t)batch * dim / 4;
  cnf_probe_kernel<<<ew_grid(n4), 256, 0, s>>>(
      reinterpret_cast<const float4*>(x), H(P.xh), H(P.xl), reinterpret_cast<float4*>(ws + P.eps), H(P.uh), H(P.ul),
      seed_dev, ordinal_dev, ordinal_offset, estimator, dim / 4, n4);
  note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());

  const int64_t boff[4] = {h.off_b0, h.off_b1, h.off_b2, h.off_b3};
  const __half* ph = x ? H(P.xh) : reinterpret_cast<const __half*>(x_hi);
  const __half* pl = x ? H(P.xl) : reinterpret_cast<const __half*>(x_lo);
  const __half* th = H(P.uh);
  const __half* tl = H(P.ul);
  float* dact = reinterpret_cast<float*>(ws + P.dact);
  int rc;
  for (int l = 0; l < 4; ++l) {
    const int K = l ? w : dim, n1 = l < 3 ? w : dim;
    const __half* wh = reinterpret_cast<const __half*>(W.wh[l]);
    const __half* wl = reinterpret_cast<const __half*>(W.wl[l]);
    __half* oph = H(l & 1 ? P.bh : P.ah);
    __half* opl = H(l & 1 ? P.bl : P.al);
    __half* oth = H(l & 1 ? P.sh : P.th);
    __half* otl = H(l & 1 ? P.sl : P.tl);
    CnfPrimalEpi pe;
    pe.bias = F(boff[l]); pe.inv_ws = W.inv_ws[l]; pe.tcol = l == 0 ? F(h.off_w0t) : nullptr; pe.t_dev = t_dev;
    pe.act = l < 3 ? act : -1; pe.dact = dact; pe.out_hi = oph; pe.out_lo = opl; pe.f = f; pe.ldo = n1; pe.t = 0.f;
    rc = launch_gemm_h3<CnfPrimalEpi, cnf_gemm_kernel<CnfPrimalEpi>>(ph, pl, batch, K, wh, wl, n1, W.ld[l], K, pe, s);
    if (rc != CFM_OK) return rc;
    CnfTangentEpi te;
    te.inv_ws = W.inv_ws[l]; te.dact = dact; te.out_hi = oth; te.out_lo = otl; te.ldo = n1;
    te.eps = l == 3 ? reinterpret_cast<const float*>(ws + P.eps) : nullptr;
    te.parts = reinterpret_cast<double*>(ws + P.parts); te.nchunk = P.nchunk;
    rc = launch_gemm_h3<CnfTangentEpi, cnf_gemm_kernel<CnfTangentEpi>>(th, tl, batch, K, wh, wl, n1, W.ld[l], K, te, s);
    if (rc != CFM_OK) return rc;
    ph = oph; pl = opl; th = oth; tl = otl;
  }
  cnf_fold_kernel<<<(batch + 255) / 256, 256, 0, s>>>(reinterpret_cast<const double*>(ws + P.parts), P.nchunk, div,
                                                       batch);
  note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}

extern "C" int cfm_cnf_tc_euler_init(cfm_cnf_tc_state* state, const float* z0, float* x, float* ll, void* x_hi,
                                     void* x_lo, float* traj, const float* t_span, int n_span, uint64_t seed,
                                     int batch, int dim, void* stream) {
  const char* what = "cfm_cnf_tc_euler_init";
  CFM_REQUIRE(state && z0 && x && ll && x_hi && x_lo && traj && t_span, "%s: null pointer", what);
  CFM_REQUIRE(n_span >= 2, "%s: n_span must be >= 2 (got %d)", what, n_span);
  if (const int rc = tc_state_shape(what, batch, dim)) return rc;
  CFM_REQUIRE(aligned16(x) && aligned16(x_hi) && aligned16(x_lo) && (reinterpret_cast<uintptr_t>(state) & 7) == 0,
              "%s: x, x_hi and x_lo must be 16-byte aligned, the state 8-byte aligned", what);
  const int64_t n4 = (int64_t)batch * dim / 4;
  cnf_euler_init_kernel<<<ew_grid((int64_t)batch * (dim + 1)), 256, 0, (cudaStream_t)stream>>>(
      state, z0, reinterpret_cast<float4*>(x), ll, reinterpret_cast<__half*>(x_hi), reinterpret_cast<__half*>(x_lo),
      traj, t_span, n_span - 1, seed, dim / 4, n4, batch);
  note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}

extern "C" int cfm_cnf_tc_euler_step(cfm_cnf_tc_state* state, float* x, float* ll, const float* f, const float* div,
                                     void* x_hi, void* x_lo, int batch, int dim, void* stream) {
  const char* what = "cfm_cnf_tc_euler_step";
  CFM_REQUIRE(state && x && ll && f && div && x_hi && x_lo, "%s: null pointer", what);
  if (const int rc = tc_state_shape(what, batch, dim)) return rc;
  CFM_REQUIRE(aligned16(x) && aligned16(f) && aligned16(x_hi) && aligned16(x_lo) &&
                  (reinterpret_cast<uintptr_t>(state) & 7) == 0,
              "%s: x, f, x_hi and x_lo must be 16-byte aligned, the state 8-byte aligned", what);
  const int64_t n4 = (int64_t)batch * dim / 4;
  cnf_euler_step_kernel<<<ew_grid(n4), 256, 0, (cudaStream_t)stream>>>(
      state, reinterpret_cast<float4*>(x), ll, reinterpret_cast<const float4*>(f), div,
      reinterpret_cast<__half*>(x_hi), reinterpret_cast<__half*>(x_lo), dim / 4, n4, batch);
  note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}
