// Sinkhorn V2: smem-staged fused sweep fed by bulk async copies (fast fp32 mode, n1 <= 8192,
// 16-byte aligned rows).  Same algorithm and outputs as sinkhorn.cu (POT sinkhorn_log, reference
// call site torchcfm/optimal_transport.py:87); different data movement:
//
//   * the CTA's row slab is streamed, R rows per stage, into an S-stage shared-memory ring with
//     cp.async.bulk (one contiguous 4*n1-byte copy per row, mbarrier complete_tx).  Thread 0 issues
//     the refill of a stage right after the per-chunk block barrier that proves every warp has
//     finished reading it, so the ring stays S chunks ahead -- across the grid barriers too (the
//     copies for the next sweep are already in flight while the column partials are combined).
//   * all 16 warps are consumers.  Thread t owns the same 4*KG columns in both phases, so v_j and the
//     running column accumulators live in registers for the whole sweep.  Per stage:
//       row phase   x = M*c2 + v_j for its columns -> warp max -> sum ex2 -> 16 per-warp partials
//                   -> one named barrier -> every warp folds the 16 partials -> u_r
//       column phase  re-reads the same smem rows, x = M*c2 + u_r, accumulates into (cm, cs)
//                   with a lazily updated reference maximum (rescale only when x > cm + 40)
//     so each element of M costs one HBM read, two smem reads and two ex2 per iteration.
//   * FACTORED path (taken on the device when span = max|M/reg|*log2(e) <= 40, the regime where
//     kernel-space Sinkhorn is finite, e.g. BASELINE config 2): E_ij = ex2(M_ij*c2 - kappa) is
//     formed ONCE per element into registers; the row phase is s_r += E*V_j with V_j = ex2(v_j - vref)
//     and the column phase c_j += E*U_r with U_r = ex2(u_r - uref): 4 instructions and ONE ex2 per
//     element per iteration instead of ~11 and two, and the smem stage is released as soon as it
//     has been read.  Ranges are safe by construction: LSE is 1-Lipschitz, so the spreads of u and
//     v are <= span and every product stays within 2^(+-3*span) << 2^127.
//   * 3-BYTE COST STREAM (factored path, when fp32 M does not fit in the L2; status[3] = 4): the factored
//     sweep only uses M through the exponent e = M*c2 - kappa in [0, span], so after the prologue it reads a
//     fixed-point copy of e instead of M: q = rint(e / a), a = fl32(span / (2^23 - 1)), 3 bytes per element
//     (12-byte groups of 4 columns, rows of ldc = align16(3*n1) bytes in the workspace).  The prologue sweep
//     still reads fp32 rows and writes the copy (float64 encode, once per solve); iterations decode with no
//     conversion instruction: the bit pattern 0x4B000000 | q is the float 2^23 + q, so e' = fmaf(F, a, -2^23 a)
//     = fl(q*a) exactly up to the final rounding.  |e' - e| <= a/2 + ulp = span * 2^-24 + ulp; 25% fewer bytes.
//     The 3-byte chunk (R rows of ldc bytes) is a quarter of the fp32 stage or less, so once the prologue has drained
//     its fp32 ring the same allocation is re-carved into a kV2QStages-deep ring of 3-byte chunks and as many
//     chunks resident for the whole solve as fit in the rest: a run of kres slab chunks in the middle of the slab,
//     filled once, read from shared memory by every later sweep.  Only the other chunks cross the ring (and HBM).
//   * 22-BIT CHUNKS (KG = 4, where the NT * 44-byte row is shorter than ldc): q = 0 at the largest cost and grows as
//     the cost falls, so a chunk whose smallest cost encodes below 2^22 never uses the top bit.  The prologue decides
//     that per chunk (the encode is monotone in M) and writes such a chunk with thread t's 16 entries packed into the
//     11 words at word 11 t of the row.  Same q, so the same e' and bit-identical results; 8% fewer bytes, and a slab
//     whose chunks are all narrow re-carves at the narrow pitch (one more resident chunk at C2).
//   * per-CTA column partials -> [cta][n1] workspace -> grid barrier -> sliced combine -> v_new,
//     marginal error -> grid barrier (identical to sinkhorn.cu).
#include <stdlib.h>

#include <algorithm>
#include <type_traits>

#include "sinkhorn_common.cuh"

namespace cfm {

// NT = threads per CTA: 512, one CTA per SM

__device__ __forceinline__ uint32_t v2_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void v2_mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(v2_smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void v2_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(v2_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void v2_mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(v2_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void v2_mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t"
      "}\n" ::"r"(v2_smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void v2_bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(v2_smem_u32(dst)), "l"(src), "r"(bytes), "r"(v2_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void v2_bulk_load_hint(void* dst, const void* src, uint32_t bytes, uint64_t* bar,
                                                  uint64_t policy) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               ::"r"(v2_smem_u32(dst)), "l"(src), "r"(bytes), "r"(v2_smem_u32(bar)), "l"(policy) : "memory");
}
__device__ __forceinline__ uint64_t v2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t v2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
template <int NT>
__device__ __forceinline__ void v2_consumer_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(NT) : "memory"); }
__device__ __forceinline__ unsigned long long v2_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// 3-byte stream: e = m*c2 - kappa in float64 (exact: a 24 x 24-bit product), quantised with one rounding and
// clamped to [0, 2^23 - 1] (at m = cost_max the fp32 kappa may put e a rounding below 0; NaN -> 0, but a NaN cost
// has already made the prologue's column potential NaN, and that reaches every potential as on the fp32 path)
__device__ __forceinline__ uint32_t v2_encode(float m, float c2, float kappa, double qinv) {
  const double e = (double)m * (double)c2 - (double)kappa;
  return (uint32_t)fmin(fmax(rint(e * qinv), 0.0), 8388607.0);
}
// e' = fl(q * qa) of the entry in the low 24 bits of w: the bit pattern 0x4B000000 | q is the float 2^23 + q (q < 2^23:
// byte 2 of an entry has its top bit clear), so subtracting 2^23 is exact and no conversion instruction is needed
__device__ __forceinline__ float v2_q_decode(uint32_t w, float qa) {
  return (__uint_as_float(0x4B000000u | (w & 0xFFFFFFu)) - 8388608.f) * qa;
}
// the same for a 22-bit entry in the low bits of w (the same float for the same q)
__device__ __forceinline__ float v2_q22_decode(uint32_t w, float qa) {
  return (__uint_as_float(0x4B000000u | (w & 0x3FFFFFu)) - 8388608.f) * qa;
}
// 22-bit chunks: a thread's 16 entries of a row (4 groups of 4 columns, in column order) fill 11 words, entry i at
// bit 22 i; the odd stride of 11 words between threads keeps the word loads free of bank conflicts
constexpr int kV2NarrowWords = 11;
constexpr uint32_t kV2NarrowRow = 512 * 4 * kV2NarrowWords;  // bytes of a 22-bit row (KG = 4: 512 threads)
constexpr uint32_t kV2NarrowLimit = 1u << 22;
// entry i of a thread's 11 words w (i is a constant once the callers' loops are unrolled)
__device__ __forceinline__ uint32_t v2_q22_field(const uint32_t* w, int i) {
  const int bit = 22 * i, wd = bit >> 5, sh = bit & 31;
  return sh + 22 <= 32 ? w[wd] >> sh : __funnelshift_r(w[wd], w[wd + 1], sh);
}
// chunks of a slab whose width the per-CTA mask records; a longer slab's later chunks keep 3 bytes
constexpr int kV2MaskWords = 8;

// Reduce R per-lane values over the warp with a shared shuffle tree: at the stage with offset
// `off` lanes whose bit `off` is set keep the odd member of each pair, the others the even one, so
// R values cost R-1 + log2(32/R) shuffles instead of 5R.  On return v[0] holds, in EVERY lane, the
// warp total of row  multi_row(lane)  (the row's index bits are lane bits 4, 3, 2 for R = 2, 4, 8).
template <int R>
__device__ __forceinline__ void multi_reduce(float (&v)[R], int lane) {
  static_assert(R == 1 || R == 2 || R == 4 || R == 8, "R must be a power of two <= 8");
  int off = 16;
#pragma unroll
  for (int n = R; n > 1; n >>= 1) {
    const bool upper = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < n / 2; ++i) {
      const float a = v[2 * i], b = v[2 * i + 1];
      const float send = upper ? a : b, keep = upper ? b : a;
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
    off >>= 1;
  }
  for (; off > 0; off >>= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], off);
}
template <int R>
__device__ __forceinline__ int multi_row(int lane) {
  int r = 0, bit = 4;
#pragma unroll
  for (int n = R, sh = 0; n > 1; n >>= 1, ++sh, --bit) r |= ((lane >> bit) & 1) << sh;
  return r;
}

// CTAs the combine step reduces in one round trip (19 partials per lane; no sm_90 part has more SMs)
constexpr int kV2MaxGrid = 152;

// Ring depth of the 3-byte stream: 2 stages leave room for 2 resident chunks at full width (3 when every chunk of the
// slab is narrow).  3 stages with 1 resident chunk gave a slower C2 step and 4096^2 shard (DESIGN.md §3.2).
constexpr int kV2QStages = 2;
// Head of the dynamic shared memory, the same in every layout: the row partials [2][R][16] and the mbarriers (8 for
// the fp32 ring, kV2QStages for the 3-byte ring, 1 for the resident chunks).  The stages follow it.
template <int NT, int R>
constexpr uint32_t v2_head_bytes() {
  return (2 * R * (NT / 32) * sizeof(float2) + (8 + kV2QStages + 1) * sizeof(uint64_t) + 127) / 128 * 128;
}

// S: depth of the fp32 ring.  qbytes: dynamic shared memory past the head, which the 3-byte stream re-carves into
// its ring and resident chunks.
template <int NT, int KG, int R>
__global__ void __launch_bounds__(NT, 1) sinkhorn_v2_kernel(const SkParams p, int S, const int qbytes) {
  constexpr int kV2Consumers = NT, kV2Warps = NT / 32;
  extern __shared__ __align__(128) unsigned char v2_smem[];
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nblk = gridDim.x, b = blockIdx.x;
  const int n0 = p.n0, n1 = p.n1, n1p = p.n1p, ng = n1p / 4;

  // auto mode: the float64 case goes to sinkhorn.cu's kernel, launched behind this one (uniform over the grid:
  // nobody reaches a grid barrier)
  if (p.precise < 0 && sk_needs_f64(p.cost_max ? __ldg(p.cost_max) : 0.f, p.normalize, p.reg)) return;

  const uint32_t stage_floats = (uint32_t)R * (uint32_t)n1p;
  float2* rowpart = reinterpret_cast<float2*>(v2_smem);  // [2][R][16]
  uint64_t* const bars = reinterpret_cast<uint64_t*>(rowpart + 2 * R * kV2Warps);
  uint64_t* full = bars;  // the ring's mbarriers: bars[0, 8) for the fp32 ring, bars[8, 8 + kV2QStages) for the 3-byte one
  uint64_t* const res_full = bars + 8 + kV2QStages;  // the resident chunks' fill
  float* stages = reinterpret_cast<float*>(v2_smem + v2_head_bytes<NT, R>());
  __shared__ double red[kV2Warps];
  __shared__ int cslice[2];  // this CTA's columns in the combine step (in smem: a register there would spill)
  // 22-bit chunks: bit c of the mask = slab chunk c of the copy is narrow (set by the prologue).  qmode, fixed for
  // the CTA after the prologue: 0 no narrow chunk (the 3-byte stream as it was), 1 every chunk narrow (stages and
  // resident chunks at the narrow pitch), 2 mixed (the 3-byte pitch, width looked up per chunk)
  __shared__ uint32_t nmask[KG == 4 ? kV2MaskWords : 1];
  __shared__ int qmode;

  if (tid == 0) {
    const int cpc = (n1 + nblk - 1) / nblk;
    cslice[0] = b * cpc;
    cslice[1] = min(n1, b * cpc + cpc);
    for (int w = 0; w < (KG == 4 ? kV2MaskWords : 1); ++w) nmask[w] = 0u;
    for (int s = 0; s < 8 + kV2QStages + 1; ++s) v2_mbar_init(&bars[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  float* u_work = reinterpret_cast<float*>(p.u_work);
  float* v_work[2] = {reinterpret_cast<float*>(p.v_work[0]), reinterpret_cast<float*>(p.v_work[1])};
  float* part_m = reinterpret_cast<float*>(p.part_m);
  float* part_s = reinterpret_cast<float*>(p.part_s);

  const float cmaxv = p.cost_max ? __ldg(p.cost_max) : 1.f;
  const float c2 = -kLog2e / (p.reg * (p.normalize ? cmaxv : 1.f));
  const float loga = -log2f((float)n0), logb = -log2f((float)n1);
  const float kappa = c2 * cmaxv;  // = min_ij M_ij*c2 (most negative exponent), so E = ex2(M*c2 - kappa) >= 1
  const bool fact = (p.cost_max != nullptr) && (-kappa <= 40.f);  // span in log2 units
  // 3-byte stream of the factored exponent (every sweep after the prologue; row pitch p.ldc bytes).  Its quantum
  // and pitch are formed where they are used: long-lived values cost registers in the combine step.
  const bool compact = fact && p.mq != nullptr;

  const SkSlab slab = sk_slab(n0, nblk, b);
  const int r_begin = slab.begin, nrows = slab.end - slab.begin;
  const int nchunks = (nrows + R - 1) / R;

  // ---- ring bookkeeping (incremental: no 64-bit div/mod in the hot loop) ----
  // chunk sequence q = 0,1,2,... over ALL sweeps; chunk q sits in stage q % S.  Slab chunks rlo .. rlo+kres-1 are
  // resident in smem (3-byte stream only, kres = 0 before it) and take no part in the sequence.
  int kres = 0, rlo = 0;
  int c_st = 0;             // consumers: stage of the next chunk to consume
  uint32_t c_par = 0;       //            parity to wait for on full[c_st]
  int p_st = 0, p_chunk = 0;  // producer (thread 0): stage / slab chunk of the next chunk to issue
  int p_dir = 1;              // sweeps alternate direction (boustrophedon): the rows a sweep ends on are
                              // the rows the next one starts on, and those are still resident in L2
  int sweep_no = 0;
  long long issued = 0, consumed_total = 0;
  bool gvalid[KG];
#pragma unroll
  for (int k = 0; k < KG; ++k) gvalid[k] = (tid + kV2Consumers * k) < ng;
  const int tcol = tid * 4;  // first owned column; group k adds 2048*k
  const bool full_cols = ng == kV2Consumers * KG;  // every thread owns KG valid float4 groups

  // L2 residency: the streamed chunks of every slab below `l2_end` are loaded evict_last (they stay in the
  // L2 from sweep to sweep), the rest evict_first (pure streaming): only the streaming part
  // crosses HBM every iteration.  p.l2_resident_frac <= 0 leaves the default policy.
  // The 3-byte stream keeps the same L2-resident BYTES (more chunks of the smaller rows) in the chunks that follow
  // the smem-resident ones; its fp32 prologue is read once and streams entirely.
  // (`l2_end` switches to the 3-byte stream's value when the producer switches format, see below)
  int l2_end = p.l2_resident_frac <= 0.f ? -1 : compact ? 0 : (int)(p.l2_resident_frac * (float)nchunks);
  // slab chunk c of the copy has 22-bit entries (uniform over the CTA)
  auto chunk_narrow = [&](int c) {
    if constexpr (KG == 4) return c < 32 * kV2MaskWords && ((nmask[c >> 5] >> (c & 31)) & 1u) != 0;
    else return false;
  };
  // thread 0: issue the bulk copies of the next chunk into its (free) stage (MODE: the CTA's qmode)
  auto issue_next = [&](auto MODE) {
    constexpr int kMode = decltype(MODE)::value;
    const int r0 = r_begin + p_chunk * R;
    const int rv = min(R, r_begin + nrows - r0);
    const bool q = compact && issued >= nchunks;  // the first nchunks chunks are the prologue's
    const uint32_t ldc = (uint32_t)p.ldc;
    const uint32_t qrow = kMode == 1 ? kV2NarrowRow : kMode == 2 && chunk_narrow(p_chunk) ? kV2NarrowRow : ldc;
    const uint32_t row_bytes = q ? qrow : (uint32_t)n1 * 4u;
    const uint32_t pitch = q ? (kMode == 1 ? kV2NarrowRow : ldc) : (uint32_t)n1p * 4u;  // a stage: R rows at this pitch
    const uint64_t pol = p_chunk < l2_end ? v2_policy_evict_last() : v2_policy_evict_first();
    v2_mbar_expect_tx(&full[p_st], (uint32_t)rv * row_bytes);
    for (int r = 0; r < rv; ++r) {
      unsigned char* dst = reinterpret_cast<unsigned char*>(stages) + ((size_t)p_st * R + r) * pitch;
      const void* src = q ? static_cast<const void*>(p.mq + (int64_t)(r0 + r) * ldc)
                          : static_cast<const void*>(p.M + (int64_t)(r0 + r) * p.ldm);
      if (l2_end < 0) v2_bulk_load(dst, src, row_bytes, &full[p_st]);
      else v2_bulk_load_hint(dst, src, row_bytes, &full[p_st], pol);
    }
    ++issued;
    p_chunk += p_dir;
    if (p_chunk >= rlo && p_chunk < rlo + kres) p_chunk = p_dir > 0 ? rlo + kres : rlo - 1;  // skip the resident run
    // at either end of the slab the next sweep runs the other way and starts with the chunk this one ended on
    if (p_chunk >= nchunks) { p_chunk = rlo + kres < nchunks ? nchunks - 1 : rlo - 1; p_dir = -1; }
    else if (p_chunk < 0) { p_chunk = rlo > 0 ? 0 : rlo + kres; p_dir = 1; }
    if (++p_st == S) p_st = 0;
  };
  // The ring runs S chunks ahead across sweeps, and the prologue's last S chunks are iteration 0's first: their
  // 3-byte rows are written after the point where the ring would issue their refills.  So no chunk of the 3-byte
  // stream is issued before the whole slab is encoded and fenced (one ring fill per solve, issued right after the
  // prologue); the copy is reused from call to call, and an early read would return the previous coupling's rows.
  auto may_issue = [&]() { return issued < nchunks || consumed_total != 0 || !compact; };
  if (tid == 0)
    for (int q = 0; q < S && may_issue(); ++q) issue_next(std::integral_constant<int, 0>{});  // initial fill (wraps into the next sweep if S > nchunks)

  // CFM_SK_TL (debug aid, scripts/sk_v2_timeline.py): %globaltimer marks of iteration 50 by thread 0: [0, 6) CTA 0
  // and [8, 14) the last CTA (sweep start, last chunk consumed, partials stored, barrier-1 exit, combine done,
  // barrier-2 exit), [16] / [17] the earliest / latest last-chunk mark of all CTAs (factored sweep only)
  unsigned long long* tl = p.tl;
  bool tl_now = false;
  auto tl_mark = [&](int slot) {
    if (!tl_now) return;
    const unsigned long long t = v2_globaltimer();
    if (slot == 1) { atomicMin(tl + 16, t); atomicMax(tl + 17, t); }
    if (b == 0 || b == nblk - 1) tl[(b == 0 ? 0 : 8) + slot] = t;
  };

  // ---- one fused sweep ----
  auto sweep = [&](bool do_row, bool do_col, const float* v_cur) {
    if (fact) {
      // ---------------- factored (kernel-space in registers) sweep ----------------
      const float vref = do_row ? __ldcg(v_cur) : 0.f;
      const float nkap = -kappa;
      float4 V[KG];
      float cs[KG][4];
#pragma unroll
      for (int k = 0; k < KG; ++k) {
        V[k] = make_float4(0.f, 0.f, 0.f, 0.f);  // idle columns: weight 0
        if (gvalid[k]) {
          if (do_row) {
            const float4 vv = __ldcg(reinterpret_cast<const float4*>(v_cur + tcol + kV2Consumers * 4 * k));
            V[k] = make_float4(ex2f(vv.x - vref), ex2f(vv.y - vref), ex2f(vv.z - vref), ex2f(vv.w - vref));
          } else {
            V[k] = make_float4(1.f, 1.f, 1.f, 1.f);
          }
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) cs[k][c] = 0.f;
      }
      float uref = 0.f;
      bool have_uref = !do_row;  // prologue: u = 0 everywhere, U = 1
      // stage format: 0 fp32 rows, 1 fp32 rows that are also encoded into the 3-byte copy, 2 the 3-byte copy
      const int fmt = !compact ? 0 : sweep_no == 0 ? 1 : 2;
      const uint32_t ldc = (uint32_t)p.ldc;
      // quantum span / (2^23 - 1) (span = 0: q = 0, e' = 0 = e) and encode scale; float64 divisions cost every
      // thread about as much as a small shape's sweep has to spare, so only the stream's sweeps form them
      const float qa = fmt != 0 ? (float)((double)(-kappa) / 8388607.0) : 0.f;
      const double qinv = fmt == 1 && qa > 0.f ? 1.0 / (double)qa : 0.0;
      // the chunk loop, compiled per qmode: mode 0 (every sweep before the stream, and a stream without narrow
      // chunks) has no width lookup and no 22-bit decode; modes 1 and 2 run only on the stream (fmt 2)
      auto chunk_loop = [&](auto MODE) {
      constexpr int kMode = decltype(MODE)::value;
      for (int cc = 0; cc < nchunks; ++cc) {
        const int chunk = (sweep_no & 1) ? nchunks - 1 - cc : cc;
        const int r0 = r_begin + chunk * R;
        const int rv = min(R, r_begin + nrows - r0);
        const bool res = (unsigned)(chunk - rlo) < (unsigned)kres;  // resident: slot S + chunk - rlo, past the ring
        const bool narrow = kMode == 1 || (kMode == 2 && chunk_narrow(chunk));
        const uint32_t qp = kMode == 1 ? kV2NarrowRow : ldc;  // row pitch of the copy's chunks in shared memory
        const float* sbase = stages + (uint32_t)c_st * stage_floats + tcol;
        const unsigned char* qbase = reinterpret_cast<const unsigned char*>(stages) +
                                     (uint32_t)(res ? S + chunk - rlo : c_st) * R * qp +
                                     (narrow ? 4 * kV2NarrowWords : 12) * tid;
        float2* rp = rowpart + (cc & 1) * R * kV2Warps;
        if (res) v2_mbar_wait(res_full, 0);
        else v2_mbar_wait(&full[c_st], c_par);
        float4 E[R][KG];
        // E of every owned group of the stage; ALL: every thread owns KG valid groups of R rows (no predicates)
        auto form_E = [&](auto FMT, auto ALL) {
          constexpr int kFmt = decltype(FMT)::value;
          constexpr bool kAll = decltype(ALL)::value;
#pragma unroll
          for (int r = 0; r < R; ++r)
#pragma unroll
            for (int k = 0; k < KG; ++k) {
              if (!kAll) E[r][k] = make_float4(0.f, 0.f, 0.f, 0.f);
              if (kAll || (gvalid[k] && r < rv)) {
                if constexpr (kFmt == 3) {
                  // 22-bit chunk: the group's 4 entries of the thread's 11 words (entry 4k + c at bit 22 (4k + c))
                  const uint32_t* w = reinterpret_cast<const uint32_t*>(qbase + r * qp);
                  E[r][k] = make_float4(ex2f(v2_q22_decode(v2_q22_field(w, 4 * k), qa)),
                                        ex2f(v2_q22_decode(v2_q22_field(w, 4 * k + 1), qa)),
                                        ex2f(v2_q22_decode(v2_q22_field(w, 4 * k + 2), qa)),
                                        ex2f(v2_q22_decode(v2_q22_field(w, 4 * k + 3), qa)));
                } else if constexpr (kFmt == 2) {
                  // 12 bytes = 4 entries; three 4-byte smem loads at a stride of 3 words (no bank conflicts)
                  const uint32_t* w = reinterpret_cast<const uint32_t*>(qbase + r * qp + 12 * kV2Consumers * k);
                  const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
                  E[r][k] = make_float4(ex2f(v2_q_decode(w0, qa)),
                                        ex2f(v2_q_decode(__funnelshift_r(w0, w1, 24), qa)),
                                        ex2f(v2_q_decode(__funnelshift_r(w1, w2, 16), qa)),
                                        ex2f(v2_q_decode(w2 >> 8, qa)));
                } else {
                  const float4 mv = *reinterpret_cast<const float4*>(sbase + r * n1p + kV2Consumers * 4 * k);
                  E[r][k] = make_float4(ex2f(fmaf(mv.x, c2, nkap)), ex2f(fmaf(mv.y, c2, nkap)),
                                        ex2f(fmaf(mv.z, c2, nkap)), ex2f(fmaf(mv.w, c2, nkap)));
                }
              }
            }
        };
        bool enc_narrow = false;
        if constexpr (KG == 4 && kMode == 0) {
          if (fmt == 1 && p.ldn != 0 && chunk < 32 * kV2MaskWords &&
              (uint32_t)qbytes >= (uint32_t)S * stage_floats * 4u + (uint32_t)p.ldn) {
            // the chunk is narrow iff its largest code, the code of its smallest cost (the encode is monotone
            // non-increasing in M), is below 2^22 and no cost is NaN
            float mn = __int_as_float(0x7f800000);
            bool nan = false;
#pragma unroll 1
            for (int r = 0; r < rv; ++r)
#pragma unroll
              for (int k = 0; k < KG; ++k)
                if (gvalid[k]) {
                  const float4 mv = *reinterpret_cast<const float4*>(sbase + r * n1p + kV2Consumers * 4 * k);
                  mn = fminf(mn, fminf(fminf(mv.x, mv.y), fminf(mv.z, mv.w)));
                  nan |= (mv.x != mv.x) | (mv.y != mv.y) | (mv.z != mv.z) | (mv.w != mv.w);
                }
            enc_narrow = !__syncthreads_or(nan || v2_encode(mn, c2, kappa, qinv) >= kV2NarrowLimit);
            if (enc_narrow && tid == 0) nmask[chunk >> 5] |= 1u << (chunk & 31);
          }
        }
        if (enc_narrow) {
          // prologue, 22-bit chunk: thread t's 16 entries of a row into the 11 words at word 11 t (entry i at bit
          // 22 i; idle groups write 0, so the whole NT * 44-byte row the stream copies is defined).  The row is
          // packed in shared memory past the fp32 ring and then stored with 16-byte coalesced writes: stored from
          // registers, each warp store would touch 44 sectors 4 bytes at a time.
          uint32_t* stg = reinterpret_cast<uint32_t*>(stages + (uint32_t)S * stage_floats);
#pragma unroll 1
          for (int r = 0; r < rv; ++r) {
            uint32_t* dst = stg + kV2NarrowWords * tid;
            uint32_t acc = 0u;  // the bits of the word being filled
#pragma unroll
            for (int k = 0; k < KG; ++k) {
              uint32_t q[4] = {0u, 0u, 0u, 0u};
              if (gvalid[k]) {
                const float4 mv = *reinterpret_cast<const float4*>(sbase + r * n1p + kV2Consumers * 4 * k);
                q[0] = v2_encode(mv.x, c2, kappa, qinv); q[1] = v2_encode(mv.y, c2, kappa, qinv);
                q[2] = v2_encode(mv.z, c2, kappa, qinv); q[3] = v2_encode(mv.w, c2, kappa, qinv);
              }
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                const int bit = 22 * (4 * k + c), sh = bit & 31;
                acc |= q[c] << sh;
                if (sh + 22 >= 32) {
                  dst[bit >> 5] = acc;
                  acc = sh + 22 > 32 ? q[c] >> (32 - sh) : 0u;
                }
              }
            }
            v2_consumer_barrier<NT>();
            const uint4* src4 = reinterpret_cast<const uint4*>(stg);
            uint4* row4 = reinterpret_cast<uint4*>(p.mq + (int64_t)(r0 + r) * ldc);
            for (int i = tid; i < p.ldn / 16; i += NT) row4[i] = src4[i];
            v2_consumer_barrier<NT>();  // the next row reuses the staging words
          }
        } else if (kMode == 0 && fmt == 1) {
          // prologue: write this stage's rows into the 3-byte copy (its own pass: E is not live yet)
#pragma unroll 1
          for (int r = 0; r < rv; ++r)
#pragma unroll
            for (int k = 0; k < KG; ++k)
              if (gvalid[k]) {
                const float4 mv = *reinterpret_cast<const float4*>(sbase + r * n1p + kV2Consumers * 4 * k);
                const uint32_t q0 = v2_encode(mv.x, c2, kappa, qinv), q1 = v2_encode(mv.y, c2, kappa, qinv);
                const uint32_t q2 = v2_encode(mv.z, c2, kappa, qinv), q3 = v2_encode(mv.w, c2, kappa, qinv);
                uint32_t* dst = reinterpret_cast<uint32_t*>(p.mq + (int64_t)(r0 + r) * ldc + 12 * (tid + kV2Consumers * k));
                dst[0] = q0 | (q1 << 24);
                dst[1] = (q1 >> 8) | (q2 << 16);
                dst[2] = (q2 >> 16) | (q3 << 8);
              }
        }
        using kT = std::true_type;
        using kF = std::false_type;
        const bool all = full_cols && rv == R;  // common case: no predicates in the hot loop
        if constexpr (kMode != 0) {
          if (narrow) { if (all) form_E(std::integral_constant<int, 3>{}, kT{}); else form_E(std::integral_constant<int, 3>{}, kF{}); }
          else if constexpr (kMode == 2) { if (all) form_E(std::integral_constant<int, 2>{}, kT{}); else form_E(std::integral_constant<int, 2>{}, kF{}); }
        } else if (fmt == 2) { if (all) form_E(std::integral_constant<int, 2>{}, kT{}); else form_E(std::integral_constant<int, 2>{}, kF{}); }
        else { if (all) form_E(std::integral_constant<int, 0>{}, kT{}); else form_E(std::integral_constant<int, 0>{}, kF{}); }
        if (!res && ++c_st == S) { c_st = 0; c_par ^= 1u; }
        if (do_row) {
          float sr[R];
#pragma unroll
          for (int r = 0; r < R; ++r) {
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < KG; ++k) {
              s = fmaf(E[r][k].x, V[k].x, s); s = fmaf(E[r][k].y, V[k].y, s);
              s = fmaf(E[r][k].z, V[k].z, s); s = fmaf(E[r][k].w, V[k].w, s);
            }
            sr[r] = s;
          }
          multi_reduce<R>(sr, lane);  // lane L now holds the warp total of row multi_row<R>(L)
          if ((lane & (32 / R - 1)) == 0) rp[multi_row<R>(lane) * kV2Warps + warp] = make_float2(sr[0], 0.f);
        }
        // every warp has now copied its part of the stage into registers: after this barrier the
        // stage is free, so thread 0 refills it with the chunk S positions ahead
        v2_consumer_barrier<NT>();
        if (tid == 0 && !res && may_issue()) issue_next(MODE);
        float U[R];
        if (do_row) {
          // fold the 16 per-warp partials: lanes 0-15 take row r, lanes 16-31 row r+1 (one tree for two rows)
#pragma unroll
          for (int rr = 0; rr < R; rr += 2) {
            const int myrow = rr + (lane >> 4);
            float pr = ((R == 1 && lane >= 16) || (lane & 15) >= kV2Warps)
                           ? 0.f : rp[(R == 1 ? 0 : myrow) * kV2Warps + (lane & 15)].x;
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) pr += __shfl_xor_sync(0xffffffffu, pr, o);
            float Srow[2];
            Srow[0] = __shfl_sync(0xffffffffu, pr, 0);
            Srow[1] = __shfl_sync(0xffffffffu, pr, 16);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = rr + h;
              if (r < R) {
                // lse_r = kappa + vref + log2(S_r); a NaN row sum (NaN cost) stays NaN: lg2_abs would read its bits
                // as 1.5 * 2^128 and give every row the same finite u
                const float S = Srow[h];
                const float u2 = loga - (kappa + vref + (S == S ? lg2_abs(S) : S));
                if (!have_uref) { uref = u2; have_uref = true; }         // first row of the slab fixes uref
                U[r] = r < rv ? ex2f(u2 - uref) : 0.f;  // padding rows: E = 0 and U = 0 (never 0*inf)
                if (warp == 0 && lane == 0 && r < rv) {
                  u_work[r0 + r] = u2;
                  p.log_u[r0 + r] = (double)u2 * kLn2d;
                }
              }
            }
          }
        } else {
#pragma unroll
          for (int r = 0; r < R; ++r) U[r] = 1.f;
        }
        if (do_col) {
#pragma unroll
          for (int r = 0; r < R; ++r)
#pragma unroll
            for (int k = 0; k < KG; ++k) {
              cs[k][0] = fmaf(E[r][k].x, U[r], cs[k][0]); cs[k][1] = fmaf(E[r][k].y, U[r], cs[k][1]);
              cs[k][2] = fmaf(E[r][k].z, U[r], cs[k][2]); cs[k][3] = fmaf(E[r][k].w, U[r], cs[k][3]);
            }
        }
      }
      };
      if constexpr (KG == 4) {
        const int qm = fmt == 2 ? qmode : 0;
        if (qm == 1) chunk_loop(std::integral_constant<int, 1>{});
        else if (qm == 2) chunk_loop(std::integral_constant<int, 2>{});
        else chunk_loop(std::integral_constant<int, 0>{});
      } else {
        chunk_loop(std::integral_constant<int, 0>{});
      }
      tl_mark(1);
      consumed_total += nchunks - kres;
      ++sweep_no;
      if (do_col) {
        // sum_i ex2(M c2 + u_i) over this slab = cs * 2^(kappa + uref): partial (max, sum) form
        const float pm = kappa + uref;
#pragma unroll
        for (int k = 0; k < KG; ++k)
          if (gvalid[k]) {
            *reinterpret_cast<float4*>(part_m + (int64_t)b * n1p + tcol + kV2Consumers * 4 * k) =
                make_float4(pm, pm, pm, pm);
            *reinterpret_cast<float4*>(part_s + (int64_t)b * n1p + tcol + kV2Consumers * 4 * k) =
                make_float4(cs[k][0], cs[k][1], cs[k][2], cs[k][3]);
          }
      }
      tl_mark(2);
      return;
    }
    // ---------------- log-domain sweep (span > 40): two smem reads per element ----------------
    float4 vreg[KG];
    float cm[KG][4], cs[KG][4];
#pragma unroll
    for (int k = 0; k < KG; ++k) {
      vreg[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (do_row && gvalid[k]) {
        const float* vp = v_cur + tcol + kV2Consumers * 4 * k;  // written before the last grid barrier
        vreg[k] = make_float4(__ldcg(vp), __ldcg(vp + 1), __ldcg(vp + 2), __ldcg(vp + 3));
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) { cm[k][c] = -1.0e30f; cs[k][c] = 0.f; }
    }
    const float inf = __int_as_float(0x7f800000);
    for (int cc = 0; cc < nchunks; ++cc) {
      const int chunk = (sweep_no & 1) ? nchunks - 1 - cc : cc;
      const int r0 = r_begin + chunk * R;
      const int rv = min(R, r_begin + nrows - r0);
      const float* sbase = stages + (uint32_t)c_st * stage_floats + tcol;
      float2* rp = rowpart + (cc & 1) * R * kV2Warps;
      v2_mbar_wait(&full[c_st], c_par);
      if (++c_st == S) { c_st = 0; c_par ^= 1u; }
      float u2[R];
      if (do_row) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
          float x[KG][4];
          float tmax = -1.0e30f;
#pragma unroll
          for (int k = 0; k < KG; ++k) {
            float4 mv = make_float4(inf, inf, inf, inf);
            if (gvalid[k] && r < rv) mv = *reinterpret_cast<const float4*>(sbase + r * n1p + kV2Consumers * 4 * k);
            x[k][0] = fmaf(mv.x, c2, vreg[k].x); x[k][1] = fmaf(mv.y, c2, vreg[k].y);
            x[k][2] = fmaf(mv.z, c2, vreg[k].z); x[k][3] = fmaf(mv.w, c2, vreg[k].w);
            tmax = fmaxf(tmax, fmaxf(fmaxf(x[k][0], x[k][1]), fmaxf(x[k][2], x[k][3])));
          }
          const float wm = warp_max(tmax);
          float s = 0.f;
#pragma unroll
          for (int k = 0; k < KG; ++k)
            s += (ex2f(x[k][0] - wm) + ex2f(x[k][1] - wm)) + (ex2f(x[k][2] - wm) + ex2f(x[k][3] - wm));
          s = warp_sum(s);
          if (lane == 0) rp[r * kV2Warps + warp] = make_float2(wm, s);
        }
      }
      v2_consumer_barrier<NT>();
#pragma unroll
      for (int r = 0; r < R; ++r) {
        u2[r] = 0.f;
        if (do_row) {
          const float2 pr = lane < kV2Warps ? rp[r * kV2Warps + lane] : make_float2(-1.0e30f, 0.f);
          const float gm = warp_max(pr.x);
          const float gs = warp_sum(pr.y * ex2f(pr.x - gm));
          u2[r] = loga - (gm + log2f(gs));
          if (warp == 0 && lane == 0 && r < rv) {
            u_work[r0 + r] = u2[r];
            p.log_u[r0 + r] = (double)u2[r] * kLn2d;
          }
        }
      }
      if (do_col) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
          if (r < rv) {
#pragma unroll
            for (int k = 0; k < KG; ++k) {
              if (gvalid[k]) {
                const float4 mv = *reinterpret_cast<const float4*>(sbase + r * n1p + kV2Consumers * 4 * k);
                const float xv[4] = {fmaf(mv.x, c2, u2[r]), fmaf(mv.y, c2, u2[r]), fmaf(mv.z, c2, u2[r]),
                                     fmaf(mv.w, c2, u2[r])};
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                  if (xv[c] > cm[k][c] + 40.f) {  // rare: reference maximum lags by more than 2^40
                    cs[k][c] *= ex2f(cm[k][c] - xv[c]);
                    cm[k][c] = xv[c];
                  }
                  cs[k][c] += ex2f(xv[c] - cm[k][c]);
                }
              }
            }
          }
        }
      }
      // the stage is read again by the column phase: it is free only once every warp is past this
      // point, which the NEXT chunk's barrier (or the one below for the last chunk) certifies
      v2_consumer_barrier<NT>();
      if (tid == 0) issue_next(std::integral_constant<int, 0>{});
    }
    consumed_total += nchunks;
    ++sweep_no;
    if (do_col) {
#pragma unroll
      for (int k = 0; k < KG; ++k)
        if (gvalid[k]) {
          *reinterpret_cast<float4*>(part_m + (int64_t)b * n1p + tcol + kV2Consumers * 4 * k) =
              make_float4(cm[k][0], cm[k][1], cm[k][2], cm[k][3]);
          *reinterpret_cast<float4*>(part_s + (int64_t)b * n1p + tcol + kV2Consumers * 4 * k) =
              make_float4(cs[k][0], cs[k][1], cs[k][2], cs[k][3]);
        }
    }
  };

  // ---- combine a slice of columns over all CTAs' partials ----
  // 64 columns per pass.  Thread t reduces column t % 64 over the CTAs c = t / 64 (mod 8), so each load of a warp is
  // 32 consecutive floats of one CTA's partial row (four full sectors; with 8 CTAs per warp load it was 8 sectors of
  // 16 useful bytes each).  The 8 (max, sum) pairs of a column then meet in smem, and thread 8k folds those of column
  // k in the order of a shuffle butterfly over 8 lanes, the order used when 8 lanes of a warp shared a column.
  static_assert(NT == 512, "the combine maps 512 threads onto 64 columns x 8 CTA residues");
  __shared__ float2 cpart[8][64];
  // v_cur not null: the column-marginal error of (u, v_cur) goes to *err_slot
  auto combine = [&](const float* v_cur, float* v_new, double* err_slot) {
    const bool have_cur = v_cur != nullptr;
    double err_local = 0.0;
    const int c_begin = cslice[0], c_end = cslice[1];
    const int sub = tid >> 6;
    for (int j0 = c_begin; j0 < c_end; j0 += 64) {
      const int j = j0 + (tid & 63);
      const bool act = j < c_end;
      float m = -1.0e30f, s = 0.f;
      if (act) {
        // every lane loads ALL its <= kV2MaxGrid / 8 (max, sum) pairs before it reduces: ONE L2 round trip per column
        // instead of three dependent ones (the combine sits between the two grid barriers: its latency is fixed cost
        // per iteration)
        float mm[kV2MaxGrid / 8], ss[kV2MaxGrid / 8];
#pragma unroll
        for (int q = 0; q < kV2MaxGrid / 8; ++q) {
          const int c = sub + q * 8;
          if (c < nblk) {
            mm[q] = __ldcg(part_m + (int64_t)c * n1p + j);
            ss[q] = __ldcg(part_s + (int64_t)c * n1p + j);
          } else { mm[q] = -1.0e30f; ss[q] = 0.f; }
        }
        float bm = m;
#pragma unroll
        for (int q = 0; q < kV2MaxGrid / 8; ++q) bm = fmaxf(bm, mm[q]);
        float acc = 0.f;
#pragma unroll
        for (int q = 0; q < kV2MaxGrid / 8; ++q) acc += ss[q] * ex2f(mm[q] - bm);
        s = acc; m = bm;
      }
      cpart[sub][tid & 63] = make_float2(m, s);
      const int jf = j0 + (tid >> 3);  // the column this thread folds when tid % 8 == 0
      const bool fold = (tid & 7) == 0 && jf < c_end;
      const float vc = fold && have_cur ? __ldcg(v_cur + jf) : 0.f;
      __syncthreads();
      if (fold) {
        float mv[8], a[8];
#pragma unroll
        for (int l = 0; l < 8; ++l) mv[l] = cpart[l][tid >> 3].x;
        float gm = mv[0];
#pragma unroll
        for (int l = 1; l < 8; ++l) gm = fmaxf(gm, mv[l]);
#pragma unroll
        for (int l = 0; l < 8; ++l) a[l] = __fmul_rn(cpart[l][tid >> 3].y, ex2f(mv[l] - gm));  // no FMA into the sums
        const float gs = ((a[0] + a[4]) + (a[2] + a[6])) + ((a[1] + a[5]) + (a[3] + a[7]));
        const float vn = logb - (gm + log2f(gs));
        v_new[jf] = vn;
        if (have_cur) {
          const double d = ((double)vc - (double)vn) * kLn2d;
          const double e = expm1(d) / (double)n1;
          err_local += e * e;
        }
      }
      if (j0 + 64 < c_end) __syncthreads();  // cpart is rewritten by the next pass (after the last, a grid barrier follows)
    }
    if (have_cur) sk_err_add(err_local, err_slot, red);
  };

  // ---- prologue: v^0 from u = 0 ----
  sk_ring_init(p);
  if (p.timeline && b == 0 && tid == 0) { tl[16] = ~0ull; tl[17] = 0ull; }

  SkLoop L;
  sweep(false, true, nullptr);
  if (compact) {
    // the 3-byte rows were written through the generic proxy; the bulk copies read them through the async
    // proxy.  Each slab is written and read by its own CTA only, so a CTA barrier suffices.
    asm volatile("fence.proxy.async.global;" ::: "memory");
    // (the narrow rows' staging words are shared memory the re-carved ring's bulk copies overwrite)
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    // The fp32 ring is drained (no 3-byte chunk is issued before this point): re-carve its memory into the 3-byte
    // ring and the resident chunks behind it, each stage and chunk R rows of qp bytes.  The resident run sits in
    // the middle of the slab: there the ring's copies are in flight while the consumers read it, so HBM stays busy.
    // (At either end of a sweep the ring is already full, and every CTA would read its resident chunks at the same
    // time while HBM idles.)
    // A slab whose chunks are all narrow carves at the narrow row pitch (more resident chunks); otherwise every stage
    // and resident chunk keeps the 3-byte pitch and a narrow chunk fills the front of its rows.
    int n_narrow = 0;
    if constexpr (KG == 4)
      for (int w = 0; w < kV2MaskWords; ++w) n_narrow += __popc(nmask[w]);
    const uint32_t ldc = (uint32_t)p.ldc;
    const int qm = n_narrow == 0 ? 0 : n_narrow == nchunks ? 1 : 2;
    const uint32_t qp = qm == 1 ? kV2NarrowRow : ldc;
    S = kV2QStages;
    full = bars + 8;
    c_st = 0; c_par = 0; p_st = 0;
    kres = max(0, min(qbytes / (int)(R * qp) - kV2QStages, nchunks));
    rlo = (nchunks - kres) / 2;
    if (tid == 0) {
      qmode = qm;  // read by the sweeps after the grid barrier below
      if (kres > 0) {
        const int rows = min(nrows - rlo * R, kres * R);
        uint32_t bytes = 0;
        for (int r = 0; r < rows; ++r) bytes += chunk_narrow(rlo + r / R) ? kV2NarrowRow : ldc;
        v2_mbar_expect_tx(res_full, bytes);
        for (int r = 0; r < rows; ++r)
          v2_bulk_load(reinterpret_cast<unsigned char*>(stages) + ((size_t)S * R + r) * qp,
                       p.mq + (int64_t)(r_begin + rlo * R + r) * ldc,
                       chunk_narrow(rlo + r / R) ? kV2NarrowRow : ldc, res_full);
      }
      if (l2_end >= 0) {  // the first streamed chunks of the slab, as many as the fp32 share's bytes
        const int l2c = (int)(p.l2_resident_frac * (float)nchunks * (4.f * (float)n1) / (float)qp);
        l2_end = min(nchunks, l2c <= rlo ? l2c : l2c + kres);
      }
      if (kres < nchunks) {
        if (qm == 1) while (issued < consumed_total + S) issue_next(std::integral_constant<int, 1>{});
        else if (qm == 2) while (issued < consumed_total + S) issue_next(std::integral_constant<int, 2>{});
        else while (issued < consumed_total + S) issue_next(std::integral_constant<int, 0>{});
      }
    }
  }
  grid.sync();
  if constexpr (KG == 4)
    if (compact && tid == 0) {  // CTA 0 cleared the count (sk_ring_init) before the barrier above
      int n_narrow = 0;
      for (int w = 0; w < kV2MaskWords; ++w) n_narrow += __popc(nmask[w]);
      if (n_narrow) atomicAdd(p.n_narrow, n_narrow);
    }
  combine(nullptr, v_work[0], nullptr);
  grid.sync();

  for (int it = 0; it < p.max_iters; ++it) {
    const SkStep st = sk_step(p, it);
    tl_now = p.timeline && it == 50 && tid == 0;
    tl_mark(0);
    const int cur = it & 1;  // v_work[cur] holds the current v (every iteration that goes on flips it)
    sweep(true, st.do_col, v_work[cur]);
    L.iters = it + 1;
    if (!st.do_col) break;
    grid.sync();
    tl_mark(3);
    double* err_slot = sk_err_slot(p, it);
    combine(st.check ? v_work[cur] : nullptr, v_work[cur ^ 1], err_slot);
    tl_mark(4);
    grid.sync();
    tl_mark(5);
    if (st.check && sk_check_stops(L, p, it)) break;
    if (st.last) break;
  }

  // ---- drain speculative prefetches so no bulk copy is in flight when the CTA exits ----
  if (tid == 0) {
    for (long long q = consumed_total; q < issued; ++q) {
      v2_mbar_wait(&full[c_st], c_par);
      if (++c_st == S) { c_st = 0; c_par ^= 1u; }
    }
    if (kres > 0) v2_mbar_wait(res_full, 0);
  }

  // kernel variant: 4 = factored on the 3-byte stream, 3 = factored, 2 = log-domain
  sk_finish(p, L, v_work[(L.iters - 1) & 1], kLn2d, 0, compact ? 4 : fact ? 3 : 2);  // the iteration that stopped
}

template <int NT, int KG, int R>
static int v2_launch_t(SkParams& p, cudaStream_t s) {
  auto kern = sinkhorn_v2_kernel<NT, KG, R>;
  // dynamic shared memory: what a block may opt in to, less the kernel's static shared memory
  // (the static size is a property of the compiled kernel: queried once, it costs the small solves host time)
  static size_t static_smem = 0;
  if (static_smem == 0) {
    cudaFuncAttributes fa;
    CFM_CUDA_OK(cudaFuncGetAttributes(&fa, kern));
    static_smem = fa.sharedSizeBytes;
  }
  int dev = 0, optin = 0;
  CFM_CUDA_OK(cudaGetDevice(&dev));
  CFM_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const size_t head = v2_head_bytes<NT, R>();
  const size_t budget = (size_t)optin - static_smem;
  const size_t stage_bytes = (size_t)R * p.n1p * 4;
  if (budget < head + 2 * stage_bytes) return 1;
  int S = (int)((budget - head) / stage_bytes);
  if (S > 8) S = 8;
  int grid = sm_count();
  if (grid > p.n0) grid = p.n0;
  if (grid > kV2MaxGrid) return 1;  // more partials per column than the combine holds in registers
  // the 3-byte stream re-carves the prologue's ring into kV2QStages stages and as many resident chunks as fit (no
  // more than the longest slab has).  Where chunks may be narrow the kernel sizes the run from their widths, so it
  // gets the whole budget.
  size_t ring = (size_t)S * stage_bytes;
  if (p.ldn != 0) {
    ring = budget - head;
  } else if (p.mq != nullptr) {
    const size_t qchunk = (size_t)R * p.ldc;
    const int slab_chunks = ((p.n0 + grid - 1) / grid + R - 1) / R;
    const int kres_max = std::max(0, std::min(slab_chunks, (int)((budget - head) / qchunk) - kV2QStages));
    ring = std::max(ring, (size_t)(kV2QStages + kres_max) * qchunk);
  }
  const int qbytes = (int)ring;
  const size_t smem = ring + head;
  CFM_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  CFM_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, NT, smem));
  if (per_sm < 1) return 1;
  void* args[] = {(void*)&p, (void*)&S, (void*)&qbytes};
  CFM_CUDA_OK(cudaLaunchCooperativeKernel((void*)kern, dim3(grid), dim3(NT), args, smem, s));
  note_launches(1);
  return CFM_OK;
}

// fp32 M streams from HBM when it takes more than 3/4 of the L2 (the potentials, the column partials and the ring
// refills share the rest); a smaller M stays resident by itself
static bool v2_streams(int n0, int n1) { return (size_t)n0 * n1 * 4 > l2_bytes() / 4 * 3; }

// Row pitch of the 3-byte cost copy when a shape takes that stream, else 0: the shapes this kernel covers
// (n1 a multiple of 4, at most 8192; the launch also needs 16-byte aligned fp32 rows) whose fp32 M streams.  An M
// that stays in the L2 keeps the fp32 sweep.  The workspace size and the launch both decide through this.
size_t sinkhorn_v2_compact_pitch(int n0, int n1) {
  if ((n1 & 3) != 0 || n1 > 8192 || !v2_streams(n0, n1)) return 0;
  return align_up((size_t)n1 * 3, 16);
}

// returns CFM_OK when launched, 1 when this shape is not covered (caller uses sinkhorn.cu), <0 on error
int sinkhorn_v2_launch(SkParams& p, cudaStream_t s) {
  if (!p.vec || p.n1p > 8192 || p.n1p != p.n1) return 1;
  p.ldc = (int64_t)sinkhorn_v2_compact_pitch(p.n0, p.n1);
  if (p.ldc == 0) p.mq = nullptr;  // (the caller points mq at the workspace region, sized by the same rule)
  // L2 policy, from the device's L2 size: M that stays resident by itself (v2_streams) keeps the default policy; a
  // larger M streams, and the part of it kept evict_last from sweep to sweep is kSkResidentShare of the L2 (CFM_SK_L2
  // overrides it with a fraction of each slab; the kernel keeps the same bytes resident on the 3-byte stream).  Solve
  // ms on an H100 80GB HBM3 (50 MB L2, 700 W limit; scripts/sk_l2_sweep.py), fp32 stream: C2 (M = 268 MB) with
  // 0 / 8 / 16 / 40 MB resident 9.61 / 9.33 / 9.36 / 9.45; a 4096 x 4096 shard (67 MB) with 0 / 4 / 10 / 20 MB
  // resident 2.91 / 2.58 / 2.51 / 2.52 -- about 10 MB, a fifth of the L2, suits both
  constexpr float kSkResidentShare = 0.2f;
  const size_t m_bytes = (size_t)p.n0 * p.n1 * 4, l2 = l2_bytes();
  const bool streams = v2_streams(p.n0, p.n1);
  static float l2frac = -2.f;
  if (l2frac < -1.f) { const char* e = getenv("CFM_SK_L2"); l2frac = e ? (float)atof(e) : -1.f; }
  p.l2_resident_frac = !streams ? 0.f : l2frac >= 0.f ? l2frac : fminf(1.f, kSkResidentShare * (float)l2 / (float)m_bytes);
  // one 512-thread CTA per SM
  const int kg = (p.n1p / 4 + 511) / 512;
  // 22-bit chunks where the kernel packs 16 entries per thread (KG = 4) into a row shorter than the 3-byte one
  // (n1 > 7509); CFM_SK_Q24=1 keeps every chunk at 3 bytes (a cross-check: both give the same bits)
  static int q24 = -1;
  if (q24 < 0) { const char* e = getenv("CFM_SK_Q24"); q24 = e && atoi(e) != 0 ? 1 : 0; }
  p.ldn = kg > 2 && !q24 && p.mq != nullptr && kV2NarrowRow < p.ldc ? (int)kV2NarrowRow : 0;
  if (kg <= 1) return v2_launch_t<512, 1, 8>(p, s);
  if (kg <= 2) return v2_launch_t<512, 2, 4>(p, s);
  return v2_launch_t<512, 4, 2>(p, s);
}

}  // namespace cfm
