// Cost matrix  M = cdist(x0, x1)**2  on the fp16 wgmma path (gemm_h3.cuh, fp16x3 scheme)
// (reference: torchcfm/optimal_transport.py:84-86).
//
// One pre-pass per input (one warp per row): |x_r|^2 in fp32, the row's absolute maximum, a power-of-two
// row scale s_r that puts max|x_r| * s_r in [2^13, 2^14) (exact; fp16 overflows at 65504 and the data range
// is the caller's), and the (hi, lo) fp16 split of the scaled row.  The GEMM epilogue undoes the scales --
// dot_ij = (acc0 + acc1 2^-11) / (s_i t_j), again exact powers of two -- and applies
// |x0_i|^2 + |x1_j|^2 - 2 dot, clamp, sqrt, square, running max exactly like the SIMT path (sqdist.cu).
#include <mutex>

#include "gemm_h3.cuh"

namespace cfm {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// ---- TMA descriptor cache ---------------------------------------------------------------------------
// A CUtensorMap is a pure function of (base pointer, shape, strides, box, element type); a training loop
// hands the same buffers to the GEMMs every step, so the encode call is made once per distinct key and the
// 128-byte descriptor is replayed from a small direct-mapped table afterwards (the only library state
// besides the error string; guarded by a mutex, safe from several host threads).
namespace {
struct MapKey {
  const void* base; int rows, d, box_rows, elem; int64_t ld;
  bool operator==(const MapKey& o) const {
    return base == o.base && rows == o.rows && d == o.d && box_rows == o.box_rows && elem == o.elem && ld == o.ld;
  }
};
struct MapSlot { MapKey key; CUtensorMap map; bool used; };
constexpr int kMapSlots = 256;
MapSlot g_maps[kMapSlots];
std::mutex g_map_mu;
inline unsigned map_hash(const MapKey& k) {
  uint64_t h = reinterpret_cast<uintptr_t>(k.base) * 0x9E3779B97F4A7C15ull;
  h ^= ((uint64_t)k.rows << 32) ^ (uint64_t)k.d ^ ((uint64_t)k.box_rows << 20) ^ ((uint64_t)k.elem << 12) ^ ((uint64_t)k.ld << 40);
  h *= 0xC2B2AE3D27D4EB4Full;
  return (unsigned)(h >> 40) % kMapSlots;
}
}  // namespace

static int make_map_cached(CUtensorMap* m, const void* base, int rows, int d, int64_t ld, int box_rows, int elem) {
  const MapKey key{base, rows, d, box_rows, elem, ld};
  const unsigned slot = map_hash(key);
  {
    std::lock_guard<std::mutex> g(g_map_mu);
    if (g_maps[slot].used && g_maps[slot].key == key) { *m = g_maps[slot].map; return CFM_OK; }
  }
  EncodeTiledFn fn = encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled not available from the driver"); return CFM_ERR_CUDA; }
  cuuint64_t dims[2] = {(cuuint64_t)d, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * (cuuint64_t)elem};
  cuuint32_t box[2] = {(cuuint32_t)(128 / elem), (cuuint32_t)box_rows};  // 128-byte swizzle atom wide
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, elem == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                  const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) rows=%d d=%d ld=%lld elem=%d", (int)r, rows, d, (long long)ld, elem);
    return CFM_ERR_CUDA;
  }
  std::lock_guard<std::mutex> g(g_map_mu);
  g_maps[slot].key = key; g_maps[slot].map = *m; g_maps[slot].used = true;
  return CFM_OK;
}

int tc_make_map_f16(CUtensorMap* m, const __half* base, int rows, int d, int64_t ld, int box_rows) {
  return make_map_cached(m, base, rows, d, ld, box_rows, 2);
}

// one warp per row; d % 4 == 0, x 16-byte aligned, ldo % 8 == 0.  `uniform_absmax` (nullable, device): scale every
// row by the power of two derived from THIS value instead of the row's own maximum (the MLP weights: one scale per
// layer, so the epilogue multiplies by a kernel-uniform constant)
__global__ void prep_rows_h3_kernel(const float* __restrict__ X, int rows, int d, __half* __restrict__ hi,
                                    __half* __restrict__ lo, int64_t ldo, float* __restrict__ sqnorm,
                                    float* __restrict__ inv_scale, const float* __restrict__ uniform_absmax) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const float4* p = reinterpret_cast<const float4*>(X + (int64_t)warp * d);
  const int n4 = d >> 2;
  float s = 0.f, am = 0.f;
  for (int k = lane; k < n4; k += 32) {
    const float4 v = __ldg(p + k);
    s = fmaf(v.x, v.x, s); s = fmaf(v.y, v.y, s); s = fmaf(v.z, v.z, s); s = fmaf(v.w, v.w, s);
    am = fmaxf(am, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
  s = warp_sum(s);
  am = warp_max(am);
  if (uniform_absmax != nullptr) am = __ldg(uniform_absmax);
  // scale = 2^(13 - floor(log2(am))); non-finite or zero rows keep scale 1 (their products are what they are)
  const float sc = h3_pow2_scale(am);
  if (lane == 0) {
    if (sqnorm) sqnorm[warp] = s;
    inv_scale[warp] = 1.f / sc;  // exact
  }
  __half* h = hi + (int64_t)warp * ldo;
  __half* l = lo + (int64_t)warp * ldo;
  for (int k = lane; k < n4; k += 32) {
    const float4 v = __ldg(p + k);  // second pass: L1-resident (a row is d*4 bytes)
    __half hh[4], ll[4];
    split_h3(v.x * sc, hh[0], ll[0]); split_h3(v.y * sc, hh[1], ll[1]);
    split_h3(v.z * sc, hh[2], ll[2]); split_h3(v.w * sc, hh[3], ll[3]);
    *reinterpret_cast<uint2*>(h + 4 * k) = pack4h(hh);
    *reinterpret_cast<uint2*>(l + 4 * k) = pack4h(ll);
  }
}

// max |X| over a (rows x d) matrix into *out (zeroed by the caller)
__global__ void absmax_h3_kernel(const float* __restrict__ X, int64_t n, float* __restrict__ out) {
  float am = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = fabsf(X[i]);
    am = (v <= 3.0e38f) ? fmaxf(am, v) : am;  // non-finite entries do not set the scale
  }
  am = warp_max(am);
  if ((threadIdx.x & 31) == 0) atomic_max_nonneg(out, am);
}

int prep_rows_h3(const float* X, int rows, int d, __half* hi, __half* lo, int64_t ldo, float* sqnorm,
                 float* inv_scale, cudaStream_t s, float* uniform_absmax) {
  if (uniform_absmax != nullptr) {
    CFM_CUDA_OK(cudaMemsetAsync(uniform_absmax, 0, sizeof(float), s));
    const int64_t n = (int64_t)rows * d;
    int blocks = (int)((n + 255) / 256);
    if (blocks > 1024) blocks = 1024;
    absmax_h3_kernel<<<blocks, 256, 0, s>>>(X, n, uniform_absmax);
    ::cfm::note_launches(1);
  }
  prep_rows_h3_kernel<<<(rows + 7) / 8, 256, 0, s>>>(X, rows, d, hi, lo, ldo, sqnorm, inv_scale, uniform_absmax);
  ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}

struct SqDistH3Epilogue {
  float* M;
  int64_t ldm;
  const float* nx;   // |x0_i|^2
  const float* ny;   // |x1_j|^2
  const float* isx;  // 1 / row scale of x0
  const float* isy;  // 1 / row scale of x1
  float* cost_max;
  int squared;
  float a, ia, tmax;
  __device__ __forceinline__ void begin_row(int row, bool ok) {
    a = ok ? __ldg(nx + row) : 0.f;
    ia = ok ? __ldg(isx + row) : 0.f;
  }
  __device__ __forceinline__ float one(float acc, float b, float ib) const {
    const float dot = (acc * ia) * ib;  // exact rescale
    const float d2 = (a + b) - 2.f * dot;
    const float v = d2 < 0.f ? 0.f : d2;  // clamp_min(0) that lets NaN through, like ATen's
    // sqrt-then-square mimics cdist(...)**2; on this path the contraction itself is good to ~1e-6 of the norms,
    // so the 2-ulp approximate square root (one MUFU, no IEEE fix-up subroutine) does not show
    float s;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(s) : "f"(v));
    return squared ? s * s : s;
  }
  __device__ __forceinline__ void store32(int row0, int lane, int col0, const float (&r)[32], int n0, int n1,
                                          float* tile) {
    const int row = row0 + lane;
    const bool ok = row < n0;
    if (col0 + 32 <= n1) {
      float o[32];
      float m = 0.f;
#pragma unroll
      for (int c = 0; c < 32; c += 4) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(ny + col0 + c));
        const float4 ib = __ldg(reinterpret_cast<const float4*>(isy + col0 + c));
        o[c] = one(r[c], b.x, ib.x); o[c + 1] = one(r[c + 1], b.y, ib.y);
        o[c + 2] = one(r[c + 2], b.z, ib.z); o[c + 3] = one(r[c + 3], b.w, ib.w);
        m = fmaxf(m, fmaxf(fmaxf(o[c], o[c + 1]), fmaxf(o[c + 2], o[c + 3])));
      }
      if (ok) tmax = fmaxf(tmax, m);
      tc_store_chunk32(tile, o, M + (int64_t)row0 * ldm + col0, ldm, n0 - row0, lane);
    } else if (ok) {
      float* dst = M + (int64_t)row * ldm + col0;
#pragma unroll
      for (int c = 0; c < 32; ++c)
        if (col0 + c < n1) {
          const float v = one(r[c], __ldg(ny + col0 + c), __ldg(isy + col0 + c));
          tmax = fmaxf(tmax, v);
          dst[c] = v;
        }
    }
  }
  __device__ __forceinline__ void finish(int lane) {
    if (cost_max == nullptr) return;
    const float m = warp_max(tmax);
    if (lane == 0) atomic_max_nonneg(cost_max, m);
  }
};

struct H3Ws { size_t ah, al, bh, bl, isx, isy, total; int64_t ld; };
static H3Ws h3_ws(int n0, int n1, int d) {
  H3Ws w;
  w.ld = (d + 7) / 8 * 8;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes, 256); return r; };
  w.ah = take((size_t)n0 * w.ld * 2); w.al = take((size_t)n0 * w.ld * 2);
  w.bh = take((size_t)n1 * w.ld * 2); w.bl = take((size_t)n1 * w.ld * 2);
  w.isx = take((size_t)n0 * 4); w.isy = take((size_t)n1 * 4);
  w.total = o;
  return w;
}

size_t sqdist_h3_workspace_bytes(int n0, int n1, int d) { return h3_ws(n0, n1, d).total; }

// nx, ny are written here (the fused pre-pass computes the norms as well)
int sqdist_h3_launch(const float* x0, const float* x1, float* M, int n0, int n1, int d, int64_t ldm, int squared,
                     float* cost_max, float* nx, float* ny, void* ws, size_t ws_bytes, cudaStream_t s) {
  const H3Ws W = h3_ws(n0, n1, d);
  CFM_REQUIRE(ws_bytes >= W.total, "sqdist fp16x3: workspace too small (%zu < %zu)", ws_bytes, W.total);
  char* w = reinterpret_cast<char*>(ws);
  __half* ah = reinterpret_cast<__half*>(w + W.ah);
  __half* al = reinterpret_cast<__half*>(w + W.al);
  __half* bh = reinterpret_cast<__half*>(w + W.bh);
  __half* bl = reinterpret_cast<__half*>(w + W.bl);
  float* isx = reinterpret_cast<float*>(w + W.isx);
  float* isy = reinterpret_cast<float*>(w + W.isy);
  int rc;
  if ((rc = prep_rows_h3(x0, n0, d, ah, al, W.ld, nx, isx, s, nullptr)) != CFM_OK) return rc;
  if ((rc = prep_rows_h3(x1, n1, d, bh, bl, W.ld, ny, isy, s, nullptr)) != CFM_OK) return rc;
  SqDistH3Epilogue epi{M, ldm, nx, ny, isx, isy, cost_max, squared, 0.f, 0.f, 0.f};
  return launch_gemm_h3(ah, al, n0, W.ld, bh, bl, n1, W.ld, d, epi, s);
}

}  // namespace cfm
