// Reusable Hopper tensor-core GEMM core:  D[m, n] = sum_k A[m, k] * B[n, k]  at fp32-grade accuracy, with each
// operand carried as a (hi, lo) pair.  The kernel (gemm_wg_kernel) is parameterised by a Scheme type that fixes the
// element type, the K-chunk and the MMAs of one k-step: the fp16x3 scheme (gemm_h3.cuh, H3Scheme).
//
// Persistent warp-specialised kernel, one CTA per SM, 384 threads = three warpgroups:
//   warpgroup 0      TMA producer (one thread): 4 tiled loads per K-chunk (A_hi, A_lo: 128 rows; B_hi, B_lo: 128
//                    rows; 128 bytes of K each, 128B swizzle) into a 3-stage shared-memory ring, mbarrier complete_tx.
//   warpgroups 1, 2  consumers: warpgroup c owns rows [64c, 64c + 64) of the 128 x 128 output tile and issues the
//                    wgmma.mma_async m64n128 instructions for them (operands straight from the swizzled stages,
//                    accumulators in registers); the stage of chunk k is handed back to the producer once the
//                    wgmma group of chunk k has retired (wait_group 1 after chunk k + 1 is issued).
//   epilogue         the consumers themselves: the accumulator fragment goes through a per-warpgroup XOR-swizzled
//                    staging tile in shared memory (64 rows x 64 columns at a time) so that a warp holds 32 rows x 32
//                    consecutive columns with thread = row, the layout the epilogue functors take:
//                      begin_row(row, ok); store32(row0, lane, col0, acc[32], n_rows, n_cols, tile); finish(lane)
//                    -- store32 is called by the whole warp, which writes the chunk coalesced via tc_store_chunk32.
//                    Meanwhile the producer already streams the next tile's stages.
// Tiles are walked M-fastest so the B panel stays hot in L2.
// Users, through gemm_h3.cuh: the fp16x3 cost matrix, the per-layer MLP and the tensor-core training step
// (train_tc.cu, the only user of split-K; see gemm_wg_body).  The PTX wrappers below are shared with
// mlp_h3.cu's fused kernel.
#pragma once
#include <cuda.h>

#include <type_traits>

#include "common.cuh"

namespace cfm {

constexpr int kTM = 128, kTN = 128;        // output tile
constexpr int kTileBytes = kTM * 128;      // 16 KB: one 128-row operand tile, 128 bytes of K per row
constexpr int kWgStages = 3;
constexpr int kWgStageBytes = 4 * kTileBytes;              // A_hi | A_lo | B_hi | B_lo
constexpr int kWgStagingBytes = 2 * 64 * 64 * 4;           // per consumer warpgroup: 64 rows x 64 fp32 columns
constexpr size_t kWgSmemBytes = (size_t)kWgStages * kWgStageBytes + kWgStagingBytes + 256;
constexpr int kWgThreads = 384;

struct TcShape {
  int n0, n1, d;          // rows of A, rows of B (= output columns), K
  int tiles_m, tiles_n;
};

// ---- PTX wrappers --------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// named barrier over `count` threads (ids 1.. are free; 0 is __syncthreads)
__device__ __forceinline__ void named_bar(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
// generic-proxy shared-memory writes -> visible to the tensor core's async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// register budget of the warp-specialised kernels: the producer warpgroup gives registers to the consumers
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// wgmma shared-memory matrix descriptor of a K-major, 128B-swizzled operand tile: rows of 128 B, 8-row groups
// 1024 B apart (stride byte offset), leading byte offset unused for swizzled K-major layouts.  Advancing along K
// inside the 128-byte atom adds the byte offset to the start address (the swizzle is applied to address bits).
__device__ __forceinline__ uint64_t wg_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3fff);       // start address, 16-byte units
  d |= (uint64_t)1 << 16;                           // leading byte offset (ignored)
  d |= (uint64_t)(1024 >> 4) << 32;                 // stride byte offset between 8-row groups
  d |= (uint64_t)1 << 62;                           // layout type: SWIZZLE_128B
  return d;
}

#define CFM_WG_ACC8(d, i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), \
                          "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define CFM_WG_ACC64(d) CFM_WG_ACC8(d, 0), CFM_WG_ACC8(d, 8), CFM_WG_ACC8(d, 16), CFM_WG_ACC8(d, 24), \
                        CFM_WG_ACC8(d, 32), CFM_WG_ACC8(d, 40), CFM_WG_ACC8(d, 48), CFM_WG_ACC8(d, 56)
#define CFM_WG_REGS64                                                                                              \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
  "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, " \
  "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"

// d[64] (+)= A(64 x 16 fp16) . B(128 x 16 fp16)^T, both K-major in shared memory; accumulate = 0 overwrites d
__device__ __forceinline__ void wg_mma_f16_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " CFM_WG_REGS64 ", %64, %65, p, 1, 1, 0, 0;\n\t}\n"
      : CFM_WG_ACC64(d)
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// Accumulator fragment of wgmma m64nN (fp32): thread (warp w of the warpgroup, lane l) holds, for every 8-column
// group i, rows 16w + l/4 and 16w + l/4 + 8 at columns 8i + 2(l%4) + {0, 1}:  d[4i + {0,1}] and d[4i + {2,3}].

// Coalesced write of one 32 x 32 fp32 chunk whose ROWS are spread over the lanes (lane = row, v[] = 32 consecutive
// columns).  Written straight from that layout a warp store instruction touches 32 different 128-byte lines, 16
// bytes each.  Here the chunk is transposed through a per-warp XOR-swizzled shared-memory tile (conflict-free
// 128-bit accesses both ways), so every store instruction writes 4 full rows x 128 contiguous bytes.
// out: &D[row0][col0], ld in floats (multiple of 4, 16-byte aligned); rows >= rows_valid are not written.
__device__ __forceinline__ void tc_store_chunk32(float* tile, const float (&v)[32], float* out, int64_t ld,
                                                 int rows_valid, int lane) {
#pragma unroll
  for (int g = 0; g < 8; ++g)
    *reinterpret_cast<float4*>(tile + lane * 32 + ((g ^ (lane & 7)) << 2)) =
        make_float4(v[4 * g], v[4 * g + 1], v[4 * g + 2], v[4 * g + 3]);
  __syncwarp();
  const int g = lane & 7;
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int r = it * 4 + (lane >> 3);
    const float4 q = *reinterpret_cast<const float4*>(tile + r * 32 + ((g ^ (r & 7)) << 2));
    if (r < rows_valid) *reinterpret_cast<float4*>(out + (int64_t)r * ld + 4 * g) = q;
  }
  __syncwarp();
}

// Split-K (kSplitK, a compile-time property of the epilogue): the work items are (tile, K-slice) pairs, item i =
// tile i % tiles, slice i / tiles, and slice s covers K-chunks [s * epi.k_chunks, (s + 1) * epi.k_chunks) of the
// epi.k_slices * epi.k_chunks >= nk chunks.  Before the epilogue of an item the consumers call epi.begin_slice(s); the
// epilogue writes a partial result per slice, which a later kernel folds.  Without split-K every item is a whole tile.
template <class Scheme, class Epi, bool kSplitK>
__device__ __forceinline__ void gemm_wg_body(const CUtensorMap& map_ah, const CUtensorMap& map_al,
                                             const CUtensorMap& map_bh, const CUtensorMap& map_bl, const TcShape& p,
                                             Epi& epi) {
  constexpr int kStages = kWgStages, kStageBytes = kWgStageBytes, kK = Scheme::kKChunk;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* stage_base = smem;
  float* staging = reinterpret_cast<float*>(smem + kStages * kStageBytes);  // [2 warpgroups][4 chunks][32 x 32]
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes + kWgStagingBytes);
  uint64_t* empty = full + kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = p.tiles_m * p.tiles_n;
  const int nk = (p.d + kK - 1) / kK;
  int num_items = num_tiles;
  if constexpr (kSplitK) num_items = num_tiles * epi.k_slices;
  // item t -> its tile and the K-chunk range [kc0, kc1)
  auto item = [&](int t, int& tile, int& kc0, int& kc1) {
    tile = t; kc0 = 0; kc1 = nk;
    if constexpr (kSplitK) {
      tile = t % num_tiles;
      kc0 = (t / num_tiles) * epi.k_chunks;
      kc1 = min(nk, kc0 + epi.k_chunks);
    }
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 256); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_items; t += gridDim.x) {
        int tile, kc0, kc1;
        item(t, tile, kc0, kc1);
        const int tm = tile % p.tiles_m, tn = tile / p.tiles_m;
        for (int kc = kc0; kc < kc1; ++kc) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sb = stage_base + stage * kStageBytes;
          mbar_expect_tx(&full[stage], kStageBytes);
          tma_load_2d(sb, &map_ah, &full[stage], kc * kK, tm * kTM);
          tma_load_2d(sb + kTileBytes, &map_al, &full[stage], kc * kK, tm * kTM);
          tma_load_2d(sb + 2 * kTileBytes, &map_bh, &full[stage], kc * kK, tn * kTN);
          tma_load_2d(sb + 3 * kTileBytes, &map_bl, &full[stage], kc * kK, tn * kTN);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: MMAs + epilogue =====================
    setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1;   // 0 / 1: rows [64 wg, 64 wg + 64) of the tile
    const int wq = warp & 3;          // warp inside the warpgroup
    float* stg = staging + wg * (4 * 1024);
    int stage = 0;
    uint32_t phase = 0;
    float acc0[64], acc1[64];
    for (int t = blockIdx.x; t < num_items; t += gridDim.x) {
      int tile, kc0, kc1;
      item(t, tile, kc0, kc1);
      const int tm = tile % p.tiles_m, tn = tile / p.tiles_m;
      int prev = -1;
      for (int kc = kc0; kc < kc1; ++kc) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(stage_base + stage * kStageBytes);
        const uint64_t ah = wg_desc_sw128(sa + wg * 8192), al = wg_desc_sw128(sa + kTileBytes + wg * 8192);
        const uint64_t bh = wg_desc_sw128(sa + 2 * kTileBytes), bl = wg_desc_sw128(sa + 3 * kTileBytes);
        wg_fence();
#pragma unroll
        for (int k = 0; k < kK / Scheme::kKStep; ++k) {
          const uint64_t koff = (uint64_t)((k * Scheme::kKStep * Scheme::kElem) >> 4);  // 32 bytes per k-step
          Scheme::mma(acc0, acc1, ah + koff, al + koff, bh + koff, bl + koff, ((kc - kc0) | k) ? 1u : 0u);
        }
        wg_commit();
        wg_wait<1>();  // the group of the previous chunk has retired: its stage goes back to the producer
        if (prev >= 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wg_wait<0>();
      if (prev >= 0) mbar_arrive(&empty[prev]);
      if constexpr (kSplitK) epi.begin_slice(t / num_tiles);

      // ---- epilogue: two 64-column halves through the warpgroup's staging tile ----
      const int fr = 16 * wq + (lane >> 2);  // fragment row (and fr + 8) inside the warpgroup's 64 rows
      const int fc = 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        named_bar(2 + wg, 128);  // the previous half's readers are done with the staging tile
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int gi = 8 * h + i;
          const int c = 8 * i + fc;  // column inside the half
          float* chunk = stg + (((fr >> 5) << 1) + (c >> 5)) * 1024;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int r = (fr + 8 * e) & 31, cc = c & 31;
            *reinterpret_cast<float2*>(chunk + r * 32 + ((((cc >> 2) ^ (r & 7))) << 2) + (cc & 3)) =
                make_float2(Scheme::combine(acc0[4 * gi + 2 * e], acc1[4 * gi + 2 * e]),
                            Scheme::combine(acc0[4 * gi + 2 * e + 1], acc1[4 * gi + 2 * e + 1]));
          }
        }
        named_bar(2 + wg, 128);
        // warp wq drains chunk wq: rows 32 (wq >> 1) .. +32, columns 32 (wq & 1) .. +32 of the half
        float* chunk = stg + wq * 1024;
        float v[32];
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          const float4 q = *reinterpret_cast<const float4*>(chunk + lane * 32 + ((g ^ (lane & 7)) << 2));
          v[4 * g] = q.x; v[4 * g + 1] = q.y; v[4 * g + 2] = q.z; v[4 * g + 3] = q.w;
        }
        __syncwarp();
        const int row0 = tm * kTM + wg * 64 + (wq >> 1) * 32;
        const int col0 = tn * kTN + h * 64 + (wq & 1) * 32;
        epi.begin_row(row0 + lane, row0 + lane < p.n0);
        if (row0 < p.n0 && col0 < p.n1) epi.store32(row0, lane, col0, v, p.n0, p.n1, chunk);  // warp-uniform
      }
    }
    epi.finish(lane);
  }
}

template <class Scheme, class Epi>
__global__ void __launch_bounds__(kWgThreads, 1)
gemm_wg_kernel(const __grid_constant__ CUtensorMap map_ah, const __grid_constant__ CUtensorMap map_al,
               const __grid_constant__ CUtensorMap map_bh, const __grid_constant__ CUtensorMap map_bl,
               const TcShape p, Epi epi) {
  gemm_wg_body<Scheme, Epi, false>(map_ah, map_al, map_bh, map_bl, p, epi);
}

// The entry of the epilogues that declare `static constexpr bool kSplitK` (the training GEMMs of train_tc.cu), with or
// without split-K; the cost-matrix and per-layer MLP epilogues declare nothing and keep gemm_wg_kernel.
template <class Scheme, class Epi>
__global__ void __launch_bounds__(kWgThreads, 1)
gemm_wg_splitk_kernel(const __grid_constant__ CUtensorMap map_ah, const __grid_constant__ CUtensorMap map_al,
                      const __grid_constant__ CUtensorMap map_bh, const __grid_constant__ CUtensorMap map_bl,
                      const TcShape p, Epi epi) {
  gemm_wg_body<Scheme, Epi, Epi::kSplitK>(map_ah, map_al, map_bh, map_bl, p, epi);
}

template <class Epi, class = void> struct wg_declares_split_k : std::false_type {};
template <class Epi> struct wg_declares_split_k<Epi, std::void_t<decltype(Epi::kSplitK)>> : std::true_type {};

// ---- host side -------------------------------------------------------------------------------------
// the default kernel entry of an epilogue: gemm_wg_splitk_kernel if it declares kSplitK, gemm_wg_kernel otherwise
template <class Scheme, class Epi>
constexpr auto wg_entry() {
  if constexpr (wg_declares_split_k<Epi>::value) return gemm_wg_splitk_kernel<Scheme, Epi>;
  else return gemm_wg_kernel<Scheme, Epi>;
}

// launch of the kernel entry `kern` on prepared tensor maps (grid = min(tiles, SMs)).  A file passes an entry of its own
// to keep its GEMMs apart from the instantiations other files' tests pin.
template <class Scheme, class Epi, auto kern = wg_entry<Scheme, Epi>()>
inline int launch_gemm_wg(const CUtensorMap& mah, const CUtensorMap& mal, const CUtensorMap& mbh,
                          const CUtensorMap& mbl, int n0, int n1, int d, Epi epi, cudaStream_t s) {
  TcShape p;
  p.n0 = n0; p.n1 = n1; p.d = d;
  p.tiles_m = (n0 + kTM - 1) / kTM;
  p.tiles_n = (n1 + kTN - 1) / kTN;
  int grid = p.tiles_m * p.tiles_n;
  if constexpr (wg_declares_split_k<Epi>::value) {
    if constexpr (Epi::kSplitK) grid *= epi.k_slices;
  }
  static bool attr_set = false;  // per kernel instantiation
  if (!attr_set) {
    CFM_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kWgSmemBytes));
    attr_set = true;
  }
  if (grid > sm_count()) grid = sm_count();
  kern<<<grid, kWgThreads, kWgSmemBytes, s>>>(mah, mal, mbh, mbl, p, epi);
  ::cfm::note_launches(1);
  CFM_CUDA_OK(cudaGetLastError());
  return CFM_OK;
}

}  // namespace cfm
