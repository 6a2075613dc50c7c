// Warp-specialised bf16 GEMM for sm_90a (Hopper).
//
//   C[g, m, n] = epilogue( sum_k A[g, m, k] * B[g, n, k] )        g in [0, G)
//
// * operands are staged by TMA (cp.async.bulk.tensor, 128B swizzle) into a
//   4-6 stage shared-memory ring;  either operand may be K-major ([.., MN, K]
//   storage) or MN-major ([.., K, MN] storage), so the same kernel serves the
//   forward (x @ w), dgrad (dy @ w^T) and wgrad (x^T @ dy) of every linear /
//   expert-FFN layer without any transposes in HBM (wgmma reads MN-major bf16
//   operands through its transpose bits);
// * two consumer warpgroups each own 64 rows of the 128 x BN tile and issue
//   wgmma.m64nBNk16 (fp32 accumulators in registers), keeping one k-block of
//   MMAs in flight while the next stage is awaited;
// * the kernel is persistent: min(tiles, SMs) CTAs walk the output tiles of all
//   groups in a fixed order (bands of kGroupM M-tiles, for L2 reuse), and the
//   producer runs ahead across tile boundaries, so the ring refills for the next
//   tile while the consumers run this tile's epilogue;
// * the output is bf16. The fused epilogue is bias, then ReLU or nothing, then a
//   ReLU-gradient mask or a residual add (never both, and neither after ReLU),
//   then a per-row scale;
// * outputs leave by TMA: each consumer warpgroup applies the epilogue in its
//   accumulator layout, writes bf16 into a 64 x 64 swizzled staging slice and one
//   thread issues a bulk tensor store, so the next tile's MMAs start without
//   waiting for global memory. The residual / ReLU-mask operand arrives the same
//   way: TMA loads it into the staging slice ahead of use and the epilogue
//   overwrites it in place. The four epilogue kinds (plain, ReLU, residual add,
//   ReLU mask) are compiled as separate specialisations, picked once per tile;
// * the general epilogue serves redirected rows only: the store target of every
//   output row comes from a row-pointer table, which is how the MoE combine
//   (expert GEMM -> NVLink peer store) is fused. It stages fp32 accumulators
//   through shared memory, 64 columns at a time, and then works on 8 adjacent
//   columns of a row per thread, so every global load and store is a 16-byte
//   row-contiguous vector.
//
// Every output tile is computed by one CTA with the same k-block order and wgmma
// shape as a one-tile-per-CTA launch, so results do not depend on the grid size.
//
// 384 threads: warps 0..7 = two consumer warpgroups, warps 8..11 = producer warpgroup
// (one thread issues TMA). The producer gives its registers to the consumers with
// setmaxnreg: the 128 fp32 accumulators plus the epilogue do not fit in the 168 registers
// per thread that a 384-thread CTA gets by default.

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <mutex>
#include <unordered_map>

#include "ptx.cuh"
#include "registry.h"
#include "tmap.h"

namespace lb {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;   // 64 bf16 = 128 bytes = one swizzle row
constexpr int kMmaK = 16;
constexpr int kNumConsumers = 256;                 // two warpgroups x 64 rows
constexpr int kNumThreads = kNumConsumers + 128;   // + the TMA producer warpgroup
constexpr int kEpiCols = 64;  // columns per epilogue staging slice
constexpr int kGroupM = 8;    // M-tiles per rasterisation band

enum Act : int { kActNone = 0, kActRelu = 1 };
enum AuxMode : int { kAuxNone = 0, kAuxReluMask = 1, kAuxAdd = 2 };
// Epilogue specialisations of the TMA-store path (bias and row scale are uniform branches
// inside each).
enum EpiKind : int { kEpiPlain = 0, kEpiRelu = 1, kEpiAdd = 2, kEpiMask = 3 };

struct GemmParams {
  int G, M, N, K;
  long long ldc;           // row stride of C (elements)
  long long c_batch;       // batch stride of C (elements)
  const float* bias;       // [G, N] fp32 or nullptr
  const __nv_bfloat16* aux;  // [G, M, N] bf16 (same strides as C) or nullptr
  const float* row_scale;  // [G, M] or nullptr
  void* const* row_ptrs;   // [G * M] destination row pointers (peer memory) or nullptr
  int act;
  int aux_mode;
  int epi;                 // EpiKind (TMA-store path only)
};

// The fused epilogue of one output element, shared by both epilogues so that they round
// alike: + bias b, activation, ReLU-gradient mask or residual add with the aux element x,
// times the row scale rs. b and rs are read only when p has a bias / row scale.
__device__ __forceinline__ float epilogue_elem(const GemmParams& p, float v, float b, int act,
                                               int aux_mode, float x, float rs) {
  if (p.bias != nullptr) v += b;
  if (act == kActRelu) v = fmaxf(v, 0.f);
  if (aux_mode == kAuxReluMask) v = x > 0.f ? v : 0.f;
  else if (aux_mode == kAuxAdd) v += x;
  if (p.row_scale != nullptr) v *= rs;
  return v;
}

// Eight adjacent output columns of one row, read row-contiguously from the staging buffer,
// through epilogue_elem to the bf16 row at `dst`. `off` is the element offset of (row, col) in
// the C-shaped aux tensor; both are 16-byte aligned.
__device__ __forceinline__ void epilogue_vec8(const GemmParams& p, float (&v)[8],
                                              __nv_bfloat16* dst, long long off,
                                              const float* bias, float rscale) {
  float b[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (bias != nullptr) {
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias));
    const float4 b1 = __ldg(reinterpret_cast<const float4*>(bias) + 1);
    b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
    b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
  }
  float x[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (p.aux_mode != kAuxNone) {
    const int4 raw = *reinterpret_cast<const int4*>(p.aux + off);
    const uint32_t w[4] = {static_cast<uint32_t>(raw.x), static_cast<uint32_t>(raw.y),
                           static_cast<uint32_t>(raw.z), static_cast<uint32_t>(raw.w)};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 t = unpack_bf16x2(w[j]);
      x[2 * j] = t.x;
      x[2 * j + 1] = t.y;
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = epilogue_elem(p, v[j], b[j], p.act, p.aux_mode, x[j], rscale);
  *reinterpret_cast<int4*>(dst) = make_int4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]),
                                            pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}

template <int BN, bool kAK, bool kBK>
__device__ __forceinline__ void wgmma_bn(float (&acc)[BN / 2], uint64_t adesc, uint64_t bdesc) {
  if constexpr (BN == 256) wgmma_m64n256k16<kAK ? 0 : 1, kBK ? 0 : 1>(acc, adesc, bdesc, 1);
  else wgmma_m64n128k16<kAK ? 0 : 1, kBK ? 0 : 1>(acc, adesc, bdesc, 1);
}

template <int BN>
struct TileShape {
  static constexpr int kStages = (BN == 256) ? 4 : 6;
  static constexpr uint32_t kABytes = kBlockM * kBlockK * 2;   // 16 KiB
  static constexpr uint32_t kBBytes = BN * kBlockK * 2;        // 32 KiB (BN=256)
  static constexpr uint32_t kStageBytes = kABytes + kBBytes;
  static constexpr uint32_t kRingBytes = kStages * kStageBytes;
  // Epilogue staging per consumer warpgroup: 64 rows x 64 columns of fp32 (general path),
  // or two 64 x 64 bf16 slices (TMA-store path, double-buffered).
  static constexpr uint32_t kStagingBytes = 2 * 64 * kEpiCols * 4;
  // full + empty ring barriers, then two aux-load barriers per consumer warpgroup
  static constexpr size_t kSmemBytes = kRingBytes + kStagingBytes + (2 * kStages + 4) * 8 + 1024;
};
constexpr uint32_t kSliceBytes = 64 * kEpiCols * 2;  // one bf16 staging slice (TMA box)

// Tiles are numbered group by group. Inside a group they go in bands of kGroupM M-tiles,
// M-fastest inside a band: the CTAs of one wave then share a few A panels and B panels in L2.
struct TileCoord {
  int g, m_blk, n_blk;
};
__device__ __forceinline__ TileCoord tile_coord(int tile, int tiles_m, int tiles_n) {
  const int per_group = tiles_m * tiles_n;
  TileCoord t;
  t.g = tile / per_group;
  const int r = tile - t.g * per_group;
  const int band = r / (kGroupM * tiles_n);
  const int first_m = band * kGroupM;
  const int rows = min(kGroupM, tiles_m - first_m);
  const int in_band = r - band * kGroupM * tiles_n;
  t.n_blk = in_band / rows;
  t.m_blk = first_m + (in_band - t.n_blk * rows);
  return t;
}

// Byte offset of the 16-byte unit u (of 16) in row r of a warpgroup's staging buffer. The
// XOR spreads both the fragment writes (4 rows x 2 units per half-warp) and the
// row-contiguous reads (8 units of one row per quarter-warp) over all 32 banks.
__device__ __forceinline__ uint32_t staging_off(int r, int u) {
  return static_cast<uint32_t>(r * (kEpiCols / 4) + (u ^ ((r & 7) << 1))) * 16;
}

// TMA-store epilogue of one warpgroup's 64 x BN block (rows row0.., columns n0..). Slices of
// 64 columns alternate between the warpgroup's two bf16 staging buffers (`stg`, 128-byte
// swizzled rows, the layout of the output / aux tensor maps). The first aux slice was loaded
// during the MMA loop; the next one is loaded as soon as its buffer's store has read it.
template <int BN, int kAct, int kAux>
__device__ __forceinline__ void epilogue_tma(const GemmParams& p, float (&acc)[BN / 2],
                                             const CUtensorMap* tmap_c,
                                             const CUtensorMap* tmap_aux, uint32_t stg,
                                             uint32_t aux_bar, uint32_t& aux_par, int row0,
                                             int n0, int g, int wg) {
  const int t = threadIdx.x & 127;
  const bool leader = t == 0;
  const int r = (t >> 5) * 16 + ((t & 31) >> 2);   // fragment rows r and r + 8
  const int q = t & 3;                              // column pair inside an 8-column chunk
  const float* bias = p.bias ? p.bias + static_cast<long long>(g) * p.N : nullptr;
  float rs[2] = {1.f, 1.f};
  if (p.row_scale != nullptr) {
#pragma unroll
    for (int i = 0; i < 2; ++i)
      if (row0 + r + 8 * i < p.M)
        rs[i] = p.row_scale[static_cast<long long>(g) * p.M + row0 + r + 8 * i];
  }
#pragma unroll
  for (int s = 0; s < BN / kEpiCols; ++s) {
    const int c0 = n0 + s * kEpiCols;
    if (c0 >= p.N) break;
    const uint32_t buf = stg + (s & 1) * kSliceBytes;
    if (kAux != kAuxNone) {
      mbar_wait(aux_bar + (s & 1) * 8, (aux_par >> (s & 1)) & 1);
      aux_par ^= 1u << (s & 1);
    } else {
      if (leader) tma_store_wait_read<1>();   // the store that last read this buffer
      named_bar_sync(1 + wg, 128);
    }
#pragma unroll
    for (int n = 0; n < kEpiCols / 8; ++n) {
      const int col = c0 + 8 * n + 2 * q;
      float2 b = make_float2(0.f, 0.f);
      if (bias != nullptr && col < p.N) b = __ldg(reinterpret_cast<const float2*>(bias + col));
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const uint32_t addr = buf + (r + 8 * i) * 128 + ((n ^ (r & 7)) << 4) + q * 4;
        const int a = 4 * (s * (kEpiCols / 8) + n) + 2 * i;
        float2 x = make_float2(0.f, 0.f);
        if (kAux != kAuxNone) {
          uint32_t w;
          asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w) : "r"(addr) : "memory");
          x = unpack_bf16x2(w);
        }
        const float v0 = epilogue_elem(p, acc[a], b.x, kAct, kAux, x.x, rs[i]);
        const float v1 = epilogue_elem(p, acc[a + 1], b.y, kAct, kAux, x.y, rs[i]);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pack_bf16x2(v0, v1)) : "memory");
      }
    }
    fence_proxy_async();
    named_bar_sync(1 + wg, 128);
    if (leader) {
      tma_store_3d(tmap_c, buf, c0, row0, g);
      tma_store_commit();
      if (kAux != kAuxNone && s + 1 < BN / kEpiCols && c0 + kEpiCols < p.N) {
        tma_store_wait_read<1>();   // slice s - 1 has left the other buffer
        const uint32_t nb = aux_bar + ((s + 1) & 1) * 8;
        mbar_arrive_expect_tx(nb, kSliceBytes);
        tma_load_3d(stg + ((s + 1) & 1) * kSliceBytes, tmap_aux, nb, c0 + kEpiCols, row0, g);
      }
    }
  }
}

// kTmaStore: out through tmap_c (and aux through tmap_aux); otherwise the general epilogue,
// which stores through p.row_ptrs and ignores both maps.
template <int BN, bool kAK, bool kBK, bool kTmaStore>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a,
                  const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_c,
                  const __grid_constant__ CUtensorMap tmap_aux, const GemmParams p) {
  using TS = TileShape<BN>;
  constexpr int kStages = TS::kStages;
  static_assert(2 * kSliceBytes <= TS::kStagingBytes / 2, "two bf16 slices per warpgroup");

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024B alignment for SWIZZLE_128B atoms.
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* staging = smem + TS::kRingBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(staging + TS::kStagingBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;
  uint64_t* aux_bars = bars + 2 * kStages;   // [wg][buffer]

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int tiles_m = (p.M + kBlockM - 1) / kBlockM;
  const int tiles_n = (p.N + BN - 1) / BN;
  const int num_tiles = p.G * tiles_m * tiles_n;
  const int num_k_blocks = (p.K + kBlockK - 1) / kBlockK;

  if (threadIdx.x == kNumConsumers) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if constexpr (kTmaStore) {
      tma_prefetch_desc(&tmap_c);
      if (p.aux_mode != kAuxNone) tma_prefetch_desc(&tmap_aux);
      for (int i = 0; i < 4; ++i) mbar_init(smem_u32(&aux_bars[i]), 1);
    }
    for (int i = 0; i < kStages; ++i) {
      mbar_init(smem_u32(&full_bar[i]), 1);
      mbar_init(smem_u32(&empty_bar[i]), kNumConsumers / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();

  // The ring position (stage, phase) runs on across tiles in both roles, so the producer
  // fills the stages for the next tile while the consumers run this tile's epilogue.
  if (warp_idx >= kNumConsumers / 32) {
    // ============================ TMA producer ============================
    setmaxnreg_dec<40>();
    if (warp_idx == kNumConsumers / 32 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const TileCoord tc = tile_coord(tile, tiles_m, tiles_n);
        const int m0 = tc.m_blk * kBlockM, n0 = tc.n_blk * BN, g = tc.g;
        for (int kb = 0; kb < num_k_blocks; ++kb) {
          mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1);
          const uint32_t fb = smem_u32(&full_bar[stage]);
          mbar_arrive_expect_tx(fb, TS::kStageBytes);
          const uint32_t sa = smem_u32(smem + stage * TS::kStageBytes);
          const uint32_t sb = sa + TS::kABytes;
          const int k0 = kb * kBlockK;
          if constexpr (kAK) {
            tma_load_3d(sa, &tmap_a, fb, k0, m0, g);
          } else {
#pragma unroll
            for (int i = 0; i < kBlockM / 64; ++i)
              tma_load_3d(sa + i * (64 * kBlockK * 2), &tmap_a, fb, m0 + 64 * i, k0, g);
          }
          if constexpr (kBK) {
            tma_load_3d(sb, &tmap_b, fb, k0, n0, g);
          } else {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i)
              tma_load_3d(sb + i * (64 * kBlockK * 2), &tmap_b, fb, n0 + 64 * i, k0, g);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ============================== consumers ==============================
  // Warpgroup wg owns tile rows [64 wg, 64 wg + 64). Its A rows start 8 KiB into the
  // stage for both majors: 64 K-major rows of 128 B, or the wg-th 64-wide MN chunk.
  setmaxnreg_inc<232>();
  const int wg = warp_idx >> 2;
  const uint32_t stg = smem_u32(staging + wg * (64 * kEpiCols * 4));
  const uint32_t aux_bar = smem_u32(&aux_bars[2 * wg]);
  const bool leader = (threadIdx.x & 127) == 0;
  uint32_t aux_par = 0;   // parity of each staging buffer's aux barrier
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const TileCoord tc = tile_coord(tile, tiles_m, tiles_n);
    const int m0 = tc.m_blk * kBlockM, n0 = tc.n_blk * BN, g = tc.g;
    const int row0 = m0 + wg * 64;
    // TMA-store path: once the previous tile's stores have read the staging buffers, load
    // this tile's first aux slice. Issued behind the first k-block's MMAs.
    auto stage_aux = [&] {
      if constexpr (kTmaStore) {
        if (leader && row0 < p.M) {
          tma_store_wait_read<0>();
          if (p.aux_mode != kAuxNone) {
            mbar_arrive_expect_tx(aux_bar, kSliceBytes);
            tma_load_3d(stg, &tmap_aux, aux_bar, n0, row0, g);
          }
        }
      }
    };

    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev_stage = 0;
    for (int kb = 0; kb < num_k_blocks; ++kb) {
      mbar_wait(smem_u32(&full_bar[stage]), phase);
      const uint32_t sa = smem_u32(smem + stage * TS::kStageBytes) + wg * (64 * 128);
      const uint32_t sb = smem_u32(smem + stage * TS::kStageBytes) + TS::kABytes;
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < kBlockK / kMmaK; ++j) {
        // K-major: advance 32 B inside the 128 B swizzle row.
        // MN-major: advance 16 K-rows of 128 B; 64-wide MN chunks are
        //           64*kBlockK*2 bytes apart (LBO), 8-row groups 1 KiB (SBO).
        const uint64_t adesc =
            kAK ? make_smem_desc_sw128(sa + j * 32, 16, 1024)
                : make_smem_desc_sw128(sa + j * (kMmaK * 128), 64 * kBlockK * 2, 1024);
        const uint64_t bdesc =
            kBK ? make_smem_desc_sw128(sb + j * 32, 16, 1024)
                : make_smem_desc_sw128(sb + j * (kMmaK * 128), 64 * kBlockK * 2, 1024);
        wgmma_bn<BN, kAK, kBK>(acc, adesc, bdesc);
      }
      wgmma_commit();
      if (kb == 0) stage_aux();
      wgmma_wait<1>();                 // the previous k-block's MMAs have retired
      __syncwarp();
      if (kb > 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[prev_stage]));
      prev_stage = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    if (num_k_blocks == 0) stage_aux();
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    __syncwarp();
    if (num_k_blocks > 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[prev_stage]));

    if constexpr (kTmaStore) {
      if (row0 < p.M) {
        switch (p.epi) {
          case kEpiPlain:
            epilogue_tma<BN, kActNone, kAuxNone>(p, acc, &tmap_c, &tmap_aux, stg, aux_bar,
                                                 aux_par, row0, n0, g, wg);
            break;
          case kEpiRelu:
            epilogue_tma<BN, kActRelu, kAuxNone>(p, acc, &tmap_c, &tmap_aux, stg, aux_bar,
                                                 aux_par, row0, n0, g, wg);
            break;
          case kEpiAdd:
            epilogue_tma<BN, kActNone, kAuxAdd>(p, acc, &tmap_c, &tmap_aux, stg, aux_bar,
                                                aux_par, row0, n0, g, wg);
            break;
          case kEpiMask:
            epilogue_tma<BN, kActNone, kAuxReluMask>(p, acc, &tmap_c, &tmap_aux, stg, aux_bar,
                                                     aux_par, row0, n0, g, wg);
            break;
        }
      }
      continue;
    }

    // ================= general epilogue (redirected rows) =================
    // Per 64-column slice: fragments -> staging (fp32), then each thread takes 8 adjacent
    // columns of a row, so every global access is a 16-byte row-contiguous vector.
    const int frow = (warp_idx & 3) * 16 + (lane >> 2);
    const int q = threadIdx.x & 7;          // 8-column chunk of the slice
    const int rsub = (threadIdx.x & 127) >> 3;
    const int first = (q >> 2) & 1;        // which half of the chunk to read first (banks)
#pragma unroll
    for (int s = 0; s < BN / kEpiCols; ++s) {
      if (n0 + s * kEpiCols >= p.N) break;
      named_bar_sync(1 + wg, 128);         // the previous slice's reads are done
#pragma unroll
      for (int n = 0; n < kEpiCols / 8; ++n) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int a = 4 * (s * (kEpiCols / 8) + n) + 2 * i;
          const uint32_t addr = stg + staging_off(frow + 8 * i, 2 * n + ((lane & 3) >> 1)) +
                                (lane & 1) * 8;
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(acc[a]),
                       "f"(acc[a + 1]) : "memory");
        }
      }
      named_bar_sync(1 + wg, 128);
      const int col = n0 + s * kEpiCols + 8 * q;
#pragma unroll
      for (int pass = 0; pass < 4; ++pass) {
        const int r = rsub + 16 * pass;
        const int row = m0 + wg * 64 + r;
        if (row >= p.M || col >= p.N) continue;
        __nv_bfloat16* dst =
            reinterpret_cast<__nv_bfloat16*>(p.row_ptrs[static_cast<long long>(g) * p.M + row]);
        if (dst == nullptr) continue;
        const long long row_off =
            static_cast<long long>(g) * p.c_batch + static_cast<long long>(row) * p.ldc;
        float4 h0, h1;
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                     : "=f"(h0.x), "=f"(h0.y), "=f"(h0.z), "=f"(h0.w)
                     : "r"(stg + staging_off(r, 2 * q + first)) : "memory");
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                     : "=f"(h1.x), "=f"(h1.y), "=f"(h1.z), "=f"(h1.w)
                     : "r"(stg + staging_off(r, 2 * q + 1 - first)) : "memory");
        const float4 lo = first ? h1 : h0, hi = first ? h0 : h1;
        float v[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
        const float rscale =
            p.row_scale != nullptr ? p.row_scale[static_cast<long long>(g) * p.M + row] : 1.f;
        const float* bias = p.bias ? p.bias + static_cast<long long>(g) * p.N + col : nullptr;
        epilogue_vec8(p, v, dst + col, row_off + col, bias, rscale);
      }
    }
  }
  // Shared memory must outlive the bulk stores that read it.
  if constexpr (kTmaStore) {
    if (leader) tma_store_wait<0>();
  }
}

// ------------------------------------------------------------------ host ----
using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                              const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                              const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeFn GetEncodeFn() {
  static EncodeFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t err = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    TORCH_CHECK(err == cudaSuccess && ptr != nullptr, "cuTensorMapEncodeTiled not available");
    fn = reinterpret_cast<EncodeFn>(ptr);
  });
  return fn;
}

CUtensorMap MakeMap(const void* base, int64_t inner, int64_t rows, int64_t groups,
                    int64_t row_stride, int64_t group_stride, int box_rows,
                    CUtensorMapDataType dt, int elem_bytes) {
  // cuTensorMapEncodeTiled is a *driver* call: make sure this thread (e.g. an
  // autograd worker that has not issued a runtime call yet) has the primary
  // context bound, otherwise it fails with CUDA_ERROR_INVALID_CONTEXT.
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    // (skipped while a stream capture is in progress: cudaFree is not capturable, and a
    // thread that reaches this point during capture already ran the warm-up steps)
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(at::cuda::getCurrentCUDAStream(), &cap);
    if (cap == cudaStreamCaptureStatusNone) {
      C10_CUDA_CHECK(cudaFree(nullptr));
      ctx_bound = true;
    }
  }
  CUtensorMap m;
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(inner), static_cast<cuuint64_t>(rows),
                        static_cast<cuuint64_t>(groups)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(row_stride * elem_bytes),
                           static_cast<cuuint64_t>(group_stride * elem_bytes)};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(128 / elem_bytes), static_cast<cuuint32_t>(box_rows), 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = GetEncodeFn()(&m, dt, 3, const_cast<void*>(base), dims, strides, box, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  TORCH_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed: ", static_cast<int>(r),
              " inner=", inner, " rows=", rows, " groups=", groups, " row_stride=", row_stride,
              " group_stride=", group_stride);
  return m;
}

template <int BN, bool kAK, bool kBK, bool kTmaStore>
static void Launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc,
                   const CUtensorMap& tx, const GemmParams& p, int sms, cudaStream_t stream) {
  constexpr size_t smem = TileShape<BN>::kSmemBytes;
  static_assert(smem <= 227 * 1024, "GEMM shared memory exceeds the sm_90 limit");
  auto kern = gemm_wgmma_kernel<BN, kAK, kBK, kTmaStore>;
  static bool configured = false;
  if (!configured) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(smem)));
    configured = true;
  }
  const int64_t tiles = static_cast<int64_t>(p.G) * ((p.M + kBlockM - 1) / kBlockM) *
                        ((p.N + BN - 1) / BN);
  TORCH_CHECK(tiles < (int64_t{1} << 31), "gemm_bf16: too many output tiles");
  const int grid = static_cast<int>(std::min<int64_t>(tiles, sms));
  kern<<<grid, kNumThreads, smem, stream>>>(ta, tb, tc, tx, p);
  CountLaunch();
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

template <int BN, bool kTmaStore>
static void Dispatch(bool ak, bool bk, const CUtensorMap& ta, const CUtensorMap& tb,
                     const CUtensorMap& tc, const CUtensorMap& tx, const GemmParams& p, int sms,
                     cudaStream_t s) {
  if (ak && bk) Launch<BN, true, true, kTmaStore>(ta, tb, tc, tx, p, sms, s);
  else if (ak && !bk) Launch<BN, true, false, kTmaStore>(ta, tb, tc, tx, p, sms, s);
  else if (!ak && bk) Launch<BN, false, true, kTmaStore>(ta, tb, tc, tx, p, sms, s);
  else Launch<BN, false, false, kTmaStore>(ta, tb, tc, tx, p, sms, s);
}

// Tile width from the shape: 256 unless N is small, or unless 128-wide tiles finish at
// least 10 % sooner under the persistent schedule (the busiest CTA runs ceil(tiles / SMs)
// tiles; a 256-wide tile costs two 128-wide ones). 128-wide tiles move 1.33x more operand
// bytes per FLOP, hence the margin.
static bool UseBn256(int64_t G, int64_t M, int64_t N, int sms) {
  if (N <= 128) return false;
  const int64_t mt = G * ((M + kBlockM - 1) / kBlockM);
  const int64_t t256 = mt * ((N + 255) / 256), t128 = mt * ((N + 127) / 128);
  const int64_t w256 = 2 * ((t256 + sms - 1) / sms), w128 = (t128 + sms - 1) / sms;
  return w128 * 10 > w256 * 9;
}

// a: [G, M, K] if a_kmajor else [G, K, M];  b: [G, N, K] if b_kmajor else [G, K, N]
// (2-D inputs are treated as G = 1).  Returns / fills the bf16 out [G, M, N]; with row_ptrs,
// row (g, m) goes to row_ptrs[g * M + m] instead (skipped where that is 0).
torch::Tensor gemm_bf16(const torch::Tensor& a_in, const torch::Tensor& b_in, bool a_kmajor,
                        bool b_kmajor, const c10::optional<torch::Tensor>& bias,
                        int64_t act, const c10::optional<torch::Tensor>& aux, int64_t aux_mode,
                        const c10::optional<torch::Tensor>& row_scale,
                        const c10::optional<torch::Tensor>& out_opt,
                        const c10::optional<torch::Tensor>& row_ptrs) {
  TORCH_CHECK(a_in.is_cuda() && b_in.is_cuda(), "gemm_bf16: CUDA tensors required");
  TORCH_CHECK(a_in.scalar_type() == torch::kBFloat16 && b_in.scalar_type() == torch::kBFloat16,
              "gemm_bf16: bf16 inputs required");
  const bool has_aux = aux.has_value() && aux->defined() && aux_mode != kAuxNone;
  TORCH_CHECK(act == kActNone || act == kActRelu,
              "gemm_bf16: act must be 0 (none) or 1 (ReLU), got ", act);
  TORCH_CHECK(aux_mode >= kAuxNone && aux_mode <= kAuxAdd,
              "gemm_bf16: aux_mode must be 0 (none), 1 (ReLU mask) or 2 (add), got ", aux_mode);
  TORCH_CHECK(act == kActNone || !has_aux, "gemm_bf16: ReLU does not combine with an aux operand");
  const c10::cuda::CUDAGuard guard(a_in.device());
  torch::Tensor a = a_in.dim() == 2 ? a_in.unsqueeze(0) : a_in;
  torch::Tensor b = b_in.dim() == 2 ? b_in.unsqueeze(0) : b_in;
  TORCH_CHECK(a.dim() == 3 && b.dim() == 3, "gemm_bf16: 2-D or 3-D operands");
  if (a.stride(2) != 1) a = a.contiguous();
  if (b.stride(2) != 1) b = b.contiguous();
  const int64_t G = a.size(0);
  TORCH_CHECK(b.size(0) == G, "gemm_bf16: group mismatch");
  const int64_t M = a_kmajor ? a.size(1) : a.size(2);
  const int64_t K = a_kmajor ? a.size(2) : a.size(1);
  const int64_t N = b_kmajor ? b.size(1) : b.size(2);
  const int64_t Kb = b_kmajor ? b.size(2) : b.size(1);
  TORCH_CHECK(K == Kb, "gemm_bf16: K mismatch ", K, " vs ", Kb);
  TORCH_CHECK(K > 0, "gemm_bf16: K must be positive, got K = ", K);
  TORCH_CHECK(N % 8 == 0, "gemm_bf16: N must be a multiple of 8");
  auto check_op = [](const torch::Tensor& t) {
    TORCH_CHECK(t.stride(1) % 8 == 0 && (t.size(0) == 1 || t.stride(0) % 8 == 0) &&
                    reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0,
                "gemm_bf16: operand rows must be 16-byte aligned");
  };
  check_op(a);
  check_op(b);

  torch::Tensor out;
  if (out_opt.has_value()) {
    out = out_opt.value();
    TORCH_CHECK(out.stride(-1) == 1, "gemm_bf16: out must be row-contiguous");
  } else {
    out = torch::empty({G, M, N}, a.options());
  }
  TORCH_CHECK(out.scalar_type() == torch::kBFloat16, "gemm_bf16: out must be bf16");
  torch::Tensor out3 = out.dim() == 2 ? out.unsqueeze(0) : out;
  TORCH_CHECK(out3.size(0) == G && out3.size(1) == M && out3.size(2) == N, "gemm_bf16: out shape");

  // The epilogue moves 8 columns per 16-byte access (row_ptrs rows must be 16-byte aligned
  // as well).
  auto aligned16 = [](const void* ptr) { return reinterpret_cast<uintptr_t>(ptr) % 16 == 0; };
  TORCH_CHECK(aligned16(out3.data_ptr()) && out3.stride(1) % 8 == 0 &&
                  (G == 1 || out3.stride(0) % 8 == 0),
              "gemm_bf16: out rows must be 16-byte aligned");

  GemmParams p;
  p.G = static_cast<int>(G); p.M = static_cast<int>(M); p.N = static_cast<int>(N);
  p.K = static_cast<int>(K);
  p.ldc = out3.stride(1);
  p.c_batch = G > 1 ? out3.stride(0) : 0;
  p.bias = nullptr; p.aux = nullptr; p.row_scale = nullptr; p.row_ptrs = nullptr;
  torch::Tensor bias_f;
  if (bias.has_value() && bias->defined()) {
    bias_f = bias->to(torch::kFloat32).contiguous();
    if (!aligned16(bias_f.data_ptr())) bias_f = bias_f.clone();
    TORCH_CHECK(bias_f.numel() == G * N, "gemm_bf16: bias must be [G, N]");
    p.bias = bias_f.data_ptr<float>();
  }
  if (has_aux) {
    torch::Tensor ax = aux.value();
    ax = ax.dim() == 2 ? ax.unsqueeze(0) : ax;
    // The aux tensor map takes out's sizes, so a smaller aux would be read past its end.
    TORCH_CHECK(ax.dim() == 3 && ax.size(0) == G && ax.size(1) == M && ax.size(2) == N,
                "gemm_bf16: aux must have out's sizes [G, M, N] = [", G, ", ", M, ", ", N,
                "] (2-D only with G = 1), got ", ax.sizes());
    TORCH_CHECK(ax.scalar_type() == torch::kBFloat16 && ax.stride(1) == p.ldc &&
                    (G == 1 || ax.stride(0) == p.c_batch) && ax.stride(2) == 1,
                "gemm_bf16: aux must be bf16 with the same strides as out");
    TORCH_CHECK(aligned16(ax.data_ptr()), "gemm_bf16: aux must be 16-byte aligned");
    p.aux = reinterpret_cast<const __nv_bfloat16*>(ax.data_ptr());
  }
  torch::Tensor rs_f;
  if (row_scale.has_value() && row_scale->defined()) {
    rs_f = row_scale->to(torch::kFloat32).contiguous();
    TORCH_CHECK(rs_f.numel() == G * M, "gemm_bf16: row_scale must be [G, M]");
    p.row_scale = rs_f.data_ptr<float>();
  }
  if (row_ptrs.has_value() && row_ptrs->defined()) {
    TORCH_CHECK(row_ptrs->scalar_type() == torch::kInt64 && row_ptrs->numel() == G * M &&
                    row_ptrs->is_contiguous(), "gemm_bf16: row_ptrs must be int64 [G, M]");
    TORCH_CHECK(row_ptrs->is_cuda() && row_ptrs->device() == a_in.device(),
                "gemm_bf16: row_ptrs must be on the device of a (the kernel reads it)");
    p.row_ptrs = reinterpret_cast<void* const*>(row_ptrs->data_ptr());
  }
  p.act = static_cast<int>(act);
  p.aux_mode = has_aux ? static_cast<int>(aux_mode) : kAuxNone;
  p.epi = p.aux_mode == kAuxAdd ? kEpiAdd
        : p.aux_mode == kAuxReluMask ? kEpiMask
        : p.act == kActRelu ? kEpiRelu : kEpiPlain;

  if (M == 0 || N == 0 || G == 0) return out;

  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  const bool bn256 = UseBn256(G, M, N, sms);
  const int bn = bn256 ? 256 : 128;
  const CUtensorMap ta = a_kmajor
      ? MakeMap(a.data_ptr(), K, M, G, a.stride(1), G > 1 ? a.stride(0) : a.stride(1) * a.size(1), kBlockM)
      : MakeMap(a.data_ptr(), M, K, G, a.stride(1), G > 1 ? a.stride(0) : a.stride(1) * a.size(1), kBlockK);
  const CUtensorMap tb = b_kmajor
      ? MakeMap(b.data_ptr(), K, N, G, b.stride(1), G > 1 ? b.stride(0) : b.stride(1) * b.size(1), bn)
      : MakeMap(b.data_ptr(), N, K, G, b.stride(1), G > 1 ? b.stride(0) : b.stride(1) * b.size(1), kBlockK);

  // Every output but the redirected-row stores leaves through TMA; the tensor maps clip
  // ragged M / N edges and follow the row and group strides of C.
  const bool tma_store = p.row_ptrs == nullptr;
  CUtensorMap tc{}, tx{};
  if (tma_store) {
    const int64_t c_group = G > 1 ? p.c_batch : p.ldc * M;
    tc = MakeMap(out3.data_ptr(), N, M, G, p.ldc, c_group, 64);
    tx = p.aux ? MakeMap(p.aux, N, M, G, p.ldc, c_group, 64) : tc;
  }

  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  if (bn256) {
    if (tma_store) Dispatch<256, true>(a_kmajor, b_kmajor, ta, tb, tc, tx, p, sms, stream);
    else Dispatch<256, false>(a_kmajor, b_kmajor, ta, tb, tc, tx, p, sms, stream);
  } else {
    if (tma_store) Dispatch<128, true>(a_kmajor, b_kmajor, ta, tb, tc, tx, p, sms, stream);
    else Dispatch<128, false>(a_kmajor, b_kmajor, ta, tb, tc, tx, p, sms, stream);
  }
  return out;
}

}  // namespace lb
