// Hopper (sm_90a) flash attention with a learned Toeplitz (T5) relative-position bias
// (SURVEY K7/K8; reference semantics `gshard_builder.py:2697-2804,1431-1514`).
//
//   O[b,i,h,:] = softmax_j( scale·q_i·k_j + rel[h, i-j+L-1] + mask(b,i,j) ) · v_j
//
// mask(b,i,j) is built in registers from packed-input metadata: keys are visible iff they
// are in the query's (non-zero) segment and, for decoders, not in its future
// (segment_pos[j] <= segment_pos[i]).  Neither the [B,H,L,L] bias, nor S, P, dP, dS ever
// reach HBM; the gradient of the bias table is folded into the backward kernel.
//
// Both kernels use the same recipe: operand tiles [128 x 128] bf16 arrive by TMA as two
// [128 rows x 64 cols] SWIZZLE_128B chunks into a shared-memory ring fed by one producer
// thread; two consumer warpgroups issue wgmma (fp32 accumulators in registers) and do the
// softmax math between the GEMMs. The same physical smem layout serves as a K-major
// operand (rows = M/N index) or an MN-major operand (rows = K index) by changing only the
// descriptor and the wgmma transpose bit, so no transposes are ever materialised.
//
// Grouped-query / multi-query attention: k and v may have Hk heads with H % Hk == 0; query
// head h reads KV head h / G, G = H / Hk (the convention of `_ExpandKv` and decode_attn.cu).
// With Hk == H every kernel does exactly what the multi-head kernels did.
//
// Soft-capped logits and an extra logit (GShard `atten_logit_cap`, `attention_extra_logit`):
//
//   z_ij = cap·tanh(scale·q_i·k_j / cap) + rel[h, i-j+L-1] + mask(b,i,j)
//   O_i  = Σ_j softmax(z_i ∪ {extra})_j · v_j      (the extra slot has value 0)
//
// The cap applies to scale·q·k only; the bias and the mask are added after it. Both are
// compile-time specialisations (flash_fwd_kernel<kCap, kExtra>, flash_bwd_kernel<kCap>), so the
// default instantiations are the plain kernels. The extra logit needs no backward code: lse
// already counts it and delta = Σ dO∘O is right because the extra slot's value is 0.
//
// Layouts: q, dO [B, L, H, D=128] and k, v [B, L, Hk, D] bf16 views (strides (*, *, D, 1));
// O [B, L, H, D] and dK, dV [B, L, Hk, D] contiguous bf16;  dq_part [Jc, B, L, H, D] fp32;
// dk_part, dv_part [S, B, L, Hk, D] fp32 (only when the group is split, S > 1);  lse, delta
// [B, H, L] fp32;  rel / drel [H, 2L-1] fp32;  segment ids / positions [B, L] int32 (optional).

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda.h>
#include <cuda_bf16.h>
#include <torch/extension.h>

#include "ptx.cuh"
#include "registry.h"
#include "tmap.h"

namespace lb {
namespace {

constexpr int kT = 128;                      // tile edge (queries / keys)
constexpr int kD = 128;                      // head dim
constexpr int kChunk = kT * 64 * 2;          // [128 x 64] SW128 chunk = 16 KiB
constexpr int kTile = 2 * kChunk;            // [128 x 128] bf16 operand = 32 KiB
constexpr int kConsumers = 256;              // two warpgroups (warps 0..7)
constexpr int kThreads = kConsumers + 128;   // + the TMA producer warpgroup (warps 8..11)
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
constexpr float kMasked = -1.0e9f;           // additive mask value (log2 domain, finite)

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float lg2(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// tanh(u) = 1 - 2r with r = 1 / (1 + e^{2u}), from a = 2u·log2e: one ex2 and one reciprocal,
// with an absolute error near fp32 rounding for every u (tanh.approx.f32 is only good to about
// 2^-11 relative, which a logit near a cap of 50 would feel). 1 - tanh(u)^2 = 4r(1 - r).
__device__ __forceinline__ float tanh_r(float a, float& r) {
  r = rcp(1.f + ex2(a));
  return fmaf(-2.f, r, 1.f);
}
// Explicit shared-space accesses: the tile base is re-aligned through integer arithmetic,
// after which the compiler can only emit *generic* LD/ST for C++ pointers into it.
__device__ __forceinline__ float lds_f32(uint32_t a) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ int lds_s32(uint32_t a) {
  int v;
  asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts_f32(uint32_t a, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory");
}
__device__ __forceinline__ void sts_f32x2(uint32_t a, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ void sts_s32(uint32_t a, int v) {
  asm volatile("st.shared.s32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}

// Byte offset of the bf16 pair (col, col + 1) of row r in a SW128 operand whose rows hold 64
// columns (128 B); 64-column chunks of `chunk_bytes` each (col < 64 for a single chunk).
__device__ __forceinline__ uint32_t sw128_off(int r, int col, uint32_t chunk_bytes) {
  const int c = col & 63;
  return static_cast<uint32_t>(col >> 6) * chunk_bytes +
         static_cast<uint32_t>(r * 128 + (((c >> 3) ^ (r & 7)) << 4) + (c & 7) * 2);
}
__device__ __forceinline__ void sts_b32(uint32_t a, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ uint64_t kdesc(uint32_t a) { return make_smem_desc_sw128(a, 16, 1024); }
__device__ __forceinline__ uint64_t mndesc(uint32_t a) { return make_smem_desc_sw128(a, kChunk, 1024); }

__device__ __forceinline__ void load_tile(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                          int h, int row0, int b) {
  tma_load_3d(dst, map, bar, h * kD, row0, b);
  tma_load_3d(dst + kChunk, map, bar, h * kD + 64, row0, b);
}

struct MaskInfo {
  const int* seg;        // [B, L] or nullptr (single segment, nothing padded)
  const int* pos;        // [B, L] or nullptr (position = index)
  const int4* blk;       // [B, L/128] (pos_min, pos_max, seg_min, seg_max) or nullptr
  int causal;
};

// Per-128-row summary of the packed-input metadata; lets every CTA skip (query block, key
// block) pairs in which nothing can be visible — the causal upper triangle, but also
// blocks that only hold other segments — without assuming anything about the positions.
__device__ __forceinline__ int4 block_meta(const MaskInfo& m, int b, int nblk, int blk) {
  if (m.blk != nullptr) return m.blk[b * nblk + blk];
  return make_int4(blk * kT, blk * kT + kT - 1, 1, 1);
}
// Every (query, key) pair of the two blocks is visible: no per-element mask needed.
__device__ __forceinline__ bool pair_full(const MaskInfo& m, const int4& qm, const int4& km) {
  return qm.z == qm.w && km.z == km.w && qm.z == km.z && qm.z != 0 &&
         (!m.causal || qm.x >= km.y);
}
__device__ __forceinline__ bool pair_visible(const MaskInfo& m, const int4& qm, const int4& km) {
  if (qm.w == 0 || km.w == 0) return false;                  // a block of pure padding
  if (km.w < qm.z || km.z > qm.w) return false;              // disjoint segment-id ranges
  if (m.causal && qm.y < km.x) return false;                 // every key lies in the future
  return true;
}

// ================================================================== forward ==
struct FwdParams {
  const float* rel;      // [H, 2L-1] or nullptr
  MaskInfo mask;
  __nv_bfloat16* out;    // [B, L, H, D]
  float* lse;            // [B, H, L] natural log
  int B, H, L;
  int G;                 // query heads per KV head
  float scale;
  float cap_l2;          // kCap: cap·log2e
  float cap_a;           // kCap: 2·scale·log2e / cap, so that tanh(scale·s / cap) = tanh_r(s·cap_a)
  float extra_l2;        // kExtra: extra·log2e
  float extra;           // kExtra: the extra logit
};

// smem: Q | (K, V) x 2 stages | P x 2 warpgroups (16 KiB each) + barriers / per-block tables.
constexpr size_t kFwdSmem = kTile * 6 + 4096 + 1024;

// K/V blocks stream through a two-stage TMA ring while each warpgroup runs
//   S = Q·K^T (wgmma, registers) | online softmax | P (bf16) -> smem | O += P·V (wgmma)
// on its 64 query rows. CTA = (query block, query head h, b); K/V come from KV head h / G.
// The heads of a group are adjacent in blockIdx.y, so their K/V tiles are re-read from L2.
template <bool kCap, bool kExtra>
__global__ void __launch_bounds__(kThreads, 1)
flash_fwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                 const __grid_constant__ CUtensorMap map_v, const FwdParams p) {
  const int nblk = p.L / kT;
  const int i_blk = nblk - 1 - static_cast<int>(blockIdx.x);      // heavy (long) rows first
  const int h = blockIdx.y, b = blockIdx.z;
  const int i0 = i_blk * kT;
  const int4 qmeta = block_meta(p.mask, b, nblk, i_blk);

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const uint32_t s_q = smem_u32(smem);
  const uint32_t s_kv = s_q + kTile;                         // stage s: K at +2s·kTile, V behind it
  const uint32_t s_p = s_kv + 4 * kTile;                     // warpgroup g: +g·kTile/2
  uint8_t* meta = smem + kTile * 6;
  uint64_t* bars = reinterpret_cast<uint64_t*>(meta);
  uint64_t* q_bar = bars;                 // 1
  uint64_t* kv_full = bars + 1;           // 2
  uint64_t* kv_empty = bars + 3;          // 2
  const uint32_t s_rel = smem_u32(meta + 128);              // float [256]
  const uint32_t s_seg = s_rel + 1024;                      // int [128]
  const uint32_t s_pos = s_seg + 512;                       // int [128]

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == kConsumers) {
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_k);
    tma_prefetch_desc(&map_v);
    mbar_init(smem_u32(q_bar), 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(smem_u32(&kv_full[s]), 1);
      mbar_init(smem_u32(&kv_empty[s]), kConsumers / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp_idx >= kConsumers / 32) {
    // ============================ TMA producer ============================
    setmaxnreg_dec<40>();
    if (threadIdx.x == kConsumers) {
      mbar_arrive_expect_tx(smem_u32(q_bar), kTile);
      load_tile(s_q, &map_q, smem_u32(q_bar), h, i0, b);
      int it = 0;
      for (int jb = 0; jb < nblk; ++jb) {
        if (!pair_visible(p.mask, qmeta, block_meta(p.mask, b, nblk, jb))) continue;
        const int s = it & 1;
        mbar_wait(smem_u32(&kv_empty[s]), ((it >> 1) & 1) ^ 1);
        const uint32_t fb = smem_u32(&kv_full[s]);
        mbar_arrive_expect_tx(fb, 2 * kTile);
        load_tile(s_kv + 2 * s * kTile, &map_k, fb, h / p.G, jb * kT, b);
        load_tile(s_kv + (2 * s + 1) * kTile, &map_v, fb, h / p.G, jb * kT, b);
        ++it;
      }
    }
    return;
  }

  // ================= softmax warpgroups (2 x 128 threads) =================
  setmaxnreg_inc<232>();
  const int wg = warp_idx >> 2;
  const int pr0 = (warp_idx & 3) * 16 + (lane >> 2);       // rows pr0, pr0 + 8 of this warpgroup
  const int cq = (lane & 3) * 2;
  const long long bl = static_cast<long long>(b) * p.L;
  const float sl2 = p.scale * kLog2e;
  const uint32_t s_pw = s_p + wg * (kTile / 2);            // this warpgroup's P: [64 x 128]
  int segq[2], posq[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int qi = i0 + wg * 64 + pr0 + 8 * i;
    segq[i] = p.mask.seg ? p.mask.seg[bl + qi] : 1;
    posq[i] = p.mask.pos ? p.mask.pos[bl + qi] : qi;
  }
  float o[64];
#pragma unroll
  for (int c = 0; c < 64; ++c) o[c] = 0.f;
  // With an extra logit the running max starts at it: exp(extra - m) then stays <= 1 and is
  // added to l at the end, and a row that sees nothing keeps m = extra, l = 0.
  const float m0 = kExtra ? p.extra_l2 : -INFINITY;
  float m_run[2] = {m0, m0}, l_run[2] = {0.f, 0.f};
  mbar_wait(smem_u32(q_bar), 0);

  int it = 0;
  for (int jb = 0; jb < nblk; ++jb) {
    const int4 kmeta = block_meta(p.mask, b, nblk, jb);
    if (!pair_visible(p.mask, qmeta, kmeta)) continue;
    const int s = it & 1;
    const int j0 = jb * kT;
    const bool full = pair_full(p.mask, qmeta, kmeta);
    named_bar_sync(1, kConsumers);                 // the previous block's tables are free
    {
      const int t = threadIdx.x;
      if (t < 255)
        sts_f32(s_rel + t * 4,
                p.rel ? p.rel[static_cast<long long>(h) * (2 * p.L - 1) + (i0 - j0 + p.L - 1) - 127 + t] * kLog2e
                      : 0.f);
      if (t < 128) {
        sts_s32(s_seg + t * 4, p.mask.seg ? p.mask.seg[bl + j0 + t] : 1);
        sts_s32(s_pos + t * 4, p.mask.pos ? p.mask.pos[bl + j0 + t] : j0 + t);
      }
    }
    named_bar_sync(1, kConsumers);
    mbar_wait(smem_u32(&kv_full[s]), (it >> 1) & 1);
    const uint32_t s_k = s_kv + 2 * s * kTile, s_v = s_k + kTile;

    float sv[64];
#pragma unroll
    for (int c = 0; c < 64; ++c) sv[c] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
      wgmma_m64n128k16<0, 0>(sv, kdesc(s_q + (kk >> 2) * kChunk + wg * 8192 + (kk & 3) * 32),
                             kdesc(s_k + (kk >> 2) * kChunk + (kk & 3) * 32), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sv);

    float mloc[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int n = 0; n < 16; ++n) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int r = wg * 64 + pr0 + 8 * i;       // query row in the tile
          const int c = n * 8 + cq + j;              // key column in the tile
          float x;
          if constexpr (kCap) {
            float rr;
            x = fmaf(p.cap_l2, tanh_r(sv[4 * n + 2 * i + j] * p.cap_a, rr), lds_f32(s_rel + (r - c + 127) * 4));
          } else {
            x = fmaf(sv[4 * n + 2 * i + j], sl2, lds_f32(s_rel + (r - c + 127) * 4));
          }
          if (!full) {
            const bool vis = (segq[i] == lds_s32(s_seg + c * 4)) && (segq[i] != 0) &&
                             (!p.mask.causal || posq[i] >= lds_s32(s_pos + c * 4));
            x = vis ? x : kMasked;
          }
          sv[4 * n + 2 * i + j] = x;
          mloc[i] = fmaxf(mloc[i], x);
        }
      }
    }
    float alpha[2], m_new[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      mloc[i] = fmaxf(mloc[i], __shfl_xor_sync(0xffffffffu, mloc[i], 1));
      mloc[i] = fmaxf(mloc[i], __shfl_xor_sync(0xffffffffu, mloc[i], 2));
      m_new[i] = fmaxf(m_run[i], mloc[i]);
      alpha[i] = ex2(m_run[i] - m_new[i]);
      m_run[i] = m_new[i];
    }
    float lsum[2] = {0.f, 0.f};
#pragma unroll
    for (int n = 0; n < 16; ++n) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float p0 = ex2(sv[4 * n + 2 * i] - m_new[i]);
        const float p1 = ex2(sv[4 * n + 2 * i + 1] - m_new[i]);
        lsum[i] += p0 + p1;
        sts_b32(s_pw + sw128_off(pr0 + 8 * i, n * 8 + cq, 8192), pack_bf16x2(p0, p1));
        o[4 * n + 2 * i] *= alpha[i];
        o[4 * n + 2 * i + 1] *= alpha[i];
      }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) l_run[i] = l_run[i] * alpha[i] + lsum[i];
    fence_proxy_async();          // P (generic-proxy stores) → visible to wgmma's async proxy
    named_bar_sync(2 + wg, 128);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)                 // O += P·V  (V is MN-major: rows = keys)
      wgmma_m64n128k16<0, 1>(o, kdesc(s_pw + (kk >> 2) * 8192 + (kk & 3) * 32),
                             mndesc(s_v + kk * 2048), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&kv_empty[s]));
    ++it;
  }
  // ---- finalize: O / l, log-sum-exp ----
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float l = l_run[i];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    if constexpr (kExtra) l += ex2(p.extra_l2 - m_run[i]);   // >= 1 when the row sees nothing
    const float inv = l > 0.f ? 1.f / l : 0.f;      // query block that sees nothing: 0
    const int qi = i0 + wg * 64 + pr0 + 8 * i;
    __nv_bfloat16* dst = p.out + ((bl + qi) * p.H + h) * kD;
#pragma unroll
    for (int n = 0; n < 16; ++n)
      *reinterpret_cast<uint32_t*>(dst + n * 8 + cq) =
          pack_bf16x2(o[4 * n + 2 * i] * inv, o[4 * n + 2 * i + 1] * inv);
    // With an extra logit, relative to it, so that a row that sees nothing (m = extra, l = 1)
    // gets lse == extra exactly.
    if ((lane & 3) == 0)
      p.lse[(static_cast<long long>(b) * p.H + h) * p.L + qi] =
          kExtra ? fmaf((m_run[i] - p.extra_l2) + lg2(l), kLn2, p.extra)
                 : (l > 0.f ? (m_run[i] + lg2(l)) * kLn2 : 0.f);
  }
}

// ================================================================= backward ==
struct BwdParams {
  const float* rel;      // [H, 2L-1] or nullptr
  MaskInfo mask;
  const float* lse;      // [B, H, L]
  const float* delta;    // [B, H, L]
  float* dq_part;        // [Jc, B, L, H, D] fp32: dQ of each key block of this launch
  __nv_bfloat16* dk;     // [B, L, Hk, D] (S == 1)
  __nv_bfloat16* dv;     // [B, L, Hk, D] (S == 1)
  float* dk_part;        // [S, B, L, Hk, D] fp32 (S > 1, else nullptr)
  float* dv_part;        // [S, B, L, Hk, D] fp32 (S > 1, else nullptr)
  float* drel_part;      // [B, H, Jc, 2L-1] fp32, zero-initialised (or nullptr)
  int B, H, L;
  int Hk, G, S;          // KV heads, query heads per KV head, runs per group
  int j_begin, jc;       // this launch covers key blocks [j_begin, j_begin + jc)
  float scale;
  float cap_l2, cap_a;   // kCap: as in FwdParams
};

// Key blocks per backward launch (the leading dimension of dq_part / drel_part).
constexpr int kJChunk = 8;
// The backward splits a group of query heads into S runs until one launch has at least this
// many CTAs (about four per SM of an H100 SXM); see flash_attn_bwd_splits.
constexpr int kBwdMinCtas = 512;

constexpr int kBwdStages = 2;
// Once the dK / dQ products have read it, the P/dS tile holds the folded fp32 dS^T of the
// half block for the dRel diagonal sums: [64 rows x 72 columns] (see flash_bwd_kernel).
constexpr int kDiagCols = 72;
constexpr int kPdsBytes = 64 * kDiagCols * 4;
static_assert(kPdsBytes >= kChunk, "the P/dS tile must hold one [128 x 64] bf16 chunk");
// K, V resident + 2 x (Q, dO) + the P/dS tile + barriers / tables.
constexpr size_t kBwdSmem = kTile * (2 + 2 * kBwdStages) + kPdsBytes + 8192 + 1024;

// CTA = (key block, h, b); warpgroup g owns keys [64g, 64g + 64) and keeps dK, dV for them in
// registers. Every visible query block is processed as two 64-row halves (FlashAttention-2
// order), with the transposed scores so that P^T / dS^T come out row = key:
//   S^T = K·Q^T, dP^T = V·dO^T | P^T = exp2(S^T - lse), dS^T = P^T∘(dP^T - delta) |
//   dV += P^T·dO | dK += dS^T·Q | dQ = dS·K -> this key block's slice of dq_part;
//   d rel[h, i-j+L-1] += Σ dS along diagonals -> this CTA's row of drel_part.
// Grouped KV heads: CTA = (key block, run r, b), where run r is the G/S query heads
// [r·G/S, (r+1)·G/S) of KV head r / S. The CTA walks (query head, visible query block) in
// that order and keeps dK, dV in registers over the whole run; lse, delta, the rel row and
// the dq_part / drel_part rows belong to the query head. S == 1: dK, dV leave as bf16; S > 1:
// as this run's slice of dk_part / dv_part, folded in run order by flash_dkv_fold_kernel.
// No atomics: the partials are folded in key-block order by the reduce kernels below, so
// the gradients are identical run to run.
// kCap: z = cap·tanh(s/cap) + rel, so dRel takes dS and dQ / dK take dS∘(1 - t²). P^T goes to
// the P/dS tile inside the element loop, which frees st[] to carry scale·(1 - t²) to the dS^T
// store while dpt[] keeps the plain dS for the diagonal sums: no third 32-float array.
template <bool kCap>
__global__ void __launch_bounds__(kThreads, 1)
flash_bwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                 const __grid_constant__ CUtensorMap map_v, const __grid_constant__ CUtensorMap map_do,
                 const BwdParams p) {
  const int nblk = p.L / kT;
  const int jrel = blockIdx.x;
  const int j_blk = p.j_begin + jrel;                         // key block (small j = long loop first)
  const int b = blockIdx.z;
  const int nh = p.G / p.S;                                   // query heads of this CTA's run
  const int h_first = blockIdx.y * nh;
  const int hkv = h_first / p.G;
  const int j0 = j_blk * kT;
  const int4 kmeta = block_meta(p.mask, b, nblk, j_blk);

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const uint32_t s_k = smem_u32(smem);
  const uint32_t s_v = s_k + kTile;
  const uint32_t s_qdo = s_v + kTile;                        // stage s: Q at +2s·kTile, dO behind it
  const uint32_t s_pds = s_qdo + 2 * kBwdStages * kTile;     // [128 keys x 64 queries], one chunk
  uint8_t* meta = smem + kTile * (2 + 2 * kBwdStages) + kPdsBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(meta);
  uint64_t* kv_bar = bars;
  uint64_t* full_bar = bars + 1;
  uint64_t* empty_bar = bars + 1 + kBwdStages;
  const uint32_t s_rel = smem_u32(meta + 128);                // float [256]
  const uint32_t s_seg = s_rel + 1024;                        // int [128]   (query block)
  const uint32_t s_pos = s_seg + 512;                         // int [128]
  const uint32_t s_lse = s_pos + 512;                         // float [128] (log2 domain)
  const uint32_t s_dlt = s_lse + 512;                         // float [128]
  const uint32_t s_diag = s_dlt + 512;                        // float [256]

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == kConsumers) {
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_k);
    tma_prefetch_desc(&map_v);
    tma_prefetch_desc(&map_do);
    mbar_init(smem_u32(kv_bar), 1);
    for (int s = 0; s < kBwdStages; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), kConsumers / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp_idx >= kConsumers / 32) {
    // ============================ TMA producer ============================
    setmaxnreg_dec<40>();
    if (threadIdx.x == kConsumers) {
      mbar_arrive_expect_tx(smem_u32(kv_bar), 2 * kTile);
      load_tile(s_k, &map_k, smem_u32(kv_bar), hkv, j0, b);
      load_tile(s_v, &map_v, smem_u32(kv_bar), hkv, j0, b);
      int it = 0;
      for (int step = 0; step < nh * nblk; ++step) {   // (query head, query block) in order
        const int h = h_first + step / nblk, ib = step % nblk;
        if (!pair_visible(p.mask, block_meta(p.mask, b, nblk, ib), kmeta)) continue;
        const int s = it % kBwdStages;
        mbar_wait(smem_u32(&empty_bar[s]), ((it / kBwdStages) & 1) ^ 1);
        const uint32_t fb = smem_u32(&full_bar[s]);
        mbar_arrive_expect_tx(fb, 2 * kTile);
        load_tile(s_qdo + (2 * s) * kTile, &map_q, fb, h, ib * kT, b);
        load_tile(s_qdo + (2 * s + 1) * kTile, &map_do, fb, h, ib * kT, b);
        ++it;
      }
    }
    return;
  }

  // ================= dS / dQ warpgroups (2 x 128 threads) =================
  setmaxnreg_inc<232>();
  const int wg = warp_idx >> 2;
  const int w16 = (warp_idx & 3) * 16 + (lane >> 2);       // fragment row (+ 8 i)
  const int cq = (lane & 3) * 2;
  const long long bl = static_cast<long long>(b) * p.L;
  const float sl2 = p.scale * kLog2e;
  int segk[2], posk[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int kj = j0 + wg * 64 + w16 + 8 * i;
    segk[i] = p.mask.seg ? p.mask.seg[bl + kj] : 1;
    posk[i] = p.mask.pos ? p.mask.pos[bl + kj] : kj;
  }
  float dv[64], dk[64];
#pragma unroll
  for (int c = 0; c < 64; ++c) { dv[c] = 0.f; dk[c] = 0.f; }
  mbar_wait(smem_u32(kv_bar), 0);

  int it = 0;
  for (int step = 0; step < nh * nblk; ++step) {     // (query head, query block) in order
    const int h = h_first + step / nblk, ib = step % nblk;
    const int4 qmeta = block_meta(p.mask, b, nblk, ib);
    if (!pair_visible(p.mask, qmeta, kmeta)) continue;
    const long long bh = static_cast<long long>(b) * p.H + h;
    const int i0 = ib * kT;
    const int s = it % kBwdStages;
    const bool full = pair_full(p.mask, qmeta, kmeta);
    named_bar_sync(1, kConsumers);                 // previous tables / P-dS tile are free
    {
      const int t = threadIdx.x;
      if (t < 255) {
        sts_f32(s_rel + t * 4,
                p.rel ? p.rel[static_cast<long long>(h) * (2 * p.L - 1) + (i0 - j0 + p.L - 1) - 127 + t] * kLog2e
                      : 0.f);
        sts_f32(s_diag + t * 4, 0.f);
      }
      if (t < 128) {
        sts_s32(s_seg + t * 4, p.mask.seg ? p.mask.seg[bl + i0 + t] : 1);
        sts_s32(s_pos + t * 4, p.mask.pos ? p.mask.pos[bl + i0 + t] : i0 + t);
        sts_f32(s_lse + t * 4, p.lse[bh * p.L + i0 + t] * kLog2e);
        sts_f32(s_dlt + t * 4, p.delta[bh * p.L + i0 + t]);
      }
    }
    named_bar_sync(1, kConsumers);
    mbar_wait(smem_u32(&full_bar[s]), (it / kBwdStages) & 1);
    const uint32_t sq = s_qdo + (2 * s) * kTile, sdo = sq + kTile;

#pragma unroll 1
    for (int hq = 0; hq < 2; ++hq) {
      if (hq == 1) named_bar_sync(1, kConsumers);  // both warpgroups' dQ MMAs left the P/dS tile
      float st[32], dpt[32];   // written by the first MMA of each chain (scale-d = 0)
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)               // S^T = K_g · Q_hq^T
        wgmma_m64n64k16<0, 0>(st, kdesc(s_k + (kk >> 2) * kChunk + wg * 8192 + (kk & 3) * 32),
                              kdesc(sq + (kk >> 2) * kChunk + hq * 8192 + (kk & 3) * 32), kk != 0);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)               // dP^T = V_g · dO_hq^T
        wgmma_m64n64k16<0, 0>(dpt, kdesc(s_v + (kk >> 2) * kChunk + wg * 8192 + (kk & 3) * 32),
                              kdesc(sdo + (kk >> 2) * kChunk + hq * 8192 + (kk & 3) * 32), kk != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(st);
      wgmma_fence_regs(dpt);
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        float pv[2][2];        // kCap: P^T of the thread's (row i, column j) at this n
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          // The column's tables are read once for both of the thread's key rows.
          const int qc = hq * 64 + n * 8 + cq + j;   // query column in the tile
          const float lse_c = lds_f32(s_lse + qc * 4), dlt_c = lds_f32(s_dlt + qc * 4);
          int seg_c = 1, pos_c = 0;
          if (!full) {
            seg_c = lds_s32(s_seg + qc * 4);
            pos_c = lds_s32(s_pos + qc * 4);
          }
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int e = 4 * n + 2 * i + j;
            const int kr = wg * 64 + w16 + 8 * i;    // key row in the tile
            float x, rr = 0.f;
            if constexpr (kCap)
              x = fmaf(p.cap_l2, tanh_r(st[e] * p.cap_a, rr), lds_f32(s_rel + (qc - kr + 127) * 4));
            else
              x = fmaf(st[e], sl2, lds_f32(s_rel + (qc - kr + 127) * 4));
            const bool vis = full || ((seg_c == segk[i]) && (segk[i] != 0) &&
                                      (!p.mask.causal || pos_c >= posk[i]));
            const float pr = vis ? ex2(x - lse_c) : 0.f;
            const float ds = pr * (dpt[e] - dlt_c);
            if constexpr (kCap) {
              pv[i][j] = pr;
              st[e] = (4.f * rr) * (1.f - rr) * p.scale;   // scale·(1 - t²)
            } else {
              st[e] = pr;
            }
            dpt[e] = ds;
          }
        }
        if constexpr (kCap) {
#pragma unroll
          for (int i = 0; i < 2; ++i)
            sts_b32(s_pds + sw128_off(wg * 64 + w16 + 8 * i, n * 8 + cq, kChunk),
                    pack_bf16x2(pv[i][0], pv[i][1]));
        }
      }
      if constexpr (!kCap) {
#pragma unroll
        for (int n = 0; n < 8; ++n)
#pragma unroll
          for (int i = 0; i < 2; ++i)
            sts_b32(s_pds + sw128_off(wg * 64 + w16 + 8 * i, n * 8 + cq, kChunk),
                    pack_bf16x2(st[4 * n + 2 * i], st[4 * n + 2 * i + 1]));
      }
      fence_proxy_async();
      named_bar_sync(2 + wg, 128);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)               // dV += P^T_g · dO_hq  (dO MN-major)
        wgmma_m64n128k16<0, 1>(dv, kdesc(s_pds + wg * 8192 + kk * 32),
                               mndesc(sdo + hq * 8192 + kk * 2048), 1);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(dv);
      named_bar_sync(2 + wg, 128);                 // P^T rows of this warpgroup are consumed
#pragma unroll
      for (int n = 0; n < 8; ++n)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int e = 4 * n + 2 * i;
          if constexpr (kCap)
            sts_b32(s_pds + sw128_off(wg * 64 + w16 + 8 * i, n * 8 + cq, kChunk),
                    pack_bf16x2(dpt[e] * st[e], dpt[e + 1] * st[e + 1]));
          else
            sts_b32(s_pds + sw128_off(wg * 64 + w16 + 8 * i, n * 8 + cq, kChunk),
                    pack_bf16x2(dpt[e] * p.scale, dpt[e + 1] * p.scale));
        }
      fence_proxy_async();
      named_bar_sync(1, kConsumers);               // dQ reads every key row of dS^T
      float dq[32];            // written by the first dQ MMA (scale-d = 0)
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)               // dK += dS^T_g · Q_hq  (Q MN-major)
        wgmma_m64n128k16<0, 1>(dk, kdesc(s_pds + wg * 8192 + kk * 32),
                               mndesc(sq + hq * 8192 + kk * 2048), 1);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)               // dQ[:, 64g..] = dS · K[:, 64g..]  (both MN-major)
        wgmma_m64n64k16<1, 1>(dq, mndesc(s_pds + kk * 2048), mndesc(s_k + wg * kChunk + kk * 2048), kk != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(dk);
      wgmma_fence_regs(dq);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int qi = i0 + hq * 64 + w16 + 8 * i;
        float* dst = p.dq_part + ((static_cast<long long>(jrel) * p.B * p.L + bl + qi) * p.H + h) * kD +
                     wg * 64 + cq;
#pragma unroll
        for (int n = 0; n < 8; ++n)
          *reinterpret_cast<float2*>(dst + n * 8) = make_float2(dq[4 * n + 2 * i], dq[4 * n + 2 * i + 1]);
      }
      if (p.drel_part != nullptr) {
        // Fixed-order diagonal sums of this half's unrounded fp32 dS^T [128 keys x 64
        // queries], in one round through the free P/dS tile. A thread's rows k and k + 8 meet
        // the same diagonals 8 columns apart, so it first adds (n, i = 0) and (n + 1, i = 1)
        // in registers: row 8w + r of the folded slab is key 16w + r of warp w, and its column
        // 8 + c holds query column c = -8..63 of that key's diagonals (c - key). The row
        // stride of 72 floats keeps both the float2 stores and the diagonal reads free of
        // bank conflicts. Thread t < 191 then sums diagonal (query - key) = t - 127 over the
        // 64 rows, in four interleaved chains combined in a fixed order.
        named_bar_sync(1, kConsumers);             // every MMA has left the tile
        {
          const uint32_t row = s_pds + (warp_idx * 8 + (lane >> 2)) * (kDiagCols * 4);
#pragma unroll
          for (int m = -1; m < 8; ++m) {
            float x[2];
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              x[j] = m >= 0 ? dpt[4 * m + j] : 0.f;
              if (m < 7) x[j] += dpt[4 * (m + 1) + 2 + j];
            }
            sts_f32x2(row + (8 * (m + 1) + cq) * 4, x[0], x[1]);
          }
        }
        named_bar_sync(1, kConsumers);
        const int t = threadIdx.x;
        if (t < 191) {
          const int dl = t - 127;
          float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int rho = 0; rho < 64; ++rho) {
            const int col = dl + (rho >> 3) * 16 + (rho & 7) + 8;
            const bool in = col >= 0 && col < kDiagCols;
            const float x = lds_f32(s_pds + (rho * kDiagCols + (in ? col : 0)) * 4);
            acc[rho & 3] += in ? x : 0.f;
          }
          const uint32_t a = s_diag + (hq * 64 + dl + 127) * 4;
          sts_f32(a, lds_f32(a) + ((acc[0] + acc[1]) + (acc[2] + acc[3])));
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&empty_bar[s]));
    if (p.drel_part != nullptr) {
      // Consecutive query blocks overlap on 127 diagonals; the barrier orders the two adds.
      named_bar_sync(1, kConsumers);
      const int t = threadIdx.x;
      float* dr = p.drel_part + ((bh * p.jc + jrel) * (2 * p.L - 1)) + (i0 - j0) + (p.L - 1) - 127;
      if (t < 255) dr[t] += lds_f32(s_diag + t * 4);
    }
    ++it;
  }
  // ---- dK, dV: registers → bf16 (or this run's fp32 partial) → global (row = key); zero
  // when no query of the run sees the block ----
  if (p.dk_part != nullptr) {
    const long long part = static_cast<long long>(blockIdx.y % p.S) * p.B * p.L;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const long long orow = ((part + bl + j0 + wg * 64 + w16 + 8 * i) * p.Hk + hkv) * kD + cq;
#pragma unroll
      for (int n = 0; n < 16; ++n) {
        *reinterpret_cast<float2*>(p.dv_part + orow + n * 8) = make_float2(dv[4 * n + 2 * i], dv[4 * n + 2 * i + 1]);
        *reinterpret_cast<float2*>(p.dk_part + orow + n * 8) = make_float2(dk[4 * n + 2 * i], dk[4 * n + 2 * i + 1]);
      }
    }
    return;
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const long long orow = ((bl + j0 + wg * 64 + w16 + 8 * i) * p.Hk + hkv) * kD + cq;
#pragma unroll
    for (int n = 0; n < 16; ++n) {
      *reinterpret_cast<uint32_t*>(p.dv + orow + n * 8) =
          pack_bf16x2(dv[4 * n + 2 * i], dv[4 * n + 2 * i + 1]);
      *reinterpret_cast<uint32_t*>(p.dk + orow + n * 8) =
          pack_bf16x2(dk[4 * n + 2 * i], dk[4 * n + 2 * i + 1]);
    }
  }
}

// (pos_min, pos_max, seg_min, seg_max) of every 128-row block; one warp per block.
__global__ void __launch_bounds__(128)
flash_blkmeta_kernel(const int* __restrict__ seg, const int* __restrict__ pos,
                     int4* __restrict__ out, int n_blocks, int blocks_per_row) {
  const int blk = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (blk >= n_blocks) return;
  const int row0 = (blk % blocks_per_row) * kT;
  int pmin = 0x7fffffff, pmax = -0x7fffffff, smin = 0x7fffffff, smax = -0x7fffffff;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const long long idx = static_cast<long long>(blk) * kT + lane * 4 + t;
    const int sv = seg ? seg[idx] : 1;
    const int pv = pos ? pos[idx] : row0 + lane * 4 + t;
    pmin = min(pmin, pv); pmax = max(pmax, pv);
    smin = min(smin, sv); smax = max(smax, sv);
  }
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) {
    pmin = min(pmin, __shfl_xor_sync(0xffffffffu, pmin, m));
    pmax = max(pmax, __shfl_xor_sync(0xffffffffu, pmax, m));
    smin = min(smin, __shfl_xor_sync(0xffffffffu, smin, m));
    smax = max(smax, __shfl_xor_sync(0xffffffffu, smax, m));
  }
  if (lane == 0) out[blk] = make_int4(pmin, pmax, smin, smax);
}

// delta[b,h,l] = Σ_d dO[b,l,h,d]·O[b,l,h,d]   (both [B, L, H, D] contiguous)
__global__ void __launch_bounds__(256)
flash_delta_kernel(const __nv_bfloat16* __restrict__ d_o, const __nv_bfloat16* __restrict__ o,
                   float* __restrict__ delta, int B, int L, int H) {
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= static_cast<long long>(B) * L * H) return;
  const int h = static_cast<int>(row % H);
  const long long bl = row / H;
  const int l = static_cast<int>(bl % L);
  const int b = static_cast<int>(bl / L);
  const uint2 a = *reinterpret_cast<const uint2*>(d_o + row * 128 + lane * 4);
  const uint2 c = *reinterpret_cast<const uint2*>(o + row * 128 + lane * 4);
  const float2 a0 = unpack_bf16x2(a.x), a1 = unpack_bf16x2(a.y);
  const float2 c0 = unpack_bf16x2(c.x), c1 = unpack_bf16x2(c.y);
  float s = a0.x * c0.x + a0.y * c0.y + a1.x * c1.x + a1.y * c1.y;
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
  if (lane == 0) delta[(static_cast<long long>(b) * H + h) * L + l] = s;
}

// dq_acc[b, l, h, :] += Σ over the launch's key blocks j visible from l's block, in order of j.
// When the launch covers every key block (dq_acc == nullptr) the sum starts from 0 and goes
// straight to the bf16 dq, which is what accumulating into a zeroed dq_acc and casting it
// would give, without the fp32 round trip.
__global__ void __launch_bounds__(256)
flash_dq_reduce_kernel(const float4* __restrict__ part, float4* __restrict__ dq_acc,
                       uint2* __restrict__ dq, MaskInfo mask, int B, int L, int H, int j_begin,
                       int jc) {
  const long long n4 = static_cast<long long>(B) * L * H * (kD / 4);
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= n4) return;
  const long long row = idx / (H * (kD / 4));                 // b * L + l
  const int b = static_cast<int>(row / L);
  const int nblk = L / kT;
  const int4 qm = block_meta(mask, b, nblk, static_cast<int>(row % L) / kT);
  float4 acc = dq_acc != nullptr ? dq_acc[idx] : make_float4(0.f, 0.f, 0.f, 0.f);
  for (int jr = 0; jr < jc; ++jr) {
    if (!pair_visible(mask, qm, block_meta(mask, b, nblk, j_begin + jr))) continue;
    const float4 v = part[static_cast<long long>(jr) * n4 + idx];
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  if (dq_acc != nullptr)
    dq_acc[idx] = acc;
  else
    dq[idx] = make_uint2(pack_bf16x2(acc.x, acc.y), pack_bf16x2(acc.z, acc.w));
}

// drel[h, t] += Σ_b Σ_j drel_part[b, h, j, t], in order of b, then j.
__global__ void __launch_bounds__(256)
flash_drel_reduce_kernel(const float* __restrict__ part, float* __restrict__ drel, int B, int H,
                         int jc, int n) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int h = blockIdx.y;
  if (t >= n) return;
  float s = 0.f;
  for (int b = 0; b < B; ++b)
    for (int jr = 0; jr < jc; ++jr) s += part[((static_cast<long long>(b) * H + h) * jc + jr) * n + t];
  drel[static_cast<long long>(h) * n + t] += s;
}

// dq (bf16) = dq_acc (fp32)
__global__ void __launch_bounds__(256)
flash_cast_kernel(const float4* __restrict__ src, uint2* __restrict__ dst, long long n4) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = src[i];
    uint2 o;
    o.x = pack_bf16x2(v.x, v.y);
    o.y = pack_bf16x2(v.z, v.w);
    dst[i] = o;
  }
}

// dk, dv (bf16) = Σ_s dk_part[s], Σ_s dv_part[s] in fp32, in order of the run s.
__global__ void __launch_bounds__(256)
flash_dkv_fold_kernel(const float4* __restrict__ dk_part, const float4* __restrict__ dv_part,
                      uint2* __restrict__ dk, uint2* __restrict__ dv, long long n4, int splits) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 a = dk_part[i], c = dv_part[i];
  for (int s = 1; s < splits; ++s) {
    const float4 x = dk_part[s * n4 + i], y = dv_part[s * n4 + i];
    a.x += x.x; a.y += x.y; a.z += x.z; a.w += x.w;
    c.x += y.x; c.y += y.y; c.z += y.z; c.w += y.w;
  }
  dk[i] = make_uint2(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w));
  dv[i] = make_uint2(pack_bf16x2(c.x, c.y), pack_bf16x2(c.z, c.w));
}

// t is a bf16 view of shape `sizes` with strides (*, *, 128, 1) and 16-byte aligned rows.
void CheckQkv(const char* op, const torch::Tensor& t, torch::IntArrayRef sizes, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == torch::kBFloat16 && t.dim() == 4 &&
                  t.sizes() == sizes && t.stride(3) == 1 && t.stride(2) == kD &&
                  t.stride(1) % 8 == 0 && t.stride(0) % 8 == 0 &&
                  reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0,
              op, ": ", name, " must be a bf16 ", sizes,
              " view with strides (*, *, 128, 1) and 16-byte aligned rows, got ", t.sizes());
}

bool Given(const c10::optional<torch::Tensor>& t) { return t.has_value() && t->defined(); }

const int* IntPtr(const c10::optional<torch::Tensor>& t) {
  return Given(t) ? t->data_ptr<int>() : nullptr;
}

// Argument checks of both entry points, made before anything is allocated or launched: every
// tensor the kernels read or write is on q's device (a host `rel` would otherwise reach the
// kernel as a host pointer), k and v are [B, L, Hk, 128] with H % Hk == 0, and rel / seg /
// pos / out / d_out / lse have the shapes the kernels index. `out`, `d_out` and `lse` are
// given by the backward only.
void CheckArgs(const char* op, const torch::Tensor& q, const torch::Tensor& k,
               const torch::Tensor& v, const c10::optional<torch::Tensor>& rel,
               const c10::optional<torch::Tensor>& seg, const c10::optional<torch::Tensor>& pos,
               const torch::Tensor* out = nullptr, const torch::Tensor* d_out = nullptr,
               const torch::Tensor* lse = nullptr) {
  TORCH_CHECK(q.is_cuda() && q.dim() == 4 && q.size(3) == kD && q.size(1) % kT == 0 &&
                  q.size(1) <= 32768,
              op, ": q must be a CUDA [B, L, H, 128] tensor with L % 128 == 0 and L <= 32768");
  const int64_t B = q.size(0), L = q.size(1), H = q.size(2);
  auto on_q = [&](const torch::Tensor& t, const char* name) {
    TORCH_CHECK(t.device() == q.device(), op, ": ", name, " is on ", t.device(),
                " but q is on ", q.device());
  };
  CheckQkv(op, q, q.sizes(), "q");
  on_q(k, "k");
  TORCH_CHECK(k.dim() == 4 && k.size(0) == B && k.size(1) == L && k.size(2) >= 1 &&
                  H % k.size(2) == 0 && k.size(3) == kD,
              op, ": k must be [B, L, Hk, 128] with q's B and L and H % Hk == 0; q is ",
              q.sizes(), ", k is ", k.sizes());
  CheckQkv(op, k, k.sizes(), "k");
  on_q(v, "v");
  CheckQkv(op, v, k.sizes(), "v");
  if (Given(rel)) {
    on_q(*rel, "rel");
    TORCH_CHECK(rel->scalar_type() == torch::kFloat32 && rel->dim() == 2 && rel->size(0) == H &&
                    rel->size(1) == 2 * L - 1, op, ": rel must be fp32 [H, 2L-1]");
  }
  for (const auto* t : {&seg, &pos}) {
    if (!Given(*t)) continue;
    const char* name = t == &seg ? "segment_ids" : "segment_pos";
    on_q(**t, name);
    TORCH_CHECK((*t)->scalar_type() == torch::kInt32 && (*t)->is_contiguous() &&
                    (*t)->sizes() == torch::IntArrayRef({B, L}),
                op, ": ", name, " must be contiguous int32 [B, L]");
  }
  if (out != nullptr) {
    on_q(*out, "out");
    TORCH_CHECK(out->scalar_type() == torch::kBFloat16 && out->is_contiguous() &&
                    out->sizes() == q.sizes(), op, ": out must be contiguous bf16 [B, L, H, 128]");
  }
  if (d_out != nullptr) {
    on_q(*d_out, "d_out");
    TORCH_CHECK(d_out->scalar_type() == torch::kBFloat16 && d_out->sizes() == q.sizes(),
                op, ": d_out must be bf16 [B, L, H, 128]");
  }
  if (lse != nullptr) {
    on_q(*lse, "lse");
    TORCH_CHECK(lse->scalar_type() == torch::kFloat32 && lse->is_contiguous() &&
                    lse->sizes() == torch::IntArrayRef({B, H, L}),
                op, ": lse must be contiguous fp32 [B, H, L]");
  }
}

// [B, L/128, 4] int32 block summaries (empty tensor when neither seg nor pos is given).
torch::Tensor BlockMeta(const int* seg, const int* pos, int64_t B, int64_t L,
                        const torch::TensorOptions& opts) {
  if (seg == nullptr && pos == nullptr) return torch::empty({0}, opts.dtype(torch::kInt32));
  auto out = torch::empty({B, L / kT, 4}, opts.dtype(torch::kInt32));
  const int n = static_cast<int>(B * (L / kT));
  flash_blkmeta_kernel<<<(n + 3) / 4, 128, 0, at::cuda::getCurrentCUDAStream()>>>(
      seg, pos, reinterpret_cast<int4*>(out.data_ptr<int>()), n, static_cast<int>(L / kT));
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return out;
}

// A negative or non-finite cap, or a non-finite extra logit, is refused before anything is
// allocated or launched.
void CheckLogitOptions(const char* op, double logit_cap, const c10::optional<double>& extra_logit) {
  TORCH_CHECK(std::isfinite(logit_cap) && logit_cap >= 0.0, op,
              ": logit_cap must be finite and >= 0 (0 = no cap), got ", logit_cap);
  TORCH_CHECK(!extra_logit.has_value() || std::isfinite(*extra_logit), op,
              ": extra_logit must be finite, got ", extra_logit.value_or(0.0));
}

// One launch of an instantiation; each instantiation sets its own dynamic shared-memory limit
// the first time it is launched.
template <bool kCap, bool kExtra>
void LaunchFwd(dim3 grid, cudaStream_t stream, const CUtensorMap& mq, const CUtensorMap& mk,
               const CUtensorMap& mv, const FwdParams& p) {
  static bool configured = false;
  if (!configured) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(flash_fwd_kernel<kCap, kExtra>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(kFwdSmem)));
    configured = true;
  }
  flash_fwd_kernel<kCap, kExtra><<<grid, kThreads, kFwdSmem, stream>>>(mq, mk, mv, p);
}

template <bool kCap>
void LaunchBwd(dim3 grid, cudaStream_t stream, const CUtensorMap& mq, const CUtensorMap& mk,
               const CUtensorMap& mv, const CUtensorMap& mdo, const BwdParams& p) {
  static bool configured = false;
  if (!configured) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(flash_bwd_kernel<kCap>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(kBwdSmem)));
    configured = true;
  }
  flash_bwd_kernel<kCap><<<grid, kThreads, kBwdSmem, stream>>>(mq, mk, mv, mdo, p);
}

}  // namespace

// Runs S into which the backward splits each group of G = H / Hk query heads: the smallest
// divisor of G for which one key-block launch, min(L/128, kJChunk) x (Hk·S) x B CTAs, has at
// least kBwdMinCtas CTAs (G when none has). It depends on the shapes only, so a problem is
// split, and its dK / dV summed, the same way on every card. Always 1 for multi-head attention.
int64_t flash_attn_bwd_splits(int64_t B, int64_t L, int64_t H, int64_t Hk) {
  TORCH_CHECK(B >= 1 && L >= kT && Hk >= 1 && H % Hk == 0,
              "flash_attn_bwd_splits: needs B >= 1, L >= 128 and H % Hk == 0");
  const int64_t g = H / Hk;
  const int64_t ctas = std::min<int64_t>(L / kT, kJChunk) * Hk * B;
  int64_t s = 1;
  while (s < g && (g % s != 0 || ctas * s < kBwdMinCtas)) ++s;
  return s;
}

// Returns (out [B,L,H,D] bf16, lse [B,H,L] fp32). logit_cap > 0 soft-caps scale·q·k;
// extra_logit adds one logit of value 0 to every softmax (lse counts it).
std::vector<torch::Tensor> flash_attn_fwd(const torch::Tensor& q, const torch::Tensor& k,
                                          const torch::Tensor& v,
                                          const c10::optional<torch::Tensor>& rel,
                                          const c10::optional<torch::Tensor>& seg,
                                          const c10::optional<torch::Tensor>& pos, double scale,
                                          bool causal, double logit_cap,
                                          const c10::optional<double>& extra_logit) {
  CheckArgs("flash_attn_fwd", q, k, v, rel, seg, pos);
  CheckLogitOptions("flash_attn_fwd", logit_cap, extra_logit);
  const int64_t B = q.size(0), L = q.size(1), H = q.size(2);
  const c10::cuda::CUDAGuard guard(q.device());
  FwdParams p;
  p.rel = nullptr;
  torch::Tensor relc;
  if (Given(rel)) {
    relc = rel->contiguous();
    p.rel = relc.data_ptr<float>();
  }
  p.mask.seg = IntPtr(seg);
  p.mask.pos = IntPtr(pos);
  p.mask.causal = causal ? 1 : 0;
  auto blk = BlockMeta(p.mask.seg, p.mask.pos, B, L, q.options());
  p.mask.blk = blk.numel() ? reinterpret_cast<const int4*>(blk.data_ptr<int>()) : nullptr;
  auto out = torch::empty({B, L, H, kD}, q.options());
  auto lse = torch::empty({B, H, L}, q.options().dtype(torch::kFloat32));
  p.out = reinterpret_cast<__nv_bfloat16*>(out.data_ptr());
  p.lse = lse.data_ptr<float>();
  p.B = static_cast<int>(B); p.H = static_cast<int>(H); p.L = static_cast<int>(L);
  p.G = static_cast<int>(H / k.size(2));
  p.scale = static_cast<float>(scale);
  const bool cap = logit_cap > 0.0, extra = extra_logit.has_value();
  p.cap_l2 = cap ? static_cast<float>(logit_cap * kLog2e) : 0.f;
  p.cap_a = cap ? static_cast<float>(2.0 * scale * kLog2e / logit_cap) : 0.f;
  p.extra = extra ? static_cast<float>(*extra_logit) : 0.f;
  p.extra_l2 = p.extra * kLog2e;
  auto mk = [&](const torch::Tensor& t) {
    return MakeMap(t.data_ptr(), t.size(2) * kD, L, B, t.stride(1), t.stride(0), kT);
  };
  const CUtensorMap mq = mk(q), mkk = mk(k), mv = mk(v);
  dim3 grid(static_cast<unsigned>(L / kT), static_cast<unsigned>(H), static_cast<unsigned>(B));
  auto stream = at::cuda::getCurrentCUDAStream();
  if (cap && extra)
    LaunchFwd<true, true>(grid, stream, mq, mkk, mv, p);
  else if (cap)
    LaunchFwd<true, false>(grid, stream, mq, mkk, mv, p);
  else if (extra)
    LaunchFwd<false, true>(grid, stream, mq, mkk, mv, p);
  else
    LaunchFwd<false, false>(grid, stream, mq, mkk, mv, p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return {out, lse};
}

// Returns (dq [B,L,H,D], dk, dv [B,L,Hk,D] bf16, drel [H,2L-1] fp32 or an empty tensor).
// logit_cap is the forward's; an extra logit needs nothing here (lse already counts it).
std::vector<torch::Tensor> flash_attn_bwd(const torch::Tensor& q, const torch::Tensor& k,
                                          const torch::Tensor& v, const torch::Tensor& out,
                                          const torch::Tensor& d_out, const torch::Tensor& lse,
                                          const c10::optional<torch::Tensor>& rel,
                                          const c10::optional<torch::Tensor>& seg,
                                          const c10::optional<torch::Tensor>& pos, double scale,
                                          bool causal, bool need_drel, double logit_cap) {
  CheckArgs("flash_attn_bwd", q, k, v, rel, seg, pos, &out, &d_out, &lse);
  CheckLogitOptions("flash_attn_bwd", logit_cap, c10::nullopt);
  const int64_t B = q.size(0), L = q.size(1), H = q.size(2), Hk = k.size(2);
  const int64_t S = flash_attn_bwd_splits(B, L, H, Hk);
  const c10::cuda::CUDAGuard guard(q.device());
  auto d_o = d_out.contiguous();
  CheckQkv("flash_attn_bwd", d_o, q.sizes(), "dO");
  auto stream = at::cuda::getCurrentCUDAStream();
  auto delta = torch::empty({B, H, L}, lse.options());
  {
    const long long rows = B * L * H;
    flash_delta_kernel<<<static_cast<int>((rows * 32 + 255) / 256), 256, 0, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(d_o.data_ptr()),
        reinterpret_cast<const __nv_bfloat16*>(out.data_ptr()), delta.data_ptr<float>(),
        static_cast<int>(B), static_cast<int>(L), static_cast<int>(H));
    C10_CUDA_KERNEL_LAUNCH_CHECK();
    CountLaunch();
  }
  BwdParams p;
  p.rel = nullptr;
  torch::Tensor relc, drel;
  if (Given(rel)) {
    relc = rel->contiguous();
    p.rel = relc.data_ptr<float>();
  }
  if (need_drel) {
    drel = torch::zeros({H, 2 * L - 1}, lse.options());
  } else {
    drel = torch::empty({0}, lse.options());
  }
  p.mask.seg = IntPtr(seg);
  p.mask.pos = IntPtr(pos);
  p.mask.causal = causal ? 1 : 0;
  auto blk = BlockMeta(p.mask.seg, p.mask.pos, B, L, q.options());
  p.mask.blk = blk.numel() ? reinterpret_cast<const int4*>(blk.data_ptr<int>()) : nullptr;
  // Key blocks go in launches of up to kJChunk; each launch's per-key-block dQ / dRel partials
  // are folded in key-block order, so the result does not depend on CTA scheduling. With one
  // launch the dQ fold writes bf16 dq directly; with several it adds into an fp32 dq_acc.
  const int nblk = static_cast<int>(L / kT);
  const int jc_max = nblk < kJChunk ? nblk : kJChunk;
  const bool one_launch = jc_max == nblk;
  auto dq = torch::empty({B, L, H, kD}, q.options());
  torch::Tensor dq_acc;
  if (!one_launch) dq_acc = torch::zeros({B, L, H, kD}, lse.options());
  auto dk = torch::empty({B, L, Hk, kD}, q.options());
  auto dv = torch::empty({B, L, Hk, kD}, q.options());
  // S > 1: every CTA writes its key block's rows of its run's slice, so no zero-fill is needed.
  torch::Tensor dk_part, dv_part;
  if (S > 1) {
    dk_part = torch::empty({S, B, L, Hk, kD}, lse.options());
    dv_part = torch::empty({S, B, L, Hk, kD}, lse.options());
  }
  p.lse = lse.data_ptr<float>();
  p.delta = delta.data_ptr<float>();
  p.dk = reinterpret_cast<__nv_bfloat16*>(dk.data_ptr());
  p.dv = reinterpret_cast<__nv_bfloat16*>(dv.data_ptr());
  p.dk_part = S > 1 ? dk_part.data_ptr<float>() : nullptr;
  p.dv_part = S > 1 ? dv_part.data_ptr<float>() : nullptr;
  p.B = static_cast<int>(B); p.H = static_cast<int>(H); p.L = static_cast<int>(L);
  p.Hk = static_cast<int>(Hk); p.G = static_cast<int>(H / Hk); p.S = static_cast<int>(S);
  p.scale = static_cast<float>(scale);
  const bool cap = logit_cap > 0.0;
  p.cap_l2 = cap ? static_cast<float>(logit_cap * kLog2e) : 0.f;
  p.cap_a = cap ? static_cast<float>(2.0 * scale * kLog2e / logit_cap) : 0.f;
  auto mk = [&](const torch::Tensor& t) {
    return MakeMap(t.data_ptr(), t.size(2) * kD, L, B, t.stride(1), t.stride(0), kT);
  };
  const CUtensorMap mq = mk(q), mkk = mk(k), mv = mk(v), mdo = mk(d_o);
  auto dq_part = torch::empty({jc_max, B, L, H, kD}, lse.options());
  p.dq_part = dq_part.data_ptr<float>();
  for (int j_begin = 0; j_begin < nblk; j_begin += jc_max) {
    const int jc = (nblk - j_begin) < jc_max ? (nblk - j_begin) : jc_max;
    p.j_begin = j_begin;
    p.jc = jc;
    torch::Tensor drel_part;
    p.drel_part = nullptr;
    if (need_drel) {
      drel_part = torch::zeros({B, H, jc, 2 * L - 1}, lse.options());
      p.drel_part = drel_part.data_ptr<float>();
    }
    dim3 grid(static_cast<unsigned>(jc), static_cast<unsigned>(Hk * S), static_cast<unsigned>(B));
    if (cap)
      LaunchBwd<true>(grid, stream, mq, mkk, mv, mdo, p);
    else
      LaunchBwd<false>(grid, stream, mq, mkk, mv, mdo, p);
    C10_CUDA_KERNEL_LAUNCH_CHECK();
    const long long n4 = B * L * H * (kD / 4);
    flash_dq_reduce_kernel<<<static_cast<int>((n4 + 255) / 256), 256, 0, stream>>>(
        reinterpret_cast<const float4*>(p.dq_part),
        one_launch ? nullptr : reinterpret_cast<float4*>(dq_acc.data_ptr<float>()),
        one_launch ? reinterpret_cast<uint2*>(dq.data_ptr()) : nullptr, p.mask, p.B, p.L, p.H,
        j_begin, jc);
    C10_CUDA_KERNEL_LAUNCH_CHECK();
    CountLaunch(2);
    if (need_drel) {
      const int n = static_cast<int>(2 * L - 1);
      flash_drel_reduce_kernel<<<dim3((n + 255) / 256, static_cast<unsigned>(H)), 256, 0, stream>>>(
          p.drel_part, drel.data_ptr<float>(), p.B, p.H, jc, n);
      C10_CUDA_KERNEL_LAUNCH_CHECK();
      CountLaunch();
    }
  }
  if (S > 1) {
    const long long n4 = B * L * Hk * (kD / 4);
    flash_dkv_fold_kernel<<<static_cast<int>((n4 + 255) / 256), 256, 0, stream>>>(
        reinterpret_cast<const float4*>(p.dk_part), reinterpret_cast<const float4*>(p.dv_part),
        reinterpret_cast<uint2*>(dk.data_ptr()), reinterpret_cast<uint2*>(dv.data_ptr()), n4,
        p.S);
    C10_CUDA_KERNEL_LAUNCH_CHECK();
    CountLaunch();
  }
  if (!one_launch) {
    const long long n4 = dq.numel() / 4;
    const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
    long long blocks = (n4 + 255) / 256;
    if (blocks > sms * 8) blocks = sms * 8;
    flash_cast_kernel<<<static_cast<int>(blocks), 256, 0, stream>>>(
        reinterpret_cast<const float4*>(dq_acc.data_ptr<float>()),
        reinterpret_cast<uint2*>(dq.data_ptr()), n4);
    C10_CUDA_KERNEL_LAUNCH_CHECK();
    CountLaunch();
  }
  return {dq, dk, dv, drel};
}

}  // namespace lb

LB_REGISTER(flash_attn) {
  m.def("flash_attn_fwd", &lb::flash_attn_fwd, py::arg("q"), py::arg("k"), py::arg("v"),
        py::arg("rel"), py::arg("seg"), py::arg("pos"), py::arg("scale"), py::arg("causal"),
        py::arg("logit_cap") = 0.0, py::arg("extra_logit") = py::none());
  m.def("flash_attn_bwd", &lb::flash_attn_bwd, py::arg("q"), py::arg("k"), py::arg("v"),
        py::arg("out"), py::arg("d_out"), py::arg("lse"), py::arg("rel"), py::arg("seg"),
        py::arg("pos"), py::arg("scale"), py::arg("causal"), py::arg("need_drel"),
        py::arg("logit_cap") = 0.0);
  m.def("flash_attn_bwd_splits", &lb::flash_attn_bwd_splits, py::arg("B"), py::arg("L"),
        py::arg("H"), py::arg("Hk"));
}
