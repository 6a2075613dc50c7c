// Split-KV ("flash-decoding") attention for one query token per sequence against a bf16 KV
// cache, fused with the in-place append of the step's key / value row.
//
//   out[b,h,:] = Σ_{j ≤ t} softmax_j( scale·q[b,h]·k[b,j,h/G] + rel[h, t-j+T-1] ) · v[b,j,h/G]
//
// with G = H / Hk query heads per KV head (grouped / multi-query attention, the
// `repeat_interleave` convention). Logits are fp32 dot products of the bf16 values, the
// softmax is fp32 and P·V accumulates in fp32; the output is rounded to bf16 once.
//
// Grid (S, Hk·⌈G/16⌉, B): CTA (s, ·, b) covers keys [s·chunk, (s+1)·chunk) of one KV head for
// up to 16 of its query heads, so every K/V tile is read from HBM once for all of them. The
// chunk depends on (B, Hk, G, T) only, never on `t` (a device scalar), so a captured CUDA graph
// replays correctly for every step; CTAs whose chunk starts after `t` exit at once.
//
// Inside a CTA each of the 4 warps streams its own 32-key tiles (round robin over the chunk)
// through a 2-stage cp.async ring: lane = key for the logits, lane = 4 head dims for P·V. The
// warps' (m, ℓ, o) are folded in warp order, then either normalised into the output (S == 1)
// or written as fp32 partials that `decode_attn_combine_kernel` folds in split order. No
// float atomics: the result is bit-identical from run to run.
//
// Cache append: the CTA whose chunk contains t writes k_new / v_new into row t. Its warps take
// key t from k_new / v_new directly and no other CTA reads row t, so there is no
// read-after-write hazard. For t outside [0, T) nothing is written and all T keys are
// visible; the `rel` index is clamped to [0, 2T-2].
//
// Layouts: q, out [B, H, 128]; k_new, v_new [B, Hk, 128]; k_cache, v_cache [B, T, Hk, 128]
// (all contiguous bf16); t 0-dim int32 / int64; rel [H, 2T-1] fp32; partials m, ℓ [B, H, S]
// and o [B, H, S, 128] fp32.

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda_bf16.h>
#include <torch/extension.h>

#include <algorithm>

#include "ptx.cuh"
#include "registry.h"

namespace lb {
namespace {

constexpr int kD = 128;                          // head dim
constexpr int kWarps = 4;
constexpr int kThreads = kWarps * 32;
constexpr int kKeys = 32;                        // keys per warp tile
constexpr int kCtaKeys = kWarps * kKeys;         // the chunk is a multiple of this
constexpr int kStages = 2;
constexpr int kRowBytes = kD * 2;                // one bf16 row = 16 chunks of 16 bytes
constexpr int kTileBytes = kKeys * kRowBytes;    // 8 KiB per operand
constexpr int kStageBytes = 2 * kTileBytes;      // K + V
constexpr int kMaxG = 16;                        // query heads per CTA

struct Params {
  const __nv_bfloat16* q;
  const __nv_bfloat16* k_new;
  const __nv_bfloat16* v_new;
  __nv_bfloat16* k_cache;
  __nv_bfloat16* v_cache;
  const void* t;
  const float* rel;       // nullptr: no bias
  float* m_part;          // S > 1 only
  float* l_part;
  float* o_part;
  __nv_bfloat16* out;
  int H, Hk, T, chunk, S, t64;
  float scale;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src),
               "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() {
  asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

__device__ __forceinline__ float warp_max(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, o));
  return x;
}
__device__ __forceinline__ float warp_sum(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

__device__ __forceinline__ long long LoadT(const Params& p) {
  return p.t64 ? *static_cast<const long long*>(p.t) : *static_cast<const int*>(p.t);
}
// Number of visible keys: t + 1 for t in [0, T), all T otherwise.
__device__ __forceinline__ int Visible(long long t, int T) {
  return (t >= 0 && t < T) ? static_cast<int>(t) + 1 : T;
}

// Byte offset of 16-byte chunk c of tile row r: XOR swizzle so that 8 lanes reading the same
// chunk of 8 consecutive rows (logits) hit 8 distinct bank groups.
__device__ __forceinline__ int Swz(int r, int c) { return r * kRowBytes + ((c ^ (r & 7)) << 4); }

// The flat-beam kernel below runs the split kernel's two inner loops through these helpers.
// s[g] = q[g]·k[lane] over the 128 head dims of a swizzled 32-key tile (lane = key).
template <int kG>
__device__ __forceinline__ void TileLogits(const unsigned char* kt, const float* q_s, int lane,
                                           float (&s)[kG]) {
#pragma unroll
  for (int g = 0; g < kG; ++g) s[g] = 0.f;
  const float4* q4 = reinterpret_cast<const float4*>(q_s);
#pragma unroll 2
  for (int c = 0; c < kD / 8; ++c) {
    const uint4 raw = *reinterpret_cast<const uint4*>(kt + Swz(lane, c));
    const float2 k0 = unpack_bf16x2(raw.x), k1 = unpack_bf16x2(raw.y);
    const float2 k2 = unpack_bf16x2(raw.z), k3 = unpack_bf16x2(raw.w);
#pragma unroll
    for (int g = 0; g < kG; ++g) {
      const float4 a = q4[g * (kD / 4) + 2 * c], e = q4[g * (kD / 4) + 2 * c + 1];
      float acc = s[g];
      acc = fmaf(a.x, k0.x, acc); acc = fmaf(a.y, k0.y, acc);
      acc = fmaf(a.z, k1.x, acc); acc = fmaf(a.w, k1.y, acc);
      acc = fmaf(e.x, k2.x, acc); acc = fmaf(e.y, k2.y, acc);
      acc = fmaf(e.z, k3.x, acc); acc = fmaf(e.w, k3.y, acc);
      s[g] = acc;
    }
  }
}

// o[g] += Σ_r pw[g][r] · v[r] for the lane's head dims [4·lane, 4·lane + 4) of a 32-key tile.
template <int kG>
__device__ __forceinline__ void TilePV(const unsigned char* vt, const float* pw, int lane,
                                       float (&o)[kG][4]) {
  const float4* p4 = reinterpret_cast<const float4*>(pw);
  const int vo = ((lane & 1) << 3);
#pragma unroll 2
  for (int r4 = 0; r4 < kKeys / 4; ++r4) {
    float vf[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int r = r4 * 4 + u;
      const uint2 raw = *reinterpret_cast<const uint2*>(vt + Swz(r, lane >> 1) + vo);
      const float2 a = unpack_bf16x2(raw.x), e = unpack_bf16x2(raw.y);
      vf[u][0] = a.x; vf[u][1] = a.y; vf[u][2] = e.x; vf[u][3] = e.y;
    }
#pragma unroll
    for (int g = 0; g < kG; ++g) {
      const float4 pp = p4[g * (kKeys / 4) + r4];
#pragma unroll
      for (int d = 0; d < 4; ++d) {
        float acc = o[g][d];
        acc = fmaf(pp.x, vf[0][d], acc); acc = fmaf(pp.y, vf[1][d], acc);
        acc = fmaf(pp.z, vf[2][d], acc); acc = fmaf(pp.w, vf[3][d], acc);
        o[g][d] = acc;
      }
    }
  }
}

template <int kG>
__global__ void __launch_bounds__(kThreads, 1) decode_attn_split_kernel(const Params p) {
  extern __shared__ __align__(128) unsigned char smem[];
  float* q_s = reinterpret_cast<float*>(smem + kWarps * kStages * kStageBytes);   // [kG][kD]
  float* p_s = q_s + kG * kD;                                                     // [kWarps][kG][kKeys]

  const int split = blockIdx.x, b = blockIdx.z;
  const int ngrp = gridDim.y / p.Hk;
  const int kh = blockIdx.y / ngrp, grp = blockIdx.y % ngrp;
  const long long t = LoadT(p);
  const int n_vis = Visible(t, p.T);
  const int wr = (t >= 0 && t < p.T) ? static_cast<int>(t) : -1;   // row to append
  const int c0 = split * p.chunk;
  if (c0 >= n_vis) return;
  const int c1 = min(c0 + p.chunk, n_vis);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int G = p.H / p.Hk;
  const int gcnt = min(kG, G - grp * kMaxG);
  const int h0 = kh * G + grp * kMaxG;
  const long long rs = static_cast<long long>(p.Hk) * kD;            // cache row stride
  const __nv_bfloat16* kc = p.k_cache + (static_cast<long long>(b) * p.T * p.Hk + kh) * kD;
  const __nv_bfloat16* vc = p.v_cache + (static_cast<long long>(b) * p.T * p.Hk + kh) * kD;
  const __nv_bfloat16* kn = p.k_new + (static_cast<long long>(b) * p.Hk + kh) * kD;
  const __nv_bfloat16* vn = p.v_new + (static_cast<long long>(b) * p.Hk + kh) * kD;

  if (wr >= c0 && grp == 0 && tid < 32) {   // c1 == wr + 1 here: row t is in this chunk
    const int c = tid & 15;
    const __nv_bfloat16* src = (tid < 16 ? kn : vn) + c * 8;
    __nv_bfloat16* dst = (tid < 16 ? p.k_cache : p.v_cache) +
                         (static_cast<long long>(b) * p.T * p.Hk + kh) * kD + wr * rs + c * 8;
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
  }
  for (int i = tid; i < kG * kD; i += kThreads) {
    const int g = i / kD;
    q_s[i] = g < gcnt ? __bfloat162float(p.q[(static_cast<long long>(b) * p.H + h0 + g) * kD + i % kD])
                      : 0.f;
  }
  __syncthreads();

  unsigned char* ring = smem + warp * kStages * kStageBytes;
  auto issue = [&](int j0, int stage) {
    unsigned char* kt = ring + stage * kStageBytes;
    unsigned char* vt = kt + kTileBytes;
#pragma unroll
    for (int i = 0; i < kKeys / 2; ++i) {
      const int r = (lane >> 4) + 2 * i, c = lane & 15, j = j0 + r;
      const bool ok = j < c1;
      const __nv_bfloat16* ks = j == wr ? kn : kc + (ok ? j : 0) * rs;
      const __nv_bfloat16* vs = j == wr ? vn : vc + (ok ? j : 0) * rs;
      cp_async16(smem_u32(kt + Swz(r, c)), ks + c * 8, ok ? 16 : 0);   // 0 bytes: zero fill
      cp_async16(smem_u32(vt + Swz(r, c)), vs + c * 8, ok ? 16 : 0);
    }
  };

  float m[kG], l[kG], o[kG][4];
#pragma unroll
  for (int g = 0; g < kG; ++g) {
    m[g] = -INFINITY;
    l[g] = 0.f;
    o[g][0] = o[g][1] = o[g][2] = o[g][3] = 0.f;
  }
  const int n_tiles = (c1 - c0 + kKeys - 1) / kKeys;
  const int relw = 2 * p.T - 1;
  float* pw = p_s + warp * kG * kKeys;
  if (warp < n_tiles) issue(c0 + warp * kKeys, 0);
  cp_async_commit();
  for (int ti = warp, it = 0; ti < n_tiles; ti += kWarps, ++it) {
    if (ti + kWarps < n_tiles) issue(c0 + (ti + kWarps) * kKeys, (it + 1) % kStages);
    cp_async_commit();
    cp_async_wait<1>();
    __syncwarp();
    const unsigned char* kt = ring + (it % kStages) * kStageBytes;
    const unsigned char* vt = kt + kTileBytes;

    // logits: lane = key
    const int j = c0 + ti * kKeys + lane;
    float s[kG];
#pragma unroll
    for (int g = 0; g < kG; ++g) s[g] = 0.f;
    const float4* q4 = reinterpret_cast<const float4*>(q_s);
#pragma unroll 2
    for (int c = 0; c < kD / 8; ++c) {
      const uint4 raw = *reinterpret_cast<const uint4*>(kt + Swz(lane, c));
      const float2 k0 = unpack_bf16x2(raw.x), k1 = unpack_bf16x2(raw.y);
      const float2 k2 = unpack_bf16x2(raw.z), k3 = unpack_bf16x2(raw.w);
#pragma unroll
      for (int g = 0; g < kG; ++g) {
        const float4 a = q4[g * (kD / 4) + 2 * c], e = q4[g * (kD / 4) + 2 * c + 1];
        float acc = s[g];
        acc = fmaf(a.x, k0.x, acc); acc = fmaf(a.y, k0.y, acc);
        acc = fmaf(a.z, k1.x, acc); acc = fmaf(a.w, k1.y, acc);
        acc = fmaf(e.x, k2.x, acc); acc = fmaf(e.y, k2.y, acc);
        acc = fmaf(e.z, k3.x, acc); acc = fmaf(e.w, k3.y, acc);
        s[g] = acc;
      }
    }
    const bool valid = j < c1;
    long long ri = t - j + p.T - 1;
    ri = ri < 0 ? 0 : (ri > relw - 1 ? relw - 1 : ri);
#pragma unroll
    for (int g = 0; g < kG; ++g) {
      float x = s[g] * p.scale;
      if (p.rel != nullptr && g < gcnt) x += p.rel[static_cast<long long>(h0 + g) * relw + ri];
      x = valid ? x : -INFINITY;
      const float m_new = fmaxf(m[g], warp_max(x));   // lane 0 is always a valid key
      const float alpha = __expf(m[g] - m_new);
      const float pv = __expf(x - m_new);
      m[g] = m_new;
      l[g] = l[g] * alpha + pv;                         // per-lane partial sum
      o[g][0] *= alpha; o[g][1] *= alpha; o[g][2] *= alpha; o[g][3] *= alpha;
      pw[g * kKeys + lane] = pv;
    }
    __syncwarp();

    // P·V: lane owns head dims [4·lane, 4·lane + 4)
    const float4* p4 = reinterpret_cast<const float4*>(pw);
    const int vo = ((lane & 1) << 3);
#pragma unroll 2
    for (int r4 = 0; r4 < kKeys / 4; ++r4) {
      float vf[4][4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int r = r4 * 4 + u;
        const uint2 raw = *reinterpret_cast<const uint2*>(vt + Swz(r, lane >> 1) + vo);
        const float2 a = unpack_bf16x2(raw.x), e = unpack_bf16x2(raw.y);
        vf[u][0] = a.x; vf[u][1] = a.y; vf[u][2] = e.x; vf[u][3] = e.y;
      }
#pragma unroll
      for (int g = 0; g < kG; ++g) {
        const float4 pp = p4[g * (kKeys / 4) + r4];
#pragma unroll
        for (int d = 0; d < 4; ++d) {
          float acc = o[g][d];
          acc = fmaf(pp.x, vf[0][d], acc); acc = fmaf(pp.y, vf[1][d], acc);
          acc = fmaf(pp.z, vf[2][d], acc); acc = fmaf(pp.w, vf[3][d], acc);
          o[g][d] = acc;
        }
      }
    }
    __syncwarp();   // the next iteration refills this stage and p_s
  }
  cp_async_wait<0>();
#pragma unroll
  for (int g = 0; g < kG; ++g) l[g] = warp_sum(l[g]);
  __syncthreads();   // every warp is done with the ring: reuse it for the warp fold

  float* wo = reinterpret_cast<float*>(smem);   // [kWarps][kG][kD]
  float* wm = wo + kWarps * kG * kD;           // [kWarps][kG]
  float* wl = wm + kWarps * kG;
#pragma unroll
  for (int g = 0; g < kG; ++g) {
    *reinterpret_cast<float4*>(wo + (warp * kG + g) * kD + 4 * lane) =
        make_float4(o[g][0], o[g][1], o[g][2], o[g][3]);
    if (lane == 0) {
      wm[warp * kG + g] = m[g];
      wl[warp * kG + g] = l[g];
    }
  }
  __syncthreads();

  const int d = tid;   // kThreads == kD
  for (int g = 0; g < gcnt; ++g) {
    float mx = -INFINITY;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) mx = fmaxf(mx, wm[w * kG + g]);
    float lsum = 0.f, osum = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {   // idle warps have m = -inf: weight 0
      const float e = __expf(wm[w * kG + g] - mx);
      lsum += wl[w * kG + g] * e;
      osum += wo[(w * kG + g) * kD + d] * e;
    }
    const long long bh = static_cast<long long>(b) * p.H + h0 + g;
    if (p.S == 1) {
      p.out[bh * kD + d] = __float2bfloat16_rn(osum / lsum);
    } else {
      p.o_part[(bh * p.S + split) * kD + d] = osum;
      if (d == 0) {
        p.m_part[bh * p.S + split] = mx;
        p.l_part[bh * p.S + split] = lsum;
      }
    }
  }
}

// Folds the live splits' partials of one (b, h) in split order.
__global__ void __launch_bounds__(kD) decode_attn_combine_kernel(const Params p) {
  const long long bh = blockIdx.x;
  const int n_live = (Visible(LoadT(p), p.T) + p.chunk - 1) / p.chunk;
  const float* m = p.m_part + bh * p.S;
  const float* l = p.l_part + bh * p.S;
  const float* o = p.o_part + bh * p.S * kD + threadIdx.x;
  float mx = -INFINITY;
  for (int s = 0; s < n_live; ++s) mx = fmaxf(mx, m[s]);
  float lsum = 0.f, osum = 0.f;
  for (int s = 0; s < n_live; ++s) {
    const float e = __expf(m[s] - mx);
    lsum += l[s] * e;
    osum += o[static_cast<long long>(s) * kD] * e;
  }
  p.out[bh * kD + threadIdx.x] = __float2bfloat16_rn(osum / lsum);
}

template <int kG>
constexpr int SmemBytes() {
  return kWarps * kStages * kStageBytes + kG * kD * 4 + kWarps * kG * kKeys * 4;
}

template <int kG>
void LaunchSplit(const Params& p, dim3 grid, cudaStream_t stream) {
  static bool configured = false;
  if (!configured) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(decode_attn_split_kernel<kG>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, SmemBytes<kG>()));
    configured = true;
  }
  decode_attn_split_kernel<kG><<<grid, kThreads, SmemBytes<kG>(), stream>>>(p);
}

void CheckBf16(const torch::Tensor& x, const char* name, const char* op = "decode_attn") {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == torch::kBFloat16 && x.is_contiguous() &&
                  x.size(-1) == kD && reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0,
              op, ": ", name, " must be a contiguous 16-byte aligned bf16 tensor with D = 128");
}

}  // namespace

// Keys per CTA: enough splits that B·Hk·⌈G/16⌉·S CTAs fill the SMs once, in multiples of 128.
namespace {
int64_t ChunkFor(int64_t units, int64_t T) {
  const int64_t sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  const int64_t want = std::max<int64_t>(1, (sms + units - 1) / units);
  const int64_t chunk = (T + want - 1) / want;
  return (chunk + kCtaKeys - 1) / kCtaKeys * kCtaKeys;
}
}  // namespace

int64_t decode_attn_chunk(int64_t B, int64_t H, int64_t Hk, int64_t T) {
  const int64_t ngrp = (H / Hk + kMaxG - 1) / kMaxG;
  return ChunkFor(B * Hk * ngrp, T);
}

// Returns out [B, H, 128] bf16; writes k_new / v_new into row t of the caches.
torch::Tensor decode_attn_fwd(const torch::Tensor& q, const torch::Tensor& k_new,
                              const torch::Tensor& v_new, const torch::Tensor& k_cache,
                              const torch::Tensor& v_cache, const torch::Tensor& t,
                              const c10::optional<torch::Tensor>& rel, double scale) {
  CheckBf16(q, "q"); CheckBf16(k_new, "k_new"); CheckBf16(v_new, "v_new");
  CheckBf16(k_cache, "k_cache"); CheckBf16(v_cache, "v_cache");
  TORCH_CHECK(q.dim() == 3 && k_cache.dim() == 4, "decode_attn: q [B,H,D], caches [B,T,Hk,D]");
  const int64_t B = q.size(0), H = q.size(1), T = k_cache.size(1), Hk = k_cache.size(2);
  TORCH_CHECK(k_cache.sizes() == v_cache.sizes() && k_cache.size(0) == B && T >= 1,
              "decode_attn: caches must both be [B, T, Hk, 128]");
  TORCH_CHECK(k_new.dim() == 3 && k_new.size(0) == B && k_new.size(1) == Hk &&
                  v_new.sizes() == k_new.sizes(), "decode_attn: k_new / v_new must be [B, Hk, 128]");
  TORCH_CHECK(Hk >= 1 && H % Hk == 0, "decode_attn: Hk must divide H");
  TORCH_CHECK(B <= 65535 && Hk * ((H / Hk + kMaxG - 1) / kMaxG) <= 65535 && T < (1 << 30),
              "decode_attn: shape out of range");
  TORCH_CHECK(t.is_cuda() && t.device() == q.device() && t.numel() == 1 &&
                  (t.scalar_type() == torch::kInt32 || t.scalar_type() == torch::kInt64),
              "decode_attn: t must be a 0-dim int32 / int64 tensor on the device of q");
  for (const auto* x : {&k_new, &v_new, &k_cache, &v_cache})
    TORCH_CHECK(x->device() == q.device(), "decode_attn: all tensors must be on one device");
  const c10::cuda::CUDAGuard guard(q.device());
  Params p;
  torch::Tensor relc;
  p.rel = nullptr;
  if (rel.has_value() && rel->defined()) {
    TORCH_CHECK(rel->is_cuda() && rel->scalar_type() == torch::kFloat32 && rel->dim() == 2 &&
                    rel->size(0) == H && rel->size(1) == 2 * T - 1,
                "decode_attn: rel must be fp32 [H, 2T-1]");
    relc = rel->contiguous();
    p.rel = relc.data_ptr<float>();
  }
  const int64_t G = H / Hk;
  const int64_t ngrp = (G + kMaxG - 1) / kMaxG;
  const int64_t chunk = decode_attn_chunk(B, H, Hk, T);
  const int64_t S = (T + chunk - 1) / chunk;
  auto out = torch::empty({B, H, kD}, q.options());
  torch::Tensor m_part, l_part, o_part;
  p.m_part = p.l_part = p.o_part = nullptr;
  if (S > 1) {
    const auto f32 = q.options().dtype(torch::kFloat32);
    m_part = torch::empty({B, H, S}, f32);
    l_part = torch::empty({B, H, S}, f32);
    o_part = torch::empty({B, H, S, kD}, f32);
    p.m_part = m_part.data_ptr<float>();
    p.l_part = l_part.data_ptr<float>();
    p.o_part = o_part.data_ptr<float>();
  }
  auto bf = [](const torch::Tensor& x) { return reinterpret_cast<__nv_bfloat16*>(x.data_ptr()); };
  p.q = bf(q); p.k_new = bf(k_new); p.v_new = bf(v_new);
  p.k_cache = bf(k_cache); p.v_cache = bf(v_cache); p.out = bf(out);
  p.t = t.data_ptr();
  p.t64 = t.scalar_type() == torch::kInt64 ? 1 : 0;
  p.H = static_cast<int>(H); p.Hk = static_cast<int>(Hk); p.T = static_cast<int>(T);
  p.chunk = static_cast<int>(chunk); p.S = static_cast<int>(S);
  p.scale = static_cast<float>(scale);
  const dim3 grid(static_cast<unsigned>(S), static_cast<unsigned>(Hk * ngrp), static_cast<unsigned>(B));
  auto stream = at::cuda::getCurrentCUDAStream();
  const int64_t gmax = std::min<int64_t>(G, kMaxG);
  if (gmax <= 1) LaunchSplit<1>(p, grid, stream);
  else if (gmax <= 2) LaunchSplit<2>(p, grid, stream);
  else if (gmax <= 4) LaunchSplit<4>(p, grid, stream);
  else if (gmax <= 8) LaunchSplit<8>(p, grid, stream);
  else LaunchSplit<16>(p, grid, stream);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  if (S > 1) {
    decode_attn_combine_kernel<<<static_cast<unsigned>(B * H), kD, 0, stream>>>(p);
    C10_CUDA_KERNEL_LAUNCH_CHECK();
    CountLaunch();
  }
  return out;
}

// ------------------------------------------------------------------ flat beam search ----
// K hypotheses per sequence share one token buffer (the KV cache). Each step appends their K
// tokens at rows slot0 … slot0+K-1, and hypothesis k attends over the rows whose bit is set in
// its visibility mask vis[b, k] (its prompt, its ancestors and itself):
//
//   out[b,k,h,:] = Σ_{j ∈ vis[b,k]} softmax_j( scale·q[b,k,h]·k[b,j,h/G]
//                                             + rel[h, qpos[b,k] - kpos[b,j] + N-1] ) · v[b,j,h/G]
//
// The kernel is the split-KV kernel above with (hypothesis, query head) pairs in place of
// query heads: a CTA serves up to 16 pairs of one KV head, pair i = k·G + (h mod G), so each
// K/V tile is read once for all K·G queries of its KV head. Only rows below slot0 + K can be
// visible, so CTAs whose chunk starts there exit at once; the launch shape depends on
// (B, K, H, Hk, N) only and slot0 is read on the device, so a captured step replays for every
// slot0. Rows slot0 … slot0+K-1 are taken from k_new / v_new by every CTA that reads them and
// written to the caches by the CTAs whose chunk holds them (key-head group 0), so no CTA reads
// a row another one writes. A 32-key tile that no pair of the CTA may see is not computed.
// A query that sees no key returns zeros.
//
// Layouts: q, out [B, K, H, 128]; k_new, v_new [B, K, Hk, 128]; caches [B, N, Hk, 128] (bf16,
// contiguous); slot0 0-dim int32 / int64; vis [B, K, ⌈N/32⌉] int32, bit j%32 of word j/32 for
// row j; qpos [B, K] and kpos [B, N] int32; rel [H, 2N-1] fp32; partials m, ℓ [B·K·H, S] and
// o [B·K·H, S, 128] fp32.
namespace {

struct BeamParams {
  const __nv_bfloat16* q;
  const __nv_bfloat16* k_new;
  const __nv_bfloat16* v_new;
  __nv_bfloat16* k_cache;
  __nv_bfloat16* v_cache;
  const void* slot0;
  const int* vis;
  const int* qpos;
  const int* kpos;
  const float* rel;       // nullptr: no bias
  float* m_part;          // S > 1 only
  float* l_part;
  float* o_part;
  __nv_bfloat16* out;
  int K, H, Hk, N, W, chunk, S, s64;
  float scale;
};

__device__ __forceinline__ long long LoadSlot0(const BeamParams& p) {
  return p.s64 ? *static_cast<const long long*>(p.slot0) : *static_cast<const int*>(p.slot0);
}
// Rows that may be visible: [0, slot0 + K) ∩ [0, N).
__device__ __forceinline__ int BeamLive(long long s0, int K, int N) {
  const long long e = s0 + K;
  return e <= 0 ? 0 : (e >= N ? N : static_cast<int>(e));
}
// The softmax max with -inf (no key seen yet) replaced by 0, so exp(x - m) stays finite.
__device__ __forceinline__ float SafeMax(float m) { return m == -INFINITY ? 0.f : m; }

template <int kG>
__global__ void __launch_bounds__(kThreads, 1) flat_beam_attn_kernel(const BeamParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  float* q_s = reinterpret_cast<float*>(smem + kWarps * kStages * kStageBytes);   // [kG][kD]
  float* p_s = q_s + kG * kD;                                                     // [kWarps][kG][kKeys]
  int* hyp_s = reinterpret_cast<int*>(p_s + kWarps * kG * kKeys);                 // [kG]
  int* qpos_s = hyp_s + kG;                                                       // [kG]
  unsigned* vis_s = reinterpret_cast<unsigned*>(qpos_s + kG);                     // [kWarps][kG]

  const int split = blockIdx.x, b = blockIdx.z;
  const int ngrp = gridDim.y / p.Hk;
  const int kh = blockIdx.y / ngrp, grp = blockIdx.y % ngrp;
  const long long s0 = LoadSlot0(p);
  const int n_live = BeamLive(s0, p.K, p.N);
  const int c0 = split * p.chunk;
  if (c0 >= n_live) return;
  const int c1 = min(c0 + p.chunk, n_live);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int G = p.H / p.Hk;
  const int gcnt = min(kG, p.K * G - grp * kMaxG);
  const long long rs = static_cast<long long>(p.Hk) * kD;            // cache row stride
  const long long cb = (static_cast<long long>(b) * p.N * p.Hk + kh) * kD;
  const __nv_bfloat16* kc = p.k_cache + cb;
  const __nv_bfloat16* vc = p.v_cache + cb;
  // row slot0 + i of this KV head in k_new / v_new
  const __nv_bfloat16* kn = p.k_new + (static_cast<long long>(b) * p.K * p.Hk + kh) * kD;
  const __nv_bfloat16* vn = p.v_new + (static_cast<long long>(b) * p.K * p.Hk + kh) * kD;
  const long long w_lo = s0 > c0 ? s0 : c0;
  const long long w_hi = s0 + p.K < c1 ? s0 + p.K : c1;

  if (grp == 0 && tid < 32) {   // append the rows of this chunk
    for (long long j = w_lo; j < w_hi; ++j) {
      const int c = tid & 15;
      const long long i = j - s0;
      const __nv_bfloat16* src = (tid < 16 ? kn : vn) + i * rs + c * 8;
      __nv_bfloat16* dst = (tid < 16 ? p.k_cache : p.v_cache) + cb + j * rs + c * 8;
      *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
    }
  }
  for (int i = tid; i < kG * kD; i += kThreads) {
    const int g = i / kD;
    float x = 0.f;
    if (g < gcnt) {
      const int pi = grp * kMaxG + g, hyp = pi / G, h = kh * G + pi % G;
      x = __bfloat162float(p.q[((static_cast<long long>(b) * p.K + hyp) * p.H + h) * kD + i % kD]);
    }
    q_s[i] = x;
  }
  if (tid < kG) {
    const int hyp = tid < gcnt ? (grp * kMaxG + tid) / G : 0;
    hyp_s[tid] = hyp;
    qpos_s[tid] = p.qpos[b * p.K + hyp];
  }
  __syncthreads();

  unsigned char* ring = smem + warp * kStages * kStageBytes;
  auto issue = [&](int j0, int stage) {
    unsigned char* kt = ring + stage * kStageBytes;
    unsigned char* vt = kt + kTileBytes;
#pragma unroll
    for (int i = 0; i < kKeys / 2; ++i) {
      const int r = (lane >> 4) + 2 * i, c = lane & 15, j = j0 + r;
      const bool ok = j < c1;
      const bool fresh = j >= s0 && j < s0 + p.K;
      const __nv_bfloat16* ks = fresh ? kn + (j - s0) * rs : kc + (ok ? j : 0) * rs;
      const __nv_bfloat16* vs = fresh ? vn + (j - s0) * rs : vc + (ok ? j : 0) * rs;
      cp_async16(smem_u32(kt + Swz(r, c)), ks + c * 8, ok ? 16 : 0);   // 0 bytes: zero fill
      cp_async16(smem_u32(vt + Swz(r, c)), vs + c * 8, ok ? 16 : 0);
    }
  };

  float m[kG], l[kG], o[kG][4];
#pragma unroll
  for (int g = 0; g < kG; ++g) {
    m[g] = -INFINITY;
    l[g] = 0.f;
    o[g][0] = o[g][1] = o[g][2] = o[g][3] = 0.f;
  }
  const int n_tiles = (c1 - c0 + kKeys - 1) / kKeys;
  const int relw = 2 * p.N - 1;
  float* pw = p_s + warp * kG * kKeys;
  unsigned* vw = vis_s + warp * kG;
  const int* vis_b = p.vis + static_cast<long long>(b) * p.K * p.W;
  if (warp < n_tiles) issue(c0 + warp * kKeys, 0);
  cp_async_commit();
  for (int ti = warp, it = 0; ti < n_tiles; ti += kWarps, ++it) {
    if (ti + kWarps < n_tiles) issue(c0 + (ti + kWarps) * kKeys, (it + 1) % kStages);
    cp_async_commit();
    const int j0 = c0 + ti * kKeys;   // a multiple of 32: one mask word per pair
    unsigned word = 0;
    if (lane < gcnt) word = static_cast<unsigned>(vis_b[hyp_s[lane] * p.W + (j0 >> 5)]);
    const bool any = __ballot_sync(0xffffffffu, word != 0) != 0;
    if (lane < kG) vw[lane] = word;
    cp_async_wait<1>();
    __syncwarp();
    if (any) {
      const unsigned char* kt = ring + (it % kStages) * kStageBytes;
      const unsigned char* vt = kt + kTileBytes;
      const int j = j0 + lane;
      float s[kG];
      TileLogits<kG>(kt, q_s, lane, s);
      const bool valid = j < c1;
      const int kp = (p.rel != nullptr && valid) ? p.kpos[static_cast<long long>(b) * p.N + j] : 0;
#pragma unroll
      for (int g = 0; g < kG; ++g) {
        float x = s[g] * p.scale;
        if (p.rel != nullptr && g < gcnt) {
          long long ri = static_cast<long long>(qpos_s[g]) - kp + p.N - 1;
          ri = ri < 0 ? 0 : (ri > relw - 1 ? relw - 1 : ri);
          const int h = kh * G + (grp * kMaxG + g) % G;
          x += p.rel[static_cast<long long>(h) * relw + ri];
        }
        x = (valid && ((vw[g] >> lane) & 1u)) ? x : -INFINITY;
        const float m_new = fmaxf(m[g], warp_max(x));
        const float ms = SafeMax(m_new);
        const float alpha = __expf(m[g] - ms);
        const float pv = __expf(x - ms);
        m[g] = m_new;
        l[g] = l[g] * alpha + pv;                         // per-lane partial sum
        o[g][0] *= alpha; o[g][1] *= alpha; o[g][2] *= alpha; o[g][3] *= alpha;
        pw[g * kKeys + lane] = pv;
      }
      __syncwarp();
      TilePV<kG>(vt, pw, lane, o);
    }
    __syncwarp();   // the next iteration refills this stage, p_s and the mask words
  }
  cp_async_wait<0>();
#pragma unroll
  for (int g = 0; g < kG; ++g) l[g] = warp_sum(l[g]);
  __syncthreads();   // every warp is done with the ring: reuse it for the warp fold

  float* wo = reinterpret_cast<float*>(smem);   // [kWarps][kG][kD]
  float* wm = wo + kWarps * kG * kD;           // [kWarps][kG]
  float* wl = wm + kWarps * kG;
#pragma unroll
  for (int g = 0; g < kG; ++g) {
    *reinterpret_cast<float4*>(wo + (warp * kG + g) * kD + 4 * lane) =
        make_float4(o[g][0], o[g][1], o[g][2], o[g][3]);
    if (lane == 0) {
      wm[warp * kG + g] = m[g];
      wl[warp * kG + g] = l[g];
    }
  }
  __syncthreads();

  const int d = tid;   // kThreads == kD
  for (int g = 0; g < gcnt; ++g) {
    float mx = -INFINITY;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) mx = fmaxf(mx, wm[w * kG + g]);
    mx = SafeMax(mx);
    float lsum = 0.f, osum = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {   // warps that saw no key have m = -inf: weight 0
      const float e = __expf(wm[w * kG + g] - mx);
      lsum += wl[w * kG + g] * e;
      osum += wo[(w * kG + g) * kD + d] * e;
    }
    const int pi = grp * kMaxG + g;
    const long long row = (static_cast<long long>(b) * p.K + pi / G) * p.H + kh * G + pi % G;
    if (p.S == 1) {
      p.out[row * kD + d] = __float2bfloat16_rn(lsum > 0.f ? osum / lsum : 0.f);
    } else {
      p.o_part[(row * p.S + split) * kD + d] = osum;
      if (d == 0) {
        p.m_part[row * p.S + split] = lsum > 0.f ? mx : -INFINITY;   // no key seen: weight 0
        p.l_part[row * p.S + split] = lsum;
      }
    }
  }
}

// Folds the live splits' partials of one (b, k, h) row in split order.
__global__ void __launch_bounds__(kD) flat_beam_attn_combine_kernel(const BeamParams p) {
  const long long row = blockIdx.x;
  const int n_live = (BeamLive(LoadSlot0(p), p.K, p.N) + p.chunk - 1) / p.chunk;
  const float* m = p.m_part + row * p.S;
  const float* l = p.l_part + row * p.S;
  const float* o = p.o_part + row * p.S * kD + threadIdx.x;
  float mx = -INFINITY;
  for (int s = 0; s < n_live; ++s) mx = fmaxf(mx, m[s]);
  mx = SafeMax(mx);
  float lsum = 0.f, osum = 0.f;
  for (int s = 0; s < n_live; ++s) {
    const float e = __expf(m[s] - mx);
    lsum += l[s] * e;
    osum += o[static_cast<long long>(s) * kD] * e;
  }
  p.out[row * kD + threadIdx.x] = __float2bfloat16_rn(lsum > 0.f ? osum / lsum : 0.f);
}

template <int kG>
constexpr int BeamSmemBytes() {
  return SmemBytes<kG>() + 2 * kG * 4 + kWarps * kG * 4;
}

template <int kG>
void LaunchBeam(const BeamParams& p, dim3 grid, cudaStream_t stream) {
  static bool configured = false;
  if (!configured) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(flat_beam_attn_kernel<kG>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        BeamSmemBytes<kG>()));
    configured = true;
  }
  flat_beam_attn_kernel<kG><<<grid, kThreads, BeamSmemBytes<kG>(), stream>>>(p);
}

void CheckInt32(const torch::Tensor& x, const torch::Tensor& q, const char* name,
                std::initializer_list<int64_t> shape) {
  TORCH_CHECK(x.is_cuda() && x.device() == q.device() && x.scalar_type() == torch::kInt32 &&
                  x.is_contiguous() && x.sizes() == c10::IntArrayRef(shape),
              "flat_beam_attn: ", name, " must be a contiguous int32 tensor of shape ",
              c10::IntArrayRef(shape), " on the device of q");
}

}  // namespace

// Keys per CTA of `flat_beam_attn_fwd`, chosen as for `decode_attn_fwd` with K·G pairs per KV head.
int64_t flat_beam_attn_chunk(int64_t B, int64_t K, int64_t H, int64_t Hk, int64_t N) {
  const int64_t ngrp = (K * (H / Hk) + kMaxG - 1) / kMaxG;
  return ChunkFor(B * Hk * ngrp, N);
}

// Returns out [B, K, H, 128] bf16; writes k_new / v_new [:, k] into row slot0 + k of the caches.
torch::Tensor flat_beam_attn_fwd(const torch::Tensor& q, const torch::Tensor& k_new,
                                 const torch::Tensor& v_new, const torch::Tensor& k_cache,
                                 const torch::Tensor& v_cache, const torch::Tensor& slot0,
                                 const torch::Tensor& vis, const torch::Tensor& qpos,
                                 const torch::Tensor& kpos, const c10::optional<torch::Tensor>& rel,
                                 double scale) {
  const char* op = "flat_beam_attn";
  CheckBf16(q, "q", op); CheckBf16(k_new, "k_new", op); CheckBf16(v_new, "v_new", op);
  CheckBf16(k_cache, "k_cache", op); CheckBf16(v_cache, "v_cache", op);
  TORCH_CHECK(q.dim() == 4 && k_cache.dim() == 4,
              "flat_beam_attn: q [B,K,H,D], caches [B,N,Hk,D]");
  const int64_t B = q.size(0), K = q.size(1), H = q.size(2);
  const int64_t N = k_cache.size(1), Hk = k_cache.size(2);
  TORCH_CHECK(K >= 1 && K <= kMaxG, "flat_beam_attn: 1 <= K <= 16 hypotheses");
  TORCH_CHECK(k_cache.sizes() == v_cache.sizes() && k_cache.size(0) == B && N >= 1,
              "flat_beam_attn: caches must both be [B, N, Hk, 128]");
  TORCH_CHECK(k_new.dim() == 4 && k_new.size(0) == B && k_new.size(1) == K &&
                  k_new.size(2) == Hk && v_new.sizes() == k_new.sizes(),
              "flat_beam_attn: k_new / v_new must be [B, K, Hk, 128]");
  TORCH_CHECK(Hk >= 1 && H % Hk == 0, "flat_beam_attn: Hk must divide H");
  const int64_t G = H / Hk;
  const int64_t ngrp = (K * G + kMaxG - 1) / kMaxG;
  TORCH_CHECK(B <= 65535 && Hk * ngrp <= 65535 && N < (1 << 30),
              "flat_beam_attn: shape out of range");
  TORCH_CHECK(slot0.is_cuda() && slot0.device() == q.device() && slot0.numel() == 1 &&
                  (slot0.scalar_type() == torch::kInt32 || slot0.scalar_type() == torch::kInt64),
              "flat_beam_attn: slot0 must be a 0-dim int32 / int64 tensor on the device of q");
  for (const auto* x : {&k_new, &v_new, &k_cache, &v_cache})
    TORCH_CHECK(x->device() == q.device(), "flat_beam_attn: all tensors must be on one device");
  const int64_t W = (N + 31) / 32;
  CheckInt32(vis, q, "vis", {B, K, W});
  CheckInt32(qpos, q, "qpos", {B, K});
  CheckInt32(kpos, q, "kpos", {B, N});
  BeamParams p;
  p.rel = nullptr;
  if (rel.has_value() && rel->defined()) {
    TORCH_CHECK(rel->is_cuda() && rel->device() == q.device() &&
                    rel->scalar_type() == torch::kFloat32 && rel->is_contiguous() &&
                    rel->dim() == 2 && rel->size(0) == H && rel->size(1) == 2 * N - 1,
                "flat_beam_attn: rel must be a contiguous fp32 [H, 2N-1] tensor on the device of q");
    p.rel = rel->data_ptr<float>();
  }
  const c10::cuda::CUDAGuard guard(q.device());
  const int64_t chunk = flat_beam_attn_chunk(B, K, H, Hk, N);
  const int64_t S = (N + chunk - 1) / chunk;
  auto out = torch::empty({B, K, H, kD}, q.options());
  torch::Tensor m_part, l_part, o_part;
  p.m_part = p.l_part = p.o_part = nullptr;
  if (S > 1) {
    const auto f32 = q.options().dtype(torch::kFloat32);
    m_part = torch::empty({B * K * H, S}, f32);
    l_part = torch::empty({B * K * H, S}, f32);
    o_part = torch::empty({B * K * H, S, kD}, f32);
    p.m_part = m_part.data_ptr<float>();
    p.l_part = l_part.data_ptr<float>();
    p.o_part = o_part.data_ptr<float>();
  }
  auto bf = [](const torch::Tensor& x) { return reinterpret_cast<__nv_bfloat16*>(x.data_ptr()); };
  p.q = bf(q); p.k_new = bf(k_new); p.v_new = bf(v_new);
  p.k_cache = bf(k_cache); p.v_cache = bf(v_cache); p.out = bf(out);
  p.slot0 = slot0.data_ptr();
  p.s64 = slot0.scalar_type() == torch::kInt64 ? 1 : 0;
  p.vis = vis.data_ptr<int>(); p.qpos = qpos.data_ptr<int>(); p.kpos = kpos.data_ptr<int>();
  p.K = static_cast<int>(K); p.H = static_cast<int>(H); p.Hk = static_cast<int>(Hk);
  p.N = static_cast<int>(N); p.W = static_cast<int>(W);
  p.chunk = static_cast<int>(chunk); p.S = static_cast<int>(S);
  p.scale = static_cast<float>(scale);
  const dim3 grid(static_cast<unsigned>(S), static_cast<unsigned>(Hk * ngrp), static_cast<unsigned>(B));
  auto stream = at::cuda::getCurrentCUDAStream();
  const int64_t gmax = std::min<int64_t>(K * G, kMaxG);
  if (gmax <= 1) LaunchBeam<1>(p, grid, stream);
  else if (gmax <= 2) LaunchBeam<2>(p, grid, stream);
  else if (gmax <= 4) LaunchBeam<4>(p, grid, stream);
  else if (gmax <= 8) LaunchBeam<8>(p, grid, stream);
  else LaunchBeam<16>(p, grid, stream);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  if (S > 1) {
    flat_beam_attn_combine_kernel<<<static_cast<unsigned>(B * K * H), kD, 0, stream>>>(p);
    C10_CUDA_KERNEL_LAUNCH_CHECK();
    CountLaunch();
  }
  return out;
}

}  // namespace lb

LB_REGISTER(decode_attn) {
  m.def("decode_attn_fwd", &lb::decode_attn_fwd, py::arg("q"), py::arg("k_new"), py::arg("v_new"),
        py::arg("k_cache"), py::arg("v_cache"), py::arg("t"), py::arg("rel"), py::arg("scale"));
  m.def("decode_attn_chunk", &lb::decode_attn_chunk, py::arg("B"), py::arg("H"), py::arg("Hk"),
        py::arg("T"));
  m.def("flat_beam_attn_fwd", &lb::flat_beam_attn_fwd, py::arg("q"), py::arg("k_new"),
        py::arg("v_new"), py::arg("k_cache"), py::arg("v_cache"), py::arg("slot0"), py::arg("vis"),
        py::arg("qpos"), py::arg("kpos"), py::arg("rel"), py::arg("scale"));
  m.def("flat_beam_attn_chunk", &lb::flat_beam_attn_chunk, py::arg("B"), py::arg("K"),
        py::arg("H"), py::arg("Hk"), py::arg("N"));
}
