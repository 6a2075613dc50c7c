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

void CheckBf16(const torch::Tensor& x, const char* name) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == torch::kBFloat16 && x.is_contiguous() &&
                  x.size(-1) == kD && reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0,
              "decode_attn: ", name, " must be a contiguous 16-byte aligned bf16 tensor with D = 128");
}

}  // namespace

// Keys per CTA: enough splits that B·Hk·⌈G/16⌉·S CTAs fill the SMs once, in multiples of 128.
int64_t decode_attn_chunk(int64_t B, int64_t H, int64_t Hk, int64_t T) {
  const int64_t ngrp = (H / Hk + kMaxG - 1) / kMaxG;
  const int64_t units = B * Hk * ngrp;
  const int64_t sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  const int64_t want = std::max<int64_t>(1, (sms + units - 1) / units);
  const int64_t chunk = (T + want - 1) / want;
  return (chunk + kCtaKeys - 1) / kCtaKeys * kCtaKeys;
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

}  // namespace lb

LB_REGISTER(decode_attn) {
  m.attr("_has_decode_attn") = true;
  m.def("decode_attn_fwd", &lb::decode_attn_fwd, py::arg("q"), py::arg("k_new"), py::arg("v_new"),
        py::arg("k_cache"), py::arg("v_cache"), py::arg("t"), py::arg("rel"), py::arg("scale"));
  m.def("decode_attn_chunk", &lb::decode_attn_chunk, py::arg("B"), py::arg("H"), py::arg("Hk"),
        py::arg("T"));
}
