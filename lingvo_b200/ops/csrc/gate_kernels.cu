// MoE router logits:  logits[T,E] = x[T,M] (bf16) · gw[M,E]   — fp32 accumulate, fp32 out.
//
// E is tiny (8 experts for the GShard LMs), so this is not tensor-core work: a 2048×8
// weight is 64 KB and the whole op is one streaming read of x. The stock path upcasts x to
// fp32 (a 64 MB write for 8k tokens) and runs an SGEMM with N = 8; here
//   forward   one warp per 4 tokens, gw transposed in shared memory ([E][M], conflict-free
//             128-bit reads, each weight reused by 4 tokens), 16-byte bf16 loads of x;
//   dx        dx[T,M] = dlogits[T,E] · gwᵀ, same tiling, bf16 out;
//   dgw       dgw[M,E] = xᵀ · dlogits: each CTA owns a token range and 2048 columns of M,
//             every thread keeps an 8×E fp32 tile in registers, partials per CTA are folded
//             by a second tiny kernel (no atomics).
// All three read x / write dx exactly once.

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "ptx.cuh"
#include "registry.h"

namespace lb {
namespace {

constexpr int kGateThreads = 256;
constexpr int kGateWarps = kGateThreads / 32;
constexpr int kTok = 4;          // tokens per warp pass
constexpr int kDgwCols = kGateThreads * 8;
constexpr int kDgwTile = 32;     // tokens staged per smem tile

__device__ __forceinline__ float gate_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void gate_load8(const __nv_bfloat16* p, float (&f)[8]) {
  const int4 v = ld_nc_v4(p);
  const uint32_t w[4] = {static_cast<uint32_t>(v.x), static_cast<uint32_t>(v.y),
                         static_cast<uint32_t>(v.z), static_cast<uint32_t>(v.w)};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 t = unpack_bf16x2(w[j]);
    f[2 * j] = t.x;
    f[2 * j + 1] = t.y;
  }
}

__device__ __forceinline__ float gate_to_float(float v) { return v; }
__device__ __forceinline__ float gate_to_float(__nv_bfloat16 v) { return __bfloat162float(v); }

// gws[e][m] = gw[m][e]
template <int E, typename WT>
__device__ __forceinline__ void stage_weights(const WT* __restrict__ gw, float* gws, int M) {
  for (int i = threadIdx.x; i < M * E; i += kGateThreads) {
    const int m = i / E, e = i % E;
    gws[e * M + m] = gate_to_float(gw[i]);
  }
  __syncthreads();
}

template <int E, typename WT>
__global__ void __launch_bounds__(kGateThreads)
gate_logits_fwd_kernel(const __nv_bfloat16* __restrict__ x, const WT* __restrict__ gw,
                       float* __restrict__ logits, int T, int M) {
  extern __shared__ __align__(16) float gws[];
  stage_weights<E, WT>(gw, gws, M);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int t0 = (blockIdx.x * kGateWarps + warp) * kTok; t0 < T;
       t0 += gridDim.x * kGateWarps * kTok) {
    float acc[kTok][E];
#pragma unroll
    for (int u = 0; u < kTok; ++u)
#pragma unroll
      for (int e = 0; e < E; ++e) acc[u][e] = 0.f;
    for (int m = lane * 8; m < M; m += 256) {
      float xf[kTok][8];
#pragma unroll
      for (int u = 0; u < kTok; ++u) {
        if (t0 + u < T) {
          gate_load8(x + static_cast<size_t>(t0 + u) * M + m, xf[u]);
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) xf[u][i] = 0.f;
        }
      }
#pragma unroll
      for (int e = 0; e < E; ++e) {
        const float4 a = *reinterpret_cast<const float4*>(gws + e * M + m);
        const float4 b = *reinterpret_cast<const float4*>(gws + e * M + m + 4);
        const float w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
        for (int u = 0; u < kTok; ++u)
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[u][e] = fmaf(xf[u][i], w[i], acc[u][e]);
      }
    }
#pragma unroll
    for (int u = 0; u < kTok; ++u) {
      float mine = 0.f;
#pragma unroll
      for (int e = 0; e < E; ++e) {
        const float s = gate_warp_sum(acc[u][e]);
        if (lane == e) mine = s;
      }
      if (lane < E && t0 + u < T) logits[static_cast<size_t>(t0 + u) * E + lane] = mine;
    }
  }
}

template <int E, typename WT>
__global__ void __launch_bounds__(kGateThreads)
gate_logits_dx_kernel(const float* __restrict__ dl, const WT* __restrict__ gw,
                      const __nv_bfloat16* __restrict__ dres, __nv_bfloat16* __restrict__ dx, int T,
                      int M) {
  // dres (optional): gradient arriving at x along another branch; added here so that
  // autograd does not launch a separate [T, M] add.
  extern __shared__ __align__(16) float gws[];
  stage_weights<E, WT>(gw, gws, M);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int t0 = (blockIdx.x * kGateWarps + warp) * kTok; t0 < T;
       t0 += gridDim.x * kGateWarps * kTok) {
    float d[kTok][E];
#pragma unroll
    for (int u = 0; u < kTok; ++u)
#pragma unroll
      for (int e = 0; e < E; ++e)
        d[u][e] = t0 + u < T ? dl[static_cast<size_t>(t0 + u) * E + e] : 0.f;
    for (int m = lane * 8; m < M; m += 256) {
      float o[kTok][8];
#pragma unroll
      for (int u = 0; u < kTok; ++u) {
        if (dres != nullptr && t0 + u < T) {
          gate_load8(dres + static_cast<size_t>(t0 + u) * M + m, o[u]);
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) o[u][i] = 0.f;
        }
      }
#pragma unroll
      for (int e = 0; e < E; ++e) {
        const float4 a = *reinterpret_cast<const float4*>(gws + e * M + m);
        const float4 b = *reinterpret_cast<const float4*>(gws + e * M + m + 4);
        const float w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
        for (int u = 0; u < kTok; ++u)
#pragma unroll
          for (int i = 0; i < 8; ++i) o[u][i] = fmaf(d[u][e], w[i], o[u][i]);
      }
#pragma unroll
      for (int u = 0; u < kTok; ++u) {
        if (t0 + u >= T) continue;
        int4 v;
        v.x = pack_bf16x2(o[u][0], o[u][1]);
        v.y = pack_bf16x2(o[u][2], o[u][3]);
        v.z = pack_bf16x2(o[u][4], o[u][5]);
        v.w = pack_bf16x2(o[u][6], o[u][7]);
        *reinterpret_cast<int4*>(dx + static_cast<size_t>(t0 + u) * M + m) = v;
      }
    }
  }
}

// part[blk][m][e] = Σ_{t in block's token range} x[t][m] · dl[t][e]
template <int E>
__global__ void __launch_bounds__(kGateThreads)
gate_logits_dgw_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ dl,
                       float* __restrict__ part, int T, int M, int tok_per_blk) {
  __shared__ float dls[kDgwTile][E];
  const int m = blockIdx.y * kDgwCols + threadIdx.x * 8;
  const bool mok = m < M;
  const int t_begin = blockIdx.x * tok_per_blk;
  const int t_end = min(T, t_begin + tok_per_blk);
  float acc[8][E];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int e = 0; e < E; ++e) acc[i][e] = 0.f;
  for (int tb = t_begin; tb < t_end; tb += kDgwTile) {
    const int n = min(kDgwTile, t_end - tb);
    __syncthreads();
    for (int i = threadIdx.x; i < n * E; i += kGateThreads)
      dls[i / E][i % E] = dl[static_cast<size_t>(tb) * E + i];
    __syncthreads();
    if (!mok) continue;
#pragma unroll 4
    for (int j = 0; j < n; ++j) {
      float xf[8];
      gate_load8(x + static_cast<size_t>(tb + j) * M + m, xf);
#pragma unroll
      for (int e = 0; e < E; ++e) {
        const float d = dls[j][e];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i][e] = fmaf(xf[i], d, acc[i][e]);
      }
    }
  }
  if (!mok) return;
  float* out = part + (static_cast<size_t>(blockIdx.x) * M + m) * E;
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int e = 0; e < E; ++e) out[i * E + e] = acc[i][e];
}

// dgw[i] = Σ_k part[k][i]: block = 32 elements × 8 partial groups (coalesced 128-byte reads).
template <typename WT>
__global__ void __launch_bounds__(256)
gate_logits_dgw_fold_kernel(const float* __restrict__ part, WT* __restrict__ dgw, int ME, int nblk) {
  __shared__ float red[8][33];
  const int cx = threadIdx.x & 31, ky = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + cx;
  float s0 = 0.f, s1 = 0.f;
  if (i < ME) {
    int k = ky;
    for (; k + 8 < nblk; k += 16) {
      s0 += part[static_cast<size_t>(k) * ME + i];
      s1 += part[static_cast<size_t>(k + 8) * ME + i];
    }
    if (k < nblk) s0 += part[static_cast<size_t>(k) * ME + i];
  }
  red[ky][cx] = s0 + s1;
  __syncthreads();
  if (ky == 0 && i < ME) {
    float s = 0.f;
#pragma unroll
    for (int r = 0; r < 8; ++r) s += red[r][cx];
    if constexpr (std::is_same<WT, float>::value) dgw[i] = s;
    else dgw[i] = __float2bfloat16(s);
  }
}

int Sms() { return at::cuda::getCurrentDeviceProperties()->multiProcessorCount; }

bool Aligned16(const torch::Tensor& t) {
  return reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0;
}

// x and dres are read with 16-byte `ld.global.nc.v4` loads (gate_load8).
void CheckArgs(const torch::Tensor& x, const torch::Tensor& gw) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == torch::kBFloat16 && x.is_contiguous() && x.dim() == 2,
              "gate_logits: x must be contiguous bf16 [T, M]");
  TORCH_CHECK(Aligned16(x), "gate_logits: x must be 16-byte aligned");
  TORCH_CHECK(gw.is_cuda() && gw.is_contiguous() && gw.dim() == 2 && gw.size(0) == x.size(1),
              "gate_logits: gw must be contiguous [M, E]");
  TORCH_CHECK(gw.device() == x.device(), "gate_logits: gw must be on x's device");
  TORCH_CHECK(gw.scalar_type() == torch::kFloat32 || gw.scalar_type() == torch::kBFloat16);
  const int64_t e = gw.size(1);
  TORCH_CHECK(e == 2 || e == 4 || e == 8 || e == 16, "gate_logits: unsupported expert count ", e);
  TORCH_CHECK(x.size(1) % 8 == 0, "gate_logits: M must be a multiple of 8");
  TORCH_CHECK(static_cast<size_t>(x.size(1)) * gw.size(1) * 4 <= 200 * 1024,
              "gate_logits: [M, E] weight does not fit in shared memory");
}

template <typename F>
void DispatchE(int64_t e, F&& f) {
  switch (e) {
    case 2: f(std::integral_constant<int, 2>()); break;
    case 4: f(std::integral_constant<int, 4>()); break;
    case 8: f(std::integral_constant<int, 8>()); break;
    case 16: f(std::integral_constant<int, 16>()); break;
    default: TORCH_CHECK(false, "gate_logits: unsupported expert count ", e);
  }
}

template <typename K>
void AllowSmem(K kernel, size_t bytes) {
  if (bytes > 48 * 1024)
    C10_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(bytes)));
}

}  // namespace

torch::Tensor gate_logits_fwd(const torch::Tensor& x, const torch::Tensor& gw) {
  CheckArgs(x, gw);
  const c10::cuda::CUDAGuard guard(x.device());
  const int T = static_cast<int>(x.size(0)), M = static_cast<int>(x.size(1));
  const int64_t E = gw.size(1);
  auto out = torch::empty({x.size(0), E}, x.options().dtype(torch::kFloat32));
  if (T == 0) return out;
  auto stream = at::cuda::getCurrentCUDAStream();
  const size_t smem = static_cast<size_t>(M) * E * 4;
  const int grid = std::min((T + kGateWarps * kTok - 1) / (kGateWarps * kTok), Sms() * 2);
  DispatchE(E, [&](auto ec) {
    constexpr int kE = decltype(ec)::value;
    auto xp = reinterpret_cast<const __nv_bfloat16*>(x.data_ptr());
    if (gw.scalar_type() == torch::kFloat32) {
      auto k = gate_logits_fwd_kernel<kE, float>;
      AllowSmem(k, smem);
      k<<<grid, kGateThreads, smem, stream>>>(xp, gw.data_ptr<float>(), out.data_ptr<float>(), T, M);
    } else {
      auto k = gate_logits_fwd_kernel<kE, __nv_bfloat16>;
      AllowSmem(k, smem);
      k<<<grid, kGateThreads, smem, stream>>>(
          xp, reinterpret_cast<const __nv_bfloat16*>(gw.data_ptr()), out.data_ptr<float>(), T, M);
    }
  });
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return out;
}

// → (dx bf16 [T, M] or undefined, dgw [M, E] in gw's dtype or undefined)
std::vector<torch::Tensor> gate_logits_bwd(const torch::Tensor& x, const torch::Tensor& gw,
                                           const torch::Tensor& dlogits, bool need_dx,
                                           bool need_dgw,
                                           const c10::optional<torch::Tensor>& dres) {
  CheckArgs(x, gw);
  TORCH_CHECK(dlogits.is_cuda() && dlogits.scalar_type() == torch::kFloat32 &&
              dlogits.is_contiguous() && dlogits.dim() == 2 && dlogits.size(0) == x.size(0) &&
              dlogits.size(1) == gw.size(1), "gate_logits_bwd: dlogits must be fp32 [T, E]");
  TORCH_CHECK(dlogits.device() == x.device(), "gate_logits_bwd: dlogits must be on x's device");
  const c10::cuda::CUDAGuard guard(x.device());
  const int T = static_cast<int>(x.size(0)), M = static_cast<int>(x.size(1));
  const int64_t E = gw.size(1);
  auto stream = at::cuda::getCurrentCUDAStream();
  torch::Tensor dx, dgw;
  auto xp = reinterpret_cast<const __nv_bfloat16*>(x.data_ptr());
  const __nv_bfloat16* drp = nullptr;
  if (dres.has_value() && dres->defined()) {
    TORCH_CHECK(dres->is_cuda() && dres->scalar_type() == torch::kBFloat16 && dres->is_contiguous() &&
                dres->numel() == x.numel(), "gate_logits_bwd: dres must be contiguous bf16 like x");
    TORCH_CHECK(dres->device() == x.device(), "gate_logits_bwd: dres must be on x's device");
    TORCH_CHECK(Aligned16(*dres), "gate_logits_bwd: dres must be 16-byte aligned");
    drp = reinterpret_cast<const __nv_bfloat16*>(dres->data_ptr());
  }
  if (need_dx) {
    dx = torch::empty_like(x);
    if (T > 0) {
      const size_t smem = static_cast<size_t>(M) * E * 4;
      const int grid = std::min((T + kGateWarps * kTok - 1) / (kGateWarps * kTok), Sms() * 2);
      DispatchE(E, [&](auto ec) {
        constexpr int kE = decltype(ec)::value;
        auto dxp = reinterpret_cast<__nv_bfloat16*>(dx.data_ptr());
        if (gw.scalar_type() == torch::kFloat32) {
          auto k = gate_logits_dx_kernel<kE, float>;
          AllowSmem(k, smem);
          k<<<grid, kGateThreads, smem, stream>>>(dlogits.data_ptr<float>(), gw.data_ptr<float>(),
                                                  drp, dxp, T, M);
        } else {
          auto k = gate_logits_dx_kernel<kE, __nv_bfloat16>;
          AllowSmem(k, smem);
          k<<<grid, kGateThreads, smem, stream>>>(
              dlogits.data_ptr<float>(), reinterpret_cast<const __nv_bfloat16*>(gw.data_ptr()), drp,
              dxp, T, M);
        }
      });
      C10_CUDA_KERNEL_LAUNCH_CHECK();
      CountLaunch();
    }
  }
  if (need_dgw) {
    dgw = torch::empty_like(gw);
    if (T == 0) {
      dgw.zero_();
    } else {
      const int nblk = std::min(Sms() * 3, (T + kDgwTile - 1) / kDgwTile);
      const int tok_per_blk = (T + nblk - 1) / nblk;
      const int used = (T + tok_per_blk - 1) / tok_per_blk;
      auto part = torch::empty({used, x.size(1), E}, x.options().dtype(torch::kFloat32));
      const dim3 grid(used, (M + kDgwCols - 1) / kDgwCols);
      DispatchE(E, [&](auto ec) {
        constexpr int kE = decltype(ec)::value;
        gate_logits_dgw_kernel<kE><<<grid, kGateThreads, 0, stream>>>(
            xp, dlogits.data_ptr<float>(), part.data_ptr<float>(), T, M, tok_per_blk);
      });
      const int me = static_cast<int>(M * E);
      if (gw.scalar_type() == torch::kFloat32)
        gate_logits_dgw_fold_kernel<float><<<(me + 31) / 32, 256, 0, stream>>>(
            part.data_ptr<float>(), dgw.data_ptr<float>(), me, used);
      else
        gate_logits_dgw_fold_kernel<__nv_bfloat16><<<(me + 31) / 32, 256, 0, stream>>>(
            part.data_ptr<float>(), reinterpret_cast<__nv_bfloat16*>(dgw.data_ptr()), me, used);
      C10_CUDA_KERNEL_LAUNCH_CHECK();
      CountLaunch(2);
    }
  }
  return {dx, dgw};
}

}  // namespace lb

LB_REGISTER(gate) {
  m.def("gate_logits_fwd", &lb::gate_logits_fwd);
  m.def("gate_logits_bwd", &lb::gate_logits_bwd);
}
