// Conformer conv-module kernel (SURVEY K10): GLU gate + padding mask + depthwise
// conv1d over time fused into one pass.
//
//   g[b,t,d]  = act[b,t,d] * sigmoid(gated[b,t,d]) * (1 - pad[b,t])      (never stored)
//   y[b,t,d]  = (1 - pad[b,t]) * sum_k w[k,d] * g[b, t + k - left, d]
//
// proj = [B, T, 2D] holds (gated | act) — the output of the `linear_start`
// GEMM (ref conformer_layer.py:300-330). `left` = K-1 for a causal conv,
// (K-1)/2 for SAME. The unfused reference path makes 3 elementwise passes plus
// a depthwise cuDNN conv; this reads proj once and writes y once. The backward
// kernel recomputes g from proj and produces d proj and d w in one pass.
//
// Tiling: block = 128 channels x TT frames of one batch row; the (TT + K - 1)
// frame halo of g (and dy in the backward) is staged in shared memory. A
// backward block walks a fixed run of kRun such tiles of one batch row and
// keeps one fp32 partial row of d w, [K, D], summed over its run in tile order.
// A fold kernel adds the B * ceil(T / (kRun * TT)) partial rows in a fixed
// order, so d w is bit-identical from run to run (no atomics). The partials
// take 4 * K * D * B * ceil(T / 64) bytes: K / 128 of the bytes of d proj in
// fp32 (K / 64 in bf16), with T rounded up to whole runs.

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda_bf16.h>
#include <torch/extension.h>

#include "registry.h"

namespace lb {
namespace {

constexpr int kCh = 128;   // channels per block (one per thread)
constexpr int kTT = 32;    // output frames per block
constexpr int kRun = 2;    // backward: T-tiles per block, one d w partial row per block

// The backward stages act, sigmoid(gated) * mask and dy' over a (kTT + K - 1)-frame halo and
// the K taps, kCh fp32 each: (4K + 3 (kTT - 1)) * kCh * 4 bytes. With kBwdSmem allowed, K <=
// kMaxK fits; both launches and glu_dwconv1d_supported refuse larger K.
constexpr int kBwdSmem = 220 * 1024;
constexpr int kMaxK = (kBwdSmem / (kCh * 4) - 3 * (kTT - 1)) / 4;
static_assert(kMaxK == 86, "backward K limit");
constexpr int kFwdSmem = 200 * 1024;
static_assert((kTT + 2 * kMaxK - 1) * kCh * 4 <= kFwdSmem, "forward fits every backward K");

size_t BwdSmemBytes(int K) { return static_cast<size_t>(3 * (kTT + K - 1) + K) * kCh * sizeof(float); }

template <typename T> __device__ __forceinline__ float ldf(const T* p);
template <> __device__ __forceinline__ float ldf<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ldf<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __bfloat162float(*p);
}
template <typename T> __device__ __forceinline__ void stf(T* p, float v);
template <> __device__ __forceinline__ void stf<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void stf<__nv_bfloat16>(__nv_bfloat16* p, float v) {
  *p = __float2bfloat16(v);
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }

template <typename T>
__global__ void __launch_bounds__(kCh)
glu_dwconv_fwd_kernel(const T* __restrict__ proj, const float* __restrict__ w,
                      const float* __restrict__ pad, T* __restrict__ y, int B, int Tn, int D,
                      int K, int left) {
  extern __shared__ float sm[];
  float* sg = sm;                          // [(kTT + K - 1)][kCh]
  float* sw = sm + (kTT + K - 1) * kCh;    // [K][kCh]
  const int d = blockIdx.x * kCh + threadIdx.x;
  const int t0 = blockIdx.y * kTT;
  const int b = blockIdx.z;
  const bool ok = d < D;
  const long long row0 = static_cast<long long>(b) * Tn;
  for (int k = 0; k < K; ++k) sw[k * kCh + threadIdx.x] = ok ? w[k * D + d] : 0.f;
  const int halo = kTT + K - 1;
  for (int j = 0; j < halo; ++j) {
    const int t = t0 - left + j;
    float g = 0.f;
    if (ok && t >= 0 && t < Tn) {
      const float m = 1.f - pad[row0 + t];
      if (m != 0.f) {
        const T* p = proj + (row0 + t) * 2 * D;
        g = ldf(p + D + d) * sigmoidf_(ldf(p + d)) * m;
      }
    }
    sg[j * kCh + threadIdx.x] = g;
  }
  __syncthreads();   // columns are private to a thread, but keep it simple & safe
  if (!ok) return;
  for (int i = 0; i < kTT; ++i) {
    const int t = t0 + i;
    if (t >= Tn) break;
    float acc = 0.f;
    for (int k = 0; k < K; ++k) acc += sw[k * kCh + threadIdx.x] * sg[(i + k) * kCh + threadIdx.x];
    stf(y + (row0 + t) * D + d, acc * (1.f - pad[row0 + t]));
  }
}

template <typename T>
__global__ void __launch_bounds__(kCh)
glu_dwconv_bwd_kernel(const T* __restrict__ proj, const float* __restrict__ w,
                      const float* __restrict__ pad, const T* __restrict__ dy,
                      T* __restrict__ dproj, float* __restrict__ dw_part /* [B * runs, K, D] */,
                      int B, int Tn, int D, int K, int left) {
  extern __shared__ float sm[];
  const int halo = kTT + K - 1;
  float* sa = sm;                    // act            [halo][kCh]   frames t0-left ..
  float* ss = sa + halo * kCh;       // sigmoid(gated) [halo][kCh]   (masked by 1-pad)
  float* sd = ss + halo * kCh;       // dy'            [halo][kCh]   frames t0-(K-1-left) ..
  float* sw = sd + halo * kCh;       // [K][kCh]
  const int d = blockIdx.x * kCh + threadIdx.x;
  const int b = blockIdx.z;
  const bool ok = d < D;
  const long long row0 = static_cast<long long>(b) * Tn;
  const int right = K - 1 - left;
  const int run0 = blockIdx.y * kRun * kTT;
  const int run_end = min(run0 + kRun * kTT, Tn);
  float* part = dw_part + (static_cast<size_t>(b) * gridDim.y + blockIdx.y) * K * D + d;
  for (int k = 0; k < K; ++k) sw[k * kCh + threadIdx.x] = ok ? w[k * D + d] : 0.f;
  for (int t0 = run0; t0 < run_end; t0 += kTT) {
    __syncthreads();                  // the previous tile is done with the halos
    for (int j = 0; j < halo; ++j) {
      const int tg = t0 - left + j;     // frame of g
      float a = 0.f, s = 0.f;
      if (ok && tg >= 0 && tg < Tn) {
        const float m = 1.f - pad[row0 + tg];
        const T* p = proj + (row0 + tg) * 2 * D;
        a = ldf(p + D + d);
        s = sigmoidf_(ldf(p + d)) * m;  // mask folded into s so g = a*s
      }
      sa[j * kCh + threadIdx.x] = a;
      ss[j * kCh + threadIdx.x] = s;
      const int td = t0 - right + j;    // frame of dy'
      float v = 0.f;
      if (ok && td >= 0 && td < Tn) v = ldf(dy + (row0 + td) * D + d) * (1.f - pad[row0 + td]);
      sd[j * kCh + threadIdx.x] = v;
    }
    __syncthreads();
    if (!ok) continue;
    // d g[s] = sum_k w[k] * dy'[s - k + left];  frame s = t0 + i lives at sd index i + right - k + left
    for (int i = 0; i < kTT; ++i) {
      const int s_t = t0 + i;
      if (s_t >= Tn) break;
      float dg = 0.f;
      for (int k = 0; k < K; ++k)
        dg += sw[k * kCh + threadIdx.x] * sd[(i + right + left - k) * kCh + threadIdx.x];
      const int gi = i + left;          // index of frame s_t in sa / ss
      const float a = sa[gi * kCh + threadIdx.x];
      const float sm_ = ss[gi * kCh + threadIdx.x];        // sigmoid * mask
      const float m = 1.f - pad[row0 + s_t];
      const float sg_ = m != 0.f ? sm_ / m : 0.f;          // plain sigmoid
      T* o = dproj + (row0 + s_t) * 2 * D;
      stf(o + D + d, dg * sm_);                            // d act
      stf(o + d, dg * m * a * sg_ * (1.f - sg_));          // d gated
    }
    // d w[k] = sum_{t in tile} dy'[t] * g[t + k - left];  dy'[t0+i] at sd[i+right], g at sa/ss[i+k].
    // The block's partial row is this thread's own column: tiles add to it in order.
    for (int k = 0; k < K; ++k) {
      float acc = 0.f;
      for (int i = 0; i < kTT; ++i) {
        const int gi = i + k;
        acc += sd[(i + right) * kCh + threadIdx.x] * sa[gi * kCh + threadIdx.x] *
               ss[gi * kCh + threadIdx.x];
      }
      float* q = part + static_cast<size_t>(k) * D;
      *q = t0 == run0 ? acc : *q + acc;
    }
  }
}

// dw[j] = sum_p part[p][j], p in order within each of 8 row groups, then the 8 group sums in
// order. Block = 32 columns x 8 row groups: coalesced 128-byte reads.
__global__ void __launch_bounds__(256)
dw_fold_kernel(const float* __restrict__ part, float* __restrict__ dw, int n, int nparts) {
  __shared__ float red[8][33];
  const int cx = threadIdx.x & 31, ky = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + cx;
  float s = 0.f;
  if (j < n)
    for (int p = ky; p < nparts; p += 8) s += part[static_cast<size_t>(p) * n + j];
  red[ky][cx] = s;
  __syncthreads();
  if (ky == 0 && j < n) {
    float t = 0.f;
#pragma unroll
    for (int r = 0; r < 8; ++r) t += red[r][cx];
    dw[j] = t;
  }
}

void Check(const torch::Tensor& proj, const torch::Tensor& w, const torch::Tensor& pad,
           int64_t left) {
  TORCH_CHECK(proj.is_cuda() && proj.dim() == 3 && proj.is_contiguous() && proj.size(2) % 2 == 0);
  TORCH_CHECK(proj.scalar_type() == torch::kBFloat16 || proj.scalar_type() == torch::kFloat32);
  TORCH_CHECK(w.is_cuda() && w.scalar_type() == torch::kFloat32 && w.is_contiguous() &&
              w.dim() == 2 && w.size(1) * 2 == proj.size(2), "glu_dwconv: w must be fp32 [K, D]");
  TORCH_CHECK(pad.is_cuda() && pad.scalar_type() == torch::kFloat32 && pad.is_contiguous() &&
              pad.numel() == proj.size(0) * proj.size(1), "glu_dwconv: pad must be fp32 [B, T]");
  TORCH_CHECK(w.size(0) >= 1 && w.size(0) <= kMaxK, "glu_dwconv: kernel size must be in [1, ",
              kMaxK, "], got ", w.size(0));
  TORCH_CHECK(left >= 0 && left < w.size(0), "glu_dwconv: left must be in [0, K), got ", left);
}

}  // namespace

torch::Tensor glu_dwconv1d_fwd(const torch::Tensor& proj, const torch::Tensor& w,
                               const torch::Tensor& pad, int64_t left) {
  Check(proj, w, pad, left);
  const c10::cuda::CUDAGuard guard(proj.device());
  const int B = proj.size(0), Tn = proj.size(1), D = proj.size(2) / 2, K = w.size(0);
  auto y = torch::empty({B, Tn, D}, proj.options());
  if (y.numel() == 0) return y;
  const size_t smem = static_cast<size_t>(kTT + 2 * K - 1) * kCh * sizeof(float);
  dim3 grid((D + kCh - 1) / kCh, (Tn + kTT - 1) / kTT, B);
  auto stream = at::cuda::getCurrentCUDAStream();
  if (proj.scalar_type() == torch::kBFloat16) {
    auto kern = glu_dwconv_fwd_kernel<__nv_bfloat16>;
    C10_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kFwdSmem));
    kern<<<grid, kCh, smem, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(proj.data_ptr()), w.data_ptr<float>(),
        pad.data_ptr<float>(), reinterpret_cast<__nv_bfloat16*>(y.data_ptr()), B, Tn, D, K,
        static_cast<int>(left));
  } else {
    auto kern = glu_dwconv_fwd_kernel<float>;
    C10_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kFwdSmem));
    kern<<<grid, kCh, smem, stream>>>(proj.data_ptr<float>(), w.data_ptr<float>(),
                                      pad.data_ptr<float>(), y.data_ptr<float>(), B, Tn, D, K,
                                      static_cast<int>(left));
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return y;
}

std::vector<torch::Tensor> glu_dwconv1d_bwd(const torch::Tensor& proj, const torch::Tensor& w,
                                            const torch::Tensor& pad, const torch::Tensor& dy,
                                            int64_t left) {
  Check(proj, w, pad, left);
  TORCH_CHECK(dy.is_cuda() && dy.is_contiguous() && dy.scalar_type() == proj.scalar_type() &&
              dy.numel() == proj.numel() / 2, "glu_dwconv: dy must be contiguous [B, T, D] of proj's dtype");
  const c10::cuda::CUDAGuard guard(proj.device());
  const int B = proj.size(0), Tn = proj.size(1), D = proj.size(2) / 2, K = w.size(0);
  auto dproj = torch::empty_like(proj);
  if (dproj.numel() == 0) return {dproj, torch::zeros_like(w)};
  auto dw = torch::empty_like(w);
  const int runs = (Tn + kRun * kTT - 1) / (kRun * kTT);
  auto part = torch::empty({static_cast<int64_t>(B) * runs, K, D}, w.options());
  const size_t smem = BwdSmemBytes(K);
  dim3 grid((D + kCh - 1) / kCh, runs, B);
  auto stream = at::cuda::getCurrentCUDAStream();
  if (proj.scalar_type() == torch::kBFloat16) {
    auto kern = glu_dwconv_bwd_kernel<__nv_bfloat16>;
    C10_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kBwdSmem));
    kern<<<grid, kCh, smem, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(proj.data_ptr()), w.data_ptr<float>(),
        pad.data_ptr<float>(), reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr()),
        reinterpret_cast<__nv_bfloat16*>(dproj.data_ptr()), part.data_ptr<float>(), B, Tn, D, K,
        static_cast<int>(left));
  } else {
    auto kern = glu_dwconv_bwd_kernel<float>;
    C10_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kBwdSmem));
    kern<<<grid, kCh, smem, stream>>>(proj.data_ptr<float>(), w.data_ptr<float>(),
                                      pad.data_ptr<float>(), dy.data_ptr<float>(),
                                      dproj.data_ptr<float>(), part.data_ptr<float>(), B, Tn, D, K,
                                      static_cast<int>(left));
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  const int n = K * D;
  dw_fold_kernel<<<(n + 31) / 32, 256, 0, stream>>>(part.data_ptr<float>(), dw.data_ptr<float>(),
                                                    n, B * runs);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch(2);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return {dproj, dw};
}

}  // namespace lb

LB_REGISTER(conv) {
  m.attr("_has_conv") = true;
  m.attr("glu_dwconv_max_k") = lb::kMaxK;
  m.def("glu_dwconv1d_fwd", &lb::glu_dwconv1d_fwd);
  m.def("glu_dwconv1d_bwd", &lb::glu_dwconv1d_bwd);
}
