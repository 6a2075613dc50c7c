// Softmax cross-entropy statistics / gradient over bf16 logits rows.
//
// The LM head computes logits = x . W^T with the wgmma GEMM (bf16 out) and
// never materialises fp32 [T, V] tensors (SURVEY K16):
//   xent_stats : per row  lse, logit[label], sum(logits), argmax      (1 read)
//   xent_bwd   : dlogits = p*a - b - onehot*c  written IN PLACE (bf16) where
//                p = exp(logit - lse) and (a, b, c) are per-row coefficients
//                built from the upstream grads of {soft-label xent, hard xent,
//                z-loss} (1 read + 1 write).
// One CTA (256 threads) per row, 16-byte loads, online softmax reduction.

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "ptx.cuh"
#include "registry.h"

namespace lb {
namespace {

constexpr int kThreads = 256;

struct MaxSum {
  float m, s;
};
__device__ __forceinline__ MaxSum combine(MaxSum a, MaxSum b) {
  const float m = fmaxf(a.m, b.m);
  MaxSum r;
  r.m = m;
  r.s = (a.m == -INFINITY ? 0.f : a.s * __expf(a.m - m)) +
        (b.m == -INFINITY ? 0.f : b.s * __expf(b.m - m));
  return r;
}

__global__ void __launch_bounds__(kThreads)
xent_stats_kernel(const __nv_bfloat16* __restrict__ logits, const long long* __restrict__ labels,
                  float* __restrict__ lse, float* __restrict__ true_logit,
                  float* __restrict__ sum_logits, long long* __restrict__ argmax, int V,
                  long long ld) {
  const int row = blockIdx.x;
  const __nv_bfloat16* lr = logits + static_cast<size_t>(row) * ld;
  MaxSum ms{-INFINITY, 0.f};
  float total = 0.f;
  float best = -INFINITY;
  int best_i = 0;
  for (int c = threadIdx.x * 8; c < V; c += kThreads * 8) {
    int4 v = *reinterpret_cast<const int4*>(lr + c);
    const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
    float f[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 t = unpack_bf16x2(w[j]);
      f[2 * j] = t.x;
      f[2 * j + 1] = t.y;
    }
    float lm = f[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) lm = fmaxf(lm, f[i]);
    float ls = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      ls += __expf(f[i] - lm);
      total += f[i];
      if (f[i] > best) { best = f[i]; best_i = c + i; }
    }
    ms = combine(ms, MaxSum{lm, ls});
  }
  __shared__ float sm_m[kThreads / 32], sm_s[kThreads / 32], sm_t[kThreads / 32],
      sm_b[kThreads / 32];
  __shared__ int sm_i[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    MaxSum other{__shfl_xor_sync(0xffffffffu, ms.m, o), __shfl_xor_sync(0xffffffffu, ms.s, o)};
    ms = combine(ms, other);
    total += __shfl_xor_sync(0xffffffffu, total, o);
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
    if (ob > best || (ob == best && oi < best_i)) { best = ob; best_i = oi; }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sm_m[warp] = ms.m; sm_s[warp] = ms.s; sm_t[warp] = total; sm_b[warp] = best; sm_i[warp] = best_i; }
  __syncthreads();
  if (threadIdx.x == 0) {
    MaxSum r{sm_m[0], sm_s[0]};
    float t = sm_t[0], b = sm_b[0];
    int bi = sm_i[0];
    for (int w = 1; w < kThreads / 32; ++w) {
      r = combine(r, MaxSum{sm_m[w], sm_s[w]});
      t += sm_t[w];
      if (sm_b[w] > b || (sm_b[w] == b && sm_i[w] < bi)) { b = sm_b[w]; bi = sm_i[w]; }
    }
    lse[row] = r.m + __logf(r.s);
    sum_logits[row] = t;
    argmax[row] = bi;
    const long long lab = labels[row];
    true_logit[row] = (lab >= 0 && lab < V) ? __bfloat162float(lr[lab]) : 0.f;
  }
}

__global__ void __launch_bounds__(kThreads)
xent_bwd_kernel(__nv_bfloat16* __restrict__ logits, const long long* __restrict__ labels,
                const float* __restrict__ lse, const float* __restrict__ coef_a,
                const float* __restrict__ coef_b, const float* __restrict__ coef_c, int V,
                long long ld) {
  const int row = blockIdx.x;
  __nv_bfloat16* lr = logits + static_cast<size_t>(row) * ld;
  const float l = lse[row], a = coef_a[row], b = coef_b[row], cc = coef_c[row];
  const long long lab = labels[row];
  for (int c = threadIdx.x * 8; c < V; c += kThreads * 8) {
    int4 v = *reinterpret_cast<const int4*>(lr + c);
    const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
    float f[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 t = unpack_bf16x2(w[j]);
      f[2 * j] = t.x;
      f[2 * j + 1] = t.y;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float d = __expf(f[i] - l) * a - b;
      if (c + i == lab) d -= cc;
      f[i] = d;
    }
    int4 o;
    o.x = pack_bf16x2(f[0], f[1]);
    o.y = pack_bf16x2(f[2], f[3]);
    o.z = pack_bf16x2(f[4], f[5]);
    o.w = pack_bf16x2(f[6], f[7]);
    *reinterpret_cast<int4*>(lr + c) = o;
  }
}

}  // namespace

std::vector<torch::Tensor> xent_stats(const torch::Tensor& logits, const torch::Tensor& labels) {
  TORCH_CHECK(logits.is_cuda() && logits.scalar_type() == torch::kBFloat16 && logits.dim() == 2 &&
              logits.stride(1) == 1);
  TORCH_CHECK(labels.scalar_type() == torch::kInt64 && labels.is_contiguous());
  const c10::cuda::CUDAGuard guard(logits.device());
  const int T = static_cast<int>(logits.size(0)), V = static_cast<int>(logits.size(1));
  TORCH_CHECK(V % 8 == 0 && logits.stride(0) % 8 == 0);
  auto f32 = logits.options().dtype(torch::kFloat32);
  auto lse = torch::empty({T}, f32), tl = torch::empty({T}, f32), sl = torch::empty({T}, f32);
  auto am = torch::empty({T}, logits.options().dtype(torch::kInt64));
  if (T > 0) {
    xent_stats_kernel<<<T, kThreads, 0, at::cuda::getCurrentCUDAStream()>>>(
        reinterpret_cast<const __nv_bfloat16*>(logits.data_ptr()), reinterpret_cast<const long long*>(labels.data_ptr<int64_t>()),
        lse.data_ptr<float>(), tl.data_ptr<float>(), sl.data_ptr<float>(),
        reinterpret_cast<long long*>(am.data_ptr<int64_t>()), V, logits.stride(0));
    C10_CUDA_KERNEL_LAUNCH_CHECK();
    CountLaunch();
  }
  return {lse, tl, sl, am};
}

// In place: logits <- dlogits.
void xent_bwd(torch::Tensor logits, const torch::Tensor& labels, const torch::Tensor& lse,
              const torch::Tensor& a, const torch::Tensor& b, const torch::Tensor& c) {
  TORCH_CHECK(logits.is_cuda() && logits.scalar_type() == torch::kBFloat16 && logits.dim() == 2);
  const c10::cuda::CUDAGuard guard(logits.device());
  const int T = static_cast<int>(logits.size(0)), V = static_cast<int>(logits.size(1));
  if (T == 0) return;
  xent_bwd_kernel<<<T, kThreads, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<__nv_bfloat16*>(logits.data_ptr()), reinterpret_cast<const long long*>(labels.data_ptr<int64_t>()),
      lse.data_ptr<float>(), a.data_ptr<float>(), b.data_ptr<float>(), c.data_ptr<float>(), V,
      logits.stride(0));
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
}

}  // namespace lb

LB_REGISTER(xent) {
  m.attr("_has_xent") = true;
  m.def("xent_stats", &lb::xent_stats);
  m.def("xent_bwd", &lb::xent_bwd);
}
