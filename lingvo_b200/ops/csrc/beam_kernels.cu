// Beam-search step hot loop (SURVEY K13; reference CPU op
// `lingvo/core/ops/beam_search_step_op_kernels.cc:100-950`).
//
// beam_topk: for every hypothesis row (one CTA per row) fuse
//     global[v] = cumulative[row] + log_probs[row, v]
//     mask EOS (handled separately by the caller) and inactive rows,
//     K best (score desc, word id asc) continuations,
//     best-in-row over ALL tokens and the row's EOS score
// in a single pass over the vocabulary: the [num_hyps, V] "global score" tensor, its
// clone with the EOS column blanked and the library top-k of the eager implementation are
// never materialised (V = 32 k, num_hyps = beams x K rows per step).
//
// Each thread keeps the K best of its strided slice in registers (insertion into a
// sorted array, strict > so lower word ids win ties), then K rounds of a block-wide
// arg-max tournament over the per-thread list heads produce the row's top-K in order.

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda_bf16.h>
#include <torch/extension.h>

#include <type_traits>

#include "registry.h"

namespace lb {
namespace {

constexpr int kMaxK = 16;
constexpr int kThreads = 256;
constexpr float kNeg = -1.0e30f;

__device__ __forceinline__ float to_float(float v) { return v; }
__device__ __forceinline__ float to_float(__nv_bfloat16 v) { return __bfloat162float(v); }

// KT: compile-time list length (>= K); every thread keeps its KT best so that all register
// array indices are static after unrolling.
template <typename T, int KT>
__global__ void __launch_bounds__(kThreads)
beam_topk_kernel(const T* __restrict__ log_probs, const float* __restrict__ cum,
                 const uint8_t* __restrict__ active, float* __restrict__ top_s,
                 long long* __restrict__ top_w, float* __restrict__ best_in_hyp,
                 float* __restrict__ eos_glob, float* __restrict__ eos_local, int V, int K,
                 int eos_id) {
  const int row = blockIdx.x;
  const T* lp = log_probs + static_cast<long long>(row) * V;
  const float c = cum[row];
  const bool act = active[row] != 0;
  float s[KT];
  int w[KT];
#pragma unroll
  for (int i = 0; i < KT; ++i) { s[i] = kNeg; w[i] = 0x7fffffff; }
  float best = kNeg;
  for (int v = threadIdx.x; v < V; v += kThreads) {
    const float g = c + to_float(lp[v]);
    best = fmaxf(best, g);
    if (v == eos_id || !act) continue;
    if (g > s[KT - 1]) {
      // sorted (descending) insertion; ascending scan ⇒ strict > keeps the smaller word id
      // ahead on ties. Bubble from the tail with compile-time indices.
      s[KT - 1] = g;
      w[KT - 1] = v;
#pragma unroll
      for (int i = KT - 1; i > 0; --i) {
        if (s[i] > s[i - 1]) {
          const float ts = s[i]; s[i] = s[i - 1]; s[i - 1] = ts;
          const int tw = w[i]; w[i] = w[i - 1]; w[i - 1] = tw;
        }
      }
    }
  }
  // ---- row-wide best over all tokens ----
  __shared__ float red_s[kThreads];
  __shared__ int red_w[kThreads];
  __shared__ int red_t[kThreads];
  red_s[threadIdx.x] = best;
  __syncthreads();
  for (int off = kThreads / 2; off > 0; off >>= 1) {
    if (threadIdx.x < off) red_s[threadIdx.x] = fmaxf(red_s[threadIdx.x], red_s[threadIdx.x + off]);
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    best_in_hyp[row] = red_s[0];
    const float el = to_float(lp[eos_id]);
    eos_local[row] = el;
    eos_glob[row] = c + el;
  }
  __syncthreads();
  // ---- K rounds of tournament over the list heads ----
  int head = 0;
  for (int r = 0; r < K; ++r) {
    float hs = kNeg;
    int hw = 0x7fffffff;
    // (register array indexed by a runtime `head`: select with a short unrolled scan)
#pragma unroll
    for (int i = 0; i < KT; ++i)
      if (i == head) { hs = s[i]; hw = w[i]; }
    red_s[threadIdx.x] = hs;
    red_w[threadIdx.x] = hw;
    red_t[threadIdx.x] = threadIdx.x;
    __syncthreads();
    for (int off = kThreads / 2; off > 0; off >>= 1) {
      if (threadIdx.x < off) {
        const float a = red_s[threadIdx.x], b = red_s[threadIdx.x + off];
        const int wa = red_w[threadIdx.x], wb = red_w[threadIdx.x + off];
        if (b > a || (b == a && wb < wa)) {
          red_s[threadIdx.x] = b;
          red_w[threadIdx.x] = wb;
          red_t[threadIdx.x] = red_t[threadIdx.x + off];
        }
      }
      __syncthreads();
    }
    const int winner = red_t[0];
    if (threadIdx.x == 0) {
      top_s[static_cast<long long>(row) * K + r] = red_s[0];
      top_w[static_cast<long long>(row) * K + r] = red_s[0] > kNeg * 0.5f ? red_w[0] : 0;
    }
    if (threadIdx.x == winner) ++head;
    __syncthreads();
  }
}

}  // namespace

// Returns (top_s [n,K] fp32, top_w [n,K] int64, best_in_hyp [n], eos_glob [n], eos_local [n]).
std::vector<torch::Tensor> beam_topk(const torch::Tensor& log_probs, const torch::Tensor& cum,
                                     const torch::Tensor& active, int64_t k, int64_t eos_id) {
  TORCH_CHECK(log_probs.is_cuda() && log_probs.dim() == 2 && log_probs.is_contiguous(),
              "beam_topk: log_probs must be a contiguous CUDA [num_hyps, V] tensor");
  TORCH_CHECK(k >= 1 && k <= kMaxK, "beam_topk: 1 <= K <= 16");
  const int64_t n = log_probs.size(0), V = log_probs.size(1);
  TORCH_CHECK(eos_id >= 0 && eos_id < V);
  const c10::cuda::CUDAGuard guard(log_probs.device());
  auto cumf = cum.to(torch::kFloat32).contiguous();
  auto act = active.to(torch::kUInt8).contiguous();
  auto fopt = log_probs.options().dtype(torch::kFloat32);
  auto top_s = torch::empty({n, k}, fopt);
  auto top_w = torch::empty({n, k}, log_probs.options().dtype(torch::kInt64));
  auto best = torch::empty({n}, fopt);
  auto eg = torch::empty({n}, fopt);
  auto el = torch::empty({n}, fopt);
  auto stream = at::cuda::getCurrentCUDAStream();
  auto launch = [&](auto* ptr) {
    using T = std::remove_cv_t<std::remove_pointer_t<decltype(ptr)>>;
    auto go = [&](auto kern) {
      kern<<<static_cast<unsigned>(n), kThreads, 0, stream>>>(
          ptr, cumf.data_ptr<float>(), act.data_ptr<uint8_t>(), top_s.data_ptr<float>(),
          reinterpret_cast<long long*>(top_w.data_ptr<int64_t>()), best.data_ptr<float>(),
          eg.data_ptr<float>(), el.data_ptr<float>(), static_cast<int>(V), static_cast<int>(k),
          static_cast<int>(eos_id));
    };
    if (k <= 4) go(beam_topk_kernel<T, 4>);
    else if (k <= 8) go(beam_topk_kernel<T, 8>);
    else go(beam_topk_kernel<T, 16>);
  };
  if (log_probs.scalar_type() == torch::kFloat32) {
    launch(log_probs.data_ptr<float>());
  } else if (log_probs.scalar_type() == torch::kBFloat16) {
    launch(reinterpret_cast<const __nv_bfloat16*>(log_probs.data_ptr()));
  } else {
    TORCH_CHECK(false, "beam_topk: fp32 or bf16 log-probs");
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return {top_s, top_w, best, eg, el};
}

}  // namespace lb

LB_REGISTER(beam) {
  m.def("beam_topk", &lb::beam_topk);
}
