// Collectives over NVLink peer memory (symmetric buffers), fused with the
// adjacent elementwise work (SURVEY K11).
//
//   allreduce_mean_bf16 : two-shot all-reduce in ONE kernel: every rank reduces
//       its 1/W shard by loading the W peer copies (fp32 accumulate), scales,
//       and stores the result into all W peers. NVSwitch gives uniform
//       any-to-any bandwidth, so the flat one-hop shape is optimal.
//   zero_adam : reduce-scatter + cast/scale + partitioned Adam + all-gather in
//       ONE kernel: shard gradients are summed from the peers, the fp32 master
//       shard and its Adam moments are updated, and the new bf16 weights are
//       stored straight into every peer's replica of the parameters.
// The device-counter flags of moe_sync order the phases across ranks.

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "adam.cuh"
#include "ptx.cuh"
#include "registry.h"

namespace lb {
namespace {

constexpr int kMaxWorld = 16;
struct PeerPtrs {
  long long p[kMaxWorld];
};

__device__ __forceinline__ void acc8(float (&a)[8], const int4& v) {
  const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float2 t = unpack_bf16x2(w[j]);
    a[2 * j] += t.x;
    a[2 * j + 1] += t.y;
  }
}

// n8 = number of 16-byte vectors in one shard; buffers hold W * n8 vectors.
// sumsq_part (optional): this CTA's Σ (a·scale)² of the unrounded fp32 mean, summed over its
// threads in a fixed order; allreduce_sumsq_fold_kernel adds the partials to sumsq.
__global__ void __launch_bounds__(512)
allreduce_mean_bf16_kernel(const PeerPtrs peers, long long n8, int rank, int world, float scale,
                           int store_all, float* __restrict__ sumsq_part) {
  __shared__ float red[16];
  float ss = 0.f;
  const long long base = static_cast<long long>(rank) * n8;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += stride) {
    float a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    int4 v[kMaxWorld];
#pragma unroll
    for (int r = 0; r < kMaxWorld; ++r)
      if (r < world) v[r] = ld_v4_relaxed_sys(reinterpret_cast<const int4*>(peers.p[r]) + base + i);
#pragma unroll
    for (int r = 0; r < kMaxWorld; ++r)
      if (r < world) acc8(a, v[r]);
    int4 o;
    o.x = pack_bf16x2(a[0] * scale, a[1] * scale);
    o.y = pack_bf16x2(a[2] * scale, a[3] * scale);
    o.z = pack_bf16x2(a[4] * scale, a[5] * scale);
    o.w = pack_bf16x2(a[6] * scale, a[7] * scale);
    if (sumsq_part != nullptr) {
#pragma unroll
      for (int k = 0; k < 8; ++k) ss += (a[k] * scale) * (a[k] * scale);
    }
    if (store_all) {
#pragma unroll
      for (int r = 0; r < kMaxWorld; ++r)
        if (r < world) st_na_v4(reinterpret_cast<int4*>(peers.p[r]) + base + i, o);
    } else {
      st_na_v4(reinterpret_cast<int4*>(peers.p[rank]) + base + i, o);
    }
  }
  if (sumsq_part != nullptr) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x == 0) {
      float s = 0.f;
      for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) s += red[w];
      sumsq_part[blockIdx.x] = s;
    }
  }
}

// *sumsq += Σ_b part[b], in a fixed order: lane l sums blocks l, l + 32, …, then a butterfly.
__global__ void __launch_bounds__(32)
allreduce_sumsq_fold_kernel(const float* __restrict__ part, int nblk, float* __restrict__ sumsq) {
  float s = 0.f;
  for (int b = threadIdx.x; b < nblk; b += 32) s += part[b];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (threadIdx.x == 0) *sumsq += s;
}

// grads: W peer bf16 buffers [W * n8 vectors]; master/m/v: local fp32 shard
// [n8 * 8]; params: W peer bf16 replica buffers [W * n8 vectors].
__global__ void __launch_bounds__(512)
zero_adam_kernel(const PeerPtrs grads, const PeerPtrs params, float* __restrict__ master,
                 float* __restrict__ m, float* __restrict__ v, long long n8, int rank, int world,
                 int grad_world, float grad_scale, const float* __restrict__ grad_scale_ptr, float lr_t, float b1,
                 float b2, float eps) {
  const long long base = static_cast<long long>(rank) * n8;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  float gs = grad_scale;
  if (grad_scale_ptr) gs *= *grad_scale_ptr;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += stride) {
    float g[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int r = 0; r < kMaxWorld; ++r)
      if (r < grad_world)
        acc8(g, ld_v4_relaxed_sys(reinterpret_cast<const int4*>(grads.p[r]) + base + i));
    float4* wp = reinterpret_cast<float4*>(master + i * 8);
    float4* mp = reinterpret_cast<float4*>(m + i * 8);
    float4* vp = reinterpret_cast<float4*>(v + i * 8);
    float w8[8], m8[8], v8[8];
    *reinterpret_cast<float4*>(w8) = wp[0]; *reinterpret_cast<float4*>(w8 + 4) = wp[1];
    *reinterpret_cast<float4*>(m8) = mp[0]; *reinterpret_cast<float4*>(m8 + 4) = mp[1];
    *reinterpret_cast<float4*>(v8) = vp[0]; *reinterpret_cast<float4*>(v8 + 4) = vp[1];
#pragma unroll
    for (int k = 0; k < 8; ++k)
      adam_update(w8[k], m8[k], v8[k], gs == 0.f ? 0.f : g[k] * gs, lr_t, b1, b2, eps);
    wp[0] = *reinterpret_cast<float4*>(w8); wp[1] = *reinterpret_cast<float4*>(w8 + 4);
    mp[0] = *reinterpret_cast<float4*>(m8); mp[1] = *reinterpret_cast<float4*>(m8 + 4);
    vp[0] = *reinterpret_cast<float4*>(v8); vp[1] = *reinterpret_cast<float4*>(v8 + 4);
    int4 o;
    o.x = pack_bf16x2(w8[0], w8[1]);
    o.y = pack_bf16x2(w8[2], w8[3]);
    o.z = pack_bf16x2(w8[4], w8[5]);
    o.w = pack_bf16x2(w8[6], w8[7]);
#pragma unroll
    for (int r = 0; r < kMaxWorld; ++r)
      if (r < world) st_na_v4(reinterpret_cast<int4*>(params.p[r]) + base + i, o);
  }
}

// The kernels dereference entries [0, used) with 16-byte vector accesses.
PeerPtrs ToPeers(const torch::Tensor& t, int64_t used) {
  TORCH_CHECK(t.device().is_cpu() && t.scalar_type() == torch::kInt64 && t.dim() == 1 &&
              t.numel() <= kMaxWorld,
              "peer pointer table must be a 1-D CPU int64 tensor of <= 16 entries");
  TORCH_CHECK(t.numel() >= used, "peer pointer table has ", t.numel(), " entries, ", used,
              " are used");
  const torch::Tensor c = t.contiguous();
  PeerPtrs p;
  for (int i = 0; i < kMaxWorld; ++i) {
    p.p[i] = i < used ? c.data_ptr<int64_t>()[i] : 0;
    TORCH_CHECK(i >= used || (p.p[i] != 0 && p.p[i] % 16 == 0),
                "peer pointer ", i, " must be nonzero and 16-byte aligned");
  }
  return p;
}

void CheckRanks(int64_t rank, int64_t world) {
  TORCH_CHECK(world >= 1 && world <= kMaxWorld, "world must be in [1, 16], got ", world);
  TORCH_CHECK(rank >= 0 && rank < world, "rank must be in [0, world), got ", rank);
}

void CheckF32(const torch::Tensor& t, const torch::Device& dev, const char* what) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == torch::kFloat32 && t.device() == dev, what,
              " must be an fp32 CUDA tensor on ", dev);
}

void CheckShard(const torch::Tensor& t, const torch::Device& dev, const char* what) {
  CheckF32(t, dev, what);
  TORCH_CHECK(t.is_contiguous() && reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0, what,
              " must be contiguous and 16-byte aligned");
}

int Blocks(long long n8) {
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  long long b = (n8 + 511) / 512;
  if (b > sms * 4) b = sms * 4;
  return b < 1 ? 1 : static_cast<int>(b);
}

}  // namespace

// `max_blocks` > 0 caps the grid: a bucket reduced on the communication stream *during*
// backward only needs enough CTAs to keep NVLink busy (≈2 µs of latency × 450 GB/s per
// direction on NVLink-4 ≈ 0.9 MB of 16-byte loads in flight ≈ 16–32 CTAs) and must leave the
// SMs to the GEMMs it overlaps with.
void allreduce_mean_bf16(const torch::Tensor& peer_ptrs_cpu, int64_t shard_elems, int64_t rank,
                         int64_t world, double scale, int64_t device, bool store_all,
                         const c10::optional<torch::Tensor>& sumsq, int64_t max_blocks) {
  TORCH_CHECK(shard_elems >= 0 && shard_elems % 8 == 0,
              "shard_elems must be a non-negative multiple of 8, got ", shard_elems);
  CheckRanks(rank, world);
  const PeerPtrs peers = ToPeers(peer_ptrs_cpu, world);
  const bool with_sumsq = sumsq.has_value() && sumsq->defined();
  const torch::Device dev(torch::kCUDA, static_cast<c10::DeviceIndex>(device));
  if (with_sumsq) {
    CheckF32(*sumsq, dev, "allreduce_mean_bf16: sumsq");
    TORCH_CHECK(sumsq->numel() >= 1, "allreduce_mean_bf16: sumsq is empty");
  }
  const c10::cuda::CUDAGuard guard(dev);
  const long long n8 = shard_elems / 8;
  int blocks = Blocks(n8);
  if (max_blocks > 0 && blocks > max_blocks) blocks = static_cast<int>(max_blocks);
  auto stream = at::cuda::getCurrentCUDAStream();
  // Per-CTA partials from the stream-ordered caching allocator (a CUDA graph's private pool
  // under capture), folded in a fixed order: sumsq is bit-identical from run to run.
  torch::Tensor part;
  if (with_sumsq) part = torch::empty({blocks}, sumsq->options());
  allreduce_mean_bf16_kernel<<<blocks, 512, 0, stream>>>(
      peers, n8, (int)rank, (int)world, (float)scale, store_all ? 1 : 0,
      with_sumsq ? part.data_ptr<float>() : nullptr);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  if (with_sumsq) {
    allreduce_sumsq_fold_kernel<<<1, 32, 0, stream>>>(part.data_ptr<float>(), blocks,
                                                       sumsq->data_ptr<float>());
    C10_CUDA_KERNEL_LAUNCH_CHECK();
  }
  CountLaunch(with_sumsq ? 2 : 1);
}

void zero_adam(const torch::Tensor& grad_peers_cpu, const torch::Tensor& param_peers_cpu,
               torch::Tensor master, torch::Tensor m, torch::Tensor v, int64_t rank, int64_t world,
               int64_t grad_world, double grad_scale, const c10::optional<torch::Tensor>& grad_scale_t, double lr_t,
               double b1, double b2, double eps) {
  TORCH_CHECK(master.is_cuda(), "zero_adam: master must be a CUDA tensor");
  const torch::Device dev = master.device();
  CheckShard(master, dev, "zero_adam: master");
  CheckShard(m, dev, "zero_adam: m");
  CheckShard(v, dev, "zero_adam: v");
  TORCH_CHECK(master.numel() % 8 == 0 && m.numel() == master.numel() && v.numel() == master.numel(),
              "zero_adam: master, m and v must have one size, a multiple of 8");
  CheckRanks(rank, world);
  TORCH_CHECK(grad_world >= 1 && grad_world <= kMaxWorld, "zero_adam: grad_world must be in [1, 16], got ",
              grad_world);
  const PeerPtrs grads = ToPeers(grad_peers_cpu, grad_world);
  const PeerPtrs params = ToPeers(param_peers_cpu, world);
  const bool with_gst = grad_scale_t.has_value() && grad_scale_t->defined();
  if (with_gst) {
    CheckF32(*grad_scale_t, dev, "zero_adam: grad_scale_t");
    TORCH_CHECK(grad_scale_t->numel() >= 1, "zero_adam: grad_scale_t is empty");
  }
  const c10::cuda::CUDAGuard guard(dev);
  const long long n8 = master.numel() / 8;
  const float* gsp = with_gst ? grad_scale_t->data_ptr<float>() : nullptr;
  zero_adam_kernel<<<Blocks(n8), 512, 0, at::cuda::getCurrentCUDAStream()>>>(
      grads, params, master.data_ptr<float>(),
      m.data_ptr<float>(), v.data_ptr<float>(), n8, (int)rank, (int)world, (int)grad_world,
      (float)grad_scale, gsp,
      (float)lr_t, (float)b1, (float)b2, (float)eps);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
}

}  // namespace lb

LB_REGISTER(comm) {
  m.attr("_has_comm") = true;
  m.def("allreduce_mean_bf16", &lb::allreduce_mean_bf16, pybind11::arg("peer_ptrs_cpu"),
        pybind11::arg("shard_elems"), pybind11::arg("rank"), pybind11::arg("world"),
        pybind11::arg("scale"), pybind11::arg("device"), pybind11::arg("store_all"),
        pybind11::arg("sumsq"), pybind11::arg("max_blocks") = 0);
  m.def("zero_adam", &lb::zero_adam);
}
