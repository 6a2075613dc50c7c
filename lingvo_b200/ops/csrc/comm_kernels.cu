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
//   tp_reduce_slabs : owner-side sum of the W partial slabs written by the
//       row-pointer epilogue of the tensor-parallel GEMM (GEMM -> reduce-scatter).
// Flags (moe_signal / moe_wait) order the phases across ranks.

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

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
__global__ void __launch_bounds__(512)
allreduce_mean_bf16_kernel(const PeerPtrs peers, long long n8, int rank, int world, float scale,
                           int store_all, float* __restrict__ sumsq) {
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
    if (sumsq != nullptr) {
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
  if (sumsq != nullptr) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(sumsq, ss);
  }
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
    for (int k = 0; k < 8; ++k) {
      const float gg = gs == 0.f ? 0.f : g[k] * gs;
      m8[k] = b1 * m8[k] + (1.f - b1) * gg;
      v8[k] = b2 * v8[k] + (1.f - b2) * gg * gg;
      w8[k] -= lr_t * m8[k] / (sqrtf(v8[k]) + eps);
    }
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

// out[row, :] = sum_w slabs[w, row, :]   (bf16 in, bf16 out, fp32 accumulate)
__global__ void tp_reduce_slabs_kernel(const __nv_bfloat16* __restrict__ slabs,
                                       __nv_bfloat16* __restrict__ out, long long n8, int world) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += stride) {
    float a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int w = 0; w < world; ++w)
      acc8(a, *(reinterpret_cast<const int4*>(slabs) + static_cast<long long>(w) * n8 + i));
    int4 o;
    o.x = pack_bf16x2(a[0], a[1]);
    o.y = pack_bf16x2(a[2], a[3]);
    o.z = pack_bf16x2(a[4], a[5]);
    o.w = pack_bf16x2(a[6], a[7]);
    *(reinterpret_cast<int4*>(out) + i) = o;
  }
}

// Same sum, but the reduced [rows, cols] block is stored at column offset
// `col_off` of a [rows, out_ld] matrix on every peer (reduce-scatter + all-gather
// = all-reduce, with the gather done by NVLink stores from the reducing rank).
__global__ void tp_reduce_bcast_kernel(const __nv_bfloat16* __restrict__ slabs, const PeerPtrs outs,
                                       int n_out, long long rows, int cols8, long long out_ld8,
                                       int col_off8, int world) {
  const long long n8 = rows * cols8;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += stride) {
    float a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int w = 0; w < world; ++w)
      acc8(a, *(reinterpret_cast<const int4*>(slabs) + static_cast<long long>(w) * n8 + i));
    int4 o;
    o.x = pack_bf16x2(a[0], a[1]);
    o.y = pack_bf16x2(a[2], a[3]);
    o.z = pack_bf16x2(a[4], a[5]);
    o.w = pack_bf16x2(a[6], a[7]);
    const long long r = i / cols8;
    const long long dst = r * out_ld8 + col_off8 + (i - r * cols8);
    for (int q = 0; q < n_out; ++q) *(reinterpret_cast<int4*>(outs.p[q]) + dst) = o;
  }
}

PeerPtrs ToPeers(const torch::Tensor& t) {
  TORCH_CHECK(t.device().is_cpu() && t.scalar_type() == torch::kInt64 && t.numel() <= kMaxWorld,
              "peer pointer table must be a CPU int64 tensor of <= 16 entries");
  PeerPtrs p;
  for (int i = 0; i < kMaxWorld; ++i) p.p[i] = i < t.numel() ? t.data_ptr<int64_t>()[i] : 0;
  return p;
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
  TORCH_CHECK(shard_elems % 8 == 0);
  const c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  const long long n8 = shard_elems / 8;
  int blocks = Blocks(n8);
  if (max_blocks > 0 && blocks > max_blocks) blocks = static_cast<int>(max_blocks);
  allreduce_mean_bf16_kernel<<<blocks, 512, 0, at::cuda::getCurrentCUDAStream()>>>(
      ToPeers(peer_ptrs_cpu), n8, (int)rank, (int)world, (float)scale, store_all ? 1 : 0,
      (sumsq.has_value() && sumsq->defined()) ? sumsq->data_ptr<float>() : nullptr);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
}

void zero_adam(const torch::Tensor& grad_peers_cpu, const torch::Tensor& param_peers_cpu,
               torch::Tensor master, torch::Tensor m, torch::Tensor v, int64_t rank, int64_t world,
               int64_t grad_world, double grad_scale, const c10::optional<torch::Tensor>& grad_scale_t, double lr_t,
               double b1, double b2, double eps) {
  TORCH_CHECK(master.is_cuda() && master.scalar_type() == torch::kFloat32 && master.is_contiguous());
  TORCH_CHECK(master.numel() % 8 == 0 && m.numel() == master.numel() && v.numel() == master.numel());
  const c10::cuda::CUDAGuard guard(master.device());
  const long long n8 = master.numel() / 8;
  const float* gsp = (grad_scale_t.has_value() && grad_scale_t->defined())
                         ? grad_scale_t->data_ptr<float>() : nullptr;
  zero_adam_kernel<<<Blocks(n8), 512, 0, at::cuda::getCurrentCUDAStream()>>>(
      ToPeers(grad_peers_cpu), ToPeers(param_peers_cpu), master.data_ptr<float>(),
      m.data_ptr<float>(), v.data_ptr<float>(), n8, (int)rank, (int)world, (int)grad_world,
      (float)grad_scale, gsp,
      (float)lr_t, (float)b1, (float)b2, (float)eps);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
}

torch::Tensor tp_reduce_slabs(const torch::Tensor& slabs, int64_t world) {
  TORCH_CHECK(slabs.is_cuda() && slabs.scalar_type() == torch::kBFloat16 && slabs.is_contiguous());
  TORCH_CHECK(slabs.size(0) == world && (slabs.numel() / world) % 8 == 0);
  const c10::cuda::CUDAGuard guard(slabs.device());
  auto sizes = slabs.sizes().vec();
  sizes.erase(sizes.begin());
  auto out = torch::empty(sizes, slabs.options());
  const long long n8 = out.numel() / 8;
  tp_reduce_slabs_kernel<<<Blocks(n8), 512, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const __nv_bfloat16*>(slabs.data_ptr()),
      reinterpret_cast<__nv_bfloat16*>(out.data_ptr()), n8, (int)world);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return out;
}

void tp_reduce_bcast(const torch::Tensor& slabs, int64_t world, const torch::Tensor& out_ptrs_cpu,
                     int64_t out_ld, int64_t col_off) {
  TORCH_CHECK(slabs.is_cuda() && slabs.scalar_type() == torch::kBFloat16 && slabs.is_contiguous() &&
              slabs.dim() == 3 && slabs.size(0) == world);
  const int64_t rows = slabs.size(1), cols = slabs.size(2);
  TORCH_CHECK(cols % 8 == 0 && out_ld % 8 == 0 && col_off % 8 == 0);
  const c10::cuda::CUDAGuard guard(slabs.device());
  const long long n8 = rows * cols / 8;
  tp_reduce_bcast_kernel<<<Blocks(n8), 512, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const __nv_bfloat16*>(slabs.data_ptr()), ToPeers(out_ptrs_cpu),
      static_cast<int>(out_ptrs_cpu.numel()), rows, static_cast<int>(cols / 8), out_ld / 8,
      static_cast<int>(col_off / 8), static_cast<int>(world));
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
}

}  // namespace lb

LB_REGISTER(comm) {
  m.def("tp_reduce_bcast", &lb::tp_reduce_bcast);
  m.attr("_has_comm") = true;
  m.def("allreduce_mean_bf16", &lb::allreduce_mean_bf16, pybind11::arg("peer_ptrs_cpu"),
        pybind11::arg("shard_elems"), pybind11::arg("rank"), pybind11::arg("world"),
        pybind11::arg("scale"), pybind11::arg("device"), pybind11::arg("store_all"),
        pybind11::arg("sumsq"), pybind11::arg("max_blocks") = 0);
  m.def("zero_adam", &lb::zero_adam);
  m.def("tp_reduce_slabs", &lb::tp_reduce_slabs);
}
