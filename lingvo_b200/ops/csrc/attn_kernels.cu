// Relative-position-bias attention support kernels (SURVEY K7/K8).
//
//   build_rel_bias : bias[b,h,i,j] = rel[h, i-j+L-1] + mask[b,i,j]  (bf16)
//       one pass, never materialises the fp32 Toeplitz or the broadcast sum.
//   rel_bias_grad  : d rel[h, i-j+L-1] = sum_b sum_{(i,j) on that diagonal} dS[b,h,i,j],
//       dS = P o (dP - delta),  P = exp(scale*QK^T + bias - lse),  dP = dO V^T.
//       wgmma kernel: both 128x128x128 GEMMs of a (h, i-block, j-block) tile are
//       computed by two warpgroups into registers, operands arrive by TMA
//       (SWIZZLE_128B) through a three-slot ring, the warpgroups recompute the
//       softmax from the saved log-sum-exp, accumulate dS over the batch in
//       registers and reduce it along diagonals in shared memory, so neither P,
//       dS nor the [H,L,L] bias gradient ever reaches HBM.
//
// Layouts: q,k,v,dO  [B, L, H, D] bf16 (BLHD, D = 128);  lse, delta [B, H, L] fp32;
//          bias [B, H, L, L] bf16;  rel / drel [H, 2L-1] fp32.

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda.h>
#include <cuda_bf16.h>
#include <torch/extension.h>

#include "ptx.cuh"
#include "registry.h"

namespace lb {

CUtensorMap MakeMap(const void* base, int64_t inner, int64_t rows, int64_t groups,
                    int64_t row_stride, int64_t group_stride, int box_rows,
                    CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, int elem_bytes = 2);

namespace {

// ------------------------------------------------------------ build_rel_bias --
__global__ void __launch_bounds__(256)
build_rel_bias_kernel(const float* __restrict__ rel, const float* __restrict__ mask,
                      __nv_bfloat16* __restrict__ bias, int B, int H, int L, int mask_b) {
  // One block per (i, b) row. A thread owns a PAIR of adjacent columns so that a
  // warp's loads (mask, reversed table) and its 4-byte stores are all contiguous;
  // the mask value is loaded once and reused for every head.
  const int i = blockIdx.x;
  const int b = blockIdx.y;
  const float* mrow = mask ? mask + (static_cast<long long>(mask_b > 1 ? b : 0) * L + i) * L : nullptr;
  for (int j = 2 * threadIdx.x; j < L; j += 2 * blockDim.x) {
    float m0 = 0.f, m1 = 0.f;
    if (mrow) {
      const float2 mm = *reinterpret_cast<const float2*>(mrow + j);
      m0 = mm.x; m1 = mm.y;
    }
    const float* r = rel + (i - j + L - 1);
    __nv_bfloat16* dst = bias + ((static_cast<long long>(b) * H) * L + i) * L + j;
#pragma unroll 4
    for (int h = 0; h < H; ++h) {
      const float f0 = fmaxf(r[0] + m0, -2.3e38f);
      const float f1 = fmaxf(r[-1] + m1, -2.3e38f);
      *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(f0, f1);
      r += 2 * L - 1;
      dst += static_cast<long long>(L) * L;
    }
  }
}

// ------------------------------------------------------------------ row_dot ----
// delta[b,h,l] = sum_d dO[b,l,h,d] * O[b,l,h,d]  (O may be a strided [B,H,L,D] view).
__global__ void __launch_bounds__(256)
attn_delta_kernel(const __nv_bfloat16* __restrict__ d_o, const __nv_bfloat16* __restrict__ o,
                  float* __restrict__ delta, int B, int L, int H, long long o_sb, long long o_sl,
                  long long o_sh) {
  // one warp per (b, l, h) row of D = 128: each lane 4 elements
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= static_cast<long long>(B) * L * H) return;
  const int h = static_cast<int>(row % H);
  const long long bl = row / H;
  const int l = static_cast<int>(bl % L);
  const int b = static_cast<int>(bl / L);
  const uint2 a = *reinterpret_cast<const uint2*>(d_o + row * 128 + lane * 4);
  const uint2 c = *reinterpret_cast<const uint2*>(o + b * o_sb + l * o_sl + h * o_sh + lane * 4);
  const float2 a0 = unpack_bf16x2(a.x), a1 = unpack_bf16x2(a.y);
  const float2 c0 = unpack_bf16x2(c.x), c1 = unpack_bf16x2(c.y);
  float s = a0.x * c0.x + a0.y * c0.y + a1.x * c1.x + a1.y * c1.y;
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
  if (lane == 0) delta[(static_cast<long long>(b) * H + h) * L + l] = s;
}

// -------------------------------------------------------------- rel_bias_grad --
constexpr int kT = 128;                       // tile edge (queries / keys)
constexpr int kD = 128;                       // head dim
constexpr int kChunkBytes = kT * 64 * 2;      // one [128 x 64] SW128 sub-tile = 16 KiB
constexpr int kTileBytes = 2 * kChunkBytes;   // [128 x 128] operand = 32 KiB
constexpr int kSlotBytes = 2 * kTileBytes;    // A + B operand of one GEMM = 64 KiB
constexpr int kSlots = 3;
constexpr int kConsumers = 256;               // two warpgroups x 64 query rows
constexpr int kThreads = kConsumers + 128;    // + the TMA producer warpgroup

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct GradParams {
  const float* lse;      // [B, H, L]
  const float* delta;    // [B, H, L]
  const __nv_bfloat16* bias;   // [B, H, L, L]
  float* drel;           // [H, 2L-1]
  int B, H, L;
  float scale;
  int causal;            // skip tiles strictly above the diagonal
};

// S = Q·K^T and dP = dO·V^T of one (i-block, j-block) tile per batch element, by wgmma into
// registers: warpgroup g owns query rows [64g, 64g + 64) and accumulates dS over the batch.
__global__ void __launch_bounds__(kThreads, 1)
rel_bias_grad_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                     const __grid_constant__ CUtensorMap map_do, const __grid_constant__ CUtensorMap map_v,
                     const GradParams p) {
  const int nblk = p.L / kT;
  const int i_blk = blockIdx.x / nblk;
  const int j_blk = blockIdx.x - i_blk * nblk;
  const int h = blockIdx.y;
  if (p.causal && j_blk > i_blk) return;      // whole CTA exits together: no barriers touched yet

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kSlots * kSlotBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kSlots;
  float* sdiag = reinterpret_cast<float*>(bars + 2 * kSlots + 2);   // [256]

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int i0 = i_blk * kT, j0 = j_blk * kT;

  if (threadIdx.x == kConsumers) {
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_k);
    tma_prefetch_desc(&map_do);
    tma_prefetch_desc(&map_v);
    for (int s = 0; s < kSlots; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), kConsumers / 32);
    }
    fence_barrier_init();
  }
  if (threadIdx.x < 256) sdiag[threadIdx.x] = 0.f;
  __syncthreads();

  if (warp_idx >= kConsumers / 32) {
    // ============================ TMA producer ============================
    setmaxnreg_dec<40>();
    if (threadIdx.x == kConsumers) {
      int slot = 0;
      uint32_t phase = 0;
      for (int b = 0; b < p.B; ++b) {
        for (int g = 0; g < 2; ++g) {
          mbar_wait(smem_u32(&empty_bar[slot]), phase ^ 1);
          const uint32_t fb = smem_u32(&full_bar[slot]);
          mbar_arrive_expect_tx(fb, kSlotBytes);
          const uint32_t sa = smem_u32(smem + slot * kSlotBytes);
          const uint32_t sb = sa + kTileBytes;
          const CUtensorMap* ma = g ? &map_do : &map_q;
          const CUtensorMap* mb = g ? &map_v : &map_k;
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            tma_load_3d(sa + c * kChunkBytes, ma, fb, h * kD + c * 64, i0, b);
            tma_load_3d(sb + c * kChunkBytes, mb, fb, h * kD + c * 64, j0, b);
          }
          if (++slot == kSlots) { slot = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ======================= softmax-recompute warpgroups ====================
  setmaxnreg_inc<232>();
  const int wg = warp_idx >> 2;
  const int row0 = wg * 64 + (warp_idx & 3) * 16 + (lane >> 2);   // tile rows row0, row0 + 8
  const int cq = (lane & 3) * 2;
  constexpr float kLog2e = 1.4426950408889634f;
  const float sl2 = p.scale * kLog2e;
  float ds[64];
#pragma unroll
  for (int c = 0; c < 64; ++c) ds[c] = 0.f;
  int slot = 0;
  uint32_t phase = 0;
  for (int b = 0; b < p.B; ++b) {
    const long long bh = static_cast<long long>(b) * p.H + h;
    float sacc[64], pacc[64];
#pragma unroll
    for (int c = 0; c < 64; ++c) { sacc[c] = 0.f; pacc[c] = 0.f; }
    int slots[2];
#pragma unroll
    for (int g = 0; g < 2; ++g) {
      slots[g] = slot;
      mbar_wait(smem_u32(&full_bar[slot]), phase);
      const uint32_t sa = smem_u32(smem + slot * kSlotBytes);
      const uint32_t sb = sa + kTileBytes;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const uint64_t adesc =
            make_smem_desc_sw128(sa + (kk >> 2) * kChunkBytes + wg * 8192 + (kk & 3) * 32, 16, 1024);
        const uint64_t bdesc = make_smem_desc_sw128(sb + (kk >> 2) * kChunkBytes + (kk & 3) * 32, 16, 1024);
        if (g == 0) wgmma_m64n128k16<0, 0>(sacc, adesc, bdesc, 1);
        else wgmma_m64n128k16<0, 0>(pacc, adesc, bdesc, 1);
      }
      wgmma_commit();
      if (++slot == kSlots) { slot = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(sacc);
    wgmma_fence_regs(pacc);
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(smem_u32(&empty_bar[slots[0]]));
      mbar_arrive(smem_u32(&empty_bar[slots[1]]));
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int qi = i0 + row0 + 8 * i;
      const float lse2 = p.lse[bh * p.L + qi] * kLog2e;
      const float delta = p.delta[bh * p.L + qi];
      const __nv_bfloat16* brow = p.bias + (bh * p.L + qi) * p.L + j0 + cq;
#pragma unroll
      for (int n = 0; n < 16; ++n) {
        const float2 bb = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(brow + n * 8));
        const int e = 4 * n + 2 * i;
        // p = exp(s·scale + bias − lse) = 2^(s·scale·log2e + (bias·log2e − lse·log2e))
        const float p0 = fast_exp2(fmaf(sacc[e], sl2, fmaf(bb.x, kLog2e, -lse2)));
        const float p1 = fast_exp2(fmaf(sacc[e + 1], sl2, fmaf(bb.y, kLog2e, -lse2)));
        ds[e] = fmaf(p0, pacc[e] - delta, ds[e]);
        ds[e + 1] = fmaf(p1, pacc[e + 1] - delta, ds[e + 1]);
      }
    }
  }
  // Diagonal (Toeplitz) reduction: element (row, col) lies on diagonal row - col.
#pragma unroll
  for (int n = 0; n < 16; ++n)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j)
        atomicAdd(&sdiag[row0 + 8 * i - (n * 8 + cq + j) + (kT - 1)], ds[4 * n + 2 * i + j]);
  named_bar_sync(1, kConsumers);
  float* out = p.drel + static_cast<long long>(h) * (2 * p.L - 1) + (i0 - j0) + (p.L - 1) - (kT - 1);
  if (threadIdx.x < 2 * kT - 1) atomicAdd(out + threadIdx.x, sdiag[threadIdx.x]);
}

}  // namespace

torch::Tensor build_rel_bias(const torch::Tensor& rel, const c10::optional<torch::Tensor>& mask,
                             int64_t batch) {
  TORCH_CHECK(rel.is_cuda() && rel.scalar_type() == torch::kFloat32 && rel.dim() == 2 &&
              rel.is_contiguous(), "build_rel_bias: rel must be fp32 [H, 2L-1]");
  const int64_t H = rel.size(0);
  const int64_t L = (rel.size(1) + 1) / 2;
  TORCH_CHECK(L % 2 == 0, "build_rel_bias: L must be even");
  const c10::cuda::CUDAGuard guard(rel.device());
  const float* mptr = nullptr;
  int mask_b = 1;
  torch::Tensor m;
  if (mask.has_value() && mask->defined()) {
    m = mask->to(torch::kFloat32).contiguous();
    TORCH_CHECK(m.numel() == L * L || m.numel() == batch * L * L, "build_rel_bias: mask shape");
    mask_b = m.numel() == L * L ? 1 : static_cast<int>(batch);
    mptr = m.data_ptr<float>();
  }
  auto bias = torch::empty({batch, H, L, L}, rel.options().dtype(torch::kBFloat16));
  dim3 grid(static_cast<unsigned>(L), static_cast<unsigned>(batch));
  build_rel_bias_kernel<<<grid, 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      rel.data_ptr<float>(), mptr, reinterpret_cast<__nv_bfloat16*>(bias.data_ptr()),
      static_cast<int>(batch), static_cast<int>(H), static_cast<int>(L), mask_b);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return bias;
}

// Returns d rel [H, 2L-1] (fp32).
// q,k,v,dO: [B, L, H, D] views with unit D stride and head stride D (slices of a fused
// qkv projection are fine); `out` is the attention output as a [B, H, L, D] view.
torch::Tensor rel_bias_grad(const torch::Tensor& q, const torch::Tensor& k, const torch::Tensor& v,
                            const torch::Tensor& d_out, const torch::Tensor& out,
                            const torch::Tensor& lse, const torch::Tensor& bias, double scale,
                            bool causal) {
  TORCH_CHECK(q.is_cuda() && q.scalar_type() == torch::kBFloat16 && q.dim() == 4,
              "rel_bias_grad: q must be bf16 [B, L, H, D]");
  const int64_t B = q.size(0), L = q.size(1), H = q.size(2), D = q.size(3);
  TORCH_CHECK(D == kD && L % kT == 0, "rel_bias_grad: needs D == 128 and L % 128 == 0");
  for (const torch::Tensor* t : {&q, &k, &v, &d_out})
    TORCH_CHECK(t->sizes() == q.sizes() && t->scalar_type() == torch::kBFloat16 &&
                    t->stride(3) == 1 && t->stride(2) == D && t->stride(1) % 8 == 0 &&
                    t->stride(0) % 8 == 0 && reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0,
                "rel_bias_grad: q/k/v/dO must be [B,L,H,D] views with strides (*, *, D, 1)");
  TORCH_CHECK(d_out.is_contiguous(), "rel_bias_grad: dO must be contiguous");
  TORCH_CHECK(out.scalar_type() == torch::kBFloat16 && out.dim() == 4 && out.size(0) == B &&
                  out.size(1) == H && out.size(2) == L && out.size(3) == D && out.stride(3) == 1,
              "rel_bias_grad: out must be a bf16 [B, H, L, D] view");
  TORCH_CHECK(lse.scalar_type() == torch::kFloat32 && lse.is_contiguous() && lse.numel() == B * H * L);
  TORCH_CHECK(bias.scalar_type() == torch::kBFloat16 && bias.is_contiguous() &&
              bias.numel() == B * H * L * L, "rel_bias_grad: bias must be bf16 [B, H, L, L]");
  const c10::cuda::CUDAGuard guard(q.device());
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
  auto drel = torch::zeros({H, 2 * L - 1}, q.options().dtype(torch::kFloat32));
  auto delta = torch::empty({B, H, L}, q.options().dtype(torch::kFloat32));
  {
    const long long rows = B * L * H;
    const int blocks = static_cast<int>((rows * 32 + 255) / 256);
    attn_delta_kernel<<<blocks, 256, 0, at::cuda::getCurrentCUDAStream()>>>(
        reinterpret_cast<const __nv_bfloat16*>(d_out.data_ptr()),
        reinterpret_cast<const __nv_bfloat16*>(out.data_ptr()), delta.data_ptr<float>(),
        static_cast<int>(B), static_cast<int>(L), static_cast<int>(H), out.stride(0),
        out.stride(2), out.stride(1));
    C10_CUDA_KERNEL_LAUNCH_CHECK();
    CountLaunch();
  }
  auto mk = [&](const torch::Tensor& t) {
    return MakeMap(t.data_ptr(), H * D, L, B, t.stride(1), t.stride(0), kT);
  };
  const CUtensorMap mq = mk(q), mkk = mk(k), mdo = mk(d_out), mv = mk(v);
  GradParams p;
  p.lse = lse.data_ptr<float>();
  p.delta = delta.data_ptr<float>();
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias.data_ptr());
  p.drel = drel.data_ptr<float>();
  p.B = static_cast<int>(B); p.H = static_cast<int>(H); p.L = static_cast<int>(L);
  p.scale = static_cast<float>(scale);
  p.causal = causal ? 1 : 0;
  constexpr size_t smem = kSlots * kSlotBytes + 1024 + 128 + 1024 + 64;
  static bool configured = false;
  if (!configured) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(rel_bias_grad_kernel,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(smem)));
    configured = true;
  }
  const int nblk = static_cast<int>(L / kT);
  dim3 grid(nblk * nblk, static_cast<unsigned>(H));
  rel_bias_grad_kernel<<<grid, kThreads, smem, at::cuda::getCurrentCUDAStream()>>>(mq, mkk, mdo, mv, p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return drel;
}

}  // namespace lb

LB_REGISTER(attn) {
  m.attr("_has_attn") = true;
  m.def("build_rel_bias", &lb::build_rel_bias, py::arg("rel"), py::arg("mask"), py::arg("batch"));
  m.def("rel_bias_grad", &lb::rel_bias_grad);
}
