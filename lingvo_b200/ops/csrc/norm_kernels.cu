// Fused normalisation kernels (bf16 activations, fp32 statistics).
//
//   rms_norm      y = x * rsqrt(mean(x^2) + eps) * scale          (GShard "_LN")
//   layer_norm    y = (x - mean) * rsqrt(var + eps) * scale + bias (core LayerNorm)
// The forward also writes each row's (mean, rstd). The backward is a dx kernel, which can add
// the gradient flowing along the residual stream (`dres_in`), and, when the parameter
// gradients are wanted, a dscale / dbias column reduction into per-row-block partials that a
// fold kernel sums in a fixed order (no atomics).
//
// Forward and dx: one warp owns a row; 16-byte vector loads; rows are streamed by a
// persistent grid (132 SMs x 8 CTAs). Memory-bound: forward reads x once and writes y once;
// the dx kernel reads x, dy once and writes dx once.

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "ptx.cuh"
#include "registry.h"

namespace lb {
namespace {

constexpr int kWarpsPerCta = 8;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&f)[8]) {
  int4 v = *reinterpret_cast<const int4*>(p);
  const uint32_t w[4] = {static_cast<uint32_t>(v.x), static_cast<uint32_t>(v.y),
                         static_cast<uint32_t>(v.z), static_cast<uint32_t>(v.w)};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float2 t = unpack_bf16x2(w[j]);
    f[2 * j] = t.x;
    f[2 * j + 1] = t.y;
  }
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&f)[8]) {
  int4 o;
  o.x = pack_bf16x2(f[0], f[1]);
  o.y = pack_bf16x2(f[2], f[3]);
  o.z = pack_bf16x2(f[4], f[5]);
  o.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<int4*>(p) = o;
}
__device__ __forceinline__ void load8f(const float* p, float (&f)[8]) {
  float4 a = *reinterpret_cast<const float4*>(p);
  float4 b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

// kCenter: true = LayerNorm (mean subtraction, optional bias), false = RMS norm.
template <bool kCenter>
__global__ void __launch_bounds__(kWarpsPerCta * 32)
norm_fwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ scale,
                const float* __restrict__ bias, __nv_bfloat16* __restrict__ y,
                float* __restrict__ stats /* [rows, 2] = (mean, rstd) */, int rows, int dim,
                float eps) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int warps_total = gridDim.x * kWarpsPerCta;
  for (int row = blockIdx.x * kWarpsPerCta + warp; row < rows; row += warps_total) {
    const __nv_bfloat16* xr = x + static_cast<size_t>(row) * dim;
    float s1 = 0.f, s2 = 0.f;
    // Unroll factors of the two passes: the fastest spill-free pair for both variants at
    // [8192, 2048] on H100 (the compiler's default spills 8 bytes in the RMS variant).
#pragma unroll 2
    for (int c = lane * 8; c < dim; c += 256) {
      float f[8];
      load8(xr + c, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) { s1 += f[i]; s2 += f[i] * f[i]; }
    }
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    const float mean = kCenter ? s1 / dim : 0.f;
    const float var = kCenter ? fmaxf(s2 / dim - mean * mean, 0.f) : s2 / dim;
    const float rstd = rsqrtf(var + eps);
    if (lane == 0 && stats) { stats[2 * row] = mean; stats[2 * row + 1] = rstd; }
#pragma unroll 4
    for (int c = lane * 8; c < dim; c += 256) {
      float f[8], sc[8];
      load8(xr + c, f);
      if (scale) load8f(scale + c, sc);
      float o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        o[i] = (f[i] - mean) * rstd;
        if (scale) o[i] *= sc[i];
      }
      if (kCenter && bias) {
        float b[8];
        load8f(bias + c, b);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] += b[i];
      }
      store8(y + static_cast<size_t>(row) * dim + c, o);
    }
  }
}

// Backward, dx only: dx = rstd * (g - mean(g) - xhat * mean(g * xhat)) with g = dy * scale
// (mean(g) only when centring), plus the gradient flowing along the residual stream when
// `dres_in` is given. dscale / dbias come from norm_dscale_kernel and the fold.
template <bool kCenter>
__global__ void __launch_bounds__(kWarpsPerCta * 32)
norm_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                const __nv_bfloat16* __restrict__ dres_in /* grad flowing on the residual stream */,
                const float* __restrict__ scale, const float* __restrict__ stats,
                __nv_bfloat16* __restrict__ dx, int rows, int dim) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int warps_total = gridDim.x * kWarpsPerCta;
  for (int row = blockIdx.x * kWarpsPerCta + warp; row < rows; row += warps_total) {
    const size_t off = static_cast<size_t>(row) * dim;
    const float mean = stats[2 * row], rstd = stats[2 * row + 1];
    float c1 = 0.f, c2 = 0.f;   // sum(g), sum(g * xhat) with g = dy * scale
    // A 64-bit index: 54 instead of 60 us with an int one, both variants at [8192, 2048] on an
    // H100 80GB HBM3 (700 W limit).
    for (size_t c = lane * 8; c < static_cast<size_t>(dim); c += 256) {
      float xf[8], gf[8], sc[8];
      load8(x + off + c, xf);
      load8(dy + off + c, gf);
      if (scale) load8f(scale + c, sc);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float xhat = (xf[i] - mean) * rstd;
        const float g = scale ? gf[i] * sc[i] : gf[i];
        c1 += g;
        c2 += g * xhat;
      }
    }
    c1 = warp_sum(c1) / dim;
    c2 = warp_sum(c2) / dim;
    if (!kCenter) c1 = 0.f;
    for (int c = lane * 8; c < dim; c += 256) {
      float xf[8], gf[8], sc[8], o[8];
      load8(x + off + c, xf);
      load8(dy + off + c, gf);
      if (scale) load8f(scale + c, sc);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float xhat = (xf[i] - mean) * rstd;
        const float g = scale ? gf[i] * sc[i] : gf[i];
        o[i] = rstd * (g - c1 - xhat * c2);
      }
      if (dres_in) {
        float r[8];
        load8(dres_in + off + c, r);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] += r[i];
      }
      store8(dx + off + c, o);
    }
  }
}

// dscale / dbias partials as a column reduction (the layout of the Adafactor statistics
// kernel): one CTA per (32-row block, 2048-column chunk), warp w sweeps the 32 rows of its
// own 256-column strip with the column sums in registers, and leaves one partial row per
// row block. Runs right after the dx kernel, so x and dy mostly come from L2.
constexpr int kDsRows = 16;
template <bool kCenter>
__global__ void __launch_bounds__(kWarpsPerCta * 32)
norm_dscale_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                   const float* __restrict__ stats, float* __restrict__ part_s,
                   float* __restrict__ part_b, int rows, int dim, int nchunk) {
  __shared__ float st[kDsRows][2];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int chunk = blockIdx.x % nchunk, blk = blockIdx.x / nchunk;
  const int r0 = blk * kDsRows;
  const int nrows = min(kDsRows, rows - r0);
  if (threadIdx.x < 2 * nrows) st[threadIdx.x >> 1][threadIdx.x & 1] = stats[2 * r0 + threadIdx.x];
  __syncthreads();
  const int c = chunk * (kWarpsPerCta * 256) + warp * 256 + lane * 8;
  if (c >= dim) return;
  float cs[8] = {0, 0, 0, 0, 0, 0, 0, 0}, cb[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const size_t base = static_cast<size_t>(r0) * dim + c;
  int r = 0;
  for (; r + 4 <= nrows; r += 4) {
    float xf[4][8], gf[4][8];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      load8(x + base + static_cast<size_t>(r + u) * dim, xf[u]);
      load8(dy + base + static_cast<size_t>(r + u) * dim, gf[u]);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float mean = st[r + u][0], rstd = st[r + u][1];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        cs[i] = fmaf(gf[u][i], (xf[u][i] - mean) * rstd, cs[i]);
        if (kCenter) cb[i] += gf[u][i];
      }
    }
  }
  for (; r < nrows; ++r) {
    float xf[8], gf[8];
    load8(x + base + static_cast<size_t>(r) * dim, xf);
    load8(dy + base + static_cast<size_t>(r) * dim, gf);
    const float mean = st[r][0], rstd = st[r][1];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      cs[i] = fmaf(gf[i], (xf[i] - mean) * rstd, cs[i]);
      if (kCenter) cb[i] += gf[i];
    }
  }
  if (part_s != nullptr) {
    float* q = part_s + static_cast<size_t>(blk) * dim + c;
    *reinterpret_cast<float4*>(q) = make_float4(cs[0], cs[1], cs[2], cs[3]);
    *reinterpret_cast<float4*>(q + 4) = make_float4(cs[4], cs[5], cs[6], cs[7]);
  }
  if (kCenter && part_b != nullptr) {
    float* q = part_b + static_cast<size_t>(blk) * dim + c;
    *reinterpret_cast<float4*>(q) = make_float4(cb[0], cb[1], cb[2], cb[3]);
    *reinterpret_cast<float4*>(q + 4) = make_float4(cb[4], cb[5], cb[6], cb[7]);
  }
}

// out[i] = Σ_k part[k][i]. Block = 32 columns × 8 row groups: coalesced 128-byte reads, the
// 8 partial sums per column meet in shared memory.
__global__ void __launch_bounds__(256)
norm_bwd_fold_kernel(const float* __restrict__ part_s, const float* __restrict__ part_b,
                     float* __restrict__ out_s, float* __restrict__ out_b, int dim, int nblk) {
  __shared__ float red[8][33];
  const float* part = blockIdx.y == 0 ? part_s : part_b;
  float* out = blockIdx.y == 0 ? out_s : out_b;
  if (part == nullptr) return;
  const int cx = threadIdx.x & 31, ky = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + cx;
  float s0 = 0.f, s1 = 0.f;
  if (i < dim) {
    int k = ky;
    for (; k + 8 < nblk; k += 16) {
      s0 += part[static_cast<size_t>(k) * dim + i];
      s1 += part[static_cast<size_t>(k + 8) * dim + i];
    }
    if (k < nblk) s0 += part[static_cast<size_t>(k) * dim + i];
  }
  red[ky][cx] = s0 + s1;
  __syncthreads();
  if (ky == 0 && i < dim) {
    float s = 0.f;
#pragma unroll
    for (int r = 0; r < 8; ++r) s += red[r][cx];
    out[i] = s;
  }
}

bool Aligned16(const torch::Tensor& t) {
  return reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0;
}

// scale / bias as the fp32 [dim] vector the kernels read with 16-byte loads.
torch::Tensor ParamVector(const torch::Tensor& v, const torch::Tensor& x, int dim,
                          const char* name) {
  TORCH_CHECK(v.device() == x.device() && v.numel() == dim, "norm: ", name, " must have ", dim,
              " elements on x's device, got ", v.numel());
  auto f = v.to(torch::kFloat32).contiguous();
  TORCH_CHECK(Aligned16(f), "norm: ", name, " must be 16-byte aligned");
  return f;
}

int GridFor(int rows) {
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  int ctas = (rows + kWarpsPerCta - 1) / kWarpsPerCta;
  return ctas < sms * 8 ? ctas : sms * 8;
}

}  // namespace

// Returns (y, stats[rows,2]).
std::vector<torch::Tensor> norm_fwd(const torch::Tensor& x,
                                    const c10::optional<torch::Tensor>& scale,
                                    const c10::optional<torch::Tensor>& bias, double eps,
                                    bool center) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == torch::kBFloat16 && x.is_contiguous(),
              "norm: x must be a contiguous CUDA bf16 tensor");
  const int dim = x.dim() > 0 ? static_cast<int>(x.size(-1)) : 0;
  TORCH_CHECK(dim > 0 && dim % 8 == 0, "norm: last dim must be a positive multiple of 8");
  TORCH_CHECK(Aligned16(x), "norm: x must be 16-byte aligned");
  torch::Tensor sc, bi;
  if (scale.has_value() && scale->defined()) sc = ParamVector(*scale, x, dim, "scale");
  if (bias.has_value() && bias->defined()) bi = ParamVector(*bias, x, dim, "bias");
  const c10::cuda::CUDAGuard guard(x.device());
  const int rows = static_cast<int>(x.numel() / dim);
  auto y = torch::empty_like(x);
  auto stats = torch::empty({rows, 2}, x.options().dtype(torch::kFloat32));
  if (rows == 0) return {y, stats};
  auto stream = at::cuda::getCurrentCUDAStream();
  const int grid = GridFor(rows);
  auto xp = reinterpret_cast<const __nv_bfloat16*>(x.data_ptr());
  auto yp = reinterpret_cast<__nv_bfloat16*>(y.data_ptr());
  if (center)
    norm_fwd_kernel<true><<<grid, kWarpsPerCta * 32, 0, stream>>>(
        xp, sc.defined() ? sc.data_ptr<float>() : nullptr,
        bi.defined() ? bi.data_ptr<float>() : nullptr, yp, stats.data_ptr<float>(), rows, dim,
        static_cast<float>(eps));
  else
    norm_fwd_kernel<false><<<grid, kWarpsPerCta * 32, 0, stream>>>(
        xp, sc.defined() ? sc.data_ptr<float>() : nullptr, nullptr, yp,
        stats.data_ptr<float>(), rows, dim, static_cast<float>(eps));
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return {y, stats};
}

// x is the norm's input, stats what norm_fwd returned for it. Returns (dx, dscale, dbias).
std::vector<torch::Tensor> norm_bwd(const torch::Tensor& x, const torch::Tensor& dy,
                                    const c10::optional<torch::Tensor>& dres,
                                    const c10::optional<torch::Tensor>& scale,
                                    const torch::Tensor& stats, bool center, bool need_dscale,
                                    bool need_dbias) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == torch::kBFloat16 && x.is_contiguous(),
              "norm_bwd: x must be a contiguous CUDA bf16 tensor");
  const int dim = x.dim() > 0 ? static_cast<int>(x.size(-1)) : 0;
  TORCH_CHECK(dim > 0 && dim % 8 == 0, "norm_bwd: last dim must be a positive multiple of 8");
  TORCH_CHECK(dy.device() == x.device() && dy.scalar_type() == torch::kBFloat16 &&
              dy.is_contiguous() && dy.sizes() == x.sizes(),
              "norm_bwd: dy must be a contiguous bf16 tensor of x's shape");
  TORCH_CHECK(Aligned16(x) && Aligned16(dy), "norm_bwd: x and dy must be 16-byte aligned");
  const int rows = static_cast<int>(x.numel() / dim);
  TORCH_CHECK(stats.device() == x.device() && stats.scalar_type() == torch::kFloat32 &&
              stats.is_contiguous() && stats.dim() == 2 && stats.size(0) == rows &&
              stats.size(1) == 2, "norm_bwd: stats must be contiguous fp32 [rows, 2]");
  const bool has_dres = dres.has_value() && dres->defined();
  if (has_dres)
    TORCH_CHECK(dres->device() == x.device() && dres->scalar_type() == torch::kBFloat16 &&
                dres->is_contiguous() && dres->numel() == x.numel() && Aligned16(*dres),
                "norm_bwd: dres must be a contiguous 16-byte-aligned bf16 tensor like x");
  torch::Tensor sc, ds, db;
  if (scale.has_value() && scale->defined()) sc = ParamVector(*scale, x, dim, "scale");
  const c10::cuda::CUDAGuard guard(x.device());
  auto dx = torch::empty_like(x);
  if (need_dscale) ds = torch::empty({dim}, x.options().dtype(torch::kFloat32));
  if (need_dbias) db = torch::empty({dim}, x.options().dtype(torch::kFloat32));
  if (rows == 0) {
    if (ds.defined()) ds.zero_();
    if (db.defined()) db.zero_();
    return {dx, ds, db};
  }
  const __nv_bfloat16* drp =
      has_dres ? reinterpret_cast<const __nv_bfloat16*>(dres->data_ptr()) : nullptr;
  auto stream = at::cuda::getCurrentCUDAStream();
  // dx: one light streaming kernel on a persistent grid; dscale / dbias: column-reduction
  // kernel + fold.
  const int grid = GridFor(rows);
  auto xp = reinterpret_cast<const __nv_bfloat16*>(x.data_ptr());
  auto dyp = reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr());
  auto dxp = reinterpret_cast<__nv_bfloat16*>(dx.data_ptr());
  const float* scp = sc.defined() ? sc.data_ptr<float>() : nullptr;
  if (center)
    norm_bwd_kernel<true><<<grid, kWarpsPerCta * 32, 0, stream>>>(
        xp, dyp, drp, scp, stats.data_ptr<float>(), dxp, rows, dim);
  else
    norm_bwd_kernel<false><<<grid, kWarpsPerCta * 32, 0, stream>>>(
        xp, dyp, drp, scp, stats.data_ptr<float>(), dxp, rows, dim);
  const bool want_b = need_dbias && center;
  if (need_dscale || want_b) {
    const int nblk = (rows + kDsRows - 1) / kDsRows;
    const int nchunk = (dim + kWarpsPerCta * 256 - 1) / (kWarpsPerCta * 256);
    torch::Tensor part_s, part_b;
    if (need_dscale) part_s = torch::empty({nblk, dim}, x.options().dtype(torch::kFloat32));
    if (want_b) part_b = torch::empty({nblk, dim}, x.options().dtype(torch::kFloat32));
    float* psp = part_s.defined() ? part_s.data_ptr<float>() : nullptr;
    float* pbp = part_b.defined() ? part_b.data_ptr<float>() : nullptr;
    if (center)
      norm_dscale_kernel<true><<<nblk * nchunk, kWarpsPerCta * 32, 0, stream>>>(
          xp, dyp, stats.data_ptr<float>(), psp, pbp, rows, dim, nchunk);
    else
      norm_dscale_kernel<false><<<nblk * nchunk, kWarpsPerCta * 32, 0, stream>>>(
          xp, dyp, stats.data_ptr<float>(), psp, pbp, rows, dim, nchunk);
    norm_bwd_fold_kernel<<<dim3((dim + 31) / 32, 2), 256, 0, stream>>>(
        psp, pbp, ds.defined() ? ds.data_ptr<float>() : nullptr,
        db.defined() ? db.data_ptr<float>() : nullptr, dim, nblk);
    CountLaunch(2);
  }
  if (need_dbias && !center) db.zero_();
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return {dx, ds.defined() ? ds : torch::Tensor(), db.defined() ? db : torch::Tensor()};
}

}  // namespace lb

LB_REGISTER(norm) {
  m.def("norm_fwd", &lb::norm_fwd);
  m.def("norm_bwd", &lb::norm_bwd);
}
