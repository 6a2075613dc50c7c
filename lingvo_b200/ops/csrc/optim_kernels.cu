// Fused optimizer kernels (fp32 master weights, bf16/fp32 gradients, optional
// bf16 compute-copy written in the same pass).
//
// Adafactor (factored second moment; reference optimizer.py:1129-1218) over a
// variable viewed as [B, R, C] is four launches with no host sync:
//   A  stats   : rowsum[B,R], colsum[B,C] of (g^2 + eps1); acc[0] += sum(w^2)
//   B  factors : EMA-update vr / vc in place, long-term mean, write the two
//                factor vectors fr[B,R], fc[B,C]
//   C  rms     : acc[1] += sum((g * fr * fc)^2)
//   D  apply   : w -= g*fr*fc * max(rms(w), eps2)*lr / max(1, rms(x)/clip);
//                bf16 copy of w written alongside.
// HBM traffic ~ 3 reads of g + read/write of w + write of the bf16 copy.
// Sums that span CTAs (row sums across column chunks, Σg², Σw², the clipping RMS) are
// written as per-CTA / per-warp partials and folded in a fixed order, never by float
// atomics, so the same inputs give bit-identical updates on every run.
//
// adam_flat: elementwise Adam on a flat fp32 shard with grad scale and bf16
// copy-out — the update half of the fused reduce-scatter + partitioned Adam.

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <map>
#include <mutex>
#include <utility>

#include "adam.cuh"
#include "ptx.cuh"
#include "registry.h"

namespace lb {
namespace {

constexpr int kRowsPerWarp = 64;
constexpr int kWarps = 8;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename GT>
__device__ __forceinline__ void load_g8(const GT* p, float (&f)[8]);
template <>
__device__ __forceinline__ void load_g8<__nv_bfloat16>(const __nv_bfloat16* p, float (&f)[8]) {
  int4 v = *reinterpret_cast<const int4*>(p);
  const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float2 t = unpack_bf16x2(w[j]);
    f[2 * j] = t.x;
    f[2 * j + 1] = t.y;
  }
}
template <>
__device__ __forceinline__ void load_g8<float>(const float* p, float (&f)[8]) {
  float4 a = *reinterpret_cast<const float4*>(p);
  float4 b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

struct Tile {
  int b, r0, r1, c0;
  bool ok;
};
// Work item = (batch b, 64-row range, 256-column strip); one warp per item.
__device__ __forceinline__ Tile get_tile(int item, int R, int C) {
  const int strips = (C + 255) / 256;
  const int ranges = (R + kRowsPerWarp - 1) / kRowsPerWarp;
  Tile t;
  t.b = item / (strips * ranges);
  const int rem = item - t.b * strips * ranges;
  const int range = rem / strips;
  t.c0 = (rem - range * strips) * 256;
  t.r0 = range * kRowsPerWarp;
  t.r1 = min(t.r0 + kRowsPerWarp, R);
  return t;
}

constexpr int kStatRows = 32;            // rows per CTA tile
constexpr int kStatCols = kWarps * 256;  // columns per CTA tile (one 256-wide strip per warp)

// One CTA per (batch b, 32-row block, 2048-column chunk); warp w sweeps the 32 rows of its
// own 256-column strip. Column sums stay in registers and leave as one partial row per
// row block (colpart[b][blk][C], plain stores, folded by adafactor_colreduce_kernel); row
// sums are warp-reduced, combined across the 8 strips in shared memory and reach global
// memory as one add per (row, chunk). No shared-memory atomics (fp32 ATOMS is a CAS spin
// loop) and no contended global atomics.
template <typename GT>
__global__ void __launch_bounds__(kWarps * 32)
adafactor_stats_kernel(const GT* __restrict__ g, const float* __restrict__ w,
                       float* __restrict__ rowsum, float* __restrict__ colpart,
                       float* __restrict__ rowpart, float* __restrict__ bpart, int B, int R,
                       int C, int nblk, int nchunk, int with_w, long long ldg) {
  // ldg: row stride of g in elements (== C unless g is a column slice of a wider matrix;
  // strided gradients are only accepted for B == 1).
  // with_w: also accumulate sum(w^2) (only on the first step of a variable; later
  // steps get it for free from the previous apply kernel, see acc[2]).
  // Statistics are of the RAW gradient (no grad scale, no eps1): both are folded in by
  // the factors kernel, which lets this pass also produce the global sum(g^2) that the
  // clipping scale is computed from.
  __shared__ float rpart[kWarps][kStatRows];
  __shared__ float wpart[kWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int chunk = blockIdx.x % nchunk;
  const int blk = (blockIdx.x / nchunk) % nblk;
  const int b = blockIdx.x / (nchunk * nblk);
  const int c = chunk * kStatCols + warp * 256 + lane * 8;
  const bool cok = c < C;
  const int r0 = blk * kStatRows;
  const int nrows = min(kStatRows, R - r0);
  const size_t base = (static_cast<size_t>(b) * R + r0) * C + c;
  const size_t gbase = (static_cast<size_t>(b) * R + r0) * ldg + c;
  float cs[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  float wsq = 0.f;
#pragma unroll 2
  for (int r = 0; r < kStatRows; r += 4) {
    float gf[4][8];
    float rs[4] = {0.f, 0.f, 0.f, 0.f};
    if (cok && r + 4 <= nrows) {           // common case: no per-row predicates
#pragma unroll
      for (int u = 0; u < 4; ++u) load_g8<GT>(g + gbase + static_cast<size_t>(r + u) * ldg, gf[u]);
      if (with_w) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float wf[8];
          load_g8<float>(w + base + static_cast<size_t>(r + u) * C, wf);
#pragma unroll
          for (int i = 0; i < 8; ++i) wsq += wf[i] * wf[i];
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float q = gf[u][i] * gf[u][i];
          cs[i] += q;
          rs[u] += q;
        }
      }
    } else if (cok) {
      for (int u = 0; u < 4 && r + u < nrows; ++u) {
        float t[8];
        load_g8<GT>(g + gbase + static_cast<size_t>(r + u) * ldg, t);
        if (with_w) {
          float wf[8];
          load_g8<float>(w + base + static_cast<size_t>(r + u) * C, wf);
#pragma unroll
          for (int i = 0; i < 8; ++i) wsq += wf[i] * wf[i];
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float q = t[i] * t[i];
          cs[i] += q;
          rs[u] += q;
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) rs[u] = warp_sum(rs[u]);
    if (lane < 4)
      rpart[warp][r + lane] = lane == 0 ? rs[0] : lane == 1 ? rs[1] : lane == 2 ? rs[2] : rs[3];
  }
  if (cok) {
    float* cp = colpart + (static_cast<size_t>(b) * nblk + blk) * C + c;
    *reinterpret_cast<float4*>(cp) = make_float4(cs[0], cs[1], cs[2], cs[3]);
    *reinterpret_cast<float4*>(cp + 4) = make_float4(cs[4], cs[5], cs[6], cs[7]);
  }
  if (with_w) {
    wsq = warp_sum(wsq);
    if (lane == 0) wpart[warp] = wsq;
  }
  __syncthreads();
  if (warp == 0) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < kWarps; ++k) s += rpart[k][lane];
    if (lane < nrows) {
      const size_t ri = static_cast<size_t>(b) * R + r0 + lane;
      if (nchunk == 1) rowsum[ri] = s;
      else rowpart[static_cast<size_t>(chunk) * B * R + ri] = s;   // folded in chunk order
    } else {
      s = 0.f;
    }
    const float tg = warp_sum(s);
    if (lane == 0) {
      float tw = 0.f;
      if (with_w) {
#pragma unroll
        for (int k = 0; k < kWarps; ++k) tw += wpart[k];
      }
      bpart[2 * blockIdx.x] = tg;        // Σg², Σw² of this CTA, folded in CTA order
      bpart[2 * blockIdx.x + 1] = tw;
    }
  }
}

// colsum[b][c] = sum over row blocks of colpart[b][blk][c].
__global__ void __launch_bounds__(256)
adafactor_colreduce_kernel(const float* __restrict__ colpart, float* __restrict__ colsum, int C,
                           int nblk) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  const int b = blockIdx.y;
  if (c >= C) return;
  const float* p = colpart + static_cast<size_t>(b) * nblk * C + c;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  int k = 0;
  for (; k + 4 <= nblk; k += 4) {
    s0 += p[static_cast<size_t>(k) * C];
    s1 += p[static_cast<size_t>(k + 1) * C];
    s2 += p[static_cast<size_t>(k + 2) * C];
    s3 += p[static_cast<size_t>(k + 3) * C];
  }
  for (; k < nblk; ++k) s0 += p[static_cast<size_t>(k) * C];
  colsum[static_cast<size_t>(b) * C + c] = (s0 + s1) + (s2 + s3);
}

// vr_is_rows: vr has shape [B,R] (mean over C is "row mean" of the reference,
// i.e. the largest dim d0 is the last dim); otherwise vr is [B,C].
__global__ void adafactor_factors_kernel(float* __restrict__ vr, float* __restrict__ vc,
                                         const float* __restrict__ rowsum,
                                         const float* __restrict__ colsum, float* __restrict__ fr,
                                         float* __restrict__ fc, int B, int R, int C, float decay,
                                         int vr_is_rows, float* __restrict__ acc, int with_w,
                                         const float* __restrict__ gscale, float eps1,
                                         const float* __restrict__ hyper) {
  if (hyper != nullptr) decay = hyper[1];   // device-resident hyper-parameters (CUDA graphs)
  // One CTA per batch element b.
  __shared__ float red[32];
  const int b = blockIdx.x;
  const float gs = gscale ? *gscale : 1.f;
  const float gs2 = gs * gs;   // mean((g*gs)^2 + eps1) = gs^2 * mean(g^2) + eps1
  if (b == 0 && threadIdx.x == 0) {
    // acc[0] = sum(w^2) for this step: freshly computed (with_w) or carried over
    // from the previous step's apply kernel (acc[2]); acc[2] restarts at 0.
    if (!with_w) acc[0] = acc[2];
    acc[2] = 0.f;
  }
  const float mix = 1.f - decay;
  const int nvr = vr_is_rows ? R : C;
  const int nvc = vr_is_rows ? C : R;
  const float* sum_r = vr_is_rows ? rowsum + static_cast<size_t>(b) * R
                                  : colsum + static_cast<size_t>(b) * C;
  const float* sum_c = vr_is_rows ? colsum + static_cast<size_t>(b) * C
                                  : rowsum + static_cast<size_t>(b) * R;
  // mean over the reduced axis: rows were summed over C, cols over R.
  const float inv_r = vr_is_rows ? 1.f / C : 1.f / R;
  const float inv_c = vr_is_rows ? 1.f / R : 1.f / C;
  float* vrb = vr + static_cast<size_t>(b) * nvr;
  float* vcb = vc + static_cast<size_t>(b) * nvc;
  float local = 0.f;
  for (int i = threadIdx.x; i < nvr; i += blockDim.x) {
    // gs == 0 marks a skipped (non-finite) step: ignore the sums, they may hold NaN/Inf.
    const float nv = vrb[i] * decay + ((gs == 0.f ? 0.f : gs2 * sum_r[i] * inv_r) + eps1) * mix;
    vrb[i] = nv;
    local += nv;
  }
  local = warp_sum(local);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) red[0] = v / nvr;
  }
  __syncthreads();
  const float ltm = red[0];
  float* f_r = vr_is_rows ? fr + static_cast<size_t>(b) * R : fc + static_cast<size_t>(b) * C;
  float* f_c = vr_is_rows ? fc + static_cast<size_t>(b) * C : fr + static_cast<size_t>(b) * R;
  for (int i = threadIdx.x; i < nvr; i += blockDim.x) f_r[i] = rsqrtf(vrb[i] / ltm);
  for (int i = threadIdx.x; i < nvc; i += blockDim.x) {
    const float nv = vcb[i] * decay + ((gs == 0.f ? 0.f : gs2 * sum_c[i] * inv_c) + eps1) * mix;
    vcb[i] = nv;
    f_c[i] = rsqrtf(nv);
  }
}

template <typename GT>
__global__ void __launch_bounds__(kWarps * 32)
adafactor_rms_kernel(const GT* __restrict__ g, const float* __restrict__ fr,
                     const float* __restrict__ fc, float* __restrict__ wpart, int B, int R, int C,
                     int items, const float* __restrict__ gscale, long long ldg) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float gs = gscale ? *gscale : 1.f;
  float s = 0.f;
  for (int item = blockIdx.x * kWarps + warp; item < items; item += gridDim.x * kWarps) {
    const Tile t = get_tile(item, R, C);
    const int c = t.c0 + lane * 8;
    if (c >= C) continue;
    float cf[8];
    load_g8<float>(fc + static_cast<size_t>(t.b) * C + c, cf);
    const GT* gp = g + (static_cast<size_t>(t.b) * R) * ldg + c;
    const float* frp = fr + static_cast<size_t>(t.b) * R;
    int r = t.r0;
    for (; r + 4 <= t.r1; r += 4) {        // 4 rows in flight, no per-row predicates
      float gf[4][8], rf[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        load_g8<GT>(gp + static_cast<size_t>(r + u) * ldg, gf[u]);
        rf[u] = frp[r + u];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float x = (gs == 0.f ? 0.f : gf[u][i] * gs) * rf[u] * cf[i];
          s += x * x;
        }
      }
    }
    for (; r < t.r1; ++r) {
      float t8[8];
      load_g8<GT>(gp + static_cast<size_t>(r) * ldg, t8);
      const float rf = frp[r];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float x = (gs == 0.f ? 0.f : t8[i] * gs) * rf * cf[i];
        s += x * x;
      }
    }
  }
  s = warp_sum(s);
  if (lane == 0) wpart[blockIdx.x * kWarps + warp] = s;
}

template <typename GT>
__global__ void __launch_bounds__(kWarps * 32)
adafactor_apply_kernel(const GT* __restrict__ g, float* __restrict__ w,
                       __nv_bfloat16* __restrict__ w_bf16, const float* __restrict__ fr,
                       const float* __restrict__ fc, const float* __restrict__ acc,
                       float* __restrict__ wpart, int B, int R,
                       int C, float lr, float eps2, float clip, int mult_by_param_scale,
                       float numel, int items, const float* __restrict__ gscale,
                       const float* __restrict__ hyper, long long ldg) {
  if (hyper != nullptr) lr = hyper[0];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float gs = gscale ? *gscale : 1.f;
  float scale = lr;
  if (mult_by_param_scale) scale *= fmaxf(sqrtf(acc[0] / numel), eps2);
  if (clip > 0.f) scale /= fmaxf(1.f, sqrtf(acc[1] / numel) / clip);
  float wsq = 0.f;
  for (int item = blockIdx.x * kWarps + warp; item < items; item += gridDim.x * kWarps) {
    const Tile t = get_tile(item, R, C);
    const int c = t.c0 + lane * 8;
    if (c >= C) continue;
    float cf[8];
    load_g8<float>(fc + static_cast<size_t>(t.b) * C + c, cf);
    // 4 rows in flight: every load issues before the first store (w aliases itself, so
    // the compiler cannot hoist the next row's loads above this row's stores).
    const size_t tb = (static_cast<size_t>(t.b) * R) * C + c;
    const size_t gtb = (static_cast<size_t>(t.b) * R) * ldg + c;
    const float* frp = fr + static_cast<size_t>(t.b) * R;
    auto update_row = [&](size_t off, float (&gf)[8], float (&wf)[8], float rf) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        wf[i] -= (gs == 0.f ? 0.f : gf[i] * gs) * rf * cf[i];
        wsq += wf[i] * wf[i];
      }
      *reinterpret_cast<float4*>(w + off) = make_float4(wf[0], wf[1], wf[2], wf[3]);
      *reinterpret_cast<float4*>(w + off + 4) = make_float4(wf[4], wf[5], wf[6], wf[7]);
      if (w_bf16 != nullptr) {
        int4 o;
        o.x = pack_bf16x2(wf[0], wf[1]);
        o.y = pack_bf16x2(wf[2], wf[3]);
        o.z = pack_bf16x2(wf[4], wf[5]);
        o.w = pack_bf16x2(wf[6], wf[7]);
        *reinterpret_cast<int4*>(w_bf16 + off) = o;
      }
    };
    int r = t.r0;
    for (; r + 4 <= t.r1; r += 4) {
      float gf[4][8], wf[4][8], rf[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const size_t off = tb + static_cast<size_t>(r + u) * C;
        load_g8<GT>(g + gtb + static_cast<size_t>(r + u) * ldg, gf[u]);
        load_g8<float>(w + off, wf[u]);
        rf[u] = frp[r + u] * scale;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) update_row(tb + static_cast<size_t>(r + u) * C, gf[u], wf[u], rf[u]);
    }
    for (; r < t.r1; ++r) {
      const size_t off = tb + static_cast<size_t>(r) * C;
      float gf[8], wf[8];
      load_g8<GT>(g + gtb + static_cast<size_t>(r) * ldg, gf);
      load_g8<float>(w + off, wf);
      update_row(off, gf, wf, frp[r] * scale);
    }
  }
  wsq = warp_sum(wsq);                       // sum(w_new^2): next step's parameter scale
  if (lane == 0) wpart[blockIdx.x * kWarps + warp] = wsq;
}

template <typename GT>
__global__ void adam_flat_kernel(float* __restrict__ w, const GT* __restrict__ g,
                                 float* __restrict__ m, float* __restrict__ v,
                                 __nv_bfloat16* __restrict__ w_bf16,
                                 const float* __restrict__ grad_scale_ptr, float lr_t, float b1,
                                 float b2, float eps, float grad_scale, long long n) {
  const float gs = grad_scale_ptr ? grad_scale * (*grad_scale_ptr) : grad_scale;
  long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 8;
  for (; i + 8 <= n; i += stride) {
    float gf[8], wf[8], mf[8], vf[8];
    load_g8<GT>(g + i, gf);
    load_g8<float>(w + i, wf);
    load_g8<float>(m + i, mf);
    load_g8<float>(v + i, vf);
#pragma unroll
    for (int k = 0; k < 8; ++k) adam_update(wf[k], mf[k], vf[k], gf[k] * gs, lr_t, b1, b2, eps);
    *reinterpret_cast<float4*>(w + i) = make_float4(wf[0], wf[1], wf[2], wf[3]);
    *reinterpret_cast<float4*>(w + i + 4) = make_float4(wf[4], wf[5], wf[6], wf[7]);
    *reinterpret_cast<float4*>(m + i) = make_float4(mf[0], mf[1], mf[2], mf[3]);
    *reinterpret_cast<float4*>(m + i + 4) = make_float4(mf[4], mf[5], mf[6], mf[7]);
    *reinterpret_cast<float4*>(v + i) = make_float4(vf[0], vf[1], vf[2], vf[3]);
    *reinterpret_cast<float4*>(v + i + 4) = make_float4(vf[4], vf[5], vf[6], vf[7]);
    if (w_bf16) {
      int4 o;
      o.x = pack_bf16x2(wf[0], wf[1]);
      o.y = pack_bf16x2(wf[2], wf[3]);
      o.z = pack_bf16x2(wf[4], wf[5]);
      o.w = pack_bf16x2(wf[6], wf[7]);
      *reinterpret_cast<int4*>(w_bf16 + i) = o;
    }
  }
}

}  // namespace

namespace {

// ---- non-factored Adafactor for many small variables in ONE launch -------------------
// table[i] = {w (fp32), g, v (fp32), w_bf16 or 0, numel, g_is_bf16}; one CTA per variable.
//   v <- decay*v + (1-decay)*((g*gs)^2 + eps1);  x = g*gs*rsqrt(v)
//   x /= max(1, RMS(x)/clip);  w -= lr * max(RMS(w), eps2)[if param scale] * x
struct SmallVar {
  long long w, g, v, wb, numel, g_bf16;
};

__global__ void __launch_bounds__(256)
adafactor_small_kernel(const SmallVar* __restrict__ table, float lr, float decay, float eps1,
                       float eps2, float clip, int mult_by_param_scale,
                       const float* __restrict__ gscale, const float* __restrict__ hyper,
                       float* __restrict__ total_sumsq_unused) {
  __shared__ float red[2][8];
  const SmallVar sv = table[blockIdx.x];
  float* w = reinterpret_cast<float*>(sv.w);
  float* v = reinterpret_cast<float*>(sv.v);
  __nv_bfloat16* wb = reinterpret_cast<__nv_bfloat16*>(sv.wb);
  const float* gf = reinterpret_cast<const float*>(sv.g);
  const __nv_bfloat16* gb = reinterpret_cast<const __nv_bfloat16*>(sv.g);
  const long long n = sv.numel;
  if (hyper != nullptr) {
    lr = hyper[0];
    decay = hyper[1];
  }
  const float gs = gscale ? *gscale : 1.f;
  const float mix = 1.f - decay;
  float wsq = 0.f, xsq = 0.f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const float g = gs == 0.f ? 0.f : (sv.g_bf16 ? __bfloat162float(gb[i]) : gf[i]) * gs;
    const float nv = v[i] * decay + (g * g + eps1) * mix;
    v[i] = nv;
    const float x = g * rsqrtf(nv);
    xsq += x * x;
    const float wi = w[i];
    wsq += wi * wi;
  }
  wsq = warp_sum(wsq);
  xsq = warp_sum(xsq);
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = wsq;
    red[1][threadIdx.x >> 5] = xsq;
  }
  __syncthreads();
  float tw = 0.f, tx = 0.f;
  for (int k = 0; k < 8; ++k) {
    tw += red[0][k];
    tx += red[1][k];
  }
  float scale = lr;
  if (mult_by_param_scale) scale *= fmaxf(sqrtf(tw / static_cast<float>(n)), eps2);
  if (clip > 0.f) scale /= fmaxf(1.f, sqrtf(tx / static_cast<float>(n)) / clip);
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const float g = gs == 0.f ? 0.f : (sv.g_bf16 ? __bfloat162float(gb[i]) : gf[i]) * gs;
    const float nw = w[i] - scale * g * rsqrtf(v[i]);
    w[i] = nw;
    if (wb != nullptr) wb[i] = __float2bfloat16(nw);
  }
}

// Σg² and Σw² over every variable of a SmallVar table: one CTA per variable, two adds.
__global__ void __launch_bounds__(256)
small_sumsq_kernel(const SmallVar* __restrict__ table, float* __restrict__ bpart) {
  __shared__ float red[2][8];
  const SmallVar sv = table[blockIdx.x];
  const float* w = reinterpret_cast<const float*>(sv.w);
  const float* gf = reinterpret_cast<const float*>(sv.g);
  const __nv_bfloat16* gb = reinterpret_cast<const __nv_bfloat16*>(sv.g);
  float gs = 0.f, ws = 0.f;
  for (long long i = threadIdx.x; i < sv.numel; i += blockDim.x) {
    const float g = sv.g_bf16 ? __bfloat162float(gb[i]) : gf[i];
    const float wi = w[i];
    gs += g * g;
    ws += wi * wi;
  }
  gs = warp_sum(gs);
  ws = warp_sum(ws);
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = gs;
    red[1][threadIdx.x >> 5] = ws;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float tg = 0.f, tw = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      tg += red[0][k];
      tw += red[1][k];
    }
    bpart[2 * blockIdx.x] = tg;
    bpart[2 * blockIdx.x + 1] = tw;
  }
}

// dst[0] += Σ_i part[i * stride] in a fixed order (one CTA): the per-CTA / per-warp partial
// sums above are combined here instead of by atomics, so every step sums in the same order.
__global__ void __launch_bounds__(256)
ordered_sum_kernel(const float* __restrict__ part, int count, int stride, float* __restrict__ dst) {
  __shared__ float red[256];
  float s = 0.f;
  for (int i = threadIdx.x; i < count; i += 256) s += part[static_cast<size_t>(i) * stride];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if (threadIdx.x < off) red[threadIdx.x] += red[threadIdx.x + off];
    __syncthreads();
  }
  if (threadIdx.x == 0) dst[0] += red[0];
}

// dst[x] = Σ_c part[c * n + x], c in order.
__global__ void __launch_bounds__(256)
chunk_sum_kernel(const float* __restrict__ part, int nchunk, long long n, float* __restrict__ dst) {
  const long long x = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (x >= n) return;
  float s = 0.f;
  for (int c = 0; c < nchunk; ++c) s += part[c * n + x];
  dst[x] = s;
}

static void OrderedSum(const float* part, int count, int stride, float* dst, cudaStream_t stream) {
  ordered_sum_kernel<<<1, 256, 0, stream>>>(part, count, stride, dst);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
}

struct AfLayout {
  float *acc, *rowsum, *colsum, *fr, *fc;
  int64_t br4, bc4;
  int items, grid;
};

// Row stride (elements) of a gradient viewed as [B, R, C]: contiguous, or — for B == 1 — a
// column slice of a wider row-major matrix (e.g. one third of a fused qkv weight gradient)
// whose rows stay 16-byte aligned.
int64_t GradRowStride(const torch::Tensor& g, const torch::Tensor& w, int64_t B, int64_t R,
                      int64_t C) {
  TORCH_CHECK(g.numel() == w.numel(), "adafactor: gradient / variable size mismatch");
  if (g.is_contiguous()) return C;
  TORCH_CHECK(B == 1 && g.dim() >= 2 && g.size(-1) == C && g.size(-2) == R && g.stride(-1) == 1,
              "adafactor: gradient must be contiguous or a column slice of a 2-D matrix");
  const int64_t ld = g.stride(-2);
  const int64_t es = g.element_size();
  TORCH_CHECK(ld >= C && (ld * es) % 16 == 0 &&
              reinterpret_cast<uintptr_t>(g.data_ptr()) % 16 == 0,
              "adafactor: strided gradient rows must be 16-byte aligned");
  return ld;
}

AfLayout Layout(const torch::Tensor& w, torch::Tensor& scratch, int64_t B, int64_t R, int64_t C) {
  TORCH_CHECK(w.is_cuda() && w.scalar_type() == torch::kFloat32 && w.is_contiguous());
  TORCH_CHECK(C % 8 == 0, "adafactor: C must be a multiple of 8");
  TORCH_CHECK(w.numel() == B * R * C);
  AfLayout l;
  l.br4 = (B * R + 3) / 4 * 4;
  l.bc4 = (B * C + 3) / 4 * 4;
  TORCH_CHECK(scratch.numel() >= 4 + 2 * l.br4 + 2 * l.bc4);
  TORCH_CHECK(reinterpret_cast<uintptr_t>(scratch.data_ptr()) % 16 == 0);
  float* sp = scratch.data_ptr<float>();
  l.acc = sp;
  l.rowsum = sp + 4;
  l.colsum = l.rowsum + l.br4;
  l.fr = l.colsum + l.bc4;
  l.fc = l.fr + l.br4;
  const int strips = static_cast<int>((C + 255) / 256);
  const int ranges = static_cast<int>((R + kRowsPerWarp - 1) / kRowsPerWarp);
  l.items = static_cast<int>(B) * strips * ranges;
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  l.grid = (l.items + kWarps - 1) / kWarps;
  if (l.grid > sms * 8) l.grid = sms * 8;
  return l;
}

// Staging buffer for the per-row-block column partials, one per (device, stream): the stats
// kernel of a variable and its fold run back to back on one stream, and the optimizer spreads
// variables over a few streams so that small tensors overlap. Grows on demand; warm-up steps
// size it before any CUDA-graph capture.
float* ColPartials(const c10::Device& dev, cudaStream_t stream, int64_t slot, int64_t floats) {
  // slot 0: the caller's own stream (whatever it is — warm-up and capture streams differ);
  // slot k > 0: the optimizer's k-th side stream.
  using Key = std::pair<int, int64_t>;
  static auto* bufs = new std::map<Key, torch::Tensor>();   // leaked: outlives the CUDA context
  static auto* mu = new std::mutex();
  std::lock_guard<std::mutex> lock(*mu);
  auto& t = (*bufs)[Key(dev.index() < 0 ? 0 : dev.index(), slot)];
  if (!t.defined() || t.numel() < floats) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(stream, &st);
    TORCH_CHECK(st == cudaStreamCaptureStatusNone,
                "adafactor_stats: staging buffer would grow during graph capture; run one "
                "eager step first");
    t = torch::empty({floats}, torch::TensorOptions().dtype(torch::kFloat32).device(dev));
  }
  return t.data_ptr<float>();
}

}  // namespace

// Phase A of the factored Adafactor step on `w` viewed as [B, R, C]: row/column sums of
// g^2 into `scratch`, optionally sum(w^2) (first step only) and the global sum(g^2).
// scratch: fp32 [4 + B*R*2 + B*C*2] = acc | rowsum | colsum | fr | fc.
//   acc[0] = sum(w^2) used now, acc[1] = clipping RMS, acc[2] = sum(w^2) carried to the
//   next step (persistent; on a fresh scratch this pass fills it), acc[3] unused.
void adafactor_stats(const torch::Tensor& w, const torch::Tensor& g, torch::Tensor scratch,
                     int64_t B, int64_t R, int64_t C, bool mult_by_param_scale,
                     bool recompute_wsq, const c10::optional<torch::Tensor>& total_sumsq,
                     int64_t slot) {
  const int64_t ldg = GradRowStride(g, w, B, R, C);
  const c10::cuda::CUDAGuard guard(w.device());
  auto stream = at::cuda::getCurrentCUDAStream();
  AfLayout l = Layout(w, scratch, B, R, C);
  if (recompute_wsq) C10_CUDA_CHECK(cudaMemsetAsync(l.acc, 0, sizeof(float) * 4, stream));
  else C10_CUDA_CHECK(cudaMemsetAsync(l.acc + 1, 0, sizeof(float), stream));
  // A fresh scratch has no carried Σw² yet: compute it here (also without the parameter
  // scale, which does not need it) so that acc[2] holds Σw² of the current weights between
  // this pass and the update, as it does on every later step (the learner's var_norm reads it).
  const int with_w = recompute_wsq ? 1 : 0;
  float* tot = (total_sumsq.has_value() && total_sumsq->defined())
                   ? total_sumsq->data_ptr<float>() : nullptr;
  const int nblk = static_cast<int>((R + kStatRows - 1) / kStatRows);
  const int nchunk = static_cast<int>((C + kStatCols - 1) / kStatCols);
  float* colpart = ColPartials(w.device(), stream.stream(), slot, B * nblk * C);
  const int grid = static_cast<int>(B) * nblk * nchunk;
  auto fopt = w.options().dtype(torch::kFloat32);
  auto bpart = torch::empty({grid, 2}, fopt);
  torch::Tensor rowpart;
  if (nchunk > 1) rowpart = torch::empty({nchunk, B * R}, fopt);
  auto run = [&](auto tag) {
    using GT = decltype(tag);
    adafactor_stats_kernel<GT><<<grid, kWarps * 32, 0, stream>>>(
        reinterpret_cast<const GT*>(g.data_ptr()), w.data_ptr<float>(), l.rowsum, colpart,
        rowpart.defined() ? rowpart.data_ptr<float>() : nullptr, bpart.data_ptr<float>(),
        (int)B, (int)R, (int)C, nblk, nchunk, with_w, (long long)ldg);
  };
  if (g.scalar_type() == torch::kBFloat16) run(__nv_bfloat16());
  else { TORCH_CHECK(g.scalar_type() == torch::kFloat32); run(float()); }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  if (nchunk > 1) {
    chunk_sum_kernel<<<static_cast<int>((B * R + 255) / 256), 256, 0, stream>>>(
        rowpart.data_ptr<float>(), nchunk, B * R, l.rowsum);
    C10_CUDA_KERNEL_LAUNCH_CHECK();
    CountLaunch();
  }
  if (tot != nullptr) OrderedSum(bpart.data_ptr<float>(), grid, 2, tot, stream);
  if (with_w) {
    OrderedSum(bpart.data_ptr<float>() + 1, grid, 2, l.acc, stream);
    C10_CUDA_CHECK(cudaMemcpyAsync(l.acc + 2, l.acc, sizeof(float), cudaMemcpyDeviceToDevice,
                                   stream));
  }
  adafactor_colreduce_kernel<<<dim3(static_cast<unsigned>((C + 255) / 256),
                                    static_cast<unsigned>(B)), 256, 0, stream>>>(
      colpart, l.colsum, (int)C, nblk);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch(2);
}

// Phase B: factors (folding grad_scale^2 and eps1 into the raw sums) -> clip RMS -> apply.
void adafactor_update(torch::Tensor w, const torch::Tensor& g, torch::Tensor vr, torch::Tensor vc,
                      torch::Tensor scratch, const c10::optional<torch::Tensor>& w_bf16,
                      int64_t B, int64_t R, int64_t C, bool vr_is_rows, double lr, double decay,
                      double eps1, double eps2, double clip, bool mult_by_param_scale,
                      const c10::optional<torch::Tensor>& grad_scale, bool recompute_wsq,
                      const c10::optional<torch::Tensor>& hyper) {
  const int64_t ldg = GradRowStride(g, w, B, R, C);
  const c10::cuda::CUDAGuard guard(w.device());
  auto stream = at::cuda::getCurrentCUDAStream();
  AfLayout l = Layout(w, scratch, B, R, C);
  const float* hp = (hyper.has_value() && hyper->defined()) ? hyper->data_ptr<float>() : nullptr;
  __nv_bfloat16* wb = nullptr;
  if (w_bf16.has_value() && w_bf16->defined()) {
    TORCH_CHECK(w_bf16->scalar_type() == torch::kBFloat16 && w_bf16->is_contiguous() &&
                w_bf16->numel() == w.numel());
    wb = reinterpret_cast<__nv_bfloat16*>(w_bf16->data_ptr());
  }
  const float numel = static_cast<float>(w.numel());
  const float* gsp = (grad_scale.has_value() && grad_scale->defined())
                         ? grad_scale->data_ptr<float>() : nullptr;
  adafactor_factors_kernel<<<static_cast<int>(B), 256, 0, stream>>>(
      vr.data_ptr<float>(), vc.data_ptr<float>(), l.rowsum, l.colsum, l.fr, l.fc, (int)B, (int)R,
      (int)C, (float)decay, vr_is_rows ? 1 : 0, l.acc,
      (recompute_wsq || !mult_by_param_scale) ? 1 : 0, gsp, (float)eps1, hp);
  auto wpart = torch::empty({2, l.grid * kWarps}, w.options().dtype(torch::kFloat32));
  float* wp_rms = wpart.data_ptr<float>();
  float* wp_apply = wp_rms + l.grid * kWarps;
  auto run = [&](auto tag) {
    using GT = decltype(tag);
    const GT* gp = reinterpret_cast<const GT*>(g.data_ptr());
    if (clip > 0) {
      adafactor_rms_kernel<GT><<<l.grid, kWarps * 32, 0, stream>>>(
          gp, l.fr, l.fc, wp_rms, (int)B, (int)R, (int)C, l.items, gsp, (long long)ldg);
      OrderedSum(wp_rms, l.grid * kWarps, 1, l.acc + 1, stream);
    }
    adafactor_apply_kernel<GT><<<l.grid, kWarps * 32, 0, stream>>>(
        gp, w.data_ptr<float>(), wb, l.fr, l.fc, l.acc, wp_apply, (int)B, (int)R, (int)C,
        (float)lr, (float)eps2, (float)clip, mult_by_param_scale ? 1 : 0, numel, l.items, gsp, hp,
        (long long)ldg);
    OrderedSum(wp_apply, l.grid * kWarps, 1, l.acc + 2, stream);
  };
  if (g.scalar_type() == torch::kBFloat16) run(__nv_bfloat16());
  else { TORCH_CHECK(g.scalar_type() == torch::kFloat32); run(float()); }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch(clip > 0 ? 3 : 2);
}

// table: int64 [n_vars, 6] device tensor of SmallVar records.
void adafactor_small(const torch::Tensor& table, double lr, double decay, double eps1, double eps2,
                     double clip, bool mult_by_param_scale,
                     const c10::optional<torch::Tensor>& grad_scale,
                     const c10::optional<torch::Tensor>& hyper) {
  TORCH_CHECK(table.is_cuda() && table.scalar_type() == torch::kInt64 && table.is_contiguous() &&
              table.dim() == 2 && table.size(1) == 6);
  const int n = static_cast<int>(table.size(0));
  if (n == 0) return;
  const c10::cuda::CUDAGuard guard(table.device());
  const float* gsp = (grad_scale.has_value() && grad_scale->defined())
                         ? grad_scale->data_ptr<float>() : nullptr;
  const float* hp = (hyper.has_value() && hyper->defined()) ? hyper->data_ptr<float>() : nullptr;
  adafactor_small_kernel<<<n, 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const SmallVar*>(table.data_ptr<int64_t>()), (float)lr, (float)decay,
      (float)eps1, (float)eps2, (float)clip, mult_by_param_scale ? 1 : 0, gsp, hp, nullptr);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
}

// out[0] += Σg², out[1] += Σw² over the table's variables.
void small_sumsq(const torch::Tensor& table, torch::Tensor out) {
  TORCH_CHECK(table.is_cuda() && table.scalar_type() == torch::kInt64 && table.is_contiguous() &&
              table.dim() == 2 && table.size(1) == 6);
  TORCH_CHECK(out.is_cuda() && out.scalar_type() == torch::kFloat32 && out.numel() >= 2);
  const int n = static_cast<int>(table.size(0));
  if (n == 0) return;
  const c10::cuda::CUDAGuard guard(table.device());
  auto stream = at::cuda::getCurrentCUDAStream();
  auto bpart = torch::empty({n, 2}, out.options());
  small_sumsq_kernel<<<n, 256, 0, stream>>>(
      reinterpret_cast<const SmallVar*>(table.data_ptr<int64_t>()), bpart.data_ptr<float>());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  OrderedSum(bpart.data_ptr<float>(), n, 2, out.data_ptr<float>(), stream);
  OrderedSum(bpart.data_ptr<float>() + 1, n, 2, out.data_ptr<float>() + 1, stream);
  CountLaunch();
}

void adam_flat(torch::Tensor w, const torch::Tensor& g, torch::Tensor m, torch::Tensor v,
               const c10::optional<torch::Tensor>& w_bf16,
               const c10::optional<torch::Tensor>& grad_scale_t, double lr_t, double b1, double b2,
               double eps, double grad_scale) {
  TORCH_CHECK(w.is_cuda() && w.scalar_type() == torch::kFloat32 && w.is_contiguous());
  const long long n = w.numel();
  TORCH_CHECK(n % 8 == 0, "adam_flat: numel must be a multiple of 8 (pad the flat buffer)");
  const c10::cuda::CUDAGuard guard(w.device());
  auto stream = at::cuda::getCurrentCUDAStream();
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  long long blocks = (n / 8 + 255) / 256;
  if (blocks > sms * 8) blocks = sms * 8;
  if (blocks < 1) blocks = 1;
  __nv_bfloat16* wb = (w_bf16.has_value() && w_bf16->defined())
                          ? reinterpret_cast<__nv_bfloat16*>(w_bf16->data_ptr()) : nullptr;
  const float* gsp = (grad_scale_t.has_value() && grad_scale_t->defined())
                         ? grad_scale_t->data_ptr<float>() : nullptr;
  if (g.scalar_type() == torch::kBFloat16)
    adam_flat_kernel<__nv_bfloat16><<<(int)blocks, 256, 0, stream>>>(
        w.data_ptr<float>(), reinterpret_cast<const __nv_bfloat16*>(g.data_ptr()),
        m.data_ptr<float>(), v.data_ptr<float>(), wb, gsp, (float)lr_t, (float)b1, (float)b2,
        (float)eps, (float)grad_scale, n);
  else
    adam_flat_kernel<float><<<(int)blocks, 256, 0, stream>>>(
        w.data_ptr<float>(), g.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(), wb,
        gsp, (float)lr_t, (float)b1, (float)b2, (float)eps, (float)grad_scale, n);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
}

}  // namespace lb

LB_REGISTER(optim) {
  m.def("adafactor_stats", &lb::adafactor_stats);
  m.def("adafactor_update", &lb::adafactor_update);
  m.def("adafactor_small", &lb::adafactor_small);
  m.def("small_sumsq", &lb::small_sumsq);
  m.def("adam_flat", &lb::adam_flat);
}
