// GShard MoE kernels: fused top-2 gate + dispatch over NVLink peer memory,
// gated combine, their backward counterparts, and the flag protocol.
//
// Layout conventions (shared with lingvo_b200/parallel/symm.py):
//   tokens on a rank          x   [G_l * S, M]            (G_l local groups)
//   expert buffer on owner    xe  [E_l, G_t * C, M]       row (e_l*G_t + g_glob)*C + c
//   combine buffer on source  yc  [E,   G_l * C, M]       row (e*G_l + g_loc)*C + c
// with E = ep * E_l experts, G_t = ep * G_l groups, rank r owning experts
// [r*E_l, (r+1)*E_l) and groups [r*G_l, (r+1)*G_l).
//
// moe_gate_dispatch (SURVEY K1+K2): one CTA-set per local group computes the
// top-2 gating of all S tokens of the group (softmax, argmax x2, exclusive
// position scan with first-choice priority, capacity), publishes (index, pos,
// keep) and then *every slot row* (e, g, c) of that group — token data or
// zeros — is stored straight into the owning rank's expert buffer through its
// peer pointer. No staging buffer, no all-to-all, no zero-fill pass.
//
// moe_scatter_rows: the same slot-major peer store for the backward pass
// (d_out = gate * dy routed back to the experts).
// moe_combine / moe_combine_bwd / moe_gather_rows: token-major local gathers.
// moe_sync: release/acquire flags at system scope replacing the collective's
// implicit barrier; the sequence number is a device counter, so it can be
// replayed from a CUDA graph.

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "ptx.cuh"
#include "registry.h"

namespace lb {
namespace {

constexpr int kGateThreads = 256;
constexpr int kMaxExperts = 32;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Copies one row of `m8` 16-byte vectors (warp-cooperative); src == nullptr
// writes zeros; `scale` != 1 rescales bf16 payload.
__device__ __forceinline__ void warp_copy_row(void* dst, const void* src, int m8, int lane,
                                              float scale) {
  int4* d = reinterpret_cast<int4*>(dst);
  if (src == nullptr) {
    const int4 z = make_int4(0, 0, 0, 0);
    for (int i = lane; i < m8; i += 32) st_na_v4(d + i, z);
    return;
  }
  const int4* s = reinterpret_cast<const int4*>(src);
  if (scale == 1.f) {
    for (int i = lane; i < m8; i += 32) st_na_v4(d + i, ld_nc_v4(s + i));
  } else {
    for (int i = lane; i < m8; i += 32) {
      int4 v = ld_nc_v4(s + i);
      uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 t = unpack_bf16x2(w[j]);
        w[j] = pack_bf16x2(t.x * scale, t.y * scale);
      }
      st_na_v4(d + i, make_int4(w[0], w[1], w[2], w[3]));
    }
  }
}

struct GateArgs {
  const float* logits;      // [G_l, S, E]
  const float* paddings;    // [G_l, S] or nullptr
  const __nv_bfloat16* x;   // [G_l * S, M]
  int* index;               // [2, G_l, S]
  int* pos;                 // [2, G_l, S]
  float* gate;              // [2, G_l, S]  (non-differentiable copy; 0 = dropped)
  int* slot_token;          // [E, G_l, C]  token id (within rank) or -1
  const long long* peer_xe; // [ep] base pointers of every rank's expert buffer
  int G_l, S, E, C, M, E_l, G_t, rank, ctas_per_group, legacy;
};

// smem: idx1/idx2 [S] uint8, g1/g2 [S] float, keep [2][S] uint8, pos [2][S] int,
//       slot map [E*C] int, scan scratch.
__global__ void __launch_bounds__(kGateThreads)
moe_gate_dispatch_kernel(const GateArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int S = a.S, E = a.E, C = a.C;
  float* g1 = reinterpret_cast<float*>(smem_raw);
  float* g2 = g1 + S;
  int* p1 = reinterpret_cast<int*>(g2 + S);
  int* p2 = p1 + S;
  int* slot_map = p2 + S;                          // [E*C]
  int* warp_tot = slot_map + E * C;                // [E][8]
  int* running = warp_tot + kMaxExperts * 8;       // [E]
  int* kept1 = running + kMaxExperts;              // [E]
  unsigned char* i1 = reinterpret_cast<unsigned char*>(kept1 + kMaxExperts);
  unsigned char* i2 = i1 + S;
  unsigned char* k1 = i2 + S;
  unsigned char* k2 = k1 + S;

  const int g = blockIdx.x / a.ctas_per_group;          // local group
  const int part = blockIdx.x % a.ctas_per_group;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* lg = a.logits + static_cast<size_t>(g) * S * E;
  const float* pad = a.paddings ? a.paddings + static_cast<size_t>(g) * S : nullptr;

  // ---- phase 1a: softmax + top-2 per token -------------------------------
  for (int t = tid; t < S; t += kGateThreads) {
    float v[kMaxExperts];
    float mx = -INFINITY;
    for (int e = 0; e < E; ++e) { v[e] = lg[static_cast<size_t>(t) * E + e]; mx = fmaxf(mx, v[e]); }
    float sum = 0.f;
    for (int e = 0; e < E; ++e) { v[e] = __expf(v[e] - mx); sum += v[e]; }
    const float inv = 1.f / sum;
    int b1 = 0;
    for (int e = 1; e < E; ++e) if (v[e] > v[b1]) b1 = e;
    const bool nonpad = pad == nullptr || pad[t] < 0.5f;
    int b2 = -1;
    if (nonpad) {
      for (int e = 0; e < E; ++e) if (e != b1 && (b2 < 0 || v[e] > v[b2])) b2 = e;
    } else {
      b2 = b1;   // reference: mask_1 == 0 for padding, so argmax repeats
    }
    i1[t] = static_cast<unsigned char>(b1);
    i2[t] = static_cast<unsigned char>(b2 < 0 ? 0 : b2);
    float a1 = nonpad ? v[b1] * inv : 0.f;
    float a2 = (nonpad && b2 >= 0) ? v[b2] * inv : 0.f;
    if (a.legacy) {
      const float den = a1 + a2 + 1e-9f;
      a1 /= den;
      a2 /= den;
    }
    g1[t] = a1;
    g2[t] = a2;
    k1[t] = nonpad ? 1 : 0;
    k2[t] = (nonpad && b2 >= 0) ? 1 : 0;
  }
  for (int i = tid; i < E * C; i += kGateThreads) slot_map[i] = -1;
  if (tid < kMaxExperts) { running[tid] = 0; kept1[tid] = 0; }
  __syncthreads();

  // ---- phase 1b: exclusive position scans (first choice, then second) -----
  for (int pass = 0; pass < 2; ++pass) {
    unsigned char* idx = pass == 0 ? i1 : i2;
    unsigned char* keep = pass == 0 ? k1 : k2;
    int* posv = pass == 0 ? p1 : p2;
    if (tid < kMaxExperts) running[tid] = pass == 0 ? 0 : kept1[tid];
    __syncthreads();
    for (int base = 0; base < S; base += kGateThreads) {
      const int t = base + tid;
      const bool active = t < S && keep[t];
      const int e_mine = active ? idx[t] : -1;
      int my_prefix = 0;
      for (int e = 0; e < E; ++e) {
        const unsigned m = __ballot_sync(0xffffffffu, e_mine == e);
        if (e_mine == e) my_prefix = __popc(m & ((1u << lane) - 1));
        if (lane == 0) warp_tot[e * 8 + warp] = __popc(m);
      }
      __syncthreads();
      if (active) {
        int off = running[e_mine];
        for (int w = 0; w < warp; ++w) off += warp_tot[e_mine * 8 + w];
        const int p = off + my_prefix;
        posv[t] = p < C ? p : 0;
        if (p >= C) keep[t] = 0;
      } else if (t < S) {
        posv[t] = 0;
      }
      __syncthreads();
      if (tid < E) {
        int tot = 0;
        for (int w = 0; w < 8; ++w) tot += warp_tot[tid * 8 + w];
        running[tid] += tot;
      }
      __syncthreads();
    }
    if (pass == 0 && tid < E) kept1[tid] = min(running[tid], C);
    __syncthreads();
  }

  // ---- phase 1c: final gates, slot map, outputs ---------------------------
  for (int t = tid; t < S; t += kGateThreads) {
    float a1 = k1[t] ? g1[t] : 0.f;
    float a2 = k2[t] ? g2[t] : 0.f;
    if (!a.legacy) {
      float den = a1 + a2;
      den = den > 0.f ? den : 1.f;
      a1 /= den;
      a2 /= den;
    }
    if (a1 != 0.f) slot_map[i1[t] * C + p1[t]] = t;
    if (a2 != 0.f) slot_map[i2[t] * C + p2[t]] = t;
    if (part == 0) {
      const size_t o = static_cast<size_t>(g) * S + t;
      const size_t o2 = static_cast<size_t>(a.G_l) * S + o;
      a.index[o] = i1[t];
      a.index[o2] = i2[t];
      a.pos[o] = p1[t];
      a.pos[o2] = p2[t];
      a.gate[o] = a1;
      a.gate[o2] = a2;
    }
  }
  __syncthreads();
  if (part == 0) {
    for (int i = tid; i < E * C; i += kGateThreads) {
      const int e = i / C, c = i - e * C;
      const int tk = slot_map[i];
      a.slot_token[(static_cast<size_t>(e) * a.G_l + g) * C + c] = tk < 0 ? -1 : g * S + tk;
    }
  }

  // ---- phase 2: slot-major peer stores ------------------------------------
  if (a.x == nullptr) return;
  const int m8 = a.M / 8;
  const size_t row_bytes = static_cast<size_t>(a.M) * 2;
  const int g_glob = a.rank * a.G_l + g;
  const int warps_per_group = a.ctas_per_group * (kGateThreads / 32);
  for (int s = part * (kGateThreads / 32) + warp; s < E * C; s += warps_per_group) {
    const int e = s / C, c = s - e * C;
    const int dest = e / a.E_l, e_l = e - dest * a.E_l;
    const size_t drow = (static_cast<size_t>(e_l) * a.G_t + g_glob) * C + c;
    char* dst = reinterpret_cast<char*>(a.peer_xe[dest]) + drow * row_bytes;
    const int tk = slot_map[s];
    const void* src = tk < 0 ? nullptr
                             : reinterpret_cast<const char*>(a.x) +
                                   (static_cast<size_t>(g) * S + tk) * row_bytes;
    warp_copy_row(dst, src, m8, lane, 1.f);
  }
}

// Slot-major scatter with per-token scale (backward of combine):
//   dst_peer[slot] = slot_token[slot] >= 0 ? scale[k?][token] * src[token] : 0
__global__ void moe_scatter_rows_kernel(const __nv_bfloat16* __restrict__ src,
                                        const int* __restrict__ slot_token,
                                        const int* __restrict__ index,   // [2, T]
                                        const float* __restrict__ gate,  // [2, T] or nullptr
                                        const long long* __restrict__ peer_dst, int E, int G_l,
                                        int C, int M, int E_l, int G_t, int rank, int T) {
  const int lane = threadIdx.x & 31;
  const int warp_g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int m8 = M / 8;
  const size_t row_bytes = static_cast<size_t>(M) * 2;
  const int slots = E * G_l * C;
  for (int s = warp_g; s < slots; s += nwarps) {
    const int e = s / (G_l * C);
    const int rem = s - e * (G_l * C);
    const int g = rem / C, c = rem - g * C;
    const int dest = e / E_l, e_l = e - dest * E_l;
    const size_t drow = (static_cast<size_t>(e_l) * G_t + rank * G_l + g) * C + c;
    char* dst = reinterpret_cast<char*>(peer_dst[dest]) + drow * row_bytes;
    const int tk = slot_token[s];
    if (tk < 0) {
      warp_copy_row(dst, nullptr, m8, lane, 1.f);
    } else {
      float sc = 1.f;
      if (gate != nullptr) {
        // Which of the token's two choices landed in this slot?
        const int k = (index[tk] == e) ? 0 : 1;
        sc = gate[static_cast<size_t>(k) * T + tk];
      }
      warp_copy_row(dst, reinterpret_cast<const char*>(src) + tk * row_bytes, m8, lane, sc);
    }
  }
}

// Token-major gated combine:  y[t] = sum_k gate[k,t] * yc[slot_k(t)].
__global__ void moe_combine_kernel(const __nv_bfloat16* __restrict__ yc,
                                   const int* __restrict__ index, const int* __restrict__ pos,
                                   const float* __restrict__ gate, __nv_bfloat16* __restrict__ y,
                                   int T, int S, int G_l, int C, int M) {
  const int lane = threadIdx.x & 31;
  const int warp_g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int t = warp_g; t < T; t += nwarps) {
    const int g = t / S;
    float gk[2];
    const __nv_bfloat16* rows[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      gk[k] = gate[static_cast<size_t>(k) * T + t];
      const size_t slot = (static_cast<size_t>(index[static_cast<size_t>(k) * T + t]) * G_l + g) * C +
                          pos[static_cast<size_t>(k) * T + t];
      rows[k] = yc + slot * M;
    }
    for (int c = lane * 8; c < M; c += 256) {
      float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        if (gk[k] != 0.f) {
          int4 v = *reinterpret_cast<const int4*>(rows[k] + c);
          const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float2 f = unpack_bf16x2(w[j]);
            acc[2 * j] += gk[k] * f.x;
            acc[2 * j + 1] += gk[k] * f.y;
          }
        }
      }
      int4 o;
      o.x = pack_bf16x2(acc[0], acc[1]);
      o.y = pack_bf16x2(acc[2], acc[3]);
      o.z = pack_bf16x2(acc[4], acc[5]);
      o.w = pack_bf16x2(acc[6], acc[7]);
      *reinterpret_cast<int4*>(y + static_cast<size_t>(t) * M + c) = o;
    }
  }
}

// d_gate[k,t] = <dy[t], yc[slot_k(t)]>   (0 for dropped choices)
__global__ void moe_combine_bwd_gate_kernel(const __nv_bfloat16* __restrict__ yc,
                                            const __nv_bfloat16* __restrict__ dy,
                                            const int* __restrict__ index,
                                            const int* __restrict__ pos,
                                            const float* __restrict__ gate,
                                            float* __restrict__ dgate, int T, int S, int G_l,
                                            int C, int M) {
  const int lane = threadIdx.x & 31;
  const int warp_g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int t = warp_g; t < T; t += nwarps) {
    const int g = t / S;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      float acc = 0.f;
      if (gate[static_cast<size_t>(k) * T + t] != 0.f) {
        const size_t slot = (static_cast<size_t>(index[static_cast<size_t>(k) * T + t]) * G_l + g) * C +
                            pos[static_cast<size_t>(k) * T + t];
        const __nv_bfloat16* r = yc + slot * M;
        const __nv_bfloat16* d = dy + static_cast<size_t>(t) * M;
        for (int c = lane * 8; c < M; c += 256) {
          int4 a = *reinterpret_cast<const int4*>(r + c);
          int4 b = *reinterpret_cast<const int4*>(d + c);
          const uint32_t wa[4] = {(uint32_t)a.x, (uint32_t)a.y, (uint32_t)a.z, (uint32_t)a.w};
          const uint32_t wb[4] = {(uint32_t)b.x, (uint32_t)b.y, (uint32_t)b.z, (uint32_t)b.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float2 fa = unpack_bf16x2(wa[j]), fb = unpack_bf16x2(wb[j]);
            acc += fa.x * fb.x + fa.y * fb.y;
          }
        }
      }
      acc = warp_sum(acc);
      if (lane == 0) dgate[static_cast<size_t>(k) * T + t] = acc;
    }
  }
}

// Token-major unweighted gather: dx[t] = sum_k keep_k * src[slot_k(t)].
__global__ void moe_gather_rows_kernel(const __nv_bfloat16* __restrict__ src,
                                       const int* __restrict__ index, const int* __restrict__ pos,
                                       const float* __restrict__ gate,
                                       __nv_bfloat16* __restrict__ out, int T, int S, int G_l,
                                       int C, int M) {
  const int lane = threadIdx.x & 31;
  const int warp_g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int t = warp_g; t < T; t += nwarps) {
    const int g = t / S;
    const __nv_bfloat16* rows[2] = {nullptr, nullptr};
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      if (gate[static_cast<size_t>(k) * T + t] != 0.f) {
        const size_t slot = (static_cast<size_t>(index[static_cast<size_t>(k) * T + t]) * G_l + g) * C +
                            pos[static_cast<size_t>(k) * T + t];
        rows[k] = src + slot * M;
      }
    }
    for (int c = lane * 8; c < M; c += 256) {
      float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        if (rows[k] != nullptr) {
          int4 v = *reinterpret_cast<const int4*>(rows[k] + c);
          const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float2 f = unpack_bf16x2(w[j]);
            acc[2 * j] += f.x;
            acc[2 * j + 1] += f.y;
          }
        }
      }
      int4 o;
      o.x = pack_bf16x2(acc[0], acc[1]);
      o.y = pack_bf16x2(acc[2], acc[3]);
      o.z = pack_bf16x2(acc[4], acc[5]);
      o.w = pack_bf16x2(acc[6], acc[7]);
      *reinterpret_cast<int4*>(out + static_cast<size_t>(t) * M + c) = o;
    }
  }
}

// One kernel = signal every peer (flags[channel][src_rank] <- seq, release at system
// scope), then wait for every peer. The sequence number lives in device memory
// (`counter[channel]`, bumped by the kernel), so the launch has no step-dependent argument
// and can be replayed from a CUDA graph.
__global__ void moe_sync_kernel(const long long* __restrict__ peer_flags,
                                const int* __restrict__ flags, int* __restrict__ counters,
                                int world, int rank, int channel) {
  __shared__ int seq_s;
  if (threadIdx.x == 0) seq_s = ++counters[channel];
  __syncthreads();
  const int seq = seq_s;
  const int r = threadIdx.x;
  if (r < world) {
    __threadfence_system();
    int* f = reinterpret_cast<int*>(peer_flags[r]) + channel * world + rank;
    st_release_sys(f, seq);
    const int* mine = flags + channel * world + r;
    while (ld_acquire_sys(mine) < seq) {
      __nanosleep(64);
    }
  }
  __syncthreads();
}

int GridWarps(int items, int warps_per_cta) {
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  int g = (items + warps_per_cta - 1) / warps_per_cta;
  return g < sms * 8 ? (g < 1 ? 1 : g) : sms * 8;
}

}  // namespace

// Returns (index[2,G,S], pos[2,G,S], gate[2,G,S], slot_token[E,G,C]).
std::vector<torch::Tensor> moe_gate_dispatch(const torch::Tensor& logits,
                                             const c10::optional<torch::Tensor>& paddings,
                                             const c10::optional<torch::Tensor>& x,
                                             const torch::Tensor& peer_xe, int64_t capacity,
                                             int64_t e_local, int64_t rank, int64_t ep,
                                             bool legacy) {
  TORCH_CHECK(logits.is_cuda() && logits.scalar_type() == torch::kFloat32 && logits.dim() == 3 &&
              logits.is_contiguous());
  const c10::cuda::CUDAGuard guard(logits.device());
  const int G = (int)logits.size(0), S = (int)logits.size(1), E = (int)logits.size(2);
  const int C = (int)capacity;
  TORCH_CHECK(E <= kMaxExperts, "at most 32 experts");
  auto i32 = logits.options().dtype(torch::kInt32);
  auto index = torch::empty({2, G, S}, i32), pos = torch::empty({2, G, S}, i32);
  auto gate = torch::empty({2, G, S}, logits.options());
  auto slot_token = torch::empty({E, G, C}, i32);
  GateArgs a;
  a.logits = logits.data_ptr<float>();
  torch::Tensor pad;
  a.paddings = nullptr;
  if (paddings.has_value() && paddings->defined()) {
    pad = paddings->to(torch::kFloat32).contiguous();
    a.paddings = pad.data_ptr<float>();
  }
  a.x = nullptr;
  a.M = 0;
  if (x.has_value() && x->defined()) {
    TORCH_CHECK(x->scalar_type() == torch::kBFloat16 && x->is_contiguous() && x->size(-1) % 8 == 0);
    a.x = reinterpret_cast<const __nv_bfloat16*>(x->data_ptr());
    a.M = (int)x->size(-1);
  }
  a.index = index.data_ptr<int>();
  a.pos = pos.data_ptr<int>();
  a.gate = gate.data_ptr<float>();
  a.slot_token = slot_token.data_ptr<int>();
  a.peer_xe = reinterpret_cast<long long*>(peer_xe.data_ptr<int64_t>());
  a.G_l = G; a.S = S; a.E = E; a.C = C; a.E_l = (int)e_local; a.G_t = (int)(ep * G);
  a.rank = (int)rank; a.legacy = legacy ? 1 : 0;
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  int cpg = a.x ? (sms * 2 + G - 1) / G : 1;
  if (cpg > (E * C + 7) / 8) cpg = (E * C + 7) / 8;
  if (cpg < 1) cpg = 1;
  a.ctas_per_group = cpg;
  const size_t smem = sizeof(float) * 2 * S + sizeof(int) * 2 * S + sizeof(int) * E * C +
                      sizeof(int) * (kMaxExperts * 8 + 2 * kMaxExperts) + 4 * S + 16;
  TORCH_CHECK(smem <= 200 * 1024, "group too large for the gate kernel: ", smem);
  if (smem > 48 * 1024)
    C10_CUDA_CHECK(cudaFuncSetAttribute(moe_gate_dispatch_kernel,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  moe_gate_dispatch_kernel<<<G * cpg, kGateThreads, smem, at::cuda::getCurrentCUDAStream()>>>(a);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return {index, pos, gate, slot_token};
}

void moe_scatter_rows(const torch::Tensor& src, const torch::Tensor& slot_token,
                      const torch::Tensor& index, const c10::optional<torch::Tensor>& gate,
                      const torch::Tensor& peer_dst, int64_t e_local, int64_t rank, int64_t ep) {
  const c10::cuda::CUDAGuard guard(src.device());
  const int E = (int)slot_token.size(0), G = (int)slot_token.size(1), C = (int)slot_token.size(2);
  const int M = (int)src.size(-1), T = (int)(src.numel() / M);
  TORCH_CHECK(src.scalar_type() == torch::kBFloat16 && src.is_contiguous() && M % 8 == 0);
  const float* gp = (gate.has_value() && gate->defined()) ? gate->data_ptr<float>() : nullptr;
  const int grid = GridWarps(E * G * C, 8);
  moe_scatter_rows_kernel<<<grid, 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const __nv_bfloat16*>(src.data_ptr()), slot_token.data_ptr<int>(),
      index.data_ptr<int>(), gp, reinterpret_cast<long long*>(peer_dst.data_ptr<int64_t>()), E, G, C, M, (int)e_local,
      (int)(ep * G), (int)rank, T);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
}

torch::Tensor moe_combine(const torch::Tensor& yc, const torch::Tensor& index,
                          const torch::Tensor& pos, const torch::Tensor& gate, int64_t S,
                          int64_t G_l, int64_t C) {
  const c10::cuda::CUDAGuard guard(yc.device());
  const int M = (int)yc.size(-1), T = (int)index.size(-1) * (int)index.size(-2);
  TORCH_CHECK(yc.scalar_type() == torch::kBFloat16 && yc.is_contiguous());
  auto y = torch::empty({T, M}, yc.options());
  moe_combine_kernel<<<GridWarps(T, 8), 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const __nv_bfloat16*>(yc.data_ptr()), index.data_ptr<int>(),
      pos.data_ptr<int>(), gate.data_ptr<float>(), reinterpret_cast<__nv_bfloat16*>(y.data_ptr()),
      T, (int)S, (int)G_l, (int)C, M);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return y;
}

torch::Tensor moe_combine_bwd_gate(const torch::Tensor& yc, const torch::Tensor& dy,
                                   const torch::Tensor& index, const torch::Tensor& pos,
                                   const torch::Tensor& gate, int64_t S, int64_t G_l, int64_t C) {
  const c10::cuda::CUDAGuard guard(yc.device());
  const int M = (int)yc.size(-1), T = (int)(dy.numel() / M);
  auto dgate = torch::empty({2, T}, gate.options());
  moe_combine_bwd_gate_kernel<<<GridWarps(T, 8), 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const __nv_bfloat16*>(yc.data_ptr()),
      reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr()), index.data_ptr<int>(),
      pos.data_ptr<int>(), gate.data_ptr<float>(), dgate.data_ptr<float>(), T, (int)S, (int)G_l,
      (int)C, M);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return dgate;
}

torch::Tensor moe_gather_rows(const torch::Tensor& src, const torch::Tensor& index,
                              const torch::Tensor& pos, const torch::Tensor& gate, int64_t S,
                              int64_t G_l, int64_t C) {
  const c10::cuda::CUDAGuard guard(src.device());
  const int M = (int)src.size(-1), T = (int)index.size(-1) * (int)index.size(-2);
  auto out = torch::empty({T, M}, src.options());
  moe_gather_rows_kernel<<<GridWarps(T, 8), 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const __nv_bfloat16*>(src.data_ptr()), index.data_ptr<int>(),
      pos.data_ptr<int>(), gate.data_ptr<float>(), reinterpret_cast<__nv_bfloat16*>(out.data_ptr()),
      T, (int)S, (int)G_l, (int)C, M);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
  return out;
}

void moe_sync(const torch::Tensor& peer_flags, const torch::Tensor& flags, torch::Tensor counters,
              int64_t world, int64_t rank, int64_t channel) {
  TORCH_CHECK(counters.is_cuda() && counters.scalar_type() == torch::kInt32);
  const c10::cuda::CUDAGuard guard(flags.device());
  moe_sync_kernel<<<1, 32, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const long long*>(peer_flags.data_ptr<int64_t>()), flags.data_ptr<int>(), counters.data_ptr<int>(), (int)world, (int)rank, (int)channel);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  CountLaunch();
}

// ---- symmetric memory (cudaMalloc + CUDA IPC) --------------------------------
torch::Tensor symm_alloc(int64_t nbytes, int64_t device) {
  const c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  void* p = nullptr;
  C10_CUDA_CHECK(cudaMalloc(&p, static_cast<size_t>(nbytes)));
  C10_CUDA_CHECK(cudaMemset(p, 0, static_cast<size_t>(nbytes)));
  auto opts = torch::TensorOptions().dtype(torch::kUInt8).device(torch::kCUDA, device);
  return torch::from_blob(p, {nbytes}, [](void* q) { cudaFree(q); }, opts);
}
pybind11::bytes symm_export(const torch::Tensor& buf) {
  cudaIpcMemHandle_t h;
  C10_CUDA_CHECK(cudaIpcGetMemHandle(&h, buf.data_ptr()));
  return pybind11::bytes(reinterpret_cast<const char*>(&h), sizeof(h));
}
int64_t symm_import(const std::string& handle, int64_t device) {
  const c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  TORCH_CHECK(handle.size() == sizeof(cudaIpcMemHandle_t));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle.data(), sizeof(h));
  void* p = nullptr;
  C10_CUDA_CHECK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  return reinterpret_cast<int64_t>(p);
}

}  // namespace lb

LB_REGISTER(moe) {
  m.def("moe_gate_dispatch", &lb::moe_gate_dispatch);
  m.def("moe_scatter_rows", &lb::moe_scatter_rows);
  m.def("moe_combine", &lb::moe_combine);
  m.def("moe_combine_bwd_gate", &lb::moe_combine_bwd_gate);
  m.def("moe_gather_rows", &lb::moe_gather_rows);
  m.def("moe_sync", &lb::moe_sync);
  m.def("symm_alloc", &lb::symm_alloc);
  m.def("symm_export", &lb::symm_export);
  m.def("symm_import", &lb::symm_import);
}
