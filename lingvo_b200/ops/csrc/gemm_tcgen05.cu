// Warp-specialised bf16 GEMM for sm_90a (Hopper).
//
//   C[g, m, n] = epilogue( sum_k A[g, m, k] * B[g, n, k] )        g in [0, G)
//
// * operands are staged by TMA (cp.async.bulk.tensor, 128B swizzle) into a
//   4-6 stage shared-memory ring;  either operand may be K-major ([.., MN, K]
//   storage) or MN-major ([.., K, MN] storage), so the same kernel serves the
//   forward (x @ w), dgrad (dy @ w^T) and wgrad (x^T @ dy) of every linear /
//   expert-FFN layer without any transposes in HBM (wgmma reads MN-major bf16
//   operands through its transpose bits);
// * two consumer warpgroups each own 64 rows of the 128 x BN tile and issue
//   wgmma.m64nBNk16 (fp32 accumulators in registers), keeping one k-block of
//   MMAs in flight while the next stage is awaited;
// * the fused epilogue (bias, activation, relu-gradient mask / residual add,
//   per-row scale, accumulate) runs on the accumulator registers and stores
//   straight to global memory.  The store target of every output row can be
//   redirected through a row-pointer table, which is how the MoE combine
//   (expert GEMM -> NVLink peer store) is fused.
//
// Grid: one CTA per output tile, 288 threads:
//   warps 0..7 = two consumer warpgroups, warp 8 = TMA producer.

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <mutex>
#include <unordered_map>

#include "ptx.cuh"
#include "registry.h"

namespace lb {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;   // 64 bf16 = 128 bytes = one swizzle row
constexpr int kMmaK = 16;
constexpr int kNumConsumers = 256;                 // two warpgroups x 64 rows
constexpr int kNumThreads = kNumConsumers + 32;    // + one TMA producer warp

enum Act : int { kActNone = 0, kActRelu = 1, kActGelu = 2, kActSilu = 3, kActGeluTanh = 4,
                 kActSquaredRelu = 5 };
enum AuxMode : int { kAuxNone = 0, kAuxReluMask = 1, kAuxAdd = 2 };

// A operand may be split along K over several tensor maps (one per NVLink peer):
// the TMA producer then *is* the all-gather (tiles are pulled straight from the
// owning rank's memory), SURVEY K5/K6 "all-gather -> GEMM".
constexpr int kMaxAMaps = 8;
struct TmapArray {
  CUtensorMap m[kMaxAMaps];
};

struct GemmParams {
  int G, M, N, K;
  void* c;                 // [G, M, N] out (bf16 or fp32)
  long long ldc;           // row stride of C (elements)
  long long c_batch;       // batch stride of C (elements)
  const float* bias;       // [G, N] fp32 or nullptr
  const __nv_bfloat16* aux;  // [G, M, N] bf16 (same strides as C) or nullptr
  void* pre_act;           // optional second output: pre-activation (bf16), same strides
  const float* row_scale;  // [G, M] or nullptr
  void* const* row_ptrs;   // [G * M] destination row pointers (peer memory) or nullptr
  void* const* nblk_ptrs;  // [tiles_n] destination base per N-tile (peer slab) or nullptr;
                           // element (row, col) goes to base[n_blk] + row*ldc + (col - n0)
  int a_k_per_map;         // K elements covered by each A tensor map (all-gather prologue)
  int act;
  int aux_mode;
  int accumulate;          // C += result (fp32 out only)
};

__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case kActRelu: return fmaxf(x, 0.f);
    case kActGelu: return 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
    case kActSilu: return x / (1.f + __expf(-x));
    case kActGeluTanh: {
      float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
      return 0.5f * x * (1.f + tanhf(u));
    }
    case kActSquaredRelu: { float r = fmaxf(x, 0.f); return r * r; }
    default: return x;
  }
}

struct EpiRow {
  void* c_row;
  long long row_off;
  const float* bias;
  float rscale;
};

// One pair of adjacent output columns (col, col + 1) of one row: bias / pre-act tap /
// activation / aux (ReLU-mask or residual add) / row scale / convert / store.
template <typename OutT>
__device__ __forceinline__ void epilogue_pair(const GemmParams& p, const EpiRow& er, float f0,
                                              float f1, int col) {
  if (er.bias != nullptr) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(er.bias + col));
    f0 += b.x; f1 += b.y;
  }
  if (p.pre_act != nullptr) {
    *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.pre_act) + er.row_off + col) =
        pack_bf16x2(f0, f1);
  }
  f0 = apply_act(f0, p.act);
  f1 = apply_act(f1, p.act);
  if (p.aux_mode != kAuxNone) {
    const float2 t = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.aux + er.row_off + col));
    if (p.aux_mode == kAuxReluMask) {
      f0 = t.x > 0.f ? f0 : 0.f;
      f1 = t.y > 0.f ? f1 : 0.f;
    } else {
      f0 += t.x;
      f1 += t.y;
    }
  }
  f0 *= er.rscale;
  f1 *= er.rscale;
  if constexpr (sizeof(OutT) == 2) {
    *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(er.c_row) + col) = pack_bf16x2(f0, f1);
  } else {
    float2* out = reinterpret_cast<float2*>(reinterpret_cast<float*>(er.c_row) + col);
    float2 o = make_float2(f0, f1);
    if (p.accumulate) {
      const float2 old = *out;
      o.x += old.x; o.y += old.y;
    }
    *out = o;
  }
}

template <int BN, bool kAK, bool kBK>
__device__ __forceinline__ void wgmma_bn(float (&acc)[BN / 2], uint64_t adesc, uint64_t bdesc) {
  if constexpr (BN == 256) wgmma_m64n256k16<kAK ? 0 : 1, kBK ? 0 : 1>(acc, adesc, bdesc, 1);
  else wgmma_m64n128k16<kAK ? 0 : 1, kBK ? 0 : 1>(acc, adesc, bdesc, 1);
}

template <int BN, bool kAK, bool kBK, typename OutT>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ TmapArray tmaps_a,
                  const __grid_constant__ CUtensorMap tmap_b, const GemmParams p) {
  constexpr int kStages = (BN == 256) ? 4 : 6;
  constexpr uint32_t kABytes = kBlockM * kBlockK * 2;   // 16 KiB
  constexpr uint32_t kBBytes = BN * kBlockK * 2;        // 32 KiB (BN=256)
  constexpr uint32_t kStageBytes = kABytes + kBBytes;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024B alignment for SWIZZLE_128B atoms.
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int tiles_m = (p.M + kBlockM - 1) / kBlockM;
  const int tiles_per_group = tiles_m * ((p.N + BN - 1) / BN);
  const int g = blockIdx.x / tiles_per_group;
  const int r = blockIdx.x - g * tiles_per_group;
  const int n_blk = r / tiles_m;
  const int m_blk = r - n_blk * tiles_m;
  const int m0 = m_blk * kBlockM, n0 = n_blk * BN;
  const int num_k_blocks = (p.K + kBlockK - 1) / kBlockK;

  if (threadIdx.x == kNumConsumers) {
    tma_prefetch_desc(&tmaps_a.m[0]);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(smem_u32(&full_bar[i]), 1);
      mbar_init(smem_u32(&empty_bar[i]), kNumConsumers / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp_idx == kNumConsumers / 32) {
    // ============================ TMA producer ============================
    if (lane == 0) {
      for (int kb = 0; kb < num_k_blocks; ++kb) {
        const int stage = kb % kStages;
        mbar_wait(smem_u32(&empty_bar[stage]), ((kb / kStages) & 1) ^ 1);
        const uint32_t fb = smem_u32(&full_bar[stage]);
        mbar_arrive_expect_tx(fb, kStageBytes);
        const uint32_t sa = smem_u32(smem + stage * kStageBytes);
        const uint32_t sb = sa + kABytes;
        const int k0 = kb * kBlockK;
        const int amap = k0 / p.a_k_per_map;
        const int ka = k0 - amap * p.a_k_per_map;
        if constexpr (kAK) {
          tma_load_3d(sa, &tmaps_a.m[amap], fb, ka, m0, g);
        } else {
#pragma unroll
          for (int i = 0; i < kBlockM / 64; ++i)
            tma_load_3d(sa + i * (64 * kBlockK * 2), &tmaps_a.m[amap], fb, m0 + 64 * i, ka, g);
        }
        if constexpr (kBK) {
          tma_load_3d(sb, &tmap_b, fb, k0, n0, g);
        } else {
#pragma unroll
          for (int i = 0; i < BN / 64; ++i)
            tma_load_3d(sb + i * (64 * kBlockK * 2), &tmap_b, fb, n0 + 64 * i, k0, g);
        }
      }
    }
    return;
  }

  // ============================== consumers ==============================
  // Warpgroup wg owns tile rows [64 wg, 64 wg + 64). Its A rows start 8 KiB into the
  // stage for both majors: 64 K-major rows of 128 B, or the wg-th 64-wide MN chunk.
  const int wg = warp_idx >> 2;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  for (int kb = 0; kb < num_k_blocks; ++kb) {
    const int stage = kb % kStages;
    mbar_wait(smem_u32(&full_bar[stage]), (kb / kStages) & 1);
    const uint32_t sa = smem_u32(smem + stage * kStageBytes) + wg * (64 * 128);
    const uint32_t sb = smem_u32(smem + stage * kStageBytes) + kABytes;
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < kBlockK / kMmaK; ++j) {
      // K-major: advance 32 B inside the 128 B swizzle row.
      // MN-major: advance 16 K-rows of 128 B; 64-wide MN chunks are
      //           64*kBlockK*2 bytes apart (LBO), 8-row groups 1 KiB (SBO).
      const uint64_t adesc =
          kAK ? make_smem_desc_sw128(sa + j * 32, 16, 1024)
              : make_smem_desc_sw128(sa + j * (kMmaK * 128), 64 * kBlockK * 2, 1024);
      const uint64_t bdesc =
          kBK ? make_smem_desc_sw128(sb + j * 32, 16, 1024)
              : make_smem_desc_sw128(sb + j * (kMmaK * 128), 64 * kBlockK * 2, 1024);
      wgmma_bn<BN, kAK, kBK>(acc, adesc, bdesc);
    }
    wgmma_commit();
    wgmma_wait<1>();                 // the previous k-block's MMAs have retired
    __syncwarp();
    if (kb > 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[(kb - 1) % kStages]));
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);

  // ============================== epilogue ==============================
  const int wrow = m0 + wg * 64 + (warp_idx & 3) * 16 + (lane >> 2);
  const int cq = (lane & 3) * 2;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = wrow + 8 * i;
    if (row >= p.M) continue;
    EpiRow er;
    er.row_off = static_cast<long long>(g) * p.c_batch + static_cast<long long>(row) * p.ldc;
    if (p.row_ptrs != nullptr) {
      er.c_row = p.row_ptrs[static_cast<long long>(g) * p.M + row];
    } else if (p.nblk_ptrs != nullptr) {
      er.c_row = reinterpret_cast<OutT*>(p.nblk_ptrs[n_blk]) + static_cast<long long>(row) * p.ldc - n0;
    } else {
      er.c_row = reinterpret_cast<OutT*>(p.c) + er.row_off;
    }
    if (er.c_row == nullptr) continue;
    er.rscale = p.row_scale != nullptr ? p.row_scale[static_cast<long long>(g) * p.M + row] : 1.f;
    er.bias = p.bias ? p.bias + static_cast<long long>(g) * p.N : nullptr;
#pragma unroll
    for (int n = 0; n < BN / 8; ++n) {
      const int col = n0 + n * 8 + cq;
      if (col < p.N) epilogue_pair<OutT>(p, er, acc[4 * n + 2 * i], acc[4 * n + 2 * i + 1], col);
    }
  }
}

// ------------------------------------------------------------------ host ----
CUtensorMap MakeMap(const void* base, int64_t inner, int64_t rows, int64_t groups,
                    int64_t row_stride, int64_t group_stride, int box_rows,
                    CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, int elem_bytes = 2);

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                              const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                              const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeFn GetEncodeFn() {
  static EncodeFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t err = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    TORCH_CHECK(err == cudaSuccess && ptr != nullptr, "cuTensorMapEncodeTiled not available");
    fn = reinterpret_cast<EncodeFn>(ptr);
  });
  return fn;
}

// 3-D bf16 map over a [G, rows, inner] view; box = [1, box_rows, 64], 128B swizzle.
CUtensorMap MakeMap(const void* base, int64_t inner, int64_t rows, int64_t groups,
                    int64_t row_stride, int64_t group_stride, int box_rows,
                    CUtensorMapDataType dt, int elem_bytes) {
  CUtensorMap m;
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(inner), static_cast<cuuint64_t>(rows),
                        static_cast<cuuint64_t>(groups)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(row_stride * elem_bytes),
                           static_cast<cuuint64_t>(group_stride * elem_bytes)};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(128 / elem_bytes), static_cast<cuuint32_t>(box_rows), 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = GetEncodeFn()(&m, dt, 3, const_cast<void*>(base), dims, strides, box, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  TORCH_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed: ", static_cast<int>(r),
              " inner=", inner, " rows=", rows, " groups=", groups, " row_stride=", row_stride,
              " group_stride=", group_stride);
  return m;
}

template <int BN, bool kAK, bool kBK, typename OutT>
static void Launch(const TmapArray& ta, const CUtensorMap& tb, const GemmParams& p,
                   cudaStream_t stream) {
  constexpr int kStages = (BN == 256) ? 4 : 6;
  constexpr size_t smem = kStages * (kBlockM * kBlockK * 2 + BN * kBlockK * 2) + 1024 + 256;
  auto kern = gemm_wgmma_kernel<BN, kAK, kBK, OutT>;
  static bool configured = false;
  if (!configured) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(smem)));
    configured = true;
  }
  const int tiles = p.G * ((p.M + kBlockM - 1) / kBlockM) * ((p.N + BN - 1) / BN);
  kern<<<tiles, kNumThreads, smem, stream>>>(ta, tb, p);
  CountLaunch();
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

template <int BN, typename OutT>
static void Dispatch(bool ak, bool bk, const TmapArray& ta, const CUtensorMap& tb,
                     const GemmParams& p, cudaStream_t s) {
  if (ak && bk) Launch<BN, true, true, OutT>(ta, tb, p, s);
  else if (ak && !bk) Launch<BN, true, false, OutT>(ta, tb, p, s);
  else if (!ak && bk) Launch<BN, false, true, OutT>(ta, tb, p, s);
  else Launch<BN, false, false, OutT>(ta, tb, p, s);
}

// Wave-quantisation heuristic switch, off by default: the 128-wide tile moves 1.33x more
// operand bytes per FLOP than the 256-wide one. LINGVO_B200_GEMM_AUTO_BN=1 turns it on.
static bool GemmAutoBn128() {
  static const bool on = [] {
    const char* e = getenv("LINGVO_B200_GEMM_AUTO_BN");
    return e != nullptr && atoi(e) != 0;
  }();
  return on;
}

// a: [G, M, K] if a_kmajor else [G, K, M];  b: [G, N, K] if b_kmajor else [G, K, N]
// (2-D inputs are treated as G = 1).  Returns / fills out [G, M, N].
torch::Tensor gemm_bf16(const torch::Tensor& a_in, const torch::Tensor& b_in, bool a_kmajor,
                        bool b_kmajor, const c10::optional<torch::Tensor>& bias,
                        int64_t act, const c10::optional<torch::Tensor>& aux, int64_t aux_mode,
                        const c10::optional<torch::Tensor>& row_scale,
                        const c10::optional<torch::Tensor>& out_opt, bool out_fp32,
                        bool accumulate, const c10::optional<torch::Tensor>& pre_act,
                        const c10::optional<torch::Tensor>& row_ptrs,
                        const c10::optional<torch::Tensor>& nblk_ptrs,
                        const c10::optional<torch::Tensor>& a_peer_ptrs, int64_t nblk_ld) {
  TORCH_CHECK(a_in.is_cuda() && b_in.is_cuda(), "gemm_bf16: CUDA tensors required");
  TORCH_CHECK(a_in.scalar_type() == torch::kBFloat16 && b_in.scalar_type() == torch::kBFloat16,
              "gemm_bf16: bf16 inputs required");
  const c10::cuda::CUDAGuard guard(a_in.device());
  // cuTensorMapEncodeTiled is a *driver* call: make sure this thread (e.g. an
  // autograd worker that has not issued a runtime call yet) has the primary
  // context bound, otherwise it fails with CUDA_ERROR_INVALID_CONTEXT.
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
  torch::Tensor a = a_in.dim() == 2 ? a_in.unsqueeze(0) : a_in;
  torch::Tensor b = b_in.dim() == 2 ? b_in.unsqueeze(0) : b_in;
  TORCH_CHECK(a.dim() == 3 && b.dim() == 3, "gemm_bf16: 2-D or 3-D operands");
  if (a.stride(2) != 1) a = a.contiguous();
  if (b.stride(2) != 1) b = b.contiguous();
  const int64_t G = a.size(0);
  TORCH_CHECK(b.size(0) == G, "gemm_bf16: group mismatch");
  const int64_t M = a_kmajor ? a.size(1) : a.size(2);
  const int64_t K = a_kmajor ? a.size(2) : a.size(1);
  const int64_t N = b_kmajor ? b.size(1) : b.size(2);
  const int64_t Kb = b_kmajor ? b.size(2) : b.size(1);
  const bool ag_prologue = a_peer_ptrs.has_value() && a_peer_ptrs->defined();
  TORCH_CHECK(ag_prologue || K == Kb, "gemm_bf16: K mismatch ", K, " vs ", Kb);
  TORCH_CHECK(N % 8 == 0, "gemm_bf16: N must be a multiple of 8");
  auto check_op = [](const torch::Tensor& t) {
    TORCH_CHECK(t.stride(1) % 8 == 0 && (t.size(0) == 1 || t.stride(0) % 8 == 0) &&
                    reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0,
                "gemm_bf16: operand rows must be 16-byte aligned");
  };
  check_op(a);
  check_op(b);

  torch::Tensor out;
  if (out_opt.has_value()) {
    out = out_opt.value();
    TORCH_CHECK(out.stride(-1) == 1, "gemm_bf16: out must be row-contiguous");
  } else {
    out = torch::empty({G, M, N}, a.options().dtype(out_fp32 ? torch::kFloat32 : torch::kBFloat16));
  }
  const bool fp32 = out.scalar_type() == torch::kFloat32;
  TORCH_CHECK(fp32 || out.scalar_type() == torch::kBFloat16, "gemm_bf16: out dtype");
  torch::Tensor out3 = out.dim() == 2 ? out.unsqueeze(0) : out;
  TORCH_CHECK(out3.size(0) == G && out3.size(1) == M && out3.size(2) == N, "gemm_bf16: out shape");

  GemmParams p;
  p.G = static_cast<int>(G); p.M = static_cast<int>(M); p.N = static_cast<int>(N);
  p.K = static_cast<int>(K);
  p.c = out3.data_ptr();
  p.ldc = out3.stride(1);
  p.c_batch = G > 1 ? out3.stride(0) : 0;
  p.bias = nullptr; p.aux = nullptr; p.row_scale = nullptr; p.pre_act = nullptr;
  p.row_ptrs = nullptr;
  p.nblk_ptrs = nullptr;
  p.a_k_per_map = static_cast<int>(K);
  torch::Tensor bias_f;
  if (bias.has_value() && bias->defined()) {
    bias_f = bias->to(torch::kFloat32).contiguous();
    TORCH_CHECK(bias_f.numel() == G * N, "gemm_bf16: bias must be [G, N]");
    p.bias = bias_f.data_ptr<float>();
  }
  if (aux.has_value() && aux->defined() && aux_mode != 0) {
    torch::Tensor ax = aux.value();
    ax = ax.dim() == 2 ? ax.unsqueeze(0) : ax;
    TORCH_CHECK(ax.scalar_type() == torch::kBFloat16 && ax.stride(1) == p.ldc &&
                    (G == 1 || ax.stride(0) == p.c_batch) && ax.stride(2) == 1,
                "gemm_bf16: aux must be bf16 with the same strides as out");
    p.aux = reinterpret_cast<const __nv_bfloat16*>(ax.data_ptr());
  }
  if (pre_act.has_value() && pre_act->defined()) {
    torch::Tensor pa = pre_act.value();
    pa = pa.dim() == 2 ? pa.unsqueeze(0) : pa;
    TORCH_CHECK(pa.scalar_type() == torch::kBFloat16 && pa.stride(1) == p.ldc &&
                    (G == 1 || pa.stride(0) == p.c_batch), "gemm_bf16: pre_act strides");
    p.pre_act = pa.data_ptr();
  }
  torch::Tensor rs_f;
  if (row_scale.has_value() && row_scale->defined()) {
    rs_f = row_scale->to(torch::kFloat32).contiguous();
    TORCH_CHECK(rs_f.numel() == G * M, "gemm_bf16: row_scale must be [G, M]");
    p.row_scale = rs_f.data_ptr<float>();
  }
  if (row_ptrs.has_value() && row_ptrs->defined()) {
    TORCH_CHECK(row_ptrs->scalar_type() == torch::kInt64 && row_ptrs->numel() == G * M &&
                    row_ptrs->is_contiguous(), "gemm_bf16: row_ptrs must be int64 [G, M]");
    p.row_ptrs = reinterpret_cast<void* const*>(row_ptrs->data_ptr());
  }
  if (nblk_ptrs.has_value() && nblk_ptrs->defined()) {
    TORCH_CHECK(nblk_ptrs->scalar_type() == torch::kInt64 && nblk_ptrs->is_cuda() &&
                    nblk_ptrs->is_contiguous(), "gemm_bf16: nblk_ptrs must be CUDA int64");
    TORCH_CHECK(G == 1, "gemm_bf16: nblk_ptrs needs G == 1");
    TORCH_CHECK(!fp32 && N > 128 && nblk_ld > 0 && nblk_ld % 8 == 0 &&
                    nblk_ptrs->numel() == (N + 255) / 256,
                "gemm_bf16: nblk_ptrs needs bf16 out, one pointer per 256-column tile and nblk_ld");
    p.nblk_ptrs = reinterpret_cast<void* const*>(nblk_ptrs->data_ptr());
    p.ldc = nblk_ld;
    TORCH_CHECK(p.aux == nullptr && p.pre_act == nullptr, "gemm_bf16: nblk_ptrs excludes aux/pre_act");
  }
  p.act = static_cast<int>(act);
  p.aux_mode = p.aux ? static_cast<int>(aux_mode) : 0;
  p.accumulate = accumulate ? 1 : 0;
  TORCH_CHECK(!accumulate || fp32, "gemm_bf16: accumulate needs fp32 out");

  if (M == 0 || N == 0 || G == 0) return out;

  // Tile-N: 256 unless N is small — or unless 128-wide tiles quantise better onto the SMs:
  // an [8192, 2048] output is 512 tiles of 128×256 = 3.88 waves on 132 SMs (4 are paid for),
  // but 1024 tiles of 128×128 = 7.76 half-cost waves. LINGVO_B200_GEMM_BN=128|256 forces one.
  bool bn256 = N > 128;
  if (bn256) {
    static const int forced = [] {
      const char* e = getenv("LINGVO_B200_GEMM_BN");
      return e ? atoi(e) : 0;
    }();
    const int sms_q = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
    const int64_t mt = (M + kBlockM - 1) / kBlockM;
    const int64_t t256 = G * mt * ((N + 255) / 256), t128 = G * mt * ((N + 127) / 128);
    const int64_t w256 = 2 * ((t256 + sms_q - 1) / sms_q), w128 = (t128 + sms_q - 1) / sms_q;
    if (forced == 128) bn256 = false;
    else if (forced == 0 && GemmAutoBn128() && w128 * 100 <= w256 * 90) bn256 = false;
  }
  const int bn = bn256 ? 256 : 128;
  TmapArray ta;
  if (a_peer_ptrs.has_value() && a_peer_ptrs->defined()) {
    // `a` is the local K-shard [M, K/W] (K-major); peers hold the other shards at
    // the given base pointers with identical strides.
    TORCH_CHECK(a_kmajor && G == 1, "all-gather prologue needs a K-major 2-D A");
    TORCH_CHECK(a_peer_ptrs->device().is_cpu() && a_peer_ptrs->scalar_type() == torch::kInt64);
    const int W = static_cast<int>(a_peer_ptrs->numel());
    TORCH_CHECK(W <= kMaxAMaps);
    const int64_t k_shard = a.size(2);
    TORCH_CHECK(k_shard % kBlockK == 0, "K shard must be a multiple of 64");
    TORCH_CHECK(Kb == k_shard * W, "B's K must equal W * shard K");
    p.K = static_cast<int>(k_shard * W);
    p.a_k_per_map = static_cast<int>(k_shard);
    for (int r = 0; r < W; ++r)
      ta.m[r] = MakeMap(reinterpret_cast<void*>(a_peer_ptrs->data_ptr<int64_t>()[r]), k_shard, M,
                        1, a.stride(1), a.stride(1) * a.size(1), kBlockM);
  } else {
    ta.m[0] = a_kmajor
        ? MakeMap(a.data_ptr(), K, M, G, a.stride(1), G > 1 ? a.stride(0) : a.stride(1) * a.size(1), kBlockM)
        : MakeMap(a.data_ptr(), M, K, G, a.stride(1), G > 1 ? a.stride(0) : a.stride(1) * a.size(1), kBlockK);
  }
  CUtensorMap tb = b_kmajor
      ? MakeMap(b.data_ptr(), Kb, N, G, b.stride(1), G > 1 ? b.stride(0) : b.stride(1) * b.size(1), bn)
      : MakeMap(b.data_ptr(), N, Kb, G, b.stride(1), G > 1 ? b.stride(0) : b.stride(1) * b.size(1), kBlockK);

  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  if (bn256) {
    if (fp32) Dispatch<256, float>(a_kmajor, b_kmajor, ta, tb, p, stream);
    else Dispatch<256, __nv_bfloat16>(a_kmajor, b_kmajor, ta, tb, p, stream);
  } else {
    if (fp32) Dispatch<128, float>(a_kmajor, b_kmajor, ta, tb, p, stream);
    else Dispatch<128, __nv_bfloat16>(a_kmajor, b_kmajor, ta, tb, p, stream);
  }
  return out;
}

}  // namespace lb
