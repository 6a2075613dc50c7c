// One Adam update of one fp32 element, shared by adam_flat (optim_kernels.cu) and zero_adam
// (comm_kernels.cu) so the two give bit-identical weights and moments. The roundings are
// spelled out (no contraction left to the compiler):
//   m = fma(m, b1, (1 − b1)·gg),  v = fma(gg, (1 − b2)·gg, v·b2),  w −= (lr_t·m) / (√v + eps)
#pragma once

namespace lb {

__device__ __forceinline__ void adam_update(float& w, float& m, float& v, float gg, float lr_t,
                                            float b1, float b2, float eps) {
  m = fmaf(m, b1, __fmul_rn(1.f - b1, gg));
  v = fmaf(gg, __fmul_rn(1.f - b2, gg), __fmul_rn(v, b2));
  w = __fsub_rn(w, __fdiv_rn(__fmul_rn(lr_t, m), __fadd_rn(sqrtf(v), eps)));
}

}  // namespace lb
