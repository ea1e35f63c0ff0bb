// Device helpers shared by the multi-agent loss heads (spo_ma_update.cu, spo_ma_ppo.cu).
#pragma once
#include <cuda_runtime.h>

// huber_loss of safepo/utils/util.py:19-22 (one-sided: 0 for e < -d) and its derivative, with the reference's op order
__device__ __forceinline__ float huber_val(float e, float d) {
  const float ae = fabsf(e);
  const float qa = (ae <= d) ? 1.f : 0.f, lb = (e > d) ? 1.f : 0.f;
  return __fadd_rn(__fdiv_rn(__fmul_rn(qa, __fmul_rn(e, e)), 2.f), __fmul_rn(__fmul_rn(lb, d), __fsub_rn(ae, __fdiv_rn(d, 2.f))));
}
__device__ __forceinline__ float huber_grad(float e, float d) { return (fabsf(e) <= d) ? e : (e > d ? d : 0.f); }
