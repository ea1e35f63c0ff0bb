// Device math shared by the multi-agent kernels (spo_ma.cu, spo_ma_update.cu, spo_ma_ppo.cu, spo_ma_trust.cu).  Each formula
// is written once here, so the kernels that evaluate it agree bit for bit:
//   ma_sigmoid / ma_std       the DiagGaussian std of act.py (sigmoid(log_std / x) * y): spo_ma_head_kernel, both actor loss
//                             and finalize kernels, spo_ma_head_jvp_kernel, spo_ma_ratio_loss_kernel, the line-search evaluation
//   ma_gauss_logp             one dimension of Normal.log_prob: the head, both actor losses, the ratio surrogate, the line search
//   ma_gauss_entropy          one dimension of Normal.entropy: both actor finalize kernels
//   ma_row_dot                a warp's head dot product feat . W[o]: the head and both actor losses
//   ma_input_ln_stats         the input LayerNorm's row statistics: the forward, its tangent and ma_ln_in_bwd_kernel
//   ma_row_ln_stats           the output LayerNorm's row statistics: the forward's epilogue, ma_ln_elu_bwd_kernel and the tangent
//   ma_stage_w_chunk          the W chunk of the block's K loop: the forward and its tangent
// The backward and the tangent recompute the LayerNorm statistics from the saved input / `pre` with the forward's own code, so
// they differentiate at exactly the mean and rstd the forward normalised with.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>
#include "spo_common.cuh"

// Block geometry of the [Linear -> ELU -> LayerNorm] kernels: a CTA owns MA_ROWS rows x all H outputs, warp w rows 4w..4w+3,
// lane l columns 128 cb + 4 l .. + 3 of every 128-column block cb < HB = H / 128.
constexpr int MA_ROWS = 32;
constexpr int MA_KC = 16;          // K chunk staged in shared memory
constexpr int MA_THREADS = 256;
constexpr int MA_MAXH = 512;

// shared memory of a block kernel: the W chunk [MA_KC][H], the input chunk [MA_ROWS][MA_KC + 4], input statistics [MA_ROWS][2]
inline size_t ma_layer_smem(int H) { return sizeof(float) * (MA_KC * H + MA_ROWS * (MA_KC + 4) + 2 * MA_ROWS); }

// f(std::integral_constant<int, HB>) for HB = H / 128; the caller has checked that H is a multiple of 128 up to MA_MAXH
template <class F>
inline void ma_launch_hb(int H, F&& f) {
  switch (H / 128) {
    case 1: f(std::integral_constant<int, 1>{}); break;
    case 2: f(std::integral_constant<int, 2>{}); break;
    case 3: f(std::integral_constant<int, 3>{}); break;
    default: f(std::integral_constant<int, 4>{}); break;
  }
}

inline bool ma_aligned(const void* p, int bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

// huber_loss of safepo/utils/util.py:19-22 (one-sided: 0 for e < -d) and its derivative, with the reference's op order
__device__ __forceinline__ float huber_val(float e, float d) {
  const float ae = fabsf(e);
  const float qa = (ae <= d) ? 1.f : 0.f, lb = (e > d) ? 1.f : 0.f;
  return __fadd_rn(__fdiv_rn(__fmul_rn(qa, __fmul_rn(e, e)), 2.f), __fmul_rn(__fmul_rn(lb, d), __fsub_rn(ae, __fdiv_rn(d, 2.f))));
}
__device__ __forceinline__ float huber_grad(float e, float d) { return (fabsf(e) <= d) ? e : (e > d ? d : 0.f); }

// sigmoid(log_std / x) and std = sigmoid(log_std / x) * y (act.py:24-43), with torch's op order
__device__ __forceinline__ float ma_sigmoid(float log_std, float x_coef) { return __fdiv_rn(1.f, 1.f + expf(-__fdiv_rn(log_std, x_coef))); }
__device__ __forceinline__ float ma_std(float log_std, float x_coef, float y_coef) { return __fmul_rn(ma_sigmoid(log_std, x_coef), y_coef); }

// Normal.log_prob of one dimension: -diff^2 / (2 std^2) - log std - log sqrt(2 pi)   (log_std = logf(std))
__device__ __forceinline__ float ma_gauss_logp(float diff, float std, float log_std) {
  const float q = __fdiv_rn(-__fmul_rn(diff, diff), __fmul_rn(2.f, __fmul_rn(std, std)));
  return __fsub_rn(__fsub_rn(q, log_std), kLogSqrt2Pi);
}

// Normal.entropy of one dimension: 0.5 + log sqrt(2 pi) + log std   (log_std = logf(std))
__device__ __forceinline__ float ma_gauss_entropy(float log_std) { return 0.5f + kLogSqrt2Pi + log_std; }

// sum_k f[k] W_row[k] over k < H by one warp (lane-strided FMA, then a warp sum): the result is in every lane
__device__ __forceinline__ float ma_row_dot(const float* f, const float* W_row, int H, int lane) {
  float s = 0.f;
  for (int k = lane; k < H; k += 32) s = fmaf(f[k], __ldg(W_row + k), s);
  return spo_warp_sum(s);
}

// Input LayerNorm statistics of the 4 rows 4 wid .. 4 wid + 3 of the CTA's block at row0, in two passes like torch's layer_norm:
// stat[2 r] = mean, stat[2 r + 1] = rstd (r the row within the CTA); rows past n get the statistics of a zero sum.
__device__ __forceinline__ void ma_input_ln_stats(const float* in, int n, int K, int row0, int wid, int lane, float* stat) {
  for (int rr = 0; rr < 4; ++rr) {
    const int r = 4 * wid + rr, g = row0 + r;
    float s = 0.f;
    if (g < n)
      for (int k = lane; k < K; k += 32) s += in[static_cast<size_t>(g) * K + k];
    s = spo_warp_sum(s);
    const float mean = s / static_cast<float>(K);
    float v = 0.f;
    if (g < n)
      for (int k = lane; k < K; k += 32) { const float d = in[static_cast<size_t>(g) * K + k] - mean; v = fmaf(d, d, v); }
    v = spo_warp_sum(v);
    if (lane == 0) { stat[2 * r] = mean; stat[2 * r + 1] = rsqrtf(v / static_cast<float>(K) + 1e-5f); }
  }
}

// LayerNorm statistics of one row of H = 128 HB values held by a warp (lane l: v[4 cb + e] = column 128 cb + 4 l + e):
// a sequential sum over c, the mean as sum / H, a sequential fmaf of the squared deviations, rstd = rsqrt(var + 1e-5).
template <int HB>
__device__ __forceinline__ void ma_row_ln_stats(const float (&v)[4 * HB], float& mean, float& rstd) {
  constexpr int H = 128 * HB;
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < 4 * HB; ++c) s += v[c];
  s = spo_warp_sum(s);
  mean = s / static_cast<float>(H);
  float q = 0.f;
#pragma unroll
  for (int c = 0; c < 4 * HB; ++c) { const float d = v[c] - mean; q = fmaf(d, d, q); }
  q = spo_warp_sum(q);
  rstd = rsqrtf(q / static_cast<float>(H) + 1e-5f);
}

// W[h][k0 .. k0 + MA_KC) of all H rows into Wc[kk][h] (transposed: conflict-free float4 reads), zero past K.  Thread tid handles
// rows tid, tid + MA_THREADS, ...; float2 loads (K is even, rows 8-byte aligned).
template <int HB>
__device__ __forceinline__ void ma_stage_w_chunk(const float* W, int K, int k0, float* Wc, int tid) {
  constexpr int H = 128 * HB;
  for (int h = tid; h < H; h += MA_THREADS) {
    const float* wp = W + static_cast<size_t>(h) * K + k0;
#pragma unroll
    for (int kk = 0; kk < MA_KC; kk += 2) {
      float2 w2 = make_float2(0.f, 0.f);
      if (k0 + kk < K) w2 = __ldg(reinterpret_cast<const float2*>(wp + kk));
      Wc[kk * H + h] = w2.x;
      Wc[(kk + 1) * H + h] = w2.y;
    }
  }
}
