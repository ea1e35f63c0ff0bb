// The single-agent forward family: one call description shared by the TMA + wgmma kernel
// (csrc/spo_tc_forward.cu) and the FFMA tile kernel (csrc/spo_forward.cu), and the per-row Gaussian
// math that both, the trust-region kernels and spo_kl_finalize evaluate.  The parity bars need these
// to agree bit for bit, so each piece is written once, in torch's operation order with unfused
// __f*_rn ops.
//
// References: safepo/common/model.py:149-170 (ActorVCritic.step), buffer.py:84-95 (store),
// safepo/single_agent/ppo_lag.py:277 and :338-348 (old distribution, KL early stop).
#pragma once
#include <cuda.h>
#include "spo_common.cuh"

enum class SpoFwdMode : int {
  kMeans,          // actor means over [count, D] -> mean_out
  kKlClose,        // KL(old || new) into ctrl->kl_sum; the last CTA closes the pass (final_kl, passes, stop)
  kKlAccumulate,   // KL(old || new) into ctrl->kl_sum only (data-parallel ranks close it with spo_kl_finalize)
  kStep,           // rollout step: sample / log-prob or critic values, optional write into slot t of the store
};

// One forward call.  CTA (blockIdx.x, blockIdx.y) walks row tiles blockIdx.x, blockIdx.x + gridDim.x, ...
// of net net_base + blockIdx.y (0 = actor, 1 = reward critic, 2 = cost critic).
struct SpoFwdArgs {
  SpoFwdMode mode;
  const float* params;
  const float* obs;            // [count, D]
  int64_t count;
  int D, A, net_base;
  float* mean_out;             // kMeans: [count, A]
  const float* old_mean;       // KL modes: [count, A]
  const float* old_log_std;    // KL modes: [A]
  int reduce;                  // kKlClose: 0 = mean over rows, 1 = mean over rows x A
  float target_kl;
  spo_update_ctrl* ctrl;
  const float* eps;            // kStep: [count, A] or null (in-kernel Philox)
  uint64_t seed, offset;
  int deterministic, has_store, t;
  float *act, *logp, *v_r, *v_c;
  spo_rollout store;           // store.steps == 1 without a store
};

__host__ __device__ inline bool spo_fwd_is_kl(SpoFwdMode m) { return m == SpoFwdMode::kKlClose || m == SpoFwdMode::kKlAccumulate; }

// One dimension of Normal.log_prob from d2 = (x - mean)^2 and var = std^2.
__device__ __forceinline__ float spo_normal_log_term(float d2, float var, float std) {
  return __fsub_rn(__fsub_rn(__fdiv_rn(-d2, __fmul_rn(2.f, var)), logf(std)), kLogSqrt2Pi);
}

// One dimension of _kl_normal_normal(p = old, q = new); ps, qs are the standard deviations.
__device__ __forceinline__ float spo_kl_term(float p_mean, float q_mean, float ps, float qs) {
  const float sr = __fdiv_rn(ps, qs);
  const float vr = __fmul_rn(sr, sr);
  const float dm = __fdiv_rn(__fsub_rn(p_mean, q_mean), qs);
  return __fmul_rn(0.5f, __fsub_rn(__fsub_rn(__fadd_rn(vr, __fmul_rn(dm, dm)), 1.f), logf(vr)));
}

// Rollout step, actor, row g: action = loc + eps * scale (host eps or Philox4x32-10 + Box-Muller), its
// log-density summed over dimensions, written to act / logp and to slot t of the store.
__device__ __forceinline__ void spo_step_actor_row(const SpoFwdArgs& a, int64_t g, const float* mu,
                                                   const float* log_std) {
  const int A = a.A, T = a.store.steps;
  float lp = 0.f;
  float* act_out = a.act ? a.act + g * A : nullptr;
  float* act_st = a.has_store ? a.store.act + (g * T + a.t) * A : nullptr;
  for (int j = 0; j < A; ++j) {
    const float std = expf(log_std[j]);
    float action = mu[j];
    if (!a.deterministic) {
      float e;
      if (a.eps) {
        e = __ldg(a.eps + g * A + j);
      } else {
        const uint4 rnd = spo_philox(make_uint4(static_cast<uint32_t>(g), static_cast<uint32_t>(j >> 1),
                                                static_cast<uint32_t>(a.offset), static_cast<uint32_t>(a.offset >> 32)),
                                     make_uint2(static_cast<uint32_t>(a.seed), static_cast<uint32_t>(a.seed >> 32)));
        const float2 z = spo_box_muller(rnd.x, rnd.y);
        e = (j & 1) ? z.y : z.x;
      }
      action = __fadd_rn(mu[j], __fmul_rn(e, std));
    }
    const float diff = __fsub_rn(action, mu[j]);
    const float term = spo_normal_log_term(__fmul_rn(diff, diff), __fmul_rn(std, std), std);
    lp = (j == 0) ? term : __fadd_rn(lp, term);
    if (act_out) act_out[j] = action;
    if (act_st) act_st[j] = action;
  }
  if (a.logp) a.logp[g] = lp;
  if (a.has_store) a.store.logp[g * T + a.t] = lp;
}

// Epilogue of row g of net `net` once its outputs mu[0..out) are known: the rollout step's sample or critic value, or
// (returned, KL modes) the row's KL(old || new) summed over dimensions.  log_std / old_log_std: [A].  The means mode
// writes its tile from each kernel's own layout (coalesced in the FFMA kernel, from registers in the wgmma one).  mu is a
// row of shared memory in both kernels, so the loops over A stay rolled: unrolled, the eight Philox instances of the
// sample would set the FFMA kernel's register count.
__device__ __forceinline__ float spo_forward_row(const SpoFwdArgs& a, int net, int64_t g, const float* mu,
                                                 const float* log_std, const float* old_log_std) {
  const int A = a.A;
  if (a.mode == SpoFwdMode::kStep) {
    if (net == 0) {
      spo_step_actor_row(a, g, mu, log_std);
    } else {
      float* vout = (net == 1) ? a.v_r : a.v_c;
      if (vout) vout[g] = mu[0];
      if (a.has_store) ((net == 1) ? a.store.value_r : a.store.value_c)[g * a.store.steps + a.t] = mu[0];
    }
  } else {
    float kl = 0.f;
    for (int j = 0; j < A; ++j) {
      const float klj = spo_kl_term(__ldg(a.old_mean + g * A + j), mu[j], expf(old_log_std[j]), expf(log_std[j]));
      kl = (j == 0) ? klj : __fadd_rn(kl, klj);
    }
    return kl;
  }
  return 0.f;
}

// Closes a KL pass on the control block: final_kl = total / denom, passes += 1, stop when above target, kl_sum reset.
__device__ __forceinline__ void spo_close_kl_pass(spo_update_ctrl* ctrl, double total, double denom, float target_kl) {
  const float kl = static_cast<float>(total / denom);
  ctrl->final_kl = kl;
  ctrl->passes += 1;
  if (kl > target_kl) ctrl->stop = 1;
  ctrl->kl_sum = 0.0;
}

// Thread 0 of every CTA of a KL pass adds its CTA's sum; in kKlClose the last CTA to arrive (ticket) closes the pass,
// so the next pass's update kernel reads ctrl->stop without a host round trip.
__device__ __forceinline__ void spo_kl_pass_add(const SpoFwdArgs& a, double cta_sum) {
  atomicAdd(&a.ctrl->kl_sum, cta_sum);
  if (a.mode != SpoFwdMode::kKlClose) return;
  __threadfence();
  if (atomicAdd(&a.ctrl->ticket, 1u) != gridDim.x - 1) return;
  __threadfence();
  const double total = *reinterpret_cast<volatile double*>(&a.ctrl->kl_sum);
  spo_close_kl_pass(a.ctrl, total, a.reduce == 0 ? static_cast<double>(a.count) : static_cast<double>(a.count) * a.A,
                    a.target_kl);
  a.ctrl->ticket = 0u;
}

// ---- launchers -------------------------------------------------------------------------------
// csrc/spo_tc_forward.cu.  The wgmma kernel needs obs_dim % 4 == 0 (16-byte TMA row pitch) and obs_dim <= 64 (K padded
// to 64), and at least 128 rows for the step and 1024 for the full-batch modes.  At obs_dim % 4 == 0 the entry points
// have already refused obs (and store->obs) that is not 16-byte aligned: both kernels read such rows as float4.
bool spo_tc_forward_applies(const SpoFwdArgs& a);
// false when cuTensorMapEncodeTiled is unavailable or rejects the observation tensor (the latter warned about once)
bool spo_tc_encode_obs_map(CUtensorMap* map, const float* obs, int64_t count, int D);
// grid: (ceil(count / 128), nets) for kStep, min(tiles, SMs) otherwise
int spo_tc_forward_launch(const CUtensorMap& map, const SpoFwdArgs& a, cudaStream_t stream);
