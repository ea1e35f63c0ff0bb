// Per-slot segment bookkeeping of the rollout (the step itself is in csrc/spo_forward.cu).
//
// Reference: safepo/single_agent/ppo_lag.py:187-234 (segment / bootstrap rule).
#include "spo_common.cuh"

namespace {

struct TransArgs {
  spo_rollout r;
  int t, epoch_end;
  const float *reward, *cost;
  const uint8_t *term, *trunc;
  const float *next_v_r, *next_v_c, *final_v_r, *final_v_c;
};

__global__ void spo_store_transition_kernel(const TransArgs a) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= a.r.num_envs) return;
  const int64_t slot = static_cast<int64_t>(n) * a.r.steps + a.t;
  a.r.reward[slot] = a.reward[n];
  a.r.cost[slot] = a.cost[n];
  const bool term = a.term[n] != 0, trunc = a.trunc[n] != 0;
  const bool end = a.epoch_end || term || trunc;
  float br = 0.f, bc = 0.f;
  if (end && !term) {
    if (a.epoch_end) { br = a.next_v_r[n]; bc = a.next_v_c[n]; }
    if (trunc && a.final_v_r) { br = a.final_v_r[n]; bc = a.final_v_c[n]; }   // overrides, ppo_lag.py:209-213
  }
  a.r.seg_end[slot] = end ? 1 : 0;
  a.r.boot_r[slot] = br;
  a.r.boot_c[slot] = bc;
}

}  // namespace

extern "C" {

int spo_store_transition(const spo_rollout* r, int t, const float* reward, const float* cost,
                         const uint8_t* terminated, const uint8_t* truncated, int epoch_end,
                         const float* next_v_r, const float* next_v_c,
                         const float* final_v_r, const float* final_v_c, void* stream) {
  SPO_REQUIRE(r && reward && cost && terminated && truncated, SPO_ERR_INVALID_ARG, "spo_store_transition: null argument");
  SPO_REQUIRE(t >= 0 && t < r->steps, SPO_ERR_INVALID_ARG, "spo_store_transition: slot t=%d outside [0,%d)", t, r->steps);
  SPO_REQUIRE(!epoch_end || (next_v_r && next_v_c), SPO_ERR_INVALID_ARG, "spo_store_transition: epoch_end needs next_v_*");
  SPO_REQUIRE((final_v_r == nullptr) == (final_v_c == nullptr), SPO_ERR_INVALID_ARG, "spo_store_transition: final_v_r/final_v_c must both be set or both NULL");
  TransArgs a{*r, t, epoch_end, reward, cost, terminated, truncated, next_v_r, next_v_c, final_v_r, final_v_c};
  const int threads = 128;
  spo_store_transition_kernel<<<(r->num_envs + threads - 1) / threads, threads, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

}  // extern "C"
