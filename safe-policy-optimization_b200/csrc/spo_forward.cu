// Forward entry points of the single-agent nets: the rollout step (ActorVCritic.step fused with buffer.store), the
// bootstrap critic values, and the full-batch actor passes (old-distribution means, the KL early-stop test).
//
// References: safepo/common/model.py:149-170 (step), safepo/common/buffer.py:84-95 (store),
// safepo/single_agent/ppo_lag.py:206,211 (bootstrap values), :277 (old_distribution = policy.actor(obs)),
// :338-348 (KL(old||new).sum(-1).mean(), break if > target_kl); cpo.py:489-491 (.mean()).
//
// Each call runs one kernel, chosen by shape: the TMA + wgmma kernel of csrc/spo_tc_forward.cu where it applies
// (spo_tc_forward_applies, and act_dim <= 8), else the FFMA tile kernel of csrc/spo_ffma_forward.cuh.  KL sums are reduced in
// fp64 and folded into the device control block by the last CTA (no host round trip: the next pass's update kernel reads
// ctrl->stop itself).
#include "spo_ffma_forward.cuh"

namespace {

__global__ void spo_kl_finalize_kernel(spo_update_ctrl* ctrl, double denom, float target_kl) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (ctrl->stop) { ctrl->kl_sum = 0.0; return; }
  spo_close_kl_pass(ctrl, ctrl->kl_sum, denom, target_kl);
}

int forward_launch(const SpoFwdArgs& a, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUtensorMap map;
  // act_dim > 8 always takes the FFMA kernel (AC = 16): the wgmma kernel's output stage holds 8 columns
  if (a.A > SPO_MAX_ACT) return spo_ffma_forward_launch_wide(a, st);
  if (spo_tc_forward_applies(a) && spo_tc_encode_obs_map(&map, a.obs, a.count, a.D)) return spo_tc_forward_launch(map, a, st);
  return ffma_forward_launch<8>(a, st);
}

SpoFwdArgs forward_args(SpoFwdMode mode, const spo_dims* d, const float* params, const float* obs, int64_t count) {
  SpoFwdArgs a{};
  a.mode = mode; a.params = params; a.obs = obs; a.count = count; a.D = d->obs_dim; a.A = d->act_dim;
  a.store.steps = 1;
  return a;
}

}  // namespace

extern "C" {

int spo_policy_step(const spo_dims* d, const float* params, const float* obs, const float* eps,
                    uint64_t seed, uint64_t offset, int deterministic, int n,
                    float* act, float* logp, float* v_r, float* v_c,
                    const spo_rollout* store, int t, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(params && obs && n > 0, SPO_ERR_INVALID_ARG, "spo_policy_step: null params/obs or n<=0");
  SpoFwdArgs a = forward_args(SpoFwdMode::kStep, d, params, obs, n);
  a.eps = eps; a.seed = seed; a.offset = offset; a.deterministic = deterministic;
  a.act = act; a.logp = logp; a.v_r = v_r; a.v_c = v_c;
  if (store) {
    SPO_REQUIRE(store->num_envs == n, SPO_ERR_INVALID_ARG, "spo_policy_step: store->num_envs=%d != n=%d", store->num_envs, n);
    SPO_REQUIRE(t >= 0 && t < store->steps, SPO_ERR_INVALID_ARG, "spo_policy_step: slot t=%d outside [0,%d) (buffer overflow)", t, store->steps);
    a.store = *store; a.has_store = 1; a.t = t;
  }
  return forward_launch(a, stream);
}

int spo_critic_values(const spo_dims* d, const float* params, const float* obs, int n,
                      float* v_r, float* v_c, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(params && obs && n > 0, SPO_ERR_INVALID_ARG, "spo_critic_values: null params/obs or n<=0");
  SpoFwdArgs a = forward_args(SpoFwdMode::kStep, d, params, obs, n);
  a.net_base = 1; a.deterministic = 1; a.v_r = v_r; a.v_c = v_c;
  return forward_launch(a, stream);
}

int spo_actor_forward(const spo_dims* d, const float* params, const float* obs, int64_t count,
                      float* mean_out, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(params && obs && mean_out && count > 0, SPO_ERR_INVALID_ARG, "spo_actor_forward: null pointer or count<=0");
  SpoFwdArgs a = forward_args(SpoFwdMode::kMeans, d, params, obs, count);
  a.mean_out = mean_out;
  return forward_launch(a, stream);
}

int spo_actor_kl(const spo_dims* d, const float* params, const float* obs, const float* old_mean,
                 const float* old_log_std, int64_t count, int reduce, float target_kl,
                 spo_update_ctrl* ctrl, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(params && obs && old_mean && old_log_std && ctrl && count > 0, SPO_ERR_INVALID_ARG, "spo_actor_kl: null pointer or count<=0");
  SPO_REQUIRE(reduce == 0 || reduce == 1, SPO_ERR_INVALID_ARG, "spo_actor_kl: reduce=%d", reduce);
  SpoFwdArgs a = forward_args(SpoFwdMode::kKlClose, d, params, obs, count);
  a.old_mean = old_mean; a.old_log_std = old_log_std; a.reduce = reduce; a.target_kl = target_kl; a.ctrl = ctrl;
  return forward_launch(a, stream);
}

int spo_actor_kl_accumulate(const spo_dims* d, const float* params, const float* obs, const float* old_mean,
                            const float* old_log_std, int64_t count, spo_update_ctrl* ctrl, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(params && obs && old_mean && old_log_std && ctrl && count > 0, SPO_ERR_INVALID_ARG, "spo_actor_kl_accumulate: null pointer or count<=0");
  SpoFwdArgs a = forward_args(SpoFwdMode::kKlAccumulate, d, params, obs, count);
  a.old_mean = old_mean; a.old_log_std = old_log_std; a.ctrl = ctrl;
  return forward_launch(a, stream);
}

int spo_kl_finalize(spo_update_ctrl* ctrl, double denom, float target_kl, void* stream) {
  SPO_REQUIRE(ctrl && denom > 0, SPO_ERR_INVALID_ARG, "spo_kl_finalize: null ctrl or denom<=0");
  spo_kl_finalize_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(ctrl, denom, target_kl);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

}  // extern "C"
