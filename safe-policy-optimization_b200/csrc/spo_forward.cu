// Forward entry points of the single-agent nets: the rollout step (ActorVCritic.step fused with buffer.store), the
// bootstrap critic values, and the full-batch actor passes (old-distribution means, the KL early-stop test).
//
// References: safepo/common/model.py:149-170 (step), safepo/common/buffer.py:84-95 (store),
// safepo/single_agent/ppo_lag.py:206,211 (bootstrap values), :277 (old_distribution = policy.actor(obs)),
// :338-348 (KL(old||new).sum(-1).mean(), break if > target_kl); cpo.py:489-491 (.mean()).
//
// Each call runs one kernel, chosen by shape: the TMA + wgmma kernel of csrc/spo_tc_forward.cu where it applies
// (spo_tc_forward_applies), else the FFMA tile kernel below.  KL sums are reduced in fp64 and folded into the device
// control block by the last CTA (no host round trip: the next pass's update kernel reads ctrl->stop itself).
#include "spo_forward.cuh"

namespace {

// 64-row tiles, weights of net net_base + blockIdx.y resident in shared memory.  Grid (ceil(n/64), nets) for the step,
// persistent min(tiles, 2 x SMs) for the full-batch modes, which therefore needs two CTAs per SM (<= 128 registers;
// no minimum-blocks launch bound: with one, ptxas spends the whole 128 on the tile loop and the obs-27 passes slow down).
__global__ void __launch_bounds__(SPO_THREADS) spo_ffma_forward_kernel(const SpoFwdArgs a) {
  extern __shared__ __align__(16) float smem[];
  __shared__ double red[SPO_THREADS / 32];
  const int tid = threadIdx.x;
  if (spo_fwd_is_kl(a.mode) && *reinterpret_cast<volatile int*>(&a.ctrl->stop)) return;
  const int net = a.net_base + blockIdx.y;
  const int D = a.D, Dp = spo_pad4(D), ldx = spo_ld(D);
  const SpoNetOff off = spo_net_off(D, a.A, net);
  const int O = off.out;
  SpoNetSmem w;
  float* p = spo_carve_net(smem, D, O, false, w);
  float* x = p;  p += SPO_ROWS * ldx;
  float* h1 = p; p += SPO_ROWS * SPO_LDH;
  float* h2 = p; p += SPO_ROWS * SPO_LDH;
  float* y = p;  // [64][8]

  spo_load_net(a.params, off, D, w, tid, SPO_THREADS);
  const int64_t n_tiles = (a.count + SPO_ROWS - 1) / SPO_ROWS;
  double acc = 0.0;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t row0 = tile * SPO_ROWS;
    const int rows = static_cast<int>(a.count - row0 < SPO_ROWS ? a.count - row0 : SPO_ROWS);
    __syncthreads();
    spo_load_rows(a.obs, D, ldx, nullptr, row0, rows, x, tid, SPO_THREADS);
    __syncthreads();
    spo_hidden_fwd(x, ldx, Dp, w.w1t, w.b1, h1, tid);
    __syncthreads();
    spo_hidden_fwd(h1, SPO_LDH, SPO_HID, w.w2t, w.b2, h2, tid);
    __syncthreads();
    spo_out_fwd(h2, w.w3, w.b3, O, y, SPO_MAX_ACT, tid, SPO_THREADS);
    __syncthreads();
    if (a.mode == SpoFwdMode::kMeans) {
      // all threads, coalesced: one thread per row would write A floats at a stride of A
      for (int i = tid; i < rows * O; i += SPO_THREADS) {
        const int r = i / O, j = i - r * O;
        a.mean_out[(row0 + r) * O + j] = y[r * SPO_MAX_ACT + j];
      }
    } else if (tid < rows) {
      acc += static_cast<double>(spo_forward_row(a, net, row0 + tid, y + tid * SPO_MAX_ACT, a.params + off.log_std, a.old_log_std));
    }
    if (a.mode == SpoFwdMode::kStep && net == 0 && a.has_store) {
      // observation rows into slot t (buffer.py:91-95), bit-exact from the shared tile
      const int T = a.store.steps;
      for (int i = tid; i < rows * D; i += SPO_THREADS) {
        const int r = i / D, c = i - r * D;
        a.store.obs[((row0 + r) * T + a.t) * D + c] = x[r * ldx + c];
      }
    }
  }
  if (!spo_fwd_is_kl(a.mode)) return;
  acc = spo_warp_sum(acc);
  if ((tid & 31) == 0) red[tid >> 5] = acc;
  __syncthreads();
  if (tid == 0) {
    double s = 0.0;
    for (int i = 0; i < SPO_THREADS / 32; ++i) s += red[i];
    spo_kl_pass_add(a, s);
  }
}

__global__ void spo_kl_finalize_kernel(spo_update_ctrl* ctrl, double denom, float target_kl) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (ctrl->stop) { ctrl->kl_sum = 0.0; return; }
  spo_close_kl_pass(ctrl, ctrl->kl_sum, denom, target_kl);
}

int ffma_forward_launch(const SpoFwdArgs& a, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    SPO_CUDA_TRY(cudaFuncSetAttribute(spo_ffma_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  const size_t smem = sizeof(float) * (spo_net_smem_floats(a.D, a.A, false) + SPO_ROWS * spo_ld(a.D) +
                                       2 * SPO_ROWS * SPO_LDH + SPO_ROWS * SPO_MAX_ACT);
  const int64_t n_tiles = (a.count + SPO_ROWS - 1) / SPO_ROWS;
  const dim3 grid = (a.mode == SpoFwdMode::kStep)
                        ? dim3(static_cast<unsigned>(n_tiles), a.net_base == 0 ? 3 : 2)
                        : dim3(static_cast<unsigned>(n_tiles < 2 * spo_sm_count() ? n_tiles : 2 * spo_sm_count()));   // 2 CTAs per SM
  spo_ffma_forward_kernel<<<grid, SPO_THREADS, smem, stream>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int forward_launch(const SpoFwdArgs& a, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUtensorMap map;
  if (spo_tc_forward_applies(a) && spo_tc_encode_obs_map(&map, a.obs, a.count, a.D)) return spo_tc_forward_launch(map, a, st);
  return ffma_forward_launch(a, st);
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
