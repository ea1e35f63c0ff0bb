// Full-batch actor passes: old-distribution means and the KL early-stop test.
//
// Reference: safepo/single_agent/ppo_lag.py:277 (old_distribution = policy.actor(obs)),
// :338-348 (KL(old||new).sum(-1).mean(), break if > target_kl); cpo.py:489-491 (.mean()).
//
// A persistent grid walks the [S,D] observation matrix in 64-row tiles with the actor's
// weights resident in shared memory; the per-row KL is reduced in fp64 and the last CTA to
// finish folds the result into the device control block (no host round trip: the next
// pass's update kernel reads ctrl->stop itself).
#include "spo_common.cuh"

// tensor-core (wgmma + TMA) implementation for large batches, csrc/spo_tc_forward.cu:
// 0 = ran, 1 = not applicable (small batch, D % 4 != 0, ...), < 0 = error
int spo_tc_forward_launch(const spo_dims* d, const float* params, const float* obs, const float* old_mean,
                          const float* old_log_std, float* mean_out, int64_t count, int mode, int reduce, float target_kl,
                          spo_update_ctrl* ctrl, cudaStream_t stream);

namespace {

struct FbArgs {
  const float* params;
  const float* obs;
  const float* old_mean;
  const float* old_log_std;
  float* mean_out;
  int64_t count;
  int D, A, mode, reduce;   // mode 0: write means, 1: KL (accumulate + finalize), 2: KL accumulate only
  float target_kl;
  spo_update_ctrl* ctrl;
};

__global__ void __launch_bounds__(SPO_THREADS) spo_fullbatch_kernel(const FbArgs a) {
  extern __shared__ __align__(16) float smem[];
  __shared__ double red[SPO_THREADS / 32];
  __shared__ bool is_last;
  const int tid = threadIdx.x;
  if (a.mode >= 1 && *reinterpret_cast<volatile int*>(&a.ctrl->stop)) return;
  const int D = a.D, A = a.A, Dp = spo_pad4(D), ldx = spo_ld(D);
  const SpoNetOff off = spo_net_off(D, A, 0);
  SpoNetSmem w;
  float* p = spo_carve_net(smem, D, A, false, w);
  float* x = p;  p += SPO_ROWS * ldx;
  float* h1 = p; p += SPO_ROWS * SPO_LDH;
  float* h2 = p; p += SPO_ROWS * SPO_LDH;
  float* y = p;

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
    spo_out_fwd(h2, w.w3, w.b3, A, y, SPO_MAX_ACT, tid, SPO_THREADS);
    __syncthreads();
    if (a.mode == 0) {
      for (int i = tid; i < rows * A; i += SPO_THREADS) {
        const int r = i / A, j = i - r * A;
        a.mean_out[(row0 + r) * A + j] = y[r * SPO_MAX_ACT + j];
      }
    } else if (tid < rows) {
      float kl = 0.f;
      for (int j = 0; j < A; ++j) {
        // _kl_normal_normal(p = old, q = new)
        const float qs = expf(__ldg(a.params + off.log_std + j));
        const float ps = expf(__ldg(a.old_log_std + j));
        const float sr = __fdiv_rn(ps, qs);
        const float vr = __fmul_rn(sr, sr);
        const float dm = __fdiv_rn(__fsub_rn(__ldg(a.old_mean + (row0 + tid) * A + j), y[tid * SPO_MAX_ACT + j]), qs);
        const float t1 = __fmul_rn(dm, dm);
        const float klj = __fmul_rn(0.5f, __fsub_rn(__fsub_rn(__fadd_rn(vr, t1), 1.f), logf(vr)));
        kl = (j == 0) ? klj : __fadd_rn(kl, klj);
      }
      acc += static_cast<double>(kl);
    }
  }
  if (a.mode == 0) return;
  acc = spo_warp_sum(acc);
  if ((tid & 31) == 0) red[tid >> 5] = acc;
  __syncthreads();
  if (tid == 0) {
    double s = 0.0;
    for (int i = 0; i < SPO_THREADS / 32; ++i) s += red[i];
    atomicAdd(&a.ctrl->kl_sum, s);
    is_last = false;
    if (a.mode == 1) {
      __threadfence();
      const unsigned t = atomicAdd(&a.ctrl->ticket, 1u);
      is_last = (t == gridDim.x - 1);
    }
  }
  __syncthreads();
  if (is_last && tid == 0) {
    __threadfence();
    const double total = *reinterpret_cast<volatile double*>(&a.ctrl->kl_sum);
    const double denom = a.reduce == 0 ? static_cast<double>(a.count) : static_cast<double>(a.count) * A;
    const float kl = static_cast<float>(total / denom);
    a.ctrl->final_kl = kl;
    a.ctrl->passes += 1;
    if (kl > a.target_kl) a.ctrl->stop = 1;
    a.ctrl->kl_sum = 0.0;
    a.ctrl->ticket = 0u;
  }
}

int launch_fullbatch(const FbArgs& a, cudaStream_t stream) {
  static bool attr_set = false;
  const size_t smem = sizeof(float) * (spo_net_smem_floats(a.D, a.A, false) + SPO_ROWS * spo_ld(a.D) +
                                       2 * SPO_ROWS * SPO_LDH + SPO_ROWS * SPO_MAX_ACT);
  if (!attr_set) {
    SPO_CUDA_TRY(cudaFuncSetAttribute(spo_fullbatch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  const int64_t n_tiles = (a.count + SPO_ROWS - 1) / SPO_ROWS;
  const int grid = static_cast<int>(n_tiles < 2 * spo_sm_count() ? n_tiles : 2 * spo_sm_count());   // 2 CTAs per SM
  spo_fullbatch_kernel<<<grid, SPO_THREADS, smem, stream>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

__global__ void spo_kl_finalize_kernel(spo_update_ctrl* ctrl, double denom, float target_kl) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (ctrl->stop) { ctrl->kl_sum = 0.0; return; }
  const float kl = static_cast<float>(ctrl->kl_sum / denom);
  ctrl->final_kl = kl;
  ctrl->passes += 1;
  if (kl > target_kl) ctrl->stop = 1;
  ctrl->kl_sum = 0.0;
}

}  // namespace

extern "C" {

int spo_actor_kl_accumulate(const spo_dims* d, const float* params, const float* obs, const float* old_mean,
                            const float* old_log_std, int64_t count, spo_update_ctrl* ctrl, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(params && obs && old_mean && old_log_std && ctrl && count > 0, SPO_ERR_INVALID_ARG, "spo_actor_kl_accumulate: null pointer or count<=0");
  rc = spo_tc_forward_launch(d, params, obs, old_mean, old_log_std, nullptr, count, 2, 0, 0.f, ctrl, static_cast<cudaStream_t>(stream));
  if (rc <= 0) return rc;
  FbArgs a{};
  a.params = params; a.obs = obs; a.old_mean = old_mean; a.old_log_std = old_log_std; a.count = count;
  a.D = d->obs_dim; a.A = d->act_dim; a.mode = 2; a.ctrl = ctrl;
  return launch_fullbatch(a, static_cast<cudaStream_t>(stream));
}

int spo_kl_finalize(spo_update_ctrl* ctrl, double denom, float target_kl, void* stream) {
  SPO_REQUIRE(ctrl && denom > 0, SPO_ERR_INVALID_ARG, "spo_kl_finalize: null ctrl or denom<=0");
  spo_kl_finalize_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(ctrl, denom, target_kl);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_actor_forward(const spo_dims* d, const float* params, const float* obs, int64_t count,
                      float* mean_out, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(params && obs && mean_out && count > 0, SPO_ERR_INVALID_ARG, "spo_actor_forward: null pointer or count<=0");
  rc = spo_tc_forward_launch(d, params, obs, nullptr, nullptr, mean_out, count, 0, 0, 0.f, nullptr, static_cast<cudaStream_t>(stream));
  if (rc <= 0) return rc;
  FbArgs a{};
  a.params = params; a.obs = obs; a.mean_out = mean_out; a.count = count; a.D = d->obs_dim; a.A = d->act_dim; a.mode = 0;
  return launch_fullbatch(a, static_cast<cudaStream_t>(stream));
}

int spo_actor_kl(const spo_dims* d, const float* params, const float* obs, const float* old_mean,
                 const float* old_log_std, int64_t count, int reduce, float target_kl,
                 spo_update_ctrl* ctrl, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(params && obs && old_mean && old_log_std && ctrl && count > 0, SPO_ERR_INVALID_ARG, "spo_actor_kl: null pointer or count<=0");
  SPO_REQUIRE(reduce == 0 || reduce == 1, SPO_ERR_INVALID_ARG, "spo_actor_kl: reduce=%d", reduce);
  rc = spo_tc_forward_launch(d, params, obs, old_mean, old_log_std, nullptr, count, 1, reduce, target_kl, ctrl, static_cast<cudaStream_t>(stream));
  if (rc <= 0) return rc;
  FbArgs a{};
  a.params = params; a.obs = obs; a.old_mean = old_mean; a.old_log_std = old_log_std; a.count = count;
  a.D = d->obs_dim; a.A = d->act_dim; a.mode = 1; a.reduce = reduce; a.target_kl = target_kl; a.ctrl = ctrl;
  return launch_fullbatch(a, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
