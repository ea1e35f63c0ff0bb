// Rollout-side kernels: fused ActorVCritic.step + buffer.store, bootstrap critic values,
// per-slot segment bookkeeping.
//
// References: safepo/common/model.py:149-170 (step), safepo/common/buffer.py:84-95
// (store), safepo/single_agent/ppo_lag.py:187-234 (segment / bootstrap rule).
#include "spo_common.cuh"

// csrc/spo_tc_forward.cu: the same step on TMA + wgmma (returns 1 when the shape does not qualify)
int spo_tc_step_launch(const spo_dims* d, const float* params, const float* obs, const float* eps, uint64_t seed, uint64_t offset,
                       int deterministic, int n, float* act, float* logp, float* v_r, float* v_c, const spo_rollout* store, int t,
                       int net_base, cudaStream_t stream);

namespace {

constexpr float kLogSqrt2Pi = 0.91893853320467274178f;  // math.log(math.sqrt(2*math.pi))

struct StepArgs {
  const float* params;
  const float* obs;   // [n,D]
  const float* eps;   // [n,A] or null
  uint64_t seed, offset;
  int deterministic, n, D, A;
  float *act, *logp, *v_r, *v_c;
  spo_rollout store;
  int has_store, t;
  int net_base;  // 0: actor + critics (grid.y = 3), 1: critics only (grid.y = 2)
};

// grid = (ceil(n/64), nets), block = 256.  One CTA evaluates one net on one 64-row tile.
__global__ void __launch_bounds__(SPO_THREADS) spo_step_kernel(const StepArgs a) {
  extern __shared__ __align__(16) float smem[];
  const int tid = threadIdx.x;
  const int net = a.net_base + blockIdx.y;
  const int D = a.D, A = a.A;
  const SpoNetOff off = spo_net_off(D, A, net);
  const int O = off.out;
  const int ldx = spo_ld(D);
  const int Dp = spo_pad4(D);

  SpoNetSmem w;
  float* p = spo_carve_net(smem, D, O, false, w);
  float* x = p;   p += SPO_ROWS * ldx;
  float* h1 = p;  p += SPO_ROWS * SPO_LDH;
  float* h2 = p;  p += SPO_ROWS * SPO_LDH;
  float* y = p;   // [64][8]

  const int64_t row0 = static_cast<int64_t>(blockIdx.x) * SPO_ROWS;
  const int rows = min(SPO_ROWS, a.n - static_cast<int>(row0));

  spo_load_net(a.params, off, D, w, tid, SPO_THREADS);
  spo_load_rows(a.obs, D, ldx, nullptr, row0, rows, x, tid, SPO_THREADS);
  __syncthreads();
  spo_hidden_fwd(x, ldx, Dp, w.w1t, w.b1, h1, tid);
  __syncthreads();
  spo_hidden_fwd(h1, SPO_LDH, SPO_HID, w.w2t, w.b2, h2, tid);
  __syncthreads();
  spo_out_fwd(h2, w.w3, w.b3, O, y, SPO_MAX_ACT, tid, SPO_THREADS);
  __syncthreads();

  const int T = a.store.steps;
  if (net == 0) {
    // sample + log-prob, one thread per row (model.py:161-167; Normal.rsample / log_prob)
    if (tid < rows) {
      const int r = tid;
      const int64_t g = row0 + r;
      float lp = 0.f;
      float* act_out = a.act ? a.act + g * A : nullptr;
      float* act_st = a.has_store ? a.store.act + (g * T + a.t) * A : nullptr;
      for (int j = 0; j < A; ++j) {
        const float mean = y[r * SPO_MAX_ACT + j];
        const float std = expf(__ldg(a.params + off.log_std + j));
        float action = mean;
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
          action = __fadd_rn(mean, __fmul_rn(e, std));  // loc + eps * scale
        }
        const float diff = __fsub_rn(action, mean);
        const float var = __fmul_rn(std, std);
        const float q = __fdiv_rn(-__fmul_rn(diff, diff), __fmul_rn(2.f, var));
        const float term = __fsub_rn(__fsub_rn(q, logf(std)), kLogSqrt2Pi);
        lp = (j == 0) ? term : __fadd_rn(lp, term);
        if (act_out) act_out[j] = action;
        if (act_st) act_st[j] = action;
      }
      if (a.logp) a.logp[g] = lp;
      if (a.has_store) a.store.logp[g * T + a.t] = lp;
    }
    if (a.has_store) {
      // obs row copy into slot t (buffer.py:91-95)
      for (int i = tid; i < rows * D; i += SPO_THREADS) {
        const int r = i / D, c = i - r * D;
        a.store.obs[((row0 + r) * T + a.t) * D + c] = x[r * ldx + c];
      }
    }
  } else {
    float* vout = (net == 1) ? a.v_r : a.v_c;
    float* vst = a.has_store ? ((net == 1) ? a.store.value_r : a.store.value_c) : nullptr;
    if (tid < rows) {
      const float v = y[tid * SPO_MAX_ACT];
      if (vout) vout[row0 + tid] = v;
      if (vst) vst[(row0 + tid) * T + a.t] = v;
    }
  }
}

size_t step_smem_bytes(int D, int O) {
  return sizeof(float) * (spo_net_smem_floats(D, O, false) + SPO_ROWS * spo_ld(D) + 2 * SPO_ROWS * SPO_LDH +
                          SPO_ROWS * SPO_MAX_ACT);
}

int launch_step(const StepArgs& a, cudaStream_t stream) {
  static bool attr_set = false;
  const size_t smem = step_smem_bytes(a.D, a.A > 1 ? a.A : 1);
  if (!attr_set) {
    SPO_CUDA_TRY(cudaFuncSetAttribute(spo_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  dim3 grid((a.n + SPO_ROWS - 1) / SPO_ROWS, a.net_base == 0 ? 3 : 2);
  spo_step_kernel<<<grid, SPO_THREADS, smem, stream>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

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

int spo_policy_step(const spo_dims* d, const float* params, const float* obs, const float* eps,
                    uint64_t seed, uint64_t offset, int deterministic, int n,
                    float* act, float* logp, float* v_r, float* v_c,
                    const spo_rollout* store, int t, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(params && obs && n > 0, SPO_ERR_INVALID_ARG, "spo_policy_step: null params/obs or n<=0");
  StepArgs a{};
  a.params = params; a.obs = obs; a.eps = eps; a.seed = seed; a.offset = offset;
  a.deterministic = deterministic; a.n = n; a.D = d->obs_dim; a.A = d->act_dim;
  a.act = act; a.logp = logp; a.v_r = v_r; a.v_c = v_c;
  a.net_base = 0;
  if (store) {
    SPO_REQUIRE(store->num_envs == n, SPO_ERR_INVALID_ARG, "spo_policy_step: store->num_envs=%d != n=%d", store->num_envs, n);
    SPO_REQUIRE(t >= 0 && t < store->steps, SPO_ERR_INVALID_ARG, "spo_policy_step: slot t=%d outside [0,%d) (buffer overflow)", t, store->steps);
    a.store = *store; a.has_store = 1; a.t = t;
  } else {
    a.store.steps = 1;
  }
  // batches of >= 128 rows with a TMA-friendly layout run on the tensor-core kernel; single rows ([D] inputs of the
  // bootstrap calls, ppo_lag.py:206,211), odd obs_dim and obs_dim > 64 on the FFMA tile kernel below
  rc = spo_tc_step_launch(d, params, obs, eps, seed, offset, deterministic, n, act, logp, v_r, v_c, store, t, 0,
                          static_cast<cudaStream_t>(stream));
  if (rc <= 0) return rc;
  return launch_step(a, static_cast<cudaStream_t>(stream));
}

int spo_critic_values(const spo_dims* d, const float* params, const float* obs, int n,
                      float* v_r, float* v_c, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(params && obs && n > 0, SPO_ERR_INVALID_ARG, "spo_critic_values: null params/obs or n<=0");
  StepArgs a{};
  a.params = params; a.obs = obs; a.n = n; a.D = d->obs_dim; a.A = d->act_dim;
  a.v_r = v_r; a.v_c = v_c; a.net_base = 1; a.store.steps = 1;
  rc = spo_tc_step_launch(d, params, obs, nullptr, 0, 0, 1, n, nullptr, nullptr, v_r, v_c, nullptr, 0, 1, static_cast<cudaStream_t>(stream));
  if (rc <= 0) return rc;
  return launch_step(a, static_cast<cudaStream_t>(stream));
}

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
