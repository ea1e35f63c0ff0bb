// Dual (reward + cost) GAE over every path of every env in one launch, and the
// advantage statistics / standardisation / Lagrange mix of buffer.get().
//
// References: safepo/common/buffer.py:97-140 (finish_path), :167-188 (discount_cumsum,
// float64 carry), :191-201 (calculate_adv_and_value_targets), :142-164 (get),
// safepo/single_agent/ppo_lag.py:280-281 (advantage mix).
//
// Layout: env-major [N,T] fp32.  A path closes at every slot with seg_end != 0; the last
// slot of an env always closes a path (the reference's epoch_end rule, ppo_lag.py:198).
//
// Recurrence per path (t descending):  delta_t = (r_t + gamma*v_{t+1}) - v_t   (fp32, unfused)
//                                      A_t     = delta_t + disc * A_{t+1}       (fp64)
// written as the affine map A_t = b_t + a_t * A_{t+1} with a_t = seg_end[t] ? 0 : disc.
// mode 0 composes the maps with a block-wide reverse scan (warp shuffles + one smem hop),
// mode 1 runs the recurrence sequentially per env (bit-exact with the reference).
#include "spo_common.cuh"

namespace {

struct GaeArgs {
  const float *reward, *cost, *value_r, *value_c;
  const uint8_t* seg_end;
  const float *boot_r, *boot_c;
  float gamma;
  double disc_r, disc_c;
  float *adv_r, *adv_c, *tgt_r, *tgt_c;
  int N, T;
};

struct Aff {  // x -> b + a*x
  double a, b;
};
// apply `first`, then `second`
__device__ __forceinline__ Aff then(const Aff& first, const Aff& second) {
  return Aff{first.a * second.a, second.a * first.b + second.b};
}
__device__ __forceinline__ Aff shfl_up_aff(const Aff& v, int d) {
  return Aff{__shfl_up_sync(0xffffffffu, v.a, d), __shfl_up_sync(0xffffffffu, v.b, d)};
}

__device__ __forceinline__ float gae_delta(float r, float vnext, float v, float gamma) {
  return __fsub_rn(__fadd_rn(r, __fmul_rn(gamma, vnext)), v);  // rewards + gamma*values[1:] - values[:-1]
}

constexpr int GAE_THREADS = 128;
constexpr int GAE_ITEMS = 4;
constexpr int GAE_TILE = GAE_THREADS * GAE_ITEMS;

// one CTA per env; tiles of 512 steps walked from the end of the epoch backwards.
__global__ void __launch_bounds__(GAE_THREADS) spo_gae_scan_kernel(const GaeArgs g) {
  __shared__ Aff warp_r[GAE_THREADS / 32], warp_c[GAE_THREADS / 32];
  const int env = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int T = g.T;
  const int64_t base = static_cast<int64_t>(env) * T;
  double carry_r = 0.0, carry_c = 0.0;  // A_{t+1} entering the current tile

  for (int hi = T - 1; hi >= 0; hi -= GAE_TILE) {
    Aff pre_r[GAE_ITEMS], pre_c[GAE_ITEMS];
    float vr[GAE_ITEMS], vc[GAE_ITEMS];
    // thread-local inclusive composition over its 4 consecutive (descending-t) items
#pragma unroll
    for (int i = 0; i < GAE_ITEMS; ++i) {
      const int t = hi - (tid * GAE_ITEMS + i);
      Aff er{1.0, 0.0}, ec{1.0, 0.0};  // identity for t < 0
      vr[i] = 0.f; vc[i] = 0.f;
      if (t >= 0) {
        const int64_t s = base + t;
        const bool end = (t == T - 1) || (g.seg_end[s] != 0);
        vr[i] = g.value_r[s];
        vc[i] = g.value_c[s];
        const float nr = end ? g.boot_r[s] : g.value_r[s + 1];
        const float nc = end ? g.boot_c[s] : g.value_c[s + 1];
        er = Aff{end ? 0.0 : g.disc_r, static_cast<double>(gae_delta(g.reward[s], nr, vr[i], g.gamma))};
        ec = Aff{end ? 0.0 : g.disc_c, static_cast<double>(gae_delta(g.cost[s], nc, vc[i], g.gamma))};
      }
      pre_r[i] = (i == 0) ? er : then(pre_r[i - 1], er);
      pre_c[i] = (i == 0) ? ec : then(pre_c[i - 1], ec);
    }
    // warp inclusive scan of thread aggregates
    Aff inc_r = pre_r[GAE_ITEMS - 1], inc_c = pre_c[GAE_ITEMS - 1];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const Aff or_ = shfl_up_aff(inc_r, d), oc_ = shfl_up_aff(inc_c, d);
      if (lane >= d) { inc_r = then(or_, inc_r); inc_c = then(oc_, inc_c); }
    }
    if (lane == 31) { warp_r[wid] = inc_r; warp_c[wid] = inc_c; }
    Aff exc_r = shfl_up_aff(inc_r, 1), exc_c = shfl_up_aff(inc_c, 1);
    if (lane == 0) { exc_r = Aff{1.0, 0.0}; exc_c = Aff{1.0, 0.0}; }
    __syncthreads();
    // value entering this thread: carry pushed through the earlier warps, then through exc
    double in_r = carry_r, in_c = carry_c;
    double tile_r = carry_r, tile_c = carry_c;
#pragma unroll
    for (int w = 0; w < GAE_THREADS / 32; ++w) {
      const Aff ar = warp_r[w], ac = warp_c[w];
      if (w < wid) { in_r = ar.b + ar.a * in_r; in_c = ac.b + ac.a * in_c; }
      tile_r = ar.b + ar.a * tile_r; tile_c = ac.b + ac.a * tile_c;
    }
    in_r = exc_r.b + exc_r.a * in_r;
    in_c = exc_c.b + exc_c.a * in_c;
#pragma unroll
    for (int i = 0; i < GAE_ITEMS; ++i) {
      const int t = hi - (tid * GAE_ITEMS + i);
      if (t >= 0) {
        const int64_t s = base + t;
        const double ar = pre_r[i].b + pre_r[i].a * in_r;
        const double ac = pre_c[i].b + pre_c[i].a * in_c;
        g.adv_r[s] = static_cast<float>(ar);
        g.adv_c[s] = static_cast<float>(ac);
        g.tgt_r[s] = static_cast<float>(ar + static_cast<double>(vr[i]));  // adv(f64) + values(f32)
        g.tgt_c[s] = static_cast<float>(ac + static_cast<double>(vc[i]));
      }
    }
    carry_r = tile_r; carry_c = tile_c;
    __syncthreads();
  }
}

// mode 1: sequential recurrence, one thread per env (cumsum = x[idx] + discount * cumsum).
__global__ void spo_gae_exact_kernel(const GaeArgs g) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= g.N) return;
  const int T = g.T;
  const int64_t base = static_cast<int64_t>(env) * T;
  double ar = 0.0, ac = 0.0;
  float vr_next = 0.f, vc_next = 0.f;
  for (int t = T - 1; t >= 0; --t) {
    const int64_t s = base + t;
    const bool end = (t == T - 1) || (g.seg_end[s] != 0);
    const float vr = g.value_r[s], vc = g.value_c[s];
    const float nr = end ? g.boot_r[s] : vr_next;
    const float nc = end ? g.boot_c[s] : vc_next;
    const double dr = static_cast<double>(gae_delta(g.reward[s], nr, vr, g.gamma));
    const double dc = static_cast<double>(gae_delta(g.cost[s], nc, vc, g.gamma));
    ar = end ? dr : __dadd_rn(dr, __dmul_rn(g.disc_r, ar));
    ac = end ? dc : __dadd_rn(dc, __dmul_rn(g.disc_c, ac));
    g.adv_r[s] = static_cast<float>(ar);
    g.adv_c[s] = static_cast<float>(ac);
    g.tgt_r[s] = static_cast<float>(__dadd_rn(ar, static_cast<double>(vr)));
    g.tgt_c[s] = static_cast<float>(__dadd_rn(ac, static_cast<double>(vc)));
    vr_next = vr; vc_next = vc;
  }
}

// ---- advantage statistics ---------------------------------------------------------------
__global__ void __launch_bounds__(256) spo_adv_stats_kernel(const float* __restrict__ adv_r,
                                                            const float* __restrict__ adv_c, int64_t count,
                                                            double* __restrict__ stats) {
  __shared__ double red[3][8];
  double s0 = 0.0, s1 = 0.0, s2 = 0.0;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < count;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const double a = adv_r[i], c = adv_c[i];
    s0 += a; s1 += a * a; s2 += c;
  }
  s0 = spo_warp_sum(s0); s1 = spo_warp_sum(s1); s2 = spo_warp_sum(s2);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { red[0][wid] = s0; red[1][wid] = s1; red[2][wid] = s2; }
  __syncthreads();
  if (threadIdx.x < 3) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += red[threadIdx.x][w];
    atomicAdd(stats + threadIdx.x, s);
  }
  if (blockIdx.x == 0 && threadIdx.x == 3) stats[3] = static_cast<double>(count);
}

__global__ void __launch_bounds__(256) spo_adv_apply_kernel(float* __restrict__ adv_r, float* __restrict__ adv_c,
                                                            int64_t count, const double* __restrict__ stats,
                                                            int std_r, int std_c, float lam, float lam_p1,
                                                            float* __restrict__ mixed) {
  const double n = stats[3];
  const double mean_d = stats[0] / n;
  const double var_d = (stats[1] - stats[0] * stats[0] / n) / (n - 1.0);  // unbiased, torch.Tensor.std default
  const float mean = static_cast<float>(mean_d);
  const float denom = __fadd_rn(static_cast<float>(sqrt(var_d < 0.0 ? 0.0 : var_d)), 1e-8f);
  const float cmean = static_cast<float>(stats[2] / n);
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < count;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float a = adv_r[i], c = adv_c[i];
    if (std_r) a = __fdiv_rn(__fsub_rn(a, mean), denom);
    if (std_c) c = __fsub_rn(c, cmean);
    adv_r[i] = a;
    adv_c[i] = c;
    if (mixed) mixed[i] = __fdiv_rn(__fsub_rn(a, __fmul_rn(lam, c)), lam_p1);
  }
}

}  // namespace

extern "C" {

int spo_gae_dual(const float* reward, const float* cost, const float* value_r, const float* value_c,
                 const uint8_t* seg_end, const float* boot_r, const float* boot_c,
                 float gamma, double disc_r, double disc_c,
                 float* adv_r, float* adv_c, float* tgt_r, float* tgt_c,
                 int num_envs, int steps, int mode, void* stream) {
  SPO_REQUIRE(reward && cost && value_r && value_c && seg_end && boot_r && boot_c && adv_r && adv_c && tgt_r && tgt_c,
              SPO_ERR_INVALID_ARG, "spo_gae_dual: null pointer argument");
  SPO_REQUIRE(num_envs >= 0 && steps >= 0, SPO_ERR_INVALID_ARG, "spo_gae_dual: negative size");
  SPO_REQUIRE(mode == 0 || mode == 1, SPO_ERR_INVALID_ARG, "spo_gae_dual: mode=%d (0 scan, 1 exact)", mode);
  if (num_envs == 0 || steps == 0) return SPO_OK;
  GaeArgs g{reward, cost, value_r, value_c, seg_end, boot_r, boot_c, gamma, disc_r, disc_c,
            adv_r, adv_c, tgt_r, tgt_c, num_envs, steps};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (mode == 0) {
    spo_gae_scan_kernel<<<num_envs, GAE_THREADS, 0, st>>>(g);
  } else {
    spo_gae_exact_kernel<<<(num_envs + 63) / 64, 64, 0, st>>>(g);
  }
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_adv_stats(const float* adv_r, const float* adv_c, int64_t count, double* stats, void* stream) {
  SPO_REQUIRE(adv_r && adv_c && stats && count > 0, SPO_ERR_INVALID_ARG, "spo_adv_stats: null pointer or count<=0");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SPO_CUDA_TRY(cudaMemsetAsync(stats, 0, 4 * sizeof(double), st));
  int blocks = static_cast<int>((count + 256 * 8 - 1) / (256 * 8));
  if (blocks > spo_sm_count() * 8) blocks = spo_sm_count() * 8;
  spo_adv_stats_kernel<<<blocks, 256, 0, st>>>(adv_r, adv_c, count, stats);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_adv_apply(float* adv_r, float* adv_c, int64_t count, const double* stats,
                  int standardize_r, int standardize_c, float lam, float lam_plus_1,
                  float* mixed, void* stream) {
  SPO_REQUIRE(adv_r && adv_c && stats && count > 0, SPO_ERR_INVALID_ARG, "spo_adv_apply: null pointer or count<=0");
  int blocks = static_cast<int>((count + 256 * 4 - 1) / (256 * 4));
  if (blocks > spo_sm_count() * 8) blocks = spo_sm_count() * 8;
  spo_adv_apply_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(adv_r, adv_c, count, stats, standardize_r,
                                                                          standardize_c, lam, lam_plus_1, mixed);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

}  // extern "C"
