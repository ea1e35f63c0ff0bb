// Multi-agent PPO loss heads of MAPPO and HAPPO (safepo/multi_agent/mappo.py:106-163, happo.py:106-171) on the device, for
// the actor and critic nets of spo_ma.cu / spo_ma_update.cu: the training forward, the backward chain, clip + Adam and PopArt
// are shared with MAPPO-Lag; what is new here is
//   - the per-dimension clipped surrogate of MAPPO (mappo.py:137-147): imp_j = exp(logp_j - old_logp_j) is [n, A] and every
//     dimension has its own clip branch, loss_row = -sum_j min(imp_j adv, clamp(imp_j) adv);
//   - HAPPO's product ratio x cross-agent factor on the plain advantage (happo.py:144-155), and MAPPO-Lag's lambda-mixed one;
//   - active masks (use_policy_active_masks / use_value_active_masks): row weights m_r / sum m instead of 1 / n, and the masked
//     entropy of act.py:69-70, (entropy() [n, A] * m).sum() / m.sum() = sum_j e_j (A times the unmasked mean over j).
// sum m is a device scalar (a torch .sum() of 0/1 floats: exact in any order below 2^24); with every row inactive it is 0 and
// the results are NaN, as the reference's 0 / 0.  Reductions over rows are per-CTA partials summed in CTA order by the
// finalize kernel (or spo_ma_partial_reduce): results do not depend on scheduling.
//
// Cost: one warp per row computes the A head dot products over H (A H FMA per row, the features read once per dimension from
// L1/L2) -- the same loop as ma_actor_loss_kernel, which it reproduces bit for bit in MAPPO-Lag's configuration.  At config 5
// (8192 rows, H 512, A 20) that is 84 MFLOP and 17 MB of feature reads: latency of the warp-serial dimension loop, not
// bandwidth, bounds it; it is one launch per update beside three layers of 2-4 GFLOP.
#include "spo_common.cuh"
#include "spo_ma_loss.cuh"

namespace {

constexpr int PPO_ROWS = 32;        // rows per CTA (4 per warp)
constexpr int PPO_THREADS = 256;
constexpr int PPO_PART = 2 + 64;    // per-CTA partials: {sum w_r loss_r, sum ratio, sum dmean_j (32), sum dstd_j (32)}
constexpr float kLogSqrt2Pi = 0.91893853320467274178f;

struct PpoActorArgs {
  const float *feat, *W, *b, *log_std, *actions, *old_logp, *adv, *cost_adv, *lamda, *factor, *masks, *mask_sum;
  float *dmean, *imp, *part;
  int n, H, A, per_dim;
  float clip_lo, clip_hi, x_coef, y_coef;
};

// One warp per row, lane j < A owns action dimension j.
//   mean = feat W^T + b;  std = sigmoid(log_std / x) y;  logp_j = -(a - mean)^2 / (2 std^2) - log std - log sqrt(2 pi)
//   adv = adv_targ (- lamda cost_adv_targ);  w_r = 1 / n, or m_r / sum m with masks;  fac = factor or 1
//   PRODUCT: imp = prod_j exp(logp_j - old_j);  loss_r = -fac min(imp adv, clamp(imp) adv)
//            d loss / d logp_j = [imp adv <= clamp(imp) adv] (-fac adv w_r) imp          (the same for every j)
//   PER_DIM: imp_j = exp(logp_j - old_j);     loss_r = -fac sum_j min(imp_j adv, clamp(imp_j) adv)
//            d loss / d logp_j = [imp_j adv <= clamp(imp_j) adv] (-fac adv w_r) imp_j
// The branch rule s1 <= s2 gives torch's total at ties (torch.min splits them 0.5 / 0.5, clamp's backward includes both edges).
__global__ void __launch_bounds__(PPO_THREADS) ma_ppo_actor_loss_kernel(const PpoActorArgs a) {
  __shared__ float red[PPO_THREADS / 32][PPO_PART];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int row0 = blockIdx.x * PPO_ROWS, A = a.A, H = a.H;
  const float inv_n = a.masks ? __fdiv_rn(1.f, *a.mask_sum) : __fdiv_rn(1.f, static_cast<float>(a.n));
  const float lam = a.lamda ? *a.lamda : 0.f;
  float std = 1.f, bj = 0.f;
  if (lane < A) {
    std = __fmul_rn(__fdiv_rn(1.f, 1.f + expf(-__fdiv_rn(a.log_std[lane], a.x_coef))), a.y_coef);   // as spo_ma_head_kernel
    bj = a.b[lane];
  }
  const float inv_var = __fdiv_rn(1.f, __fmul_rn(std, std)), log_std_v = logf(std);
  float sum_loss = 0.f, sum_ratio = 0.f, sum_dm = 0.f, sum_ds = 0.f;
  for (int r = 0; r < 4; ++r) {
    const int g = row0 + 4 * wid + r;
    if (g >= a.n) break;                                   // warp-uniform
    const float* f = a.feat + static_cast<size_t>(g) * H;
    float mu = 0.f;
    for (int j = 0; j < A; ++j) {
      float s = 0.f;
      for (int k = lane; k < H; k += 32) s = fmaf(f[k], __ldg(a.W + j * H + k), s);
      s = spo_warp_sum(s);
      if (lane == j) mu = s + bj;
    }
    float ratio = 1.f, diff = 0.f;
    if (lane < A) {
      const float act = a.actions[static_cast<size_t>(g) * A + lane];
      diff = __fsub_rn(act, mu);
      const float q = __fdiv_rn(-__fmul_rn(diff, diff), __fmul_rn(2.f, __fmul_rn(std, std)));
      const float logp = __fsub_rn(__fsub_rn(q, log_std_v), kLogSqrt2Pi);
      ratio = expf(__fsub_rn(logp, a.old_logp[static_cast<size_t>(g) * A + lane]));
    }
    const float adv = a.cost_adv ? __fsub_rn(a.adv[g], __fmul_rn(lam, a.cost_adv[g])) : a.adv[g];
    const float fac = a.factor ? a.factor[g] : 1.f;
    const float wr = a.masks ? __fmul_rn(a.masks[g], inv_n) : inv_n;
    const float gw = -__fmul_rn(__fmul_rn(fac, adv), wr);
    float crow;
    if (!a.per_dim) {
      float imp = ratio;
#pragma unroll
      for (int m = 16; m > 0; m >>= 1) imp *= __shfl_xor_sync(0xffffffffu, imp, m);
      const float s1 = __fmul_rn(imp, adv);
      const float s2 = __fmul_rn(fminf(fmaxf(imp, a.clip_lo), a.clip_hi), adv);
      crow = __fmul_rn((s1 <= s2) ? gw : 0.f, imp);
      if (lane == 0) {
        a.imp[g] = imp;
        const float l = -__fmul_rn(fac, fminf(s1, s2));
        sum_loss += a.masks ? __fmul_rn(l, a.masks[g]) : l;
        sum_ratio += imp;
      }
    } else {
      const float s1 = __fmul_rn(ratio, adv);
      const float s2 = __fmul_rn(fminf(fmaxf(ratio, a.clip_lo), a.clip_hi), adv);
      crow = __fmul_rn((s1 <= s2) ? gw : 0.f, ratio);
      const float row_min = spo_warp_sum(lane < A ? fminf(s1, s2) : 0.f);
      const float row_ratio = spo_warp_sum(lane < A ? ratio : 0.f);
      if (lane < A) a.imp[static_cast<size_t>(g) * A + lane] = ratio;
      if (lane == 0) {
        const float l = -__fmul_rn(fac, row_min);
        sum_loss += a.masks ? __fmul_rn(l, a.masks[g]) : l;
        sum_ratio += row_ratio;
      }
    }
    if (lane < A) {
      const float dm = __fmul_rn(crow, __fmul_rn(diff, inv_var));
      // d logp / d std = (a - mean)^2 / std^3 - 1 / std
      const float ds = __fmul_rn(crow, __fsub_rn(__fmul_rn(__fmul_rn(diff, diff), __fdiv_rn(inv_var, std)), __fdiv_rn(1.f, std)));
      a.dmean[static_cast<size_t>(g) * A + lane] = dm;
      sum_dm += dm;
      sum_ds += ds;
    }
  }
  if (lane == 0) { red[wid][0] = sum_loss; red[wid][1] = sum_ratio; }
  red[wid][2 + lane] = sum_dm;
  red[wid][2 + 32 + lane] = sum_ds;
  __syncthreads();
  if (tid < PPO_PART) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < PPO_THREADS / 32; ++w) s += red[w][tid];
    a.part[static_cast<size_t>(blockIdx.x) * PPO_PART + tid] = s;
  }
}

// One CTA: sums the partials over the CTAs in order and finishes the scalars and the small gradients.
//   policy_loss = sum w-less loss_r (masked: m_r loss_r) / (n or sum m);  mean ratio = sum ratio / (n or n A)
//   entropy = mean_j e_j without masks, q sum_j e_j with them (q = sum m / sum m: 1, or NaN when every row is inactive),
//   e_j = 0.5 + log sqrt(2 pi) + log std_j (act.py:57-60, 69-70)
//   g_b[j] = sum_r dmean_j;  g_log_std[j] = (sum_r dstd_j - c_j) d std / d log_std, c_j = entropy_coef / (A std_j) or q entropy_coef / std_j
struct PpoFinalArgs {
  const float *part, *log_std, *mask_sum;
  float *g_b, *g_log_std, *scalars;    // scalars[0] = policy_loss, [1] = dist_entropy, [2] = mean importance weight
  int nblk, n, A, per_dim;
  float x_coef, y_coef, entropy_coef;
};

__global__ void __launch_bounds__(128) ma_ppo_actor_final_kernel(const PpoFinalArgs a) {
  __shared__ float tot[PPO_PART];
  __shared__ float ent[32];
  const int tid = threadIdx.x;
  if (tid < PPO_PART) {
    float s = 0.f;
    for (int b = 0; b < a.nblk; ++b) s += a.part[static_cast<size_t>(b) * PPO_PART + tid];
    tot[tid] = s;
  }
  if (tid < 32) ent[tid] = 0.f;
  __syncthreads();
  const float msum = a.mask_sum ? *a.mask_sum : 0.f;
  const float q = __fdiv_rn(msum, msum);
  if (tid < a.A) {
    const float sg = __fdiv_rn(1.f, 1.f + expf(-__fdiv_rn(a.log_std[tid], a.x_coef)));
    const float std = __fmul_rn(sg, a.y_coef);
    const float dstd_dls = __fdiv_rn(__fmul_rn(a.y_coef, __fmul_rn(sg, 1.f - sg)), a.x_coef);
    const float c = a.mask_sum ? __fdiv_rn(__fmul_rn(q, a.entropy_coef), std)
                               : __fdiv_rn(a.entropy_coef, __fmul_rn(static_cast<float>(a.A), std));
    a.g_log_std[tid] = __fmul_rn(tot[2 + 32 + tid] - c, dstd_dls);
    a.g_b[tid] = tot[2 + tid];
    ent[tid] = 0.5f + kLogSqrt2Pi + logf(std);          // 0.5 + 0.5 log(2 pi) + log std
  }
  __syncthreads();
  if (tid == 0) {
    float e = 0.f;
    for (int j = 0; j < a.A; ++j) e += ent[j];
    a.scalars[0] = __fdiv_rn(tot[0], a.mask_sum ? msum : static_cast<float>(a.n));
    a.scalars[1] = a.mask_sum ? __fmul_rn(q, e) : __fdiv_rn(e, static_cast<float>(a.A));
    a.scalars[2] = __fdiv_rn(tot[1], static_cast<float>(a.per_dim ? a.n * a.A : a.n));
  }
}

// Value loss with row weights (happo.py:106-122 with use_value_active_masks): the clipped one-sided-Huber loss of
// ma_value_loss_kernel, torch.max's tie rule included, each row weighted by w_r = m_r / sum m.
//   dv[r] = coef w_r dL_r / dv;  part[blk] = {sum w_r L_r, sum dv}  (the loss is the sum of the first entries)
struct MaskedValueArgs {
  const float *v, *vp, *rn_c, *rn_o, *masks, *mask_sum;
  float *dv, *part;
  int n;
  float clip, delta, coef;
};

__global__ void __launch_bounds__(256) ma_value_loss_masked_kernel(const MaskedValueArgs a) {
  __shared__ float red[8][2];
  const int i = blockIdx.x * 256 + threadIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float L = 0.f, dv = 0.f;
  if (i < a.n) {
    const float wr = __fmul_rn(a.masks[i], __fdiv_rn(1.f, *a.mask_sum));
    const float v = a.v[i], vp = a.vp[i];
    const float dlt = __fsub_rn(v, vp);
    const float vpc = __fadd_rn(vp, fminf(fmaxf(dlt, -a.clip), a.clip));
    const float ec = __fsub_rn(a.rn_c[i], vpc), eo = __fsub_rn(a.rn_o[i], v);
    const float hc = huber_val(ec, a.delta), ho = huber_val(eo, a.delta);
    L = __fmul_rn(wr, fmaxf(ho, hc));
    const float wo = (ho > hc) ? 1.f : (ho == hc ? 0.5f : 0.f);
    const float inr = (dlt >= -a.clip && dlt <= a.clip) ? 1.f : 0.f;
    dv = __fmul_rn(a.coef, wr) * (wo * (-huber_grad(eo, a.delta)) + (1.f - wo) * inr * (-huber_grad(ec, a.delta)));
    a.dv[i] = dv;
  }
  L = spo_warp_sum(L);
  dv = spo_warp_sum(dv);
  if (lane == 0) { red[wid][0] = L; red[wid][1] = dv; }
  __syncthreads();
  if (threadIdx.x < 2) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
    a.part[blockIdx.x * 2 + threadIdx.x] = s;
  }
}

}  // namespace

extern "C" {

int spo_ma_ppo_actor_loss(const float* feat, int n, int H, const float* W, const float* b, const float* log_std, int A, const float* actions,
                          const float* old_logp, const float* adv, const float* cost_adv, const float* lamda, const float* factor,
                          const float* active_masks, const float* mask_sum, int ratio_mode, float clip_lo, float clip_hi, float std_x_coef,
                          float std_y_coef, float* dmean, float* imp, float* part, void* stream) {
  SPO_REQUIRE(feat && W && b && log_std && actions && old_logp && adv && dmean && imp && part && n > 0 && H > 0, SPO_ERR_INVALID_ARG,
              "spo_ma_ppo_actor_loss: null argument or empty shape");
  SPO_REQUIRE((cost_adv == nullptr) == (lamda == nullptr), SPO_ERR_INVALID_ARG,
              "spo_ma_ppo_actor_loss: the Lagrangian needs both lamda and cost_adv (or neither)");
  SPO_REQUIRE((active_masks == nullptr) == (mask_sum == nullptr), SPO_ERR_INVALID_ARG,
              "spo_ma_ppo_actor_loss: active masks need both active_masks and mask_sum (or neither)");
  SPO_REQUIRE(ratio_mode == SPO_MA_RATIO_PRODUCT || ratio_mode == SPO_MA_RATIO_PER_DIM, SPO_ERR_INVALID_ARG,
              "spo_ma_ppo_actor_loss: ratio_mode=%d must be SPO_MA_RATIO_PRODUCT or SPO_MA_RATIO_PER_DIM", ratio_mode);
  SPO_REQUIRE(A >= 1 && A <= 32, SPO_ERR_UNSUPPORTED, "spo_ma_ppo_actor_loss: act_dim=%d must be in 1..32", A);
  PpoActorArgs a{feat, W, b, log_std, actions, old_logp, adv, cost_adv, lamda, factor, active_masks, mask_sum, dmean, imp, part,
                 n, H, A, ratio_mode == SPO_MA_RATIO_PER_DIM, clip_lo, clip_hi, std_x_coef, std_y_coef};
  ma_ppo_actor_loss_kernel<<<(n + PPO_ROWS - 1) / PPO_ROWS, PPO_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_ppo_actor_finalize(const float* part, int nblk, int n, const float* mask_sum, int ratio_mode, const float* log_std, int A,
                              float std_x_coef, float std_y_coef, float entropy_coef, float* g_b, float* g_log_std, float* scalars, void* stream) {
  SPO_REQUIRE(part && log_std && g_b && g_log_std && scalars && nblk > 0 && n > 0, SPO_ERR_INVALID_ARG,
              "spo_ma_ppo_actor_finalize: null argument or empty shape");
  SPO_REQUIRE(ratio_mode == SPO_MA_RATIO_PRODUCT || ratio_mode == SPO_MA_RATIO_PER_DIM, SPO_ERR_INVALID_ARG,
              "spo_ma_ppo_actor_finalize: ratio_mode=%d must be SPO_MA_RATIO_PRODUCT or SPO_MA_RATIO_PER_DIM", ratio_mode);
  SPO_REQUIRE(A >= 1 && A <= 32, SPO_ERR_UNSUPPORTED, "spo_ma_ppo_actor_finalize: act_dim=%d must be in 1..32", A);
  SPO_REQUIRE(nblk == (n + PPO_ROWS - 1) / PPO_ROWS, SPO_ERR_INVALID_ARG, "spo_ma_ppo_actor_finalize: nblk=%d is not ceil(n/32) for n=%d",
              nblk, n);
  PpoFinalArgs a{part, log_std, mask_sum, g_b, g_log_std, scalars, nblk, n, A, ratio_mode == SPO_MA_RATIO_PER_DIM, std_x_coef, std_y_coef,
                 entropy_coef};
  ma_ppo_actor_final_kernel<<<1, 128, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_value_loss_masked(const float* v, const float* value_preds, const float* ret_norm_clipped, const float* ret_norm_orig,
                             const float* active_masks, const float* mask_sum, int n, float clip, float huber_delta, float coef, float* dv,
                             float* part, void* stream) {
  SPO_REQUIRE(v && value_preds && ret_norm_clipped && ret_norm_orig && active_masks && mask_sum && dv && part && n > 0, SPO_ERR_INVALID_ARG,
              "spo_ma_value_loss_masked: null argument or n<=0");
  MaskedValueArgs a{v, value_preds, ret_norm_clipped, ret_norm_orig, active_masks, mask_sum, dv, part, n, clip, huber_delta, coef};
  ma_value_loss_masked_kernel<<<(n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

}  // extern "C"
