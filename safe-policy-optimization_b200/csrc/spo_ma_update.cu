// Multi-agent (MAPPO-Lag, BASELINE config 5) network UPDATE: the device side of MAPPO_L_Trainer.ppo_update
// (safepo/multi_agent/mappolag.py:135-199) for one agent -- SURVEY section 8f rank 3, second slice.
//
// The three nets of an agent (MultiAgentActor / MultiAgentCritic x 2, safepo/common/model.py:172-363) are trained on the WHOLE
// batch per step (num_mini_batch 1, mappolag/config.yaml), so unlike the single-agent path this is throughput work: the
// forward of spo_ma.cu (run with its activations kept), then per layer
//     dz   = LayerNorm'(ELU'(.)) applied to the incoming gradient            (ma_ln_elu_bwd_kernel, one warp per row)
//     dW   = dz^T x   (reduction over the n rows, split over the grid)       (ma_gemm_tn_kernel + ma_partial_reduce_kernel)
//     dx   = dz W                                                            (ma_gemm_nn_kernel)
// and the loss heads (clipped surrogate on the product of per-dimension ratios with the Lagrangian-mixed advantage;
// PopArt-normalised, clipped, one-sided-Huber value loss), the joint-norm clip and Adam on the packed parameter buffer.
// Every reduction over rows is a two-stage sum in a fixed order (per-CTA partials, then one thread per output over the CTAs):
// results do not depend on scheduling.  The products run on the tensor pipe as mma.sync 3xTF32 tiles (128 x 64 x 32); moving them to
// wgmma with the 3xTF32 operand copies of spo_tc_forward.cu is the next step for this path (DESIGN.md section 8).
#include "spo_common.cuh"
#include "spo_ma_loss.cuh"
#include "spo_mma.cuh"

namespace {

constexpr int MU_ROWS = 32;        // rows per CTA of the row-wise kernels
constexpr int MU_THREADS = 256;
constexpr float kLogSqrt2Pi = 0.91893853320467274178f;

// ------------------------------------------------------------------------------------------------------------------
// LayerNorm + ELU backward of one [Linear -> ELU -> LayerNorm] block (mlp.py:18-27).
//   pre = ELU(z) (kept by the training forward), y = LN(pre) * gamma + beta, dy = d loss / d y
//   xhat = (pre - mean) * rstd;  dxhat = dy * gamma;  dpre = rstd * (dxhat - mean(dxhat) - xhat * mean(dxhat * xhat))
//   dz = dpre * (pre > 0 ? 1 : pre + 1)          [ELU'(z) = exp(z) = ELU(z) + 1 for z <= 0]
// Per-CTA partial column sums: part[blk][0] = sum_r dy * xhat (d gamma), [1] = sum_r dy (d beta), [2] = sum_r dz (d bias).
// Warp w holds rows 4w..4w+3 of the CTA's 32 completely: lane l owns columns 128 cb + 4 l .. + 3.
// ------------------------------------------------------------------------------------------------------------------
struct LnEluBwdArgs {
  const float *dy, *pre, *ln_w;
  float *dz, *part;
  int n, H;
};

template <int HB>
__global__ void __launch_bounds__(MU_THREADS) ma_ln_elu_bwd_kernel(const LnEluBwdArgs a) {
  constexpr int H = 128 * HB;
  __shared__ float acc_s[3][H];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int row0 = blockIdx.x * MU_ROWS;
  float pg[4 * HB], pb[4 * HB], pz[4 * HB], gam[4 * HB];
#pragma unroll
  for (int cb = 0; cb < HB; ++cb) {
    const float4 g4 = __ldg(reinterpret_cast<const float4*>(a.ln_w + 128 * cb + 4 * lane));
    gam[4 * cb] = g4.x; gam[4 * cb + 1] = g4.y; gam[4 * cb + 2] = g4.z; gam[4 * cb + 3] = g4.w;
  }
#pragma unroll
  for (int c = 0; c < 4 * HB; ++c) { pg[c] = 0.f; pb[c] = 0.f; pz[c] = 0.f; }
  for (int r = 0; r < 4; ++r) {
    const int g = row0 + 4 * wid + r;
    if (g >= a.n) break;                                   // warp-uniform
    float e[4 * HB], d[4 * HB];
    float s = 0.f;
#pragma unroll
    for (int cb = 0; cb < HB; ++cb) {
      const float4 e4 = *reinterpret_cast<const float4*>(a.pre + static_cast<size_t>(g) * H + 128 * cb + 4 * lane);
      const float4 d4 = *reinterpret_cast<const float4*>(a.dy + static_cast<size_t>(g) * H + 128 * cb + 4 * lane);
      e[4 * cb] = e4.x; e[4 * cb + 1] = e4.y; e[4 * cb + 2] = e4.z; e[4 * cb + 3] = e4.w;
      d[4 * cb] = d4.x; d[4 * cb + 1] = d4.y; d[4 * cb + 2] = d4.z; d[4 * cb + 3] = d4.w;
      s += (e4.x + e4.y) + (e4.z + e4.w);
    }
    s = spo_warp_sum(s);
    const float mean = s / static_cast<float>(H);
    float q = 0.f;
#pragma unroll
    for (int c = 0; c < 4 * HB; ++c) { const float t = e[c] - mean; q = fmaf(t, t, q); }
    q = spo_warp_sum(q);
    const float rstd = rsqrtf(q / static_cast<float>(H) + 1e-5f);     // same statistics as the forward (spo_ma.cu)
    float s1 = 0.f, s2 = 0.f;
    float xh[4 * HB];
#pragma unroll
    for (int c = 0; c < 4 * HB; ++c) {
      xh[c] = (e[c] - mean) * rstd;
      const float dx = d[c] * gam[c];
      s1 += dx;
      s2 = fmaf(dx, xh[c], s2);
    }
    s1 = spo_warp_sum(s1) / static_cast<float>(H);
    s2 = spo_warp_sum(s2) / static_cast<float>(H);
    float o[4 * HB];
#pragma unroll
    for (int c = 0; c < 4 * HB; ++c) {
      const float dx = d[c] * gam[c];
      const float dpre = rstd * (dx - s1 - xh[c] * s2);
      o[c] = dpre * (e[c] > 0.f ? 1.f : e[c] + 1.f);
      pg[c] = fmaf(d[c], xh[c], pg[c]);
      pb[c] += d[c];
      pz[c] += o[c];
    }
#pragma unroll
    for (int cb = 0; cb < HB; ++cb)
      *reinterpret_cast<float4*>(a.dz + static_cast<size_t>(g) * H + 128 * cb + 4 * lane) = make_float4(o[4 * cb], o[4 * cb + 1], o[4 * cb + 2], o[4 * cb + 3]);
  }
  // the eight warps add their column partials one after the other: a fixed order
  for (int w = 0; w < MU_THREADS / 32; ++w) {
    if (wid == w) {
#pragma unroll
      for (int cb = 0; cb < HB; ++cb)
#pragma unroll
        for (int e4 = 0; e4 < 4; ++e4) {
          const int c = 128 * cb + 4 * lane + e4;
          if (w == 0) { acc_s[0][c] = pg[4 * cb + e4]; acc_s[1][c] = pb[4 * cb + e4]; acc_s[2][c] = pz[4 * cb + e4]; }
          else { acc_s[0][c] += pg[4 * cb + e4]; acc_s[1][c] += pb[4 * cb + e4]; acc_s[2][c] += pz[4 * cb + e4]; }
        }
    }
    __syncthreads();
  }
  float* dst = a.part + static_cast<size_t>(blockIdx.x) * 3 * H;
  for (int i = tid; i < 3 * H; i += MU_THREADS) dst[i] = acc_s[i / H][i % H];
}

// ------------------------------------------------------------------------------------------------------------------
// Parameter gradients of the input LayerNorm (feature_norm, mlp.py:46-47): dxn = d loss / d LN(x)
//   part[blk][0][c] = sum_r dxn[r][c] * xhat[r][c],  part[blk][1][c] = sum_r dxn[r][c]   (no gradient flows into x itself)
// ------------------------------------------------------------------------------------------------------------------
struct LnInBwdArgs {
  const float *dxn, *x;
  float* part;
  int n, K;
};

__global__ void __launch_bounds__(MU_THREADS) ma_ln_in_bwd_kernel(const LnInBwdArgs a) {
  __shared__ float stat[MU_ROWS][2];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int row0 = blockIdx.x * MU_ROWS, K = a.K;
  for (int rr = 0; rr < 4; ++rr) {
    const int r = 4 * wid + rr, g = row0 + r;
    float s = 0.f;
    if (g < a.n)
      for (int k = lane; k < K; k += 32) s += a.x[static_cast<size_t>(g) * K + k];
    s = spo_warp_sum(s);
    const float mean = s / static_cast<float>(K);
    float v = 0.f;
    if (g < a.n)
      for (int k = lane; k < K; k += 32) { const float d = a.x[static_cast<size_t>(g) * K + k] - mean; v = fmaf(d, d, v); }
    v = spo_warp_sum(v);
    if (lane == 0) { stat[r][0] = mean; stat[r][1] = rsqrtf(v / static_cast<float>(K) + 1e-5f); }
  }
  __syncthreads();
  const int rows = min(MU_ROWS, a.n - row0);
  float* dst = a.part + static_cast<size_t>(blockIdx.x) * 2 * K;
  for (int c = tid; c < K; c += MU_THREADS) {
    float sg = 0.f, sb = 0.f;
    for (int r = 0; r < rows; ++r) {
      const size_t i = static_cast<size_t>(row0 + r) * K + c;
      const float d = a.dxn[i];
      sg = fmaf(d, (a.x[i] - stat[r][0]) * stat[r][1], sg);
      sb += d;
    }
    dst[c] = sg;
    dst[K + c] = sb;
  }
}

// out_s[j] = scale * sum_b part[b * stride + s * len + j]  for up to three segments s (out_s may be null): one thread per
// output, CTAs in order
struct ReduceArgs {
  const float* part;
  float* out[3];
  int nblk, stride, len, nseg;
  float scale;
};

__global__ void __launch_bounds__(256) ma_partial_reduce_kernel(const ReduceArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.nseg * a.len) return;
  const int s = i / a.len, j = i - s * a.len;
  if (!a.out[s]) return;
  float acc = 0.f;
  for (int b = 0; b < a.nblk; ++b) acc += a.part[static_cast<size_t>(b) * a.stride + i];
  a.out[s][j] = acc * a.scale;
}

// ------------------------------------------------------------------------------------------------------------------
// Tile products on the tensor pipe: mma.sync m16n8k8 TF32 with the 3xTF32 split in registers (spo_mma.cuh: lo*hi + hi*lo + hi*hi,
// small terms first -- fp32-grade results, ~1e-6 relative).  128 x 64 output tile, 32-deep chunks; warp w of 8 owns a 64 x 16 patch
// (4 x 2 mma tiles: 20 operand loads per 24 mma).  Both operand tiles are staged k-major with leading dimensions = 8 (mod 32), which
// makes the fragment loads of both operands bank-conflict free (the same rule as in spo_update.cu).
//   NN: C[M][N] = A[M][Kd] B[Kd][N]                         (dx = dz W;  d feat = d mean W_out)
//   TN: C[M][N] = sum_r A[r][M] B[r][N], r in the z-th slice of R rows -> part[z][M][N]   (dW = dz^T x)
// All operands row-major fp32; edges are guarded element-wise, no alignment requirement beyond 4 bytes.
// (The first version of these products was a 64 x 64 x 16 FFMA tile, 4 x 4 per thread: 16.5 TFLOP/s for a whole update.)
// ------------------------------------------------------------------------------------------------------------------
constexpr int GTM = 128, GTN = 64, GK = 32;
constexpr int LDA_S = GTM + 8, LDB_S = GTN + 8;

struct GemmArgs {
  const float *A, *B;
  float* C;
  int M, N, Kd;      // TN: Kd = R (rows reduced over), rows_per_slice = slice length
  int rows_per_slice;
};

__device__ __forceinline__ void tile_store(const float (&acc)[4][2][4], float* C, int M, int N, int m_base, int n_base) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int gm = m_base + 16 * mt + g + ((e >> 1) << 3), gn = n_base + 8 * nt + 2 * t + (e & 1);
        if (gm < M && gn < N) C[static_cast<size_t>(gm) * N + gn] = acc[mt][nt][e];
      }
}

__global__ void __launch_bounds__(256) ma_gemm_nn_kernel(const GemmArgs a) {
  __shared__ __align__(16) float As[GK * LDA_S];   // [k][m]
  __shared__ __align__(16) float Bs[GK * LDB_S];   // [k][n]
  const int tid = threadIdx.x, wid = tid >> 5;
  const int m0 = blockIdx.y * GTM, n0 = blockIdx.x * GTN;
  const int wm = (wid & 1) * 64, wn = (wid >> 1) * 16;
  float acc[4][2][4];
  spo_mma_zero<4>(acc);
  for (int k0 = 0; k0 < a.Kd; k0 += GK) {
    {   // A tile 128 x 32: thread -> row tid >> 1, sixteen consecutive k
      const int r = tid >> 1, kb = (tid & 1) * 16, gm = m0 + r;
      const float* src = a.A + static_cast<size_t>(gm) * a.Kd + k0 + kb;
#pragma unroll
      for (int e = 0; e < 16; ++e) As[(kb + e) * LDA_S + r] = (gm < a.M && k0 + kb + e < a.Kd) ? src[e] : 0.f;
    }
    {   // B tile 32 x 64: thread -> k rows tid >> 4 and + 16, four consecutive n
      const int kk = tid >> 4, cb = (tid & 15) * 4;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int gk = k0 + kk + 16 * h;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int gn = n0 + cb + e;
          Bs[(kk + 16 * h) * LDB_S + cb + e] = (gk < a.Kd && gn < a.N) ? a.B[static_cast<size_t>(gk) * a.N + gn] : 0.f;
        }
      }
    }
    __syncthreads();
    spo_warp_mma_3xtf32<4>(acc, As, 1, LDA_S, Bs, LDB_S, 1, wm, wn, GK);
    __syncthreads();
  }
  tile_store(acc, a.C, a.M, a.N, m0 + wm, n0 + wn);
}

__global__ void __launch_bounds__(256) ma_gemm_tn_kernel(const GemmArgs a) {
  __shared__ __align__(16) float As[GK * LDA_S];   // [r][m]
  __shared__ __align__(16) float Bs[GK * LDB_S];   // [r][n]
  const int tid = threadIdx.x, wid = tid >> 5;
  const int m0 = blockIdx.y * GTM, n0 = blockIdx.x * GTN;
  const int wm = (wid & 1) * 64, wn = (wid >> 1) * 16;
  const int r_begin = blockIdx.z * a.rows_per_slice;
  const int r_end = min(a.Kd, r_begin + a.rows_per_slice);
  float acc[4][2][4];
  spo_mma_zero<4>(acc);
  for (int r0 = r_begin; r0 < r_end; r0 += GK) {
    {   // A tile 32 x 128: thread -> rows tid >> 5 + 8 i, four consecutive m
      const int cb = (tid & 31) * 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int kk = (tid >> 5) + 8 * i, gr = r0 + kk;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int gm = m0 + cb + e;
          As[kk * LDA_S + cb + e] = (gr < r_end && gm < a.M) ? a.A[static_cast<size_t>(gr) * a.M + gm] : 0.f;
        }
      }
    }
    {   // B tile 32 x 64
      const int kk = tid >> 4, cb = (tid & 15) * 4;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int gr = r0 + kk + 16 * h;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int gn = n0 + cb + e;
          Bs[(kk + 16 * h) * LDB_S + cb + e] = (gr < r_end && gn < a.N) ? a.B[static_cast<size_t>(gr) * a.N + gn] : 0.f;
        }
      }
    }
    __syncthreads();
    spo_warp_mma_3xtf32<4>(acc, As, 1, LDA_S, Bs, LDB_S, 1, wm, wn, GK);
    __syncthreads();
  }
  tile_store(acc, a.C + static_cast<size_t>(blockIdx.z) * a.M * a.N, a.M, a.N, m0 + wm, n0 + wn);
}

// ------------------------------------------------------------------------------------------------------------------
// Actor head, loss and d loss / d mean (mappolag.py:147-166; distributions.py:8-9,38-42; act.py:45-60).  One warp per row
// (4 rows per warp, 32 per CTA); lane j < A owns action dimension j.
//   mean = feat W^T + b;  std = sigmoid(log_std / x) * y;  logp_j = -(a - mean)^2 / (2 std^2) - log std - log sqrt(2 pi)
//   imp = prod_j exp(logp_j - old_logp_j);  adv = adv_targ - lamda * cost_adv_targ
//   loss_row = -factor * min(imp * adv, clamp(imp, lo, hi) * adv);   policy_loss = mean_rows(loss_row)
//   d policy_loss / d logp_j = [imp * adv <= clamp(imp) * adv] * (-factor * adv / n) * imp       (the same for every j)
// part[blk] = { sum loss_row, 0, sum_r dmean_j (A), sum_r dstd_j (A) }   (2 + 2 * 32 floats per CTA)
// ------------------------------------------------------------------------------------------------------------------
constexpr int ACT_PART = 2 + 64;

struct ActorLossArgs {
  const float *feat, *W, *b, *log_std, *actions, *old_logp, *adv, *cost_adv, *factor, *lamda;
  float *dmean, *imp, *part;
  int n, H, A;
  float clip_lo, clip_hi, x_coef, y_coef;
};

__global__ void __launch_bounds__(MU_THREADS) ma_actor_loss_kernel(const ActorLossArgs a) {
  __shared__ float red[MU_THREADS / 32][ACT_PART];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int row0 = blockIdx.x * MU_ROWS, A = a.A, H = a.H;
  const float inv_n = __fdiv_rn(1.f, static_cast<float>(a.n));
  const float lam = *a.lamda;
  float std = 1.f, bj = 0.f;
  if (lane < A) {
    std = __fmul_rn(__fdiv_rn(1.f, 1.f + expf(-__fdiv_rn(a.log_std[lane], a.x_coef))), a.y_coef);   // as spo_ma_head_kernel
    bj = a.b[lane];
  }
  const float inv_var = __fdiv_rn(1.f, __fmul_rn(std, std)), log_std_v = logf(std);
  float sum_loss = 0.f, sum_dm = 0.f, sum_ds = 0.f;
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
    float imp = ratio;
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) imp *= __shfl_xor_sync(0xffffffffu, imp, m);
    const float adv = __fsub_rn(a.adv[g], __fmul_rn(lam, a.cost_adv[g]));
    const float fac = a.factor[g];
    const float s1 = __fmul_rn(imp, adv);
    const float s2 = __fmul_rn(fminf(fmaxf(imp, a.clip_lo), a.clip_hi), adv);
    const float gi = (s1 <= s2) ? -__fmul_rn(__fmul_rn(fac, adv), inv_n) : 0.f;
    const float crow = __fmul_rn(gi, imp);
    if (lane == 0) {
      a.imp[g] = imp;
      sum_loss += -__fmul_rn(fac, fminf(s1, s2));
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
  if (lane == 0) { red[wid][0] = sum_loss; red[wid][1] = 0.f; }
  red[wid][2 + lane] = sum_dm;
  red[wid][2 + 32 + lane] = sum_ds;
  __syncthreads();
  if (tid < ACT_PART) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < MU_THREADS / 32; ++w) s += red[w][tid];
    a.part[static_cast<size_t>(blockIdx.x) * ACT_PART + tid] = s;
  }
}

// one CTA: sums the actor partials over the CTAs in order and finishes the scalars and the small gradients
//   policy_loss = sum loss_row / n;   entropy = mean_j (0.5 + 0.5 log(2 pi) + log std_j)   (act.py:57-60: mean over [n][A])
//   g_b[j] = sum_r dmean_j;   g_log_std[j] = (sum_r dstd_j - entropy_coef / (A std_j)) * d std / d log_std
struct ActorFinalArgs {
  const float *part, *log_std;
  float *g_b, *g_log_std, *scalars;    // scalars[0] = policy_loss, [1] = dist_entropy
  int nblk, n, A;
  float x_coef, y_coef, entropy_coef;
};

__global__ void __launch_bounds__(128) ma_actor_final_kernel(const ActorFinalArgs a) {
  __shared__ float tot[ACT_PART];
  __shared__ float ent[32];
  const int tid = threadIdx.x;
  if (tid < ACT_PART) {
    float s = 0.f;
    for (int b = 0; b < a.nblk; ++b) s += a.part[static_cast<size_t>(b) * ACT_PART + tid];
    tot[tid] = s;
  }
  if (tid < 32) ent[tid] = 0.f;
  __syncthreads();
  if (tid < a.A) {
    const float sg = __fdiv_rn(1.f, 1.f + expf(-__fdiv_rn(a.log_std[tid], a.x_coef)));
    const float std = __fmul_rn(sg, a.y_coef);
    const float dstd_dls = __fdiv_rn(__fmul_rn(a.y_coef, __fmul_rn(sg, 1.f - sg)), a.x_coef);
    const float gs = tot[2 + 32 + tid] - __fdiv_rn(a.entropy_coef, __fmul_rn(static_cast<float>(a.A), std));
    a.g_log_std[tid] = __fmul_rn(gs, dstd_dls);
    a.g_b[tid] = tot[2 + tid];
    ent[tid] = 0.5f + kLogSqrt2Pi + logf(std);          // 0.5 + 0.5 log(2 pi) + log std
  }
  __syncthreads();
  if (tid == 0) {
    float e = 0.f;
    for (int j = 0; j < a.A; ++j) e += ent[j];
    a.scalars[0] = __fdiv_rn(tot[0], static_cast<float>(a.n));
    a.scalars[1] = __fdiv_rn(e, static_cast<float>(a.A));
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Value loss (mappolag.py:121-133 with use_clipped_value_loss, use_huber_loss; util.py:19-22):
//   vpc = vp + clamp(v - vp, -clip, clip);  ec = rn_c - vpc;  eo = rn_o - v;  L = mean(max(huber(eo), huber(ec)))
//   (rn_c, rn_o: the two PopArt normalisations of the returns -- the reference normalises twice and UPDATES the statistics both times)
//   huber(e) = e^2 / 2 for |e| <= d, d (|e| - d / 2) for e > d, 0 for e < -d (sic);  dv = scale * dL/dv, scale = value_loss_coef / n
// part[blk] = { sum L_row, sum dv }
// ------------------------------------------------------------------------------------------------------------------
struct ValueLossArgs {
  const float *v, *vp, *rn_c, *rn_o;
  float *dv, *part;
  int n;
  float clip, delta, scale;
};

__global__ void __launch_bounds__(256) ma_value_loss_kernel(const ValueLossArgs a) {
  __shared__ float red[8][2];
  const int i = blockIdx.x * 256 + threadIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float L = 0.f, dv = 0.f;
  if (i < a.n) {
    const float v = a.v[i], vp = a.vp[i];
    const float dlt = __fsub_rn(v, vp);
    const float vpc = __fadd_rn(vp, fminf(fmaxf(dlt, -a.clip), a.clip));
    const float ec = __fsub_rn(a.rn_c[i], vpc), eo = __fsub_rn(a.rn_o[i], v);
    const float hc = huber_val(ec, a.delta), ho = huber_val(eo, a.delta);
    L = fmaxf(ho, hc);
    const float wo = (ho > hc) ? 1.f : (ho == hc ? 0.5f : 0.f);
    const float inr = (dlt >= -a.clip && dlt <= a.clip) ? 1.f : 0.f;
    dv = a.scale * (wo * (-huber_grad(eo, a.delta)) + (1.f - wo) * inr * (-huber_grad(ec, a.delta)));
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

// ------------------------------------------------------------------------------------------------------------------
// PopArt.forward on a [n] batch (popart.py:76-112 with norm_axes 1, one output): update the running statistics with the
// batch moments, then normalise.  state = {running_mean, running_mean_sq, debiasing_term}.  One CTA.
// ------------------------------------------------------------------------------------------------------------------
struct PopArtArgs {
  const float* x;
  float *state, *out;
  int n;
  float w, one_minus_w, eps;
};

__global__ void __launch_bounds__(1024) ma_popart_kernel(const PopArtArgs a) {
  __shared__ float red[32][2];
  __shared__ float mv[2];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  float s = 0.f, q = 0.f;
  for (int i = tid; i < a.n; i += 1024) { const float v = a.x[i]; s += v; q = fmaf(v, v, q); }
  s = spo_warp_sum(s);
  q = spo_warp_sum(q);
  if (lane == 0) { red[wid][0] = s; red[wid][1] = q; }
  __syncthreads();
  if (tid == 0) {
    float ts = 0.f, tq = 0.f;
    for (int w = 0; w < 32; ++w) { ts += red[w][0]; tq += red[w][1]; }
    const float bm = __fdiv_rn(ts, static_cast<float>(a.n)), bq = __fdiv_rn(tq, static_cast<float>(a.n));
    const float rm = __fadd_rn(__fmul_rn(a.state[0], a.w), __fmul_rn(bm, a.one_minus_w));
    const float rq = __fadd_rn(__fmul_rn(a.state[1], a.w), __fmul_rn(bq, a.one_minus_w));
    const float db = __fadd_rn(__fmul_rn(a.state[2], a.w), a.one_minus_w);
    a.state[0] = rm; a.state[1] = rq; a.state[2] = db;
    const float den = fmaxf(db, a.eps);
    const float mean = __fdiv_rn(rm, den), msq = __fdiv_rn(rq, den);
    mv[0] = mean;
    mv[1] = sqrtf(fmaxf(__fsub_rn(msq, __fmul_rn(mean, mean)), 1e-2f));
  }
  __syncthreads();
  const float mean = mv[0], sd = mv[1];
  for (int i = tid; i < a.n; i += 1024) a.out[i] = __fdiv_rn(__fsub_rn(a.x[i], mean), sd);
}

// ------------------------------------------------------------------------------------------------------------------
// Lagrange multiplier step (mappolag.py:169-172): delta = -((mean(aver_episode_costs) - cost_limit) (1 - gamma) + imp * cost_adv).mean()
//   lamda <- relu(lamda - delta * rate).  One CTA.
// ------------------------------------------------------------------------------------------------------------------
struct LagrArgs {
  const float *imp, *cost_adv, *aver_costs;
  float* lamda;
  int n;
  float cost_limit, one_minus_gamma, rate;
};

__global__ void __launch_bounds__(1024) ma_lagrange_kernel(const LagrArgs a) {
  __shared__ float red[32][2];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  float s = 0.f, c = 0.f;
  for (int i = tid; i < a.n; i += 1024) { s = fmaf(a.imp[i], a.cost_adv[i], s); c += a.aver_costs[i]; }
  s = spo_warp_sum(s);
  c = spo_warp_sum(c);
  if (lane == 0) { red[wid][0] = s; red[wid][1] = c; }
  __syncthreads();
  if (tid == 0) {
    float ts = 0.f, tc = 0.f;
    for (int w = 0; w < 32; ++w) { ts += red[w][0]; tc += red[w][1]; }
    const float nf = static_cast<float>(a.n);
    const float c0 = __fmul_rn(__fsub_rn(__fdiv_rn(tc, nf), a.cost_limit), a.one_minus_gamma);
    const float delta = -__fadd_rn(c0, __fdiv_rn(ts, nf));
    *a.lamda = fmaxf(__fsub_rn(*a.lamda, __fmul_rn(delta, a.rate)), 0.f);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// clip_grad_norm_ + Adam on a packed parameter buffer (torch.optim.Adam single-tensor path; weight_decay adds wd * p to the
// gradient first).  Stage 1: per-CTA sums of squares; stage 2 (one CTA): norm -> out, clip coefficient; stage 3: the update.
// ------------------------------------------------------------------------------------------------------------------
struct SumsqArgs {
  const float* g;
  float* part;
  int count;
};

__global__ void __launch_bounds__(256) ma_sumsq_kernel(const SumsqArgs a) {
  __shared__ float red[8];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float s = 0.f;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < a.count; i += gridDim.x * 256) { const float v = a.g[i]; s = fmaf(v, v, s); }
  s = spo_warp_sum(s);
  if (lane == 0) red[wid] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w];
    a.part[blockIdx.x] = t;
  }
}

struct NormArgs {
  const float* part;
  float* norm_coef;     // [0] = total norm, [1] = clip coefficient min(max_norm / (norm + 1e-6), 1)
  int nblk;
  float max_norm;
};

__global__ void ma_norm_kernel(const NormArgs a) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    float t = 0.f;
    for (int b = 0; b < a.nblk; ++b) t += a.part[b];
    const float norm = sqrtf(t);
    a.norm_coef[0] = norm;
    a.norm_coef[1] = fminf(__fdiv_rn(a.max_norm, __fadd_rn(norm, 1e-6f)), 1.f);
  }
}

struct AdamArgs {
  float *p, *m, *v;
  const float *g, *norm_coef;
  int count;
  float w1, b2, w2, bc2_sqrt, eps, step_size, wd;    // w1 = 1 - beta1, w2 = 1 - beta2, step_size = lr / (1 - beta1^t)
};

__global__ void __launch_bounds__(256) ma_adam_kernel(const AdamArgs a) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= a.count) return;
  const float coef = a.norm_coef[1];
  const float p = a.p[i];
  float g = __fmul_rn(a.g[i], coef);
  if (a.wd != 0.f) g = fmaf(a.wd, p, g);
  float m = a.m[i], v = a.v[i];
  m = fmaf(a.w1, __fsub_rn(g, m), m);                                           // exp_avg.lerp_(grad, 1 - beta1)
  v = __fadd_rn(__fmul_rn(v, a.b2), __fmul_rn(__fmul_rn(a.w2, g), g));          // mul_(beta2).addcmul_(grad, grad, 1 - beta2)
  const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), a.bc2_sqrt), a.eps);
  a.p[i] = __fadd_rn(p, __fdiv_rn(__fmul_rn(-a.step_size, m), denom));     // addcdiv_(exp_avg, denom, value=-step_size)
  a.m[i] = m;
  a.v[i] = v;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" {

int spo_ma_ln_elu_bwd(const float* dy, const float* pre, const float* ln_w, int n, int H, float* dz, float* part, void* stream) {
  SPO_REQUIRE(dy && pre && ln_w && dz && part && n > 0, SPO_ERR_INVALID_ARG, "spo_ma_ln_elu_bwd: null argument or n<=0");
  SPO_REQUIRE(H >= 128 && H <= 512 && (H & 127) == 0, SPO_ERR_UNSUPPORTED, "spo_ma_ln_elu_bwd: H=%d must be a multiple of 128 up to 512", H);
  SPO_REQUIRE(aligned16(dy) && aligned16(pre) && aligned16(ln_w) && aligned16(dz), SPO_ERR_INVALID_ARG, "spo_ma_ln_elu_bwd: 16-byte alignment required");
  LnEluBwdArgs a{dy, pre, ln_w, dz, part, n, H};
  const int grid = (n + MU_ROWS - 1) / MU_ROWS;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (H / 128) {
    case 1: ma_ln_elu_bwd_kernel<1><<<grid, MU_THREADS, 0, st>>>(a); break;
    case 2: ma_ln_elu_bwd_kernel<2><<<grid, MU_THREADS, 0, st>>>(a); break;
    case 3: ma_ln_elu_bwd_kernel<3><<<grid, MU_THREADS, 0, st>>>(a); break;
    default: ma_ln_elu_bwd_kernel<4><<<grid, MU_THREADS, 0, st>>>(a); break;
  }
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_ln_in_bwd(const float* dxn, const float* x, int n, int K, float* part, void* stream) {
  SPO_REQUIRE(dxn && x && part && n > 0 && K > 0, SPO_ERR_INVALID_ARG, "spo_ma_ln_in_bwd: null argument or empty shape");
  LnInBwdArgs a{dxn, x, part, n, K};
  ma_ln_in_bwd_kernel<<<(n + MU_ROWS - 1) / MU_ROWS, MU_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_partial_reduce(const float* part, int nblk, int stride, int nseg, int len, float* out0, float* out1, float* out2, float scale,
                          void* stream) {
  SPO_REQUIRE(part && nblk > 0 && nseg >= 1 && nseg <= 3 && len > 0 && stride >= nseg * len, SPO_ERR_INVALID_ARG,
              "spo_ma_partial_reduce: bad shape (nblk=%d stride=%d nseg=%d len=%d)", nblk, stride, nseg, len);
  ReduceArgs a{part, {out0, out1, out2}, nblk, stride, len, nseg, scale};
  ma_partial_reduce_kernel<<<(nseg * len + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_gemm_nn(const float* A, const float* B, float* C, int M, int N, int Kd, void* stream) {
  SPO_REQUIRE(A && B && C && M > 0 && N > 0 && Kd > 0, SPO_ERR_INVALID_ARG, "spo_ma_gemm_nn: null argument or empty shape");
  GemmArgs a{A, B, C, M, N, Kd, 0};
  dim3 grid((N + GTN - 1) / GTN, (M + GTM - 1) / GTM, 1);
  SPO_REQUIRE(grid.y <= 65535, SPO_ERR_UNSUPPORTED, "spo_ma_gemm_nn: M=%d too large", M);
  ma_gemm_nn_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_gemm_tn(const float* A, const float* B, float* part, int R, int M, int N, int slices, void* stream) {
  SPO_REQUIRE(A && B && part && R > 0 && M > 0 && N > 0 && slices >= 1 && slices <= 1024, SPO_ERR_INVALID_ARG,
              "spo_ma_gemm_tn: null argument or bad shape");
  const int rps = ((R + slices - 1) / slices + GK - 1) / GK * GK;
  SPO_REQUIRE(static_cast<long long>(rps) * (slices - 1) < R, SPO_ERR_INVALID_ARG, "spo_ma_gemm_tn: %d slices leave an empty slice for R=%d", slices, R);
  GemmArgs a{A, B, part, M, N, R, rps};
  dim3 grid((N + GTN - 1) / GTN, (M + GTM - 1) / GTM, slices);
  ma_gemm_tn_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_actor_loss(const float* feat, int n, int H, const float* W, const float* b, const float* log_std, int A, const float* actions,
                      const float* old_logp, const float* adv, const float* cost_adv, const float* factor, const float* lamda,
                      float clip_lo, float clip_hi, float std_x_coef, float std_y_coef, float* dmean, float* imp, float* part, void* stream) {
  SPO_REQUIRE(feat && W && b && log_std && actions && old_logp && adv && cost_adv && factor && lamda && dmean && imp && part && n > 0 && H > 0,
              SPO_ERR_INVALID_ARG, "spo_ma_actor_loss: null argument or empty shape");
  SPO_REQUIRE(A >= 1 && A <= 32, SPO_ERR_UNSUPPORTED, "spo_ma_actor_loss: act_dim=%d must be in 1..32", A);
  ActorLossArgs a{feat, W, b, log_std, actions, old_logp, adv, cost_adv, factor, lamda, dmean, imp, part, n, H, A, clip_lo, clip_hi, std_x_coef, std_y_coef};
  ma_actor_loss_kernel<<<(n + MU_ROWS - 1) / MU_ROWS, MU_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_actor_finalize(const float* part, int nblk, int n, const float* log_std, int A, float std_x_coef, float std_y_coef, float entropy_coef,
                          float* g_b, float* g_log_std, float* scalars, void* stream) {
  SPO_REQUIRE(part && log_std && g_b && g_log_std && scalars && nblk > 0 && n > 0 && A >= 1 && A <= 32, SPO_ERR_INVALID_ARG,
              "spo_ma_actor_finalize: null argument or bad shape");
  ActorFinalArgs a{part, log_std, g_b, g_log_std, scalars, nblk, n, A, std_x_coef, std_y_coef, entropy_coef};
  ma_actor_final_kernel<<<1, 128, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_value_loss(const float* v, const float* value_preds, const float* ret_norm_clipped, const float* ret_norm_orig, int n, float clip,
                      float huber_delta, float scale, float* dv, float* part, void* stream) {
  SPO_REQUIRE(v && value_preds && ret_norm_clipped && ret_norm_orig && dv && part && n > 0, SPO_ERR_INVALID_ARG,
              "spo_ma_value_loss: null argument or n<=0");
  ValueLossArgs a{v, value_preds, ret_norm_clipped, ret_norm_orig, dv, part, n, clip, huber_delta, scale};
  ma_value_loss_kernel<<<(n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_popart_normalize(const float* x, int n, float* state, double beta, float epsilon, float* out, void* stream) {
  SPO_REQUIRE(x && state && out && n > 0, SPO_ERR_INVALID_ARG, "spo_ma_popart_normalize: null argument or n<=0");
  // weight and (1.0 - weight) are Python floats in popart.py:92-100; each is rounded to fp32 once where it meets a tensor
  PopArtArgs a{x, state, out, n, static_cast<float>(beta), static_cast<float>(1.0 - beta), epsilon};
  ma_popart_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_lagrange_step(const float* imp, const float* cost_adv, const float* aver_episode_costs, int n, float cost_limit, double gamma,
                         float rate, float* lamda, void* stream) {
  SPO_REQUIRE(imp && cost_adv && aver_episode_costs && lamda && n > 0, SPO_ERR_INVALID_ARG, "spo_ma_lagrange_step: null argument or n<=0");
  LagrArgs a{imp, cost_adv, aver_episode_costs, lamda, n, cost_limit, static_cast<float>(1.0 - gamma), rate};
  ma_lagrange_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_clip_adam(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int count, float max_grad_norm, double lr, double beta1,
                     double beta2, double eps, double weight_decay, int step, float* work, float* norm_out, void* stream) {
  SPO_REQUIRE(params && grads && exp_avg && exp_avg_sq && work && norm_out && count > 0 && step >= 1, SPO_ERR_INVALID_ARG,
              "spo_ma_clip_adam: null argument, count<=0 or step<1");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nblk = min(1024, (count + 255) / 256);
  ma_sumsq_kernel<<<nblk, 256, 0, st>>>(SumsqArgs{grads, work, count});
  ma_norm_kernel<<<1, 32, 0, st>>>(NormArgs{work, norm_out, nblk, max_grad_norm});
  // the scalar factors as torch's Python floats compute them (float64), rounded once
  const double bc1 = 1.0 - pow(beta1, step), bc2 = 1.0 - pow(beta2, step);
  AdamArgs a{params, exp_avg, exp_avg_sq, grads, norm_out, count,
             static_cast<float>(1.0 - beta1), static_cast<float>(beta2), static_cast<float>(1.0 - beta2),
             static_cast<float>(sqrt(bc2)), static_cast<float>(eps), static_cast<float>(lr / bc1), static_cast<float>(weight_decay)};
  ma_adam_kernel<<<(count + 255) / 256, 256, 0, st>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

}  // extern "C"
