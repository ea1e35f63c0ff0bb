// Multi-agent trust-region step (MACPO, safepo/multi_agent/macpo.py:153-380): the Fisher-vector product of the LayerNorm/ELU
// actor, the ratio surrogate head, the conjugate-gradient vector steps, the step direction and the line-search evaluation.
//
// Fisher-vector product.  F is the Hessian of mean_rows(sum_j KL_j(old || new)) at new = old (macpo.py:153-166,187-198).  There
// dKL/dmean is exactly 0, so the mean block is Gauss-Newton: F_mean v = J^T W J v with J = d mean / d params and the per-dimension
// weight W_j = 2 / (1e-8 + 2 std_j^2) / n.  J v is a forward-mode pass through the net (spo_ma_mlp_layer_jvp per block,
// spo_ma_head_jvp for the mean layer, which also applies W); J^T is the existing backward chain (spo_ma_gemm_tn / _nn,
// spo_ma_ln_elu_bwd, spo_ma_ln_in_bwd).  The log_std block is diagonal and closed-form (spo_ma_fvp_finalize); the mixed
// mean / log_std block is zero at new = old.
//
// Vector kernels (CG, dots, step, line search) run over the net's packed parameter buffer, zero padding included: every
// element-wise update maps 0 to 0 on the padding, so it stays exactly 0.  Their sums are deterministic: a fixed grid of
// VCTAS = 256 CTAs, a fixed-order block reduction per CTA, and the last CTA to finish sums the per-CTA partials in CTA order.
#include "spo_ma_math.cuh"

namespace {

constexpr int VT = 256;            // threads of the vector kernels
constexpr int VCTAS = 256;         // fixed grid of the vector reductions: results do not depend on the device
constexpr int VMAXS = 4;           // sums per reduction

// block sum (fixed order); the result is valid in thread 0
__device__ __forceinline__ float block_sum(float v, float* sh) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  v = spo_warp_sum(v);
  __syncthreads();
  if (lane == 0) sh[wid] = v;
  __syncthreads();
  if (wid == 0) {
    v = lane < (blockDim.x >> 5) ? sh[lane] : 0.f;
    v = spo_warp_sum(v);
  }
  return v;
}

// Two-stage deterministic reduction of S sums: every CTA stores its partials, the last CTA to arrive adds them in CTA order.
// Returns true in the last CTA, where tot[0..S) holds the totals (in shared memory, valid after the call in every thread).
template <int S>
__device__ bool grid_reduce(float (&v)[S], float* work, float* tot) {
  __shared__ float sh[32];
  __shared__ bool last;
  float* part = work;
  unsigned* counter = reinterpret_cast<unsigned*>(work + VCTAS * VMAXS);
#pragma unroll
  for (int s = 0; s < S; ++s) {
    const float b = block_sum(v[s], sh);
    if (threadIdx.x == 0) part[blockIdx.x * VMAXS + s] = b;
  }
  if (threadIdx.x == 0) {
    __threadfence();
    last = atomicAdd(counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return false;
  __threadfence();
#pragma unroll
  for (int s = 0; s < S; ++s) {
    const float x = threadIdx.x < gridDim.x ? __ldcg(part + threadIdx.x * VMAXS + s) : 0.f;
    const float b = block_sum(x, sh);
    if (threadIdx.x == 0) tot[s] = b;
  }
  if (threadIdx.x == 0) *counter = 0u;
  __syncthreads();
  return true;
}

int vec_grid(long long count) { return static_cast<int>(std::min<long long>(VCTAS, (count + VT - 1) / VT)); }

// ---------------- forward-mode tangent of one [Linear -> ELU -> LayerNorm] block ----------------
struct MaJvpArgs {
  const float *in, *din;                       // [n][K] block input and its tangent (din unused with the input LayerNorm)
  const float *W, *dW, *db;                    // [H][K], [H][K], [H]
  const float *pre, *ln_w, *dln_w, *dln_b;     // saved ELU output [n][H]; output LayerNorm weight and the tangents of its affine
  const float *lin_w, *lin_b, *dlin_w, *dlin_b;  // input LayerNorm (feature_norm) and its tangents, or null
  float* dout;                                 // [n][H]
  int n, K, H;
};

// dz = dx W^T + x dW^T + db as ONE K loop over both products (chunks 0..nk-1: the tangent input against W, nk..2nk-1: the input
// against dW), then ELU' from the saved ELU output (h > 0 -> 1, else h + 1 = exp(z)) and the LayerNorm tangent with the forward's
// row statistics of `pre` (ma_row_ln_stats):  dout = g * rstd (dh - mean(dh) - hn mean(dh hn)) + dg hn + dbeta,  hn = (h - mean) rstd.
template <int HB>
__global__ void __launch_bounds__(MA_THREADS) spo_ma_layer_jvp_kernel(const MaJvpArgs a) {
  extern __shared__ __align__(16) float smem[];
  constexpr int H = 128 * HB;
  float* Wc = smem;                            // [MA_KC][H]
  float* xs = Wc + MA_KC * H;                  // [MA_ROWS][MA_KC + 4]
  float* stat = xs + MA_ROWS * (MA_KC + 4);    // [MA_ROWS][2]
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int row0 = blockIdx.x * MA_ROWS;
  const int K = a.K;

  if (a.lin_w) ma_input_ln_stats(a.in, a.n, K, row0, wid, lane, stat);
  __syncthreads();

  float acc[4][4 * HB];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4 * HB; ++c) acc[r][c] = 0.f;

  const int nk = (K + MA_KC - 1) / MA_KC;
  for (int c = 0; c < 2 * nk; ++c) {
    const bool tang = c < nk;
    const int k0 = (tang ? c : c - nk) * MA_KC;
    ma_stage_w_chunk<HB>(tang ? a.W : a.dW, K, k0, Wc, tid);
    {
      const int r = tid >> 3, kk = (tid & 7) * 2, g = row0 + r;
      float2 v = make_float2(0.f, 0.f);
      if (g < a.n && k0 + kk < K) {
        if (a.lin_w) {
          const float2 x = __ldg(reinterpret_cast<const float2*>(a.in + static_cast<size_t>(g) * K + k0 + kk));
          const float mean = stat[2 * r], rstd = stat[2 * r + 1];
          const float h0 = (x.x - mean) * rstd, h1 = (x.y - mean) * rstd;
          const float* sw = tang ? a.dlin_w : a.lin_w;
          const float* sb = tang ? a.dlin_b : a.lin_b;
          v.x = fmaf(h0, sw[k0 + kk], sb[k0 + kk]);
          v.y = fmaf(h1, sw[k0 + kk + 1], sb[k0 + kk + 1]);
        } else {
          v = __ldg(reinterpret_cast<const float2*>((tang ? a.din : a.in) + static_cast<size_t>(g) * K + k0 + kk));
        }
      }
      xs[r * (MA_KC + 4) + kk] = v.x;
      xs[r * (MA_KC + 4) + kk + 1] = v.y;
    }
    __syncthreads();
#pragma unroll
    for (int kq = 0; kq < MA_KC; kq += 4) {
      float4 xv[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) xv[r] = *reinterpret_cast<const float4*>(xs + (4 * wid + r) * (MA_KC + 4) + kq);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int cb = 0; cb < HB; ++cb) {
          const float4 wv = *reinterpret_cast<const float4*>(Wc + (kq + kk) * H + 128 * cb + 4 * lane);
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const float xk = (kk == 0) ? xv[r].x : (kk == 1) ? xv[r].y : (kk == 2) ? xv[r].z : xv[r].w;
            acc[r][4 * cb + 0] = fmaf(xk, wv.x, acc[r][4 * cb + 0]);
            acc[r][4 * cb + 1] = fmaf(xk, wv.y, acc[r][4 * cb + 1]);
            acc[r][4 * cb + 2] = fmaf(xk, wv.z, acc[r][4 * cb + 2]);
            acc[r][4 * cb + 3] = fmaf(xk, wv.w, acc[r][4 * cb + 3]);
          }
        }
      }
    }
    __syncthreads();
  }

  const float invH = 1.f / static_cast<float>(H);
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int g = row0 + 4 * wid + r;          // the whole warp shares g: the warp sums below are safe for g >= n
    float h[4 * HB];
#pragma unroll
    for (int cb = 0; cb < HB; ++cb) {
      float4 pv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (g < a.n) pv = __ldg(reinterpret_cast<const float4*>(a.pre + static_cast<size_t>(g) * H + 128 * cb + 4 * lane));
      h[4 * cb] = pv.x; h[4 * cb + 1] = pv.y; h[4 * cb + 2] = pv.z; h[4 * cb + 3] = pv.w;
    }
    float mean, rstd;
    ma_row_ln_stats<HB>(h, mean, rstd);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int cb = 0; cb < HB; ++cb) {
      const float4 bv = __ldg(reinterpret_cast<const float4*>(a.db + 128 * cb + 4 * lane));
      const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = 4 * cb + e;
        const float dh = (acc[r][c] + bb[e]) * (h[c] > 0.f ? 1.f : h[c] + 1.f);
        acc[r][c] = dh;
        h[c] = (h[c] - mean) * rstd;           // hn from here on
        s1 += dh;
        s2 = fmaf(dh, h[c], s2);
      }
    }
    const float m1 = spo_warp_sum(s1) * invH, m2 = spo_warp_sum(s2) * invH;
    if (g < a.n) {
#pragma unroll
      for (int cb = 0; cb < HB; ++cb) {
        const int col = 128 * cb + 4 * lane;
        const float4 gw = __ldg(reinterpret_cast<const float4*>(a.ln_w + col));
        const float4 dg = __ldg(reinterpret_cast<const float4*>(a.dln_w + col));
        const float4 dbt = __ldg(reinterpret_cast<const float4*>(a.dln_b + col));
        const float gg[4] = {gw.x, gw.y, gw.z, gw.w}, dgg[4] = {dg.x, dg.y, dg.z, dg.w}, dbb[4] = {dbt.x, dbt.y, dbt.z, dbt.w};
        float o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int c = 4 * cb + e;
          const float dhn = rstd * (acc[r][c] - m1 - h[c] * m2);
          o[e] = fmaf(gg[e], dhn, fmaf(dgg[e], h[c], dbb[e]));
        }
        *reinterpret_cast<float4*>(a.dout + static_cast<size_t>(g) * H + col) = make_float4(o[0], o[1], o[2], o[3]);
      }
    }
  }
}

// ---------------- mean-layer tangent with the Fisher weight ----------------
struct MaHeadJvpArgs {
  const float *feat, *dfeat, *W, *dW, *db, *log_std;   // [n][H] x2, [A][H] x2, [A], [A]
  float *dmean, *part;                                 // [n][A]; [ceil(n/32)][A] column sums of dmean
  int n, H, A;
  float x_coef, y_coef;
};

// a CTA owns 32 rows (4 per warp): dmean[r][o] = w_o (dfeat W^T + feat dW^T + db)[r][o], w_o = 2 / (1e-8 + 2 std_o^2) / n
__global__ void __launch_bounds__(256) spo_ma_head_jvp_kernel(const MaHeadJvpArgs a) {
  __shared__ float sm[32][33];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int rr = 0; rr < 4; ++rr) {
    const int r = 4 * wid + rr, row = blockIdx.x * 32 + r;
    for (int o = 0; o < a.A; ++o) {
      float s = 0.f;
      if (row < a.n) {
        const float* f = a.feat + static_cast<size_t>(row) * a.H;
        const float* df = a.dfeat + static_cast<size_t>(row) * a.H;
        for (int k = lane; k < a.H; k += 32)
          s = fmaf(df[k], __ldg(a.W + o * a.H + k), fmaf(f[k], __ldg(a.dW + o * a.H + k), s));
      }
      s = spo_warp_sum(s);
      if (lane == 0) {
        float v = 0.f;
        if (row < a.n) {
          const float sd = ma_std(a.log_std[o], a.x_coef, a.y_coef);
          const float w = __fdiv_rn(__fdiv_rn(2.f, 1e-8f + 2.f * sd * sd), static_cast<float>(a.n));
          v = w * (s + a.db[o]);
          a.dmean[static_cast<size_t>(row) * a.A + o] = v;
        }
        sm[r][o] = v;
      }
    }
  }
  __syncthreads();
  if (threadIdx.x < a.A) {
    float s = 0.f;
    for (int r = 0; r < 32; ++r) s += sm[r][threadIdx.x];
    a.part[static_cast<size_t>(blockIdx.x) * a.A + threadIdx.x] = s;
  }
}

// ---------------- closed-form log_std block + damping ----------------
// Per dimension, with s = std(log_std), s0 = s^2 at new = old, D = 1e-8 + 2 s^2:  KL_j = log s_old - log s + s0 / D - 1/2,
//   f'(s) = -1/s - 4 s s0 / D^2,   f''(s) = 1/s^2 - 4 s0 / D^2 + 32 s^2 s0 / D^3,
//   s' = y sg (1 - sg) / x,   s'' = y sg (1 - sg)(1 - 2 sg) / x^2,   d^2 KL_j / d log_std_j^2 = f'' s'^2 + f' s''.
// The reference's log terms enter with the sign opposite to KL(old || new)'s, so f'(s_old) = -2 / s (up to the 1e-8) is not 0 and
// the s'' term stays.  Evaluated in double.
__device__ double ma_logstd_curv(float log_std, float x_coef, float y_coef) {
  const double x = x_coef, y = y_coef;
  const double sg = 1.0 / (1.0 + exp(-static_cast<double>(log_std) / x));
  const double s = y * sg, s0 = s * s, D = 1e-8 + 2.0 * s0;
  const double f1 = -1.0 / s - 4.0 * s * s0 / (D * D);
  const double f2 = 1.0 / s0 - 4.0 * s0 / (D * D) + 32.0 * s0 * s0 / (D * D * D);
  const double d1 = y * sg * (1.0 - sg) / x, d2 = y * sg * (1.0 - sg) * (1.0 - 2.0 * sg) / (x * x);
  return f2 * d1 * d1 + f1 * d2;
}

__global__ void __launch_bounds__(VT) spo_ma_fvp_finalize_kernel(const float* __restrict__ gn, const float* __restrict__ v, float* __restrict__ out,
                                                                 int P, const float* __restrict__ log_std, int ls_off, int A, float x_coef,
                                                                 float y_coef, float damping) {
  for (int i = blockIdx.x * VT + threadIdx.x; i < P; i += gridDim.x * VT) {
    const float vi = v[i];
    const int j = i - ls_off;
    float f;
    if (j >= 0 && j < A) f = static_cast<float>(ma_logstd_curv(log_std[j], x_coef, y_coef) * static_cast<double>(vi));
    else f = gn[i];
    out[i] = __fadd_rn(f, __fmul_rn(damping, vi));
  }
}

// ---------------- ratio surrogate head ----------------
// One warp per 32 rows, lane = row.  ratio = prod_j exp(logp_j - old_logp_j);  loss = sign * mean(ratio * factor * adv);
// dmean[n][A] = d loss / d mean;  part[blk][3][A] = {sum ratio*factor*adv (at [0]), sum dmean_j, sum d loss / d log_std_j}.
__global__ void __launch_bounds__(32) spo_ma_ratio_loss_kernel(const float* __restrict__ mean, int n, const float* __restrict__ log_std, int A,
                                                               const float* __restrict__ actions, const float* __restrict__ old_logp,
                                                               const float* __restrict__ adv, const float* __restrict__ factor, float sign,
                                                               float x_coef, float y_coef, float* __restrict__ dmean, float* __restrict__ part) {
  const int lane = threadIdx.x, row = blockIdx.x * 32 + lane;
  const bool ok = row < n;
  float ratio = 1.f;
  if (ok)
    for (int j = 0; j < A; ++j) {
      const float sd = ma_std(log_std[j], x_coef, y_coef);
      const float diff = __fsub_rn(actions[static_cast<size_t>(row) * A + j], mean[static_cast<size_t>(row) * A + j]);
      const float lp = ma_gauss_logp(diff, sd, logf(sd));
      ratio = __fmul_rn(ratio, expf(__fsub_rn(lp, old_logp[static_cast<size_t>(row) * A + j])));
    }
  const float fa = ok ? __fmul_rn(factor[row], adv[row]) : 0.f;
  const float term = ok ? __fmul_rn(ratio, fa) : 0.f;
  const float c = sign * term / static_cast<float>(n);     // d loss / d logp_j of this row
  float* pb = part + static_cast<size_t>(blockIdx.x) * 3 * A;
  const float tsum = spo_warp_sum(term);
  if (lane == 0) pb[0] = tsum;
  for (int j = 0; j < A; ++j) {
    float dm = 0.f, ds = 0.f;
    if (ok) {
      const float lsj = log_std[j];
      const float sd = ma_std(lsj, x_coef, y_coef);
      const float sg = 1.f / (1.f + expf(-lsj / x_coef));
      const float diff = actions[static_cast<size_t>(row) * A + j] - mean[static_cast<size_t>(row) * A + j];
      dm = c * diff / (sd * sd);
      ds = c * (diff * diff / (sd * sd * sd) - 1.f / sd) * (y_coef * sg * (1.f - sg) / x_coef);
      dmean[static_cast<size_t>(row) * A + j] = dm;
    }
    dm = spo_warp_sum(dm);
    ds = spo_warp_sum(ds);
    if (lane == 0) {
      if (j > 0) pb[j] = 0.f;
      pb[A + j] = dm;
      pb[2 * A + j] = ds;
    }
  }
}

// ---------------- vector kernels ----------------
struct Dots { const float* a[VMAXS]; const float* b[VMAXS]; };

template <int S>
__global__ void __launch_bounds__(VT) spo_ma_dots_kernel(const Dots d, int P, float* work, float* out) {
  __shared__ float tot[VMAXS];
  float v[S];
#pragma unroll
  for (int s = 0; s < S; ++s) v[s] = 0.f;
  for (int i = blockIdx.x * VT + threadIdx.x; i < P; i += gridDim.x * VT)
#pragma unroll
    for (int s = 0; s < S; ++s) v[s] = fmaf(d.a[s][i], d.b[s][i], v[s]);
  if (grid_reduce<S>(v, work, tot) && threadIdx.x < S) out[threadIdx.x] = tot[threadIdx.x];
}

// state = {rdotr, p.Ap, beta, done}
__global__ void __launch_bounds__(VT) spo_ma_cg_begin_kernel(const float* __restrict__ b, float* __restrict__ x, float* __restrict__ r,
                                                             float* __restrict__ p, int P, float* work, float* state) {
  __shared__ float tot[VMAXS];
  float v[1] = {0.f};
  for (int i = blockIdx.x * VT + threadIdx.x; i < P; i += gridDim.x * VT) {
    const float bi = b[i];
    x[i] = 0.f; r[i] = bi; p[i] = bi;
    v[0] = fmaf(bi, bi, v[0]);
  }
  if (grid_reduce<1>(v, work, tot) && threadIdx.x == 0) { state[0] = tot[0]; state[1] = 0.f; state[2] = 0.f; state[3] = 0.f; }
}

// MACPO's CG step (macpo.py:168-185): alpha = rdotr / (p.Ap + 1e-8), x += alpha p, r -= alpha Ap, beta = r.r / rdotr (no eps),
// stop once the NEW rdotr < residual_tol (rdotr itself, not its square root).  A stopped solve leaves x, r, p untouched.
__global__ void __launch_bounds__(VT) spo_ma_cg_update_kernel(float* __restrict__ x, float* __restrict__ r, const float* __restrict__ p,
                                                              const float* __restrict__ Ap, int P, float residual_tol, float* work,
                                                              float* state) {
  __shared__ float tot[VMAXS];
  if (state[3] != 0.f) return;                 // uniform over the grid: no CTA reaches the reduction
  const float rdotr = state[0];
  const float alpha = __fdiv_rn(rdotr, __fadd_rn(state[1], 1e-8f));
  float v[1] = {0.f};
  for (int i = blockIdx.x * VT + threadIdx.x; i < P; i += gridDim.x * VT) {
    x[i] = __fadd_rn(x[i], __fmul_rn(alpha, p[i]));
    const float ri = __fsub_rn(r[i], __fmul_rn(alpha, Ap[i]));
    r[i] = ri;
    v[0] = fmaf(ri, ri, v[0]);
  }
  if (grid_reduce<1>(v, work, tot) && threadIdx.x == 0) {
    const float nr = tot[0];
    state[2] = __fdiv_rn(nr, rdotr);
    state[0] = nr;
    if (nr < residual_tol) state[3] = 1.f;
  }
}

__global__ void __launch_bounds__(VT) spo_ma_cg_direction_kernel(const float* __restrict__ r, float* __restrict__ p, int P, const float* state) {
  if (state[3] != 0.f) return;
  const float beta = state[2];
  for (int i = blockIdx.x * VT + threadIdx.x; i < P; i += gridDim.x * VT) p[i] = __fadd_rn(r[i], __fmul_rn(beta, p[i]));
}

// x = c (xg + nu xb)  (use_a) or  nu xb  (macpo.py:323-325)
__global__ void __launch_bounds__(VT) spo_ma_step_dir_kernel(const float* __restrict__ xg, const float* __restrict__ xb, float c, float nu,
                                                             int use_a, float* __restrict__ x, int P) {
  for (int i = blockIdx.x * VT + threadIdx.x; i < P; i += gridDim.x * VT) {
    const float nb = __fmul_rn(nu, xb[i]);
    x[i] = use_a ? __fmul_rn(c, __fadd_rn(xg[i], nb)) : nb;
  }
}

// one line-search trial (macpo.py:343-348): x <- x * 0.5 / |x| when |x| > 0.5 (|x|^2 in xsq[0]), out = old - coef x
__global__ void __launch_bounds__(VT) spo_ma_ls_trial_kernel(const float* __restrict__ old, float* __restrict__ x, const float* __restrict__ xsq,
                                                             float coef, float* __restrict__ out, int P) {
  const float nrm = sqrtf(xsq[0]);
  const bool rescale = nrm > 0.5f;
  for (int i = blockIdx.x * VT + threadIdx.x; i < P; i += gridDim.x * VT) {
    float xi = x[i];
    if (rescale) { xi = __fdiv_rn(__fmul_rn(xi, 0.5f), nrm); x[i] = xi; }
    out[i] = __fsub_rn(old[i], __fmul_rn(coef, xi));
  }
}

// line-search evaluation (macpo.py:349-368): out = {new reward loss, new cost loss, mean KL(old || new), mean ratio}
__global__ void __launch_bounds__(VT) spo_ma_linesearch_eval_kernel(const float* __restrict__ mean_new, const float* __restrict__ mean_old,
                                                                    const float* __restrict__ ls_new, const float* __restrict__ ls_old, int A,
                                                                    const float* __restrict__ actions, const float* __restrict__ old_logp,
                                                                    const float* __restrict__ adv, const float* __restrict__ cost_adv,
                                                                    const float* __restrict__ factor, int n, float x_coef, float y_coef,
                                                                    float* work, float* out) {
  __shared__ float tot[VMAXS];
  float v[4] = {0.f, 0.f, 0.f, 0.f};
  for (int row = blockIdx.x * VT + threadIdx.x; row < n; row += gridDim.x * VT) {
    float ratio = 1.f, kl = 0.f;
    for (int j = 0; j < A; ++j) {
      const float sn = ma_std(ls_new[j], x_coef, y_coef), so = ma_std(ls_old[j], x_coef, y_coef);
      const size_t e = static_cast<size_t>(row) * A + j;
      const float mn = mean_new[e], mo = mean_old[e];
      const float diff = __fsub_rn(actions[e], mn);
      const float lsn = logf(sn), lso = logf(so);
      const float lp = ma_gauss_logp(diff, sn, lsn);
      ratio = __fmul_rn(ratio, expf(__fsub_rn(lp, old_logp[e])));
      const float dm = __fsub_rn(mo, mn);
      const float num = __fadd_rn(__fmul_rn(so, so), __fmul_rn(dm, dm));
      const float den = __fadd_rn(1e-8f, __fmul_rn(2.f, __fmul_rn(sn, sn)));
      kl += __fsub_rn(__fadd_rn(__fsub_rn(lso, lsn), __fdiv_rn(num, den)), 0.5f);
    }
    const float rf = __fmul_rn(ratio, factor[row]);
    v[0] += __fmul_rn(rf, adv[row]);
    v[1] += __fmul_rn(rf, cost_adv[row]);
    v[2] += kl;
    v[3] += ratio;
  }
  if (grid_reduce<4>(v, work, tot) && threadIdx.x == 0) {
    const float fn = static_cast<float>(n);
    out[0] = -(tot[0] / fn);
    out[1] = tot[1] / fn;
    out[2] = tot[2] / fn;
    out[3] = tot[3] / fn;
  }
}

}  // namespace

extern "C" {

int spo_ma_mlp_layer_jvp(const float* in, const float* din, int n, int K, const float* W, const float* dW, const float* db, const float* pre,
                         const float* ln_w, const float* dln_w, const float* dln_b, int H, const float* ln_in_w, const float* ln_in_b,
                         const float* dln_in_w, const float* dln_in_b, float* dout, void* stream) {
  SPO_REQUIRE(in && W && dW && db && pre && ln_w && dln_w && dln_b && dout && n > 0, SPO_ERR_INVALID_ARG,
              "spo_ma_mlp_layer_jvp: null argument or n<=0");
  const bool lin = ln_in_w != nullptr;
  SPO_REQUIRE(lin ? (ln_in_b && dln_in_w && dln_in_b) : (din && !ln_in_b && !dln_in_w && !dln_in_b), SPO_ERR_INVALID_ARG,
              "spo_ma_mlp_layer_jvp: pass din, or the input LayerNorm with both tangents");
  SPO_REQUIRE(K >= 2 && (K & 1) == 0 && H >= 128 && H <= MA_MAXH && (H & 127) == 0, SPO_ERR_UNSUPPORTED,
              "spo_ma_mlp_layer_jvp: K=%d must be even, H=%d a multiple of 128 up to %d", K, H, MA_MAXH);
  SPO_REQUIRE(ma_aligned(in, 8) && (lin || ma_aligned(din, 8)) && ma_aligned(W, 8) && ma_aligned(dW, 8) && ma_aligned(db, 16) &&
                  ma_aligned(pre, 16) && ma_aligned(ln_w, 16) && ma_aligned(dln_w, 16) && ma_aligned(dln_b, 16) && ma_aligned(dout, 16),
              SPO_ERR_INVALID_ARG, "spo_ma_mlp_layer_jvp: in / din / W / dW must be 8-byte, the H-sized buffers 16-byte aligned");
  MaJvpArgs a{in, din, W, dW, db, pre, ln_w, dln_w, dln_b, ln_in_w, ln_in_b, dln_in_w, dln_in_b, dout, n, K, H};
  ma_launch_hb(H, [&](auto hb) {
    spo_ma_layer_jvp_kernel<hb.value><<<(n + MA_ROWS - 1) / MA_ROWS, MA_THREADS, ma_layer_smem(H), static_cast<cudaStream_t>(stream)>>>(a);
  });
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_head_jvp(const float* feat, const float* dfeat, int n, int H, const float* W, const float* dW, const float* db, int A,
                    const float* log_std, float std_x_coef, float std_y_coef, float* dmean, float* part, void* stream) {
  SPO_REQUIRE(feat && dfeat && W && dW && db && log_std && dmean && part && n > 0 && H > 0, SPO_ERR_INVALID_ARG,
              "spo_ma_head_jvp: null argument or empty shape");
  SPO_REQUIRE(A >= 1 && A <= 32, SPO_ERR_UNSUPPORTED, "spo_ma_head_jvp: act_dim=%d must be in 1..32", A);
  MaHeadJvpArgs a{feat, dfeat, W, dW, db, log_std, dmean, part, n, H, A, std_x_coef, std_y_coef};
  spo_ma_head_jvp_kernel<<<(n + 31) / 32, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_fvp_finalize(const float* gn, const float* v, float* out, int P, const float* log_std, int log_std_offset, int A, float std_x_coef,
                        float std_y_coef, float damping, void* stream) {
  SPO_REQUIRE(gn && v && out && log_std && P > 0 && A >= 1 && log_std_offset >= 0 && log_std_offset + A <= P, SPO_ERR_INVALID_ARG,
              "spo_ma_fvp_finalize: null argument or log_std block outside [0, P)");
  spo_ma_fvp_finalize_kernel<<<vec_grid(P), VT, 0, static_cast<cudaStream_t>(stream)>>>(gn, v, out, P, log_std, log_std_offset, A, std_x_coef,
                                                                                         std_y_coef, damping);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_ratio_loss(const float* mean, int n, const float* log_std, int A, const float* actions, const float* old_logp, const float* adv,
                      const float* factor, float sign, float std_x_coef, float std_y_coef, float* dmean, float* part, void* stream) {
  SPO_REQUIRE(mean && log_std && actions && old_logp && adv && factor && dmean && part && n > 0, SPO_ERR_INVALID_ARG,
              "spo_ma_ratio_loss: null argument or n<=0");
  SPO_REQUIRE(A >= 1 && A <= 32, SPO_ERR_UNSUPPORTED, "spo_ma_ratio_loss: act_dim=%d must be in 1..32", A);
  spo_ma_ratio_loss_kernel<<<(n + 31) / 32, 32, 0, static_cast<cudaStream_t>(stream)>>>(mean, n, log_std, A, actions, old_logp, adv, factor, sign,
                                                                                        std_x_coef, std_y_coef, dmean, part);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_dots(const float* a0, const float* b0, const float* a1, const float* b1, const float* a2, const float* b2, const float* a3,
                const float* b3, int ndot, int P, float* work, float* out, void* stream) {
  SPO_REQUIRE(ndot >= 1 && ndot <= VMAXS && P > 0 && work && out, SPO_ERR_INVALID_ARG, "spo_ma_dots: ndot=%d must be in 1..4, P > 0", ndot);
  Dots d{{a0, a1, a2, a3}, {b0, b1, b2, b3}};
  for (int s = 0; s < ndot; ++s) SPO_REQUIRE(d.a[s] && d.b[s], SPO_ERR_INVALID_ARG, "spo_ma_dots: pair %d is null", s);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int g = vec_grid(P);
  switch (ndot) {
    case 1: spo_ma_dots_kernel<1><<<g, VT, 0, st>>>(d, P, work, out); break;
    case 2: spo_ma_dots_kernel<2><<<g, VT, 0, st>>>(d, P, work, out); break;
    case 3: spo_ma_dots_kernel<3><<<g, VT, 0, st>>>(d, P, work, out); break;
    default: spo_ma_dots_kernel<4><<<g, VT, 0, st>>>(d, P, work, out); break;
  }
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_work_floats(void) { return VCTAS * VMAXS + 4; }

int spo_ma_cg_begin(const float* b, float* x, float* r, float* p, int P, float* work, float* state, void* stream) {
  SPO_REQUIRE(b && x && r && p && work && state && P > 0, SPO_ERR_INVALID_ARG, "spo_ma_cg_begin: null argument or P<=0");
  spo_ma_cg_begin_kernel<<<vec_grid(P), VT, 0, static_cast<cudaStream_t>(stream)>>>(b, x, r, p, P, work, state);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_cg_update(float* x, float* r, float* p, const float* Ap, int P, float residual_tol, float* work, float* state, void* stream) {
  SPO_REQUIRE(x && r && p && Ap && work && state && P > 0, SPO_ERR_INVALID_ARG, "spo_ma_cg_update: null argument or P<=0");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  spo_ma_cg_update_kernel<<<vec_grid(P), VT, 0, st>>>(x, r, p, Ap, P, residual_tol, work, state);
  SPO_CUDA_TRY(cudaGetLastError());
  spo_ma_cg_direction_kernel<<<vec_grid(P), VT, 0, st>>>(r, p, P, state);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_step_dir(const float* xg, const float* xb, float c, float nu, int use_a, float* x, int P, void* stream) {
  SPO_REQUIRE(xb && x && (xg || !use_a) && P > 0, SPO_ERR_INVALID_ARG, "spo_ma_step_dir: null argument or P<=0");
  spo_ma_step_dir_kernel<<<vec_grid(P), VT, 0, static_cast<cudaStream_t>(stream)>>>(xg, xb, c, nu, use_a, x, P);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_ls_trial(const float* old, float* x, const float* xsq, float coef, float* out, int P, void* stream) {
  SPO_REQUIRE(old && x && xsq && out && P > 0, SPO_ERR_INVALID_ARG, "spo_ma_ls_trial: null argument or P<=0");
  spo_ma_ls_trial_kernel<<<vec_grid(P), VT, 0, static_cast<cudaStream_t>(stream)>>>(old, x, xsq, coef, out, P);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_linesearch_eval(const float* mean_new, const float* mean_old, const float* log_std_new, const float* log_std_old, int A,
                           const float* actions, const float* old_logp, const float* adv, const float* cost_adv, const float* factor, int n,
                           float std_x_coef, float std_y_coef, float* work, float* out, void* stream) {
  SPO_REQUIRE(mean_new && mean_old && log_std_new && log_std_old && actions && old_logp && adv && cost_adv && factor && work && out && n > 0 && A >= 1,
              SPO_ERR_INVALID_ARG, "spo_ma_linesearch_eval: null argument or empty shape");
  spo_ma_linesearch_eval_kernel<<<vec_grid(n), VT, 0, static_cast<cudaStream_t>(stream)>>>(mean_new, mean_old, log_std_new, log_std_old, A, actions,
                                                                                          old_logp, adv, cost_adv, factor, n, std_x_coef,
                                                                                          std_y_coef, work, out);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

}  // extern "C"
