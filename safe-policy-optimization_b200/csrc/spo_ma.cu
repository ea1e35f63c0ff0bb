// Multi-agent (MAPPO-Lag, BASELINE config 5) network forward: the rollout-side `get_actions` of
// safepo/multi_agent/mappolag.py:69-82 -- MultiAgentActor / MultiAgentCritic of safepo/common/model.py:172-363 built from
// safepo/utils/mlp.py:9-61 (LayerNorm -> [Linear -> ELU -> LayerNorm] x (1 + layer_N)) and the DiagGaussian head of
// safepo/utils/distributions.py:21-42 / act.py:24-43 (std = sigmoid(log_std / x_coef) * y_coef, per-dimension log-probs).
//
// First slice of SURVEY section 8f rank 3: the forward, fp32 FFMA tiles; with `pre` / `xn` outputs the same kernel is the training
// forward of the update (second slice, spo_ma_update.cu).  One
// launch per hidden layer: a CTA owns 32 rows x ALL H outputs, so the LayerNorm over the H outputs of a row is a warp-level
// reduction in the epilogue (warp w holds rows 4w..4w+3 completely: lane l owns columns 4l..4l+3 of every 128-column block).
// The K loop stages 16-wide chunks of W (transposed to [k][h]: conflict-free float4 reads) and of the input rows (with the
// optional input LayerNorm applied on the fly) in shared memory: 256 FMA per 20 shared-memory float4 loads per thread.
// Algorithmic cost per row and layer: 2 K H FLOP, 4 (K + H) bytes; at config 5 (N = 8192, K = 398 / 512, H = 512) a layer is
// 3.3 / 4.3 GFLOP and FFMA-bound.  A tensor-pipe variant (mma.sync 3xTF32 with the truncating register split, LayerNorm statistics
// exchanged between eight column groups) measured 15 % faster but 3x less accurate through three layers and was not kept
// (DESIGN.md section 4.6); the wgmma version (K-major operand tiles do not fit one SM's shared memory: a cluster would split H
// and exchange the LayerNorm statistics) is the next step, DESIGN.md section 8.
#include "spo_ma_math.cuh"

namespace {

struct MaLayerArgs {
  const float* in;      // [n][K]
  const float *W, *b, *ln_w, *ln_b;   // [H][K], [H], [H], [H]
  const float *lin_w, *lin_b;         // input LayerNorm over K (feature_norm) or null
  float* out;           // [n][H]
  int n, K, H;
  float* pre;           // training: ELU(z) before the output LayerNorm [n][H], or null
  float* xn;            // training: the input after the input LayerNorm [n][K], or null
};

// HB = H / 128 column blocks per lane (H = 128 * HB)
template <int HB>
__global__ void __launch_bounds__(MA_THREADS) spo_ma_layer_kernel(const MaLayerArgs a) {
  extern __shared__ __align__(16) float smem[];
  constexpr int H = 128 * HB;
  float* Wc = smem;                       // [MA_KC][H]
  float* xs = Wc + MA_KC * H;             // [MA_ROWS][MA_KC + 4]
  float* stat = xs + MA_ROWS * (MA_KC + 4);   // [MA_ROWS][2] mean, rstd of the input rows (input LayerNorm)
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

  for (int k0 = 0; k0 < K; k0 += MA_KC) {
    ma_stage_w_chunk<HB>(a.W, K, k0, Wc, tid);
    // input chunk: 32 rows x 16 k = 256 float2
    {
      const int r = tid >> 3, kk = (tid & 7) * 2, g = row0 + r;
      float2 v = make_float2(0.f, 0.f);
      if (g < a.n && k0 + kk < K) {
        v = __ldg(reinterpret_cast<const float2*>(a.in + static_cast<size_t>(g) * K + k0 + kk));
        if (a.lin_w) {
          const float mean = stat[2 * r], rstd = stat[2 * r + 1];
          v.x = fmaf((v.x - mean) * rstd, a.lin_w[k0 + kk], a.lin_b[k0 + kk]);
          v.y = fmaf((v.y - mean) * rstd, a.lin_w[k0 + kk + 1], a.lin_b[k0 + kk + 1]);
          if (a.xn) *reinterpret_cast<float2*>(a.xn + static_cast<size_t>(g) * K + k0 + kk) = v;
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

  // epilogue: bias, ELU, LayerNorm over the H outputs of each row (the warp holds the whole row), write-back
#pragma unroll
  for (int r = 0; r < 4; ++r) {
#pragma unroll
    for (int cb = 0; cb < HB; ++cb) {
      const float4 bv = __ldg(reinterpret_cast<const float4*>(a.b + 128 * cb + 4 * lane));
      const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float v = acc[r][4 * cb + e] + bb[e];
        acc[r][4 * cb + e] = v > 0.f ? v : expm1f(v);     // ELU(alpha = 1)
      }
    }
    float mean, rstd;
    ma_row_ln_stats<HB>(acc[r], mean, rstd);
    const int g = row0 + 4 * wid + r;
    if (g < a.n) {
      if (a.pre) {
#pragma unroll
        for (int cb = 0; cb < HB; ++cb)
          *reinterpret_cast<float4*>(a.pre + static_cast<size_t>(g) * H + 128 * cb + 4 * lane) =
              make_float4(acc[r][4 * cb], acc[r][4 * cb + 1], acc[r][4 * cb + 2], acc[r][4 * cb + 3]);
      }
#pragma unroll
      for (int cb = 0; cb < HB; ++cb) {
        const float4 gw = __ldg(reinterpret_cast<const float4*>(a.ln_w + 128 * cb + 4 * lane));
        const float4 gb = __ldg(reinterpret_cast<const float4*>(a.ln_b + 128 * cb + 4 * lane));
        float4 o;
        o.x = fmaf((acc[r][4 * cb + 0] - mean) * rstd, gw.x, gb.x);
        o.y = fmaf((acc[r][4 * cb + 1] - mean) * rstd, gw.y, gb.y);
        o.z = fmaf((acc[r][4 * cb + 2] - mean) * rstd, gw.z, gb.z);
        o.w = fmaf((acc[r][4 * cb + 3] - mean) * rstd, gw.w, gb.w);
        *reinterpret_cast<float4*>(a.out + static_cast<size_t>(g) * H + 128 * cb + 4 * lane) = o;
      }
    }
  }
}

struct MaHeadArgs {
  const float *feat, *W, *b, *log_std, *eps;   // [n][H], [O][H], [O], [O] or null (value head), [n][O] or null (deterministic)
  float *out, *logp;                           // actions / values [n][O], per-dimension log-probs [n][O] or null
  int n, H, O;
  float x_coef, y_coef;
};

// one warp per row: out[o] = b[o] + feat[row] . W[o]; actor: action = mean + std * eps, log-prob per dimension
__global__ void __launch_bounds__(256) spo_ma_head_kernel(const MaHeadArgs a) {
  const int lane = threadIdx.x & 31, row = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= a.n) return;
  const float* f = a.feat + static_cast<size_t>(row) * a.H;
  for (int o = 0; o < a.O; ++o) {
    const float s = ma_row_dot(f, a.W + o * a.H, a.H, lane);
    if (lane == 0) {
      const float mean = s + a.b[o];
      if (!a.log_std) {
        a.out[static_cast<size_t>(row) * a.O + o] = mean;
      } else {
        const float std = ma_std(a.log_std[o], a.x_coef, a.y_coef);
        float action = mean;
        if (a.eps) action = __fadd_rn(mean, __fmul_rn(a.eps[static_cast<size_t>(row) * a.O + o], std));
        a.out[static_cast<size_t>(row) * a.O + o] = action;
        if (a.logp) a.logp[static_cast<size_t>(row) * a.O + o] = ma_gauss_logp(__fsub_rn(action, mean), std, logf(std));
      }
    }
  }
}

}  // namespace

extern "C" {

static int ma_layer_launch(const float* in, int n, int K, const float* W, const float* b, const float* ln_w, const float* ln_b, int H,
                           const float* ln_in_w, const float* ln_in_b, float* out, float* pre, float* xn, void* stream, const char* who) {
  SPO_REQUIRE(in && W && b && ln_w && ln_b && out && n > 0, SPO_ERR_INVALID_ARG, "%s: null argument or n<=0", who);
  SPO_REQUIRE((ln_in_w == nullptr) == (ln_in_b == nullptr), SPO_ERR_INVALID_ARG, "%s: input LayerNorm needs weight and bias", who);
  SPO_REQUIRE(K >= 2 && (K & 1) == 0 && H >= 128 && H <= MA_MAXH && (H & 127) == 0, SPO_ERR_UNSUPPORTED,
              "%s: K=%d must be even, H=%d a multiple of 128 up to %d", who, K, H, MA_MAXH);
  SPO_REQUIRE(ma_aligned(in, 8) && ma_aligned(W, 8) && ma_aligned(out, 16), SPO_ERR_INVALID_ARG, "%s: in / W must be 8-byte, out 16-byte aligned",
              who);
  SPO_REQUIRE(ma_aligned(pre, 16) && ma_aligned(xn, 8), SPO_ERR_INVALID_ARG, "%s: pre must be 16-byte, xn 8-byte aligned", who);
  SPO_REQUIRE(!xn || ln_in_w, SPO_ERR_INVALID_ARG, "%s: xn is the output of the input LayerNorm, which is not requested", who);
  MaLayerArgs a{in, W, b, ln_w, ln_b, ln_in_w, ln_in_b, out, n, K, H, pre, xn};
  ma_launch_hb(H, [&](auto hb) {
    spo_ma_layer_kernel<hb.value><<<(n + MA_ROWS - 1) / MA_ROWS, MA_THREADS, ma_layer_smem(H), static_cast<cudaStream_t>(stream)>>>(a);
  });
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_ma_mlp_layer(const float* in, int n, int K, const float* W, const float* b, const float* ln_w, const float* ln_b, int H,
                     const float* ln_in_w, const float* ln_in_b, float* out, void* stream) {
  return ma_layer_launch(in, n, K, W, b, ln_w, ln_b, H, ln_in_w, ln_in_b, out, nullptr, nullptr, stream, "spo_ma_mlp_layer");
}

int spo_ma_mlp_layer_train(const float* in, int n, int K, const float* W, const float* b, const float* ln_w, const float* ln_b, int H,
                           const float* ln_in_w, const float* ln_in_b, float* out, float* pre, float* xn, void* stream) {
  SPO_REQUIRE(pre, SPO_ERR_INVALID_ARG, "spo_ma_mlp_layer_train: pre is null");
  return ma_layer_launch(in, n, K, W, b, ln_w, ln_b, H, ln_in_w, ln_in_b, out, pre, xn, stream, "spo_ma_mlp_layer_train");
}

int spo_ma_head(const float* feat, int n, int H, const float* W, const float* b, int O, const float* log_std, float std_x_coef,
                float std_y_coef, const float* eps, float* out, float* logp, void* stream) {
  SPO_REQUIRE(feat && W && b && out && n > 0 && O > 0 && H > 0, SPO_ERR_INVALID_ARG, "spo_ma_head: null argument or empty shape");
  MaHeadArgs a{feat, W, b, log_std, eps, out, logp, n, H, O, std_x_coef, std_y_coef};
  spo_ma_head_kernel<<<(n + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

}  // extern "C"
