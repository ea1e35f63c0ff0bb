// Trust-region pieces of CPO / TRPO-Lag on the device.
//
// Reference: safepo/single_agent/cpo.py:70-157 (flat params, conjugate_gradients, fvp),
// :353-519 (losses, line search); trpo_lag.py:363-442.
//
//   spo_surrogate_grad   L = mean_i ratio_i * adv_i  and  dL/dtheta over the full batch
//   spo_fvp              (H + damping I) v,  H = Hessian of mean_{S*A} KL(old || new) at new = old.
//                        For a Gaussian with state-independent log_std this is
//                          [ 2 v_ls / A ;  J^T diag(sigma^-2) J v_mean / (S A) ]
//                        (SURVEY fact 7): one JVP and one VJP through the mean MLP, no
//                        autograd graph -- 8 tile GEMMs per 64 rows instead of ~12.
//   spo_linesearch_eval  mean(ratio*adv_a), mean(ratio*adv_b), mean_{S*A} KL(old||new)
//   spo_conjugate_gradient  cpo.py:81-106 with every dot / axpy / the residual test on device
//
// All three full-batch kernels share one persistent tile loop: one CTA per SM walk
// the [S,D] observations in 64-row tiles with the actor (and, for the FVP, the tangent
// vector reshaped as a second set of weights) resident in shared memory; parameter-shaped
// results are accumulated in registers across tiles and flushed once per CTA with atomics.
#include "spo_forward.cuh"

namespace {

enum { MODE_GRAD = 0, MODE_FVP = 1, MODE_EVAL = 2 };

struct TrArgs {
  const float* params;
  const float *obs, *act, *logp_old, *adv_a, *adv_b, *old_mean, *old_log_std;
  const float* v;     // FVP: tangent, actor-flat
  float* out;         // GRAD/FVP: [P_a] accumulated with atomics (pre-zeroed); EVAL: out3
  float* out_loss;    // GRAD: scalar (pre-zeroed)
  int64_t count;
  int D, A;
};

// tangent vector viewed as a second set of actor weights (same packed order, offset by -0:
// v is actor-flat so the SpoNetOff of net 0 applies directly)
__device__ inline void load_tangent(const float* __restrict__ v, const SpoNetOff& o, int D, const SpoNetSmem& s, int tid) {
  spo_load_net(v, o, D, s, tid, SPO_THREADS);
}

template <int MODE, int NT1>
__global__ void __launch_bounds__(SPO_THREADS, 1) spo_trust_kernel(const TrArgs a) {
  extern __shared__ __align__(16) float smem[];
  __shared__ double red[3][SPO_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int D = a.D, A = a.A, Dp = spo_pad4(D), ldx = spo_ld(D);
  const SpoNetOff off = spo_net_off(D, A, 0);

  SpoNetSmem w, tv;
  float* p = spo_carve_net(smem, D, A, true, w);
  if (MODE == MODE_FVP) p = spo_carve_net(p, D, A, false, tv);
  float* x = p;   p += SPO_ROWS * ldx;
  float* h1 = p;  p += SPO_ROWS * SPO_LDH;
  float* h2 = p;  p += SPO_ROWS * SPO_LDH;
  // one [64][LDH] buffer holds, in turn, dh1 and dh2 (FVP), dz2 and dz1: a GEMM that reads it keeps its result in
  // registers until a barrier, then overwrites it (one buffer less keeps the FVP within 227 KB at obs 128 / act 8)
  float* dz = p;  p += SPO_ROWS * SPO_LDH;
  float* y = p;   p += SPO_ROWS * SPO_MAX_ACT;
  float* gy = p;  p += SPO_ROWS * SPO_MAX_ACT;
  float* gl = p;  p += SPO_ROWS * SPO_MAX_ACT;   // GRAD: per-row d/dlog_std
  float* gsmall = p; p += 672;                   // b1[64] b2[64] w3[A*64] b3[A] log_std[A]
  float* ls = p;  p += 8;

  spo_load_net(a.params, off, D, w, tid, SPO_THREADS);
  if (MODE == MODE_FVP) load_tangent(a.v, off, D, tv, tid);
  if (tid < A) ls[tid] = a.params[off.log_std + tid];
  const int SP = 2 * SPO_HID + A * SPO_HID + 2 * A;
  for (int i = tid; i < 672; i += SPO_THREADS) gsmall[i] = 0.f;

  const int j0 = spo_m0(tid), k0 = spo_nb(tid);   // 4x4 parameter tile (W2[j0..][k0..]; W1 tile 0 likewise)
  const int rs = spo_ns(tid);                      // rows rs, rs+4, rs+8, rs+12 of the n-major GEMMs
  float gW2[4][4], gW1[NT1][4][4];
  spo_zero(gW2);
#pragma unroll
  for (int i = 0; i < NT1; ++i) spo_zero(gW1[i]);
  double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0;
  const float inv_s = 1.f / static_cast<float>(a.count);
  const float inv_sa = 1.f / (static_cast<float>(a.count) * A);

  const int64_t n_tiles = (a.count + SPO_ROWS - 1) / SPO_ROWS;
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
    if (MODE != MODE_FVP) {
      spo_out_fwd(h2, w.w3, w.b3, A, y, SPO_MAX_ACT, tid, SPO_THREADS);
      __syncthreads();
    }

    if (MODE == MODE_EVAL || MODE == MODE_GRAD) {
      if (tid < SPO_ROWS) {
        const int r = tid;
        const bool valid = r < rows;
        const int64_t g = row0 + (valid ? r : 0);
        float lp = 0.f, kl = 0.f;
        float dmu[SPO_MAX_ACT], dl[SPO_MAX_ACT];
#pragma unroll
        for (int j = 0; j < SPO_MAX_ACT; ++j) {
          dmu[j] = dl[j] = 0.f;
          if (j < A) {
            const float mean = y[r * SPO_MAX_ACT + j];
            const float std = expf(ls[j]);
            const float var = __fmul_rn(std, std);
            const float diff = __fsub_rn(__ldg(a.act + g * A + j), mean);
            const float d2 = __fmul_rn(diff, diff);
            const float term = spo_normal_log_term(d2, var, std);
            lp = (j == 0) ? term : __fadd_rn(lp, term);
            dmu[j] = __fdiv_rn(diff, var);
            dl[j] = __fsub_rn(__fdiv_rn(d2, var), 1.f);
            if (MODE == MODE_EVAL) kl += spo_kl_term(__ldg(a.old_mean + g * A + j), mean, expf(__ldg(a.old_log_std + j)), std);
          }
        }
        const float ratio = expf(__fsub_rn(lp, __ldg(a.logp_old + g)));
        const float adv = __ldg(a.adv_a + g);
        if (valid) {
          acc0 += static_cast<double>(__fmul_rn(ratio, adv));
          if (MODE == MODE_EVAL) {
            if (a.adv_b) acc1 += static_cast<double>(__fmul_rn(ratio, __ldg(a.adv_b + g)));
            acc2 += static_cast<double>(kl);
          }
        }
        if (MODE == MODE_GRAD) {
          const float c = valid ? __fmul_rn(__fmul_rn(adv, ratio), inv_s) : 0.f;
#pragma unroll
          for (int j = 0; j < SPO_MAX_ACT; ++j) {
            gy[r * SPO_MAX_ACT + j] = __fmul_rn(c, dmu[j]);
            gl[r * SPO_MAX_ACT + j] = __fmul_rn(c, dl[j]);
          }
        }
      }
      if (MODE == MODE_EVAL) continue;
      __syncthreads();
    }

    if (MODE == MODE_FVP) {
      // ---- JVP ----
      {  // dh1 = (x V1^T + c1) * (1 - h1^2)     -> dz
        float acc[4][4];
        spo_zero(acc);
        spo_tile_mma<true>(acc, tv.w1t, SPO_LDH, x, ldx, j0, rs, Dp);   // m: unit j0.., n: rows rs + 4*ni
        const float4 c = *reinterpret_cast<const float4*>(tv.b1 + j0);
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
          const float4 h = *reinterpret_cast<const float4*>(h1 + (rs + 4 * ni) * SPO_LDH + j0);
          float4 o;
          o.x = (acc[0][ni] + c.x) * (1.f - h.x * h.x);
          o.y = (acc[1][ni] + c.y) * (1.f - h.y * h.y);
          o.z = (acc[2][ni] + c.z) * (1.f - h.z * h.z);
          o.w = (acc[3][ni] + c.w) * (1.f - h.w * h.w);
          *reinterpret_cast<float4*>(dz + (rs + 4 * ni) * SPO_LDH + j0) = o;
        }
      }
      __syncthreads();
      {  // dh2 = (dh1 W2^T + h1 V2^T + c2) * (1 - h2^2)     -> dz, over dh1
        float acc[4][4];
        spo_zero(acc);
        spo_tile_mma<true>(acc, w.w2t, SPO_LDH, dz, SPO_LDH, j0, rs, SPO_HID);
        spo_tile_mma<true>(acc, tv.w2t, SPO_LDH, h1, SPO_LDH, j0, rs, SPO_HID);
        __syncthreads();   // every read of dh1 is done
        const float4 c = *reinterpret_cast<const float4*>(tv.b2 + j0);
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
          const float4 h = *reinterpret_cast<const float4*>(h2 + (rs + 4 * ni) * SPO_LDH + j0);
          float4 o;
          o.x = (acc[0][ni] + c.x) * (1.f - h.x * h.x);
          o.y = (acc[1][ni] + c.y) * (1.f - h.y * h.y);
          o.z = (acc[2][ni] + c.z) * (1.f - h.z * h.z);
          o.w = (acc[3][ni] + c.w) * (1.f - h.w * h.w);
          *reinterpret_cast<float4*>(dz + (rs + 4 * ni) * SPO_LDH + j0) = o;
        }
      }
      __syncthreads();
      // dmu = dh2 W3^T + h2 V3^T + c3 ; g_mu = dmu * sigma^-2 / (S A)
      spo_out_fwd(dz, w.w3, tv.b3, A, y, SPO_MAX_ACT, tid, SPO_THREADS);   // dh2 W3^T + c3
      for (int wi = tid; wi < SPO_ROWS * A; wi += SPO_THREADS) {           // + h2 V3^T
        const int r = wi / A, o = wi - r * A;
        const float4* hp = reinterpret_cast<const float4*>(h2 + r * SPO_LDH);
        const float4* vp = reinterpret_cast<const float4*>(tv.w3 + o * SPO_HID);
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < SPO_HID / 4; ++k) {
          const float4 aa = hp[k], bb = vp[k];
          s = fmaf(aa.x, bb.x, s); s = fmaf(aa.y, bb.y, s); s = fmaf(aa.z, bb.z, s); s = fmaf(aa.w, bb.w, s);
        }
        gy[r * SPO_MAX_ACT + o] = s;
      }
      __syncthreads();
      for (int wi = tid; wi < SPO_ROWS * SPO_MAX_ACT; wi += SPO_THREADS) {
        const int r = wi >> 3, o = wi & 7;
        float gval = 0.f;
        if (o < A && r < rows) gval = (y[wi] + gy[wi]) * expf(-2.f * ls[o]) * inv_sa;
        gy[wi] = gval;
      }
      __syncthreads();
    }

    // ---- backward / VJP of the mean MLP with output cotangent gy[r][o] ----
    for (int i = tid; i < A * SPO_HID + A + (MODE == MODE_GRAD ? A : 0); i += SPO_THREADS) {
      float s = 0.f;
      if (i < A * SPO_HID) {
        const int o = i >> 6, k = i & 63;
#pragma unroll 8
        for (int r = 0; r < SPO_ROWS; ++r) s = fmaf(gy[r * SPO_MAX_ACT + o], h2[r * SPO_LDH + k], s);
      } else if (i < A * SPO_HID + A) {
        const int o = i - A * SPO_HID;
        for (int r = 0; r < SPO_ROWS; ++r) s += gy[r * SPO_MAX_ACT + o];
      } else {
        const int j = i - A * SPO_HID - A;
        for (int r = 0; r < SPO_ROWS; ++r) s += gl[r * SPO_MAX_ACT + j];
      }
      gsmall[2 * SPO_HID + i] += s;
    }
    if (MODE == MODE_FVP) __syncthreads();   // dh2 (dz) was read by nobody else; dz2 overwrites it below
    {
      const int r0 = (tid >> 4) * 4, kk = (tid & 15) * 4;
#pragma unroll
      for (int ri = 0; ri < 4; ++ri) {
        const int r = r0 + ri;
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int o = 0; o < A; ++o) {
          const float d = gy[r * SPO_MAX_ACT + o];
          const float4 wv = *reinterpret_cast<const float4*>(w.w3 + o * SPO_HID + kk);
          s.x = fmaf(d, wv.x, s.x); s.y = fmaf(d, wv.y, s.y); s.z = fmaf(d, wv.z, s.z); s.w = fmaf(d, wv.w, s.w);
        }
        const float4 h = *reinterpret_cast<const float4*>(h2 + r * SPO_LDH + kk);
        s.x *= (1.f - h.x * h.x); s.y *= (1.f - h.y * h.y); s.z *= (1.f - h.z * h.z); s.w *= (1.f - h.w * h.w);
        *reinterpret_cast<float4*>(dz + r * SPO_LDH + kk) = s;
      }
    }
    __syncthreads();
    spo_tile_mma<false>(gW2, dz, SPO_LDH, h1, SPO_LDH, j0, k0, SPO_ROWS);
    if (tid < SPO_HID) {
      float s = 0.f;
#pragma unroll 8
      for (int r = 0; r < SPO_ROWS; ++r) s += dz[r * SPO_LDH + tid];
      gsmall[SPO_HID + tid] += s;
    }
    {  // dz1 = (dz2 W2) * (1 - h1^2)     -> dz, over dz2
      float acc[4][4];
      spo_zero(acc);
      spo_tile_mma<true>(acc, w.w2, SPO_LDH, dz, SPO_LDH, j0, rs, SPO_HID);   // m: input unit, n: rows rs + 4*ni
      __syncthreads();   // every read of dz2 is done
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        const float4 h = *reinterpret_cast<const float4*>(h1 + (rs + 4 * ni) * SPO_LDH + j0);
        float4 o4;
        o4.x = acc[0][ni] * (1.f - h.x * h.x);
        o4.y = acc[1][ni] * (1.f - h.y * h.y);
        o4.z = acc[2][ni] * (1.f - h.z * h.z);
        o4.w = acc[3][ni] * (1.f - h.w * h.w);
        *reinterpret_cast<float4*>(dz + (rs + 4 * ni) * SPO_LDH + j0) = o4;
      }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < NT1; ++i) {
      const int tj = (i == 0) ? j0 : (tid & 15) * 4, tk = (i == 0) ? k0 : 64 + (tid >> 4) * 4;
      if (tk < Dp) spo_tile_mma<false>(gW1[i], dz, SPO_LDH, x, ldx, tj, tk, SPO_ROWS);
    }
    if (tid < SPO_HID) {
      float s = 0.f;
#pragma unroll 8
      for (int r = 0; r < SPO_ROWS; ++r) s += dz[r * SPO_LDH + tid];
      gsmall[tid] += s;
    }
  }

  // ---- flush ----
  if (MODE == MODE_EVAL || MODE == MODE_GRAD) {
    acc0 = spo_warp_sum(acc0); acc1 = spo_warp_sum(acc1); acc2 = spo_warp_sum(acc2);
    if (lane == 0) { red[0][wid] = acc0; red[1][wid] = acc1; red[2][wid] = acc2; }
    __syncthreads();
    if (tid == 0) {
      double s0 = 0, s1 = 0, s2 = 0;
      for (int i = 0; i < SPO_THREADS / 32; ++i) { s0 += red[0][i]; s1 += red[1][i]; s2 += red[2][i]; }
      const double S = static_cast<double>(a.count);
      if (MODE == MODE_GRAD) {
        atomicAdd(a.out_loss, static_cast<float>(s0 / S));
      } else {
        atomicAdd(a.out + 0, static_cast<float>(s0 / S));
        atomicAdd(a.out + 1, static_cast<float>(s1 / S));
        atomicAdd(a.out + 2, static_cast<float>(s2 / (S * A)));
      }
    }
    if (MODE == MODE_EVAL) return;
  }
  __syncthreads();
  if (a.out) {
#pragma unroll
    for (int mi = 0; mi < 4; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) atomicAdd(a.out + off.w2 + (j0 + mi) * SPO_HID + k0 + ni, gW2[mi][ni]);
#pragma unroll
    for (int i = 0; i < NT1; ++i) {
      const int tj = (i == 0) ? j0 : (tid & 15) * 4, tk = (i == 0) ? k0 : 64 + (tid >> 4) * 4;
      if (tk < Dp) {
#pragma unroll
        for (int mi = 0; mi < 4; ++mi)
#pragma unroll
          for (int ni = 0; ni < 4; ++ni)
            if (tk + ni < D) atomicAdd(a.out + off.w1 + (tj + mi) * D + tk + ni, gW1[i][mi][ni]);
      }
    }
    for (int i = tid; i < SP; i += SPO_THREADS) {
      int g;
      if (i < SPO_HID) g = off.b1 + i;
      else if (i < 2 * SPO_HID) g = off.b2 + (i - SPO_HID);
      else if (i < 2 * SPO_HID + A * SPO_HID) g = off.w3 + (i - 2 * SPO_HID);
      else if (i < 2 * SPO_HID + A * SPO_HID + A) g = off.b3 + (i - 2 * SPO_HID - A * SPO_HID);
      else g = off.log_std + (i - 2 * SPO_HID - A * SPO_HID - A);
      if (MODE == MODE_FVP && g < A) continue;   // log_std block has its own closed form
      atomicAdd(a.out + g, gsmall[i]);
    }
  }
}

// out += damping * v ; log_std block: out = 2 v / A + damping v   (cpo.py:157 and fact 7)
__global__ void spo_fvp_finalize_kernel(float* out, const float* v, int P, int A, float damping) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const float vi = v[i];
  out[i] = (i < A) ? fmaf(damping, vi, 2.f * vi / static_cast<float>(A)) : fmaf(damping, vi, out[i]);
}

size_t trust_smem_bytes(int D, int A, int mode) {
  size_t f = spo_net_smem_floats(D, A, true) + (mode == MODE_FVP ? spo_net_smem_floats(D, A, false) : 0) +
             SPO_ROWS * spo_ld(D) + 3 * SPO_ROWS * SPO_LDH + 3 * SPO_ROWS * SPO_MAX_ACT + 672 + 8;
  return f * sizeof(float);
}

template <int MODE>
int launch_trust(const TrArgs& a, cudaStream_t st) {
  const size_t smem = trust_smem_bytes(a.D, a.A, MODE);
  SPO_REQUIRE(smem <= 227 * 1024, SPO_ERR_UNSUPPORTED, "trust-region kernel: obs_dim=%d needs %zu B shared memory", a.D, smem);
  const int64_t n_tiles = (a.count + SPO_ROWS - 1) / SPO_ROWS;
  const int grid = static_cast<int>(n_tiles < spo_sm_count() ? n_tiles : spo_sm_count());
  if (spo_pad4(a.D) <= 64) {
    SPO_CUDA_TRY(cudaFuncSetAttribute(spo_trust_kernel<MODE, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    spo_trust_kernel<MODE, 1><<<grid, SPO_THREADS, smem, st>>>(a);
  } else {
    SPO_CUDA_TRY(cudaFuncSetAttribute(spo_trust_kernel<MODE, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    spo_trust_kernel<MODE, 2><<<grid, SPO_THREADS, smem, st>>>(a);
  }
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

// ---- conjugate gradient vector kernel (single CTA; P_a ~ 1e4) ---------------------------
// state: x (out), r, p, z in work[0..3P), scalars at work + 4P: [0] rdotr [1] done
__device__ float block_dot(const float* a, const float* b, int n, float* red) {
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s = fmaf(a[i], b[i], s);
  s = spo_warp_sum(s);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < (blockDim.x >> 5); ++i) t += red[i];
  return t;
}

__global__ void __launch_bounds__(1024) spo_cg_init_kernel(const float* b, float* x, float* r, float* p, float* sc, int n) {
  __shared__ float red[32];
  for (int i = threadIdx.x; i < n; i += blockDim.x) { x[i] = 0.f; r[i] = b[i]; p[i] = b[i]; }   // fvp(0) == 0 exactly (cpo.py:91)
  __syncthreads();
  const float rr = block_dot(r, r, n, red);
  if (threadIdx.x == 0) { sc[0] = rr; sc[1] = 0.f; }
}

__global__ void __launch_bounds__(1024) spo_cg_step_kernel(float* x, float* r, float* p, const float* z, float* sc, int n,
                                                           float tol, float eps) {
  __shared__ float red[32];
  if (sc[1] != 0.f) return;   // residual test tripped earlier (cpo.py:101)
  const float rdotr = sc[0];
  const float pz = block_dot(p, z, n, red);
  const float alpha = rdotr / (pz + eps);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    x[i] = fmaf(alpha, p[i], x[i]);
    r[i] = fmaf(-alpha, z[i], r[i]);
  }
  __syncthreads();
  const float nrr = block_dot(r, r, n, red);
  if (sqrtf(nrr) < tol) {
    if (threadIdx.x == 0) sc[1] = 1.f;
    return;
  }
  const float mu = nrr / (rdotr + eps);
  for (int i = threadIdx.x; i < n; i += blockDim.x) p[i] = fmaf(mu, p[i], r[i]);
  if (threadIdx.x == 0) sc[0] = nrr;
}

int check_trust_args(const spo_dims* d, const float* params, const float* obs, int64_t count, const char* who) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(params && obs && count > 0, SPO_ERR_INVALID_ARG, "%s: null params/obs or count<=0", who);
  return SPO_OK;
}

}  // namespace

extern "C" {

int spo_surrogate_grad(const spo_dims* d, const float* params, const float* obs, const float* act,
                       const float* logp_old, const float* adv, int64_t count,
                       float* out_loss, float* grad, void* stream) {
  int rc = check_trust_args(d, params, obs, count, "spo_surrogate_grad");
  if (rc) return rc;
  SPO_REQUIRE(act && logp_old && adv && out_loss && grad, SPO_ERR_INVALID_ARG, "spo_surrogate_grad: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const SpoNetOff off = spo_net_off(d->obs_dim, d->act_dim, 0);
  SPO_CUDA_TRY(cudaMemsetAsync(grad, 0, sizeof(float) * off.count, st));
  SPO_CUDA_TRY(cudaMemsetAsync(out_loss, 0, sizeof(float), st));
  TrArgs a{};
  a.params = params; a.obs = obs; a.act = act; a.logp_old = logp_old; a.adv_a = adv; a.out = grad; a.out_loss = out_loss;
  a.count = count; a.D = d->obs_dim; a.A = d->act_dim;
  return launch_trust<MODE_GRAD>(a, st);
}

int spo_fvp(const spo_dims* d, const float* params, const float* obs, int64_t count,
            const float* v, float damping, float* out, void* stream) {
  int rc = check_trust_args(d, params, obs, count, "spo_fvp");
  if (rc) return rc;
  SPO_REQUIRE(v && out && v != out, SPO_ERR_INVALID_ARG, "spo_fvp: null or aliased v/out");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const SpoNetOff off = spo_net_off(d->obs_dim, d->act_dim, 0);
  SPO_CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(float) * off.count, st));
  TrArgs a{};
  a.params = params; a.obs = obs; a.v = v; a.out = out; a.count = count; a.D = d->obs_dim; a.A = d->act_dim;
  rc = launch_trust<MODE_FVP>(a, st);
  if (rc) return rc;
  spo_fvp_finalize_kernel<<<(off.count + 255) / 256, 256, 0, st>>>(out, v, off.count, d->act_dim, damping);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_linesearch_eval(const spo_dims* d, const float* params, const float* obs, const float* act,
                        const float* logp_old, const float* adv_a, const float* adv_b,
                        const float* old_mean, const float* old_log_std, int64_t count,
                        float* out3, void* stream) {
  int rc = check_trust_args(d, params, obs, count, "spo_linesearch_eval");
  if (rc) return rc;
  SPO_REQUIRE(act && logp_old && adv_a && old_mean && old_log_std && out3, SPO_ERR_INVALID_ARG, "spo_linesearch_eval: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SPO_CUDA_TRY(cudaMemsetAsync(out3, 0, 3 * sizeof(float), st));
  TrArgs a{};
  a.params = params; a.obs = obs; a.act = act; a.logp_old = logp_old; a.adv_a = adv_a; a.adv_b = adv_b;
  a.old_mean = old_mean; a.old_log_std = old_log_std; a.out = out3; a.count = count; a.D = d->obs_dim; a.A = d->act_dim;
  return launch_trust<MODE_EVAL>(a, st);
}

// Data-parallel ranks cannot use the monolithic solver below: every Fisher-vector product has to be averaged across the
// ranks before the step that consumes it (SURVEY section 8e, exchange 3').  The same two vector kernels, one call each:
//   spo_cg_begin   x = 0, r = p = b, rdotr = r.r                (work: r | p | z | - | scalars, like spo_conjugate_gradient)
//   (host)         spo_fvp(p = work + P  ->  z = work + 2P), all-reduce z, ...
//   spo_cg_update  one iteration of cpo.py:92-105 with the z it finds in work + 2P
int spo_cg_begin(const spo_dims* d, const float* b, float* x, float* work, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(b && x && work, SPO_ERR_INVALID_ARG, "spo_cg_begin: null argument");
  const int P = spo_net_off(d->obs_dim, d->act_dim, 0).count;
  spo_cg_init_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(b, x, work, work + P, work + 4 * P, P);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_cg_update(const spo_dims* d, float* x, float* work, float residual_tol, float eps, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(x && work, SPO_ERR_INVALID_ARG, "spo_cg_update: null argument");
  const int P = spo_net_off(d->obs_dim, d->act_dim, 0).count;
  spo_cg_step_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(x, work, work + P, work + 2 * P, work + 4 * P, P, residual_tol, eps);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_conjugate_gradient(const spo_dims* d, const float* params, const float* obs, int64_t count,
                           const float* b, int iters, float damping, float residual_tol, float eps,
                           float* x, float* work, void* stream) {
  int rc = check_trust_args(d, params, obs, count, "spo_conjugate_gradient");
  if (rc) return rc;
  SPO_REQUIRE(b && x && work && iters >= 0, SPO_ERR_INVALID_ARG, "spo_conjugate_gradient: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int P = spo_net_off(d->obs_dim, d->act_dim, 0).count;
  float *r = work, *p = work + P, *z = work + 2 * P, *sc = work + 4 * P;
  spo_cg_init_kernel<<<1, 1024, 0, st>>>(b, x, r, p, sc, P);
  SPO_CUDA_TRY(cudaGetLastError());
  for (int it = 0; it < iters; ++it) {
    rc = spo_fvp(d, params, obs, count, p, damping, z, stream);
    if (rc) return rc;
    spo_cg_step_kernel<<<1, 1024, 0, st>>>(x, r, p, z, sc, P, residual_tol, eps);
    SPO_CUDA_TRY(cudaGetLastError());
  }
  return SPO_OK;
}

}  // extern "C"
