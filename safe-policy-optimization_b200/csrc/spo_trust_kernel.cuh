// The persistent full-batch kernel of the trust-region pieces (csrc/spo_trust.cu), templated on the action capacity.
// act_dim <= 8 runs the AC = 8 instantiations, compiled in spo_trust.cu; 9..16 the AC = 16 ones, compiled in
// spo_trust_wide.cu.  Keeping the two apart keeps the AC = 8 code exactly what it was before AC existed: with both in one
// translation unit the compiler's inlining choices for the shared helpers change.
#pragma once
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

}  // namespace

// the AC = 16 launcher (spo_trust_wide.cu); args: a TrArgs.  (TrArgs keeps internal linkage: given external linkage, the
// compiler's choices for the AC = 8 code change too.)
int spo_trust_launch_wide(int mode, const void* args, cudaStream_t st);

namespace {

// tangent vector viewed as a second set of actor weights (same packed order, offset by -0:
// v is actor-flat so the SpoNetOff of net 0 applies directly)
__device__ inline void load_tangent(const float* __restrict__ v, const SpoNetOff& o, int D, const SpoNetSmem& s, int tid) {
  spo_load_net(v, o, D, s, tid, SPO_THREADS);
}

// Action capacity AC (8 or 16): the per-row output buffers y / gy / gl are [64][AC]; act_dim <= 8 runs AC = 8.
// Small-parameter gradient slots: b1[64] b2[64] w3[A*64] b3[A] log_std[A], padded (672 floats at AC = 8).
template <int AC>
__host__ __device__ constexpr int trust_gsmall_floats() { return AC * (SPO_HID + 2) + 2 * SPO_HID + 16; }
// The FVP has no use for gl; at AC = 16 it leaves it out, which keeps obs_dim 128 / act_dim 16 under 227 KB.
template <int MODE, int AC>
__host__ __device__ constexpr bool trust_has_gl() { return !(MODE == MODE_FVP && AC > 8); }

template <int MODE, int NT1, int AC>
__global__ void __launch_bounds__(SPO_THREADS, 1) spo_trust_kernel(const TrArgs a) {
  constexpr int GSN = trust_gsmall_floats<AC>();
  static_assert(trust_gsmall_floats<8>() == 672, "AC = 8 layout");
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
  float* y = p;   p += SPO_ROWS * AC;
  float* gy = p;  p += SPO_ROWS * AC;
  float* gl = p;  if (trust_has_gl<MODE, AC>()) p += SPO_ROWS * AC;   // GRAD: per-row d/dlog_std
  float* gsmall = p; p += GSN;                   // b1[64] b2[64] w3[A*64] b3[A] log_std[A]
  float* ls = p;  p += AC;

  spo_load_net(a.params, off, D, w, tid, SPO_THREADS);
  if (MODE == MODE_FVP) load_tangent(a.v, off, D, tv, tid);
  if (tid < A) ls[tid] = a.params[off.log_std + tid];
  const int SP = 2 * SPO_HID + A * SPO_HID + 2 * A;
  for (int i = tid; i < GSN; i += SPO_THREADS) gsmall[i] = 0.f;

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
      spo_out_fwd(h2, w.w3, w.b3, A, y, AC, tid, SPO_THREADS);
      __syncthreads();
    }

    if (MODE == MODE_EVAL || MODE == MODE_GRAD) {
      if (tid < SPO_ROWS) {
        const int r = tid;
        const bool valid = r < rows;
        const int64_t g = row0 + (valid ? r : 0);
        float lp = 0.f, kl = 0.f;
        float dmu[AC], dl[AC];
#pragma unroll
        for (int j = 0; j < AC; ++j) {
          dmu[j] = dl[j] = 0.f;
          if (j < A) {
            const float mean = y[r * AC + j];
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
          for (int j = 0; j < AC; ++j) {
            gy[r * AC + j] = __fmul_rn(c, dmu[j]);
            gl[r * AC + j] = __fmul_rn(c, dl[j]);
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
      spo_out_fwd(dz, w.w3, tv.b3, A, y, AC, tid, SPO_THREADS);   // dh2 W3^T + c3
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
        gy[r * AC + o] = s;
      }
      __syncthreads();
      constexpr int AC_LOG2 = AC == 8 ? 3 : 4;
      for (int wi = tid; wi < SPO_ROWS * AC; wi += SPO_THREADS) {
        const int r = wi >> AC_LOG2, o = wi & (AC - 1);
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
        for (int r = 0; r < SPO_ROWS; ++r) s = fmaf(gy[r * AC + o], h2[r * SPO_LDH + k], s);
      } else if (i < A * SPO_HID + A) {
        const int o = i - A * SPO_HID;
        for (int r = 0; r < SPO_ROWS; ++r) s += gy[r * AC + o];
      } else {
        const int j = i - A * SPO_HID - A;
        for (int r = 0; r < SPO_ROWS; ++r) s += gl[r * AC + j];
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
          const float d = gy[r * AC + o];
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

// FVP at obs_dim 128: 221 920 B at act_dim 8 (AC = 8), 230 272 B at act_dim 16 (AC = 16, no gl buffer)
template <int MODE, int AC>
size_t trust_smem_bytes(int D, int A) {
  size_t f = spo_net_smem_floats(D, A, true) + (MODE == MODE_FVP ? spo_net_smem_floats(D, A, false) : 0) +
             SPO_ROWS * spo_ld(D) + 3 * SPO_ROWS * SPO_LDH + (trust_has_gl<MODE, AC>() ? 3 : 2) * SPO_ROWS * AC +
             trust_gsmall_floats<AC>() + AC;
  return f * sizeof(float);
}

template <int MODE, int AC>
int launch_trust_ac(const TrArgs& a, cudaStream_t st) {
  const size_t smem = trust_smem_bytes<MODE, AC>(a.D, a.A);
  SPO_REQUIRE(smem <= 227 * 1024, SPO_ERR_UNSUPPORTED, "trust-region kernel: obs_dim=%d needs %zu B shared memory", a.D, smem);
  const int64_t n_tiles = (a.count + SPO_ROWS - 1) / SPO_ROWS;
  const int grid = static_cast<int>(n_tiles < spo_sm_count() ? n_tiles : spo_sm_count());
  if (spo_pad4(a.D) <= 64) {
    SPO_CUDA_TRY(cudaFuncSetAttribute(spo_trust_kernel<MODE, 1, AC>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    spo_trust_kernel<MODE, 1, AC><<<grid, SPO_THREADS, smem, st>>>(a);
  } else {
    SPO_CUDA_TRY(cudaFuncSetAttribute(spo_trust_kernel<MODE, 2, AC>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    spo_trust_kernel<MODE, 2, AC><<<grid, SPO_THREADS, smem, st>>>(a);
  }
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

}  // namespace
