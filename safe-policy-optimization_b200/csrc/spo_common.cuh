// Shared device/host helpers of libspo (sm_90a).
//
// Tile convention used by every MLP kernel in this library: a CTA of 256 threads works on
// a tile of 64 rows (samples).  Activations live in shared memory sample-major,
// act[r][f] with row stride LDH=68 floats (68 = 4*17: float4-aligned rows whose 16-byte
// chunks rotate through all eight bank groups).  A layer is a 64x64xK register-tiled FFMA
// GEMM: each thread owns a 4x4 output tile, both operands are read as float4.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "spo.h"

#define SPO_HID 64        // hidden width (both layers)
#define SPO_ROWS 64       // rows (samples) per CTA tile
#define SPO_THREADS 256   // threads per CTA: 16x16 thread tiles of 4x4
#define SPO_LDH 68        // row stride of 64-wide sample-major activations / transposed weights
#define SPO_MAX_OBS 128
#define SPO_MAX_ACT 8        // action capacity of the narrow kernel instantiations and of the wgmma forward kernel
#define SPO_MAX_ACT_WIDE 16  // act_dim limit of the single-agent API: 9..16 run the kernels' AC = 16 instantiations

void spo_set_error(const char* fmt, ...);

#define SPO_CUDA_TRY(expr)                                                            \
  do {                                                                                \
    cudaError_t e__ = (expr);                                                         \
    if (e__ != cudaSuccess) {                                                         \
      spo_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
      return SPO_ERR_CUDA;                                                            \
    }                                                                                 \
  } while (0)

#define SPO_REQUIRE(cond, code, ...)                                                  \
  do {                                                                                \
    if (!(cond)) {                                                                    \
      spo_set_error(__VA_ARGS__);                                                     \
      return (code);                                                                  \
    }                                                                                 \
  } while (0)

int spo_check_dims(const spo_dims* d);
// Observation rows are read as float4 (spo_load_rows, the wgmma kernel's TMA map) whenever obs_dim % 4 == 0, so such
// an obs array must be 16-byte aligned; other obs_dims are read one float at a time.
inline bool spo_obs_aligned(const float* obs, int D) { return (D & 3) != 0 || (reinterpret_cast<uintptr_t>(obs) & 15) == 0; }
// streaming multiprocessors of the current device (sizes the persistent grids; queried once per process)
int spo_sm_count();

// ---- packed parameter layout ---------------------------------------------------------
struct SpoNetOff {
  int log_std, w1, b1, w2, b2, w3, b3, count, out;  // absolute float offsets; log_std = -1 for critics
};

__host__ __device__ inline SpoNetOff spo_net_off(int D, int A, int net) {
  const int H = SPO_HID;
  const int actor_count = A + H * D + H + H * H + H + A * H + A;
  const int critic_count = H * D + H + H * H + H + H + 1;
  SpoNetOff o;
  int base = 0;
  if (net == 0) {
    o.log_std = 0;
    base = A;
    o.out = A;
    o.count = actor_count;
  } else {
    o.log_std = -1;
    base = actor_count + (net - 1) * critic_count;
    o.out = 1;
    o.count = critic_count;
  }
  o.w1 = base;
  o.b1 = o.w1 + H * D;
  o.w2 = o.b1 + H;
  o.b2 = o.w2 + H * H;
  o.w3 = o.b2 + H;
  o.b3 = o.w3 + o.out * H;
  return o;
}

__host__ __device__ inline int spo_pad4(int k) { return (k + 3) & ~3; }
// leading dimension (floats) of a sample-major [rows][K] tile: float4 aligned and
// == 4 (mod 8) so that rows 4 apart fall in different bank groups.
__host__ __device__ inline int spo_ld(int k) {
  int k4 = spo_pad4(k);
  return (k4 % 8 == 0) ? k4 + 4 : k4;
}

// ---- shared-memory images of one net's weights -----------------------------------------
// w1t [Dp][LDH]  (transposed: w1t[k][j] = W1[j][k]; rows k >= D are zero)
// w2t [64][LDH]  (w2t[k][j] = W2[j][k])
// w2  [64][LDH]  (natural; only for backward / JVP kernels)
// w3  [O][64], b1 b2 [64], b3 [O]
struct SpoNetSmem {
  float *w1t, *b1, *w2t, *b2, *w3, *b3, *w2;
};

__host__ __device__ inline int spo_net_smem_floats(int D, int O, bool with_w2) {
  return spo_pad4(D) * SPO_LDH + SPO_HID + SPO_HID * SPO_LDH + SPO_HID + spo_pad4(O * SPO_HID) + spo_pad4(O) +
         (with_w2 ? SPO_HID * SPO_LDH : 0);
}

__device__ inline float* spo_carve_net(float* p, int D, int O, bool with_w2, SpoNetSmem& s) {
  s.w1t = p; p += spo_pad4(D) * SPO_LDH;
  s.b1 = p;  p += SPO_HID;
  s.w2t = p; p += SPO_HID * SPO_LDH;
  s.b2 = p;  p += SPO_HID;
  s.w3 = p;  p += spo_pad4(O * SPO_HID);
  s.b3 = p;  p += spo_pad4(O);
  s.w2 = nullptr;
  if (with_w2) { s.w2 = p; p += SPO_HID * SPO_LDH; }
  return p;
}

// Load one net from the packed global buffer into its smem image (all threads of the CTA).
__device__ inline void spo_load_net(const float* __restrict__ params, const SpoNetOff& o, int D,
                                    const SpoNetSmem& s, int tid, int nthreads) {
  const int Dp = spo_pad4(D);
  for (int i = tid; i < SPO_HID * D; i += nthreads) {
    int j = i / D, k = i - j * D;
    s.w1t[k * SPO_LDH + j] = __ldg(params + o.w1 + i);
  }
  for (int i = tid; i < (Dp - D) * SPO_HID; i += nthreads) {
    int k = D + i / SPO_HID, j = i % SPO_HID;
    s.w1t[k * SPO_LDH + j] = 0.f;
  }
  for (int i = tid; i < SPO_HID * SPO_HID; i += nthreads) {
    int j = i >> 6, k = i & 63;
    float w = __ldg(params + o.w2 + i);
    s.w2t[k * SPO_LDH + j] = w;
    if (s.w2) s.w2[j * SPO_LDH + k] = w;
  }
  for (int i = tid; i < SPO_HID; i += nthreads) {
    s.b1[i] = __ldg(params + o.b1 + i);
    s.b2[i] = __ldg(params + o.b2 + i);
  }
  for (int i = tid; i < o.out * SPO_HID; i += nthreads) s.w3[i] = __ldg(params + o.w3 + i);
  for (int i = tid; i < o.out; i += nthreads) s.b3[i] = __ldg(params + o.b3 + i);
}

// ---- register-tiled smem GEMM ----------------------------------------------------------
// Thread -> output tile map of a 64x64 output (256 threads, 4x4 outputs each).  A warp owns a
// 32(m) x 16(n) patch: its 32 lanes cover 8 m-tiles x 4 n-tiles, so one warp-wide LDS.128 of
// the A operand touches 8 distinct 16-byte chunks (128 contiguous bytes, one wavefront) and
// one of the B operand 4 (a 16 x 2 arrangement keeps the LSU busier than the FMA pipe).
//   m0           = first of 4 consecutive m
//   spo_nb(tid)  = first of 4 consecutive n          (B k-major: float4 along n)
//   spo_ns(tid)  = first of 4 n spaced 4 apart       (B n-major: rows ns, ns+4, ns+8, ns+12 --
//                  the 4 n-tiles of a warp then read 4 consecutive rows per LDS, which are
//                  conflict-free for every leading dimension == 4 (mod 8))
__device__ __forceinline__ int spo_m0(int tid) { return ((((tid >> 5) & 1) << 3) + (tid & 7)) << 2; }
__device__ __forceinline__ int spo_nb(int tid) { return (((tid >> 6) << 2) + ((tid >> 3) & 3)) << 2; }
__device__ __forceinline__ int spo_ns(int tid) { return ((tid >> 6) << 4) + ((tid >> 3) & 3); }

// acc[mi][ni] += sum_k A[k][m0+mi] * B(n(ni), k),  k in [0,K), K % 4 == 0.
//   A is reduction-major: A[k*lda + m]   (float4 along m)
//   B_N_MAJOR : B[n*ldb + k] (float4 along k), n(ni) = n0 + 4*ni     (pass n0 = spo_ns(tid))
//   else      : B[k*ldb + n] (float4 along n), n(ni) = n0 + ni       (pass n0 = spo_nb(tid))
template <bool B_N_MAJOR>
__device__ __forceinline__ void spo_tile_mma(float (&acc)[4][4], const float* __restrict__ A, int lda,
                                             const float* __restrict__ B, int ldb, int m0, int n0, int K) {
#pragma unroll 2
  for (int k = 0; k < K; k += 4) {
    float4 a[4], b[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const float4*>(A + (k + i) * lda + m0);
    if (B_N_MAJOR) {
#pragma unroll
      for (int i = 0; i < 4; ++i) b[i] = *reinterpret_cast<const float4*>(B + (n0 + 4 * i) * ldb + k);
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        const float bk[4] = {b[ni].x, b[ni].y, b[ni].z, b[ni].w};
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          acc[0][ni] = fmaf(a[kk].x, bk[kk], acc[0][ni]);
          acc[1][ni] = fmaf(a[kk].y, bk[kk], acc[1][ni]);
          acc[2][ni] = fmaf(a[kk].z, bk[kk], acc[2][ni]);
          acc[3][ni] = fmaf(a[kk].w, bk[kk], acc[3][ni]);
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) b[i] = *reinterpret_cast<const float4*>(B + (k + i) * ldb + n0);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const float bn[4] = {b[kk].x, b[kk].y, b[kk].z, b[kk].w};
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
          acc[0][ni] = fmaf(a[kk].x, bn[ni], acc[0][ni]);
          acc[1][ni] = fmaf(a[kk].y, bn[ni], acc[1][ni]);
          acc[2][ni] = fmaf(a[kk].z, bn[ni], acc[2][ni]);
          acc[3][ni] = fmaf(a[kk].w, bn[ni], acc[3][ni]);
        }
      }
    }
  }
}

__device__ __forceinline__ void spo_zero(float (&acc)[4][4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
}

// torch's tanh on CPU is the correctly-rounded-ish libm/sleef tanhf; CUDA tanhf is
// <= 1-2 ulp.  (Never tanh.approx here: parity bar is 1e-5 relative on losses.)
__device__ __forceinline__ float spo_tanh(float x) { return tanhf(x); }

// tanh for the epilogues: 1 - 2/(exp(2|x|)+1) on the SFU (ex2 + rcp) for |x| >= 0.04 and
// the odd Taylor polynomial below that (absolute error < 3e-7 overall, relative < 2e-7 near
// 0); tanhf costs ~25 dependent instructions per element, which made the v1 epilogue
// the bottleneck of this kernel.
__device__ __forceinline__ float spo_tanh_fast(float x) {
  const float ax = fabsf(x);
  const float x2 = x * x;
  const float poly = x * fmaf(x2, fmaf(x2, fmaf(x2, -0.053968254f, 0.13333334f), -0.33333334f), 1.f);
  const float e = __expf(2.f * ax);
  const float big = copysignf(1.f - __fdividef(2.f, e + 1.f), x);
  return ax < 0.04f ? poly : big;
}


// Hidden layer forward for a 64-row tile:  out[r][j] = tanh(b[j] + sum_k in[r][k] * wt[k][j]).
// in: sample-major [64][ldin] with K (multiple of 4) valid columns; out: [64][LDH].
// Thread tile: units j = m0..m0+3, rows r = ns, ns+4, ns+8, ns+12.
__device__ __forceinline__ void spo_hidden_fwd(const float* __restrict__ in, int ldin, int K,
                                               const float* __restrict__ wt, const float* __restrict__ bias,
                                               float* __restrict__ out, int tid) {
  const int m0 = spo_m0(tid), ns = spo_ns(tid);
  float acc[4][4];
  spo_zero(acc);
  spo_tile_mma<true>(acc, wt, SPO_LDH, in, ldin, m0, ns, K);
  const float4 b = *reinterpret_cast<const float4*>(bias + m0);
#pragma unroll
  for (int ni = 0; ni < 4; ++ni) {
    float4 h;
    h.x = spo_tanh(acc[0][ni] + b.x);
    h.y = spo_tanh(acc[1][ni] + b.y);
    h.z = spo_tanh(acc[2][ni] + b.z);
    h.w = spo_tanh(acc[3][ni] + b.w);
    *reinterpret_cast<float4*>(out + (ns + 4 * ni) * SPO_LDH + m0) = h;
  }
}

// Output layer: y[r][o] = b3[o] + sum_k h2[r][k] * w3[o][k], O <= 8.  Work items (r,o)
// are spread over the CTA; result written to out[r*ldo + o].
__device__ __forceinline__ void spo_out_fwd(const float* __restrict__ h2, const float* __restrict__ w3,
                                            const float* __restrict__ b3, int O, float* __restrict__ out,
                                            int ldo, int tid, int nthreads) {
  for (int w = tid; w < SPO_ROWS * O; w += nthreads) {
    const int r = w / O, o = w - r * O;
    const float4* hp = reinterpret_cast<const float4*>(h2 + r * SPO_LDH);
    const float4* wp = reinterpret_cast<const float4*>(w3 + o * SPO_HID);
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
    for (int k = 0; k < SPO_HID / 4; ++k) {
      float4 a = hp[k], b = wp[k];
      s0 = fmaf(a.x, b.x, s0); s1 = fmaf(a.y, b.y, s1); s2 = fmaf(a.z, b.z, s2); s3 = fmaf(a.w, b.w, s3);
    }
    out[r * ldo + o] = ((s0 + s1) + (s2 + s3)) + b3[o];
  }
}

// Load `rows` observation rows (global row-major, D floats each, row r at src + idx(r)*D)
// into a zero-padded sample-major smem tile x[64][ldx].  gather != nullptr: idx(r) =
// gather[r] else idx(r) = row0 + r.  Rows >= rows and columns >= D are zeroed.
__device__ __forceinline__ void spo_load_rows(const float* __restrict__ src, int D, int ldx,
                                              const int64_t* __restrict__ gather, int64_t row0, int rows,
                                              float* __restrict__ x, int tid, int nthreads) {
  const int Dp = spo_pad4(D);
  if ((D & 3) == 0) {
    const int c4 = D >> 2;
    for (int i = tid; i < SPO_ROWS * c4; i += nthreads) {
      const int r = i / c4, c = i - r * c4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < rows) {
        const int64_t g = gather ? gather[r] : row0 + r;
        v = __ldg(reinterpret_cast<const float4*>(src + g * D) + c);
      }
      *reinterpret_cast<float4*>(x + r * ldx + 4 * c) = v;
    }
  } else {
    for (int i = tid; i < SPO_ROWS * Dp; i += nthreads) {
      const int r = i / Dp, c = i - r * Dp;
      float v = 0.f;
      if (r < rows && c < D) {
        const int64_t g = gather ? gather[r] : row0 + r;
        v = __ldg(src + g * D + c);
      }
      x[r * ldx + c] = v;
    }
  }
}

// ---- reductions ------------------------------------------------------------------------
__device__ __forceinline__ float spo_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double spo_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- Philox4x32-10 + Box-Muller (perf-mode sampling; parity mode takes eps from host) ---
__device__ __forceinline__ uint4 spo_philox(uint4 ctr, uint2 key) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += 0x9E3779B9u;
    key.y += 0xBB67AE85u;
  }
  return ctr;
}
__device__ __forceinline__ float2 spo_box_muller(uint32_t a, uint32_t b) {
  const float u1 = (static_cast<float>(a) + 0.5f) * 2.3283064365386963e-10f;  // (0,1)
  const float u2 = (static_cast<float>(b) + 0.5f) * 2.3283064365386963e-10f;
  const float rad = sqrtf(-2.f * logf(u1));
  float s, c;
  sincosf(6.283185307179586f * u2, &s, &c);
  return make_float2(rad * c, rad * s);
}
