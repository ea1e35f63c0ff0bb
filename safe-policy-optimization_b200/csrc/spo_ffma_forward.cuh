// The FFMA tile kernel of the single-agent forward family (csrc/spo_forward.cu), templated on the action capacity AC.
// act_dim <= 8 runs AC = 8, instantiated in spo_forward.cu; 9..16 runs AC = 16, instantiated in spo_forward_wide.cu.  Keeping
// the two apart keeps the AC = 8 code exactly what it was before AC existed: with both in one translation unit the compiler's
// inlining choices for the shared helpers change.
#pragma once
#include "spo_forward.cuh"

// the AC = 16 launcher (spo_forward_wide.cu)
int spo_ffma_forward_launch_wide(const SpoFwdArgs& a, cudaStream_t stream);

namespace {

// 64-row tiles, weights of net net_base + blockIdx.y resident in shared memory.  Grid (ceil(n/64), nets) for the step,
// persistent min(tiles, 2 x SMs) for the full-batch modes, which therefore needs two CTAs per SM (<= 128 registers;
// no minimum-blocks launch bound: with one, ptxas spends the whole 128 on the tile loop and the obs-27 passes slow down).
// AC: action capacity, the row stride of the output staging tile y (8 for act_dim <= 8, 16 for 9..16).
template <int AC>
__global__ void __launch_bounds__(SPO_THREADS) spo_ffma_forward_kernel(const SpoFwdArgs a) {
  extern __shared__ __align__(16) float smem[];
  __shared__ double red[SPO_THREADS / 32];
  const int tid = threadIdx.x;
  if (spo_fwd_is_kl(a.mode) && *reinterpret_cast<volatile int*>(&a.ctrl->stop)) return;
  const int net = a.net_base + blockIdx.y;
  const int D = a.D, Dp = spo_pad4(D), ldx = spo_ld(D);
  const SpoNetOff off = spo_net_off(D, a.A, net);
  const int O = off.out;
  SpoNetSmem w;
  float* p = spo_carve_net(smem, D, O, false, w);
  float* x = p;  p += SPO_ROWS * ldx;
  float* h1 = p; p += SPO_ROWS * SPO_LDH;
  float* h2 = p; p += SPO_ROWS * SPO_LDH;
  float* y = p;  // [64][AC]

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
    spo_out_fwd(h2, w.w3, w.b3, O, y, AC, tid, SPO_THREADS);
    __syncthreads();
    if (a.mode == SpoFwdMode::kMeans) {
      // all threads, coalesced: one thread per row would write A floats at a stride of A
      for (int i = tid; i < rows * O; i += SPO_THREADS) {
        const int r = i / O, j = i - r * O;
        a.mean_out[(row0 + r) * O + j] = y[r * AC + j];
      }
    } else if (tid < rows) {
      acc += static_cast<double>(spo_forward_row(a, net, row0 + tid, y + tid * AC, a.params + off.log_std, a.old_log_std));
    }
    if (a.mode == SpoFwdMode::kStep && net == 0 && a.has_store) {
      // observation rows into slot t (buffer.py:91-95), bit-exact from the shared tile
      const int T = a.store.steps;
      for (int i = tid; i < rows * D; i += SPO_THREADS) {
        const int r = i / D, c = i - r * D;
        a.store.obs[((row0 + r) * T + a.t) * D + c] = x[r * ldx + c];
      }
    }
  }
  if (!spo_fwd_is_kl(a.mode)) return;
  acc = spo_warp_sum(acc);
  if ((tid & 31) == 0) red[tid >> 5] = acc;
  __syncthreads();
  if (tid == 0) {
    double s = 0.0;
    for (int i = 0; i < SPO_THREADS / 32; ++i) s += red[i];
    spo_kl_pass_add(a, s);
  }
}

template <int AC>
int ffma_forward_launch(const SpoFwdArgs& a, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    SPO_CUDA_TRY(cudaFuncSetAttribute(spo_ffma_forward_kernel<AC>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  const size_t smem = sizeof(float) * (spo_net_smem_floats(a.D, a.A, false) + SPO_ROWS * spo_ld(a.D) +
                                       2 * SPO_ROWS * SPO_LDH + SPO_ROWS * AC);
  const int64_t n_tiles = (a.count + SPO_ROWS - 1) / SPO_ROWS;
  const dim3 grid = (a.mode == SpoFwdMode::kStep)
                        ? dim3(static_cast<unsigned>(n_tiles), a.net_base == 0 ? 3 : 2)
                        : dim3(static_cast<unsigned>(n_tiles < 2 * spo_sm_count() ? n_tiles : 2 * spo_sm_count()));   // 2 CTAs per SM
  spo_ffma_forward_kernel<AC><<<grid, SPO_THREADS, smem, stream>>>(a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

}  // namespace
