// MLP forward passes on the Hopper tensor cores (wgmma + TMA).
//
// Serves (a) spo_actor_forward / spo_actor_kl / spo_actor_kl_accumulate for large batches
// (reference: safepo/single_agent/ppo_lag.py:277 and :338-344 -- policy.actor(data["obs"])
// over S = 1,024,000 observations and the KL against the old distribution), and
// (b) spo_policy_step / spo_critic_values, the rollout forward of all three nets
// (safepo/common/model.py:149-170 ActorVCritic.step fused with buffer.py:84-95 store): one launch,
// grid (row tiles, nets); the actor CTAs sample, evaluate the log-density and write the
// transition straight into slot t of the env-major rollout arrays from the epilogue.
//
// Per 128-row tile of a persistent CTA (two warpgroups, warpgroup g owns rows [64g, 64g+64)):
//   TMA      obs tile [128 x D] -> smem, as a 3-D box (16-byte k-chunk, row, chunk index) so the
//            bytes land directly in the canonical K-major / no-swizzle wgmma operand layout
//            (chunks >= D/4 are zero-filled by the TMA unit: K is padded to 64 for free)
//   split    x -> (hi, lo) TF32 pair, hi = rna_tf32(x), lo = rna_tf32(x - hi)       (all 8 warps)
//   layer 1  D1[64x64] (registers) = Xhi*W1hi + Xhi*W1lo + Xlo*W1hi     24 x wgmma m64n64k8 tf32
//   epi 1    +b1 -> tanh -> (hi, lo) -> smem operand tile of layer 2 (own rows only)
//   layer 2  D2[64x64] (registers) = H1hi*W2hi + H1hi*W2lo + H1lo*W2hi
//   epi 2    +b2 -> tanh -> fp32 staging tile -> output layer (A <= 8 outputs) on CUDA cores,
//            one thread per (row, column half) -> mean write-back or KL(old || new) accumulation
// The next tile's observations are fetched by TMA as soon as both warpgroups have consumed the
// current x tile, under the two epilogues.
//
// 3xTF32 with rounded splits and small terms accumulated first reproduces fp32 GEMM
// accuracy (max |err| ~8e-7 on |values| <= 2.8 at K = 64), which the 1e-5 parity bar needs;
// single-pass TF32 (~7e-4) does not.
#include <cuda.h>
#include "spo_forward.cuh"

namespace {

constexpr int TC_ROWS = 128;                 // rows per tile = two wgmma M=64 blocks
constexpr int TC_THREADS = 256;              // two warpgroups
constexpr uint32_t X_LBO = TC_ROWS * 16;     // 2048 B between k-chunks of the 128-row tiles (TMA box order)
constexpr uint32_t W_LBO = SPO_HID * 16;     // 1024 B between k-chunks of the 64-row weight tiles
constexpr uint32_t SBO = 128;                // 8 rows x 16 B core matrices back to back
constexpr uint32_t X_TILE_BYTES = TC_ROWS * 64 * 4;   // 32 KB
constexpr uint32_t W_TILE_BYTES = SPO_HID * 64 * 4;   // 16 KB

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ float rna_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

__device__ __forceinline__ float tanh_fast(float x) { return spo_tanh_fast(x); }

// wgmma shared-memory matrix descriptor, K-major without swizzle: LBO = bytes between the two
// 16-byte k-chunks of one k8 step, SBO = bytes between 8-row core matrices (layout type 0).
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr, uint32_t lbo) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>((lbo >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((SBO >> 4) & 0x3FFF) << 32;
  return d;
}

// D[64 x 64] (+)= A[64 x 8] * B[64 x 8]^T, both operands TF32 from shared memory.  Fragment of
// thread (warp w of the warpgroup, lane): d[i] = D(16w + lane/4 + 8((i>>1)&1), 8(i>>2) + 2(lane%4) + (i&1)).
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t da, uint64_t db, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "%32, %33, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accum));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  const long long t0 = clock64();
  while (!done) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}\n"
                 : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    if (!done && clock64() - t0 > 4000000000ll) asm volatile("trap;");   // ~2 s: a lost arrival must not hang the GPU
  }
}

__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(dst)),
               "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

// weight tile [64 out][64 in] of W (row-major [64][K], K <= 64) -> canonical (hi, lo) operand images
__device__ void load_weight_tile(const float* __restrict__ W, int K, float* hi, float* lo, int tid, int nthreads) {
  for (int i = tid; i < SPO_HID * 16; i += nthreads) {
    const int j = i >> 4, c = i & 15;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    float* pv = &v.x;
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (4 * c + e < K) pv[e] = __ldg(W + j * K + 4 * c + e);
    float4 h, l;
    h.x = rna_tf32(v.x); h.y = rna_tf32(v.y); h.z = rna_tf32(v.z); h.w = rna_tf32(v.w);
    l.x = rna_tf32(v.x - h.x); l.y = rna_tf32(v.y - h.y); l.z = rna_tf32(v.z - h.z); l.w = rna_tf32(v.w - h.w);
    const uint32_t off = c * W_LBO + j * 16;
    *reinterpret_cast<float4*>(reinterpret_cast<uint8_t*>(hi) + off) = h;
    *reinterpret_cast<float4*>(reinterpret_cast<uint8_t*>(lo) + off) = l;
  }
}

// 3xTF32 product of this warpgroup's 64 rows of an activation tile with a 64-row weight tile, K = 64, small
// terms first; returns with the products complete (the operand tiles may be overwritten afterwards).
__device__ __forceinline__ void wg_layer(float (&d)[32], const float* a_hi, const float* a_lo, const float* w_hi, const float* w_lo,
                                         int wg) {
  const uint32_t row_off = static_cast<uint32_t>(wg) * 64 * 16;
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
  uint32_t accum = 0;
#pragma unroll
  for (int pass = 0; pass < 3; ++pass) {
    const float* ap = (pass == 0) ? a_lo : a_hi;          // lo*hi, hi*lo, hi*hi
    const float* wp = (pass == 1) ? w_lo : w_hi;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      wgmma_tf32(d, wgmma_desc(smem_u32(ap) + row_off + ks * 2 * X_LBO, X_LBO), wgmma_desc(smem_u32(wp) + ks * 2 * W_LBO, W_LBO), accum);
      accum = 1;
    }
  }
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}

// fp32 staging tile [128][64] of the layer-2 activations, columns XOR-swizzled by row so that the
// row-per-lane reads of the output layer hit 32 distinct banks
__device__ __forceinline__ int stage_idx(int r, int c) { return r * SPO_HID + (c ^ (r & 31)); }

__global__ void __launch_bounds__(TC_THREADS, 1) spo_tc_forward_kernel(const __grid_constant__ CUtensorMap obs_map, const SpoFwdArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  float* x_hi = reinterpret_cast<float*>(smem);                          // TMA destination, rounded in place
  float* x_lo = reinterpret_cast<float*>(smem + X_TILE_BYTES);
  float* h_hi = reinterpret_cast<float*>(smem + 2 * X_TILE_BYTES);
  float* h_lo = reinterpret_cast<float*>(smem + 3 * X_TILE_BYTES);
  float* w1_hi = reinterpret_cast<float*>(smem + 4 * X_TILE_BYTES);
  float* w1_lo = w1_hi + W_TILE_BYTES / 4;
  float* w2_hi = w1_lo + W_TILE_BYTES / 4;
  float* w2_lo = w2_hi + W_TILE_BYTES / 4;
  float* small = w2_lo + W_TILE_BYTES / 4;                                // b1[64] b2[64] w3[A*64] b3[8] ls[8] ols[8]
  float* stage = x_lo;   // free between layer 1 of a tile and the split of the next one
  __shared__ __align__(8) uint64_t bar_x_full;
  __shared__ double red[8];
  __shared__ float pmean[TC_ROWS][SPO_MAX_ACT];   // partial output-layer sums of the upper column half, then the outputs

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;
  if (spo_fwd_is_kl(a.mode) && *reinterpret_cast<volatile int*>(&a.ctrl->stop)) return;
  const int D = a.D;
  const int net = a.net_base + static_cast<int>(blockIdx.y);
  const SpoNetOff off = spo_net_off(D, a.A, net);
  const int A = off.out;      // outputs of this net's last layer (act_dim for the actor, 1 for a critic)
  float* b1 = small; float* b2 = small + 64; float* w3 = small + 128; float* b3 = w3 + A * 64; float* ls = b3 + 8; float* ols = ls + 8;

  load_weight_tile(a.params + off.w1, D, w1_hi, w1_lo, tid, TC_THREADS);
  load_weight_tile(a.params + off.w2, SPO_HID, w2_hi, w2_lo, tid, TC_THREADS);
  for (int i = tid; i < SPO_HID; i += TC_THREADS) { b1[i] = a.params[off.b1 + i]; b2[i] = a.params[off.b2 + i]; }
  for (int i = tid; i < A * SPO_HID; i += TC_THREADS) w3[i] = a.params[off.w3 + i];
  if (tid < A) {
    b3[tid] = a.params[off.b3 + tid];
    ls[tid] = (net == 0) ? a.params[off.log_std + tid] : 0.f;
    ols[tid] = a.old_log_std ? a.old_log_std[tid] : 0.f;
  }
  if (tid == 0) {
    mbar_init(&bar_x_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;");
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // weight images -> visible to wgmma
  __syncthreads();

  const int64_t n_tiles = (a.count + TC_ROWS - 1) / TC_ROWS;
  double kl_acc = 0.0;
  // (the step launches one CTA per tile: the loop body runs once)
  uint32_t phase = 0;
  if (tid == 0 && static_cast<int64_t>(blockIdx.x) < n_tiles) {   // first tile's observations
    mbar_expect_tx(&bar_x_full, X_TILE_BYTES);
    tma_load_3d(x_hi, &obs_map, 0, static_cast<int>(static_cast<int64_t>(blockIdx.x) * TC_ROWS), 0, &bar_x_full);
  }
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, phase ^= 1) {
    const int64_t row0 = tile * TC_ROWS;
    // ---- split x into the TF32 pair (rows beyond the tensor were zero-filled by TMA) ----
    {
      const int quad = warp & 3, half = warp >> 2;
      const int r = quad * 32 + lane;
      mbar_wait(&bar_x_full, phase);
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const uint32_t o = (half * 8 + c) * X_LBO + r * 16;
        float4* ph = reinterpret_cast<float4*>(reinterpret_cast<uint8_t*>(x_hi) + o);
        float4* pl = reinterpret_cast<float4*>(reinterpret_cast<uint8_t*>(x_lo) + o);
        const float4 v = *ph;
        float4 h, l;
        h.x = rna_tf32(v.x); h.y = rna_tf32(v.y); h.z = rna_tf32(v.z); h.w = rna_tf32(v.w);
        l.x = rna_tf32(v.x - h.x); l.y = rna_tf32(v.y - h.y); l.z = rna_tf32(v.z - h.z); l.w = rna_tf32(v.w - h.w);
        *ph = h; *pl = l;
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    float d[32];
    wg_layer(d, x_hi, x_lo, w1_hi, w1_lo, wg);
    // the x tile is free once both warpgroups have consumed it: fetch the next tile's observations now,
    // under the two epilogues of this tile
    __syncthreads();
    if (tid == 0) {
      const int64_t next = tile + gridDim.x;
      if (next < n_tiles) {
        mbar_expect_tx(&bar_x_full, X_TILE_BYTES);
        tma_load_3d(x_hi, &obs_map, 0, static_cast<int>(next * TC_ROWS), 0, &bar_x_full);
      }
    }
    const int wr = 64 * wg + 16 * (warp & 3) + (lane >> 2);   // fragment rows wr and wr + 8
    // ---- epilogue 1: h1 = tanh(D1 + b1) -> operand tile of layer 2 (this warpgroup's rows) ----
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int r = wr + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + 2 * (lane & 3);
      const float t0 = tanh_fast(d[i] + b1[c]), t1 = tanh_fast(d[i + 1] + b1[c + 1]);
      float2 h, l;
      h.x = rna_tf32(t0); h.y = rna_tf32(t1);
      l.x = rna_tf32(t0 - h.x); l.y = rna_tf32(t1 - h.y);
      const uint32_t o = (c >> 2) * X_LBO + r * 16 + (c & 3) * 4;
      *reinterpret_cast<float2*>(reinterpret_cast<uint8_t*>(h_hi) + o) = h;
      *reinterpret_cast<float2*>(reinterpret_cast<uint8_t*>(h_lo) + o) = l;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");   // this warpgroup's rows only
    // ---- layer 2 and epilogue 2: h2 = tanh(D2 + b2) -> staging tile ----
    wg_layer(d, h_hi, h_lo, w2_hi, w2_lo, wg);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int r = wr + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      stage[stage_idx(r, c)] = tanh_fast(d[i] + b2[c]);
    }
    asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
    // ---- output layer: thread (row r of this warpgroup, column half) ----
    const int r = 64 * wg + (tid & 63), half = (tid >> 6) & 1;
    float mean[SPO_MAX_ACT];
#pragma unroll
    for (int j = 0; j < SPO_MAX_ACT; ++j) mean[j] = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) {
      const float t = stage[stage_idx(r, half * 32 + k)];
#pragma unroll
      for (int j = 0; j < SPO_MAX_ACT; ++j)
        if (j < A) mean[j] = fmaf(t, w3[j * 64 + half * 32 + k], mean[j]);
    }
    if (half == 1) {
#pragma unroll
      for (int j = 0; j < SPO_MAX_ACT; ++j)
        if (j < A) pmean[r][j] = mean[j];
    }
    asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
    const int64_t g = row0 + r;
    if (half == 0 && g < a.count) {
      // the means go straight from registers to global memory; the other epilogues read the row back from pmean
#pragma unroll
      for (int j = 0; j < SPO_MAX_ACT; ++j)
        if (j < A) {
          const float mu = (mean[j] + pmean[r][j]) + b3[j];
          if (a.mode == SpoFwdMode::kMeans) a.mean_out[g * A + j] = mu;
          else pmean[r][j] = mu;
        }
      if (a.mode != SpoFwdMode::kMeans) kl_acc += static_cast<double>(spo_forward_row(a, net, g, pmean[r], ls, ols));
    }
    if (a.mode == SpoFwdMode::kStep && net == 0 && a.has_store) {
      // observation rows into slot t (buffer.py:91-95): bit-exact copy from global (the smem tile holds the TF32 split)
      const int rows = static_cast<int>((a.count - row0) < TC_ROWS ? (a.count - row0) : TC_ROWS), c4 = D >> 2;
      const int T = a.store.steps;
      for (int i = tid; i < rows * c4; i += TC_THREADS) {
        const int rr = i / c4, c = i - rr * c4;
        const float4 v = __ldg(reinterpret_cast<const float4*>(a.obs + (row0 + rr) * D) + c);
        *(reinterpret_cast<float4*>(a.store.obs + ((row0 + rr) * T + a.t) * D) + c) = v;
      }
    }
    // one CTA-wide rendezvous per tile: the staging tile (x_lo), pmean and the h tiles are reused by the next tile
    __syncthreads();
  }

  if (spo_fwd_is_kl(a.mode)) {
    kl_acc = spo_warp_sum(kl_acc);
    if (lane == 0) red[warp] = kl_acc;
    __syncthreads();
    if (tid == 0) spo_kl_pass_add(a, ((red[0] + red[1]) + (red[2] + red[3])) + ((red[4] + red[5]) + (red[6] + red[7])));
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
    (void)cudaGetLastError();
  }
  return fn;
}

}  // namespace

bool spo_tc_forward_applies(const SpoFwdArgs& a) {
  const bool step = a.mode == SpoFwdMode::kStep;
  return (a.D & 3) == 0 && a.D <= 64 && a.count >= (step ? TC_ROWS : 8 * TC_ROWS);
}

bool spo_tc_encode_obs_map(CUtensorMap* map, const float* obs, int64_t count, int D) {
  EncodeTiledFn encode = get_encode_fn();
  if (!encode) return false;
  const cuuint64_t gdim[3] = {4, static_cast<cuuint64_t>(count), static_cast<cuuint64_t>(D / 4)};
  const cuuint64_t gstride[2] = {static_cast<cuuint64_t>(D) * 4, 16};      // bytes: row pitch, k-chunk pitch
  const cuuint32_t box[3] = {4, TC_ROWS, 16};
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(obs), gdim, gstride, box, estr,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    static bool warned = false;
    if (!warned) {
      warned = true;
      fprintf(stderr, "libspo: cuTensorMapEncodeTiled failed (%d) for obs [%lld,%d]; using the FFMA tile kernel\n", static_cast<int>(r),
              static_cast<long long>(count), D);
    }
    return false;
  }
  return true;
}

constexpr size_t TC_SMEM_BYTES = 4 * X_TILE_BYTES + 4 * W_TILE_BYTES + sizeof(float) * (128 + SPO_MAX_ACT * 64 + 24);   // 198.6 KB

int spo_tc_forward_launch(const CUtensorMap& map, const SpoFwdArgs& a, cudaStream_t stream) {
  static bool attr_set = false;   // per process: one process drives one GPU
  if (!attr_set) {
    SPO_CUDA_TRY(cudaFuncSetAttribute(spo_tc_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  const int64_t n_tiles = (a.count + TC_ROWS - 1) / TC_ROWS;
  const dim3 grid = (a.mode == SpoFwdMode::kStep)
                        ? dim3(static_cast<unsigned>(n_tiles), a.net_base == 0 ? 3 : 2)
                        : dim3(static_cast<unsigned>(n_tiles < spo_sm_count() ? n_tiles : spo_sm_count()));   // one CTA per SM
  spo_tc_forward_kernel<<<grid, TC_THREADS, TC_SMEM_BYTES, stream>>>(map, a);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}
