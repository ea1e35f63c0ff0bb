// The minibatch update loop as one persistent launch per pass -- round-2 design: every net is spread over FOUR
// SMs of one 12-CTA thread-block cluster; the CTAs exchange activations by pushing 2-4 KB blocks into each other's
// shared memory with the bulk-copy engine (cp.async.bulk shared -> peer shared, complete_tx on the receiver's mbarrier).
// There is no cluster barrier inside the loop.
//
// Reference: safepo/single_agent/ppo_lag.py:297-336 (PPO-Lag), focops.py:309-357 (FOCOPS), cpo.py:543-571 /
// trpo_lag.py:466-494 (critic regression).  Per minibatch: forward of the three nets, losses, backward, critic L2
// term, ONE joint grad-norm clip over all three nets (ppo_lag.py:325), three Adam steps.
//
// Why: the chain of minibatch steps is strictly serial (each step needs the previous step's weights), so the only
// figure of merit is the latency of ONE step.  One CTA per net would leave five 64x64x64 GEMMs and every per-parameter /
// per-row phase to a single SM; here the hidden layer is split by UNITS: CTA (net n, quarter q) owns hidden units [16q, 16q+16) of both layers -- the matching rows of W1 and W2,
// their biases, the matching columns of W3, and the Adam moments of exactly those parameters (in registers).  Nothing
// is replicated except b3 / log_std (<= 16 floats), no weight ever moves; what moves per step is activations:
//
//   forward   h1[:, slice] = tanh(x W1[slice]^T)          -> all-gather of the 64x16 slices inside the net (3 x 4 KB in)
//             h2[:, slice] = tanh(h1 W2[slice]^T)         (needs all of h1, local afterwards)
//             y partial    = h2[:, slice] W3[:, slice]^T  -> all-gather of the 64 x O partial sums (3 x 2 KB in)
//   loss rows              (replicated in the four CTAs of a net: every CTA holds all 64 rows of y)
//   backward  dz2[:, slice], dW2[slice, :] = dz2[:, slice]^T h1, dW3[:, slice]       (local)
//             dh1 partial  = dz2[:, slice] W2[slice, :]   -> reduce-scatter by column quarter (3 x 4 KB in), hidden
//                                                            behind the dW2 product and the dW3 / db3 / dlog_std sums
//             dz1[:, slice], dW1[slice, :] = dz1[:, slice]^T x                       (local)
//   clip      (sum g^2, sum theta^2) of the slice         -> all-to-all of 16 bytes between the 12 CTAs = the step barrier
//   Adam      on the slice, weights rewritten in place in shared memory: W1 / b1 at the end of the step, speculatively with
//             clip = 1 (their (theta, m, v) backed up: 15 KB at NT1 = 1); W2, b2, W3, b3, log_std in the next step's h1
//             window with the actual clip (the last step of a launch: in the epilogue)
//
// How the CTAs talk was chosen with the probes tools/cluster_probe.cu and tools/dsmem_probe.cu (12-CTA cluster): pulls
// with ld.shared::cluster need a cluster barrier in front and local stores behind, st.async + mbarrier showed a long fixed
// latency for blocks, while cp.async.bulk pushes are issued by one thread, land with the lowest latency and leave the LSU alone.
// So every activation exchange is: producers write their block (fence.proxy.async + __syncthreads), one elected thread per
// destination pushes it, consumers wait on their own mbarrier (armed with the byte count).  The 16-byte all-to-all of the
// norms is the exception: there is no block to stage, so twelve threads store their registers into the peers with st.async
// (complete_tx on the same kind of mbarrier); on H100 this took the norm push from 612 to 336 cycles per step and the
// whole step from 15 003 to 14 643 (clock64 phase marks, tools/phase_timers.py).  The activation exchanges
// stay on the bulk copy: sending the 2 KB partial-output rows with st.async instead measured no faster.  Buffer reuse is safe because a CTA
// pushes its 16 bytes of the step barrier only after its last read of any exchanged buffer, and nothing of the next
// step is pushed before all 12 of them arrived; the step barrier alternates between two mbarriers so that a CTA a whole
// step ahead cannot complete_tx into a phase that is still open at a slower one.
//
// GEMMs: warp-level mma.sync.m16n8k8 TF32 with the 3xTF32 split in registers (csrc/spo_mma.cuh); every product of
// the step is 64x16x64 (or its transposes).  The operands change every step (each is produced by the previous phase),
// so there is nothing for TMA to prefetch and what counts is the issue-to-result latency of small products.  The
// full-batch and rollout kernels (csrc/spo_tc_forward.cu), where tiles are independent, are the wgmma ones.
//
// Shared-memory tiles use leading dimensions == 8 (mod 32): k-pair 64-bit loads for [m][k] x [n][k] products and 32-bit
// loads for transposed operands are then bank-conflict free; h1 lives in four XOR-swizzled [64][16] slice blocks (one
// block = one contiguous 4 KB push) with the same property for both of its uses.
//
// Minibatch rows: the permutation of a pass is known before the pass starts, so the entry point first runs
// spo_pack_tiles over the whole grid, which writes the pass's rows out in step order as one contiguous record per 64-row
// tile, laid out exactly like a tile slot in shared memory ([64][ldx] observations, then [64][AUXW] side data, zero
// padding).  The update kernel keeps a ring of NSLOT such slots; one thread brings a whole tile in with a single
// cp.async.bulk global -> shared copy NSLOT tiles ahead, and the top of a tile waits on the slot's mbarrier.  No other
// thread touches the gather, and no register stages it.
//
// Data-parallel ranks (spo_pg_update_dp): every CTA pushes its slice of the gradient to the same CTA of every peer
// GPU as 8-byte {value, sequence} words (posted NVLink stores into peer-mapped staging memory), dW2 / dW3 / db2 as soon
// as they exist (dh1 exchange and the dW1 product still ahead), the rest after dW1; a receiver polls the words
// themselves -- no fence, no flag, no barrier (the sequence number in every word is the flag).  Sums run in rank
// order on every rank, so the replicas stay bit-identical.
// act_dim <= 8 runs the AC = 8 instantiations, compiled in spo_update.cu; 9..16 the AC = 16 ones, compiled in
// spo_update_wide.cu.  Keeping them apart keeps the AC = 8 module what it was before AC existed (same instructions, same
// kernels in the object file).
#pragma once
#include <cooperative_groups.h>
#include <stdlib.h>
#include "spo_common.cuh"
#include "spo_mma.cuh"

namespace cg = cooperative_groups;

// the memory pool of the packed tiles (spo_update.cu): the library's own, on the current device, keeping its blocks
// across calls so that a pass's allocation is served without a device-wide synchronisation
int spo_update_tile_pool(cudaMemPool_t* pool);

#ifdef SPO_PHASE_TIMERS
__device__ unsigned long long g_phase_cycles[16][24];
#define PHASE_MARK(idx)                                                   \
  do {                                                                    \
    if (tid == 0) {                                                       \
      const long long now__ = clock64();                                  \
      sm_phase__[idx] += static_cast<unsigned long long>(now__ - phase_t__); \
      phase_t__ = now__;                                                  \
    }                                                                     \
  } while (0)
#else
#define PHASE_MARK(idx) do { } while (0)
#endif

namespace {

constexpr int UT = 256;                 // threads per CTA: 8 warps, 2 per scheduler
constexpr int NQ = 4;                   // CTAs per net
constexpr int SL = SPO_HID / NQ;        // hidden units per CTA (16)
constexpr int NCTA = 3 * NQ;            // working CTAs of the cluster
constexpr int LDA = 72;                 // leading dimension of 64-wide tiles   (== 8 mod 32)
constexpr int LDS = 40;                 // leading dimension of SL-wide slices  (== 8 mod 32)

// Everything sized by the action capacity AC (8 or 16; the kernel is instantiated for both, act_dim <= 8 runs AC = 8):
//   per-row side data   act[AC] | logp adv target_r target_c | old_mean[AC] | old_std[AC]
//   small parameters    b1[SL] b2[SL] w3[AC][SL] b3[AC] log_std[AC] of a slice; thread i owns entries i, i + UT, ...
//                       (SPN = 176 at AC = 8: one per thread; 320 at AC = 16: two for the first 64 threads)
template <int AC>
struct UpdShape {
  static_assert(AC == 8 || AC == 16, "action capacity 8 or 16");
  static constexpr int AUXW = 3 * AC + 4;
  // the cost critic reads its target from AUX_TGT + 1
  static constexpr int AUX_LOGP = AC, AUX_ADV = AC + 1, AUX_TGT = AC + 2, AUX_OMEAN = AC + 4, AUX_OSTD = 2 * AC + 4;
  static constexpr int SP_B1 = 0, SP_B2 = SL, SP_W3 = 2 * SL, SP_B3 = 2 * SL + AC * SL, SP_LS = SP_B3 + AC;
  static constexpr int SPN = SP_LS + AC;
  static constexpr int SPT = (SPN + UT - 1) / UT;   // small-parameter entries per thread
  static constexpr int YQ = SPO_ROWS * AC;          // floats per partial-output block
  static constexpr int DH = AC / 4;                 // action dims per thread in the loss rows (4 lanes per row)
};
static_assert(UpdShape<8>::SPN == 176 && UpdShape<8>::SPT == 1 && UpdShape<16>::SPN == 320 && UpdShape<16>::SPT == 2, "layout");

__host__ __device__ constexpr int upd_ldx(int nt1) { return 64 * nt1 + 8; }
// one packed tile = one shared-memory tile slot: [64][ldx] observations, then [64][AUXW] side data
template <int NT1, int AC>
__host__ __device__ constexpr int upd_tile_floats() { return SPO_ROWS * (upd_ldx(NT1) + UpdShape<AC>::AUXW); }
static_assert(upd_tile_floats<1, 8>() * 4 == 25600 && upd_tile_floats<2, 8>() * 4 == 41984 && upd_tile_floats<2, 16>() * 4 % 16 == 0,
              "bulk copies move multiples of 16 bytes");
// per-CTA gradient slot of the cross-GPU exchange, in 8-byte {value, seq} words: W2 frags, W1 frags, small
__host__ __device__ constexpr int dp_slot_words(int nt1) { return UT * 4 * (1 + nt1) + UT; }

template <int N> struct IC { static constexpr int value = N; };

struct UpdArgs {
  float *params, *adam_m, *adam_v;
  int* adam_t;
  float* tiles;     // the pass's packed tiles (written by spo_pack_tiles, read by the update kernel)
  spo_batch data;
  const int64_t* perm;
  int64_t perm_len;
  int batch, kind, D, A;
  int actor_only;   // CUP projection stage: the critic CTAs only take part in the step barrier
  spo_hparams hp;
  spo_update_ctrl* ctrl;
  spo_comm comm;    // world <= 1: single GPU
};

// ---- PTX helpers -----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ uint32_t mapa(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
// mbarrier + bulk-copy engine: the two 12 KB activation exchanges of a step (h1 all-gather, dh1 reduce-scatter) are PUSHED
// as 4 KB cp.async.bulk copies shared -> peer shared that complete_tx on the receiver's mbarrier: 695 cycles from issue to
// "all three slices landed" measured (tools/dsmem_probe.cu BULK) against ~1000 for 3 x float4 ld.shared::cluster per
// thread plus the barrier in front of them plus the local stores behind them; and the copy engine, not the LSU, moves the bytes.
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t a = smem_u32(bar);
  uint32_t ok = 0;
  while (!ok) {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"(a), "r"(parity) : "memory");
  }
}
// the same wait with acquire semantics at cluster scope: for data that peers wrote with st.async (generic proxy)
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  const uint32_t a = smem_u32(bar);
  uint32_t ok = 0;
  while (!ok) {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"(a), "r"(parity) : "memory");
  }
}
// 16 bytes from registers into a peer's shared memory; complete_tx (release, cluster scope) on the peer's mbarrier
__device__ __forceinline__ void st_async16(uint32_t remote_dst, float4 v, uint32_t remote_bar) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];"
               ::"r"(remote_dst), "r"(__float_as_uint(v.x)), "r"(__float_as_uint(v.y)), "r"(__float_as_uint(v.z)),
               "r"(__float_as_uint(v.w)), "r"(remote_bar) : "memory");
}
__device__ __forceinline__ void bulk_push(uint32_t remote_dst, const void* local_src, uint32_t bytes, uint32_t remote_bar) {
  asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(remote_dst), "r"(smem_u32(local_src)), "r"(bytes), "r"(remote_bar) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// a packed tile global -> own shared memory (complete_tx on the own mbarrier), and the same bytes into L2 only
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_prefetch_l2(const void* gmem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem_src), "r"(bytes) : "memory");
}
// cross-GPU words: {value, seq} as one 8-byte access (single-copy atomic), system scope, no caching games
__device__ __forceinline__ void st_ll(float2* p, float v, unsigned seq) {
  asm volatile("st.relaxed.sys.global.v2.b32 [%0], {%1, %2};" ::"l"(p), "r"(__float_as_uint(v)), "r"(seq) : "memory");
}

// One Adam step on a scalar in torch's _multi_tensor_adam op order:
//   m = lerp(m, g, 1-b1) (fused mul-add);  v = v*b2 + ((1-b2)*g)*g;
//   denom = sqrt(v)/sqrt(bc2) + eps;  p = p + (step_size*m)/denom,  step_size = -lr/bc1.
// sqrt and the division use the SFU approximations (sqrt.approx / div.approx, <= 2 ulp), 1/sqrt(bc2) is a precomputed
// factor (measured error of whole chains: tests/test_gpu_parity.py prints it).
struct AdamK {
  float w1, b2, w2, ibc2s, eps, ss;  // w1 = 1-b1, w2 = 1-b2, ibc2s = 1/sqrt(1-b2^t)
};
__device__ __forceinline__ float sqrt_approx(float x) {
  float r;
  asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float adam_update(float p, float g, float& m, float& v, const AdamK& k) {
  m = fmaf(k.w1, __fsub_rn(g, m), m);
  v = __fadd_rn(__fmul_rn(v, k.b2), __fmul_rn(__fmul_rn(k.w2, g), g));
  const float denom = fmaf(sqrt_approx(v), k.ibc2s, k.eps);
  return __fadd_rn(p, __fdividef(__fmul_rn(k.ss, m), denom));
}

// One 16-row m-tile x NTL 8-column n-tiles of C (+)= A * B on the tensor pipe, 3xTF32 with the three partial
// products in separate accumulator chains (lo*hi, hi*lo, hi*hi; small terms are added first at the end).
//   A(m, k) = A[m * a_sm + k * a_sk]      B(k, n) = B[k * b_sk + n * b_sn]      (shared memory, K = 8 * KSTEPS)
// Fragment ownership (g = lane >> 2, t = lane & 3): acc[nt][0..3] = C(m0+g, n0+8nt+2t), (.., +1), (m0+g+8, ..), (.., +1)
// With two warps per scheduler nothing hides a load -> split -> mma chain: all operand fragments of a chunk of (up to)
// eight k-steps are requested before the first split, then the chunk's splits and mmas run from registers.
template <int NTL, int KSTEPS, bool ACCUM>
__device__ __forceinline__ void warp_gemm(float (&acc)[NTL][4], const float* __restrict__ A, int a_sm, int a_sk,
                                          const float* __restrict__ B, int b_sk, int b_sn, int m0, int n0) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const float* a_ptr = A + (m0 + g) * a_sm + t * a_sk;
  const float* b_ptr = B + t * b_sk + (n0 + g) * b_sn;
  float c_lh[NTL][4], c_hl[NTL][4], c_hh[NTL][4];
#pragma unroll
  for (int nt = 0; nt < NTL; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) { c_lh[nt][e] = 0.f; c_hl[nt][e] = 0.f; c_hh[nt][e] = 0.f; }
  constexpr int CH = KSTEPS < 8 ? KSTEPS : 8;
#pragma unroll
  for (int kc = 0; kc < KSTEPS; kc += CH) {
    float af[CH][4], bf[CH][NTL][2];
#pragma unroll
    for (int ks = 0; ks < CH; ++ks) {
      const float* p = a_ptr + (kc + ks) * 8 * a_sk;
      af[ks][0] = p[0]; af[ks][1] = p[8 * a_sm]; af[ks][2] = p[4 * a_sk]; af[ks][3] = p[8 * a_sm + 4 * a_sk];
#pragma unroll
      for (int nt = 0; nt < NTL; ++nt) {
        const float* pb = b_ptr + nt * 8 * b_sn + (kc + ks) * 8 * b_sk;
        bf[ks][nt][0] = pb[0]; bf[ks][nt][1] = pb[4 * b_sk];
      }
    }
#pragma unroll
    for (int ks = 0; ks < CH; ++ks) {
      uint32_t ah[4], al[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) spo_split_tf32(af[ks][i], ah[i], al[i]);
#pragma unroll
      for (int nt = 0; nt < NTL; ++nt) {
        uint32_t bh[2], bl[2];
        spo_split_tf32(bf[ks][nt][0], bh[0], bl[0]);
        spo_split_tf32(bf[ks][nt][1], bh[1], bl[1]);
        spo_mma_tf32(c_lh[nt], al, bh);
        spo_mma_tf32(c_hl[nt], ah, bl);
        spo_mma_tf32(c_hh[nt], ah, bh);
      }
    }
  }
#pragma unroll
  for (int nt = 0; nt < NTL; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float s = (c_lh[nt][e] + c_hl[nt][e]) + c_hh[nt][e];
      acc[nt][e] = ACCUM ? acc[nt][e] + s : s;
    }
}

// The same product when BOTH operands are contiguous along k (A[m][k], B[n][k]: the two forward layers): the mma's k
// slots are bound to memory as slot t <-> k0 + 2t, slot t + 4 <-> k0 + 2t + 1, so that a thread's two k values of a row are
// one 8-byte load.  With leading dimensions == 8 (mod 32) a half-warp's 64-bit accesses (g = 0..3, t = 0..3: banks
// 8g + 2t, +1) are conflict-free, whereas the 32-bit fragment loads of warp_gemm collide two-way for this orientation
// (banks 8g + t repeat for g and g + 4) -- 32 % of all shared-memory wavefronts of the first version of this kernel.
template <int KSTEPS>
__device__ __forceinline__ void warp_gemm_kk(float (&acc)[1][4], const float* __restrict__ A, int lda,
                                             const float* __restrict__ B, int ldb, int m0, int n0) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const float* a_ptr = A + (m0 + g) * lda + 2 * t;
  const float* b_ptr = B + (n0 + g) * ldb + 2 * t;
  float c_lh[4] = {0.f, 0.f, 0.f, 0.f}, c_hl[4] = {0.f, 0.f, 0.f, 0.f}, c_hh[4] = {0.f, 0.f, 0.f, 0.f};
  constexpr int CH = KSTEPS < 8 ? KSTEPS : 8;
#pragma unroll
  for (int kc = 0; kc < KSTEPS; kc += CH) {
    float2 a0[CH], a1[CH], bb[CH];
#pragma unroll
    for (int ks = 0; ks < CH; ++ks) {
      a0[ks] = *reinterpret_cast<const float2*>(a_ptr + (kc + ks) * 8);
      a1[ks] = *reinterpret_cast<const float2*>(a_ptr + 8 * lda + (kc + ks) * 8);
      bb[ks] = *reinterpret_cast<const float2*>(b_ptr + (kc + ks) * 8);
    }
#pragma unroll
    for (int ks = 0; ks < CH; ++ks) {
      uint32_t ah[4], al[4], bh[2], bl[2];
      spo_split_tf32(a0[ks].x, ah[0], al[0]);
      spo_split_tf32(a1[ks].x, ah[1], al[1]);
      spo_split_tf32(a0[ks].y, ah[2], al[2]);
      spo_split_tf32(a1[ks].y, ah[3], al[3]);
      spo_split_tf32(bb[ks].x, bh[0], bl[0]);
      spo_split_tf32(bb[ks].y, bh[1], bl[1]);
      spo_mma_tf32(c_lh, al, bh);
      spo_mma_tf32(c_hl, ah, bl);
      spo_mma_tf32(c_hh, ah, bh);
    }
  }
#pragma unroll
  for (int e = 0; e < 4; ++e) acc[0][e] = (c_lh[e] + c_hl[e]) + c_hh[e];
}

// h1 lives as four slice blocks [quarter][64 rows][16 columns] (each 4 KB contiguous: one bulk copy per peer) with the
// column index XOR-ed by 8 on rows whose bit 1 is set.  Both access patterns of the mma fragments are then conflict-free:
// k-pair 64-bit loads of the layer-2 A operand (half-warp rows g = 0..3: banks 16(g&1) + 8((g>>1)^x) + 2t, +1) and the 32-bit
// loads of the dW2 B operand (rows k0 + t: banks 16(t&1) + 8((t>>1)^x) + g).
constexpr int H1Q = SPO_ROWS * SL;   // floats per slice block
// element (row r, unit c): h1[(c >> 4) * H1Q + r * SL + ((c & 15) ^ (((r >> 1) & 1) << 3))]

// layer 2: acc[16 x 8 tile at (m0, n0)] = h1[m0.., :] * W2slice[n0.., :]^T   (A from the swizzled blocks, B = w2s [n][k], k-pair mapping)
__device__ __forceinline__ void warp_gemm_l2(float (&acc)[1][4], const float* __restrict__ h1, const float* __restrict__ B, int ldb, int m0, int n0) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int r0 = m0 + g, sw = ((r0 >> 1) & 1) << 3;          // row r0 + 8 has the same swizzle
  const float* b_ptr = B + (n0 + g) * ldb + 2 * t;
  float c_lh[4] = {0.f, 0.f, 0.f, 0.f}, c_hl[4] = {0.f, 0.f, 0.f, 0.f}, c_hh[4] = {0.f, 0.f, 0.f, 0.f};
  float2 a0[8], a1[8], bb[8];
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {
    const float* blk = h1 + (ks >> 1) * H1Q + ((((ks & 1) << 3) + 2 * t) ^ sw);
    a0[ks] = *reinterpret_cast<const float2*>(blk + r0 * SL);
    a1[ks] = *reinterpret_cast<const float2*>(blk + (r0 + 8) * SL);
    bb[ks] = *reinterpret_cast<const float2*>(b_ptr + ks * 8);
  }
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {
    uint32_t ah[4], al[4], bh[2], bl[2];
    spo_split_tf32(a0[ks].x, ah[0], al[0]);
    spo_split_tf32(a1[ks].x, ah[1], al[1]);
    spo_split_tf32(a0[ks].y, ah[2], al[2]);
    spo_split_tf32(a1[ks].y, ah[3], al[3]);
    spo_split_tf32(bb[ks].x, bh[0], bl[0]);
    spo_split_tf32(bb[ks].y, bh[1], bl[1]);
    spo_mma_tf32(c_lh, al, bh);
    spo_mma_tf32(c_hl, ah, bl);
    spo_mma_tf32(c_hh, ah, bh);
  }
#pragma unroll
  for (int e = 0; e < 4; ++e) acc[0][e] = (c_lh[e] + c_hl[e]) + c_hh[e];
}

// dW2 slice: acc[16 (own units j) x 8 columns at n0] += dz2s^T * h1   (A(m = j, k = r) = dz2s[r][j]; B(k = r, n) = h1[r][n] swizzled)
__device__ __forceinline__ void warp_gemm_dw2(float (&acc)[1][4], const float* __restrict__ dz, int ldz, const float* __restrict__ h1, int n0) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const float* a_ptr = dz + t * ldz + g;
  const int n = n0 + g, sw = ((t >> 1) & 1) << 3;            // rows 8ks + t and 8ks + t + 4 share the swizzle of t
  const float* b_ptr = h1 + (n >> 4) * H1Q + t * SL + ((n & 15) ^ sw);
  float c_lh[4] = {0.f, 0.f, 0.f, 0.f}, c_hl[4] = {0.f, 0.f, 0.f, 0.f}, c_hh[4] = {0.f, 0.f, 0.f, 0.f};
  float af[8][4], bf[8][2];
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {
    const float* p = a_ptr + ks * 8 * ldz;
    af[ks][0] = p[0]; af[ks][1] = p[8]; af[ks][2] = p[4 * ldz]; af[ks][3] = p[4 * ldz + 8];
    const float* pb = b_ptr + ks * 8 * SL;
    bf[ks][0] = pb[0]; bf[ks][1] = pb[4 * SL];
  }
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {
    uint32_t ah[4], al[4], bh[2], bl[2];
#pragma unroll
    for (int i = 0; i < 4; ++i) spo_split_tf32(af[ks][i], ah[i], al[i]);
    spo_split_tf32(bf[ks][0], bh[0], bl[0]);
    spo_split_tf32(bf[ks][1], bh[1], bl[1]);
    spo_mma_tf32(c_lh, al, bh);
    spo_mma_tf32(c_hl, ah, bl);
    spo_mma_tf32(c_hh, ah, bh);
  }
#pragma unroll
  for (int e = 0; e < 4; ++e) acc[0][e] += (c_lh[e] + c_hl[e]) + c_hh[e];
}

// dynamic shared memory of spo_update_kernel<NT1, AC, *> without its tile slots, and the number of slots: two wherever
// they fit in 227 KB, so that a tile is copied in a whole step ahead; one at (NT1, AC) = (2, 16).
//   (1, 8): 121 152 + 2 x 25 600 = 172 352 B    (2, 8): 137 536 + 2 x 41 984 = 221 504 B
//   (1, 16): 136 768 + 2 x 31 744 = 200 256 B   (2, 16): 153 152 + 1 x 48 128 = 201 280 B
template <int NT1, int AC>
__host__ __device__ constexpr size_t update_fixed_smem_bytes() {
  using S = UpdShape<AC>;
  return sizeof(float) * (4 * AC + 16 + SL * upd_ldx(NT1) + SL * LDA + 2 * S::SPN + NQ * SPO_ROWS * SL + 3 * SPO_ROWS * LDS +
                          (3 + NQ) * SPO_ROWS * AC + 2 * NQ * SPO_ROWS * SL + 64 + 128 + 3 * (4 * NT1 + 1) * UT);
}
template <int NT1, int AC>
__host__ __device__ constexpr int update_nslot() {
  return update_fixed_smem_bytes<NT1, AC>() + 2 * sizeof(float) * upd_tile_floats<NT1, AC>() <= 227 * 1024 ? 2 : 1;
}
template <int NT1, int AC>
__host__ __device__ constexpr size_t update_smem_bytes() {
  return update_fixed_smem_bytes<NT1, AC>() + update_nslot<NT1, AC>() * sizeof(float) * upd_tile_floats<NT1, AC>();
}
static_assert(update_smem_bytes<1, 8>() == 172352 && update_smem_bytes<2, 8>() == 221504 && update_smem_bytes<1, 16>() == 200256 &&
              update_smem_bytes<2, 16>() == 201280, "shared-memory figures in the comment above");

// Packs the rows of one pass in step order: tile t = (step s, sub u) = t / tps, t % tps is one contiguous record, laid out
// like a tile slot of the update kernel.  Row r is sample perm[s * batch + 64 u + r] while 64 u + r < rows of step s, zeros
// past it; observation columns D .. ldx-1 are zero, and so is every side column without a source for the kind.  One warp
// per row; values are copied bit for bit.  Returns at once after a KL early stop, like the update kernel.
template <int NT1, int AC>
__global__ void __launch_bounds__(256) spo_pack_tiles(const UpdArgs a, int64_t n_tiles) {
  using S = UpdShape<AC>;
  if (*reinterpret_cast<volatile int*>(&a.ctrl->stop)) return;
  constexpr int ldx = upd_ldx(NT1), AUXW = S::AUXW, TILEF = upd_tile_floats<NT1, AC>();
  const int D = a.D, A = a.A, lane = threadIdx.x & 31;
  const int tps = (a.batch + SPO_ROWS - 1) / SPO_ROWS;
  const bool actor = a.kind != SPO_LOSS_CRITIC_ONLY, focops = a.kind == SPO_LOSS_FOCOPS;
  const int64_t n_rows = n_tiles * SPO_ROWS, wstride = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  for (int64_t w = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; w < n_rows; w += wstride) {
    const int64_t t = w / SPO_ROWS, step = t / tps;
    const int r = static_cast<int>(w - t * SPO_ROWS), row = static_cast<int>(t - step * tps) * SPO_ROWS + r;
    int64_t rows_step = a.perm_len - step * a.batch;
    if (rows_step > a.batch) rows_step = a.batch;
    const bool valid = row < rows_step;
    const int64_t g = valid ? a.perm[step * a.batch + row] : 0;
    float* xo = a.tiles + t * TILEF + r * ldx;
    float* ao = a.tiles + t * TILEF + SPO_ROWS * ldx + r * AUXW;
    const float* xs = a.data.obs + g * D;
    for (int c = lane; c < ldx; c += 32) xo[c] = (valid && c < D) ? xs[c] : 0.f;
    for (int c = lane; c < AUXW; c += 32) {
      const float* src = nullptr;
      int64_t i = g;
      if (c < A) { if (actor) { src = a.data.act; i = g * A + c; } }
      else if (c == S::AUX_LOGP) { if (actor) src = a.data.logp; }
      else if (c == S::AUX_ADV) { if (actor) src = a.data.adv; }
      else if (c == S::AUX_TGT) src = a.data.target_r;
      else if (c == S::AUX_TGT + 1) src = a.data.target_c;
      else if (c >= S::AUX_OMEAN && c < S::AUX_OMEAN + A) { if (focops) { src = a.data.old_mean; i = g * A + c - S::AUX_OMEAN; } }
      else if (c >= S::AUX_OSTD && c < S::AUX_OSTD + A) { if (focops) { src = a.data.old_std; i = g * A + c - S::AUX_OSTD; } }
      ao[c] = (valid && src) ? src[i] : 0.f;
    }
  }
}

// DP = false: the single-GPU instantiation carries none of the cross-GPU code (its 24-register polling buffers would sit
// on top of an already full register file).  AC: action capacity (UpdShape); DP exists only at AC = 8.
template <int NT1, int AC, bool DP>
__global__ void __launch_bounds__(UT, 1) spo_update_kernel(const UpdArgs a) {
  static_assert(!(DP && AC != 8), "the cross-GPU gradient slots hold one small parameter per thread");
  using S = UpdShape<AC>;
  constexpr int AUXW = S::AUXW, AUX_LOGP = S::AUX_LOGP, AUX_ADV = S::AUX_ADV, AUX_TGT = S::AUX_TGT, AUX_OMEAN = S::AUX_OMEAN,
                AUX_OSTD = S::AUX_OSTD;
  constexpr int SP_B1 = S::SP_B1, SP_B2 = S::SP_B2, SP_W3 = S::SP_W3, SP_B3 = S::SP_B3, SP_LS = S::SP_LS, SPN = S::SPN;
  constexpr int SPT = S::SPT, YQ = S::YQ, DH = S::DH;
  constexpr int NSLOT = update_nslot<NT1, AC>(), TILEF = upd_tile_floats<NT1, AC>();
  constexpr uint32_t TILEB = TILEF * sizeof(float);
  extern __shared__ __align__(16) float smem[];
  __shared__ __align__(8) uint64_t bar_h1, bar_dh, bar_y, bar_ss[2];   // complete_tx targets of the four pushed exchanges
  __shared__ __align__(8) uint64_t bar_tile[NSLOT];                    // ... and of the tile copies, one per slot
  __shared__ int comm_dead;   // a peer GPU never showed up: stop waiting (ctrl->stop = 2 tells the host)
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank();
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  spo_update_ctrl* ctrl = a.ctrl;
  if (*reinterpret_cast<volatile int*>(&ctrl->stop)) return;  // whole cluster takes this branch together

  const int D = a.D, A = a.A;
  constexpr int ldx = upd_ldx(NT1);
  const bool idle = rank >= NCTA;                 // fallback cluster of 16: the last four CTAs only join the barriers
  const int net = idle ? 2 : static_cast<int>(rank) / NQ;
  const int q = static_cast<int>(rank) % NQ;      // hidden-unit quarter
  const unsigned grp0 = static_cast<unsigned>(net * NQ);
  const bool is_actor = (net == 0);
  const bool active = !idle && !(is_actor && a.kind == SPO_LOSS_CRITIC_ONLY) && !(!is_actor && a.actor_only);
  const SpoNetOff off = spo_net_off(D, A, net);
  const int O = off.out;
  const int g8 = lane >> 2, t4 = lane & 3;

  // ---- shared memory carve-up -------------------------------------------------------------------------------
  float* p = smem;
  float* lsc = p; p += 4 * AC;                    // per action dim: std, 1/var, log(std), spare (refreshed every step)
  float* adk = p; p += 16;                        // Adam scalars by step parity: [step & 1][8]
  float* w1s = p; p += SL * ldx;                  // W1[16q + j][k]
  float* w2s = p; p += SL * LDA;                  // W2[16q + j][k]
  float* sp = p;  p += SPN;                       // small parameters (layout SP_*)
  float* gsmall = p; p += SPN;                    // their gradients
  float* slots = p; p += NSLOT * TILEF;           // tile slots, each [64][ldx] observations + [64][AUXW] side data
  float* x = slots;                               // the current tile's slot ...
  float* aux = x + SPO_ROWS * ldx;                // ... and its per-row side data
  float* h1 = p;  p += NQ * H1Q;                  // all 64 units as four swizzled slice blocks: own + the three pushed by the peers
  float* h2s = p; p += SPO_ROWS * LDS;            // own slice
  float* dz2s = p; p += SPO_ROWS * LDS;
  float* dz1s = p; p += SPO_ROWS * LDS;           // apart from h2s: the dW3 sums still read h2 while dz1 is formed
  float* yblk = p; p += NQ * YQ;                  // [quarter][64][AC] partial outputs: own block written here, the other three pushed in
  float* y = p;   p += SPO_ROWS * AC;
  float* dy = p;  p += SPO_ROWS * AC;
  float* dls = p; p += SPO_ROWS * AC;             // per-row d loss / d log_std
  float* dh1b = p; p += NQ * H1Q;                 // own partial of dh1 as [destination quarter][64][16]: block d is pushed to CTA d
  float* dh1in = p; p += NQ * H1Q;                // [source quarter][64][16]: the partials the three peers pushed for the own columns
  float* red = p; p += 64;                        // block-reduction scratch
  float* bk = p;  p += 3 * (4 * NT1 + 1) * UT;    // (theta, m, v) of this thread's W1 / b1 entries before a speculative Adam step
  float* xin = p; p += 2 * 16 * 4;                // [parity][source CTA]{sum g^2, sum theta^2, -, -}: own entry written here, 11 pushed in
  float* b1s = sp + SP_B1; float* b2s = sp + SP_B2; float* w3s = sp + SP_W3; float* b3 = sp + SP_B3; float* log_std = sp + SP_LS;

  const int tps = (a.batch + SPO_ROWS - 1) / SPO_ROWS;                    // tiles per step
  const int64_t n_steps = (a.perm_len + a.batch - 1) / a.batch;
  const int64_t n_tiles = n_steps * tps;
  // packed tile t -> slot t % NSLOT (one thread; the slot's previous tile has been read by every thread and fenced).  With a
  // single slot the copy has only the tail of a step to land in, so the tile after it is prefetched into L2 a step ahead.
  auto issue_tile = [&](int64_t t) {
    if (t >= n_tiles) return;
    const int s = static_cast<int>(t % NSLOT);
    mbar_expect_tx(&bar_tile[s], TILEB);
    bulk_load(slots + s * TILEF, a.tiles + t * TILEF, TILEB, &bar_tile[s]);
    if (NSLOT == 1 && t + 1 < n_tiles) bulk_prefetch_l2(a.tiles + (t + 1) * TILEF, TILEB);
  };

  if (tid == 0) {
    comm_dead = 0;
    mbar_init(&bar_h1, 1);
    mbar_init(&bar_dh, 1);
    mbar_init(&bar_y, 1);
    mbar_init(&bar_ss[0], 1);
    mbar_init(&bar_ss[1], 1);
#pragma unroll
    for (int s = 0; s < NSLOT; ++s) mbar_init(&bar_tile[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    if (!idle) { mbar_expect_tx(&bar_ss[0], (NCTA - 1) * 16); mbar_expect_tx(&bar_ss[1], (NCTA - 1) * 16); }
    for (int b = 0; b < 2; ++b) {   // the step-independent Adam scalars (fp64 like torch's Python floats)
      adk[8 * b + 0] = static_cast<float>(1.0 - static_cast<double>(a.hp.beta1));
      adk[8 * b + 1] = a.hp.beta2;
      adk[8 * b + 2] = static_cast<float>(1.0 - static_cast<double>(a.hp.beta2));
      adk[8 * b + 4] = a.hp.adam_eps;
    }
    if (active) {
      mbar_expect_tx(&bar_h1, (NQ - 1) * H1Q * 4);
      mbar_expect_tx(&bar_dh, (NQ - 1) * H1Q * 4);
      mbar_expect_tx(&bar_y, (NQ - 1) * YQ * 4);
#pragma unroll
      for (int t = 0; t < NSLOT; ++t) issue_tile(t);
    }
  }

  // ---- small-parameter entries of this thread: tid, and tid + UT at AC = 16 (threads < SPN - UT) ----
  // Entry 1 is written out beside entry 0 rather than as [SPT] arrays and loops over them: the AC = 8 instantiation then
  // compiles to exactly the instructions of the kernel before the action capacity was a parameter.
  bool sp_valid = false, sp_counted = false;
  int sp_goff = 0;
  if (tid < SPN && !idle) {
    const int i = tid;
    sp_counted = true;
    if (i < SP_B2) { sp_valid = true; sp_goff = off.b1 + SL * q + i; }
    else if (i < SP_W3) { sp_valid = true; sp_goff = off.b2 + SL * q + (i - SP_B2); }
    else if (i < SP_B3) { const int o = (i - SP_W3) / SL, kk = (i - SP_W3) % SL; sp_valid = o < O; sp_goff = off.w3 + o * SPO_HID + SL * q + kk; }
    else if (i < SP_LS) { const int o = i - SP_B3; sp_valid = o < O; sp_goff = off.b3 + o; sp_counted = (q == 0); }
    else { const int j = i - SP_LS; sp_valid = is_actor && j < A; sp_goff = off.log_std + j; sp_counted = (q == 0); }
  }
  float sp_m = 0.f, sp_v = 0.f;
  bool sp_valid1 = false, sp_counted1 = false;   // entry 1: i = tid + UT >= UT > SP_W3, so w3 rows, b3 or log_std
  int sp_goff1 = 0;
  float sp_m1 = 0.f, sp_v1 = 0.f;
  if constexpr (SPT > 1) {
    static_assert(UT > SP_W3, "entry 1 lies past b1 / b2");
    const int i = tid + UT;
    if (i < SPN && !idle) {
      sp_counted1 = true;
      if (i < SP_B3) { const int o = (i - SP_W3) / SL, kk = (i - SP_W3) % SL; sp_valid1 = o < O; sp_goff1 = off.w3 + o * SPO_HID + SL * q + kk; }
      else if (i < SP_LS) { const int o = i - SP_B3; sp_valid1 = o < O; sp_goff1 = off.b3 + o; sp_counted1 = (q == 0); }
      else { const int j = i - SP_LS; sp_valid1 = is_actor && j < A; sp_goff1 = off.log_std + j; sp_counted1 = (q == 0); }
    }
  }

  // ---- one-time loads ----
  if (!idle) {
    for (int i = tid; i < SL * ldx; i += UT) {
      const int j = i / ldx, k = i - j * ldx;
      w1s[i] = (k < D) ? __ldg(a.params + off.w1 + (SL * q + j) * D + k) : 0.f;
    }
    for (int i = tid; i < SL * LDA; i += UT) {
      const int j = i / LDA, k = i - j * LDA;
      w2s[i] = (k < SPO_HID) ? __ldg(a.params + off.w2 + (SL * q + j) * SPO_HID + k) : 0.f;
    }
    if (tid < SPN) {
      sp[tid] = sp_valid ? a.params[sp_goff] : 0.f;
      gsmall[tid] = 0.f;
      if (sp_valid) { sp_m = a.adam_m[sp_goff]; sp_v = a.adam_v[sp_goff]; }
    }
    if constexpr (SPT > 1) {
      if (tid + UT < SPN) {
        sp[tid + UT] = sp_valid1 ? a.params[sp_goff1] : 0.f;
        gsmall[tid + UT] = 0.f;
        if (sp_valid1) { sp_m1 = a.adam_m[sp_goff1]; sp_v1 = a.adam_v[sp_goff1]; }
      }
    }
  }
  // Adam moments of this thread's accumulator-fragment elements.  Fragment e of the dW2 slice product (warp w = n-tile w):
  //   (j, k) = (g + 8*(e>>1), 8w + 2t + (e&1));  the dW1 slice product has n-tiles w + 8*i, i < NT1.
  float mW2[4], vW2[4], mW1[NT1][4], vW1[NT1][4];
  auto frag_jk = [&](int e, int ntile, int& j, int& k) { j = g8 + ((e >> 1) << 3); k = 8 * ntile + 2 * t4 + (e & 1); };
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    int j, k;
    frag_jk(e, wid, j, k);
    mW2[e] = active ? a.adam_m[off.w2 + (SL * q + j) * SPO_HID + k] : 0.f;
    vW2[e] = active ? a.adam_v[off.w2 + (SL * q + j) * SPO_HID + k] : 0.f;
#pragma unroll
    for (int i = 0; i < NT1; ++i) {
      frag_jk(e, wid + 8 * i, j, k);
      const bool ok = active && k < D;
      mW1[i][e] = ok ? a.adam_m[off.w1 + (SL * q + j) * D + k] : 0.f;
      vW1[i][e] = ok ? a.adam_v[off.w1 + (SL * q + j) * D + k] : 0.f;
    }
  }
  const int t0 = a.adam_t[net];
  double b1pow = pow(static_cast<double>(a.hp.beta1), static_cast<double>(t0));   // threads UT - 32 / UT - 64 keep them current
  double b2pow = pow(static_cast<double>(a.hp.beta2), static_cast<double>(t0));
  const float lr = (net == 0) ? a.hp.lr_actor : (net == 1 ? a.hp.lr_reward : a.hp.lr_cost);
  const float extra_sumsq = (is_actor && q == 0 && a.kind == SPO_LOSS_CRITIC_ONLY && !idle) ? ctrl->extra_sumsq : 0.f;
  const float vcoef = (net == 1) ? a.hp.value_coef : 1.f;
  const float reg = is_actor ? 0.f : __fmul_rn(vcoef, __fmul_rn(a.hp.critic_l2, 2.f));

  int64_t step_idx = 0;
#ifdef SPO_PHASE_TIMERS
  __shared__ unsigned long long sm_phase__[24];
  if (tid < 24) sm_phase__[tid] = 0ull;
  long long phase_t__ = clock64();
#endif
  // column sums over the 64 rows of a [64][LDS] slice: thread (c = tid >> 4, rg = tid & 15) adds rows rg + 16 i
  auto colsum_into = [&](const float* buf, float* dst) {
    const int c = tid >> 4, rg = tid & 15;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) s += buf[(rg + 16 * i) * LDS + c];
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    s += __shfl_xor_sync(0xffffffffu, s, 8);
    if (rg == 0) dst[c] += s;
  };

  // shared::cluster addresses of the buffers this CTA pulls from: the four CTAs of its net, all CTAs for the norm
  uint32_t ph_x = 0;     // phase parity of bar_h1 / bar_y / bar_dh (one phase per tile of an active net)
  uint32_t tcount = 0;   // tiles done: the step barrier of tile n uses bar_ss[n & 1], phase parity (n >> 1) & 1 -- two barriers in
                         // alternation, so that a peer that is a whole step ahead can never complete_tx into a phase still open here

  // gradient accumulators = accumulator fragments of the dW products (persist across the tiles of a step)
  float gW2[1][4], gW1[NT1][4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    gW2[0][e] = 0.f;
#pragma unroll
    for (int i = 0; i < NT1; ++i) gW1[i][e] = 0.f;
  }
  double acc_loss = 0.0;        // thread 0 of quarter 0: sum over steps of this net's logged loss
  float step_loss = 0.f, step_aux0 = 0.f, step_aux1 = 0.f;   // thread 0: loss numerators of the current step

  // cross-GPU staging of this CTA: [parity][source rank][cta][dp_slot_words] 8-byte words
  const int world = DP ? a.comm.world : 1, me = DP ? a.comm.rank : 0;
  constexpr int DPW = dp_slot_words(NT1);
  const int mt = wid & 3, ntl = wid >> 2;     // 16 x 8 tile of the 64 x 16 slice products
  const int rA = mt * 16 + g8, cA = ntl * 8 + 2 * t4;
  const int r4 = tid >> 2, k4 = tid & 3;      // (row, quarter-of-a-slice) mapping of the element-wise phases

  cluster.sync();   // nobody pushes into a peer's shared memory before every CTA of the cluster has armed its mbarriers
  if (idle) {       // fallback cluster of 16: the last four CTAs only keep the cluster alive
    cluster.sync();
    return;
  }

  // ---- pieces of the step that run at two places (speculative Adam, see the end of the step) ----
  bool pending = false;      // the norms of the last finished step have been pushed but not yet checked
  int pend_par = 0;
  float pend_inv_b = 0.f;
  // The step barrier = the all-to-all of (sum g^2, sum theta^2): every CTA pushes 16 bytes to each of the other 11 and waits
  // for 11 x 16 bytes on its own mbarrier.  A CTA pushes only after its last read of any exchanged buffer and checks the norms
  // before it pushes anything of the next step, so nobody can overwrite h1 / the partial-output blocks / the dh1 slots of a
  // CTA that still reads them (every caller has passed a __syncthreads after its last such read).
  // Thread p < 12 holds (ssq, t2) in registers and stores them straight into CTA p's slot with st.async: no local staging
  // copy, proxy fence or block barrier in front, and twelve independent stores instead of eleven bulk copies that one SM's
  // copy engine issues one after the other.  Thread `rank` writes the own slot; a __syncthreads precedes every resolve_clip.
  auto step_barrier_push = [&](int par, float ssq, float t2) {
    if (tid < NCTA) {
      float* mine = xin + (par * 16 + static_cast<int>(rank)) * 4;
      const float4 v = make_float4(ssq, t2, 0.f, 0.f);
      if (tid == static_cast<int>(rank)) *reinterpret_cast<float4*>(mine) = v;
      else st_async16(mapa(smem_u32(mine), tid), v, mapa(smem_u32(&bar_ss[tcount & 1u]), tid));
    }
  };
  auto step_barrier_wait = [&]() {
    uint64_t* bar = &bar_ss[tcount & 1u];
    mbar_wait_cluster(bar, (tcount >> 1) & 1u);
    if (tid == 0) mbar_expect_tx(bar, (NCTA - 1) * 16);
    ++tcount;
  };
  // layer 1 of the forward: own 16 units of h1 into the own (swizzled) slice block
  auto layer1 = [&]() {
    float acc[1][4];
    warp_gemm_kk<8 * NT1>(acc, x, ldx, w1s, ldx, mt * 16, ntl * 8);
    const float2 bb = *reinterpret_cast<const float2*>(b1s + cA);
    const int cs = cA ^ (((rA >> 1) & 1) << 3);     // swizzled column inside the own slice block (rows rA and rA + 8 alike)
    *reinterpret_cast<float2*>(h1 + q * H1Q + rA * SL + cs) = make_float2(spo_tanh_fast(acc[0][0] + bb.x), spo_tanh_fast(acc[0][1] + bb.y));
    *reinterpret_cast<float2*>(h1 + q * H1Q + (rA + 8) * SL + cs) = make_float2(spo_tanh_fast(acc[0][2] + bb.x), spo_tanh_fast(acc[0][3] + bb.y));
    fence_proxy_async();                            // the slice is read by the bulk-copy engine next
  };
  // the twelve (sum g^2, sum theta^2) pairs of a finished step -> the clip coefficient (all that gates the next h1 push)
  auto resolve_clip = [&](int par) -> float {
    float total = 0.f;
#pragma unroll
    for (int b = 0; b < NCTA; ++b) total += xin[(par * 16 + b) * 4];   // every thread adds them in CTA order
    // clip coefficient max_norm / (norm + 1e-6), capped at 1 (SFU sqrt and division: <= 2 ulp, exactly 1 below the limit)
    return fminf(__fdividef(a.hp.max_grad_norm, __fadd_rn(sqrt_approx(total), 1e-6f)), 1.f);
  };
  // ... and the logged loss of that step (thread 0 of quarter 0, ppo_lag.py:330-336): critics include the L2 term over the
  // whole net.  Runs before the loss rows of the next step add to step_loss.
  auto log_loss = [&](int par, float inv_b) {
    if (tid != 0) return;
    if (q == 0 && active) {
      float t2net = 0.f;
#pragma unroll
      for (int b = 0; b < NCTA; ++b)
        if (b / NQ == net) t2net += xin[(par * 16 + b) * 4 + 1];
      float L;
      if (!is_actor) L = fmaf(a.hp.critic_l2, t2net, __fmul_rn(step_loss, inv_b));
      else if (a.kind == SPO_LOSS_PPO_CLIP) L = __fmul_rn(step_loss, inv_b);
      else L = __fsub_rn(__fmul_rn(step_loss, inv_b),
                         __fmul_rn(__fmul_rn(__fdiv_rn(1.f, a.hp.focops_lam), __fmul_rn(step_aux0, inv_b)), __fmul_rn(step_aux1, inv_b)));
      acc_loss += static_cast<double>(L);
    }
    step_loss = 0.f; step_aux0 = 0.f; step_aux1 = 0.f;
  };
  auto adam_k = [&](int par) {
    const float* kp = adk + 8 * par;
    AdamK k;
    k.w1 = kp[0]; k.b2 = kp[1]; k.w2 = kp[2]; k.ibc2s = kp[3]; k.eps = kp[4]; k.ss = kp[5];
    return k;
  };
  // Adam is split by what the next step needs first.  Layer 1 needs W1 / b1 only: their Adam runs at the end of a step,
  // speculatively with clip = 1 (adam_l1 with save: (theta, m, v) go to the backup first).  W2, b2, W3, b3 and log_std get
  // theirs in the next step while the h1 blocks travel, once the clip is known (adam_rest): no backup, no redo.
  // In both: all loads first, then the arithmetic, then all stores -- shared-memory loads cannot be moved across possibly
  // aliasing stores by the compiler, which would serialise the load -> sqrt -> rcp -> store chains of a thread.
  constexpr int NWB = 4 * NT1 + 1;   // backed-up entries per thread: 4 per block of W1, the b1 entry (threads < SL)
  auto adam_l1 = [&](float clip, bool save, const AdamK& k) {
    float w1v[NT1][4];
    float bv = 0.f, bg = 0.f;
#pragma unroll
    for (int e = 0; e < 4; e += 2) {
#pragma unroll
      for (int i = 0; i < NT1; ++i) {
        int j, kc;
        frag_jk(e, wid + 8 * i, j, kc);
        const float2 t = *reinterpret_cast<const float2*>(w1s + j * ldx + kc);   // columns >= D are zero padding
        w1v[i][e] = t.x; w1v[i][e + 1] = t.y;
      }
    }
    if (tid < SP_B2) { bv = sp[tid]; bg = gsmall[tid]; }
    if (save) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
#pragma unroll
        for (int i = 0; i < NT1; ++i) {
          bk[(0 * NWB + 4 * i + e) * UT + tid] = w1v[i][e];
          bk[(1 * NWB + 4 * i + e) * UT + tid] = mW1[i][e];
          bk[(2 * NWB + 4 * i + e) * UT + tid] = vW1[i][e];
        }
      }
      if (tid < SP_B2) {
        bk[(0 * NWB + NWB - 1) * UT + tid] = bv;
        bk[(1 * NWB + NWB - 1) * UT + tid] = sp_m;
        bk[(2 * NWB + NWB - 1) * UT + tid] = sp_v;
      }
    }
#pragma unroll
    for (int e = 0; e < 4; e += 2) {
#pragma unroll
      for (int i = 0; i < NT1; ++i) {
        // padded columns (kc >= D): gradient 0, moments 0 -> the update is exactly 0, the padding stays 0
        w1v[i][e] = adam_update(w1v[i][e], __fmul_rn(gW1[i][e], clip), mW1[i][e], vW1[i][e], k);
        w1v[i][e + 1] = adam_update(w1v[i][e + 1], __fmul_rn(gW1[i][e + 1], clip), mW1[i][e + 1], vW1[i][e + 1], k);
      }
    }
    if (tid < SP_B2) bv = adam_update(bv, __fmul_rn(bg, clip), sp_m, sp_v, k);
#pragma unroll
    for (int e = 0; e < 4; e += 2) {
#pragma unroll
      for (int i = 0; i < NT1; ++i) {
        int j, kc;
        frag_jk(e, wid + 8 * i, j, kc);
        *reinterpret_cast<float2*>(w1s + j * ldx + kc) = make_float2(w1v[i][e], w1v[i][e + 1]);
      }
    }
    if (tid < SP_B2) sp[tid] = bv;
  };
  // undo a speculative W1 / b1 step: weights back into shared memory, moments back into the registers
  auto adam_l1_restore = [&]() {
#pragma unroll
    for (int e = 0; e < 4; e += 2) {
#pragma unroll
      for (int i = 0; i < NT1; ++i) {
        int j, kc;
        frag_jk(e, wid + 8 * i, j, kc);
        *reinterpret_cast<float2*>(w1s + j * ldx + kc) =
            make_float2(bk[(0 * NWB + 4 * i + e) * UT + tid], bk[(0 * NWB + 4 * i + e + 1) * UT + tid]);
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
#pragma unroll
      for (int i = 0; i < NT1; ++i) {
        mW1[i][e] = bk[(1 * NWB + 4 * i + e) * UT + tid];
        vW1[i][e] = bk[(2 * NWB + 4 * i + e) * UT + tid];
      }
    }
    if (tid < SP_B2) {
      sp[tid] = bk[(0 * NWB + NWB - 1) * UT + tid];
      sp_m = bk[(1 * NWB + NWB - 1) * UT + tid];
      sp_v = bk[(2 * NWB + NWB - 1) * UT + tid];
    }
  };
  // the W1 / b1 gradients are cleared once the clip is known (the redo of a clipped step still reads them)
  auto clear_l1_grads = [&]() {
#pragma unroll
    for (int e = 0; e < 4; ++e)
#pragma unroll
      for (int i = 0; i < NT1; ++i) gW1[i][e] = 0.f;
    if (tid < SP_B2) gsmall[tid] = 0.f;
  };
  // row-independent pieces of the Gaussian log-density of action dim j from its log_std
  auto set_lsc = [&](int j, float ls) {
    const float sd = expf(ls);
    lsc[4 * j + 0] = sd;
    lsc[4 * j + 1] = __fdiv_rn(1.f, __fmul_rn(sd, sd));
    lsc[4 * j + 2] = logf(sd);
  };
  // Adam with the actual clip on the rest of this thread's parameters (W2 fragments, small entries past b1), then their
  // gradients are cleared for the step that follows.  The owners of log_std refresh lsc from the new value at once.
  auto adam_rest = [&](float clip, const AdamK& k) {
    float2 w2v[2];
    float spv = 0.f, spg = 0.f, spv1 = 0.f, spg1 = 0.f;   // small entries tid and tid + UT
    const bool own0 = tid >= SP_B2 && tid < SPN;
#pragma unroll
    for (int e = 0; e < 4; e += 2) {
      int j, kc;
      frag_jk(e, wid, j, kc);
      w2v[e >> 1] = *reinterpret_cast<const float2*>(w2s + j * LDA + kc);
    }
    if (own0) { spv = sp[tid]; spg = gsmall[tid]; }
    if constexpr (SPT > 1) {
      if (tid + UT < SPN) { spv1 = sp[tid + UT]; spg1 = gsmall[tid + UT]; }
    }
#pragma unroll
    for (int e = 0; e < 4; e += 2) {
      w2v[e >> 1].x = adam_update(w2v[e >> 1].x, __fmul_rn(gW2[0][e], clip), mW2[e], vW2[e], k);
      w2v[e >> 1].y = adam_update(w2v[e >> 1].y, __fmul_rn(gW2[0][e + 1], clip), mW2[e + 1], vW2[e + 1], k);
    }
    if (own0 && sp_valid) {
      spv = adam_update(spv, __fmul_rn(spg, clip), sp_m, sp_v, k);
      if (tid >= SP_LS) set_lsc(tid - SP_LS, spv);   // valid log_std entries: actor, j < A
    }
    if constexpr (SPT > 1) {
      if (tid + UT < SPN && sp_valid1) {
        spv1 = adam_update(spv1, __fmul_rn(spg1, clip), sp_m1, sp_v1, k);
        if (tid + UT >= SP_LS) set_lsc(tid + UT - SP_LS, spv1);
      }
    }
#pragma unroll
    for (int e = 0; e < 4; e += 2) {
      int j, kc;
      frag_jk(e, wid, j, kc);
      *reinterpret_cast<float2*>(w2s + j * LDA + kc) = w2v[e >> 1];
    }
    if (own0) { sp[tid] = spv; gsmall[tid] = 0.f; }
    if constexpr (SPT > 1) {
      if (tid + UT < SPN) { sp[tid + UT] = spv1; gsmall[tid + UT] = 0.f; }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) gW2[0][e] = 0.f;
  };

  int64_t step = 0;
  int sub = 0;
  auto next_tile = [&]() { if (++sub == tps) { sub = 0; ++step; } };
  for (int64_t qt = 0; qt < n_tiles; ++qt, next_tile()) {
    x = slots + (qt % NSLOT) * TILEF;
    aux = x + SPO_ROWS * ldx;
    int64_t rs64 = a.perm_len - step * a.batch;
    if (rs64 > a.batch) rs64 = a.batch;
    const int rows_step = static_cast<int>(rs64);
    int rows = rows_step - sub * SPO_ROWS;
    rows = rows < 0 ? 0 : (rows > SPO_ROWS ? SPO_ROWS : rows);
    const bool last_tile = (sub == tps - 1);
    const float inv_b = __fdiv_rn(1.f, static_cast<float>(rows_step));
    const unsigned seq = static_cast<unsigned>(a.comm.seq_base + static_cast<unsigned long long>(step_idx) + 1ull);
    const int par = static_cast<int>(step_idx & 1);
    // Cross-GPU exchange: every word goes to every peer (one NVLink hop), each rank sums all copies itself in rank order.
    // (A two-hop variant -- every word reduced by one owner rank and redistributed, 3.6x less NVLink traffic at 8 GPUs --
    // was built and dropped: the second hop cost more than the bytes it saved.)
    // push `n` of this thread's gradient values (words (w0 + i) * UT + tid of the CTA slot) to every peer GPU
    auto dp_push = [&](const float* vals, auto n_c, int w0) {
      constexpr int n = decltype(n_c)::value;
      const size_t base = ((static_cast<size_t>(seq & 1u) * world + me) * NCTA + rank) * DPW;
      for (int r = 0; r < world; ++r) {
        if (r == me) continue;
        float2* dst = reinterpret_cast<float2*>(a.comm.grad_bufs[r]) + base;
#pragma unroll
        for (int i = 0; i < n; ++i) st_ll(dst + (w0 + i) * UT + tid, vals[i], seq);
      }
    };
    // the receive for 4..8 ranks: three words of ALL peers per round (up to 21 requests in flight) instead of all words of one
    // peer per round: 3 L2 round trips at 8 GPUs instead of 7
    auto dp_sum_wide = [&](float (&g2)[4], float (&g1)[NT1][4], float& gs) {
      constexpr int NW = 4 * (1 + NT1) + 1, G = 3;
      const unsigned limit = a.comm.spin_limit ? a.comm.spin_limit : 400000000u;
      const float inv_w = __fdiv_rn(1.f, static_cast<float>(world));
      float val[NW];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        val[e] = g2[e];
#pragma unroll
        for (int i = 0; i < NT1; ++i) val[4 * (1 + i) + e] = g1[i][e];
      }
      val[NW - 1] = gs;
      const float2* slot0 = reinterpret_cast<const float2*>(a.comm.grad_bufs[me]) + (static_cast<size_t>(seq & 1u) * world * NCTA + rank) * DPW + tid;
      const size_t rstride = static_cast<size_t>(NCTA) * DPW;
#pragma unroll
      for (int i0 = 0; i0 < NW; i0 += G) {
        unsigned need = 0;
#pragma unroll
        for (int j = 0; j < G; ++j)
          if (i0 + j < NW && ((i0 + j < NW - 1) || tid < SPN))
#pragma unroll
            for (int r = 0; r < 8; ++r)
              if (r < world && r != me) need |= 1u << (r * G + j);
        unsigned got = 0, polls = 0;
        float v[8][G];
        while (got != need) {
          unsigned wa[8][G], wb[8][G];
#pragma unroll
          for (int r = 0; r < 8; ++r)
#pragma unroll
            for (int j = 0; j < G; ++j)
              if (((need & ~got) >> (r * G + j)) & 1u)
                asm volatile("ld.relaxed.sys.global.v2.b32 {%0, %1}, [%2];" : "=r"(wa[r][j]), "=r"(wb[r][j]) : "l"(slot0 + r * rstride + (i0 + j) * UT) : "memory");
#pragma unroll
          for (int r = 0; r < 8; ++r)
#pragma unroll
            for (int j = 0; j < G; ++j)
              if ((((need & ~got) >> (r * G + j)) & 1u) && wb[r][j] == seq) { v[r][j] = __uint_as_float(wa[r][j]); got |= 1u << (r * G + j); }
          if (got != need) {
            if (*reinterpret_cast<volatile int*>(&comm_dead)) break;
            if (++polls > limit) { comm_dead = 1; atomicExch(&ctrl->stop, 2); break; }
          }
        }
#pragma unroll
        for (int j = 0; j < G; ++j)
          if (i0 + j < NW) {
            float acc = 0.f;
#pragma unroll
            for (int r = 0; r < 8; ++r)
              if (r < world) acc += (r == me) ? val[i0 + j] : (((got >> (r * G + j)) & 1u) ? v[r][j] : 0.f);
            val[i0 + j] = __fmul_rn(acc, inv_w);
          }
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        g2[e] = val[e];
#pragma unroll
        for (int i = 0; i < NT1; ++i) g1[i][e] = val[4 * (1 + i) + e];
      }
      gs = val[NW - 1];
    };
    // rank-ordered sum of ALL of this thread's gradient words (4 of dW2, 4 per block of dW1, one small entry for
    // tid < SPN) with the words received from every peer GPU, scaled by 1/world.  The words of a peer are requested
    // together and tested afterwards: a sys-scope load is an L2 round trip (~0.35 us), nine of them one after the other
    // were most of the +3.9 us per step of the first version at 2 GPUs.
    auto dp_sum_all = [&](float (&g2)[4], float (&g1)[NT1][4], float& gs) {
      constexpr int NW = 4 * (1 + NT1) + 1;
      const unsigned limit = a.comm.spin_limit ? a.comm.spin_limit : 400000000u;
      const unsigned need = (tid < SPN) ? ((1u << NW) - 1u) : ((1u << (NW - 1)) - 1u);
      float acc[NW];
#pragma unroll
      for (int i = 0; i < NW; ++i) acc[i] = 0.f;
      for (int r = 0; r < world; ++r) {
        if (r == me) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            acc[e] += g2[e];
#pragma unroll
            for (int i = 0; i < NT1; ++i) acc[4 * (1 + i) + e] += g1[i][e];
          }
          acc[NW - 1] += gs;
          continue;
        }
        const float2* src = reinterpret_cast<const float2*>(a.comm.grad_bufs[me]) + ((static_cast<size_t>(seq & 1u) * world + r) * NCTA + rank) * DPW + tid;
        unsigned got = 0, polls = 0;
        float v[NW];
#pragma unroll
        for (int i = 0; i < NW; ++i) v[i] = 0.f;
        while (got != need) {
          unsigned wa[NW], wb[NW];
#pragma unroll
          for (int i = 0; i < NW; ++i)
            if (!((got >> i) & 1u) && ((need >> i) & 1u))
              asm volatile("ld.relaxed.sys.global.v2.b32 {%0, %1}, [%2];" : "=r"(wa[i]), "=r"(wb[i]) : "l"(src + i * UT) : "memory");
#pragma unroll
          for (int i = 0; i < NW; ++i)
            if (!((got >> i) & 1u) && ((need >> i) & 1u) && wb[i] == seq) { v[i] = __uint_as_float(wa[i]); got |= 1u << i; }
          if (got != need) {
            if (*reinterpret_cast<volatile int*>(&comm_dead)) break;
            if (++polls > limit) { comm_dead = 1; atomicExch(&ctrl->stop, 2); break; }
          }
        }
#pragma unroll
        for (int i = 0; i < NW; ++i) acc[i] += v[i];
      }
      const float inv_w = __fdiv_rn(1.f, static_cast<float>(world));
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        g2[e] = __fmul_rn(acc[e], inv_w);
#pragma unroll
        for (int i = 0; i < NT1; ++i) g1[i][e] = __fmul_rn(acc[4 * (1 + i) + e], inv_w);
      }
      gs = __fmul_rn(acc[NW - 1], inv_w);
    };

    if (active) mbar_wait(&bar_tile[qt % NSLOT], static_cast<uint32_t>(qt / NSLOT) & 1u);   // tile qt has landed
    __syncthreads();   // Adam's weight writes visible
    PHASE_MARK(0);   // top of the step: slot wait + barrier

    // ---------------- forward, layer 1: own 16 units ----------------
    if (active) layer1();
    PHASE_MARK(2);   // layer-1 product + tanh
    // The norms of the PREVIOUS step have been travelling since its end (SPECULATION, see the end of the step): W1 / b1 already
    // had their Adam step with clip = 1.  Now, before anything of this step leaves the CTA, check them.
    const bool defer = pending;    // the previous step's Adam on W2, b2, W3, b3, log_std runs in this tile's h1 window
    float clip = 1.f;
    if (pending) {
      pending = false;
      step_barrier_wait();
      PHASE_MARK(9);   // wait for the previous step's norms
      clip = resolve_clip(pend_par);
      if (active) {
        if (clip < 1.f) {          // rare: the joint norm exceeded max_grad_norm -- undo W1 / b1, redo with the clip, redo layer 1
          __syncthreads();
          adam_l1_restore();
          adam_l1(clip, false, adam_k(pend_par));
          __syncthreads();
          layer1();
        }
        clear_l1_grads();
      }
    }
    PHASE_MARK(1);   // resolve clip (+ rollback)
    float yv[AC];                                     // output-layer rows of this thread's row r4 (after the y exchange)
    if (active) {
      __syncthreads();                                // own slice complete (and fenced towards the async proxy)
      if (lane == 0 && wid < NQ && wid != q)          // all-gather of h1: the own 4 KB block goes to the three peers of the net
        bulk_push(mapa(smem_u32(h1 + q * H1Q), grp0 + wid), h1 + q * H1Q, H1Q * 4, mapa(smem_u32(&bar_h1), grp0 + wid));
      // while the blocks travel: the rest of the previous step's Adam step, with the actual clip (so never redone)
      if (defer) {
        adam_rest(clip, adam_k(pend_par));
        __syncthreads();                              // W2 / b2 / W3 / b3 / log_std and lsc final before layer 2 reads them
      } else if (qt == 0 && is_actor && tid >= UT - 32 && tid - (UT - 32) < A) {
        set_lsc(tid - (UT - 32), log_std[tid - (UT - 32)]);   // first tile of the launch (later tiles of a step keep theirs)
      }
      PHASE_MARK(19);  // h1 push, Adam on W2 .. log_std
      mbar_wait(&bar_h1, ph_x);                       // ... and theirs have landed here
      if (tid == 0) mbar_expect_tx(&bar_h1, (NQ - 1) * H1Q * 4);
      PHASE_MARK(3);   // h1 all-gather (pushed)
      // ---------------- forward, layer 2 + partial output layer ----------------
      {
        float acc[1][4];
        warp_gemm_l2(acc, h1, w2s, LDA, mt * 16, ntl * 8);
        const float2 bb = *reinterpret_cast<const float2*>(b2s + cA);
        *reinterpret_cast<float2*>(h2s + rA * LDS + cA) = make_float2(spo_tanh_fast(acc[0][0] + bb.x), spo_tanh_fast(acc[0][1] + bb.y));
        *reinterpret_cast<float2*>(h2s + (rA + 8) * LDS + cA) = make_float2(spo_tanh_fast(acc[0][2] + bb.x), spo_tanh_fast(acc[0][3] + bb.y));
      }
      __syncthreads();
      // output layer, partial over the own 16 hidden units: thread (row r4, quarter of the slice k4), two shuffles
      {
        const float4 hv = *reinterpret_cast<const float4*>(h2s + r4 * LDS + 4 * k4);
        for (int o = 0; o < O; o += 2) {     // two outputs per trip: their shuffle chains overlap (rows >= O of w3 are allocated)
          const float4 wa = *reinterpret_cast<const float4*>(w3s + o * SL + 4 * k4);
          const float4 wb = *reinterpret_cast<const float4*>(w3s + (o + 1) * SL + 4 * k4);
          float sa = fmaf(hv.x, wa.x, hv.y * wa.y) + fmaf(hv.z, wa.z, hv.w * wa.w);
          float sb = fmaf(hv.x, wb.x, hv.y * wb.y) + fmaf(hv.z, wb.z, hv.w * wb.w);
          sa += __shfl_xor_sync(0xffffffffu, sa, 1);
          sb += __shfl_xor_sync(0xffffffffu, sb, 1);
          sa += __shfl_xor_sync(0xffffffffu, sa, 2);
          sb += __shfl_xor_sync(0xffffffffu, sb, 2);
          if (k4 == (o & 3)) yblk[q * YQ + r4 * AC + o] = sa;
          if (k4 == ((o + 1) & 3) && o + 1 < O) yblk[q * YQ + r4 * AC + o + 1] = sb;
        }
        fence_proxy_async();
      }
      __syncthreads();
      if (lane == 0 && wid < NQ && wid != q)          // all-gather of the partial outputs: 2 KB to each peer of the net
        bulk_push(mapa(smem_u32(yblk + q * YQ), grp0 + wid), yblk + q * YQ, YQ * 4, mapa(smem_u32(&bar_y), grp0 + wid));
      PHASE_MARK(4);   // layer 2 + partial output layer
      // the row's side data, read while the partial outputs travel
      float pa[DH], psd[DH], piv[DH], pls[DH], plogp = 0.f, padv = 0.f, ptgt = 0.f;
#pragma unroll
      for (int h = 0; h < DH; ++h) pa[h] = 0.f;
#pragma unroll
      for (int h = 0; h < DH; ++h) psd[h] = 1.f;
#pragma unroll
      for (int h = 0; h < DH; ++h) piv[h] = 1.f;
#pragma unroll
      for (int h = 0; h < DH; ++h) pls[h] = 0.f;
      {
        const float* axp = aux + r4 * AUXW;
        if (is_actor) {
#pragma unroll
          for (int h = 0; h < DH; ++h) {
            const int j = k4 + 4 * h;
            if (j < A) { pa[h] = axp[j]; psd[h] = lsc[4 * j]; piv[h] = lsc[4 * j + 1]; pls[h] = lsc[4 * j + 2]; }
          }
          plogp = axp[AUX_LOGP];
          padv = axp[AUX_ADV];
        } else if (k4 == 0) {
          ptgt = axp[AUX_TGT + (net == 2 ? 1 : 0)];
        }
      }
      // ... and bookkeeping nobody needs before the loss rows: the previous step's logged loss (it reads step_loss before
      // this step's loss rows add to it), the bias-corrected Adam scalars of this step (read at its end and in the next
      // step's first tile; double-buffered by step parity, as the previous step's set is still read there)
      if (defer) log_loss(pend_par, pend_inv_b);
      if (last_tile) {
        float* kp = adk + 8 * par;
        if (tid == UT - 32) {
          b1pow *= static_cast<double>(a.hp.beta1);
          kp[5] = -__fdiv_rn(lr, static_cast<float>(1.0 - b1pow));
        } else if (tid == UT - 64) {
          b2pow *= static_cast<double>(a.hp.beta2);
          kp[3] = __fdiv_rn(1.f, sqrtf(static_cast<float>(1.0 - b2pow)));
        }
      }
      mbar_wait(&bar_y, ph_x);
      if (tid == 0) mbar_expect_tx(&bar_y, (NQ - 1) * YQ * 4);
      PHASE_MARK(5);   // y all-gather (pushed)
      // y[r][o] = b3[o] + sum over the four quarters: lane k4 of a row reads quarter k4's partial, a butterfly over the
      // four lanes finishes the sum (fixed order (p0 + p1) + (p2 + p3) in every CTA)
      {
        const float4* yp = reinterpret_cast<const float4*>(yblk + k4 * YQ + r4 * AC);
#pragma unroll
        for (int c = 0; c < AC / 4; ++c) {
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (c == 0 || O > 4 * c) v = yp[c];
          yv[4 * c] = v.x; yv[4 * c + 1] = v.y; yv[4 * c + 2] = v.z; yv[4 * c + 3] = v.w;
        }
#pragma unroll
        for (int o = 0; o < AC; ++o) {
          if (o < O) {     // O is uniform over the CTA
            yv[o] += __shfl_xor_sync(0xffffffffu, yv[o], 1);
            yv[o] += __shfl_xor_sync(0xffffffffu, yv[o], 2);
            yv[o] = __fadd_rn(yv[o], b3[o]);
          }
        }
      }
      // ---------------- loss and d loss / d output: thread (row r4, action dims j = k4 + 4h, h < AC / 4) ----------------
      float part0 = 0.f, part1 = 0.f, part2 = 0.f;
      {
        const int r = r4;
        const bool valid = r < rows;
        float* ax = aux + r * AUXW;
        if (!is_actor) {
          if (k4 == 0) {
            const float dv = __fsub_rn(yv[0], ptgt);
            part0 = valid ? __fmul_rn(dv, dv) : 0.f;
            dy[r * AC] = valid ? __fmul_rn(__fmul_rn(__fmul_rn(2.f, dv), inv_b), vcoef) : 0.f;
          }
        } else {
          float term[DH], klj[DH], dmu_lp[DH], dls_lp[DH], dmu_kl[DH], dls_kl[DH];
#pragma unroll
          for (int h = 0; h < DH; ++h) term[h] = 0.f;
#pragma unroll
          for (int h = 0; h < DH; ++h) klj[h] = 0.f;
#pragma unroll
          for (int h = 0; h < DH; ++h) dmu_kl[h] = 0.f;
#pragma unroll
          for (int h = 0; h < DH; ++h) dls_kl[h] = 0.f;
#pragma unroll
          for (int h = 0; h < DH; ++h) {
            const int j = k4 + 4 * h;
            dmu_lp[h] = 0.f; dls_lp[h] = 0.f;
            if (j < A) {
              // yv[j] with a compile-time index: j = k4 + 4h
              float mean;
              if constexpr (DH == 2) {   // (this form keeps the AC = 8 instruction stream of the narrow-only kernel)
                const float m_lo = (k4 == 0) ? yv[0] : (k4 == 1) ? yv[1] : (k4 == 2) ? yv[2] : yv[3];
                const float m_hi = (k4 == 0) ? yv[4] : (k4 == 1) ? yv[5] : (k4 == 2) ? yv[6] : yv[7];
                mean = h ? m_hi : m_lo;
              } else {
                mean = (k4 == 0) ? yv[4 * h] : (k4 == 1) ? yv[4 * h + 1] : (k4 == 2) ? yv[4 * h + 2] : yv[4 * h + 3];
              }
              const float std = psd[h], inv_var = piv[h];
              const float diff = __fsub_rn(pa[h], mean);
              const float d2 = __fmul_rn(diff, diff);
              const float q2 = __fmul_rn(d2, inv_var);           // (a - mu)^2 / var
              term[h] = __fsub_rn(__fsub_rn(__fmul_rn(-0.5f, q2), pls[h]), kLogSqrt2Pi);
              dmu_lp[h] = __fmul_rn(diff, inv_var);
              dls_lp[h] = __fsub_rn(q2, 1.f);
              if (a.kind == SPO_LOSS_FOCOPS) {
                // KL(new || old), torch _kl_normal_normal(p=new, q=old); padded rows carry zeros: keep them finite
                const float os = valid ? ax[AUX_OSTD + j] : 1.f, om = ax[AUX_OMEAN + j];
                const float ios = __fdiv_rn(1.f, os);
                const float sr = __fmul_rn(std, ios);
                const float vr = __fmul_rn(sr, sr);
                const float dm = __fmul_rn(__fsub_rn(mean, om), ios);
                const float t1 = __fmul_rn(dm, dm);
                klj[h] = __fmul_rn(0.5f, __fsub_rn(__fsub_rn(__fadd_rn(vr, t1), 1.f), logf(vr)));
                dmu_kl[h] = __fmul_rn(dm, ios);
                dls_kl[h] = __fsub_rn(vr, 1.f);
              }
            }
          }
          // sums over the action dims: the 4 lanes of a row, AC / 4 dims each
          float lp = term[0], kl = klj[0];
#pragma unroll
          for (int h = 1; h < DH; ++h) { lp += term[h]; kl += klj[h]; }
          lp += __shfl_xor_sync(0xffffffffu, lp, 1);
          lp += __shfl_xor_sync(0xffffffffu, lp, 2);
          if (a.kind == SPO_LOSS_FOCOPS) {
            kl += __shfl_xor_sync(0xffffffffu, kl, 1);
            kl += __shfl_xor_sync(0xffffffffu, kl, 2);
          }
          const float ratio = expf(__fsub_rn(lp, plogp));
          const float adv = padv;
          if (a.kind == SPO_LOSS_PPO_CLIP) {
            const float s1 = __fmul_rn(ratio, adv);
            const float s2 = __fmul_rn(fminf(fmaxf(ratio, a.hp.clip_lo), a.hp.clip_hi), adv);
            if (k4 == 0) part0 = valid ? -fminf(s1, s2) : 0.f;
            // d(-mean(min))/d logp = -(1/B) * adv * ratio where the unclipped branch is active
            const float gl = (valid && s1 <= s2) ? -__fmul_rn(__fmul_rn(adv, ratio), inv_b) : 0.f;
#pragma unroll
            for (int h = 0; h < DH; ++h) {
              const int j = k4 + 4 * h;
              if (j < A) {
                dy[r * AC + j] = __fmul_rn(gl, dmu_lp[h]);
                dls[r * AC + j] = __fmul_rn(gl, dls_lp[h]);
              }
            }
          } else {
            // FOCOPS needs mean(mask) over the minibatch before gradients can be formed: stash per-row pieces,
            // finish after the block reduction below
            const float mask = (valid && kl <= a.hp.focops_kl) ? 1.f : 0.f;
            if (k4 == 0) {
              part0 = valid ? __fmul_rn(kl, mask) : 0.f;
              part1 = valid ? __fmul_rn(ratio, adv) : 0.f;
              part2 = mask;
            }
            const float gl = valid ? __fmul_rn(__fmul_rn(adv, ratio), inv_b) : 0.f;
#pragma unroll
            for (int h = 0; h < DH; ++h) {
              const int j = k4 + 4 * h;
              if (j < A) {
                dy[r * AC + j] = __fmul_rn(__fmul_rn(mask, inv_b), dmu_kl[h]);
                dls[r * AC + j] = __fmul_rn(__fmul_rn(mask, inv_b), dls_kl[h]);
                y[r * AC + j] = __fmul_rn(gl, dmu_lp[h]);
                ax[AUX_OMEAN + j] = __fmul_rn(gl, dls_lp[h]);   // the old-mean slot of the row is free now
              }
            }
          }
        }
        part0 = spo_warp_sum(part0);
        if (is_actor && a.kind == SPO_LOSS_FOCOPS) { part1 = spo_warp_sum(part1); part2 = spo_warp_sum(part2); }
        if (lane == 0) { red[wid * 4 + 0] = part0; red[wid * 4 + 1] = part1; red[wid * 4 + 2] = part2; }
      }
      __syncthreads();
      if (is_actor && a.kind == SPO_LOSS_FOCOPS) {
        // This formulation needs the whole minibatch in one tile (batch <= 64).  (focops.py uses batch 64.)
        float msum = 0.f;
#pragma unroll
        for (int w = 0; w < UT / 32; ++w) msum += red[w * 4 + 2];
        const float mbar = __fmul_rn(msum, inv_b);
        const float c2 = -__fmul_rn(__fdiv_rn(1.f, a.hp.focops_lam), mbar);
        const float* ax = aux + r4 * AUXW;
#pragma unroll
        for (int h = 0; h < DH; ++h) {
          const int j = k4 + 4 * h;
          if (j < A) {
            dy[r4 * AC + j] = __fadd_rn(dy[r4 * AC + j], __fmul_rn(c2, y[r4 * AC + j]));
            dls[r4 * AC + j] = __fadd_rn(dls[r4 * AC + j], __fmul_rn(c2, ax[AUX_OMEAN + j]));
          }
        }
        __syncthreads();
      }
      PHASE_MARK(6);   // y pull + loss rows

      // ---------------- backward ----------------
      // (b) dz2[r][kk] = (sum_o dy[r][o] * w3[o][kk]) * (1 - h2[r][kk]^2), own 16 columns
      {
        float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int o = 0; o < O; ++o) {
          const float d = dy[r4 * AC + o];
          const float4 wv = *reinterpret_cast<const float4*>(w3s + o * SL + 4 * k4);
          s4.x = fmaf(d, wv.x, s4.x); s4.y = fmaf(d, wv.y, s4.y); s4.z = fmaf(d, wv.z, s4.z); s4.w = fmaf(d, wv.w, s4.w);
        }
        const float4 h = *reinterpret_cast<const float4*>(h2s + r4 * LDS + 4 * k4);
        s4.x *= (1.f - h.x * h.x); s4.y *= (1.f - h.y * h.y); s4.z *= (1.f - h.z * h.z); s4.w *= (1.f - h.w * h.w);
        *reinterpret_cast<float4*>(dz2s + r4 * LDS + 4 * k4) = s4;
      }
      __syncthreads();
      PHASE_MARK(7);   // dz2
      // (c) dh1 partial [64 x 64] = dz2[:, slice] W2[slice, :], stored by destination quarter; block d is pushed to CTA d
      {
        float acc[4][4];
        warp_gemm<4, 2, false>(acc, dz2s, LDS, 1, w2s, LDA, 1, mt * 16, (wid >> 2) * 32);
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int c = (wid >> 2) * 32 + nt * 8 + 2 * t4;
          float* blk = dh1b + (c >> 4) * H1Q + (c & 15);
          *reinterpret_cast<float2*>(blk + rA * SL) = make_float2(acc[nt][0], acc[nt][1]);
          *reinterpret_cast<float2*>(blk + (rA + 8) * SL) = make_float2(acc[nt][2], acc[nt][3]);
        }
        fence_proxy_async();
      }
      __syncthreads();
      if (lane == 0 && wid < NQ && wid != q)          // reduce-scatter of dh1: the partial for CTA d's columns goes to its slot [q]
        bulk_push(mapa(smem_u32(dh1in + q * H1Q), grp0 + wid), dh1b + wid * H1Q, H1Q * 4, mapa(smem_u32(&bar_dh), grp0 + wid));
      PHASE_MARK(8);   // dh1 partial product + push
      // (d) dW2[slice j][k] += sum_r dz2[r][j] * h1[r][k] (warp w: columns 8w..8w+7);  db2[j] += sum_r dz2[r][j]
      //     -- runs while the 12 KB of dh1 partials travel
      if (tid == 0) {   // the loss numerators of the tile (the block reduction of the loss rows; red is next written at the sum of squares)
        float l0 = 0.f, l1 = 0.f, l2 = 0.f;
#pragma unroll
        for (int w = 0; w < UT / 32; ++w) { l0 += red[w * 4]; l1 += red[w * 4 + 1]; l2 += red[w * 4 + 2]; }
        step_loss += l0;
        step_aux0 += l1;
        step_aux1 += l2;
      }
      warp_gemm_dw2(gW2, dz2s, LDS, h1, wid * 8);
      colsum_into(dz2s, gsmall + SP_B2);
      PHASE_MARK(10);  // loss numerators, dW2 + db2 (dh1 partials in flight)
      // (a) small grads of the output layer, own 16 columns: dW3[o][kk] = sum_r dy[r][o] h2[r][kk];
      //     -- nothing before the step's end needs them, so they too run while the dh1 partials travel;
      //     thread (kk = tid >> 4, rg = tid & 15) adds rows rg + 16 i, four shuffles finish each sum.
      //     db3[o] / dlog_std[j] (replicated in the four CTAs): column sums of dy / dls, same split.
      {
        const int kk = tid >> 4, rg = tid & 15;
        float hv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) hv[i] = h2s[(rg + 16 * i) * LDS + kk];
        // the column sums for db3 / dlog_std ride along with the first pair of dW3 sums (independent shuffle chains).
        // AC = 8: kk < 8 sums dy column kk (db3), kk >= 8 dls column kk - 8 (dlog_std); AC = 16: thread kk sums both columns kk.
        if constexpr (AC == 8) {
          const int col = kk & 7;
          const bool need = (kk < 8) ? (col < O) : (is_actor && col < A);
          const float* src = (kk < 8) ? dy : dls;
          float sc = 0.f;
          if (need) {
#pragma unroll
            for (int i = 0; i < 4; ++i) sc += src[(rg + 16 * i) * AC + col];
          }
          for (int o = 0; o < O; o += 2) {           // column o + 1 of dy exists (AC columns); its sum is dropped when >= O
            float sa = 0.f, sb = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float2 d = *reinterpret_cast<const float2*>(dy + (rg + 16 * i) * AC + o);
              sa = fmaf(d.x, hv[i], sa);
              sb = fmaf(d.y, hv[i], sb);
            }
#pragma unroll
            for (int m = 1; m < 16; m <<= 1) {
              sa += __shfl_xor_sync(0xffffffffu, sa, m);
              sb += __shfl_xor_sync(0xffffffffu, sb, m);
              if (o == 0) sc += __shfl_xor_sync(0xffffffffu, sc, m);
            }
            if (rg == 0) {
              gsmall[SP_W3 + o * SL + kk] += sa;
              if (o + 1 < O) gsmall[SP_W3 + (o + 1) * SL + kk] += sb;
            }
          }
          if (need && rg == 0) gsmall[(kk < 8 ? SP_B3 : SP_LS) + col] += sc;
        } else {
          const bool need_b3 = kk < O, need_ls = is_actor && kk < A;
          float sc = 0.f, sl = 0.f;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            if (need_b3) sc += dy[(rg + 16 * i) * AC + kk];
            if (need_ls) sl += dls[(rg + 16 * i) * AC + kk];
          }
          for (int o = 0; o < O; o += 2) {
            float sa = 0.f, sb = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float2 d = *reinterpret_cast<const float2*>(dy + (rg + 16 * i) * AC + o);
              sa = fmaf(d.x, hv[i], sa);
              sb = fmaf(d.y, hv[i], sb);
            }
#pragma unroll
            for (int m = 1; m < 16; m <<= 1) {
              sa += __shfl_xor_sync(0xffffffffu, sa, m);
              sb += __shfl_xor_sync(0xffffffffu, sb, m);
              if (o == 0) { sc += __shfl_xor_sync(0xffffffffu, sc, m); sl += __shfl_xor_sync(0xffffffffu, sl, m); }
            }
            if (rg == 0) {
              gsmall[SP_W3 + o * SL + kk] += sa;
              if (o + 1 < O) gsmall[SP_W3 + (o + 1) * SL + kk] += sb;
            }
          }
          if (rg == 0) {
            if (need_b3) gsmall[SP_B3 + kk] += sc;
            if (need_ls) gsmall[SP_LS + kk] += sl;
          }
        }
      }
      PHASE_MARK(20);  // dW3 / db3 / dlog_std (dh1 partials in flight)
      if (DP && world > 1 && last_tile) {
        // data-parallel ranks: dW2 / db2 / dW3 / db3 / dlog_std leave for the peer GPUs now, ahead of the dW1 product
        __syncthreads();                                   // gsmall[b2, w3, b3, log_std] complete
        float sv = (tid >= SP_B2 && tid < SPN) ? gsmall[tid] : 0.f;
        dp_push(gW2[0], IC<4>{}, 0);
        if (tid >= SP_B2 && tid < SPN) dp_push(&sv, IC<1>{}, 4 * (1 + NT1));
      }
      mbar_wait(&bar_dh, ph_x);
      if (tid == 0) mbar_expect_tx(&bar_dh, (NQ - 1) * H1Q * 4);
      // (e) dz1[r][jj] = (sum over the four partials, quarter order) * (1 - h1[r][16q + jj]^2)
      {
        float4 v[NQ];
#pragma unroll
        for (int d = 0; d < NQ; ++d) {
          const float* src = (d == q) ? dh1b + q * H1Q : dh1in + d * H1Q;
          v[d] = *reinterpret_cast<const float4*>(src + r4 * SL + 4 * k4);
        }
        float4 s4 = v[0];
#pragma unroll
        for (int d = 1; d < NQ; ++d) { s4.x += v[d].x; s4.y += v[d].y; s4.z += v[d].z; s4.w += v[d].w; }
        const float4 h = *reinterpret_cast<const float4*>(h1 + q * H1Q + r4 * SL + ((4 * k4) ^ (((r4 >> 1) & 1) << 3)));
        s4.x *= (1.f - h.x * h.x); s4.y *= (1.f - h.y * h.y); s4.z *= (1.f - h.z * h.z); s4.w *= (1.f - h.w * h.w);
        *reinterpret_cast<float4*>(dz1s + r4 * LDS + 4 * k4) = s4;
      }
      __syncthreads();
      PHASE_MARK(11);  // dh1 reduce + dz1
      // (f) dW1[slice j][k] += sum_r dz1[r][j] * x[r][k];  db1[j] += sum_r dz1[r][j]
#pragma unroll
      for (int i = 0; i < NT1; ++i)
        warp_gemm<1, 8, true>(reinterpret_cast<float (&)[1][4]>(gW1[i]), dz1s, 1, LDS, x, ldx, 1, 0, (wid + 8 * i) * 8);
      colsum_into(dz1s, gsmall + SP_B1);
      fence_proxy_async();   // the slot's reads (dW1 last) and the FOCOPS scratch writes precede the next bulk copy into it
      PHASE_MARK(12);  // dW1 + db1
    }

    __syncthreads();       // gsmall complete; every read and write of this tile's slot is done
    if (active && tid == UT - 32) issue_tile(qt + NSLOT);   // (a thread outside warp 0, which pushes the norms next)
    ph_x ^= active ? 1u : 0u;   // both pushed exchanges of this tile are consumed
    if (!last_tile) {
      // more tiles of the same step follow: the exchange only orders the buffer reuse
      step_barrier_push(par, 0.f, 0.f);
      step_barrier_wait();
      continue;
    }

    // ---------------- cross-GPU gradient sum (data-parallel ranks), in rank order ----------------
    if (DP && world > 1 && active) {
      float sv = 0.f;
      if (tid < SP_B2) { sv = gsmall[tid]; dp_push(&sv, IC<1>{}, 4 * (1 + NT1)); }
#pragma unroll
      for (int i = 0; i < NT1; ++i) dp_push(gW1[i], IC<4>{}, 4 * (1 + i));
      sv = (tid < SPN) ? gsmall[tid] : 0.f;
      if (world >= 4 && world <= 8) dp_sum_wide(gW2[0], gW1, sv);
      else dp_sum_all(gW2[0], gW1, sv);
      if (tid < SPN) gsmall[tid] = sv;
    }
    PHASE_MARK(13);  // cross-GPU gradient exchange

    // ---------------- joint gradient norm (cluster-wide), clip, Adam ----------------
    if (active) {
      float ss = 0.f, th2 = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        int j, k;
        frag_jk(e, wid, j, k);
        if (!is_actor) {
          const float th = w2s[j * LDA + k];
          gW2[0][e] = fmaf(reg, th, gW2[0][e]);
          th2 = fmaf(th, th, th2);
        }
        ss = fmaf(gW2[0][e], gW2[0][e], ss);
#pragma unroll
        for (int i = 0; i < NT1; ++i) {
          frag_jk(e, wid + 8 * i, j, k);
          if (k < D) {
            if (!is_actor) {
              const float t1 = w1s[j * ldx + k];
              gW1[i][e] = fmaf(reg, t1, gW1[i][e]);
              th2 = fmaf(t1, t1, th2);
            }
            ss = fmaf(gW1[i][e], gW1[i][e], ss);
          } else {
            gW1[i][e] = 0.f;   // padded observation columns are exact zeros anyway
          }
        }
      }
      if (tid < SPN && sp_valid) {
        const float th = sp[tid];
        const float g = fmaf(reg, th, gsmall[tid]);
        gsmall[tid] = g;
        if (sp_counted) { ss = fmaf(g, g, ss); th2 = fmaf(th, th, th2); }
      }
      if constexpr (SPT > 1) {
        if (tid + UT < SPN && sp_valid1) {
          const float th = sp[tid + UT];
          const float g = fmaf(reg, th, gsmall[tid + UT]);
          gsmall[tid + UT] = g;
          if (sp_counted1) { ss = fmaf(g, g, ss); th2 = fmaf(th, th, th2); }
        }
      }
      ss = spo_warp_sum(ss);
      if (!is_actor) th2 = spo_warp_sum(th2);
      if (lane == 0) *reinterpret_cast<float2*>(red + 16 + 2 * wid) = make_float2(ss, th2);
      __syncthreads();
    }
    {
      float s = 0.f, t2 = 0.f;
      if (tid < NCTA && active) {   // the twelve threads that push the pair, each with the same sum
#pragma unroll
        for (int w = 0; w < UT / 32; w += 2) {
          const float4 v = *reinterpret_cast<const float4*>(red + 16 + 2 * w);
          s += v.x + v.z; t2 += v.y + v.w;
        }
      }
      PHASE_MARK(14);  // regulariser + sum of squares
      step_barrier_push(par, s + extra_sumsq, t2);
      PHASE_MARK(17);  // norms pushed
    }
    // SPECULATION: the joint norm almost never exceeds max_grad_norm (clip = min(max_norm / (norm + 1e-6), 1) is exactly 1 then),
    // so W1 / b1 -- all that the next step's layer 1 reads -- get their Adam step NOW with clip = 1 ((theta, m, v) saved first),
    // and the next step's stage-in and layer-1 product follow while the twelve 16-byte pushes travel; the norms are checked
    // before that step pushes anything (top of the loop), and the rest of the Adam step runs there with the actual clip.  A step
    // whose norm does exceed the limit has its W1 / b1 step undone and redone there: results are bit-identical either way.
    if (active) adam_l1(1.f, true, adam_k(par));
    pending = true;
    pend_par = par;
    pend_inv_b = inv_b;
    PHASE_MARK(16);  // Adam on W1 / b1 + backup
    ++step_idx;
    // the __syncthreads at the top of the next iteration orders these weight writes before the next forward
  }
  if (pending) {         // the last step of the launch: its clip check and the rest of its Adam step, as at the top of a step
    __syncthreads();     // the own slot of the norms, written by one thread, is read by all
    step_barrier_wait();
    const float clip = resolve_clip(pend_par);
    if (active) {
      if (clip < 1.f) {
        __syncthreads();
        adam_l1_restore();
        adam_l1(clip, false, adam_k(pend_par));
      }
      log_loss(pend_par, pend_inv_b);
      adam_rest(clip, adam_k(pend_par));
    }
  }
  __syncthreads();

  // ---- write back: weights, moments, step counters, logged losses ----
  if (active) {
    for (int i = tid; i < SL * D; i += UT) {
      const int j = i / D, kx = i - j * D;
      a.params[off.w1 + (SL * q + j) * D + kx] = w1s[j * ldx + kx];
    }
    for (int i = tid; i < SL * SPO_HID; i += UT)
      a.params[off.w2 + (SL * q + (i >> 6)) * SPO_HID + (i & 63)] = w2s[(i >> 6) * LDA + (i & 63)];
    if (tid < SPN && sp_valid && (sp_counted || tid < SP_B3)) {
      a.params[sp_goff] = sp[tid];
      a.adam_m[sp_goff] = sp_m;
      a.adam_v[sp_goff] = sp_v;
    }
    if constexpr (SPT > 1) {
      if (tid + UT < SPN && sp_valid1 && (sp_counted1 || tid + UT < SP_B3)) {
        a.params[sp_goff1] = sp[tid + UT];
        a.adam_m[sp_goff1] = sp_m1;
        a.adam_v[sp_goff1] = sp_v1;
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      int j, kc;
      frag_jk(e, wid, j, kc);
      a.adam_m[off.w2 + (SL * q + j) * SPO_HID + kc] = mW2[e];
      a.adam_v[off.w2 + (SL * q + j) * SPO_HID + kc] = vW2[e];
#pragma unroll
      for (int i = 0; i < NT1; ++i) {
        frag_jk(e, wid + 8 * i, j, kc);
        if (kc < D) {
          a.adam_m[off.w1 + (SL * q + j) * D + kc] = mW1[i][e];
          a.adam_v[off.w1 + (SL * q + j) * D + kc] = vW1[i][e];
        }
      }
    }
    if (tid == 0 && q == 0) {
      a.adam_t[net] = t0 + static_cast<int>(n_steps);
      const int slot = (net == 0) ? 2 : (net == 1 ? 0 : 1);
      atomicAdd(&ctrl->loss_sum[slot], acc_loss);
    }
  }
#ifdef SPO_PHASE_TIMERS
  if (tid < 24) atomicAdd(&g_phase_cycles[rank & 15][tid], sm_phase__[tid]);
#endif
  if (rank == NQ && tid == 0) atomicAdd(reinterpret_cast<unsigned long long*>(&ctrl->steps), static_cast<unsigned long long>(n_steps));
  cluster.sync();  // no CTA may exit while a peer can still read its shared memory
}

inline int64_t upd_n_tiles(const UpdArgs& a) {
  return (a.perm_len + a.batch - 1) / a.batch * ((a.batch + SPO_ROWS - 1) / SPO_ROWS);
}

template <int NT1, int AC>
int launch_pack(const UpdArgs& a, cudaStream_t stream) {
  const int64_t n_tiles = upd_n_tiles(a);
  const int64_t blocks = (n_tiles * SPO_ROWS + 7) / 8;   // one warp per row, grid-stride beyond 2^16 blocks
  spo_pack_tiles<NT1, AC><<<static_cast<unsigned>(blocks < 65536 ? blocks : 65536), 256, 0, stream>>>(a, n_tiles);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

template <int NT1, int AC, bool DP>
int launch_update_kernel(const UpdArgs& a, cudaStream_t stream) {
  constexpr size_t smem = update_smem_bytes<NT1, AC>();
  static_assert(smem <= 227 * 1024, "shared memory of the update kernel");
  // 12 CTAs are needed; clusters above 8 are "non-portable" sizes: 12 is tried first, 16 (four CTAs idle) second.
  // The choice is cached per process: one process drives one GPU (torchrun-style data parallelism).
  static int cluster_size = 0;
  SPO_CUDA_TRY(cudaFuncSetAttribute(spo_update_kernel<NT1, AC, DP>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  SPO_CUDA_TRY(cudaFuncSetAttribute(spo_update_kernel<NT1, AC, DP>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  if (!cluster_size) {
    const char* env = getenv("SPO_CLUSTER");   // debugging aid: pin the cluster size (12 or 16)
    if (env && atoi(env) >= NCTA && atoi(env) <= 16) cluster_size = atoi(env);
  }
  for (int attempt = 0; attempt < 2; ++attempt) {
    const int cs = cluster_size ? cluster_size : (attempt == 0 ? NCTA : 16);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(cs);
    cfg.blockDim = dim3(UT);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cs;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, spo_update_kernel<NT1, AC, DP>, a);
    if (e == cudaSuccess) { cluster_size = cs; return SPO_OK; }
    if (cluster_size || attempt == 1) {
      spo_set_error("spo_pg_update: launch failed (cluster=%d): %s", cs, cudaGetErrorString(e));
      return SPO_ERR_CUDA;
    }
    (void)cudaGetLastError();  // clear and retry with the other cluster size
  }
  return SPO_ERR_CUDA;
}

// one pass: the packed tiles of the pass are allocated stream-ordered, written by spo_pack_tiles, read by the update
// kernel and freed, all on `stream`
template <int NT1, int AC, bool DP>
int launch_update(UpdArgs a, cudaStream_t stream) {
  cudaMemPool_t pool;
  int rc = spo_update_tile_pool(&pool);
  if (rc) return rc;
  const size_t bytes = static_cast<size_t>(upd_n_tiles(a)) * upd_tile_floats<NT1, AC>() * sizeof(float);
  SPO_CUDA_TRY(cudaMallocFromPoolAsync(reinterpret_cast<void**>(&a.tiles), bytes, pool, stream));
  rc = launch_pack<NT1, AC>(a, stream);
  if (rc == SPO_OK) rc = launch_update_kernel<NT1, AC, DP>(a, stream);
  const cudaError_t e = cudaFreeAsync(a.tiles, stream);
  if (rc == SPO_OK && e != cudaSuccess) {
    spo_set_error("spo_pg_update: cudaFreeAsync failed: %s", cudaGetErrorString(e));
    return SPO_ERR_CUDA;
  }
  return rc;
}

}  // namespace

// the AC = 16 launcher (spo_update_wide.cu); args: an UpdArgs, which keeps internal linkage like the kernel.
// pack_only: only spo_pack_tiles, into args->tiles (the test hook spo_debug_pack_tiles)
int spo_update_launch_wide(int nt1, const void* args, cudaStream_t stream, bool pack_only);
