// Warp-level tile GEMM on the legacy tensor path (mma.sync.m16n8k8 TF32) with 3xTF32 error
// compensation done in registers.
//
// Why this path for the 64-row tiles: a 4x4
// register-tiled FFMA GEMM pulls 2 B of shared-memory operands per FMA and is bound by the
// 128 B/clk shared-memory return bandwidth (4.1 k cycles per 64^3 GEMM); mma fragments need
// 0.19 B per FMA, the split x = hi + lo costs two
// full-rate ALU ops per loaded element, and lo*hi + hi*lo + hi*hi
// (small terms first) matches fp32 accumulation to ~3e-7 relative.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// hi = x with the 13 low mantissa bits cleared (what the tensor core would read anyway),
// lo = x - hi exactly (<= 13 significant bits; the hardware keeps its top 11).  One LOP3 and one
// FADD on the full-rate pipes -- cvt.rna.tf32.f32 is a quarter-rate conversion and was a
// co-bottleneck of the tile GEMMs.  Accuracy with small terms first: of the order of 1e-6 max abs error on
// |values| <= 2.8 at K = 64, slightly worse than rounded splits.
__device__ __forceinline__ void spo_split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(x) & 0xFFFFE000u;
  lo = __float_as_uint(x - __uint_as_float(hi));
}

__device__ __forceinline__ void spo_mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

template <int MT>
__device__ __forceinline__ void spo_mma_zero(float (&acc)[MT][2][4]) {
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;
}

// acc (warp patch of 16*MT rows x 16 cols at (m_base, n_base)) += A * B over k in [0, K), K % 8 == 0.
//   A(m, k) = A[m * a_sm + k * a_sk]      B(k, n) = B[k * b_sk + n * b_sn]      (shared memory)
// Fragment ownership (g = lane >> 2, t = lane & 3), per 16 x 8 mma tile (mt, nt):
//   acc[mt][nt][0..3] = C(m_base+16mt+g, n_base+8nt+2t), (.., +1), (row+8, ..), (row+8, +1)
template <int MT>
__device__ __forceinline__ void spo_warp_mma_3xtf32(float (&acc)[MT][2][4], const float* __restrict__ A, int a_sm, int a_sk,
                                                    const float* __restrict__ B, int b_sk, int b_sn, int m_base, int n_base, int K) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const float* a_ptr = A + (m_base + g) * a_sm + t * a_sk;
  const float* b_ptr = B + t * b_sk + (n_base + g) * b_sn;
#pragma unroll 4
  for (int k0 = 0; k0 < K; k0 += 8) {
    uint32_t ah[MT][4], al[MT][4], bh[2][2], bl[2][2];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      const float* p = a_ptr + mt * 16 * a_sm + k0 * a_sk;
      spo_split_tf32(p[0], ah[mt][0], al[mt][0]);
      spo_split_tf32(p[8 * a_sm], ah[mt][1], al[mt][1]);
      spo_split_tf32(p[4 * a_sk], ah[mt][2], al[mt][2]);
      spo_split_tf32(p[8 * a_sm + 4 * a_sk], ah[mt][3], al[mt][3]);
    }
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      const float* p = b_ptr + nt * 8 * b_sn + k0 * b_sk;
      spo_split_tf32(p[0], bh[nt][0], bl[nt][0]);
      spo_split_tf32(p[4 * b_sk], bh[nt][1], bl[nt][1]);
    }
    // small terms first; the two column tiles alternate so that an mma never directly follows the one
    // it depends on
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      spo_mma_tf32(acc[mt][0], al[mt], bh[0]);
      spo_mma_tf32(acc[mt][1], al[mt], bh[1]);
      spo_mma_tf32(acc[mt][0], ah[mt], bl[0]);
      spo_mma_tf32(acc[mt][1], ah[mt], bl[1]);
      spo_mma_tf32(acc[mt][0], ah[mt], bh[0]);
      spo_mma_tf32(acc[mt][1], ah[mt], bh[1]);
    }
  }
}
