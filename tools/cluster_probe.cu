// Bring-up probe for the round-2 update kernel (csrc/spo_update.cu): can a cluster of 12 / 16 CTAs be launched,
// and what does one exchange cost when it is built from st.async (remote shared-memory stores that complete_tx on the
// receiver's mbarrier) instead of barrier.cluster?
//   (a) all-gather inside groups of 4 CTAs: every CTA writes a 64x16 fp32 slice into all 4 members (16 KB landed per CTA)
//   (b) all-to-all of one float2 between all active CTAs (the joint-gradient-norm exchange)
//   (c) barrier.cluster.arrive + wait, for reference
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/cluster_probe tools/cluster_probe.cu
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
namespace cg = cooperative_groups;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ uint32_t mapa(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
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
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"(a), "r"(parity) : "memory");
  }
}
__device__ __forceinline__ void st_async_f2(uint32_t remote_addr, float x, float y, uint32_t remote_bar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.f32 [%0], {%1, %2}, [%3];"
               ::"r"(remote_addr), "f"(x), "f"(y), "r"(remote_bar) : "memory");
}

constexpr int NT = 256, GRP = 4, SL = 16, LDS = 72;

__global__ void __launch_bounds__(NT, 1) probe(int active, int iters, unsigned long long* cyc, int* errors) {
  __shared__ __align__(16) float h1[64 * LDS];
  __shared__ __align__(16) float xch[2][16][2];
  __shared__ __align__(8) uint64_t bar_h1, bar_ss;
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank();
  const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const bool act = static_cast<int>(rank) < active;
  const unsigned grp0 = rank & ~3u, q = rank & 3u;
  if (tid == 0) {
    mbar_init(&bar_h1, 1);
    mbar_init(&bar_ss, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    if (act) { mbar_expect_tx(&bar_h1, 64 * 64 * 4); mbar_expect_tx(&bar_ss, active * 8); }
  }
  cluster.sync();
  unsigned long long t_ag = 0, t_ss = 0, t_cb = 0;
  int bad = 0;
  if (act) {
    const int mt = wid & 3, nt = wid >> 2;   // 16 x 8 tile of the 64 x 16 slice
    const uint32_t h1a = smem_u32(h1), bh = smem_u32(&bar_h1), bs = smem_u32(&bar_ss);
    for (int it = 0; it < iters; ++it) {
      const uint32_t par = it & 1;
      // (a) all-gather of the slice into the 4 members of the group
      long long c0 = clock64();
      const int r0 = mt * 16 + g, c = q * SL + nt * 8 + 2 * t;
      const float v = static_cast<float>(it * 1000 + static_cast<int>(q));
#pragma unroll
      for (unsigned d = 0; d < GRP; ++d) {
        const uint32_t base = mapa(h1a, grp0 + d), rb = mapa(bh, grp0 + d);
        st_async_f2(base + (r0 * LDS + c) * 4, v, v + 0.5f, rb);
        st_async_f2(base + ((r0 + 8) * LDS + c) * 4, v, v + 0.5f, rb);
      }
      mbar_wait(&bar_h1, par);
      if (tid == 0) mbar_expect_tx(&bar_h1, 64 * 64 * 4);
      long long c1 = clock64();
      // check: column block s of every row carries it*1000 + s
      for (int i = tid; i < 64 * 64; i += NT) {
        const int r = i >> 6, cc = i & 63;
        const float want = static_cast<float>(it * 1000 + (cc >> 4)) + ((cc & 1) ? 0.5f : 0.f);
        if (h1[r * LDS + cc] != want) ++bad;
      }
      __syncthreads();
      // (b) all-to-all of one float2
      long long c2 = clock64();
      if (tid < active) {
        const uint32_t dst = mapa(smem_u32(&xch[par][rank][0]), tid);
        st_async_f2(dst, static_cast<float>(rank + it), 1.f, mapa(bs, tid));
      }
      mbar_wait(&bar_ss, par);
      if (tid == 0) mbar_expect_tx(&bar_ss, active * 8);
      float tot = 0.f;
      for (int s = 0; s < active; ++s) tot += xch[par][s][0];
      long long c3 = clock64();
      const float want_tot = static_cast<float>(active * (active - 1) / 2 + active * it);
      if (tot != want_tot) ++bad;
      t_ag += c1 - c0;
      t_ss += c3 - c2;
      __syncthreads();
    }
  }
  cluster.sync();
  for (int it = 0; it < iters; ++it) {
    long long c0 = clock64();
    asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
    t_cb += clock64() - c0;
  }
  // (c2) __syncthreads + fence by one thread + relaxed arrive + wait   (c3) cluster.sync()   (d) barrier + pull of 3 float4 per thread
  unsigned long long t_c2 = 0, t_c3 = 0, t_pull = 0, t_pull_only = 0;
  for (int it = 0; it < iters; ++it) {
    long long c0 = clock64();
    __syncthreads();
    if (tid == 0) asm volatile("fence.acq_rel.cluster;" ::: "memory");
    asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
    t_c2 += clock64() - c0;
  }
  for (int it = 0; it < iters; ++it) {
    long long c0 = clock64();
    cluster.sync();
    t_c3 += clock64() - c0;
  }
  {
    const int r4 = tid >> 2, k4 = tid & 3;
    float keep = 0.f;
    for (int it = 0; it < iters; ++it) {
      h1[r4 * LDS + 16 * (rank & 3) + 4 * k4] = static_cast<float>(it);
      __syncthreads();
      asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
      asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
      long long c0 = clock64();
      float4 v[4];
#pragma unroll
      for (unsigned d = 0; d < 4; ++d) {
        if (d == (rank & 3)) continue;
        const uint32_t a = mapa(smem_u32(h1), (rank & ~3u) + d) + (r4 * LDS + 16 * d + 4 * k4) * 4;
        asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v[d].x), "=f"(v[d].y), "=f"(v[d].z), "=f"(v[d].w) : "r"(a) : "memory");
      }
      float sacc = 0.f;
#pragma unroll
      for (unsigned d = 0; d < 4; ++d) if (d != (rank & 3)) sacc += v[d].x;
      keep += sacc;
      long long c1 = clock64();
#pragma unroll
      for (unsigned d = 0; d < 4; ++d) if (d != (rank & 3)) *reinterpret_cast<float4*>(h1 + r4 * LDS + 16 * d + 4 * k4) = v[d];
      __syncthreads();
      long long c2 = clock64();
      t_pull_only += c1 - c0;
      t_pull += c2 - c0;
      asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
      asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
    }
    if (keep == 12345.f) errors[1] = 1;
  }
  if (tid == 0) {
    cyc[rank * 3 + 0] = t_ag;
    cyc[rank * 3 + 1] = t_ss;
    cyc[rank * 3 + 2] = t_cb;
    if (rank == 0) printf("   [rank 0] sync+fence+barrier %.0f   cluster.sync() %.0f   pull 3xfloat4: loads %.0f, +stores+sync %.0f cycles\n",
                          double(t_c2) / iters, double(t_c3) / iters, double(t_pull_only) / iters, double(t_pull) / iters);
  }
  if (bad) atomicAdd(errors, bad);
}

static int run(int cs, int active, int iters) {
  unsigned long long* cyc;
  int* err;
  cudaMalloc(&cyc, sizeof(unsigned long long) * 3 * 16);
  cudaMalloc(&err, 2 * sizeof(int));
  cudaMemset(cyc, 0, sizeof(unsigned long long) * 3 * 16);
  cudaMemset(err, 0, 2 * sizeof(int));
  cudaError_t e = cudaFuncSetAttribute(probe, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  if (e != cudaSuccess) printf("  set non-portable: %s\n", cudaGetErrorString(e));
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(cs);
  cfg.blockDim = dim3(NT);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int maxc = -1;
  e = cudaOccupancyMaxActiveClusters(&maxc, probe, &cfg);
  printf("cluster=%d active=%d: cudaOccupancyMaxActiveClusters -> %d (%s)\n", cs, active, maxc, cudaGetErrorString(e));
  (void)cudaGetLastError();
  e = cudaLaunchKernelEx(&cfg, probe, active, iters, cyc, err);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    printf("  launch/run FAILED: %s\n", cudaGetErrorString(e));
    (void)cudaGetLastError();
    return 1;
  }
  unsigned long long h[48];
  int herr = 0;
  cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
  cudaMemcpy(&herr, err, sizeof(int), cudaMemcpyDeviceToHost);
  printf("  errors=%d   cycles per round (rank 0 / max over ranks): all-gather 16KB x4: %.0f / ", herr, double(h[0]) / iters);
  unsigned long long m0 = 0, m1 = 0, m2 = 0;
  for (int r = 0; r < cs; ++r) { if (h[r * 3] > m0) m0 = h[r * 3]; if (h[r * 3 + 1] > m1) m1 = h[r * 3 + 1]; if (h[r * 3 + 2] > m2) m2 = h[r * 3 + 2]; }
  printf("%.0f   float2 all-to-all: %.0f / %.0f   barrier.cluster: %.0f / %.0f\n", double(m0) / iters, double(h[1]) / iters, double(m1) / iters,
         double(h[2]) / iters, double(m2) / iters);
  cudaFree(cyc);
  cudaFree(err);
  return 0;
}

int main() {
  cudaDeviceProp p;
  cudaGetDeviceProperties(&p, 0);
  printf("%s, %d SMs\n", p.name, p.multiProcessorCount);
  const int iters = 500;
  run(4, 4, iters);
  run(8, 8, iters);
  run(12, 12, iters);
  run(16, 12, iters);
  run(16, 16, iters);
  return 0;
}
