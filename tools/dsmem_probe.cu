// What does a cluster-wide "everyone's shared-memory data is in place, now read a peer" cost, and which part of
// it is the barrier, the L1 invalidate that barrier.cluster.wait.acquire drags in (CCTL.IVALL in SASS), or the
// ld.shared::cluster round trip itself?  12-CTA cluster, 256 threads, thread-0 clock64 deltas averaged over ITERS rounds.
//   raw    : dependent chain of remote float4 loads, no synchronisation at all           -> DSMEM latency
//   raw3   : 3 independent remote float4 loads per thread, all threads                    -> DSMEM throughput
//   S1     : __syncthreads + barrier.cluster (relaxed arrive, acquire wait) + 1 remote float4 load per thread
//   S1L    : same, but the load after the barrier is LOCAL shared memory                  -> cost the barrier leaves behind
//   S2     : __syncthreads + one remote mbarrier.arrive per peer (release.cluster) + try_wait (acquire.cta) + remote load
//   S2r    : same with relaxed arrives / relaxed wait
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/dsmem_probe tools/dsmem_probe.cu
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
namespace cg = cooperative_groups;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ uint32_t mapa(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ float4 ld_dsmem_f4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
template <bool RELAXED>
__device__ __forceinline__ void mbar_remote_arrive(uint32_t remote_bar) {
  if (RELAXED) asm volatile("mbarrier.arrive.relaxed.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote_bar) : "memory");
  else asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote_bar) : "memory");
}
template <bool RELAXED>
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t a = smem_u32(bar);
  uint32_t ok = 0;
  while (!ok) {
    if (RELAXED)
      asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.relaxed.cta.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(a), "r"(parity) : "memory");
    else
      asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(a), "r"(parity) : "memory");
  }
}

constexpr int NT = 256, NC = 12, LD = 72;

__global__ void __launch_bounds__(NT, 1) probe(int iters, double* out) {
  __shared__ __align__(16) float buf[64 * LD];
  __shared__ __align__(8) uint64_t bar;
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank();
  const int tid = threadIdx.x;
  for (int i = tid; i < 64 * LD; i += NT) buf[i] = 0.f;
  if (tid == 0) {
    mbar_init(&bar, NC);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  cluster.sync();
  const unsigned peer = (rank + 1) % NC;
  const int r4 = tid >> 2, k4 = tid & 3;
  const uint32_t my = smem_u32(buf) + (r4 * LD + 4 * k4) * 4;
  const uint32_t rem = mapa(smem_u32(buf), peer) + (r4 * LD + 4 * k4) * 4;
  float keep = 0.f;
  long long t[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  // raw: dependent chain (the loaded value, always 0, feeds the next address)
  {
    long long c0 = clock64();
    uint32_t a = rem;
    for (int it = 0; it < iters; ++it) {
      float4 v = ld_dsmem_f4(a);
      a = rem + static_cast<uint32_t>(v.x);
      keep += v.y;
    }
    t[0] = clock64() - c0;
  }
  cluster.sync();
  // raw3: three independent loads from three peers per thread
  {
    const uint32_t r1 = mapa(smem_u32(buf), (rank + 1) % NC) + (r4 * LD + 16 + 4 * k4) * 4;
    const uint32_t r2 = mapa(smem_u32(buf), (rank + 2) % NC) + (r4 * LD + 32 + 4 * k4) * 4;
    const uint32_t r3 = mapa(smem_u32(buf), (rank + 3) % NC) + (r4 * LD + 48 + 4 * k4) * 4;
    long long c0 = clock64();
    for (int it = 0; it < iters; ++it) {
      float4 a = ld_dsmem_f4(r1), b = ld_dsmem_f4(r2), c = ld_dsmem_f4(r3);
      keep += a.x + b.x + c.x;
      __syncthreads();
    }
    t[1] = clock64() - c0;
  }
  cluster.sync();
  // S1 / S1L
  for (int variant = 0; variant < 2; ++variant) {
    long long c0 = clock64();
    for (int it = 0; it < iters; ++it) {
      __syncthreads();
      asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
      asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
      if (variant == 0) { float4 v = ld_dsmem_f4(rem); keep += v.x; }
      else { float4 v; asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(my) : "memory"); keep += v.x; }
      if (keep == 1234.5f) buf[tid] = keep;   // force the load to complete inside the round
    }
    t[2 + variant] = clock64() - c0;
    cluster.sync();
  }
  // S2 / S2r: mbarrier all-to-all (12 arrivals per phase)
  uint32_t parity = 0;
  for (int variant = 0; variant < 2; ++variant) {
    long long c0 = clock64();
    for (int it = 0; it < iters; ++it) {
      __syncthreads();
      if (tid < NC) {
        const uint32_t rb = mapa(smem_u32(&bar), tid);
        if (variant == 0) mbar_remote_arrive<false>(rb); else mbar_remote_arrive<true>(rb);
      }
      if (variant == 0) mbar_wait<false>(&bar, parity); else mbar_wait<true>(&bar, parity);
      parity ^= 1u;
      float4 v = ld_dsmem_f4(rem);
      keep += v.x;
      if (keep == 1234.5f) buf[tid] = keep;
    }
    t[4 + variant] = clock64() - c0;
    cluster.sync();
  }
  // S3: barrier.cluster with the default release arrive (what cluster.sync() does) + remote load
  {
    long long c0 = clock64();
    for (int it = 0; it < iters; ++it) {
      asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
      asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
      float4 v = ld_dsmem_f4(rem);
      keep += v.x;
      if (keep == 1234.5f) buf[tid] = keep;
    }
    t[6] = clock64() - c0;
  }
  cluster.sync();
  // BULK: all-gather inside groups of 4 with the bulk-copy engine: every CTA owns a contiguous 4 KB slice and sends it to
  // its three group peers with cp.async.bulk.shared::cluster (complete_tx on the receiver's mbarrier); receivers wait for
  // 3 x 4 KB.  Time = issue -> all three slices landed (thread 0).
  {
    __shared__ __align__(128) float slices[4][1024];
    __shared__ __align__(8) uint64_t bar2;
    if (tid == 0) {
      mbar_init(&bar2, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    cluster.sync();
    const unsigned g0 = rank & ~3u, qq = rank & 3u;
    uint32_t par2 = 0;
    long long acc_t = 0;
    for (int it = 0; it < iters; ++it) {
      for (int i = tid; i < 1024; i += NT) slices[qq][i] = static_cast<float>(it + i);
      if (tid == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar2)), "r"(3 * 4096) : "memory");
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncthreads();
      asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");   // receivers armed, sources written
      asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
      long long c0 = clock64();
      if (tid < 4 && tid != qq) {
        const uint32_t dst = mapa(smem_u32(&slices[qq][0]), g0 + tid), rb = mapa(smem_u32(&bar2), g0 + tid);
        asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(dst), "r"(smem_u32(&slices[qq][0])), "r"(4096), "r"(rb) : "memory");
      }
      mbar_wait<false>(&bar2, par2);
      par2 ^= 1u;
      acc_t += clock64() - c0;
      float chk = slices[(qq + 1) & 3][tid];
      if (chk != static_cast<float>(it + tid)) keep += 1e9f;
      __syncthreads();
    }
    t[7] = acc_t;
  }
  cluster.sync();
  if (tid == 0 && rank == 0)
    for (int i = 0; i < 8; ++i) out[i] = double(t[i]) / iters;
  if (tid == 0 && rank == 0) out[8] = keep;
}

int main() {
  double* out;
  cudaMalloc(&out, 16 * sizeof(double));
  cudaMemset(out, 0, 16 * sizeof(double));
  cudaFuncSetAttribute(probe, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(NC);
  cfg.blockDim = dim3(NT);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = NC;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, probe, 1000, out);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("FAILED: %s\n", cudaGetErrorString(e)); return 1; }
  double h[16];
  cudaMemcpy(h, out, sizeof(h), cudaMemcpyDeviceToHost);
  printf("cycles per round, cluster of %d CTAs x %d threads (thread 0 of CTA 0):\n", NC, NT);
  printf("  raw  dependent remote float4 load (DSMEM latency)                      %.0f\n", h[0]);
  printf("  raw3 three independent remote float4 loads per thread + __syncthreads  %.0f\n", h[1]);
  printf("  S1   __syncthreads + barrier.cluster(relaxed/acquire) + remote load     %.0f\n", h[2]);
  printf("  S1L  __syncthreads + barrier.cluster(relaxed/acquire) + LOCAL load      %.0f\n", h[3]);
  printf("  S2   __syncthreads + 12 remote mbarrier arrives (release) + wait + remote load   %.0f\n", h[4]);
  printf("  S2r  same, relaxed arrives / relaxed wait                              %.0f\n", h[5]);
  printf("  S3   barrier.cluster(release/acquire) + remote load                    %.0f\n", h[6]);
  printf("  BULK 3 x 4 KB cp.async.bulk smem->peer smem + mbarrier wait (12 KB in)   %.0f   (check value %.3g: > 1e8 means wrong data)\n", h[7], h[8]);
  return 0;
}
