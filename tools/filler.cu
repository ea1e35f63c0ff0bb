// Experiment: does a 12-CTA kernel with a > 32 KB loop body run faster when the other SMs of the GPU are busy?
// A filler kernel occupies `ctas` SMs until a flag is set or a cycle limit is hit.  mode 0: nanosleep loop; 1: FFMA spin; 2: idle wait on clock only.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -shared -Xcompiler -fPIC tools/filler.cu -o tools/libfiller.so
#include <cuda_runtime.h>

__global__ void filler_kernel(volatile int* stop, long long max_cycles, int mode, float* sink) {
  const long long t0 = clock64();
  float x = threadIdx.x * 1e-3f, y = 1.0001f;
  while (!*stop && clock64() - t0 < max_cycles) {
    if (mode == 0) {
      __nanosleep(500);
    } else if (mode == 1) {
#pragma unroll 64
      for (int i = 0; i < 256; ++i) x = fmaf(x, y, 1e-7f);
    }
  }
  if (x == 123.456f) *sink = x;
}

extern "C" int filler_launch(int ctas, int threads, int mode, int* stop, long long max_cycles, float* sink, void* stream) {
  filler_kernel<<<ctas, threads, 200 * 1024, static_cast<cudaStream_t>(stream)>>>(stop, max_cycles, mode, sink);
  return static_cast<int>(cudaGetLastError());
}
extern "C" int filler_prepare() {
  return static_cast<int>(cudaFuncSetAttribute(filler_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
}
