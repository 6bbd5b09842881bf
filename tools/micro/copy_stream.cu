// copy_stream — the HBM copy ceiling with the access types of the streaming stencils: every thread moves
// 16-byte vectors with ld.global.cs / st.global.cs (evict-first), U = 4 loads in flight before the stores.
// tools/kernel_bench.py builds it into a temporary directory and times it beside torch's copy_:
//   nvcc -O3 -shared -Xcompiler -fPIC -gencode arch=compute_90a,code=sm_90a -o copy_stream.so copy_stream.cu
#include <cuda_runtime.h>
#include <stdint.h>

namespace {
constexpr int kThreads = 256, kU = 4;

__global__ void __launch_bounds__(kThreads) k_copy_stream(const float4* __restrict__ in, float4* __restrict__ out,
                                                          int64_t nvec) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  for (; i + (kU - 1) * stride < nvec; i += kU * stride) {
    float4 v[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) v[u] = __ldcs(in + i + u * stride);
#pragma unroll
    for (int u = 0; u < kU; ++u) __stcs(out + i + u * stride, v[u]);
  }
  for (; i < nvec; i += stride) __stcs(out + i, __ldcs(in + i));
}
}  // namespace

// n_bytes must be a multiple of 16 and both pointers 16-byte aligned; blocks_per_sm x SMs blocks, grid-stride.
extern "C" int copy_stream(const void* in, void* out, int64_t n_bytes, int blocks_per_sm, void* stream) {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  k_copy_stream<<<sms * blocks_per_sm, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const float4*>(in), static_cast<float4*>(out), n_bytes / 16);
  return (int)cudaGetLastError();
}
