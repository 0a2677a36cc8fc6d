// Read-only vs copy HBM bandwidth: what is the roofline of a pass that only READS?
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o readbw readbw.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
template <int MODE>
__global__ void __launch_bounds__(256) rd(const float4* __restrict__ a, const float4* __restrict__ b, float4* __restrict__ c, size_t n, float* out) {
  float acc = 0.f;
  for (size_t i = (size_t)blockIdx.x * 512 + threadIdx.x; i < n; i += (size_t)gridDim.x * 512) {
    float4 x = __ldcs(a + i), y = __ldcs(b + i);
    float4 x2 = (i + 256 < n) ? __ldcs(a + i + 256) : x, y2 = (i + 256 < n) ? __ldcs(b + i + 256) : y;
    if (MODE == 0) { acc += x.x + y.y + x2.z + y2.w; }
    else { float4 z = make_float4(x.x + y.x, x.y + y.y, x.z + y.z, x.w + y.w); __stcs(c + i, z);
           if (i + 256 < n) { float4 z2 = make_float4(x2.x + y2.x, x2.y + y2.y, x2.z + y2.z, x2.w + y2.w); __stcs(c + i + 256, z2); } }
  }
  if (MODE == 0 && acc == 123.456f) *out = acc;
}
int main(int argc, char** argv) {
  // default: 64 Mi float4 = 1 GiB per array; pass a float4 count to mimic a short pass
  // (BERT-Small pass 1 reads 2 x 115 MB: ./readbw 7191168)
  const size_t n = argc > 1 ? (size_t)atoll(argv[1]) : (size_t)64 << 20;
  float4 *a, *b, *c; float* out;
  cudaMalloc(&a, n * 16); cudaMalloc(&b, n * 16); cudaMalloc(&c, n * 16 > ((size_t)512 << 20) ? n * 16 : ((size_t)512 << 20)); cudaMalloc(&out, 4);
  cudaMemset(a, 0, n * 16); cudaMemset(b, 0, n * 16);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  int num_sms = 0; cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, 0);
  for (int mode = 0; mode < 2; ++mode)
    for (int per_sm : {3, 8}) {
      int grid = num_sms * per_sm;
      float best = 1e9;
      for (int it = 0; it < 6; ++it) {
        if (n < ((size_t)16 << 20)) cudaMemsetAsync(c, 0, 512u << 20);   // evict a and b from L2 (c is >= 512 MB only when n is large: guard below)
        cudaEventRecord(e0);
        if (mode == 0) rd<0><<<grid, 256>>>(a, b, c, n, out); else rd<1><<<grid, 256>>>(a, b, c, n, out);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1); if (it && ms < best) best = ms;
      }
      double bytes = (mode == 0 ? 2.0 : 3.0) * n * 16;
      printf("%s  %d CTAs/SM x256thr (4 LDG.128 in flight/thread): %.1f us  %.0f GB/s\n", mode == 0 ? "read-only 2 streams " : "read 2 + write 1     ", per_sm, best * 1e3, bytes / best / 1e6);
    }
  return 0;
}
