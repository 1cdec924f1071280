// Micro-benchmark: issue rate of FP64 FMA (and FP32 FMA for comparison) per SM sub-partition on the GPU at hand.
// One CTA, W warps, each lane runs 8 independent FMA chains; cycles from clock64() on warp 0.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/fp64_rate.bin scripts/fp64_rate.cu
#include <cstdio>
#include <cuda_runtime.h>

template <class T>
__global__ void k_rate(T* out, long long* cyc, int iters, int active_lanes) {
  T a[8];
  for (int i = 0; i < 8; ++i) a[i] = (T)(threadIdx.x + i) * (T)1e-3;
  const T b = (T)1.0000001, c = (T)1e-7;
  __syncthreads();
  const long long t0 = clock64();
  if ((threadIdx.x & 31) < active_lanes) {
    for (int it = 0; it < iters; ++it) {
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = a[i] * b + c;
    }
  }
  __syncthreads();
  const long long t1 = clock64();
  T s = 0;
  for (int i = 0; i < 8; ++i) s += a[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <class T>
void run(const char* name, int warps, int lanes, int blocks) {
  T* out; long long* cyc;
  cudaMalloc(&out, sizeof(T) * 1024 * blocks); cudaMalloc(&cyc, sizeof(long long) * blocks);
  const int iters = 2000;
  k_rate<T><<<blocks, 32 * warps>>>(out, cyc, iters, lanes);
  k_rate<T><<<blocks, 32 * warps>>>(out, cyc, iters, lanes);
  cudaDeviceSynchronize();
  long long h[1024]; cudaMemcpy(h, cyc, sizeof(long long) * blocks, cudaMemcpyDeviceToHost);
  long long mx = 0; for (int i = 0; i < blocks; ++i) mx = h[i] > mx ? h[i] : mx;
  const double fma_warp = (double)iters * 8;                 // warp-level FMA instructions per warp
  const double per_smsp = fma_warp * ((warps + 3) / 4);      // warps sharing one sub-partition
  printf("%s warps/CTA=%d active_lanes=%d CTAs=%d: %lld cycles; %.2f cycles per warp-FMA per sub-partition; %.1f lane-FMA/clk/SM\n",
         name, warps, lanes, blocks, mx, mx / per_smsp, fma_warp * warps * lanes / (double)mx);
  cudaFree(out); cudaFree(cyc);
}

int main() {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  printf("%s, %d SMs, clock %d kHz\n", p.name, p.multiProcessorCount, p.clockRate);
  for (int w : {1, 2, 4, 8, 16}) run<double>("fp64", w, 32, 1);
  for (int l : {1, 4, 8, 16}) run<double>("fp64", 4, l, 1);
  run<double>("fp64", 8, 32, p.multiProcessorCount);
  run<double>("fp64", 8, 32, 2 * p.multiProcessorCount);
  for (int w : {1, 4, 8, 16}) run<float>("fp32", w, 32, 1);
  return 0;
}
