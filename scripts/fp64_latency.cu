// Micro-benchmark: DEPENDENT-chain latencies that bound the tail kernel's diagonal blocks (one warp, clock64()):
// DFMA -> DFMA, the 1/sqrt sequence of tail_diag.cuh (MUFU.RSQ64H + two Newton steps), shared-memory load -> use, CTA barrier.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/fp64_latency.bin scripts/fp64_latency.cu
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ double rsq(double p) {
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(p));
  const double hp = 0.5 * p;
  y = y * (1.5 - hp * y * y);
  y = y * (1.5 - hp * y * y);
  return y;
}

__global__ void k_lat(double* out, long long* cyc, int iters) {
  __shared__ int chase[256];
  __shared__ double sd[256];
  const int tid = threadIdx.x;
  chase[tid] = (tid * 37 + 11) & 255;
  sd[tid] = 1.0 + 1e-9 * tid;
  __syncthreads();
  double a = 1.0 + 1e-6 * tid;
  const double b = 1.0000001, c = 1e-7;
  long long t0, t1;
  // 1. dependent DFMA
  t0 = clock64();
  for (int i = 0; i < iters; ++i) a = a * b + c;
  t1 = clock64();
  if (tid == 0) cyc[0] = t1 - t0;
  // 2. dependent rsqrt sequence (p_{k+1} = rsq(p_k) + 1)
  double p = 2.0 + a * 1e-9;
  t0 = clock64();
  for (int i = 0; i < iters; ++i) p = rsq(p) + 1.0;
  t1 = clock64();
  if (tid == 0) cyc[1] = t1 - t0;
  // 3. shared-memory pointer chase
  int q = tid;
  t0 = clock64();
  for (int i = 0; i < iters; ++i) q = chase[q];
  t1 = clock64();
  if (tid == 0) cyc[2] = t1 - t0;
  // 4. shared double load -> DFMA -> store -> load (read-modify-write chain on one address per thread)
  t0 = clock64();
  for (int i = 0; i < iters; ++i) { sd[tid] = sd[tid] * b + c; }
  t1 = clock64();
  if (tid == 0) cyc[3] = t1 - t0;
  // 5. CTA barrier
  t0 = clock64();
  for (int i = 0; i < iters; ++i) __syncthreads();
  t1 = clock64();
  if (tid == 0) cyc[4] = t1 - t0;
  // 6. a pivot step of the 4x4 micro-block: rsq -> mul -> fma (next pivot)
  double d = 2.0 + 1e-9 * q, l = 0.5;
  t0 = clock64();
  for (int i = 0; i < iters; ++i) { const double iv = rsq(d); const double m = l * iv; d = 3.0 - m * m; }
  t1 = clock64();
  if (tid == 0) cyc[5] = t1 - t0;
  out[tid] = a + p + q + sd[tid] + d;
}

int main() {
  cudaDeviceProp pr; cudaGetDeviceProperties(&pr, 0);
  printf("%s, clock %d kHz\n", pr.name, pr.clockRate);
  double* out; long long* cyc;
  cudaMalloc(&out, 8 * 256); cudaMalloc(&cyc, 8 * 8);
  const int iters = 4000;
  const char* names[6] = {"dependent DFMA", "1/sqrt sequence (MUFU.RSQ64H + 2 Newton) + DADD", "shared-memory pointer chase (LDS -> LDS)",
                          "shared RMW (LDS.64 -> DFMA -> STS.64 -> LDS.64)", "__syncthreads()", "pivot step (rsq -> DMUL -> DFMA)"};
  for (int threads : {32, 256}) {
    k_lat<<<1, threads>>>(out, cyc, iters);
    k_lat<<<1, threads>>>(out, cyc, iters);
    cudaDeviceSynchronize();
    long long h[8]; cudaMemcpy(h, cyc, 8 * 8, cudaMemcpyDeviceToHost);
    for (int i = 0; i < 6; ++i) printf("threads=%3d  %-60s %.1f cycles\n", threads, names[i], (double)h[i] / iters);
  }
  return 0;
}
