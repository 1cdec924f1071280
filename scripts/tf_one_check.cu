// Stand-alone check of tf_factor_one (tail_diag.cuh) as the engine runs it: a cluster of two CTAs factorises a 32 x 32
// pair (CTA 0: A following CTA 1's flags for G, G rank-deficient), compared with a host reference.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I msckf_mono_b200/csrc -o scripts/tf_one_check.bin scripts/tf_one_check.cu
#include <cooperative_groups.h>
#include <cmath>
#include <cstdio>
#include <vector>
#include "tail_diag.cuh"
namespace cg = cooperative_groups;
using namespace mb;

__global__ void __cluster_dims__(2, 1, 1) k_check(const double* Ain, const double* Gin, double* LIout, int* rk_out, int nb, int reps, double* pivr) {
  __shared__ __align__(16) double D[kFB * kFLD], LI[kFB * kFLD];
  __shared__ double idv[kFB], d0[kFB + 2];
  __shared__ unsigned s_words[kFB / 4];
  __shared__ int s_timeout;
  cg::cluster_group cluster = cg::this_cluster();
  const int crank = cluster.block_rank(), tid = threadIdx.x;
  if (tid < kFB / 4) s_words[tid] = 0u;
  cluster.sync();
  TfLink lk;
  lk.words = s_words;
  lk.timed_out = &s_timeout;
  if (crank == 1) lk.words = cluster.map_shared_rank(s_words, 0);
  int rk = 0;
  for (int rep = 0; rep < reps; ++rep) {
    const double* M = crank ? Gin : Ain;
    for (int e = tid; e < kFB * kFLD; e += 256) { const int i = e / kFLD, j = e % kFLD; D[e] = (i < nb && j <= i) ? M[i * 32 + j] : 0.0; }
    for (int k = tid; k < kFB; k += 256) d0[k] = Gin[k * 32 + k];
    __syncthreads();
    rk = tf_factor_one(D, LI, idv, d0, 0, nb, 1e-11, 32, crank ? 1 : 0, 0, tid, 256, (unsigned)rep + 1u, lk, pivr + crank * 32);
    cluster.sync();
  }
  for (int e = tid; e < kFB * kFLD; e += 256) LIout[crank * kFB * kFLD + e] = LI[e];
  if (tid == 0) rk_out[crank] = rk;
}

int main() {
  const int n = 32;
  std::vector<double> A(n * n), G(n * n), B(n * n), C(n * n);
  unsigned s = 12345;
  auto rnd = [&]() { s = s * 1664525u + 1013904223u; return (double)(s >> 8) / (1 << 24) - 0.5; };
  for (auto& v : B) v = rnd();
  for (auto& v : C) v = rnd();
  for (int i : {5, 13, 14, 30}) for (int k = 0; k < n; ++k) C[i * n + k] = 0.3 * C[(i - 1) * n + k] - 0.7 * C[(i - 3) * n + k];  // dependent rows -> rank-deficient G
  for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) {
    double a = 0, g = 0;
    for (int k = 0; k < n; ++k) { a += B[i * n + k] * B[j * n + k]; g += C[i * n + k] * C[j * n + k]; }
    A[i * n + j] = a + (i == j ? 1.0 : 0.0); G[i * n + j] = g;
  }
  // host reference: G decides (pivot > 1e-11 * original diagonal), A follows; inverse of the factor restricted to kept indices
  std::vector<double> LG = G, LA = A; std::vector<int> keep(n, 0);
  for (int j = 0; j < n; ++j) {
    const bool k = LG[j * n + j] > 1e-11 * G[j * n + j];
    keep[j] = k;
    for (int M = 0; M < 2; ++M) {
      auto& L = M ? LG : LA;
      const double iv = k ? 1.0 / std::sqrt(L[j * n + j]) : 0.0;
      for (int i = j; i < n; ++i) L[i * n + j] *= iv;
      for (int b = j + 1; b < n; ++b) for (int i = b; i < n; ++i) L[i * n + b] -= L[i * n + j] * L[b * n + j];
    }
  }
  auto inv = [&](const std::vector<double>& L) {  // Linv of the kept part (rows / cols of dropped pivots zero)
    std::vector<double> X(n * n, 0.0);
    for (int c = 0; c < n; ++c) if (keep[c]) {
      for (int i = c; i < n; ++i) if (keep[i]) {
        double v = (i == c) ? 1.0 : 0.0;
        for (int k = c; k < i; ++k) v -= L[i * n + k] * X[k * n + c];
        X[i * n + c] = v / L[i * n + i];
      }
    }
    return X;
  };
  const auto XA = inv(LA), XG = inv(LG);
  double *dA, *dG, *dL; int* dr;
  cudaMalloc(&dA, 8 * n * n); cudaMalloc(&dG, 8 * n * n); cudaMalloc(&dL, 8 * 2 * kFB * kFLD); cudaMalloc(&dr, 8); double* dP; cudaMalloc(&dP, 8 * 64);
  cudaMemcpy(dA, A.data(), 8 * n * n, cudaMemcpyHostToDevice); cudaMemcpy(dG, G.data(), 8 * n * n, cudaMemcpyHostToDevice);
  for (int reps : {1, 50}) {
    k_check<<<2, 256>>>(dA, dG, dL, dr, n, reps, dP);
    cudaError_t e = cudaDeviceSynchronize();
    std::vector<double> L(2 * kFB * kFLD); int rk[2];
    cudaMemcpy(L.data(), dL, 8 * L.size(), cudaMemcpyDeviceToHost); cudaMemcpy(rk, dr, 8, cudaMemcpyDeviceToHost);
    double ea = 0, eg = 0, na = 0, ng = 0;
    for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) {  // (extra row c of the identity ends as column c of L^-T: LI[i][j] = Linv[i][j])
      const double da = L[i * kFLD + j] - XA[i * n + j], dg = L[kFB * kFLD + i * kFLD + j] - XG[i * n + j];
      ea = fmax(ea, fabs(da)); eg = fmax(eg, fabs(dg)); na = fmax(na, fabs(XA[i * n + j])); ng = fmax(ng, fabs(XG[i * n + j]));
    }
    int nk = 0; for (int k : keep) nk += k;
    printf("reps=%d: %s  rank A %d G %d (host %d)  max |Linv - ref| A %.3e (of %.2e)  G %.3e (of %.2e)\n", reps, cudaGetErrorString(e), rk[0], rk[1], nk, ea, na, eg, ng);
  }
  return 0;
}
