// Phase timings (SM clocks) of the Cholesky's diagonal-block kernel, one launch on a 64×64 SPD block.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o /tmp/potf2_probe tests/studies/potf2_probe.cu && /tmp/potf2_probe
#include <cstdio>
#include <cmath>
#include <vector>
#include <cuda_runtime.h>
#define KBO_NB 64
#define KBO_POTF2_PROBE
#include "../../kubeflow_b200/csrc/potf2.cuh"

int main() {
  const int n = 64, lda = 64;
  std::vector<double> A(n * n);
  for (int i = 0; i < n; i++)
    for (int j = 0; j < n; j++) A[i * n + j] = std::exp(-0.05 * (i - j) * (i - j)) + (i == j ? 1e-3 : 0.0);
  double *dA, *dL;
  int* info;
  long long* probe;
  cudaMalloc(&dA, sizeof(double) * n * n);
  cudaMalloc(&dL, sizeof(double) * n * n);
  cudaMalloc(&info, sizeof(int));
  cudaMalloc(&probe, sizeof(long long) * 16);
  const int smem = 2 * KBO_NB * (KBO_NB + 1) * (int)sizeof(double);
  cudaFuncSetAttribute(potf2_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  float best = 1e9f;
  long long hp[16];
  for (int it = 0; it < 20; it++) {
    cudaMemcpy(dA, A.data(), sizeof(double) * n * n, cudaMemcpyHostToDevice);
    cudaMemset(info, 0, sizeof(int));
    cudaEventRecord(e0);
    potf2_inv_kernel<<<1, POTF2_THREADS, smem>>>(dA, lda, n, 0, dL, info, nullptr, 0, probe);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
  }
  cudaMemcpy(hp, probe, sizeof(hp), cudaMemcpyDeviceToHost);
  int hinfo;
  cudaMemcpy(&hinfo, info, sizeof(int), cudaMemcpyDeviceToHost);
  std::vector<double> L(n * n), Li(n * n);
  cudaMemcpy(L.data(), dA, sizeof(double) * n * n, cudaMemcpyDeviceToHost);
  cudaMemcpy(Li.data(), dL, sizeof(double) * n * n, cudaMemcpyDeviceToHost);
  double err = 0.0, erri = 0.0;   // ‖L·Lᵀ − A‖∞ and ‖Linv·L − I‖∞ over the lower triangle
  for (int i = 0; i < n; i++)
    for (int j = 0; j <= i; j++) {
      double s = 0.0, u = 0.0;
      for (int k = 0; k <= j; k++) s += L[i * n + k] * L[j * n + k];
      for (int k = j; k <= i; k++) u += Li[i * n + k] * L[k * n + j];
      err = fmax(err, fabs(s - A[i * n + j]));
      erri = fmax(erri, fabs(u - (i == j ? 1.0 : 0.0)));
    }
  printf("info %d  event time %.1f us  |LLt-A| %.2e  |Linv L - I| %.2e\n", hinfo, best * 1e3, err, erri);
  const char* names[] = {"load", "factor16 (kb=0)", "inverse16 (kb=0)", "trsm (kb=0)", "update (kb=0)", "all four 16-blocks", "doubling b=16", "doubling b=32"};
  for (int i = 1; i < 8; i++) printf("  %-22s %8lld clk (since mark %d)\n", names[i], hp[i] - hp[i == 5 ? 0 : i - 1], i == 5 ? 0 : i - 1);
  return 0;
}
