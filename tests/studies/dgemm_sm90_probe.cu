// Throughput of the fit's FP64 GEMM (csrc/dgemm_sm90.cuh: m16n8k8, cp.async ring) beside csrc/dgemm.cuh (m8n8k4) on the shapes the
// Cholesky uses, in one binary.  Answers: DESIGN.md §3 "The fit".
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o /tmp/dgemm_sm90_probe tests/studies/dgemm_sm90_probe.cu && /tmp/dgemm_sm90_probe
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#include "../../kubeflow_b200/csrc/dgemm.cuh"
#include "../../kubeflow_b200/csrc/dgemm_sm90.cuh"

int main() {
  const int N = 8192;
  double *A, *C;
  cudaMalloc(&A, sizeof(double) * (size_t)N * N);
  cudaMalloc(&C, sizeof(double) * (size_t)N * N);
  cudaMemset(A, 0, sizeof(double) * (size_t)N * N);
  cudaMemset(C, 0, sizeof(double) * (size_t)N * N);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  struct Case { const char* name; int M, Nn, K, lower; };
  const Case cases[] = {{"syrk update 7936 x 7936 x 256 (lower)", 7936, 7936, 256, 1}, {"syrk update 4096 x 4096 x 256 (lower)", 4096, 4096, 256, 1},
                        {"syrk update 7680 x 7680 x 512 (lower)", 7680, 7680, 512, 1}, {"column block 7936 x 256 x 256", 7936, 256, 256, 0},
                        {"square 4096 x 4096 x 4096", 4096, 4096, 4096, 0}, {"next diagonal block 256 x 256 x 256 (lower)", 256, 256, 256, 1},
                        {"in-panel update 192 x 192 x 64 (lower)", 192, 192, 64, 1}};
  for (int sm90 = 0; sm90 < 2; sm90++)
    for (const Case& c : cases) {
      float best = 1e9f;
      for (int rep = 0; rep < 4; rep++) {
        cudaEventRecord(e0);
        if (sm90)
          dgemm_sm90_launch<true>(0, c.M, c.Nn, c.K, A, N, A + 300, N, C, N, -1.0, 1.0, KM_FULL, 0, c.lower ? TS_LOWER : TS_NONE);
        else
          dgemm64_launch<true, EPI_STORE>(0, c.M, c.Nn, c.K, A, N, A + 300, N, C, N, -1.0, 1.0, KM_FULL, 0, c.lower ? TS_LOWER : TS_NONE);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) best = ms;
      }
      const double flops = 2.0 * c.M * c.Nn * c.K * (c.lower ? 0.5 : 1.0);
      printf("%-9s %-44s %8.3f ms  %6.2f TFLOP/s  (%s)\n", sm90 ? "m16n8k8" : "m8n8k4", c.name, best, flops / best * 1e-9, cudaGetErrorString(cudaGetLastError()));
    }
  return 0;
}
