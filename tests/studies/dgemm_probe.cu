// Throughput of the FP64 tensor-core GEMM building block (csrc/dgemm.cuh) on the shapes the Cholesky uses.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o /tmp/dgemm_probe tests/studies/dgemm_probe.cu && /tmp/dgemm_probe
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#include "../../kubeflow_b200/csrc/dgemm.cuh"
#ifdef DGEMM_V2
#include "../../kubeflow_b200/csrc/dgemm2.cuh"
#endif

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
                        {"square 4096 x 4096 x 4096", 4096, 4096, 4096, 0}};
  for (const Case& c : cases) {
    float best = 1e9f;
    for (int rep = 0; rep < 4; rep++) {
      cudaEventRecord(e0);
#ifdef DGEMM_V2
      dgemm2_launch_nt(0, c.M, c.Nn, c.K, A, N, A + 300, N, C, N, -1.0, 1.0, c.lower ? TS_LOWER : TS_NONE);
#else
      dgemm64_launch<true, EPI_STORE>(0, c.M, c.Nn, c.K, A, N, A + 300, N, C, N, -1.0, 1.0, KM_FULL, 0, c.lower ? TS_LOWER : TS_NONE);
#endif
      cudaEventRecord(e1);
      cudaEventSynchronize(e1);
      float ms;
      cudaEventElapsedTime(&ms, e0, e1);
      if (ms < best) best = ms;
    }
    const double flops = 2.0 * c.M * c.Nn * c.K * (c.lower ? 0.5 : 1.0);
    printf("%-44s %8.3f ms  %6.2f TFLOP/s  (%s)\n", c.name, best, flops / best * 1e-9, cudaGetErrorString(cudaGetLastError()));
  }
  return 0;
}
