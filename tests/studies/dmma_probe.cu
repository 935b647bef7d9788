// Peak FP64 tensor-core rate by mma shape (register-resident operands, independent accumulators).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/dmma_probe tests/studies/dmma_probe.cu && /tmp/dmma_probe
#include <cstdio>
#include <cuda_runtime.h>

template <int SHAPE>
__global__ void __launch_bounds__(256) probe(double* out, int iters) {
  double a[8], b[4], c[8][4];
  for (int i = 0; i < 8; i++) a[i] = threadIdx.x * 1e-3 + i;
  for (int i = 0; i < 4; i++) b[i] = threadIdx.x * 1e-4 + i;
  for (int j = 0; j < 8; j++)
    for (int i = 0; i < 4; i++) c[j][i] = 0.0;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int j = 0; j < 8; j++) {
      if (SHAPE == 0)
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[j][0]), "+d"(c[j][1]) : "d"(a[0]), "d"(b[0]));
      if (SHAPE == 1)
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                     : "+d"(c[j][0]), "+d"(c[j][1]), "+d"(c[j][2]), "+d"(c[j][3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
      if (SHAPE == 2)
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+d"(c[j][0]), "+d"(c[j][1]), "+d"(c[j][2]), "+d"(c[j][3]) : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
      if (SHAPE == 3)
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
                     : "+d"(c[j][0]), "+d"(c[j][1]), "+d"(c[j][2]), "+d"(c[j][3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
    }
  }
  double s = 0.0;
  for (int j = 0; j < 8; j++)
    for (int i = 0; i < 4; i++) s += c[j][i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void __launch_bounds__(256) probe_dfma(double* out, int iters) {
  double c[16], a = threadIdx.x * 1e-3, b = 1.0000001;
  for (int i = 0; i < 16; i++) c[i] = i;
  for (int it = 0; it < iters; it++)
#pragma unroll
    for (int i = 0; i < 16; i++) c[i] = fma(a, c[i], b);
  double s = 0.0;
  for (int i = 0; i < 16; i++) s += c[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  double* out;
  cudaMalloc(&out, sizeof(double) * sms * 4 * 256);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  const int iters = 20000;
  const double fl[4] = {2.0 * 8 * 8 * 4, 2.0 * 16 * 8 * 4, 2.0 * 16 * 8 * 8, 2.0 * 16 * 8 * 16};
  const char* nm[4] = {"m8n8k4", "m16n8k4", "m16n8k8", "m16n8k16"};
  for (int ctas = 1; ctas <= 4; ctas *= 2)
    for (int sh = 0; sh < 5; sh++) {
      float best = 1e9f;
      for (int rep = 0; rep < 3; rep++) {
        cudaEventRecord(e0);
        if (sh == 0) probe<0><<<sms * ctas, 256>>>(out, iters);
        if (sh == 1) probe<1><<<sms * ctas, 256>>>(out, iters);
        if (sh == 2) probe<2><<<sms * ctas, 256>>>(out, iters);
        if (sh == 3) probe<3><<<sms * ctas, 256>>>(out, iters);
        if (sh == 4) probe_dfma<<<sms * ctas, 256>>>(out, iters);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) best = ms;
      }
      const double flops = sh < 4 ? fl[sh] * 8.0 * iters * 8 /*warps*/ * sms * ctas : 2.0 * 16 * iters * 256.0 * sms * ctas;
      printf("%d CTA/SM  %-9s %8.3f ms  %7.2f TFLOP/s  (%s)\n", ctas, sh < 4 ? nm[sh] : "dfma", best, flops / best * 1e-9, cudaGetErrorString(cudaGetLastError()));
    }
  return 0;
}
