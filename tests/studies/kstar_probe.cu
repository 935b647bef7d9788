// Where do the cycles of tc_kstar_kernel go?  Restates its tile loop at cfg3's shape (262 144 candidate rows, Npad 8192, D 32,
// Matérn-5/2, a pruning pass that stores the first 8 of 64 trial tiles) with compile-time switches, and times, in one run:
//   (a) the whole tile loop, as the parent built it (both warpgroups in lock-step, pairs by LDG, stores under a predicate), as it
//       is now (still lock-step, pairs staged in shared memory with the trial planes, a mean-only body), and the same with the two
//       warpgroups ping-ponged by named turn barriers (one's MMAs under the other's epilogue), which measured slower
//   Its answers are recorded in DESIGN.md §3 (tc_kstar.cu).
//   (b) MMA only: the epilogue replaced by one FADD per accumulator into a sink
//   (c) epilogue only: no wgmma, the accumulator a cheap function of the column
//   (d) MUFU.EX2 / MUFU.SQRT / MUFU.RSQ throughput per SM with 1 and 2 warps per SMSP
// Cycles per tile per SM come from clock64() around each CTA (one CTA per SM), so they do not depend on the clock the card ran at.
// Operand contents are arbitrary finite fp16: they set no timing.  Loads use plain bulk copies instead of tensor maps.
//
// Build: nvcc -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -o /tmp/kstar_probe tests/studies/kstar_probe.cu
// Run:   nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv && /tmp/kstar_probe
#include <cstdio>
#include <cstdlib>
#include <type_traits>
#include <vector>

#include "../../kubeflow_b200/csrc/tc_common.cuh"

using namespace tcx;

constexpr int BM = 128, BN = 128, BK = 32, STAGES = 4, CONSUMERS = 256, THREADS = CONSUMERS + 32;
constexpr int ROWS = 262144, NPAD = 8192, NT = NPAD / BN, STORE_TILES = 8;
constexpr int A_BYTES = BM * BK * 2 * 2, STAGE_BYTES = BN * BK * 2 * 2, NX_BYTES = BN * 8;
constexpr size_t SMEM = 1024 + A_BYTES + STAGES * (STAGE_BYTES + NX_BYTES) + 256;
enum { FULL = 0, MMA_ONLY = 1, EPI_ONLY = 2 };

#define CK(x)                                                                              \
  do {                                                                                     \
    cudaError_t e = (x);                                                                   \
    if (e != cudaSuccess) {                                                                \
      fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e));   \
      exit(1);                                                                             \
    }                                                                                      \
  } while (0)

__device__ __forceinline__ float ex2_ftz(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float sqrt_ftz(float x) {
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float rsq_ftz(float x) {
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float matern(float dot, float nsum, float log2amp) {   // tc_kstar.cu's ks_kernel_value<1>
  const float d2 = fmaf(-2.f, dot, nsum);
  const float s = sqrt_ftz(fabsf(d2));
  const float p = fmaf(fmaf(s, 0.33333334f, 1.f), s, 1.f);
  return p * ex2_ftz(fmaf(s, -1.4426950408889634f, log2amp));
}

// PP: ping-pong turn barriers.  NEW: pairs from shared memory (stage held over the epilogue) and a mean-only body for tiles past
// STORE_TILES; otherwise pairs by LDG straight after the MMAs and one body with the stores under a predicate.
template <int MODE, bool PP, bool NEW>
__global__ void __launch_bounds__(THREADS, 1)
probe_kernel(const __half* __restrict__ A, const __half* __restrict__ B, const float4* __restrict__ nxal4, const float* __restrict__ ncand,
             float log2amp, __half* __restrict__ out, float* __restrict__ mun, long long* __restrict__ cyc) {
  extern __shared__ unsigned char raw[];
  unsigned char* smA = (unsigned char*)(((uintptr_t)raw + 1023) & ~(uintptr_t)1023);
  unsigned char* ring = smA + A_BYTES;
  unsigned char* nxs = ring + STAGES * STAGE_BYTES;
  uint64_t* full = (uint64_t*)(nxs + STAGES * NX_BYTES);
  uint64_t* empty = full + STAGES;
  uint64_t* a_full = empty + STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == CONSUMERS) {
    for (int i = 0; i < STAGES; i++) {
      mbar_init(smem_u32(&full[i]), 1);
      mbar_init(smem_u32(&empty[i]), 2);
    }
    mbar_init(smem_u32(a_full), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const long long t_start = clock64();
  if (warp == CONSUMERS / 32) {
    if (lane == 0) {
      mbar_expect_tx(smem_u32(a_full), A_BYTES);
      bulk_load(smem_u32(smA), A + (size_t)blockIdx.x * (A_BYTES / 2), A_BYTES, smem_u32(a_full));
      for (int t = 0; t < NT; t++) {
        const uint32_t st = t % STAGES, use = t / STAGES;
        mbar_wait(smem_u32(&empty[st]), (use & 1) ^ 1);
        const uint32_t bar = smem_u32(&full[st]);
        mbar_expect_tx(bar, STAGE_BYTES + (NEW ? NX_BYTES : 0));
        bulk_load(smem_u32(ring + st * STAGE_BYTES), B + (size_t)t * (STAGE_BYTES / 2), STAGE_BYTES, bar);
        if (NEW) bulk_load(smem_u32(nxs + st * NX_BYTES), nxal4 + (size_t)t * (BN / 2), NX_BYTES, bar);
      }
    }
    __syncwarp();
  } else {
    const int wg = threadIdx.x >> 7, wl = (threadIdx.x >> 5) & 3, q = lane & 3;
    const int r0 = blockIdx.x * BM + wg * 64 + wl * 16 + (lane >> 2), r1 = r0 + 8;
    const bool signal = (threadIdx.x & 127) == 0;
    const float nc0 = ncand[r0], nc1 = ncand[r1];
    __half* out0 = out + (size_t)r0 * (STORE_TILES * BN);
    __half* out1 = out + (size_t)r1 * (STORE_TILES * BN);
    double mu0 = 0.0, mu1 = 0.0;
    float sink = 0.f;
    float acc[64];
    mbar_wait(smem_u32(a_full), 0);
    if (PP && wg == 1) named_bar_arrive(1, CONSUMERS);
    for (int t = 0; t < NT; t++) {
      const uint32_t st = t % STAGES, use = t / STAGES;
      if (PP) named_bar_sync(1 + wg, CONSUMERS);
      mbar_wait(smem_u32(&full[st]), use & 1);
      if (MODE != EPI_ONLY) {
        const uint32_t a_hi = smem_u32(smA) + wg * (A_BYTES / 8), a_lo = a_hi + A_BYTES / 2;
        const uint32_t b_hi = smem_u32(ring + st * STAGE_BYTES), b_lo = b_hi + STAGE_BYTES / 2;
        wgmma_fence();
#pragma unroll
        for (int prod = 0; prod < 4; prod++) {
          const uint32_t a = (prod < 2) ? a_lo : a_hi, b = (prod & 1) ? b_hi : b_lo;
#pragma unroll
          for (int k = 0; k < BK / 16; k++) wgmma_f16_n128(acc, gmma_desc_sw64(a + k * 32), gmma_desc_sw64(b + k * 32), (prod > 0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
      } else {
#pragma unroll
        for (int j = 0; j < 64; j++) acc[j] = fmaf((float)t, 1e-3f, (float)j * 0.01f);
      }
      if (PP && (wg == 0 || t + 1 < NT)) named_bar_arrive(2 - wg, CONSUMERS);
      if (MODE != EPI_ONLY) {
        wgmma_wait<0>();
        acc_fence(acc);
      }
      if (!NEW && signal) mbar_arrive(smem_u32(&empty[st]));
      if (MODE == MMA_ONLY) {
#pragma unroll
        for (int j = 0; j < 64; j++) sink += acc[j];
      } else {
        const int n_base = t * BN;
        const uint32_t nx = smem_u32(nxs + st * NX_BYTES) + q * 16;
        auto body = [&](auto store_tag) {
          constexpr bool STORE = decltype(store_tag)::value;
          float ma0 = 0.f, mb0 = 0.f, ma1 = 0.f, mb1 = 0.f;
#pragma unroll
          for (int i = 0; i < BN / 8; i++) {
            const int n = n_base + 8 * i + 2 * q;
            const float4 na = NEW ? lds128(nx + i * 64) : __ldg(nxal4 + (n >> 1));
            const float k00 = matern(acc[4 * i], nc0 + na.x, log2amp), k01 = matern(acc[4 * i + 1], nc0 + na.z, log2amp);
            const float k10 = matern(acc[4 * i + 2], nc1 + na.x, log2amp), k11 = matern(acc[4 * i + 3], nc1 + na.z, log2amp);
            ma0 = fmaf(k00, na.y, ma0);
            mb0 = fmaf(k01, na.w, mb0);
            ma1 = fmaf(k10, na.y, ma1);
            mb1 = fmaf(k11, na.w, mb1);
            if (STORE && (NEW || t < STORE_TILES)) {
              *reinterpret_cast<__half2*>(out0 + n) = __floats2half2_rn(k00, k01);
              *reinterpret_cast<__half2*>(out1 + n) = __floats2half2_rn(k10, k11);
            }
          }
          mu0 += (double)(ma0 + mb0);
          mu1 += (double)(ma1 + mb1);
        };
        if (!NEW || t < STORE_TILES)
          body(std::true_type{});
        else
          body(std::false_type{});
      }
      if (NEW) {
        named_bar_sync(3 + wg, 128);
        if (signal) mbar_arrive(smem_u32(&empty[st]));
      }
    }
    if ((lane & 3) == 0) {
      mun[r0] = (float)mu0 + sink;
      mun[r1] = (float)mu1;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) cyc[blockIdx.x] = clock64() - t_start;
}

template <int OP>
__global__ void mufu_kernel(float* out, long long* cyc, int iters) {
  float x[8];
#pragma unroll
  for (int k = 0; k < 8; k++) x[k] = 0.5f + 0.01f * (threadIdx.x + k);
  __syncthreads();
  const long long t0 = clock64();
  for (int it = 0; it < iters; it++)
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = OP == 0 ? ex2_ftz(-x[k]) : OP == 1 ? sqrt_ftz(x[k]) : rsq_ftz(x[k]);
  __syncthreads();
  if (threadIdx.x == 0) cyc[blockIdx.x] = clock64() - t0;
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < 8; k++) s += x[k];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

static double mean_cycles(const long long* d, int n) {
  std::vector<long long> h(n);
  CK(cudaMemcpy(h.data(), d, sizeof(long long) * n, cudaMemcpyDeviceToHost));
  double s = 0;
  for (long long v : h) s += (double)v;
  return s / n;
}

template <int MODE, bool PP, bool NEW>
static void run(const char* label, const __half* A, const __half* B, const float4* nx, const float* nc, __half* out, float* mun, long long* cyc) {
  auto k = probe_kernel<MODE, PP, NEW>;
  CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM));
  const int grid = ROWS / BM;
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  k<<<grid, THREADS, SMEM>>>(A, B, nx, nc, 0.f, out, mun, cyc);
  CK(cudaGetLastError());
  const int reps = 5;
  CK(cudaEventRecord(e0));
  for (int r = 0; r < reps; r++) k<<<grid, THREADS, SMEM>>>(A, B, nx, nc, 0.f, out, mun, cyc);
  CK(cudaEventRecord(e1));
  CK(cudaEventSynchronize(e1));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  const double cpt = mean_cycles(cyc, grid) / NT;
  printf("%-58s %8.3f ms/launch  %7.0f cycles/tile/SM\n", label, ms / reps, cpt);
}

template <int OP>
static void run_mufu(const char* label, int nsm, float* buf, long long* cyc) {
  const int iters = 1 << 14;
  for (int warps_per_smsp = 1; warps_per_smsp <= 2; warps_per_smsp++) {
    const int threads = 128 * warps_per_smsp;
    CK(cudaFuncSetAttribute(mufu_kernel<OP>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));   // one CTA per SM
    mufu_kernel<OP><<<nsm, threads, 160 * 1024>>>(buf, cyc, iters);
    mufu_kernel<OP><<<nsm, threads, 160 * 1024>>>(buf, cyc, iters);
    CK(cudaDeviceSynchronize());
    const double c = mean_cycles(cyc, nsm);
    printf("%-10s %d warp(s)/SMSP: %6.2f results/clk/SM\n", label, warps_per_smsp, (double)threads * iters * 8 / c);
  }
}

int main() {
  cudaDeviceProp p;
  CK(cudaGetDeviceProperties(&p, 0));
  printf("%s, %d SMs; cfg3 shape: %d rows, Npad %d, D %d, Matern-5/2, first %d of %d tiles stored\n", p.name, p.multiProcessorCount, ROWS, NPAD, BK,
         STORE_TILES, NT);
  std::vector<__half> hA((size_t)ROWS * BK * 2), hB((size_t)NPAD * BK * 2);
  srand(1);
  for (auto& v : hA) v = __float2half((rand() / (float)RAND_MAX - 0.5f) * 0.5f);
  for (auto& v : hB) v = __float2half((rand() / (float)RAND_MAX - 0.5f) * 0.5f);
  std::vector<float> hnx((size_t)NPAD * 2), hnc(ROWS);
  for (int n = 0; n < NPAD; n++) {
    hnx[2 * n] = 2.f + rand() / (float)RAND_MAX;
    hnx[2 * n + 1] = rand() / (float)RAND_MAX - 0.5f;
  }
  for (auto& v : hnc) v = 2.f + rand() / (float)RAND_MAX;
  __half *A, *B, *out;
  float *nx, *nc, *mun, *buf;
  long long* cyc;
  CK(cudaMalloc(&A, hA.size() * 2));
  CK(cudaMalloc(&B, hB.size() * 2));
  CK(cudaMalloc(&nx, hnx.size() * 4));
  CK(cudaMalloc(&nc, hnc.size() * 4));
  CK(cudaMalloc(&out, (size_t)ROWS * STORE_TILES * BN * 2));
  CK(cudaMalloc(&mun, (size_t)ROWS * 4));
  CK(cudaMalloc(&cyc, sizeof(long long) * (ROWS / BM)));
  CK(cudaMalloc(&buf, sizeof(float) * 1024 * 1024));
  CK(cudaMemcpy(A, hA.data(), hA.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(B, hB.data(), hB.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(nx, hnx.data(), hnx.size() * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(nc, hnc.data(), hnc.size() * 4, cudaMemcpyHostToDevice));
  const float4* nx4 = (const float4*)nx;
  run<FULL, false, false>("(a) full, parent: lock-step, LDG pairs, predicated stores", A, B, nx4, nc, out, mun, cyc);
  run<FULL, false, true>("(a) full, now: lock-step, LDS pairs, mean-only body", A, B, nx4, nc, out, mun, cyc);
  run<FULL, true, true>("(a) full, ping-pong, LDS pairs, mean-only body", A, B, nx4, nc, out, mun, cyc);
  run<MMA_ONLY, false, false>("(b) MMA only, lock-step", A, B, nx4, nc, out, mun, cyc);
  run<MMA_ONLY, true, false>("(b) MMA only, ping-pong", A, B, nx4, nc, out, mun, cyc);
  run<EPI_ONLY, false, false>("(c) epilogue only, parent body", A, B, nx4, nc, out, mun, cyc);
  run<EPI_ONLY, false, true>("(c) epilogue only, new body", A, B, nx4, nc, out, mun, cyc);
  run_mufu<0>("MUFU.EX2", p.multiProcessorCount, buf, cyc);
  run_mufu<1>("MUFU.SQRT", p.multiProcessorCount, buf, cyc);
  run_mufu<2>("MUFU.RSQ", p.multiProcessorCount, buf, cyc);
  printf("MUFU bound of (a): 2 MUFU x %d x %d elements per tile; at 16/clk/SM that is %d cycles/tile/SM\n", BM, BN, 2 * BM * BN / 16);
  return 0;
}
