// FP64 GEMM on Hopper's m16n8k8 DMMA: the FP64 GEMMs of the fit (Cholesky updates, shadows, W_PP, rows of L⁻¹).
// Same operation, tile and K-range clipping as dgemm64_kernel (dgemm.cuh): C[M×N] = alpha · A[M×K] · op(B) + beta · C.
// Why a second kernel: on an H100 the m8n8k4 DMMA runs at half the FP64 tensor rate and m16n8k{4,8,16} at the full rate
// (DESIGN.md §3 "The fit"), and the register-prefetch feed of dgemm64_kernel leaves the load latency of every K-slab exposed
// in the small GEMMs on the chain's 8 SMs.  Here a three-stage cp.async ring keeps two slabs in flight.
// Why k8 and not k16: beside 64 accumulator registers per thread, m16n8k16's 20 live fragment doubles spill at the 128-register
// cap that two CTAs per SM need; m16n8k8's 10 do not, and the k8 kernel was 4–6 % faster on every Cholesky shape of
// tests/studies/dgemm_sm90_probe.cu.
#pragma once
#include "dgemm.cuh"

#define DS_STAGES 3
#define DS_SMEM_BYTES (DS_STAGES * DG_STAGE_DOUBLES * 8)

// D(16×8) += A(16×8)·B(8×8).  Fragments (lane = 4g + t): a = A[g][t], A[g+8][t], A[g][t+4], A[g+8][t+4]; b = B[t][g], B[t+4][g];
// c = C[g][2t], C[g][2t+1], C[g+8][2t], C[g+8][2t+1].  One instruction carries 1024 FMAs (four times m8n8k4's).
__device__ __forceinline__ void dmma_m16n8k8(double (&d)[4], const double (&a)[4], const double (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}

// 8-byte asynchronous copy global → shared; ok = false writes 0.0 and reads nothing (src must still be a valid address)
__device__ __forceinline__ void cp_async8(double* dst, const double* src, bool ok) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(s), "l"(src), "r"(ok ? 8 : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

// TRANSB = true: B is N×K row-major (C = A·Bᵀ, "NT"); false: B is K×N row-major ("NN").  128×64 CTA tile, 8 warps in a 4×2 grid,
// each warp a 32×32 sub-tile = 2×4 m16n8 tiles (32 accumulator doubles per thread), two k8 steps per 16-wide K-slab.  The
// shared-memory layout is dgemm64_kernel's: [row][k] with pitch 20 and NN's B as [k][n] with pitch 68, so each half-warp's fragment
// loads (lanes (g, t) = (row, k) or (k, n)) land on 16 distinct 8-byte banks.  Per 16-wide K-slab a warp loads 8 KB for 32 K flop: half of what shared memory can deliver
// at the full DMMA rate.  No split-K: every element of C is one fixed-order sum, so the fit stays bit-identical across ranks.
template <bool TRANSB>
__global__ void __launch_bounds__(256, 2)
dgemm_sm90_kernel(int M, int N, int K, const double* __restrict__ A, int lda, const double* __restrict__ B, int ldb,
                  double* __restrict__ C, int ldc, double alpha, double beta, int kmode, int kbegin, int tileskip,
                  long long strideA, long long strideB, long long strideC) {
  A += (long long)blockIdx.z * strideA;
  B += (long long)blockIdx.z * strideB;
  C += (long long)blockIdx.z * strideC;
  extern __shared__ __align__(16) double ds_smem[];
  const int m0 = blockIdx.y * DG_BM, n0 = blockIdx.x * DG_BN;
  if (tileskip == TS_LOWER && n0 > m0 + DG_BM - 1) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  int kb = kbegin, ke = K;
  if (kmode == KM_UPTO_N) ke = min(K, n0 + DG_BN);
  if (kmode == KM_FROM_N) kb = max(kbegin, n0);
  if (kmode == KM_UPTO_M) ke = min(K, m0 + DG_BM);
  if (kmode == KM_FROM_M) kb = max(kbegin, m0);
  kb = kb & ~(DG_BK - 1);

  // stage s: A as [row][k] (pitch DG_LDK), then B as [n][k] (NT) or [k][n] (NN).  Thread tid copies k = tid & 15 of rows
  // tid/16 + 16i (NN's B: n = tid & 63 of k-rows tid/64 + 4i); one base pointer per operand keeps the copy loop's registers low
  const int lr = tid >> 4, lk = tid & 15;
  const double* Ag = A + (size_t)(m0 + lr) * lda + lk;
  const double* Bg = TRANSB ? B + (size_t)(n0 + lr) * ldb + lk : B + (size_t)(tid >> 6) * ldb + n0 + (tid & 63);
  auto load = [&](int s, int k0) {
    double* As = ds_smem + s * DG_STAGE_DOUBLES;
    double* Bs = As + DG_A_DOUBLES;
    const bool kok = k0 + lk < ke && k0 + lk >= kbegin;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const bool ok = kok && m0 + lr + 16 * i < M;
      cp_async8(As + (lr + 16 * i) * DG_LDK + lk, ok ? Ag + (size_t)(16 * i) * lda + k0 : A, ok);
    }
    if (TRANSB) {
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const bool ok = kok && n0 + lr + 16 * i < N;
        cp_async8(Bs + (lr + 16 * i) * DG_LDK + lk, ok ? Bg + (size_t)(16 * i) * ldb + k0 : B, ok);
      }
    } else {
      const int n = tid & 63;
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int k = (tid >> 6) + 4 * i, gk = k0 + k;
        const bool ok = n0 + n < N && gk < ke && gk >= kbegin;
        cp_async8(Bs + k * DG_LDB + n, ok ? Bg + (size_t)(4 * i + k0) * ldb : B, ok);
      }
    }
  };
  // the first DS_STAGES − 1 slabs are requested before C is read; one commit group per slab, empty past the end
#pragma unroll
  for (int s = 0; s < DS_STAGES - 1; s++) {
    if (kb + s * DG_BK < ke) load(s, kb + s * DG_BK);
    cp_async_commit();
  }

  // alpha = ±1, beta = 1: the accumulators start from alpha·C (as in dgemm64_kernel), read while the first slabs are in flight
  const bool preload = beta == 1.0 && (alpha == 1.0 || alpha == -1.0);
  double acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; i++)
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
      for (int e = 0; e < 4; e++) acc[i][j][e] = 0.0;
  if (preload) {
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
      for (int j = 0; j < 4; j++)
#pragma unroll
        for (int e = 0; e < 4; e++) {
          const int gm = m0 + wm + 16 * i + g + 8 * (e >> 1), gn = n0 + wn + 8 * j + 2 * t + (e & 1);
          if (gm < M && gn < N) acc[i][j][e] = alpha * C[(size_t)gm * ldc + gn];
        }
  }

  int s = 0;
  for (int k0 = kb; k0 < ke; k0 += DG_BK) {
    cp_async_wait<DS_STAGES - 2>();   // this thread's copies of slab k0 have landed ...
    __syncthreads();                  // ... everyone's have, and the slot loaded below was consumed by all warps last iteration
    {
      const int kn = k0 + (DS_STAGES - 1) * DG_BK, sn = s == 0 ? DS_STAGES - 1 : s - 1;
      if (kn < ke) load(sn, kn);
      cp_async_commit();
    }
    const double* As = ds_smem + s * DG_STAGE_DOUBLES;
    const double* Bs = As + DG_A_DOUBLES;
#pragma unroll
    for (int kh = 0; kh < DG_BK; kh += 8) {
      double a[2][4];
#pragma unroll
      for (int i = 0; i < 2; i++)
#pragma unroll
        for (int q = 0; q < 2; q++) {
          a[i][2 * q] = As[(wm + 16 * i + g) * DG_LDK + kh + t + 4 * q];
          a[i][2 * q + 1] = As[(wm + 16 * i + 8 + g) * DG_LDK + kh + t + 4 * q];
        }
#pragma unroll
      for (int j = 0; j < 4; j++) {
        double b[2];
#pragma unroll
        for (int q = 0; q < 2; q++)
          b[q] = TRANSB ? Bs[(wn + 8 * j + g) * DG_LDK + kh + t + 4 * q] : Bs[(kh + t + 4 * q) * DG_LDB + wn + 8 * j + g];
        dmma_m16n8k8(acc[0][j], a[0], b);
        dmma_m16n8k8(acc[1][j], a[1], b);
      }
    }
    s = s == DS_STAGES - 1 ? 0 : s + 1;
  }
  cp_async_wait<0>();   // no copy may still target shared memory when the CTA exits

#pragma unroll
  for (int i = 0; i < 2; i++)
#pragma unroll
    for (int e2 = 0; e2 < 2; e2++) {
      const int gm = m0 + wm + 16 * i + g + 8 * e2;
      if (gm >= M) continue;
#pragma unroll
      for (int j = 0; j < 4; j++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int gn = n0 + wn + 8 * j + 2 * t + e;
          if (gn >= N) continue;
          double* c = C + (size_t)gm * ldc + gn;
          const double v = acc[i][j][2 * e2 + e];
          *c = (beta == 0.0 || preload) ? alpha * v : alpha * v + beta * (*c);
        }
    }
}

// More than 48 KB of dynamic shared memory needs the opt-in, once per instantiation and device.  Callers that capture launches
// into a CUDA graph call this before the capture begins: no attribute call may run inside one.
template <bool TRANSB>
static inline void dgemm_sm90_opt_in() {
  static bool attr_set[16] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 16 && !attr_set[dev]) {
    cudaFuncSetAttribute(dgemm_sm90_kernel<TRANSB>, cudaFuncAttributeMaxDynamicSharedMemorySize, DS_SMEM_BYTES);
    attr_set[dev] = true;
  }
}

template <bool TRANSB>
static inline void dgemm_sm90_launch(cudaStream_t s, int M, int N, int K, const double* A, int lda, const double* B, int ldb, double* C,
                                     int ldc, double alpha, double beta, int kmode, int kbegin, int tileskip, int batch = 1,
                                     long long strideA = 0, long long strideB = 0, long long strideC = 0) {
  dim3 grid((N + DG_BN - 1) / DG_BN, (M + DG_BM - 1) / DG_BM, batch);
  dgemm_sm90_opt_in<TRANSB>();
  dgemm_sm90_kernel<TRANSB><<<grid, 256, DS_SMEM_BYTES, s>>>(M, N, K, A, lda, B, ldb, C, ldc, alpha, beta, kmode, kbegin, tileskip, strideA,
                                                             strideB, strideC);
}
