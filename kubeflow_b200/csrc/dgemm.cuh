// FP64 GEMM building block on the FP64 tensor cores (DMMA m8n8k4).
// C[M×N] = alpha · A[M×K] · op(B) + beta · C, with per-tile K-range clipping for triangular operands.
// Used by the FP64 (checker-precision) variance contraction, the LML gradient and CMA-ES; the fit's GEMMs use the m16n8k8 kernel
// of dgemm_sm90.cuh, which shares this file's tile constants and K-range modes.
#pragma once
#include <cuda_runtime.h>

enum { KM_FULL = 0, KM_UPTO_N = 1, KM_FROM_N = 2, KM_UPTO_M = 3, KM_FROM_M = 4 };
enum { EPI_STORE = 0, EPI_ROWSUMSQ = 1 };
enum { TS_NONE = 0, TS_LOWER = 1 };

#define DG_BM 128
#define DG_BN 64
#define DG_BK 16
// Shared-memory tiles are [row][k] with a row pitch of 20 doubles (NN's B tile: [k][n], pitch 68).  A 64-bit shared access is
// served per half-warp over 16 eight-byte banks, so both access patterns must touch 16 distinct banks per half-warp:
//  * the slab store — lanes = 16 consecutive k of one row — is contiguous;
//  * the DMMA fragment load — lanes (g, t) = (row, k) — lands on bank (g·pitch + t) mod 16 = 4g + t for g < 4: distinct.
// (The first layout, [k][row] with pitch ≡ 8, had the loads 2-way and the stores 8-way conflicted: ncu showed the tensor pipe 53 %
// active, `mio_throttle` the top stall.)
#define DG_LDK (DG_BK + 4)
#define DG_LDB (DG_BN + 4)
#define DG_A_DOUBLES (DG_BM * DG_LDK)
#define DG_B_DOUBLES (DG_BN * DG_LDK > DG_BK * DG_LDB ? DG_BN * DG_LDK : DG_BK * DG_LDB)
#define DG_STAGE_DOUBLES (DG_A_DOUBLES + DG_B_DOUBLES)
#define DG_SMEM_BYTES (2 * DG_STAGE_DOUBLES * 8 + 2 * DG_BM * 8)   // two slabs + the row-sum epilogue's scratch

// FP64 tensor-core MMA (DMMA), warp-level: D(8×8) += A(8×4)·B(4×8).  Fragments (lane = 4g + t): a = A[g][t], b = B[t][g],
// c/d = C[g][2t], C[g][2t+1].  DMMA and plain DFMA peak rates: tests/studies/dmma_probe.cu; the point of
// the tensor form is that one fragment load feeds 256 FMAs, so the FP64 GEMM-shaped work (FP64 variance contraction, LML
// gradient, CMA-ES products) is not bound by shared-memory loads.
__device__ __forceinline__ void dmma_m8n8k4(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

// TRANSB = true : B is N×K row-major (C = A·Bᵀ, "NT");  false: B is K×N row-major ("NN").
// 128×64 CTA tile, 8 warps in a 4×2 grid, each warp a 32×32 sub-tile = 4×4 DMMA tiles (32 accumulator doubles per
// thread).  The next K-slab is prefetched into registers while the current one is consumed.
template <bool TRANSB, int EPI>
__global__ void __launch_bounds__(256, 2)
dgemm64_kernel(int M, int N, int K, const double* __restrict__ A, int lda, const double* __restrict__ B, int ldb,
               double* __restrict__ C, int ldc, double alpha, double beta, int kmode, int kbegin, int tileskip,
               long long strideA, long long strideB, long long strideC) {
  A += (long long)blockIdx.z * strideA;
  B += (long long)blockIdx.z * strideB;
  C += (long long)blockIdx.z * strideC;
  // two slabs of shared memory: the next slab is stored while the current one is consumed, one barrier per slab
  extern __shared__ __align__(16) double dg_smem[];
  double(*As)[DG_LDK] = reinterpret_cast<double(*)[DG_LDK]>(dg_smem);
  double* Bs_raw = dg_smem + DG_A_DOUBLES;
  double(*Bt)[DG_LDK] = reinterpret_cast<double(*)[DG_LDK]>(Bs_raw);   // TRANSB: [n][k]
  double(*Bn)[DG_LDB] = reinterpret_cast<double(*)[DG_LDB]>(Bs_raw);   // NN:     [k][n]
  auto flip = [&](int buf) {
    As = reinterpret_cast<double(*)[DG_LDK]>(dg_smem + buf * DG_STAGE_DOUBLES);
    Bs_raw = dg_smem + buf * DG_STAGE_DOUBLES + DG_A_DOUBLES;
    Bt = reinterpret_cast<double(*)[DG_LDK]>(Bs_raw);
    Bn = reinterpret_cast<double(*)[DG_LDB]>(Bs_raw);
  };
  const int m0 = blockIdx.y * DG_BM, n0 = blockIdx.x * DG_BN;
  if (tileskip == TS_LOWER && n0 > m0 + DG_BM - 1) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;   // this warp's sub-tile origin inside the CTA tile
  int kb = kbegin, ke = K;
  if (kmode == KM_UPTO_N) ke = min(K, n0 + DG_BN);
  if (kmode == KM_FROM_N) kb = max(kbegin, n0);
  if (kmode == KM_UPTO_M) ke = min(K, m0 + DG_BM);
  if (kmode == KM_FROM_M) kb = max(kbegin, m0);
  kb = kb & ~(DG_BK - 1);

  // alpha = ±1, beta = 1 (every update of the factorisation): the accumulators START from ±C, so the tile of C is read while the
  // first slab is in flight instead of in a serialised read-modify-write epilogue — at K = 256 that epilogue was a quarter of the
  // kernel.  (Accumulating onto C instead of adding C last changes the rounding order, not the error bound.)
  const bool preload = EPI == EPI_STORE && beta == 1.0 && (alpha == 1.0 || alpha == -1.0);
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j][0] = acc[i][j][1] = 0.0;
  if (preload) {
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int gm = m0 + wm + 8 * i + g;
#pragma unroll
      for (int j = 0; j < 4; j++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int gn = n0 + wn + 8 * j + 2 * t + e;
          if (gm < M && gn < N) acc[i][j][e] = alpha * C[(size_t)gm * ldc + gn];
        }
    }
  }

  double pa[8], pb[4];
  auto prefetch = [&](int k0) {
    {
      const int k = tid & 15, gk = k0 + k;
      const bool kok = gk < ke && gk >= kbegin;
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const int gm = m0 + (tid >> 4) + 16 * i;
        pa[i] = (kok && gm < M) ? A[(size_t)gm * lda + gk] : 0.0;
      }
    }
    if (TRANSB) {
      const int k = tid & 15, gk = k0 + k;
      const bool kok = gk < ke && gk >= kbegin;
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int gn = n0 + (tid >> 4) + 16 * i;
        pb[i] = (kok && gn < N) ? B[(size_t)gn * ldb + gk] : 0.0;
      }
    } else {
      const int gn = n0 + (tid & 63);
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int gk = k0 + (tid >> 6) + 4 * i;
        pb[i] = (gn < N && gk < ke && gk >= kbegin) ? B[(size_t)gk * ldb + gn] : 0.0;
      }
    }
  };
  auto commit = [&]() {
#pragma unroll
    for (int i = 0; i < 8; i++) As[(tid >> 4) + 16 * i][tid & 15] = pa[i];
    if (TRANSB) {
#pragma unroll
      for (int i = 0; i < 4; i++) Bt[(tid >> 4) + 16 * i][tid & 15] = pb[i];
    } else {
#pragma unroll
      for (int i = 0; i < 4; i++) Bn[(tid >> 6) + 4 * i][tid & 63] = pb[i];
    }
  };
  if (kb < ke) {
    prefetch(kb);
    commit();
    if (kb + DG_BK < ke) prefetch(kb + DG_BK);
  }
  __syncthreads();
  int buf = 0;
  for (int k0 = kb; k0 < ke; k0 += DG_BK) {
    const bool more = k0 + DG_BK < ke;
    if (more) {   // the next slab (in registers since the previous iteration) goes to the other buffer, the one after it is requested
      double(*Ac)[DG_LDK] = As;
      double(*Btc)[DG_LDK] = Bt;
      double(*Bnc)[DG_LDB] = Bn;
      flip(buf ^ 1);
      commit();
      if (k0 + 2 * DG_BK < ke) prefetch(k0 + 2 * DG_BK);
      As = Ac;
      Bt = Btc;
      Bn = Bnc;
    }
#pragma unroll
    for (int k4 = 0; k4 < DG_BK; k4 += 4) {
      double a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; i++) a[i] = As[wm + 8 * i + g][k4 + t];
#pragma unroll
      for (int j = 0; j < 4; j++) b[j] = TRANSB ? Bt[wn + 8 * j + g][k4 + t] : Bn[k4 + t][wn + 8 * j + g];
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) dmma_m8n8k4(acc[i][j][0], acc[i][j][1], a[i], b[j]);
    }
    if (more) flip(buf ^ 1);
    buf ^= 1;
    __syncthreads();
  }

  // accumulator (i, j, e) is C[m0 + wm + 8i + g][n0 + wn + 8j + 2t + e]
  if (EPI == EPI_STORE) {
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int gm = m0 + wm + 8 * i + g;
      if (gm >= M) continue;
#pragma unroll
      for (int j = 0; j < 4; j++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int gn = n0 + wn + 8 * j + 2 * t + e;
          if (gn >= N) continue;
          double* c = C + (size_t)gm * ldc + gn;
          *c = (beta == 0.0 || preload) ? alpha * acc[i][j][e] : alpha * acc[i][j][e] + beta * (*c);
        }
    }
  } else {  // EPI_ROWSUMSQ: C is part[M × ldc], column = this block's n-tile; fixed reduction order
    double(*rs)[DG_BM] = reinterpret_cast<double(*)[DG_BM]>(dg_smem + 2 * DG_STAGE_DOUBLES);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      double s = 0.0;
#pragma unroll
      for (int j = 0; j < 4; j++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int gn = n0 + wn + 8 * j + 2 * t + e;
          if (gn < N) s = fma(acc[i][j][e], acc[i][j][e], s);
        }
      s += __shfl_xor_sync(0xffffffffu, s, 1);   // the 4 lanes of a row group
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      if (t == 0) rs[warp & 1][wm + 8 * i + g] = s;
    }
    __syncthreads();
    if (tid < DG_BM && m0 + tid < M) C[(size_t)(m0 + tid) * ldc + blockIdx.x] = rs[0][tid] + rs[1][tid];
  }
}

template <bool TRANSB, int EPI>
static inline void dgemm64_launch(cudaStream_t s, int M, int N, int K, const double* A, int lda, const double* B, int ldb,
                                  double* C, int ldc, double alpha, double beta, int kmode, int kbegin, int tileskip,
                                  int batch = 1, long long strideA = 0, long long strideB = 0, long long strideC = 0) {
  dim3 grid((N + DG_BN - 1) / DG_BN, (M + DG_BM - 1) / DG_BM, batch);
  static bool attr_set[16] = {};   // per instantiation and device: more than 48 KB of dynamic shared memory needs the opt-in
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 16 && !attr_set[dev]) {
    cudaFuncSetAttribute(dgemm64_kernel<TRANSB, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, DG_SMEM_BYTES);
    attr_set[dev] = true;
  }
  dgemm64_kernel<TRANSB, EPI><<<grid, 256, DG_SMEM_BYTES, s>>>(M, N, K, A, lda, B, ldb, C, ldc, alpha, beta, kmode, kbegin, tileskip,
                                                   strideA, strideB, strideC);
}
