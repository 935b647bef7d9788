// tell(): GaussianProcessRegressor.fit at fixed θ on the device, FP64 throughout.
//   $SK/_gpr.py:275-280 normalise y | :349-350 K = k(X,X)+alpha·I | :352 L = cholesky(K) | :363 alpha_ = cho_solve
//   $SK/kernels.py:1559-1570 RBF, :1713-1729 Matern(nu=2.5)
// Why FP64 here (not fp32/tensor cores): the posterior mean is K*·alpha with |alpha|₂ up to ~3e3 for the
// workloads of record; fp32 L/alpha moves EI by 1e-4 (measured, DESIGN.md §numerics) against a 1e-5 contract.
// H100 has a full FP64 pipe, and the fit is O(N³/3) once per suggestion next to the O(M·N²) sweep.
#include <stdlib.h>

#include "kbo_internal.cuh"
#include "dgemm_sm90.cuh"
#include "ktab.cuh"

// ------------------------------------------------------------------------------------------------
// Xs = X / ℓ, nx = |Xs|² (one thread per trial row)
__global__ void prep_x_kernel(const double* __restrict__ X, int N, int D, const double* __restrict__ inv_ls, int n_ls,
                              double* __restrict__ Xs, double* __restrict__ XsT, int ldx, double* __restrict__ nx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  double s = 0.0;
  for (int d = 0; d < D; d++) {
    const double v = X[(size_t)i * D + d] * inv_ls[n_ls == 1 ? 0 : d];
    Xs[(size_t)i * D + d] = v;
    XsT[(size_t)d * ldx + i] = v;
    s = fma(v, v, s);
  }
  nx[i] = s;
}

// mean / population std / min of y and the normalised yn — one CTA, fixed-order tree reductions.
__global__ void __launch_bounds__(1024) prep_y_kernel(const double* __restrict__ y, int N, int normalize, double* __restrict__ yn,
                                                      double* __restrict__ scal) {
  __shared__ double red[1024];
  __shared__ double s_mean, s_std;
  const int t = threadIdx.x;
  double a = 0.0, mn = INFINITY;
  for (int i = t; i < N; i += 1024) {
    a += y[i];
    mn = fmin(mn, y[i]);
  }
  red[t] = a;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (t < o) red[t] += red[t + o];
    __syncthreads();
  }
  if (t == 0) s_mean = red[0] / N;
  __syncthreads();
  red[t] = mn;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (t < o) red[t] = fmin(red[t], red[t + o]);
    __syncthreads();
  }
  const double ymin = red[0];
  __syncthreads();
  const double mean = s_mean;
  a = 0.0;
  for (int i = t; i < N; i += 1024) {
    const double d = y[i] - mean;
    a = fma(d, d, a);
  }
  red[t] = a;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (t < o) red[t] += red[t + o];
    __syncthreads();
  }
  if (t == 0) {
    double sd = sqrt(red[0] / N);
    if (sd < 10.0 * 2.220446049250313e-16) sd = 1.0;  // sklearn _handle_zeros_in_scale
    s_std = sd;
  }
  __syncthreads();
  const double m = normalize ? s_mean : 0.0, sd = normalize ? s_std : 1.0;
  for (int i = t; i < N; i += 1024) yn[i] = (y[i] - m) / sd;
  if (t == 0) {
    scal[S_YMEAN] = m;
    scal[S_YSTD] = sd;
    scal[S_YOPT] = ymin;
  }
}

// K = amp·k(Xs,Xs) + noise·I.  Exact pairwise differences (as scipy cdist does), lower tiles computed
// and mirrored.  64×64 tile, 4×4 per thread, D consumed in chunks of 16 through shared memory.
__global__ void __launch_bounds__(256) gram_kernel(const double* __restrict__ Xs, int N, int D, int kind, double amp, double noise,
                                                   double* __restrict__ K, int ldk, int tile0) {
  const int m0 = blockIdx.y * 64, n0 = (blockIdx.x + tile0) * 64;
  if (n0 > m0) return;
  __shared__ double Xi[16][66], Xj[16][66];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  double acc[4][4] = {};
  for (int d0 = 0; d0 < D; d0 += 16) {
    const int d = tid & 15;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int r = (tid >> 4) + 16 * i;
      Xi[d][r] = (m0 + r < N && d0 + d < D) ? Xs[(size_t)(m0 + r) * D + d0 + d] : 0.0;
      Xj[d][r] = (n0 + r < N && d0 + d < D) ? Xs[(size_t)(n0 + r) * D + d0 + d] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int dd = 0; dd < 16; dd++) {
      double a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; i++) a[i] = Xi[dd][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; j++) b[j] = Xj[dd][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const double df = a[i] - b[j];
          acc[i][j] = fma(df, df, acc[i][j]);
        }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int gm = m0 + ty + 16 * i;
    if (gm >= N) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int gn = n0 + tx + 16 * j;
      if (gn >= N) continue;
      double v = amp * kbo_kernel_exact(acc[i][j], kind);
      if (gm == gn) v += noise;
      K[(size_t)gm * ldk + gn] = v;
      if (m0 != n0) K[(size_t)gn * ldk + gm] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Blocked right-looking Cholesky (lower), NB = 64.
// potf2_inv: factor one diagonal block in shared memory and invert it (for the panel solve).  1024 threads:
// thread (i, q) owns row i = t/16 and columns [4q, 4q+4).  Right-looking with ONE barrier per column: the trailing
// update of column j reads the still-unscaled column j and writes only columns > j; column j itself is rescaled after
// the barrier, when nobody reads it any more.
__device__ __forceinline__ void tri_inverse_64(double (*S)[KBO_NB + 1], double (*T)[KBO_NB + 1], double* invd, int t) {
  // T = S⁻¹ (lower), forward substitution per column, 16 threads per column; invd[i] = 1/S[i][i]
  if (t < KBO_NB) invd[t] = 1.0 / S[t][t];
  __syncthreads();
  const int c = t >> 4, q = t & 15;
  for (int i = 0; i < KBO_NB; i++) {
    double s = 0.0;
    for (int k = c + q; k < i; k += 16) s = fma(S[i][k], T[k][c], s);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (q == 0) T[i][c] = (i < c) ? 0.0 : (i == c ? invd[i] : -s * invd[i]);
    __syncwarp();
  }
}

#include <algorithm>
#include <chrono>
#include "potf2.cuh"

// batched inverse of the 64×64 diagonal blocks of a lower-triangular L (for kbo_trtri); one CTA per block
__global__ void __launch_bounds__(1024) diag_inv_kernel(const double* __restrict__ L, int N, int ldl, double* __restrict__ W, int ldw) {
  extern __shared__ double sm[];
  double(*S)[KBO_NB + 1] = reinterpret_cast<double(*)[KBO_NB + 1]>(sm);
  double(*T)[KBO_NB + 1] = reinterpret_cast<double(*)[KBO_NB + 1]>(sm + KBO_NB * (KBO_NB + 1));
  __shared__ double invd[KBO_NB];
  const int t = threadIdx.x, k0 = blockIdx.x * KBO_NB, jb = min(KBO_NB, N - k0);
  for (int e = t; e < KBO_NB * KBO_NB; e += 1024) {
    const int r = e >> 6, c = e & 63;
    S[r][c] = (r < jb && c <= r) ? L[(size_t)(k0 + r) * ldl + k0 + c] : (r == c ? 1.0 : 0.0);
  }
  __syncthreads();
  tri_inverse_64(S, T, invd, t);
  __syncthreads();
  for (int e = t; e < KBO_NB * KBO_NB; e += 1024) {
    const int r = e >> 6, c = e & 63;
    if (r < jb && c < jb) W[(size_t)(k0 + r) * ldw + k0 + c] = T[r][c];
  }
}

// panel solve: P ← P · Linvᵀ for a 64-row slab of the panel below the diagonal block (in place, rows owned by the CTA)
__global__ void __launch_bounds__(256) trsm_panel_kernel(double* __restrict__ P, int lda, int rows, int jb,
                                                         const double* __restrict__ Linv, const int* __restrict__ info) {
  if (*info != 0) return;
  extern __shared__ double sm[];
  double(*Ps)[KBO_NB + 1] = reinterpret_cast<double(*)[KBO_NB + 1]>(sm);
  double(*Ls)[KBO_NB + 1] = reinterpret_cast<double(*)[KBO_NB + 1]>(sm + KBO_NB * (KBO_NB + 1));
  const int t = threadIdx.x, r0 = blockIdx.x * 64;
  for (int e = t; e < 64 * 64; e += 256) {
    const int r = e >> 6, c = e & 63;
    Ps[r][c] = (r0 + r < rows && c < jb) ? P[(size_t)(r0 + r) * lda + c] : 0.0;
    Ls[r][c] = Linv[e];
  }
  __syncthreads();
  const int tx = t & 15, ty = t >> 4;
  double acc[4][4] = {};
  for (int k = 0; k < jb; k++) {
    double a[4], b[4];
#pragma unroll
    for (int i = 0; i < 4; i++) a[i] = Ps[ty + 16 * i][k];
#pragma unroll
    for (int j = 0; j < 4; j++) b[j] = Ls[tx + 16 * j][k];  // (P·Linvᵀ)[r,c] = Σ_k P[r,k]·Linv[c,k]
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int j = 0; j < 4; j++) acc[i][j] = fma(a[i], b[j], acc[i][j]);
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int r = r0 + ty + 16 * i;
    if (r >= rows) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int c = tx + 16 * j;
      if (c < jb) P[(size_t)r * lda + c] = acc[i][j];
    }
  }
}

// `panel_done` (optional) is called after each 256-column outer panel is final — all rows of L in those columns, before the
// trailing update of the rest is enqueued — with the number of finished columns; the fit uses it to interleave L⁻¹.
template <typename Hook>
static int potrf_impl(kbo_handle* h, double* A, int N, int lda, int* info_dev, cudaStream_t s, Hook panel_done, double* Linv_lane = nullptr) {
  if (!Linv_lane) KBO_TRY(kbo_reserve(h, h->Linv, KBO_NB * KBO_NB));
  const int smem = 2 * KBO_NB * (KBO_NB + 1) * (int)sizeof(double);
  if (!h->attr_fit) {
    KBO_CUDA(h, cudaFuncSetAttribute(potf2_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    KBO_CUDA(h, cudaFuncSetAttribute(trsm_panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    KBO_CUDA(h, cudaFuncSetAttribute(diag_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    h->attr_fit = true;
  }
  KBO_CUDA(h, cudaMemsetAsync(info_dev, 0, sizeof(int), s));
  double* Linv = Linv_lane ? Linv_lane : h->Linv.p;   // inverted diagonal block of the current step (one per concurrent factorisation)
  // Two-level blocking: 64-wide diagonal blocks (one CTA each) inside 256-wide outer panels.  Inside a panel only the
  // panel's own remaining columns are updated after each 64-block (K = 64, ≤ 192 columns); the rest of the trailing
  // matrix sees ONE update per outer panel with K = 256 — 4× less read-modify-write traffic on the trailing matrix than
  // updating it after every 64-block (that version was memory bound: 46 GB of traffic at N = 8192).
  const int OW = 256;
  for (int K0 = 0; K0 < N; K0 += OW) {
    const int W = min(OW, N - K0);
    for (int k = K0; k < K0 + W; k += KBO_NB) {
      const int jb = min(KBO_NB, N - k);
      double* Akk = A + (size_t)k * lda + k;
      potf2_inv_kernel<<<1, POTF2_THREADS, smem, s>>>(Akk, lda, jb, k, Linv, info_dev);
      KBO_LAUNCH_CHECK(h);
      const int rows = N - k - jb;
      if (rows > 0) {
        double* P = A + (size_t)(k + jb) * lda + k;
        trsm_panel_kernel<<<(rows + 63) / 64, 256, smem, s>>>(P, lda, rows, jb, Linv, info_dev);
        KBO_LAUNCH_CHECK(h);
        const int cin = K0 + W - (k + jb);  // columns of the outer panel still to be factorised
        if (cin > 0) {
          double* C = A + (size_t)(k + jb) * lda + (k + jb);
          dgemm_sm90_launch<true>(s, rows, cin, jb, P, lda, P, lda, C, lda, -1.0, 1.0, KM_FULL, 0, TS_LOWER);
          KBO_LAUNCH_CHECK(h);
        }
      }
    }
    KBO_TRY(panel_done(K0, W));
    const int rows_t = N - (K0 + W);
    if (rows_t > 0) {
      const double* Pp = A + (size_t)(K0 + W) * lda + K0;  // rows below the panel × the panel's W columns
      double* C = A + (size_t)(K0 + W) * lda + (K0 + W);
      dgemm_sm90_launch<true>(s, rows_t, rows_t, W, Pp, lda, Pp, lda, C, lda, -1.0, 1.0, KM_FULL, 0, TS_LOWER);
      KBO_LAUNCH_CHECK(h);
    }
  }
  return KBO_OK;
}

int kbo_i_potrf(kbo_handle* h, double* A, int N, int lda, int* info_dev, cudaStream_t s) {
  return potrf_impl(h, A, N, lda, info_dev, s, [](int, int) { return (int)KBO_OK; });
}

// W = L^-1 by recursive doubling: [[W11,0],[−W22·L21·W11, W22]] — log2(N/64) levels of two batched GEMMs.
// T: N × ldw scratch (nullptr: the handle's)
int kbo_i_trtri(kbo_handle* h, const double* L, int N, int ldl, double* W, int ldw, cudaStream_t s, double* T) {
  const int smem = 2 * KBO_NB * (KBO_NB + 1) * (int)sizeof(double);
  KBO_CUDA(h, cudaFuncSetAttribute(diag_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  if (!T) {
    KBO_TRY(kbo_reserve(h, h->T, (size_t)N * ldw));
    T = h->T.p;
  }
  KBO_CUDA(h, cudaMemsetAsync(W, 0, sizeof(double) * (size_t)N * ldw, s));
  diag_inv_kernel<<<(N + KBO_NB - 1) / KBO_NB, 1024, smem, s>>>(L, N, ldl, W, ldw);
  KBO_LAUNCH_CHECK(h);
  for (long long b = KBO_NB; b < N; b *= 2) {
    const int full = (int)(N / (2 * b));
    const long long sL = 2 * b * (long long)ldl + 2 * b, sW = 2 * b * (long long)ldw + 2 * b;
    if (full > 0) {
      // T21 = L21 · W11   (W11 lower-triangular: k >= n)
      dgemm_sm90_launch<false>(s, (int)b, (int)b, (int)b, L + b * ldl, ldl, W, ldw, T + b * ldw, ldw, 1.0, 0.0, KM_FROM_N, 0,
                               TS_NONE, full, sL, sW, sW);
      KBO_LAUNCH_CHECK(h);
      // W21 = −W22 · T21  (W22 lower-triangular: k <= m)
      dgemm_sm90_launch<false>(s, (int)b, (int)b, (int)b, W + b * ldw + b, ldw, T + b * ldw, ldw, W + b * ldw, ldw, -1.0, 0.0,
                               KM_UPTO_M, 0, TS_NONE, full, sW, sW, sW);
      KBO_LAUNCH_CHECK(h);
    }
    const long long r0 = (long long)full * 2 * b;
    if (r0 + b < N) {  // ragged last pair: second half has rows2 < b rows
      const int rows2 = (int)(N - (r0 + b));
      const double* L21 = L + (r0 + b) * ldl + r0;
      const double* W11 = W + r0 * ldw + r0;
      double* T21 = T + (r0 + b) * ldw + r0;
      double* W21 = W + (r0 + b) * ldw + r0;
      const double* W22 = W + (r0 + b) * ldw + (r0 + b);
      dgemm_sm90_launch<false>(s, rows2, (int)b, (int)b, L21, ldl, W11, ldw, T21, ldw, 1.0, 0.0, KM_FROM_N, 0, TS_NONE);
      KBO_LAUNCH_CHECK(h);
      dgemm_sm90_launch<false>(s, rows2, (int)b, rows2, W22, ldw, T21, ldw, W21, ldw, -1.0, 0.0, KM_UPTO_M, 0, TS_NONE);
      KBO_LAUNCH_CHECK(h);
    }
  }
  return KBO_OK;
}

// ------------------------------------------------------------------------------------------------
// Events of the multi-stream factorisation below: the handle keeps at least n of them.
static int fit_events(kbo_handle* h, int n) {
  while ((int)h->ev_panel.size() < n) {
    cudaEvent_t e;
    KBO_CUDA(h, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    h->ev_panel.push_back(e);
  }
  return KBO_OK;
}

// ------------------------------------------------------------------------------------------------
// L = chol(K) and (rows of) W = L⁻¹ TOGETHER: the chain on its OWN SMs, the panel below it solved in its shadow.
// The Cholesky of N = 8192 is a chain of 128 single-CTA diagonal blocks with small panel kernels in between — most of the GPU
// idles — and the inverse W_i,<i = −W_ii·(L_i,<i·W_<i,<i) of row panel i needs only the rows of L the Cholesky has already
// finished, so it runs on another stream under the chain.  The dependent chain of a 256-column panel works on its 256×256
// DIAGONAL block only (four single-CTA factorisations, ≤ 3-CTA solves, ≤ 9-CTA updates), and the trailing update LOOKS AHEAD:
// the next column blocks are updated first, so the next panel's chain starts as soon as its own column block is up to date,
// while the rest of the update and the inverse's row panels fill the SMs the chain leaves idle.
// On SMs shared with the updates that chain is slow (KBO_FIT_TRACE, N = 8192): the four single-CTA factorisations of a panel take
// more than twice as long while trailing updates run as on an idle GPU — the update GEMMs hold two 128-register CTAs per SM, i.e.
// the whole register file, so a chain kernel waits until an SM drains (stream priority orders pending CTAs; it does not preempt) —
// and inverting the diagonal block and solving the panel below it with one GEMM against that inverse, on the chain's stream, add
// dependent launches per panel.  Here
//  * a GREEN CONTEXT (CUDA 12.4+) gives the chain stream 8 SMs of its own; everything else runs on the rest.  If the
//    driver cannot split the device the same streams are created unpartitioned and only the second point applies;
//  * the rows below the diagonal block are solved column block by column block on a second stream AS the chain produces the
//    64×64 inverses (four buffers): after the last factorisation only one 64-column solve remains before the trailing update
//    can start.  W_PP (for L⁻¹ and the triangular solves) is formed on a stream of its own, off the critical path.
// Driver entry points come from cudaGetDriverEntryPoint: libkbo links the runtime only.
#include <cuda.h>
namespace {
struct DrvApi {
  CUresult (*DeviceGet)(CUdevice*, int) = nullptr;
  CUresult (*DeviceGetDevResource)(CUdevice, CUdevResource*, CUdevResourceType) = nullptr;
  CUresult (*DevSmResourceSplitByCount)(CUdevResource*, unsigned int*, const CUdevResource*, CUdevResource*, unsigned int, unsigned int) = nullptr;
  CUresult (*DevResourceGenerateDesc)(CUdevResourceDesc*, CUdevResource*, unsigned int) = nullptr;
  CUresult (*GreenCtxCreate)(CUgreenCtx*, CUdevResourceDesc, CUdevice, unsigned int) = nullptr;
  CUresult (*GreenCtxDestroy)(CUgreenCtx) = nullptr;
  CUresult (*GreenCtxStreamCreate)(CUstream*, CUgreenCtx, unsigned int, int) = nullptr;
  bool ok = false;
};
DrvApi load_drv() {
  DrvApi d;
  auto get = [](const char* name, void** fn) {
    cudaDriverEntryPointQueryResult q;
    return cudaGetDriverEntryPoint(name, fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess && *fn;
  };
  d.ok = get("cuDeviceGet", (void**)&d.DeviceGet) && get("cuDeviceGetDevResource", (void**)&d.DeviceGetDevResource) &&
         get("cuDevSmResourceSplitByCount", (void**)&d.DevSmResourceSplitByCount) && get("cuDevResourceGenerateDesc", (void**)&d.DevResourceGenerateDesc) &&
         get("cuGreenCtxCreate", (void**)&d.GreenCtxCreate) && get("cuGreenCtxDestroy", (void**)&d.GreenCtxDestroy) &&
         get("cuGreenCtxStreamCreate", (void**)&d.GreenCtxStreamCreate);
  if (!d.ok) cudaGetLastError();
  return d;
}
const DrvApi& drv() {
  static const DrvApi d = load_drv();
  return d;
}
}  // namespace

// ncu / nsys cannot instrument kernels launched into a green context ("Failed to prepare kernel for profiling" ends the process),
// compute-sanitizer can: with a profiler's injection library mapped the fit keeps the plain streams.
static bool profiler_attached() {
  static const bool attached = [] {
    FILE* f = fopen("/proc/self/maps", "r");
    if (!f) return false;
    char line[1024];
    bool hit = false;
    while (!hit && fgets(line, sizeof line, f))
      hit = strstr(line, "nsight-compute") || strstr(line, "libcuda-injection") || strstr(line, "libnvperf_") || strstr(line, "nsight-systems") ||
            strstr(line, "ToolsInjection");
    fclose(f);
    return hit;
  }();
  return attached;
}

// The streams of the v3 factorisation (roles: kbo_internal.cuh).  partitioned = true asks for the green-context set (created once;
// falls back to the plain set if the driver cannot split the device).
#define FIT_NSTREAMS 10
static int fit_partition(kbo_handle* h, bool partitioned, cudaStream_t (&out)[FIT_NSTREAMS]) {
  int lo = 0, hi = 0;
  KBO_CUDA(h, cudaDeviceGetStreamPriorityRange(&lo, &hi));
  int prio[FIT_NSTREAMS];   // numerically lower = more urgent
  prio[0] = prio[1] = prio[2] = prio[3] = hi;
  for (int k = 2; k <= 4; k++) prio[2 + k] = min(lo, hi + (k - 1));
  prio[7] = max(hi, lo - 1);
  prio[8] = lo;
  prio[9] = hi;
  static const bool off = getenv("KBO_FIT_NO_PARTITION") != nullptr;
  const DrvApi& d = drv();
  if (partitioned && !h->part_tried && !off && d.ok && !profiler_attached()) {
    h->part_tried = true;
    CUdevice dev;
    CUdevResource all, chain, rest;
    unsigned int nb = 1;
    CUdevResourceDesc dc = nullptr, dr = nullptr;
    CUgreenCtx gc = nullptr, gr = nullptr;
    bool ok = d.DeviceGet(&dev, h->device) == CUDA_SUCCESS && d.DeviceGetDevResource(dev, &all, CU_DEV_RESOURCE_TYPE_SM) == CUDA_SUCCESS &&
              d.DevSmResourceSplitByCount(&chain, &nb, &all, &rest, 0, 8) == CUDA_SUCCESS && nb == 1 && rest.sm.smCount >= 64 &&
              d.DevResourceGenerateDesc(&dc, &chain, 1) == CUDA_SUCCESS && d.DevResourceGenerateDesc(&dr, &rest, 1) == CUDA_SUCCESS &&
              d.GreenCtxCreate(&gc, dc, dev, CU_GREEN_CTX_DEFAULT_STREAM) == CUDA_SUCCESS;
    ok = ok && d.GreenCtxCreate(&gr, dr, dev, CU_GREEN_CTX_DEFAULT_STREAM) == CUDA_SUCCESS;
    for (int i = 0; ok && i < FIT_NSTREAMS; i++)
      ok = d.GreenCtxStreamCreate((CUstream*)&h->s3g[i], (i < 2 || i == 9) ? gc : gr, CU_STREAM_NON_BLOCKING, prio[i]) == CUDA_SUCCESS;
    if (ok) {
      h->gctx_chain = gc;
      h->gctx_rest = gr;
      h->part_ok = true;
      static const bool trace = getenv("KBO_FIT_TRACE") != nullptr;
      if (trace) fprintf(stderr, "[kbo fit] SM partition: chain %u SMs, rest %u SMs\n", chain.sm.smCount, rest.sm.smCount);
    } else {
      for (auto& st : h->s3g)
        if (st) {
          cudaStreamDestroy(st);
          st = nullptr;
        }
      if (gc) d.GreenCtxDestroy(gc);
      if (gr) d.GreenCtxDestroy(gr);
      cudaGetLastError();
    }
  }
  if (partitioned && h->part_ok) {
    for (int i = 0; i < FIT_NSTREAMS; i++) out[i] = h->s3g[i];
    return KBO_OK;
  }
  if (!h->s3p[0])
    for (int i = 0; i < FIT_NSTREAMS; i++) KBO_CUDA(h, cudaStreamCreateWithPriority(&h->s3p[i], cudaStreamNonBlocking, prio[i]));
  for (int i = 0; i < FIT_NSTREAMS; i++) out[i] = h->s3p[i];
  return KBO_OK;
}
static void fit_graph_drop(kbo_handle* h);
void kbo_i_fit_partition_free(kbo_handle* h) {
  fit_graph_drop(h);   // its kernel nodes belong to the green contexts below
  if (h->s_cap) cudaStreamDestroy(h->s_cap);
  h->s_cap = nullptr;
  for (auto* set : {&h->s3g, &h->s3p})
    for (auto& st : *set)
      if (st) {
        cudaStreamDestroy(st);
        st = nullptr;
      }
  if (h->gctx_chain) drv().GreenCtxDestroy((CUgreenCtx)h->gctx_chain);
  if (h->gctx_rest) drv().GreenCtxDestroy((CUgreenCtx)h->gctx_rest);
  h->gctx_chain = h->gctx_rest = nullptr;
}

// The Gram matrix's columns past its first `tile0` 64-column tiles (which hold everything the first panel's chain and shadows read).
struct GramRest {
  const double* Xs;
  int N, D, kind;
  double amp, noise;
  double* K;
  int ldk, tile0;
  dim3 grid() const { return dim3((N + 63) / 64 - tile0, (N + 63) / 64); }
};

// Set the graph's Gram node to this fit's arguments: θ (amp, noise) is passed by value, and a replay must not reuse a stale one.
static int gram_node_set(kbo_handle* h, const GramRest& g) {
  void* args[] = {(void*)&g.Xs, (void*)&g.N, (void*)&g.D, (void*)&g.kind, (void*)&g.amp, (void*)&g.noise, (void*)&g.K, (void*)&g.ldk, (void*)&g.tile0};
  cudaKernelNodeParams p = {};
  p.func = (void*)gram_kernel;
  p.gridDim = g.grid();
  p.blockDim = dim3(256);
  p.kernelParams = args;
  KBO_CUDA(h, cudaGraphExecKernelNodeSetParams(h->fit_exec, h->fit_gram_node, &p));
  return KBO_OK;
}

static int fit_graph_replay(kbo_handle* h, cudaStream_t s, const GramRest* gram, bool zsolve) {
  if (gram) KBO_TRY(gram_node_set(h, *gram));
  KBO_CUDA(h, cudaGraphLaunch(h->fit_exec, s));
  h->launches += h->fit_graph_launches;
  h->fit_graph_stat[3]++;
  if (zsolve) h->z_ready = true;
  return KBO_OK;
}

static void fit_graph_drop(kbo_handle* h) {
  if (h->fit_exec) cudaGraphExecDestroy(h->fit_exec);
  if (h->fit_graph) cudaGraphDestroy(h->fit_graph);
  h->fit_exec = nullptr;
  h->fit_graph = nullptr;
  h->fit_gram_node = nullptr;
  h->fit_key.clear();
}

// The factorisation is ~3000 launches, event records and waits over ten streams.  Enqueued call by call, the host is barely ahead
// of the chain: the GPU is idle when a fit starts (every ask ends in a synchronisation), and the chain needs a panel's launches about
// as fast as the host issues them.  So the schedule is captured once into a CUDA graph and replayed with one cudaGraphLaunch for as
// long as what it bakes in holds (the key below): the same kernels, arguments and dependencies, so the same results bit for bit.
// KBO_FIT_TRACE and kbo_debug_fit_stream_path enqueue it call by call.
static int factor_and_invert_v3(kbo_handle* h, double* A, int N, int lda, double* W, int ldw, int* info_dev, cudaStream_t s, int lead,
                                const GramRest* gram = nullptr) {
  // gram (optional): the first column block of A is complete and info / W are zeroed (the caller did both on s); this launches the
  // rest of A.  The chain-side streams then start on the first column block; everything that touches other column blocks waits for
  // the whole matrix.
  // panel width 256: four 64-blocks per panel
  const int OW = 256, NB = KBO_NB, n_panels = (N + OW - 1) / OW;
  // look-ahead depth: column blocks at distance 1..Dn from the panel get their own GEMM (and stream) per panel, the bulk of the
  // trailing update covers the rest — the chain can run Dn − 1 panels ahead of the bulk
  const int Dn = 3;
  // merged bulks: the bulk updates of panels (P, P+1), P even, run as ONE K = 512 GEMM after panel P+1 (a faster GEMM shape, half
  // the passes over the trailing matrix); the even panel covers the column block the merged region misses with one more distance GEMM
  auto kmax_of = [&](int P) { return P % 2 == 0 ? Dn + 1 : Dn; };
  const int CBW = Dn + 2;   // events per column block: distances 1..Dn+1
  // the event layout below: six per panel (+ 2), CBW per column block, 32 singles, and W_PP's per panel
  KBO_TRY(fit_events(h, 6 * n_panels + 2 + (n_panels + 8) * CBW + 32 + n_panels));
  // the SM partition pays when trailing updates big enough to fill the GPU run beside the chain; small factorisations (and any
  // process a profiler is attached to) use plain priority streams
  cudaStream_t st5[FIT_NSTREAMS];
  KBO_TRY(fit_partition(h, N >= 2048, st5));
  const bool partitioned = st5[0] == h->s3g[0] && h->part_ok;
  KBO_TRY(kbo_reserve(h, h->T, (size_t)N * ldw));
  KBO_TRY(kbo_reserve(h, h->T2, (size_t)N * OW));
  KBO_TRY(kbo_reserve(h, h->Linv4, (size_t)NB * NB * 4 * 2));   // two sets of the four block inverses
  const int smem = 2 * NB * (NB + 1) * (int)sizeof(double);
  if (!h->attr_fit) {
    KBO_CUDA(h, cudaFuncSetAttribute(potf2_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    KBO_CUDA(h, cudaFuncSetAttribute(trsm_panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    KBO_CUDA(h, cudaFuncSetAttribute(diag_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    h->attr_fit = true;
  }
  dgemm_sm90_opt_in<true>();
  dgemm_sm90_opt_in<false>();
  // a lazy fit takes alpha from triangular solves: the forward one (z = L⁻¹·yn) is carried along, one panel behind (solve.cu)
  const bool zsolve = lead < N && A == h->K.p && W == h->W.p && N == h->N && lda == h->ld;
  if (zsolve) KBO_TRY(kbo_i_zsolve_reserve(h));
  if (gram && !h->ev_gram) KBO_CUDA(h, cudaEventCreateWithFlags(&h->ev_gram, cudaEventDisableTiming));
  static const bool trace = getenv("KBO_FIT_TRACE") != nullptr;
  const bool graph = !trace && !h->fit_stream_path;
  if (graph && !h->s_cap) KBO_CUDA(h, cudaStreamCreateWithFlags(&h->s_cap, cudaStreamNonBlocking));
  // Everything above allocates or sets attributes; nothing below may (a capture forbids it).
  std::vector<intptr_t> key;
  if (graph) {
    key = {N, lda, ldw, lead, zsolve, gram != nullptr, partitioned, (intptr_t)A, (intptr_t)W, (intptr_t)h->T.p, (intptr_t)h->T2.p, (intptr_t)h->Linv4.p,
           (intptr_t)info_dev, zsolve ? (intptr_t)h->zf.p : 0, zsolve ? (intptr_t)h->yn.p : 0, gram ? gram->tile0 : 0};
    if (h->fit_exec && key == h->fit_key) return fit_graph_replay(h, s, gram, zsolve);
  }
  // the caller's stream, or the capture's origin stream: the graph is then launched on s
  const cudaStream_t so = graph ? h->s_cap : s;
  const cudaEvent_t e_early = gram ? h->ev_gram : nullptr;
  double* T = h->T.p;
  double* T2 = h->T2.p;
  // the 64×64 inverses of a panel's diagonal blocks, two sets: the chain of panel P+1 starts when the NEAR shadow of panel P is done,
  // the far shadow of panel P may still be reading its set (it is done before the chain of panel P+2 can start: that one waits for
  // the near shadow of P+1, which waits for the distance-1 update of P, which waits for the far shadow of P)
  double* Linv_sets = h->Linv4.p;
  cudaStream_t sc = st5[0], sn = st5[1], ss = st5[2], su = st5[3], sb = st5[7], si = st5[8], sw = st5[9];
  cudaStream_t* colS = st5 + 2;   // colS[k]: column-block updates at distance k (colS[1] == su)
  cudaEvent_t* ev_solve = h->ev_panel.data();                     // [n_panels]     the FAR rows below the diagonal block (past the next block) are L
  cudaEvent_t* ev_col = h->ev_panel.data() + n_panels;            // [n_panels + 1] column block P, rows below its diagonal block, carries every earlier update
  cudaEvent_t* ev_chain = h->ev_panel.data() + 2 * n_panels + 1;  // [n_panels]     diagonal block factored, its 64-block inverses in W
  cudaEvent_t* ev_near = h->ev_panel.data() + 3 * n_panels + 1;   // [n_panels + 1] diagonal block P carries every earlier update: the chain may start
  cudaEvent_t* ev_nsolve = h->ev_panel.data() + 4 * n_panels + 2; // [n_panels]     the NEAR rows (the next diagonal block's rows) of panel P are L
  cudaEvent_t* ev_rest = h->ev_panel.data() + 5 * n_panels + 2;   // [n_panels]     trailing update of panel P done
  cudaEvent_t* ev_cb = h->ev_panel.data() + 6 * n_panels + 2;     // [(n_panels + 8) × CBW] column block j updated through distance k
  cudaEvent_t* ev_x = ev_cb + (size_t)(n_panels + 8) * CBW;  // pf[8], tr[8], start, joins
  cudaEvent_t *ev_pf = ev_x, *ev_tr = ev_x + 8, e_start = ev_x[16], *e_join = ev_x + 17;
  std::vector<cudaStream_t> all_streams = {sc, sn, ss, sb, si, sw};
  cudaEvent_t* ev_wpp = ev_x + 32;   // [n_panels] W_PP complete
  for (int k = 1; k <= Dn + 1; k++) all_streams.push_back(colS[k]);
  cudaEvent_t tr[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  std::vector<cudaEvent_t> tp;   // per panel on the chain stream: enqueued | column block ready | diagonal block done
  auto mark = [&]() {
    if (!trace) return;
    cudaEvent_t e;
    cudaEventCreate(&e);
    cudaEventRecord(e, sc);
    tp.push_back(e);
  };
  // KBO_FIT_TRACE=2: a timeline of one panel in eight (when each piece of the schedule finished, ms after the Gram matrix)
  static const bool timeline = trace && atoi(getenv("KBO_FIT_TRACE")) >= 2;
  struct TL { cudaEvent_t e; const char* what; int P; };
  std::vector<TL> tl;
  auto tmark = [&](cudaStream_t st, const char* what, int P) {
    if (!timeline || (P % 8 != 2 && P % 8 != 3)) return;
    cudaEvent_t e;
    cudaEventCreate(&e);
    cudaEventRecord(e, st);
    tl.push_back({e, what, P});
  };
  if (trace) {
    for (auto& e : tr) cudaEventCreate(&e);
    cudaEventRecord(tr[0], s);
  }
  const int launches0 = h->launches;
  if (graph) KBO_CUDA(h, cudaStreamBeginCapture(so, cudaStreamCaptureModeThreadLocal));
  cudaGraphNode_t gram_node = nullptr;
  double host_ms = 0.0;
  const int rc = [&]() -> int {
  if (gram) {
    KBO_CUDA(h, cudaEventRecord(e_early, so));
    gram_kernel<<<gram->grid(), 256, 0, so>>>(gram->Xs, gram->N, gram->D, gram->kind, gram->amp, gram->noise, gram->K, gram->ldk, gram->tile0);
    KBO_LAUNCH_CHECK(h);
    if (graph) {
      cudaStreamCaptureStatus cs;
      const cudaGraphNode_t* deps = nullptr;
      size_t nd = 0;
      KBO_CUDA(h, cudaStreamGetCaptureInfo(so, &cs, nullptr, nullptr, &deps, &nd));
      if (nd != 1) KBO_FAIL(h, KBO_ERR_CUDA, "fit graph capture: the Gram launch is not the origin stream's last node");
      gram_node = deps[0];
    }
  } else {
    KBO_CUDA(h, cudaMemsetAsync(info_dev, 0, 2 * sizeof(int), so));   // h->info: the pivot and who set it
    KBO_CUDA(h, cudaMemsetAsync(W, 0, sizeof(double) * (size_t)N * ldw, so));   // on the caller's stream: all SMs, not the chain's 8
  }
  if (zsolve) KBO_TRY(kbo_i_zsolve_begin(h, so));
  KBO_CUDA(h, cudaEventRecord(e_start, so));
  for (cudaStream_t st : all_streams) {
    const bool chain_side = st == sc || st == sn || st == sw;
    KBO_CUDA(h, cudaStreamWaitEvent(st, e_early && chain_side ? e_early : e_start, 0));
  }
  const int RW = 512;
  int rp0 = 0;
  auto body = [&]() -> int {
    for (int K0 = 0, P = 0; K0 < N; K0 += OW, P++) {
      const int Wd = min(OW, N - K0), rows_t = N - (K0 + Wd);
      const int nblk = (Wd + NB - 1) / NB;
      double* Linv4 = Linv_sets + (size_t)(P & 1) * 4 * NB * NB;
      mark();
      if (P > 0) KBO_CUDA(h, cudaStreamWaitEvent(sc, ev_near[P], 0));
      mark();
      tmark(sc, "chain starts", P);
      // ---- the chain (own SMs): the diagonal block only ------------------------------------------------------------------
      for (int b = 0; b < nblk; b++) {
        const int k = K0 + b * NB, jb = min(NB, N - k);
        double* Li = Linv4 + (size_t)b * NB * NB;
        potf2_inv_kernel<<<1, POTF2_THREADS, smem, sc>>>(A + (size_t)k * lda + k, lda, jb, k, Li, info_dev, W + (size_t)k * ldw + k, ldw);
        KBO_LAUNCH_CHECK(h);
        KBO_CUDA(h, cudaEventRecord(ev_pf[b], sc));
        const int rows_in = K0 + Wd - (k + jb);
        if (rows_in > 0) {
          double* Pn = A + (size_t)(k + jb) * lda + k;
          trsm_panel_kernel<<<(rows_in + 63) / 64, 256, smem, sc>>>(Pn, lda, rows_in, jb, Li, info_dev);
          KBO_LAUNCH_CHECK(h);
          KBO_CUDA(h, cudaEventRecord(ev_tr[b], sc));
          dgemm_sm90_launch<true>(sc, rows_in, rows_in, jb, Pn, lda, Pn, lda, A + (size_t)(k + jb) * lda + (k + jb), lda, -1.0, 1.0, KM_FULL, 0,
                                  TS_LOWER);
          KBO_LAUNCH_CHECK(h);
        }
      }
      mark();
      tmark(sc, "chain done", P);
      KBO_CUDA(h, cudaEventRecord(ev_chain[P], sc));
      // ---- W_PP = L_PP⁻¹ by recursive doubling from the 64-block inverses, on the chain's partition, as the chain produces the blocks:
      // the first pair and the lower-left product after the second block, the second pair and the last product after the fourth
      {
        double* Wpp = W + (size_t)K0 * ldw + K0;
        const double* Lpp = A + (size_t)K0 * lda + K0;
        auto level = [&](int bsz, int r0) -> int {   // W21 = −W22·(L21·W11) for the pair of bsz-blocks at r0
          if (r0 + bsz >= Wd) return KBO_OK;
          const int rows2 = min(bsz, Wd - (r0 + bsz));
          double* T21 = T + (size_t)(K0 + r0 + bsz) * ldw + K0 + r0;
          dgemm_sm90_launch<false>(sw, rows2, bsz, bsz, Lpp + (size_t)(r0 + bsz) * lda + r0, lda, Wpp + (size_t)r0 * ldw + r0, ldw, T21, ldw, 1.0, 0.0,
                                   KM_FROM_N, 0, TS_NONE);
          KBO_LAUNCH_CHECK(h);
          dgemm_sm90_launch<false>(sw, rows2, bsz, rows2, Wpp + (size_t)(r0 + bsz) * ldw + r0 + bsz, ldw, T21, ldw,
                                   Wpp + (size_t)(r0 + bsz) * ldw + r0, ldw, -1.0, 0.0, KM_UPTO_M, 0, TS_NONE);
          KBO_LAUNCH_CHECK(h);
          return KBO_OK;
        };
        if (nblk == 4) {
          KBO_CUDA(h, cudaStreamWaitEvent(sw, ev_pf[1], 0));   // blocks 0, 1 factored (and L[1][0] solved before block 1 was)
          KBO_TRY(level(NB, 0));
          KBO_CUDA(h, cudaStreamWaitEvent(sw, ev_chain[P], 0));
          KBO_TRY(level(NB, 2 * NB));
          KBO_TRY(level(2 * NB, 0));
        } else {
          KBO_CUDA(h, cudaStreamWaitEvent(sw, ev_chain[P], 0));
          for (int bsz = NB; bsz < Wd; bsz *= 2)
            for (int r0 = 0; r0 + bsz < Wd; r0 += 2 * bsz) KBO_TRY(level(bsz, r0));
        }
        KBO_CUDA(h, cudaEventRecord(ev_wpp[P], sw));
      }
      KBO_CUDA(h, cudaStreamWaitEvent(si, ev_wpp[P], 0));
      // ---- the shadows: rows below the diagonal block, one 64-column block behind the chain.  NEAR = the rows of the next diagonal
      // block (on the chain's SMs: 4-CTA kernels that must not queue behind GEMM blocks) — all the next panel's chain waits for is
      // their solve and the 256×256 update of its diagonal block; FAR = the rest, on the big partition ------------------------------
      if (rows_t > 0) {
        const int n_near = min(OW, rows_t), n_far = rows_t - n_near;
        auto shadow = [&](cudaStream_t st, int r0, int nrows, cudaEvent_t ready) -> int {
          if (ready) KBO_CUDA(h, cudaStreamWaitEvent(st, ready, 0));   // these rows of the column block carry the earlier updates too
          for (int b = 0; b < nblk; b++) {
            const int k = K0 + b * NB, jb = min(NB, N - k);
            KBO_CUDA(h, cudaStreamWaitEvent(st, ev_pf[b], 0));
            double* Xb = A + (size_t)r0 * lda + k;
            trsm_panel_kernel<<<(nrows + 63) / 64, 256, smem, st>>>(Xb, lda, nrows, jb, Linv4 + (size_t)b * NB * NB, info_dev);
            KBO_LAUNCH_CHECK(h);
            const int ncols = K0 + Wd - (k + jb);   // the panel's columns right of this block
            if (ncols > 0) {
              KBO_CUDA(h, cudaStreamWaitEvent(st, ev_tr[b], 0));   // L of the diagonal block's rows in this column block (the chain's trsm)
              dgemm_sm90_launch<true>(st, nrows, ncols, jb, Xb, lda, A + (size_t)(k + jb) * lda + k, lda, Xb + jb, lda, -1.0, 1.0, KM_FULL, 0, TS_NONE);
              KBO_LAUNCH_CHECK(h);
            }
          }
          return KBO_OK;
        };
        const int rn = K0 + Wd, rf = rn + n_near;
        // block (P+1, P) got its last update from the previous panel's distance-1 update
        KBO_TRY(shadow(sn, rn, n_near, P > 0 ? ev_col[P] : nullptr));
        KBO_CUDA(h, cudaEventRecord(ev_nsolve[P], sn));
        tmark(sn, "near shadow done", P);
        // What was added to a column block last before this panel's distance-k update: panel P−1's update at distance k+1 if it made
        // one, else the last bulk issued (by panel P−1)
        auto pred_of = [&](int k) -> cudaEvent_t {
          if (P == 0) return nullptr;
          return k + 1 <= kmax_of(P - 1) ? ev_cb[(size_t)(P + k) * CBW + k + 1] : ev_rest[P - 1];
        };
        cudaEvent_t pred1 = pred_of(1);
        // the next diagonal block's own update (after the previous panel's distance-2 update of the same block)
        if (P == 0 && e_early) KBO_CUDA(h, cudaStreamWaitEvent(sn, e_start, 0));   // that block is not in the first column block
        if (pred1) KBO_CUDA(h, cudaStreamWaitEvent(sn, pred1, 0));
        const double* Ln = A + (size_t)rn * lda + K0;
        dgemm_sm90_launch<true>(sn, n_near, n_near, Wd, Ln, lda, Ln, lda, A + (size_t)rn * lda + rn, lda, -1.0, 1.0, KM_FULL, 0, TS_LOWER);
        KBO_LAUNCH_CHECK(h);
        KBO_CUDA(h, cudaEventRecord(ev_near[P + 1], sn));
        tmark(sn, "next diagonal block updated", P);
        if (n_far > 0) {
          // FAR rows: one GEMM against W_PP (L_far = A_far·W_PPᵀ, out of place + copy) instead of seven 64-column steps — under the bulk
          // updates every small kernel of the big partition waits for SM slots (KBO_FIT_TRACE=2 timeline: the seven steps queue,
          // 0.2 for this)
          if (P > 0) KBO_CUDA(h, cudaStreamWaitEvent(ss, ev_col[P], 0));
          KBO_CUDA(h, cudaStreamWaitEvent(ss, ev_wpp[P], 0));
          double* Pf = A + (size_t)rf * lda + K0;
          dgemm_sm90_launch<true>(ss, n_far, Wd, Wd, Pf, lda, W + (size_t)K0 * ldw + K0, ldw, T2, OW, 1.0, 0.0, KM_UPTO_N, 0, TS_NONE);
          KBO_LAUNCH_CHECK(h);
          KBO_CUDA(h, cudaMemcpy2DAsync(Pf, sizeof(double) * lda, T2, sizeof(double) * OW, sizeof(double) * Wd, n_far, cudaMemcpyDeviceToDevice, ss));
          KBO_CUDA(h, cudaEventRecord(ev_solve[P], ss));
          tmark(ss, "far shadow done", P);
          // ---- trailing update.  Distance 1: the next column block's FAR rows (the next panel's far shadow waits for it)
          KBO_CUDA(h, cudaStreamWaitEvent(su, ev_solve[P], 0));
          KBO_CUDA(h, cudaStreamWaitEvent(su, ev_nsolve[P], 0));
          if (pred1) KBO_CUDA(h, cudaStreamWaitEvent(su, pred1, 0));
          const double* Lf = A + (size_t)rf * lda + K0;
          dgemm_sm90_launch<true>(su, n_far, n_near, Wd, Lf, lda, Ln, lda, A + (size_t)rf * lda + rn, lda, -1.0, 1.0, KM_FULL, 0, TS_NONE);
          KBO_LAUNCH_CHECK(h);
          KBO_CUDA(h, cudaEventRecord(ev_col[P + 1], su));
          tmark(su, "distance-1 update done", P);
          // distances 2..kmax_of(P): column block j = P + k, rows from its diagonal block down; each after what was added to that block before
          // (distance k + 1 of the previous panel, or — the farthest — the previous panel's bulk)
          for (int k = 2; k <= kmax_of(P); k++) {
            const int j = P + k, c0 = j * OW;
            if (c0 >= N) break;
            cudaStream_t st = colS[k];
            KBO_CUDA(h, cudaStreamWaitEvent(st, ev_solve[P], 0));
            if (cudaEvent_t pe = pred_of(k)) KBO_CUDA(h, cudaStreamWaitEvent(st, pe, 0));
            const double* Lc = A + (size_t)c0 * lda + K0;
            dgemm_sm90_launch<true>(st, N - c0, min(OW, N - c0), Wd, Lc, lda, Lc, lda, A + (size_t)c0 * lda + c0, lda, -1.0, 1.0, KM_FULL, 0, TS_LOWER);
            KBO_LAUNCH_CHECK(h);
            KBO_CUDA(h, cudaEventRecord(ev_cb[(size_t)j * CBW + k], st));
            tmark(st, k == 2 ? "distance-2 update done" : k == 3 ? "distance-3 update done" : "distance-4 update done", P);
          }
          // the bulk: every column block farther than that, merged for the pair (P−1, P) after the odd panel
          if (P % 2 == 1) {
            const int Pb = P - 1;   // first panel of the bulk
            const int cB = (Pb + kmax_of(Pb) + 1) * OW, Kb = 2 * OW;
            if (cB < N) {
              KBO_CUDA(h, cudaStreamWaitEvent(sb, ev_solve[P], 0));
              const double* Lb = A + (size_t)cB * lda + (size_t)Pb * OW;
              dgemm_sm90_launch<true>(sb, N - cB, N - cB, Kb, Lb, lda, Lb, lda, A + (size_t)cB * lda + cB, lda, -1.0, 1.0, KM_FULL, 0, TS_LOWER);
              KBO_LAUNCH_CHECK(h);
              KBO_CUDA(h, cudaEventRecord(ev_rest[P], sb));
              tmark(sb, "bulk update done", P);
            }
          }
        }
      }
      if (zsolve) {
        KBO_TRY(kbo_i_zsolve_diag(h, K0, Wd, si));
        if (rows_t > 0) {
          KBO_CUDA(h, cudaStreamWaitEvent(si, ev_nsolve[P], 0));
          if (rows_t > OW) KBO_CUDA(h, cudaStreamWaitEvent(si, ev_solve[P], 0));
          KBO_TRY(kbo_i_zsolve_update(h, K0, Wd, si));
        }
      }
      const int done = K0 + Wd;
      if (rp0 < lead && (done - rp0 >= RW || done >= N)) {
        const int P0 = rp0, Pw = done - rp0;
        rp0 = done;
        if (P > 0) {   // rows [P0, done) of L left of this panel: the earlier panels' shadows
          // (panel P − 1 had far rows only if more than one 256-row block lay below it: a graph capture may wait only on events
          // recorded inside it)
          if (N - K0 > OW) KBO_CUDA(h, cudaStreamWaitEvent(si, ev_solve[P - 1], 0));
          KBO_CUDA(h, cudaStreamWaitEvent(si, ev_nsolve[P - 1], 0));
        }
        double* Wrp = W + (size_t)P0 * ldw + P0;
        const double* Lrp = A + (size_t)P0 * lda + P0;
        for (int b = OW; b < Pw; b *= 2)
          for (int r0 = 0; r0 + b < Pw; r0 += 2 * b) {
            const int rows2 = min(b, Pw - (r0 + b));
            double* T21 = T + (size_t)(P0 + r0 + b) * ldw + P0 + r0;
            dgemm_sm90_launch<false>(si, rows2, b, b, Lrp + (size_t)(r0 + b) * lda + r0, lda, Wrp + (size_t)r0 * ldw + r0, ldw, T21, ldw, 1.0, 0.0,
                                     KM_FROM_N, 0, TS_NONE);
            KBO_LAUNCH_CHECK(h);
            dgemm_sm90_launch<false>(si, rows2, b, rows2, Wrp + (size_t)(r0 + b) * ldw + r0 + b, ldw, T21, ldw,
                                     Wrp + (size_t)(r0 + b) * ldw + r0, ldw, -1.0, 0.0, KM_UPTO_M, 0, TS_NONE);
            KBO_LAUNCH_CHECK(h);
          }
        if (P0 > 0) {
          double* Trow = T + (size_t)P0 * ldw;
          dgemm_sm90_launch<false>(si, Pw, P0, P0, A + (size_t)P0 * lda, lda, W, ldw, Trow, ldw, 1.0, 0.0, KM_FROM_N, 0, TS_NONE);
          KBO_LAUNCH_CHECK(h);
          dgemm_sm90_launch<false>(si, Pw, P0, Pw, Wrp, ldw, Trow, ldw, W + (size_t)P0 * ldw, ldw, -1.0, 0.0, KM_UPTO_M, 0, TS_NONE);
          KBO_LAUNCH_CHECK(h);
        }
      }
    }
    return KBO_OK;
  };
  const auto host_t0 = std::chrono::steady_clock::now();
  const int rc = body();
  host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count();
  {
    int j = 0;
    for (cudaStream_t st : all_streams) {
      cudaEventRecord(e_join[j], st);
      cudaStreamWaitEvent(so, e_join[j], 0);
      j++;
    }
  }
  return rc;
  }();
  if (graph) {
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(so, &g);
    if (rc != KBO_OK) {
      if (g) cudaGraphDestroy(g);
      return rc;
    }
    if (e != cudaSuccess) KBO_FAIL(h, KBO_ERR_CUDA, "fit graph capture failed: %s", cudaGetErrorString(e));
    h->fit_graph_stat[0]++;
    h->fit_graph_launches = h->launches - launches0;
    h->launches = launches0;   // counted again by the replay
    // the same schedule over moved buffers keeps its topology: update the executable graph in place; otherwise instantiate anew
    cudaGraphExecUpdateResultInfo ui;
    if (h->fit_exec && (!gram) == (!h->fit_gram_node) && cudaGraphExecUpdate(h->fit_exec, g, &ui) == cudaSuccess) {
      cudaGraphDestroy(g);   // the nodes of the graph fit_exec was instantiated from still address it (fit_gram_node)
      h->fit_graph_stat[1]++;
    } else {
      cudaGetLastError();
      fit_graph_drop(h);
      // node priorities: the chain's streams are the most urgent, and a graph otherwise runs every node at the priority of the
      // stream it is launched into
      const cudaError_t ei = cudaGraphInstantiateWithFlags(&h->fit_exec, g, cudaGraphInstantiateFlagUseNodePriority);
      if (ei != cudaSuccess) {
        cudaGraphDestroy(g);
        h->fit_exec = nullptr;
        KBO_FAIL(h, KBO_ERR_CUDA, "fit graph instantiation failed: %s", cudaGetErrorString(ei));
      }
      h->fit_graph = g;
      h->fit_gram_node = gram_node;
      h->fit_graph_stat[2]++;
    }
    h->fit_key = key;
    return fit_graph_replay(h, s, gram, zsolve);
  }
  if (tr[0]) {
    int j = 1;
    for (cudaStream_t st : {sc, ss, sb, si}) cudaEventRecord(tr[j++], st);
    for (cudaStream_t st : all_streams) cudaStreamSynchronize(st);
    float t[5] = {0, 0, 0, 0, 0};
    for (int i = 1; i < 5; i++) cudaEventElapsedTime(&t[i], tr[0], tr[i]);
    fprintf(stderr, "[kbo fit v3 N=%d%s] chain stream done at %.3f ms, shadow %.3f, bulk update %.3f, inverse %.3f ms\n", N, partitioned ? ", partitioned" : "", t[1],
            t[2], t[3], t[4]);
    double sum[2] = {0, 0};
    for (size_t i = 0; i + 2 < tp.size(); i += 3) {
      float w, d;
      cudaEventElapsedTime(&w, tp[i], tp[i + 1]);
      cudaEventElapsedTime(&d, tp[i + 1], tp[i + 2]);
      sum[0] += w;
      sum[1] += d;
      if ((i / 3) % 8 == 0) fprintf(stderr, "   panel %2d: wait for column block %.3f | diagonal block %.3f ms\n", (int)(i / 3), w, d);
    }
    fprintf(stderr, "   chain totals: waiting %.3f | diagonal blocks %.3f ms; host enqueue of the whole factorisation %.3f ms\n", sum[0], sum[1],
            host_ms);
    if (!tl.empty()) {
      std::vector<std::pair<float, size_t>> order;
      for (size_t i = 0; i < tl.size(); i++) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, tr[0], tl[i].e);
        order.push_back({ms, i});
      }
      std::sort(order.begin(), order.end());
      for (auto& o : order) fprintf(stderr, "   %8.3f ms  panel %2d  %s\n", o.first, tl[o.second].P, tl[o.second].what);
      for (auto& t : tl) cudaEventDestroy(t.e);
    }
    for (auto& e : tr) cudaEventDestroy(e);
    for (auto& e : tp) cudaEventDestroy(e);
  }
  (void)host_ms;
  if (zsolve && rc == KBO_OK) h->z_ready = true;
  return rc;
}

// Test hook: the cached graph's kernel nodes by the context they run in — counts[0] the chain's green context, [1] the rest's,
// [2] any other (the plain streams of an unpartitioned fit, and the Gram launch on the caller's side).  No graph: all zero.
int kbo_i_fit_graph_nodes(kbo_handle* h, int32_t* counts) {
  counts[0] = counts[1] = counts[2] = 0;
  if (!h->fit_graph) return KBO_OK;
  CUresult (*node_params)(CUgraphNode, CUDA_KERNEL_NODE_PARAMS*) = nullptr;
  CUresult (*from_green)(CUcontext*, CUgreenCtx) = nullptr;
  cudaDriverEntryPointQueryResult q;
  KBO_CUDA(h, cudaGetDriverEntryPoint("cuGraphKernelNodeGetParams", (void**)&node_params, cudaEnableDefault, &q));
  KBO_CUDA(h, cudaGetDriverEntryPoint("cuCtxFromGreenCtx", (void**)&from_green, cudaEnableDefault, &q));
  if (!node_params || !from_green) KBO_FAIL(h, KBO_ERR_CUDA, "kbo_debug_fit_graph: driver entry points missing");
  CUcontext chain = nullptr, rest = nullptr;
  if (h->gctx_chain && (from_green(&chain, (CUgreenCtx)h->gctx_chain) != CUDA_SUCCESS || from_green(&rest, (CUgreenCtx)h->gctx_rest) != CUDA_SUCCESS))
    KBO_FAIL(h, KBO_ERR_CUDA, "kbo_debug_fit_graph: cuCtxFromGreenCtx failed");
  size_t n = 0;
  KBO_CUDA(h, cudaGraphGetNodes(h->fit_graph, nullptr, &n));
  std::vector<cudaGraphNode_t> nodes(n);
  KBO_CUDA(h, cudaGraphGetNodes(h->fit_graph, nodes.data(), &n));
  for (cudaGraphNode_t nd : nodes) {
    cudaGraphNodeType t;
    KBO_CUDA(h, cudaGraphNodeGetType(nd, &t));
    if (t != cudaGraphNodeTypeKernel) continue;
    CUDA_KERNEL_NODE_PARAMS p = {};
    if (node_params((CUgraphNode)nd, &p) != CUDA_SUCCESS) KBO_FAIL(h, KBO_ERR_CUDA, "kbo_debug_fit_graph: cuGraphKernelNodeGetParams failed");
    counts[chain && p.ctx == chain ? 0 : rest && p.ctx == rest ? 1 : 2]++;
  }
  return KBO_OK;
}

// ------------------------------------------------------------------------------------------------
// z = W·yn (one warp per row, lower triangle only) ; alpha = Wᵀ·z (one thread per column, coalesced across k)
__global__ void trmv_lower_kernel(const double* __restrict__ W, int N, int ldw, const double* __restrict__ x, double* __restrict__ z) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= N) return;
  double s = 0.0;
#pragma unroll 8   // eight loads in flight per lane; the accumulation order is unchanged
  for (int k = lane; k <= row; k += 32) s = fma(W[(size_t)row * ldw + k], x[k], s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) z[row] = s;
}
// alpha = Wᵀ·z: block (x = 128 columns, y = row slab of 256) accumulates a partial; a second pass sums the slabs in order
__global__ void trmv_lower_t_kernel(const double* __restrict__ W, int N, int ldw, const double* __restrict__ z, double* __restrict__ part) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int i0 = blockIdx.y * 256, i1 = min(N, i0 + 256);
  if (k >= N) return;
  double s = 0.0;
  for (int i = max(i0, k); i < i1; i++) s = fma(W[(size_t)i * ldw + k], z[i], s);
  part[(size_t)blockIdx.y * N + k] = s;
}
__global__ void trmv_t_reduce_kernel(const double* __restrict__ part, int N, int nslab, double* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= N) return;
  double s = 0.0;
  for (int b = 0; b < nslab; b++) s += part[(size_t)b * N + k];
  out[k] = s;
}
// LML = −½ ynᵀalpha − Σ log L_ii − N/2 log 2π  ($SK/_gpr.py:604-618)
__global__ void __launch_bounds__(1024) lml_kernel(const double* __restrict__ L, int N, int ldl, const double* __restrict__ yn,
                                                   const double* __restrict__ alpha, double* __restrict__ scal) {
  __shared__ double r1[1024], r2[1024];
  const int t = threadIdx.x;
  double q = 0.0, ld = 0.0;
  for (int i = t; i < N; i += 1024) {
    q = fma(yn[i], alpha[i], q);
    ld += log(L[(size_t)i * ldl + i]);
  }
  r1[t] = q;
  r2[t] = ld;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (t < o) {
      r1[t] += r1[t + o];
      r2[t] += r2[t + o];
    }
    __syncthreads();
  }
  if (t == 0) {
    scal[S_QUAD] = r1[0];
    scal[S_LOGDET] = r2[0];
    scal[S_LML] = -0.5 * r1[0] - r2[0] - 0.5 * N * 1.8378770664093453;
  }
}

// max |W| (order-independent: bit pattern of a non-negative double is monotone as uint64)
__global__ void absmax_kernel(const double* __restrict__ W, int N, int ldw, unsigned long long* __restrict__ out) {
  double m = 0.0;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < (size_t)N * N; e += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(e / N), c = (int)(e % N);
    if (c <= r) m = fmax(m, fabs(W[(size_t)r * ldw + c]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, (unsigned long long)__double_as_longlong(m));
}
// fp16 hi/lo planes of 2^s·W (s chosen so max|2^s W| ∈ [2^13, 2^14)); zero above the diagonal and in the padding.
__global__ void split_w_kernel(const double* __restrict__ W, int N, int ldw, int Npad, const unsigned long long* __restrict__ amax,
                               __half* __restrict__ Wh, __half* __restrict__ Wl, double* __restrict__ scale_out) {
  const double mx = __longlong_as_double((long long)*amax);
  int e;
  frexp(mx > 0.0 ? mx : 1.0, &e);  // mx = f·2^e, f ∈ [0.5,1)
  const double sc = ldexp(1.0, 14 - e);
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
    scale_out[0] = sc;
    scale_out[1] = 1.0 / sc;
  }
  const int r = blockIdx.y;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < Npad; c += gridDim.x * blockDim.x) {
    double v = (r < N && c <= r) ? W[(size_t)r * ldw + c] * sc : 0.0;
    const __half hi = __double2half(v);
    const __half lo = __double2half(v - (double)__half2float(hi));
    Wh[(size_t)r * Npad + c] = hi;
    Wl[(size_t)r * Npad + c] = lo;
  }
}

__global__ void zero_upper_kernel(double* __restrict__ A, int N, int lda) {
  const int r = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < N && c > r) A[(size_t)r * lda + c] = 0.0;
}
int kbo_i_zero_upper(kbo_handle* h, double* A, int N, int lda, cudaStream_t s) {
  dim3 g((N + 255) / 256, N);
  zero_upper_kernel<<<g, 256, 0, s>>>(A, N, lda);
  KBO_LAUNCH_CHECK(h);
  return KBO_OK;
}

int kbo_i_gram(kbo_handle* h, const double* Xs, int N, int D, int kernel, double amp, double noise, double* K, int ldk, cudaStream_t s) {
  dim3 grid((N + 63) / 64, (N + 63) / 64);
  gram_kernel<<<grid, 256, 0, s>>>(Xs, N, D, kernel, amp, noise, K, ldk, 0);
  KBO_LAUNCH_CHECK(h);
  return KBO_OK;
}
// alpha = Wᵀ(W yn), LML, and (when the tensor-core sweep may be used) the fp16 hi/lo planes of W — shared by fit and append
static int fit_finish(kbo_handle* h, cudaStream_t s, bool new_center) {
  const int N = h->N, ld = h->ld;
  const kbo_params* p = &h->prm;
  static const bool trace = getenv("KBO_FIT_TRACE") != nullptr;
  cudaEvent_t fe[5];
  if (trace) {
    for (auto& e : fe) cudaEventCreate(&e);
    cudaEventRecord(fe[0], s);
  }
  if (!h->w_full) {
    KBO_TRY(kbo_i_alpha_by_solves(h, s));   // alpha = L⁻ᵀ(L⁻¹ yn): two panel solves instead of Wᵀ(W yn)
  } else {
  trmv_lower_kernel<<<(N + 7) / 8, 256, 0, s>>>(h->W.p, N, ld, h->yn.p, h->z.p);
  KBO_LAUNCH_CHECK(h);
  {
    const int nslab = (N + 255) / 256;
    KBO_TRY(kbo_reserve(h, h->T, (size_t)nslab * N));  // the trtri scratch doubles as the slab partials
    dim3 g((N + 127) / 128, nslab);
    trmv_lower_t_kernel<<<g, 128, 0, s>>>(h->W.p, N, ld, h->z.p, h->T.p);
    KBO_LAUNCH_CHECK(h);
    trmv_t_reduce_kernel<<<(N + 127) / 128, 128, 0, s>>>(h->T.p, N, nslab, h->alpha.p);
    KBO_LAUNCH_CHECK(h);
  }
  }
  if (trace) cudaEventRecord(fe[1], s);
  lml_kernel<<<1, 1024, 0, s>>>(h->K.p, N, ld, h->yn.p, h->alpha.p, h->scal.p);
  KBO_LAUNCH_CHECK(h);
  if (trace) cudaEventRecord(fe[2], s);
  if (p->var_mode == KBO_VAR_TC_F16X3 || (p->var_mode == KBO_VAR_AUTO && N > 1024)) {
    h->have_planes = true;
    const int Npad = h->Npad;
    KBO_TRY(kbo_reserve(h, h->Wh, (size_t)Npad * Npad));
    KBO_TRY(kbo_reserve(h, h->Wl, (size_t)Npad * Npad));
    unsigned long long* amax = reinterpret_cast<unsigned long long*>(h->scal.p + S_WAMAX);  // a uint64 in a double slot (same size and alignment)
    KBO_CUDA(h, cudaMemsetAsync(amax, 0, sizeof(unsigned long long), s));
    // with a lazy inverse only the leading w_lead rows of W exist: planes (and their scale) cover those rows; kbo_i_ensure_w redoes both
    const int Nw = h->w_full ? N : h->w_lead;
    absmax_kernel<<<h->sm_count * 4, 256, 0, s>>>(h->W.p, Nw, ld, amax);
    KBO_LAUNCH_CHECK(h);
    dim3 g((Npad + 255) / 256, h->w_full ? Npad : round_up(Nw, 256));
    split_w_kernel<<<g, 256, 0, s>>>(h->W.p, Nw, ld, Npad, amax, h->Wh.p, h->Wl.p, h->scal.p + S_WSCALE);
    KBO_LAUNCH_CHECK(h);
    if (trace) cudaEventRecord(fe[3], s);
    // trial-side operands of the tensor-core K* kernel (alpha changes with every fit / append / rebase)
    KBO_TRY(kbo_i_tc_trials_prep(h, new_center, s));
  } else {
    // auto at N <= 1024 builds no planes.  Planes left by an earlier, larger fit of this handle (a rebase or an append that
    // went back below 1024) hold another history's W at another Npad as row stride: the sweep must not contract with them.
    h->have_planes = false;
    h->ks_ready = false;
    if (trace) cudaEventRecord(fe[3], s);
  }
  if (trace) {
    cudaEventRecord(fe[4], s);
    cudaEventSynchronize(fe[4]);
    float a, b, c, d;
    cudaEventElapsedTime(&a, fe[0], fe[1]);
    cudaEventElapsedTime(&b, fe[1], fe[2]);
    cudaEventElapsedTime(&c, fe[2], fe[3]);
    cudaEventElapsedTime(&d, fe[3], fe[4]);
    fprintf(stderr, "[kbo fit finish N=%d] alpha %.3f ms | lml %.3f ms | planes %.3f ms | trial operands %.3f ms\n", N, a, b, c, d);
    for (auto& e : fe) cudaEventDestroy(e);
  }
  return KBO_OK;
}

int kbo_i_fit(kbo_handle* h, const double* X, const double* y, int N, int D, const kbo_params* p, cudaStream_t s) {
  if (N < 1 || D < 1 || D > 512) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_fit: need N >= 1 and 1 <= D <= 512 (got N=%d D=%d)", N, D);
  if (p->n_length_scale != 1 && p->n_length_scale != D)
    KBO_FAIL(h, KBO_ERR_INVALID, "kbo_fit: n_length_scale must be 1 or D=%d (got %d)", D, p->n_length_scale);
  if (!(p->noise >= 0.0) || !(p->amplitude > 0.0)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_fit: amplitude must be > 0 and noise >= 0");
  if (p->var_mode < KBO_VAR_F64 || p->var_mode > KBO_VAR_AUTO) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_fit: unknown var_mode %d", p->var_mode);
  if (p->kernel != KBO_KERNEL_RBF && p->kernel != KBO_KERNEL_MATERN52) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_fit: unknown kernel %d", p->kernel);
  for (int d = 0; d < p->n_length_scale; d++)
    if (!(p->length_scale[d] > 0.0)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_fit: length_scale[%d] must be > 0", d);
  h->fitted = false;
  h->have_planes = false;
  h->ks_ready = false;
  h->N = N;
  h->D = D;
  h->ld = round_up(N, 64);
  h->Npad = round_up(N, 256);
  h->prm = *p;
  h->inv_ls.resize(p->n_length_scale);
  for (int d = 0; d < p->n_length_scale; d++) h->inv_ls[d] = 1.0 / p->length_scale[d];
  h->prm.length_scale = nullptr;
  const int ld = h->ld;
  KBO_TRY(kbo_reserve(h, h->d_inv_ls, 512));
  // rows are reserved up to the pitch (ld = N rounded up to 64) so kbo_fit_append can add trials in place until the pitch is
  // full; past it the caller refits.  Only ld bounds how many appended rows stack on one factorisation: kbo_fit_rebase keeps ld
  // and lowers N, so after a rebase to n_keep another ld − n_keep rows (the dropped rows plus up to 63) can be appended, each
  // l = W·k formed with the W rows of the appends before it.  Measured on an H100 80GB HBM3 at 511 stacked rows and noise 1e-6,
  // their backward errors stay below a fresh fit's worst tile (tests/test_gpu_append_scale.py).
  KBO_TRY(kbo_reserve(h, h->Xs, (size_t)ld * D));
  KBO_TRY(kbo_reserve(h, h->XsT, (size_t)D * ld));
  KBO_TRY(kbo_reserve(h, h->nx, ld));
  KBO_TRY(kbo_reserve(h, h->yn, ld));
  KBO_TRY(kbo_reserve(h, h->yraw, ld));
  KBO_TRY(kbo_reserve(h, h->K, (size_t)ld * ld));
  KBO_TRY(kbo_reserve(h, h->W, (size_t)ld * ld));
  KBO_TRY(kbo_reserve(h, h->alpha, ld));
  KBO_TRY(kbo_reserve(h, h->z, ld));
  KBO_CUDA(h, kbo_copy(h->yraw.p, y, N, cudaMemcpyDeviceToDevice, s));
  KBO_TRY(kbo_reserve(h, h->scal, 16));
  KBO_TRY(kbo_reserve(h, h->info, 4));
  // inv_ls is tiny: stage through pageable memory is fine, but keep it async-safe by copying from the vector we own
  KBO_CUDA(h, kbo_copy(h->d_inv_ls.p, h->inv_ls.data(), h->inv_ls.size(), cudaMemcpyHostToDevice, s));
  prep_x_kernel<<<(N + 127) / 128, 128, 0, s>>>(X, N, D, h->d_inv_ls.p, p->n_length_scale, h->Xs.p, h->XsT.p, ld, h->nx.p);
  KBO_LAUNCH_CHECK(h);
  prep_y_kernel<<<1, 1024, 0, s>>>(y, N, p->normalize_y, h->yn.p, h->scal.p);
  KBO_LAUNCH_CHECK(h);
  // KBO_FIT_TRACE=1: per-phase CUDA-event timings on stderr (debug aid; adds stream syncs)
  static const bool trace = getenv("KBO_FIT_TRACE") != nullptr;
  cudaEvent_t te[6];
  if (trace)
    for (auto& e : te) cudaEventCreate(&e);
  if (trace) cudaEventRecord(te[0], s);
  // the one-stream reference: Cholesky, then recursive-doubling inverse (kbo_potrf, kbo_trtri)
  static const bool serial = getenv("KBO_FIT_SERIAL") != nullptr;
  // v3 starts on the first column block of the Gram matrix: the first 8 64-column tiles are launched here, the rest by v3
  const bool early = !serial && N >= 1024;
  const GramRest gram_rest{h->Xs.p, N, D, p->kernel, p->amplitude, p->noise, h->K.p, ld, 8};
  if (early) {
    KBO_CUDA(h, cudaMemsetAsync(h->info.p, 0, sizeof *h->info.p * 2, s));
    KBO_CUDA(h, cudaMemsetAsync(h->W.p, 0, sizeof *h->W.p * N * ld, s));
    gram_kernel<<<dim3(gram_rest.tile0, (N + 63) / 64), 256, 0, s>>>(h->Xs.p, N, D, p->kernel, p->amplitude, p->noise, h->K.p, ld, 0);
    KBO_LAUNCH_CHECK(h);
  } else {
    KBO_TRY(kbo_i_gram(h, h->Xs.p, N, D, p->kernel, p->amplitude, p->noise, h->K.p, ld, s));
  }
  if (trace) cudaEventRecord(te[1], s);
  h->w_full = true;
  h->w_lead = N;
  if (serial) {
    KBO_CUDA(h, cudaMemsetAsync(h->info.p, 0, sizeof *h->info.p * 2, s));   // kbo_i_potrf resets only the pivot
    KBO_TRY(kbo_i_potrf(h, h->K.p, N, ld, h->info.p, s));
    if (trace) cudaEventRecord(te[2], s);
    KBO_TRY(kbo_i_trtri(h, h->K.p, N, ld, h->W.p, ld, s));
  } else {
    {
      // Lazy inverse: a tensor-core fit whose sweeps will prune (kbo_set_rank_prefix) forms only the rows of W the pruning pass
      // contracts with — the first 512·P1 — and leaves the rest to kbo_i_ensure_w, which runs if something asks for all of W.
      int lead = N;
      const bool planes = p->var_mode == KBO_VAR_TC_F16X3 || (p->var_mode == KBO_VAR_AUTO && N > 1024);
      if (h->lazy_w && planes && h->rank_tc && h->rank_prefix != 0 && h->tc_fast && D <= 128) {
        const int P1 = kbo_prefix_pairs(h);
        if (P1 >= 1 && P1 < kbo_tile_pairs(h->Npad) && P1 * 512 + 512 <= N) lead = round_up(P1 * 512, 512);
      }
      KBO_TRY(factor_and_invert_v3(h, h->K.p, N, ld, h->W.p, ld, h->info.p, s, lead, early ? &gram_rest : nullptr));
      h->w_lead = lead < N ? lead : N;
      h->w_full = lead >= N;
    }
    if (trace) cudaEventRecord(te[2], s);
  }
  if (trace) cudaEventRecord(te[3], s);
  KBO_TRY(fit_finish(h, s, true));
  if (trace) {
    cudaEventRecord(te[4], s);
    cudaEventSynchronize(te[4]);
    float g, c, t, r;
    cudaEventElapsedTime(&g, te[0], te[1]);
    cudaEventElapsedTime(&c, te[1], te[2]);
    cudaEventElapsedTime(&t, te[2], te[3]);
    cudaEventElapsedTime(&r, te[3], te[4]);
    fprintf(stderr, "[kbo fit N=%d] gram %.3f ms | potrf %.3f ms | trtri %.3f ms | alpha+lml+split %.3f ms\n", N, g, c, t, r);
    for (auto& e : te) cudaEventDestroy(e);
  }
  h->fitted = true;
  return KBO_OK;
}

// ------------------------------------------------------------------------------------------------
// The rows of W a lazy fit left out (and the full fp16 planes): row panels [w_lead, N) of W_i,<i = −W_ii·(L_i,<i·W_<i,<i), the
// 512-wide diagonal blocks first.  What the lazy fit saved; paid only by callers that need all of W.
int kbo_i_ensure_w(kbo_handle* h, cudaStream_t s) {
  if (!h->fitted && !h->w_lead) return KBO_OK;
  if (h->w_full) return KBO_OK;
  const int N = h->N, ld = h->ld, OW = 256, RW = 512;
  double* A = h->K.p;
  double* W = h->W.p;
  KBO_TRY(kbo_reserve(h, h->T, (size_t)N * ld));
  double* T = h->T.p;
  for (int P0 = h->w_lead; P0 < N; P0 += RW) {
    const int Pw = min(RW, N - P0);
    double* Wrp = W + (size_t)P0 * ld + P0;
    const double* Lrp = A + (size_t)P0 * ld + P0;
    for (int b = OW; b < Pw; b *= 2)
      for (int r0 = 0; r0 + b < Pw; r0 += 2 * b) {
        const int rows2 = min(b, Pw - (r0 + b));
        double* T21 = T + (size_t)(P0 + r0 + b) * ld + P0 + r0;
        dgemm_sm90_launch<false>(s, rows2, b, b, Lrp + (size_t)(r0 + b) * ld + r0, ld, Wrp + (size_t)r0 * ld + r0, ld, T21, ld, 1.0, 0.0, KM_FROM_N, 0,
                                 TS_NONE);
        KBO_LAUNCH_CHECK(h);
        dgemm_sm90_launch<false>(s, rows2, b, rows2, Wrp + (size_t)(r0 + b) * ld + r0 + b, ld, T21, ld, Wrp + (size_t)(r0 + b) * ld + r0, ld, -1.0,
                                 0.0, KM_UPTO_M, 0, TS_NONE);
        KBO_LAUNCH_CHECK(h);
      }
    if (P0 > 0) {
      double* Trow = T + (size_t)P0 * ld;
      dgemm_sm90_launch<false>(s, Pw, P0, P0, A + (size_t)P0 * ld, ld, W, ld, Trow, ld, 1.0, 0.0, KM_FROM_N, 0, TS_NONE);
      KBO_LAUNCH_CHECK(h);
      dgemm_sm90_launch<false>(s, Pw, P0, Pw, Wrp, ld, Trow, ld, W + (size_t)P0 * ld, ld, -1.0, 0.0, KM_UPTO_M, 0, TS_NONE);
      KBO_LAUNCH_CHECK(h);
    }
  }
  h->w_full = true;
  h->w_lead = N;
  if (h->have_planes) {
    const int Npad = h->Npad;
    unsigned long long* amax = reinterpret_cast<unsigned long long*>(h->scal.p + S_WAMAX);  // a uint64 in a double slot (same size and alignment)
    KBO_CUDA(h, cudaMemsetAsync(amax, 0, sizeof(unsigned long long), s));
    absmax_kernel<<<h->sm_count * 4, 256, 0, s>>>(h->W.p, N, ld, amax);
    KBO_LAUNCH_CHECK(h);
    dim3 g((Npad + 255) / 256, Npad);
    split_w_kernel<<<g, 256, 0, s>>>(h->W.p, N, ld, Npad, amax, h->Wh.p, h->Wl.p, h->scal.p + S_WSCALE);
    KBO_LAUNCH_CHECK(h);
  }
  return KBO_OK;
}

// ------------------------------------------------------------------------------------------------
// kbo_lml_batch: log-marginal likelihood of G hyper-parameter settings at once ($SK/_gpr.py:604-618 per θ; the loop being
// replaced is sklearn's optimiser evaluating them one after another, :299-339, :658-667; SURVEY.md §8(f)1).
// The Cholesky of a few-thousand-trial history is a CHAIN of single-CTA diagonal blocks — most of the GPU idles — so the G
// factorisations are enqueued on G streams and hide each other's latency: 8 θ at N = 2048 cost about as much as 2 fits.
// Per θ only what the LML needs is computed: Gram, Cholesky, z = L⁻¹·yn by blocked forward substitution (no inverse, no
// alpha: ynᵀK⁻¹yn = zᵀz), Σ log L_ii.
__global__ void __launch_bounds__(256)
trsv_lml_kernel(const double* __restrict__ L, int N, int ldl, const double* __restrict__ yn, const int* __restrict__ info, double* __restrict__ out) {
  extern __shared__ double zs[];            // z, N doubles
  __shared__ double rhs[KBO_NB];
  __shared__ double Lb[KBO_NB][KBO_NB + 1];   // the diagonal block: the substitution below is a dependent chain, keep it off global memory
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  if (*info != 0) {
    if (t == 0) out[0] = -INFINITY;
    return;
  }
  double logdet = 0.0, quad = 0.0;
  for (int b0 = 0; b0 < N; b0 += KBO_NB) {
    const int jb = min(KBO_NB, N - b0);
    // rhs_r = yn_r − Σ_{k < b0} L[r][k]·z[k]: one warp per 8 rows, lanes stride the columns, fixed-order butterfly
    for (int rr = warp; rr < jb; rr += 8) {
      const double* row = L + (size_t)(b0 + rr) * ldl;
      double a = 0.0;
      for (int k = lane; k < b0; k += 32) a = fma(row[k], zs[k], a);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      if (lane == 0) rhs[rr] = yn[b0 + rr] - a;
    }
    for (int e = t; e < KBO_NB * KBO_NB; e += 256) {
      const int r = e >> 6, c = e & 63;
      Lb[r][c] = (r < jb && c <= r) ? L[(size_t)(b0 + r) * ldl + b0 + c] : 0.0;
    }
    __syncthreads();
    if (warp == 0) {   // forward substitution inside the 64-block: lanes own rows lane and lane+32
      double r0 = lane < jb ? rhs[lane] : 0.0, r1 = lane + 32 < jb ? rhs[lane + 32] : 0.0;
      for (int c = 0; c < jb; c++) {
        const double lcc = Lb[c][c];
        const double zc = __shfl_sync(0xffffffffu, c < 32 ? r0 : r1, c & 31) / lcc;
        if (lane == (c & 31)) {
          if (c < 32) r0 = zc; else r1 = zc;
        }
        if (lane > c && lane < jb) r0 = fma(-Lb[lane][c], zc, r0);
        if (lane + 32 > c && lane + 32 < jb) r1 = fma(-Lb[lane + 32][c], zc, r1);
        if (lane == 0) {
          logdet += log(lcc);
          quad = fma(zc, zc, quad);
        }
      }
      if (lane < jb) zs[b0 + lane] = r0;
      if (lane + 32 < jb) zs[b0 + lane + 32] = r1;
    }
    __syncthreads();
  }
  if (t == 0) out[0] = -0.5 * quad - logdet - 0.5 * N * 1.8378770664093453;
}

struct LmlLane {
  cudaStream_t s = nullptr;
  DevBuf<double> K, Xs, XsT, nx, inv_ls, Linv, out;
  DevBuf<int> info;
  DevBuf<double> W, T, z, alpha, part;   // kbo_lml_grad_batch only: W = L⁻¹, the trtri / transpose scratch, alpha, gradient partials
};

// Checks shared by kbo_lml_batch and kbo_lml_grad_batch; makes G lanes and the kernels' shared-memory opt-ins.
static int lml_lanes_prepare(kbo_handle* h, const char* name, int N, int D, int G, const kbo_params* params, std::vector<LmlLane>*& lanes) {
  if (N < 1 || D < 1 || D > 512 || G < 1 || G > 64) KBO_FAIL(h, KBO_ERR_INVALID, "%s: need N >= 1, 1 <= D <= 512, 1 <= G <= 64", name);
  for (int g = 0; g < G; g++) {
    const kbo_params* p = params + g;
    if (!p->length_scale || (p->n_length_scale != 1 && p->n_length_scale != D)) KBO_FAIL(h, KBO_ERR_INVALID, "%s: theta %d: n_length_scale must be 1 or D", name, g);
    if (!(p->noise >= 0.0) || !(p->amplitude > 0.0)) KBO_FAIL(h, KBO_ERR_INVALID, "%s: theta %d: amplitude must be > 0 and noise >= 0", name, g);
    if (p->kernel != KBO_KERNEL_RBF && p->kernel != KBO_KERNEL_MATERN52) KBO_FAIL(h, KBO_ERR_INVALID, "%s: theta %d: unknown kernel", name, g);
    for (int d = 0; d < p->n_length_scale; d++)
      if (!(p->length_scale[d] > 0.0)) KBO_FAIL(h, KBO_ERR_INVALID, "%s: theta %d: length_scale[%d] must be > 0", name, g, d);
  }
  if ((int)sizeof(double) * N > 200 * 1024) KBO_FAIL(h, KBO_ERR_INVALID, "%s: N <= 25600 supported (got %d)", name, N);
  lanes = (std::vector<LmlLane>*)h->lml_lanes;
  if (!lanes) h->lml_lanes = lanes = new std::vector<LmlLane>();
  if ((int)lanes->size() < G) lanes->resize(G);
  const int smem_pf = 2 * KBO_NB * (KBO_NB + 1) * (int)sizeof(double);
  if (!h->attr_fit) {
    KBO_CUDA(h, cudaFuncSetAttribute(potf2_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_pf));
    KBO_CUDA(h, cudaFuncSetAttribute(trsm_panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_pf));
    KBO_CUDA(h, cudaFuncSetAttribute(diag_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_pf));
    h->attr_fit = true;
  }
  return KBO_OK;
}

// y statistics are θ-independent: normalise once on the caller's stream, which every lane then waits for
static int lml_lanes_prep_y(kbo_handle* h, const double* y_dev, int N, int ld, int normalize_y, cudaStream_t s) {
  KBO_TRY(kbo_reserve(h, h->lml_yn, ld));
  KBO_TRY(kbo_reserve(h, h->lml_scal, 16));
  prep_y_kernel<<<1, 1024, 0, s>>>(y_dev, N, normalize_y, h->lml_yn.p, h->lml_scal.p);
  KBO_LAUNCH_CHECK(h);
  if (!h->lml_ev) KBO_CUDA(h, cudaEventCreateWithFlags(&h->lml_ev, cudaEventDisableTiming));
  KBO_CUDA(h, cudaEventRecord(h->lml_ev, s));
  return KBO_OK;
}

// One θ on its lane: X/ℓ, Gram, Cholesky in L.K (pivot in L.info).
static int lml_lane_factor(kbo_handle* h, LmlLane& L, const double* X_dev, int N, int D, int ld, const kbo_params* p, std::vector<double>& inv) {
  if (!L.s) KBO_CUDA(h, cudaStreamCreateWithFlags(&L.s, cudaStreamNonBlocking));
  KBO_TRY(kbo_reserve(h, L.K, (size_t)ld * ld));
  KBO_TRY(kbo_reserve(h, L.Xs, (size_t)ld * D));
  KBO_TRY(kbo_reserve(h, L.XsT, (size_t)D * ld));
  KBO_TRY(kbo_reserve(h, L.nx, ld));
  KBO_TRY(kbo_reserve(h, L.inv_ls, 512));
  KBO_TRY(kbo_reserve(h, L.Linv, KBO_NB * KBO_NB));
  KBO_TRY(kbo_reserve(h, L.info, 4));
  KBO_TRY(kbo_reserve(h, L.out, 2));
  KBO_CUDA(h, cudaStreamWaitEvent(L.s, h->lml_ev, 0));
  for (int d = 0; d < p->n_length_scale; d++) inv[d] = 1.0 / p->length_scale[d];
  KBO_CUDA(h, kbo_copy(L.inv_ls.p, inv.data(), p->n_length_scale, cudaMemcpyHostToDevice, L.s));   // pageable: staged before return
  prep_x_kernel<<<(N + 127) / 128, 128, 0, L.s>>>(X_dev, N, D, L.inv_ls.p, p->n_length_scale, L.Xs.p, L.XsT.p, ld,
                                                 L.nx.p);
  KBO_LAUNCH_CHECK(h);
  KBO_TRY(kbo_i_gram(h, L.Xs.p, N, D, p->kernel, p->amplitude, p->noise, L.K.p, ld, L.s));
  KBO_TRY(potrf_impl(h, L.K.p, N, ld, L.info.p, L.s, [](int, int) { return (int)KBO_OK; }, L.Linv.p));
  return KBO_OK;
}

int kbo_i_lml_batch(kbo_handle* h, const double* X_dev, const double* y_dev, int N, int D, int G, const kbo_params* params, double* lml_host,
                    int32_t* info_host, cudaStream_t s) {
  std::vector<LmlLane>* lanes = nullptr;
  KBO_TRY(lml_lanes_prepare(h, "kbo_lml_batch", N, D, G, params, lanes));
  const int ld = round_up(N, 64);
  const int zs_bytes = (int)sizeof(double) * N;
  KBO_CUDA(h, cudaFuncSetAttribute(trsv_lml_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, zs_bytes));
  KBO_TRY(lml_lanes_prep_y(h, y_dev, N, ld, params[0].normalize_y, s));
  std::vector<double> inv(512);
  for (int g = 0; g < G; g++) {
    LmlLane& L = (*lanes)[g];
    KBO_TRY(lml_lane_factor(h, L, X_dev, N, D, ld, params + g, inv));
    trsv_lml_kernel<<<1, 256, zs_bytes, L.s>>>(L.K.p, N, ld, h->lml_yn.p, L.info.p, L.out.p);
    KBO_LAUNCH_CHECK(h);
  }
  for (int g = 0; g < G; g++) {
    LmlLane& L = (*lanes)[g];
    int inf = 0;
    KBO_CUDA(h, kbo_copy(lml_host + g, L.out.p, 1, cudaMemcpyDeviceToHost, L.s));
    KBO_CUDA(h, kbo_copy(&inf, L.info.p, 1, cudaMemcpyDeviceToHost, L.s));
    KBO_CUDA(h, cudaStreamSynchronize(L.s));
    if (info_host) info_host[g] = inf;
  }
  return KBO_OK;
}

// ------------------------------------------------------------------------------------------------
// kbo_lml_grad_batch: LML and ∂LML/∂θ of G settings over one history — what sklearn's L-BFGS-B asks of
// log_marginal_likelihood(theta, eval_gradient=True) once per start and iteration ($SK/_gpr.py:541-655), for the starts of a
// restart search in lockstep.  Per θ on its lane stream: Gram, Cholesky (as kbo_lml_batch), W = L⁻¹ (kbo_i_trtri with the
// lane's scratch), alpha = Wᵀ(W·yn) and the LML (the fit's kernels), then K⁻¹ and the gradient (kbo_i_lml_grad_from_w, the
// kernels kbo_lml_grad runs).  Every reduction has a fixed order and nothing is shared between lanes, so a θ's result does not
// depend on the batch it is in.  Lane memory: L / K⁻¹, W and the scratch plane, 3·ld² doubles, plus the small vectors.
size_t kbo_i_lml_grad_lane_bytes(int N, int D, int P) {
  const size_t ld = (size_t)round_up(N, 64), nb = (size_t)(N + 63) / 64;
  return sizeof(double) * (3 * ld * ld + 2 * ld * D + 3 * ld + nb * nb * (2 + P) + (2 + P) + KBO_NB * KBO_NB + 512 + 16) + sizeof(int) * 4;
}

int kbo_i_lml_grad_batch(kbo_handle* h, const double* X_dev, const double* y_dev, int N, int D, int G, const kbo_params* params, double* lml_host,
                         double* grad_host, int32_t* info_host, cudaStream_t s) {
  std::vector<LmlLane>* lanes = nullptr;
  KBO_TRY(lml_lanes_prepare(h, "kbo_lml_grad_batch", N, D, G, params, lanes));
  const int P = params[0].n_length_scale;
  for (int g = 1; g < G; g++)
    if (params[g].n_length_scale != P) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_lml_grad_batch: theta %d: every theta needs the same n_length_scale", g);
  const size_t need = (size_t)G * kbo_i_lml_grad_lane_bytes(N, D, P);   // checked before anything is allocated or launched
  if (need > h->scratch_limit)
    KBO_FAIL(h, KBO_ERR_INVALID, "kbo_lml_grad_batch: %d thetas at N = %d, D = %d need %zu bytes of lane memory, over the scratch limit of %llu bytes",
             G, N, D, need, (unsigned long long)h->scratch_limit);
  const int ld = round_up(N, 64), nb = (N + 63) / 64, ncomp = 2 + P, nslab = (N + 255) / 256;
  KBO_TRY(lml_lanes_prep_y(h, y_dev, N, ld, params[0].normalize_y, s));
  std::vector<double> inv(512);
  for (int g = 0; g < G; g++) {
    LmlLane& L = (*lanes)[g];
    const kbo_params* p = params + g;
    KBO_TRY(kbo_reserve(h, L.W, (size_t)ld * ld));
    KBO_TRY(kbo_reserve(h, L.T, (size_t)ld * ld));
    KBO_TRY(kbo_reserve(h, L.z, ld));
    KBO_TRY(kbo_reserve(h, L.alpha, ld));
    KBO_TRY(kbo_reserve(h, L.part, (size_t)nb * nb * ncomp + ncomp));
    KBO_TRY(kbo_reserve(h, L.out, 16));   // the LML kernel writes S_QUAD, S_LOGDET, S_LML
    KBO_TRY(lml_lane_factor(h, L, X_dev, N, D, ld, p, inv));
    double *K = L.K.p, *W = L.W.p, *T = L.T.p, *alpha = L.alpha.p, *out = L.out.p;
    KBO_TRY(kbo_i_trtri(h, K, N, ld, W, ld, L.s, T));
    trmv_lower_kernel<<<(N + 7) / 8, 256, 0, L.s>>>(W, N, ld, h->lml_yn.p, L.z.p);
    KBO_LAUNCH_CHECK(h);
    trmv_lower_t_kernel<<<dim3((N + 127) / 128, nslab), 128, 0, L.s>>>(W, N, ld, L.z.p, T);   // slab partials in the scratch plane
    KBO_LAUNCH_CHECK(h);
    trmv_t_reduce_kernel<<<(N + 127) / 128, 128, 0, L.s>>>(T, N, nslab, alpha);
    KBO_LAUNCH_CHECK(h);
    lml_kernel<<<1, 1024, 0, L.s>>>(K, N, ld, h->lml_yn.p, alpha, out);   // LML in out[S_LML]; L is not read after this
    KBO_LAUNCH_CHECK(h);
    double* part = L.part.p;
    KBO_TRY(kbo_i_lml_grad_from_w(h, L.Xs.p, N, D, p->kernel, p->amplitude, p->noise, alpha, W, T, K, ld, P, part,
                                  part + (size_t)nb * nb * ncomp, L.s));
  }
  for (int g = 0; g < G; g++) {
    LmlLane& L = (*lanes)[g];
    int inf = 0;
    double lml = 0.0;
    double* gh = grad_host + (size_t)g * ncomp;
    KBO_CUDA(h, kbo_copy(&lml, L.out.p + S_LML, 1, cudaMemcpyDeviceToHost, L.s));
    KBO_CUDA(h, kbo_copy(gh, L.part.p + (size_t)nb * nb * ncomp, ncomp, cudaMemcpyDeviceToHost, L.s));
    KBO_CUDA(h, kbo_copy(&inf, L.info.p, 1, cudaMemcpyDeviceToHost, L.s));
    KBO_CUDA(h, cudaStreamSynchronize(L.s));
    if (inf != 0) {   // the lane ran on a partly factored L: nothing it computed after the pivot means anything
      lml = -INFINITY;
      for (int c = 0; c < ncomp; c++) gh[c] = 0.0;
    }
    lml_host[g] = lml;
    if (info_host) info_host[g] = inf;
  }
  return KBO_OK;
}

void kbo_i_lml_batch_free(kbo_handle* h) {
  auto* lanes = (std::vector<LmlLane>*)h->lml_lanes;
  if (!lanes) return;
  for (auto& L : *lanes)
    if (L.s) cudaStreamDestroy(L.s);
  delete lanes;
  h->lml_lanes = nullptr;
}

// ------------------------------------------------------------------------------------------------
// kbo_fit_append: one more trial at the fitted θ without refactorising (SURVEY.md §8(f)2, constant-liar asks and the
// steady state of a Katib experiment, where each request adds a trial or two to a history the service already holds).
// With W = L⁻¹ resident the bordered factorisation is three matrix-vector passes:
//   k = amp·k(X, x) ;  l = W k ;  d = sqrt(amp + noise − l·l) ;  L ← [[L,0],[lᵀ,d]] ;  W ← [[W,0],[−(Wᵀl)ᵀ/d, 1/d]]
// followed by the same finish as a fit (y statistics change with every trial, so yn, alpha and the LML are recomputed).
__global__ void append_x_kernel(const double* __restrict__ x, int D, const double* __restrict__ inv_ls, int n_ls, double* __restrict__ Xs,
                                double* __restrict__ XsT, int ldx, double* __restrict__ nx, int row, double y, double* __restrict__ yraw) {
  for (int d = threadIdx.x; d < D; d += 256) {
    const double v = x[d] * inv_ls[n_ls == 1 ? 0 : d];
    Xs[(size_t)row * D + d] = v;
    XsT[(size_t)d * ldx + row] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;   // same left-to-right fma chain over d as prep_x_kernel: nx is bit-identical to a refit's
    for (int d = 0; d < D; d++) {
      const double v = Xs[(size_t)row * D + d];
      t = fma(v, v, t);
    }
    nx[row] = t;
    yraw[row] = y;
  }
}
// k_j = amp·k(x_row, x_j) for j < row, written into row `row` of the K/L buffer (exact differences, like gram_kernel)
__global__ void gram_row_kernel(const double* __restrict__ Xs, int D, int row, int kind, double amp, double* __restrict__ Krow) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= row) return;
  double d2 = 0.0;
  for (int d = 0; d < D; d++) {
    const double df = Xs[(size_t)row * D + d] - Xs[(size_t)j * D + d];
    d2 = fma(df, df, d2);
  }
  Krow[j] = amp * kbo_kernel_exact(d2, kind);
}
// after l = W k: d² = amp + noise − Σ l², L row ← (l, d, 0…), and the info flag if the bordered matrix is not PD
__global__ void __launch_bounds__(1024) append_diag_kernel(const double* __restrict__ l, int row, int ld, double knn, double* __restrict__ Lrow,
                                                          double* __restrict__ dinv, int* __restrict__ info) {
  __shared__ double red[1024];
  const int t = threadIdx.x;
  double a = 0.0;
  for (int j = t; j < row; j += 1024) a = fma(l[j], l[j], a);
  red[t] = a;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (t < o) red[t] += red[t + o];
    __syncthreads();
  }
  const double d2 = knn - red[0];
  const bool ok = d2 > 0.0;
  const double d = ok ? sqrt(d2) : 1.0;
  for (int j = t; j < ld; j += 1024) Lrow[j] = j < row ? l[j] : (j == row ? d : 0.0);
  if (t == 0) {
    *dinv = 1.0 / d;
    if (!ok && info[0] == 0) {
      info[0] = row + 1;
      info[1] = 1;   // the rows above are intact: a rebase below this row recovers (kbo_i_fit_rebase)
    }
  }
}
// W row ← (−(Wᵀl)/d, 1/d, 0…)
__global__ void append_wrow_kernel(const double* __restrict__ wtl, int row, int ld, const double* __restrict__ dinv, double* __restrict__ Wrow) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= ld) return;
  const double di = *dinv;
  Wrow[j] = j < row ? -wtl[j] * di : (j == row ? di : 0.0);
}

int kbo_i_fit_append(kbo_handle* h, const double* x_dev, double y, cudaStream_t s) {
  if (!h->fitted) KBO_FAIL(h, KBO_ERR_STATE, "kbo_fit_append: call kbo_fit first");
  KBO_TRY(kbo_i_ensure_w(h, s));   // the bordered row is l = W·k
  const int row = h->N, ld = h->ld, D = h->D;
  if (row + 1 > ld) KBO_FAIL(h, KBO_ERR_STATE, "kbo_fit_append: no room (N=%d fills its %d-row pitch): call kbo_fit with the whole history", row, ld);
  double* Krow = h->K.p + (size_t)row * ld;
  double* Wrow = h->W.p + (size_t)row * ld;
  KBO_TRY(kbo_reserve(h, h->lrow, (size_t)ld * 2 + 8));
  double* l = h->lrow.p;
  double* wtl = l + ld;
  double* dinv = wtl + ld;
  append_x_kernel<<<1, 256, 0, s>>>(x_dev, D, h->d_inv_ls.p, h->prm.n_length_scale, h->Xs.p, h->XsT.p, ld,
                                    h->nx.p, row, y, h->yraw.p);
  KBO_LAUNCH_CHECK(h);
  if (row > 0) {
    gram_row_kernel<<<(row + 127) / 128, 128, 0, s>>>(h->Xs.p, D, row, h->prm.kernel, h->prm.amplitude, Krow);
    KBO_LAUNCH_CHECK(h);
    trmv_lower_kernel<<<(row + 7) / 8, 256, 0, s>>>(h->W.p, row, ld, Krow, l);
    KBO_LAUNCH_CHECK(h);
  }
  append_diag_kernel<<<1, 1024, 0, s>>>(l, row, ld, h->prm.amplitude + h->prm.noise, Krow, dinv, h->info.p);
  KBO_LAUNCH_CHECK(h);
  {
    const int nslab = (row + 255) / 256;
    KBO_TRY(kbo_reserve(h, h->T, (size_t)(nslab + 1) * ld));
    if (row > 0) {
      dim3 g((row + 127) / 128, nslab);
      trmv_lower_t_kernel<<<g, 128, 0, s>>>(h->W.p, row, ld, l, h->T.p);
      KBO_LAUNCH_CHECK(h);
      trmv_t_reduce_kernel<<<(row + 127) / 128, 128, 0, s>>>(h->T.p, row, nslab, wtl);
      KBO_LAUNCH_CHECK(h);
    }
    append_wrow_kernel<<<(ld + 255) / 256, 256, 0, s>>>(wtl, row, ld, dinv, Wrow);
    KBO_LAUNCH_CHECK(h);
  }
  h->N = row + 1;
  h->Npad = round_up(h->N, 256);   // a rebase may have shrunk it below the new N; the planes are rebuilt at this extent by fit_finish
  prep_y_kernel<<<1, 1024, 0, s>>>(h->yraw.p, h->N, h->prm.normalize_y, h->yn.p, h->scal.p);
  KBO_LAUNCH_CHECK(h);
  KBO_TRY(fit_finish(h, s, false));
  return KBO_OK;
}

// kbo_fit_rebase: keep the first n_keep trials of the fitted history (the leading blocks of L and W = L⁻¹ ARE the factors of
// the shorter history), optionally with new y values — y enters only through yn/alpha/LML.  Drops constant-liar rows before
// the real trials are appended, and replaces a lie by the observed value when the trial finishes.
// A failure is cleared only if every kept row was factored: a failed append leaves just its own row unwritten, a failed fit its
// whole failing 64-block (potf2_inv_kernel returns before writing the block back, and the rows below it are never solved).
__global__ void clear_info_above_kernel(int* info, int n_keep) {
  const int bad = info[0];
  if (bad == 0) return;
  const int factored = info[1] ? bad - 1 : (bad - 1) / KBO_NB * KBO_NB;
  if (n_keep <= factored) info[0] = info[1] = 0;
}
int kbo_i_fit_rebase(kbo_handle* h, int n_keep, const double* y_dev, cudaStream_t s) {
  if (!h->fitted) KBO_FAIL(h, KBO_ERR_STATE, "kbo_fit_rebase: call kbo_fit first");
  if (n_keep < 1 || n_keep > h->N) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_fit_rebase: need 1 <= n_keep <= N=%d (got %d)", h->N, n_keep);
  KBO_TRY(kbo_i_ensure_w(h, s));   // keeps the bookkeeping simple: a rebased history carries all of W
  if (y_dev) KBO_CUDA(h, kbo_copy(h->yraw.p, y_dev, n_keep, cudaMemcpyDeviceToDevice, s));
  h->N = n_keep;
  h->Npad = round_up(n_keep, 256);
  clear_info_above_kernel<<<1, 1, 0, s>>>(h->info.p, n_keep);
  KBO_LAUNCH_CHECK(h);
  prep_y_kernel<<<1, 1024, 0, s>>>(h->yraw.p, h->N, h->prm.normalize_y, h->yn.p, h->scal.p);
  KBO_LAUNCH_CHECK(h);
  KBO_TRY(fit_finish(h, s, false));
  return KBO_OK;
}
