// ∂LML/∂θ on the device, θ = (log amplitude, log noise, log ℓ_1..ℓ_P)  — SURVEY.md §8(f)1, $SK/_gpr.py:621-653:
//   ∂LML/∂θ = ½ Σ_ij (α_i α_j − K⁻¹_ij) ∂K_ij/∂θ,   K = a·k(r) + σ²I,  r² = Σ_d Δ_d²  (Δ = scaled difference)
//   ∂K/∂log a = a·k ; ∂K/∂log σ² = σ²·I ; ∂K/∂log ℓ_d = a·q(r)·Δ_d²,  q = k (RBF), (5/3)(1+s)e^{−s} (Matérn-5/2, s = √5 r)
// K⁻¹ = WᵀW is formed as the lower triangle of Wt·Wtᵀ (Wt = Wᵀ, FP64 GEMM with the triangular K-range cut: N³/3 flop);
// one fused pass over the lower-triangular 64×64 pair tiles then accumulates every component (off-diagonal pairs count
// twice), per-block partials are reduced in a fixed order.  Everything FP64; kbo_lml_grad runs it after kbo_fit at the same θ,
// kbo_lml_grad_batch (fit.cu) on each θ's lane.
#include "kbo_internal.cuh"
#include "dgemm.cuh"
#include "ktab.cuh"

__global__ void transpose_kernel(const double* __restrict__ A, int N, int lda, double* __restrict__ At, int ldt) {
  __shared__ double t[32][33];
  const int x = blockIdx.x * 32 + threadIdx.x, y0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += 8)
    if (x < N && y0 + j < N) t[j][threadIdx.x] = A[(size_t)(y0 + j) * lda + x];
  __syncthreads();
  const int xo = blockIdx.y * 32 + threadIdx.x, yo0 = blockIdx.x * 32;
  for (int j = threadIdx.y; j < 32; j += 8)
    if (xo < N && yo0 + j < N) At[(size_t)(yo0 + j) * ldt + xo] = t[threadIdx.x][j];
}

// one block per lower-triangular 64×64 tile of trial pairs; partial[blk][0]=Σ G·a·k, [1]=Σ_diag G, [2+d]=Σ G·a·q·Δ_d²
__global__ void __launch_bounds__(256)
lml_grad_kernel(const double* __restrict__ Xs, int N, int D, int kind, double amp, const double* __restrict__ alpha,
                const double* __restrict__ Kinv, int ldk, int P, double* __restrict__ partial, int ncomp) {
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  if (n0 > m0) return;
  __shared__ double Xi[16][66], Xj[16][66];
  __shared__ double red[8];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4, lane = tid & 31, warp = tid >> 5;
  const int blk = blockIdx.y * gridDim.x + blockIdx.x;
  double* out = partial + (size_t)blk * ncomp;
  auto load_chunk = [&](int d0) {
    const int d = tid & 15;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int r = (tid >> 4) + 16 * i;
      Xi[d][r] = (m0 + r < N && d0 + d < D) ? Xs[(size_t)(m0 + r) * D + d0 + d] : 0.0;
      Xj[d][r] = (n0 + r < N && d0 + d < D) ? Xs[(size_t)(n0 + r) * D + d0 + d] : 0.0;
    }
  };
  auto block_sum = [&](double v) -> double {   // fixed order: lanes by shuffle tree, then warps 0..7
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double s = 0.0;
    for (int w = 0; w < 8; w++) s += red[w];
    return s;
  };
  double d2[4][4] = {};
  for (int d0 = 0; d0 < D; d0 += 16) {
    load_chunk(d0);
    __syncthreads();
#pragma unroll
    for (int dd = 0; dd < 16; dd++)
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const double df = Xi[dd][ty + 16 * i] - Xj[dd][tx + 16 * j];
          d2[i][j] = fma(df, df, d2[i][j]);
        }
    __syncthreads();
  }
  double c[4][4];
  double s_amp = 0.0, s_diag = 0.0;
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int gi = m0 + ty + 16 * i, gj = n0 + tx + 16 * j;
      double w = (gi < N && gj < N && gj <= gi) ? (gi == gj ? 1.0 : 2.0) : 0.0;   // lower triangle, off-diagonal pairs twice
      double G = 0.0, k = 0.0, q = 0.0;
      if (w != 0.0) {
        G = alpha[gi] * alpha[gj] - Kinv[(size_t)gi * ldk + gj];
        const double r2 = d2[i][j];
        if (kind == KBO_KERNEL_RBF) {
          k = kbo_exp_nonpos(-0.5 * r2);
          q = k;
        } else {
          const double s = kbo_sqrt_nonneg(5.0 * r2);
          const double e = kbo_exp_nonpos(-s);
          k = fma(s, fma(s, 1.0 / 3.0, 1.0), 1.0) * e;
          q = (5.0 / 3.0) * (1.0 + s) * e;
        }
        if (gi == gj) s_diag += G;
      }
      s_amp = fma(w * G, amp * k, s_amp);
      c[i][j] = w * G * amp * q;
    }
  {
    const double a = block_sum(s_amp), b = block_sum(s_diag);
    if (tid == 0) {
      out[0] = a;
      out[1] = b;
    }
  }
  double iso = 0.0;
  for (int d0 = 0; d0 < D; d0 += 16) {
    load_chunk(d0);
    __syncthreads();
    for (int dd = 0; dd < 16 && d0 + dd < D; dd++) {
      double s = 0.0;
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const double df = Xi[dd][ty + 16 * i] - Xj[dd][tx + 16 * j];
          s = fma(c[i][j], df * df, s);
        }
      if (P == 1) {
        iso += s;
      } else {
        const double t = block_sum(s);
        if (tid == 0) out[2 + d0 + dd] = t;
      }
    }
    __syncthreads();
  }
  if (P == 1) {
    const double t = block_sum(iso);
    if (tid == 0) out[2] = t;
  }
}

__global__ void lml_grad_reduce_kernel(const double* __restrict__ partial, int nblk_x, int nblk_y, int ncomp, double noise,
                                       double* __restrict__ grad) {
  const int cidx = blockIdx.x * blockDim.x + threadIdx.x;
  if (cidx >= ncomp) return;
  double s = 0.0;
  for (int by = 0; by < nblk_y; by++)
    for (int bx = 0; bx <= by && bx < nblk_x; bx++) s += partial[(size_t)(by * nblk_x + bx) * ncomp + cidx];
  grad[cidx] = cidx == 1 ? 0.5 * noise * s : 0.5 * s;
}

// K⁻¹ (lower triangle of Wt·Wtᵀ, Wt = Wᵀ) into Kinv, then the 2 + P gradient components into grad_dev.  Every operand is the
// caller's: kbo_lml_grad passes the handle's fit state, kbo_lml_grad_batch each lane's own planes.  part: nb²·(2 + P) doubles.
int kbo_i_lml_grad_from_w(kbo_handle* h, const double* Xs, int N, int D, int kind, double amp, double noise, const double* alpha,
                          const double* W, double* Wt, double* Kinv, int ld, int P, double* part, double* grad_dev, cudaStream_t s) {
  const int ncomp = 2 + P, nb = (N + 63) / 64;
  dim3 tg((N + 31) / 32, (N + 31) / 32), tb(32, 8);
  transpose_kernel<<<tg, tb, 0, s>>>(W, N, ld, Wt, ld);
  KBO_LAUNCH_CHECK(h);
  dgemm64_launch<true, EPI_STORE>(s, N, N, N, Wt, ld, Wt, ld, Kinv, ld, 1.0, 0.0, KM_FROM_M, 0, TS_LOWER);
  KBO_LAUNCH_CHECK(h);
  dim3 g(nb, nb);
  lml_grad_kernel<<<g, 256, 0, s>>>(Xs, N, D, kind, amp, alpha, Kinv, ld, P, part, ncomp);
  KBO_LAUNCH_CHECK(h);
  lml_grad_reduce_kernel<<<(ncomp + 63) / 64, 64, 0, s>>>(part, nb, nb, ncomp, noise, grad_dev);
  KBO_LAUNCH_CHECK(h);
  return KBO_OK;
}

extern "C" int kbo_lml_grad(kbo_handle* h, double* grad_host, int32_t n_out, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!h->fitted) KBO_FAIL(h, KBO_ERR_STATE, "kbo_lml_grad: call kbo_fit first");
  KBO_TRY(kbo_i_ensure_w(h, (cudaStream_t)stream));   // K⁻¹ = WᵀW
  const int N = h->N, D = h->D, ld = h->ld, P = (int)h->inv_ls.size(), ncomp = 2 + P;
  if (!grad_host || n_out != ncomp) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_lml_grad: output must hold 2 + n_length_scale = %d doubles", ncomp);
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  // Wt = Wᵀ into the trtri scratch, K⁻¹ (lower) into the K* fp64 scratch
  KBO_TRY(kbo_reserve(h, h->T, (size_t)N * ld));
  KBO_TRY(kbo_reserve(h, h->Ks64, (size_t)N * ld));
  const int nb = (N + 63) / 64;
  KBO_TRY(kbo_reserve(h, h->part, (size_t)nb * nb * ncomp + ncomp));
  double* grad_dev = h->part.p + (size_t)nb * nb * ncomp;
  KBO_TRY(kbo_i_lml_grad_from_w(h, h->Xs.p, N, D, h->prm.kernel, h->prm.amplitude, h->prm.noise, h->alpha.p,
                                h->W.p, h->T.p, h->Ks64.p, ld, P, h->part.p, grad_dev, s));
  int inf = 0;
  KBO_CUDA(h, cudaMemcpyAsync(grad_host, grad_dev, sizeof(double) * ncomp, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, kbo_copy(&inf, h->info.p, 1, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  // a failed fit leaves L (and so K⁻¹) partly unfactored: the gradient built from it is meaningless
  if (inf != 0) KBO_FAIL(h, KBO_ERR_NOT_PD, "kernel matrix is not positive definite (pivot %d); increase `noise`", inf);
  return KBO_OK;
}
