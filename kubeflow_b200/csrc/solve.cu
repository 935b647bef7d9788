// Triangular solves with the Cholesky factor, FP64, by 256-row panels — what the product path uses INSTEAD of the explicit
// inverse W = L⁻¹ ($SK/_gpr.py:363 alpha_ = cho_solve(L, y); :460 V = solve_triangular(L, K*ᵀ)).
//
// The pruned sweep needs exact variances for a handful of candidates and alpha for one right-hand side; forming W costs N³/3
// FP64 flop (a large share of the fit) to serve them.  A solve needs the factor L and the inverses of its 256×256
// diagonal blocks, which the look-ahead factorisation computes anyway (fit.cu: W_PP, kept in the diagonal blocks of the W
// buffer).  Forward, right-looking:   v_P = W_PP·b_P ;  b_>P −= L_>P,P·v_P      (P = 0, 1, …)
// backward (alpha = L⁻ᵀ z):            a_P = W_PPᵀ·z_P ; z_<P −= (L_P,<P)ᵀ·a_P   (P = last, …, 0)
// Up to 8 right-hand sides ride together (row-major N × 8): one pass over the triangle of L (268 MB at N = 8192) serves all of
// them, in one cooperative launch per solve (two grid barriers per panel).  Every right-hand side goes through the same operations in the same order whatever
// rides beside it, so a candidate's value does not depend on which other survivors it was grouped with.
#include "kbo_internal.cuh"

#define SV_P 256   // panel width = the factorisation's outer panel
#define SV_R 8     // right-hand sides per pass

namespace {

// Grid-wide barrier of a cooperative launch: every CTA adds one to a counter and spins until it reaches the running target.
// Release / acquire through __threadfence around the atomic: the panels written before the barrier are read (with plain,
// L2 loads: __ldcg — B, V, Z, A carry no __restrict__/const) after it.
__device__ __forceinline__ void sv_grid_barrier(unsigned* ctr, unsigned& target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    target += gridDim.x;
    __threadfence();
    atomicAdd(ctr, 1u);
    unsigned v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
    } while (v < target);
    __threadfence();
  }
  __syncthreads();
}

// V = L⁻¹·B, the whole solve in ONE cooperative launch (one CTA per SM, two grid barriers per panel) — 64 dependent launches
// per solve cost more than the 268 MB of L they read.  Per panel P:
//   (a) V_P = W_PP·B_P — one warp per row of the panel (the first 32 CTAs), B_P in shared memory as [rhs][k];
//   (b) B_>P −= L_>P,P·V_P — one warp per row below, grid-strided, V_P in shared memory as [rhs][k] (conflict-free).
// Fixed-order butterfly reductions: a right-hand side's result does not depend on the grid size or on what rides beside it.
template <bool SINGLE>   // SINGLE: one group (the usual case: alpha, one survivor) — the group loops vanish at compile time
__global__ void __launch_bounds__(256)
sv_forward_kernel(const double* __restrict__ L, const double* __restrict__ W, int N, int ld, double* B, double* V, unsigned* bar, int G_rt, size_t gstride) {
  const int G = SINGLE ? 1 : G_rt;
  // G groups of 8 right-hand sides ride one launch (group g at B + g·gstride): the rows of L and W_PP are loaded once and every group
  // goes through the arithmetic of a single-group solve, so a right-hand side's result does not depend on G either
  extern __shared__ double vs_all[];   // [G][SV_R][SV_P]
  unsigned target = 0;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gwarp = blockIdx.x * 8 + warp, nwarps = gridDim.x * 8;
  for (int K0 = 0; K0 < N; K0 += SV_P) {
    const int Wd = min(SV_P, N - K0);
    if (blockIdx.x * 8 < Wd) {   // (a)
      for (int e = threadIdx.x; e < G * SV_P * SV_R; e += 256) {
        const int g = e / (SV_P * SV_R), k = (e / SV_R) % SV_P, q = e % SV_R;
        vs_all[(size_t)g * SV_R * SV_P + q * SV_P + k] = k < Wd ? __ldcg(B + g * gstride + (size_t)(K0 + k) * SV_R + q) : 0.0;
      }
      __syncthreads();
      const int r = gwarp;
      if (r < Wd) {
        const double* w = W + (size_t)(K0 + r) * ld + K0;
        double wv[SV_P / 32];
#pragma unroll
        for (int i = 0; i < SV_P / 32; i++) wv[i] = lane + 32 * i <= r ? w[lane + 32 * i] : 0.0;
        for (int g = 0; g < G; g++) {
          const double* vs = vs_all + (size_t)g * SV_R * SV_P;
          double acc[SV_R];
#pragma unroll
          for (int q = 0; q < SV_R; q++) acc[q] = 0.0;
#pragma unroll
          for (int i = 0; i < SV_P / 32; i++)
#pragma unroll
            for (int q = 0; q < SV_R; q++) acc[q] = fma(wv[i], vs[q * SV_P + lane + 32 * i], acc[q]);
#pragma unroll
          for (int q = 0; q < SV_R; q++) {
            double v = acc[q];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0) V[g * gstride + (size_t)(K0 + r) * SV_R + q] = v;
          }
        }
      }
    }
    sv_grid_barrier(bar, target);
    const int below = N - (K0 + Wd);
    if (below > 0) {   // (b)
      for (int e = threadIdx.x; e < G * SV_P * SV_R; e += 256) {
        const int g = e / (SV_P * SV_R), k = (e / SV_R) % SV_P, q = e % SV_R;
        vs_all[(size_t)g * SV_R * SV_P + q * SV_P + k] = k < Wd ? __ldcg(V + g * gstride + (size_t)(K0 + k) * SV_R + q) : 0.0;
      }
      __syncthreads();
      for (int r = gwarp; r < below; r += nwarps) {
        const double* l = L + (size_t)(K0 + Wd + r) * ld + K0;
        double lv[SV_P / 32];
#pragma unroll
        for (int i = 0; i < SV_P / 32; i++) lv[i] = lane + 32 * i < Wd ? l[lane + 32 * i] : 0.0;
        for (int g = 0; g < G; g++) {
          const double* vs = vs_all + (size_t)g * SV_R * SV_P;
          double acc[SV_R];
#pragma unroll
          for (int q = 0; q < SV_R; q++) acc[q] = 0.0;
#pragma unroll
          for (int i = 0; i < SV_P / 32; i++)
#pragma unroll
            for (int q = 0; q < SV_R; q++) acc[q] = fma(lv[i], vs[q * SV_P + lane + 32 * i], acc[q]);
#pragma unroll
          for (int q = 0; q < SV_R; q++) {
            double v = acc[q];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0) {
              double* o = B + g * gstride + (size_t)(K0 + Wd + r) * SV_R + q;
              *o = __ldcg(o) - v;
            }
          }
        }
      }
      sv_grid_barrier(bar, target);
    }
  }
}

// One 32-column unit of a transposed panel product:  out[c][q] (−)= Σ_r M[r][c0 + c]·x[r][q], r < rows.  Lanes own the columns
// (coalesced 256-byte row segments), the 8 warps take rows r ≡ warp (mod 8) with all their loads in flight, and the 8
// partial sums meet in shared memory in warp order.
template <bool TRI, bool SUB>
__device__ __forceinline__ void sv_unit_t(const double* __restrict__ M, int ldm, int rows, int c0, int ncols, const double* xs /* smem [r][q] */,
                                          double* red /* smem [8][32][SV_R] */, double* out /* global, row c0.. */) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = c0 + lane;
  double acc[SV_R];
#pragma unroll
  for (int q = 0; q < SV_R; q++) acc[q] = 0.0;
  for (int rb = 0; rb < SV_P / 8; rb += 16) {
    double mv[16];
#pragma unroll
    for (int i = 0; i < 16; i++) {
      const int r = (rb + i) * 8 + warp;
      mv[i] = (r < rows && lane < ncols && (!TRI || r >= c)) ? M[(size_t)r * ldm + c] : 0.0;
    }
#pragma unroll
    for (int i = 0; i < 16; i++) {
      const int r = min((rb + i) * 8 + warp, rows - 1);
#pragma unroll
      for (int q = 0; q < SV_R; q++) acc[q] = fma(mv[i], xs[r * SV_R + q], acc[q]);
    }
  }
#pragma unroll
  for (int q = 0; q < SV_R; q++) red[(warp * 32 + lane) * SV_R + q] = acc[q];
  __syncthreads();
  {
    const int cc = threadIdx.x >> 3, q = threadIdx.x & 7;   // 32 columns × 8 right-hand sides = 256 threads
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < 8; w++) v += red[(w * 32 + cc) * SV_R + q];
    if (cc < ncols) {
      double* o = out + (size_t)(c0 + cc) * SV_R + q;
      *o = SUB ? __ldcg(o) - v : v;
    }
  }
  __syncthreads();
}

// A = L⁻ᵀ·Z in one cooperative launch.  Per panel P, last to first:
//   (a) A_P = W_PPᵀ·Z_P — 8 units of 32 columns;   (b) Z_<P −= (L_P,<P)ᵀ·A_P — K0/32 units, grid-strided.
__global__ void __launch_bounds__(256)
sv_backward_kernel(const double* __restrict__ L, const double* __restrict__ W, int N, int ld, double* Z, double* A, unsigned* bar) {
  __shared__ double xs[SV_P * SV_R];
  __shared__ double red[8 * 32 * SV_R];
  unsigned target = 0;
  const int last = (N - 1) / SV_P * SV_P;
  for (int K0 = last; K0 >= 0; K0 -= SV_P) {
    const int Wd = min(SV_P, N - K0);
    const int units_a = (Wd + 31) / 32;
    if ((int)blockIdx.x < units_a) {   // (a)
      for (int e = threadIdx.x; e < Wd * SV_R; e += 256) xs[e] = __ldcg(Z + (size_t)K0 * SV_R + e);
      __syncthreads();
      for (int u = blockIdx.x; u < units_a; u += gridDim.x)
        sv_unit_t<true, false>(W + (size_t)K0 * ld + K0, ld, Wd, u * 32, min(32, Wd - u * 32), xs, red, A + (size_t)K0 * SV_R);
    }
    sv_grid_barrier(bar, target);
    if (K0 > 0) {   // (b)
      for (int e = threadIdx.x; e < Wd * SV_R; e += 256) xs[e] = __ldcg(A + (size_t)K0 * SV_R + e);
      __syncthreads();
      for (int u = blockIdx.x; u < K0 / 32; u += gridDim.x) sv_unit_t<false, true>(L + (size_t)K0 * ld, ld, Wd, u * 32, 32, xs, red, Z);
      sv_grid_barrier(bar, target);
    }
  }
}

// right-hand sides of one group: B[j][q] = Ks[(c0 + q)·ld + j] (q < nq; the rest zero)
__global__ void sv_pack_kernel(const double* __restrict__ Ks, int ld, int N, int c0, int nq, double* __restrict__ B) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
#pragma unroll
  for (int q = 0; q < SV_R; q++) B[(size_t)j * SV_R + q] = q < nq ? Ks[(size_t)(c0 + q) * ld + j] : 0.0;
}
// varn[c0 + q] = amp − Σ_j V[j][q]² : one CTA per right-hand side, fixed-order tree
__global__ void __launch_bounds__(256) sv_sumsq_kernel(const double* __restrict__ V, int N, double amp, double* __restrict__ varn) {
  __shared__ double red[256];
  const int q = blockIdx.x;
  double a = 0.0;
  for (int j = threadIdx.x; j < N; j += 256) {
    const double v = V[(size_t)j * SV_R + q];
    a = fma(v, v, a);
  }
  red[threadIdx.x] = a;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) varn[q] = amp - red[0];
}
__global__ void sv_col_kernel(const double* __restrict__ src, int N, int stride_src, double* __restrict__ dst, int stride_dst) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < N) dst[(size_t)j * stride_dst] = src[(size_t)j * stride_src];
}

}  // namespace

#define SV_GMAX 8   // groups of 8 right-hand sides per forward launch (16 KB of shared memory each)
static int sv_bar_reset(kbo_handle* h, cudaStream_t s) {
  KBO_TRY(kbo_reserve(h, h->sv_bar, 64));
  KBO_CUDA(h, cudaMemsetAsync(h->sv_bar.p, 0, sizeof *h->sv_bar.p, s));
  return KBO_OK;
}
// B (G groups of N × 8, overwritten: scratch) -> V = L⁻¹·B.  Needs the diagonal-block inverses in W's diagonal 256-blocks.
int kbo_i_solve_fwd(kbo_handle* h, double* B, double* V, cudaStream_t s, int G, size_t gstride) {
  KBO_TRY(sv_bar_reset(h, s));
  const double* L = h->K.p;
  const double* W = h->W.p;
  int N = h->N, ld = h->ld;
  unsigned* bar = h->sv_bar.p;
  const size_t smem = sizeof(double) * (size_t)G * SV_R * SV_P;
  static bool attr = false;
  if (!attr) {
    KBO_CUDA(h, cudaFuncSetAttribute(sv_forward_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(double) * SV_GMAX * SV_R * SV_P)));
    attr = true;
  }
  void* args[] = {(void*)&L, (void*)&W, (void*)&N, (void*)&ld, (void*)&B, (void*)&V, (void*)&bar, (void*)&G, (void*)&gstride};
  const void* fn = G == 1 ? (const void*)sv_forward_kernel<true> : (const void*)sv_forward_kernel<false>;
  KBO_CUDA(h, cudaLaunchCooperativeKernel(fn, dim3(h->sm_count), dim3(256), args, smem, s));   // one CTA per SM: co-resident
  return KBO_OK;
}
// Z (N × 8, overwritten) -> A = L⁻ᵀ·Z (N × 8)
int kbo_i_solve_bwd(kbo_handle* h, double* Z, double* A, cudaStream_t s) {
  KBO_TRY(sv_bar_reset(h, s));
  const double* L = h->K.p;
  const double* W = h->W.p;
  int N = h->N, ld = h->ld;
  unsigned* bar = h->sv_bar.p;
  void* args[] = {(void*)&L, (void*)&W, (void*)&N, (void*)&ld, (void*)&Z, (void*)&A, (void*)&bar};
  KBO_CUDA(h, cudaLaunchCooperativeKernel((const void*)sv_backward_kernel, dim3(h->sm_count), dim3(256), args, 0, s));
  return KBO_OK;
}

// ---- z = L⁻¹·yn one panel behind the factorisation (fit.cu, lazy fits): the forward half of alpha rides in the factorisation's
// shadow — a panel's step needs W_PP and the rows of L below the panel, both final as soon as that panel is — so fit_finish pays
// for the backward half only.  One right-hand side, plain vectors b (consumed) and z.
namespace {
__global__ void __launch_bounds__(256) sv_zdiag_kernel(const double* __restrict__ Wpp, int ldw, int Wd, const double* __restrict__ b, double* __restrict__ z) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= Wd) return;
  const double* w = Wpp + (size_t)r * ldw;
  double a = 0.0;
#pragma unroll
  for (int i = 0; i < SV_P / 32; i++) {
    const int k = lane + 32 * i;
    if (k <= r) a = fma(w[k], b[k], a);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (lane == 0) z[r] = a;
}
__global__ void __launch_bounds__(256) sv_zupdate_kernel(const double* __restrict__ Lp, int ldl, int rows, int Wd, const double* __restrict__ zP,
                                                         double* __restrict__ b) {
  __shared__ double zs[SV_P];
  for (int k = threadIdx.x; k < SV_P; k += 256) zs[k] = k < Wd ? zP[k] : 0.0;
  __syncthreads();
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const double* l = Lp + (size_t)r * ldl;
  double lv[SV_P / 32];
#pragma unroll
  for (int i = 0; i < SV_P / 32; i++) lv[i] = lane + 32 * i < Wd ? l[lane + 32 * i] : 0.0;
  double a = 0.0;
#pragma unroll
  for (int i = 0; i < SV_P / 32; i++) a = fma(lv[i], zs[lane + 32 * i], a);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (lane == 0) b[r] -= a;
}
}  // namespace
int kbo_i_zsolve_reserve(kbo_handle* h) { return kbo_reserve(h, h->zf, (size_t)(h->N + SV_P) * 2); }
// after kbo_i_zsolve_reserve: it allocates nothing, so a graph capture may contain it
int kbo_i_zsolve_begin(kbo_handle* h, cudaStream_t s) {
  KBO_CUDA(h, kbo_copy(h->zf.p, h->yn.p, h->N, cudaMemcpyDeviceToDevice, s));
  h->z_ready = false;
  return KBO_OK;
}
// panel [K0, K0 + Wd): z_P = W_PP·b_P (needs W's diagonal 256-block) ...
int kbo_i_zsolve_diag(kbo_handle* h, int K0, int Wd, cudaStream_t s) {
  double* b = h->zf.p;
  double* z = b + h->N + SV_P;
  sv_zdiag_kernel<<<(Wd + 7) / 8, 256, 0, s>>>(h->W.p + (size_t)K0 * h->ld + K0, h->ld, Wd, b + K0, z + K0);
  KBO_LAUNCH_CHECK(h);
  return KBO_OK;
}
// ... then b_>P −= L_>P,P·z_P (needs the rows of L below the panel)
int kbo_i_zsolve_update(kbo_handle* h, int K0, int Wd, cudaStream_t s) {
  const int N = h->N, rows = N - (K0 + Wd);
  if (rows <= 0) return KBO_OK;
  double* b = h->zf.p;
  double* z = b + N + SV_P;
  sv_zupdate_kernel<<<(rows + 7) / 8, 256, 0, s>>>(h->K.p + (size_t)(K0 + Wd) * h->ld + K0, h->ld, rows, Wd, z + K0, b + K0 + Wd);
  KBO_LAUNCH_CHECK(h);
  return KBO_OK;
}

// alpha = L⁻ᵀ(L⁻¹·yn) into h->alpha (what fit_finish computes as Wᵀ(W·yn) when W is formed)
int kbo_i_alpha_by_solves(kbo_handle* h, cudaStream_t s) {
  const int N = h->N;
  KBO_TRY(kbo_reserve(h, h->sv_B, (size_t)(N + SV_P) * SV_R));
  KBO_TRY(kbo_reserve(h, h->sv_V, (size_t)(N + SV_P) * SV_R));
  double* B = h->sv_B.p;
  double* V = h->sv_V.p;
  if (h->z_ready) {   // the factorisation already carried z = L⁻¹·yn along (kbo_i_zsolve_*)
    KBO_CUDA(h, cudaMemsetAsync(V, 0, sizeof(double) * (size_t)N * SV_R, s));
    sv_col_kernel<<<(N + 255) / 256, 256, 0, s>>>(h->zf.p + N + SV_P, N, 1, V, SV_R);
    KBO_LAUNCH_CHECK(h);
    h->z_ready = false;
  } else {
    KBO_CUDA(h, cudaMemsetAsync(B, 0, sizeof(double) * (size_t)N * SV_R, s));
    sv_col_kernel<<<(N + 255) / 256, 256, 0, s>>>(h->yn.p, N, 1, B, SV_R);
    KBO_LAUNCH_CHECK(h);
    KBO_TRY(kbo_i_solve_fwd(h, B, V, s, 1, 0));      // V[:,0] = z
  }
  KBO_TRY(kbo_i_solve_bwd(h, V, B, s));      // B[:,0] = alpha (V is consumed)
  sv_col_kernel<<<(N + 255) / 256, 256, 0, s>>>(B, N, SV_R, h->alpha.p, 1);
  KBO_LAUNCH_CHECK(h);
  return KBO_OK;
}

// varn64[c] = amp − ‖L⁻¹ k*_c‖² for the n rows of Ks (n × ld, FP64 K*): up to 64 right-hand sides (8 groups of 8) per forward solve
int kbo_i_variance_by_solves(kbo_handle* h, const double* Ks, int n, double* varn64, cudaStream_t s) {
  const int N = h->N, ld = h->ld;
  const size_t gstride = (size_t)(N + SV_P) * SV_R;
  KBO_TRY(kbo_reserve(h, h->sv_B, gstride * SV_GMAX));
  KBO_TRY(kbo_reserve(h, h->sv_V, gstride * SV_GMAX));
  double* B = h->sv_B.p;
  double* V = h->sv_V.p;
  for (int c0 = 0; c0 < n; c0 += SV_R * SV_GMAX) {
    const int nc = n - c0 < SV_R * SV_GMAX ? n - c0 : SV_R * SV_GMAX, G = (nc + SV_R - 1) / SV_R;
    for (int g = 0; g < G; g++) {
      const int nq = nc - g * SV_R < SV_R ? nc - g * SV_R : SV_R;
      sv_pack_kernel<<<(N + 255) / 256, 256, 0, s>>>(Ks, ld, N, c0 + g * SV_R, nq, B + g * gstride);
      KBO_LAUNCH_CHECK(h);
    }
    KBO_TRY(kbo_i_solve_fwd(h, B, V, s, G, gstride));
    for (int g = 0; g < G; g++) {
      const int nq = nc - g * SV_R < SV_R ? nc - g * SV_R : SV_R;
      sv_sumsq_kernel<<<nq, 256, 0, s>>>(V + g * gstride, N, h->prm.amplitude, varn64 + c0 + g * SV_R);
      KBO_LAUNCH_CHECK(h);
    }
  }
  return KBO_OK;
}
