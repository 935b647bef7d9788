// ask(): predict(return_std=True) + acquisition + first-index argmax over the candidate grid.
//   $SK/_gpr.py:446 K* = k(Xc,X) | :447-450 mean | :460 V = L⁻¹K*ᵀ (here V = K*·Wᵀ, W = L⁻¹) | :480-500 variance
//   skopt.acquisition.gaussian_ei / gaussian_lcb / gaussian_pi ; Optimizer._tell: X_cand[np.argmin(values)]
// Per candidate chunk:  cross_mean_kernel (FP64: K*, μ = K*·alpha)  →  variance contraction (FP64 SIMT GEMM with a
// fused Σv² epilogue, or the wgmma kernel in tc_var.cu)  →  once per sweep: acquisition + argmax.
#include <algorithm>
#include <cstring>
#include <type_traits>

#include "kbo_internal.cuh"
#include "dgemm.cuh"
#include "ktab.cuh"
#include "kbo_acq.cuh"

// ------------------------------------------------------------------------------------------------
// K* kernel.  A CTA owns 128 candidates and walks all 64-trial tiles (so μ = K*·alpha needs no atomics).
// The dot products are an FP64 GEMM with K = D: 8×4 outputs per thread (12 LDS per 32 DFMA keeps the FP64 pipe, not
// shared memory, the limiter), the trial matrix is read from its TRANSPOSE (XsT, D × ldx) so global loads coalesce and
// shared stores are conflict-free, and the next 32-dimension slab is prefetched into registers while the current one
// is consumed (one __syncthreads per slab).  Epilogue per element: d² → branch-free FP64 kernel value (ktab.cuh) → μ FMA →
// MODE 0: fp64 K* (chunk × ldks)   MODE 1: fp16 hi/lo planes (chunk_pad × Npad).
#ifndef KBO_CM_MINB
#define KBO_CM_MINB 2
#endif
#define CM_BM 128
#define CM_BN 64
#define CM_DC 32
template <typename XT, typename MT, int MODE>
__global__ void __launch_bounds__(256, KBO_CM_MINB)
cross_mean_kernel(const XT* __restrict__ Xc, int64_t rows, int D, const double* __restrict__ inv_ls, int n_ls,
                  const double* __restrict__ XsT, int ldx, const double* __restrict__ nx, int N, const double* __restrict__ alpha, int kind,
                  double amp, double* __restrict__ Ks64, int ldks, __half* __restrict__ Ksh,
                  __half* __restrict__ Ksl, int Npad, MT* __restrict__ mun, double* __restrict__ mu_part) {
  // gridDim.y > 1: the trial tiles are split over blockIdx.y (few candidate rows — the calibration rows — would otherwise leave
  // half of the SMs idle); each split writes its partial mean to mu_part[split][row], summed in split order by mu_parts_kernel
  extern __shared__ __align__(16) unsigned char smraw[];
  const int Dp = (D + CM_DC - 1) / CM_DC * CM_DC;
  double* As = reinterpret_cast<double*>(smraw);        // [Dp][130]
  double* Bs = As + (size_t)Dp * 130;                   // [2][32][66]
  double* nc = Bs + 2 * CM_DC * 66;                     // [128]
  double* nxs = nc + CM_BM;                             // [2][64]
  double* als = nxs + 2 * CM_BN;                        // [2][64]
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = (int64_t)blockIdx.x * CM_BM;

  for (int e = tid; e < CM_BM * Dp; e += 256) {
    const int r = e / Dp, d = e % Dp;
    double v = 0.0;
    if (m0 + r < rows && d < D) v = (double)Xc[(m0 + r) * D + d] * inv_ls[n_ls == 1 ? 0 : d];
    As[d * 130 + r] = v;
  }
  __syncthreads();
  if (tid < CM_BM) {
    double s = 0.0;
    for (int d = 0; d < D; d++) s = fma(As[d * 130 + tid], As[d * 130 + tid], s);
    nc[tid] = s;
  }
  const int nd = Dp / CM_DC;
  const int ntiles = (N + CM_BN - 1) / CM_BN;
  const int tps = (ntiles + gridDim.y - 1) / gridDim.y;
  const int tile0 = blockIdx.y * tps, tile1 = min(ntiles, tile0 + tps);
  const int total = max(0, tile1 - tile0) * nd;
  double pf[8];
  double pf_nx = 0.0, pf_al = 0.0;
  // slab `it` = (tile it / nd, dims [ (it % nd)·32, +32 ) ): thread loads n = tid & 63, dd = (tid >> 6) + 4q
  auto prefetch = [&](int it) {
    const int n0 = (tile0 + it / nd) * CM_BN, d0 = (it % nd) * CM_DC;
    const int n = n0 + (tid & 63);
#pragma unroll
    for (int q = 0; q < 8; q++) {
      const int d = d0 + (tid >> 6) + 4 * q;
      pf[q] = (n < N && d < D) ? XsT[(size_t)d * ldx + n] : 0.0;
    }
    if ((it % nd) == 0 && tid < CM_BN) {
      pf_nx = n < N ? nx[n] : 0.0;
      pf_al = n < N ? alpha[n] : 0.0;
    }
  };
  auto commit = [&](int it) {
    double* B = Bs + (it & 1) * CM_DC * 66;
#pragma unroll
    for (int q = 0; q < 8; q++) B[((tid >> 6) + 4 * q) * 66 + (tid & 63)] = pf[q];
    if ((it % nd) == 0 && tid < CM_BN) {
      const int tb = (it / nd) & 1;
      nxs[tb * CM_BN + tid] = pf_nx;
      als[tb * CM_BN + tid] = pf_al;
    }
  };
  double musum[8];
#pragma unroll
  for (int i = 0; i < 8; i++) musum[i] = 0.0;
  double acc[8][4];
  if (total > 0) {
    prefetch(0);
    commit(0);
  }
  __syncthreads();
  for (int it = 0; it < total; it++) {
    const int tile = tile0 + it / nd, dchunk = it % nd;
    if (dchunk == 0) {
#pragma unroll
      for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0.0;
    }
    if (it + 1 < total) prefetch(it + 1);
    {
      const double* B = Bs + (it & 1) * CM_DC * 66;
      const double* A = As + (size_t)dchunk * CM_DC * 130;
#pragma unroll 8
      for (int dd = 0; dd < CM_DC; dd++) {
        double a[8], b[4];
#pragma unroll
        for (int i = 0; i < 8; i++) a[i] = A[dd * 130 + ty + 16 * i];
#pragma unroll
        for (int j = 0; j < 4; j++) b[j] = B[dd * 66 + tx + 16 * j];
#pragma unroll
        for (int i = 0; i < 8; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) acc[i][j] = fma(a[i], b[j], acc[i][j]);
      }
    }
    if (dchunk == nd - 1) {
      // branch-free epilogue: all 32 kernel values are computed unconditionally (inputs are always finite), so the whole
      // block is one scheduling region with 32 independent FP64 dependency chains to interleave.  Interior tiles (the
      // overwhelming majority) skip the row/column masks altogether; edge tiles mask the results at the end.
      const int n0 = tile * CM_BN, tb = (it / nd) & 1;
      double nxv[4], alv[4];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int c = tx + 16 * j;
        nxv[j] = nxs[tb * CM_BN + c];
        alv[j] = als[tb * CM_BN + c];
      }
      auto epilogue = [&](auto masked_tag) {
        constexpr bool MASKED = decltype(masked_tag)::value;
#pragma unroll
        for (int i = 0; i < 8; i++) {
          const int r = ty + 16 * i;
          const bool rok = !MASKED || m0 + r < rows;
          const double ncr = nc[r];
          double kv[4];
#pragma unroll
          for (int j = 0; j < 4; j++) kv[j] = amp * kbo_kernel_exact(fma(-2.0, acc[i][j], ncr + nxv[j]), kind);
#pragma unroll
          for (int j = 0; j < 4; j++) {
            const bool ok = !MASKED || (rok && n0 + tx + 16 * j < N);
            if (MASKED) kv[j] = ok ? kv[j] : 0.0;
            musum[i] = fma(kv[j], alv[j], musum[i]);   // alpha is zero-padded past N, kv is masked: padding adds exactly 0
            const int c = tx + 16 * j;
            if (MODE == 0) {
              if (ok) Ks64[(size_t)(m0 + r) * ldks + n0 + c] = kv[j];
            } else {  // 16 lanes × 2 B = one full 32-byte sector per (row, 16-column group): no staging needed
              const __half hi = __double2half(kv[j]);
              const size_t g = (size_t)(m0 + r) * Npad + n0 + c;
              Ksh[g] = hi;
              Ksl[g] = __double2half(kv[j] - (double)__half2float(hi));
            }
          }
        }
      };
      if (m0 + CM_BM <= rows && n0 + CM_BN <= N)
        epilogue(std::false_type{});
      else
        epilogue(std::true_type{});
    }
    if (it + 1 < total) commit(it + 1);
    __syncthreads();
  }
  if (MODE == 1 && blockIdx.y == gridDim.y - 1) {  // zero the padding columns [ntiles·64, Npad) of this CTA's rows (W is zero there, but 0·NaN must not happen)
    const int c0 = ntiles * CM_BN, w = Npad - c0;
    if (w > 0) {
      const int segs = w / 8;
      for (int e = tid; e < CM_BM * segs; e += 256) {
        const int r = e / segs, sgm = e % segs;
        const size_t g = (size_t)(m0 + r) * Npad + c0 + sgm * 8;
        *reinterpret_cast<uint4*>(Ksh + g) = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4*>(Ksl + g) = make_uint4(0, 0, 0, 0);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; i++) {
    double s = musum[i];
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const int64_t gm = m0 + ty + 16 * i;
    if (tx == 0 && gm < rows) {
      if (gridDim.y > 1)
        mu_part[(size_t)blockIdx.y * rows + gm] = s;
      else
        mun[gm] = (MT)s;
    }
  }
}
template <typename MT>
__global__ void mu_parts_kernel(const double* __restrict__ part, int64_t rows, int nsplit, MT* __restrict__ mun) {
  const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= rows) return;
  double s = 0.0;
  for (int j = 0; j < nsplit; j++) s += part[(size_t)j * rows + m];
  mun[m] = (MT)s;
}

__global__ void var_from_parts_kernel(const double* __restrict__ part, int64_t rows, int njt, double amp, double* __restrict__ varn) {
  const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= rows) return;
  double s = 0.0;
  for (int j = 0; j < njt; j++) s += part[m * njt + j];
  varn[m] = amp - s;
}

// ------------------------------------------------------------------------------------------------
// Acquisition + argmax.  T = double (checker precision) or float (8 B/candidate in, the HBM-bound pass).
struct BlockBest {
  double v;
  long long i;
};

// One pass: 8 B/candidate in (μ_n, σ²_n as fp32), optional 4 B out.  Persistent-style grid (≤ 2 CTAs per SM, 256 threads),
// each thread streams groups of 4 candidates with TWO groups (4×16 B loads) in flight before any math, so a 12 MB pass is
// not latency-bound on a single load→erfc→store chain per thread.
// fp32 path of the HBM-bound pass, specialised per acquisition kind (no runtime switch inside the candidate loop):
//   σ = σ²·rsqrt(σ²)·y_std (MUFU.RSQ), z = imp/σ (MUFU.RCP), φ(z) = exp2(−z²·log2e/2)/√(2π) (MUFU.EX2),
//   Φ(z) = erfc(−z/√2)/2 with erfc(x ≥ 0) = t·exp(−x² + P(t)), t = 1/(1 + x/2), P = the degree-9 Chebyshev fit of
//   Numerical Recipes §6.2 (`erfcc`): FRACTIONAL error ≤ 1.2e-7 everywhere, so candidates whose EI is ~1e-30 still rank
//   correctly (an absolute-error Φ — Abramowitz–Stegun 26.2.17 — mis-ranked that tail; tests/test_gpu_parity.py edge cases),
//   at ~16 instructions instead of erfcf's ~35.  |ΔEI| ≲ 3e-7 for |imp| ≲ 4; the fp64 instantiation keeps erfc/exp.
__device__ __forceinline__ float kbo_ex2_ftz(float x) {   // MUFU.EX2 alone; results below 2^-126 flush to zero
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float kbo_erfc_nonneg_f32(float x) {
  const float t = __fdividef(1.f, fmaf(0.5f, x, 1.f));
  float p = 0.17087277f;
  p = fmaf(p, t, -0.82215223f);
  p = fmaf(p, t, 1.48851587f);
  p = fmaf(p, t, -1.13520398f);
  p = fmaf(p, t, 0.27886807f);
  p = fmaf(p, t, -0.18628806f);
  p = fmaf(p, t, 0.09678418f);
  p = fmaf(p, t, 0.37409196f);
  p = fmaf(p, t, 1.00002368f);
  p = fmaf(p, t, -1.26551223f);
  return t * kbo_ex2_ftz(1.44269504088896340736f * fmaf(-x, x, p));
}
// The fp32 acquisition is evaluated in NORMALISED units, never at the raw y scale: an fp32 μ = y_mean + y_std·μ_n rounds at
// the scale of y_mean (half an ulp is 1e-3 at |y_mean| = 2e4 — a Katib metric in µs), which is above every slack of the
// bounds below.  c_n = (y_opt − ξ − y_mean)/y_std is formed once in FP64 and carried as an fp32 hi/lo pair, so the
// improvement c_n − μ_n is as accurate as μ_n itself.  The values returned are
//   EI: imp_n·Φ(z) + σ_n·φ(z) = EI / y_std     PI: Φ(z) = PI     LCB: κσ_n − μ_n = (LCB value + y_mean) / y_std
// — increasing maps of the raw value (y_std > 0), so they rank the same; acq_raw() undoes the map where a raw value is wanted.
struct AcqFrame {
  float chi, clo, kp;
};
__device__ __forceinline__ AcqFrame acq_frame(double ymean, double ystd, double yopt, double xi, double kappa) {
  const double c = (yopt - xi - ymean) / ystd;
  AcqFrame f;
  f.chi = (float)c;
  f.clo = (float)(c - (double)f.chi);
  f.kp = (float)kappa;
  return f;
}
__device__ __forceinline__ double acq_raw(int acq, double a, double ymean, double ystd) {
  return acq == KBO_ACQ_PI ? a : acq == KBO_ACQ_LCB ? fma(ystd, a, -ymean) : ystd * a;
}
template <int ACQ>
__device__ __forceinline__ float acq_value_f32(float mun, float varn, const AcqFrame& f) {
  const float var = fmaxf(varn, 0.f);
  const float sd = var > 0.f ? var * rsqrtf(var) : 0.f;
  if (ACQ == KBO_ACQ_LCB) return fmaf(f.kp, sd, -mun);
  if (!(sd > 0.f)) return 0.f;
  const float imp = (f.chi - mun) + f.clo;
  const float z = __fdividef(imp, sd);   // MUFU.RCP + FMUL (2 ulp), no IEEE-division subroutine
  const float q = 0.5f * kbo_erfc_nonneg_f32(0.70710678118654752440f * fabsf(z));   // tail beyond |z|
  const float cdf = z <= 0.f ? q : 1.f - q;
  if (ACQ == KBO_ACQ_PI) return cdf;
  const float pdf = 0.3989422804014327f * kbo_ex2_ftz(-0.72134752044448170368f * z * z);
  return fmaf(imp, cdf, sd * pdf);
}

// FAST_ACQ = −1: generic path (runtime acquisition kind, erfc/exp/sqrt in T, optional fp64 μ/σ outputs);
// FAST_ACQ = 0/1/2: the fp32 specialisation for EI / LCB / PI chosen on the host — no per-candidate switch.
template <typename T, int FAST_ACQ>
__global__ void __launch_bounds__(256)
acq_kernel(const T* __restrict__ mun, const T* __restrict__ varn, int64_t M, int64_t goff, int acq, double ymean, double ystd,
           double yopt, const double* __restrict__ scal_dev, double xi, double kappa, double* __restrict__ mu_out,
           double* __restrict__ std_out, double* __restrict__ acq_out, float* __restrict__ acq_out32,
           BlockBest* __restrict__ partial, unsigned int* __restrict__ ticket, kbo_best* __restrict__ best) {
  if (scal_dev) {  // composed path: y statistics stay on the device, no host round trip
    ymean = scal_dev[S_YMEAN];
    ystd = scal_dev[S_YSTD];
    yopt = scal_dev[S_YOPT];
  }
  double bv = -INFINITY;
  long long bi = 0x7fffffffffffffffLL;
  const AcqFrame fr = acq_frame(ymean, ystd, yopt, xi, kappa);
  constexpr int FA = FAST_ACQ >= 0 ? FAST_ACQ : 0;
  // fp32 specialisation: ranking values are normalised (acq_value_f32); what leaves the kernel is the raw value
  const float ysf = (float)ystd, ymf = (float)ymean;
  auto raw32 = [&](float a) { return FA == KBO_ACQ_PI ? a : FA == KBO_ACQ_LCB ? fmaf(ysf, a, -ymf) : ysf * a; };
  const int64_t stride = (int64_t)gridDim.x * 256 * 4;
  auto load4 = [&](int64_t base, T (&m4)[4], T (&v4)[4]) {
    if (base + 3 < M) {
      if (sizeof(T) == 4) {
        const float4 a = __ldcs(reinterpret_cast<const float4*>(mun + base));
        const float4 b = __ldcs(reinterpret_cast<const float4*>(varn + base));
        m4[0] = a.x; m4[1] = a.y; m4[2] = a.z; m4[3] = a.w;
        v4[0] = b.x; v4[1] = b.y; v4[2] = b.z; v4[3] = b.w;
      } else {
        const double2 a0 = *reinterpret_cast<const double2*>(mun + base), a1 = *reinterpret_cast<const double2*>(mun + base + 2);
        const double2 b0 = *reinterpret_cast<const double2*>(varn + base), b1 = *reinterpret_cast<const double2*>(varn + base + 2);
        m4[0] = a0.x; m4[1] = a0.y; m4[2] = a1.x; m4[3] = a1.y;
        v4[0] = b0.x; v4[1] = b0.y; v4[2] = b1.x; v4[3] = b1.y;
      }
    } else {
#pragma unroll
      for (int q = 0; q < 4; q++) {
        m4[q] = base + q < M ? mun[base + q] : (T)0;
        v4[q] = base + q < M ? varn[base + q] : (T)0;
      }
    }
  };
  // Per-thread running best is kept in the value type VT with a strict '>' (indices only grow inside a thread, so the
  // first maximum wins without an index compare); it is widened to (double, int64) once, before the cross-thread reduce.
  // The generic path evaluates in FP64 also for fp32 inputs (the arrays of a tensor-core sweep): an fp32 μ = y_mean + y_std·μ_n
  // would round at the scale of y_mean.
  constexpr bool fast32 = FAST_ACQ >= 0;
  using VT = typename std::conditional<fast32, T, double>::type;
  VT tbest = -(VT)INFINITY;
  int64_t tidx = 0x7fffffffffffffffLL;
  auto process4 = [&](int64_t base, const T (&m4)[4], const T (&v4)[4]) {
    if (base >= M) return;
    const bool full = base + 3 < M;
    if (fast32 && full) {
      // the hot path: four values, one vector store, ONE compare against the running best per group (the first maximum
      // inside the group is located only when the group wins) — ~40 instructions per candidate in total
      float a4[4];
#pragma unroll
      for (int q = 0; q < 4; q++)
        a4[q] = acq_value_f32<FA>((float)m4[q], (float)v4[q], fr);
      if (acq_out32) __stcs(reinterpret_cast<float4*>(acq_out32 + base), make_float4(raw32(a4[0]), raw32(a4[1]), raw32(a4[2]), raw32(a4[3])));
      if (acq_out) {
#pragma unroll
        for (int q = 0; q < 4; q++) acq_out[base + q] = acq_raw(FA, (double)a4[q], ymean, ystd);
      }
      const float gm = fmaxf(fmaxf(a4[0], a4[1]), fmaxf(a4[2], a4[3]));   // fmaxf ignores NaN operands
      if ((VT)gm > tbest || tidx == 0x7fffffffffffffffLL) {
        const int q = a4[0] == gm ? 0 : a4[1] == gm ? 1 : a4[2] == gm ? 2 : a4[3] == gm ? 3 : -1;   // −1: all four are NaN
        if (q >= 0) {
          tbest = (VT)gm;
          tidx = base + q;
        }
      }
      return;
    }
    float o4[4];
#pragma unroll
    for (int q = 0; q < 4; q++) {
      double mu = 0.0, sd = 0.0;
      VT a;
      if (fast32) {
        const float fm = (float)m4[q], fv = (float)v4[q];
        a = (VT)acq_value_f32<FA>(fm, fv, fr);
        o4[q] = raw32((float)a);
      } else {
        a = (VT)acq_value<double>((double)m4[q], (double)v4[q], acq, ymean, ystd, yopt, xi, kappa, &mu, &sd);
        o4[q] = (float)a;
      }
      if (full || base + q < M) {
        if (!fast32) {
          if (mu_out) mu_out[base + q] = (double)mu;
          if (std_out) std_out[base + q] = (double)sd;
        }
        if (acq_out) acq_out[base + q] = fast32 ? acq_raw(FA, (double)a, ymean, ystd) : (double)a;
        if (a > tbest || (tidx == 0x7fffffffffffffffLL && a == a)) {  // NaN never wins; −inf can (all-hopeless grids)
          tbest = a;
          tidx = base + q;
        }
      }
    }
    if (acq_out32) {
      if (full) {
        __stcs(reinterpret_cast<float4*>(acq_out32 + base), make_float4(o4[0], o4[1], o4[2], o4[3]));
      } else {
        for (int q = 0; q < 4 && base + q < M; q++) acq_out32[base + q] = o4[q];
      }
    }
  };
  // software-pipelined stream: the loads of trip t+1 (two groups of 4 candidates, 4×16 B) are in flight while trip t is computed
  {
    int64_t base = ((int64_t)blockIdx.x * 256 + threadIdx.x) * 4;
    T ma[4], va[4], mb[4], vb[4];
    if (base < M) load4(base, ma, va);
    if (base + stride < M) load4(base + stride, mb, vb);
    while (base < M) {
      const int64_t nbase = base + 2 * stride;
      T na[4], nva[4], nb[4], nvb[4];
      if (nbase < M) load4(nbase, na, nva);
      if (nbase + stride < M) load4(nbase + stride, nb, nvb);
      process4(base, ma, va);
      if (base + stride < M) process4(base + stride, mb, vb);
#pragma unroll
      for (int q = 0; q < 4; q++) {
        ma[q] = na[q]; va[q] = nva[q]; mb[q] = nb[q]; vb[q] = nvb[q];
      }
      base = nbase;
    }
  }
  if (tidx != 0x7fffffffffffffffLL) {
    bv = (double)tbest;
    bi = goff + tidx;
  }
  // warp-shuffle argmax (lowest index wins ties), then across the 8 warps through shared memory
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (better(ov, oi, bv, bi)) {
      bv = ov;
      bi = oi;
    }
  }
  __shared__ double sv[8];
  __shared__ long long si[8];
  __shared__ unsigned int s_last;
  if ((threadIdx.x & 31) == 0) {
    sv[threadIdx.x >> 5] = bv;
    si[threadIdx.x >> 5] = bi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; w++)
      if (better(sv[w], si[w], bv, bi)) {
        bv = sv[w];
        bi = si[w];
      }
    partial[blockIdx.x].v = bv;
    partial[blockIdx.x].i = bi;
    __threadfence();
    s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (!s_last) return;
  // last block to finish: final reduce over the per-block partials (a max under a total order: order-independent)
  __threadfence();
  bv = -INFINITY;
  bi = 0x7fffffffffffffffLL;
  for (int e = threadIdx.x; e < (int)gridDim.x; e += 256) {
    const double pv = ((volatile BlockBest*)partial)[e].v;
    const long long pi = ((volatile BlockBest*)partial)[e].i;
    if (better(pv, pi, bv, bi)) {
      bv = pv;
      bi = pi;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (better(ov, oi, bv, bi)) {
      bv = ov;
      bi = oi;
    }
  }
  if ((threadIdx.x & 31) == 0) {
    sv[threadIdx.x >> 5] = bv;
    si[threadIdx.x >> 5] = bi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; w++)
      if (better(sv[w], si[w], bv, bi)) {
        bv = sv[w];
        bi = si[w];
      }
    best->value = fast32 && bv > -INFINITY ? acq_raw(FA, bv, ymean, ystd) : bv;   // no pick: −inf, whatever the y statistics
    best->index = bi;
    const int64_t l = bi - goff;
    if (l >= 0 && l < M) {
      const double var = (double)varn[l] > 0.0 ? (double)varn[l] : 0.0;
      best->mu = ystd * (double)mun[l] + ymean;
      best->std = sqrt(var * ystd * ystd);
    } else {
      best->mu = 0.0;
      best->std = 0.0;
    }
    *ticket = 0;  // re-arm for the next launch on this stream
  }
}

// ------------------------------------------------------------------------------------------------
// FP64 refinement of the suggestion in tensor-core mode.  The sweep's fp32 acquisition values carry the ~1e-6 error of the
// fp16×3 contraction; a near-tie could therefore pick a different index than the fp64 reference.  Every candidate whose
// (recomputed, bit-identical) fp32 value is within `delta` of the maximum is a contender: its row goes through the FP64
// K*/variance path again and the first-index argmax is taken over those FP64 values.  Contenders are a handful, so this is
// one pass plus a few small launches; the arrays returned for parity tests are not touched.
#define KBO_REFINE_CAP 4096
__global__ void __launch_bounds__(256)
contender_kernel(const float* __restrict__ mun, const float* __restrict__ varn, int64_t M, int acq, const double* __restrict__ scal, double xi,
                 double kappa, const kbo_best* __restrict__ best, int64_t goff, double delta, int* __restrict__ list, int* __restrict__ count) {
  const AcqFrame f = acq_frame(scal[S_YMEAN], scal[S_YSTD], scal[S_YOPT], xi, kappa);
  auto value = [&](int64_t i) {
    return acq == KBO_ACQ_EI    ? acq_value_f32<KBO_ACQ_EI>(mun[i], varn[i], f)
           : acq == KBO_ACQ_LCB ? acq_value_f32<KBO_ACQ_LCB>(mun[i], varn[i], f)
                                : acq_value_f32<KBO_ACQ_PI>(mun[i], varn[i], f);
  };
  // the window is centred on the pick's own normalised fp32 value (delta is in normalised units: delta·y_std raw); a pick
  // that is not the fp32 maximum only widens it.  No pick (every value NaN: the index is the sentinel): no window.
  const int64_t l = best->index - goff;
  const float thr = (l >= 0 && l < M) ? value(l) - (float)delta : INFINITY;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < M; i += (int64_t)gridDim.x * 256) {
    const float a = value(i);
    if (a >= thr || (l >= 0 && l < M && !(mun[i] == mun[i] && varn[i] == varn[i]))) {   // a NaN mean or variance is never pruned
      const int slot = atomicAdd(count, 1);
      if (slot < KBO_REFINE_CAP) list[slot] = (int)i;
    }
  }
}
template <typename XT>
__global__ void gather_rows_kernel(const XT* __restrict__ Xc, int D, const int* __restrict__ list, int n, double* __restrict__ Xg) {
  const int r = blockIdx.x;
  if (r >= n) return;
  const int64_t src = list[r];
  for (int d = threadIdx.x; d < D; d += blockDim.x) Xg[(size_t)r * D + d] = (double)Xc[src * D + d];
}
// The FP64 decision of up to three acquisitions over the UNION of their survivors: the union's rows (uidx, ascending) carry
// FP64 mean / variance evaluated once; acquisition k takes the first-index argmax over its own survivors, pos[off_k .. off_k+n_k)
// (ascending positions into the union).  One CTA per acquisition.
struct UnionPick {
  int nk;
  int acq[3], off[3], n[3];
  kbo_best* best[3];
};
__global__ void __launch_bounds__(1024)
refine_best_union_kernel(const double* __restrict__ mun, const double* __restrict__ varn, const int* __restrict__ uidx, const int* __restrict__ pos,
                         UnionPick up, const double* __restrict__ scal, double xi, double kappa, int64_t goff) {
  __shared__ double sv[1024];
  __shared__ int sp[1024];
  const int k = blockIdx.x;   // selects, not a dynamic index: the parameter block stays out of local memory
  const int acq = k == 0 ? up.acq[0] : k == 1 ? up.acq[1] : up.acq[2];
  const int n = k == 0 ? up.n[0] : k == 1 ? up.n[1] : up.n[2];
  const int* ps = pos + (k == 0 ? up.off[0] : k == 1 ? up.off[1] : up.off[2]);
  kbo_best* best = k == 0 ? up.best[0] : k == 1 ? up.best[1] : up.best[2];
  const double ym = scal[S_YMEAN], ys = scal[S_YSTD], yo = scal[S_YOPT];
  double bv = -INFINITY;
  int bp = 0x7fffffff;
  for (int p = threadIdx.x; p < n; p += 1024) {
    double mu, sd;
    const double a = acq_value<double>(mun[ps[p]], varn[ps[p]], acq, ym, ys, yo, xi, kappa, &mu, &sd);
    if (a > bv || (bp == 0x7fffffff && a == a)) {   // positions only grow inside a thread: first maximum kept
      bv = a;
      bp = p;
    }
  }
  sv[threadIdx.x] = bv;
  sp[threadIdx.x] = bp;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      const double ov = sv[threadIdx.x + o];
      const int op = sp[threadIdx.x + o];
      if (ov > sv[threadIdx.x] || (ov == sv[threadIdx.x] && op < sp[threadIdx.x])) {
        sv[threadIdx.x] = ov;
        sp[threadIdx.x] = op;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0 && sp[0] == 0x7fffffff) {   // every FP64 value NaN: what acq_kernel reports when nothing is picked
    best->value = -INFINITY;
    best->index = 0x7fffffffffffffffLL;
    best->mu = 0.0;
    best->std = 0.0;
  }
  if (threadIdx.x == 0 && sp[0] != 0x7fffffff) {
    const int q = ps[sp[0]];
    double mu, sd;
    const double a = acq_value<double>(mun[q], varn[q], acq, ym, ys, yo, xi, kappa, &mu, &sd);
    best->value = a;
    best->index = goff + uidx[q];
    best->mu = mu;
    best->std = sd;
  }
}

// K* row of a contender in FP64, one thread per (contender, trial): scaled differences summed in d order, exact kernel
__global__ void __launch_bounds__(256)
refine_cross_kernel(const double* __restrict__ Xg, int D, const double* __restrict__ inv_ls, int n_ls, const double* __restrict__ XsT, int ld,
                    int N, int kind, double amp, double* __restrict__ Ks) {
  __shared__ double xs[512];
  const int c = blockIdx.y;
  for (int d = threadIdx.x; d < D; d += 256) xs[d] = Xg[(size_t)c * D + d] * inv_ls[n_ls == 1 ? 0 : d];
  __syncthreads();
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= N) return;
  double d2 = 0.0;
  for (int d = 0; d < D; d++) {
    const double df = xs[d] - XsT[(size_t)d * ld + j];
    d2 = fma(df, df, d2);
  }
  Ks[(size_t)c * ld + j] = amp * kbo_kernel_exact(d2, kind);
}
// normalised mean K*·alpha of one contender per CTA, fixed-order reduction
__global__ void __launch_bounds__(256)
refine_mu_kernel(const double* __restrict__ Ks, int ld, int N, const double* __restrict__ alpha, double* __restrict__ mun) {
  __shared__ double red[256];
  const double* k = Ks + (size_t)blockIdx.x * ld;
  double a = 0.0;
  for (int j = threadIdx.x; j < N; j += 256) a = fma(k[j], alpha[j], a);
  red[threadIdx.x] = a;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) mun[blockIdx.x] = red[0];
}
// Σ_i (W k*)_i² for a handful of contender rows: CTA (bx, by) takes W rows [8·bx, 8·bx+8) and contenders [C·by, C·by+C);
// a warp owns one W row, lanes stride the columns, butterfly reduction — the summation order depends on neither
// the contender's position nor their number, so a candidate's refined value is bit-reproducible however the grid is sharded.
template <int KBO_RV_C>
__global__ void __launch_bounds__(256)
refine_var_kernel(const double* __restrict__ W, int ld, int N, const double* __restrict__ Ks, int n, double* __restrict__ part, int nblk) {
  __shared__ double ssq[8][KBO_RV_C];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.y * KBO_RV_C;
  const double* ks[KBO_RV_C];
#pragma unroll
  for (int c = 0; c < KBO_RV_C; c++) ks[c] = Ks + (size_t)min(c0 + c, n - 1) * ld;
  double sq[KBO_RV_C];
#pragma unroll
  for (int c = 0; c < KBO_RV_C; c++) sq[c] = 0.0;
  const int i = blockIdx.x * 8 + warp;   // one W row per warp: N/8 CTAs keep enough loads in flight to stream the triangle
  if (i < N) {
    const double* w = W + (size_t)i * ld;
    double acc[KBO_RV_C];
#pragma unroll
    for (int c = 0; c < KBO_RV_C; c++) acc[c] = 0.0;
#pragma unroll 8
    for (int j = lane; j <= i; j += 32) {
      const double wv = w[j];
#pragma unroll
      for (int c = 0; c < KBO_RV_C; c++) acc[c] = fma(wv, ks[c][j], acc[c]);
    }
#pragma unroll
    for (int c = 0; c < KBO_RV_C; c++) {
      double v = acc[c];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      sq[c] = v * v;
    }
  }
  if (lane == 0)
#pragma unroll
    for (int c = 0; c < KBO_RV_C; c++) ssq[warp][c] = sq[c];
  __syncthreads();
  if (threadIdx.x < KBO_RV_C && c0 + threadIdx.x < n) {
    double t = 0.0;
    for (int w8 = 0; w8 < 8; w8++) t += ssq[w8][threadIdx.x];
    part[(size_t)(c0 + threadIdx.x) * nblk + blockIdx.x] = t;
  }
}

static int acq_grid(kbo_handle* h, int64_t M) {
  int64_t g = (M + 2047) / 2048;   // two groups of 4 candidates per thread per trip (1024 per CTA measured slower at 1M: more partials/atomics)
  const int64_t cap = (int64_t)h->sm_count * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

template <typename T>
static int launch_acq(kbo_handle* h, const T* mun, const T* varn, int64_t M, int64_t goff, int acq, double ymean, double ystd, double yopt,
                      const double* scal_dev, double xi, double kappa, double* mu_out, double* std_out, double* acq_out, float* acq_out32, kbo_best* best_dev,
                      cudaStream_t s) {
  const int g = acq_grid(h, M);
  if (h->blockbest.cap == 0) {
    KBO_TRY(kbo_reserve(h, h->blockbest, (size_t)h->sm_count * 8 + 4));
    KBO_CUDA(h, cudaMemsetAsync(h->blockbest.p, 0, sizeof *h->blockbest.p * h->blockbest.cap, s));
  }
  // the last-block ticket lives in the 64 bytes past the partials (BlockBest entries are 16-byte aligned)
  unsigned int* ticket = reinterpret_cast<unsigned int*>(h->blockbest.p + (size_t)h->sm_count * 8);
#define KBO_ACQ_LAUNCH(FA)                                                                                                     \
  acq_kernel<T, FA><<<g, 256, 0, s>>>(mun, varn, M, goff, acq, ymean, ystd, yopt, scal_dev, xi, kappa, mu_out, std_out, acq_out, \
                                      acq_out32, h->blockbest.p, ticket, best_dev)
  if (sizeof(T) == 4 && !mu_out && !std_out) {
    if (acq == KBO_ACQ_EI) KBO_ACQ_LAUNCH(KBO_ACQ_EI);
    else if (acq == KBO_ACQ_LCB) KBO_ACQ_LAUNCH(KBO_ACQ_LCB);
    else KBO_ACQ_LAUNCH(KBO_ACQ_PI);
  } else {
    KBO_ACQ_LAUNCH(-1);
  }
#undef KBO_ACQ_LAUNCH
  KBO_LAUNCH_CHECK(h);
  return KBO_OK;
}

int kbo_i_acq_argmax_f32(kbo_handle* h, const float* mu_n, const float* var_n, int64_t M, int64_t goff, int acq, double y_mean,
                         double y_std, double y_opt, double xi, double kappa, double amp, float* acq_out, kbo_best* best_dev,
                         cudaStream_t s) {
  (void)amp;
  if (M < 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_acq_argmax: M must be >= 1");
  if (((uintptr_t)mu_n | (uintptr_t)var_n | (uintptr_t)acq_out) & 15) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_acq_argmax: pointers must be 16-byte aligned");
  return launch_acq<float>(h, mu_n, var_n, M, goff, acq, y_mean, y_std, y_opt, nullptr, xi, kappa, nullptr, nullptr, nullptr, acq_out, best_dev, s);
}

// ------------------------------------------------------------------------------------------------
static size_t cross_smem_bytes(int D, int mode) {
  const int Dp = (D + CM_DC - 1) / CM_DC * CM_DC;
  size_t b = sizeof(double) * ((size_t)Dp * 130 + 2 * CM_DC * 66 + CM_BM + 4 * CM_BN);
  (void)mode;
  return b;
}

template <typename XT, typename MT, int MODE>
static int launch_cross(kbo_handle* h, const XT* Xc, int64_t rows, int64_t rows_grid, double* Ks64, int ldks, __half* Ksh, __half* Ksl, MT* mun,
                        cudaStream_t s) {
  const size_t smem = cross_smem_bytes(h->D, MODE);
  KBO_CUDA(h, cudaFuncSetAttribute(cross_mean_kernel<XT, MT, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const unsigned gx = (unsigned)((rows_grid + CM_BM - 1) / CM_BM);
  // fewer CTAs than one wave (two per SM): split the trial tiles so every SM works — the 74 CTAs of the calibration rows left half
  // of the GPU idle
  const int ntiles = (h->N + CM_BN - 1) / CM_BN;
  int nsplit = 1;
  if (gx < 2u * h->sm_count) nsplit = (int)min((unsigned)min(ntiles, 16), max(1u, 2u * h->sm_count / gx));
  double* part = nullptr;
  if (nsplit > 1) {
    KBO_TRY(kbo_reserve(h, h->mu_part, (size_t)nsplit * rows));
    part = h->mu_part.p;
  }
  cross_mean_kernel<XT, MT, MODE><<<dim3(gx, nsplit), 256, smem, s>>>(
      Xc, rows, h->D, h->d_inv_ls.p, (int)h->inv_ls.size(), h->XsT.p, h->ld, h->nx.p, h->N,
      h->alpha.p, h->prm.kernel, h->prm.amplitude, Ks64, ldks, Ksh, Ksl, h->Npad, mun, part);
  KBO_LAUNCH_CHECK(h);
  if (nsplit > 1) {
    mu_parts_kernel<MT><<<(unsigned)((rows + 255) / 256), 256, 0, s>>>(part, rows, nsplit, mun);
    KBO_LAUNCH_CHECK(h);
  }
  return KBO_OK;
}

static cudaEvent_t* ev_pair(kbo_handle* h, std::vector<std::pair<cudaEvent_t, cudaEvent_t>>& v, size_t& used) {
  if (used == v.size()) {
    std::pair<cudaEvent_t, cudaEvent_t> p;
    cudaEventCreate(&p.first);
    cudaEventCreate(&p.second);
    v.push_back(p);
  }
  return &v[used++].first;
}
#define KBO_TIME_BEGIN(vec, used)                      \
  cudaEvent_t* _ev = nullptr;                          \
  if (h->time_kernels) {                               \
    _ev = ev_pair(h, h->vec, h->used);                 \
    cudaEventRecord(_ev[0], s);                        \
  }
#define KBO_TIME_END()                                 \
  if (_ev) cudaEventRecord((&_ev[0])[1], s);

#define KBO_SOLVE_CAP 256   // survivors a lazy fit evaluates by triangular solves with L before it forms the rest of L⁻¹ instead

// One acquisition's way through the stages of a sweep.  kbo_sweep decides one; kbo_sweep_multi several over one posterior, each
// leaving at the first stage where its own survivor list fits its cap — the stage its single sweep would have decided at.
struct AcqDecision {
  int acq;
  kbo_best* best;
  bool done;
  int unrefined, contenders, prefix_survivors;   // what kbo_last_unrefined / _contenders / _prefix_survivors report for it
};

// The survivors of the acquisitions a stage decides, collected on the host (each list is read back once its count is known,
// before the next acquisition reuses the device list) and evaluated together by refine_union.
struct StagePicks {
  int nk = 0;
  AcqDecision* d[3];
  std::vector<int> list[3];
};
static int take_list(kbo_handle* h, StagePicks& sp, AcqDecision& d, const int* list_dev, int n, cudaStream_t s) {
  std::vector<int>& l = sp.list[sp.nk];
  l.resize(n);
  KBO_CUDA(h, cudaMemcpyAsync(l.data(), list_dev, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  sp.d[sp.nk++] = &d;
  return KBO_OK;
}

// FP64 decision of every acquisition in sp over the UNION of their survivor lists: K*, mean and variance of each union row are
// evaluated once (a candidate's FP64 values depend on neither its position nor the number of rows evaluated with it — see
// refine_var_kernel and the panel solves), then each acquisition takes the first-index argmax over its own survivors.  A lazy
// fit evaluates the variance by panel solves with L in groups, whatever the union's size: it never forms W here.
#define KBO_UNION_BATCH 4096   // union rows per K* / variance batch
static int refine_union(kbo_handle* h, const void* Xc, int xc_dtype, int64_t goff, StagePicks& sp, cudaStream_t s) {
  if (sp.nk == 0) return KBO_OK;
  const int N = h->N, D = h->D, ld = h->ld;
  std::vector<int> U;
  for (int k = 0; k < sp.nk; k++) {
    std::sort(sp.list[k].begin(), sp.list[k].end());   // ascending indices: first maximum = lowest index
    U.insert(U.end(), sp.list[k].begin(), sp.list[k].end());
  }
  std::sort(U.begin(), U.end());
  U.erase(std::unique(U.begin(), U.end()), U.end());
  const int nu = (int)U.size();
  UnionPick up{};
  up.nk = sp.nk;
  std::vector<int> host(U);   // [union indices][positions of acquisition 0][... 1][... 2]
  for (int k = 0; k < sp.nk; k++) {
    up.acq[k] = sp.d[k]->acq;
    up.best[k] = sp.d[k]->best;
    up.off[k] = (int)host.size() - nu;
    up.n[k] = (int)sp.list[k].size();
    for (int idx : sp.list[k]) host.push_back((int)(std::lower_bound(U.begin(), U.end(), idx) - U.begin()));
  }
  KBO_TRY(kbo_reserve(h, h->un_idx, host.size()));
  KBO_TRY(kbo_reserve(h, h->un_mv, (size_t)nu * 2));
  int* uidx = h->un_idx.p;
  double* mun64 = h->un_mv.p;
  double* varn64 = mun64 + nu;
  KBO_CUDA(h, cudaMemcpyAsync(uidx, host.data(), sizeof(int) * host.size(), cudaMemcpyHostToDevice, s));
  const int njt = (N + 7) / 8;   // row blocks of refine_var_kernel (8 rows of W per CTA)
  for (int b0 = 0; b0 < nu; b0 += KBO_UNION_BATCH) {
    const int m = nu - b0 < KBO_UNION_BATCH ? nu - b0 : KBO_UNION_BATCH;
    KBO_TRY(kbo_reserve(h, h->refine_x, (size_t)m * D));
    KBO_TRY(kbo_reserve(h, h->Ks64, (size_t)m * ld));
    KBO_TRY(kbo_reserve(h, h->part, (size_t)m * njt));
    double* Xg = h->refine_x.p;
    if (xc_dtype == KBO_F64)
      gather_rows_kernel<double><<<m, 64, 0, s>>>((const double*)Xc, D, uidx + b0, m, Xg);
    else
      gather_rows_kernel<float><<<m, 64, 0, s>>>((const float*)Xc, D, uidx + b0, m, Xg);
    KBO_LAUNCH_CHECK(h);
    refine_cross_kernel<<<dim3((N + 255) / 256, m), 256, 0, s>>>(Xg, D, h->d_inv_ls.p, (int)h->inv_ls.size(), h->XsT.p, ld, N,
                                                                 h->prm.kernel, h->prm.amplitude, h->Ks64.p);
    KBO_LAUNCH_CHECK(h);
    refine_mu_kernel<<<m, 256, 0, s>>>(h->Ks64.p, ld, N, h->alpha.p, mun64 + b0);
    KBO_LAUNCH_CHECK(h);
    if (!h->w_full) {
      // lazy inverse: ‖L⁻¹k*‖² by panel solves with the factor itself (solve.cu) — no W
      KBO_TRY(kbo_i_variance_by_solves(h, h->Ks64.p, m, varn64 + b0, s));
    } else {
      if (m <= 2)   // the usual case: one contender — no point carrying eight accumulators through the triangle of W
        refine_var_kernel<1><<<dim3(njt, m), 256, 0, s>>>(h->W.p, ld, N, h->Ks64.p, m, h->part.p, njt);
      else
        refine_var_kernel<8><<<dim3(njt, (m + 7) / 8), 256, 0, s>>>(h->W.p, ld, N, h->Ks64.p, m, h->part.p, njt);
      KBO_LAUNCH_CHECK(h);
      var_from_parts_kernel<<<(m + 255) / 256, 256, 0, s>>>(h->part.p, m, njt, h->prm.amplitude, varn64 + b0);
      KBO_LAUNCH_CHECK(h);
    }
  }
  refine_best_union_kernel<<<sp.nk, 1024, 0, s>>>(mun64, varn64, uidx, uidx + nu, up, h->scal.p, h->prm.xi, h->prm.kappa, goff);
  KBO_LAUNCH_CHECK(h);
  // the host copies above must outlive the asynchronous H2D copy
  KBO_CUDA(h, cudaStreamSynchronize(s));
  for (int k = 0; k < sp.nk; k++) sp.d[k]->done = true;
  sp.nk = 0;
  return KBO_OK;
}

// Test hook (kbo_debug_record_stages): one stage's bounds (fs[] as the stage's survivor kernel read it) and its survivor list.
// Off by default; when off, nothing is read back and the sweep's launches and synchronisation are unchanged.
enum { KBO_STAGE_LAZY_PRUNE = 0, KBO_STAGE_PRUNE = 1, KBO_STAGE_PRUNE_INTERVAL = 2, KBO_STAGE_INTERVAL = 3, KBO_STAGE_WINDOW = 4 };
static int record_stage(kbo_handle* h, int stage, int acq, int cal_n, const float* fs_dev, const int* count_dev, const int* list_dev, int cap,
                        float delta, cudaStream_t s) {
  if (!h->record_stages) return KBO_OK;
  kbo_handle::StageRec r{};
  r.stage = stage;
  r.acq = acq;
  r.cal_n = cal_n;
  float fs[5];
  for (float& v : fs) v = NAN;
  if (fs_dev) KBO_CUDA(h, cudaMemcpyAsync(fs, fs_dev, sizeof fs, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaMemcpyAsync(&r.n, count_dev, sizeof(int), cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  r.list.resize(r.n < cap ? r.n : cap);
  if (!r.list.empty()) {
    KBO_CUDA(h, cudaMemcpyAsync(r.list.data(), list_dev, sizeof(int) * r.list.size(), cudaMemcpyDeviceToHost, s));
    KBO_CUDA(h, cudaStreamSynchronize(s));
  }
  float lb = NAN;
  if (fs_dev) {   // from_ordered_bits on the host; 0 (no bound set) decodes to NaN, as the survivor kernels read it
    unsigned u;
    memcpy(&u, &fs[1], sizeof u);
    u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
    memcpy(&lb, &u, sizeof lb);
  }
  const float f[7] = {fs[0], fs[3], fs[2], fs[4], lb, lb - 1e-5f * fmaxf(1.f, fabsf(lb)), delta};
  for (int k = 0; k < 7; k++) r.f[k] = f[k];
  h->stage_recs.push_back(std::move(r));
  return KBO_OK;
}

// contenders of the three-product sweep's window (see below) for one acquisition; a list that fits is handed to sp
static int refine_suggestion(kbo_handle* h, int64_t M, int64_t goff, AcqDecision& d, StagePicks& sp, cudaStream_t s) {
  const double* scal = h->scal.p;
  KBO_TRY(kbo_reserve(h, h->refine, KBO_REFINE_CAP + 16));
  int* list = h->refine.p;
  int* count = list + KBO_REFINE_CAP;
  // contenders: within delta of the fp32 maximum, in normalised units (2e-4·y_std on the raw scale; for LCB the raw value is
  // ≈ −y_mean, whose fp32 ulp alone can exceed any absolute window).  2e-4 is ≥ 10× the tensor-core mode's acquisition error
  // bound; when more than the cap lie inside it (a flat landscape, or a late-stage experiment whose best EI is itself below 2e-4·y_std) the window is
  // narrowed until the cap holds and the FP64 decision is taken among the best by fp32 value (last_unrefined = 1); only
  // exact fp32 ties beyond the cap — e.g. thousands of identical candidates — keep the tensor-core pick (last_unrefined = 2),
  // which is then the lowest index among them, as the reference's argmin is.
  double delta = 2e-4;
  int n = 0, first_n = 0;
  d.unrefined = 0;
  for (int round = 0; round < 24; round++) {
    KBO_CUDA(h, cudaMemsetAsync(count, 0, sizeof(int), s));
    contender_kernel<<<acq_grid(h, M), 256, 0, s>>>(kbo_view<float>(h->mun), kbo_view<float>(h->varn), M, d.acq, scal, h->prm.xi, h->prm.kappa,
                                                    d.best, goff, delta, list, count);
    KBO_LAUNCH_CHECK(h);
    KBO_CUDA(h, cudaMemcpyAsync(&n, count, sizeof(int), cudaMemcpyDeviceToHost, s));
    KBO_CUDA(h, cudaStreamSynchronize(s));
    if (round == 0) first_n = n;
    if (n <= KBO_REFINE_CAP) break;
    d.unrefined = 1;
    delta = round < 22 ? delta * 0.25 : 0.0;   // the last attempt: exact ties of the maximum only
  }
  d.contenders = first_n;
  KBO_TRY(record_stage(h, KBO_STAGE_WINDOW, d.acq, 0, nullptr, count, list, KBO_REFINE_CAP, (float)delta, s));
  if (n < 1 || n > KBO_REFINE_CAP) {
    d.unrefined = 2;
    d.done = true;   // keeps the tensor-core pick
    return KBO_OK;
  }
  return take_list(h, sp, d, list, n, s);
}

// ------------------------------------------------------------------------------------------------
// Ranking pass with ONE fp16 product (kbo_set_tc_fast, default on for array-free tensor-core sweeps).  With the suggestion
// decided in FP64 by the refinement, the sweep only has to RANK: keep every candidate that could still be the maximum given
// the error of a cheaper variance.  The pass computes Σv² with the hi planes alone (a third of the MMAs, half the bytes);
// its error bound E on σ² is calibrated per sweep against the three-product kernel on the first wave of rows (8× the largest
// difference seen + 1e-6).  Candidate i survives iff  max(acq(μ_i, σ²_i ± E)) ≥ max_j min(acq(μ_j, σ²_j ± E)) − slack  — EI
// and LCB grow with σ, PI is monotone either way, so the two ends bound the value over the interval.  Survivors (typically a
// handful: EI is sharply peaked) go through the FP64 refinement; more than 4096 of them and the sweep is redone with the
// three-product kernel.
__device__ __forceinline__ float acq_any_f32(int acq, float mu, float var, const AcqFrame& f) {
  return acq == KBO_ACQ_EI    ? acq_value_f32<KBO_ACQ_EI>(mu, var, f)
         : acq == KBO_ACQ_LCB ? acq_value_f32<KBO_ACQ_LCB>(mu, var, f)
                              : acq_value_f32<KBO_ACQ_PI>(mu, var, f);
}
__device__ __forceinline__ unsigned ordered_bits(float v) {   // monotone float -> uint
  const unsigned b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float from_ordered_bits(unsigned u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u); }
// the calibration maxima propagate NaN (fmaxf drops it): a NaN error must not leave a tight bound behind.  A NaN E or Eμ makes
// every bound NaN, so no lower bound is found, nothing is pruned and the sweep falls back to three products / the FP64 path.
__device__ __forceinline__ float max_nan(float a, float b) { return (a != a || a > b) ? a : b; }

// Calibration of the ranking pass on STRATIFIED rows: row i·M/n of the grid, i < n (n = one wave of the variance kernel, or all
// rows of a small grid), so a sorted / clustered / blocked candidate order is sampled across its whole extent.  Those rows went
// through the FP64 K* kernel and the three-product contraction (v_ex, mu_ex); v_rk / mu_rk are the ranking arithmetic's values,
// of the whole grid (row idx[i] goes with calibration row i) or, idx = nullptr, of the calibration rows themselves.
// fs[0] = E (bound on |σ̃² − σ²|), fs[1] (as uint) = ordered bits of the best lower bound, fs[2] = raw max |dσ²|,
// fs[3] = Eμ (bound on |μ̃ − μ|, normalised units), fs[4] = raw max |dμ|.  acq < 0: the lower bound is reset below every ordered
// value; otherwise it is the best value of that acquisition on the calibration rows, less their own error.
__global__ void cal_index_kernel(int* __restrict__ list, int n, int64_t M) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) list[i] = (int)(((int64_t)i * M) / n);
}
__global__ void __launch_bounds__(1024)
calib_kernel(const float* __restrict__ v_rk, const float* __restrict__ v_ex, const float* __restrict__ mu_rk, const float* __restrict__ mu_ex,
             const int* __restrict__ idx, int n, int acq, const double* __restrict__ scal, double xi, double kappa, float* __restrict__ fs) {
  __shared__ float red[1024], redm[1024], redl[1024];
  const AcqFrame f = acq >= 0 ? acq_frame(scal[S_YMEAN], scal[S_YSTD], scal[S_YOPT], xi, kappa) : AcqFrame{};
  float m = 0.f, mm = 0.f, lb = -INFINITY;
  for (int i = threadIdx.x; i < n; i += 1024) {
    const int g = idx ? idx[i] : i;
    m = max_nan(m, fabsf(v_rk[g] - v_ex[i]));
    mm = max_nan(mm, fabsf(mu_rk[g] - mu_ex[i]));
    if (acq >= 0) {
      const float a = acq_any_f32(acq, mu_ex[i], v_ex[i], f);   // three-product value: |error| ~ 1e-6
      if (a > lb) lb = a;
    }
  }
  red[threadIdx.x] = m;
  redm[threadIdx.x] = mm;
  redl[threadIdx.x] = lb;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      red[threadIdx.x] = max_nan(red[threadIdx.x], red[threadIdx.x + o]);
      redm[threadIdx.x] = max_nan(redm[threadIdx.x], redm[threadIdx.x + o]);
      redl[threadIdx.x] = fmaxf(redl[threadIdx.x], redl[threadIdx.x + o]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    fs[0] = 8.f * red[0] + 1e-6f;
    fs[2] = red[0];
    fs[3] = 8.f * redm[0] + 1e-7f;
    fs[4] = redm[0];
    const float l = redl[0] - 2e-5f * fmaxf(1.f, fabsf(redl[0]));   // the calibration values' own error, generously
    ((unsigned*)fs)[1] = acq >= 0 && l > -INFINITY ? ordered_bits(l) : 0u;   // 0: below every ordered value
  }
}
// Bounds of the acquisition value over the box (μ ± Eμ) × (σ² ± E): all three kinds fall with μ; EI and LCB grow with σ, PI is
// monotone in σ either way — so the corners bound the value.
// A NaN mean, variance, E or Eμ gives NaN bounds (the clamps and maxima below would drop it and bound at σ = 0): a NaN upper
// bound survives every interval test, a NaN lower bound never enters the maximum.
__device__ __forceinline__ void acq_bounds_f32(int acq, float mu, float var, float E, float Em, const AcqFrame& f,
                                               float* lb, float* ub) {
  if (!(mu == mu && var == var && E == E && Em == Em)) {
    *lb = *ub = __int_as_float(0x7fc00000);
    return;
  }
  const float vlo = fmaxf(var - E, 0.f), vhi = var + E;
  const float u0 = acq_any_f32(acq, mu - Em, vlo, f), u1 = acq_any_f32(acq, mu - Em, vhi, f);
  const float l0 = acq_any_f32(acq, mu + Em, vlo, f), l1 = acq_any_f32(acq, mu + Em, vhi, f);
  *ub = fmaxf(u0, u1);
  *lb = fminf(l0, l1);
  // PI where the box reaches σ = 0: acq_value_f32 gives 0 there, but Φ(imp/σ) → 1 as σ → 0 with a positive improvement — that
  // supremum (as in acq_prefix_ub_f32), or a saturated PI near a trial would be pruned below a maximum of 1
  if (acq == KBO_ACQ_PI && !(vlo > 0.f) && (f.chi - (mu - Em)) + f.clo > 0.f) *ub = 1.f;
}
// The interval test: the best lower bound over the M rows (the whole grid, or the pruning pass's survivors), then the rows whose
// upper bound can still reach it — src[i] is row i's index in the grid (nullptr: i itself)
__global__ void __launch_bounds__(256)
bound_max_kernel(const float* __restrict__ mun, const float* __restrict__ varn, int64_t M, int acq, const double* __restrict__ scal, double xi,
                 double kappa, float* __restrict__ fs) {
  const AcqFrame f = acq_frame(scal[S_YMEAN], scal[S_YSTD], scal[S_YOPT], xi, kappa);
  const float E = fs[0], Em = fs[3];
  float best = -INFINITY;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < M; i += (int64_t)gridDim.x * 256) {
    float lb, ub;
    acq_bounds_f32(acq, mun[i], varn[i], E, Em, f, &lb, &ub);
    if (lb > best) best = lb;   // NaN never enters
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0 && best > -INFINITY) atomicMax((unsigned*)fs + 1, ordered_bits(best));
}
__global__ void __launch_bounds__(256)
survivor_kernel(const float* __restrict__ mun, const float* __restrict__ varn, const int* __restrict__ src, int64_t M, int acq,
                const double* __restrict__ scal, double xi, double kappa, const float* __restrict__ fs, int* __restrict__ list, int* __restrict__ count) {
  const AcqFrame f = acq_frame(scal[S_YMEAN], scal[S_YSTD], scal[S_YOPT], xi, kappa);
  const float E = fs[0], Em = fs[3];
  const float lbmax = from_ordered_bits(((const unsigned*)fs)[1]);
  const float thr = lbmax - 1e-5f * fmaxf(1.f, fabsf(lbmax));   // fp32 evaluation and fp32 storage of μ
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < M; i += (int64_t)gridDim.x * 256) {
    float lb, ub;
    acq_bounds_f32(acq, mun[i], varn[i], E, Em, f, &lb, &ub);
    if (!(ub < thr)) {   // NaN survives
      const int slot = atomicAdd(count, 1);
      if (slot < KBO_REFINE_CAP) list[slot] = src ? src[i] : (int)i;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Pruning pass (kbo_set_rank_prefix).  sigma² = amp − Σ_j v_j² with every v_j² >= 0, so the sum over a PREFIX of the trial
// tiles gives an upper bound on sigma² — and EI / LCB grow with sigma, so acq(mu, sigma²_prefix) bounds the acquisition value
// from above at the prefix's share of the triangular contraction (the first eighth of the trials: 1/64 of the MMAs).  A lower
// bound on the maximum comes for free: the calibration rows carry (near-)exact values.  Every candidate whose upper bound stays
// below it is out; the few that remain (tens to hundreds of a million on the workload of record — EI is decided by the mean
// far more than by sigma) get the full contraction, the interval test of the ranking pass and the FP64 decision, exactly as
// before.  A landscape too flat to prune this way falls back to the full ranking pass over the grid.
//   fs[0] = E, fs[1] = ordered bits of the lower bound on the maximum, fs[2] = raw max |d sigma²|, fs[3] = Emu, fs[4] = raw max |d mu|
// supremum of the acquisition value over mu in [mu ± Em], sigma² in (0, var_ub]
__device__ __forceinline__ float acq_prefix_ub_f32(int acq, float mu, float var_ub, float Em, const AcqFrame& f) {
  if (!(mu == mu && var_ub == var_ub && Em == Em)) return __int_as_float(0x7fc00000);   // NaN: survives
  if (acq == KBO_ACQ_PI) {   // Φ(imp/σ): falls with σ where imp > 0 — its supremum there is 1
    const float imp = (f.chi - (mu - Em)) + f.clo;
    if (imp > 0.f) return 1.f;
  }
  return acq_any_f32(acq, mu - Em, var_ub, f);
}
__global__ void __launch_bounds__(256)
prefix_survivor_kernel(const float* __restrict__ mun, const float* __restrict__ var_ub, int64_t M, int acq, const double* __restrict__ scal, double xi,
                       double kappa, const float* __restrict__ fs, int* __restrict__ list, int* __restrict__ count, int cap) {
  const AcqFrame f = acq_frame(scal[S_YMEAN], scal[S_YSTD], scal[S_YOPT], xi, kappa);
  const float E = fs[0], Em = fs[3];
  const float lb = from_ordered_bits(((const unsigned*)fs)[1]);
  const float thr = lb - 1e-5f * fmaxf(1.f, fabsf(lb));
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < M; i += (int64_t)gridDim.x * 256) {
    const float v = var_ub[i];
    const float ub = acq_prefix_ub_f32(acq, mun[i], v == v ? fmaxf(v, 0.f) + E : v, Em, f);
    if (!(ub < thr)) {   // NaN survives
      const int slot = atomicAdd(count, 1);
      if (slot < cap) list[slot] = (int)i;
    }
  }
}

static int calibration_rows(kbo_handle* h, const void* Xc, int xc_dtype, int64_t M, int* cal_n_out, cudaStream_t s, int jtiles = -1);

// lower bound of the acquisition value over sigma² in (0, var_ub] at mean mu_n (normalised): EI and LCB grow with sigma, so the
// bound is their sigma -> 0 limit (max(improvement, 0) and −mu: no variance needed at all); PI falls with sigma where the
// improvement is positive, so its bound there sits at var_ub
__device__ __forceinline__ float acq_lower_f32(int acq, float mu_n, float var_ub, const AcqFrame& f) {
  if (acq == KBO_ACQ_LCB) return -mu_n;
  const float imp = (f.chi - mu_n) + f.clo;
  if (acq == KBO_ACQ_EI) return fmaxf(imp, 0.f);
  return imp > 0.f ? acq_any_f32(acq, mu_n, var_ub, f) : 0.f;
}
__global__ void __launch_bounds__(256)
grid_lower_bound_kernel(const float* __restrict__ mun, const float* __restrict__ var_ub, int64_t M, int acq, const double* __restrict__ scal, double xi,
                        double kappa, float* __restrict__ fs) {
  const AcqFrame f = acq_frame(scal[S_YMEAN], scal[S_YSTD], scal[S_YOPT], xi, kappa);
  const float E = fs[0], Em = fs[3];
  if (!(E == E && Em == Em)) return;   // no bound from a NaN calibration: the lower bound stays unset and nothing is pruned
  float best = -INFINITY;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < M; i += (int64_t)gridDim.x * 256) {
    const float m = mun[i], v = var_ub[i];
    if (!(m == m && v == v)) continue;
    const float lb = acq_lower_f32(acq, m + Em, fmaxf(v, 0.f) + E, f);
    if (lb > best) best = lb;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0 && best > -INFINITY) atomicMax((unsigned*)fs + 1, ordered_bits(best - 1e-5f * fmaxf(1.f, fabsf(best))));
}

#define KBO_PRUNE_CAP 16384
// The grid pass of the pruning sweeps: per chunk, the mean over all trials and the variance bound from the first P1 tile pairs
// (only their 512·P1 columns of K̃* are stored).
static int prefix_grid_pass(kbo_handle* h, const void* Xc, int xc_dtype, int64_t M, int64_t chunk, int P1, cudaStream_t s) {
  const size_t esz = xc_dtype == KBO_F64 ? 8 : 4;
  for (int64_t c0 = 0; c0 < M; c0 += chunk) {
    const int64_t rows = (M - c0 < chunk) ? (M - c0) : chunk;
    const unsigned char* xc = (const unsigned char*)Xc + (size_t)c0 * h->D * esz;
    h->tim.chunks++;
    {
      KBO_TIME_BEGIN(ev_cross, ev_cross_used);
      KBO_TRY(kbo_i_tc_kstar(h, xc, xc_dtype, rows, h->Ksh.p, kbo_view<float>(h->mun) + c0, s, P1 * 512));
      KBO_TIME_END();
    }
    {
      KBO_TIME_BEGIN(ev_var, ev_var_used);
      KBO_TRY(kbo_i_tc_rank(h, h->Ksh.p, round_up64(rows, 256), h->Wh.p, h->Npad, h->prm.amplitude,
                            kbo_view<float>(h->varn) + c0, s, 0, P1));
      KBO_TIME_END();
    }
  }
  return KBO_OK;
}

// Reads back the survivor count at `count` (into *n, if given) together with the bounds that follow it (fs = count + 4) and
// reports the raw calibration maxima (kbo_last_rank_error, kbo_last_rank_mu_error).
static int read_bounds(kbo_handle* h, const int* count, int* n, cudaStream_t s) {
  struct { int n; int pad[3]; float fs[8]; } host;
  KBO_CUDA(h, cudaMemcpyAsync(&host, count, sizeof host, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (n) *n = host.n;
  h->last_rank_err = host.fs[2];
  h->last_rank_mu_err = host.fs[4];
  return KBO_OK;
}

// The pruning sweep of a LAZY fit (only the leading rows of W exist): everything it touches is the factor L, alpha, and the
// leading block of W.  Calibration: exact mean (FP64 K* kernel) and exact PREFIX variance (three products over the prefix's
// tiles) against the ranking arithmetic over the same prefix -> E, Emu.  Lower bound on the maximum: the sigma -> 0 limit of
// the acquisition function over the whole grid (for EI: the largest predicted improvement) — free.  Candidates whose prefix
// upper bound reaches it (normally a handful) are evaluated EXACTLY in FP64 by panel solves with L and the first-index
// argmax is taken over those values: no ranking pass, no interval test.  An acquisition left undecided (more than 256 such
// candidates, or no usable lower bound) goes on to the caller, which forms the rest of W and runs the sweep of a full fit.
// The grid pass is shared by every acquisition in dec[]; the bound, the survivor list and the FP64 decision are per kind.
static int prune_sweep_lead(kbo_handle* h, const void* Xc, int xc_dtype, int64_t M, int64_t goff, int64_t chunk, AcqDecision* dec, int n_acq,
                            cudaStream_t s) {
  const int Npad = h->Npad;
  const double* scal = h->scal.p;
  const int P1 = kbo_prefix_pairs(h);
  if (P1 < 1 || P1 >= kbo_tile_pairs(Npad) || P1 * 512 > h->w_lead) return KBO_OK;
  KBO_TRY(kbo_reserve(h, h->refine, KBO_REFINE_CAP + 16));
  int* count = h->refine.p + KBO_REFINE_CAP;
  float* fs = reinterpret_cast<float*>(count + 4);   // the bounds after the count (see h->refine)
  KBO_TRY(kbo_reserve(h, h->pr_list, KBO_PRUNE_CAP + 16));
  int* plist = h->pr_list.p;
  int* pcount = plist + KBO_PRUNE_CAP;
  int cal_n = 0;
  {
    KBO_TIME_BEGIN(ev_cal, ev_cal_used);
    KBO_TRY(calibration_rows(h, Xc, xc_dtype, M, &cal_n, s, 2 * P1));   // cal_mu exact, var_cal = exact prefix bound
    const int64_t cal_pad = round_up64(cal_n, 256);
    KBO_TRY(kbo_reserve(h, h->cal_mu_rk, (size_t)(cal_pad + 256)));
    KBO_TRY(kbo_reserve(h, h->cal_var_rk, (size_t)(cal_pad + 256)));
    KBO_TRY(kbo_i_tc_kstar(h, h->cal_x.p, KBO_F64, cal_n, h->Ksh.p, h->cal_mu_rk.p, s, P1 * 512));
    KBO_TRY(kbo_i_tc_rank(h, h->Ksh.p, cal_pad, h->Wh.p, Npad, h->prm.amplitude, h->cal_var_rk.p, s, 0, P1));
    calib_kernel<<<1, 1024, 0, s>>>(h->cal_var_rk.p, h->var_cal.p, h->cal_mu_rk.p, h->cal_mu.p,
                                    nullptr, cal_n, -1, nullptr, 0.0, 0.0, fs);
    KBO_LAUNCH_CHECK(h);
    KBO_TIME_END();
  }
  KBO_TRY(prefix_grid_pass(h, Xc, xc_dtype, M, chunk, P1, s));
  KBO_TIME_BEGIN(ev_acq, ev_acq_used);
  StagePicks sp;
  for (int k = 0; k < n_acq; k++) {
    AcqDecision& d = dec[k];
    if (d.done) continue;
    KBO_CUDA(h, cudaMemsetAsync(pcount, 0, sizeof(int), s));
    KBO_CUDA(h, cudaMemsetAsync(fs + 1, 0, sizeof(float), s));   // this kind's lower bound starts below every ordered value
    grid_lower_bound_kernel<<<acq_grid(h, M), 256, 0, s>>>(kbo_view<float>(h->mun), kbo_view<float>(h->varn), M, d.acq, scal, h->prm.xi, h->prm.kappa, fs);
    KBO_LAUNCH_CHECK(h);
    prefix_survivor_kernel<<<acq_grid(h, M), 256, 0, s>>>(kbo_view<float>(h->mun), kbo_view<float>(h->varn), M, d.acq, scal, h->prm.xi, h->prm.kappa, fs, plist,
                                                         pcount, KBO_PRUNE_CAP);
    KBO_LAUNCH_CHECK(h);
    int n1 = 0;
    KBO_CUDA(h, cudaMemcpyAsync(&n1, pcount, sizeof(int), cudaMemcpyDeviceToHost, s));
    KBO_TRY(read_bounds(h, count, nullptr, s));
    d.prefix_survivors = n1;
    KBO_TRY(record_stage(h, KBO_STAGE_LAZY_PRUNE, d.acq, cal_n, fs, pcount, plist, KBO_PRUNE_CAP, NAN, s));
    if (n1 < 1 || n1 > KBO_SOLVE_CAP) continue;
    d.contenders = n1;
    d.unrefined = 0;
    KBO_TRY(take_list(h, sp, d, plist, n1, s));
  }
  KBO_TRY(refine_union(h, Xc, xc_dtype, goff, sp, s));   // panel solves with L: the lazy fit stays lazy
  KBO_TIME_END();
  return KBO_OK;
}


// The pruning sweep.  An acquisition whose survivors fit (prefix bound, then interval test) is decided here in FP64 (done);
// one with too many survivors goes on to the caller's full ranking pass; the calibration buffers stay valid for it.  The
// calibration rows' ranking arithmetic and the grid pass are shared by every acquisition in dec[].
static int prune_sweep(kbo_handle* h, const void* Xc, int xc_dtype, int64_t M, int64_t goff, int cal_n, int64_t chunk, AcqDecision* dec, int n_acq,
                       cudaStream_t s) {
  const int D = h->D, Npad = h->Npad;
  const double* scal = h->scal.p;
  int P1 = kbo_prefix_pairs(h);
  if (P1 < 1) P1 = 1;
  if (P1 >= kbo_tile_pairs(Npad)) return KBO_OK;   // nothing to save: the caller's full pass is the prefix
  KBO_TRY(kbo_reserve(h, h->refine, KBO_REFINE_CAP + 16));
  int* list = h->refine.p;
  int* count = list + KBO_REFINE_CAP;
  float* fs = reinterpret_cast<float*>(count + 4);   // the bounds after the count (see h->refine)
  KBO_TRY(kbo_reserve(h, h->pr_list, KBO_PRUNE_CAP + 16));
  int* plist = h->pr_list.p;
  int* pcount = plist + KBO_PRUNE_CAP;
  const int64_t cal_pad = round_up64(cal_n, 256);
  KBO_TRY(kbo_reserve(h, h->cal_mu_rk, (size_t)(cal_pad + 256)));
  KBO_TRY(kbo_reserve(h, h->cal_var_rk, (size_t)(cal_pad + 256)));
  {
    KBO_TIME_BEGIN(ev_cal, ev_cal_used);
    // the ranking arithmetic on the calibration rows (all tile pairs): what E and Emu are measured from
    KBO_TRY(kbo_i_tc_kstar(h, h->cal_x.p, KBO_F64, cal_n, h->Ksh.p, h->cal_mu_rk.p, s));
    KBO_TRY(kbo_i_tc_rank(h, h->Ksh.p, cal_pad, h->Wh.p, Npad, h->prm.amplitude, h->cal_var_rk.p, s));
    KBO_TIME_END();
  }
  // pass 1 over the grid: mean over all trials, variance bound from the first P1 tile pairs
  KBO_TRY(prefix_grid_pass(h, Xc, xc_dtype, M, chunk, P1, s));
  KBO_TIME_BEGIN(ev_acq, ev_acq_used);
  StagePicks sp;
  for (int k = 0; k < n_acq; k++) {
    AcqDecision& d = dec[k];
    if (d.done) continue;
    // E, Emu and this kind's lower bound on the maximum from the calibration rows (one CTA over one wave of rows)
    calib_kernel<<<1, 1024, 0, s>>>(h->cal_var_rk.p, h->var_cal.p, h->cal_mu_rk.p, h->cal_mu.p,
                                    nullptr, cal_n, d.acq, scal, h->prm.xi, h->prm.kappa, fs);
    KBO_LAUNCH_CHECK(h);
    KBO_CUDA(h, cudaMemsetAsync(pcount, 0, sizeof(int), s));
    prefix_survivor_kernel<<<acq_grid(h, M), 256, 0, s>>>(kbo_view<float>(h->mun), kbo_view<float>(h->varn), M, d.acq, scal, h->prm.xi, h->prm.kappa, fs, plist,
                                                         pcount, KBO_PRUNE_CAP);
    KBO_LAUNCH_CHECK(h);
    int n1 = 0;
    KBO_CUDA(h, cudaMemcpyAsync(&n1, pcount, sizeof(int), cudaMemcpyDeviceToHost, s));
    KBO_TRY(read_bounds(h, count, nullptr, s));
    d.prefix_survivors = n1;
    KBO_TRY(record_stage(h, KBO_STAGE_PRUNE, d.acq, cal_n, fs, pcount, plist, KBO_PRUNE_CAP, NAN, s));
    if (n1 < 1 || n1 > KBO_PRUNE_CAP) continue;
    // pass 2: the survivors' rows through the whole ranking pass, then the interval test and the FP64 decision
    const int64_t n1_pad = round_up64(n1, 256);
    KBO_TRY(kbo_reserve(h, h->pr_x, (size_t)n1_pad * D));
    KBO_TRY(kbo_reserve(h, h->pr_mu, (size_t)(n1_pad + 256)));
    KBO_TRY(kbo_reserve(h, h->pr_var, (size_t)(n1_pad + 256)));
    if (xc_dtype == KBO_F64)
      gather_rows_kernel<double><<<n1, 64, 0, s>>>((const double*)Xc, D, plist, n1, h->pr_x.p);
    else
      gather_rows_kernel<float><<<n1, 64, 0, s>>>((const float*)Xc, D, plist, n1, h->pr_x.p);
    KBO_LAUNCH_CHECK(h);
    KBO_TRY(kbo_i_tc_kstar(h, h->pr_x.p, KBO_F64, n1, h->Ksh.p, h->pr_mu.p, s));
    KBO_TRY(kbo_i_tc_rank(h, h->Ksh.p, n1_pad, h->Wh.p, Npad, h->prm.amplitude, h->pr_var.p, s));
    KBO_CUDA(h, cudaMemsetAsync(count, 0, sizeof(int), s));
    const int g2 = (n1 + 255) / 256;
    bound_max_kernel<<<g2, 256, 0, s>>>(h->pr_mu.p, h->pr_var.p, n1, d.acq, scal, h->prm.xi, h->prm.kappa, fs);
    KBO_LAUNCH_CHECK(h);
    survivor_kernel<<<g2, 256, 0, s>>>(h->pr_mu.p, h->pr_var.p, plist, n1, d.acq, scal, h->prm.xi, h->prm.kappa, fs, list,
                                       count);
    KBO_LAUNCH_CHECK(h);
    int n2 = 0;
    KBO_CUDA(h, cudaMemcpyAsync(&n2, count, sizeof(int), cudaMemcpyDeviceToHost, s));
    KBO_CUDA(h, cudaStreamSynchronize(s));
    d.contenders = n2;
    KBO_TRY(record_stage(h, KBO_STAGE_PRUNE_INTERVAL, d.acq, cal_n, fs, count, list, KBO_REFINE_CAP, NAN, s));
    if (n2 < 1 || n2 > KBO_REFINE_CAP) continue;
    d.unrefined = 0;
    KBO_TRY(take_list(h, sp, d, list, n2, s));
  }
  KBO_TRY(refine_union(h, Xc, xc_dtype, goff, sp, s));
  KBO_TIME_END();
  return KBO_OK;
}

// The interval test of the full ranking pass for one acquisition; survivors that fit go to sp.  Not handed over: they do not
// fit (the caller redoes the sweep with three products).
static int fast_pick(kbo_handle* h, int64_t M, int cal_n, AcqDecision& d, StagePicks& sp, cudaStream_t s) {
  const double* scal = h->scal.p;
  KBO_TRY(kbo_reserve(h, h->refine, KBO_REFINE_CAP + 16));
  int* list = h->refine.p;
  int* count = list + KBO_REFINE_CAP;
  float* fs = reinterpret_cast<float*>(count + 4);   // the bounds after the count (see h->refine)
  KBO_CUDA(h, cudaMemsetAsync(count, 0, sizeof(int), s));
  calib_kernel<<<1, 1024, 0, s>>>(kbo_view<float>(h->varn), h->var_cal.p, kbo_view<float>(h->mun), h->cal_mu.p,
                                  h->cal_idx.p, cal_n, -1, nullptr, 0.0, 0.0, fs);
  KBO_LAUNCH_CHECK(h);
  bound_max_kernel<<<acq_grid(h, M), 256, 0, s>>>(kbo_view<float>(h->mun), kbo_view<float>(h->varn), M, d.acq, scal, h->prm.xi, h->prm.kappa, fs);
  KBO_LAUNCH_CHECK(h);
  survivor_kernel<<<acq_grid(h, M), 256, 0, s>>>(kbo_view<float>(h->mun), kbo_view<float>(h->varn), nullptr, M, d.acq, scal, h->prm.xi, h->prm.kappa, fs,
                                                 list, count);
  KBO_LAUNCH_CHECK(h);
  int n = 0;
  KBO_TRY(read_bounds(h, count, &n, s));
  d.contenders = n;
  KBO_TRY(record_stage(h, KBO_STAGE_INTERVAL, d.acq, cal_n, fs, count, list, KBO_REFINE_CAP, NAN, s));
  if (n < 1 || n > KBO_REFINE_CAP) return KBO_OK;
  d.unrefined = 0;
  return take_list(h, sp, d, list, n, s);
}

// The stratified calibration rows of a ranking sweep through the FP64 K* kernel and the three-product contraction:
// cal_idx (row indices), cal_mu (normalised mean), var_cal (normalised variance).  Uses the K* scratch planes, so it runs
// before the first chunk.
static int calibration_rows(kbo_handle* h, const void* Xc, int xc_dtype, int64_t M, int* cal_n_out, cudaStream_t s, int jtiles) {
  // one wave of the three-product cluster kernel: sm_count / 2 clusters × 128 rows.  The bounds are 8 × the largest error seen on
  // these rows; the errors are sums of thousands of rounding terms (light-tailed: the maximum over 1e6 rows of a Gaussian exceeds
  // the maximum over 1e4 by ~1.2×), so the sample size is not what the margin hinges on — its being stratified is.
  int64_t want = (int64_t)h->sm_count * 64;
  const int cal_n = (int)(M < want ? M : want);
  const int64_t cal_pad = round_up64(cal_n, 128);
  KBO_TRY(kbo_reserve(h, h->cal_idx, (size_t)cal_pad));
  KBO_TRY(kbo_reserve(h, h->cal_x, (size_t)cal_pad * h->D));
  KBO_TRY(kbo_reserve(h, h->cal_mu, (size_t)cal_pad));
  KBO_TRY(kbo_reserve(h, h->var_cal, (size_t)cal_pad));
  cal_index_kernel<<<(cal_n + 255) / 256, 256, 0, s>>>(h->cal_idx.p, cal_n, M);
  KBO_LAUNCH_CHECK(h);
  if (xc_dtype == KBO_F64)
    gather_rows_kernel<double><<<cal_n, 64, 0, s>>>((const double*)Xc, h->D, h->cal_idx.p, cal_n, h->cal_x.p);
  else
    gather_rows_kernel<float><<<cal_n, 64, 0, s>>>((const float*)Xc, h->D, h->cal_idx.p, cal_n, h->cal_x.p);
  KBO_LAUNCH_CHECK(h);
  KBO_TRY((launch_cross<double, float, 1>(h, h->cal_x.p, cal_n, cal_pad, nullptr, 0, h->Ksh.p, h->Ksl.p,
                                          h->cal_mu.p, s)));
  // jtiles > 0: the exact variance bound from a PREFIX of the trial tiles (needs the leading rows of W only)
  KBO_TRY(kbo_i_tc_variance(h, h->Ksh.p, h->Ksl.p, cal_pad, h->Wh.p, h->Wl.p, h->Npad,
                            0.0, h->prm.amplitude, h->var_cal.p, h->prm.tc_k_span, s, 3, jtiles));
  *cal_n_out = cal_n;
  return KBO_OK;
}

static int sweep_impl(kbo_handle* h, const void* Xc, int xc_dtype, int64_t M, int64_t goff, double* mu_out, double* std_out, double* acq_out,
                      AcqDecision* dec, int n_acq, cudaStream_t s, bool force_three);

int kbo_i_debug_cross_planes(kbo_handle* h, const void* Xc, int xc_dtype, int64_t M, cudaStream_t s) {
  const int64_t rows_pad = round_up64(M, 128);
  if (xc_dtype == KBO_F64)
    return launch_cross<double, float, 1>(h, (const double*)Xc, M, rows_pad, nullptr, 0, h->Ksh.p, h->Ksl.p, kbo_view<float>(h->mun), s);
  return launch_cross<float, float, 1>(h, (const float*)Xc, M, rows_pad, nullptr, 0, h->Ksh.p, h->Ksl.p, kbo_view<float>(h->mun), s);
}

// Test hook: the ranking arithmetic of M rows as the pruning pass (tile_pairs >= 1: the first tile_pairs pairs of trial tiles, only
// their columns of K̃* stored) or the full ranking pass (tile_pairs < 0, or all pairs) computes it: tensor-core K* and mean, then
// the wgmma contraction.  A lazy fit forms the rest of W first where the pairs reach past its leading rows.
int kbo_i_debug_rank_rows(kbo_handle* h, const void* Xc, int xc_dtype, int64_t M, int tile_pairs, float* mun_out, float* varn_out, cudaStream_t s) {
  if (!h->fitted || !h->have_planes || !h->ks_ready)
    KBO_FAIL(h, KBO_ERR_STATE, "kbo_debug_rank_rows: needs a fit with tensor-core planes and K* operands (D <= 128)");
  const int Npad = h->Npad, n_pairs = kbo_tile_pairs(Npad);
  if (tile_pairs == 0) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_debug_rank_rows: tile_pairs must be >= 1 or < 0");
  const int P1 = (tile_pairs < 0 || tile_pairs > n_pairs) ? n_pairs : tile_pairs;
  if (!h->w_full && (P1 == n_pairs || P1 * 512 > h->w_lead)) KBO_TRY(kbo_i_ensure_w(h, s));
  const int64_t rows_pad = round_up64(M, 256);
  KBO_TRY(kbo_reserve(h, h->Ksh, (size_t)rows_pad * Npad));
  const size_t bytes = sizeof(float) * (size_t)(rows_pad + 256);
  KBO_TRY(kbo_reserve(h, h->mun, bytes));
  KBO_TRY(kbo_reserve(h, h->varn, bytes));
  KBO_TRY(kbo_i_tc_kstar(h, Xc, xc_dtype, M, h->Ksh.p, kbo_view<float>(h->mun), s, P1 < n_pairs ? P1 * 512 : -1));
  KBO_TRY(kbo_i_tc_rank(h, h->Ksh.p, rows_pad, h->Wh.p, Npad, h->prm.amplitude, kbo_view<float>(h->varn), s, 0, P1));
  KBO_CUDA(h, kbo_copy(mun_out, kbo_view<float>(h->mun), M, cudaMemcpyDeviceToDevice, s));
  KBO_CUDA(h, kbo_copy(varn_out, kbo_view<float>(h->varn), M, cudaMemcpyDeviceToDevice, s));
  return KBO_OK;
}

static void record_decisions(kbo_handle* h, const AcqDecision* dec, int n_acq) {
  h->dec_n = n_acq;
  for (int k = 0; k < n_acq; k++) {
    h->dec_unrefined[k] = dec[k].unrefined;
    h->dec_contenders[k] = dec[k].contenders;
    h->dec_prefix_survivors[k] = dec[k].prefix_survivors;
  }
}

int kbo_i_sweep(kbo_handle* h, const void* Xc, int xc_dtype, int64_t M, int64_t goff, double* mu_out, double* std_out, double* acq_out,
                kbo_best* best_dev, cudaStream_t s) {
  AcqDecision d{h->prm.acq, best_dev, false, h->last_unrefined, h->last_contenders, h->last_prefix_survivors};
  h->stage_recs.clear();
  const int r = sweep_impl(h, Xc, xc_dtype, M, goff, mu_out, std_out, acq_out, &d, 1, s, false);
  h->last_unrefined = d.unrefined;
  h->last_contenders = d.contenders;
  h->last_prefix_survivors = d.prefix_survivors;
  record_decisions(h, &d, 1);
  return r;
}

int kbo_i_sweep_multi(kbo_handle* h, const void* Xc, int xc_dtype, int64_t M, int64_t goff, int n_acq, const int32_t* acqs, kbo_best* best_dev,
                      cudaStream_t s) {
  if (n_acq < 1 || n_acq > 3) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sweep_multi: n_acq must be 1, 2 or 3 (got %d)", n_acq);
  AcqDecision dec[3];
  for (int k = 0; k < n_acq; k++) {
    if (acqs[k] < KBO_ACQ_EI || acqs[k] > KBO_ACQ_PI) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sweep_multi: unknown acquisition %d", acqs[k]);
    for (int j = 0; j < k; j++)
      if (acqs[j] == acqs[k]) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sweep_multi: acquisition %d requested twice", acqs[k]);
    dec[k] = AcqDecision{acqs[k], best_dev + k, false, 0, 0, -1};
  }
  const float rank_err = h->last_rank_err, rank_mu_err = h->last_rank_mu_err;   // kbo_last_* keep reporting the last kbo_sweep
  h->stage_recs.clear();
  const int r = sweep_impl(h, Xc, xc_dtype, M, goff, nullptr, nullptr, nullptr, dec, n_acq, s, false);
  h->last_rank_err = rank_err;
  h->last_rank_mu_err = rank_mu_err;
  record_decisions(h, dec, n_acq);
  return r;
}

// Every acquisition in dec[] that is not done yet is decided over ONE posterior: the calibration rows, the K* planes, the
// contractions and the mean are computed once per stage and shared; the bounds, survivor lists and FP64 decisions are per kind.
// Each kind leaves at the first stage where its own list fits its cap — where kbo_sweep with that kind alone would have.
static int sweep_impl(kbo_handle* h, const void* Xc, int xc_dtype, int64_t M, int64_t goff, double* mu_out, double* std_out, double* acq_out,
                      AcqDecision* dec, int n_acq, cudaStream_t s, bool force_three) {
  if (!h->fitted) KBO_FAIL(h, KBO_ERR_STATE, "kbo_sweep: call kbo_fit first");
  if (M < 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sweep: M must be >= 1 (got %lld)", (long long)M);
  if (xc_dtype != KBO_F64 && xc_dtype != KBO_F32) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sweep: xc_dtype must be KBO_F64 or KBO_F32");
  if (h->D > 256) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sweep: D <= 256 supported (got %d)", h->D);
  const int N = h->N, D = h->D, ld = h->ld, Npad = h->Npad;
  if (N > Npad || N > ld) KBO_FAIL(h, KBO_ERR_STATE, "kbo_sweep: inconsistent fit state (N=%d, Npad=%d, ld=%d)", N, Npad, ld);
  // The fp16 K* planes hold amplitude·k: above 1e4 the entries near the trials approach the fp16 range (65504) and the
  // contraction overflows, so such fits take the FP64 path in every mode.  The tensor-core error grows with the amplitude
  // (|dσ²| ∝ amplitude): `auto` keeps the 1e-5 bound on returned arrays by using the tensor cores for array sweeps up to
  // amplitude 10 only (DESIGN.md §1).  Array-free sweeps are decided in FP64 whatever the amplitude.
  const double amp = h->prm.amplitude;
  const bool arrays = mu_out || std_out || acq_out;
  const bool tc = amp <= 1e4 && (h->prm.var_mode == KBO_VAR_TC_F16X3 ||
                                 (h->prm.var_mode == KBO_VAR_AUTO && (amp <= 10.0 || !arrays) && h->have_planes &&
                                  (double)M * h->N * h->N > 2e11));
  const size_t esz = xc_dtype == KBO_F64 ? 8 : 4;
  const double* scal = h->scal.p;
  // array-free tensor-core sweeps rank with one fp16 product and let the FP64 refinement decide (fast_pick above)
  const bool fast = tc && !force_three && h->tc_fast && !mu_out && !std_out && !acq_out && M < 0x7fffffff;
  // ... and, by default, build that pass's K̃* on the tensor cores and contract it with wgmma MMAs (tc_kstar.cu, tc_rank.cu)
  const bool rank_tc = fast && h->rank_tc && h->ks_ready;
  int cal_n = 0;
  int64_t chunk;
  if (tc) {
    const int64_t wave = (int64_t)h->sm_count * 128;
    const int64_t cal_pad = fast ? round_up64(M < wave ? M : wave, 128) : 0;
    if (rank_tc) {
      // one fp16 plane per chunk; the ranking kernel deals (256-row group, tile pair) items, so any multiple of 256 rows will do
      chunk = (int64_t)(h->scratch_limit / ((size_t)Npad * 2)) / 256 * 256;
      if (chunk < 256) chunk = 256;
      if (chunk > round_up64(M, 256)) chunk = round_up64(M, 256);
      int64_t rows_sh = chunk > round_up64(cal_pad, 256) ? chunk : round_up64(cal_pad, 256);
      const int64_t prune_rows = round_up64(M < 16384 ? M : 16384, 256);          // the pruning pass re-runs up to 16384 survivors in one go
      if (rows_sh < prune_rows) rows_sh = prune_rows;
      KBO_TRY(kbo_reserve(h, h->Ksh, (size_t)rows_sh * Npad));
      KBO_TRY(kbo_reserve(h, h->Ksl, (size_t)cal_pad * Npad));   // the lo plane exists for the calibration rows only
    } else {
      // wave-aligned chunks: the variance kernel runs one 128-row CTA per SM, the K* kernel two — a chunk that is a multiple
      // of sm_count·128 rows leaves no partial wave
      chunk = (int64_t)(h->scratch_limit / ((size_t)Npad * 4));
      chunk = chunk >= wave ? chunk / wave * wave : chunk / 128 * 128;
      if (chunk < 128) chunk = 128;
      if (chunk > round_up64(M, 128)) chunk = round_up64(M, 128);
      const int64_t rows_sh = chunk > cal_pad ? chunk : cal_pad;
      KBO_TRY(kbo_reserve(h, h->Ksh, (size_t)rows_sh * Npad));
      KBO_TRY(kbo_reserve(h, h->Ksl, (size_t)rows_sh * Npad));
    }
    const size_t bytes = sizeof(float) * (size_t)(round_up64(M, 256) + 256);
    KBO_TRY(kbo_reserve(h, h->mun, bytes));
    KBO_TRY(kbo_reserve(h, h->varn, bytes));
  } else {
    chunk = (int64_t)(h->scratch_limit / ((size_t)ld * 8)) / 64 * 64;
    if (chunk < 64) chunk = 64;
    if (chunk > round_up64(M, 64)) chunk = round_up64(M, 64);
    KBO_TRY(kbo_reserve(h, h->Ks64, (size_t)chunk * ld));
    KBO_TRY(kbo_reserve(h, h->part, (size_t)chunk * ((N + 63) / 64)));
    const size_t bytes = sizeof(double) * (size_t)M;
    KBO_TRY(kbo_reserve(h, h->mun, bytes));
    KBO_TRY(kbo_reserve(h, h->varn, bytes));
  }
  h->tim.chunks = 0;
  auto all_done = [&]() {
    for (int k = 0; k < n_acq; k++)
      if (!dec[k].done) return false;
    return true;
  };
  for (int k = 0; k < n_acq; k++)
    if (!force_three && !dec[k].done) dec[k].prefix_survivors = -1;   // (a three-product redo keeps what the failed ranking attempt recorded)
  if (!h->w_full) {
    // a lazy fit: try the sweep that needs the leading rows of W only; anything else forms the rest first
    if (tc && rank_tc && h->rank_prefix != 0) {
      KBO_TRY(prune_sweep_lead(h, Xc, xc_dtype, M, goff, chunk, dec, n_acq, s));
      if (all_done()) return KBO_OK;
      h->tim.chunks = 0;
    }
    KBO_TRY(kbo_i_ensure_w(h, s));
  }
  if (fast) {   // the calibration rows borrow the K* scratch, so they go first
    KBO_TIME_BEGIN(ev_cal, ev_cal_used);
    KBO_TRY(calibration_rows(h, Xc, xc_dtype, M, &cal_n, s));
    KBO_TIME_END();
  }
  if (rank_tc && h->rank_prefix != 0) {
    KBO_TRY(prune_sweep(h, Xc, xc_dtype, M, goff, cal_n, chunk, dec, n_acq, s));
    if (all_done()) return KBO_OK;
    h->tim.chunks = 0;   // not prunable: the full ranking pass below starts over
  }
  for (int64_t c0 = 0; c0 < M; c0 += chunk) {
    const int64_t rows = (M - c0 < chunk) ? (M - c0) : chunk;
    const unsigned char* xc = (const unsigned char*)Xc + (size_t)c0 * D * esz;
    h->tim.chunks++;
    if (rank_tc) {
      {
        KBO_TIME_BEGIN(ev_cross, ev_cross_used);
        KBO_TRY(kbo_i_tc_kstar(h, xc, xc_dtype, rows, h->Ksh.p, kbo_view<float>(h->mun) + c0, s));
        KBO_TIME_END();
      }
      {
        KBO_TIME_BEGIN(ev_var, ev_var_used);
        KBO_TRY(kbo_i_tc_rank(h, h->Ksh.p, round_up64(rows, 256), h->Wh.p, Npad, h->prm.amplitude,
                              kbo_view<float>(h->varn) + c0, s));
        KBO_TIME_END();
      }
    } else if (tc) {
      const int64_t rows_pad = round_up64(rows, 128);
      float* mun = kbo_view<float>(h->mun) + c0;
      {
        KBO_TIME_BEGIN(ev_cross, ev_cross_used);
        if (xc_dtype == KBO_F64)
          KBO_TRY((launch_cross<double, float, 1>(h, (const double*)xc, rows, rows_pad, nullptr, 0, h->Ksh.p, h->Ksl.p, mun, s)));
        else
          KBO_TRY((launch_cross<float, float, 1>(h, (const float*)xc, rows, rows_pad, nullptr, 0, h->Ksh.p, h->Ksl.p, mun, s)));
        KBO_TIME_END();
      }
      {
        KBO_TIME_BEGIN(ev_var, ev_var_used);
        KBO_TRY(kbo_i_tc_variance(h, h->Ksh.p, h->Ksl.p, rows_pad, h->Wh.p, h->Wl.p,
                                  Npad, 0.0, h->prm.amplitude, kbo_view<float>(h->varn) + c0, fast ? 1024 : h->prm.tc_k_span, s, fast ? 1 : 3));
        KBO_TIME_END();
      }
    } else {
      double* mun = kbo_view<double>(h->mun) + c0;
      {
        KBO_TIME_BEGIN(ev_cross, ev_cross_used);
        if (xc_dtype == KBO_F64)
          KBO_TRY((launch_cross<double, double, 0>(h, (const double*)xc, rows, rows, h->Ks64.p, ld, nullptr, nullptr, mun, s)));
        else
          KBO_TRY((launch_cross<float, double, 0>(h, (const float*)xc, rows, rows, h->Ks64.p, ld, nullptr, nullptr, mun, s)));
        KBO_TIME_END();
      }
      {
        KBO_TIME_BEGIN(ev_var, ev_var_used);
        const int njt = (N + 63) / 64;
        dgemm64_launch<true, EPI_ROWSUMSQ>(s, (int)rows, N, N, h->Ks64.p, ld, h->W.p, ld, h->part.p, njt,
                                           1.0, 0.0, KM_UPTO_N, 0, TS_NONE);
        KBO_LAUNCH_CHECK(h);
        var_from_parts_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, s>>>(h->part.p, rows, njt, h->prm.amplitude,
                                                                            kbo_view<double>(h->varn) + c0);
        KBO_LAUNCH_CHECK(h);
        KBO_TIME_END();
      }
    }
  }
  // acquisition over the whole grid; y statistics are read from the fit's device scalars (no host sync)
  {
    KBO_TIME_BEGIN(ev_acq, ev_acq_used);
    if (fast) {
      StagePicks sp;
      for (int k = 0; k < n_acq; k++)
        if (!dec[k].done) KBO_TRY(fast_pick(h, M, cal_n, dec[k], sp, s));
      KBO_TRY(refine_union(h, Xc, xc_dtype, goff, sp, s));
      KBO_TIME_END();
      // the kinds whose survivors overflowed: one three-product sweep for all of them
      if (!all_done()) return sweep_impl(h, Xc, xc_dtype, M, goff, mu_out, std_out, acq_out, dec, n_acq, s, true);
      return KBO_OK;
    }
    StagePicks sp;
    for (int k = 0; k < n_acq; k++) {
      AcqDecision& d = dec[k];
      if (d.done) continue;
      if (tc) {
        KBO_TRY(launch_acq<float>(h, kbo_view<float>(h->mun), kbo_view<float>(h->varn), M, goff, d.acq, 0.0, 1.0, 0.0, scal, h->prm.xi,
                                  h->prm.kappa, mu_out, std_out, acq_out, nullptr, d.best, s));
        d.unrefined = 2;
        if (M < 0x7fffffff)
          KBO_TRY(refine_suggestion(h, M, goff, d, sp, s));
        else
          d.done = true;
      } else {
        d.unrefined = 0;
        KBO_TRY(launch_acq<double>(h, kbo_view<double>(h->mun), kbo_view<double>(h->varn), M, goff, d.acq, 0.0, 1.0, 0.0, scal, h->prm.xi,
                                   h->prm.kappa, mu_out, std_out, acq_out, nullptr, d.best, s));
        d.done = true;
      }
    }
    KBO_TRY(refine_union(h, Xc, xc_dtype, goff, sp, s));
    KBO_TIME_END();
  }
  return KBO_OK;
}

// ------------------------------------------------------------------------------------------------
// FP64 posterior mean at a few points, raw y scale: the refinement's K* row and fixed-order mean (refine_cross_kernel,
// refine_mu_kernel) — alpha only, never W, so a lazy fit stays lazy.  What gp_hedge's gains update reads at the last picks.
template <typename XT>
__global__ void rows_to_f64_kernel(const XT* __restrict__ X, int64_t n, int D, double* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n * D) out[e] = (double)X[e];
}
__global__ void raw_mean_kernel(const double* __restrict__ mun, int n, const double* __restrict__ scal, double* __restrict__ mu) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) mu[i] = scal[S_YSTD] * mun[i] + scal[S_YMEAN];   // as acq_value forms μ
}

int kbo_i_predict_mean(kbo_handle* h, const void* X, int x_dtype, int n, double* mu_host, cudaStream_t s) {
  if (!h->fitted) KBO_FAIL(h, KBO_ERR_STATE, "kbo_predict_mean: call kbo_fit first");
  if (x_dtype != KBO_F64 && x_dtype != KBO_F32) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_predict_mean: xc_dtype must be KBO_F64 or KBO_F32");
  if (h->D > 256) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_predict_mean: D <= 256 supported (got %d)", h->D);
  const int N = h->N, D = h->D, ld = h->ld;
  const int B = n < 1024 ? n : 1024;   // rows per batch: K* scratch of B × ld doubles
  KBO_TRY(kbo_reserve(h, h->refine_x, (size_t)B * D));
  KBO_TRY(kbo_reserve(h, h->Ks64, (size_t)B * ld));
  KBO_TRY(kbo_reserve(h, h->part, (size_t)B * 2));
  double* Xg = h->refine_x.p;
  double* mun = h->part.p;
  double* mu = mun + B;
  const size_t esz = x_dtype == KBO_F64 ? 8 : 4;
  for (int r0 = 0; r0 < n; r0 += B) {
    const int m = n - r0 < B ? n - r0 : B;
    const unsigned char* x = (const unsigned char*)X + (size_t)r0 * D * esz;
    const unsigned g = (unsigned)(((int64_t)m * D + 255) / 256);
    if (x_dtype == KBO_F64)
      rows_to_f64_kernel<double><<<g, 256, 0, s>>>((const double*)x, m, D, Xg);
    else
      rows_to_f64_kernel<float><<<g, 256, 0, s>>>((const float*)x, m, D, Xg);
    KBO_LAUNCH_CHECK(h);
    refine_cross_kernel<<<dim3((N + 255) / 256, m), 256, 0, s>>>(Xg, D, h->d_inv_ls.p, (int)h->inv_ls.size(), h->XsT.p, ld, N,
                                                                 h->prm.kernel, h->prm.amplitude, h->Ks64.p);
    KBO_LAUNCH_CHECK(h);
    refine_mu_kernel<<<m, 256, 0, s>>>(h->Ks64.p, ld, N, h->alpha.p, mun);
    KBO_LAUNCH_CHECK(h);
    raw_mean_kernel<<<(m + 255) / 256, 256, 0, s>>>(mun, m, h->scal.p, mu);
    KBO_LAUNCH_CHECK(h);
    KBO_CUDA(h, cudaMemcpyAsync(mu_host + r0, mu, sizeof(double) * (size_t)m, cudaMemcpyDeviceToHost, s));
    KBO_CUDA(h, cudaStreamSynchronize(s));
  }
  int inf = 0;
  KBO_CUDA(h, kbo_copy(&inf, h->info.p, 1, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (inf != 0) KBO_FAIL(h, KBO_ERR_NOT_PD, "kernel matrix is not positive definite (pivot %d); increase `noise`", inf);
  return KBO_OK;
}
