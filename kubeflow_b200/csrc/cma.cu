// (μ/μ_w, λ)-CMA-ES generation on the device, FP64 — the sampler behind Katib's `cmaes` algorithm (goptuna; SURVEY.md §8(a) A9).
// N. Hansen, "The CMA Evolution Strategy: A Tutorial" (arXiv:1604.00772), active-weights variant as in CyberAgent `cmaes`:
//   ask : z ~ N(0,I) (Philox4x32-10 + Box–Muller, or caller-supplied), y = B·(d∘z), x = m + σ·y
//   tell: rank by fitness (NumPy order, NaN last; ties → lower sample index), y_w, m, p_σ, σ, h_σ, p_c,
//         C ← a·C + c1·p_c p_cᵀ + cμ·Σ w°_i y_i y_iᵀ, then C = B diag(d²) Bᵀ by one-sided Jacobi warm-started from the previous
//         basis (G = C·B_prev), d_j² = b_jᵀ C b_j.  Over the cfg4 run (D = 128, λ = 4096, Rastrigin) the warm start still
//         takes 6–7 sweeps, counting the last one that rotates nothing (10 at most), measured on an H100.
// Everything is tiny (D ≤ 128, λ ≤ 8192: C is 128 KiB) — the generation is launch/latency bound, so each phase is one
// kernel and the whole state lives in HBM/L2 between them; nothing returns to the host until the caller asks.
#include <cmath>

#include "kbo_internal.cuh"
#include "dgemm.cuh"
#include "kbo_rng.cuh"

#define CMA_EPS 1e-8
#define CMA_MAXD 128

struct CmaMarginDim;

struct kbo_cma {
  int D = 0, lambda = 0, mu = 0, lam_pow2 = 0, lam_pad = 0;  // lam_pad: λ rounded up to the 256-wide split-K slices
  uint64_t seed = 0;
  long long gen = 0;    // strategy generation: back to 0 at every restart (h_σ and the termination test read it)
  long long draws = 0;  // Philox counter of the built-in sampler: one per tell, never reset, so no restart repeats a draw
  // strategy parameters (host copies)
  double mu_eff, c1, cmu, cm, c_sigma, d_sigma, cc, chi_n, wsum;
  // termination test (`cmaes`' should_stop): constants of the current run, fitness history ring of 2·term doubles
  int term = 0;
  double tolx = 0.0;
  DevBuf<double> mean, C, B, Dv, ps, pc, weights, Z, Zs, Y, Ys, YwT, zn2, R, G, scal, yw, hist;
  DevBuf<int> order;
  DevBuf<unsigned> flags;
  bool asked = false;
  // CMA-ES with Margin (kbo_cma_set_margin): off while n_disc == 0, and then no margin buffer is touched
  int n_disc = 0;
  double alpha = 0.0, alpha_set = 0.0;  // alpha_set: the caller's α, or 0 for the default 1/(D·λ) recomputed at restarts
  DevBuf<double> A;                     // A
  DevBuf<CmaMarginDim> mdim;            // per-dimension level descriptors
  DevBuf<double> mlev, mprev, mpre;     // level tables; (m, σ) before the tell; m before the correction
  // learning-rate adaptation (kbo_cma_set_lr_adapt): off while !lra, and then no LRA buffer is touched
  bool lra = false;
  DevBuf<double> lprev, lC0;                    // (m, σ) and C before the tell
  DevBuf<double> lW, lP, lS, lT, lL;            // B·diag(1/d); P₀ = C^{-1/2}; S = ΔΣ/σ′²; P₀·S; P₀·S·P₀ (all D×D)
  DevBuf<double> lE, lscal;                     // E_m (D) then E_Σ (D×D); V_m, V_Σ, η_m, η_Σ, η_m before the last tell
};

// A discrete dimension's sorted levels in cube coordinates: levels[off, off + count) of the table, or, for ranges too long
// for a table (kind 2), level k = first + k·step.  Continuous dimensions have kind 0.
struct CmaMarginDim {
  double first, step;
  long long count, off;
  int kind;
};

enum CmaScal { CS_SIGMA = 0, CS_ALPHA_C = 1, CS_BEST_F = 2, CS_SWEEPS = 3, CS_COUNT = 8 };

// ------------------------------------------------------------------------------------------------ RNG (philox4x32_10: kbo_rng.cuh)
// two standard normals per call from 128 random bits (53-bit uniforms, Box–Muller in FP64)
__global__ void cma_normal_kernel(double* __restrict__ Z, int64_t n, uint64_t seed, uint64_t gen) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;  // pair index
  if (2 * p >= n) return;
  uint32_t r[4];
  philox4x32_10((uint32_t)p, (uint32_t)(p >> 32), (uint32_t)gen, (uint32_t)(gen >> 32), (uint32_t)seed, (uint32_t)(seed >> 32), r);
  const double u1 = ((((uint64_t)r[0] << 21) ^ (uint64_t)(r[1] >> 11)) + 1.0) * (1.0 / 9007199254740993.0);  // (0,1]
  const double u2 = (((uint64_t)r[2] << 21) ^ (uint64_t)(r[3] >> 11)) * (1.0 / 9007199254740992.0);          // [0,1)
  const double rad = sqrt(-2.0 * log(u1));
  double s, c;
  sincospi(2.0 * u2, &s, &c);
  Z[2 * p] = rad * c;
  if (2 * p + 1 < n) Z[2 * p + 1] = rad * s;
}

// Zs = Z∘d, zn2[k] = ‖z_k‖²  (one warp per sample)
__global__ void cma_scale_kernel(const double* __restrict__ Z, const double* __restrict__ Dv, int lambda, int D, double* __restrict__ Zs,
                                 double* __restrict__ zn2) {
  const int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (k >= lambda) return;
  double s = 0.0;
  for (int d = lane; d < D; d += 32) {
    const double z = Z[(size_t)k * D + d];
    Zs[(size_t)k * D + d] = z * Dv[d];
    s = fma(z, z, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) zn2[k] = s;
}
__global__ void cma_x_kernel(const double* __restrict__ Y, const double* __restrict__ mean, const double* __restrict__ scal, int64_t n, int D,
                             double* __restrict__ X) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) X[e] = fma(scal[CS_SIGMA], Y[e], mean[e % D]);
}
// synthetic fitness for the benchmark of record (cfg4): 0 = sphere, 1 = Rastrigin (one warp per sample)
__global__ void cma_fitness_kernel(const double* __restrict__ X, int lambda, int D, int kind, double* __restrict__ f) {
  const int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (k >= lambda) return;
  double s = 0.0;
  for (int d = lane; d < D; d += 32) {
    const double x = X[(size_t)k * D + d];
    s += kind == 0 ? x * x : (x * x - 10.0 * cospi(2.0 * x) + 10.0);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) f[k] = s;
}

// ------------------------------------------------------------------------------------------------ rank
// single-CTA bitonic sort of (fitness, index) in shared memory, in NumPy's order (what the oracle's lexsort gives):
// -inf < finite < +inf < NaN, -0 == +0, every NaN equal; ties → lower index first.  Padding rows are NaN with indices
// past lambda, so they sort after every real sample.
__global__ void __launch_bounds__(1024) cma_sort_kernel(const double* __restrict__ f, int lambda, int n2, int* __restrict__ order,
                                                        double* __restrict__ scal) {
  extern __shared__ unsigned char smc[];
  double* key = reinterpret_cast<double*>(smc);
  int* idx = reinterpret_cast<int*>(key + n2);
  for (int i = threadIdx.x; i < n2; i += 1024) {
    key[i] = i < lambda ? f[i] : NAN;
    idx[i] = i;
  }
  __syncthreads();
  for (int k = 2; k <= n2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n2; i += 1024) {
        const int l = i ^ j;
        if (l > i) {
          const bool up = (i & k) == 0;
          const double a = key[i], b = key[l];
          const int ia = idx[i], ib = idx[l];
          const bool an = a != a, bn = b != b;
          const bool gt = an != bn ? an : (a > b || (!(a < b) && ia > ib));
          if (gt == up) {
            key[i] = b; key[l] = a;
            idx[i] = ib; idx[l] = ia;
          }
        }
      }
      __syncthreads();
    }
  for (int i = threadIdx.x; i < lambda; i += 1024) order[i] = idx[i];
  if (threadIdx.x == 0) scal[CS_BEST_F] = key[0];
}

// Ys[r] = Y[order[r]];  YwT[d][r] = w°_r·Ys[r][d],  w°_r = w_r (w_r ≥ 0) or w_r·n/(‖z‖²+ε)
// rows r >= lambda (padding up to lam_pad) are written as zeros so the split-K GEMM can use uniform 256-wide slices
__global__ void cma_gather_kernel(const double* __restrict__ Y, const int* __restrict__ order, const double* __restrict__ w,
                                  const double* __restrict__ zn2, int lambda, int lam_pad, int D, double* __restrict__ Ys,
                                  double* __restrict__ YwT) {
  const int r = blockIdx.x;
  const bool live = r < lambda;
  const int src = live ? order[r] : 0;
  const double wr = live ? w[r] : 0.0;
  const double wio = wr >= 0.0 ? wr : wr * (double)D / (zn2[src] + CMA_EPS);
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const double v = live ? Y[(size_t)src * D + d] : 0.0;
    Ys[(size_t)r * D + d] = v;
    YwT[(size_t)d * lam_pad + r] = wio * v;
  }
}

// ------------------------------------------------------------------------------------------------ update (one CTA)
struct CmaConst {
  double mu_eff, c1, cmu, cm, c_sigma, d_sigma, cc, chi_n, wsum;
  int mu;
  long long gen;
};
__global__ void __launch_bounds__(1024) cma_update_kernel(const double* __restrict__ Ys, const double* __restrict__ w, int D, CmaConst k,
                                                          double* __restrict__ mean, const double* __restrict__ B,
                                                          const double* __restrict__ Dv, double* __restrict__ ps, double* __restrict__ pc,
                                                          double* __restrict__ scal, double* __restrict__ yw_out) {
  __shared__ double yw[CMA_MAXD], u[CMA_MAXD], red[1024];
  __shared__ double s_norm;
  const int t = threadIdx.x;
  // y_w = Σ_{r<μ} w_r Ys[r]: 1024/D threads per coordinate, fixed-order combine
  {
    const int per = 1024 / CMA_MAXD;  // 8 partial sums per coordinate
    const int d = t % CMA_MAXD, part = t / CMA_MAXD;
    double s = 0.0;
    if (d < D)
      for (int r = part; r < k.mu; r += per) s = fma(w[r], Ys[(size_t)r * D + d], s);
    red[t] = s;
    __syncthreads();
    if (t < D) {
      double a = 0.0;
      for (int p = 0; p < per; p++) a += red[p * CMA_MAXD + t];
      yw[t] = a;
      yw_out[t] = a;
    }
    __syncthreads();
  }
  const double sigma = scal[CS_SIGMA];
  if (t < D) mean[t] = fma(k.cm * sigma, yw[t], mean[t]);
  // C^{-1/2} y_w = B·((Bᵀ y_w)/d)
  if (t < D) {
    double a = 0.0;
    for (int i = 0; i < D; i++) a = fma(B[(size_t)i * D + t], yw[i], a);
    u[t] = a / Dv[t];
  }
  __syncthreads();
  if (t < D) {
    double a = 0.0;
    for (int j = 0; j < D; j++) a = fma(B[(size_t)t * D + j], u[j], a);
    const double v = (1.0 - k.c_sigma) * ps[t] + sqrt(k.c_sigma * (2.0 - k.c_sigma) * k.mu_eff) * a;
    ps[t] = v;
    red[t] = v * v;
  }
  __syncthreads();
  if (t == 0) {
    double a = 0.0;
    for (int i = 0; i < D; i++) a += red[i];
    s_norm = sqrt(a);
  }
  __syncthreads();
  const double norm_ps = s_norm;
  const double h_left = norm_ps / sqrt(1.0 - pow(1.0 - k.c_sigma, 2.0 * (double)(k.gen + 1)));
  const double h_sigma = h_left < (1.4 + 2.0 / (D + 1.0)) * k.chi_n ? 1.0 : 0.0;
  if (t < D) pc[t] = (1.0 - k.cc) * pc[t] + h_sigma * sqrt(k.cc * (2.0 - k.cc) * k.mu_eff) * yw[t];
  if (t == 0) {
    const double delta_h = (1.0 - h_sigma) * k.cc * (2.0 - k.cc);
    scal[CS_ALPHA_C] = 1.0 + k.c1 * delta_h - k.c1 - k.cmu * k.wsum;
    scal[CS_SIGMA] = sigma * exp((k.c_sigma / k.d_sigma) * (norm_ps / k.chi_n - 1.0));
  }
}
// C ← a·C + c1·p_c p_cᵀ + cμ·R, symmetrised ((C+Cᵀ)/2 as the reference does before its eigendecomposition)
// R arrives as `nsl` split-K partial sums (D×D each), added here in slice order (deterministic)
__global__ void cma_c_finalize_kernel(double* __restrict__ C, const double* __restrict__ R, int nsl, const double* __restrict__ pc,
                                      const double* __restrict__ scal, int D, double c1, double cmu) {
  const int i = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= D || j > i) return;
  const double a = scal[CS_ALPHA_C];
  double rij = 0.0, rji = 0.0;
  for (int z = 0; z < nsl; z++) {
    rij += R[(size_t)z * D * D + (size_t)i * D + j];
    rji += R[(size_t)z * D * D + (size_t)j * D + i];
  }
  const double v = a * 0.5 * (C[(size_t)i * D + j] + C[(size_t)j * D + i]) + c1 * pc[i] * pc[j] + cmu * 0.5 * (rij + rji);
  C[(size_t)i * D + j] = v;
  C[(size_t)j * D + i] = v;
}

// ------------------------------------------------------------------------------------------------ eigendecomposition
// One-sided (Hestenes) Jacobi on the columns of G = C·B_prev in shared memory (column-major, one column contiguous).
// Round-robin ordering: D/2 disjoint column pairs per step, 16 threads per pair.  On exit column j of G is λ_j·b_j.
// Rotations stop at |g_a·g_b| ≤ 1e-13·‖g_a‖‖g_b‖ (orthogonality of B to ~1e-13; the last quadratic sweep to 1e-16 buys nothing).
// DT = compile-time D (128: fully unrolled 8-row loops, loads pipelined) or 0 = runtime D.
template <int DT>
__global__ void __launch_bounds__(1024) cma_jacobi_kernel(const double* __restrict__ G, int Drt, double* __restrict__ B, double* __restrict__ scal,
                                                          int max_sweeps) {
  const int D = DT > 0 ? DT : Drt;
  extern __shared__ double Gt[];  // [Dp][D+1], Dp = D rounded up to even
  __shared__ int s_rot;
  const int Dp = (D + 1) & ~1, ldg = D + 1;
  const int t = threadIdx.x, pair = t >> 4, q = t & 15, npairs = Dp >> 1;
  for (int e = t; e < Dp * D; e += 1024) {
    const int j = e / D, i = e % D;
    Gt[j * ldg + i] = j < D ? G[(size_t)i * D + j] : 0.0;
  }
  __syncthreads();
  int sweep = 0;
  for (; sweep < max_sweeps; sweep++) {
    if (t == 0) s_rot = 0;
    __syncthreads();
    for (int step = 0; step < Dp - 1; step++) {
      for (int pk0 = 0; pk0 < npairs; pk0 += 64) {   // warp-uniform trip count: every lane takes part in the shuffles
        const int pk = pk0 + pair;
        const bool live = pk < npairs;
        int a = 0, b = 0;
        if (live) {
          if (pk == 0) {
            a = Dp - 1;
            b = step;
          } else {
            a = (step + pk) % (Dp - 1);
            b = (step - pk + Dp - 1) % (Dp - 1);
          }
        }
        const bool real = live && a < D && b < D;
        double* ga = Gt + a * ldg;
        double* gb = Gt + b * ldg;
        double al = 0.0, be = 0.0, ga_ = 0.0;
        if (real) {
#pragma unroll
          for (int i = q; i < D; i += 16) {
            const double x = ga[i], y = gb[i];
            al = fma(x, x, al);
            be = fma(y, y, be);
            ga_ = fma(x, y, ga_);
          }
        }
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) {
          al += __shfl_xor_sync(0xffffffffu, al, o);
          be += __shfl_xor_sync(0xffffffffu, be, o);
          ga_ += __shfl_xor_sync(0xffffffffu, ga_, o);
        }
        if (real && fabs(ga_) > 1e-13 * sqrt(al * be) && al > 0.0 && be > 0.0) {
          const double zeta = (be - al) / (2.0 * ga_);
          const double tt = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
          const double c = rsqrt(1.0 + tt * tt), s = c * tt;
#pragma unroll
          for (int i = q; i < D; i += 16) {
            const double x = ga[i], y = gb[i];
            ga[i] = c * x - s * y;
            gb[i] = s * x + c * y;
          }
          if (q == 0) s_rot = 1;
        }
      }
      __syncthreads();
    }
    const int rotated = s_rot;
    __syncthreads();
    if (!rotated) break;
  }
  // normalised columns are the eigenvectors (up to sign: a column's norm is |λ_j|, so cma_eigval_kernel takes λ_j itself).
  // Every nonzero column is written, a NaN one included (so a broken C shows in B instead of leaving it stale).  An exactly
  // zero column was never rotated (pairs with a zero column are skipped), so its warm-start vector, left in place, is the
  // eigenvector C annihilates; its d_j is the floor.
  for (int j0 = 0; j0 < D; j0 += 64) {
    const int j = j0 + pair;
    double n2 = 0.0;
    if (j < D)
      for (int i = q; i < D; i += 16) n2 = fma(Gt[j * ldg + i], Gt[j * ldg + i], n2);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) n2 += __shfl_xor_sync(0xffffffffu, n2, o);
    if (j < D && n2 != 0.0) {
      const double inv = 1.0 / sqrt(n2);
      for (int i = q; i < D; i += 16) B[(size_t)i * D + j] = Gt[j * ldg + i] * inv;
    }
  }
  if (t == 0) scal[CS_SWEEPS] = (double)(sweep + 1);
}
// d_j = √λ_j with λ_j = b_jᵀ C b_j (the Rayleigh quotient keeps the sign a column norm loses); only λ_j ≤ 0 is floored,
// at CMA_EPS, as the oracle does.  One CTA per eigenpair: thread (part, i) sums every 8th term of (C b_j)_i from column i
// of C (= row i, C being symmetric, so the loads coalesce) with all 16 loads in flight; fixed-order reductions.
__global__ void __launch_bounds__(1024) cma_eigval_kernel(const double* __restrict__ C, const double* __restrict__ B, int D,
                                                          double* __restrict__ Dv) {
  constexpr int PARTS = 1024 / CMA_MAXD;
  __shared__ double b[CMA_MAXD], red[1024];
  const int j = blockIdx.x, t = threadIdx.x, i = t % CMA_MAXD, part = t / CMA_MAXD;
  if (t < D) b[t] = B[(size_t)t * D + j];
  __syncthreads();
  double s = 0.0;
  if (i < D) {
    double c[CMA_MAXD / PARTS];
#pragma unroll
    for (int u = 0; u < CMA_MAXD / PARTS; u++) {
      const int k = part + u * PARTS;
      c[u] = k < D ? C[(size_t)k * D + i] : 0.0;
    }
#pragma unroll
    for (int u = 0; u < CMA_MAXD / PARTS; u++) {
      const int k = part + u * PARTS;
      if (k < D) s = fma(c[u], b[k], s);
    }
  }
  red[t] = s;
  __syncthreads();
  if (t < CMA_MAXD) {
    double a = 0.0;
    for (int p = 0; p < PARTS; p++) a += red[p * CMA_MAXD + t];
    red[t] = t < D ? a * b[t] : 0.0;
  }
  __syncthreads();
  for (int o = CMA_MAXD / 2; o > 0; o >>= 1) {
    if (t < o) red[t] += red[t + o];
    __syncthreads();
  }
  if (t == 0) {
    const double lam = red[0];
    Dv[j] = sqrt(lam <= 0.0 ? CMA_EPS : lam);
  }
}

__global__ void cma_init_kernel(double* __restrict__ C, double* __restrict__ B, double* __restrict__ Dv, double* __restrict__ ps,
                                double* __restrict__ pc, int D) {
  const int i = blockIdx.x, j = threadIdx.x;
  if (j < D) {
    C[(size_t)i * D + j] = i == j ? 1.0 : 0.0;
    B[(size_t)i * D + j] = i == j ? 1.0 : 0.0;
  }
  if (j == 0) {
    Dv[i] = 1.0;
    ps[i] = 0.0;
    pc[i] = 0.0;
  }
}

// ------------------------------------------------------------------------------------------------ termination test
// Criteria 4 and 5 are exact equality tests, so every rounding is the one `cmaes` makes in NumPy: products by __dmul_rn and
// sums by __dadd_rn (never contracted into a DFMA), and √c and max(d)/min(d) correctly rounded by the integer routines
// below (the library's FP64 sqrt and division are DFMA Newton sequences; these give the same IEEE results without one).
#define CMA_TOLXUP 1e4
#define CMA_TOLFUN 1e-12
#define CMA_TOLCONDCOV 1e14
enum CmaStop { STOP_TOLFUN = 1, STOP_TOLX = 2, STOP_TOLXUP = 4, STOP_NOEFFECTCOORD = 8, STOP_NOEFFECTAXIS = 16, STOP_CONDITIONCOV = 32 };

// RN(√x): digit-by-digit root of the 53-bit significand scaled to a 54-bit root, rounded to nearest-even by the remainder
__device__ double cma_sqrt_rn(double x) {
  if (x != x || x < 0.0) return __longlong_as_double(0x7ff8000000000000LL);
  if (x == 0.0 || x > 1.7976931348623157e308) return x;
  const unsigned long long bits = (unsigned long long)__double_as_longlong(x);
  int e = (int)(bits >> 52);
  unsigned long long m = bits & 0xfffffffffffffULL;
  if (e == 0) {                                   // subnormal: normalise the significand
    e = 1;
    while (!(m & (1ULL << 52))) { m <<= 1; e--; }
  } else {
    m |= 1ULL << 52;
  }
  int E = e - 1075;                               // x = m·2^E
  if (E & 1) { m <<= 1; E--; }                    // m < 2^54, E even
  unsigned long long r = 0, rem = 0;              // √(m·2^54) = r + rem-fraction, r < 2^54
  for (int i = 53; i >= 0; i--) {
    const unsigned long long pair = i >= 27 ? (m >> (2 * (i - 27))) & 3ULL : 0ULL;
    rem = (rem << 2) | pair;
    const unsigned long long trial = (r << 2) | 1ULL;
    if (rem >= trial) { rem -= trial; r = (r << 1) | 1ULL; } else { r <<= 1; }
  }
  unsigned long long q = r >> 1;                  // 53 bits; r's last bit is the guard, rem != 0 the sticky bit
  if ((r & 1ULL) && (rem != 0 || (q & 1ULL))) q++;
  const int k = (E - 54) / 2 + 1;                 // √x = q·2^k
  return __longlong_as_double((long long)((((unsigned long long)(k + 1074)) << 52) + q));
}
// RN(a/b) for positive normal a, b with a ≥ b (max(d)/min(d)): long division of the significands to 54 quotient bits
__device__ double cma_div_rn(double a, double b) {
  const unsigned long long ba = (unsigned long long)__double_as_longlong(a), bb = (unsigned long long)__double_as_longlong(b);
  unsigned long long ma = (ba & 0xfffffffffffffULL) | (1ULL << 52), mb = (bb & 0xfffffffffffffULL) | (1ULL << 52);
  int k = (int)(ba >> 52) - (int)(bb >> 52) - 52;  // a/b = (ma/mb)·2^(k+52)
  if (ma < mb) { ma <<= 1; k--; }
  unsigned long long Q = 0, rem = ma;
  for (int i = 0; i < 54; i++) {
    Q <<= 1;
    if (rem >= mb) { rem -= mb; Q |= 1ULL; }
    rem <<= 1;
  }
  unsigned long long q = Q >> 1;                  // a/b ≈ q·2^k, q in [2^52, 2^53)
  if ((Q & 1ULL) && (rem != 0 || (q & 1ULL))) q++;
  if (k + 1075 > 2046) return __longlong_as_double(0x7ff0000000000000LL);
  return __longlong_as_double((long long)((((unsigned long long)(k + 1074)) << 52) + q));   // q = 2^53 carries into the exponent
}

// One CTA of CMA_MAXD threads, after the tell on the tell's stream: records this generation's best and worst fitness
// (NumPy order, so the worst is NaN when any sample is) in slot 2·(g mod term) of the ring, then evaluates all six criteria
// on the updated state (g = strategy generation after the increment, i = g mod D for the axis test).
__global__ void __launch_bounds__(CMA_MAXD) cma_stop_kernel(const double* __restrict__ f, const int* __restrict__ order, int lambda, int D,
                                                            const double* __restrict__ mean, const double* __restrict__ C,
                                                            const double* __restrict__ B, const double* __restrict__ Dv,
                                                            const double* __restrict__ pc, const double* __restrict__ scal, double* hist,
                                                            int term, long long g, double tolx, unsigned* __restrict__ flags) {
  __shared__ double s_hi[CMA_MAXD / 32], s_lo[CMA_MAXD / 32], s_dhi[CMA_MAXD / 32], s_dlo[CMA_MAXD / 32];
  __shared__ int s_nan[CMA_MAXD / 32], s_dnan[CMA_MAXD / 32];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int slot = (int)(2 * (g % term));
  if (t == 0) hist[slot] = f[order[0]];
  if (t == 1) hist[slot + 1] = f[order[lambda - 1]];
  __syncthreads();
  // max / min of the history and of d, with NumPy's NaN propagation kept as a separate flag
  int hnan = 0, dnan = 0;
  double hi = -INFINITY, lo = INFINITY, dhi = -INFINITY, dlo = INFINITY;
  for (int i = t; i < 2 * term; i += CMA_MAXD) {
    const double v = hist[i];
    hnan |= v != v;
    hi = fmax(hi, v);
    lo = fmin(lo, v);
  }
  const double sigma = scal[CS_SIGMA];
  bool tolx_all = true, coord_any = false, axis_all = true;
  if (t < D) {
    const double c = C[(size_t)t * D + t], m = mean[t], d = Dv[t];
    dnan = d != d;
    dhi = d;
    dlo = d;
    tolx_all = __dmul_rn(sigma, c) < tolx && __dmul_rn(sigma, pc[t]) < tolx;
    coord_any = m == __dadd_rn(m, __dmul_rn(__dmul_rn(0.2, sigma), cma_sqrt_rn(c)));
    const int ax = (int)(g % D);
    axis_all = m == __dadd_rn(m, __dmul_rn(__dmul_rn(__dmul_rn(0.1, sigma), Dv[ax]), B[(size_t)t * D + ax]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    hnan |= __shfl_xor_sync(0xffffffffu, hnan, o);
    dnan |= __shfl_xor_sync(0xffffffffu, dnan, o);
    hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    dhi = fmax(dhi, __shfl_xor_sync(0xffffffffu, dhi, o));
    dlo = fmin(dlo, __shfl_xor_sync(0xffffffffu, dlo, o));
  }
  if (lane == 0) { s_hi[w] = hi; s_lo[w] = lo; s_dhi[w] = dhi; s_dlo[w] = dlo; s_nan[w] = hnan; s_dnan[w] = dnan; }
  tolx_all = __syncthreads_and(tolx_all);
  coord_any = __syncthreads_or(coord_any);
  axis_all = __syncthreads_and(axis_all);
  if (t == 0) {
    for (int i = 1; i < CMA_MAXD / 32; i++) {
      hi = fmax(hi, s_hi[i]); lo = fmin(lo, s_lo[i]); dhi = fmax(dhi, s_dhi[i]); dlo = fmin(dlo, s_dlo[i]);
      hnan |= s_nan[i]; dnan |= s_dnan[i];
    }
    unsigned fl = 0;
    if (g > term && !hnan && __dadd_rn(hi, -lo) < CMA_TOLFUN) fl |= STOP_TOLFUN;   // inf − inf is NaN: false
    if (tolx_all) fl |= STOP_TOLX;
    if (!dnan && __dmul_rn(sigma, dhi) > CMA_TOLXUP) fl |= STOP_TOLXUP;
    if (coord_any) fl |= STOP_NOEFFECTCOORD;
    if (axis_all) fl |= STOP_NOEFFECTAXIS;
    if (!dnan && (dhi > 1.7976931348623157e308 ? dlo <= 1.7976931348623157e308 : cma_div_rn(dhi, dlo) > CMA_TOLCONDCOV))
      fl |= STOP_CONDITIONCOV;                                                    // inf/finite = inf, inf/inf = NaN
    *flags = fl;
  }
}

// ------------------------------------------------------------------------------------------------ margin (CMAwM)
// CMA-ES with Margin (Hamano et al., GECCO 2022) as in CyberAgent `cmaes`: oracle/cma_margin_oracle.py states each rule.
// Levels and thresholds ℓ_k = (v_k + v_{k+1})/2 round as NumPy does (DMUL / DADD, never a contracted DFMA), so a sample
// encodes to the same level on both sides of a threshold.
__device__ __forceinline__ double cma_level(const CmaMarginDim& m, const double* __restrict__ lev, long long k) {
  return m.kind == 1 ? lev[m.off + k] : __dadd_rn(m.first, __dmul_rn((double)k, m.step));
}
__device__ __forceinline__ double cma_threshold(const CmaMarginDim& m, const double* __restrict__ lev, long long k) {
  return __dmul_rn(__dadd_rn(cma_level(m, lev, k), cma_level(m, lev, k + 1)), 0.5);
}
// number of thresholds ℓ_k (k < count − 1) with ℓ_k < x (below = false) or ℓ_k ≤ x (below = true), by binary search
__device__ __forceinline__ long long cma_rank(const CmaMarginDim& m, const double* __restrict__ lev, double x, bool below) {
  long long lo = 0, hi = m.count - 1;
  while (lo < hi) {
    const long long mid = lo + ((hi - lo) >> 1);
    const double l = cma_threshold(m, lev, mid);
    if (below ? l <= x : l < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// x = m + σ·(A∘y); a discrete coordinate encodes to the level whose interval (ℓ_{k−1}, ℓ_k] holds x (margin-free: cma_x_kernel)
__global__ void cma_x_margin_kernel(const double* __restrict__ Y, const double* __restrict__ mean, const double* __restrict__ scal,
                                    const double* __restrict__ A, const CmaMarginDim* __restrict__ md, const double* __restrict__ lev,
                                    int64_t n, int D, double* __restrict__ X) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int d = (int)(e % D);
  const double x = fma(scal[CS_SIGMA], A[d] * Y[e], mean[d]);
  const CmaMarginDim m = md[d];
  X[e] = m.kind == 0 ? x : cma_level(m, lev, cma_rank(m, lev, x, false));
}

// One CTA of CMA_MAXD threads, one per dimension, after cma_eigval_kernel.  The mean step of cma_update_kernel is redone
// with A from the (m, σ) it started from — m ← m + c_m·σ·A∘y_w, the same DFMA, so A_j = 1 reproduces it bit for bit —
// then each discrete dimension gets the margin correction of m_j and A_j at the updated σ and C.
__global__ void __launch_bounds__(CMA_MAXD) cma_margin_kernel(const double* __restrict__ mprev, const double* __restrict__ yw, double cm,
                                                              const double* __restrict__ scal, const double* __restrict__ C,
                                                              const CmaMarginDim* __restrict__ md, const double* __restrict__ lev, int D,
                                                              double alpha, double* __restrict__ mean, double* __restrict__ A,
                                                              double* __restrict__ mpre) {
  const int t = threadIdx.x;
  if (t >= D) return;
  const double a = A[t];
  double m = fma(cm * mprev[D], a * yw[t], mprev[t]);
  mpre[t] = m;
  const CmaMarginDim dm = md[t];
  if (dm.kind != 0) {
    const long long r = cma_rank(dm, lev, m, true);
    const double l_lo = cma_threshold(dm, lev, r == 0 ? 0 : r - 1);
    const double l_up = cma_threshold(dm, lev, r == dm.count - 1 ? r - 1 : r);
    const double sc = sqrt(C[(size_t)t * D + t]);
    const double s = __dmul_rn(__dmul_rn(scal[CS_SIGMA], a), sc);
    const double p_lo = normcdf(__dadd_rn(l_lo, -m) / s);
    const double p_up = normcdf(__dadd_rn(m, -l_up) / s);
    const double p_mid = __dadd_rn(__dadd_rn(1.0, -p_lo), -p_up);
    if (fmax(p_lo, p_up) > 0.5) {
      if (fmin(p_lo, p_up) < alpha) {
        const double sg = m > l_up ? 1.0 : (m < l_up ? -1.0 : 0.0);
        m = __dadd_rn(l_up, __dmul_rn(sg, __dmul_rn(s, -normcdfinv(alpha))));
      }
    } else {
      const double h = 0.5 * alpha;
      const double lo = fmax(p_lo, h), up = fmax(p_up, h);
      const double over = __dadd_rn(__dadd_rn(__dadd_rn(1.0, -lo), -up), -p_mid);
      const double den = __dadd_rn(__dadd_rn(__dadd_rn(lo, p_mid), up), -3.0 * h);
      double q_lo = __dadd_rn(lo, __dmul_rn(over, __dadd_rn(lo, -h)) / den);
      double q_up = __dadd_rn(up, __dmul_rn(over, __dadd_rn(up, -h)) / den);
      q_lo = fmin(fmax(q_lo, 1e-10), 0.5 - 1e-10);
      q_up = fmin(fmax(q_up, 1e-10), 0.5 - 1e-10);
      const double chi_lo = -normcdfinv(q_lo), chi_up = -normcdfinv(q_up);
      const double chi = __dadd_rn(chi_lo, chi_up);
      A[t] = __dadd_rn(l_up, -l_lo) / __dmul_rn(__dmul_rn(chi, scal[CS_SIGMA]), sc);
      m = __dadd_rn(__dmul_rn(l_lo, chi_up), __dmul_rn(l_up, chi_lo)) / chi;
    }
  }
  mean[t] = m;
}

// ------------------------------------------------------------------------------------------------ learning-rate adaptation (LRA)
// LRA-CMA-ES (Nomura, Akimoto & Ono, GECCO 2023) as in CyberAgent `cmaes`: oracle/cma_lra_oracle.py states each rule.
// The covariance side works in units of the plain update's σ′²: S = ΔΣ/σ′² = C′ − r²·C with r = σ/σ′, and the blended
// Σ/σ′² = r²·C + η_Σ·S goes into C for the unchanged eigendecomposition, so no σ² is ever formed.
#define LRA_ALPHA 1.4
#define LRA_BETA_M 0.1
#define LRA_BETA_S 0.03
#define LRA_GAMMA 0.1
#define LRA_SIGMA_MAX 1e32
enum LraScal { LS_V_M = 0, LS_V_S = 1, LS_ETA_M = 2, LS_ETA_S = 3, LS_ETA_M_PREV = 4, LS_COUNT = 5 };

// W = B·diag(1/d) of the basis from before the tell (P₀ = W·Bᵀ = C^{-1/2}), and S = C′ − r²·C_prev (exactly symmetric)
__global__ void cma_lra_prep_kernel(const double* __restrict__ B, const double* __restrict__ Dv, const double* __restrict__ C,
                                    const double* __restrict__ C0, const double* __restrict__ prev, const double* __restrict__ scal, int D,
                                    double* __restrict__ W, double* __restrict__ S) {
  const int i = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= D) return;
  const double r = prev[D] / scal[CS_SIGMA];
  const size_t e = (size_t)i * D + j;
  W[e] = B[e] / Dv[j];
  S[e] = C[e] - (r * r) * C0[e];
}

// The next η from one moving average's ‖E‖² and V; when V − ‖E‖² is not positive and finite, η stays (a stated departure)
__device__ __forceinline__ double cma_lra_eta(double eta, double E2, double V, double beta) {
  const double den = V - E2;
  if (!(den > 0.0 && den < INFINITY)) return eta;
  const double snr = (E2 - beta / (2.0 - beta) * V) / den;
  const double rel = fmin(fmax(snr / LRA_ALPHA / eta - 1.0, -1.0), 1.0);
  return fmin(eta * exp(fmin(LRA_GAMMA * eta, beta) * rel), 1.0);
}

// One CTA, after cma_c_finalize_kernel (mean = m′, σ′ in scal, C = C′) and the three products (L = P₀·S·P₀): local
// differences Δ̃m = P₀·Δm/σ and Δ̃Σ = L/(r²·√2), the moving averages, both SNRs and η, then m ← m + η_m·Δm and
// C ← r²·C_prev + η_Σ·S.  Per-thread sums in a fixed stride order, then a fixed tree: no atomics.
__global__ void __launch_bounds__(1024) cma_lra_kernel(const double* __restrict__ prev, const double* __restrict__ C0,
                                                       const double* __restrict__ P, const double* __restrict__ S,
                                                       const double* __restrict__ L, const double* __restrict__ scal, int D,
                                                       double* __restrict__ E, double* __restrict__ ls, double* __restrict__ mean,
                                                       double* __restrict__ C) {
  __shared__ double dm[CMA_MAXD], red[4][1024];
  __shared__ double s_eta[2];
  const int t = threadIdx.x;
  const double s0 = prev[D], r = s0 / scal[CS_SIGMA];
  const double cs = 0.7071067811865476 / (r * r);
  if (t < D) dm[t] = mean[t] - prev[t];
  __syncthreads();
  double a = 0.0, b = 0.0, a2 = 0.0, b2 = 0.0;
  if (t < D) {
    double u = 0.0;
    for (int j = 0; j < D; j++) u = fma(P[(size_t)t * D + j], dm[j], u);
    const double x = u / s0;
    const double e = (1.0 - LRA_BETA_M) * E[t] + LRA_BETA_M * x;
    E[t] = e;
    a = x * x;
    b = e * e;
  }
  double* ES = E + D;
  for (int k = t; k < D * D; k += 1024) {
    const double x = cs * L[k];
    const double e = (1.0 - LRA_BETA_S) * ES[k] + LRA_BETA_S * x;
    ES[k] = e;
    a2 = fma(x, x, a2);
    b2 = fma(e, e, b2);
  }
  red[0][t] = a; red[1][t] = b; red[2][t] = a2; red[3][t] = b2;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (t < o)
      for (int q = 0; q < 4; q++) red[q][t] += red[q][t + o];
    __syncthreads();
  }
  if (t == 0) {
    const double vm = (1.0 - LRA_BETA_M) * ls[LS_V_M] + LRA_BETA_M * red[0][0];
    const double vs = (1.0 - LRA_BETA_S) * ls[LS_V_S] + LRA_BETA_S * red[2][0];
    const double em = ls[LS_ETA_M];
    ls[LS_V_M] = vm;
    ls[LS_V_S] = vs;
    ls[LS_ETA_M_PREV] = em;
    s_eta[0] = ls[LS_ETA_M] = cma_lra_eta(em, red[1][0], vm, LRA_BETA_M);
    s_eta[1] = ls[LS_ETA_S] = cma_lra_eta(ls[LS_ETA_S], red[3][0], vs, LRA_BETA_S);
  }
  __syncthreads();
  const double eta_m = s_eta[0], eta_s = s_eta[1], r2 = r * r;
  if (t < D) mean[t] = fma(eta_m, dm[t], prev[t]);
  for (int k = t; k < D * D; k += 1024) C[k] = fma(eta_s, S[k], r2 * C0[k]);
}

// One CTA, after cma_eigval_kernel on the blended C = Σ/σ′²: σ = σ′·exp(Σ_j log d_j / D) (= exp(log det Σ / 2D), d_j²
// floored as cma_eigval_kernel floors), capped; C and d are divided by g = (σ/σ′)² and √g, so det C = 1; then the
// step-size correction σ·η_m(before)/η_m(after).  Runs before cma_stop_kernel, which reads the final state.
__global__ void __launch_bounds__(1024) cma_lra_finish_kernel(const double* __restrict__ ls, int D, double* __restrict__ Dv,
                                                              double* __restrict__ C, double* __restrict__ scal) {
  __shared__ double red[CMA_MAXD];
  __shared__ double s_r;
  const int t = threadIdx.x;
  if (t < CMA_MAXD) red[t] = t < D ? log(Dv[t]) : 0.0;
  __syncthreads();
  for (int o = CMA_MAXD / 2; o > 0; o >>= 1) {
    if (t < o) red[t] += red[t + o];
    __syncthreads();
  }
  if (t == 0) {
    const double s1 = scal[CS_SIGMA];
    double sn = s1 * exp(red[0] / D);
    if (sn > LRA_SIGMA_MAX) sn = LRA_SIGMA_MAX;
    s_r = sn / s1;
    scal[CS_SIGMA] = sn * ls[LS_ETA_M_PREV] / ls[LS_ETA_M];
  }
  __syncthreads();
  const double rr = s_r, g = rr * rr;
  if (t < D) Dv[t] = Dv[t] / rr;
  for (int k = t; k < D * D; k += 1024) C[k] = C[k] / g;
}

// The LRA step between cma_c_finalize_kernel and the eigendecomposition: W and S, P₀ = W·Bᵀ, L = (P₀·S)·P₀, the blend
static int cma_lra_blend(kbo_handle* h, kbo_cma* c, cudaStream_t s) {
  const int D = c->D;
  double *W = c->lW.p, *P = c->lP.p, *S = c->lS.p, *T = c->lT.p, *L = c->lL.p;
  cma_lra_prep_kernel<<<dim3((D + 127) / 128, D), 128, 0, s>>>(c->B.p, c->Dv.p, c->C.p,
                                                                c->lC0.p, c->lprev.p,
                                                                c->scal.p, D, W, S);
  KBO_LAUNCH_CHECK(h);
  dgemm64_launch<true, EPI_STORE>(s, D, D, D, W, D, c->B.p, D, P, D, 1.0, 0.0, KM_FULL, 0, TS_NONE);
  KBO_LAUNCH_CHECK(h);
  dgemm64_launch<false, EPI_STORE>(s, D, D, D, P, D, S, D, T, D, 1.0, 0.0, KM_FULL, 0, TS_NONE);
  KBO_LAUNCH_CHECK(h);
  dgemm64_launch<false, EPI_STORE>(s, D, D, D, T, D, P, D, L, D, 1.0, 0.0, KM_FULL, 0, TS_NONE);
  KBO_LAUNCH_CHECK(h);
  cma_lra_kernel<<<1, 1024, 0, s>>>(c->lprev.p, c->lC0.p, P, S, L, c->scal.p, D,
                                    c->lE.p, c->lscal.p, c->mean.p, c->C.p);
  KBO_LAUNCH_CHECK(h);
  return KBO_OK;
}

// ------------------------------------------------------------------------------------------------ separable CMA-ES (sep-CMA)
// sep-CMA-ES (Ros & Hansen, PPSN 2008) as CyberAgent `cmaes`' SepCMA: oracle/sepcma_oracle.py states each rule.  C is kept
// as its diagonal and d = √C, so a generation is O(λ·D) and D goes to SEP_MAXD.  The ask is cma_normal_kernel,
// cma_scale_kernel (y = d∘z; its ‖z‖² is not used) and cma_x_kernel; the tell is cma_sort_kernel and the three kernels
// below.  Every reduction has a fixed order and there are no atomics, so a run replays bit for bit.
#define SEP_MAXD 4096
#define SEP_UPD_THREADS 256
#define SEP_FIN_THREADS 1024
#define SEP_STOP_THREADS 256
#define SEP_SIGMA_MAX 1e32

struct kbo_sepcma {
  int D = 0, lambda = 0, mu = 0, lam_pow2 = 0, nparts = 0;  // nparts: CTAs of sepcma_update_kernel
  uint64_t seed = 0;
  long long gen = 0;    // strategy generation: back to 0 at every restart
  long long draws = 0;  // Philox counter of the built-in sampler: one per tell, never reset
  double mu_eff, c1, cmu, cm, c_sigma, d_sigma, cc, chi_n;
  int term = 0;
  double tolx = 0.0;
  DevBuf<double> mean, C, Dv, ps, pc, weights, Z, Y, zn2, scal, yw, wy2, part, hist;  // C, Dv: the diagonal and √ of it
  DevBuf<int> order;
  DevBuf<unsigned> flags;
  bool asked = false;
};

struct SepConst {
  double mu_eff, c1, cmu, cm, c_sigma, d_sigma, cc, chi_n;
};

// One thread per dimension j: over the μ best samples in rank order, y_w,j = Σ w_r y_r,j and Σ w_r y_r,j²; then
// m_j ← m_j + c_m·σ·y_w,j and p_σ,j ← (1 − c_σ)·p_σ,j + √(c_σ(2 − c_σ)μ_eff)·y_w,j/d_j (d from before the tell).  Each CTA
// writes its Σ p_σ,j² by a fixed tree to part[blockIdx.x].
__global__ void __launch_bounds__(SEP_UPD_THREADS) sepcma_update_kernel(const double* __restrict__ Y, const int* __restrict__ order,
                                                                        const double* __restrict__ w, int D, int mu, SepConst k,
                                                                        double* __restrict__ mean, const double* __restrict__ Dv,
                                                                        double* __restrict__ ps, const double* __restrict__ scal,
                                                                        double* __restrict__ yw, double* __restrict__ wy2,
                                                                        double* __restrict__ part) {
  __shared__ double red[SEP_UPD_THREADS];
  const int t = threadIdx.x, j = blockIdx.x * SEP_UPD_THREADS + t;
  double v2 = 0.0;
  if (j < D) {
    double a = 0.0, b = 0.0;
#pragma unroll 4
    for (int r = 0; r < mu; r++) {
      const double y = Y[(size_t)order[r] * D + j], wr = w[r];
      a = fma(wr, y, a);
      b = fma(wr * y, y, b);
    }
    yw[j] = a;
    wy2[j] = b;
    mean[j] = fma(k.cm * scal[CS_SIGMA], a, mean[j]);
    const double v = (1.0 - k.c_sigma) * ps[j] + sqrt(k.c_sigma * (2.0 - k.c_sigma) * k.mu_eff) * (a / Dv[j]);
    ps[j] = v;
    v2 = v * v;
  }
  red[t] = v2;
  __syncthreads();
  for (int o = SEP_UPD_THREADS / 2; o > 0; o >>= 1) {
    if (t < o) red[t] += red[t + o];
    __syncthreads();
  }
  if (t == 0) part[blockIdx.x] = red[0];
}

// One CTA: ‖p_σ‖ from the partials in CTA order, then σ (capped), h_σ, and per dimension p_c, C and d = √C (C_j ≤ 0
// floored at CMA_EPS under the root, as the oracle does).
__global__ void __launch_bounds__(SEP_FIN_THREADS) sepcma_finish_kernel(const double* __restrict__ part, int nparts, int D, SepConst k,
                                                                        long long gen, const double* __restrict__ yw,
                                                                        const double* __restrict__ wy2, double* __restrict__ pc,
                                                                        double* __restrict__ C, double* __restrict__ Dv,
                                                                        double* __restrict__ scal) {
  __shared__ double s_h;
  const int t = threadIdx.x;
  if (t == 0) {
    double a = 0.0;
    for (int i = 0; i < nparts; i++) a += part[i];
    const double norm_ps = sqrt(a);
    const double h_left = norm_ps / sqrt(1.0 - pow(1.0 - k.c_sigma, 2.0 * (double)(gen + 1)));
    s_h = h_left < (1.4 + 2.0 / (D + 1.0)) * k.chi_n ? 1.0 : 0.0;
    const double sigma = scal[CS_SIGMA] * exp((k.c_sigma / k.d_sigma) * (norm_ps / k.chi_n - 1.0));
    scal[CS_SIGMA] = sigma > SEP_SIGMA_MAX ? SEP_SIGMA_MAX : sigma;
  }
  __syncthreads();
  const double h = s_h;
  const double a = 1.0 + k.c1 * ((1.0 - h) * k.cc * (2.0 - k.cc)) - k.c1 - k.cmu;
  const double pcoef = h * sqrt(k.cc * (2.0 - k.cc) * k.mu_eff);
  for (int j = t; j < D; j += SEP_FIN_THREADS) {
    const double p = (1.0 - k.cc) * pc[j] + pcoef * yw[j];
    pc[j] = p;
    const double c = a * C[j] + k.c1 * (p * p) + k.cmu * wy2[j];
    C[j] = c;
    Dv[j] = sqrt(c <= 0.0 ? CMA_EPS : c);
  }
}

// One CTA striding over D, after the tell: the history ring and five of cma_stop_kernel's criteria with its rounding
// rules (no NOEFFECTAXIS: there is no basis).  TOLX tests σ·C_j, as cma_stop_kernel tests σ·C_ii.
__global__ void __launch_bounds__(SEP_STOP_THREADS) sepcma_should_stop_kernel(const double* __restrict__ f, const int* __restrict__ order,
                                                                       int lambda, int D, const double* __restrict__ mean,
                                                                       const double* __restrict__ C, const double* __restrict__ Dv,
                                                                       const double* __restrict__ pc, const double* __restrict__ scal,
                                                                       double* hist, int term, long long g, double tolx,
                                                                       unsigned* __restrict__ flags) {
  constexpr int NW = SEP_STOP_THREADS / 32;
  __shared__ double s_hi[NW], s_lo[NW], s_dhi[NW], s_dlo[NW];
  __shared__ int s_nan[NW], s_dnan[NW];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int slot = (int)(2 * (g % term));
  if (t == 0) hist[slot] = f[order[0]];
  if (t == 1) hist[slot + 1] = f[order[lambda - 1]];
  __syncthreads();
  int hnan = 0, dnan = 0;
  double hi = -INFINITY, lo = INFINITY, dhi = -INFINITY, dlo = INFINITY;
  for (int i = t; i < 2 * term; i += SEP_STOP_THREADS) {
    const double v = hist[i];
    hnan |= v != v;
    hi = fmax(hi, v);
    lo = fmin(lo, v);
  }
  const double sigma = scal[CS_SIGMA];
  const double s02 = __dmul_rn(0.2, sigma);
  bool tolx_all = true, coord_any = false;
  for (int j = t; j < D; j += SEP_STOP_THREADS) {
    const double c = C[j], m = mean[j], d = Dv[j];
    dnan |= d != d;
    dhi = fmax(dhi, d);
    dlo = fmin(dlo, d);
    tolx_all &= __dmul_rn(sigma, c) < tolx && __dmul_rn(sigma, pc[j]) < tolx;
    coord_any |= m == __dadd_rn(m, __dmul_rn(s02, cma_sqrt_rn(c)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    hnan |= __shfl_xor_sync(0xffffffffu, hnan, o);
    dnan |= __shfl_xor_sync(0xffffffffu, dnan, o);
    hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    dhi = fmax(dhi, __shfl_xor_sync(0xffffffffu, dhi, o));
    dlo = fmin(dlo, __shfl_xor_sync(0xffffffffu, dlo, o));
  }
  if (lane == 0) { s_hi[w] = hi; s_lo[w] = lo; s_dhi[w] = dhi; s_dlo[w] = dlo; s_nan[w] = hnan; s_dnan[w] = dnan; }
  tolx_all = __syncthreads_and(tolx_all);
  coord_any = __syncthreads_or(coord_any);
  if (t == 0) {
    for (int i = 1; i < NW; i++) {
      hi = fmax(hi, s_hi[i]); lo = fmin(lo, s_lo[i]); dhi = fmax(dhi, s_dhi[i]); dlo = fmin(dlo, s_dlo[i]);
      hnan |= s_nan[i]; dnan |= s_dnan[i];
    }
    unsigned fl = 0;
    if (g > term && !hnan && __dadd_rn(hi, -lo) < CMA_TOLFUN) fl |= STOP_TOLFUN;
    if (tolx_all) fl |= STOP_TOLX;
    if (!dnan && __dmul_rn(sigma, dhi) > CMA_TOLXUP) fl |= STOP_TOLXUP;
    if (coord_any) fl |= STOP_NOEFFECTCOORD;
    if (!dnan && (dhi > 1.7976931348623157e308 ? dlo <= 1.7976931348623157e308 : cma_div_rn(dhi, dlo) > CMA_TOLCONDCOV))
      fl |= STOP_CONDITIONCOV;
    *flags = fl;
  }
}

// ------------------------------------------------------------------------------------------------ host side
static int cma_generation_tell(kbo_handle* h, kbo_cma* c, const double* fitness, cudaStream_t s) {
  const int D = c->D, lam = c->lambda;
  const int smem_sort = c->lam_pow2 * 12;
  cma_sort_kernel<<<1, 1024, smem_sort, s>>>(fitness, lam, c->lam_pow2, c->order.p, c->scal.p);
  KBO_LAUNCH_CHECK(h);
  cma_gather_kernel<<<c->lam_pad, 128, 0, s>>>(c->Y.p, c->order.p, c->weights.p, c->zn2.p, lam,
                                               c->lam_pad, D, c->Ys.p, c->YwT.p);
  KBO_LAUNCH_CHECK(h);
  CmaConst k{c->mu_eff, c->c1, c->cmu, c->cm, c->c_sigma, c->d_sigma, c->cc, c->chi_n, c->wsum, c->mu, c->gen};
  if (c->n_disc) {   // (m, σ) the update starts from, for the margin kernel's A-scaled mean step
    KBO_CUDA(h, kbo_copy(c->mprev.p, c->mean.p, (size_t)D, cudaMemcpyDeviceToDevice, s));
    KBO_CUDA(h, kbo_copy(c->mprev.p + D, c->scal.p, 1, cudaMemcpyDeviceToDevice, s));
  }
  if (c->lra) {      // (m, σ) and C the update starts from, for the learning-rate adaptation after it
    KBO_CUDA(h, kbo_copy(c->lprev.p, c->mean.p, (size_t)D, cudaMemcpyDeviceToDevice, s));
    KBO_CUDA(h, kbo_copy(c->lprev.p + D, c->scal.p, 1, cudaMemcpyDeviceToDevice, s));
    KBO_CUDA(h, kbo_copy(c->lC0.p, c->C.p, (size_t)D * D, cudaMemcpyDeviceToDevice, s));
  }
  cma_update_kernel<<<1, 1024, 0, s>>>(c->Ys.p, c->weights.p, D, k, c->mean.p, c->B.p,
                                       c->Dv.p, c->ps.p, c->pc.p, c->scal.p, c->yw.p);
  KBO_LAUNCH_CHECK(h);
  // R = Σ w°_i y_i y_iᵀ  (D×D = YwT[D×λ]·Ys[λ×D]) as split-K over 256-sample slices: a 128×128 output is only two
  // tiles of the GEMM, so without the split a K = 4096 product ran on 2 CTAs; the slices fill 2·λ/256 CTAs
  const int nsl = c->lam_pad / 256;
  dgemm64_launch<false, EPI_STORE>(s, D, D, 256, c->YwT.p, c->lam_pad, c->Ys.p, D, c->R.p, D, 1.0, 0.0, KM_FULL,
                                   0, TS_NONE, nsl, 256, 256LL * D, (long long)D * D);
  KBO_LAUNCH_CHECK(h);
  dim3 g((D + 127) / 128, D);
  cma_c_finalize_kernel<<<g, 128, 0, s>>>(c->C.p, c->R.p, nsl, c->pc.p, c->scal.p, D, c->c1,
                                          c->cmu);
  KBO_LAUNCH_CHECK(h);
  if (c->lra) KBO_TRY(cma_lra_blend(h, c, s));   // B and Dv are still C_prev's here; C becomes the blended Σ/σ′²
  // G = C·B_prev, then Jacobi
  dgemm64_launch<false, EPI_STORE>(s, D, D, D, c->C.p, D, c->B.p, D, c->G.p, D, 1.0, 0.0, KM_FULL, 0, TS_NONE);
  KBO_LAUNCH_CHECK(h);
  const int Dp = (D + 1) & ~1;
  if (D == 128)
    cma_jacobi_kernel<128><<<1, 1024, sizeof(double) * Dp * (D + 1), s>>>(c->G.p, D, c->B.p, c->scal.p, 30);
  else
    cma_jacobi_kernel<0><<<1, 1024, sizeof(double) * Dp * (D + 1), s>>>(c->G.p, D, c->B.p, c->scal.p, 30);
  KBO_LAUNCH_CHECK(h);
  cma_eigval_kernel<<<D, 1024, 0, s>>>(c->C.p, c->B.p, D, c->Dv.p);
  KBO_LAUNCH_CHECK(h);
  if (c->n_disc) {
    cma_margin_kernel<<<1, CMA_MAXD, 0, s>>>(c->mprev.p, c->yw.p, c->cm, c->scal.p,
                                             c->C.p, c->mdim.p, c->mlev.p, D, c->alpha,
                                             c->mean.p, c->A.p, c->mpre.p);
    KBO_LAUNCH_CHECK(h);
  }
  if (c->lra) {
    cma_lra_finish_kernel<<<1, 1024, 0, s>>>(c->lscal.p, D, c->Dv.p, c->C.p, c->scal.p);
    KBO_LAUNCH_CHECK(h);
  }
  cma_stop_kernel<<<1, CMA_MAXD, 0, s>>>(fitness, c->order.p, lam, D, c->mean.p, c->C.p,
                                         c->B.p, c->Dv.p, c->pc.p, c->scal.p,
                                         c->hist.p, c->term, c->gen + 1, c->tolx, c->flags.p);
  KBO_LAUNCH_CHECK(h);
  c->gen++;
  c->draws++;
  c->asked = false;
  return KBO_OK;
}

static int cma_generation_ask(kbo_handle* h, kbo_cma* c, double* X, const double* z_in, cudaStream_t s) {
  const int D = c->D, lam = c->lambda;
  const int64_t n = (int64_t)lam * D;
  const double* Z = z_in;
  if (!Z) {
    cma_normal_kernel<<<(unsigned)((n / 2 + 1 + 255) / 256), 256, 0, s>>>(c->Z.p, n, c->seed, (uint64_t)c->draws);
    KBO_LAUNCH_CHECK(h);
    Z = c->Z.p;
  }
  cma_scale_kernel<<<(lam + 7) / 8, 256, 0, s>>>(Z, c->Dv.p, lam, D, c->Zs.p, c->zn2.p);
  KBO_LAUNCH_CHECK(h);
  // Y[k,i] = Σ_j Zs[k,j]·B[i,j]
  dgemm64_launch<true, EPI_STORE>(s, lam, D, D, c->Zs.p, D, c->B.p, D, c->Y.p, D, 1.0, 0.0, KM_FULL, 0, TS_NONE);
  KBO_LAUNCH_CHECK(h);
  if (c->n_disc)
    cma_x_margin_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(c->Y.p, c->mean.p, c->scal.p,
                                                                     c->A.p, c->mdim.p,
                                                                     c->mlev.p, n, D, X);
  else
    cma_x_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(c->Y.p, c->mean.p, c->scal.p, n, D, X);
  KBO_LAUNCH_CHECK(h);
  c->asked = true;
  return KBO_OK;
}

// Strategy parameters for population λ (tutorial Table 1; active weights as in `cmaes`), the buffers they size, and the
// termination constants of a run starting at σ0.  Shared by create and restart; uploads the weights (synchronous copy).
static int cma_configure(kbo_handle* h, kbo_cma* c, int lambda, double sigma0) {
  const int D = c->D;
  c->lambda = lambda;
  c->mu = lambda / 2;
  int p2 = 1;
  while (p2 < lambda) p2 <<= 1;
  c->lam_pow2 = p2;
  c->lam_pad = round_up(lambda, 256);
  std::vector<double> w(lambda);
  const int mu = c->mu, n = D;
  double s1 = 0, s2 = 0, m1 = 0, m2 = 0;
  for (int i = 0; i < lambda; i++) {
    w[i] = log((lambda + 1) / 2.0) - log((double)(i + 1));
    if (i < mu) { s1 += w[i]; s2 += w[i] * w[i]; } else { m1 += w[i]; m2 += w[i] * w[i]; }
  }
  const double mu_eff = s1 * s1 / s2, mu_eff_minus = m1 * m1 / m2, alpha_cov = 2.0;
  const double c1 = alpha_cov / ((n + 1.3) * (n + 1.3) + mu_eff);
  double cmu = alpha_cov * (mu_eff - 2 + 1 / mu_eff) / ((n + 2.0) * (n + 2.0) + alpha_cov * mu_eff / 2);
  if (cmu > 1 - c1 - 1e-8) cmu = 1 - c1 - 1e-8;
  double min_alpha = 1 + c1 / cmu;
  if (1 + (2 * mu_eff_minus) / (mu_eff + 2) < min_alpha) min_alpha = 1 + (2 * mu_eff_minus) / (mu_eff + 2);
  if ((1 - c1 - cmu) / (n * cmu) < min_alpha) min_alpha = (1 - c1 - cmu) / (n * cmu);
  double pos = 0, neg = 0;
  for (int i = 0; i < lambda; i++) (w[i] > 0 ? pos : neg) += fabs(w[i]);
  double wsum = 0;
  for (int i = 0; i < lambda; i++) {
    w[i] = w[i] >= 0 ? w[i] / pos : min_alpha / neg * w[i];
    wsum += w[i];
  }
  c->mu_eff = mu_eff; c->c1 = c1; c->cmu = cmu; c->cm = 1.0; c->wsum = wsum;
  c->c_sigma = (mu_eff + 2) / (n + mu_eff + 5);
  const double t = sqrt((mu_eff - 1) / (n + 1)) - 1;
  c->d_sigma = 1 + 2 * (t > 0 ? t : 0) + c->c_sigma;
  c->cc = (4 + mu_eff / n) / (n + 4 + 2 * mu_eff / n);
  c->chi_n = sqrt((double)n) * (1.0 - 1.0 / (4.0 * n) + 1.0 / (21.0 * n * n));
  c->term = 10 + (30 * n + lambda - 1) / lambda;   // 10 + ⌈30·n/λ⌉
  c->tolx = 1e-12 * sigma0;
  const size_t LD = (size_t)lambda * D, LPD = (size_t)c->lam_pad * D;
  KBO_TRY(kbo_reserve(h, c->mean, D));
  KBO_TRY(kbo_reserve(h, c->C, (size_t)D * D));
  KBO_TRY(kbo_reserve(h, c->B, (size_t)D * D));
  KBO_TRY(kbo_reserve(h, c->Dv, D));
  KBO_TRY(kbo_reserve(h, c->ps, D));
  KBO_TRY(kbo_reserve(h, c->pc, D));
  KBO_TRY(kbo_reserve(h, c->weights, lambda));
  KBO_TRY(kbo_reserve(h, c->Z, LD + 2));
  KBO_TRY(kbo_reserve(h, c->Zs, LD));
  KBO_TRY(kbo_reserve(h, c->Y, LD));
  KBO_TRY(kbo_reserve(h, c->Ys, LPD));
  KBO_TRY(kbo_reserve(h, c->YwT, LPD));
  KBO_TRY(kbo_reserve(h, c->zn2, lambda));
  KBO_TRY(kbo_reserve(h, c->order, lambda));
  KBO_TRY(kbo_reserve(h, c->R, (size_t)D * D * (c->lam_pad / 256)));
  KBO_TRY(kbo_reserve(h, c->G, (size_t)D * D));
  KBO_TRY(kbo_reserve(h, c->scal, CS_COUNT));
  KBO_TRY(kbo_reserve(h, c->yw, D));
  KBO_TRY(kbo_reserve(h, c->hist, (size_t)c->term * 2));
  KBO_TRY(kbo_reserve(h, c->flags, 1));
  KBO_TRY(kbo_upload(h, c->weights, w.data(), lambda));
  return KBO_OK;
}

// A run's starting state: mean0, σ0, C = B = I, d = 1, zero paths, history and flags, strategy generation 0.
static int cma_start_run(kbo_handle* h, kbo_cma* c, const double* mean0, double sigma0) {
  const int D = c->D;
  double sc[CS_COUNT] = {sigma0, 0, 0, 0, 0, 0, 0, 0};
  cudaMemcpy(c->mean.p, mean0, sizeof *c->mean.p * D, cudaMemcpyHostToDevice);
  cudaMemcpy(c->scal.p, sc, sizeof sc, cudaMemcpyHostToDevice);
  cma_init_kernel<<<D, 128>>>(c->C.p, c->B.p, c->Dv.p, c->ps.p, c->pc.p, D);
  cudaMemset(c->hist.p, 0, sizeof *c->hist.p * 2 * (size_t)c->term);
  cudaMemset(c->flags.p, 0, sizeof *c->flags.p);
  KBO_CUDA(h, cudaDeviceSynchronize());
  c->gen = 0;
  c->asked = false;
  return KBO_OK;
}

// A run's margin state: A = 1, and α = the caller's or the default 1/(D·λ) of the current λ (synchronous)
static int cma_margin_reset(kbo_handle* h, kbo_cma* c) {
  if (!c->n_disc) return KBO_OK;
  c->alpha = c->alpha_set > 0.0 ? c->alpha_set : 1.0 / ((double)c->D * c->lambda);
  const std::vector<double> ones(c->D, 1.0);
  KBO_TRY(kbo_upload(h, c->A, ones.data(), c->D));
  return KBO_OK;
}

// A run's LRA state: E = 0, V = 0, η = 1 (synchronous)
static int cma_lra_reset(kbo_handle* h, kbo_cma* c) {
  if (!c->lra) return KBO_OK;
  const double ls[LS_COUNT] = {0.0, 0.0, 1.0, 1.0, 1.0};
  KBO_CUDA(h, cudaMemset(c->lE.p, 0, sizeof *c->lE.p * (size_t)c->D * (c->D + 1)));
  KBO_TRY(kbo_upload(h, c->lscal, ls, LS_COUNT));
  return KBO_OK;
}

extern "C" {

int kbo_cma_set_lr_adapt(kbo_handle* h, kbo_cma* c, int32_t on) {
  if (!h || !c) return KBO_ERR_INVALID;
  if (c->asked) KBO_FAIL(h, KBO_ERR_STATE, "kbo_cma_set_lr_adapt: the last ask has not been told");
  if (on && c->n_disc) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_set_lr_adapt: learning-rate adaptation is not available with margin dimensions");
  KBO_CUDA(h, cudaSetDevice(h->device));
  KBO_CUDA(h, cudaDeviceSynchronize());            // a tell in flight may still use the state about to be reset
  c->lra = false;
  if (!on) return KBO_OK;
  const size_t D = c->D, DD = D * D;
  KBO_TRY(kbo_reserve(h, c->lprev, D + 1));
  KBO_TRY(kbo_reserve(h, c->lC0, DD));
  KBO_TRY(kbo_reserve(h, c->lW, DD));
  KBO_TRY(kbo_reserve(h, c->lP, DD));
  KBO_TRY(kbo_reserve(h, c->lS, DD));
  KBO_TRY(kbo_reserve(h, c->lT, DD));
  KBO_TRY(kbo_reserve(h, c->lL, DD));
  KBO_TRY(kbo_reserve(h, c->lE, D * (D + 1)));
  KBO_TRY(kbo_reserve(h, c->lscal, LS_COUNT));
  c->lra = true;
  return cma_lra_reset(h, c);
}

int kbo_cma_lra_state(kbo_handle* h, kbo_cma* c, double* E_mean_host, double* E_Sigma_host, double* V_host, double* eta_host, void* stream) {
  if (!h || !c) return KBO_ERR_INVALID;
  if (!c->lra) KBO_FAIL(h, KBO_ERR_STATE, "kbo_cma_lra_state: learning-rate adaptation is off");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t D = c->D;
  double ls[LS_COUNT];
  KBO_CUDA(h, kbo_d2h(E_mean_host, c->lE.p, D, s));
  KBO_CUDA(h, kbo_d2h(E_Sigma_host, c->lE.p + D, D * D, s));
  KBO_CUDA(h, kbo_copy(ls, c->lscal.p, LS_COUNT, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (V_host) { V_host[0] = ls[LS_V_M]; V_host[1] = ls[LS_V_S]; }
  if (eta_host) { eta_host[0] = ls[LS_ETA_M]; eta_host[1] = ls[LS_ETA_S]; }
  return KBO_OK;
}

int kbo_cma_set_margin(kbo_handle* h, kbo_cma* c, int32_t n_discrete, const int32_t* dims, const int64_t* level_offsets,
                       const double* levels, const double* arith, double alpha) {
  if (!h || !c) return KBO_ERR_INVALID;
  if (c->asked) KBO_FAIL(h, KBO_ERR_STATE, "kbo_cma_set_margin: the last ask has not been told");
  if (n_discrete < 0 || n_discrete > c->D) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_set_margin: 0 <= n_discrete <= D required (got %d)", n_discrete);
  if (!(alpha == 0.0 || (alpha > 0.0 && alpha < 1.0))) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_set_margin: alpha must be in (0, 1), or 0 for 1/(D*lambda)");
  if (n_discrete && c->lra) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_set_margin: margin dimensions are not available with learning-rate adaptation");
  if (n_discrete && (!dims || !level_offsets)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_set_margin: dims and level_offsets must be given");
  const int D = c->D;
  std::vector<CmaMarginDim> md(D, CmaMarginDim{0.0, 0.0, 0, 0, 0});
  const int64_t n_lev = n_discrete ? level_offsets[n_discrete] : 0;
  if (level_offsets && (level_offsets[0] != 0 || n_lev < 0)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_set_margin: level_offsets must start at 0");
  if (n_lev && !levels) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_set_margin: null levels");
  for (int i = 0; i < n_discrete; i++) {
    const int d = dims[i];
    if (d < 0 || d >= D || (i && d <= dims[i - 1])) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_set_margin: dims must be increasing in [0, D)");
    const int64_t off = level_offsets[i], k = level_offsets[i + 1] - off;
    if (k < 0 || level_offsets[i + 1] > n_lev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_set_margin: level_offsets must be non-decreasing");
    if (k) {
      for (int64_t j = 0; j < k; j++)
        if (!std::isfinite(levels[off + j]) || (j && !(levels[off + j] > levels[off + j - 1])))
          KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_set_margin: dimension %d: levels must be finite and increasing", d);
      if (k < 2) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_set_margin: dimension %d: a discrete dimension needs 2 or more levels", d);
      md[d] = CmaMarginDim{0.0, 0.0, (long long)k, (long long)off, 1};
    } else {
      if (!arith) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_set_margin: dimension %d has no level table and arith is null", d);
      const double first = arith[3 * i], step = arith[3 * i + 1], cnt = arith[3 * i + 2];
      if (!std::isfinite(first) || !(step > 0.0) || !std::isfinite(step) || !(cnt >= 2.0 && cnt <= 9007199254740992.0) || cnt != std::floor(cnt))
        KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_set_margin: dimension %d: arithmetic levels need finite first, step > 0 and an integer count >= 2", d);
      md[d] = CmaMarginDim{first, step, (long long)cnt, 0, 2};
    }
  }
  KBO_CUDA(h, cudaSetDevice(h->device));
  KBO_CUDA(h, cudaDeviceSynchronize());            // a tell in flight may still read the tables about to be replaced
  c->n_disc = 0;
  if (!n_discrete) return KBO_OK;
  KBO_TRY(kbo_reserve(h, c->A, (size_t)D));
  KBO_TRY(kbo_reserve(h, c->mprev, (size_t)(D + 1)));
  KBO_TRY(kbo_reserve(h, c->mpre, (size_t)D));
  KBO_TRY(kbo_upload(h, c->mdim, md.data(), D));
  KBO_TRY(kbo_upload(h, c->mlev, levels, (size_t)n_lev));
  KBO_CUDA(h, cudaMemcpy(c->mpre.p, c->mean.p, sizeof *c->mpre.p * D, cudaMemcpyDeviceToDevice));
  c->n_disc = n_discrete;
  c->alpha_set = alpha;
  return cma_margin_reset(h, c);
}

int kbo_cma_margin_state(kbo_handle* h, kbo_cma* c, double* A_host, double* mean_before_host, double* alpha_host, void* stream) {
  if (!h || !c) return KBO_ERR_INVALID;
  if (!c->n_disc) KBO_FAIL(h, KBO_ERR_STATE, "kbo_cma_margin_state: no margin is set");
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, kbo_d2h(A_host, c->A.p, (size_t)c->D, s));
  KBO_CUDA(h, kbo_d2h(mean_before_host, c->mpre.p, (size_t)c->D, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (alpha_host) *alpha_host = c->alpha;
  return KBO_OK;
}

int kbo_cma_create(kbo_handle* h, kbo_cma** out, int32_t D, int32_t lambda, const double* mean0, double sigma0, uint64_t seed) {
  if (!h || !out) return KBO_ERR_INVALID;
  *out = nullptr;
  if (D < 1 || D > CMA_MAXD) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_create: 1 <= D <= %d supported (got %d)", CMA_MAXD, D);
  if (lambda < 4 || lambda > 8192) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_create: 4 <= lambda <= 8192 supported (got %d)", lambda);
  if (!mean0 || !(sigma0 > 0.0)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_create: mean0 must be given and sigma0 > 0");
  KBO_CUDA(h, cudaSetDevice(h->device));
  std::unique_ptr<kbo_cma> c(new (std::nothrow) kbo_cma());
  if (!c) return KBO_ERR_NOMEM;
  c->D = D;
  c->seed = seed;
  KBO_TRY(cma_configure(h, c.get(), lambda, sigma0));
  cudaFuncSetAttribute(cma_jacobi_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(double) * CMA_MAXD * (CMA_MAXD + 1)));
  cudaFuncSetAttribute(cma_jacobi_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(double) * CMA_MAXD * (CMA_MAXD + 1)));
  cudaFuncSetAttribute(cma_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 12);
  KBO_TRY(cma_start_run(h, c.get(), mean0, sigma0));
  *out = c.release();
  return KBO_OK;
}

int kbo_cma_restart(kbo_handle* h, kbo_cma* c, int32_t lambda, const double* mean0, double sigma0) {
  if (!h || !c) return KBO_ERR_INVALID;
  if (lambda < 4 || lambda > 8192) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_restart: 4 <= lambda <= 8192 supported (got %d)", lambda);
  if (!mean0 || !(sigma0 > 0.0)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_restart: mean0 must be given and sigma0 > 0");
  KBO_CUDA(h, cudaSetDevice(h->device));
  KBO_CUDA(h, cudaDeviceSynchronize());            // the last tell may still be reading buffers that are about to grow
  KBO_TRY(cma_configure(h, c, lambda, sigma0));
  KBO_TRY(cma_margin_reset(h, c));
  KBO_TRY(cma_lra_reset(h, c));
  return cma_start_run(h, c, mean0, sigma0);
}

int kbo_cma_stop_flags(kbo_handle* h, kbo_cma* c, uint32_t* flags_host, double* funhist_host, int32_t* term_host, void* stream) {
  if (!h || !c) return KBO_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, kbo_d2h(flags_host, c->flags.p, 1, s));
  KBO_CUDA(h, kbo_d2h(funhist_host, c->hist.p, (size_t)c->term * 2, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (term_host) *term_host = c->term;
  return KBO_OK;
}

void kbo_cma_destroy(kbo_cma* c) {
  if (c) delete c;
}

int kbo_cma_ask(kbo_handle* h, kbo_cma* c, double* X_dev, const double* z_in_dev, void* stream) {
  if (!h || !c) return KBO_ERR_INVALID;
  if (!X_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_ask: null output");
  return cma_generation_ask(h, c, X_dev, z_in_dev, (cudaStream_t)stream);
}

int kbo_cma_tell(kbo_handle* h, kbo_cma* c, const double* fitness_dev, void* stream) {
  if (!h || !c) return KBO_ERR_INVALID;
  if (!fitness_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_tell: null fitness");
  if (!c->asked) KBO_FAIL(h, KBO_ERR_STATE, "kbo_cma_tell: call kbo_cma_ask first (tell ranks the samples of the last ask)");
  return cma_generation_tell(h, c, fitness_dev, (cudaStream_t)stream);
}

int kbo_cma_state(kbo_handle* h, kbo_cma* c, double* mean, double* sigma, double* C, double* p_sigma, double* p_c, double* B, double* Dv,
                  double* Y_last, int64_t* generation, void* stream) {
  if (!h || !c) return KBO_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  const size_t D = c->D;
  KBO_CUDA(h, kbo_d2h(mean, c->mean.p, D, s));
  KBO_CUDA(h, kbo_d2h(sigma, c->scal.p, 1, s));
  KBO_CUDA(h, kbo_d2h(C, c->C.p, D * D, s));
  KBO_CUDA(h, kbo_d2h(p_sigma, c->ps.p, D, s));
  KBO_CUDA(h, kbo_d2h(p_c, c->pc.p, D, s));
  KBO_CUDA(h, kbo_d2h(B, c->B.p, D * D, s));
  KBO_CUDA(h, kbo_d2h(Dv, c->Dv.p, D, s));
  KBO_CUDA(h, kbo_d2h(Y_last, c->Y.p, D * c->lambda, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (generation) *generation = c->gen;
  return KBO_OK;
}

int kbo_cma_run_synthetic(kbo_handle* h, kbo_cma* c, int32_t fitness_kind, int32_t generations, double* best_f_host, float* elapsed_ms,
                          double* jacobi_sweeps_last) {
  if (!h || !c) return KBO_ERR_INVALID;
  if (fitness_kind < 0 || fitness_kind > 1 || generations < 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_cma_run_synthetic: bad argument");
  cudaStream_t s = 0;
  DevBuf<double> X, f;
  KBO_TRY(kbo_reserve(h, X, (size_t)c->lambda * c->D));
  KBO_TRY(kbo_reserve(h, f, (size_t)c->lambda));
  cudaEventRecord(h->ev[5], s);
  int r = KBO_OK;
  for (int g = 0; g < generations && r == KBO_OK; g++) {
    r = cma_generation_ask(h, c, X.p, nullptr, s);
    if (r != KBO_OK) break;
    cma_fitness_kernel<<<(c->lambda + 7) / 8, 256, 0, s>>>(X.p, c->lambda, c->D, fitness_kind, f.p);
    h->launches++;
    r = cma_generation_tell(h, c, f.p, s);
  }
  cudaEventRecord(h->ev[6], s);
  double sc[CS_COUNT];
  kbo_copy(sc, c->scal.p, CS_COUNT, cudaMemcpyDeviceToHost, s);
  cudaError_t e = cudaStreamSynchronize(s);
  if (r != KBO_OK) return r;
  if (e != cudaSuccess) KBO_FAIL(h, KBO_ERR_CUDA, "kbo_cma_run_synthetic: %s", cudaGetErrorString(e));
  if (best_f_host) *best_f_host = sc[CS_BEST_F];
  if (jacobi_sweeps_last) *jacobi_sweeps_last = sc[CS_SWEEPS];
  if (elapsed_ms) cudaEventElapsedTime(elapsed_ms, h->ev[5], h->ev[6]);
  return KBO_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ separable CMA-ES: host side
// Strategy parameters for population λ (positive weights only; sep-CMA's c_c, c1 and (D + 2)/3-scaled cμ, capped at
// 1 − c1 − 1e-8 as the full path caps it), the buffers
// they size, and the termination constants of a run starting at σ0.  Shared by create and restart.
static int sepcma_configure(kbo_handle* h, kbo_sepcma* c, int lambda, double sigma0) {
  const int D = c->D, mu = lambda / 2;
  const double n = D;
  c->lambda = lambda;
  c->mu = mu;
  int p2 = 1;
  while (p2 < lambda) p2 <<= 1;
  c->lam_pow2 = p2;
  c->nparts = (D + SEP_UPD_THREADS - 1) / SEP_UPD_THREADS;
  std::vector<double> w(mu);
  double s1 = 0, s2 = 0;
  for (int i = 0; i < mu; i++) {
    w[i] = log((lambda + 1) / 2.0) - log((double)(i + 1));
    s1 += w[i];
  }
  for (int i = 0; i < mu; i++) {
    w[i] /= s1;
    s2 += w[i] * w[i];
  }
  const double mu_eff = 1.0 / s2;
  c->mu_eff = mu_eff;
  c->cm = 1.0;
  c->c_sigma = (mu_eff + 2) / (n + mu_eff + 5);
  const double t = sqrt((mu_eff - 1) / (n + 1)) - 1;
  c->d_sigma = 1 + 2 * (t > 0 ? t : 0) + c->c_sigma;
  c->cc = 4.0 / (n + 4.0);
  c->c1 = 2.0 / ((n + 1.3) * (n + 1.3) + mu_eff);
  const double r = (2 * mu_eff - 1) / ((n + 2) * (n + 2) + mu_eff);
  c->cmu = (n + 2) / 3.0 * (2.0 / mu_eff / ((n + sqrt(2.0)) * (n + sqrt(2.0))) + (1 - 1 / mu_eff) * (r < 1 ? r : 1.0));
  if (c->cmu > 1 - c->c1 - 1e-8) c->cmu = 1 - c->c1 - 1e-8;   // past 1 at large λ, C's own coefficient would turn negative
  c->chi_n = sqrt(n) * (1.0 - 1.0 / (4.0 * n) + 1.0 / (21.0 * n * n));
  c->term = 10 + (30 * D + lambda - 1) / lambda;   // 10 + ⌈30·n/λ⌉
  c->tolx = 1e-12 * sigma0;
  const size_t LD = (size_t)lambda * D;
  KBO_TRY(kbo_reserve(h, c->mean, D));
  KBO_TRY(kbo_reserve(h, c->C, D));
  KBO_TRY(kbo_reserve(h, c->Dv, D));
  KBO_TRY(kbo_reserve(h, c->ps, D));
  KBO_TRY(kbo_reserve(h, c->pc, D));
  KBO_TRY(kbo_reserve(h, c->Z, LD + 2));
  KBO_TRY(kbo_reserve(h, c->Y, LD));
  KBO_TRY(kbo_reserve(h, c->zn2, lambda));
  KBO_TRY(kbo_reserve(h, c->order, lambda));
  KBO_TRY(kbo_reserve(h, c->scal, CS_COUNT));
  KBO_TRY(kbo_reserve(h, c->yw, D));
  KBO_TRY(kbo_reserve(h, c->wy2, D));
  KBO_TRY(kbo_reserve(h, c->part, c->nparts));
  KBO_TRY(kbo_reserve(h, c->hist, (size_t)c->term * 2));
  KBO_TRY(kbo_reserve(h, c->flags, 1));
  KBO_TRY(kbo_upload(h, c->weights, w.data(), mu));
  return KBO_OK;
}

// A run's starting state: mean0, σ0, C = d = 1, zero paths, history and flags, strategy generation 0 (synchronous).
static int sepcma_start_run(kbo_handle* h, kbo_sepcma* c, const double* mean0, double sigma0) {
  const int D = c->D;
  const double sc[CS_COUNT] = {sigma0, 0, 0, 0, 0, 0, 0, 0};
  const std::vector<double> ones(D, 1.0);
  KBO_CUDA(h, cudaMemcpy(c->mean.p, mean0, sizeof *c->mean.p * D, cudaMemcpyHostToDevice));
  KBO_CUDA(h, cudaMemcpy(c->scal.p, sc, sizeof sc, cudaMemcpyHostToDevice));
  KBO_CUDA(h, cudaMemcpy(c->C.p, ones.data(), sizeof *c->C.p * D, cudaMemcpyHostToDevice));
  KBO_CUDA(h, cudaMemcpy(c->Dv.p, ones.data(), sizeof *c->Dv.p * D, cudaMemcpyHostToDevice));
  KBO_CUDA(h, cudaMemset(c->ps.p, 0, sizeof *c->ps.p * D));
  KBO_CUDA(h, cudaMemset(c->pc.p, 0, sizeof *c->pc.p * D));
  KBO_CUDA(h, cudaMemset(c->hist.p, 0, sizeof *c->hist.p * 2 * (size_t)c->term));
  KBO_CUDA(h, cudaMemset(c->flags.p, 0, sizeof *c->flags.p));
  KBO_CUDA(h, cudaDeviceSynchronize());
  c->gen = 0;
  c->asked = false;
  return KBO_OK;
}

static int sepcma_generation_ask(kbo_handle* h, kbo_sepcma* c, double* X, const double* z_in, cudaStream_t s) {
  const int D = c->D, lam = c->lambda;
  const int64_t n = (int64_t)lam * D;
  const double* Z = z_in;
  if (!Z) {
    cma_normal_kernel<<<(unsigned)((n / 2 + 1 + 255) / 256), 256, 0, s>>>(c->Z.p, n, c->seed, (uint64_t)c->draws);
    KBO_LAUNCH_CHECK(h);
    Z = c->Z.p;
  }
  cma_scale_kernel<<<(lam + 7) / 8, 256, 0, s>>>(Z, c->Dv.p, lam, D, c->Y.p, c->zn2.p);   // Y = d∘z
  KBO_LAUNCH_CHECK(h);
  cma_x_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(c->Y.p, c->mean.p, c->scal.p, n, D, X);
  KBO_LAUNCH_CHECK(h);
  c->asked = true;
  return KBO_OK;
}

static int sepcma_generation_tell(kbo_handle* h, kbo_sepcma* c, const double* fitness, cudaStream_t s) {
  const int D = c->D, lam = c->lambda;
  const SepConst k{c->mu_eff, c->c1, c->cmu, c->cm, c->c_sigma, c->d_sigma, c->cc, c->chi_n};
  cma_sort_kernel<<<1, 1024, c->lam_pow2 * 12, s>>>(fitness, lam, c->lam_pow2, c->order.p, c->scal.p);
  KBO_LAUNCH_CHECK(h);
  sepcma_update_kernel<<<c->nparts, SEP_UPD_THREADS, 0, s>>>(c->Y.p, c->order.p, c->weights.p, D, c->mu, k, c->mean.p, c->Dv.p,
                                                             c->ps.p, c->scal.p, c->yw.p, c->wy2.p, c->part.p);
  KBO_LAUNCH_CHECK(h);
  sepcma_finish_kernel<<<1, SEP_FIN_THREADS, 0, s>>>(c->part.p, c->nparts, D, k, c->gen, c->yw.p, c->wy2.p, c->pc.p, c->C.p,
                                                     c->Dv.p, c->scal.p);
  KBO_LAUNCH_CHECK(h);
  sepcma_should_stop_kernel<<<1, SEP_STOP_THREADS, 0, s>>>(fitness, c->order.p, lam, D, c->mean.p, c->C.p, c->Dv.p, c->pc.p, c->scal.p,
                                                    c->hist.p, c->term, c->gen + 1, c->tolx, c->flags.p);
  KBO_LAUNCH_CHECK(h);
  c->gen++;
  c->draws++;
  c->asked = false;
  return KBO_OK;
}

extern "C" {

int kbo_sepcma_create(kbo_handle* h, kbo_sepcma** out, int32_t D, int32_t lambda, const double* mean0, double sigma0, uint64_t seed) {
  if (!h || !out) return KBO_ERR_INVALID;
  *out = nullptr;
  if (D < 1 || D > SEP_MAXD) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sepcma_create: 1 <= D <= %d supported (got %d)", SEP_MAXD, D);
  if (lambda < 4 || lambda > 8192) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sepcma_create: 4 <= lambda <= 8192 supported (got %d)", lambda);
  if (!mean0 || !(sigma0 > 0.0)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sepcma_create: mean0 must be given and sigma0 > 0");
  KBO_CUDA(h, cudaSetDevice(h->device));
  std::unique_ptr<kbo_sepcma> c(new (std::nothrow) kbo_sepcma());
  if (!c) return KBO_ERR_NOMEM;
  c->D = D;
  c->seed = seed;
  KBO_TRY(sepcma_configure(h, c.get(), lambda, sigma0));
  cudaFuncSetAttribute(cma_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 12);
  KBO_TRY(sepcma_start_run(h, c.get(), mean0, sigma0));
  *out = c.release();
  return KBO_OK;
}

void kbo_sepcma_destroy(kbo_sepcma* c) {
  if (c) delete c;
}

int kbo_sepcma_restart(kbo_handle* h, kbo_sepcma* c, int32_t lambda, const double* mean0, double sigma0) {
  if (!h || !c) return KBO_ERR_INVALID;
  if (lambda < 4 || lambda > 8192) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sepcma_restart: 4 <= lambda <= 8192 supported (got %d)", lambda);
  if (!mean0 || !(sigma0 > 0.0)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sepcma_restart: mean0 must be given and sigma0 > 0");
  KBO_CUDA(h, cudaSetDevice(h->device));
  KBO_CUDA(h, cudaDeviceSynchronize());            // the last tell may still be reading buffers that are about to grow
  KBO_TRY(sepcma_configure(h, c, lambda, sigma0));
  return sepcma_start_run(h, c, mean0, sigma0);
}

int kbo_sepcma_ask(kbo_handle* h, kbo_sepcma* c, double* X_dev, const double* z_in_dev, void* stream) {
  if (!h || !c) return KBO_ERR_INVALID;
  if (!X_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sepcma_ask: null output");
  return sepcma_generation_ask(h, c, X_dev, z_in_dev, (cudaStream_t)stream);
}

int kbo_sepcma_tell(kbo_handle* h, kbo_sepcma* c, const double* fitness_dev, void* stream) {
  if (!h || !c) return KBO_ERR_INVALID;
  if (!fitness_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sepcma_tell: null fitness");
  if (!c->asked) KBO_FAIL(h, KBO_ERR_STATE, "kbo_sepcma_tell: call kbo_sepcma_ask first (tell ranks the samples of the last ask)");
  return sepcma_generation_tell(h, c, fitness_dev, (cudaStream_t)stream);
}

int kbo_sepcma_state(kbo_handle* h, kbo_sepcma* c, double* mean, double* sigma, double* C_diag, double* p_sigma, double* p_c, double* Dv,
                     double* Y_last, int64_t* generation, void* stream) {
  if (!h || !c) return KBO_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  const size_t D = c->D;
  KBO_CUDA(h, kbo_d2h(mean, c->mean.p, D, s));
  KBO_CUDA(h, kbo_d2h(sigma, c->scal.p, 1, s));
  KBO_CUDA(h, kbo_d2h(C_diag, c->C.p, D, s));
  KBO_CUDA(h, kbo_d2h(p_sigma, c->ps.p, D, s));
  KBO_CUDA(h, kbo_d2h(p_c, c->pc.p, D, s));
  KBO_CUDA(h, kbo_d2h(Dv, c->Dv.p, D, s));
  KBO_CUDA(h, kbo_d2h(Y_last, c->Y.p, D * c->lambda, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (generation) *generation = c->gen;
  return KBO_OK;
}

int kbo_sepcma_stop_flags(kbo_handle* h, kbo_sepcma* c, uint32_t* flags_host, double* funhist_host, int32_t* term_host, void* stream) {
  if (!h || !c) return KBO_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, kbo_d2h(flags_host, c->flags.p, 1, s));
  KBO_CUDA(h, kbo_d2h(funhist_host, c->hist.p, (size_t)c->term * 2, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (term_host) *term_host = c->term;
  return KBO_OK;
}

}  // extern "C"
