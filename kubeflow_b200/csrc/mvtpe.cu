// Multivariate Parzen estimator on the device — Katib's `multivariate-tpe` algorithm (Optuna 3.x's
// TPESampler(multivariate=True) on a flat space; the FP64 restatement that is the contract is oracle/mvtpe_oracle.py,
// DESIGN.md §7 "multivariate-tpe").
//   history : values in parameter units (grid values for integers, category indices for categoricals) and FP64 losses,
//             appended as trials are told; NaN losses and values outside a parameter's domain are refused
//   models  : one stable radix sort of the losses splits the history into the n_below = min(ceil(0.1·n), 25) best ("below")
//             and the rest ("above"), both in told order.  Each group is a mixture of one component per observation (its
//             values as means, one shared sigma per parameter) plus the prior; mvtpe_model_kernel writes every component's
//             constant c_k in FP64, mvtpe_table_kernel the integer offset tables
//   ask     : candidate vectors come from Philox4x32-10 keyed by (seed, ask, point, candidate, slot) — slot 0 picks a
//             component of the below mixture, slot 1 + d inverts parameter d's CDF under it — or from the caller.  Every
//             candidate is scored in FP32 (mvtpe_score_kernel: candidates × components register tiles over parameter slabs,
//             exact differences, online log-sum-exp with ex2.approx) with an error bound; whatever can still be the maximum is
//             re-scored in FP64 (mvtpe_decide_kernel) and the first index of the FP64 maximum wins.
#include <algorithm>
#include <cmath>

#include <cub/device/device_radix_sort.cuh>

#include "kbo_internal.cuh"
#include "kbo_rng.cuh"
#include "kbo_tpe_common.cuh"

#define MV_BM 64              // candidates per score block: 16 thread rows × 4
#define MV_BN 128             // components per tile: 16 thread columns × 8
#define MV_DS 32              // float parameters per staged slab
#define MV_DDS 16             // integer / categorical parameters per staged slab
#define MV_LCAP (1 << 16)     // integer parameters with at most this many levels score through an offset table
#define MV_MAXM (1 << 24)
#define MV_MAXD 65535
#define MV_PW 1.0             // Optuna's prior_weight
#define MV_T2 40.0f           // log2 distance below the maximum past which a term counts as "far" in the error bound
#define MV_RESCALE 64.0f      // a thread's running maximum is raised only when a tile's maximum passes it by this much (log2)
#define MV_H2 0.72134752044448170  // ½·log2(e)
#define MV_EPS_EX2 9.5367432e-7f   // 2^-20: relative error allowed for ex2.approx.ftz.f32 (the PTX ISA documents about 2 ulp)
#define MV_LN_SQRT_2PI 0.91893853320467274
#define MV_LOG2E 1.4426950408889634

struct MvParam {
  int kind;     // kbo_mvtpe_kind
  int slot;     // index among the float parameters, or among the discrete (integer + categorical) ones
  int levels;   // integer: grid points lo, lo + q, ..., hi; categorical: categories
  int pad;
  long long tab;       // integer with levels <= MV_LCAP: offset of its table in a group's tables; else -1
  double lo, hi, q;    // integer: hi is the last grid point
  double lo2, hi2;     // integer: lo - q/2, hi + q/2; float: lo, hi
  double pm, ps;       // the prior component: (lo2 + hi2) / 2, hi2 - lo2
  double lpm;          // log of the prior's N(pm, ps²) mass over [lo2, hi2]
  double lcat, b;      // categorical: log(pw/C) - log(pw + 1) (a row's shared normaliser), log(pw/C + 1) - log(pw/C) (the match)
};
struct MvHdr {  // one per group
  int m, pad;             // observation components
  double lwp;             // log of the prior's normalised weight
  float Bsum, XM;         // Σ match bonuses (log2), max over float parameters of the scaled range
  unsigned kCmax, kCabs;  // ordered keys of max c2 and max |c2| (log2 units), written by mvtpe_model_kernel
};
struct MvModels {
  const MvParam* prm;
  const int *flt, *dsc, *idx, *dv;
  const double *vals, *w, *c64, *sg, *fs, *tab64;
  const float *c2, *mu32, *tab32;
  const MvHdr* hdr;
  int D, Df, Dd, mcap;
  long long ltab;      // entries of a group's tables (the sum of the tabled integers' levels)
};

struct kbo_mvtpe {
  int D = 0, Df = 0, Dd = 0, lmax = 1;
  long long ltab = 0;
  std::vector<MvParam> prm;
  std::vector<int> flt, dsc, tabd;
  uint64_t seed = 0;
  uint32_t asks = 0;
  int n = 0, cap = 0, built_n = -1, nb = 0, mcap = 0;
  uint32_t pick_ask = 0;            // the last shard ask: its ask number, k, n_candidates and history size, for kbo_mvtpe_pick
  int pick_k = 0, pick_M = 0, pick_n = -1;
  DevBuf<MvParam> d_prm;
  DevBuf<int> d_flt, d_dsc, d_tabd;
  DevBuf<double> vals, loss;
  DevBuf<int> err;
  DevBuf<uint64_t> lkey, lkey2;
  DevBuf<int> lidx, lidx2, below, grp, pos;
  DevBuf<unsigned char> tmp;
  DevBuf<int> idx, dv;
  DevBuf<double> w, c64, sg, fs, tab64;
  DevBuf<float> c2, mu32, tab32;
  DevBuf<MvHdr> hdr;
  DevBuf<double> draws, prior;
  DevBuf<float2> sc;
  DevBuf<unsigned> lb;
  DevBuf<int> surv;
  DevBuf<TpeBest> bb;
  std::vector<int> last_surv;
  EventSet<5> ev;
  float last_ms[4] = {};
};

// ------------------------------------------------------------------------------------------------ FP64 helpers
// log Φ(x) without underflow or cancellation (Optuna's _log_ndtr)
__device__ __forceinline__ double mv_log_ndtr(double x) {
  if (x > 5.0) return log1p(-normcdf(-x));
  if (x > -1.0) return log(normcdf(x));
  return log(0.5 * erfcx(-x * 0.70710678118654752)) - 0.5 * x * x;
}
// log of the N(0, 1) mass of [a, b], a < b (Optuna's _log_gauss_mass): in a tail the difference of two log Φ through expm1,
// mirrored so that it is always the left tail; across 0 the mass as a sum of two erfs, so neither side cancels
__device__ __forceinline__ double mv_log_gauss_mass(double a, double b) {
  if (a > 0.0) {
    const double t = a;
    a = -b;
    b = -t;
  }
  if (b <= 0.0) {
    const double la = mv_log_ndtr(a), lb = mv_log_ndtr(b);
    return lb + log(-expm1(la - lb));
  }
  return log(0.5 * (erf(b * 0.70710678118654752) + erf(-a * 0.70710678118654752)));
}
__device__ __forceinline__ int mv_level(const MvParam& P, double x) { return (int)rint((x - P.lo) / P.q); }
__device__ __forceinline__ double mv_grid(const MvParam& P, int j) { return __dadd_rn(P.lo, __dmul_rn((double)j, P.q)); }
// f_d(j) in nats: log mass of the offset j·q under the group's sigma (observation means lie on the grid)
__device__ __forceinline__ double mv_int_term64(const MvParam& P, double sg, int j) {
  const double r = P.q / sg;
  return mv_log_gauss_mass(((double)j - 0.5) * r, ((double)j + 0.5) * r);
}

// ------------------------------------------------------------------------------------------------ history
// a told row is usable: finite float values in [lo, hi], integers on their grid, category indices in range, loss not NaN
__global__ void mvtpe_check_kernel(const MvParam* __restrict__ prm, int D, const double* __restrict__ X, const double* __restrict__ loss, int n,
                                   int* __restrict__ err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (loss[i] != loss[i]) atomicMax(err, 1);
  for (int d = 0; d < D; d++) {
    const MvParam P = prm[d];
    const double x = X[(size_t)i * D + d];
    bool ok;
    if (P.kind == KBO_MVTPE_FLOAT) {
      ok = x >= P.lo && x <= P.hi;
    } else if (P.kind == KBO_MVTPE_INT) {
      const double j = rint((x - P.lo) / P.q);
      ok = j >= 0.0 && j < (double)P.levels && x == mv_grid(P, (int)j);
    } else {
      ok = x >= 0.0 && x < (double)P.levels && x == floor(x);
    }
    if (!ok) atomicMax(err, 2);
  }
}

// ------------------------------------------------------------------------------------------------ model build
// idx[g][pos] = trial: each group's members in told order
__global__ void mvtpe_members_kernel(const int* __restrict__ grp, const int* __restrict__ pos, int n, int mcap, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) idx[(size_t)grp[i] * mcap + pos[i]] = i;
}
// Optuna's default_weights(m) in told order, prior_weight appended, normalised; one CTA per group
__global__ void __launch_bounds__(256) mvtpe_weights_kernel(int mcap, MvHdr* __restrict__ hdr, double* __restrict__ W) {
  const int g = blockIdx.x, m = hdr[g].m;
  double* w = W + (size_t)g * (mcap + 1);
  double part = 0.0;
  for (int k = threadIdx.x; k < m; k += blockDim.x) part += tpe_lfw(k, m);
  const double sum = tpe_block_reduce<false>(part) + MV_PW;
  for (int k = threadIdx.x; k < m; k += blockDim.x) w[k] = tpe_lfw(k, m) / sum;
  if (threadIdx.x == 0) {
    w[m] = MV_PW / sum;
    hdr[g].lwp = log(MV_PW / sum);
  }
}
// per observation component k of group g: c_k = log w_k + Σ_float (-log σ - ½log 2π - log mass over [lo, hi])
// + Σ_int (-log mass over [lo2, hi2]) + Σ_cat (log(pw/C) - log(pw + 1)), in FP64 (c64, nats) and FP32 (c2, log2 units);
// the scaled float means and the discrete values in the score kernel's layouts
__global__ void __launch_bounds__(256) mvtpe_model_kernel(MvModels md, double* __restrict__ C64, float* __restrict__ C2, float* __restrict__ MU32,
                                                          int* __restrict__ DV, MvHdr* __restrict__ hdr) {
  const int g = blockIdx.y, k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= md.hdr[g].m) return;
  const int i = md.idx[(size_t)g * md.mcap + k];
  double c = log(md.w[(size_t)g * (md.mcap + 1) + k]);
  for (int d = 0; d < md.D; d++) {
    const MvParam P = md.prm[d];
    const double x = md.vals[(size_t)i * md.D + d];
    if (P.kind == KBO_MVTPE_CAT) {
      c += P.lcat;
      DV[((size_t)g * md.Dd + P.slot) * md.mcap + k] = (int)x;
      continue;
    }
    const double sg = md.sg[(size_t)g * md.D + d];
    c -= mv_log_gauss_mass((P.lo2 - x) / sg, (P.hi2 - x) / sg);
    if (P.kind == KBO_MVTPE_FLOAT) {
      c -= log(sg) + MV_LN_SQRT_2PI;
      MU32[((size_t)g * md.Df + P.slot) * md.mcap + k] = (float)((x - P.pm) * md.fs[(size_t)g * md.Df + P.slot]);
    } else {
      DV[((size_t)g * md.Dd + P.slot) * md.mcap + k] = mv_level(P, x);
    }
  }
  C64[(size_t)g * md.mcap + k] = c;
  const float c2 = (float)(c * MV_LOG2E);
  C2[(size_t)g * md.mcap + k] = c2;
  atomicMax(&hdr[g].kCmax, tpe_fkey(c2));
  atomicMax(&hdr[g].kCabs, tpe_fkey(fabsf(c2)));
}
// the offset tables of the integer parameters with at most MV_LCAP levels: f(j), j = 0 .. levels - 1, in nats and log2 units
__global__ void mvtpe_table_kernel(MvModels md, const int* __restrict__ tabd, double* __restrict__ T64, float* __restrict__ T32) {
  const int g = blockIdx.z, d = tabd[blockIdx.y], j = blockIdx.x * blockDim.x + threadIdx.x;
  const MvParam P = md.prm[d];
  if (j >= P.levels) return;
  const double v = mv_int_term64(P, md.sg[(size_t)g * md.D + d], j);
  T64[(size_t)g * md.ltab + P.tab + j] = v;
  T32[(size_t)g * md.ltab + P.tab + j] = (float)(v * MV_LOG2E);
}

// ------------------------------------------------------------------------------------------------ ask: candidates
// candidate m of point p: a component of the below mixture ∝ w_k (slot 0), then every parameter from that component (slot
// 1 + d): floats and integers by the truncated normal's inverse CDF (integers on [lo2, hi2), then rounded to the grid and
// clipped), categories from the component's row; parameter d goes to x[d * stride]
__device__ __forceinline__ void mv_draw(const MvModels& md, uint64_t seed, uint32_t ask, int p, int m, double* __restrict__ x_out, size_t stride) {
  const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t r[4];
  philox4x32_10((uint32_t)m, 0u, (uint32_t)p, ask, k0, k1, r);
  const double u1 = tpe_u01(r[0], r[1]);
  const int nc = md.hdr[0].m;
  const double* w = md.w;
  int k = 0;
  double cum = w[0];
  while (k < nc && !(u1 < cum)) cum += w[++k];
  const int trial = k < nc ? md.idx[k] : -1;   // -1: the prior
  for (int d = 0; d < md.D; d++) {
    const MvParam P = md.prm[d];
    philox4x32_10((uint32_t)m, (uint32_t)(d + 1), (uint32_t)p, ask, k0, k1, r);
    const double u2 = tpe_u01_open(r[2], r[3]);
    double x;
    if (P.kind == KBO_MVTPE_CAT) {
      const double C = (double)P.levels, a = MV_PW / C;
      int c;
      if (trial < 0) {
        c = (int)(u2 * C);
      } else {   // row: a / (pw + 1) everywhere plus 1 / (pw + 1) at the observed category o
        const int o = (int)md.vals[(size_t)trial * md.D + d];
        const double v = u2 * (MV_PW + 1.0);
        if (v < a * o) c = (int)(v / a);
        else if (v < a * (o + 1) + 1.0) c = o;
        else c = max(o + 1, (int)((v - 1.0) / a));
      }
      x = (double)min(max(c, 0), P.levels - 1);
    } else {
      const double mu = trial < 0 ? P.pm : md.vals[(size_t)trial * md.D + d];
      const double sg = trial < 0 ? P.ps : md.sg[d];
      x = tpe_truncnorm_draw(P.lo2, P.hi2, mu, sg, u2);
      if (P.kind == KBO_MVTPE_INT) x = mv_grid(P, min(max((int)rint((x - P.lo) / P.q), 0), P.levels - 1));
    }
    x_out[d * stride] = x;
  }
}
// every candidate of every point: local candidate m is global candidate m0 + m (m0 = 0 but for a shard ask)
__global__ void mvtpe_draw_kernel(MvModels md, int M, int m0, uint64_t seed, uint32_t ask, double* __restrict__ X) {
  const int p = blockIdx.y, m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  mv_draw(md, seed, ask, p, m0 + m, X + (size_t)p * md.D * M + m, (size_t)M);
}
// a shard ask's winners, regenerated from their global indices (the draw's values are already those mvtpe_prep_kernel keeps);
// an index outside [0, M) is an error
__global__ void mvtpe_pick_kernel(MvModels md, int k, int M, uint64_t seed, uint32_t ask, const long long* __restrict__ idx,
                                  double* __restrict__ x_out, int* __restrict__ err) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= k) return;
  const long long m = idx[p];
  double* x = x_out + (size_t)p * md.D;
  if (!(m >= 0 && m < M)) {
    atomicExch(err, 1);
    for (int d = 0; d < md.D; d++) x[d] = NAN;
    return;
  }
  mv_draw(md, seed, ask, p, (int)m, x, 1);
}
// every candidate into the working buffer (integers rounded to the grid and clipped; floats outside [lo, hi] and invalid
// category indices are an error) with the prior component's log density in FP64 (without its weight, which is per group)
// Xs and Xw may be the same buffer (the engine's own draws): each element is read, then written, by one thread
__global__ void mvtpe_prep_kernel(MvModels md, int M, const double* Xs, double* Xw, double* __restrict__ prior,
                                  int* __restrict__ err) {
  const int p = blockIdx.y, m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  double lp = 0.0;
  for (int d = 0; d < md.D; d++) {
    const MvParam P = md.prm[d];
    const size_t o = ((size_t)p * md.D + d) * M + m;
    double x = Xs[o];
    if (P.kind == KBO_MVTPE_FLOAT) {
      if (!(x >= P.lo && x <= P.hi)) atomicMax(err, 3);
      const double z = (x - P.pm) / P.ps;
      lp += -0.5 * z * z - log(P.ps) - MV_LN_SQRT_2PI - P.lpm;
    } else if (P.kind == KBO_MVTPE_INT) {
      if (!isfinite(x)) {
        atomicMax(err, 3);
        x = P.lo;
      }
      x = mv_grid(P, (int)fmin(fmax(rint((x - P.lo) / P.q), 0.0), (double)(P.levels - 1)));
      lp += mv_log_gauss_mass((x - 0.5 * P.q - P.pm) / P.ps, (x + 0.5 * P.q - P.pm) / P.ps) - P.lpm;
    } else {
      if (!(x >= 0.0 && x < (double)P.levels && x == floor(x))) atomicMax(err, 3);
      lp -= log((double)P.levels);
    }
    Xw[o] = x;
  }
  prior[(size_t)p * M + m] = lp;
}

// ------------------------------------------------------------------------------------------------ ask: FP32 score
// Error of L = m + log2 S, one group's FP32 log2-density at one candidate, against the exact value.  DESIGN.md §7
// "multivariate-tpe" derives it; u = 2^-24, R bounds Σ_float z² + |Σ_int f| of every term within T of the maximum.
__device__ __forceinline__ float mv_lse_err(const MvHdr& hd, int Df, int nterms, float m, float S, float L, float p2, int ntiles, int nres) {
  const float u = 5.9604645e-8f;
  const float Cmax = tpe_funkey(hd.kCmax), Cabs = tpe_funkey(hd.kCabs);
  float dt = 1.02f * u * fabsf(p2);   // the prior term: FP64, rounded once to FP32
  if (hd.m > 0) {
    const float R = fmaxf(0.f, Cmax + hd.Bsum - m + MV_T2 + 1.f);
    const float zeta = 2.02f * u * (hd.XM * sqrtf((float)Df * R) + R) + 2.05f * u * u * ((float)Df * hd.XM * hd.XM + R);
    const float acc = u * (float)nterms * (Cabs + hd.Bsum + R);
    const float dto = 1.01f * (u * (Cabs + hd.Bsum + R) + zeta + acc) + 1e-13f * (Cabs + hd.Bsum + R);
    dt = fmaxf(dt, dto);
  }
  if (!(dt <= 0.5f)) return INFINITY;   // the near / far split above assumes every near exponent is off by less than 1
  const float eS = 1.01f * (u * (float)(7 + ntiles + nres + 2 * 4 + 2) + MV_EPS_EX2 * (float)(1 + nres + 4 + 1));
  const float far = 2.f * (float)(hd.m + 1) * 1.8189894e-12f;   // 2^-39 per term
  return dt + u * (MV_T2 + MV_RESCALE) * (float)(1 + nres + 5) + 1.4426950f * (eS + far) + 2.f * u * fabsf(log2f(S)) + u * fabsf(L);
}

// log l(x) - log g(x) in FP32 with its error bound for MV_BM candidates per block.  Per group, the observation components
// pass through shared memory in tiles of MV_BN; each thread keeps a 4 × 8 register tile of exponents (candidates ×
// components), initialised to c2 and accumulated over float slabs of MV_DS parameters as -(x' - μ')² with x' = (x - pm)·fs,
// fs = sqrt(½ log2 e) / σ (one FADD and one FFMA per pair and parameter), then over discrete slabs (table entries for
// integers, the match bonus for categories).  Each tile folds into a per-thread running (max, sum) with ex2.approx; the 16
// threads of a candidate row merge by shuffles, then the prior term (FP64, per candidate) joins as one more term.
// lb[p] = max over candidates of (score - bound), the lower bound on the maximum the decision prunes with.
__global__ void __launch_bounds__(256) mvtpe_score_kernel(MvModels md, int M, const double* __restrict__ X, const double* __restrict__ prior,
                                                          float2* __restrict__ sc, float* __restrict__ score_out, unsigned* __restrict__ lb) {
  __shared__ __align__(16) float xs[MV_DS][MV_BM];
  __shared__ __align__(16) float ms[MV_DS][MV_BN];
  __shared__ __align__(16) int xd[MV_DDS][MV_BM];
  __shared__ __align__(16) int mdv[MV_DDS][MV_BN];
  __shared__ float cs[MV_BN];
  __shared__ long long dk[MV_DDS];   // per staged discrete parameter: table offset, -1 categorical, -2 integer without a table
  __shared__ float db[MV_DDS];    // categorical: match bonus (log2)
  __shared__ double dr[MV_DDS];   // integer without a table: q / σ
  const int p = blockIdx.y, m0 = blockIdx.x * MV_BM;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int D = md.D, Df = md.Df, Dd = md.Dd;
  const int nfs = (Df + MV_DS - 1) / MV_DS, nds = (Dd + MV_DDS - 1) / MV_DDS;
  float Lb[4], Eb[4], La[4], Ea[4];   // below / above: log2-density and its bound
  for (int g = 0; g < 2; g++) {
    const MvHdr hd = md.hdr[g];
    const int ntiles = (hd.m + MV_BN - 1) / MV_BN;
    const double* fs = md.fs + (size_t)g * Df;
    auto stage_x = [&](int s) {
      const int dn = min(MV_DS, Df - s * MV_DS);
      for (int e = threadIdx.x; e < dn * MV_BM; e += 256) {
        const int dd = e / MV_BM, c = e % MV_BM, d = md.flt[s * MV_DS + dd], m = min(m0 + c, M - 1);
        xs[dd][c] = (float)((X[((size_t)p * D + d) * M + m] - md.prm[d].pm) * fs[s * MV_DS + dd]);
      }
    };
    float mref[4], S[4];
    int nres[4];
#pragma unroll
    for (int c = 0; c < 4; c++) { mref[c] = -INFINITY; S[c] = 0.f; nres[c] = 0; }
    if (nfs == 1 && ntiles) {
      __syncthreads();
      stage_x(0);
    }
    for (int t = 0; t < ntiles; t++) {
      const int k0 = t * MV_BN;
      __syncthreads();
      for (int i = threadIdx.x; i < MV_BN; i += 256) cs[i] = k0 + i < hd.m ? md.c2[(size_t)g * md.mcap + k0 + i] : -INFINITY;
      __syncthreads();
      float acc[4][8];
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const float c0 = cs[(j < 4 ? 0 : 64) + tx * 4 + (j & 3)];
#pragma unroll
        for (int c = 0; c < 4; c++) acc[c][j] = c0;
      }
      for (int s = 0; s < nfs; s++) {
        const int dn = min(MV_DS, Df - s * MV_DS);
        __syncthreads();
        if (nfs > 1) stage_x(s);
        for (int e = threadIdx.x; e < dn * MV_BN; e += 256) {
          const int dd = e / MV_BN, i = e % MV_BN;
          ms[dd][i] = k0 + i < hd.m ? md.mu32[((size_t)g * Df + s * MV_DS + dd) * md.mcap + k0 + i] : 0.f;
        }
        __syncthreads();
        for (int dd = 0; dd < dn; dd++) {
          const float4 xv = *reinterpret_cast<const float4*>(&xs[dd][ty * 4]);
          const float4 ma = *reinterpret_cast<const float4*>(&ms[dd][tx * 4]);
          const float4 mb = *reinterpret_cast<const float4*>(&ms[dd][64 + tx * 4]);
          const float xa[4] = {xv.x, xv.y, xv.z, xv.w};
          const float mu[8] = {ma.x, ma.y, ma.z, ma.w, mb.x, mb.y, mb.z, mb.w};
#pragma unroll
          for (int c = 0; c < 4; c++)
#pragma unroll
            for (int j = 0; j < 8; j++) {
              const float z = xa[c] - mu[j];
              acc[c][j] = fmaf(-z, z, acc[c][j]);
            }
        }
      }
      for (int s = 0; s < nds; s++) {
        const int dn = min(MV_DDS, Dd - s * MV_DDS);
        __syncthreads();
        if (threadIdx.x < dn) {
          const MvParam P = md.prm[md.dsc[s * MV_DDS + threadIdx.x]];
          dk[threadIdx.x] = P.kind == KBO_MVTPE_CAT ? -1 : (P.tab >= 0 ? P.tab : -2);
          db[threadIdx.x] = (float)(P.b * MV_LOG2E);
          dr[threadIdx.x] = P.kind == KBO_MVTPE_INT ? P.q / md.sg[(size_t)g * D + md.dsc[s * MV_DDS + threadIdx.x]] : 0.0;
        }
        for (int e = threadIdx.x; e < dn * MV_BM; e += 256) {
          const int dd = e / MV_BM, c = e % MV_BM, d = md.dsc[s * MV_DDS + dd], m = min(m0 + c, M - 1);
          const MvParam& P = md.prm[d];
          const double x = X[((size_t)p * D + d) * M + m];
          xd[dd][c] = P.kind == KBO_MVTPE_CAT ? (int)x : mv_level(P, x);
        }
        for (int e = threadIdx.x; e < dn * MV_BN; e += 256) {
          const int dd = e / MV_BN, i = e % MV_BN;
          mdv[dd][i] = k0 + i < hd.m ? md.dv[((size_t)g * Dd + s * MV_DDS + dd) * md.mcap + k0 + i] : 0;
        }
        __syncthreads();
        for (int dd = 0; dd < dn; dd++) {
          const long long kind = dk[dd];
          const int4 xv = *reinterpret_cast<const int4*>(&xd[dd][ty * 4]);
          const int4 ma = *reinterpret_cast<const int4*>(&mdv[dd][tx * 4]);
          const int4 mb = *reinterpret_cast<const int4*>(&mdv[dd][64 + tx * 4]);
          const int xa[4] = {xv.x, xv.y, xv.z, xv.w};
          const int mv[8] = {ma.x, ma.y, ma.z, ma.w, mb.x, mb.y, mb.z, mb.w};
          if (kind == -1) {
            const float b = db[dd];
#pragma unroll
            for (int c = 0; c < 4; c++)
#pragma unroll
              for (int j = 0; j < 8; j++) acc[c][j] += xa[c] == mv[j] ? b : 0.f;
          } else if (kind >= 0) {
            const float* tab = md.tab32 + (size_t)g * md.ltab + kind;
#pragma unroll
            for (int c = 0; c < 4; c++)
#pragma unroll
              for (int j = 0; j < 8; j++) acc[c][j] += __ldg(tab + abs(xa[c] - mv[j]));
          } else {   // more levels than MV_LCAP: each term in FP64, one evaluation per iteration, added where it belongs
            const double r = dr[dd];
#pragma unroll 1
            for (int q = 0; q < 32; q++) {
              const int c = q >> 3, j = q & 7;
              const double jj = (double)abs(xd[dd][ty * 4 + c] - mdv[dd][(j < 4 ? 0 : 64) + tx * 4 + (j & 3)]);
              const float v = (float)(mv_log_gauss_mass((jj - 0.5) * r, (jj + 0.5) * r) * MV_LOG2E);
#pragma unroll
              for (int cc = 0; cc < 4; cc++)
#pragma unroll
                for (int jc = 0; jc < 8; jc++)
                  if (q == cc * 8 + jc) acc[cc][jc] += v;
            }
          }
        }
      }
#pragma unroll
      for (int c = 0; c < 4; c++) {
        float tmax = acc[c][0];
#pragma unroll
        for (int j = 1; j < 8; j++) tmax = fmaxf(tmax, acc[c][j]);
        if (tmax > mref[c] + MV_RESCALE) {
          S[c] *= tpe_ex2(mref[c] - tmax);
          mref[c] = tmax;
          nres[c]++;
        }
        if (mref[c] > -INFINITY) {
          float loc = 0.f;
#pragma unroll
          for (int j = 0; j < 8; j++) loc += tpe_ex2(acc[c][j] - mref[c]);
          S[c] += loc;
        }
      }
    }
    // the 16 threads of a candidate row (one half-warp) merge their (max, sum); then the prior term
#pragma unroll
    for (int c = 0; c < 4; c++) {
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, mref[c], o), S2 = __shfl_xor_sync(0xffffffffu, S[c], o);
        nres[c] = max(nres[c], __shfl_xor_sync(0xffffffffu, nres[c], o));
        const float mn = fmaxf(mref[c], m2);
        const float f1 = mref[c] > -INFINITY ? tpe_ex2(mref[c] - mn) : 0.f, f2 = m2 > -INFINITY ? tpe_ex2(m2 - mn) : 0.f;
        S[c] = fmaf(S[c], f1, S2 * f2);
        mref[c] = mn;
      }
      const int m = min(m0 + ty * 4 + c, M - 1);
      const float p2 = (float)((prior[(size_t)p * M + m] + hd.lwp) * MV_LOG2E);
      const float mn = fmaxf(mref[c], p2);
      const float f1 = mref[c] > -INFINITY ? tpe_ex2(mref[c] - mn) : 0.f;
      S[c] = fmaf(S[c], f1, tpe_ex2(p2 - mn));
      const float L = mn + log2f(S[c]);
      const float E = mv_lse_err(hd, Df, Df + Dd, mn, S[c], L, p2, ntiles, nres[c]);
      if (g == 0) {
        Lb[c] = L;
        Eb[c] = E;
      } else {
        La[c] = L;
        Ea[c] = E;
      }
    }
  }
  const float u = 5.9604645e-8f;
  float best_lo = -INFINITY;
#pragma unroll
  for (int c = 0; c < 4; c++) {
    const int m = m0 + ty * 4 + c;
    const float s2 = Lb[c] - La[c];
    const float s = s2 * 0.69314718f;
    const float e = 1.05f * (0.69314718f * (Eb[c] + Ea[c] + u * fabsf(s2)) + 2.f * u * fabsf(s)) + 1e-9f;
    if (m < M && tx == 0) {
      sc[(size_t)p * M + m] = make_float2(s, e);
      if (score_out) {
        score_out[2 * ((size_t)p * M + m)] = s;
        score_out[2 * ((size_t)p * M + m) + 1] = e;
      }
    }
    if (m < M && tx == 0) best_lo = fmaxf(best_lo, s - e);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best_lo = fmaxf(best_lo, __shfl_xor_sync(0xffffffffu, best_lo, o));
  if ((threadIdx.x & 31) == 0 && best_lo > -INFINITY) atomicMax(lb + p, tpe_fkey(best_lo));
}

// ------------------------------------------------------------------------------------------------ ask: FP64 decision
// log of one group's density at candidate (p, mm) in FP64: one warp, lanes over the observation components (online
// log-sum-exp per lane, merged by shuffles), then the prior term
__device__ double mv_lse64(const MvModels& md, int g, const double* __restrict__ X, int M, int p, int mm, double lprior, int lane) {
  const int nc = md.hdr[g].m, D = md.D;
  double mx = -INFINITY, s = 0.0;
  for (int k = lane; k < nc; k += 32) {
    const int i = md.idx[(size_t)g * md.mcap + k];
    double t = md.c64[(size_t)g * md.mcap + k];
    for (int d = 0; d < D; d++) {
      const MvParam& P = md.prm[d];
      const double x = X[((size_t)p * D + d) * M + mm];
      if (P.kind == KBO_MVTPE_FLOAT) {
        const double z = (x - md.vals[(size_t)i * D + d]) / md.sg[(size_t)g * D + d];
        t -= 0.5 * z * z;
      } else if (P.kind == KBO_MVTPE_INT) {
        const int j = abs(mv_level(P, x) - md.dv[((size_t)g * md.Dd + P.slot) * md.mcap + k]);
        t += P.tab >= 0 ? md.tab64[(size_t)g * md.ltab + P.tab + j] : mv_int_term64(P, md.sg[(size_t)g * D + d], j);
      } else if ((int)x == md.dv[((size_t)g * md.Dd + P.slot) * md.mcap + k]) {
        t += P.b;
      }
    }
    if (t > mx) {
      s = s * exp(mx - t) + 1.0;
      mx = t;
    } else {
      s += exp(t - mx);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double m2 = __shfl_xor_sync(0xffffffffu, mx, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    const double mn = fmax(mx, m2);
    s = (mx > -INFINITY ? s * exp(mx - mn) : 0.0) + (m2 > -INFINITY ? s2 * exp(m2 - mn) : 0.0);
    mx = mn;
  }
  const double mn = fmax(mx, lprior);
  s = (mx > -INFINITY ? s * exp(mx - mn) : 0.0) + exp(lprior - mn);
  return mn + log(s);
}
// every candidate whose upper bound reaches the lower bound on the maximum is re-scored in FP64 by one warp; per block, the
// first index of the FP64 maximum among them
__global__ void __launch_bounds__(256) mvtpe_decide_kernel(MvModels md, int M, const double* __restrict__ X, const double* __restrict__ prior,
                                                           const float2* __restrict__ sc, const unsigned* __restrict__ lb, TpeBest* __restrict__ bb,
                                                           int nbb, int* __restrict__ surv) {
  const int p = blockIdx.y, m = blockIdx.x * 256 + threadIdx.x, lane = threadIdx.x & 31;
  const float LB = tpe_funkey(lb[p]);
  bool keep = false;
  if (m < M) {
    const float2 v = sc[(size_t)p * M + m];
    keep = !(v.x + v.y < LB);
  }
  unsigned mask = __ballot_sync(0xffffffffu, keep);
  if (lane == 0 && mask) atomicAdd(surv + p, __popc(mask));
  const double lw0 = md.hdr[0].lwp, lw1 = md.hdr[1].lwp;
  TpeBest best{0.0, -1};
  while (mask) {
    const int src = __ffs(mask) - 1;
    mask &= mask - 1;
    const int mm = m - lane + src;
    const double lp = prior[(size_t)p * M + mm];
    const double v = mv_lse64(md, 0, X, M, p, mm, lp + lw0, lane) - mv_lse64(md, 1, X, M, p, mm, lp + lw1, lane);
    if (tpe_better(v, mm, best)) { best.s = v; best.i = mm; }
  }
  best = tpe_block_best(best);
  if (threadIdx.x == 0) bb[(size_t)p * nbb + blockIdx.x] = best;
}
// per point: the winner over the per-block results, and its vector
__global__ void __launch_bounds__(256) mvtpe_final_kernel(int D, int M, const double* __restrict__ X, const TpeBest* __restrict__ bb, int nbb,
                                                          double* __restrict__ x_out, long long* __restrict__ idx_out) {
  const int p = blockIdx.x;
  TpeBest best{0.0, -1};
  for (int i = threadIdx.x; i < nbb; i += blockDim.x) {
    const TpeBest b = bb[(size_t)p * nbb + i];
    if (tpe_better(b.s, b.i, best)) best = b;
  }
  best = tpe_block_best(best);
  __shared__ long long win;
  if (threadIdx.x == 0) {
    win = best.i;
    if (idx_out) idx_out[p] = best.i;
  }
  __syncthreads();
  for (int d = threadIdx.x; d < D; d += blockDim.x) x_out[(size_t)p * D + d] = win >= 0 ? X[((size_t)p * D + d) * M + win] : NAN;
}

// ------------------------------------------------------------------------------------------------ host side
static double host_log_gauss_mass_central(double h) { return std::log(std::erf(h * 0.70710678118654752)); }   // [-h, h]

static MvModels mv_models(kbo_mvtpe* t) {
  MvModels md;
  md.prm = t->d_prm.p;
  md.flt = t->d_flt.p;
  md.dsc = t->d_dsc.p;
  md.idx = t->idx.p;
  md.dv = t->dv.p;
  md.vals = t->vals.p;
  md.w = t->w.p;
  md.c64 = t->c64.p;
  md.sg = t->sg.p;
  md.fs = t->fs.p;
  md.tab64 = t->tab64.p;
  md.c2 = t->c2.p;
  md.mu32 = t->mu32.p;
  md.tab32 = t->tab32.p;
  md.hdr = t->hdr.p;
  md.D = t->D;
  md.Df = t->Df;
  md.Dd = t->Dd;
  md.mcap = t->mcap;
  md.ltab = t->ltab;
  return md;
}

// Optuna's sigma for a group of m observations in a space of D parameters: 0.2·max(m, 1)^(-1/(D + 4))·(hi2 - lo2), clipped
// to [(hi2 - lo2) / min(100, m + 2), hi2 - lo2]
static double mv_sigma(const MvParam& P, int m, int D) {
  const double r = P.hi2 - P.lo2;
  const double s = 0.2 * std::pow((double)std::max(m, 1), -1.0 / (D + 4)) * r;
  return std::min(std::max(s, r / std::min(100.0, 1.0 + (double)(m + 1))), r);
}

static int mv_build(kbo_handle* h, kbo_mvtpe* t, cudaStream_t s) {
  const int n = t->n, D = t->D;
  t->nb = n ? std::min((int)std::ceil(0.1 * (double)n), TPE_LF) : 0;
  const int nb = t->nb, m[2] = {nb, n - nb};
  t->mcap = round_up(std::max(n, 1), MV_BN);
  const size_t mc = t->mcap;
  KBO_TRY(kbo_reserve(h, t->idx, mc * 2));
  KBO_TRY(kbo_reserve(h, t->w, (mc + 1) * 2));
  KBO_TRY(kbo_reserve(h, t->c64, mc * 2));
  KBO_TRY(kbo_reserve(h, t->c2, mc * 2));
  KBO_TRY(kbo_reserve(h, t->mu32, mc * std::max(t->Df, 1) * 2));
  KBO_TRY(kbo_reserve(h, t->dv, mc * std::max(t->Dd, 1) * 2));
  KBO_TRY(kbo_reserve(h, t->sg, (size_t)D * 2));
  KBO_TRY(kbo_reserve(h, t->fs, (size_t)std::max(t->Df, 1) * 2));
  KBO_TRY(kbo_reserve(h, t->tab64, (size_t)std::max(t->ltab, 1ll) * 2));
  KBO_TRY(kbo_reserve(h, t->tab32, (size_t)std::max(t->ltab, 1ll) * 2));
  KBO_TRY(kbo_reserve(h, t->hdr, 2));
  // per group: sigma, the float scales, and the error-bound constants the host knows
  std::vector<double> sg(2 * D, NAN), fs(2 * std::max(t->Df, 1), 0.0);
  MvHdr hd[2];
  for (int g = 0; g < 2; g++) {
    memset(&hd[g], 0, sizeof hd[g]);
    hd[g].m = m[g];
    double xm = 0.0, bs = 0.0;
    for (int d = 0; d < D; d++) {
      const MvParam& P = t->prm[d];
      if (P.kind == KBO_MVTPE_CAT) {
        bs += P.b * MV_LOG2E;
        continue;
      }
      sg[g * D + d] = mv_sigma(P, m[g], D);
      if (P.kind == KBO_MVTPE_FLOAT) {
        const double f = std::sqrt(MV_H2) / sg[g * D + d];
        fs[g * t->Df + P.slot] = f;
        xm = std::max(xm, (P.hi - P.lo) * f);
      }
    }
    hd[g].Bsum = (float)(bs * 1.0001);
    hd[g].XM = (float)(xm * 1.0001);
  }
  KBO_CUDA(h, kbo_copy(t->sg.p, sg.data(), sg.size(), cudaMemcpyHostToDevice, s));
  KBO_CUDA(h, kbo_copy(t->fs.p, fs.data(), fs.size(), cudaMemcpyHostToDevice, s));
  KBO_CUDA(h, kbo_copy(t->hdr.p, hd, 2, cudaMemcpyHostToDevice, s));
  if (n > 0) {
    KBO_TRY(kbo_reserve(h, t->lkey, (size_t)n));
    KBO_TRY(kbo_reserve(h, t->lkey2, (size_t)n));
    KBO_TRY(kbo_reserve(h, t->lidx, (size_t)n));
    KBO_TRY(kbo_reserve(h, t->lidx2, (size_t)n));
    KBO_TRY(kbo_reserve(h, t->below, TPE_LF));
    KBO_TRY(kbo_reserve(h, t->grp, (size_t)n));
    KBO_TRY(kbo_reserve(h, t->pos, (size_t)n));
    size_t b1 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b1, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int*)nullptr, (int*)nullptr, n, 0, 64, s);
    KBO_TRY(kbo_reserve(h, t->tmp, std::max<size_t>(b1, 16)));
    // the stable loss order (NumPy's argsort(kind='stable'); NaN losses are refused by tell)
    tpe_loss_keys_kernel<<<(n + 255) / 256, 256, 0, s>>>(t->loss.p, n, t->lkey.p, t->lidx.p);
    KBO_LAUNCH_CHECK(h);
    size_t bytes = t->tmp.cap;
    KBO_CUDA(h, cub::DeviceRadixSort::SortPairs(t->tmp.p, bytes, t->lkey.p, t->lkey2.p, t->lidx.p,
                                               t->lidx2.p, n, 0, 64, s));
    tpe_split_kernel<<<1, 32, 0, s>>>(t->lidx2.p, nb, t->below.p);
    KBO_LAUNCH_CHECK(h);
    tpe_group_kernel<<<(n + 255) / 256, 256, 0, s>>>(t->below.p, nb, n, t->grp.p, t->pos.p);
    KBO_LAUNCH_CHECK(h);
    mvtpe_members_kernel<<<(n + 255) / 256, 256, 0, s>>>(t->grp.p, t->pos.p, n, t->mcap, t->idx.p);
    KBO_LAUNCH_CHECK(h);
  }
  mvtpe_weights_kernel<<<2, 256, 0, s>>>(t->mcap, t->hdr.p, t->w.p);
  KBO_LAUNCH_CHECK(h);
  const MvModels md = mv_models(t);
  if (n > 0) {
    mvtpe_model_kernel<<<dim3((n + 255) / 256, 2), 256, 0, s>>>(md, t->c64.p, t->c2.p, t->mu32.p, t->dv.p,
                                                               t->hdr.p);
    KBO_LAUNCH_CHECK(h);
  }
  if (!t->tabd.empty()) {
    mvtpe_table_kernel<<<dim3((t->lmax + 255) / 256, (unsigned)t->tabd.size(), 2), 256, 0, s>>>(md, t->d_tabd.p, t->tab64.p,
                                                                                               t->tab32.p);
    KBO_LAUNCH_CHECK(h);
  }
  KBO_CUDA(h, cudaStreamSynchronize(s));   // the host vectors above are read by the copies
  t->built_n = n;
  return KBO_OK;
}

extern "C" {

int kbo_mvtpe_create(kbo_handle* h, kbo_mvtpe** out, int32_t D, const int32_t* kinds, const double* lo, const double* hi, const double* q,
                     const int32_t* levels, uint64_t seed) {
  if (!h || !out) return KBO_ERR_INVALID;
  *out = nullptr;
  if (D < 1 || D > MV_MAXD) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_create: 1 <= D <= %d supported (got %d)", MV_MAXD, D);
  if (!kinds) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_create: null kinds");
  KBO_CUDA(h, cudaSetDevice(h->device));
  std::unique_ptr<kbo_mvtpe> t(new (std::nothrow) kbo_mvtpe());
  if (!t) return KBO_ERR_NOMEM;
  t->D = D;
  t->seed = seed;
  t->prm.resize(D);
  const double lpm = host_log_gauss_mass_central(0.5);   // the prior's mass over its own range: [pm - ps/2, pm + ps/2]
  for (int d = 0; d < D; d++) {
    MvParam& P = t->prm[d];
    memset(&P, 0, sizeof P);
    P.kind = kinds[d];
    P.tab = -1;
    if (P.kind == KBO_MVTPE_CAT) {
      if (!levels || levels[d] < 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_create: parameter %d: a categorical needs >= 1 categories", d);
      P.levels = levels[d];
      P.slot = t->Dd++;
      t->dsc.push_back(d);
      const double a = MV_PW / P.levels;
      P.lcat = std::log(a) - std::log(MV_PW + 1.0);
      P.b = std::log(a + 1.0) - std::log(a);
      continue;
    }
    if (P.kind != KBO_MVTPE_FLOAT && P.kind != KBO_MVTPE_INT) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_create: parameter %d: unknown kind %d", d, kinds[d]);
    if (!lo || !hi || !std::isfinite(lo[d]) || !std::isfinite(hi[d]) || !(lo[d] <= hi[d]) || (P.kind == KBO_MVTPE_FLOAT && !(lo[d] < hi[d])))
      KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_create: parameter %d: need finite lo < hi (lo <= hi for an integer)", d);
    P.lo = lo[d];
    P.hi = hi[d];
    P.lo2 = P.lo;
    P.hi2 = P.hi;
    if (P.kind == KBO_MVTPE_INT) {
      if (!q || !(q[d] > 0.0) || !std::isfinite(q[d])) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_create: parameter %d: step must be > 0", d);
      P.q = q[d];
      const double L = std::floor((P.hi - P.lo) / P.q) + 1.0;
      if (!(L >= 1.0 && L < 2147483647.0)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_create: parameter %d: too many levels", d);
      P.levels = (int)L;
      P.hi = P.lo + (double)(P.levels - 1) * P.q;
      P.lo2 = P.lo - 0.5 * P.q;
      P.hi2 = P.hi + 0.5 * P.q;
      P.slot = t->Dd++;
      t->dsc.push_back(d);
      if (P.levels <= MV_LCAP) {
        P.tab = t->ltab;
        t->ltab += P.levels;
        t->lmax = std::max(t->lmax, P.levels);
        t->tabd.push_back(d);
      }
    } else {
      P.slot = t->Df++;
      t->flt.push_back(d);
    }
    P.pm = 0.5 * (P.lo2 + P.hi2);
    P.ps = P.hi2 - P.lo2;
    P.lpm = lpm;
  }
  KBO_TRY(kbo_upload(h, t->d_prm, t->prm.data(), D));
  KBO_TRY(kbo_upload(h, t->d_flt, t->flt.data(), t->flt.size()));
  KBO_TRY(kbo_upload(h, t->d_dsc, t->dsc.data(), t->dsc.size()));
  KBO_TRY(kbo_upload(h, t->d_tabd, t->tabd.data(), t->tabd.size()));
  KBO_TRY(kbo_reserve(h, t->err, 1));
  KBO_TRY(t->ev.create());
  *out = t.release();
  return KBO_OK;
}

void kbo_mvtpe_destroy(kbo_mvtpe* t) {
  if (t) delete t;
}

int kbo_mvtpe_tell(kbo_handle* h, kbo_mvtpe* t, const double* X, const double* loss, int32_t n_new, int on_host, void* stream) {
  if (!h || !t) return KBO_ERR_INVALID;
  if (n_new < 0) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_tell: n_new must be >= 0 (got %d)", n_new);
  if (n_new == 0) return KBO_OK;
  if (!X || !loss) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_tell: null argument");
  if ((int64_t)t->n + n_new > (1 << 24)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_tell: at most 2^24 trials supported");
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  KBO_TRY(tpe_history_append(h, t, X, loss, n_new, on_host, s));
  const double* Xn = t->vals.p + (size_t)t->D * t->n;   // the new rows: checked before n counts them
  const double* Ln = t->loss.p + t->n;
  KBO_CUDA(h, cudaMemsetAsync(t->err.p, 0, sizeof *t->err.p, s));
  mvtpe_check_kernel<<<(n_new + 255) / 256, 256, 0, s>>>(t->d_prm.p, t->D, Xn, Ln, n_new, t->err.p);
  KBO_LAUNCH_CHECK(h);
  int err = 0;
  KBO_CUDA(h, kbo_copy(&err, t->err.p, 1, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (err == 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_tell: a trial has a NaN loss (nothing was told)");
  if (err) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_tell: a value is outside its parameter's domain: floats in [lo, hi], integers on their grid, category indices in range (nothing was told)");
  t->n += n_new;
  return KBO_OK;
}

// One ask over local candidates [0, M), which are global candidates [m0, m0 + M) of n_candidates = Mall.  With val_dev null
// it is kbo_mvtpe_ask (m0 = 0, M = Mall): the winners' vectors go to x_dev.  With val_dev it is a shard ask: each point
// writes its FP64 winner and global index to val_dev / idx_dev, and M = 0 (an empty shard) is legal.
static int mv_ask_run(kbo_handle* h, kbo_mvtpe* t, int k, int M, int m0, int Mall, const double* cand_dev, double* x_dev, int64_t* idx_dev,
                      double* cand_out_dev, float* score_out_dev, double* val_dev, cudaStream_t s) {
  KBO_CUDA(h, cudaSetDevice(h->device));
  cudaEventRecord(t->ev[0], s);
  if (t->built_n != t->n) KBO_TRY(mv_build(h, t, s));
  const uint32_t ask = t->asks++;
  const int D = t->D;
  if (val_dev) {
    t->pick_ask = ask;
    t->pick_k = k;
    t->pick_M = Mall;
    t->pick_n = t->n;
    if (M == 0) {
      tpe_shard_best_kernel<<<k, 256, 0, s>>>(nullptr, 0, m0, Mall, val_dev, (long long*)idx_dev);
      KBO_LAUNCH_CHECK(h);
      t->last_surv.assign(k, 0);
      std::fill(t->last_ms, t->last_ms + 4, 0.f);
      KBO_CUDA(h, cudaStreamSynchronize(s));
      return KBO_OK;
    }
  }
  const size_t KM = (size_t)k * M;
  const int nbb = (M + 255) / 256;
  KBO_TRY(kbo_reserve(h, t->surv, (size_t)k));
  KBO_TRY(kbo_reserve(h, t->bb, (size_t)k * nbb));
  KBO_TRY(kbo_reserve(h, t->prior, KM));
  KBO_TRY(kbo_reserve(h, t->sc, KM));
  KBO_TRY(kbo_reserve(h, t->lb, (size_t)k));
  KBO_CUDA(h, cudaMemsetAsync(t->surv.p, 0, sizeof *t->surv.p * (size_t)k, s));
  KBO_CUDA(h, cudaMemsetAsync(t->lb.p, 0, sizeof *t->lb.p * (size_t)k, s));
  KBO_CUDA(h, cudaMemsetAsync(t->err.p, 0, sizeof *t->err.p, s));
  const MvModels md = mv_models(t);
  double* Xw = cand_out_dev;   // the working candidates: the caller's output buffer if it wants them, else the handle's
  if (!Xw) {
    KBO_TRY(kbo_reserve(h, t->draws, KM * D));
    Xw = t->draws.p;
  }
  const dim3 gm((M + 255) / 256, k);
  if (!cand_dev) {
    mvtpe_draw_kernel<<<gm, 256, 0, s>>>(md, M, m0, t->seed, ask, Xw);
    KBO_LAUNCH_CHECK(h);
  }
  mvtpe_prep_kernel<<<gm, 256, 0, s>>>(md, M, cand_dev ? cand_dev : Xw, Xw, t->prior.p, t->err.p);
  KBO_LAUNCH_CHECK(h);
  cudaEventRecord(t->ev[1], s);
  mvtpe_score_kernel<<<dim3((M + MV_BM - 1) / MV_BM, k), 256, 0, s>>>(md, M, Xw, t->prior.p, t->sc.p, score_out_dev,
                                                                       t->lb.p);
  KBO_LAUNCH_CHECK(h);
  cudaEventRecord(t->ev[2], s);
  mvtpe_decide_kernel<<<dim3(nbb, k), 256, 0, s>>>(md, M, Xw, t->prior.p, t->sc.p, t->lb.p,
                                                   t->bb.p, nbb, t->surv.p);
  KBO_LAUNCH_CHECK(h);
  cudaEventRecord(t->ev[3], s);
  if (val_dev) tpe_shard_best_kernel<<<k, 256, 0, s>>>(t->bb.p, nbb, m0, Mall, val_dev, (long long*)idx_dev);
  else mvtpe_final_kernel<<<k, 256, 0, s>>>(D, M, Xw, t->bb.p, nbb, x_dev, (long long*)idx_dev);
  KBO_LAUNCH_CHECK(h);
  cudaEventRecord(t->ev[4], s);
  t->last_surv.assign(k, 0);
  int err = 0;
  KBO_CUDA(h, kbo_copy(t->last_surv.data(), t->surv.p, (size_t)k, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, kbo_copy(&err, t->err.p, 1, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  for (int i = 0; i < 4; i++) cudaEventElapsedTime(&t->last_ms[i], t->ev[i], t->ev[i + 1]);
  if (err) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_ask: a supplied candidate is outside its parameter's domain (a float outside [lo, hi] or an invalid category index)");
  return KBO_OK;
}

int kbo_mvtpe_ask(kbo_handle* h, kbo_mvtpe* t, int32_t k, int32_t M, const double* cand_dev, double* x_dev, int64_t* idx_dev, double* cand_out_dev,
                  float* score_out_dev, void* stream) {
  if (!h || !t) return KBO_ERR_INVALID;
  if (!x_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_ask: null output");
  if (k < 1 || k > 65535) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_ask: 1 <= k <= 65535 supported (got %d)", k);
  if (M < 1 || M > MV_MAXM) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_ask: 1 <= n_candidates <= 2^24 supported (got %d)", M);
  return mv_ask_run(h, t, k, M, 0, M, cand_dev, x_dev, idx_dev, cand_out_dev, score_out_dev, nullptr, (cudaStream_t)stream);
}

int kbo_mvtpe_ask_shard(kbo_handle* h, kbo_mvtpe* t, int32_t k, int32_t M, int32_t lo, int32_t hi, const double* cand_dev, double* val_dev,
                        int64_t* idx_dev, void* stream) {
  if (!h || !t) return KBO_ERR_INVALID;
  if (cand_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_ask_shard: caller-supplied candidates are not accepted (the shards draw their own)");
  if (!val_dev || !idx_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_ask_shard: null output");
  if (k < 1 || k > 65535) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_ask_shard: 1 <= k <= 65535 supported (got %d)", k);
  if (M < 1 || M > MV_MAXM) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_ask_shard: 1 <= n_candidates <= 2^24 supported (got %d)", M);
  if (!(0 <= lo && lo <= hi && hi <= M)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_ask_shard: need 0 <= lo <= hi <= n_candidates (got [%d, %d) of %d)", lo, hi, M);
  return mv_ask_run(h, t, k, hi - lo, lo, M, nullptr, nullptr, idx_dev, nullptr, nullptr, val_dev, (cudaStream_t)stream);
}

int kbo_mvtpe_pick(kbo_handle* h, kbo_mvtpe* t, int32_t k, const int64_t* idx_dev, double* x_dev, void* stream) {
  if (!h || !t) return KBO_ERR_INVALID;
  if (!idx_dev || !x_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_pick: null argument");
  if (t->pick_k == 0 || t->pick_n != t->n) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_pick: no shard ask since the last tell");
  if (k != t->pick_k) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_pick: k must be the last shard ask's (%d, got %d)", t->pick_k, k);
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  KBO_CUDA(h, cudaMemsetAsync(t->err.p, 0, sizeof *t->err.p, s));
  mvtpe_pick_kernel<<<(k + 255) / 256, 256, 0, s>>>(mv_models(t), k, t->pick_M, t->seed, t->pick_ask, (const long long*)idx_dev, x_dev,
                                                    t->err.p);
  KBO_LAUNCH_CHECK(h);
  int err = 0;
  KBO_CUDA(h, kbo_copy(&err, t->err.p, 1, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (err) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_pick: a winning index is outside [0, n_candidates)");
  return KBO_OK;
}

int kbo_mvtpe_state(kbo_handle* h, kbo_mvtpe* t, int32_t group, double* w, double* sigma, double* mu, double* cat_rows, int32_t cap,
                    int32_t* n_obs, int32_t* n_below, void* stream) {
  if (!h || !t) return KBO_ERR_INVALID;
  if (group < 0 || group > 1 || cap < 0) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_mvtpe_state: bad argument");
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  if (t->built_n != t->n) KBO_TRY(mv_build(h, t, s));
  const int D = t->D, m = group ? t->n - t->nb : t->nb, c = std::min(cap, m);
  KBO_CUDA(h, kbo_d2h(w, t->w.p + (size_t)group * (t->mcap + 1), (size_t)std::min(cap, m + 1), s));
  KBO_CUDA(h, kbo_d2h(sigma, t->sg.p + (size_t)group * D, (size_t)D, s));
  if (mu && c > 0) {
    std::vector<int> idx(c);
    KBO_CUDA(h, kbo_copy(idx.data(), t->idx.p + (size_t)group * t->mcap, (size_t)c, cudaMemcpyDeviceToHost, s));
    KBO_CUDA(h, cudaStreamSynchronize(s));
    for (int k = 0; k < c; k++)
      KBO_CUDA(h, kbo_copy(mu + (size_t)k * D, t->vals.p + (size_t)idx[k] * D, (size_t)D, cudaMemcpyDeviceToHost, s));
  }
  if (cat_rows)
    for (int d = 0; d < D; d++) {
      const MvParam& P = t->prm[d];
      const bool cat = P.kind == KBO_MVTPE_CAT;
      cat_rows[2 * d] = cat ? std::exp(P.lcat + P.b) : NAN;
      cat_rows[2 * d + 1] = cat ? std::exp(P.lcat) : NAN;
    }
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (n_obs) *n_obs = m;
  if (n_below) *n_below = t->nb;
  return KBO_OK;
}

int kbo_mvtpe_last_survivors(kbo_handle* h, kbo_mvtpe* t, int32_t* out, int32_t n) {
  if (!h || !t) return KBO_ERR_INVALID;
  for (int i = 0; out && i < n && i < (int)t->last_surv.size(); i++) out[i] = t->last_surv[i];
  return (int)t->last_surv.size();
}

int kbo_mvtpe_last_timings(kbo_handle* h, kbo_mvtpe* t, float* ms, int32_t n) {
  if (!h || !t) return KBO_ERR_INVALID;
  for (int i = 0; ms && i < n && i < 4; i++) ms[i] = t->last_ms[i];
  return 4;
}

}  // extern "C"
