// Tree-structured Parzen estimator on the device — Katib's `tpe` algorithm (hyperopt's tpe.suggest on a flat space; the
// FP64 restatement that is the contract is oracle/tpe_oracle.py, DESIGN.md §7 "tpe").
//   history : values in parameter units (category index for choices) and FP64 losses, appended as trials are told
//   models  : one stable radix sort of the losses (NumPy order, NaN last) splits the history into the n_below best
//             ("below") and the rest ("above"); a stable segmented sort orders each numeric parameter's values in both
//             groups; tpe_model_kernel turns them into adaptive Parzen mixtures (w, mu, sigma) with the prior inserted,
//             plus per-component constants; tpe_cat_kernel builds the categorical tables
//   ask     : candidates come from Philox4x32-10 keyed by (seed, ask, point, parameter, candidate), drawn from the below
//             model truncated to [lo, hi) by inverse CDF (tpe_draw_kernel), or are supplied by the caller.  Continuous parameters are scored
//             in FP32 (tpe_score_kernel: online log-sum-exp over components staged in shared memory, ex2.approx) with a
//             per-candidate error bound; whatever can still be the maximum is re-scored in FP64 (tpe_decide_kernel) and the
//             first index of the FP64 maximum wins.  Quantized and categorical parameters score each distinct value present
//             once, in FP64 (tpe_level_kernel, tpe_disc_score_kernel).
#include <algorithm>
#include <cmath>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include "kbo_internal.cuh"
#include "kbo_rng.cuh"
#include "kbo_tpe_common.cuh"

#define TPE_CB 32          // slots of a below mixture (<= 25 observations + the prior)
#define TPE_CHUNK 1024     // components staged in shared memory at a time by the score kernel
#define TPE_CPT 4          // candidates per thread in the score kernel (each staged component is read once for all four)
#define TPE_THREADS 256
#define TPE_LCAP 65536     // quantized / categorical parameters with at most this many levels are deduplicated by a level table
#define TPE_MAXM (1 << 24)
#define TPE_T2 40.0f       // log2 distance below the running maximum past which a term counts as "far" in the error bound
#define TPE_H2 0.72134752f // 0.5 * log2(e)
#define TPE_EPS_EX2 9.5367432e-7f  // 2^-20: relative error allowed for ex2.approx.ftz.f32 (the PTX ISA documents about 2 ulp)

struct TpeParam {
  int kind;     // kbo_tpe_kind
  int slot;     // numeric parameters: mixture slot; choices: table slot
  int levels;   // quantized: multiples of q reachable from [lo, hi); choice: categories
  int pad;
  double lo, hi, q, base;  // base = rint(lo / q)
  double pm, ps;           // prior mu = (lo + hi) / 2, prior sigma = hi - lo
};
struct TpeHdr {  // one per (numeric parameter, group)
  int ncomp, pad;
  double p_acc;
  float A, B, C2max, C2abs;  // error-bound constants of the FP32 arithmetic: max r', max r'|mu'|, max c2, max |c2|
};
struct TpeModels {
  const TpeParam* prm;
  const double *w, *mu, *sg, *lc, *cdf;
  const float4* f4;  // (mu', r', c2, 0): mu' = (mu - pm) / ps, r' = ps / sigma, c2 = log2 of the component's coefficient
  const TpeHdr* hdr;
  const double *cat_sc, *cat_cum;
  int ms, lcat;
};

struct kbo_tpe {
  int D = 0, Dc = 0, Dd = 0, Dnum = 0, Dcat = 0, lcat = 1, lt = 1;
  std::vector<TpeParam> prm;
  std::vector<int> cont, disc, num, cat;
  double gamma = 0.25, pw = 1.0;
  uint64_t seed = 0;
  uint32_t asks = 0;
  int n = 0, cap = 0, built_n = -1, nb = 0, ms = 0;
  uint32_t pick_ask = 0;            // the last shard ask: its ask number, k, n_candidates and history size, for kbo_tpe_pick
  int pick_k = 0, pick_M = 0, pick_n = -1;
  DevBuf<TpeParam> d_prm;
  DevBuf<int> d_cont, d_disc, d_num, d_cat;
  DevBuf<double> vals, loss;
  DevBuf<uint64_t> lkey, lkey2, skey, skey2;
  DevBuf<int> lidx, lidx2, below, grp, pos, sval, sval2, segb, sege;
  DevBuf<unsigned char> tmp;
  DevBuf<double> w, mu, sg, lc, cdf, cat_p, cat_sc, cat_cum;
  DevBuf<float4> f4;
  DevBuf<TpeHdr> hdr;
  DevBuf<double> draws;
  DevBuf<float2> sc;
  DevBuf<unsigned> lb, first;
  DevBuf<int> surv, err;
  DevBuf<TpeBest> bb;
  std::vector<int> last_surv;
  EventSet<6> ev;
  float last_ms[5] = {};
};

// ------------------------------------------------------------------------------------------------ device helpers
// hyperopt's normal_cdf: 0.5 * (1 + erf((x - mu) / max(sqrt(2) * sigma, 1e-12)))
__device__ __forceinline__ double tpe_ncdf(double x, double mu, double sigma) {
  return 0.5 * (1.0 + erf((x - mu) / fmax(1.4142135623730951 * sigma, 1e-12)));
}
__device__ __forceinline__ size_t tpe_moff(int slot, int g, int ms) { return (size_t)slot * ms + (g ? TPE_CB : 0); }

// one draw from the below model: choices from p_below; numeric parameters from the mixture truncated to [lo, hi) —
// component k with probability ∝ w_k·mass_k (what hyperopt's rejection loop amounts to), then that component's truncated
// normal by inverse CDF on the side of the mean where the tail probabilities keep their relative precision
__device__ double tpe_draw(const TpeModels& md, const TpeParam& P, uint64_t seed, uint32_t ask, int point, int d, int m) {
  uint32_t r[4];
  philox4x32_10((uint32_t)m, (uint32_t)d, (uint32_t)point, ask, (uint32_t)seed, (uint32_t)(seed >> 32), r);
  const double u1 = tpe_u01(r[0], r[1]), u2 = tpe_u01_open(r[2], r[3]);
  if (P.kind == KBO_TPE_CHOICE) {
    const double* cum = md.cat_cum + (size_t)P.slot * md.lcat;
    int c = 0;
    while (c < P.levels - 1 && !(u1 < cum[c])) c++;
    return (double)c;
  }
  const size_t o = tpe_moff(P.slot, 0, md.ms);
  const int nc = md.hdr[2 * P.slot].ncomp;
  int k = 0;
  while (k < nc - 1 && !(u1 < md.cdf[o + k])) k++;
  return tpe_truncnorm_draw(P.lo, P.hi, md.mu[o + k], md.sg[o + k], u2);
}
// every candidate of every (point, parameter), before quantization: local candidate m is global candidate m0 + m (m0 = 0
// but for a shard ask)
__global__ void tpe_draw_kernel(TpeModels md, int D, int M, int m0, uint64_t seed, uint32_t ask, double* __restrict__ X) {
  const int pd = blockIdx.y, p = pd / D, d = pd % D;
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m < M) X[(size_t)pd * M + m] = tpe_draw(md, md.prm[d], seed, ask, p, d, m0 + m);
}
// a shard ask's winners, regenerated from their global indices and taken to their values as tpe_final_kernel does;
// an index outside [0, M) is an error
__global__ void tpe_pick_kernel(TpeModels md, int KD, int D, int M, uint64_t seed, uint32_t ask, const long long* __restrict__ idx,
                                double* __restrict__ x_out, int* __restrict__ err) {
  const int pd = blockIdx.x * blockDim.x + threadIdx.x;
  if (pd >= KD) return;
  const int p = pd / D, d = pd % D;
  const long long m = idx[pd];
  if (!(m >= 0 && m < M)) {
    atomicExch(err, 1);
    x_out[pd] = NAN;
    return;
  }
  const TpeParam P = md.prm[d];
  double x = tpe_draw(md, P, seed, ask, p, d, (int)m);
  if (P.kind == KBO_TPE_QUNIFORM) x = rint(x / P.q) * P.q;
  x_out[pd] = x;
}
// level index of a candidate of a quantized (rint(x/q) - rint(lo/q)) or categorical (the index itself) parameter; -1 if invalid
__device__ __forceinline__ long long tpe_level(const TpeParam& P, double x) {
  double j;
  if (P.kind == KBO_TPE_CHOICE) {
    if (!(x == floor(x))) return -1;
    j = x;
  } else {
    j = rint(x / P.q) - P.base;
  }
  if (!(j >= 0.0 && j < (double)P.levels)) return -1;
  return (long long)j;
}

// ---- FP64 scores (the decision) -----------------------------------------------------------------------------------------
// GMM1_lpdf, continuous: logsumexp_k(lc_k - ½((x-mu_k)/max(sigma_k,1e-12))²), lc_k = log(w_k / sqrt(2π sigma_k²) / p_accept);
// one warp, lanes over components
__device__ double tpe_lse64(const TpeModels& md, size_t o, int n, double x, int lane) {
  double m = -INFINITY;
  for (int k = lane; k < n; k += 32) {
    const double z = (x - md.mu[o + k]) / fmax(md.sg[o + k], 1e-12);
    m = fmax(m, fma(-0.5, z * z, md.lc[o + k]));
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, off));
  double s = 0.0;
  for (int k = lane; k < n; k += 32) {
    const double z = (x - md.mu[o + k]) / fmax(md.sg[o + k], 1e-12);
    s += exp(fma(-0.5, z * z, md.lc[o + k]) - m);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  return log(s) + m;
}
// GMM1_lpdf, quantized: log Σ_k w_k (Φ_k(min(v+q/2, hi)) - Φ_k(max(v-q/2, lo))) - log p_accept
__device__ double tpe_qlpdf64(const TpeModels& md, size_t o, int n, double p_acc, const TpeParam& P, double v, int lane) {
  const double ub = fmin(v + P.q / 2.0, P.hi), lb = fmax(v - P.q / 2.0, P.lo);
  double s = 0.0;
  for (int k = lane; k < n; k += 32) {
    const double w = md.w[o + k], mu = md.mu[o + k], sg = md.sg[o + k];
    double inc = w * tpe_ncdf(ub, mu, sg);
    inc -= w * tpe_ncdf(lb, mu, sg);
    s += inc;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  return log(s) - log(p_acc);
}

// ---- FP32 bound -----------------------------------------------------------------------------------------------------------
// Error of L = m + log2(S), the FP32 log2-sum-exp of one mixture at one candidate, against the exact value (log2 units).
// DESIGN.md §7 "tpe" derives it; in short, with u = 2^-24 and z_k = (x' - mu'_k) r'_k:
//  * every |z_k| <= Zall = A|x'| + B; a term within T2 of the maximum has z_k² <= (C2max - m + T2 + 1) / h2
//  * such a term's computed exponent t_k = c2_k - h2 z_k² is off by at most dt (inputs, products, the fma, the shift by m);
//    log-sum-exp is 1-Lipschitz in the ∞-norm, so the near terms move L by at most dt
//  * far terms (more than T2 below the maximum) add at most 2·n·2^-T2 to S relative to its value
//  * S itself: at most TPE_CHUNK + 3·chunks + 4 roundings on any path into the sum, and one ex2.approx per term and per merge
__device__ __forceinline__ float tpe_lse_err(float m, float S, float L, const TpeHdr& hd, float ax, int nchunks) {
  const float u = 5.9604645e-8f;
  const float Zall = fmaf(hd.A, ax, hd.B) * 1.001f;
  const float Z2 = fminf(Zall * Zall, fmaxf(0.f, hd.C2max - m + TPE_T2 + 1.f) * (1.f / TPE_H2));
  const float Z = sqrtf(Z2);
  const float zeta = u * (3.01f * Z + 1.01f * Zall);
  const float dt = 1.01f * (2.f * u * hd.C2abs + TPE_H2 * (2.f * Z * zeta + zeta * zeta + 3.f * u * Z2) + u * TPE_T2);
  const float eS = (float)(TPE_CHUNK + 3 * nchunks + 4) * u + (float)(1 + nchunks) * TPE_EPS_EX2 + 2.f * (float)hd.ncomp * 9.094947e-13f;  // 2^-40
  return dt + 1.01f * eS * 1.4426950f + 2.f * u * fabsf(log2f(S)) + u * fabsf(L);
}

// ------------------------------------------------------------------------------------------------ model build
// segment (numeric parameter j, group g) holds that group's values of parameter j at [j·n + (g ? nb : 0), ...)
__global__ void tpe_seg_fill_kernel(const double* __restrict__ vals, int n, int nb, int D, const int* __restrict__ num, const int* __restrict__ grp,
                                    const int* __restrict__ pos, uint64_t* __restrict__ key, int* __restrict__ val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (i >= n) return;
  const int g = grp[i], ps = pos[i];
  const size_t off = (size_t)j * n + (g ? nb : 0) + ps;
  key[off] = tpe_ordered(vals[(size_t)i * D + num[j]]);
  val[off] = ps;
}

// adaptive_parzen_normal for (numeric parameter j, group g): the sorted observations with the prior inserted at
// searchsorted(prior_mu), sigma = the larger neighbour gap clipped to [ps / min(100, 1 + #components), ps] (prior: ps),
// linear-forgetting weights by told order, prior_weight for the prior, normalised; then p_accept and the per-component
// constants of both scoring paths, and (below group) the sampler's cumulative component probabilities
__global__ void __launch_bounds__(256) tpe_model_kernel(const TpeParam* __restrict__ prm, const int* __restrict__ num, int n, int nb,
                                                        const uint64_t* __restrict__ skey, const int* __restrict__ sval, int ms, double pw,
                                                        double* __restrict__ W, double* __restrict__ MU, double* __restrict__ SG,
                                                        double* __restrict__ LC, float4* __restrict__ F4, double* __restrict__ CDF,
                                                        TpeHdr* __restrict__ hdr) {
  const int j = blockIdx.x, g = blockIdx.y, t = threadIdx.x;
  const TpeParam P = prm[num[j]];
  const int N = g ? n - nb : nb, nc = N + 1;
  const uint64_t* key = skey + (size_t)j * n + (g ? nb : 0);
  const int* gp = sval + (size_t)j * n + (g ? nb : 0);
  const size_t o = tpe_moff(j, g, ms);
  __shared__ int s_pp;
  if (t == 0) {
    int pp = 0;
    if (N == 1) {
      pp = P.pm < tpe_unordered(key[0]) ? 0 : 1;
    } else if (N >= 2) {  // searchsorted(sorted, prior_mu, side='left')
      int lo = 0, hi = N;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (tpe_unordered(key[mid]) < P.pm) lo = mid + 1; else hi = mid;
      }
      pp = lo;
    }
    s_pp = pp;
  }
  __syncthreads();
  const int pp = s_pp;
  auto srt = [&](int i) -> double { return i < pp ? tpe_unordered(key[i]) : (i == pp ? P.pm : tpe_unordered(key[i - 1])); };
  const double minsg = P.ps / fmin(100.0, 1.0 + (double)nc), maxsg = P.ps;
  double part = 0.0;
  for (int i = t; i < nc; i += blockDim.x) {
    const double mu = srt(i);
    double sg;
    if (N == 0) sg = P.ps;
    else if (N == 1) sg = 0.5 * P.ps;
    else if (i == 0) sg = srt(1) - srt(0);
    else if (i == nc - 1) sg = srt(nc - 1) - srt(nc - 2);
    else sg = fmax(mu - srt(i - 1), srt(i + 1) - mu);
    sg = fmin(fmax(sg, minsg), maxsg);
    if (i == pp) sg = P.ps;
    const double w = i == pp ? pw : tpe_lfw(gp[i < pp ? i : i - 1], N);
    MU[o + i] = mu;
    SG[o + i] = sg;
    W[o + i] = w;
    part += w;
  }
  const double wsum = tpe_block_reduce<false>(part);
  part = 0.0;
  for (int i = t; i < nc; i += blockDim.x) {
    const double w = W[o + i] / wsum;
    W[o + i] = w;
    part += w * (tpe_ncdf(P.hi, MU[o + i], SG[o + i]) - tpe_ncdf(P.lo, MU[o + i], SG[o + i]));
  }
  const double p_acc = tpe_block_reduce<false>(part);
  double A = 0.0, B = 0.0, C2max = -INFINITY, C2abs = 0.0;
  for (int i = t; i < nc; i += blockDim.x) {
    const double sg = SG[o + i];
    const double lc = log(W[o + i] / sqrt(2.0 * 3.141592653589793 * (sg * sg)) / p_acc);
    LC[o + i] = lc;
    const float c2 = (float)(lc * 1.4426950408889634);
    const float mup = (float)((MU[o + i] - P.pm) / P.ps), rp = (float)(P.ps / fmax(sg, 1e-12));
    F4[o + i] = make_float4(mup, rp, c2, 0.f);
    A = fmax(A, (double)rp);
    B = fmax(B, (double)rp * fabs((double)mup));
    C2max = fmax(C2max, (double)c2);
    C2abs = fmax(C2abs, fabs((double)c2));
  }
  A = tpe_block_reduce<true>(A);
  B = tpe_block_reduce<true>(B);
  C2max = tpe_block_reduce<true>(C2max);
  C2abs = tpe_block_reduce<true>(C2abs);
  if (t == 0) {
    TpeHdr hd;
    hd.ncomp = nc;
    hd.pad = 0;
    hd.p_acc = p_acc;
    hd.A = (float)A;
    hd.B = (float)B;
    hd.C2max = (float)C2max;
    hd.C2abs = (float)C2abs;
    hdr[2 * j + g] = hd;
    if (g == 0) {
      double cum = 0.0;
      for (int i = 0; i < nc; i++) {
        cum += W[o + i] * (tpe_ncdf(P.hi, MU[o + i], SG[o + i]) - tpe_ncdf(P.lo, MU[o + i], SG[o + i]));
        CDF[o + i] = cum;
      }
      for (int i = 0; i < nc; i++) CDF[o + i] /= cum;
      CDF[o + nc - 1] = 1.0;
    }
  }
}

// ap_categorical_sampler's tables: p_g = bincount(observations of group g, linear-forgetting weights) + prior_weight,
// normalised (each category's count summed in told order, as bincount does); score table log p_below - log p_above; the
// sampler's cumulative p_below
__global__ void __launch_bounds__(256) tpe_cat_kernel(const TpeParam* __restrict__ prm, const int* __restrict__ cat, int n, int nb, int D,
                                                      const double* __restrict__ vals, const int* __restrict__ grp, const int* __restrict__ pos,
                                                      double pw, int lcat, double* __restrict__ CP, double* __restrict__ SC,
                                                      double* __restrict__ CUM) {
  const int j = blockIdx.x, d = cat[j], t = threadIdx.x;
  const int L = prm[d].levels;
  for (int g = 0; g < 2; g++) {
    const int N = g ? n - nb : nb;
    double* p = CP + ((size_t)j * 2 + g) * lcat;
    double part = 0.0;
    for (int c = t; c < L; c += blockDim.x) {
      double acc = 0.0;
      for (int i = 0; i < n; i++)
        if (grp[i] == g && vals[(size_t)i * D + d] == (double)c) acc += tpe_lfw(pos[i], N);
      const double v = acc + pw;
      p[c] = v;
      part += v;
    }
    const double sum = tpe_block_reduce<false>(part);
    for (int c = t; c < L; c += blockDim.x) p[c] /= sum;
  }
  __syncthreads();
  const double* pb = CP + (size_t)j * 2 * lcat;
  const double* pa = pb + lcat;
  for (int c = t; c < L; c += blockDim.x) SC[(size_t)j * lcat + c] = log(pb[c]) - log(pa[c]);
  if (t == 0) {
    double cum = 0.0;
    for (int c = 0; c < L; c++) {
      cum += pb[c];
      CUM[(size_t)j * lcat + c] = cum;
    }
    CUM[(size_t)j * lcat + L - 1] = 1.0;
  }
}

// ------------------------------------------------------------------------------------------------ ask: continuous parameters
// log2 of one mixture's density (with the 1/p_accept folded into c2) at the thread's TPE_CPT scaled candidates, and its bound
__device__ __forceinline__ void tpe_mix_lse32(float4* comp, const float4* __restrict__ src, const TpeHdr hd, const float (&xs)[TPE_CPT],
                                              float (&L)[TPE_CPT], float (&E)[TPE_CPT]) {
  float mt[TPE_CPT], st[TPE_CPT];
#pragma unroll
  for (int c = 0; c < TPE_CPT; c++) { mt[c] = -INFINITY; st[c] = 0.f; }
  int nchunks = 0;
  for (int base = 0; base < hd.ncomp; base += TPE_CHUNK) {
    nchunks++;
    const int n = min(TPE_CHUNK, hd.ncomp - base);
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += TPE_THREADS) comp[i] = src[base + i];
    __syncthreads();
    float mc[TPE_CPT], sn[TPE_CPT];
#pragma unroll
    for (int c = 0; c < TPE_CPT; c++) { mc[c] = -INFINITY; sn[c] = 0.f; }
    for (int i = 0; i < n; i++) {
      const float4 cc = comp[i];
#pragma unroll
      for (int c = 0; c < TPE_CPT; c++) {
        const float z = (xs[c] - cc.x) * cc.y;
        mc[c] = fmaxf(mc[c], fmaf(-TPE_H2, z * z, cc.z));
      }
    }
    for (int i = 0; i < n; i++) {
      const float4 cc = comp[i];
#pragma unroll
      for (int c = 0; c < TPE_CPT; c++) {
        const float z = (xs[c] - cc.x) * cc.y;
        sn[c] += tpe_ex2(fmaf(-TPE_H2, z * z, cc.z) - mc[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < TPE_CPT; c++) {
      const float mn = fmaxf(mt[c], mc[c]);
      st[c] = st[c] * tpe_ex2(mt[c] - mn) + sn[c] * tpe_ex2(mc[c] - mn);
      mt[c] = mn;
    }
  }
#pragma unroll
  for (int c = 0; c < TPE_CPT; c++) {
    L[c] = mt[c] + log2f(st[c]);
    E[c] = tpe_lse_err(mt[c], st[c], L[c], hd, fabsf(xs[c]), nchunks);
  }
}

// FP32 score log l(x) - log g(x) and its error bound for TPE_CPT candidates per thread; the components of each mixture pass
// through shared memory in chunks of TPE_CHUNK (a broadcast LDS.128 per component, shared by the thread's candidates).  Per
// chunk: the maximum exponent, then Σ ex2(t - max), merged into the running (max, sum).  lb[pair] = max over candidates of
// (score - bound), the lower bound on the maximum the decision prunes with.
__global__ void __launch_bounds__(TPE_THREADS) tpe_score_kernel(TpeModels md, const int* __restrict__ cont, int Dc, int D, int M,
                                                                const double* __restrict__ X, float2* __restrict__ sc, float* __restrict__ score_out, unsigned* __restrict__ lb) {
  __shared__ float4 comp[TPE_CHUNK];
  const int pair = blockIdx.y, p = pair / Dc, d = cont[pair % Dc];
  const TpeParam P = md.prm[d];
  const int m0 = blockIdx.x * (TPE_THREADS * TPE_CPT) + threadIdx.x;
  float xs[TPE_CPT];
#pragma unroll
  for (int c = 0; c < TPE_CPT; c++) {
    const int m = m0 + c * TPE_THREADS;
    const double x = m < M ? X[((size_t)p * D + d) * M + m] : P.pm;
    xs[c] = (float)((x - P.pm) / P.ps);
  }
  float Lb[TPE_CPT], Eb[TPE_CPT], La[TPE_CPT], Ea[TPE_CPT];
  tpe_mix_lse32(comp, md.f4 + tpe_moff(P.slot, 0, md.ms), md.hdr[2 * P.slot], xs, Lb, Eb);
  tpe_mix_lse32(comp, md.f4 + tpe_moff(P.slot, 1, md.ms), md.hdr[2 * P.slot + 1], xs, La, Ea);
  const float u = 5.9604645e-8f;
  float best_lo = -INFINITY;
#pragma unroll
  for (int c = 0; c < TPE_CPT; c++) {
    const int m = m0 + c * TPE_THREADS;
    const float s2 = Lb[c] - La[c];
    const float s = s2 * 0.69314718f;
    const float e = 1.05f * (0.69314718f * (Eb[c] + Ea[c] + u * fabsf(s2)) + 2.f * u * fabsf(s)) + 1e-9f;
    if (m < M) {
      sc[(size_t)pair * M + m] = make_float2(s, e);
      if (score_out) {
        const size_t q = ((size_t)p * D + d) * M + m;
        score_out[2 * q] = s;
        score_out[2 * q + 1] = e;
      }
      best_lo = fmaxf(best_lo, s - e);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best_lo = fmaxf(best_lo, __shfl_xor_sync(0xffffffffu, best_lo, o));
  if ((threadIdx.x & 31) == 0 && best_lo > -INFINITY) atomicMax(lb + pair, tpe_fkey(best_lo));
}

// every candidate whose upper bound reaches the lower bound on the maximum is re-scored in FP64 by one warp; per block, the
// first index of the FP64 maximum among them
__global__ void __launch_bounds__(256) tpe_decide_kernel(TpeModels md, const int* __restrict__ cont, int Dc, int D, int M,
                                                         const double* __restrict__ X, const float2* __restrict__ sc, const unsigned* __restrict__ lb,
                                                         TpeBest* __restrict__ bb, int nbb, int* __restrict__ surv) {
  const int pair = blockIdx.y, p = pair / Dc, d = cont[pair % Dc], pd = p * D + d;
  const TpeParam P = md.prm[d];
  const int m = blockIdx.x * 256 + threadIdx.x, lane = threadIdx.x & 31;
  const float LB = tpe_funkey(lb[pair]);
  bool keep = false;
  if (m < M) {
    const float2 v = sc[(size_t)pair * M + m];
    keep = !(v.x + v.y < LB);
  }
  unsigned mask = __ballot_sync(0xffffffffu, keep);
  if (lane == 0 && mask) atomicAdd(surv + pd, __popc(mask));
  const size_t ob = tpe_moff(P.slot, 0, md.ms), oa = tpe_moff(P.slot, 1, md.ms);
  const int nb = md.hdr[2 * P.slot].ncomp, na = md.hdr[2 * P.slot + 1].ncomp;
  TpeBest best{0.0, -1};
  while (mask) {
    const int src = __ffs(mask) - 1;
    mask &= mask - 1;
    const int mm = m - lane + src;
    const double x = X[(size_t)pd * M + mm];
    const double v = tpe_lse64(md, ob, nb, x, lane) - tpe_lse64(md, oa, na, x, lane);
    if (tpe_better(v, mm, best)) { best.s = v; best.i = mm; }
  }
  best = tpe_block_best(best);
  if (threadIdx.x == 0) bb[(size_t)pd * nbb + blockIdx.x] = best;
}

// ------------------------------------------------------------------------------------------------ ask: quantized / categorical
// first occurrence of every level present among the candidates (parameters with at most TPE_LCAP levels)
__global__ void tpe_level_kernel(TpeModels md, const int* __restrict__ disc, int Dd, int D, int M, const double* __restrict__ X,
                                 unsigned* __restrict__ first, int lt,
                                 int* __restrict__ err) {
  const int pair = blockIdx.y, p = pair / Dd, d = disc[pair % Dd];
  const TpeParam P = md.prm[d];
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const double x = X[((size_t)p * D + d) * M + m];
  const long long j = tpe_level(P, x);
  if (j < 0) {
    atomicExch(err, 1);
    return;
  }
  if (P.levels <= TPE_LCAP) atomicMin(first + (size_t)pair * lt + j, (unsigned)m);
}
// FP64 score of each level present (table mode) or of each candidate (more levels than TPE_LCAP); equal values score equal,
// so the first index of the maximum over candidates is the best level's first occurrence
__global__ void __launch_bounds__(256) tpe_disc_score_kernel(TpeModels md, const int* __restrict__ disc, int Dd, int D, int M,
                                                             const double* __restrict__ X, const unsigned* __restrict__ first, int lt,
                                                             TpeBest* __restrict__ bb, int nbb, int* __restrict__ surv) {
  const int pair = blockIdx.y, p = pair / Dd, d = disc[pair % Dd], pd = p * D + d;
  const TpeParam P = md.prm[d];
  const bool table = P.levels <= TPE_LCAP;
  const int e = blockIdx.x * 256 + threadIdx.x, lane = threadIdx.x & 31;
  const int entries = table ? P.levels : M;
  bool present = false;
  if (e < entries) present = table ? first[(size_t)pair * lt + e] != 0xFFFFFFFFu : true;
  unsigned mask = __ballot_sync(0xffffffffu, present);
  if (lane == 0 && mask) atomicAdd(surv + pd, __popc(mask));
  TpeBest best{0.0, -1};
  while (mask) {
    const int src = __ffs(mask) - 1;
    mask &= mask - 1;
    const int ee = e - lane + src;
    long long idx, j;
    if (table) {
      idx = first[(size_t)pair * lt + ee];
      j = ee;
    } else {
      idx = ee;
      j = tpe_level(P, X[(size_t)pd * M + ee]);
      if (j < 0) continue;  // reported by tpe_level_kernel
    }
    double v;
    if (P.kind == KBO_TPE_CHOICE) {
      v = md.cat_sc[(size_t)P.slot * md.lcat + j];
    } else {
      const double x = ((double)j + P.base) * P.q;
      const size_t ob = tpe_moff(P.slot, 0, md.ms), oa = tpe_moff(P.slot, 1, md.ms);
      const TpeHdr hb = md.hdr[2 * P.slot], ha = md.hdr[2 * P.slot + 1];
      v = tpe_qlpdf64(md, ob, hb.ncomp, hb.p_acc, P, x, lane) - tpe_qlpdf64(md, oa, ha.ncomp, ha.p_acc, P, x, lane);
    }
    if (tpe_better(v, idx, best)) { best.s = v; best.i = idx; }
  }
  best = tpe_block_best(best);
  if (threadIdx.x == 0) bb[(size_t)pd * nbb + blockIdx.x] = best;
}

// per (point, parameter): the winner over the per-block results, and its value (quantized values rint(x/q)·q)
__global__ void __launch_bounds__(256) tpe_final_kernel(TpeModels md, int D, int M, const double* __restrict__ X,
                                                        const TpeBest* __restrict__ bb, int nbb, double* __restrict__ x_out,
                                                        long long* __restrict__ idx_out) {
  const int pd = blockIdx.x, d = pd % D;
  TpeBest best{0.0, -1};
  for (int i = threadIdx.x; i < nbb; i += blockDim.x) {
    const TpeBest b = bb[(size_t)pd * nbb + i];
    if (tpe_better(b.s, b.i, best)) best = b;
  }
  best = tpe_block_best(best);
  if (threadIdx.x == 0) {
    const TpeParam P = md.prm[d];
    double x = NAN;
    if (best.i >= 0) {
      x = X[(size_t)pd * M + best.i];
      if (P.kind == KBO_TPE_QUNIFORM) x = rint(x / P.q) * P.q;
    }
    x_out[pd] = x;
    if (idx_out) idx_out[pd] = best.i;
  }
}

// ------------------------------------------------------------------------------------------------ host side
static TpeModels tpe_models(kbo_tpe* t) {
  TpeModels md;
  md.prm = t->d_prm.p;
  md.w = t->w.p;
  md.mu = t->mu.p;
  md.sg = t->sg.p;
  md.lc = t->lc.p;
  md.cdf = t->cdf.p;
  md.f4 = t->f4.p;
  md.hdr = t->hdr.p;
  md.cat_sc = t->cat_sc.p;
  md.cat_cum = t->cat_cum.p;
  md.ms = t->ms;
  md.lcat = t->lcat;
  return md;
}

static int tpe_build(kbo_handle* h, kbo_tpe* t, cudaStream_t s) {
  const int n = t->n, D = t->D;
  t->nb = n ? std::min((int)std::ceil(t->gamma * std::sqrt((double)n)), TPE_LF) : 0;
  const int nb = t->nb, nn = std::max(n, 1);
  t->ms = TPE_CB + round_up(n + 1, 32);
  const size_t slots = (size_t)std::max(t->Dnum, 1) * t->ms;
  KBO_TRY(kbo_reserve(h, t->w, slots));
  KBO_TRY(kbo_reserve(h, t->mu, slots));
  KBO_TRY(kbo_reserve(h, t->sg, slots));
  KBO_TRY(kbo_reserve(h, t->lc, slots));
  KBO_TRY(kbo_reserve(h, t->cdf, slots));
  KBO_TRY(kbo_reserve(h, t->f4, slots));
  KBO_TRY(kbo_reserve(h, t->hdr, std::max(t->Dnum, 1) * 2));
  KBO_TRY(kbo_reserve(h, t->cat_p, (size_t)std::max(t->Dcat, 1) * t->lcat * 2));
  KBO_TRY(kbo_reserve(h, t->cat_sc, (size_t)std::max(t->Dcat, 1) * t->lcat));
  KBO_TRY(kbo_reserve(h, t->cat_cum, (size_t)std::max(t->Dcat, 1) * t->lcat));
  KBO_TRY(kbo_reserve(h, t->grp, (size_t)nn));
  KBO_TRY(kbo_reserve(h, t->pos, (size_t)nn));
  const size_t ns = (size_t)std::max(t->Dnum, 1) * nn;
  KBO_TRY(kbo_reserve(h, t->skey, ns));
  KBO_TRY(kbo_reserve(h, t->skey2, ns));
  KBO_TRY(kbo_reserve(h, t->sval, ns));
  KBO_TRY(kbo_reserve(h, t->sval2, ns));
  if (n > 0) {
    KBO_TRY(kbo_reserve(h, t->lkey, (size_t)n));
    KBO_TRY(kbo_reserve(h, t->lkey2, (size_t)n));
    KBO_TRY(kbo_reserve(h, t->lidx, (size_t)n));
    KBO_TRY(kbo_reserve(h, t->lidx2, (size_t)n));
    KBO_TRY(kbo_reserve(h, t->below, TPE_LF));
    KBO_TRY(kbo_reserve(h, t->segb, (size_t)std::max(t->Dnum, 1) * 2));
    KBO_TRY(kbo_reserve(h, t->sege, (size_t)std::max(t->Dnum, 1) * 2));
    size_t b1 = 0, b2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b1, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int*)nullptr, (int*)nullptr, n, 0, 64, s);
    if (t->Dnum)
      cub::DeviceSegmentedSort::StableSortPairs(nullptr, b2, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int*)nullptr, (int*)nullptr,
                                                t->Dnum * n, 2 * t->Dnum, (const int*)nullptr, (const int*)nullptr, s);
    KBO_TRY(kbo_reserve(h, t->tmp, std::max<size_t>(std::max(b1, b2), 16)));
    // the stable loss order (NumPy's argsort(kind='mergesort'), NaN last)
    tpe_loss_keys_kernel<<<(n + 255) / 256, 256, 0, s>>>(t->loss.p, n, t->lkey.p, t->lidx.p);
    KBO_LAUNCH_CHECK(h);
    size_t bytes = t->tmp.cap;
    KBO_CUDA(h, cub::DeviceRadixSort::SortPairs(t->tmp.p, bytes, t->lkey.p, t->lkey2.p, t->lidx.p,
                                               t->lidx2.p, n, 0, 64, s));
    tpe_split_kernel<<<1, 32, 0, s>>>(t->lidx2.p, nb, t->below.p);
    KBO_LAUNCH_CHECK(h);
    tpe_group_kernel<<<(n + 255) / 256, 256, 0, s>>>(t->below.p, nb, n, t->grp.p, t->pos.p);
    KBO_LAUNCH_CHECK(h);
    if (t->Dnum) {
      std::vector<int> sb(2 * t->Dnum), se(2 * t->Dnum);
      for (int j = 0; j < t->Dnum; j++) {
        sb[2 * j] = j * n;
        se[2 * j] = j * n + nb;
        sb[2 * j + 1] = j * n + nb;
        se[2 * j + 1] = (j + 1) * n;
      }
      KBO_CUDA(h, kbo_copy(t->segb.p, sb.data(), sb.size(), cudaMemcpyHostToDevice, s));
      KBO_CUDA(h, kbo_copy(t->sege.p, se.data(), se.size(), cudaMemcpyHostToDevice, s));
      tpe_seg_fill_kernel<<<dim3((n + 255) / 256, t->Dnum), 256, 0, s>>>(t->vals.p, n, nb, D, t->d_num.p,
                                                                        t->grp.p, t->pos.p, t->skey2.p,
                                                                        t->sval2.p);
      KBO_LAUNCH_CHECK(h);
      bytes = t->tmp.cap;
      const int *segb = t->segb.p, *sege = t->sege.p;   // the offset types the size query above was made with
      KBO_CUDA(h, cub::DeviceSegmentedSort::StableSortPairs(t->tmp.p, bytes, t->skey2.p, t->skey.p,
                                                            t->sval2.p, t->sval.p, t->Dnum * n, 2 * t->Dnum, segb, sege, s));
      // the host vectors above must outlive the copies (pageable memory: staged before cudaMemcpyAsync returns)
    }
  }
  if (t->Dnum) {
    tpe_model_kernel<<<dim3(t->Dnum, 2), 256, 0, s>>>(t->d_prm.p, t->d_num.p, n, nb, t->skey.p,
                                                      t->sval.p, t->ms, t->pw, t->w.p, t->mu.p, t->sg.p,
                                                      t->lc.p, t->f4.p, t->cdf.p, t->hdr.p);
    KBO_LAUNCH_CHECK(h);
  }
  if (t->Dcat) {
    tpe_cat_kernel<<<t->Dcat, 256, 0, s>>>(t->d_prm.p, t->d_cat.p, n, nb, D, t->vals.p,
                                           t->grp.p, t->pos.p, t->pw, t->lcat, t->cat_p.p,
                                           t->cat_sc.p, t->cat_cum.p);
    KBO_LAUNCH_CHECK(h);
  }
  t->built_n = n;
  return KBO_OK;
}

extern "C" {

int kbo_tpe_create(kbo_handle* h, kbo_tpe** out, int32_t D, const int32_t* kinds, const double* lo, const double* hi, const double* q,
                   const int32_t* levels, double gamma, double prior_weight, uint64_t seed) {
  if (!h || !out) return KBO_ERR_INVALID;
  *out = nullptr;
  if (D < 1 || D > 65535) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_create: 1 <= D <= 65535 supported (got %d)", D);
  if (!kinds) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_create: null kinds");
  if (!(gamma > 0.0 && gamma < 1.0)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_create: gamma must be in (0, 1) (got %g)", gamma);
  if (!(prior_weight > 0.0) || !std::isfinite(prior_weight)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_create: prior_weight must be > 0 (got %g)", prior_weight);
  KBO_CUDA(h, cudaSetDevice(h->device));
  std::unique_ptr<kbo_tpe> t(new (std::nothrow) kbo_tpe());
  if (!t) return KBO_ERR_NOMEM;
  t->D = D;
  t->gamma = gamma;
  t->pw = prior_weight;
  t->seed = seed;
  t->prm.resize(D);
  for (int d = 0; d < D; d++) {
    TpeParam& P = t->prm[d];
    memset(&P, 0, sizeof P);
    P.kind = kinds[d];
    if (P.kind == KBO_TPE_CHOICE) {
      if (!levels || levels[d] < 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_create: parameter %d: a choice needs >= 1 categories", d);
      P.levels = levels[d];
      P.slot = t->Dcat++;
      t->cat.push_back(d);
      t->disc.push_back(d);
      t->lcat = std::max(t->lcat, P.levels);
      if (P.levels <= TPE_LCAP) t->lt = std::max(t->lt, P.levels);
      continue;
    }
    if (P.kind != KBO_TPE_UNIFORM && P.kind != KBO_TPE_QUNIFORM) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_create: parameter %d: unknown kind %d", d, kinds[d]);
    if (!lo || !hi || !std::isfinite(lo[d]) || !std::isfinite(hi[d]) || !(lo[d] < hi[d]))
      KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_create: parameter %d: need finite lo < hi", d);
    P.lo = lo[d];
    P.hi = hi[d];
    P.pm = 0.5 * (P.hi + P.lo);
    P.ps = 1.0 * (P.hi - P.lo);
    P.slot = t->Dnum++;
    t->num.push_back(d);
    if (P.kind == KBO_TPE_QUNIFORM) {
      if (!q || !(q[d] > 0.0) || !std::isfinite(q[d])) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_create: parameter %d: q must be > 0", d);
      P.q = q[d];
      P.base = std::nearbyint(P.lo / P.q);
      const double L = std::nearbyint(P.hi / P.q) - P.base + 1.0;
      if (!(L >= 1.0 && L < 2147483647.0)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_create: parameter %d: too many levels", d);
      P.levels = (int)L;
      t->disc.push_back(d);
      if (P.levels <= TPE_LCAP) t->lt = std::max(t->lt, P.levels);
    } else {
      t->cont.push_back(d);
    }
  }
  t->Dc = (int)t->cont.size();
  t->Dd = (int)t->disc.size();
  KBO_TRY(kbo_upload(h, t->d_prm, t->prm.data(), D));
  KBO_TRY(kbo_upload(h, t->d_cont, t->cont.data(), t->cont.size()));
  KBO_TRY(kbo_upload(h, t->d_disc, t->disc.data(), t->disc.size()));
  KBO_TRY(kbo_upload(h, t->d_num, t->num.data(), t->num.size()));
  KBO_TRY(kbo_upload(h, t->d_cat, t->cat.data(), t->cat.size()));
  KBO_TRY(t->ev.create());
  *out = t.release();
  return KBO_OK;
}

void kbo_tpe_destroy(kbo_tpe* t) {
  if (t) delete t;
}

int kbo_tpe_tell(kbo_handle* h, kbo_tpe* t, const double* X, const double* loss, int32_t n_new, int on_host, void* stream) {
  if (!h || !t) return KBO_ERR_INVALID;
  if (n_new < 0) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_tell: n_new must be >= 0 (got %d)", n_new);
  if (n_new == 0) return KBO_OK;
  if (!X || !loss) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_tell: null argument");
  if ((int64_t)t->n + n_new > (1 << 24)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_tell: at most 2^24 trials supported");
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  KBO_TRY(tpe_history_append(h, t, X, loss, n_new, on_host, s));
  if (on_host) KBO_CUDA(h, cudaStreamSynchronize(s));   // the caller may free its host arrays on return
  t->n += n_new;
  return KBO_OK;
}

// One ask over local candidates [0, M), which are global candidates [m0, m0 + M) of n_candidates = Mall.  With val_dev null
// it is kbo_tpe_ask (m0 = 0, M = Mall): the winners' values go to x_dev.  With val_dev it is a shard ask: each (point,
// parameter) writes its FP64 winner and global index to val_dev / idx_dev, and M = 0 (an empty shard) is legal.
static int tpe_ask_run(kbo_handle* h, kbo_tpe* t, int k, int M, int m0, int Mall, const double* cand_dev, double* x_dev, int64_t* idx_dev,
                       double* cand_out_dev, float* score_out_dev, double* val_dev, cudaStream_t s) {
  KBO_CUDA(h, cudaSetDevice(h->device));
  cudaEventRecord(t->ev[0], s);
  if (t->built_n != t->n) KBO_TRY(tpe_build(h, t, s));
  const uint32_t ask = t->asks++;
  const int D = t->D, KD = k * D;
  if (val_dev) {
    t->pick_ask = ask;
    t->pick_k = k;
    t->pick_M = Mall;
    t->pick_n = t->n;
    if (M == 0) {
      tpe_shard_best_kernel<<<KD, 256, 0, s>>>(nullptr, 0, m0, Mall, val_dev, (long long*)idx_dev);
      KBO_LAUNCH_CHECK(h);
      t->last_surv.assign(KD, 0);
      std::fill(t->last_ms, t->last_ms + 5, 0.f);
      KBO_CUDA(h, cudaStreamSynchronize(s));
      return KBO_OK;
    }
  }
  const int nbb = (std::max(M, t->Dd ? t->lt : 1) + 255) / 256;
  KBO_TRY(kbo_reserve(h, t->surv, (size_t)KD));
  KBO_TRY(kbo_reserve(h, t->bb, (size_t)KD * nbb));
  KBO_TRY(kbo_reserve(h, t->err, 1));
  KBO_CUDA(h, cudaMemsetAsync(t->surv.p, 0, sizeof *t->surv.p * (size_t)KD, s));
  KBO_CUDA(h, cudaMemsetAsync(t->err.p, 0, sizeof *t->err.p, s));
  const TpeModels md = tpe_models(t);
  const double* X = cand_dev;
  if (!X) {   // the draws go to the caller's buffer if it wants them, else to the handle's
    double* Xw = cand_out_dev;
    if (!Xw) {
      KBO_TRY(kbo_reserve(h, t->draws, (size_t)KD * M));
      Xw = t->draws.p;
    }
    tpe_draw_kernel<<<dim3((M + 255) / 256, KD), 256, 0, s>>>(md, D, M, m0, t->seed, ask, Xw);
    KBO_LAUNCH_CHECK(h);
    X = Xw;
  } else if (cand_out_dev) {
    KBO_CUDA(h, cudaMemcpyAsync(cand_out_dev, cand_dev, 8 * (size_t)KD * M, cudaMemcpyDeviceToDevice, s));
  }
  cudaEventRecord(t->ev[1], s);
  if (t->Dc) {
    const int pairs = k * t->Dc;
    KBO_TRY(kbo_reserve(h, t->sc, (size_t)pairs * M));
    KBO_TRY(kbo_reserve(h, t->lb, (size_t)pairs));
    KBO_CUDA(h, cudaMemsetAsync(t->lb.p, 0, sizeof *t->lb.p * (size_t)pairs, s));
    tpe_score_kernel<<<dim3((M + TPE_THREADS * TPE_CPT - 1) / (TPE_THREADS * TPE_CPT), pairs), TPE_THREADS, 0, s>>>(
        md, t->d_cont.p, t->Dc, D, M, X, t->sc.p, score_out_dev, t->lb.p);
    KBO_LAUNCH_CHECK(h);
    cudaEventRecord(t->ev[2], s);
    tpe_decide_kernel<<<dim3(nbb, pairs), 256, 0, s>>>(md, t->d_cont.p, t->Dc, D, M, X, t->sc.p,
                                                       t->lb.p, t->bb.p, nbb, t->surv.p);
    KBO_LAUNCH_CHECK(h);
  } else {
    cudaEventRecord(t->ev[2], s);
  }
  cudaEventRecord(t->ev[3], s);
  if (t->Dd) {
    const int pairs = k * t->Dd;
    KBO_TRY(kbo_reserve(h, t->first, (size_t)pairs * t->lt));
    KBO_CUDA(h, cudaMemsetAsync(t->first.p, 0xFF, sizeof *t->first.p * (size_t)pairs * t->lt, s));
    tpe_level_kernel<<<dim3((M + 255) / 256, pairs), 256, 0, s>>>(md, t->d_disc.p, t->Dd, D, M, X, t->first.p, t->lt,
                                                                  t->err.p);
    KBO_LAUNCH_CHECK(h);
    tpe_disc_score_kernel<<<dim3(nbb, pairs), 256, 0, s>>>(md, t->d_disc.p, t->Dd, D, M, X, t->first.p, t->lt, t->bb.p, nbb, t->surv.p);
    KBO_LAUNCH_CHECK(h);
  }
  cudaEventRecord(t->ev[4], s);
  if (val_dev) tpe_shard_best_kernel<<<KD, 256, 0, s>>>(t->bb.p, nbb, m0, Mall, val_dev, (long long*)idx_dev);
  else tpe_final_kernel<<<KD, 256, 0, s>>>(md, D, M, X, t->bb.p, nbb, x_dev, (long long*)idx_dev);
  KBO_LAUNCH_CHECK(h);
  cudaEventRecord(t->ev[5], s);
  t->last_surv.assign(KD, 0);
  int err = 0;
  KBO_CUDA(h, kbo_copy(t->last_surv.data(), t->surv.p, (size_t)KD, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, kbo_copy(&err, t->err.p, 1, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  for (int i = 0; i < 5; i++) cudaEventElapsedTime(&t->last_ms[i], t->ev[i], t->ev[i + 1]);
  if (err) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_ask: a supplied candidate of a quantized or categorical parameter is outside its levels");
  return KBO_OK;
}

int kbo_tpe_ask(kbo_handle* h, kbo_tpe* t, int32_t k, int32_t M, const double* cand_dev, double* x_dev, int64_t* idx_dev, double* cand_out_dev,
                float* score_out_dev, void* stream) {
  if (!h || !t) return KBO_ERR_INVALID;
  if (!x_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_ask: null output");
  if (k < 1 || k > 65535) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_ask: 1 <= k <= 65535 supported (got %d)", k);
  if (M < 1 || M > TPE_MAXM) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_ask: 1 <= n_candidates <= 2^24 supported (got %d)", M);
  if ((int64_t)k * t->D > 65535) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_ask: k * D must be <= 65535");
  if ((int64_t)k * t->D * M > (1ll << 31)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_ask: k * D * n_candidates must be <= 2^31");
  return tpe_ask_run(h, t, k, M, 0, M, cand_dev, x_dev, idx_dev, cand_out_dev, score_out_dev, nullptr, (cudaStream_t)stream);
}

int kbo_tpe_ask_shard(kbo_handle* h, kbo_tpe* t, int32_t k, int32_t M, int32_t lo, int32_t hi, const double* cand_dev, double* val_dev,
                      int64_t* idx_dev, void* stream) {
  if (!h || !t) return KBO_ERR_INVALID;
  if (cand_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_ask_shard: caller-supplied candidates are not accepted (the shards draw their own)");
  if (!val_dev || !idx_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_ask_shard: null output");
  if (k < 1 || k > 65535) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_ask_shard: 1 <= k <= 65535 supported (got %d)", k);
  if (M < 1 || M > TPE_MAXM) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_ask_shard: 1 <= n_candidates <= 2^24 supported (got %d)", M);
  if (!(0 <= lo && lo <= hi && hi <= M)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_ask_shard: need 0 <= lo <= hi <= n_candidates (got [%d, %d) of %d)", lo, hi, M);
  if ((int64_t)k * t->D > 65535) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_ask_shard: k * D must be <= 65535");
  if ((int64_t)k * t->D * (hi - lo) > (1ll << 31)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_ask_shard: k * D * (hi - lo) must be <= 2^31");
  return tpe_ask_run(h, t, k, hi - lo, lo, M, nullptr, nullptr, idx_dev, nullptr, nullptr, val_dev, (cudaStream_t)stream);
}

int kbo_tpe_pick(kbo_handle* h, kbo_tpe* t, int32_t k, const int64_t* idx_dev, double* x_dev, void* stream) {
  if (!h || !t) return KBO_ERR_INVALID;
  if (!idx_dev || !x_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_pick: null argument");
  if (t->pick_k == 0 || t->pick_n != t->n) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_pick: no shard ask since the last tell");
  if (k != t->pick_k) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_pick: k must be the last shard ask's (%d, got %d)", t->pick_k, k);
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  KBO_TRY(kbo_reserve(h, t->err, 1));
  KBO_CUDA(h, cudaMemsetAsync(t->err.p, 0, sizeof *t->err.p, s));
  const int KD = k * t->D;
  tpe_pick_kernel<<<(KD + 255) / 256, 256, 0, s>>>(tpe_models(t), KD, t->D, t->pick_M, t->seed, t->pick_ask, (const long long*)idx_dev,
                                                   x_dev, t->err.p);
  KBO_LAUNCH_CHECK(h);
  int err = 0;
  KBO_CUDA(h, kbo_copy(&err, t->err.p, 1, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (err) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_pick: a winning index is outside [0, n_candidates)");
  return KBO_OK;
}

int kbo_tpe_state(kbo_handle* h, kbo_tpe* t, int32_t param, int32_t group, double* w, double* mu, double* sigma, int32_t cap, int32_t* ncomp,
                  double* p_accept, int32_t* n_below, void* stream) {
  if (!h || !t) return KBO_ERR_INVALID;
  if (param < 0 || param >= t->D || group < 0 || group > 1 || cap < 0) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_tpe_state: bad argument");
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  if (t->built_n != t->n) KBO_TRY(tpe_build(h, t, s));
  const TpeParam& P = t->prm[param];
  int nc;
  double pa = 1.0;
  if (P.kind == KBO_TPE_CHOICE) {
    nc = P.levels;
    if (w) KBO_CUDA(h, kbo_copy(w, t->cat_p.p + ((size_t)P.slot * 2 + group) * t->lcat, (size_t)std::min(cap, nc),
                                       cudaMemcpyDeviceToHost, s));
  } else {
    TpeHdr hd;
    KBO_CUDA(h, kbo_copy(&hd, t->hdr.p + 2 * P.slot + group, 1, cudaMemcpyDeviceToHost, s));
    KBO_CUDA(h, cudaStreamSynchronize(s));
    nc = hd.ncomp;
    pa = hd.p_acc;
    const size_t o = (size_t)P.slot * t->ms + (group ? TPE_CB : 0), c = (size_t)std::min(cap, nc);
    KBO_CUDA(h, kbo_d2h(w, t->w.p + o, c, s));
    KBO_CUDA(h, kbo_d2h(mu, t->mu.p + o, c, s));
    KBO_CUDA(h, kbo_d2h(sigma, t->sg.p + o, c, s));
  }
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (ncomp) *ncomp = nc;
  if (p_accept) *p_accept = pa;
  if (n_below) *n_below = t->nb;
  return KBO_OK;
}

int kbo_tpe_last_survivors(kbo_handle* h, kbo_tpe* t, int32_t* out, int32_t n) {
  if (!h || !t) return KBO_ERR_INVALID;
  for (int i = 0; out && i < n && i < (int)t->last_surv.size(); i++) out[i] = t->last_surv[i];
  return (int)t->last_surv.size();
}

int kbo_tpe_last_timings(kbo_handle* h, kbo_tpe* t, float* ms, int32_t n) {
  if (!h || !t) return KBO_ERR_INVALID;
  for (int i = 0; ms && i < n && i < 5; i++) ms[i] = t->last_ms[i];
  return 5;
}

}  // extern "C"
