// FP64 acquisition values and the first-index argmax order, shared by the GP sweep (sweep.cu), the forest sweep (forest.cu) and
// the GBRT sweep (gbrt.cu): skopt.acquisition.gaussian_ei / gaussian_lcb / gaussian_pi on a posterior mean and variance.
#pragma once
#include "../../include/kbo.h"

// (v, i) beats (bv, bi): larger value, lowest index among equals (np.argmin(-values)).
__device__ __forceinline__ bool better(double v, long long i, double bv, long long bi) { return v > bv || (v == bv && i < bi); }

// The acquisition at mean mu and standard deviation sd as they are: LCB takes any sd (the GBRT sweep's may be negative where its
// quantiles cross), EI and PI are 0 where sd <= 0.
template <typename T>
__device__ __forceinline__ T acq_of_sd(T mu, T sd, int acq, T yopt, T xi, T kappa) {
  if (acq == KBO_ACQ_LCB) return -(mu - kappa * sd);
  if (!(sd > (T)0)) return sd == sd ? (T)0 : sd;   // σ = 0: no improvement possible; a NaN σ (NaN y statistics) stays NaN
  const T imp = yopt - xi - mu;
  const T z = imp / sd;
  const T cdf = (T)0.5 * erfc(-z * (T)0.70710678118654752440);
  if (acq == KBO_ACQ_PI) return cdf;
  const T pdf = exp((T)-0.5 * z * z) * (T)0.39894228040143267794;
  return imp * cdf + sd * pdf;
}

template <typename T>
__device__ __forceinline__ T acq_value(T mun, T varn, int acq, T ymean, T ystd, T yopt, T xi, T kappa, T* mu_o, T* sd_o) {
  const T var = varn > (T)0 ? varn : (T)0;  // $SK/_gpr.py:485-491
  const T mu = ystd * mun + ymean;          // :450
  const T sd = sqrt(var * ystd * ystd);     // :494,:500
  *mu_o = mu;
  *sd_o = sd;
  return acq_of_sd(mu, sd, acq, yopt, xi, kappa);
}
