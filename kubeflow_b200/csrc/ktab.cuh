// Kernel function k = f(d²) in FP64, branch-free, in registers.
// (A Taylor-table variant was measured first: two data-dependent 16-byte loads per element made the kernel L1-gather
//  bound, slower than this polynomial — so the table is gone.)
//   exp(x), x <= 0:  n = rint(x·log2e) by the 1.5·2⁵² trick, f = x·log2e − n (two-term log2e), 2^f by a degree-11
//   polynomial in f (|f·ln2| ≤ 0.3466, truncation 6e-15 relative), scaled by 2ⁿ through the exponent bits.
//   Results below 2⁻¹⁰²⁰ flush to 0 (irrelevant next to the 1e-5 contract).
#pragma once
#include <cuda_runtime.h>

__device__ __forceinline__ double kbo_exp_nonpos(double x) {
  const double t = x * 1.4426950408889634;
  const double u = t + 6755399441055744.0;          // 1.5·2^52: rounds t to nearest integer in the low word
  const int ni = __double2loint(u);
  const double nf = u - 6755399441055744.0;
  double f = fma(x, 1.4426950408889634, -nf);
  f = fma(x, 2.0355273740931033e-17, f);             // low part of log2(e)
  // 2^f = Σ (ln2)^k/k! · f^k, |f| ≤ 1/2 (the ln2 factor folded into the coefficients: one DMUL less per value)
  double p = 4.44553827187081e-10;
  p = fma(p, f, 7.054911620801121e-09);
  p = fma(p, f, 1.0178086009239696e-07);
  p = fma(p, f, 1.3215486790144305e-06);
  p = fma(p, f, 1.5252733804059838e-05);
  p = fma(p, f, 0.00015403530393381606);
  p = fma(p, f, 0.0013333558146428441);
  p = fma(p, f, 0.009618129107628477);
  p = fma(p, f, 0.055504108664821576);
  p = fma(p, f, 0.2402265069591007);
  p = fma(p, f, 0.6931471805599453);
  p = fma(p, f, 1.0);
  const int hi = __double2hiint(p) + (ni << 20);
  const double r = __hiloint2double(hi, __double2loint(p));
  return ni < -1020 ? 0.0 : r;
}

// branch-free sqrt for x >= 0: fp32 MUFU.RSQ seed (~2^-22), ONE Newton step for 1/sqrt in FP64 (→ ~1e-13), then the
// Newton correction on s = x·y itself, which squares the error again (≤ 1 ulp).
// x is floored at 1e-30 so the seed is finite; sqrt(0) comes out as 1e-15, i.e. k(0) = 1 − O(1e-30).
__device__ __forceinline__ double kbo_sqrt_nonneg(double x) {
  x = fmax(x, 1e-30);
  double y = (double)rsqrtf((float)x);
  y = y * fma(-0.5 * x, y * y, 1.5);
  const double s = x * y;
  return fma(fma(-s, s, x), 0.5 * y, s);
}

__device__ __forceinline__ double kbo_kernel_exact(double d2, int kind) {
  d2 = fmax(d2, 0.0);
  if (kind == 0 /*KBO_KERNEL_RBF*/) return kbo_exp_nonpos(-0.5 * d2);
  const double s = kbo_sqrt_nonneg(5.0 * d2);
  return fma(s, fma(s, 1.0 / 3.0, 1.0), 1.0) * kbo_exp_nonpos(-s);
}
