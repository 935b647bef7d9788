// Code shared by the Parzen-estimator samplers: tpe.cu (hyperopt's tpe.suggest) and mvtpe.cu (Optuna's multivariate
// TPESampler).  Loss keys in NumPy's order and the below / above split, the truncated-normal inverse-CDF draw, first-index
// argmax bookkeeping, block reductions and the MUFU exponential; on the host, the told history's append.
#pragma once
#include <stdint.h>
#include <algorithm>

#include "kbo_internal.cuh"

#define TPE_LF 25  // hyperopt's DEFAULT_LF and Optuna's ramp length: linear forgetting, and the cap on n_below

__device__ __forceinline__ uint64_t tpe_ordered(double v) {  // doubles as unsigned keys in NumPy's order: -0 == +0, NaN last
  if (v != v) return ~0ull;
  if (v == 0.0) v = 0.0;
  const uint64_t b = (uint64_t)__double_as_longlong(v);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double tpe_unordered(uint64_t k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k));
}
__device__ __forceinline__ unsigned tpe_fkey(float f) {  // floats as unsigned keys (0 is below every float)
  const unsigned b = __float_as_uint(f);
  return (b >> 31) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float tpe_funkey(unsigned k) { return __uint_as_float((k >> 31) ? (k & 0x7FFFFFFFu) : ~k); }
__device__ __forceinline__ float tpe_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// hyperopt's linear_forgetting_weights(N, 25)[j], and Optuna's default_weights(N)[j]: ones for N <= 25, else
// linspace(1/N, 1, N - 25) then 25 ones
__device__ __forceinline__ double tpe_lfw(int j, int N) {
  if (N <= TPE_LF) return 1.0;
  const int nr = N - TPE_LF;
  if (j >= nr) return 1.0;
  const double start = 1.0 / N;
  if (nr == 1) return start;
  if (j == nr - 1) return 1.0;
  return (double)j * ((1.0 - start) / (double)(nr - 1)) + start;
}

struct TpeBest {
  double s;
  long long i;  // -1: none
};
// first index of the maximum, NaN above everything (np.argmax)
__device__ __forceinline__ bool tpe_better(double s, long long i, const TpeBest& b) {
  if (i < 0) return false;
  if (b.i < 0) return true;
  const bool an = s != s, bn = b.s != b.s;
  if (an != bn) return an;
  if (!an && s != b.s) return s > b.s;
  return i < b.i;
}
__device__ __forceinline__ TpeBest tpe_block_best(TpeBest b) {
  __shared__ double ss[32];
  __shared__ long long si[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double s = __shfl_xor_sync(0xffffffffu, b.s, o);
    const long long i = __shfl_xor_sync(0xffffffffu, b.i, o);
    if (tpe_better(s, i, b)) { b.s = s; b.i = i; }
  }
  if (lane == 0) { ss[warp] = b.s; si[warp] = b.i; }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int k = 1; k < (int)(blockDim.x >> 5); k++)
      if (tpe_better(ss[k], si[k], b)) { b.s = ss[k]; b.i = si[k]; }
  __syncthreads();
  return b;  // valid in thread 0
}
// a shard ask's result per row (tpe: (point, parameter); mvtpe: point): the winner over the row's nbb per-block results as
// (FP64 value, global index lo + local index).  A row with no candidate (nbb = 0: an empty shard) reports (-inf, sentinel):
// sentinel is n_candidates, past every real index, so it loses even to a real -inf under the first-index rule.
static __global__ void __launch_bounds__(256) tpe_shard_best_kernel(const TpeBest* __restrict__ bb, int nbb, long long lo, long long sentinel,
                                                                    double* __restrict__ val, long long* __restrict__ idx) {
  const int r = blockIdx.x;
  TpeBest best{0.0, -1};
  for (int i = threadIdx.x; i < nbb; i += blockDim.x) {
    const TpeBest b = bb[(size_t)r * nbb + i];
    if (tpe_better(b.s, b.i, best)) best = b;
  }
  best = tpe_block_best(best);
  if (threadIdx.x == 0) {
    val[r] = best.i >= 0 ? best.s : -INFINITY;
    idx[r] = best.i >= 0 ? lo + best.i : sentinel;
  }
}
template <bool MAX>
__device__ __forceinline__ double tpe_block_reduce(double v) {
  __shared__ double red[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double u = __shfl_xor_sync(0xffffffffu, v, o);
    v = MAX ? fmax(v, u) : v + u;
  }
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int k = 1; k < (int)(blockDim.x >> 5); k++) v = MAX ? fmax(v, red[k]) : v + red[k];
  if (threadIdx.x == 0) red[0] = v;
  __syncthreads();
  return red[0];
}

// a draw from N(mu, sg²) truncated to [lo, hi) by inverse CDF, u2 in (0, 1): on the side of the mean where the tail
// probabilities keep their relative precision; the result is clamped into [lo, hi)
__device__ __forceinline__ double tpe_truncnorm_draw(double lo, double hi, double mu, double sg, double u2) {
  const double a = (lo - mu) / sg, b = (hi - mu) / sg;
  double z;
  if (a + b > 0.0) {
    const double pl = normcdf(-b), pu = normcdf(-a);
    z = -normcdfinv(pl + u2 * (pu - pl));
  } else {
    const double pl = normcdf(a), pu = normcdf(b);
    z = normcdfinv(pl + u2 * (pu - pl));
  }
  double x = fma(sg, z, mu);
  if (!(x >= lo)) x = lo;
  if (x >= hi) x = nextafter(hi, lo);
  return x;
}
// the two uniforms of a Philox block: u1 in [0, 1) from r[0..1], u2 in (0, 1) from r[2..3], 53 bits each
__device__ __forceinline__ double tpe_u01(uint32_t a, uint32_t b) {
  return (double)((((uint64_t)a) << 21) ^ (uint64_t)(b >> 11)) * (1.0 / 9007199254740992.0);
}
__device__ __forceinline__ double tpe_u01_open(uint32_t a, uint32_t b) {
  return ((double)((((uint64_t)a) << 21) ^ (uint64_t)(b >> 11)) + 0.5) * (1.0 / 9007199254740992.0);
}

// ---- the split ---------------------------------------------------------------------------------------------------------
static __global__ void tpe_loss_keys_kernel(const double* __restrict__ loss, int n, uint64_t* __restrict__ key, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    key[i] = tpe_ordered(loss[i]);
    idx[i] = i;
  }
}
// below trials in told order (the first n_below <= TPE_LF of the stable loss order, sorted by index)
static __global__ void tpe_split_kernel(const int* __restrict__ order, int nb, int* __restrict__ below) {
  if (threadIdx.x != 0) return;
  int b[TPE_LF];
  for (int j = 0; j < nb; j++) {
    int v = order[j], k = j;
    while (k > 0 && b[k - 1] > v) { b[k] = b[k - 1]; k--; }
    b[k] = v;
  }
  for (int j = 0; j < nb; j++) below[j] = b[j];
}
// group (0 below, 1 above) and position within the group in told order
static __global__ void tpe_group_kernel(const int* __restrict__ below, int nb, int n, int* __restrict__ grp, int* __restrict__ pos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int c = 0;
  bool isb = false;
  for (int j = 0; j < nb; j++) {
    const int b = below[j];
    c += b < i;
    isb |= b == i;
  }
  grp[i] = isb ? 0 : 1;
  pos[i] = isb ? c : i - c;
}

// ---- the told history (host) -----------------------------------------------------------------------------------------
// Queues the copy of n_new trials (D values and one loss each) into rows t->n .. t->n + n_new - 1 of t->vals / t->loss on s,
// growing both by doubling first.  Rows already told survive a failed growth; t->n is left for the caller to advance.
template <class Sampler>
static int tpe_history_append(kbo_handle* h, Sampler* t, const double* X, const double* loss, int n_new, int on_host, cudaStream_t s) {
  const size_t D = t->D;
  if (t->n + n_new > t->cap) {
    const int cap = std::max({2 * t->cap, t->n + n_new, 64});
    DevBuf<double> v, l;
    KBO_TRY(kbo_reserve(h, v, D * cap));
    KBO_TRY(kbo_reserve(h, l, (size_t)cap));
    if (t->n) {
      KBO_CUDA(h, kbo_copy(v.p, t->vals.p, D * t->n, cudaMemcpyDeviceToDevice, s));
      KBO_CUDA(h, kbo_copy(l.p, t->loss.p, (size_t)t->n, cudaMemcpyDeviceToDevice, s));
      KBO_CUDA(h, cudaStreamSynchronize(s));
    }
    t->vals = std::move(v);
    t->loss = std::move(l);
    t->cap = cap;
  }
  const cudaMemcpyKind kind = on_host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
  KBO_CUDA(h, kbo_copy(t->vals.p + D * t->n, X, D * n_new, kind, s));
  KBO_CUDA(h, kbo_copy(t->loss.p + t->n, loss, (size_t)n_new, kind, s));
  return KBO_OK;
}
