// Code shared by the tree surrogates: forest.cu (RF / ET) and gbrt.cu (GBRT).  On the device, the stable warp partition of the
// fits, the finite check and column presort of the history, and the sweeps' first-index argmax, per CTA and across CTAs; on the
// host, the state both models hold and the plumbing of their fit, sweep, predict and timing entry points.  As in
// kbo_tpe_common.cuh, kernels and host helpers are static: each surrogate's translation unit compiles its own copy.
#pragma once
#include <stdint.h>
#include <algorithm>

#include <cub/device/device_segmented_radix_sort.cuh>

#include "kbo_internal.cuh"
#include "kbo_acq.cuh"

// The state of a fitted tree model: its history (X, y), the flag of its finite check, its presorted columns (order: D × N row
// indices, each column sorted by value), the sweep's per-CTA argmax partials, and the fit (ev[0] → ev[1]) and sweep (ev[2] →
// ev[3]) events.
struct TreeCore {
  int N = 0, D = 0;
  bool fitted = false;
  DevBuf<float> X;
  DevBuf<double> y;
  DevBuf<int> flag, order_in, order, seg;
  DevBuf<uint32_t> keys, keys2;
  DevBuf<unsigned char> sort_tmp;
  DevBuf<kbo_best> part;
  float last_ms[2] = {0.f, 0.f};     // fit, sweep
  EventSet<4> ev;
};

// Stable partition of one segment seg[0, c) by pred, by one warp: lefts in place (a left is never written past the positions the
// warp has read), rights through tr[] and back.  Returns the left count.
template <typename P>
__device__ __forceinline__ int warp_partition(int* seg, int* tr, int c, P pred) {
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  int nl = 0, nr = 0;
  for (int j0 = 0; j0 < c; j0 += 32) {
    const int j = j0 + lane;
    const bool valid = j < c;
    const int i = valid ? seg[j] : 0;
    const bool L = valid && pred(i), R = valid && !L;
    __syncwarp();
    const unsigned ml = __ballot_sync(0xffffffffu, L), mr = __ballot_sync(0xffffffffu, R);
    if (L) seg[nl + __popc(ml & lt)] = i;
    if (R) tr[nr + __popc(mr & lt)] = i;
    nl += __popc(ml);
    nr += __popc(mr);
  }
  __syncwarp();
  for (int j = lane; j < nr; j += 32) seg[nl + j] = tr[j];
  __syncwarp();
  return nl;
}

__device__ __forceinline__ uint32_t f32_key(float x) {   // order-preserving map of a float to uint32
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// ---- checks, presort -------------------------------------------------------------------------------------------------------
static __global__ void tree_check_kernel(const float* __restrict__ X, const double* __restrict__ y, int N, int D, int* __restrict__ bad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N && !isfinite(y[i])) atomicOr(bad, 1);
  if (i < (int64_t)N * D && !isfinite(X[i])) atomicOr(bad, 2);
}

// Column-major keys (e = f·N + i) and row indices of the presort, and its D + 1 segment offsets: the grid covers max(N·D, D + 1).
static __global__ void tree_keys_kernel(const float* __restrict__ X, int N, int D, uint32_t* __restrict__ keys, int* __restrict__ idx,
                                        int* __restrict__ seg) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e <= D) seg[e] = (int)e * N;
  if (e >= (int64_t)N * D) return;
  const int f = (int)(e / N), i = (int)(e % N);
  keys[e] = f32_key(X[(size_t)i * D + f]);
  idx[e] = i;
}

// ---- the sweeps' first-index argmax ------------------------------------------------------------------------------------------
// One thread's best candidate for each of up to three acquisitions, then its 256-thread CTA's, written to part[blockIdx.x·3 + q].
struct TreeArgmax {
  kbo_best b[3] = {{-INFINITY, INT64_MAX, 0.0, 0.0}, {-INFINITY, INT64_MAX, 0.0, 0.0}, {-INFINITY, INT64_MAX, 0.0, 0.0}};

  __device__ __forceinline__ void keep(int q, double v, int64_t m, double mu, double sd) {
    if (v > b[q].value) b[q] = kbo_best{v, m, mu, sd};   // indices only grow inside a thread: the first maximum stays
  }

  __device__ __forceinline__ void write(int n_acq, kbo_best* __restrict__ part) {
    if (n_acq == 0) return;
    __shared__ kbo_best sp[3][8];
    const int tid = threadIdx.x;
#pragma unroll
    for (int q = 0; q < 3; q++) {
      if (q >= n_acq) break;
      kbo_best x = b[q];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const kbo_best y{__shfl_xor_sync(0xffffffffu, x.value, o), __shfl_xor_sync(0xffffffffu, x.index, o),
                         __shfl_xor_sync(0xffffffffu, x.mu, o), __shfl_xor_sync(0xffffffffu, x.std, o)};
        if (better(y.value, y.index, x.value, x.index)) x = y;
      }
      if ((tid & 31) == 0) sp[q][tid >> 5] = x;
    }
    __syncthreads();
    if (tid < n_acq) {
      kbo_best x = sp[tid][0];
      for (int w = 1; w < 8; w++)
        if (better(sp[tid][w].value, sp[tid][w].index, x.value, x.index)) x = sp[tid][w];
      part[(size_t)blockIdx.x * 3 + tid] = x;
    }
  }
};

// The argmax across the sweep's nblocks CTAs: one warp per acquisition, global_offset added to the index.
static __global__ void tree_reduce_kernel(const kbo_best* __restrict__ part, int nblocks, int n_acq, int64_t goff, kbo_best* __restrict__ best) {
  const int q = blockIdx.x;
  kbo_best b{-INFINITY, INT64_MAX, 0.0, 0.0};
  for (int k = threadIdx.x; k < nblocks; k += 32) {
    const kbo_best& p = part[(size_t)k * 3 + q];
    if (better(p.value, p.index, b.value, b.index)) b = p;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const kbo_best y{__shfl_xor_sync(0xffffffffu, b.value, o), __shfl_xor_sync(0xffffffffu, b.index, o),
                     __shfl_xor_sync(0xffffffffu, b.mu, o), __shfl_xor_sync(0xffffffffu, b.std, o)};
    if (better(y.value, y.index, b.value, b.index)) b = y;
  }
  if (threadIdx.x == 0 && q < n_acq) {
    b.index += goff;
    best[q] = b;
  }
}

// ---- host plumbing; fn names the entry point and what the model in error messages ----------------------------------------------
// Fit prologue: (X, y) copied into t after the fit's first event, both checked finite (synchronises).
static int tree_fit_begin(kbo_handle* h, TreeCore* t, const float* X, const double* y, int N, int D, const char* fn, cudaStream_t s) {
  t->fitted = false;
  const size_t ND = (size_t)N * D;
  KBO_TRY(kbo_reserve(h, t->X, ND));
  KBO_TRY(kbo_reserve(h, t->y, (size_t)N));
  KBO_TRY(kbo_reserve(h, t->flag, 1));
  KBO_CUDA(h, cudaEventRecord(t->ev[0], s));
  KBO_CUDA(h, kbo_copy(t->X.p, X, ND, cudaMemcpyDeviceToDevice, s));
  KBO_CUDA(h, kbo_copy(t->y.p, y, (size_t)N, cudaMemcpyDeviceToDevice, s));
  KBO_CUDA(h, cudaMemsetAsync(t->flag.p, 0, sizeof *t->flag.p, s));
  tree_check_kernel<<<(unsigned)((ND + 255) / 256), 256, 0, s>>>(t->X.p, t->y.p, N, D, t->flag.p);
  KBO_LAUNCH_CHECK(h);
  int bad = 0;
  KBO_CUDA(h, kbo_copy(&bad, t->flag.p, 1, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (bad & 1) KBO_FAIL(h, KBO_ERR_INVALID, "%s: y contains NaN or infinity", fn);
  if (bad & 2) KBO_FAIL(h, KBO_ERR_INVALID, "%s: X contains NaN or infinity", fn);
  return KBO_OK;
}

// Presort every column of t->X once: stable segmented radix sort of (order-preserving key, row index) into t->order.
static int tree_presort(kbo_handle* h, TreeCore* t, int N, int D, cudaStream_t s) {
  const size_t ND = (size_t)N * D;
  KBO_TRY(kbo_reserve(h, t->keys, ND));
  KBO_TRY(kbo_reserve(h, t->keys2, ND));
  KBO_TRY(kbo_reserve(h, t->order_in, ND));
  KBO_TRY(kbo_reserve(h, t->order, ND));
  KBO_TRY(kbo_reserve(h, t->seg, (size_t)(D + 1)));
  size_t tb = 0;
  const int* seg = t->seg.p;
  KBO_CUDA(h, cub::DeviceSegmentedRadixSort::SortPairs(nullptr, tb, t->keys.p, t->keys2.p, t->order_in.p, t->order.p, (int)ND, D, seg,
                                                       seg + 1, 0, 32, s));
  KBO_TRY(kbo_reserve(h, t->sort_tmp, std::max<size_t>(tb, 16)));
  tree_keys_kernel<<<(unsigned)((std::max(ND, (size_t)D + 1) + 255) / 256), 256, 0, s>>>(t->X.p, N, D, t->keys.p, t->order_in.p, t->seg.p);
  KBO_LAUNCH_CHECK(h);
  KBO_CUDA(h, cub::DeviceSegmentedRadixSort::SortPairs(t->sort_tmp.p, tb, t->keys.p, t->keys2.p, t->order_in.p, t->order.p, (int)ND, D,
                                                       seg, seg + 1, 0, 32, s));
  return KBO_OK;
}

// Fit epilogue: the fit's last event, a synchronise (host copies made during the fit must land before it returns), its time.
static int tree_fit_end(kbo_handle* h, TreeCore* t, int N, int D, cudaStream_t s) {
  KBO_CUDA(h, cudaEventRecord(t->ev[1], s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  KBO_CUDA(h, cudaEventElapsedTime(&t->last_ms[0], t->ev[0], t->ev[1]));
  t->N = N;
  t->D = D;
  t->fitted = true;
  return KBO_OK;
}

// Sweep prologue: the arguments' checks, then the sweep's first event.
static int tree_sweep_begin(kbo_handle* h, TreeCore* t, int64_t M, int n_acq, const int32_t* acqs, double y_opt, const kbo_best* best_dev,
                            const char* fn, const char* what, cudaStream_t s) {
  if (!t->fitted) KBO_FAIL(h, KBO_ERR_STATE, "%s: %s is not fitted", fn, what);
  if (M < 1) KBO_FAIL(h, KBO_ERR_INVALID, "%s: M must be >= 1 (got %lld)", fn, (long long)M);
  if (n_acq < 0 || n_acq > 3 || (n_acq > 0 && (!acqs || !best_dev))) KBO_FAIL(h, KBO_ERR_INVALID, "%s: 0 <= n_acq <= 3 with acqs and best_dev", fn);
  for (int i = 0; i < n_acq; i++) {
    if (acqs[i] < KBO_ACQ_EI || acqs[i] > KBO_ACQ_PI) KBO_FAIL(h, KBO_ERR_INVALID, "%s: unknown acquisition %d", fn, acqs[i]);
    for (int j = 0; j < i; j++)
      if (acqs[j] == acqs[i]) KBO_FAIL(h, KBO_ERR_INVALID, "%s: acquisition %d given twice", fn, acqs[i]);
  }
  if (!std::isfinite(y_opt)) KBO_FAIL(h, KBO_ERR_INVALID, "%s: y_opt must be finite", fn);
  KBO_CUDA(h, cudaSetDevice(h->device));
  KBO_CUDA(h, cudaEventRecord(t->ev[2], s));
  return KBO_OK;
}

// Sweep epilogue: the argmax across the nblocks CTAs of the sweep kernel into best_dev, then the sweep's last event.
static int tree_sweep_end(kbo_handle* h, TreeCore* t, int nblocks, int n_acq, int64_t goff, kbo_best* best_dev, cudaStream_t s) {
  if (n_acq > 0) {
    tree_reduce_kernel<<<n_acq, 32, 0, s>>>(t->part.p, nblocks, n_acq, goff, best_dev);
    KBO_LAUNCH_CHECK(h);
  }
  KBO_CUDA(h, cudaEventRecord(t->ev[3], s));
  return KBO_OK;
}

// Predict prologue: the n rows of X on the device, as given or (x_on_host) copied into the handle's staging buffer.
static int tree_predict_rows(kbo_handle* h, const TreeCore* t, const float* X, int n, int x_on_host, const float** Xd, const char* fn,
                             const char* what, cudaStream_t s) {
  if (!t->fitted) KBO_FAIL(h, KBO_ERR_STATE, "%s: %s is not fitted", fn, what);
  KBO_CUDA(h, cudaSetDevice(h->device));
  *Xd = X;
  if (x_on_host) {
    const size_t bytes = (size_t)n * t->D * sizeof(float);
    KBO_TRY(kbo_reserve(h, h->stage_Xc, bytes));
    KBO_CUDA(h, cudaMemcpyAsync(h->stage_Xc.p, X, bytes, cudaMemcpyHostToDevice, s));
    *Xd = kbo_view<float>(h->stage_Xc);
  }
  return KBO_OK;
}

// kbo_<kind>_last_timings: the last fit's and the last finished sweep's milliseconds.
static int tree_last_timings(kbo_handle* h, TreeCore* t, float* ms, int32_t n) {
  if (!h || !t) return KBO_ERR_INVALID;
  float sweep = 0.f;
  if (cudaEventQuery(t->ev[3]) == cudaSuccess && cudaEventElapsedTime(&sweep, t->ev[2], t->ev[3]) == cudaSuccess) t->last_ms[1] = sweep;
  cudaGetLastError();
  for (int i = 0; ms && i < n && i < 2; i++) ms[i] = t->last_ms[i];
  return 2;
}
