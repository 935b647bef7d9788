// skopt's GBRT surrogate of Katib's `bayesianoptimization`: GradientBoostingQuantileRegressor, three quantile-loss boosting chains
// (GradientBoostingRegressor(loss="quantile", n_estimators=30), trees of depth <= 3, learning rate 0.1), fitted and swept on the
// device.  FP64 NumPy restatement: oracle/gbrt_oracle.py, which cites the scikit-learn 1.9.0 sources line by line.
//
// Fit (gbrt_fit_kernel): one CTA per chain, the three chains at once, every stage on the device with no host round trip.
//   Init: np.percentile(y, 100·α), NumPy's linear rule, from y sorted once (gbrt_init_kernel).
//   X is presorted once per fit (a stable segmented radix sort of each column), shared by every chain and stage.  Each stage
//   copies that order into the chain's columns and splits breadth-first, nodes in heap slots (children of k are 2k+1, 2k+2),
//   stably partitioning every column's node segment so every segment stays sorted.
//   Split search: every gradient is α or α − 1, so sklearn's proxy ranks splits as (pl²·nr + pr²·nl) / (nl·nr) does, pl / pr the
//   rows with y >= raw going left / right.  A warp owns a feature and scans its segment 32 rows at a time: one ballot of the
//   y >= raw bits, a popc prefix gives pl at every position, and the scores are compared exactly by cross-multiplying in 128-bit
//   integers.  Ties go to the lowest position, then the lowest feature.  A split after sorted position p is valid where
//   v[p+1] > fl32(v[p] + 1e-7); the threshold is v[p]/2 + v[p+1]/2 in FP64, v[p] where that rounds to v[p+1] or overflows.
//   A node is a leaf at depth 3, below 2 rows, when it is pure (no row or every row with y >= raw) or has no valid split.
//   Leaf value: the k-th smallest residual fl(y − raw) of the leaf, k = ceil(t) − 1, t = fl(fl(fl(100·α)/100)·n) (sklearn's
//   _weighted_percentile with unit weights), by an 8-pass radix select on order-preserving 64-bit keys.
//   Raw update: raw += fl(0.1·value), __dmul_rn then __dadd_rn.
// Sweep (gbrt_sweep_kernel): the whole model (3 × stages trees of 15 heap slots: 8-byte nodes whose threshold is RD_f32 of the
// FP64 one — for float32 x, x <= t  <=>  x <= RD_f32(t) — and the leaves' fl(0.1·value)) is staged in shared memory once per
// CTA, and a tile of 256 candidate rows with it where they fit, so each tree's gather of a feature reads shared memory.  Each
// chain sums from its init in stage order with __dadd_rn; μ = chain(0.5), σ = fl(chain(hi) − chain(lo)) / 2 (negative where the
// quantiles cross), then EI / LCB / PI (kbo_acq.cuh) and a first-index argmax per acquisition.
#include <float.h>
#include <math.h>
#include <algorithm>
#include <vector>

#include <cub/device/device_radix_sort.cuh>

#include "kbo_tree.cuh"

#define GBRT_FIT_THREADS 1024
#define GBRT_CHAINS 3
#define GBRT_SLOTS 15          // heap slots of a tree of depth <= 3
#define GBRT_DEPTH 3
#define GBRT_LEAF 0xFFFFFFFFu
#define GBRT_MAX_N 65536
#define GBRT_MAX_D 1024
#define GBRT_MAX_STAGES 128

struct kbo_gbrt : TreeCore {
  int S = 30;
  double alpha[GBRT_CHAINS] = {0.16, 0.5, 0.84};
  DevBuf<double> ysort, raw, alpha_dev, init;
  DevBuf<int> cols, tmp;
  DevBuf<unsigned char> pos, side, leaf, ysort_tmp;
  DevBuf<unsigned long long> rkey;
  // per (chain, stage, slot): the tree in heap layout (export) and the packed model (sweep)
  DevBuf<int> feat, nn, np_;
  DevBuf<double> thr, value, mval;
  DevBuf<uint2> mnode;
  double h_init[GBRT_CHAINS] = {0.0, 0.0, 0.0};
};

__device__ __forceinline__ unsigned long long gbrt_f64_key(double x) {   // order-preserving, -0.0 taken as +0.0
  const unsigned long long u = (unsigned long long)__double_as_longlong(x == 0.0 ? 0.0 : x);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double gbrt_key_f64(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k));
}

// ---- init -------------------------------------------------------------------------------------------------------------------
// np.percentile(y, 100·α) with the linear rule (numpy/lib/_function_base_impl.py _quantile / _lerp): virtual index (n − 1)·q,
// q = fl(100·α) / 100; γ its fractional part; a + (b − a)·γ, or b − (b − a)·(1 − γ) where γ >= 0.5; the last value past n − 1.
__global__ void gbrt_init_kernel(const double* __restrict__ ys, int N, const double* __restrict__ alpha, double* __restrict__ init) {
  const int c = threadIdx.x;
  if (c >= GBRT_CHAINS) return;
  const double q = __ddiv_rn(__dmul_rn(100.0, alpha[c]), 100.0);
  const double v = __dmul_rn((double)(N - 1), q);
  if (v >= (double)(N - 1)) {
    init[c] = ys[N - 1];
    return;
  }
  const double lo = floor(v);
  const int i = (int)lo;
  const double g = __dadd_rn(v, -lo);
  const double a = ys[i], b = ys[i + 1];
  const double d = __dadd_rn(b, -a);
  init[c] = g >= 0.5 ? __dadd_rn(b, -__dmul_rn(d, __dadd_rn(1.0, -g))) : __dadd_rn(a, __dmul_rn(d, g));
}

// ---- fit --------------------------------------------------------------------------------------------------------------------
struct GbrtFitArgs {
  const float* X;
  const double* y;
  const int* order;       // D × N presorted row indices
  const double* alpha;    // 3
  const double* init;     // 3
  int N, D, S;
  int* cols;              // per chain D × N
  int* tmp;
  unsigned char* pos;     // per chain N: y >= raw
  unsigned char* side;
  unsigned char* leaf;    // per chain N: heap slot of each row's leaf
  unsigned long long* rkey;   // per chain N: residual keys in column-0 order
  double* raw;            // per chain N
  int* feat;              // per (chain, stage) 15 slots: -2 leaf, -3 unused
  double* thr;
  double* value;
  int* nn;
  int* np_;
  uint2* mnode;
  double* mval;
};

struct GbrtSplit {
  unsigned long long num, den;   // den == 0: no split
  int feat, nl;
  double thr;
};

__device__ __forceinline__ bool gbrt_gt(unsigned long long n1, unsigned long long d1, unsigned long long n2, unsigned long long d2) {
  if (d1 == 0) return false;
  if (d2 == 0) return true;
  return (unsigned __int128)n1 * d2 > (unsigned __int128)n2 * d1;
}

__global__ void __launch_bounds__(GBRT_FIT_THREADS, 1) gbrt_fit_kernel(GbrtFitArgs a) {
  const int ch = blockIdx.x, N = a.N, D = a.D;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const size_t ND = (size_t)N * D;
  int* cols = a.cols + (size_t)ch * ND;
  int* tmp = a.tmp + (size_t)ch * ND;
  unsigned char* pos = a.pos + (size_t)ch * N;
  unsigned char* side = a.side + (size_t)ch * N;
  unsigned char* leaf = a.leaf + (size_t)ch * N;
  unsigned long long* rkey = a.rkey + (size_t)ch * N;
  double* raw = a.raw + (size_t)ch * N;
  const float* __restrict__ X = a.X;
  const double* __restrict__ y = a.y;
  const double alpha = a.alpha[ch], u = __dadd_rn(1.0, -alpha);
  const double prank = __ddiv_rn(__dmul_rn(100.0, alpha), 100.0);

  __shared__ int s_start[GBRT_SLOTS], s_end[GBRT_SLOTS], s_state[GBRT_SLOTS];   // state: 0 unused, 1 split, 2 leaf
  __shared__ double s_val[GBRT_SLOTS];
  __shared__ GbrtSplit s_best[32];
  __shared__ GbrtSplit s_win;
  __shared__ int s_hist[256];
  __shared__ int s_rank;
  __shared__ unsigned long long s_prefix;

  for (int i = tid; i < N; i += blockDim.x) raw[i] = a.init[ch];
  for (int st = 0; st < a.S; st++) {
    const size_t ob = ((size_t)ch * a.S + st) * GBRT_SLOTS;
    __syncthreads();
    for (int i = tid; i < N; i += blockDim.x) pos[i] = y[i] >= raw[i] ? 1 : 0;
    for (size_t e = tid; e < ND; e += blockDim.x) cols[e] = a.order[e];
    if (tid < GBRT_SLOTS) {
      s_state[tid] = 0;
      s_val[tid] = 0.0;
    }
    if (tid == 0) {
      s_start[0] = 0;
      s_end[0] = N;
      s_state[0] = 1;
    }
    __syncthreads();
    for (int k = 0; k < GBRT_SLOTS; k++) {
      if (s_state[k] == 0) {   // below a leaf
        if (tid == 0) {
          a.feat[ob + k] = -3;
          a.thr[ob + k] = -2.0;
          a.value[ob + k] = 0.0;
          a.nn[ob + k] = 0;
          a.np_[ob + k] = 0;
          a.mnode[ob + k] = make_uint2(0u, GBRT_LEAF);
          a.mval[ob + k] = 0.0;
        }
        continue;
      }
      const int s = s_start[k], e = s_end[k], c = e - s;
      const int depth = k < 1 ? 0 : k < 3 ? 1 : k < 7 ? 2 : 3;
      int P = 0;
      for (int j0 = 0; j0 < c; j0 += blockDim.x) {
        const int j = j0 + tid;
        P += __syncthreads_count(j < c && pos[cols[s + j]]);
      }
      bool is_leaf = depth >= GBRT_DEPTH || c < 2 || P == 0 || P == c;
      if (!is_leaf) {
        GbrtSplit best{0ull, 0ull, 0x7fffffff, 0, 0.0};
        for (int f = warp; f < D; f += 32) {
          const int* col = cols + (size_t)f * N + s;
          int before = 0;   // rows with y >= raw in the chunks already scanned
          for (int j0 = 0; j0 < c; j0 += 32) {
            const int j = j0 + lane;
            const bool valid = j < c;
            const int i = valid ? col[j] : 0;
            const float v = valid ? X[(size_t)i * D + f] : 0.f;
            const unsigned m = __ballot_sync(0xffffffffu, valid && pos[i]);
            const int pl = before + __popc(m << (31 - lane));
            float vn = __shfl_down_sync(0xffffffffu, v, 1);
            if (lane == 31 && j + 1 < c) vn = X[(size_t)col[j + 1] * D + f];
            const int nl = j + 1, nr = c - nl, pr = P - pl;
            const bool cand = valid && j + 1 < c && !(vn <= __fadd_rn(v, 1e-7f));
            unsigned long long num = 0ull, den = 0ull;
            if (cand) {
              num = (unsigned long long)pl * pl * nr + (unsigned long long)pr * pr * nl;
              den = (unsigned long long)nl * nr;
            }
            // first maximum of the chunk
            unsigned long long bn = num, bd = den;
            int bl = lane;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
              const unsigned long long on = __shfl_xor_sync(0xffffffffu, bn, o), od = __shfl_xor_sync(0xffffffffu, bd, o);
              const int ol = __shfl_xor_sync(0xffffffffu, bl, o);
              const bool take = gbrt_gt(on, od, bn, bd) || (!gbrt_gt(bn, bd, on, od) && od != 0 && ol < bl);
              if (take) {
                bn = on;
                bd = od;
                bl = ol;
              }
            }
            if (gbrt_gt(bn, bd, best.num, best.den)) {
              const float va = __shfl_sync(0xffffffffu, v, bl), vb = __shfl_sync(0xffffffffu, vn, bl);
              double th = (double)va / 2.0 + (double)vb / 2.0;
              if (th == (double)vb || isinf(th)) th = (double)va;
              best = GbrtSplit{bn, bd, f, j0 + bl + 1, th};
            }
            before += __popc(m);
          }
        }
        if (lane == 0) s_best[warp] = best;
        __syncthreads();
        if (tid == 0) {
          GbrtSplit b = s_best[0];
          for (int w = 1; w < 32; w++) {
            const GbrtSplit& o = s_best[w];
            if (gbrt_gt(o.num, o.den, b.num, b.den) || (o.den != 0 && !gbrt_gt(b.num, b.den, o.num, o.den) && o.feat < b.feat)) b = o;
          }
          s_win = b;
        }
        __syncthreads();
        is_leaf = s_win.den == 0;   // no valid split
      }
      if (is_leaf) {
        if (tid == 0) s_state[k] = 2;
        continue;   // its value comes with the other leaves'
      }
      const GbrtSplit w = s_win;
      const int* wcol = cols + (size_t)w.feat * N + s;
      for (int j = tid; j < c; j += blockDim.x) side[wcol[j]] = j < w.nl ? 1 : 0;
      __syncthreads();
      for (int f = warp; f < D; f += 32)
        if (f != w.feat) warp_partition(cols + (size_t)f * N + s, tmp + (size_t)f * N + s, c, [&](int i) { return side[i] != 0; });
      if (tid == 0) {
        a.feat[ob + k] = w.feat;
        a.thr[ob + k] = w.thr;
        a.value[ob + k] = __ddiv_rn(__dadd_rn(__dmul_rn((double)P, alpha), -__dmul_rn((double)(c - P), u)), (double)c);
        a.nn[ob + k] = c;
        a.np_[ob + k] = P;
        a.mnode[ob + k] = make_uint2(__float_as_uint(__double2float_rd(w.thr)), (uint32_t)w.feat);
        a.mval[ob + k] = 0.0;
        s_state[k] = 1;
        s_start[2 * k + 1] = s;
        s_end[2 * k + 1] = s + w.nl;
        s_start[2 * k + 2] = s + w.nl;
        s_end[2 * k + 2] = e;
        s_state[2 * k + 1] = s_state[2 * k + 2] = 1;
      }
      __syncthreads();
    }
    // leaves: the residual percentile by radix select over the leaf's rows (column 0 holds every node's rows contiguously)
    for (int k = 0; k < GBRT_SLOTS; k++) {
      __syncthreads();
      if (s_state[k] != 2) continue;
      const int s = s_start[k], c = s_end[k] - s;
      for (int j = tid; j < c; j += blockDim.x) {
        const int i = cols[s + j];
        leaf[i] = (unsigned char)k;
        rkey[s + j] = gbrt_f64_key(__dadd_rn(y[i], -raw[i]));
      }
      if (tid == 0) {
        double t = __dmul_rn(prank, (double)c);
        if (t == 0.0) t = __longlong_as_double(1ll);   // nextafter(0, 1)
        int r = (int)ceil(t) - 1;
        s_rank = r < 0 ? 0 : r > c - 1 ? c - 1 : r;
        s_prefix = 0ull;
      }
      unsigned long long mask = 0ull;
      for (int sh = 56; sh >= 0; sh -= 8) {
        if (tid < 256) s_hist[tid] = 0;
        __syncthreads();
        const unsigned long long pre = s_prefix;
        for (int j = tid; j < c; j += blockDim.x) {
          const unsigned long long key = rkey[s + j];
          if ((key & mask) == pre) atomicAdd(&s_hist[(int)((key >> sh) & 255ull)], 1);
        }
        __syncthreads();
        if (tid == 0) {
          int r = s_rank, b = 0;
          while (s_hist[b] <= r) r -= s_hist[b++];
          s_rank = r;
          s_prefix = pre | ((unsigned long long)b << sh);
        }
        mask |= 255ull << sh;
        __syncthreads();
      }
      int P = 0;
      for (int j0 = 0; j0 < c; j0 += blockDim.x) {
        const int j = j0 + tid;
        P += __syncthreads_count(j < c && pos[cols[s + j]]);
      }
      if (tid == 0) {
        const double v = gbrt_key_f64(s_prefix);
        s_val[k] = v;
        a.feat[ob + k] = -2;
        a.thr[ob + k] = -2.0;
        a.value[ob + k] = v;
        a.nn[ob + k] = c;
        a.np_[ob + k] = P;
        a.mnode[ob + k] = make_uint2(0u, GBRT_LEAF);
        a.mval[ob + k] = __dmul_rn(0.1, v);
      }
    }
    __syncthreads();
    for (int i = tid; i < N; i += blockDim.x) raw[i] = __dadd_rn(raw[i], __dmul_rn(0.1, s_val[leaf[i]]));
  }
}

// ---- sweep ------------------------------------------------------------------------------------------------------------------
struct GbrtSweepArgs {
  const uint2* mnode;    // 3 × S × 15
  const double* mval;
  const double* init;
  int S;
  const float* Xc;
  int64_t M;
  int D, ld;             // ld: row pitch of the staged tile (D rounded up to odd)
  int n_acq, acq0, acq1, acq2;
  double yopt, xi, kappa;
  double* mu_out;
  double* sd_out;
  double* q_out;         // 3 × M chain predictions
  kbo_best* part;
};

// ACQ = false (predict): the chain sums alone, so the instance's SASS shows they are never contracted into a DFMA.
template <bool STAGE_X, bool ACQ>
__global__ void __launch_bounds__(256) gbrt_sweep_kernel(GbrtSweepArgs a) {
  extern __shared__ double2 gsm[];
  const int tid = threadIdx.x;
  const int nslots = GBRT_CHAINS * a.S * GBRT_SLOTS;
  double* vals = reinterpret_cast<double*>(gsm);
  uint2* nodes = reinterpret_cast<uint2*>(vals + nslots);
  float* xs = reinterpret_cast<float*>(nodes + nslots);
  for (int i = tid; i < nslots; i += 256) {
    vals[i] = a.mval[i];
    nodes[i] = a.mnode[i];
  }
  const double init0 = a.init[0], init1 = a.init[1], init2 = a.init[2];
  TreeArgmax best;
  const int acqs[3] = {a.acq0, a.acq1, a.acq2};
  const int64_t ntiles = (a.M + 255) / 256;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t m0 = tile * 256, m = m0 + tid;
    const float* row;
    if (STAGE_X) {
      __syncthreads();
      const int64_t nrow = a.M - m0 < 256 ? a.M - m0 : 256;
      for (int e = tid; e < (int)nrow * a.D; e += 256) {
        const int r = e / a.D, f = e - r * a.D;
        xs[r * a.ld + f] = __ldg(a.Xc + (size_t)m0 * a.D + e);
      }
      __syncthreads();
      row = xs + tid * a.ld;
    } else {
      row = a.Xc + (size_t)(m < a.M ? m : 0) * a.D;
    }
    if (m >= a.M) continue;
    double q[3] = {init0, init1, init2};
#pragma unroll
    for (int c = 0; c < GBRT_CHAINS; c++) {
      const int base0 = c * a.S * GBRT_SLOTS;
      for (int st = 0; st < a.S; st++) {
        const int base = base0 + st * GBRT_SLOTS;
        int k = 0;
        uint2 nd = nodes[base];
        while (nd.y != GBRT_LEAF) {
          const float x = STAGE_X ? row[nd.y] : __ldg(row + nd.y);
          k = 2 * k + (x <= __uint_as_float(nd.x) ? 1 : 2);
          nd = nodes[base + k];
        }
        q[c] = __dadd_rn(q[c], vals[base + k]);
      }
    }
    const double mu = q[1];
    const double sd = __dmul_rn(__dadd_rn(q[2], -q[0]), 0.5);
    if (a.mu_out) a.mu_out[m] = mu;
    if (a.sd_out) a.sd_out[m] = sd;
    if (a.q_out) {
      a.q_out[m] = q[0];
      a.q_out[a.M + m] = q[1];
      a.q_out[2 * a.M + m] = q[2];
    }
    if constexpr (ACQ) {
#pragma unroll
      for (int qq = 0; qq < 3; qq++) {
        if (qq >= a.n_acq) break;
        best.keep(qq, acq_of_sd<double>(mu, sd, acqs[qq], a.yopt, a.xi, a.kappa), m, mu, sd);
      }
    }
  }
  if constexpr (ACQ) best.write(a.n_acq, a.part);
}

// ---- C ABI ------------------------------------------------------------------------------------------------------------------
static int gbrt_sweep_launch(kbo_handle* h, kbo_gbrt* g, const float* Xc, int64_t M, int n_acq, const int32_t* acqs, double yopt, double xi,
                             double kappa, double* mu_out, double* sd_out, double* q_out, int* nblocks_out, cudaStream_t s) {
  const int ld = g->D | 1;   // an odd pitch: the 32 rows a warp reads hit 32 different banks
  const size_t model = (size_t)GBRT_CHAINS * g->S * GBRT_SLOTS * (sizeof(double) + sizeof(uint2));
  const size_t tile = (size_t)256 * ld * sizeof(float);
  const bool stage = model + tile <= 113 * 1024;
  const size_t smem = stage ? model + tile : model;
  GbrtSweepArgs a{g->mnode.p, g->mval.p, g->init.p, g->S, Xc, M, g->D, ld, n_acq,
                  n_acq > 0 ? acqs[0] : 0, n_acq > 1 ? acqs[1] : 0, n_acq > 2 ? acqs[2] : 0, yopt, xi, kappa, mu_out, sd_out, q_out, nullptr};
  void (*k)(GbrtSweepArgs) = stage ? (n_acq > 0 ? gbrt_sweep_kernel<true, true> : gbrt_sweep_kernel<true, false>)
                                   : (n_acq > 0 ? gbrt_sweep_kernel<false, true> : gbrt_sweep_kernel<false, false>);
  int occ = 0;
  KBO_CUDA(h, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  KBO_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, 256, smem));
  const int64_t ntiles = (M + 255) / 256;
  const int nb = (int)std::min<int64_t>(ntiles, (int64_t)h->sm_count * std::max(occ, 1));
  KBO_TRY(kbo_reserve(h, g->part, (size_t)nb * 3));
  a.part = g->part.p;
  k<<<nb, 256, smem, s>>>(a);
  KBO_LAUNCH_CHECK(h);
  *nblocks_out = nb;
  return KBO_OK;
}

extern "C" {

int kbo_gbrt_create(kbo_handle* h, kbo_gbrt** out, const double* quantiles, int32_t n_estimators) {
  if (!h || !out) return KBO_ERR_INVALID;
  *out = nullptr;
  if (n_estimators < 1 || n_estimators > GBRT_MAX_STAGES)
    KBO_FAIL(h, KBO_ERR_INVALID, "kbo_gbrt_create: 1 <= n_estimators <= %d (got %d)", GBRT_MAX_STAGES, n_estimators);
  if (quantiles) {
    for (int c = 0; c < GBRT_CHAINS; c++)
      if (!(quantiles[c] > 0.0 && quantiles[c] < 1.0)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_gbrt_create: quantiles must lie in (0, 1)");
    if (!(quantiles[0] < quantiles[1] && quantiles[1] < quantiles[2]))
      KBO_FAIL(h, KBO_ERR_INVALID, "kbo_gbrt_create: quantiles must be increasing (lower, middle, upper)");
  }
  KBO_CUDA(h, cudaSetDevice(h->device));
  std::unique_ptr<kbo_gbrt> g(new (std::nothrow) kbo_gbrt());
  if (!g) return KBO_ERR_NOMEM;
  g->S = n_estimators;
  if (quantiles)
    for (int c = 0; c < GBRT_CHAINS; c++) g->alpha[c] = quantiles[c];
  KBO_TRY(kbo_upload(h, g->alpha_dev, g->alpha, GBRT_CHAINS));
  KBO_TRY(g->ev.create());
  *out = g.release();
  return KBO_OK;
}

void kbo_gbrt_destroy(kbo_gbrt* g) {
  if (g) delete g;
}

int kbo_gbrt_fit(kbo_handle* h, kbo_gbrt* g, const float* X, const double* y, int32_t N, int32_t D, void* stream) {
  if (!h || !g || !X || !y) return KBO_ERR_INVALID;
  if (N < 1 || N > GBRT_MAX_N) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_gbrt_fit: 1 <= N <= %d (got %d)", GBRT_MAX_N, N);
  if (D < 1 || D > GBRT_MAX_D) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_gbrt_fit: 1 <= D <= %d (got %d)", GBRT_MAX_D, D);
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  KBO_TRY(tree_fit_begin(h, g, X, y, N, D, "kbo_gbrt_fit", s));
  const size_t ND = (size_t)N * D;
  // init: y sorted once, the linear percentile per chain
  KBO_TRY(kbo_reserve(h, g->ysort, (size_t)N));
  KBO_TRY(kbo_reserve(h, g->init, GBRT_CHAINS));
  size_t tb = 0;
  KBO_CUDA(h, cub::DeviceRadixSort::SortKeys(nullptr, tb, g->y.p, g->ysort.p, N, 0, 64, s));
  KBO_TRY(kbo_reserve(h, g->ysort_tmp, std::max<size_t>(tb, 16)));
  KBO_CUDA(h, cub::DeviceRadixSort::SortKeys(g->ysort_tmp.p, tb, g->y.p, g->ysort.p, N, 0, 64, s));
  gbrt_init_kernel<<<1, 32, 0, s>>>(g->ysort.p, N, g->alpha_dev.p, g->init.p);
  KBO_LAUNCH_CHECK(h);
  KBO_TRY(tree_presort(h, g, N, D, s));
  const size_t C = GBRT_CHAINS, TS = C * g->S * GBRT_SLOTS;
  KBO_TRY(kbo_reserve(h, g->cols, C * ND));
  KBO_TRY(kbo_reserve(h, g->tmp, C * ND));
  KBO_TRY(kbo_reserve(h, g->pos, C * N));
  KBO_TRY(kbo_reserve(h, g->side, C * N));
  KBO_TRY(kbo_reserve(h, g->leaf, C * N));
  KBO_TRY(kbo_reserve(h, g->rkey, C * N));
  KBO_TRY(kbo_reserve(h, g->raw, C * N));
  KBO_TRY(kbo_reserve(h, g->feat, TS));
  KBO_TRY(kbo_reserve(h, g->thr, TS));
  KBO_TRY(kbo_reserve(h, g->value, TS));
  KBO_TRY(kbo_reserve(h, g->nn, TS));
  KBO_TRY(kbo_reserve(h, g->np_, TS));
  KBO_TRY(kbo_reserve(h, g->mnode, TS));
  KBO_TRY(kbo_reserve(h, g->mval, TS));
  GbrtFitArgs a{g->X.p, g->y.p, g->order.p, g->alpha_dev.p, g->init.p, N, D, g->S, g->cols.p, g->tmp.p, g->pos.p, g->side.p, g->leaf.p,
                g->rkey.p, g->raw.p, g->feat.p, g->thr.p, g->value.p, g->nn.p, g->np_.p, g->mnode.p, g->mval.p};
  gbrt_fit_kernel<<<GBRT_CHAINS, GBRT_FIT_THREADS, 0, s>>>(a);
  KBO_LAUNCH_CHECK(h);
  KBO_CUDA(h, kbo_copy(g->h_init, g->init.p, GBRT_CHAINS, cudaMemcpyDeviceToHost, s));
  return tree_fit_end(h, g, N, D, s);
}

int kbo_gbrt_sweep(kbo_handle* h, kbo_gbrt* g, const float* Xc, int64_t M, int64_t global_offset, int32_t n_acq, const int32_t* acqs, double y_opt,
                   double xi, double kappa, kbo_best* best_dev, double* mu_out, double* sigma_out, double* quantiles_out, void* stream) {
  if (!h || !g || !Xc) return KBO_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  KBO_TRY(tree_sweep_begin(h, g, M, n_acq, acqs, y_opt, best_dev, "kbo_gbrt_sweep", "the model", s));
  int nb = 0;
  KBO_TRY(gbrt_sweep_launch(h, g, Xc, M, n_acq, acqs, y_opt, xi, kappa, mu_out, sigma_out, quantiles_out, &nb, s));
  return tree_sweep_end(h, g, nb, n_acq, global_offset, best_dev, s);
}

int kbo_gbrt_predict(kbo_handle* h, kbo_gbrt* g, const float* X, int32_t n, int x_on_host, double* mu_host, double* sigma_host,
                     double* quantiles_host, void* stream) {
  if (!h || !g || !X || n < 1) return KBO_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  const float* Xd = nullptr;
  KBO_TRY(tree_predict_rows(h, g, X, n, x_on_host, &Xd, "kbo_gbrt_predict", "the model", s));
  KBO_TRY(kbo_reserve(h, h->stage_y, (size_t)n * 5));
  double* mu = h->stage_y.p;
  int nb = 0;
  KBO_TRY(gbrt_sweep_launch(h, g, Xd, n, 0, nullptr, 0.0, 0.0, 0.0, mu, mu + n, mu + 2 * (size_t)n, &nb, s));
  KBO_CUDA(h, kbo_d2h(mu_host, mu, n, s));
  KBO_CUDA(h, kbo_d2h(sigma_host, mu + n, n, s));
  KBO_CUDA(h, kbo_d2h(quantiles_host, mu + 2 * (size_t)n, 3 * (size_t)n, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  return KBO_OK;
}

int kbo_gbrt_export(kbo_handle* h, kbo_gbrt* g, int32_t chain, int32_t stage, int32_t* feature, double* threshold, int32_t* left, int32_t* right,
                    double* value, int32_t* n_node_samples, int32_t* n_pos, int32_t cap, int32_t* n_nodes, double* init, void* stream) {
  if (!h || !g) return KBO_ERR_INVALID;
  if (!g->fitted) KBO_FAIL(h, KBO_ERR_STATE, "kbo_gbrt_export: the model is not fitted");
  if (chain < 0 || chain >= GBRT_CHAINS) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_gbrt_export: chain %d out of range [0, %d)", chain, GBRT_CHAINS);
  if (stage < 0 || stage >= g->S) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_gbrt_export: stage %d out of range [0, %d)", stage, g->S);
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  const size_t ob = ((size_t)chain * g->S + stage) * GBRT_SLOTS;
  int hf[GBRT_SLOTS], hn[GBRT_SLOTS], hp[GBRT_SLOTS];
  double ht[GBRT_SLOTS], hv[GBRT_SLOTS];
  KBO_CUDA(h, kbo_copy(hf, g->feat.p + ob, GBRT_SLOTS, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, kbo_copy(ht, g->thr.p + ob, GBRT_SLOTS, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, kbo_copy(hv, g->value.p + ob, GBRT_SLOTS, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, kbo_copy(hn, g->nn.p + ob, GBRT_SLOTS, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, kbo_copy(hp, g->np_.p + ob, GBRT_SLOTS, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (init) *init = g->h_init[chain];
  // heap slots to sklearn's depth-first preorder, left first
  int id[GBRT_SLOTS], slot[GBRT_SLOTS], n = 0, stack[GBRT_SLOTS], sp = 0;
  stack[sp++] = 0;
  while (sp) {
    const int k = stack[--sp];
    id[k] = n;
    slot[n++] = k;
    if (hf[k] >= 0) {
      stack[sp++] = 2 * k + 2;
      stack[sp++] = 2 * k + 1;
    }
  }
  if (n_nodes) *n_nodes = n;
  if (cap < n) return KBO_OK;   // size query
  for (int j = 0; j < n; j++) {
    const int k = slot[j];
    const bool inner = hf[k] >= 0;
    if (feature) feature[j] = inner ? hf[k] : -2;
    if (threshold) threshold[j] = inner ? ht[k] : -2.0;
    if (left) left[j] = inner ? id[2 * k + 1] : -1;
    if (right) right[j] = inner ? id[2 * k + 2] : -1;
    if (value) value[j] = hv[k];
    if (n_node_samples) n_node_samples[j] = hn[k];
    if (n_pos) n_pos[j] = hp[k];
  }
  return KBO_OK;
}

int kbo_gbrt_last_timings(kbo_handle* h, kbo_gbrt* g, float* ms, int32_t n) { return tree_last_timings(h, g, ms, n); }

}  // extern "C"
