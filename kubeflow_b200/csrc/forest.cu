// Tree-ensemble surrogates of Katib's `bayesianoptimization` with base_estimator RF / ET: skopt's cook_estimator forests
// (RandomForestRegressor / ExtraTreesRegressor, 100 trees, min_samples_leaf = 3), fitted and swept on the device.  FP64 NumPy
// restatement: oracle/forest_oracle.py, which cites the scikit-learn 1.9.0 sources ($SKT = sklearn/tree) line by line.
//
// Fit (forest_fit_kernel): one CTA per tree, every tree of a batch at once, no host round trip per node or level.  Nodes are
// split in breadth-first order (node k's children get the next two ids, left first) from a FIFO the CTA walks.
//   RF: X is presorted once per forest (a stable segmented radix sort of each column); each tree compacts the columns to its
//       in-bag samples, and every split stably partitions each column's node segment, so every segment stays sorted.  A warp
//       owns a feature and scans the segment with warp prefix sums of (w, w·y): the split after sorted position p is valid
//       where v[p+1] > fl32(v[p] + 1e-7) ($SKT/_partitioner.pyx:210-213, FEATURE_THRESHOLD is a float32) and both sides keep
//       min_samples_leaf DISTINCT samples; the proxy is sum_l²/w_l + sum_r²/w_r ($SKT/_criterion.pyx:944-973), the threshold
//       v[p]/2 + v[p+1]/2 in FP64, or v[p] when that rounds to v[p+1] or overflows ($SKT/_splitter.pyx:~455-465).
//   ET: a warp owns a feature: min / max over the node (float32), skip if max <= fl32(min + 1e-7), threshold = (max − min)·u + min
//       with u a Philox 53-bit uniform keyed (seed, tree, node, feature), min where it equals max ($SKT/_splitter.pyx:616-655);
//       then the left count and (w, w·y) sums of x <= threshold.
//   Both: within a feature the first (lowest-threshold) maximum of the proxy wins, across features the lowest feature index.
//   A node is a leaf when it holds fewer than 2·min_samples_leaf samples or its impurity is <= DBL_EPSILON ($SKT/_tree.pyx:230-251).
//   Leaf value = Σw·y / Σw, impurity = Σ(w·y)·y / Σw − value² (MSE.node_impurity, $SKT/_criterion.pyx:938-940).
//   Bootstrap (RF): draw d of tree t is sample (u32·N) >> 32, u32 = Philox4x32-10(counter (d, t, 0, 0), key seed)[0]; the
//   draw counts are the sample weights, as sklearn's forest passes them ($SK-ensemble/_forest.py _parallel_build_trees).
// Sweep (forest_sweep_kernel): candidates in blocks of 256·CPT; each tree in turn is staged in shared memory (leaf records,
// then 8-byte nodes whose threshold is RD_f32 of the FP64 one: for float32 x, x <= t  <=>  x <= RD_f32(t)), every candidate
// walks it, and the leaf's value v and v² + max(impurity, 0) are added in tree order with __dadd_rn.  Then skopt's
// _return_std: μ = Σv / T, σ² = Σ(v² + var) / T − μ², negatives to 0, σ = √σ², and EI / LCB / PI on the raw μ, σ with the
// GP path's FP64 formulas (kbo_acq.cuh), with a first-index argmax per acquisition.
#include <float.h>
#include <algorithm>
#include <vector>

#include "kbo_rng.cuh"
#include "kbo_tree.cuh"

#define FOREST_FIT_THREADS 1024
#define FOREST_LEAF 0xFFFFFFFFu
#define FOREST_MAX_N 65536
#define FOREST_MAX_D 1024
#define FOREST_MAX_T 1024

struct kbo_forest : TreeCore {
  int kind = 0, T = 0, msl = 3;
  uint64_t seed = 0;
  int n_cap = 0;                     // node capacity per tree
  DevBuf<int> cnt;
  DevBuf<int> cols, tmp, nstart, nend;
  DevBuf<unsigned char> side;
  DevBuf<int> feat, left, right, nns, nnodes, nleaves;
  DevBuf<double> thr, value, imp, wn;
  DevBuf<unsigned char> blob;
  DevBuf<long long> tree_off;
  DevBuf<uint32_t> ex_mn, ex_mx;
  std::vector<int> h_nnodes, h_nleaves;
  std::vector<long long> h_off;
  size_t max_tree_bytes = 0;
  int last_launch[6] = {};           // the last sweep's (staged, CPT, CTAs per SM, CTAs, static smem, opt-in limit)
};

__device__ __forceinline__ float key_f32(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }

// NumPy's random_standard_uniform from two 32-bit words: (a >> 5, b >> 6) → 53 bits / 2^53.
__device__ __forceinline__ double u53(uint32_t a, uint32_t b) { return ((double)(a >> 5) * 67108864.0 + (double)(b >> 6)) * (1.0 / 9007199254740992.0); }

__device__ __forceinline__ double et_threshold(uint64_t seed, int t, int node, int f, float mn, float mx) {
  uint32_t r[4];
  philox4x32_10((uint32_t)node, (uint32_t)t, (uint32_t)f, 1u, (uint32_t)seed, (uint32_t)(seed >> 32), r);
  const double lo = (double)mn, hi = (double)mx;
  double th = __dadd_rn(__dmul_rn(__dadd_rn(hi, -lo), u53(r[0], r[1])), lo);
  if (th == hi) th = lo;
  return th;
}

// ---- bootstrap counts --------------------------------------------------------------------------------------------------
__global__ void forest_bootstrap_kernel(int* __restrict__ cnt, int N, uint64_t seed) {
  const int t = blockIdx.y, d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= N) return;
  uint32_t r[4];
  philox4x32_10((uint32_t)d, (uint32_t)t, 0u, 0u, (uint32_t)seed, (uint32_t)(seed >> 32), r);
  const int i = (int)(((uint64_t)r[0] * (uint64_t)N) >> 32);
  atomicAdd(&cnt[(size_t)t * N + i], 1);
}

// ---- fit -----------------------------------------------------------------------------------------------------------------
struct FitArgs {
  const float* X;
  const double* y;
  const int* cnt;     // T × N draw counts (RF) or nullptr (ET: every weight 1)
  const int* order;   // D × N presorted sample indices (RF)
  int N, D, msl, kind, t0, cap;
  uint64_t seed;
  int* cols;          // per batch tree: D × N (RF) or N (ET)
  int* tmp;
  unsigned char* side;
  int* nstart;
  int* nend;
  int* feat;
  double* thr;
  int* left;
  int* right;
  double* value;
  double* imp;
  int* nns;
  double* wn;
  int* nnodes;
};

struct SplitRec {
  double proxy, thr;
  int feat, nl;
};

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__global__ void __launch_bounds__(FOREST_FIT_THREADS, 1) forest_fit_kernel(FitArgs a) {
  const int bt = blockIdx.x, t = a.t0 + bt, N = a.N, D = a.D;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool rf = a.kind == KBO_FOREST_RF;
  const int* cnt = a.cnt ? a.cnt + (size_t)t * N : nullptr;
  const size_t per = rf ? (size_t)D * N : (size_t)N;
  int* cols = a.cols + (size_t)bt * per;
  int* tmp = a.tmp + (size_t)bt * per;
  unsigned char* side = a.side + (size_t)bt * N;
  int* nstart = a.nstart + (size_t)bt * a.cap;
  int* nend = a.nend + (size_t)bt * a.cap;
  const size_t ob = (size_t)t * a.cap;
  const double* __restrict__ y = a.y;
  const float* __restrict__ X = a.X;
  auto wt = [&](int i) { return cnt ? cnt[i] : 1; };

  __shared__ int s_n, s_nn, s_leaf;
  __shared__ double s_red[3][32];
  __shared__ double s_sw, s_swy;
  __shared__ SplitRec s_best[32];
  __shared__ SplitRec s_win;

  // root: the in-bag samples (count > 0), each column in presorted order
  if (rf) {
    for (int f = warp; f < D; f += 32) {
      int n = 0;
      const int* o = a.order + (size_t)f * N;
      for (int j0 = 0; j0 < N; j0 += 32) {
        const int j = j0 + lane;
        const int i = j < N ? o[j] : 0;
        const bool keep = j < N && wt(i) > 0;
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (keep) cols[(size_t)f * N + n + __popc(m & ((1u << lane) - 1u))] = i;
        n += __popc(m);
      }
      if (f == 0 && lane == 0) s_n = n;
    }
  } else {
    for (int i = tid; i < N; i += blockDim.x) cols[i] = i;
    if (tid == 0) s_n = N;
  }
  __syncthreads();
  if (tid == 0) {
    nstart[0] = 0;
    nend[0] = s_n;
    s_nn = 1;
  }
  __syncthreads();

  for (int k = 0; k < s_nn; k++) {
    const int s = nstart[k], e = nend[k], c = e - s;
    // node statistics over its samples (fixed reduction order)
    {
      const int* seg = cols + s;
      double sw = 0.0, swy = 0.0, swyy = 0.0;
      for (int j = tid; j < c; j += blockDim.x) {
        const int i = seg[j];
        const double w = (double)wt(i), yi = y[i];
        const double wy = __dmul_rn(w, yi);
        sw = __dadd_rn(sw, w);
        swy = __dadd_rn(swy, wy);
        swyy = __dadd_rn(swyy, __dmul_rn(wy, yi));
      }
      sw = warp_sum_d(sw);
      swy = warp_sum_d(swy);
      swyy = warp_sum_d(swyy);
      if (lane == 0) {
        s_red[0][warp] = sw;
        s_red[1][warp] = swy;
        s_red[2][warp] = swyy;
      }
      __syncthreads();
      if (tid == 0) {
        double a0 = 0.0, a1 = 0.0, a2 = 0.0;
        for (int w = 0; w < 32; w++) {
          a0 = __dadd_rn(a0, s_red[0][w]);
          a1 = __dadd_rn(a1, s_red[1][w]);
          a2 = __dadd_rn(a2, s_red[2][w]);
        }
        const double val = __ddiv_rn(a1, a0);
        const double im = __dadd_rn(__ddiv_rn(a2, a0), -__dmul_rn(val, val));
        s_sw = a0;
        s_swy = a1;
        a.value[ob + k] = val;
        a.imp[ob + k] = im;
        a.nns[ob + k] = c;
        a.wn[ob + k] = a0;
        a.feat[ob + k] = -2;   // sklearn's TREE_UNDEFINED / TREE_LEAF until a split is taken
        a.thr[ob + k] = -2.0;
        a.left[ob + k] = -1;
        a.right[ob + k] = -1;
        s_leaf = (c < 2 * a.msl || im <= DBL_EPSILON) ? 1 : 0;
      }
      __syncthreads();
    }
    if (s_leaf) continue;
    const double sw = s_sw, swy = s_swy;
    // best split of each warp's features
    SplitRec best;
    best.proxy = -INFINITY;
    best.thr = 0.0;
    best.feat = 0x7fffffff;
    best.nl = 0;
    for (int f = warp; f < D; f += 32) {
      if (rf) {
        const int* col = cols + (size_t)f * N + s;
        double cw = 0.0, cwy = 0.0;
        for (int j0 = 0; j0 < c; j0 += 32) {
          const int j = j0 + lane;
          const bool valid = j < c;
          const int i = valid ? col[j] : 0;
          const float v = valid ? X[(size_t)i * D + f] : 0.f;
          const double w = valid ? (double)wt(i) : 0.0;
          double iw = w, iwy = valid ? __dmul_rn(w, y[i]) : 0.0;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const double pw = __shfl_up_sync(0xffffffffu, iw, o), pwy = __shfl_up_sync(0xffffffffu, iwy, o);
            if (lane >= o) {
              iw = __dadd_rn(iw, pw);
              iwy = __dadd_rn(iwy, pwy);
            }
          }
          const double wl = __dadd_rn(cw, iw), sl = __dadd_rn(cwy, iwy);
          float vn = __shfl_down_sync(0xffffffffu, v, 1);
          if (lane == 31 && j + 1 < c) vn = X[(size_t)col[j + 1] * D + f];
          const int nl = j + 1;
          const bool cand = valid && j + 1 < c && !(vn <= __fadd_rn(v, 1e-7f)) && nl >= a.msl && c - nl >= a.msl;
          double proxy = -INFINITY;
          if (cand) {
            const double wr = __dadd_rn(sw, -wl), sr = __dadd_rn(swy, -sl);
            proxy = __dadd_rn(__ddiv_rn(__dmul_rn(sl, sl), wl), __ddiv_rn(__dmul_rn(sr, sr), wr));
          }
          // first maximum of the chunk
          double bp = proxy;
          int bl = lane;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            const double op = __shfl_xor_sync(0xffffffffu, bp, o);
            const int ol = __shfl_xor_sync(0xffffffffu, bl, o);
            if (op > bp || (op == bp && ol < bl)) {
              bp = op;
              bl = ol;
            }
          }
          if (bp > best.proxy) {
            const float va = __shfl_sync(0xffffffffu, v, bl), vb = __shfl_sync(0xffffffffu, vn, bl);
            double th = (double)va / 2.0 + (double)vb / 2.0;
            if (th == (double)vb || isinf(th)) th = (double)va;
            best.proxy = bp;
            best.thr = th;
            best.feat = f;
            best.nl = j0 + bl + 1;
          }
          cw = __shfl_sync(0xffffffffu, wl, 31);
          cwy = __shfl_sync(0xffffffffu, sl, 31);
        }
      } else {
        const int* seg = cols + s;
        float mn = INFINITY, mx = -INFINITY;
        for (int j = lane; j < c; j += 32) {
          const float v = X[(size_t)seg[j] * D + f];
          mn = fminf(mn, v);
          mx = fmaxf(mx, v);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        }
        if (mx <= __fadd_rn(mn, 1e-7f)) continue;   // constant in this node
        const double th = et_threshold(a.seed, t, k, f, mn, mx);
        double wl = 0.0, sl = 0.0;
        int nl = 0;
        for (int j = lane; j < c; j += 32) {
          const int i = seg[j];
          if ((double)X[(size_t)i * D + f] <= th) {
            const double w = (double)wt(i);
            wl = __dadd_rn(wl, w);
            sl = __dadd_rn(sl, __dmul_rn(w, y[i]));
            nl++;
          }
        }
        wl = warp_sum_d(wl);
        sl = warp_sum_d(sl);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) nl += __shfl_xor_sync(0xffffffffu, nl, o);
        if (nl < a.msl || c - nl < a.msl) continue;
        const double wr = __dadd_rn(sw, -wl), sr = __dadd_rn(swy, -sl);
        const double proxy = __dadd_rn(__ddiv_rn(__dmul_rn(sl, sl), wl), __ddiv_rn(__dmul_rn(sr, sr), wr));
        if (proxy > best.proxy) {
          best.proxy = proxy;
          best.thr = th;
          best.feat = f;
          best.nl = nl;
        }
      }
    }
    if (lane == 0) s_best[warp] = best;
    __syncthreads();
    if (tid == 0) {
      SplitRec b = s_best[0];
      for (int w = 1; w < 32; w++) {
        const SplitRec& o = s_best[w];
        if (o.proxy > b.proxy || (o.proxy == b.proxy && o.feat < b.feat)) b = o;
      }
      s_win = b;
      s_leaf = b.proxy == -INFINITY ? 1 : 0;   // no valid split: sklearn's split.pos == end
    }
    __syncthreads();
    if (s_leaf) continue;
    const SplitRec w = s_win;
    if (rf) {
      const int* bcol = cols + (size_t)w.feat * N + s;
      for (int j = tid; j < c; j += blockDim.x) side[bcol[j]] = j < w.nl ? 1 : 0;
      __syncthreads();
      for (int f = warp; f < D; f += 32)
        if (f != w.feat)
          warp_partition(cols + (size_t)f * N + s, tmp + (size_t)f * N + s, c, [&](int i) { return side[i] != 0; });
    } else if (warp == 0) {
      warp_partition(cols + s, tmp + s, c, [&](int i) { return (double)X[(size_t)i * D + w.feat] <= w.thr; });
    }
    __syncthreads();
    if (tid == 0) {
      const int l = s_nn;
      a.feat[ob + k] = w.feat;
      a.thr[ob + k] = w.thr;
      a.left[ob + k] = l;
      a.right[ob + k] = l + 1;
      nstart[l] = s;
      nend[l] = s + w.nl;
      nstart[l + 1] = s + w.nl;
      nend[l + 1] = e;
      s_nn = l + 2;
    }
    __syncthreads();
  }
  if (tid == 0) a.nnodes[t] = s_nn;
}

// ---- packing for the sweep: per tree [leaf records (v, v² + max(impurity, 0)) × L][nodes uint2 × n, padded to 16 B] ---------
// A node is (RD_f32(threshold) bits, left << 10 | feature), the right child being left + 1 (breadth-first ids); a leaf is
// (leaf slot, FOREST_LEAF).
__global__ void forest_count_leaves_kernel(const int* __restrict__ left, const int* __restrict__ nnodes, int cap, int* __restrict__ nleaves) {
  const int t = blockIdx.x;
  int c = 0;
  for (int k = threadIdx.x; k < nnodes[t]; k += blockDim.x) c += left[(size_t)t * cap + k] < 0;
  __shared__ int s;
  if (threadIdx.x == 0) s = 0;
  __syncthreads();
  atomicAdd(&s, c);
  __syncthreads();
  if (threadIdx.x == 0) nleaves[t] = s;
}

__global__ void __launch_bounds__(1024) forest_pack_kernel(const int* __restrict__ feat, const double* __restrict__ thr, const int* __restrict__ left,
                                                           const double* __restrict__ value, const double* __restrict__ imp,
                                                           const int* __restrict__ nnodes, const int* __restrict__ nleaves, int cap,
                                                           const long long* __restrict__ off, unsigned char* __restrict__ blob) {
  const int t = blockIdx.x, n = nnodes[t];
  const size_t ob = (size_t)t * cap;
  double2* leaves = reinterpret_cast<double2*>(blob + off[t]);
  uint2* nodes = reinterpret_cast<uint2*>(blob + off[t] + (size_t)nleaves[t] * 16);
  __shared__ int s_base;
  if (threadIdx.x == 0) s_base = 0;
  __syncthreads();
  typedef cub::BlockScan<int, 1024> Scan;
  __shared__ typename Scan::TempStorage ts;
  for (int k0 = 0; k0 < n; k0 += 1024) {
    const int k = k0 + threadIdx.x;
    const bool leaf = k < n && left[ob + k] < 0;
    int slot, total;
    Scan(ts).ExclusiveSum(leaf ? 1 : 0, slot, total);
    slot += s_base;
    if (k < n) {
      if (leaf) {
        const double v = value[ob + k], im = imp[ob + k];
        leaves[slot] = make_double2(v, __dadd_rn(im > 0.0 ? im : 0.0, __dmul_rn(v, v)));   // var_tree + mean_tree ** 2
        nodes[k] = make_uint2((uint32_t)slot, FOREST_LEAF);
      } else {
        nodes[k] = make_uint2(__float_as_uint(__double2float_rd(thr[ob + k])), ((uint32_t)left[ob + k] << 10) | (uint32_t)feat[ob + k]);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) s_base += total;
    __syncthreads();
  }
}

// ---- sweep ------------------------------------------------------------------------------------------------------------------
struct SweepArgs {
  const unsigned char* blob;
  const long long* off;
  const int* nleaves;
  int T;
  const float* Xc;
  int64_t M;
  int D;
  int n_acq, acq0, acq1, acq2;
  double yopt, xi, kappa;
  double* mu_out;
  double* sd_out;
  kbo_best* part;
};

template <int CPT, bool STAGED>
__global__ void __launch_bounds__(256) forest_sweep_kernel(SweepArgs a) {
  extern __shared__ int4 smem[];
  const int tid = threadIdx.x;
  const int64_t ntiles = (a.M + 256 * CPT - 1) / (256 * CPT);
  TreeArgmax best;
  const int acqs[3] = {a.acq0, a.acq1, a.acq2};
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    int64_t m[CPT];
    double amu[CPT], aq[CPT];
#pragma unroll
    for (int c = 0; c < CPT; c++) {
      m[c] = tile * 256 * CPT + c * 256 + tid;
      amu[c] = 0.0;
      aq[c] = 0.0;
    }
    for (int t = 0; t < a.T; t++) {
      const unsigned char* src = a.blob + a.off[t];
      const int nl = a.nleaves[t];
      const double2* leaves;
      const uint2* nodes;
      if (STAGED) {
        const int n16 = (int)((a.off[t + 1] - a.off[t]) >> 4);
        __syncthreads();
        for (int i = tid; i < n16; i += 256) smem[i] = __ldg(reinterpret_cast<const int4*>(src) + i);
        __syncthreads();
        leaves = reinterpret_cast<const double2*>(smem);
        nodes = reinterpret_cast<const uint2*>(reinterpret_cast<const unsigned char*>(smem) + (size_t)nl * 16);
      } else {
        leaves = reinterpret_cast<const double2*>(src);
        nodes = reinterpret_cast<const uint2*>(src + (size_t)nl * 16);
      }
      uint2 nd[CPT];
      const float* xr[CPT];
#pragma unroll
      for (int c = 0; c < CPT; c++) {
        nd[c] = nodes[0];
        xr[c] = a.Xc + (size_t)(m[c] < a.M ? m[c] : 0) * a.D;
      }
      bool more = true;
      while (more) {   // the CPT walks advance in lockstep, so their loads overlap
        more = false;
#pragma unroll
        for (int c = 0; c < CPT; c++) {
          if (nd[c].y != FOREST_LEAF) {
            const float x = __ldg(xr[c] + (nd[c].y & 1023u));
            nd[c] = nodes[(nd[c].y >> 10) + (x <= __uint_as_float(nd[c].x) ? 0u : 1u)];
            more = true;
          }
        }
      }
#pragma unroll
      for (int c = 0; c < CPT; c++) {
        const double2 lv = leaves[nd[c].x];
        amu[c] = __dadd_rn(amu[c], lv.x);
        aq[c] = __dadd_rn(aq[c], lv.y);
      }
    }
    const double T = (double)a.T;
#pragma unroll
    for (int c = 0; c < CPT; c++) {
      if (m[c] >= a.M) continue;
      const double mu = __ddiv_rn(amu[c], T);
      double s2 = __dadd_rn(__ddiv_rn(aq[c], T), -__dmul_rn(mu, mu));
      if (s2 < 0.0) s2 = 0.0;
      const double sd = __dsqrt_rn(s2);
      if (a.mu_out) a.mu_out[m[c]] = mu;
      if (a.sd_out) a.sd_out[m[c]] = sd;
#pragma unroll
      for (int q = 0; q < 3; q++) {
        if (q >= a.n_acq) break;
        double mo, so;
        best.keep(q, acq_value<double>(mu, s2, acqs[q], 0.0, 1.0, a.yopt, a.xi, a.kappa, &mo, &so), m[c], mu, sd);
      }
    }
  }
  best.write(a.n_acq, a.part);
}

// ---- export: the per-node min / max of each feature over the node's samples, to restate the ET draws --------------------
__global__ void forest_route_minmax_kernel(const float* __restrict__ X, int N, int D, const int* __restrict__ feat, const double* __restrict__ thr,
                                           const int* __restrict__ left, uint32_t* __restrict__ mn, uint32_t* __restrict__ mx) {
  const int i = blockIdx.x;
  int k = 0;
  while (true) {
    const int l = left[k];
    if (l < 0) break;
    for (int f = threadIdx.x; f < D; f += blockDim.x) {
      const uint32_t key = f32_key(X[(size_t)i * D + f]);
      atomicMin(&mn[(size_t)k * D + f], key);
      atomicMax(&mx[(size_t)k * D + f], key);
    }
    k = (double)X[(size_t)i * D + feat[k]] <= thr[k] ? l : l + 1;
  }
}

__global__ void forest_draws_kernel(const uint32_t* __restrict__ mn, const uint32_t* __restrict__ mx, const int* __restrict__ left, int n, int D,
                                    uint64_t seed, int t, double* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)n * D) return;
  const int k = (int)(e / D), f = (int)(e % D);
  double th = NAN;
  if (left[k] >= 0) {
    const float a = key_f32(mn[e]), b = key_f32(mx[e]);
    if (!(b <= __fadd_rn(a, 1e-7f))) th = et_threshold(seed, t, k, f, a, b);
  }
  out[e] = th;
}

// ---- C ABI ------------------------------------------------------------------------------------------------------------------
static int forest_sweep_launch(kbo_handle* h, kbo_forest* f, const float* Xc, int64_t M, int n_acq, const int32_t* acqs, double yopt, double xi,
                               double kappa, double* mu_out, double* sd_out, int* nblocks_out, cudaStream_t s) {
  const int cpt = (M + 1023) / 1024 >= 2 * h->sm_count ? 4 : 1;
  // The largest tree is staged in shared memory when it fits there beside the kernel's own static shared memory (TreeArgmax's
  // partials): a block may opt in to smem_optin bytes of both together.  Larger trees are walked in global memory.
  void (*k)(SweepArgs) = cpt == 4 ? forest_sweep_kernel<4, true> : forest_sweep_kernel<1, true>;
  cudaFuncAttributes fa;
  KBO_CUDA(h, cudaFuncGetAttributes(&fa, k));
  const bool staged = f->max_tree_bytes + fa.sharedSizeBytes <= (size_t)h->smem_optin;
  const size_t sm = staged ? f->max_tree_bytes : 0;
  if (staged) {
    KBO_CUDA(h, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  } else {
    k = cpt == 4 ? forest_sweep_kernel<4, false> : forest_sweep_kernel<1, false>;
  }
  int occ = 0;
  KBO_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, 256, sm));
  const int64_t ntiles = (M + 256 * cpt - 1) / (256 * cpt);
  const int nb = (int)std::min<int64_t>(ntiles, (int64_t)h->sm_count * std::max(occ, 1));
  KBO_TRY(kbo_reserve(h, f->part, (size_t)nb * 3));
  SweepArgs a{f->blob.p, f->tree_off.p, f->nleaves.p, f->T, Xc, M, f->D, n_acq,
              n_acq > 0 ? acqs[0] : 0, n_acq > 1 ? acqs[1] : 0, n_acq > 2 ? acqs[2] : 0, yopt, xi, kappa, mu_out, sd_out, f->part.p};
  k<<<nb, 256, sm, s>>>(a);
  KBO_LAUNCH_CHECK(h);
  const int launch[6] = {staged ? 1 : 0, cpt, occ, nb, (int)fa.sharedSizeBytes, h->smem_optin};
  std::copy(launch, launch + 6, f->last_launch);
  *nblocks_out = nb;
  return KBO_OK;
}

extern "C" {

int kbo_forest_create(kbo_handle* h, kbo_forest** out, int32_t kind, int32_t n_trees, int32_t min_samples_leaf, uint64_t seed) {
  if (!h || !out) return KBO_ERR_INVALID;
  *out = nullptr;
  if (kind != KBO_FOREST_RF && kind != KBO_FOREST_ET) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_forest_create: kind must be RF (0) or ET (1), got %d", kind);
  if (n_trees < 1 || n_trees > FOREST_MAX_T) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_forest_create: 1 <= n_trees <= %d (got %d)", FOREST_MAX_T, n_trees);
  if (min_samples_leaf < 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_forest_create: min_samples_leaf must be >= 1 (got %d)", min_samples_leaf);
  KBO_CUDA(h, cudaSetDevice(h->device));
  std::unique_ptr<kbo_forest> f(new (std::nothrow) kbo_forest());
  if (!f) return KBO_ERR_NOMEM;
  f->kind = kind;
  f->T = n_trees;
  f->msl = min_samples_leaf;
  f->seed = seed;
  KBO_TRY(f->ev.create());
  *out = f.release();
  return KBO_OK;
}

void kbo_forest_destroy(kbo_forest* f) {
  if (f) delete f;
}

int kbo_forest_fit(kbo_handle* h, kbo_forest* f, const float* X, const double* y, int32_t N, int32_t D, const int32_t* counts, void* stream) {
  if (!h || !f || !X || !y) return KBO_ERR_INVALID;
  if (N < 1 || N > FOREST_MAX_N) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_forest_fit: 1 <= N <= %d (got %d)", FOREST_MAX_N, N);
  if (D < 1 || D > FOREST_MAX_D) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_forest_fit: 1 <= D <= %d (got %d)", FOREST_MAX_D, D);
  if (counts && f->kind != KBO_FOREST_RF) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_forest_fit: bootstrap counts are for RF forests only");
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  KBO_TRY(tree_fit_begin(h, f, X, y, N, D, "kbo_forest_fit", s));
  const int T = f->T;
  const bool rf = f->kind == KBO_FOREST_RF;
  const size_t ND = (size_t)N * D;
  if (rf) {
    KBO_TRY(kbo_reserve(h, f->cnt, (size_t)T * N));
    if (counts) {
      KBO_CUDA(h, kbo_copy(f->cnt.p, counts, (size_t)T * N, cudaMemcpyDeviceToDevice, s));
    } else {
      KBO_CUDA(h, cudaMemsetAsync(f->cnt.p, 0, sizeof *f->cnt.p * T * N, s));
      forest_bootstrap_kernel<<<dim3((N + 255) / 256, T), 256, 0, s>>>(f->cnt.p, N, f->seed);
      KBO_LAUNCH_CHECK(h);
    }
    KBO_TRY(tree_presort(h, f, N, D, s));
  }
  // node capacity: every leaf holds >= min_samples_leaf samples (or is the root)
  const int cap = 2 * std::max(1, N / f->msl) + 1;
  f->n_cap = cap;
  const size_t TC = (size_t)T * cap;
  KBO_TRY(kbo_reserve(h, f->feat, TC));
  KBO_TRY(kbo_reserve(h, f->thr, TC));
  KBO_TRY(kbo_reserve(h, f->left, TC));
  KBO_TRY(kbo_reserve(h, f->right, TC));
  KBO_TRY(kbo_reserve(h, f->value, TC));
  KBO_TRY(kbo_reserve(h, f->imp, TC));
  KBO_TRY(kbo_reserve(h, f->nns, TC));
  KBO_TRY(kbo_reserve(h, f->wn, TC));
  KBO_TRY(kbo_reserve(h, f->nnodes, (size_t)T));
  KBO_TRY(kbo_reserve(h, f->nleaves, (size_t)T));
  // trees in batches whose column scratch stays within 2 GiB
  const size_t per = rf ? ND : (size_t)N;   // column scratch ints per tree
  const int batch = (int)std::max<size_t>(1, std::min<size_t>((size_t)T, (2ull << 30) / (2 * sizeof(int) * per + N + 8ull * cap)));
  KBO_TRY(kbo_reserve(h, f->cols, per * batch));
  KBO_TRY(kbo_reserve(h, f->tmp, per * batch));
  KBO_TRY(kbo_reserve(h, f->side, (size_t)N * batch));
  KBO_TRY(kbo_reserve(h, f->nstart, (size_t)cap * batch));
  KBO_TRY(kbo_reserve(h, f->nend, (size_t)cap * batch));
  for (int t0 = 0; t0 < T; t0 += batch) {
    FitArgs a{f->X.p, f->y.p, rf ? f->cnt.p : nullptr, rf ? f->order.p : nullptr, N, D, f->msl,
              f->kind, t0, cap, f->seed, f->cols.p, f->tmp.p, f->side.p, f->nstart.p, f->nend.p,
              f->feat.p, f->thr.p, f->left.p, f->right.p, f->value.p, f->imp.p, f->nns.p,
              f->wn.p, f->nnodes.p};
    forest_fit_kernel<<<std::min(batch, T - t0), FOREST_FIT_THREADS, 0, s>>>(a);
    KBO_LAUNCH_CHECK(h);
  }
  forest_count_leaves_kernel<<<T, 256, 0, s>>>(f->left.p, f->nnodes.p, cap, f->nleaves.p);
  KBO_LAUNCH_CHECK(h);
  f->h_nnodes.assign(T, 0);
  f->h_nleaves.assign(T, 0);
  KBO_CUDA(h, kbo_copy(f->h_nnodes.data(), f->nnodes.p, (size_t)T, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, kbo_copy(f->h_nleaves.data(), f->nleaves.p, (size_t)T, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  f->h_off.assign(T + 1, 0);
  f->max_tree_bytes = 0;
  for (int t = 0; t < T; t++) {
    const size_t bytes = (size_t)f->h_nleaves[t] * 16 + (size_t)round_up(f->h_nnodes[t], 2) * 8;
    f->h_off[t + 1] = f->h_off[t] + (long long)bytes;
    f->max_tree_bytes = std::max(f->max_tree_bytes, bytes);
  }
  KBO_TRY(kbo_reserve(h, f->blob, (size_t)f->h_off[T]));
  KBO_TRY(kbo_reserve(h, f->tree_off, (size_t)(T + 1)));
  KBO_CUDA(h, kbo_copy(f->tree_off.p, f->h_off.data(), (size_t)(T + 1), cudaMemcpyHostToDevice, s));
  KBO_CUDA(h, cudaMemsetAsync(f->blob.p, 0, (size_t)f->h_off[T], s));
  forest_pack_kernel<<<T, 1024, 0, s>>>(f->feat.p, f->thr.p, f->left.p, f->value.p,
                                        f->imp.p, f->nnodes.p, f->nleaves.p, cap,
                                        f->tree_off.p, f->blob.p);
  KBO_LAUNCH_CHECK(h);
  return tree_fit_end(h, f, N, D, s);   // synchronises: the host copy of tree_off must outlive its transfer
}

int kbo_forest_sweep(kbo_handle* h, kbo_forest* f, const float* Xc, int64_t M, int64_t global_offset, int32_t n_acq, const int32_t* acqs, double y_opt,
                     double xi, double kappa, kbo_best* best_dev, double* mu_out, double* sigma_out, void* stream) {
  if (!h || !f || !Xc) return KBO_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  KBO_TRY(tree_sweep_begin(h, f, M, n_acq, acqs, y_opt, best_dev, "kbo_forest_sweep", "the forest", s));
  int nb = 0;
  KBO_TRY(forest_sweep_launch(h, f, Xc, M, n_acq, acqs, y_opt, xi, kappa, mu_out, sigma_out, &nb, s));
  return tree_sweep_end(h, f, nb, n_acq, global_offset, best_dev, s);
}

int kbo_forest_predict(kbo_handle* h, kbo_forest* f, const float* X, int32_t n, int x_on_host, double* mu_host, double* sigma_host, void* stream) {
  if (!h || !f || !X || n < 1) return KBO_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  const float* Xd = nullptr;
  KBO_TRY(tree_predict_rows(h, f, X, n, x_on_host, &Xd, "kbo_forest_predict", "the forest", s));
  KBO_TRY(kbo_reserve(h, h->stage_y, (size_t)n * 2));
  double* mu = h->stage_y.p;
  int nb = 0;
  KBO_TRY(forest_sweep_launch(h, f, Xd, n, 0, nullptr, 0.0, 0.0, 0.0, mu, mu + n, &nb, s));
  KBO_CUDA(h, kbo_d2h(mu_host, mu, n, s));
  KBO_CUDA(h, kbo_d2h(sigma_host, mu + n, n, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  return KBO_OK;
}

int kbo_forest_export(kbo_handle* h, kbo_forest* f, int32_t tree, int32_t* feature, double* threshold, int32_t* left, int32_t* right, double* value,
                      double* impurity, int32_t* n_node_samples, double* weighted_n, double* et_draws, int32_t cap, int32_t* n_nodes, int32_t* counts,
                      void* stream) {
  if (!h || !f) return KBO_ERR_INVALID;
  if (!f->fitted) KBO_FAIL(h, KBO_ERR_STATE, "kbo_forest_export: the forest is not fitted");
  if (tree < 0 || tree >= f->T) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_forest_export: tree %d out of range [0, %d)", tree, f->T);
  if (et_draws && f->kind != KBO_FOREST_ET) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_forest_export: et_draws is for ET forests only");
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  const int n = f->h_nnodes[tree];
  if (n_nodes) *n_nodes = n;
  if (counts) {
    if (f->kind == KBO_FOREST_RF) {
      KBO_CUDA(h, kbo_copy(counts, f->cnt.p + (size_t)tree * f->N, (size_t)f->N, cudaMemcpyDeviceToHost, s));
    } else {
      for (int i = 0; i < f->N; i++) counts[i] = 1;
    }
  }
  if (cap < n) {
    KBO_CUDA(h, cudaStreamSynchronize(s));
    return KBO_OK;   // size query
  }
  const size_t ob = (size_t)tree * f->n_cap;
  KBO_CUDA(h, kbo_d2h(feature, f->feat.p + ob, n, s));
  KBO_CUDA(h, kbo_d2h(threshold, f->thr.p + ob, n, s));
  KBO_CUDA(h, kbo_d2h(left, f->left.p + ob, n, s));
  KBO_CUDA(h, kbo_d2h(right, f->right.p + ob, n, s));
  KBO_CUDA(h, kbo_d2h(value, f->value.p + ob, n, s));
  KBO_CUDA(h, kbo_d2h(impurity, f->imp.p + ob, n, s));
  KBO_CUDA(h, kbo_d2h(n_node_samples, f->nns.p + ob, n, s));
  KBO_CUDA(h, kbo_d2h(weighted_n, f->wn.p + ob, n, s));
  if (et_draws) {
    const size_t nd = (size_t)n * f->D;
    KBO_TRY(kbo_reserve(h, f->ex_mn, nd));
    KBO_TRY(kbo_reserve(h, f->ex_mx, nd));
    KBO_TRY(kbo_reserve(h, h->stage_X, nd));
    KBO_CUDA(h, cudaMemsetAsync(f->ex_mn.p, 0xFF, sizeof *f->ex_mn.p * nd, s));
    KBO_CUDA(h, cudaMemsetAsync(f->ex_mx.p, 0x00, sizeof *f->ex_mx.p * nd, s));
    forest_route_minmax_kernel<<<f->N, 128, 0, s>>>(f->X.p, f->N, f->D, f->feat.p + ob, f->thr.p + ob,
                                                    f->left.p + ob, f->ex_mn.p, f->ex_mx.p);
    KBO_LAUNCH_CHECK(h);
    forest_draws_kernel<<<(unsigned)((nd + 255) / 256), 256, 0, s>>>(f->ex_mn.p, f->ex_mx.p, f->left.p + ob,
                                                                     n, f->D, f->seed, tree, h->stage_X.p);
    KBO_LAUNCH_CHECK(h);
    KBO_CUDA(h, kbo_copy(et_draws, h->stage_X.p, nd, cudaMemcpyDeviceToHost, s));
  }
  KBO_CUDA(h, cudaStreamSynchronize(s));
  return KBO_OK;
}

int kbo_forest_last_timings(kbo_handle* h, kbo_forest* f, float* ms, int32_t n) { return tree_last_timings(h, f, ms, n); }

// Test hook: how the last sweep or predict was launched, stats[6] = (staged, CPT, CTAs per SM, CTAs, the kernel's static shared
// memory, the device's per-block opt-in limit).
int kbo_debug_forest_sweep(kbo_handle* h, kbo_forest* f, int32_t* stats) {
  if (!h || !f) return KBO_ERR_INVALID;
  if (!stats) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_debug_forest_sweep: bad argument");
  std::copy(f->last_launch, f->last_launch + 6, stats);
  return KBO_OK;
}

}  // extern "C"
