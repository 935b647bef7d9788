// Internal declarations shared by the libkbo translation units (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <memory>
#include <string>
#include <vector>

#include "../../include/kbo.h"

#define KBO_NB 64  // Cholesky / trtri block size (one diagonal block = one CTA in shared memory)

// A device array of T owned by its holder: freed when the holder is destroyed, grown only by kbo_reserve.  cap counts elements.
template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) {
      if (p) cudaFree(p);
      p = o.p;
      cap = o.cap;
      o.p = nullptr;
      o.cap = 0;
    }
    return *this;
  }
  ~DevBuf() {
    if (p) cudaFree(p);
  }
};

// A byte buffer holds data with no single element type (one of two dtypes, CUB temporary storage, packed tree nodes); this is
// the one place it is read as U.
template <class U>
static inline U* kbo_view(const DevBuf<unsigned char>& b) { return reinterpret_cast<U*>(b.p); }

// The fixed timing events of one object: create() makes all of them, the destructor destroys them.
template <int N>
struct EventSet {
  cudaEvent_t e[N] = {};
  EventSet() = default;
  EventSet(const EventSet&) = delete;
  EventSet& operator=(const EventSet&) = delete;
  ~EventSet() {
    for (cudaEvent_t x : e)
      if (x) cudaEventDestroy(x);
  }
  int create() {
    for (cudaEvent_t& x : e)
      if (cudaEventCreate(&x) != cudaSuccess) {
        x = nullptr;
        return KBO_ERR_CUDA;
      }
    return KBO_OK;
  }
  cudaEvent_t operator[](int i) const { return e[i]; }
};

struct BlockBest;  // sweep.cu

struct kbo_handle {
  int device = 0;
  int sm_count = 132;
  int smem_optin = 227 * 1024;  // shared memory a block may opt in to, static and dynamic together
  std::string err;
  uint64_t scratch_limit = 4ull << 30;

  // ---- fit state -------------------------------------------------------------------------
  bool fitted = false;
  bool have_planes = false;  // fp16 hi/lo planes of W built by the last fit
  int N = 0, D = 0, ld = 0;  // ld = leading dimension of L / W (multiple of 64)
  int Npad = 0;              // multiple of 256: extent of the fp16 W planes and of K* scratch rows
  kbo_params prm{};
  std::vector<double> inv_ls;  // 1/ℓ_d, host copy
  DevBuf<double> d_inv_ls;     // D doubles
  DevBuf<double> XsT;          // Xs transposed: D × ld (coalesced trial-tile loads in the K* kernel)
  DevBuf<double> Xs, nx, yn, K, W, Linv, T, alpha, z;
  DevBuf<double> yraw, lrow;  // raw y (re-normalised on append) and the append's work vectors
  DevBuf<__half> Wh, Wl;      // fp16 planes Npad×Npad (TC mode)
  DevBuf<double> scal;        // device scalars, see ScalIdx
  DevBuf<int> info;           // [0] potrf info; [1] 1 if an append set it (only that row is unfactored), 0 after a fit (its whole
                              // failing 64-block is)
  DevBuf<double> stage_X, stage_y;  // H2D staging for host-pointer entry points
  DevBuf<unsigned char> stage_Xc;   // the same for candidates, fp64 or fp32 (xc_dtype)
  // ---- sweep workspace ---------------------------------------------------------------------
  DevBuf<double> Ks64;         // chunk × ldks fp64 (F64 mode)
  DevBuf<__half> Ksh, Ksl;     // chunk × Npad fp16 planes (TC mode)
  DevBuf<unsigned char> mun;   // M (fp64 in F64 mode, fp32 in TC mode)
  DevBuf<double> part;         // chunk × n_jtiles partial Σv² (fp64) — F64 mode
  DevBuf<unsigned char> varn;  // M (same dtype as mun)
  DevBuf<BlockBest> blockbest; // per-block argmax partials
  DevBuf<kbo_best> best;       // one kbo_best for suggest_host
  // contender list of the FP64 refinement (tensor-core mode); at KBO_REFINE_CAP the survivor count padded to 4 ints, then
  // 8 floats of stage bounds (slot 1 holds ordered unsigned bits): both types, all 4 bytes wide and 4-byte aligned
  DevBuf<int> refine;
  DevBuf<double> refine_x;     // gathered rows of the FP64 refinement
  int last_contenders = 0;
  float last_rank_err = 0.f;   // largest |σ²(1 product) − σ²(3 products)| over the calibration rows of the last fast sweep
  bool tc_fast = true;      // array-free tensor-core sweeps rank with ONE fp16 product and let the FP64 refinement decide
  DevBuf<float> var_cal;    // three-product variance of the calibration rows
  kbo_timings tim{};
  EventSet<8> ev;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev_var, ev_cross, ev_acq, ev_cal;
  size_t ev_var_used = 0, ev_cross_used = 0, ev_acq_used = 0, ev_cal_used = 0;
  int launches = 0;
  bool time_kernels = false;
  bool attr_fit = false, attr_tc = false;   // cudaFuncSetAttribute done for this handle's device
  // ---- tensor-core K* generation (tc_kstar.cu) and wgmma ranking kernel (tc_rank.cu) ---------------------------
  bool rank_tc = true;        // kbo_set_rank_tc: the ranking pass builds K̃* on the tensor cores and contracts with wgmma MMAs
  bool ks_ready = false;      // trial-side operands below match the current fit
  DevBuf<double> ks_center;   // D doubles: centre subtracted from the scaled coordinates (any fixed vector is valid)
  DevBuf<__half> ks_Xh, ks_Xl; // trials, fp16 hi/lo planes, round_up(N,256) × round_up(D,32)
  DevBuf<float> ks_nxal;      // (|x̂_n|², alpha_n) float pairs
  DevBuf<__half> ks_Ch, ks_Cl; // candidate planes of the current chunk
  DevBuf<float> ks_nc;        // squared norms of the current chunk
  DevBuf<float> rk_part;      // [tile pairs][rows] partial Σ v² of the ranking kernel
  struct RkSched {
    int key[5] = {-1, -1, -1, -1, -1};  // (row groups, j-tiles, CTAs, first tile pair, end tile pair)
    DevBuf<int> dev;
    std::vector<int> host;
  } rk_sched[8];
  int rk_sched_next = 0;
  bool attr_rank = false;
  int rank_prefix = -1;            // kbo_set_rank_prefix: tile pairs of the pruning pass (-1: an eighth of them, 0: no pruning pass)
  int last_prefix_survivors = -1;  // candidates whose prefix upper bound reached the calibration rows' best value (-1: pass not run)
  DevBuf<int> pr_list;             // pruning pass: survivor indices
  DevBuf<double> pr_x;             // their gathered rows
  DevBuf<float> pr_mu, pr_var;     // their ranking-pass mean / variance
  DevBuf<float> cal_mu_rk, cal_var_rk;  // the ranking arithmetic on the calibration rows
  DevBuf<double> mu_part;          // FP64 K* kernel with the trial tiles split over blockIdx.y: partial means [split][row]
  DevBuf<int> cal_idx;             // stratified calibration rows of the ranking pass: indices
  DevBuf<double> cal_x;            // their gathered rows
  DevBuf<float> cal_mu;            // their FP64-path mean
  float last_rank_mu_err = 0.f;    // largest |μ̃ − μ| (normalised units) on the calibration rows of the last ranking sweep
  int last_unrefined = 0;          // 1: the last tensor-core sweep could not decide in FP64 (more near-ties than the cap)
  int dec_n = 0;                   // acquisitions the last kbo_sweep / kbo_sweep_multi decided, and how (kbo_last_decisions)
  int dec_unrefined[3] = {}, dec_contenders[3] = {}, dec_prefix_survivors[3] = {};
  DevBuf<int> un_idx;              // FP64 decision over the union of several acquisitions' survivors: indices / positions
  DevBuf<double> un_mv;            // their mean + variance
  // test hook (kbo_debug_record_stages): what each stage of the last kbo_sweep / kbo_sweep_multi kept, read back only when switched on
  struct StageRec {
    int stage, acq, cal_n, n;      // n: survivors counted; list holds the first min(n, the stage's cap) of them (grid-local indices)
    float f[7];                    // E, Eμ, raw max |dσ²|, raw max |dμ|, lower bound on the maximum, threshold, window delta
    std::vector<int> list;
  };
  bool record_stages = false;
  std::vector<StageRec> stage_recs;
  cudaStream_t s_copy = nullptr;   // the candidate grid's host-to-device copy, beside the fit (api.cu)
  // ---- fit: the chain runs on its own SM partition (green contexts); shadow panel solve / trailing update / inverse share the rest (fit.cu)
  DevBuf<double> T2;                // N × 256 scratch of the far rows' panel solve
  bool part_tried = false, part_ok = false;
  void *gctx_chain = nullptr, *gctx_rest = nullptr;   // CUgreenCtx
  // stream roles: 0 chain, 1 near shadow (both on the chain's partition), 2 far shadow, 3..6 column-block updates at distance 1..4,
  // 7 bulk trailing update, 8 inverse, 9 W_PP (on the chain's partition)
  cudaStream_t s3g[10] = {};       // green-context set
  cudaStream_t s3p[10] = {};       // the same roles as plain priority streams (small N, profilers, no green contexts)
  DevBuf<double> Linv4;             // the four 64×64 block inverses of the current panel
  std::vector<cudaEvent_t> ev_panel;
  cudaEvent_t ev_gram = nullptr;   // the first column block of the Gram matrix is complete (the factorisation starts on it)
  // The factorisation as one CUDA graph (fit.cu, factor_and_invert_v3): captured on s_cap (the caller's stream may be the legacy
  // default stream, which cannot capture), replayed on the caller's stream while the key (shape, mode, device pointers) holds.
  cudaStream_t s_cap = nullptr;
  cudaGraph_t fit_graph = nullptr;          // the graph fit_exec was instantiated from (its nodes address fit_exec's)
  cudaGraphExec_t fit_exec = nullptr;
  cudaGraphNode_t fit_gram_node = nullptr;  // the Gram matrix's second launch: θ by value, set before every replay
  std::vector<intptr_t> fit_key;
  int fit_graph_launches = 0;               // kernel launches in the graph (counted into `launches` on every replay)
  bool fit_stream_path = false;             // kbo_debug_fit_stream_path: enqueue the factorisation call by call
  int fit_graph_stat[4] = {};               // captures, executable updates, instantiations, replays
  // ---- lazy inverse (fit.cu, solve.cu): the product path never needs all of W = L⁻¹ -----------------------------------------
  bool lazy_w = true;              // kbo_set_lazy_inverse: tensor-core fits form only the leading rows of W the pruning pass reads
  bool w_full = true;              // all rows of W (and the full fp16 planes) exist
  int w_lead = 0;                  // rows of W formed so far (the diagonal 256-blocks exist for every panel)
  DevBuf<double> sv_B, sv_V;       // N × 8 right-hand sides / solutions of the panel solves
  DevBuf<unsigned> sv_bar;         // grid-barrier counter of the cooperative solve kernels
  DevBuf<double> zf;               // b (consumed) and z = L⁻¹·yn of the forward substitution carried along by the factorisation
  bool z_ready = false;            // zf holds z of the current factorisation
  // ---- kbo_lml_batch: concurrent factorisations for several θ (fit.cu) --------------------------------------------------
  void* lml_lanes = nullptr;       // std::vector<LmlLane>*
  DevBuf<double> lml_yn, lml_scal;
  cudaEvent_t lml_ev = nullptr;
  // ---- multi-GPU exchange (comm.cu): NCCL communicator bound at run time ------------------------------------------------
  void* comm = nullptr;            // ncclComm_t
  int comm_ranks = 1, comm_rank = 0;
  DevBuf<kbo_best> comm_buf;       // n_ranks kbo_best gathered
};

// h->scal holds 16 doubles.  The first S_COUNT are the fit's scalars; S_WSCALE and S_WSCALE + 1 hold 2^s and 2^-s of the fp16 W
// planes, and S_WAMAX, past S_COUNT, holds max |W| as the bit pattern of a uint64 (the atomic max of absmax_kernel).
enum ScalIdx { S_YMEAN = 0, S_YSTD = 1, S_YOPT = 2, S_LML = 3, S_LOGDET = 4, S_QUAD = 5, S_WSCALE = 6, S_COUNT = 8, S_WAMAX = 8 };

#define KBO_FAIL(h, code, ...)                         \
  do {                                                 \
    char _b[512];                                      \
    snprintf(_b, sizeof _b, __VA_ARGS__);              \
    (h)->err = _b;                                     \
    return (code);                                     \
  } while (0)

#define KBO_CUDA(h, expr)                                                                          \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      KBO_FAIL(h, KBO_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

#define KBO_LAUNCH_CHECK(h)                                                                        \
  do {                                                                                             \
    (h)->launches++;                                                                               \
    cudaError_t _e = cudaGetLastError();                                                           \
    if (_e != cudaSuccess)                                                                         \
      KBO_FAIL(h, KBO_ERR_CUDA, "kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

#define KBO_TRY(expr)          \
  do {                         \
    int _r = (expr);           \
    if (_r != KBO_OK) return _r; \
  } while (0)
// Room for n elements in b: grow-only, and the old contents are not kept.
template <class T>
static inline int kbo_reserve(kbo_handle* h, DevBuf<T>& b, size_t n) {
  if (n <= b.cap) return KBO_OK;
  if (b.p) cudaFree(b.p);
  b.p = nullptr;
  b.cap = 0;
  const size_t bytes = sizeof(T) * n;
  cudaError_t e = cudaMalloc(&b.p, bytes);
  if (e != cudaSuccess) KBO_FAIL(h, KBO_ERR_NOMEM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
  b.cap = n;
  return KBO_OK;
}
// n elements of host data into b, synchronously (at least 4 bytes reserved, so an empty list still has a device pointer)
template <class T>
static inline int kbo_upload(kbo_handle* h, DevBuf<T>& b, const T* host, size_t n) {
  KBO_TRY(kbo_reserve(h, b, std::max(n, (4 + sizeof(T) - 1) / sizeof(T))));
  if (n) KBO_CUDA(h, cudaMemcpy(b.p, host, sizeof(T) * n, cudaMemcpyHostToDevice));
  return KBO_OK;
}
// n elements from src to dst on s (cudaMemcpyAsync); the element types must agree
template <class T>
static inline cudaError_t kbo_copy(T* dst, const T* src, size_t n, cudaMemcpyKind kind, cudaStream_t s) {
  return cudaMemcpyAsync(dst, src, sizeof(T) * n, kind, s);
}
// n elements of device data to out on s (cudaMemcpyAsync), or nothing when the caller passed no out
template <class T>
static inline cudaError_t kbo_d2h(T* out, const T* src, size_t n, cudaStream_t s) {
  return out ? cudaMemcpyAsync(out, src, sizeof(T) * n, cudaMemcpyDeviceToHost, s) : cudaSuccess;
}

static inline int round_up(int x, int m) { return (x + m - 1) / m * m; }
static inline int64_t round_up64(int64_t x, int64_t m) { return (x + m - 1) / m * m; }
// Pairs of 256-trial tiles the ranking pass contracts over, and the pairs the pruning pass takes by default (an eighth of them;
// kbo_set_rank_prefix sets another count, 0 turns the pass off).  Callers check the range they need themselves.
static inline int kbo_tile_pairs(int Npad) { return (Npad / 256 + 1) / 2; }
static inline int kbo_prefix_pairs(const kbo_handle* h) { return h->rank_prefix < 0 ? (kbo_tile_pairs(h->Npad) + 7) / 8 : h->rank_prefix; }

// ---- fit.cu ------------------------------------------------------------------------------------
int kbo_i_gram(kbo_handle* h, const double* Xs, int N, int D, int kernel, double amp, double noise, double* K, int ldk,
               cudaStream_t s);
int kbo_i_potrf(kbo_handle* h, double* A, int N, int lda, int* info_dev, cudaStream_t s);
int kbo_i_fit_append(kbo_handle* h, const double* x_dev, double y, cudaStream_t s);
int kbo_i_fit_rebase(kbo_handle* h, int n_keep, const double* y_dev, cudaStream_t s);
int kbo_i_trtri(kbo_handle* h, const double* L, int N, int ldl, double* W, int ldw, cudaStream_t s, double* T = nullptr);
int kbo_i_zero_upper(kbo_handle* h, double* A, int N, int lda, cudaStream_t s);
int kbo_i_fit(kbo_handle* h, const double* X_dev, const double* y_dev, int N, int D, const kbo_params* p, cudaStream_t s);
int kbo_i_lml_batch(kbo_handle* h, const double* X_dev, const double* y_dev, int N, int D, int G, const kbo_params* params, double* lml_host,
                    int32_t* info_host, cudaStream_t s);
int kbo_i_lml_grad_batch(kbo_handle* h, const double* X_dev, const double* y_dev, int N, int D, int G, const kbo_params* params, double* lml_host,
                         double* grad_host, int32_t* info_host, cudaStream_t s);
size_t kbo_i_lml_grad_lane_bytes(int N, int D, int P);   // device memory one θ of kbo_lml_grad_batch takes
void kbo_i_lml_batch_free(kbo_handle* h);
void kbo_i_fit_partition_free(kbo_handle* h);
int kbo_i_fit_graph_nodes(kbo_handle* h, int32_t* counts);   // test hook: kernel nodes of the cached graph per context
int kbo_i_ensure_w(kbo_handle* h, cudaStream_t s);   // form the rest of W and the full planes if the fit left them out
int kbo_i_debug_rank_rows(kbo_handle* h, const void* Xc, int xc_dtype, int64_t M, int tile_pairs, float* mun_out, float* varn_out, cudaStream_t s);
// ---- lmlgrad.cu ---------------------------------------------------------------------------------
int kbo_i_lml_grad_from_w(kbo_handle* h, const double* Xs, int N, int D, int kind, double amp, double noise, const double* alpha,
                          const double* W, double* Wt, double* Kinv, int ld, int P, double* part, double* grad_dev, cudaStream_t s);
// ---- solve.cu ----------------------------------------------------------------------------------
int kbo_i_alpha_by_solves(kbo_handle* h, cudaStream_t s);
int kbo_i_variance_by_solves(kbo_handle* h, const double* Ks, int n, double* varn64, cudaStream_t s);
int kbo_i_zsolve_reserve(kbo_handle* h);
int kbo_i_zsolve_begin(kbo_handle* h, cudaStream_t s);
int kbo_i_zsolve_diag(kbo_handle* h, int K0, int Wd, cudaStream_t s);
int kbo_i_zsolve_update(kbo_handle* h, int K0, int Wd, cudaStream_t s);
// ---- sweep.cu ----------------------------------------------------------------------------------
int kbo_i_sweep(kbo_handle* h, const void* Xc_dev, int xc_dtype, int64_t M, int64_t goff, double* mu_out, double* std_out,
                double* acq_out, kbo_best* best_dev, cudaStream_t s);
int kbo_i_sweep_multi(kbo_handle* h, const void* Xc_dev, int xc_dtype, int64_t M, int64_t goff, int n_acq, const int32_t* acqs, kbo_best* best_dev,
                      cudaStream_t s);
int kbo_i_predict_mean(kbo_handle* h, const void* X_dev, int x_dtype, int n, double* mu_host, cudaStream_t s);
int kbo_i_debug_cross_planes(kbo_handle* h, const void* Xc, int xc_dtype, int64_t M, cudaStream_t s);   // FP64 K* → Ksh/Ksl, mun (test hook)
int kbo_i_acq_argmax_f32(kbo_handle* h, const float* mu_n, const float* var_n, int64_t M, int64_t goff, int acq, double y_mean,
                         double y_std, double y_opt, double xi, double kappa, double amp, float* acq_out, kbo_best* best_dev,
                         cudaStream_t s);
int kbo_i_encode_map_f16(kbo_handle* h, CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint32_t box_inner,
                         uint32_t box_outer);
// ---- tc_kstar.cu / tc_rank.cu ------------------------------------------------------------------
int kbo_i_tc_trials_prep(kbo_handle* h, bool new_center, cudaStream_t s);
// store_cols: leading columns of the plane actually written (-1: all); the mean always runs over every trial
int kbo_i_tc_kstar(kbo_handle* h, const void* Xc, int xc_dtype, int64_t rows, __half* Ksh, float* mun, cudaStream_t s, int store_cols = -1);
int kbo_i_tc_rank(kbo_handle* h, const __half* Ksh, int64_t rows, const __half* Wh, int Npad, double amp, float* var_n_out, cudaStream_t s,
                  int p_begin = 0, int p_end = -1);
// ---- tc_var.cu ---------------------------------------------------------------------------------
// var_n[m] = amp − Σ_j (Σ_k K*[m,k] W[j,k])²  for the rows of one chunk, on the wgmma tensor cores.
int kbo_i_tc_variance(kbo_handle* h, const __half* Ksh, const __half* Ksl, int64_t rows, const __half* Wh, const __half* Wl,
                      int Npad, double w_scale_inv, double amp, float* var_n_out, int k_span, cudaStream_t s, int nprod = 3, int jtiles = -1);
