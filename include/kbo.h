/*
 * kbo.h — C ABI of libkbo.so, the H100 (sm_90a) GP-suggestion engine.
 *
 * This is the drop-in boundary (SURVEY.md §8(b) "B-inner").  The reference platform repo
 * (/root/reference = kubeflow/kubeflow @ 6d6b78bc) reaches the suggestion service only through
 * Kubernetes (testing/katib_studyjob_test.py:155-161, testing/kfctl/kf_is_ready_test.py:65-70) and
 * holds no FFI for it; the arithmetic these entry points replace is the one Katib's
 * `bayesianoptimization` service executes (SURVEY.md §8(a), upstream kubeflow/katib
 * pkg/suggestion/v1beta1/skopt/base_service.py -> skopt.Optimizer.tell/ask ->
 * sklearn.gaussian_process.GaussianProcessRegressor).  Each entry point cites the
 * scikit-learn 1.9.0 lines ($SK = sklearn/gaussian_process) or the skopt function it replaces.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes; no C++/torch types.
 *   - every call returns KBO_OK (0) or a negative kbo_status; kbo_last_error(h) gives the text.
 *   - "dev" pointers are device memory owned by the caller (e.g. torch tensors), row-major,
 *     contiguous, 16-byte aligned.  The library never frees caller memory.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Calls are
 *     asynchronous on that stream unless the name ends in _host or the doc says "synchronises".
 *   - one handle per device per thread; a handle owns its workspace (grow-only device buffers).
 *   - there is NO CPU fallback: without a CUDA device kbo_create fails with KBO_ERR_CUDA.
 */
#ifndef KBO_H_
#define KBO_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KBO_VERSION 100 /* 0.1.0 */

typedef struct kbo_handle kbo_handle;

typedef enum kbo_status {
  KBO_OK = 0,
  KBO_ERR_INVALID = -1, /* bad argument (maps to gRPC INVALID_ARGUMENT)            */
  KBO_ERR_CUDA = -2,    /* CUDA runtime/driver error (maps to gRPC INTERNAL)       */
  KBO_ERR_NOT_PD = -3,  /* Cholesky met a non-positive pivot ($SK/_gpr.py:353-362) */
  KBO_ERR_NOMEM = -4,
  KBO_ERR_STATE = -5    /* sweep before fit, etc.                                   */
} kbo_status;

typedef enum kbo_kernel_kind {
  KBO_KERNEL_RBF = 0,     /* $SK/kernels.py:1559-1570 */
  KBO_KERNEL_MATERN52 = 1 /* $SK/kernels.py:1713-1729 (nu = 2.5; skopt's default GP kernel) */
} kbo_kernel_kind;

typedef enum kbo_acq_kind {
  KBO_ACQ_EI = 0,  /* skopt.acquisition.gaussian_ei  */
  KBO_ACQ_LCB = 1, /* skopt.acquisition.gaussian_lcb (value reported is -(mu - kappa*sigma)) */
  KBO_ACQ_PI = 2   /* skopt.acquisition.gaussian_pi  */
} kbo_acq_kind;

typedef enum kbo_var_mode {
  KBO_VAR_F64 = 0,     /* variance contraction V = K* W^T on the FP64 SIMT pipe (checker precision) */
  KBO_VAR_TC_F16X3 = 1, /* wgmma tensor cores, fp16 hi/lo split (3 MMAs per product), fp32 accum */
  KBO_VAR_AUTO = 2      /* FP64 while M·N² <= 2e11 (a few ms of FP64 pipe), tensor cores above that    */
} kbo_var_mode;

typedef enum kbo_dtype { KBO_F64 = 0, KBO_F32 = 1 } kbo_dtype;

/* Fixed hyper-parameters θ and acquisition settings of one tell/ask (SURVEY.md §7 "parity at fixed θ"). */
typedef struct kbo_params {
  int32_t kernel;          /* kbo_kernel_kind */
  int32_t acq;             /* kbo_acq_kind */
  int32_t normalize_y;     /* 1 = $SK/_gpr.py:275-280 */
  int32_t var_mode;        /* kbo_var_mode */
  double amplitude;        /* ConstantKernel value ($SK/kernels.py:1278) */
  double noise;            /* GaussianProcessRegressor.alpha, added to diag(K) ($SK/_gpr.py:350) */
  double xi;               /* EI / PI offset (skopt default 0.01) */
  double kappa;            /* LCB weight (skopt default 1.96) */
  const double* length_scale; /* HOST pointer, n_length_scale entries */
  int32_t n_length_scale;  /* 1 (isotropic) or D (anisotropic) */
  int32_t tc_k_span;       /* TC mode: trials accumulated by the tensor cores before a drain into a second fp32 register sum; 0 = default */
} kbo_params;

/* Result of one sweep: best acquisition value and its GLOBAL candidate index (lowest index wins ties,
 * = np.argmin(-values) in skopt Optimizer._tell), with the posterior at that point (raw y scale). */
typedef struct kbo_best {
  double value;
  int64_t index;
  double mu;
  double std;
} kbo_best;

/* Timings of the last kbo_suggest_host call, milliseconds (CUDA events on the call's stream). */
typedef struct kbo_timings {
  float h2d_ms, fit_ms, sweep_ms, d2h_ms, total_ms;
  float var_kernel_ms;   /* sum over chunks of the variance-contraction kernel */
  float cross_kernel_ms; /* sum over chunks of the K* / mean kernel           */
  float acq_kernel_ms;   /* acquisition + argmax kernels                      */
  int32_t launches;      /* kernels launched by the call                      */
  int32_t chunks;
  float calib_ms;        /* ranking pass: the stratified calibration rows (FP64 K* + three-product contraction) */
} kbo_timings;

int kbo_version(void);
int kbo_create(kbo_handle** out, int device);
void kbo_destroy(kbo_handle* h);
const char* kbo_last_error(const kbo_handle* h);
/* cap (bytes) on the per-sweep K* scratch; default 4 GiB.  Determines the candidate chunk size (rounded down to a
 * multiple of sm_count*128 rows so every launch is a whole number of waves).  Also caps the lane memory of one
 * kbo_lml_grad_batch call. */
int kbo_set_scratch_limit(kbo_handle* h, uint64_t bytes);
/* Tensor-core mode re-evaluates on the FP64 path every candidate whose fp32 acquisition value is within 2e-4 of the maximum
 * (at most 4096 of them) and takes the first-index argmax over those FP64 values, so the returned suggestion (index, value,
 * mu, std) has FP64 accuracy; this costs one extra pass over (mu, sigma²) and one stream synchronisation.
 * kbo_last_contenders returns how many candidates the last sweep refined (> 4096: refinement skipped). */
int kbo_last_contenders(kbo_handle* h);
/* Tensor-core sweeps that return only the suggestion (no mu/std/acq arrays) rank the grid with ONE fp16 product per term —
 * a third of the MMAs — and keep every candidate that could still be the maximum given that pass's error on sigma²
 * (calibrated per sweep against the three-product kernel on sm_count·64 rows stratified over the grid, x8 + 1e-6); the survivors are decided
 * by the FP64 refinement above, so the returned suggestion is unchanged.  More than 4096 survivors: the sweep is redone
 * with three products.  Default on.  kbo_last_rank_error returns the
 * largest |sigma²(1 product) - sigma²(3 products)| seen on the calibration rows of the last such sweep. */
int kbo_set_tc_fast(kbo_handle* h, int enabled);
double kbo_last_rank_error(kbo_handle* h);
/* The ranking pass builds its K* plane on the tensor cores (c·x as wgmma MMAs of fp16 hi/lo splits, kernel values in fp32,
 * only the hi plane written, the mean accumulated on the fly) and contracts it with wgmma m64n256k16 MMAs; 0 selects the FP64 K*
 * kernel + single-CTA-MMA cluster kernel of round 1 for that pass.  Default 1 (needs D <= 128; wider spaces use the FP64
 * kernel).  Either way the calibration rows are STRATIFIED over the grid (row i*M/n) and go through the FP64 K* kernel and
 * the three-product contraction; kbo_last_rank_mu_error is the largest |mean(ranking) - mean(FP64)| seen on them, in
 * normalised-y units (0 with the FP64 K* kernel). */
int kbo_set_rank_tc(kbo_handle* h, int enabled);
double kbo_last_rank_mu_error(kbo_handle* h);
/* Pruning pass in front of the ranking pass (needs kbo_set_rank_tc).  sigma² = amp - sum_j v_j² with every term >= 0, so the sum
 * over a PREFIX of the trial tiles bounds sigma² from above, and with it EI / LCB (they grow with sigma; PI is bounded by 1 where
 * the improvement is positive) — at the prefix's share of the triangular contraction: the first eighth of the trials costs 1/64
 * of the MMAs.  The calibration rows' (near-exact) values give a lower bound on the maximum for free.  Candidates whose upper
 * bound stays below it are out; the rest (at most 16384, else the full ranking pass runs as before) get the full contraction,
 * the interval test and the FP64 decision.  tile_pairs: 512-trial tile pairs in the prefix; -1 (default) = an eighth of them,
 * 0 = no pruning pass.  kbo_last_prefix_survivors: how many candidates the last pruning pass kept (-1: it did not run). */
int kbo_set_rank_prefix(kbo_handle* h, int tile_pairs);
/* Lazy inverse (default on).  A tensor-core fit whose sweeps will prune forms only the rows of W = L^-1 the pruning pass reads
 * (the first 512·tile_pairs; plus the 256×256 diagonal blocks of every panel, which the look-ahead factorisation needs anyway):
 * alpha comes from two panel solves with L, the survivors' exact variances from panel solves with L (solve.cu), the lower bound
 * on the maximum from the sigma -> 0 limit of the acquisition function.  N³/3 FP64 flop — a third of the fit — are not spent.
 * The rest of W (and the full fp16 planes) are formed on demand by anything that needs them: array-returning sweeps, FP64-mode
 * sweeps, kbo_fit_append / kbo_fit_rebase, kbo_lml_grad, kbo_fit_state, and the sweep itself when more than 64 candidates
 * pass the prefix bound.  0 = always form W in kbo_fit.  Results do not depend on the setting beyond FP64 rounding. */
int kbo_set_lazy_inverse(kbo_handle* h, int enabled);
int kbo_last_prefix_survivors(kbo_handle* h);
/* How the last tensor-core sweep decided its suggestion: 0 = FP64 evaluation of every candidate that could still be the
 * maximum; 1 = more such candidates than the cap (4096), FP64 decision among the best 4096 by fp32 value; 2 = not refined
 * (exact fp32 ties beyond the cap, or a grid of 2^31 or more rows): the suggestion carries the mode's own accuracy. */
int kbo_last_unrefined(kbo_handle* h);

/* ---- tell: GaussianProcessRegressor.fit at fixed θ ($SK/_gpr.py:275-280, 349-368) ---------------
 * X: N×D fp64, y: N fp64, device pointers (x_on_host = 0) or host pointers (x_on_host = 1).
 * Computes X/ℓ, normalised y, K = amp·k(X,X)+noise·I, L = chol(K), W = L^-1, alpha = W^T W y, LML, and
 * (TC mode) the fp16 hi/lo split of W.  All on the device; asynchronous on `stream` except that a
 * non-positive pivot is reported by the next synchronising call (kbo_fit_info / kbo_best_to_host). */
int kbo_fit(kbo_handle* h, const double* X, const double* y, int32_t N, int32_t D, const kbo_params* p,
            int x_on_host, void* stream);
/* Append ONE trial (x: D doubles, y) to the fitted history at the same theta without refactorising: the bordered Cholesky
 * row l = W k, d = sqrt(amp + noise - l.l), the matching row of W = L^-1, then the y statistics, alpha, LML and the fp16
 * planes are brought up to date — O(N^2) instead of O(N^3) (SURVEY.md 8(f)2: skopt's constant-liar `ask(n_points=k)` tells
 * k-1 lies one after another, `Optimizer.tell` refits each time).  Works in place up to the row pitch of the last kbo_fit
 * (its N rounded up to 64).  kbo_fit_rebase keeps that pitch, so after a rebase to n_keep up to pitch - n_keep rows can be
 * appended on the same factorisation, not just the rest of one 64-row block.  kbo_fit_room() says how many more trials can
 * be appended (0: call kbo_fit with the whole history).  Not positive definite
 * is reported by kbo_fit_info like after a fit; the handle then needs a kbo_fit.  Results equal a refit's to ~1e-12. */
int kbo_fit_append(kbo_handle* h, const double* x, double y, int x_on_host, void* stream);
int kbo_fit_room(kbo_handle* h);
/* Keep the first n_keep trials of the fitted history, optionally with new targets y[0..n_keep) (NULL: unchanged).  The
 * leading blocks of L and L^-1 are the factors of the shorter history and y enters only through yn / alpha / LML, so this is
 * O(N^2): it drops constant-liar rows before the real trials are appended and replaces a lie by the observed value.
 * After a non-positive pivot p (kbo_fit_info's info) the rebase recovers only if every kept row was factored: after a failed
 * kbo_fit_append, n_keep <= p - 1; after a failed kbo_fit, n_keep <= 64*floor((p - 1)/64), because the fit stops at the
 * failing 64-row block as a whole.  A rebase into that block keeps reporting KBO_ERR_NOT_PD: the shorter history needs a
 * kbo_fit. */
int kbo_fit_rebase(kbo_handle* h, int32_t n_keep, const double* y, int y_on_host, void* stream);

/* synchronises; any out pointer may be NULL.  info = 0 or 1-based index of the failed pivot. */
int kbo_fit_info(kbo_handle* h, double* lml, double* y_mean, double* y_std, double* y_opt, int32_t* info,
                 void* stream);
/* Gradient of the log-marginal likelihood of the last kbo_fit w.r.t. θ = (log amplitude, log noise, log ℓ_1..ℓ_P), P =
 * n_length_scale of that fit ($SK/_gpr.py:621-653).  grad_host: n_out = 2 + P doubles.  Synchronises.  KBO_ERR_NOT_PD
 * (grad_host then holds no gradient) if that fit met a non-positive pivot. */
int kbo_lml_grad(kbo_handle* h, double* grad_host, int32_t n_out, void* stream);
/* Log-marginal likelihood of G hyper-parameter settings over ONE history (X, y as for kbo_fit), for theta search: what sklearn's
 * optimiser evaluates one theta after another ($SK/_gpr.py:299-339, :604-618, :658-667).  The G factorisations run on G streams
 * and hide each other's latency (a Cholesky of a few thousand trials is a chain of single-CTA blocks): 8 thetas cost about two
 * fits.  Per theta: Gram, Cholesky, z = L^-1 yn by forward substitution, LML = -z.z/2 - sum log L_ii - N/2 log 2pi.  Does not
 * touch the handle's fitted state.  params: G entries (kernel, amplitude, noise, length_scale, n_length_scale, normalize_y of
 * entry 0 used); lml_host: G doubles (-inf where the Gram matrix is not positive definite); info_host (may be NULL): G failed
 * pivots (0 = ok).  Synchronises.  1 <= G <= 64. */
int kbo_lml_batch(kbo_handle* h, const double* X, const double* y, int32_t N, int32_t D, int32_t G, const kbo_params* params,
                  int x_on_host, double* lml_host, int32_t* info_host, void* stream);
/* Log-marginal likelihood AND its gradient for G hyper-parameter settings over ONE history, for gradient-based theta fitting
 * with several starts in lockstep: what sklearn's L-BFGS-B asks of log_marginal_likelihood(theta, eval_gradient=True) once
 * per start and iteration ($SK/_gpr.py:541-655).  Arguments as kbo_lml_batch; every entry must have the same n_length_scale P.
 * Per theta, on its own stream: Gram, Cholesky, W = L^-1, alpha = W^T W yn, the LML, K^-1 = W^T W and the kbo_lml_grad
 * gradient.  grad_host: G x (2 + P) doubles, row g in kbo_lml_grad's order (log amplitude, log noise, log l_1..l_P).  A theta
 * whose Gram matrix is not positive definite gets lml = -inf, a zero gradient and its pivot in info_host; the others are
 * unaffected.  Each theta's (lml, gradient) is bit-identical whatever batch or position it is computed in.  Memory: about
 * 3 * 8 * ld^2 bytes per theta (ld = N rounded up to 64; 1.5 GiB at N = 8192), kept by the handle for the next call; a batch
 * needing more than kbo_set_scratch_limit fails with KBO_ERR_INVALID (naming the bytes needed) before any work.  Does not
 * touch the handle's fitted state.  Synchronises.  1 <= G <= 64, 1 <= D <= 512, N <= 25600. */
int kbo_lml_grad_batch(kbo_handle* h, const double* X, const double* y, int32_t N, int32_t D, int32_t G, const kbo_params* params,
                       int x_on_host, double* lml_host, double* grad_host, int32_t* info_host, void* stream);
/* copies the fit state into caller-owned DEVICE buffers (any may be NULL): L_out, W_out are N×N row-major
 * (L: lower Cholesky factor, strict upper part zeroed; W = L^-1), alpha_out has N entries. For parity tests. */
int kbo_fit_state(kbo_handle* h, double* L_out, double* W_out, double* alpha_out, void* stream);

/* ---- ask: predict(return_std) + acquisition + first-index argmax over M candidates ---------------
 * ($SK/_gpr.py:445-500; skopt gaussian_ei/lcb/pi; Optimizer._tell `X_cand[np.argmin(values)]`).
 * Xc: M×D, dtype xc_dtype, device (xc_on_host=0) or host.  global_offset is added to reported indices
 * (the rank's row offset when the grid is sharded, SURVEY.md §8(e)).
 * Optional device outputs (NULL to skip): mu_out, std_out, acq_out — fp64, M entries each.
 * best_dev: device kbo_best written at the end of the stream work. */
int kbo_sweep(kbo_handle* h, const void* Xc, int32_t xc_dtype, int64_t M, int64_t global_offset, int xc_on_host,
              double* mu_out, double* std_out, double* acq_out, kbo_best* best_dev, void* stream);
/* Several acquisitions over ONE candidate grid, as skopt's gp_hedge evaluates EI, LCB and PI on the same candidates.
 * acqs: n_acq (1-3) distinct kbo_acq_kind values, host memory; best_dev: n_acq device kbo_best.  best_dev[i] is what kbo_sweep
 * with acq = acqs[i] returns on the same fit and grid.  The posterior (calibration rows, K* planes, contractions, mean) is
 * computed once per stage for every acquisition still undecided; each acquisition keeps its own bounds, survivor lists and FP64
 * decision and finishes at the first stage where its own list fits — where its single sweep would have.  Array-free.
 * The FP64 decisions a stage takes are one evaluation over the union of those kinds' survivors.
 * Duplicate or unknown kinds: KBO_ERR_INVALID.  kbo_last_decisions reports each kind's decision; kbo_last_unrefined,
 * kbo_last_contenders, kbo_last_prefix_survivors, kbo_last_rank_error and kbo_last_rank_mu_error keep reporting the last
 * kbo_sweep. */
int kbo_sweep_multi(kbo_handle* h, const void* Xc, int32_t xc_dtype, int64_t M, int64_t global_offset, int xc_on_host, int32_t n_acq,
                    const int32_t* acqs, kbo_best* best_dev, void* stream);
/* Per acquisition of the last kbo_sweep (one) or kbo_sweep_multi (n_acq, in request order): what kbo_last_unrefined,
 * kbo_last_contenders and kbo_last_prefix_survivors report for a single sweep.  Fills up to n entries of each non-NULL array;
 * returns the number of acquisitions the last sweep decided. */
int kbo_last_decisions(kbo_handle* h, int32_t n, int32_t* unrefined, int32_t* contenders, int32_t* prefix_survivors);
/* FP64 posterior mean (raw y scale) at n points X (n×D, dtype x_dtype, device or host): K*·alpha as the sweep's FP64
 * refinement forms it.  Needs alpha only — a lazy fit's inverse is not formed.  mu_out_host: n doubles.  Synchronises. */
int kbo_predict_mean(kbo_handle* h, const void* X, int32_t x_dtype, int32_t n, int x_on_host, double* mu_out_host, void* stream);
/* synchronises `stream`, copies *best_dev to host, and returns KBO_ERR_NOT_PD if the fit failed. */
int kbo_best_to_host(kbo_handle* h, const kbo_best* best_dev, kbo_best* best_host, void* stream);

/* ---- multi-GPU: the grid shards by rows, one exchange step (SURVEY.md 8(e)) ---------------------------------------------
 * One process (or thread) per GPU, one handle each.  Rank r sweeps rows [lo_r, hi_r) of the grid with global_offset = lo_r;
 * kbo_allreduce_argmax then replaces *best_dev on every rank by the global first-index argmax (maximum value, lowest global
 * index among equals = np.argmin(-values) over the concatenated grid): ONE ncclAllGather of 32 bytes per rank on `stream`
 * plus a one-thread reduce.  NCCL is bound at run time (dlopen libnccl.so.2): kbo_comm_unique_id on one rank gives the
 * 128-byte ncclUniqueId the caller distributes by any means (the gRPC SPMD server broadcasts it); kbo_comm_init is
 * collective over the n_ranks handles.  Without a communicator (or with one rank) kbo_allreduce_argmax is a no-op. */
#define KBO_COMM_ID_BYTES 128
int kbo_comm_unique_id(void* id_out /* KBO_COMM_ID_BYTES */);
int kbo_comm_init(kbo_handle* h, int32_t n_ranks, int32_t rank, const void* id /* KBO_COMM_ID_BYTES */);
int kbo_comm_destroy(kbo_handle* h);
int kbo_comm_size(kbo_handle* h);
int kbo_allreduce_argmax(kbo_handle* h, kbo_best* best_dev, void* stream);

/* ---- one call, HOST buffers in, host result out (tell + ask); synchronises -----------------------
 * The end-to-end entry: H2D of X, y, Xc and D2H of the result are inside the call.  With a communicator (kbo_comm_init) the
 * call is collective: every rank passes its row block and global_offset, and best_host is the global argmax on every rank. */
int kbo_suggest_host(kbo_handle* h, const double* X, const double* y, int32_t N, int32_t D, const void* Xc,
                     int32_t xc_dtype, int64_t M, int64_t global_offset, const kbo_params* p,
                     kbo_best* best_host, kbo_timings* timings /* may be NULL */);
int kbo_last_timings(kbo_handle* h, kbo_timings* out);

/* ---- building blocks, caller-owned device memory (used by the parity tests one kernel at a time) --
 * kbo_gram:  K (N×ldk, fp64) = amplitude·k(Xs,Xs) + noise·I, Xs already divided by ℓ. ($SK/kernels.py:1561,1716)
 * kbo_potrf: in-place lower Cholesky of A (N×lda); the strict upper triangle is scratch afterwards; info_dev = 0 or failed pivot. ($SK/_gpr.py:352)
 * kbo_trtri: W (N×ldw, zero upper) = L^-1 for lower-triangular L.  Needs the potrf of the same handle just before
 *            (reuses its inverted diagonal blocks).
 * kbo_acq_argmax: standalone acquisition + argmax pass over (mu, var) in the NORMALISED y scale:
 *            mu_n, var_n fp32 (8 B/candidate read) -> optional acq fp32 (4 B write) + best. The HBM-bound kernel
 *            whose GB/s the headline metric asks for.  y_std must be finite and > 0 (KBO_ERR_INVALID otherwise):
 *            the values are ranked in units of y_std. */
int kbo_gram(kbo_handle* h, const double* Xs, int32_t N, int32_t D, int32_t kernel, double amplitude, double noise,
             double* K, int32_t ldk, void* stream);
int kbo_potrf(kbo_handle* h, double* A, int32_t N, int32_t lda, int32_t* info_dev, void* stream);
int kbo_trtri(kbo_handle* h, const double* L, int32_t N, int32_t ldl, double* W, int32_t ldw, void* stream);
int kbo_acq_argmax(kbo_handle* h, const float* mu_n, const float* var_n, int64_t M, int64_t global_offset,
                   int32_t acq, double y_mean, double y_std, double y_opt, double xi, double kappa,
                   float* acq_out, kbo_best* best_dev, void* stream);

/* ---- request ingestion (host only; SURVEY.md 8(f)3) -------------------------------------------------------------------
 * A serialized api.v1.beta1.GetSuggestionsRequest (kubeflow/katib pkg/apis/manager/v1beta1/api.proto; what grpc hands the
 * suggestion service before `GetSuggestionsRequest.FromString`) scanned into flat arrays, replacing the walk over the parsed
 * message that katib's pkg/suggestion/v1beta1/internal/trial.py `Trial.convert` + skopt/base_service.py `getSuggestions`
 * do per request.  `bytes` must stay alive while the kbo_req is open; offsets are relative to it.
 * kbo_req_trials fills one row per trial (any output pointer may be NULL), n_params columns in the order of param_names:
 *   usable          condition SUCCEEDED/EARLYSTOPPED and the objective metric present (Trial.convert's filter)
 *   objective       strtod of the objective metric value; objective_flags bit0 = plain decimal literal (else NaN)
 *   values / flags  strtod of the assignment; bit0 = plain decimal literal, bit1 = integer literal (<= 15 digits);
 *                   value_len 0xFFFFFFFF = the trial has no assignment of that name
 * Values that are not plain literals are left to the caller (Python float()/int() semantics, categorical strings).
 * select (NULL = all): per-trial mask; assignments of unselected trials are not looked at (their rows read as missing) —
 * a steady request parses numbers only for the trials the service has not seen (strtod dominates the scan). */
typedef struct kbo_req kbo_req;
int kbo_req_open(const void* bytes, uint64_t len, kbo_req** out);
void kbo_req_close(kbo_req* r);
int kbo_req_header(const kbo_req* r, uint64_t* experiment_off, uint64_t* experiment_len, int32_t* current_request_number,
                   int32_t* total_request_number, int32_t* n_trials);
int kbo_req_trials(const kbo_req* r, int32_t n_params, const char* const* param_names, uint64_t* name_off, uint32_t* name_len,
                   uint64_t* name_hash, int32_t* condition, uint8_t* usable, double* objective, uint8_t* objective_flags,
                   uint64_t* objective_off, uint32_t* objective_len, double* values, uint8_t* value_flags, uint64_t* value_off,
                   uint32_t* value_len, const uint8_t* select);
uint64_t kbo_hash64(const void* bytes, uint64_t len);   /* the FNV-1a hash kbo_req_trials puts in name_hash */

/* ---- CMA-ES (Katib algorithm `cmaes`, goptuna; N. Hansen's tutorial arXiv:1604.00772, active weights) ---------------
 * State (mean, sigma, C, evolution paths, eigenbasis) lives on the device.  One generation = ask + tell:
 *   kbo_cma_ask : X (lambda×D, device, fp64) = m + sigma·B·(d∘z); z from the built-in Philox stream (seed, generation) or,
 *                 for parity tests, from z_in_dev (lambda×D device, may be NULL).
 *   kbo_cma_tell: fitness (lambda, device, minimised) for the X of the last ask → rank-μ/rank-1 covariance update,
 *                 step-size control and a warm-started Jacobi eigendecomposition C = B diag(d²) Bᵀ.
 *                 Ranking is NumPy's sort order: -inf < finite < +inf < NaN, -0 == +0, every NaN equal (a diverged trial
 *                 that reports nan ranks last, after inf); ties → lower sample index.
 *                 d_j² is the eigenvalue λ_j itself (b_jᵀ C b_j); only λ_j ≤ 0 is replaced, by 1e-8.
 *                 Every tell ends with the termination test of CyberAgent `cmaes` (should_stop) on the updated state, on the
 *                 device: the generation's best and worst fitness go to slot 2·(g mod term) of a history ring of 2·term
 *                 doubles (term = 10 + ⌈30·D/lambda⌉, g = strategy generation after the tell), and six criteria set bits:
 *                 TOLFUN=1 (g > term and max−min of the history < 1e-12), TOLX=2 (all σ·C_ii and σ·p_c,i < 1e-12·σ0),
 *                 TOLXUP=4 (σ·max d > 1e4), NOEFFECTCOORD=8 (some m_i == m_i + 0.2σ·√C_ii), NOEFFECTAXIS=16
 *                 (m == m + 0.1σ·d_i·b_i, i = g mod D, b_i column i of this library's Jacobi basis), CONDITIONCOV=32
 *                 (max d / min d > 1e14).  NaN anywhere in a criterion's operands makes it false, as in NumPy.
 * The built-in Philox stream is keyed by a draw counter that advances once per tell and is never reset (without a
 * restart it equals the generation), so the draws of a restarted run never repeat earlier ones.
 * Limits: 1 <= D <= 128, 4 <= lambda <= 8192.  kbo_cma_state copies to HOST buffers (any may be NULL) and synchronises;
 * its `generation` is the strategy generation of the current run.
 * kbo_cma_stop_flags copies the flags word (0 before the first tell of a run) and, if funhist_host is given, the 2·term
 * history, writes term, and synchronises.
 * kbo_cma_restart starts a new run in place (IPOP / BIPOP restarts): population lambda (buffers grow as needed, weights
 * and constants are recomputed), mean0_host, sigma0, C = B = I, d = 1, zero paths, history and flags, strategy generation
 * 0.  Same limits and error codes as kbo_cma_create; after a failed restart the instance may only be destroyed.
 * kbo_cma_run_synthetic runs `generations` ask/fitness/tell rounds entirely on the device with a built-in fitness
 * (0 = sphere, 1 = Rastrigin) — the BASELINE.json config-4 benchmark.
 * kbo_cma_set_margin turns on CMA-ES with Margin (CMAwM, Hamano et al. GECCO 2022, as in CyberAgent `cmaes`) for
 * n_discrete dimensions dims[] (increasing).  Dimension dims[i] has the sorted levels levels[level_offsets[i],
 * level_offsets[i+1]) (2 or more, increasing; level_offsets has n_discrete + 1 entries from 0) or, when that range is
 * empty, the arithmetic levels first + k·step, k < count, from arith[3i .. 3i+2] = (first, step, count).  alpha is the
 * margin α in (0, 1), or 0 for 1/(D·lambda), recomputed at every restart.  Then kbo_cma_ask returns x = m + σ·(A∘y) with
 * each discrete coordinate encoded to its level (the interval (ℓ_{k−1}, ℓ_k] of thresholds ℓ_k = (v_k + v_{k+1})/2 that
 * holds it); the tell's mean step is m + c_m·σ·A∘y_w, and after the eigendecomposition a one-CTA kernel corrects m_j and
 * A_j of each discrete dimension (oracle/cma_margin_oracle.py).  A starts at 1 and a restart resets it.  n_discrete = 0
 * turns the margin off: every kernel is then the margin-free one.  Not between an ask and its tell (KBO_ERR_STATE).
 * kbo_cma_margin_state copies A, the mean before the last correction and α to HOST (any may be NULL) and synchronises.
 * Margin dimensions are refused (KBO_ERR_INVALID) while learning-rate adaptation is on.
 * kbo_cma_set_lr_adapt turns learning-rate adaptation on (on != 0) or off (LRA-CMA-ES, Nomura, Akimoto & Ono, GECCO 2023,
 * as in CyberAgent `cmaes`; oracle/cma_lra_oracle.py).  Each tell then blends the plain update with the state it started
 * from: m ← m + η_m·Δm, Σ ← σ²C + η_Σ·ΔΣ, with η_m and η_Σ in (0, 1] driven by the signal-to-noise ratios of moving
 * averages of Δm and ΔΣ in the local coordinates Σ^{-1/2}; σ is taken from log det Σ so that det C = 1, then scaled by
 * η_m(before)/η_m(after).  Turning it on or off resets E = V = 0 and η = 1, and so does every restart.  Not between an
 * ask and its tell (KBO_ERR_STATE); refused with margin dimensions set (KBO_ERR_INVALID).  Off, no LRA work is done.
 * kbo_cma_lra_state copies E_m (D), E_Σ (D×D), V = (V_m, V_Σ) and eta = (η_m, η_Σ) to HOST (any may be NULL) and
 * synchronises; KBO_ERR_STATE while the adaptation is off. */
typedef struct kbo_cma kbo_cma;
int kbo_cma_create(kbo_handle* h, kbo_cma** out, int32_t D, int32_t lambda, const double* mean0_host, double sigma0, uint64_t seed);
void kbo_cma_destroy(kbo_cma* c);
int kbo_cma_ask(kbo_handle* h, kbo_cma* c, double* X_dev, const double* z_in_dev, void* stream);
int kbo_cma_tell(kbo_handle* h, kbo_cma* c, const double* fitness_dev, void* stream);
int kbo_cma_state(kbo_handle* h, kbo_cma* c, double* mean, double* sigma, double* C, double* p_sigma, double* p_c, double* B,
                  double* d, double* Y_last, int64_t* generation, void* stream);
int kbo_cma_stop_flags(kbo_handle* h, kbo_cma* c, uint32_t* flags_host, double* funhist_host, int32_t* term_host, void* stream);
int kbo_cma_restart(kbo_handle* h, kbo_cma* c, int32_t lambda, const double* mean0_host, double sigma0);
int kbo_cma_run_synthetic(kbo_handle* h, kbo_cma* c, int32_t fitness_kind, int32_t generations, double* best_f_host,
                          float* elapsed_ms, double* jacobi_sweeps_last);
int kbo_cma_set_margin(kbo_handle* h, kbo_cma* c, int32_t n_discrete, const int32_t* dims, const int64_t* level_offsets,
                       const double* levels, const double* arith, double alpha);
int kbo_cma_margin_state(kbo_handle* h, kbo_cma* c, double* A_host, double* mean_before_host, double* alpha_host, void* stream);
int kbo_cma_set_lr_adapt(kbo_handle* h, kbo_cma* c, int32_t on);
int kbo_cma_lra_state(kbo_handle* h, kbo_cma* c, double* E_mean_host, double* E_Sigma_host, double* V_host, double* eta_host,
                      void* stream);

/* ---- separable CMA-ES (`cmaes` with use_separable_cma; Ros & Hansen, PPSN 2008, as CyberAgent `cmaes`' SepCMA) ------
 * A separate object from kbo_cma: C is kept as its diagonal and d = √C, so sampling and update are O(lambda·D) and no D×D
 * object exists (oracle/sepcma_oracle.py states each rule).  Positive recombination weights only (μ = ⌊lambda/2⌋);
 * c_c = 4/(D+4), c1 = 2/((D+1.3)² + μ_eff) and the rank-μ rate scaled by (D+2)/3, capped at 1 − c1 − 1e-8.
 *   kbo_sepcma_ask : X (lambda×D, device, fp64) = m + sigma·(d∘z); z from the built-in Philox stream (the same convention
 *                    and never-reset draw counter as kbo_cma_ask) or from z_in_dev (lambda×D device, may be NULL).
 *   kbo_sepcma_tell: fitness (lambda, device, minimised, ranked in kbo_cma_tell's NumPy order) for the X of the last ask →
 *                    mean, p_σ, σ (capped at 1e32), h_σ, p_c, C and d = √C (C_j <= 0 floored at 1e-8 under the root).  It
 *                    ends with kbo_cma_tell's termination test without NOEFFECTAXIS (bit 16 is never set): TOLFUN, TOLX
 *                    (all σ·C_j and σ·p_c,j < 1e-12·σ0), TOLXUP, NOEFFECTCOORD (some m_j == m_j + 0.2σ·√C_j), CONDITIONCOV.
 * Limits: 1 <= D <= 4096, 4 <= lambda <= 8192.  kbo_sepcma_state copies mean, sigma, the diagonal C_diag, p_sigma, p_c, d and
 * the last ask's steps Y (lambda×D) to HOST buffers (any may be NULL) and synchronises; `generation` is the strategy
 * generation of the current run.  kbo_sepcma_stop_flags and kbo_sepcma_restart behave as kbo_cma_stop_flags and
 * kbo_cma_restart (restart: C = d = 1, zero paths, history and flags, generation 0; the draw counter goes on). */
typedef struct kbo_sepcma kbo_sepcma;
int kbo_sepcma_create(kbo_handle* h, kbo_sepcma** out, int32_t D, int32_t lambda, const double* mean0_host, double sigma0, uint64_t seed);
void kbo_sepcma_destroy(kbo_sepcma* c);
int kbo_sepcma_ask(kbo_handle* h, kbo_sepcma* c, double* X_dev, const double* z_in_dev, void* stream);
int kbo_sepcma_tell(kbo_handle* h, kbo_sepcma* c, const double* fitness_dev, void* stream);
int kbo_sepcma_state(kbo_handle* h, kbo_sepcma* c, double* mean, double* sigma, double* C_diag, double* p_sigma, double* p_c, double* d,
                     double* Y_last, int64_t* generation, void* stream);
int kbo_sepcma_stop_flags(kbo_handle* h, kbo_sepcma* c, uint32_t* flags_host, double* funhist_host, int32_t* term_host, void* stream);
int kbo_sepcma_restart(kbo_handle* h, kbo_sepcma* c, int32_t lambda, const double* mean0_host, double sigma0);

/* ---- TPE (Katib algorithm `tpe`: hyperopt's tpe.suggest on a flat space; FP64 restatement oracle/tpe_oracle.py) -------
 * Parameter kinds: UNIFORM = uniform(lo, hi); QUNIFORM = quniform(lo, hi, q), values rint(x/q)·q; CHOICE = choice over
 * `levels` categories, observed and reported as the category index.
 *   kbo_tpe_create: D parameters (HOST arrays kinds, lo, hi, q, levels; lo/hi/q are read for numeric kinds, levels for
 *                   choices), gamma in (0, 1), prior_weight > 0, seed (random_state).
 *   kbo_tpe_tell  : appends n_new trials in told order: X (n_new×D, parameter units) and losses (minimised; non-finite losses
 *                   rank in NumPy's order, NaN last).  Device pointers, or host pointers with on_host = 1 (then synchronises).
 *   kbo_tpe_ask   : k points, each with its own n_candidates draws per parameter from the below model (Philox4x32-10 keyed by
 *                   (seed, ask counter, point, parameter, candidate)), or the caller's candidates cand_dev (k×D×n_candidates,
 *                   device, fp64: numeric values before quantization, category indices for choices).  Each parameter takes
 *                   the candidate at the first index of the maximum of log l(x) - log g(x); continuous parameters are scored
 *                   in FP32 with an error bound and every candidate that can still be the maximum is decided in FP64;
 *                   quantized and categorical parameters score each distinct value present once, in FP64.
 *                   x_dev: k×D fp64 suggestions (device); optional device outputs: idx_dev (k×D winning candidate indices),
 *                   cand_out_dev (k×D×n_candidates: the draws), score_out_dev (k×D×n_candidates×2 floats: FP32 score and
 *                   its bound, continuous parameters only).  Synchronises.  1 <= n_candidates <= 2^24, k·D <= 65535.
 *   kbo_tpe_state : the models of the current history (built on demand), HOST outputs, any may be NULL: for a numeric
 *                   parameter the group's (0 below, 1 above) mixture weights, means, sigmas (first cap of ncomp components) and
 *                   p_accept; for a choice the group's category probabilities (w, ncomp = categories).  Synchronises.
 *   kbo_tpe_last_survivors: per (point, parameter) of the last ask, the candidates decided in FP64 (continuous) or the
 *                   distinct values scored (quantized, categorical).  Returns k·D, fills up to n entries.
 *   kbo_tpe_last_timings: milliseconds of the last ask's phases (models, FP32 score, FP64 decision, discrete parameters, final
 *                   reduction), CUDA events on its stream.  Returns 5, fills up to n entries.
 *   kbo_tpe_ask_shard: one shard of an ask sharded over ranks: as kbo_tpe_ask, but only candidates [lo, hi) of n_candidates
 *                   are drawn (keyed by their global index) and scored; quantized and categorical parameters score the
 *                   distinct values present in the shard.  Per (point, parameter) it writes the shard's winner to val_dev
 *                   (k×D fp64, device: its FP64 score) and idx_dev (k×D, device: its global index).  lo == hi is an empty
 *                   shard, which writes (-inf, n_candidates) and never wins.  The ask counter advances as one kbo_tpe_ask
 *                   advances it.  cand_dev must be NULL.  Synchronises.  The exchange of (value, index) pairs is the
 *                   caller's: the first index of the maximum over all shards is the winner one kbo_tpe_ask would pick.
 *   kbo_tpe_pick  : after a shard ask and before the next tell, the values of the winning global indices idx_dev (k×D,
 *                   device, each in [0, n_candidates)), regenerated from Philox and quantized as kbo_tpe_ask does, to x_dev
 *                   (k×D fp64, device).  k must be the shard ask's.  Synchronises. */
typedef enum kbo_tpe_kind { KBO_TPE_UNIFORM = 0, KBO_TPE_QUNIFORM = 1, KBO_TPE_CHOICE = 2 } kbo_tpe_kind;
typedef struct kbo_tpe kbo_tpe;
int kbo_tpe_create(kbo_handle* h, kbo_tpe** out, int32_t D, const int32_t* kinds, const double* lo, const double* hi, const double* q,
                   const int32_t* levels, double gamma, double prior_weight, uint64_t seed);
void kbo_tpe_destroy(kbo_tpe* t);
int kbo_tpe_tell(kbo_handle* h, kbo_tpe* t, const double* X, const double* loss, int32_t n_new, int on_host, void* stream);
int kbo_tpe_ask(kbo_handle* h, kbo_tpe* t, int32_t k, int32_t n_candidates, const double* cand_dev, double* x_dev, int64_t* idx_dev,
                double* cand_out_dev, float* score_out_dev, void* stream);
int kbo_tpe_state(kbo_handle* h, kbo_tpe* t, int32_t param, int32_t group, double* w, double* mu, double* sigma, int32_t cap,
                  int32_t* ncomp, double* p_accept, int32_t* n_below, void* stream);
int kbo_tpe_last_survivors(kbo_handle* h, kbo_tpe* t, int32_t* out, int32_t n);
int kbo_tpe_last_timings(kbo_handle* h, kbo_tpe* t, float* ms, int32_t n);
int kbo_tpe_ask_shard(kbo_handle* h, kbo_tpe* t, int32_t k, int32_t n_candidates, int32_t lo, int32_t hi, const double* cand_dev,
                      double* val_dev, int64_t* idx_dev, void* stream);
int kbo_tpe_pick(kbo_handle* h, kbo_tpe* t, int32_t k, const int64_t* idx_dev, double* x_dev, void* stream);

/* ---- multivariate TPE (Katib algorithm `multivariate-tpe`: Optuna's TPESampler(multivariate=True) on a flat space; FP64
 * restatement oracle/mvtpe_oracle.py) ------------------------------------------------------------------------------------
 * Parameter kinds: FLOAT on [lo, hi]; INT on the grid lo, lo + q, ... <= hi (q = step), values are grid points; CAT over
 * `levels` categories, observed and reported as the category index.  Optuna's defaults are fixed: consider_prior,
 * prior_weight = 1, consider_magic_clip, no endpoints.
 *   kbo_mvtpe_create: D parameters (HOST arrays kinds, lo, hi, q, levels; lo/hi are read for FLOAT and INT, q for INT, levels
 *                   for CAT), seed (random_state).  1 <= D <= 65535.
 *   kbo_mvtpe_tell  : appends n_new trials in told order: X (n_new×D, parameter units) and losses (minimised; ±inf rank).
 *                   Device pointers, or host pointers with on_host = 1.  A NaN loss, a float outside [lo, hi], an integer
 *                   off its grid or an invalid category index fails the call and tells nothing.  Synchronises.
 *   kbo_mvtpe_ask   : k points, each the best of its own n_candidates candidate vectors drawn from the below mixture
 *                   (Philox4x32-10 keyed by (seed, ask counter, point, candidate, slot)), or of the caller's candidates
 *                   cand_dev (k×D×n_candidates, device, fp64; integers are rounded to the grid and clipped, a float outside
 *                   [lo, hi] or an invalid category index is an error).  The winner is the candidate at the first index of
 *                   the maximum of log l(x) - log g(x): every candidate is scored in FP32 with an error bound and every one
 *                   that can still be the maximum is decided in FP64.  x_dev: k×D fp64 suggestions (device); optional
 *                   device outputs: idx_dev (k winning candidate indices), cand_out_dev (k×D×n_candidates: the candidates
 *                   as scored), score_out_dev (k×n_candidates×2 floats: FP32 score and its bound).  Synchronises.
 *                   1 <= k <= 65535, 1 <= n_candidates <= 2^24.
 *   kbo_mvtpe_state : the models of the current history (built on demand) for group 0 (below) or 1 (above), HOST outputs, any
 *                   may be NULL: w (the first cap of n_obs + 1 weights: observations in told order, then the prior), sigma
 *                   (D; NaN for categoricals), mu (the first cap observations' values, cap×D), cat_rows (2×D: an observation
 *                   row's entry at its own category and elsewhere; NaN for other kinds), n_obs, n_below.  Synchronises.
 *   kbo_mvtpe_last_survivors: per point of the last ask, the candidates decided in FP64.  Returns k, fills up to n entries.
 *   kbo_mvtpe_last_timings: milliseconds of the last ask's phases (models and draws, FP32 score, FP64 decision, final
 *                   reduction), CUDA events on its stream.  Returns 4, fills up to n entries.
 *   kbo_mvtpe_ask_shard: one shard of an ask sharded over ranks: as kbo_mvtpe_ask, but only candidates [lo, hi) of
 *                   n_candidates are drawn (keyed by their global index) and scored.  Per point it writes the shard's winner
 *                   to val_dev (k fp64, device: its FP64 score) and idx_dev (k, device: its global index).  lo == hi is an
 *                   empty shard, which writes (-inf, n_candidates) and never wins.  The ask counter advances as one
 *                   kbo_mvtpe_ask advances it.  cand_dev must be NULL.  Synchronises.
 *   kbo_mvtpe_pick  : after a shard ask and before the next tell, the vectors of the winning global indices idx_dev (k,
 *                   device, each in [0, n_candidates)), regenerated from Philox as kbo_mvtpe_ask draws them, to x_dev (k×D
 *                   fp64, device).  k must be the shard ask's.  Synchronises. */
typedef enum kbo_mvtpe_kind { KBO_MVTPE_FLOAT = 0, KBO_MVTPE_INT = 1, KBO_MVTPE_CAT = 2 } kbo_mvtpe_kind;
typedef struct kbo_mvtpe kbo_mvtpe;
int kbo_mvtpe_create(kbo_handle* h, kbo_mvtpe** out, int32_t D, const int32_t* kinds, const double* lo, const double* hi, const double* q,
                     const int32_t* levels, uint64_t seed);
void kbo_mvtpe_destroy(kbo_mvtpe* t);
int kbo_mvtpe_tell(kbo_handle* h, kbo_mvtpe* t, const double* X, const double* loss, int32_t n_new, int on_host, void* stream);
int kbo_mvtpe_ask(kbo_handle* h, kbo_mvtpe* t, int32_t k, int32_t n_candidates, const double* cand_dev, double* x_dev, int64_t* idx_dev,
                  double* cand_out_dev, float* score_out_dev, void* stream);
int kbo_mvtpe_state(kbo_handle* h, kbo_mvtpe* t, int32_t group, double* w, double* sigma, double* mu, double* cat_rows, int32_t cap,
                    int32_t* n_obs, int32_t* n_below, void* stream);
int kbo_mvtpe_last_survivors(kbo_handle* h, kbo_mvtpe* t, int32_t* out, int32_t n);
int kbo_mvtpe_last_timings(kbo_handle* h, kbo_mvtpe* t, float* ms, int32_t n);
int kbo_mvtpe_ask_shard(kbo_handle* h, kbo_mvtpe* t, int32_t k, int32_t n_candidates, int32_t lo, int32_t hi, const double* cand_dev,
                        double* val_dev, int64_t* idx_dev, void* stream);
int kbo_mvtpe_pick(kbo_handle* h, kbo_mvtpe* t, int32_t k, const int64_t* idx_dev, double* x_dev, void* stream);

/* ---- tree forests (Katib algorithm `bayesianoptimization` with base_estimator RF / ET: skopt's RandomForestRegressor /
 * ExtraTreesRegressor surrogates; FP64 restatement oracle/forest_oracle.py) --------------------------------------------------
 * Trees follow scikit-learn 1.9.0's DecisionTreeRegressor(min_samples_leaf) with the squared-error criterion and every feature
 * considered at every node: X is float32, y and every statistic FP64; node ids are breadth-first (children of node k are the next
 * two ids, left first); ties between splits go to the lowest feature, then the lowest threshold.
 *   kbo_forest_create: kind RF (bootstrap; best split over the sorted values) or ET (no bootstrap; one uniform threshold per feature
 *                   per node), n_trees (1..1024), min_samples_leaf (>= 1), seed.  Random draws are Philox4x32-10 keyed by seed:
 *                   RF bootstrap draw d of tree t is sample (u32·N) >> 32, u32 = word 0 of counter (d, t, 0, 0); the ET threshold
 *                   of (tree t, node k, feature f) is (max - min)·u + min (min where it equals max), u = the 53-bit uniform of
 *                   words 0 and 1 of counter (k, t, f, 1), NumPy's (a >> 5, b >> 6) construction.
 *   kbo_forest_fit  : X (N×D fp32), y (N fp64), device pointers.  counts (RF only, may be NULL): T×N int32 device bootstrap counts
 *                   that replace the drawn ones.  NaN or infinite X or y: KBO_ERR_INVALID.  Synchronises.
 *                   1 <= N <= 65536, 1 <= D <= 1024.
 *   kbo_forest_sweep: skopt's forest predict with return_std (mean over trees of the leaf values; sigma² = mean over trees of
 *                   max(impurity, 0) + value², minus mean², negatives to 0), then n_acq (0-3, distinct kbo_acq_kind, HOST acqs)
 *                   acquisitions on the raw mean and sigma (EI / PI with y_opt and xi, LCB with kappa; EI = PI = 0 where sigma = 0)
 *                   over M fp32 candidates Xc (M×D, device).  best_dev: n_acq device kbo_best, the first-index argmax of each, with
 *                   global_offset added to the index.  mu_out / sigma_out: optional device fp64 arrays of M.  Asynchronous.
 *   kbo_forest_predict: mean and sigma as above at n points (device, or host with x_on_host = 1) into HOST arrays.  Synchronises.
 *   kbo_forest_export: one tree's arrays into HOST buffers (any may be NULL), sklearn's tree_ conventions: feature (-2 at leaves),
 *                   threshold (-2 at leaves), left / right (-1 at leaves), value, impurity, n_node_samples (distinct samples),
 *                   weighted_n (bootstrap weight).  et_draws (ET only): n_nodes×D, the threshold drawn for each feature of each
 *                   internal node, NaN where the feature is constant in the node and on leaves.  counts (may be NULL): N int32, the
 *                   tree's bootstrap counts (all 1 for ET).  n_nodes receives the tree's node count; with cap < n_nodes only n_nodes
 *                   and counts are written.  Synchronises.
 *   kbo_forest_last_timings: milliseconds of the last fit and the last sweep, CUDA events on their streams.  Returns 2. */
typedef enum kbo_forest_kind { KBO_FOREST_RF = 0, KBO_FOREST_ET = 1 } kbo_forest_kind;
typedef struct kbo_forest kbo_forest;
int kbo_forest_create(kbo_handle* h, kbo_forest** out, int32_t kind, int32_t n_trees, int32_t min_samples_leaf, uint64_t seed);
void kbo_forest_destroy(kbo_forest* f);
int kbo_forest_fit(kbo_handle* h, kbo_forest* f, const float* X, const double* y, int32_t N, int32_t D, const int32_t* counts, void* stream);
int kbo_forest_sweep(kbo_handle* h, kbo_forest* f, const float* Xc, int64_t M, int64_t global_offset, int32_t n_acq, const int32_t* acqs, double y_opt,
                     double xi, double kappa, kbo_best* best_dev, double* mu_out, double* sigma_out, void* stream);
int kbo_forest_predict(kbo_handle* h, kbo_forest* f, const float* X, int32_t n, int x_on_host, double* mu_host, double* sigma_host, void* stream);
int kbo_forest_export(kbo_handle* h, kbo_forest* f, int32_t tree, int32_t* feature, double* threshold, int32_t* left, int32_t* right, double* value,
                      double* impurity, int32_t* n_node_samples, double* weighted_n, double* et_draws, int32_t cap, int32_t* n_nodes, int32_t* counts,
                      void* stream);
int kbo_forest_last_timings(kbo_handle* h, kbo_forest* f, float* ms, int32_t n);

/* ---- GBRT (Katib algorithm `bayesianoptimization` with skopt's GBRT surrogate: GradientBoostingQuantileRegressor, three
 * GradientBoostingRegressor(loss="quantile", n_estimators) chains; FP64 restatement oracle/gbrt_oracle.py) ------------------------
 * Each chain follows scikit-learn 1.9.0: init np.percentile(y, 100·α) (linear); per stage a squared-error tree of depth <= 3 on
 * the negative gradient (α where y >= raw, α − 1 elsewhere) over float32 X, its leaves replaced by the inverted-CDF percentile of
 * the residuals y − raw, and raw += fl(0.1·value).  Splits maximise (pl²·nr + pr²·nl) / (nl·nr) exactly (counts of rows going
 * left / right and of those with y >= raw); ties go to the lowest feature, then the lowest threshold; a node whose rows are all
 * on one side of raw is a leaf.
 *   kbo_gbrt_create: quantiles (3 increasing values in (0, 1), NULL: skopt's 0.16, 0.5, 0.84), n_estimators (1..128).
 *   kbo_gbrt_fit    : X (N×D fp32), y (N fp64), device pointers, 1 <= N <= 65536, 1 <= D <= 1024.  NaN or infinite X or y:
 *                   KBO_ERR_INVALID.  Synchronises.
 *   kbo_gbrt_sweep  : skopt's predict with return_std: mean = chain 1, sigma = fl(chain 2 − chain 0) / 2, negative where the quantiles cross; then n_acq (0-3, distinct kbo_acq_kind, HOST
 *                   acqs) acquisitions on them (EI / PI with y_opt and xi, 0 where sigma <= 0; LCB with kappa and sigma as it
 *                   is) over M fp32 candidates Xc (M×D, device).  best_dev: n_acq device kbo_best, the first-index argmax of
 *                   each, with global_offset added to the index.  mu_out / sigma_out (M) and quantiles_out (3×M, chain-major):
 *                   optional device fp64 arrays.  Asynchronous.
 *   kbo_gbrt_predict: mean, sigma and the three chains as above at n points (device, or host with x_on_host = 1) into HOST
 *                   arrays (any may be NULL).  Synchronises.
 *   kbo_gbrt_export : one stage's tree of one chain into HOST buffers (any may be NULL) in sklearn's tree_ layout (depth-first
 *                   preorder, left first): feature (-2 at leaves), threshold (-2 at leaves), left / right (-1 at leaves), value
 *                   (leaves: the replaced value; inner nodes: the mean negative gradient), n_node_samples, n_pos (rows with
 *                   y >= raw).  n_nodes receives the node count; with cap < n_nodes only n_nodes and init are written.  init: the
 *                   chain's init.  Synchronises.
 *   kbo_gbrt_last_timings: milliseconds of the last fit and the last sweep, CUDA events on their streams.  Returns 2. */
typedef struct kbo_gbrt kbo_gbrt;
int kbo_gbrt_create(kbo_handle* h, kbo_gbrt** out, const double* quantiles, int32_t n_estimators);
void kbo_gbrt_destroy(kbo_gbrt* g);
int kbo_gbrt_fit(kbo_handle* h, kbo_gbrt* g, const float* X, const double* y, int32_t N, int32_t D, void* stream);
int kbo_gbrt_sweep(kbo_handle* h, kbo_gbrt* g, const float* Xc, int64_t M, int64_t global_offset, int32_t n_acq, const int32_t* acqs, double y_opt,
                   double xi, double kappa, kbo_best* best_dev, double* mu_out, double* sigma_out, double* quantiles_out, void* stream);
int kbo_gbrt_predict(kbo_handle* h, kbo_gbrt* g, const float* X, int32_t n, int x_on_host, double* mu_host, double* sigma_host,
                     double* quantiles_host, void* stream);
int kbo_gbrt_export(kbo_handle* h, kbo_gbrt* g, int32_t chain, int32_t stage, int32_t* feature, double* threshold, int32_t* left, int32_t* right,
                    double* value, int32_t* n_node_samples, int32_t* n_pos, int32_t cap, int32_t* n_nodes, double* init, void* stream);
int kbo_gbrt_last_timings(kbo_handle* h, kbo_gbrt* g, float* ms, int32_t n);

/* ---- ENAS controller (Katib algorithm `enas`: the macro-search LSTM controller of ENAS and its REINFORCE training; FP64
 * restatement oracle/enas_oracle.py) -----------------------------------------------------------------------------------------
 * Parameters, in this order in every flat buffer (FP32, row-major): w_lstm (2H × 4H; gates i, f, o, g), g_emb (H), w_emb
 * (n_ops × H), w_soft (H × n_ops), w_attn_1 (H × H), w_attn_2 (H × H), v_attn (H).  An arc holds L(L+1)/2 decisions: per layer l,
 * its op, then skip_0 .. skip_{l-1}.
 *   kbo_enas_settings: temperature / tanh_const <= 0 mean None (the factor is skipped); entropy_weight and skip_weight are >= 0
 *                   (None is 0); baseline_decay in [0, 1]; learning_rate in (0, 1]; skip_target in (0, 1).
 *   kbo_enas_create: 1 <= L <= 64, 1 <= H <= 128, 1 <= n_ops <= 4096.  Parameters start U(-0.1, 0.1) (Philox4x32-10 keyed by
 *                   seed, counter (element lo, hi, 2^32 - 1, 2^32 - 1)); moments, baseline, step and draw counter start at 0.
 *   kbo_enas_train  : `steps` (0..10000) REINFORCE steps on a fixed reward in ONE launch: sample an arc (draw counter + step),
 *                   forward, backward, TF Adam (β1 = 0, β2 = 0.999, ε̂ = 1e-3, lr_t = lr·sqrt(1 - β2^t), t over the controller's
 *                   life).  arcs (device, steps × L(L+1)/2 int32, may be NULL): imposed arcs (teacher forcing).  stats (device,
 *                   may be NULL): steps × 6 floats nll, ent, mean kl, loss, baseline, skip rate.  Advances the draw counter by
 *                   `steps`.  Synchronises.
 *   kbo_enas_sample : k (1..1024) arcs into arcs (device, k × L(L+1)/2 int32); decision d of arc a draws u = (word 0 >> 8)·2^-24
 *                   of counter (draw counter lo, hi, a, d) unless uniforms (device, k × L(L+1)/2 floats) are imposed; a
 *                   decision is the first bin whose prefix sum of exp(s - max) exceeds u·total.  Optional device outputs:
 *                   op_probs (k × L × n_ops), skip_probs (k × L(L-1)/2, P(skip = 1)).  Advances the draw counter by 1.
 *                   Synchronises.
 *   kbo_enas_state  : HOST copies (any may be NULL) of the parameters, Adam moments m and v (flat, as above), baseline, Adam
 *                   step count and draw counter.  Synchronises.
 *   kbo_enas_set_params: HOST parameters, optional moments (NULL: zero), baseline and step; the draw counter is kept.
 *   kbo_enas_last_timings: milliseconds of the last train and the last sample call, CUDA events on their streams.  Returns 2. */
typedef struct kbo_enas_settings {
  double temperature, tanh_const, entropy_weight, baseline_decay, learning_rate, skip_target, skip_weight;
} kbo_enas_settings;
typedef struct kbo_enas kbo_enas;
int kbo_enas_create(kbo_handle* h, kbo_enas** out, int32_t L, int32_t H, int32_t n_ops, const kbo_enas_settings* settings, uint64_t seed);
void kbo_enas_destroy(kbo_enas* e);
int kbo_enas_train(kbo_handle* h, kbo_enas* e, double reward, int32_t steps, const int32_t* arcs, float* stats, void* stream);
int kbo_enas_sample(kbo_handle* h, kbo_enas* e, int32_t k, int32_t* arcs, const float* uniforms, float* op_probs, float* skip_probs, void* stream);
int kbo_enas_state(kbo_handle* h, kbo_enas* e, float* params, float* m, float* v, float* baseline, int64_t* step, int64_t* draws, void* stream);
int kbo_enas_set_params(kbo_handle* h, kbo_enas* e, const float* params, const float* m, const float* v, float baseline, int64_t step,
                        void* stream);
int kbo_enas_last_timings(kbo_handle* h, kbo_enas* e, float* ms, int32_t n);

#ifdef __cplusplus
}
#endif
#endif /* KBO_H_ */
