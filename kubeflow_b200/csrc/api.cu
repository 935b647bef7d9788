// extern "C" surface of libkbo.so (include/kbo.h).  No exceptions cross this boundary; every failure is a
// negative kbo_status plus kbo_last_error() text.  There is no CPU path: without a device kbo_create fails.
#include "kbo_internal.cuh"
#include "dgemm_sm90.cuh"

static const char* kNoHandle = "kbo: null handle";

extern "C" {

int kbo_version(void) { return KBO_VERSION; }

int kbo_create(kbo_handle** out, int device) {
  if (!out) return KBO_ERR_INVALID;
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0 || device < 0 || device >= n) return KBO_ERR_CUDA;
  if (cudaSetDevice(device) != cudaSuccess) return KBO_ERR_CUDA;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return KBO_ERR_CUDA;
  std::unique_ptr<kbo_handle> h(new (std::nothrow) kbo_handle());
  if (!h) return KBO_ERR_NOMEM;
  h->device = device;
  h->sm_count = prop.multiProcessorCount;
  h->smem_optin = (int)prop.sharedMemPerBlockOptin;   // cudaDevAttrMaxSharedMemoryPerBlockOptin
  if (prop.major != 9) {
    // sm_90a cubin only: refuse politely instead of failing at the first launch
    h->err = "libkbo is built for sm_90a (H100) only";
  }
  KBO_TRY(h->ev.create());
  *out = h.release();
  return KBO_OK;
}

// Device memory and the fixed events go with `delete h`; what has to be torn down in order (the communicator, streams,
// green contexts and the events the fit and sweep create on demand) is released here first.
void kbo_destroy(kbo_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  kbo_comm_destroy(h);
  kbo_i_lml_batch_free(h);
  if (h->lml_ev) cudaEventDestroy(h->lml_ev);
  for (auto& e : h->ev_panel) cudaEventDestroy(e);
  if (h->ev_gram) cudaEventDestroy(h->ev_gram);
  kbo_i_fit_partition_free(h);
  if (h->s_copy) cudaStreamDestroy(h->s_copy);
  for (auto* v : {&h->ev_var, &h->ev_cross, &h->ev_acq, &h->ev_cal})
    for (auto& p : *v) {
      cudaEventDestroy(p.first);
      cudaEventDestroy(p.second);
    }
  delete h;
}

const char* kbo_last_error(const kbo_handle* h) { return h ? h->err.c_str() : kNoHandle; }

int kbo_set_scratch_limit(kbo_handle* h, uint64_t bytes) {
  if (!h) return KBO_ERR_INVALID;
  if (bytes < (64ull << 20)) KBO_FAIL(h, KBO_ERR_INVALID, "scratch limit must be >= 64 MiB");
  h->scratch_limit = bytes;
  return KBO_OK;
}

int kbo_set_tc_fast(kbo_handle* h, int enabled) {
  if (!h) return KBO_ERR_INVALID;
  h->tc_fast = enabled != 0;
  return KBO_OK;
}

double kbo_last_rank_error(kbo_handle* h) { return h ? (double)h->last_rank_err : -1.0; }

double kbo_last_rank_mu_error(kbo_handle* h) { return h ? (double)h->last_rank_mu_err : -1.0; }

int kbo_last_unrefined(kbo_handle* h) { return h ? h->last_unrefined : KBO_ERR_INVALID; }

int kbo_set_rank_prefix(kbo_handle* h, int tile_pairs) {
  if (!h) return KBO_ERR_INVALID;
  h->rank_prefix = tile_pairs < 0 ? -1 : tile_pairs;
  return KBO_OK;
}

int kbo_last_prefix_survivors(kbo_handle* h) { return h ? h->last_prefix_survivors : KBO_ERR_INVALID; }

int kbo_set_lazy_inverse(kbo_handle* h, int enabled) {
  if (!h) return KBO_ERR_INVALID;
  h->lazy_w = enabled != 0;
  return KBO_OK;
}

int kbo_set_rank_tc(kbo_handle* h, int enabled) {
  if (!h) return KBO_ERR_INVALID;
  h->rank_tc = enabled != 0;
  return KBO_OK;
}

int kbo_last_contenders(kbo_handle* h) { return h ? h->last_contenders : KBO_ERR_INVALID; }

int kbo_fit(kbo_handle* h, const double* X, const double* y, int32_t N, int32_t D, const kbo_params* p, int x_on_host, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!X || !y || !p || !p->length_scale) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_fit: null argument");
  if (N < 1 || D < 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_fit: need N >= 1 and D >= 1 (got N=%d D=%d)", N, D);
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  if (x_on_host) {
    KBO_TRY(kbo_reserve(h, h->stage_X, (size_t)N * D));
    KBO_TRY(kbo_reserve(h, h->stage_y, (size_t)N));
    KBO_CUDA(h, kbo_copy(h->stage_X.p, X, (size_t)N * D, cudaMemcpyHostToDevice, s));
    KBO_CUDA(h, kbo_copy(h->stage_y.p, y, (size_t)N, cudaMemcpyHostToDevice, s));
    X = h->stage_X.p;
    y = h->stage_y.p;
  }
  return kbo_i_fit(h, X, y, N, D, p, s);
}

int kbo_lml_batch(kbo_handle* h, const double* X, const double* y, int32_t N, int32_t D, int32_t G, const kbo_params* params, int x_on_host,
                  double* lml_host, int32_t* info_host, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!X || !y || !params || !lml_host) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_lml_batch: null argument");
  if (N < 1 || D < 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_lml_batch: need N >= 1 and D >= 1");
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  if (x_on_host) {
    KBO_TRY(kbo_reserve(h, h->stage_X, (size_t)N * D));
    KBO_TRY(kbo_reserve(h, h->stage_y, (size_t)N));
    KBO_CUDA(h, kbo_copy(h->stage_X.p, X, (size_t)N * D, cudaMemcpyHostToDevice, s));
    KBO_CUDA(h, kbo_copy(h->stage_y.p, y, (size_t)N, cudaMemcpyHostToDevice, s));
    X = h->stage_X.p;
    y = h->stage_y.p;
  }
  return kbo_i_lml_batch(h, X, y, N, D, G, params, lml_host, info_host, s);
}

int kbo_lml_grad_batch(kbo_handle* h, const double* X, const double* y, int32_t N, int32_t D, int32_t G, const kbo_params* params, int x_on_host,
                       double* lml_host, double* grad_host, int32_t* info_host, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!X || !y || !params || !lml_host || !grad_host) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_lml_grad_batch: null argument");
  if (N < 1 || D < 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_lml_grad_batch: need N >= 1 and D >= 1");
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  if (x_on_host) {
    KBO_TRY(kbo_reserve(h, h->stage_X, (size_t)N * D));
    KBO_TRY(kbo_reserve(h, h->stage_y, (size_t)N));
    KBO_CUDA(h, kbo_copy(h->stage_X.p, X, (size_t)N * D, cudaMemcpyHostToDevice, s));
    KBO_CUDA(h, kbo_copy(h->stage_y.p, y, (size_t)N, cudaMemcpyHostToDevice, s));
    X = h->stage_X.p;
    y = h->stage_y.p;
  }
  return kbo_i_lml_grad_batch(h, X, y, N, D, G, params, lml_host, grad_host, info_host, s);
}

int kbo_fit_append(kbo_handle* h, const double* x, double y, int x_on_host, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!x) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_fit_append: null argument");
  if (!h->fitted) KBO_FAIL(h, KBO_ERR_STATE, "kbo_fit_append: call kbo_fit first");
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  if (x_on_host) {
    KBO_TRY(kbo_reserve(h, h->stage_X, (size_t)h->D));
    KBO_CUDA(h, kbo_copy(h->stage_X.p, x, (size_t)h->D, cudaMemcpyHostToDevice, s));
    x = h->stage_X.p;
  }
  return kbo_i_fit_append(h, x, y, s);
}

int kbo_fit_rebase(kbo_handle* h, int32_t n_keep, const double* y, int y_on_host, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!h->fitted) KBO_FAIL(h, KBO_ERR_STATE, "kbo_fit_rebase: call kbo_fit first");
  if (n_keep < 1 || n_keep > h->N) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_fit_rebase: need 1 <= n_keep <= N=%d (got %d)", h->N, n_keep);
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  if (y && y_on_host) {
    KBO_TRY(kbo_reserve(h, h->stage_y, (size_t)n_keep));
    KBO_CUDA(h, kbo_copy(h->stage_y.p, y, (size_t)n_keep, cudaMemcpyHostToDevice, s));
    y = h->stage_y.p;
  }
  return kbo_i_fit_rebase(h, n_keep, y, s);
}

int kbo_fit_room(kbo_handle* h) { return (h && h->fitted) ? h->ld - h->N : 0; }

int kbo_fit_info(kbo_handle* h, double* lml, double* y_mean, double* y_std, double* y_opt, int32_t* info, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!h->fitted) KBO_FAIL(h, KBO_ERR_STATE, "kbo_fit_info: call kbo_fit first");
  cudaStream_t s = (cudaStream_t)stream;
  double sc[S_COUNT];
  int inf = 0;
  KBO_CUDA(h, kbo_copy(sc, h->scal.p, S_COUNT, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, kbo_copy(&inf, h->info.p, 1, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (lml) *lml = sc[S_LML];
  if (y_mean) *y_mean = sc[S_YMEAN];
  if (y_std) *y_std = sc[S_YSTD];
  if (y_opt) *y_opt = sc[S_YOPT];
  if (info) *info = inf;
  if (inf != 0) KBO_FAIL(h, KBO_ERR_NOT_PD, "kernel matrix is not positive definite (pivot %d); increase `noise` ($SK/_gpr.py:353-362)", inf);
  return KBO_OK;
}

int kbo_fit_state(kbo_handle* h, double* L_out, double* W_out, double* alpha_out, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!h->fitted) KBO_FAIL(h, KBO_ERR_STATE, "kbo_fit_state: call kbo_fit first");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t N = h->N, ld = h->ld;
  if (W_out) KBO_TRY(kbo_i_ensure_w(h, s));
  if (L_out) {
    KBO_CUDA(h, cudaMemcpy2DAsync(L_out, N * 8, h->K.p, ld * 8, N * 8, N, cudaMemcpyDeviceToDevice, s));
    KBO_TRY(kbo_i_zero_upper(h, L_out, (int)N, (int)N, s));
  }
  if (W_out) KBO_CUDA(h, cudaMemcpy2DAsync(W_out, N * 8, h->W.p, ld * 8, N * 8, N, cudaMemcpyDeviceToDevice, s));
  if (alpha_out) KBO_CUDA(h, kbo_copy(alpha_out, h->alpha.p, N, cudaMemcpyDeviceToDevice, s));
  return KBO_OK;
}

int kbo_sweep(kbo_handle* h, const void* Xc, int32_t xc_dtype, int64_t M, int64_t global_offset, int xc_on_host, double* mu_out,
              double* std_out, double* acq_out, kbo_best* best_dev, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!Xc || !best_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sweep: null argument");
  if (M < 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sweep: M must be >= 1");
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  if (xc_on_host) {
    const size_t bytes = (size_t)M * h->D * (xc_dtype == KBO_F64 ? 8 : 4);
    KBO_TRY(kbo_reserve(h, h->stage_Xc, bytes));
    KBO_CUDA(h, cudaMemcpyAsync(h->stage_Xc.p, Xc, bytes, cudaMemcpyHostToDevice, s));
    Xc = h->stage_Xc.p;
  }
  return kbo_i_sweep(h, Xc, xc_dtype, M, global_offset, mu_out, std_out, acq_out, best_dev, s);
}

static int stage_rows(kbo_handle* h, const void** X, int32_t dtype, int64_t rows, cudaStream_t s) {
  const size_t bytes = (size_t)rows * h->D * (dtype == KBO_F64 ? 8 : 4);
  KBO_TRY(kbo_reserve(h, h->stage_Xc, bytes));
  KBO_CUDA(h, cudaMemcpyAsync(h->stage_Xc.p, *X, bytes, cudaMemcpyHostToDevice, s));
  *X = h->stage_Xc.p;
  return KBO_OK;
}

int kbo_sweep_multi(kbo_handle* h, const void* Xc, int32_t xc_dtype, int64_t M, int64_t global_offset, int xc_on_host, int32_t n_acq,
                    const int32_t* acqs, kbo_best* best_dev, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!Xc || !acqs || !best_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sweep_multi: null argument");
  if (M < 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_sweep_multi: M must be >= 1");
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  if (xc_on_host) KBO_TRY(stage_rows(h, &Xc, xc_dtype, M, s));
  return kbo_i_sweep_multi(h, Xc, xc_dtype, M, global_offset, n_acq, acqs, best_dev, s);
}

int kbo_last_decisions(kbo_handle* h, int32_t n, int32_t* unrefined, int32_t* contenders, int32_t* prefix_survivors) {
  if (!h) return KBO_ERR_INVALID;
  if (n < 0) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_last_decisions: n must be >= 0");
  for (int k = 0; k < n && k < h->dec_n; k++) {
    if (unrefined) unrefined[k] = h->dec_unrefined[k];
    if (contenders) contenders[k] = h->dec_contenders[k];
    if (prefix_survivors) prefix_survivors[k] = h->dec_prefix_survivors[k];
  }
  return h->dec_n;
}

int kbo_predict_mean(kbo_handle* h, const void* X, int32_t x_dtype, int32_t n, int x_on_host, double* mu_out_host, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!X || !mu_out_host) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_predict_mean: null argument");
  if (n < 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_predict_mean: n must be >= 1");
  if (!h->fitted) KBO_FAIL(h, KBO_ERR_STATE, "kbo_predict_mean: call kbo_fit first");
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  if (x_on_host) KBO_TRY(stage_rows(h, &X, x_dtype, n, s));
  return kbo_i_predict_mean(h, X, x_dtype, n, mu_out_host, s);
}

int kbo_best_to_host(kbo_handle* h, const kbo_best* best_dev, kbo_best* best_host, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!best_dev || !best_host) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_best_to_host: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  int inf = 0;
  KBO_CUDA(h, cudaMemcpyAsync(best_host, best_dev, sizeof(kbo_best), cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, kbo_copy(&inf, h->info.p, 1, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (inf != 0) KBO_FAIL(h, KBO_ERR_NOT_PD, "kernel matrix is not positive definite (pivot %d); increase `noise`", inf);
  return KBO_OK;
}

static float sum_pairs(std::vector<std::pair<cudaEvent_t, cudaEvent_t>>& v, size_t used) {
  float t = 0.f;
  for (size_t i = 0; i < used; i++) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, v[i].first, v[i].second);
    t += ms;
  }
  return t;
}

int kbo_suggest_host(kbo_handle* h, const double* X, const double* y, int32_t N, int32_t D, const void* Xc, int32_t xc_dtype, int64_t M,
                     int64_t global_offset, const kbo_params* p, kbo_best* best_host, kbo_timings* timings) {
  if (!h) return KBO_ERR_INVALID;
  if (!X || !y || !Xc || !p || !best_host) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_suggest_host: null argument");
  cudaStream_t s = 0;
  KBO_CUDA(h, cudaSetDevice(h->device));
  KBO_TRY(kbo_reserve(h, h->best, 1));
  h->launches = 0;
  h->time_kernels = true;
  h->ev_var_used = h->ev_cross_used = h->ev_acq_used = h->ev_cal_used = 0;
  cudaEventRecord(h->ev[0], s);
  // X, y go up first and the fit is enqueued; the candidate grid (the bulk of the bytes) is copied on a second stream WHILE the
  // fit runs — it is not needed before the sweep.  (Issued after the fit's launches so that a pageable source, whose copy
  // blocks the host, still overlaps the device work; a pinned source overlaps either way.)
  int r = kbo_fit(h, X, y, N, D, p, 1, s);
  cudaEventRecord(h->ev[1], s);
  if (r == KBO_OK) {
    const size_t bytes = (size_t)M * D * (xc_dtype == KBO_F64 ? 8 : 4);
    r = kbo_reserve(h, h->stage_Xc, bytes);
    if (r == KBO_OK && !h->s_copy) {
      cudaError_t e = cudaStreamCreateWithFlags(&h->s_copy, cudaStreamNonBlocking);
      if (e != cudaSuccess) {
        h->err = std::string("cudaStreamCreate failed: ") + cudaGetErrorString(e);
        r = KBO_ERR_CUDA;
      }
    }
    if (r == KBO_OK) {
      cudaEventRecord(h->ev[5], h->s_copy);
      cudaError_t e = cudaMemcpyAsync(h->stage_Xc.p, Xc, bytes, cudaMemcpyHostToDevice, h->s_copy);
      cudaEventRecord(h->ev[6], h->s_copy);
      if (e != cudaSuccess) {
        h->err = std::string("H2D of candidates failed: ") + cudaGetErrorString(e);
        r = KBO_ERR_CUDA;
      } else {
        cudaStreamWaitEvent(s, h->ev[6], 0);
      }
    }
  }
  cudaEventRecord(h->ev[2], s);
  if (r == KBO_OK) r = kbo_i_sweep(h, h->stage_Xc.p, xc_dtype, M, global_offset, nullptr, nullptr, nullptr, h->best.p, s);
  if (r == KBO_OK && h->comm) r = kbo_allreduce_argmax(h, h->best.p, s);   // sharded grid: the global first-index argmax
  cudaEventRecord(h->ev[3], s);
  if (r == KBO_OK) r = kbo_best_to_host(h, h->best.p, best_host, s);
  cudaEventRecord(h->ev[4], s);
  cudaEventSynchronize(h->ev[4]);
  h->time_kernels = false;
  kbo_timings t{};
  cudaEventElapsedTime(&t.fit_ms, h->ev[0], h->ev[1]);    // includes H2D of X, y
  if (r == KBO_OK) cudaEventElapsedTime(&t.h2d_ms, h->ev[5], h->ev[6]);    // H2D of the candidate grid (second stream, overlapped with the fit)
  cudaEventElapsedTime(&t.sweep_ms, h->ev[2], h->ev[3]);
  cudaEventElapsedTime(&t.d2h_ms, h->ev[3], h->ev[4]);
  cudaEventElapsedTime(&t.total_ms, h->ev[0], h->ev[4]);
  t.var_kernel_ms = sum_pairs(h->ev_var, h->ev_var_used);
  t.cross_kernel_ms = sum_pairs(h->ev_cross, h->ev_cross_used);
  t.acq_kernel_ms = sum_pairs(h->ev_acq, h->ev_acq_used);
  t.calib_ms = sum_pairs(h->ev_cal, h->ev_cal_used);
  t.launches = h->launches;
  t.chunks = h->tim.chunks;
  h->tim = t;
  if (timings) *timings = t;
  return r;
}

int kbo_last_timings(kbo_handle* h, kbo_timings* out) {
  if (!h || !out) return KBO_ERR_INVALID;
  *out = h->tim;
  return KBO_OK;
}

int kbo_gram(kbo_handle* h, const double* Xs, int32_t N, int32_t D, int32_t kernel, double amplitude, double noise, double* K, int32_t ldk,
             void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!Xs || !K || N < 1 || D < 1 || ldk < N) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_gram: bad argument");
  if (kernel != KBO_KERNEL_RBF && kernel != KBO_KERNEL_MATERN52) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_gram: unknown kernel %d", kernel);
  return kbo_i_gram(h, Xs, N, D, kernel, amplitude, noise, K, ldk, (cudaStream_t)stream);
}

int kbo_potrf(kbo_handle* h, double* A, int32_t N, int32_t lda, int32_t* info_dev, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!A || !info_dev || N < 1 || lda < N) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_potrf: bad argument");
  return kbo_i_potrf(h, A, N, lda, info_dev, (cudaStream_t)stream);
}

int kbo_trtri(kbo_handle* h, const double* L, int32_t N, int32_t ldl, double* W, int32_t ldw, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!L || !W || N < 1 || ldl < N || ldw < N) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_trtri: bad argument");
  return kbo_i_trtri(h, L, N, ldl, W, ldw, (cudaStream_t)stream);
}

int kbo_acq_argmax(kbo_handle* h, const float* mu_n, const float* var_n, int64_t M, int64_t global_offset, int32_t acq, double y_mean,
                   double y_std, double y_opt, double xi, double kappa, float* acq_out, kbo_best* best_dev, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!mu_n || !var_n || !best_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_acq_argmax: null argument");
  if (acq < KBO_ACQ_EI || acq > KBO_ACQ_PI) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_acq_argmax: unknown acquisition %d", acq);
  if (!(y_std > 0.0) || !(y_std < INFINITY)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_acq_argmax: y_std must be finite and > 0 (got %g)", y_std);
  return kbo_i_acq_argmax_f32(h, mu_n, var_n, M, global_offset, acq, y_mean, y_std, y_opt, xi, kappa, 1.0, acq_out, best_dev,
                              (cudaStream_t)stream);
}

}  // extern "C"

// Test hook (not in kbo.h): the FP64 tensor-core rate of this GPU — DMMA on register-resident operands, 8 independent accumulator
// tiles per warp, 8 warps per CTA, one CTA per SM — the denominator bench.py's fit roofline uses (there is no FP64 entry in
// MEASURED_PEAKS.json).  Both shapes the FP64 GEMMs issue are timed and the faster is reported: on an H100 m8n8k4 reaches half the
// rate of m16n8k8, which the fit's GEMMs (dgemm_sm90.cuh) use.  Same loops as tests/studies/dmma_probe.cu.
template <bool K8>
__global__ void __launch_bounds__(256) fp64_peak_kernel(double* out, int iters) {
  double a[4], b[2], c[8][4];
#pragma unroll
  for (int i = 0; i < 4; i++) a[i] = threadIdx.x * 1e-3 + i;
#pragma unroll
  for (int i = 0; i < 2; i++) b[i] = threadIdx.x * 1e-4 + 1.0 + i;
#pragma unroll
  for (int j = 0; j < 8; j++) c[j][0] = c[j][1] = c[j][2] = c[j][3] = 0.0;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int j = 0; j < 8; j++) {
      if (K8)
        dmma_m16n8k8(c[j], a, b);
      else
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[j][0]), "+d"(c[j][1]) : "d"(a[0]), "d"(b[0]));
    }
  }
  double s = 0.0;
#pragma unroll
  for (int j = 0; j < 8; j++) s += c[j][0] + c[j][1] + c[j][2] + c[j][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
extern "C" {
int kbo_debug_fp64_peak(kbo_handle* h, double* tflops_out) {
  if (!h || !tflops_out) return KBO_ERR_INVALID;
  cudaSetDevice(h->device);
  const int iters = 20000, ctas = h->sm_count;
  DevBuf<double> buf;
  KBO_TRY(kbo_reserve(h, buf, (size_t)ctas * 256));
  double* out = buf.p;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  double peak = 0.0;
  for (int k8 = 0; k8 < 2; k8++) {
    const int its = k8 ? iters / 2 : iters;   // one m16n8k8 is four m8n8k4s of work: half the iterations, twice the time at twice the rate
    float best = 1e30f;
    for (int rep = 0; rep < 4; rep++) {
      cudaEventRecord(e0, 0);
      if (k8)
        fp64_peak_kernel<true><<<ctas, 256>>>(out, its);
      else
        fp64_peak_kernel<false><<<ctas, 256>>>(out, its);
      cudaEventRecord(e1, 0);
      cudaEventSynchronize(e1);
      float ms = 0.f;
      cudaEventElapsedTime(&ms, e0, e1);
      if (rep > 0 && ms < best) best = ms;
    }
    const double flop_per_mma = k8 ? 2.0 * 16 * 8 * 8 : 2.0 * 8 * 8 * 4;
    peak = fmax(peak, flop_per_mma * 8.0 * its * 8 * ctas / (best * 1e-3) * 1e-12);
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  KBO_CUDA(h, cudaGetLastError());
  *tflops_out = peak;
  return KBO_OK;
}

// Test hook (not in kbo.h): one dgemm_sm90_kernel launch on caller-owned device buffers (row-major; transb = 1: B is N×K, C = A·Bᵀ;
// 0: B is K×N), on the given stream.  For the tests that check the fit's FP64 GEMM against a host product.
int kbo_debug_dgemm_sm90(kbo_handle* h, int32_t transb, int32_t M, int32_t N, int32_t K, const double* A, int32_t lda, const double* B, int32_t ldb,
                         double* C, int32_t ldc, double alpha, double beta, int32_t kmode, int32_t kbegin, int32_t tileskip, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!A || !B || !C || M < 1 || N < 1 || K < 0 || lda < K || ldb < (transb ? K : N) || ldc < N || kmode < KM_FULL || kmode > KM_FROM_M ||
      (tileskip != TS_NONE && tileskip != TS_LOWER))
    KBO_FAIL(h, KBO_ERR_INVALID, "kbo_debug_dgemm_sm90: bad argument");
  cudaSetDevice(h->device);
  if (transb)
    dgemm_sm90_launch<true>((cudaStream_t)stream, M, N, K, A, lda, B, ldb, C, ldc, alpha, beta, kmode, kbegin, tileskip);
  else
    dgemm_sm90_launch<false>((cudaStream_t)stream, M, N, K, A, lda, B, ldb, C, ldc, alpha, beta, kmode, kbegin, tileskip);
  KBO_CUDA(h, cudaGetLastError());
  return KBO_OK;
}

// Test hook (not in kbo.h): the ranking pass alone over M candidates (device pointer), normalised mean / variance copied to
// caller-owned DEVICE float arrays.  mode 0 = FP64 K* kernel + one-product cluster kernel, 1 = tensor-core K* + wgmma
// ranking kernel.  plane_out (optional, M × Npad fp16, M <= one chunk) receives the K* hi plane the contraction consumed.
int kbo_debug_rank_pass(kbo_handle* h, const void* Xc, int32_t xc_dtype, int64_t M, int32_t mode, float* mun_out, float* varn_out, void* plane_out,
                        void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!h->fitted || !h->have_planes) KBO_FAIL(h, KBO_ERR_STATE, "kbo_debug_rank_pass: needs a fit with tensor-core planes");
  cudaStream_t s = (cudaStream_t)stream;
  const int Npad = h->Npad;
  const int64_t rows_pad = round_up64(M, 256);
  KBO_TRY(kbo_reserve(h, h->Ksh, (size_t)rows_pad * Npad));
  KBO_TRY(kbo_reserve(h, h->Ksl, (size_t)rows_pad * Npad));
  const size_t bytes = sizeof(float) * (size_t)(rows_pad + 256);
  KBO_TRY(kbo_reserve(h, h->mun, bytes));
  KBO_TRY(kbo_reserve(h, h->varn, bytes));
  KBO_TRY(kbo_i_ensure_w(h, s));
  if (mode == 1) {
    if (!h->ks_ready) KBO_FAIL(h, KBO_ERR_STATE, "kbo_debug_rank_pass: tensor-core K* operands not available (D > 128?)");
    KBO_TRY(kbo_i_tc_kstar(h, Xc, xc_dtype, M, h->Ksh.p, kbo_view<float>(h->mun), s));
    KBO_TRY(kbo_i_tc_rank(h, h->Ksh.p, rows_pad, h->Wh.p, Npad, h->prm.amplitude, kbo_view<float>(h->varn), s));
  } else {
    KBO_TRY(kbo_i_debug_cross_planes(h, Xc, xc_dtype, M, s));
    KBO_TRY(kbo_i_tc_variance(h, h->Ksh.p, h->Ksl.p, round_up64(M, 128), h->Wh.p, h->Wl.p,
                              Npad, 0.0, h->prm.amplitude, kbo_view<float>(h->varn), 1024, s, 1));
  }
  KBO_CUDA(h, kbo_copy(mun_out, kbo_view<float>(h->mun), M, cudaMemcpyDeviceToDevice, s));
  KBO_CUDA(h, kbo_copy(varn_out, kbo_view<float>(h->varn), M, cudaMemcpyDeviceToDevice, s));
  if (plane_out) KBO_CUDA(h, kbo_copy(static_cast<__half*>(plane_out), h->Ksh.p, (size_t)M * Npad, cudaMemcpyDeviceToDevice, s));
  return KBO_OK;
}

// Test hook (not in kbo.h): the tensor-core K* kernel alone over M candidates (device pointer), writing straight into caller-owned
// DEVICE buffers: mun_out (rows_pad floats) and plane_out (rows_pad × Npad fp16), rows_pad = M rounded up to 256.  store_cols < 0
// stores every column; otherwise only the 128-column tiles covering the first store_cols, and the rest of plane_out is not written.
int kbo_debug_kstar(kbo_handle* h, const void* Xc, int32_t xc_dtype, int64_t M, int32_t store_cols, float* mun_out, void* plane_out, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!Xc || !mun_out || !plane_out || M < 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_debug_kstar: bad argument");
  if (!h->fitted || !h->ks_ready) KBO_FAIL(h, KBO_ERR_STATE, "kbo_debug_kstar: needs a fit with tensor-core K* operands (D <= 128)");
  cudaSetDevice(h->device);
  KBO_TRY(kbo_i_tc_kstar(h, Xc, xc_dtype, M, (__half*)plane_out, mun_out, (cudaStream_t)stream, store_cols));
  return KBO_OK;
}

// Test hook (not in kbo.h): the pruning pass's (tile_pairs >= 1) or the full ranking pass's (tile_pairs < 0) normalised mean and
// variance of M candidate rows (device pointer) into caller-owned DEVICE float arrays.  Scratch is M × Npad fp16: callers slice
// large grids (a row's values do not depend on the rows swept with it).
int kbo_debug_rank_rows(kbo_handle* h, const void* Xc, int32_t xc_dtype, int64_t M, int32_t tile_pairs, float* mun_out, float* varn_out, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!Xc || !mun_out || !varn_out || M < 1) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_debug_rank_rows: bad argument");
  cudaSetDevice(h->device);
  return kbo_i_debug_rank_rows(h, Xc, xc_dtype, M, tile_pairs, mun_out, varn_out, (cudaStream_t)stream);
}

// Test hooks (not in kbo.h): with recording on, each kbo_sweep / kbo_sweep_multi keeps, per stage it ran and per acquisition, the
// bounds that stage pruned with and its survivor list (kbo_handle::StageRec); recording adds read-backs, never arithmetic.
int kbo_debug_record_stages(kbo_handle* h, int32_t on) {
  if (!h) return KBO_ERR_INVALID;
  h->record_stages = on != 0;
  h->stage_recs.clear();
  return KBO_OK;
}
// Test hooks (not in kbo.h): with on != 0, kbo_fit enqueues its factorisation call by call instead of replaying the cached graph
// (the path KBO_FIT_TRACE measures).  stats[8] = graph captures, executable updates, instantiations, replays since the handle was
// made; then the cached graph's kernel nodes in the chain's green context, in the rest's, elsewhere; kernel launches per replay.
int kbo_debug_fit_stream_path(kbo_handle* h, int32_t on) {
  if (!h) return KBO_ERR_INVALID;
  h->fit_stream_path = on != 0;
  return KBO_OK;
}
int kbo_debug_fit_graph(kbo_handle* h, int32_t* stats) {
  if (!h) return KBO_ERR_INVALID;
  if (!stats) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_debug_fit_graph: bad argument");
  cudaSetDevice(h->device);
  for (int i = 0; i < 4; i++) stats[i] = h->fit_graph_stat[i];
  stats[7] = h->fit_graph_launches;
  return kbo_i_fit_graph_nodes(h, stats + 4);
}
int kbo_debug_stage_count(kbo_handle* h) { return h ? (int)h->stage_recs.size() : KBO_ERR_INVALID; }
// ints[4] = (stage, acquisition, calibration rows, survivors counted), floats[7] = (E, Eμ, raw max |dσ²|, raw max |dμ|, lower bound,
// threshold, window delta); the first min(cap, list length) survivors go to list.  Returns the list length.
int kbo_debug_stage(kbo_handle* h, int32_t i, int32_t* ints, float* floats, int32_t* list, int32_t cap) {
  if (!h) return KBO_ERR_INVALID;
  if (i < 0 || i >= (int)h->stage_recs.size() || !ints || !floats || cap < 0) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_debug_stage: bad argument");
  const kbo_handle::StageRec& r = h->stage_recs[i];
  ints[0] = r.stage;
  ints[1] = r.acq;
  ints[2] = r.cal_n;
  ints[3] = r.n;
  for (int k = 0; k < 7; k++) floats[k] = r.f[k];
  const int n = (int)r.list.size();
  if (list)
    for (int k = 0; k < n && k < cap; k++) list[k] = r.list[k];
  return n;
}

}  // extern "C"
