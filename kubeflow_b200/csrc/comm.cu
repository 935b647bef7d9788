// Multi-GPU exchange behind the C ABI (SURVEY.md §8(e), §8(b) `kbo_allreduce_argmax`): the candidate grid shards by rows, every
// rank sweeps its rows with a global offset, and the only exchange is the argmax — ONE ncclAllGather of 32 bytes per rank
// (value, global index, mu, std) followed by a one-thread reduce that every rank runs identically: maximum value, lowest
// global index among equals = np.argmin(-values) over the concatenated grid (skopt Optimizer._tell).  NCCL is bound at run
// time (dlopen of libnccl.so.2 — inside a PyTorch process that is the copy torch already loaded), so libkbo.so itself has no
// link-time dependency on it and single-GPU callers never touch it.
#include <dlfcn.h>

#include "kbo_internal.cuh"

namespace {

typedef struct { char internal[128]; } nccl_unique_id;   // ncclUniqueId (NCCL_UNIQUE_ID_BYTES = 128)
typedef int (*pfn_get_unique_id)(nccl_unique_id*);
typedef int (*pfn_comm_init_rank)(void**, int, nccl_unique_id, int);
typedef int (*pfn_comm_destroy)(void*);
typedef int (*pfn_all_gather)(const void*, void*, size_t, int /*ncclDataType_t*/, void*, cudaStream_t);
typedef const char* (*pfn_get_error_string)(int);

struct NcclApi {
  void* lib = nullptr;
  pfn_get_unique_id get_unique_id = nullptr;
  pfn_comm_init_rank comm_init_rank = nullptr;
  pfn_comm_destroy comm_destroy = nullptr;
  pfn_all_gather all_gather = nullptr;
  pfn_get_error_string get_error_string = nullptr;
  std::string err;
};

NcclApi* nccl_api() {
  static NcclApi api;
  if (api.lib || !api.err.empty()) return &api;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (api.lib) break;
  }
  if (!api.lib) {
    api.err = std::string("libnccl.so.2 not found: ") + (dlerror() ? dlerror() : "");
    return &api;
  }
  api.get_unique_id = (pfn_get_unique_id)dlsym(api.lib, "ncclGetUniqueId");
  api.comm_init_rank = (pfn_comm_init_rank)dlsym(api.lib, "ncclCommInitRank");
  api.comm_destroy = (pfn_comm_destroy)dlsym(api.lib, "ncclCommDestroy");
  api.all_gather = (pfn_all_gather)dlsym(api.lib, "ncclAllGather");
  api.get_error_string = (pfn_get_error_string)dlsym(api.lib, "ncclGetErrorString");
  if (!api.get_unique_id || !api.comm_init_rank || !api.comm_destroy || !api.all_gather) api.err = "libnccl.so.2 lacks a required symbol";
  return &api;
}

// first-index argmax over the ranks' results; NaN never wins; one thread — n_ranks is at most a few dozen
__global__ void argmax_reduce_kernel(const kbo_best* __restrict__ all, int n, kbo_best* __restrict__ out) {
  kbo_best b = all[0];
  bool have = b.value == b.value;
  for (int r = 1; r < n; r++) {
    const kbo_best c = all[r];
    if (!(c.value == c.value)) continue;
    if (!have || c.value > b.value || (c.value == b.value && c.index < b.index)) {
      b = c;
      have = true;
    }
  }
  *out = b;
}

}  // namespace

extern "C" {

int kbo_comm_unique_id(void* id_out) {
  if (!id_out) return KBO_ERR_INVALID;
  NcclApi* a = nccl_api();
  if (!a->err.empty()) return KBO_ERR_STATE;
  nccl_unique_id id;
  if (a->get_unique_id(&id) != 0) return KBO_ERR_CUDA;
  memcpy(id_out, &id, sizeof id);
  return KBO_OK;
}

int kbo_comm_init(kbo_handle* h, int32_t n_ranks, int32_t rank, const void* id) {
  if (!h) return KBO_ERR_INVALID;
  if (!id || n_ranks < 1 || rank < 0 || rank >= n_ranks) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_comm_init: need 0 <= rank < n_ranks and a 128-byte id");
  NcclApi* a = nccl_api();
  if (!a->err.empty()) KBO_FAIL(h, KBO_ERR_STATE, "kbo_comm_init: %s", a->err.c_str());
  if (h->comm) KBO_FAIL(h, KBO_ERR_STATE, "kbo_comm_init: communicator already initialised (kbo_comm_destroy first)");
  KBO_CUDA(h, cudaSetDevice(h->device));
  nccl_unique_id uid;
  memcpy(&uid, id, sizeof uid);
  void* comm = nullptr;
  const int r = a->comm_init_rank(&comm, n_ranks, uid, rank);
  if (r != 0) KBO_FAIL(h, KBO_ERR_CUDA, "ncclCommInitRank failed: %s", a->get_error_string ? a->get_error_string(r) : "?");
  h->comm = comm;
  h->comm_ranks = n_ranks;
  h->comm_rank = rank;
  return kbo_reserve(h, h->comm_buf, (size_t)n_ranks);
}

int kbo_comm_destroy(kbo_handle* h) {
  if (!h) return KBO_ERR_INVALID;
  if (h->comm) {
    NcclApi* a = nccl_api();
    cudaSetDevice(h->device);
    if (a->comm_destroy) a->comm_destroy(h->comm);
    h->comm = nullptr;
    h->comm_ranks = 1;
    h->comm_rank = 0;
  }
  return KBO_OK;
}

int kbo_comm_size(kbo_handle* h) { return h ? h->comm_ranks : KBO_ERR_INVALID; }

int kbo_allreduce_argmax(kbo_handle* h, kbo_best* best_dev, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  if (!best_dev) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_allreduce_argmax: null argument");
  if (!h->comm || h->comm_ranks == 1) return KBO_OK;   // one rank: the local result is the global one
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  NcclApi* a = nccl_api();
  const int r = a->all_gather(best_dev, h->comm_buf.p, sizeof(kbo_best) / sizeof(double), 8 /* ncclFloat64 */, h->comm, s);
  if (r != 0) KBO_FAIL(h, KBO_ERR_CUDA, "ncclAllGather failed: %s", a->get_error_string ? a->get_error_string(r) : "?");
  argmax_reduce_kernel<<<1, 1, 0, s>>>(h->comm_buf.p, h->comm_ranks, best_dev);
  KBO_LAUNCH_CHECK(h);
  return KBO_OK;
}

}  // extern "C"
