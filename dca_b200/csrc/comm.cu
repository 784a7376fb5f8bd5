// Gradient exchange of the data-parallel training step INSIDE the library: one NCCL communicator per engine, the
// all-reduce of the flat gradient buffer enqueued by the same C call that launches the kernels, so that
//   phase 1 (forward + loss + head backward)  ->  all-reduce(head bucket)  ||  phase 2 (hidden / encoder backward)
//   ->  all-reduce(rest)  ->  join
// is ONE captured CUDA graph with zero Python between the kernels (SURVEY.md 8b names dca_allreduce, 8e the
// exchange; the reference has no multi-GPU path: dca/train.py:91-98 is a single-process Keras fit).
// libnccl is resolved at run time (dlopen of the copy torch has already mapped, else the system one), so
// libdca_b200.so carries no link-time dependency on it and loads on boxes without NCCL.
#include <dlfcn.h>
#include <nccl.h>
#include <cstdlib>
#include <cstring>
#include "dca_internal.cuh"
#include "engine.h"

namespace dca {

namespace {

struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
  bool ok = false;
};

NcclApi& api() {
  static NcclApi a;
  static bool tried = false;
  if (tried) return a;
  tried = true;
  // the copy already mapped into the process (torch's bundled NCCL) wins, so both users share one version
  a.lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
  if (!a.lib) a.lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!a.lib) a.lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!a.lib) return a;
#define DCA_SYM(field, name) *(void**)(&a.field) = dlsym(a.lib, name)
  DCA_SYM(GetUniqueId, "ncclGetUniqueId"); DCA_SYM(CommInitRank, "ncclCommInitRank"); DCA_SYM(CommDestroy, "ncclCommDestroy");
  DCA_SYM(AllReduce, "ncclAllReduce"); DCA_SYM(GroupStart, "ncclGroupStart"); DCA_SYM(GroupEnd, "ncclGroupEnd");
  DCA_SYM(GetErrorString, "ncclGetErrorString"); DCA_SYM(GetVersion, "ncclGetVersion");
#undef DCA_SYM
  a.ok = a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.AllReduce && a.GetErrorString;
  return a;
}

int need_api() {
  if (!api().ok) { set_error("NCCL is not available: libnccl.so.2 could not be loaded (%s)", dlerror() ? dlerror() : "missing symbols"); return DCA_ERR_UNSUPPORTED; }
  return DCA_OK;
}

#define DCA_NCCL_OK(expr)                                                                         \
  do {                                                                                            \
    ncclResult_t _r = (expr);                                                                     \
    if (_r != ncclSuccess) { set_error("%s failed: %s", #expr, api().GetErrorString(_r)); return DCA_ERR_CUDA; } \
  } while (0)

}  // namespace

int Engine::comm_init(const void* id128, int rank_, int world_) {
  DCA_TRY(need_api());
  if (!id128 || world_ < 1 || rank_ < 0 || rank_ >= world_) { set_error("dca_comm_init: bad rank / world (%d / %d)", rank_, world_); return DCA_ERR_BAD_ARG; }
  DCA_TRY(comm_destroy());
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  ncclComm_t c = nullptr;
  DCA_NCCL_OK(api().CommInitRank(&c, world_, id, rank_));
  comm = c; comm_world = world_; comm_rank = rank_;
  int least = 0, greatest = 0;
  DCA_CUDA_OK(cudaDeviceGetStreamPriorityRange(&least, &greatest));
  DCA_CUDA_OK(cudaStreamCreateWithPriority(&comm_stream, cudaStreamNonBlocking, greatest));
  DCA_CUDA_OK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
  DCA_CUDA_OK(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
  return DCA_OK;
}

int Engine::comm_destroy() {
  for (auto& c : graphs) if (c.phase == 3 && c.exec) { cudaGraphExecDestroy(c.exec); c.exec = nullptr; c.seen = 0; }
  if (comm) { if (api().ok) api().CommDestroy((ncclComm_t)comm); comm = nullptr; }
  if (comm_stream) { cudaStreamDestroy(comm_stream); comm_stream = nullptr; }
  if (ev_fork) { cudaEventDestroy(ev_fork); ev_fork = nullptr; }
  if (ev_join) { cudaEventDestroy(ev_join); ev_join = nullptr; }
  comm_world = 1; comm_rank = 0;
  return DCA_OK;
}

// sum all-reduce of grads[lo, hi) in place
int Engine::allreduce_range(int64_t lo, int64_t hi, cudaStream_t s) {
  if (!comm) { set_error("dca_allreduce: no communicator (dca_comm_init)"); return DCA_ERR_BAD_ARG; }
  if (hi <= lo) return DCA_OK;
  DCA_NCCL_OK(api().AllReduce(gp(lo), gp(lo), (size_t)(hi - lo), ncclFloat, ncclSum, (ncclComm_t)comm, s));
  count_launch(1);
  return DCA_OK;
}

int Engine::bn_allreduce(double* a, double* b, int n, cudaStream_t s) {
  if (!bn_synced()) return DCA_OK;
  if (api().GroupStart && b) DCA_NCCL_OK(api().GroupStart());
  DCA_NCCL_OK(api().AllReduce(a, a, (size_t)n, ncclDouble, ncclSum, (ncclComm_t)comm, s));
  if (b) DCA_NCCL_OK(api().AllReduce(b, b, (size_t)n, ncclDouble, ncclSum, (ncclComm_t)comm, s));
  if (api().GroupEnd && b) DCA_NCCL_OK(api().GroupEnd());
  count_launch(1);
  return DCA_OK;
}

// phase 1 -> [comm stream: all-reduce of the head gradients] || phase 2 -> all-reduce(rest) -> join.
// tensor-core path with several heads: phase 1 itself launches the head backward per head and enqueues each head's all-reduce as
// soon as that head's gradients are final (engine.cu), so only the loss slot / theta tail is left for the comm stream here.
int Engine::train_step_dp_body(const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf, const int32_t* rows,
                               int Bn, cudaStream_t s) {
  const int64_t hb = x_kind ? 0 : head_W[0];
  const bool split = !x_kind && tc_heads && !fused_heads && n_slots > 1 && split_heads_enabled();
  dp_split_heads = split;
  const int st1 = train_step_body(X, ldx, Y, ldy, sf, rows, Bn, s, 1);
  dp_split_heads = false;
  DCA_TRY(st1);
  DCA_CUDA_OK(cudaEventRecord(ev_fork, s));
  DCA_CUDA_OK(cudaStreamWaitEvent(comm_stream, ev_fork, 0));
  if (split) {
    // what the per-head all-reduces have not covered: everything behind the last head tensor (theta, loss slot, flag)
    int64_t tail = hb;
    for (int k = 0; k < n_slots; ++k) { const int64_t e = head_b[slot_head[k]] + cfg.n_out; if (e > tail) tail = e; }
    DCA_TRY(allreduce_range(tail, P + 2, comm_stream));
  } else {
    DCA_TRY(allreduce_range(hb, P + 2, comm_stream));
  }
  DCA_CUDA_OK(cudaEventRecord(ev_join, comm_stream));
  // The persistent kernels of phase 2 take one CTA (and most of the shared memory) of EVERY SM; the collective's CTAs then
  // only become resident when those retire and the "overlap" is a queue.  DCA_DP_RESERVE_SMS=n keeps n SMs free of them.
  static const int reserve = [] { const char* e = getenv("DCA_DP_RESERVE_SMS"); const int v = e ? atoi(e) : 0; return v < 0 ? 0 : (v > 100 ? 100 : v); }();
  dp_reserve_sms = reserve;
  const int st2 = train_step_body(X, ldx, Y, ldy, sf, rows, Bn, s, 2);
  dp_reserve_sms = 0;
  DCA_TRY(st2);
  DCA_TRY(allreduce_range(0, hb, s));
  DCA_CUDA_OK(cudaStreamWaitEvent(s, ev_join, 0));
  return DCA_OK;
}

bool Engine::split_heads_enabled() {
  // measured at N = 2 (C5 shard): three head-backward launches cost +32 us, more than the overlap returns -> opt-in
  static const bool on = [] { const char* e = getenv("DCA_DP_SPLIT_HEADS"); return e && e[0] == '1'; }();
  return on;
}

}  // namespace dca

using namespace dca;

extern "C" int dca_comm_unique_id(void* id128) {
  if (!id128) { set_error("dca_comm_unique_id: NULL"); return DCA_ERR_BAD_ARG; }
  DCA_TRY(need_api());
  ncclUniqueId id;
  DCA_NCCL_OK(api().GetUniqueId(&id));
  memcpy(id128, &id, sizeof(id));
  return DCA_OK;
}
extern "C" int dca_comm_init(dca_handle* h, const void* id128, int32_t rank, int32_t world) {
  if (!h) { set_error("dca_comm_init: handle is NULL"); return DCA_ERR_BAD_ARG; }
  return h->e.comm_init(id128, rank, world);
}
extern "C" int dca_comm_destroy(dca_handle* h) {
  if (!h) return DCA_OK;
  return h->e.comm_destroy();
}
extern "C" int dca_allreduce(dca_handle* h, void* stream) {
  if (!h) { set_error("dca_allreduce: handle is NULL"); return DCA_ERR_BAD_ARG; }
  return h->e.allreduce_range(0, h->e.P + 2, (cudaStream_t)stream);
}
extern "C" int dca_train_step_dp(dca_handle* h, const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf,
                                 const int32_t* rows, int32_t batch, void* stream) {
  if (!h) { set_error("dca_train_step_dp: handle is NULL"); return DCA_ERR_BAD_ARG; }
  if (!h->e.comm) { set_error("dca_train_step_dp: no communicator (dca_comm_init)"); return DCA_ERR_BAD_ARG; }
  return h->e.train_step(X, ldx, Y, ldy, sf, rows, batch, (cudaStream_t)stream, 3);
}
