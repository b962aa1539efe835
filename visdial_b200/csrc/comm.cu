// Data-parallel gradient all-reduce (SURVEY.md §8e): one ncclAllReduce(SUM) of the flat fp32 gradient per
// training step.  The reference has no counterpart (train.lua is single-GPU).  NCCL is bound with dlopen so
// that the library loads (and every single-GPU path works) on a host without libnccl, and so that a Python
// process that already carries torch's libnccl.so.2 reuses that copy instead of loading a second one.
#include "engine.h"
#include <dlfcn.h>
#include <string.h>
#include <stdlib.h>
#include <utility>

namespace vd {
namespace {
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
enum { ncclFloat32 = 7, ncclSum = 0 };

struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};

NcclApi& api() {
  static NcclApi a;
  if (a.handle) return a;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    a.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (a.handle) break;
  }
  VD_REQUIRE(a.handle != nullptr, VD_E_COMM, "cannot dlopen libnccl.so.2");
  a.GetUniqueId = (decltype(a.GetUniqueId))dlsym(a.handle, "ncclGetUniqueId");
  a.CommInitRank = (decltype(a.CommInitRank))dlsym(a.handle, "ncclCommInitRank");
  a.AllReduce = (decltype(a.AllReduce))dlsym(a.handle, "ncclAllReduce");
  a.CommDestroy = (decltype(a.CommDestroy))dlsym(a.handle, "ncclCommDestroy");
  a.GetErrorString = (decltype(a.GetErrorString))dlsym(a.handle, "ncclGetErrorString");
  a.GroupStart = (decltype(a.GroupStart))dlsym(a.handle, "ncclGroupStart");
  a.GroupEnd = (decltype(a.GroupEnd))dlsym(a.handle, "ncclGroupEnd");
  VD_REQUIRE(a.GetUniqueId && a.CommInitRank && a.AllReduce && a.CommDestroy, VD_E_COMM, "libnccl lacks required symbols");
  return a;
}

void nccl_check(ncclResult_t r, const char* what) {
  if (r == 0) return;
  char buf[256];
  snprintf(buf, sizeof(buf), "NCCL %s failed: %s", what, api().GetErrorString ? api().GetErrorString(r) : "?");
  throw CudaError(VD_E_COMM, buf);
}
}  // namespace

void comm_unique_id(void* out) {
  ncclUniqueId id;
  nccl_check(api().GetUniqueId(&id), "ncclGetUniqueId");
  static_assert(sizeof(ncclUniqueId) == VD_COMM_ID_BYTES, "unique id size");
  memcpy(out, &id, sizeof(id));
}

void comm_init(Engine* e, const void* idbytes, int rank, int world) {
  VD_REQUIRE(world >= 1 && rank >= 0 && rank < world, VD_E_BADARG, "bad rank/world");
  VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
  if (e->nccl_comm) { api().CommDestroy((ncclComm_t)e->nccl_comm); e->nccl_comm = nullptr; }
  e->rank = rank; e->world = world;
  if (world == 1) return;
  ncclUniqueId id;
  memcpy(&id, idbytes, sizeof(id));
  ncclComm_t comm;
  nccl_check(api().CommInitRank(&comm, world, id, rank), "ncclCommInitRank");
  e->nccl_comm = comm;
}

void comm_destroy(Engine* e) {
  if (e->comm_stream) {
    cudaStreamSynchronize(e->comm_stream);
    cudaStreamDestroy(e->comm_stream); e->comm_stream = nullptr;
    if (e->ev_comm_dep) cudaEventDestroy(e->ev_comm_dep);
    if (e->ev_comm_done) cudaEventDestroy(e->ev_comm_done);
    e->ev_comm_dep = e->ev_comm_done = nullptr;
  }
  if (e->nccl_comm) { api().CommDestroy((ncclComm_t)e->nccl_comm); e->nccl_comm = nullptr; }
}

void Engine::arm_grad_sync() {
  seg_reduced.assign(lay.segs.size(), 0);
  ar_armed = world > 1 && ar_overlap && nccl_comm != nullptr;
}

// one ncclAllReduce(SUM) of dW[off, off+count) on the communication stream, ordered behind `producer` (or its event)
void Engine::reduce_range(int64_t off, int64_t count, cudaStream_t producer, cudaEvent_t producer_event) {
  VD_REQUIRE(nccl_comm != nullptr, VD_E_STATE, "communicator not initialised");
  if (!comm_stream) {
    int lo = 0, hi = 0;
    VD_CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    VD_CUDA_CHECK(cudaStreamCreateWithPriority(&comm_stream, cudaStreamNonBlocking, hi));
    VD_CUDA_CHECK(cudaEventCreateWithFlags(&ev_comm_dep, cudaEventDisableTiming));
    VD_CUDA_CHECK(cudaEventCreateWithFlags(&ev_comm_done, cudaEventDisableTiming));
  }
  if (!producer_event) {
    VD_CUDA_CHECK(cudaEventRecord(ev_comm_dep, producer));
    producer_event = ev_comm_dep;
  }
  VD_CUDA_CHECK(cudaStreamWaitEvent(comm_stream, producer_event, 0));
  cudaStream_t prev = cx.stream;
  cx.stream = comm_stream;
  {
    LaunchCtx::Scope sc(&cx, "allreduce", 0.0, 2.0 * 4.0 * (double)count);
    nccl_check(api().AllReduce(dW + off, dW + off, (size_t)count, ncclFloat32, ncclSum, (ncclComm_t)nccl_comm, comm_stream), "ncclAllReduce");
  }
  cx.stream = prev;
  comm_pending = true;
}

void Engine::reduce_segments(int first, int last, cudaStream_t producer, cudaEvent_t producer_event) {
  if (!ar_armed) return;
  VD_REQUIRE(first >= 0 && last >= first && last < (int)lay.segs.size(), VD_E_STATE, "reduce_segments: range");
  for (int i = first; i <= last; ++i) {
    VD_REQUIRE(!seg_reduced[i], VD_E_STATE, "gradient bucket reduced twice");
    seg_reduced[i] = 1;
  }
  const int64_t off = lay.segs[first].off;
  const int64_t end = last + 1 < (int)lay.segs.size() ? lay.segs[last + 1].off : nparams;
  reduce_range(off, end - off, producer, producer_event);
}

void Engine::reduce_remaining() {
  if (world <= 1) return;
  VD_REQUIRE(nccl_comm != nullptr, VD_E_STATE, "communicator not initialised");
  join_options_backward();
  if (seg_reduced.size() != lay.segs.size()) seg_reduced.assign(lay.segs.size(), 0);
  const int n = (int)lay.segs.size();
  // the segments still local (at least the word embedding, which every branch writes; with the option stream also opt.lstm,
  // final at the same moment) go out as ONE grouped launch: one collective latency at the exposed end of the step
  std::vector<std::pair<int64_t, int64_t>> runs;
  for (int i = 0; i < n;) {
    if (seg_reduced[i]) { ++i; continue; }
    int j = i;
    while (j + 1 < n && !seg_reduced[j + 1]) ++j;
    for (int k = i; k <= j; ++k) seg_reduced[k] = 1;
    const int64_t off = lay.segs[i].off;
    const int64_t end = j + 1 < n ? lay.segs[j + 1].off : nparams;
    runs.emplace_back(off, end - off);
    i = j + 1;
  }
  if (!runs.empty()) {
    const bool grouped = runs.size() > 1 && api().GroupStart && api().GroupEnd;
    if (grouped) nccl_check(api().GroupStart(), "ncclGroupStart");
    for (size_t r = 0; r < runs.size(); ++r) reduce_range(runs[r].first, runs[r].second, main_stream, nullptr);
    if (grouped) nccl_check(api().GroupEnd(), "ncclGroupEnd");
  }
  if (comm_pending) {
    VD_CUDA_CHECK(cudaEventRecord(ev_comm_done, comm_stream));
    VD_CUDA_CHECK(cudaStreamWaitEvent(main_stream, ev_comm_done, 0));
    comm_pending = false;
  }
  ar_armed = false;
}

void Engine::allreduce_grads() { reduce_remaining(); }

}  // namespace vd
