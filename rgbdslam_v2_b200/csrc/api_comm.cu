// api_comm.cu -- the ONE exchange step of the multi-GPU path (SURVEY.md 8e): frame pairs are sharded over ranks
// without any data-path collective; the resulting fixed-size edge records (rgbdslam_b200_pair_result) are
// all-gathered once over NCCL (NVLink 5 / NVSwitch) before the replicated pose-graph solve.
// NCCL is bound at run time (dlsym on the already loaded library of the host process, else dlopen) so that the
// library itself loads on machines without NCCL / libcuda (CPU build check).
#include <dlfcn.h>

#include <cstring>
#include <mutex>

#include "comm.h"
#include "state.h"

namespace rb200 {

NcclApi g_nccl;

int load_nccl() {
  if (g_nccl.ok) return 0;
  void* h = RTLD_DEFAULT;
  if (!dlsym(h, "ncclAllGather")) {
    h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) {
      set_error(std::string("NCCL not available: ") + dlerror());
      return RGBDSLAM_B200_ERR_NCCL;
    }
  }
  g_nccl.GetUniqueId = (decltype(g_nccl.GetUniqueId))dlsym(h, "ncclGetUniqueId");
  g_nccl.CommInitRank = (decltype(g_nccl.CommInitRank))dlsym(h, "ncclCommInitRank");
  g_nccl.CommDestroy = (decltype(g_nccl.CommDestroy))dlsym(h, "ncclCommDestroy");
  g_nccl.AllGather = (decltype(g_nccl.AllGather))dlsym(h, "ncclAllGather");
  g_nccl.GetErrorString = (decltype(g_nccl.GetErrorString))dlsym(h, "ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.CommDestroy || !g_nccl.AllGather) {
    set_error("NCCL symbols missing");
    return RGBDSLAM_B200_ERR_NCCL;
  }
  g_nccl.ok = true;
  return 0;
}

int nccl_fail(ncclResult_t r, const char* what) {
  set_error(std::string("NCCL error in ") + what + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?"));
  return RGBDSLAM_B200_ERR_NCCL;
}

Comm* get_comm(uint64_t h) {
  Comm* c = (Comm*)(uintptr_t)h;
  if (!c || c->magic != Comm::kMagic) {
    set_error("invalid communicator handle");
    return nullptr;
  }
  return c;
}

}  // namespace rb200

using namespace rb200;

extern "C" {

int rgbdslam_b200_comm_unique_id(uint8_t* id128) {
  std::lock_guard<std::mutex> lk(g_state.mu);
  int rc = load_nccl();
  if (rc) return rc;
  if (!id128) {
    set_error("comm_unique_id: null output");
    return RGBDSLAM_B200_ERR_ARG;
  }
  ncclUniqueId id;
  ncclResult_t r = g_nccl.GetUniqueId(&id);
  if (r != 0) return nccl_fail(r, "ncclGetUniqueId");
  memcpy(id128, &id, 128);
  return 0;
}

int rgbdslam_b200_comm_init(int rank, int world, const uint8_t* id128, uint64_t* comm_handle) {
  RB200_ENTER_INITED();
  if (int rc = load_nccl()) return rc;
  if (!id128 || !comm_handle || world < 1 || rank < 0 || rank >= world) {
    set_error("comm_init: bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  Comm* c = new Comm();
  c->rank = rank;
  c->world = world;
  ncclUniqueId id;
  memcpy(&id, id128, 128);
  ncclResult_t r = g_nccl.CommInitRank(&c->comm, world, id, rank);
  if (r != 0) {
    delete c;
    return nccl_fail(r, "ncclCommInitRank");
  }
  *comm_handle = (uint64_t)(uintptr_t)c;
  g_state.comm_count++;
  return 0;
}

int rgbdslam_b200_comm_destroy(uint64_t comm_handle) {
  std::lock_guard<std::mutex> lk(g_state.mu);
  Comm* c = get_comm(comm_handle);
  if (!c) return RGBDSLAM_B200_ERR_ARG;
  if (g_nccl.ok && c->comm) g_nccl.CommDestroy(c->comm);
  c->send.release();
  c->recv.release();
  for (int k = 0; k < kSlots; k++) c->slot_recv[k].release();
  if (c->gstream) cudaStreamDestroy(c->gstream);
  c->magic = 0;
  delete c;
  g_state.comm_count--;
  return 0;
}

int rgbdslam_b200_allgather_edges(uint64_t comm_handle, const rgbdslam_b200_pair_result* local, int n_per_rank,
                                  rgbdslam_b200_pair_result* all) {
  RB200_ENTER_INITED();
  Comm* c = get_comm(comm_handle);
  if (!c) return RGBDSLAM_B200_ERR_ARG;
  if (n_per_rank < 0 || (n_per_rank > 0 && (!local || !all))) {
    set_error("allgather_edges: bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (n_per_rank == 0) return 0;
  const size_t bytes = sizeof(rgbdslam_b200_pair_result) * (size_t)n_per_rank;
  int rc;
  if ((rc = c->send.ensure(bytes)) || (rc = c->recv.ensure(bytes * c->world))) return rc;
  cudaStream_t st = g_state.stream;
  RB200_CUDA(cudaMemcpyAsync(c->send.ptr, local, bytes, cudaMemcpyHostToDevice, st));
  ncclResult_t r = g_nccl.AllGather(c->send.ptr, c->recv.ptr, bytes, 0 /* ncclInt8 */, c->comm, st);
  if (r != 0) return nccl_fail(r, "ncclAllGather");
  RB200_CUDA(cudaMemcpyAsync(all, c->recv.ptr, bytes * c->world, cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// The exchange step of a batch in flight: the edge records of slot `slot` (still on the device) are all-gathered on the
// communicator's own stream as soon as the slot's kernels have finished, and land in `all` (host, world * n_per_rank records);
// rgbdslam_b200_match_pairs_wait(slot) also waits for this.  No host round trip, the next batch can be submitted meanwhile.
// Every rank must issue these calls in the same slot order.
int rgbdslam_b200_allgather_slot_edges(uint64_t comm_handle, int slot, int n_per_rank, rgbdslam_b200_pair_result* all) {
  RB200_ENTER_INITED();
  Comm* c = get_comm(comm_handle);
  Workspace* ws = c ? get_slot(slot) : nullptr;
  if (!ws) return RGBDSLAM_B200_ERR_ARG;
  if (n_per_rank < 0 || (n_per_rank > 0 && !all)) {
    set_error("allgather_slot_edges: bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  Workspace& w = *ws;
  if (!w.pending || n_per_rank == 0) {
    set_error("allgather_slot_edges: the slot has no batch in flight (call it right after match_pairs*_submit)");
    return RGBDSLAM_B200_ERR_STATE;
  }
  const size_t bytes = sizeof(rgbdslam_b200_pair_result) * (size_t)n_per_rank;
  if (w.d_results.cap < bytes) {
    set_error("allgather_slot_edges: n_per_rank exceeds the batch submitted on this slot");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (!c->gstream) RB200_CUDA(cudaStreamCreateWithFlags(&c->gstream, cudaStreamNonBlocking));
  if (int rc = c->slot_recv[slot].ensure(bytes * c->world)) return rc;
  RB200_CUDA(cudaEventRecord(w.ev[kEvGatherDep], w.stream));  // everything the slot has queued so far
  RB200_CUDA(cudaStreamWaitEvent(c->gstream, w.ev[kEvGatherDep], 0));
  ncclResult_t r = g_nccl.AllGather(w.d_results.ptr, c->slot_recv[slot].ptr, bytes, 0 /* ncclInt8 */, c->comm, c->gstream);
  if (r != 0) return nccl_fail(r, "ncclAllGather");
  RB200_CUDA(cudaMemcpyAsync(all, c->slot_recv[slot].ptr, bytes * c->world, cudaMemcpyDeviceToHost, c->gstream));
  RB200_CUDA(cudaEventRecord(w.ev_gather, c->gstream));
  w.gather_pending = true;
  return 0;
}

}  // extern "C"
