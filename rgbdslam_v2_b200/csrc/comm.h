// comm.h -- NCCL binding shared by the api_*.cu translation units (api_comm.cu owns the definitions).
#pragma once
#include <cuda_runtime.h>

#include "state.h"

namespace rb200 {

typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;

struct NcclApi {
  bool ok = false;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, int /*ncclDataType_t*/, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
extern NcclApi g_nccl;

struct Comm {
  static constexpr uint32_t kMagic = 0x434f4d4du;
  uint32_t magic = kMagic;
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1;
  DevBuf send, recv;
  cudaStream_t gstream = nullptr;        // the collectives of in-flight slots, in submission order
  DevBuf slot_recv[kSlots];
};

int load_nccl();
int nccl_fail(ncclResult_t r, const char* what);
Comm* get_comm(uint64_t h);  // nullptr (and last_error set) unless h is a live communicator handle

}  // namespace rb200
