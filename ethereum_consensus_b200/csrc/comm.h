// Process-global communicator of the library (comm.cu): one rank per process / per GPU.
#pragma once
#include "engine.h"

namespace b200 {

struct Comm {
    bool ready = false;
    int rank = 0, world = 1;
    void* nccl = nullptr;  // ncclComm_t when world > 1
    int nccl_version = 0;
};
Comm& comm();

// every rank contributes `bytes_per_rank` bytes; recv holds world x bytes_per_rank, rank-major.  Issued on `stream`.
int32_t comm_all_gather(Engine& e, const void* send, void* recv, size_t bytes_per_rank, cudaStream_t stream);

}  // namespace b200
