// Process-global engine context: one CUDA device, one stream, grow-only device/pinned buffers.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <mutex>
#include <string>

#include "../../include/b200_consensus.h"

namespace b200 {

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    // grow-only; contents are NOT preserved
    cudaError_t reserve(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = n + n / 8 + 4096;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

struct PinnedBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        size_t want = n + n / 8 + 4096;
        cudaError_t e = cudaMallocHost(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
};

struct Engine {
    bool ready = false;
    int device = -1;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaEvent_t ev_copy[17] = {nullptr};  // H2D slice k done (copy stream) -> compute stream may hash slice k
    std::mutex mu;
    std::string last_error;
    uint64_t launches = 0;
    uint64_t collectives = 0;  // NCCL collectives issued by the library (comm.cu)
    float last_kernel_ms = 0.f;
    // SSZ scratch (one-shot calls)
    DevBuf arena, fields, planbuf;
    PinnedBuf staging;
    DevBuf xch_dev;        // b200_comm_all_gather_bytes scratch
    PinnedBuf xch_host;
    uint32_t* d_zero = nullptr;  // 65 zero-subtree hashes, word form
    // BLS scratch lives in bls_engine (opaque here)
    void* bls = nullptr;
};

Engine& engine();

// The Validator records (121 bytes each, back to back, pubkey first) of a single-GPU resident state in HBM: *records and
// *n (nullptr and 0 for an empty list).  B200_ERR_BAD_ARG for a NULL or sharded handle.  The records move
// when the list outgrows its reserved region, so the pointer holds until the state's next call; the caller holds the
// engine lock.
int32_t state_validator_records(const b200_state* h, const uint8_t** records, uint64_t* n);

// eth_aggregate_public_keys (strict) of the public keys of Validator records index[0 .. n) (device) in HBM, the keys packed
// and validated on the device: *code and out48 as b200_eth_aggregate_public_keys_batch gives them for one group; keys48
// (host, n x 48) receives the keys.  The caller holds the engine lock (capi_bls.cu).
int32_t aggregate_record_keys(const uint8_t* records, const uint64_t* index, uint32_t n, uint8_t* keys48, uint8_t out48[48],
                              int32_t* code);

// Every entry point holds the engine lock for the whole call.
struct Guard {
    std::unique_lock<std::mutex> lk;
    explicit Guard(Engine& e) : lk(e.mu) {}
};

// B200_SUCCESS when b200_init succeeded; binds the calling thread to the engine's device
inline int32_t check_ready(Engine& e) {
    if (!e.ready) { e.last_error = "b200_init has not been called (or failed)"; return B200_ERR_NOT_INITIALIZED; }
    cudaError_t ce = cudaSetDevice(e.device);
    if (ce != cudaSuccess) { e.last_error = cudaGetErrorString(ce); return B200_ERR_CUDA; }
    return B200_SUCCESS;
}

#define B200_CUDA_TRY(expr)                                                                   \
    do {                                                                                      \
        cudaError_t e__ = (expr);                                                             \
        if (e__ != cudaSuccess) {                                                             \
            engine().last_error = std::string(#expr) + ": " + cudaGetErrorString(e__);        \
            return B200_ERR_CUDA;                                                             \
        }                                                                                     \
    } while (0)

}  // namespace b200
