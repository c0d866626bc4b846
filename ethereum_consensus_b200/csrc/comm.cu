// Multi-GPU exchange INSIDE the library (SURVEY.md §8e, include/b200_consensus.h "multi-GPU"): one process per GPU, one
// NCCL communicator per process, every collective issued on the engine's own stream so it is ordered with the kernels
// that produce / consume its buffers — no host round trip between "hash my slice" and "finish the tree".
//
// NCCL is bound at run time (dlopen "libnccl.so.2"): a host process that already carries NCCL (PyTorch bundles one)
// shares that copy instead of loading a second, and a single-GPU deployment never needs the library at all.
// The reference has no counterpart (it is single-process, SURVEY.md §2a); the messages are tiny (160 B of subtree
// roots, 4 B per verdict, 576 B of Gt) so the collectives are latency-bound over NVLink — one per call.
// b200_comm_init_loopback puts a test transport behind the same comm_all_gather (comm_loopback.h): one file shared by
// processes on one GPU, so the sharded paths run at world > 1 where two GPUs are not available.
#include <dlfcn.h>
#include <nccl.h>

#include <cstring>

#include "comm.h"
#include "comm_loopback.h"

namespace b200 {
namespace {

struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    ncclResult_t (*GetVersion)(int*) = nullptr;
};
NcclApi g_nccl;
Comm g_comm;
Loopback g_loop;   // active between b200_comm_init_loopback and b200_comm_destroy

template <class F>
bool bind(F& fn, const char* name) {
    fn = reinterpret_cast<F>(dlsym(g_nccl.handle, name));
    return fn != nullptr;
}

int32_t load_nccl(Engine& e) {
    if (g_nccl.handle) return B200_SUCCESS;
    const char* names[] = {getenv("B200_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
        if (!n || !*n) continue;
        g_nccl.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (g_nccl.handle) break;
    }
    if (!g_nccl.handle) {
        e.last_error = std::string("NCCL not found (dlopen libnccl.so.2): ") + (dlerror() ? dlerror() : "");
        return B200_ERR_COMM;
    }
    bool ok = bind(g_nccl.GetUniqueId, "ncclGetUniqueId") && bind(g_nccl.CommInitRank, "ncclCommInitRank") &&
              bind(g_nccl.CommDestroy, "ncclCommDestroy") && bind(g_nccl.AllGather, "ncclAllGather") &&
              bind(g_nccl.GetErrorString, "ncclGetErrorString") &&
              bind(g_nccl.GetVersion, "ncclGetVersion");
    if (!ok) {
        e.last_error = "NCCL library lacks a required symbol";
        dlclose(g_nccl.handle);
        g_nccl = NcclApi();
        return B200_ERR_COMM;
    }
    return B200_SUCCESS;
}

int32_t nccl_fail(Engine& e, const char* what, ncclResult_t r) {
    e.last_error = std::string(what) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "NCCL error");
    return B200_ERR_COMM;
}

// The all-gather through the loopback file: the send bytes go to this rank's slot once the stream has produced them,
// the ranks meet at the file's barrier, and the world slots are copied to `recv` on the stream.
int32_t loopback_all_gather(Engine& e, const void* send, void* recv, size_t bytes_per_rank, cudaStream_t stream) {
    uint8_t* mine = g_loop.send_slot(bytes_per_rank, e.last_error);
    if (!mine) return B200_ERR_COMM;
    if (bytes_per_rank) B200_CUDA_TRY(cudaMemcpyAsync(mine, send, bytes_per_rank, cudaMemcpyDeviceToHost, stream));
    B200_CUDA_TRY(cudaStreamSynchronize(stream));
    const uint8_t* all = g_loop.arrive(e.last_error);
    if (!all) return B200_ERR_COMM;
    for (int r = 0; r < g_comm.world && bytes_per_rank; r++)
        B200_CUDA_TRY(cudaMemcpyAsync(static_cast<uint8_t*>(recv) + size_t(r) * bytes_per_rank, all + size_t(r) * g_loop.slot_bytes(),
                                      bytes_per_rank, cudaMemcpyHostToDevice, stream));
    e.collectives++;
    return B200_SUCCESS;
}

}  // namespace

Comm& comm() { return g_comm; }

int32_t comm_all_gather(Engine& e, const void* send, void* recv, size_t bytes_per_rank, cudaStream_t stream) {
    Comm& c = g_comm;
    if (!c.ready) { e.last_error = "b200_comm_init has not been called"; return B200_ERR_NOT_INITIALIZED; }
    if (c.world == 1) {
        if (send != recv && bytes_per_rank)
            B200_CUDA_TRY(cudaMemcpyAsync(recv, send, bytes_per_rank, cudaMemcpyDeviceToDevice, stream));
        return B200_SUCCESS;
    }
    if (g_loop.active()) return loopback_all_gather(e, send, recv, bytes_per_rank, stream);
    ncclResult_t r = g_nccl.AllGather(send, recv, bytes_per_rank, ncclUint8, static_cast<ncclComm_t>(c.nccl), stream);
    if (r != ncclSuccess) return nccl_fail(e, "ncclAllGather", r);
    e.collectives++;
    return B200_SUCCESS;
}

}  // namespace b200

using namespace b200;

extern "C" {

int32_t b200_comm_unique_id(uint8_t out_id[B200_COMM_ID_BYTES]) {
    Engine& e = engine();
    std::unique_lock<std::mutex> lk(e.mu);
    if (!out_id) return B200_ERR_BAD_ARG;
    int32_t rc = load_nccl(e);
    if (rc) return rc;
    static_assert(sizeof(ncclUniqueId) == B200_COMM_ID_BYTES, "ncclUniqueId is 128 bytes");
    ncclUniqueId id;
    ncclResult_t r = g_nccl.GetUniqueId(&id);
    if (r != ncclSuccess) return nccl_fail(e, "ncclGetUniqueId", r);
    memcpy(out_id, &id, sizeof(id));
    return B200_SUCCESS;
}

int32_t b200_comm_init(const uint8_t id[B200_COMM_ID_BYTES], int32_t rank, int32_t world) {
    Engine& e = engine();
    std::unique_lock<std::mutex> lk(e.mu);
    if (!e.ready) { e.last_error = "b200_init must precede b200_comm_init"; return B200_ERR_NOT_INITIALIZED; }
    if (world < 1 || rank < 0 || rank >= world || (world > 1 && !id)) return B200_ERR_BAD_ARG;
    Comm& c = g_comm;
    if (c.ready) return (c.rank == rank && c.world == world) ? B200_SUCCESS : B200_ERR_BAD_ARG;
    B200_CUDA_TRY(cudaSetDevice(e.device));
    if (world > 1) {
        int32_t rc = load_nccl(e);
        if (rc) return rc;
        ncclUniqueId nid;
        memcpy(&nid, id, sizeof(nid));
        ncclComm_t nc = nullptr;
        ncclResult_t r = g_nccl.CommInitRank(&nc, world, nid, rank);
        if (r != ncclSuccess) return nccl_fail(e, "ncclCommInitRank", r);
        c.nccl = nc;
        g_nccl.GetVersion(&c.nccl_version);
    }
    c.rank = rank; c.world = world; c.ready = true;
    return B200_SUCCESS;
}

int32_t b200_comm_init_loopback(const char* path, int32_t rank, int32_t world, uint64_t slot_bytes, uint32_t timeout_ms) {
    Engine& e = engine();
    std::unique_lock<std::mutex> lk(e.mu);
    if (!e.ready) { e.last_error = "b200_init must precede b200_comm_init_loopback"; return B200_ERR_NOT_INITIALIZED; }
    if (!path || world < 1 || rank < 0 || rank >= world || !slot_bytes) return B200_ERR_BAD_ARG;
    Comm& c = g_comm;
    if (c.ready) return (c.rank == rank && c.world == world) ? B200_SUCCESS : B200_ERR_BAD_ARG;
    B200_CUDA_TRY(cudaSetDevice(e.device));
    if (!g_loop.open(path, rank, world, slot_bytes, timeout_ms, e.last_error)) return B200_ERR_COMM;
    c.rank = rank; c.world = world; c.ready = true;
    return B200_SUCCESS;
}

int32_t b200_comm_info(int32_t* rank, int32_t* world, int32_t* nccl_version) {
    Comm& c = g_comm;
    if (!c.ready) return B200_ERR_NOT_INITIALIZED;
    if (rank) *rank = c.rank;
    if (world) *world = c.world;
    if (nccl_version) *nccl_version = c.nccl_version;
    return B200_SUCCESS;
}

uint64_t b200_collective_count(void) { return engine().collectives; }

// Host-buffer all-gather for the hosts' own small exchanges (e.g. per-shard verdict vectors when every rank verified a
// DIFFERENT batch): staged through the engine's pinned + device scratch, one ncclAllGather on the engine stream.
int32_t b200_comm_all_gather_bytes(const uint8_t* send, size_t bytes_per_rank, uint8_t* recv) {
    Engine& e = engine();
    std::unique_lock<std::mutex> lk(e.mu);
    if (!e.ready) return B200_ERR_NOT_INITIALIZED;
    Comm& c = g_comm;
    if (!c.ready) { e.last_error = "b200_comm_init has not been called"; return B200_ERR_NOT_INITIALIZED; }
    if ((!send || !recv) && bytes_per_rank) return B200_ERR_BAD_ARG;
    if (!bytes_per_rank) return B200_SUCCESS;
    B200_CUDA_TRY(cudaSetDevice(e.device));
    const size_t padded = (bytes_per_rank + 15) & ~size_t(15), total = padded * size_t(c.world);
    B200_CUDA_TRY(e.xch_dev.reserve(padded + total));
    B200_CUDA_TRY(e.xch_host.reserve(padded + total));
    uint8_t* h = static_cast<uint8_t*>(e.xch_host.p);
    uint8_t* d = static_cast<uint8_t*>(e.xch_dev.p);
    memcpy(h, send, bytes_per_rank);
    B200_CUDA_TRY(cudaMemcpyAsync(d, h, padded, cudaMemcpyHostToDevice, e.stream));
    int32_t rc = comm_all_gather(e, d, d + padded, padded, e.stream);
    if (rc) return rc;
    B200_CUDA_TRY(cudaMemcpyAsync(h + padded, d + padded, total, cudaMemcpyDeviceToHost, e.stream));
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    for (int r = 0; r < c.world; r++) memcpy(recv + size_t(r) * bytes_per_rank, h + padded + size_t(r) * padded, bytes_per_rank);
    return B200_SUCCESS;
}

void b200_comm_destroy(void) {
    Engine& e = engine();
    std::unique_lock<std::mutex> lk(e.mu);
    Comm& c = g_comm;
    if (!c.ready) return;
    if (e.ready) { cudaSetDevice(e.device); cudaStreamSynchronize(e.stream); }
    if (c.nccl && g_nccl.CommDestroy) g_nccl.CommDestroy(static_cast<ncclComm_t>(c.nccl));
    g_loop.close();
    c = Comm();
}

}  // extern "C"
