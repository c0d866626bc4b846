// The loopback communicator's file and barrier (ethereum_consensus_b200/csrc/comm_loopback.h) built for the host, one
// communicator per process, with host memcpy where comm.cu copies to and from the device (tests/test_sharded_cases.py).
#include <cstring>
#include <string>

#include "../../ethereum_consensus_b200/csrc/comm_loopback.h"

namespace {
b200::Loopback g_loop;
std::string g_err;
int g_world = 1;
constexpr int kErrComm = 0x106;   // B200_ERR_COMM
}  // namespace

extern "C" {

__attribute__((visibility("default"))) int lb_open(const char* path, int rank, int world, unsigned long long slot_bytes,
                                                    unsigned timeout_ms) {
    g_world = world;
    return g_loop.open(path, rank, world, slot_bytes, timeout_ms, g_err) ? 0 : kErrComm;
}

// recv: world x bytes, rank-major
__attribute__((visibility("default"))) int lb_all_gather(const void* send, size_t bytes, void* recv) {
    uint8_t* mine = g_loop.send_slot(bytes, g_err);
    if (!mine) return kErrComm;
    if (bytes) memcpy(mine, send, bytes);
    const uint8_t* all = g_loop.arrive(g_err);
    if (!all) return kErrComm;
    for (int r = 0; r < g_world && bytes; r++) memcpy(static_cast<uint8_t*>(recv) + size_t(r) * bytes, all + size_t(r) * g_loop.slot_bytes(), bytes);
    return 0;
}

__attribute__((visibility("default"))) const char* lb_error() { return g_err.c_str(); }

__attribute__((visibility("default"))) void lb_close() { g_loop.close(); }

}  // extern "C"
