// Loopback communicator: the all-gather of comm.cu through one file that every rank maps (MAP_SHARED), so that several
// processes on ONE GPU can run the sharded entry points at world > 1.  Test use only (b200_comm_init_loopback): it stands
// in for NCCL behind comm_all_gather and is not a production transport.  No CUDA here, so that a host test can compile it
// with g++ and run the barrier in plain processes; comm.cu moves the bytes between the device and the slots.
//
// File layout: a 64-byte header (magic, world, slot size, arrival counter), then two generations of `world` slots of
// `slot_bytes`.  Gather number g of a rank: write its slot of parity g & 1, arrive (counter + 1), wait until the counter
// reaches world * (g + 1), read the world slots of that parity.  Two parities suffice: a rank writes generation g + 2
// only after every rank arrived at g + 1, i.e. after every rank finished reading generation g.  The file must be new
// (or all zero) for each communicator.
#pragma once
#include <fcntl.h>
#include <sched.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <time.h>
#include <unistd.h>

#include <cstdint>
#include <cstring>
#include <string>

namespace b200 {

struct LoopbackHeader {
    uint64_t magic;      // written last by the rank that initialised the header
    uint64_t world;
    uint64_t slot_bytes;
    uint64_t arrived;    // arrivals since the file was made: generation g is complete at world * (g + 1)
    uint64_t claim;      // 0 -> 1 by the one rank that initialises the header
    uint64_t pad[3];
};
static_assert(sizeof(LoopbackHeader) == 64, "the slots start at byte 64");

class Loopback {
public:
    static constexpr uint64_t kMagic = 0x6b6f6f6c30303262ull;   // "b200look"

    bool active() const { return base_ != nullptr; }
    uint64_t generation() const { return gen_; }

    // Maps `path` (created if missing) for `world` ranks of `slot_bytes` each.  False, with `err`, when the file cannot be
    // mapped, when its header names another world or slot size, or when no rank initialises it within the timeout.
    bool open(const char* path, int rank, int world, uint64_t slot_bytes, uint32_t timeout_ms, std::string& err) {
        close();
        if (!path || world < 1 || rank < 0 || rank >= world || !slot_bytes || slot_bytes > (uint64_t(1) << 40) / uint64_t(world)) {
            err = "loopback: bad arguments";
            return false;
        }
        const size_t len = sizeof(LoopbackHeader) + 2 * size_t(world) * size_t(slot_bytes);
        const int fd = ::open(path, O_RDWR | O_CREAT, 0600);
        if (fd < 0) { err = std::string("loopback: cannot open ") + path; return false; }
        struct stat st;
        // grow only: a rank that would shrink the file under another's mapping reads the header and is refused instead
        bool ok = fstat(fd, &st) == 0 && (size_t(st.st_size) >= len || ftruncate(fd, off_t(len)) == 0);
        void* p = ok ? mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0) : MAP_FAILED;
        ::close(fd);
        if (p == MAP_FAILED) { err = std::string("loopback: cannot map ") + path; return false; }
        base_ = static_cast<uint8_t*>(p);
        len_ = len;
        LoopbackHeader* h = header();
        uint64_t zero = 0;
        if (__atomic_compare_exchange_n(&h->claim, &zero, 1, false, __ATOMIC_ACQ_REL, __ATOMIC_ACQUIRE)) {
            h->world = uint64_t(world);
            h->slot_bytes = slot_bytes;
            __atomic_store_n(&h->arrived, 0, __ATOMIC_RELAXED);
            __atomic_store_n(&h->magic, kMagic, __ATOMIC_RELEASE);
        }
        const uint64_t t0 = now_ms();
        for (unsigned spin = 0; __atomic_load_n(&h->magic, __ATOMIC_ACQUIRE) != kMagic; spin++) {
            if (now_ms() - t0 > timeout_ms) { err = "loopback: the file header was never initialised"; close(); return false; }
            backoff(spin);
        }
        if (h->world != uint64_t(world) || h->slot_bytes != slot_bytes) {
            err = "loopback: the file was made for world " + std::to_string(h->world) + ", slot " + std::to_string(h->slot_bytes) +
                  " B, not world " + std::to_string(world) + ", slot " + std::to_string(slot_bytes) + " B";
            close();
            return false;
        }
        rank_ = rank; world_ = world; slot_ = slot_bytes; timeout_ms_ = timeout_ms;
        gen_ = 0;
        poisoned_ = false;
        return true;
    }

    // This rank's slot of the next generation, to be filled with `bytes` bytes; nullptr (with `err`) when the call is larger
    // than a slot or an earlier gather timed out.
    uint8_t* send_slot(size_t bytes, std::string& err) {
        if (poisoned_) { err = "loopback: an earlier all-gather timed out; the communicator is unusable"; return nullptr; }
        if (bytes > slot_) {
            err = "loopback: " + std::to_string(bytes) + " B per rank exceeds the slot of " + std::to_string(slot_) + " B";
            return nullptr;
        }
        return slots(gen_) + size_t(rank_) * slot_;
    }

    // Arrive at the current generation and wait for every rank; then the world slots (slot_bytes apart, rank-major) of
    // that generation, and the generation advances.  nullptr (with `err`) on timeout, which poisons the communicator.
    const uint8_t* arrive(std::string& err) {
        if (poisoned_) { err = "loopback: an earlier all-gather timed out; the communicator is unusable"; return nullptr; }
        LoopbackHeader* h = header();
        const uint64_t need = uint64_t(world_) * (gen_ + 1);
        __atomic_add_fetch(&h->arrived, 1, __ATOMIC_ACQ_REL);   // release: this rank's slot bytes
        const uint64_t t0 = now_ms();
        uint64_t got;
        for (unsigned spin = 0; (got = __atomic_load_n(&h->arrived, __ATOMIC_ACQUIRE)) < need; spin++) {
            if (now_ms() - t0 > timeout_ms_) {
                const uint64_t here = got > uint64_t(world_) * gen_ ? got - uint64_t(world_) * gen_ : 0;
                err = "loopback: all-gather generation " + std::to_string(gen_) + " timed out after " + std::to_string(timeout_ms_) +
                      " ms with " + std::to_string(here) + " of " + std::to_string(world_) + " ranks arrived";
                poisoned_ = true;
                return nullptr;
            }
            backoff(spin);
        }
        return slots(gen_++);
    }

    uint64_t slot_bytes() const { return slot_; }

    void close() {
        if (base_) munmap(base_, len_);
        base_ = nullptr;
        len_ = 0;
        gen_ = 0;
        poisoned_ = false;
    }

    ~Loopback() { close(); }

private:
    LoopbackHeader* header() const { return reinterpret_cast<LoopbackHeader*>(base_); }
    uint8_t* slots(uint64_t g) const { return base_ + sizeof(LoopbackHeader) + size_t(g & 1) * size_t(world_) * slot_; }

    static uint64_t now_ms() {
        timespec ts;
        clock_gettime(CLOCK_MONOTONIC, &ts);
        return uint64_t(ts.tv_sec) * 1000u + uint64_t(ts.tv_nsec) / 1000000u;
    }
    // a short spin, then sleeps growing to 1 ms: the ranks share one GPU, and a waiting rank must not take its CPU
    static void backoff(unsigned spin) {
        if (spin < 64) { sched_yield(); return; }
        const long us = spin < 1024 ? 10 + long(spin - 64) : 1000;
        timespec ts{0, (us < 1000 ? us : 1000) * 1000};
        nanosleep(&ts, nullptr);
    }

    uint8_t* base_ = nullptr;
    size_t len_ = 0;
    int rank_ = 0, world_ = 1;
    uint64_t slot_ = 0, gen_ = 0;
    uint32_t timeout_ms_ = 0;
    bool poisoned_ = false;
};

}  // namespace b200
