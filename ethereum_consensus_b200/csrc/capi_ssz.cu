// extern "C" entry points — engine life cycle and the SSZ half of include/b200_consensus.h.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <vector>

#include "comm.h"
#include "engine.h"
#include "epoch.h"
#include "sha256.cuh"
#include "sha256_hd.cuh"
#include "shuffle.h"
#include "ssz_plan.h"

namespace b200 {

Engine& engine() {
    static Engine e;
    return e;
}

namespace {

// crypto::hash on the device: one thread, arbitrary length (parity helper; not a throughput path)
__global__ void k_sha256_bytes(const uint8_t* data, size_t len, uint32_t* out_words) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    uint32_t st[8], w[16];
    sha256_init(st);
    size_t nblocks = (len + 9 + 63) / 64;
    for (size_t b = 0; b < nblocks; b++) {
        for (int i = 0; i < 16; i++) {
            uint32_t v = 0;
            for (int k = 0; k < 4; k++) {
                size_t pos = b * 64 + size_t(i) * 4 + size_t(k);
                uint32_t byte = 0;
                if (pos < len) byte = data[pos];
                else if (pos == len) byte = 0x80;
                else if (pos >= nblocks * 64 - 8) byte = uint32_t((uint64_t(len) * 8) >> (8 * (nblocks * 64 - 1 - pos))) & 0xff;
                v = (v << 8) | byte;
            }
            w[i] = v;
        }
        sha256_compress(st, w);
    }
    for (int i = 0; i < 8; i++) out_words[i] = st[i];
}

int32_t run_oneshot(Engine& e, SszPlan& plan, const std::vector<uint32_t>& outputs, uint8_t* out) {
    return plan.run(e, e.arena, e.fields, e.planbuf, COPY_ALL, outputs, out);
}

}  // namespace
}  // namespace b200

using namespace b200;

struct b200_state {
    SszPlan plan;
    std::vector<uint32_t> outputs;
    DevBuf arena, fields, planbuf, selbuf, scatter;
    // ---- incremental re-hash (b200_state_update_* / b200_state_root_incremental) ----
    // Host shadow of the serialization with everything EXCEPT the five big lists filled in (their byte ranges are never
    // written or read: untouched zero pages of an anonymous mapping): small-field updates patch it and the plan is
    // rebuilt from it.  `shadow_cap` bytes are allocated, so that a reshape (b200_state_append_elements /
    // b200_state_set_field) moves the bytes after the changed field in place; past that it is re-allocated.
    uint8_t* shadow = nullptr;
    size_t len = 0, shadow_cap = 0;
    int preset = 0;
    StateOffsets so;
    uint64_t cap[5] = {0, 0, 0, 0, 0};   // elements each big list's device regions are reserved for
    // per chain (5 big lists, then block_roots / state_roots / randao_mixes / slashings): changed first-job inputs
    // (Validator records / 32-byte chunks), unsorted
    std::vector<uint32_t> dirty[9];
    std::vector<char> rehash = std::vector<char>(9, 0);  // chains to re-hash in full at the next root
    bool small_dirty = false;
    std::vector<std::pair<const uint8_t*, const uint8_t*>> small_ranges;  // patched shadow bytes since the last root
    uint8_t* pinned_head = nullptr;   // page-locked ranges of the shadow (registration is an optimisation)
    uint8_t* pinned_tail = nullptr;
    bool sharded = false;   // b200_state_upload_deneb_sharded: this rank's slices only; root is a collective, no updates
    // ---- beacon committees (b200_state_committee_count_per_slot ... b200_state_attesting_indices) ----
    // Bumped by every write into the Validator records (chain 0): a cached epoch built under another generation is stale.
    uint64_t records_gen = 0;
    // One epoch's shuffled active list, valid while its seed (recomputed from the shadow on every call) and the records'
    // generation are those it was built with; `pos` (the inverse map, one u32 per validator) is built on first use.
    struct CommitteeEpoch {
        bool used = false, pos_ready = false;
        uint64_t epoch = 0, gen = 0, n_active = 0, cps = 0, last_use = 0;
        uint8_t seed[32] = {0};
        DevBuf shuffled, pos;
    };
    static constexpr int kCommitteeEpochs = 4;   // previous, current and next, and one more asked epoch
    CommitteeEpoch committees[kCommitteeEpochs];
    uint64_t committee_tick = 0;
    DevBuf committee_work;   // per-call inputs and outputs of the committee kernels
    ~b200_state() {  // callers hold the engine lock and have selected the device
        if (pinned_head) cudaHostUnregister(pinned_head);
        if (pinned_tail) cudaHostUnregister(pinned_tail);
        free(shadow);
        arena.release(); fields.release(); planbuf.release(); selbuf.release(); scatter.release();
        for (CommitteeEpoch& c : committees) { c.shuffled.release(); c.pos.release(); }
        committee_work.release();
    }
};

namespace {
// a single-GPU resident state: the calls that update, read or compute duties on a state take only these
bool resident(const b200_state* h) { return h && !h->sharded; }
// chain c of the handle's plan (ssz_plan.h: StateChain)
StateChain chain(const b200_state* h, int c) { return state_chain(h->so, preset_of(h->preset), c); }
// Device address of chain c's bytes on a resident handle.  Its plan stages all nine chains, and a big list's region is
// reserved for its capacity even while the list is empty.
uint8_t* chain_dev(const b200_state* h, int c) {
    uint64_t field_off = 0; size_t nbytes = 0;
    h->plan.chain_field(c, &field_off, &nbytes);
    return static_cast<uint8_t*>(h->fields.p) + field_off;
}
// Elements reserved beyond a big list's length when its device regions are (re)allocated: 2^16 (one 8 MB slab of
// Validator records) or a sixteenth of the list, whichever is larger.  Deposits then append in place for many blocks;
// crossing the capacity relocates the list on the device.
inline uint64_t headroom(uint64_t n) { return std::max<uint64_t>(uint64_t(1) << 16, n / 16); }
constexpr size_t kShadowSlack = 64 << 10;   // shadow bytes beyond the reserved lists: header / summaries growth

size_t shadow_bytes_for(const b200_state* h) {
    size_t b = h->len + kShadowSlack;
    for (int f = 0; f < 5; f++) b += size_t(h->cap[f] - chain(h, f).len) * chain(h, f).elem;
    const SmallList votes = appendable_small_list(B200_FIELD_ETH1_DATA_VOTES, preset_of(h->preset));
    return b + size_t(votes.limit * votes.elem) - (h->so.var[2] - h->so.var[1]);
}

// Page-lock the head of the shadow up to eth1_data_votes (the fixed part and historical_roots: it never changes size),
// and the tail (latest_execution_payload_header, the two withdrawal indices, historical_summaries) while it stays where
// it is.  A staged copy lies wholly inside or wholly outside each range (eth1_data_votes starts where the head ends).
void pin_shadow(b200_state* h, bool tail) {
    if (cudaHostRegister(h->shadow, h->so.var[1], cudaHostRegisterDefault) == cudaSuccess) h->pinned_head = h->shadow;
    if (tail && cudaHostRegister(h->shadow + h->so.var[7], h->len - h->so.var[7], cudaHostRegisterDefault) == cudaSuccess)
        h->pinned_tail = h->shadow + h->so.var[7];
    cudaGetLastError();  // pageable copies work too
}
void unpin_tail(b200_state* h) {
    if (h->pinned_tail) cudaHostUnregister(h->pinned_tail);
    h->pinned_tail = nullptr;
}

// Resize variable-size field k (StateOffsets::var index) of the shadow to `new_size` bytes: the shadow's bytes after it
// move, the offset words after it are rewritten, h->len follows.  The field's own bytes are the caller's to fill; call
// reparse() after.  Refuses (leaving everything as it was) a serialization beyond the 32-bit offsets' reach.
int32_t reshape_shadow(Engine& e, b200_state* h, int k, size_t new_size) {
    const size_t old_size = h->so.var[k + 1] - h->so.var[k];
    if (new_size == old_size) return B200_SUCCESS;
    const uint64_t new_len = uint64_t(h->len) - old_size + new_size;
    if (new_len > 0xffffffffull) { e.last_error = "state reshape: the serialization would exceed 4 GiB"; return B200_ERR_LIMIT; }
    if (new_len > h->shadow_cap) {
        const size_t want = shadow_bytes_for(h) + (new_len - h->len);
        uint8_t* ns = static_cast<uint8_t*>(calloc(want, 1));
        if (!ns) { e.last_error = "out of host memory for the state shadow"; return B200_ERR_CUDA; }
        memcpy(ns, h->shadow, h->so.var[2]);
        memcpy(ns + h->so.var[7], h->shadow + h->so.var[7], h->len - h->so.var[7]);
        if (h->pinned_head) cudaHostUnregister(h->pinned_head);
        h->pinned_head = nullptr;
        unpin_tail(h);
        free(h->shadow);
        h->shadow = ns; h->shadow_cap = want;
        pin_shadow(h, false);
    }
    // the shadow holds nothing of the big lists: what moves is [max(end of field k, start of the header), len)
    const size_t from = std::max<size_t>(h->so.var[k + 1], h->so.var[7]);
    unpin_tail(h);   // the tail moves or changes size: it stays pageable from now on (a few KB to copy)
    if (from < h->len) memmove(h->shadow + (from + new_size - old_size), h->shadow + from, h->len - from);
    for (int i = k + 1; i < 9; i++) {
        const uint32_t v = uint32_t(h->so.var[i] + new_size - old_size);
        uint8_t* w = h->shadow + h->so.var_word[i];
        w[0] = uint8_t(v); w[1] = uint8_t(v >> 8); w[2] = uint8_t(v >> 16); w[3] = uint8_t(v >> 24);
    }
    for (int i = k + 1; i < 10; i++) h->so.var[i] = uint32_t(h->so.var[i] + new_size - old_size);
    h->len = size_t(new_len);
    return B200_SUCCESS;
}
bool reparse(b200_state* h) { return parse_beacon_state(h->shadow, h->len, h->preset, h->so); }

// every small staged field: re-copied and re-hashed at the next root (their field-buffer and arena places follow the
// sizes of eth1_data_votes / the header / historical_summaries)
void mark_all_small(b200_state* h) {
    h->small_dirty = true;
    h->small_ranges.emplace_back(h->shadow, h->shadow + h->so.var[2]);
    h->small_ranges.emplace_back(h->shadow + h->so.var[7], h->shadow + h->len);
}

// after a root: every dirty path, full re-hash and patched small field is in it
void mark_clean(b200_state* h) {
    for (auto& d : h->dirty) d.clear();
    std::fill(h->rehash.begin(), h->rehash.end(), 0);
    h->small_dirty = false;
    h->small_ranges.clear();
}

// [lo, hi) of the serialization in the places that hold it: pieces of the host shadow (chain -1: everything outside the
// five big lists, [0, var[2]) and [var[7], len)), then pieces of chains in HBM, `at` bytes into the chain.  The four big
// vectors (chains 5..8) are held in both places.
struct Piece {
    int chain;
    uint64_t x, y, at;
};
std::vector<Piece> split_range(const b200_state* h, uint64_t lo, uint64_t hi) {
    std::vector<Piece> out;
    auto add = [&](int c, uint64_t a, uint64_t b) {
        const uint64_t x = std::max(a, lo), y = std::min(b, hi);
        if (x < y) out.push_back(Piece{c, x, y, x - a});
    };
    add(-1, 0, h->so.var[2]);
    add(-1, h->so.var[7], h->len);
    for (int c = 0; c < 9; c++) {
        const StateChain L = chain(h, c);
        add(c, L.lo, L.hi);
    }
    return out;
}

// grow a device buffer keeping its contents
int32_t grow_keep(Engine& e, DevBuf& b, size_t n) {
    if (n <= b.cap) return B200_SUCCESS;
    DevBuf nb;
    B200_CUDA_TRY(nb.reserve(n));
    if (b.p) {
        cudaError_t ce = cudaMemcpyAsync(nb.p, b.p, b.cap, cudaMemcpyDeviceToDevice, e.stream);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(e.stream);
        if (ce != cudaSuccess) { nb.release(); e.last_error = cudaGetErrorString(ce); return B200_ERR_CUDA; }
    }
    b.release();
    b = nb;
    return B200_SUCCESS;
}

// Make `np` (planned from the shadow as it is now) the handle's plan.  Chains whose job sequence changed are re-hashed in
// full at the next root.  When a chain's regions moved (a big list outgrew its capacity), the nine chains are copied into
// new device buffers on the device — field bytes and every arena level — except the arena of a chain whose capacity
// changed, which is re-hashed in full from its copied bytes; the small fields are re-staged.
int32_t adopt_plan(Engine& e, b200_state* h, SszPlan& np, std::vector<uint32_t>& outs) {
    bool moved = false;
    for (int c = 0; c < 9; c++) moved = moved || !np.same_chain_layout(h->plan, c);
    const size_t need_arena = np.arena_nodes() * 32, need_fields = np.field_bytes() + 256;
    if (!moved) {
        int32_t rc = grow_keep(e, h->arena, need_arena);
        if (rc) return rc;
        rc = grow_keep(e, h->fields, need_fields);
        if (rc) return rc;
    } else {
        DevBuf na, nf;
        cudaError_t ce = na.reserve(need_arena);
        if (ce == cudaSuccess) ce = nf.reserve(need_fields);
        std::vector<char> full(9, 0);
        for (int c = 0; c < 9 && ce == cudaSuccess; c++) {
            uint64_t fo = 0, fn = 0; size_t nb = 0;
            h->plan.chain_field(c, &fo, &nb);
            np.chain_field(c, &fn, &nb);
            const size_t ro = h->plan.chain_region_bytes(c), rn = np.chain_region_bytes(c);
            uint8_t* nfp = static_cast<uint8_t*>(nf.p);
            ce = cudaMemcpyAsync(nfp + fn, static_cast<uint8_t*>(h->fields.p) + fo, std::min(ro, rn), cudaMemcpyDeviceToDevice, e.stream);
            if (ce == cudaSuccess && rn > ro) ce = cudaMemsetAsync(nfp + fn + ro, 0, rn - ro, e.stream);
            const auto& ao = h->plan.chain_arena(c);
            const auto& an = np.chain_arena(c);
            bool same_shape = ao.size() == an.size();
            for (size_t i = 0; same_shape && i < ao.size(); i++) same_shape = ao[i].second == an[i].second;
            if (!same_shape) { full[size_t(c)] = 1; continue; }
            for (size_t i = 0; ce == cudaSuccess && i < ao.size(); i++)
                ce = cudaMemcpyAsync(static_cast<uint32_t*>(na.p) + an[i].first * 8, static_cast<uint32_t*>(h->arena.p) + ao[i].first * 8,
                                     ao[i].second * 32, cudaMemcpyDeviceToDevice, e.stream);
        }
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(e.stream);
        if (ce != cudaSuccess) {
            na.release(); nf.release();
            e.last_error = std::string("state relocation: ") + cudaGetErrorString(ce);
            return B200_ERR_CUDA;
        }
        h->arena.release(); h->fields.release();
        h->arena = na; h->fields = nf;
        h->records_gen++;
        for (int c = 0; c < 9; c++) if (full[size_t(c)]) h->rehash[size_t(c)] = 1;
        mark_all_small(h);
    }
    for (int c = 0; c < 9; c++)
        if (!np.same_chain_jobs(h->plan, c)) h->rehash[size_t(c)] = 1;
    h->plan = std::move(np);
    h->outputs = outs;
    return B200_SUCCESS;
}
}  // namespace

// the registry's view of a resident state (capi_bls.cu: b200_registry_load_state / b200_registry_sync_state)
int32_t b200::state_validator_records(const b200_state* h, const uint8_t** records, uint64_t* n) {
    if (!resident(h)) return B200_ERR_BAD_ARG;
    *n = chain(h, 0).len;
    *records = *n ? chain_dev(h, 0) : nullptr;
    return B200_SUCCESS;
}

extern "C" {

int32_t b200_init(int32_t device) {
    Engine& e = engine();
    Guard g(e);
    if (e.ready) return e.device == device ? B200_SUCCESS : B200_ERR_BAD_ARG;
    int n = 0;
    cudaError_t ce = cudaGetDeviceCount(&n);
    if (ce != cudaSuccess || n == 0) {
        e.last_error = std::string("no CUDA device: ") + cudaGetErrorString(ce);
        return B200_ERR_NO_DEVICE;
    }
    if (device < 0 || device >= n) { e.last_error = "device index out of range"; return B200_ERR_BAD_ARG; }
    B200_CUDA_TRY(cudaSetDevice(device));
    B200_CUDA_TRY(cudaStreamCreateWithFlags(&e.stream, cudaStreamNonBlocking));
    B200_CUDA_TRY(cudaStreamCreateWithFlags(&e.copy_stream, cudaStreamNonBlocking));
    B200_CUDA_TRY(cudaEventCreate(&e.ev0));
    B200_CUDA_TRY(cudaEventCreate(&e.ev1));
    for (auto& ev : e.ev_copy) B200_CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    e.device = device;
    e.ready = true;
    return ensure_zero_nodes(e);
}

void b200_shutdown(void) {
    Engine& e = engine();
    Guard g(e);
    if (!e.ready) return;
    cudaSetDevice(e.device);
    cudaStreamSynchronize(e.stream);
    e.arena.release(); e.fields.release(); e.planbuf.release(); e.staging.release();
    if (e.d_zero) cudaFree(e.d_zero);
    e.d_zero = nullptr;
    cudaEventDestroy(e.ev0); cudaEventDestroy(e.ev1);
    for (auto& ev : e.ev_copy) cudaEventDestroy(ev);
    cudaStreamDestroy(e.stream); cudaStreamDestroy(e.copy_stream);
    e.ready = false;
}

const char* b200_last_error(void) { return engine().last_error.c_str(); }
uint64_t b200_launch_count(void) { return engine().launches; }
float b200_last_kernel_ms(void) { return engine().last_kernel_ms; }

int32_t b200_sha256(const uint8_t* data, size_t len, uint8_t out[32]) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!out || (!data && len)) return B200_ERR_BAD_ARG;
    B200_CUDA_TRY(e.fields.reserve(len + 64));
    B200_CUDA_TRY(e.staging.reserve(64));
    if (len) B200_CUDA_TRY(cudaMemcpyAsync(e.fields.p, data, len, cudaMemcpyHostToDevice, e.stream));
    uint32_t* d_out = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(e.fields.p) + ((len + 31) & ~size_t(31)));
    k_sha256_bytes<<<1, 32, 0, e.stream>>>(static_cast<const uint8_t*>(e.fields.p), len, d_out);
    e.launches++;
    B200_CUDA_TRY(cudaGetLastError());
    B200_CUDA_TRY(cudaMemcpyAsync(e.staging.p, d_out, 32, cudaMemcpyDeviceToHost, e.stream));
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    const uint32_t* w = static_cast<const uint32_t*>(e.staging.p);
    for (int k = 0; k < 8; k++) {
        out[4 * k] = uint8_t(w[k] >> 24); out[4 * k + 1] = uint8_t(w[k] >> 16);
        out[4 * k + 2] = uint8_t(w[k] >> 8); out[4 * k + 3] = uint8_t(w[k]);
    }
    return B200_SUCCESS;
}

int32_t b200_merkleize(const uint8_t* chunks, size_t n_chunks, uint64_t limit, uint8_t out[32]) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!out || (!chunks && n_chunks)) return B200_ERR_BAD_ARG;
    if (limit == 0) limit = n_chunks ? n_chunks : 1;
    if (limit > (uint64_t(1) << 63)) return B200_ERR_BAD_ARG;
    if (n_chunks > limit) return B200_ERR_LIMIT;
    SszPlan p;
    std::vector<uint32_t> outs{p.wide_chunks(p.stage_field(chunks, 32 * n_chunks), n_chunks, depth_for(limit))};
    return run_oneshot(e, p, outs, out);
}

int32_t b200_mix_in_length(const uint8_t root[32], uint64_t length, uint8_t out[32]) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!root || !out) return B200_ERR_BAD_ARG;
    SszPlan p;
    std::vector<uint32_t> outs{p.mix_in_length(p.leaf(root), length)};
    return run_oneshot(e, p, outs, out);
}

int32_t b200_is_valid_merkle_branch(const uint8_t leaf[32], const uint8_t* branch, size_t depth, uint64_t index,
                                    const uint8_t root[32], int32_t* ok) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!leaf || !root || !ok || (!branch && depth) || depth > 64) return B200_ERR_BAD_ARG;
    SszPlan p;
    uint32_t v = p.leaf(leaf);
    for (size_t i = 0; i < depth; i++) {
        uint32_t sib = p.leaf(branch + 32 * i);
        v = ((index >> i) & 1) ? p.hash2(sib, v) : p.hash2(v, sib);
    }
    uint8_t got[32];
    std::vector<uint32_t> outs{v};
    rc = run_oneshot(e, p, outs, got);
    if (rc) return rc;
    *ok = memcmp(got, root, 32) == 0 ? 1 : 0;
    return B200_SUCCESS;
}

int32_t b200_htr_validators(const uint8_t* ssz, size_t n, uint64_t limit, uint8_t out[32]) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!out || (!ssz && n)) return B200_ERR_BAD_ARG;
    if (limit == 0) limit = n ? n : 1;
    if (limit > (uint64_t(1) << 63)) return B200_ERR_BAD_ARG;
    if (n > limit) return B200_ERR_LIMIT;
    SszPlan p;
    uint32_t r = p.wide_records(JOB_VALIDATORS, p.stage_field(ssz, 121 * n), n, depth_for(limit));
    std::vector<uint32_t> outs{p.mix_in_length(r, n)};
    return run_oneshot(e, p, outs, out);
}

int32_t b200_htr_packed(const uint8_t* data, size_t nbytes, uint64_t limit_chunks, int32_t is_list, uint64_t length,
                        uint8_t out[32]) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!out || (!data && nbytes)) return B200_ERR_BAD_ARG;
    uint64_t n = (nbytes + 31) / 32;
    if (limit_chunks == 0) limit_chunks = n ? n : 1;
    if (limit_chunks > (uint64_t(1) << 63)) return B200_ERR_BAD_ARG;
    if (n > limit_chunks) return B200_ERR_LIMIT;
    SszPlan p;
    uint32_t r = p.wide_chunks(p.stage_field(data, nbytes), n, depth_for(limit_chunks));
    if (is_list) r = p.mix_in_length(r, length);
    std::vector<uint32_t> outs{r};
    return run_oneshot(e, p, outs, out);
}

int32_t b200_htr_beacon_state_deneb(const uint8_t* ssz, size_t len, int32_t preset, uint8_t out[32]) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!ssz || !out) return B200_ERR_BAD_ARG;
    SszPlan p;
    std::vector<uint32_t> outs;
    rc = build_beacon_state_plan(p, ssz, len, preset, outs);
    if (rc) { e.last_error = "malformed deneb BeaconState SSZ"; return rc; }
    return run_oneshot(e, p, outs, out);
}

int32_t b200_state_upload_deneb(const uint8_t* ssz, size_t len, int32_t preset, b200_state** out_handle) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!ssz || !out_handle) return B200_ERR_BAD_ARG;
    std::unique_ptr<b200_state> h(new b200_state());
    if (!parse_beacon_state(ssz, len, preset, h->so)) { e.last_error = "malformed deneb BeaconState SSZ"; return B200_ERR_SSZ_MALFORMED; }
    h->len = len; h->preset = preset;
    for (int f = 0; f < 5; f++) h->cap[f] = chain(h.get(), f).len + headroom(chain(h.get(), f).len);
    {
        SszPlan first;  // reads the caller's buffer
        std::vector<uint32_t> outs;
        rc = build_beacon_state_plan(first, ssz, len, preset, outs, h->cap);
        if (rc) { e.last_error = "malformed deneb BeaconState SSZ"; return rc; }
        uint8_t root[32];
        rc = first.run(e, h->arena, h->fields, h->planbuf, COPY_ALL, outs, root);  // uploads + first hash
        if (rc) return rc;  // ~b200_state releases the device buffers
    }
    // keep what is needed to re-plan without the caller's buffer: the serialization minus the big lists
    h->shadow_cap = shadow_bytes_for(h.get());
    h->shadow = static_cast<uint8_t*>(calloc(h->shadow_cap, 1));
    if (!h->shadow) { e.last_error = "out of host memory for the state shadow"; return B200_ERR_CUDA; }
    memcpy(h->shadow, ssz, h->so.var[2]);
    memcpy(h->shadow + h->so.var[7], ssz + h->so.var[7], len - h->so.var[7]);
    // page-lock the populated ranges (a few MB) so that re-staging a patched small field is a real async DMA
    pin_shadow(h.get(), true);
    rc = build_beacon_state_plan(h->plan, h->shadow, len, preset, h->outputs, h->cap);  // same layout: lengths and caps
    if (rc) return rc;
    *out_handle = h.release();
    return B200_SUCCESS;
}

// pending small-field updates or reshapes: re-plan from the shadow (the chains stay where they are; fresh small leaves,
// lengths and finisher ops)
static int32_t replan_if_small_dirty(Engine& e, b200_state* h) {
    if (!h->small_dirty) return B200_SUCCESS;
    SszPlan np;
    std::vector<uint32_t> outs;
    int32_t rc = build_beacon_state_plan(np, h->shadow, h->len, h->preset, outs, h->cap);
    if (rc) return rc;
    return adopt_plan(e, h, np, outs);
}

int32_t b200_state_root(b200_state* h, uint8_t out[32]) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!h || !out) return B200_ERR_BAD_ARG;
    if (h->sharded)   // every rank of the communicator calls this together: stages | ncclAllGather | finisher
        return h->plan.run(e, h->arena, h->fields, h->planbuf, COPY_NONE, h->outputs, out);
    rc = replan_if_small_dirty(e, h);  // updates made through b200_state_update_* are honoured here too
    if (rc) return rc;
    rc = h->plan.run(e, h->arena, h->fields, h->planbuf, h->small_dirty ? COPY_SMALL_ONLY : COPY_NONE, h->outputs, out,
                     nullptr, nullptr, &h->small_ranges);
    if (rc) return rc;
    mark_clean(h);
    return B200_SUCCESS;
}

void b200_state_free(b200_state* h) {
    if (!h) return;
    Engine& e = engine();
    Guard g(e);
    if (e.ready) { cudaSetDevice(e.device); cudaStreamSynchronize(e.stream); }
    delete h;
}

int32_t b200_state_update_elements(b200_state* h, int32_t field, const uint64_t* indices, const uint8_t* values, size_t n) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || field < 0 || field > 4 || (n && (!indices || !values)) || n > 0xffffffffull) return B200_ERR_BAD_ARG;
    if (!n) return B200_SUCCESS;
    const StateChain L = chain(h, field);
    for (size_t i = 0; i < n; i++)
        if (indices[i] >= L.len) { e.last_error = "state_update_elements: index beyond the list length"; return B200_ERR_BAD_ARG; }
    const uint32_t elem = L.elem;
    // [indices | values] through pinned staging, then a scatter kernel into the resident list
    const size_t off_vals = n * 8;
    const size_t total = off_vals + n * elem;
    B200_CUDA_TRY(e.staging.reserve(total));
    B200_CUDA_TRY(h->scatter.reserve(total));
    memcpy(e.staging.p, indices, n * 8);
    memcpy(static_cast<uint8_t*>(e.staging.p) + off_vals, values, n * elem);
    B200_CUDA_TRY(cudaMemcpyAsync(h->scatter.p, e.staging.p, total, cudaMemcpyHostToDevice, e.stream));
    launch_scatter(chain_dev(h, field), static_cast<const uint64_t*>(h->scatter.p),
                   static_cast<const uint8_t*>(h->scatter.p) + off_vals, uint32_t(n), elem, e.stream);
    e.launches++;
    B200_CUDA_TRY(cudaGetLastError());
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    for (size_t i = 0; i < n; i++) h->dirty[field].push_back(L.input_of(indices[i]));
    if (field == 0) h->records_gen++;
    return B200_SUCCESS;
}

static int32_t update_bytes(Engine& e, b200_state* h, uint64_t ssz_offset, const uint8_t* data, size_t n);

int32_t b200_state_update_bytes(b200_state* h, uint64_t ssz_offset, const uint8_t* data, size_t n) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    return update_bytes(e, h, ssz_offset, data, n);
}

// b200_state_update_bytes with the engine lock held (the sync-committee rotation writes through it too)
static int32_t update_bytes(Engine& e, b200_state* h, uint64_t ssz_offset, const uint8_t* data, size_t n) {
    if (!resident(h) || (n && !data) || ssz_offset > h->len || n > h->len - ssz_offset) return B200_ERR_BAD_ARG;
    if (!n) return B200_SUCCESS;
    const uint64_t lo = ssz_offset;
    const std::vector<Piece> pieces = split_range(h, lo, lo + n);
    // (1) the shadow's pieces: patch them; the variable-size offsets must not change
    std::vector<uint8_t> saved;
    for (const Piece& p : pieces) {
        if (p.chain >= 0) continue;
        saved.insert(saved.end(), h->shadow + p.x, h->shadow + p.y);
        memcpy(h->shadow + p.x, data + (p.x - lo), p.y - p.x);
        h->small_ranges.emplace_back(h->shadow + p.x, h->shadow + p.y);
    }
    if (!saved.empty()) {
        StateOffsets so2;
        bool ok = parse_beacon_state(h->shadow, h->len, h->preset, so2);
        for (int i = 0; ok && i < 10; i++) ok = so2.var[i] == h->so.var[i];
        if (!ok) {  // would move or resize a variable-size field: not an in-place update
            size_t pos = 0;
            for (const Piece& p : pieces) {
                if (p.chain >= 0) continue;
                memcpy(h->shadow + p.x, saved.data() + pos, p.y - p.x);
                pos += p.y - p.x;
            }
            // (the ranges stay recorded: re-copying unchanged bytes is harmless)
            e.last_error = "state_update_bytes: the update changes a variable-size field's offset or length; use state_append_elements / state_set_field";
            return B200_ERR_BAD_ARG;
        }
        h->small_dirty = true;
    }
    // (2) the pieces inside big lists and inside the four big vectors: copy into the resident chain, mark the covered
    //     inputs dirty
    for (const Piece& p : pieces) {
        if (p.chain < 0) continue;
        B200_CUDA_TRY(e.staging.reserve(p.y - p.x));
        memcpy(e.staging.p, data + (p.x - lo), p.y - p.x);
        B200_CUDA_TRY(cudaMemcpyAsync(chain_dev(h, p.chain) + p.at, e.staging.p, p.y - p.x, cudaMemcpyHostToDevice, e.stream));
        B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
        const uint32_t unit = chain(h, p.chain).unit;
        for (uint64_t u = p.at / unit; u <= (p.at + (p.y - p.x) - 1) / unit; u++) h->dirty[p.chain].push_back(uint32_t(u));
        if (p.chain == 0) h->records_gen++;
    }
    return B200_SUCCESS;
}

// Field ids of the reshaping calls beyond the five big lists (include/b200_consensus.h)
static constexpr int32_t kFieldVotes = B200_FIELD_ETH1_DATA_VOTES, kFieldHeader = B200_FIELD_LATEST_EXECUTION_PAYLOAD_HEADER;

// append to a big list: shadow offsets, then (past the capacity) relocation on the device, then the appended bytes H2D
static int32_t append_big(Engine& e, b200_state* h, int f, const uint8_t* values, size_t n) {
    const StateChain L = chain(h, f);
    const uint64_t old_n = L.len, new_n = old_n + n, limit = preset_of(h->preset).validator_registry_limit;
    if (n > limit || new_n > limit) { e.last_error = "state_append_elements: beyond the list limit"; return B200_ERR_LIMIT; }
    const uint32_t elem = L.elem;
    if (uint64_t(n) * elem > 0xffffffffull) { e.last_error = "state_append_elements: the serialization would exceed 4 GiB"; return B200_ERR_LIMIT; }
    const size_t old_bytes = size_t(old_n) * elem, new_bytes = size_t(new_n) * elem;
    int32_t rc = reshape_shadow(e, h, L.var, new_bytes);
    if (rc) return rc;
    auto undo = [&]() { reshape_shadow(e, h, L.var, old_bytes); reparse(h); };
    if (!reparse(h)) { undo(); return B200_ERR_SSZ_MALFORMED; }
    if (new_n > h->cap[f]) {   // relocate the list (and re-place the chains after it) with fresh headroom
        const uint64_t old_cap = h->cap[f];
        h->cap[f] = new_n + headroom(new_n);
        SszPlan np;
        std::vector<uint32_t> outs;
        rc = build_beacon_state_plan(np, h->shadow, h->len, h->preset, outs, h->cap);
        if (!rc) rc = adopt_plan(e, h, np, outs);
        if (rc) { h->cap[f] = old_cap; undo(); return rc; }
    }
    B200_CUDA_TRY(e.staging.reserve(n * elem));
    memcpy(e.staging.p, values, n * elem);
    B200_CUDA_TRY(cudaMemcpyAsync(chain_dev(h, f) + old_bytes, e.staging.p, n * elem, cudaMemcpyHostToDevice, e.stream));
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    if (f == 0) h->records_gen++;
    // appended inputs are dirty; the old ragged last chunk is among them when the first appended element shares it
    for (uint64_t u = L.input_of(old_n); u <= L.input_of(new_n - 1); u++) h->dirty[f].push_back(uint32_t(u));
    // new length mix-in and finisher ops; the finisher nodes of the lists' tops are allocated ahead of the small fields'
    // arena levels, so those move with them and are re-hashed
    mark_all_small(h);
    return B200_SUCCESS;
}

// replace small variable-size field k (StateOffsets::var index) of the shadow with `len` bytes
static int32_t set_small(Engine& e, b200_state* h, int k, const uint8_t* data, size_t len) {
    const std::vector<uint8_t> saved(h->shadow + h->so.var[k], h->shadow + h->so.var[k + 1]);
    int32_t rc = reshape_shadow(e, h, k, len);
    if (rc) return rc;
    if (len) memcpy(h->shadow + h->so.var[k], data, len);
    if (!reparse(h)) {
        reshape_shadow(e, h, k, saved.size());
        if (!saved.empty()) memcpy(h->shadow + h->so.var[k], saved.data(), saved.size());
        reparse(h);
        e.last_error = "state_set_field: malformed encoding";
        return B200_ERR_SSZ_MALFORMED;
    }
    mark_all_small(h);
    return B200_SUCCESS;
}

int32_t b200_state_append_elements(b200_state* h, int32_t field, const uint8_t* values, size_t n) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || (n && !values)) return B200_ERR_BAD_ARG;
    if (field >= 0 && field <= 4) return n ? append_big(e, h, field, values, n) : B200_SUCCESS;
    const SmallList l = appendable_small_list(field, preset_of(h->preset));
    if (l.var < 0) { e.last_error = "state_append_elements: unknown field"; return B200_ERR_BAD_ARG; }
    if (!n) return B200_SUCCESS;
    const size_t old_bytes = h->so.var[l.var + 1] - h->so.var[l.var];
    if (n > l.limit || old_bytes / l.elem + n > l.limit) { e.last_error = "state_append_elements: beyond the list limit"; return B200_ERR_LIMIT; }
    std::vector<uint8_t> buf(old_bytes + n * l.elem);
    memcpy(buf.data(), h->shadow + h->so.var[l.var], old_bytes);
    memcpy(buf.data() + old_bytes, values, n * l.elem);
    return set_small(e, h, l.var, buf.data(), buf.size());
}

int32_t b200_state_set_field(b200_state* h, int32_t field, const uint8_t* ssz, size_t len) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || (len && !ssz)) return B200_ERR_BAD_ARG;
    if (field == kFieldVotes) {
        const SmallList votes = appendable_small_list(field, preset_of(h->preset));
        if (len % votes.elem) { e.last_error = "state_set_field: eth1_data_votes not a multiple of 72 bytes"; return B200_ERR_SSZ_MALFORMED; }
        if (len / votes.elem > votes.limit) { e.last_error = "state_set_field: beyond ETH1_DATA_VOTES_BOUND"; return B200_ERR_LIMIT; }
        return set_small(e, h, votes.var, ssz, len);
    }
    if (field == kFieldHeader) {
        // 584 fixed bytes whose only offset (extra_data, at byte 436) is 584, then 0..32 bytes of extra_data
        if (len < 584 || len > 584 + 32 || le32(ssz + 436) != 584) {
            e.last_error = "state_set_field: malformed ExecutionPayloadHeader";
            return B200_ERR_SSZ_MALFORMED;
        }
        return set_small(e, h, 7, ssz, len);
    }
    e.last_error = "state_set_field: unknown field";
    return B200_ERR_BAD_ARG;
}

int32_t b200_state_root_incremental(b200_state* h, uint8_t out[32]) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!h || !out) return B200_ERR_BAD_ARG;
    rc = replan_if_small_dirty(e, h);
    if (rc) return rc;
    std::vector<std::vector<uint32_t>> dirty(h->plan.n_chains());
    for (int f = 0; f < 9 && size_t(f) < dirty.size(); f++) {
        dirty[size_t(f)] = h->dirty[f];
        std::sort(dirty[size_t(f)].begin(), dirty[size_t(f)].end());
        dirty[size_t(f)].erase(std::unique(dirty[size_t(f)].begin(), dirty[size_t(f)].end()), dirty[size_t(f)].end());
    }
    rc = h->plan.run(e, h->arena, h->fields, h->planbuf, h->small_dirty ? COPY_SMALL_ONLY : COPY_NONE, h->outputs, out,
                     &dirty, &h->selbuf, &h->small_ranges, &h->rehash);
    if (rc) return rc;
    mark_clean(h);
    return B200_SUCCESS;
}

int32_t b200_htr_beacon_state_deneb_shard(const uint8_t* ssz, size_t len, int32_t preset, int32_t rank, int32_t world,
                                          uint8_t* out_roots) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!ssz || !out_roots) return B200_ERR_BAD_ARG;
    SszPlan p;
    std::vector<uint32_t> outs;
    rc = build_beacon_state_shard_plan(p, ssz, len, preset, rank, world, outs);
    if (rc) return rc;
    return run_oneshot(e, p, outs, out_roots);
}

int32_t b200_htr_beacon_state_deneb_combine(const uint8_t* ssz, size_t len, int32_t preset, int32_t world,
                                            const uint8_t* all_roots, uint8_t out[32]) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!ssz || !all_roots || !out) return B200_ERR_BAD_ARG;
    SszPlan p;
    std::vector<uint32_t> outs;
    rc = build_beacon_state_combine_plan(p, ssz, len, preset, world, all_roots, outs);
    if (rc) return rc;
    return run_oneshot(e, p, outs, out);
}

// get_active_validator_indices + compute_shuffled_indices on a device-resident state: the registry never leaves HBM;
// only the shuffled index list (8 B per active validator) comes back.
int32_t b200_state_shuffled_active_indices(b200_state* h, uint64_t epoch, const uint8_t seed[32], uint32_t rounds, uint64_t* out,
                                           size_t* out_n) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || !seed || !out_n) return B200_ERR_BAD_ARG;
    *out_n = 0;
    const uint64_t n = chain(h, 0).len;
    if (n == 0) return B200_SUCCESS;
    if (!out) return B200_ERR_BAD_ARG;
    uint64_t *d_act, *d_out;
    rc = shuffle_scratch(e, n, &d_act, &d_out);
    if (rc) return rc;
    B200_CUDA_TRY(cudaEventRecord(e.ev0, e.stream));
    uint64_t cnt = 0;
    rc = active_indices_on_device(e, chain_dev(h, 0), n, epoch, d_act, &cnt);
    if (rc) return rc;
    rc = shuffle_on_device(e, d_act, cnt, seed, rounds, d_out);
    if (rc) return rc;
    B200_CUDA_TRY(cudaEventRecord(e.ev1, e.stream));
    if (cnt) B200_CUDA_TRY(cudaMemcpyAsync(out, d_out, cnt * 8, cudaMemcpyDeviceToHost, e.stream));
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    B200_CUDA_TRY(cudaEventElapsedTime(&e.last_kernel_ms, e.ev0, e.ev1));
    *out_n = size_t(cnt);
    return B200_SUCCESS;
}

// ---- duties on a resident state: proposer lookahead and sync committees (deneb/spec/mod.rs) ----
namespace {
constexpr uint8_t kDomainBeaconProposer[4] = {0, 0, 0, 0}, kDomainSyncCommittee[4] = {7, 0, 0, 0};   // domains.rs:19-30
constexpr size_t kSlotOffset = 40;   // genesis_time (8), genesis_validators_root (32), then slot

uint64_t shadow_slot(const b200_state* h) { return le64(h->shadow + kSlotOffset); }
void sha256_host(const uint8_t* data, size_t len, uint8_t out[32]) {
    Sha256Ctx c;
    sha_init(c);
    sha_update(c, data, len);
    sha_final(c, out);
}
// get_seed (deneb/spec/mod.rs:2713-2748): SHA-256(domain || le64(epoch) || randao_mixes[(epoch + EPHV - 2) mod EPHV]),
// the mix index in wrapping u64 (EPHV divides 2^64, so the wrap does not change it); the mixes are read from the shadow
void state_seed(const b200_state* h, uint64_t epoch, const uint8_t domain[4], uint8_t out[32]) {
    const Preset& P = preset_of(h->preset);
    const uint64_t mix = (epoch + P.epochs_per_historical_vector - 2) % P.epochs_per_historical_vector;
    uint8_t in[44];
    memcpy(in, domain, 4);
    for (int k = 0; k < 8; k++) in[4 + k] = uint8_t(epoch >> (8 * k));
    memcpy(in + 12, h->shadow + h->so.randao_mixes + 32 * mix, 32);
    sha256_host(in, sizeof(in), out);
}

// get_active_validator_indices(state, epoch) into the shuffle scratch: *d_act (device) holds *n_active indices, *d_out
// (device) has room for max(N, min_out) more; *recs: the Validator records in HBM.  No active validator (the reference's
// CollectionCannotBeEmpty, or its `i % 0` panic for the sync committee) -> B200_ERR_BAD_ARG.
int32_t duty_active(Engine& e, b200_state* h, uint64_t epoch, uint64_t min_out, const uint8_t** recs, uint64_t** d_act,
                    uint64_t** d_out, uint64_t* n_active) {
    const uint64_t n = chain(h, 0).len;
    if (n == 0) { e.last_error = "duties: no active validator"; return B200_ERR_BAD_ARG; }
    *recs = chain_dev(h, 0);
    int32_t rc = shuffle_scratch(e, std::max(n, min_out), d_act, d_out);
    if (rc) return rc;
    rc = active_indices_on_device(e, *recs, n, epoch, *d_act, n_active);
    if (rc) return rc;
    if (*n_active == 0) { e.last_error = "duties: no active validator"; return B200_ERR_BAD_ARG; }
    return B200_SUCCESS;
}

// get_next_sync_committee (deneb/spec/mod.rs:1973-2060) with the engine lock held: indices (host, SIZE) and the SyncCommittee
// bytes (host, SIZE x 48 keys then the 48-byte aggregate; zero on a non-zero *code)
int32_t next_sync_committee(Engine& e, b200_state* h, uint64_t* out_indices, uint8_t* out_committee, int32_t* out_code) {
    const Preset& P = preset_of(h->preset);
    const uint64_t epoch = shadow_slot(h) / P.slots_per_epoch + 1;
    uint8_t seed[32];
    state_seed(h, epoch, kDomainSyncCommittee, seed);
    const uint8_t* recs;
    uint64_t *d_act, *d_idx, cnt = 0;
    B200_CUDA_TRY(cudaEventRecord(e.ev0, e.stream));
    int32_t rc = duty_active(e, h, epoch, P.sync_committee_size, &recs, &d_act, &d_idx, &cnt);
    if (rc) return rc;
    rc = sample_committee_on_device(e, seed, P.sync_committee_size, P.shuffle_round_count, d_act, cnt, recs, d_idx);
    if (rc) return rc;
    const size_t size = P.sync_committee_size;
    rc = aggregate_record_keys(recs, d_idx, uint32_t(size), out_committee, out_committee + size * 48, out_code);
    if (rc) return rc;
    B200_CUDA_TRY(cudaEventRecord(e.ev1, e.stream));
    B200_CUDA_TRY(cudaMemcpyAsync(out_indices, d_idx, size * 8, cudaMemcpyDeviceToHost, e.stream));
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    B200_CUDA_TRY(cudaEventElapsedTime(&e.last_kernel_ms, e.ev0, e.ev1));
    if (*out_code) memset(out_committee, 0, size * 48 + 48);
    return B200_SUCCESS;
}
// process_sync_committee_updates with the engine lock held (b200_state_sync_committee_updates, b200_state_process_epoch)
int32_t sync_committee_updates(Engine& e, b200_state* h, int32_t* rotated, int32_t* out_code) {
    const Preset& P = preset_of(h->preset);
    const uint64_t next_epoch = shadow_slot(h) / P.slots_per_epoch + 1;
    if (next_epoch % P.epochs_per_sync_committee_period != 0) {
        *rotated = 0; *out_code = B200_SUCCESS;
        return B200_SUCCESS;
    }
    // current_sync_committee <- next_sync_committee <- get_next_sync_committee: the two fields are adjacent, one patch
    const size_t committee = (size_t(P.sync_committee_size) + 1) * 48;
    std::vector<uint8_t> both(2 * committee);
    std::vector<uint64_t> idx(P.sync_committee_size);
    memcpy(both.data(), h->shadow + h->so.next_sync_committee, committee);
    int32_t code = B200_SUCCESS;
    int32_t rc = next_sync_committee(e, h, idx.data(), both.data() + committee, &code);
    if (rc) return rc;
    *out_code = code;
    *rotated = 0;
    if (code) return B200_SUCCESS;   // the reference's `?` before mem::replace: the state stays as it was
    rc = update_bytes(e, h, h->so.current_sync_committee, both.data(), both.size());
    if (rc) return rc;
    *rotated = 1;
    return B200_SUCCESS;
}
}  // namespace

int32_t b200_state_get_seed(b200_state* h, uint64_t epoch, const uint8_t domain_type[4], uint8_t out[32]) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || !domain_type || !out) return B200_ERR_BAD_ARG;
    state_seed(h, epoch, domain_type, out);
    return B200_SUCCESS;
}

int32_t b200_state_proposer_indices(b200_state* h, uint64_t epoch, uint64_t* out) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || !out) return B200_ERR_BAD_ARG;
    const Preset& P = preset_of(h->preset);
    if (epoch > ~uint64_t(0) / P.slots_per_epoch) { e.last_error = "proposer_indices: epoch * SLOTS_PER_EPOCH overflows u64"; return B200_ERR_BAD_ARG; }
    // get_beacon_proposer_index (deneb/spec/mod.rs:2822-2856) for every slot of the epoch: seed SHA-256(get_seed(epoch,
    // BeaconProposer) || le64(slot)), the active set and the balances being those of the epoch
    uint8_t epoch_seed[32], in[40];
    state_seed(h, epoch, kDomainBeaconProposer, epoch_seed);
    memcpy(in, epoch_seed, 32);
    std::vector<uint8_t> slot_seeds(P.slots_per_epoch * 32);
    for (uint64_t j = 0; j < P.slots_per_epoch; j++) {
        const uint64_t slot = epoch * P.slots_per_epoch + j;
        for (int k = 0; k < 8; k++) in[32 + k] = uint8_t(slot >> (8 * k));
        sha256_host(in, sizeof(in), slot_seeds.data() + 32 * j);
    }
    const uint8_t* recs;
    uint64_t *d_act, *d_out, cnt = 0;
    B200_CUDA_TRY(cudaEventRecord(e.ev0, e.stream));
    rc = duty_active(e, h, epoch, 0, &recs, &d_act, &d_out, &cnt);
    if (rc) return rc;
    std::vector<uint64_t> res(P.slots_per_epoch);
    rc = sample_proposers_on_device(e, slot_seeds.data(), uint32_t(P.slots_per_epoch), P.shuffle_round_count, d_act, cnt, recs, res.data());
    if (rc) return rc;
    B200_CUDA_TRY(cudaEventRecord(e.ev1, e.stream));
    B200_CUDA_TRY(cudaEventSynchronize(e.ev1));
    B200_CUDA_TRY(cudaEventElapsedTime(&e.last_kernel_ms, e.ev0, e.ev1));
    memcpy(out, res.data(), res.size() * 8);
    return B200_SUCCESS;
}

int32_t b200_state_next_sync_committee(b200_state* h, uint64_t* out_indices, uint8_t* out_committee, int32_t* out_code) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || !out_indices || !out_committee || !out_code) return B200_ERR_BAD_ARG;
    return next_sync_committee(e, h, out_indices, out_committee, out_code);
}

int32_t b200_state_sync_committee_updates(b200_state* h, int32_t* rotated, int32_t* out_code) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || !rotated || !out_code) return B200_ERR_BAD_ARG;
    return sync_committee_updates(e, h, rotated, out_code);
}

int32_t b200_state_sync_committee_indices(b200_state* h, int32_t which, uint64_t* out) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || !out || (which != 0 && which != 1)) return B200_ERR_BAD_ARG;
    const Preset& P = preset_of(h->preset);
    const uint8_t* keys = h->shadow + (which ? h->so.next_sync_committee : h->so.current_sync_committee);
    const uint64_t n = chain(h, 0).len;
    const uint8_t* recs = n ? chain_dev(h, 0) : nullptr;
    B200_CUDA_TRY(cudaEventRecord(e.ev0, e.stream));
    std::vector<uint64_t> res(P.sync_committee_size);
    rc = match_committee_keys_on_device(e, recs, n, keys, P.sync_committee_size, res.data());
    if (rc) return rc;
    B200_CUDA_TRY(cudaEventRecord(e.ev1, e.stream));
    B200_CUDA_TRY(cudaEventSynchronize(e.ev1));
    B200_CUDA_TRY(cudaEventElapsedTime(&e.last_kernel_ms, e.ev0, e.ev1));
    memcpy(out, res.data(), res.size() * 8);
    return B200_SUCCESS;
}

// ---- beacon committees on a resident state (phase0/helpers.rs:741-806, 896-974; deneb/block_processing.rs:53-100) ----
namespace {
constexpr uint8_t kDomainBeaconAttester[4] = {1, 0, 0, 0};   // domains.rs:19-30
constexpr size_t kMaxAttestations = size_t(1) << 20;         // b200_state_attesting_indices' bound per call
using CommitteeEpoch = b200_state::CommitteeEpoch;

// get_committee_count_per_slot (:741-773) for n active validators
uint64_t committees_per_slot(const Preset& P, uint64_t n) {
    return std::max<uint64_t>(1, std::min<uint64_t>(P.max_committees_per_slot, n / P.slots_per_epoch / P.target_committee_size));
}

// The cached committee source of `epoch`: get_active_validator_indices(epoch) shuffled by get_seed(epoch, BeaconAttester)
// on the device.  A hit needs the same seed (recomputed from the shadow) and the same records generation; a miss rebuilds
// the least recently used entry.  Every launch is on the engine stream, so later kernels of the call see the list.
int32_t committee_epoch(Engine& e, b200_state* h, uint64_t epoch, CommitteeEpoch** out) {
    const Preset& P = preset_of(h->preset);
    uint8_t seed[32];
    state_seed(h, epoch, kDomainBeaconAttester, seed);
    CommitteeEpoch* lru = &h->committees[0];
    for (CommitteeEpoch& c : h->committees) {
        if (c.used && c.epoch == epoch && c.gen == h->records_gen && !memcmp(c.seed, seed, 32)) {
            c.last_use = ++h->committee_tick;
            *out = &c;
            return B200_SUCCESS;
        }
        if (!c.used || (lru->used && c.last_use < lru->last_use)) lru = &c;
    }
    CommitteeEpoch& c = *lru;
    c.used = false;
    c.pos_ready = false;
    const uint64_t n = chain(h, 0).len;
    uint64_t cnt = 0;
    if (n) {
        uint64_t *d_act, *d_out;
        int32_t rc = shuffle_scratch(e, n, &d_act, &d_out);
        if (rc) return rc;
        rc = active_indices_on_device(e, chain_dev(h, 0), n, epoch, d_act, &cnt);
        if (rc) return rc;
        B200_CUDA_TRY(c.shuffled.reserve(cnt * 8 + 64));
        rc = shuffle_on_device(e, d_act, cnt, seed, uint32_t(P.shuffle_round_count), static_cast<uint64_t*>(c.shuffled.p));
        if (rc) return rc;
    }
    c.epoch = epoch;
    c.gen = h->records_gen;
    memcpy(c.seed, seed, 32);
    c.n_active = cnt;
    c.cps = committees_per_slot(P, cnt);
    c.last_use = ++h->committee_tick;
    c.used = true;
    *out = &c;
    return B200_SUCCESS;
}

// the entry's inverse position map (built on first use)
int32_t committee_positions(Engine& e, b200_state* h, CommitteeEpoch& c) {
    if (c.pos_ready) return B200_SUCCESS;
    const uint64_t n = chain(h, 0).len;
    B200_CUDA_TRY(c.pos.reserve(n * 4 + 64));
    int32_t rc = committee_positions_on_device(e, static_cast<const uint64_t*>(c.shuffled.p), c.n_active, n, static_cast<uint32_t*>(c.pos.p));
    if (rc) return rc;
    c.pos_ready = true;
    return B200_SUCCESS;
}

int32_t begin_timed(Engine& e) {
    B200_CUDA_TRY(cudaEventRecord(e.ev0, e.stream));
    return B200_SUCCESS;
}
int32_t end_timed(Engine& e) {
    B200_CUDA_TRY(cudaEventRecord(e.ev1, e.stream));
    B200_CUDA_TRY(cudaEventSynchronize(e.ev1));
    B200_CUDA_TRY(cudaEventElapsedTime(&e.last_kernel_ms, e.ev0, e.ev1));
    return B200_SUCCESS;
}

// attesting_indices' work buffer: jobs | Bitlist bytes | output indices
size_t o_bits_of(size_t n_jobs) { return (n_jobs * sizeof(AttestingJob) + 255) & ~size_t(255); }
size_t o_out_of(size_t n_jobs, size_t n_bits_bytes) { return (o_bits_of(n_jobs) + n_bits_bytes + 255) & ~size_t(255); }

// Bitlist[MAX_VALIDATORS_PER_COMMITTEE] length in bits of `len` SSZ bytes; false when malformed (no delimiter bit: empty
// or a zero last byte, or more than `max_bits` bits)
bool bitlist_len(const uint8_t* b, size_t len, uint64_t max_bits, uint64_t* bits) {
    if (len == 0 || b[len - 1] == 0 || len > max_bits / 8 + 1) return false;
    *bits = 8 * uint64_t(len - 1) + uint64_t(31 - __builtin_clz(uint32_t(b[len - 1])));
    return *bits <= max_bits;
}
}  // namespace

int32_t b200_state_committee_count_per_slot(b200_state* h, uint64_t epoch, uint64_t* out) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || !out) return B200_ERR_BAD_ARG;
    CommitteeEpoch* c;
    if ((rc = begin_timed(e)) || (rc = committee_epoch(e, h, epoch, &c)) || (rc = end_timed(e))) return rc;
    *out = c->cps;
    return B200_SUCCESS;
}

int32_t b200_state_beacon_committees(b200_state* h, uint64_t epoch, uint64_t* out_indices, uint32_t* out_offsets, uint64_t* out_cps,
                                     size_t* out_n) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || !out_indices || !out_offsets || !out_cps || !out_n) return B200_ERR_BAD_ARG;
    const Preset& P = preset_of(h->preset);
    CommitteeEpoch* c;
    if ((rc = begin_timed(e)) || (rc = committee_epoch(e, h, epoch, &c))) return rc;
    if (c->n_active == 0) { e.last_error = "beacon_committees: no active validator"; return B200_ERR_BAD_ARG; }
    if ((rc = end_timed(e))) return rc;   // the device time of the kernels; the list then goes to the host
    B200_CUDA_TRY(cudaMemcpyAsync(out_indices, c->shuffled.p, c->n_active * 8, cudaMemcpyDeviceToHost, e.stream));
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    const uint64_t count = P.slots_per_epoch * c->cps, n = c->n_active;
    for (uint64_t k = 0; k <= count; k++) out_offsets[k] = uint32_t(n * k / count);
    *out_cps = c->cps;
    *out_n = size_t(n);
    return B200_SUCCESS;
}

int32_t b200_state_attester_duties(b200_state* h, uint64_t epoch, const uint64_t* validators, size_t n, uint64_t* out) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || (n && !out) || n > 0xffffffffull) return B200_ERR_BAD_ARG;
    const Preset& P = preset_of(h->preset);
    const uint64_t N = chain(h, 0).len;
    if (!validators && n != N) { e.last_error = "attester_duties: validators == NULL asks for all N validators"; return B200_ERR_BAD_ARG; }
    for (size_t i = 0; validators && i < n; i++)
        if (validators[i] >= N) { e.last_error = "attester_duties: validator index beyond the registry"; return B200_ERR_BAD_ARG; }
    if (epoch > shadow_slot(h) / P.slots_per_epoch + 1) { e.last_error = "attester_duties: epoch after the next epoch"; return B200_ERR_BAD_ARG; }
    if (epoch > ~uint64_t(0) / P.slots_per_epoch) { e.last_error = "attester_duties: epoch * SLOTS_PER_EPOCH overflows u64"; return B200_ERR_BAD_ARG; }
    if (!n) return B200_SUCCESS;
    CommitteeEpoch* c;
    if ((rc = begin_timed(e)) || (rc = committee_epoch(e, h, epoch, &c)) || (rc = committee_positions(e, h, *c))) return rc;
    // work: requested indices | rows
    const size_t o_rows = validators ? ((n * 8 + 255) & ~size_t(255)) : 0;
    B200_CUDA_TRY(h->committee_work.reserve(o_rows + n * 40));
    uint8_t* w = static_cast<uint8_t*>(h->committee_work.p);
    if (validators) {
        B200_CUDA_TRY(e.staging.reserve(n * 8));
        memcpy(e.staging.p, validators, n * 8);
        B200_CUDA_TRY(cudaMemcpyAsync(w, e.staging.p, n * 8, cudaMemcpyHostToDevice, e.stream));
    }
    rc = attester_duties_on_device(e, static_cast<const uint32_t*>(c->pos.p), validators ? reinterpret_cast<const uint64_t*>(w) : nullptr,
                                   n, c->n_active, c->cps, P.slots_per_epoch, epoch, reinterpret_cast<uint64_t*>(w + o_rows));
    if (rc) return rc;
    if ((rc = end_timed(e))) return rc;
    B200_CUDA_TRY(cudaMemcpyAsync(out, w + o_rows, n * 40, cudaMemcpyDeviceToHost, e.stream));
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    return B200_SUCCESS;
}

int32_t b200_state_attesting_indices(b200_state* h, size_t n_att, const uint8_t* data, const uint8_t* bits, const uint32_t* bits_offsets,
                                     uint64_t* out_indices, uint32_t* out_offsets, int32_t* out_codes) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || n_att > kMaxAttestations) return B200_ERR_BAD_ARG;
    if (!n_att) {
        if (out_offsets) out_offsets[0] = 0;
        e.last_kernel_ms = 0.f;
        return B200_SUCCESS;
    }
    if (!data || !bits_offsets || !out_indices || !out_offsets || !out_codes) return B200_ERR_BAD_ARG;
    if (bits_offsets[0] != 0) { e.last_error = "attesting_indices: bits_offsets[0] must be 0"; return B200_ERR_BAD_ARG; }
    for (size_t a = 0; a < n_att; a++)
        if (bits_offsets[a + 1] < bits_offsets[a]) { e.last_error = "attesting_indices: bits_offsets decrease"; return B200_ERR_BAD_ARG; }
    const size_t n_bits_bytes = bits_offsets[n_att];
    if (n_bits_bytes && !bits) return B200_ERR_BAD_ARG;

    // ---- the host step: process_attestation's checks from the shadow and the cached committees ----
    const Preset& P = preset_of(h->preset);
    const uint64_t state_slot = shadow_slot(h), cur = state_slot / P.slots_per_epoch, prev = cur ? cur - 1 : 0;
    if ((rc = begin_timed(e))) return rc;
    CommitteeEpoch* ce[2] = {nullptr, nullptr};   // previous, current (built when first asked)
    std::vector<AttestingJob> jobs;
    uint32_t total = 0;
    out_offsets[0] = 0;
    for (size_t a = 0; a < n_att; a++) {
        const uint8_t* d = data + 128 * a;
        const uint8_t* b = bits + bits_offsets[a];
        const size_t nb = bits_offsets[a + 1] - bits_offsets[a];
        const uint64_t slot = le64(d), index = le64(d + 8), target = le64(d + 88);
        uint64_t len = 0;
        int32_t code = B200_SUCCESS;
        CommitteeEpoch* c = nullptr;
        if (!bitlist_len(b, nb, P.max_validators_per_committee, &len)) code = B200_ATTESTATION_MALFORMED_BITS;
        else if (target != prev && target != cur) code = B200_ATTESTATION_INVALID_TARGET_EPOCH;
        else if (slot / P.slots_per_epoch != target) code = B200_ATTESTATION_INVALID_SLOT;
        else if (slot + P.min_attestation_inclusion_delay > state_slot) code = B200_ATTESTATION_NO_DELAY;   // wraps, as a release build
        else {
            CommitteeEpoch*& slot_entry = ce[target == cur ? 1 : 0];
            if (!slot_entry && (rc = committee_epoch(e, h, target, &slot_entry))) return rc;
            c = slot_entry;
            if (index >= c->cps) code = B200_ATTESTATION_INVALID_INDEX;
        }
        uint32_t set = 0;
        if (!code) {
            const uint64_t count = P.slots_per_epoch * c->cps, k = (slot % P.slots_per_epoch) * c->cps + index;
            const uint64_t start = c->n_active * k / count, end = c->n_active * (k + 1) / count;
            if (len != end - start) code = B200_ATTESTATION_BITFIELD;
            else {
                for (size_t i = 0; i < nb; i++) set += uint32_t(__builtin_popcount(b[i]));
                set -= 1;   // the delimiter
                if (!set) code = B200_ATTESTATION_INDICES_EMPTY;
                else jobs.push_back({static_cast<const uint64_t*>(c->shuffled.p) + start, uint32_t(len), bits_offsets[a], total, 0});
            }
        }
        out_codes[a] = code;
        if (!code) total += set;
        out_offsets[a + 1] = total;
    }

    // ---- the gather on the device ----
    if (!jobs.empty()) {
        const size_t o_bits = o_bits_of(jobs.size()), o_out = o_out_of(jobs.size(), n_bits_bytes);
        B200_CUDA_TRY(h->committee_work.reserve(o_out + size_t(total) * 8));
        B200_CUDA_TRY(e.staging.reserve(o_out));
        uint8_t* hs = static_cast<uint8_t*>(e.staging.p);
        memcpy(hs, jobs.data(), jobs.size() * sizeof(AttestingJob));
        memcpy(hs + o_bits, bits, n_bits_bytes);
        uint8_t* w = static_cast<uint8_t*>(h->committee_work.p);
        B200_CUDA_TRY(cudaMemcpyAsync(w, hs, o_out, cudaMemcpyHostToDevice, e.stream));
        rc = attesting_indices_on_device(e, reinterpret_cast<const AttestingJob*>(w), uint32_t(jobs.size()), w + o_bits,
                                         reinterpret_cast<uint64_t*>(w + o_out));
        if (rc) return rc;
    }
    if ((rc = end_timed(e))) return rc;
    if (!jobs.empty()) {
        B200_CUDA_TRY(cudaMemcpyAsync(out_indices, static_cast<uint8_t*>(h->committee_work.p) + o_out_of(jobs.size(), n_bits_bytes),
                                      size_t(total) * 8, cudaMemcpyDeviceToHost, e.stream));
        B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    }
    return B200_SUCCESS;
}

// ---- process_epoch on a resident state (deneb/spec/mod.rs:965-1003) ----
namespace {
// floor(sqrt(x)) exactly (u64::integer_sqrt): Newton's iteration on integers from above
uint64_t integer_sqrt(uint64_t x) {
    if (x < 2) return x;
    unsigned __int128 r = x, y = (r + 1) / 2;
    while (y < r) { r = y; y = (r + x / r) / 2; }
    return uint64_t(r);
}
// get_block_root (:2552, :2582) from the shadow's block_roots; false where the reference returns SlotOutOfRange
bool block_root(const b200_state* h, const Preset& P, uint64_t slot, uint64_t epoch, const uint8_t** root) {
    const uint64_t at = epoch * P.slots_per_epoch;
    if (at >= slot || slot > at + P.slots_per_historical_root) return false;
    *root = h->shadow + h->so.block_roots + 32 * (at % P.slots_per_historical_root);
    return true;
}
constexpr uint32_t kPerValidatorSteps = B200_EPOCH_INACTIVITY_UPDATES | B200_EPOCH_REWARDS_AND_PENALTIES |
                                        B200_EPOCH_REGISTRY_UPDATES | B200_EPOCH_SLASHINGS | B200_EPOCH_EFFECTIVE_BALANCE_UPDATES;
// get_total_balance (:2857-2868) of sum k of the totals pass: the checked sum, then at least one increment
uint64_t total_balance(const EpochTotals& T, int k, uint64_t inc) { return std::max(T.lo[k], inc); }
// The scalars of the reward deltas, shared by b200_state_process_epoch and b200_state_epoch_deltas.  `read` has bit k set
// for every sum k of T the caller's sub-steps read; one that overflows u64 refuses with B200_ERR_LIMIT before anything is
// filled.  Otherwise fills p's total_active, base_per_inc (get_base_reward_per_increment, the exact integer_sqrt),
// active_inc, part_inc, increment and inactivity_denominator.
int32_t reward_scalars(Engine& e, const EpochTotals& T, const Preset& P, uint32_t read, const char* who, EpochParams* p) {
    for (int k = 0; k < 5; k++)
        if ((read >> k & 1) && T.hi[k]) {
            e.last_error = std::string(who) + ": get_total_balance overflows u64";
            return B200_ERR_LIMIT;
        }
    const uint64_t inc = P.effective_balance_increment;
    p->total_active = total_balance(T, 0, inc);
    p->base_per_inc = inc * P.base_reward_factor / integer_sqrt(p->total_active);
    p->active_inc = p->total_active / inc;
    for (int f = 0; f < 3; f++) p->part_inc[f] = total_balance(T, 1 + f, inc) / inc;
    p->increment = inc;
    p->inactivity_denominator = P.inactivity_score_bias * P.inactivity_penalty_quotient_bellatrix;
    return B200_SUCCESS;
}
// is_in_inactivity_leak; get_finality_delay wraps
bool inactivity_leak(const Preset& P, uint64_t prev, uint64_t finalized_epoch) {
    return prev - finalized_epoch > P.min_epochs_to_inactivity_penalty;
}
}  // namespace

int32_t b200_state_process_epoch(b200_state* h, uint32_t steps, int32_t* out_code) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || !out_code || (steps & ~uint32_t(B200_EPOCH_ALL))) return B200_ERR_BAD_ARG;
    *out_code = B200_SUCCESS;
    const Preset& P = preset_of(h->preset);
    const uint64_t n = chain(h, 0).len;
    for (int f = 1; f < 5; f++)
        if (chain(h, f).len != n) { e.last_error = "process_epoch: the five big lists differ in length"; return B200_ERR_BAD_ARG; }
    uint8_t* dev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};   // validators, balances, participation x 2, scores
    for (int f = 0; f < 5 && n; f++) dev[f] = chain_dev(h, f);
    const uint64_t slot = shadow_slot(h), cur = slot / P.slots_per_epoch, prev = cur ? cur - 1 : 0, next = cur + 1;
    const uint64_t inc = P.effective_balance_increment;
    B200_CUDA_TRY(cudaEventRecord(e.ev0, e.stream));
    EpochTotals T;
    rc = epoch_totals_on_device(e, dev[0], dev[2], dev[3], n, cur, prev, P.ejection_balance, &T);
    if (rc) return rc;

    // ---- the host step: every refusal is decided here, before anything is written ----
    const bool run_jf = (steps & B200_EPOCH_JUSTIFICATION_AND_FINALIZATION) && cur > 1;
    const bool run_inactivity = (steps & B200_EPOCH_INACTIVITY_UPDATES) && cur > 0;
    const bool run_rewards = (steps & B200_EPOCH_REWARDS_AND_PENALTIES) && cur > 0;
    const bool run_sync = (steps & B200_EPOCH_SYNC_COMMITTEE_UPDATES) && next % P.epochs_per_sync_committee_period == 0;
    const bool run_summary = (steps & B200_EPOCH_HISTORICAL_SUMMARIES_UPDATE) &&
                             next % (P.slots_per_historical_root / P.slots_per_epoch) == 0;
    // get_total_balance: the sums a selected sub-step reads
    const bool total_read = run_jf || run_rewards || (steps & B200_EPOCH_SLASHINGS);
    const uint32_t read = (total_read ? 1u : 0u) | (run_jf ? 0x14u : 0u) | (run_rewards ? 0xeu : 0u);
    EpochParams p{};
    if ((rc = reward_scalars(e, T, P, read, "process_epoch", &p))) return rc;
    auto total = [&](int k) { return total_balance(T, k, inc); };
    uint8_t jf[121];   // justification_bits, previous_justified, current_justified, finalized (adjacent)
    memcpy(jf, h->shadow + h->so.justification_bits, sizeof(jf));
    if (run_jf) {   // weigh_justification_and_finalization (:1469-1520)
        const uint64_t old_pj = le64(jf + 1), old_cj = le64(jf + 41);
        uint8_t cp_pj[40], cp_cj[40];
        memcpy(cp_pj, jf + 1, 40); memcpy(cp_cj, jf + 41, 40);
        memcpy(jf + 1, cp_cj, 40);
        uint8_t bits = uint8_t(((jf[0] << 1) & 0x0e) | (jf[0] & 0xf0));
        const uint64_t active = total(0);
        const uint64_t targets[2] = {total(2), total(4)}, epochs[2] = {prev, cur};
        for (int k = 0; k < 2; k++) {
            if (targets[k] * 3 < active * 2) continue;
            const uint8_t* root;
            if (!block_root(h, P, slot, epochs[k], &root)) { e.last_error = "process_epoch: get_block_root out of range"; return B200_ERR_BAD_ARG; }
            for (int b = 0; b < 8; b++) jf[41 + b] = uint8_t(epochs[k] >> (8 * b));
            memcpy(jf + 49, root, 32);
            bits |= uint8_t(k == 0 ? 2 : 1);
        }
        jf[0] = bits;
        if ((bits & 0x0e) == 0x0e && old_pj + 3 == cur) memcpy(jf + 81, cp_pj, 40);
        if ((bits & 0x06) == 0x06 && old_pj + 2 == cur) memcpy(jf + 81, cp_pj, 40);
        if ((bits & 0x07) == 0x07 && old_cj + 2 == cur) memcpy(jf + 81, cp_cj, 40);
        if ((bits & 0x03) == 0x03 && old_cj + 1 == cur) memcpy(jf + 81, cp_cj, 40);
    }
    p.steps = steps & kPerValidatorSteps;
    if (!run_inactivity) p.steps &= ~uint32_t(B200_EPOCH_INACTIVITY_UPDATES);
    if (!run_rewards) p.steps &= ~uint32_t(B200_EPOCH_REWARDS_AND_PENALTIES);
    p.cur = cur; p.prev = prev;
    p.finalized_epoch = le64(jf + 81);
    p.leak = inactivity_leak(P, prev, p.finalized_epoch);
    // the exit queue (initiate_validator_exit, :3062-3111) in closed form, and the activation churn
    p.churn = std::max(P.min_per_epoch_churn_limit, T.n_active_cur / P.churn_limit_quotient);
    p.activation_epoch = cur + 1 + P.max_seed_lookahead;
    const uint64_t max_exit = T.max_exit_plus1 - 1;
    p.exit0 = T.max_exit_plus1 ? std::max(max_exit, p.activation_epoch) : p.activation_epoch;
    p.c0 = T.max_exit_plus1 && max_exit == p.exit0 ? T.n_at_max_exit : 0;
    if ((steps & B200_EPOCH_REGISTRY_UPDATES) && T.n_eject) {
        const uint64_t k = T.n_eject - 1;
        const unsigned __int128 last = p.c0 < p.churn ? (unsigned __int128)p.exit0 + (p.c0 + k) / p.churn
                                                      : (unsigned __int128)p.exit0 + 1 + k / p.churn;
        if (last + P.min_validator_withdrawability_delay > ~uint64_t(0)) {
            e.last_error = "process_epoch: an ejected validator's withdrawable_epoch overflows u64";
            return B200_ERR_LIMIT;
        }
    }
    p.activation_limit = (steps & B200_EPOCH_REGISTRY_UPDATES) ? uint32_t(std::min(P.max_per_epoch_activation_churn_limit, p.churn)) : 0;
    p.slash_epoch = cur + P.epochs_per_slashings_vector / 2;
    uint64_t slashings_sum = 0;   // `.sum::<Gwei>()` wraps in a release build
    for (uint64_t k = 0; k < P.epochs_per_slashings_vector; k++) slashings_sum += le64(h->shadow + h->so.slashings + 8 * k);
    p.adjusted_slashing = std::min(slashings_sum * P.proportional_slashing_multiplier_bellatrix, p.total_active);
    p.max_effective = P.max_effective_balance;
    p.ejection_balance = P.ejection_balance;
    p.hysteresis_down = inc / P.hysteresis_quotient * P.hysteresis_downward_multiplier;
    p.hysteresis_up = inc / P.hysteresis_quotient * P.hysteresis_upward_multiplier;
    p.score_bias = P.inactivity_score_bias;
    p.score_recovery = P.inactivity_score_recovery_rate;
    p.withdraw_delay = P.min_validator_withdrawability_delay;
    if (run_sync && T.n_active_next == 0) { e.last_error = "process_epoch: no active validator for the next sync committee"; return B200_ERR_BAD_ARG; }
    const uint64_t n_summaries = (h->so.var[9] - h->so.var[8]) / 64;
    if (run_summary && n_summaries + 1 > P.historical_roots_limit) {
        e.last_error = "process_epoch: historical_summaries is full";
        return B200_ERR_LIMIT;
    }

    // ---- the per-validator steps and the participation rotation on the device ----
    if (p.steps && n) {
        const uint32_t* changed = nullptr;
        uint64_t n_changed = 0;
        rc = epoch_apply_on_device(e, dev[0], reinterpret_cast<uint64_t*>(dev[1]), reinterpret_cast<uint64_t*>(dev[4]), dev[2], n,
                                   p, &changed, &n_changed);
        if (rc) return rc;
        if (n_changed) h->records_gen++;
        // changed records: re-hash their paths, or the whole list once they are more than a sixteenth of it
        if (n_changed > std::max<uint64_t>(4096, n / 16)) {
            h->rehash[0] = 1;
        } else if (n_changed) {
            std::vector<uint32_t> idx(n_changed);
            B200_CUDA_TRY(cudaMemcpyAsync(idx.data(), changed, n_changed * 4, cudaMemcpyDeviceToHost, e.stream));
            B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
            h->dirty[0].insert(h->dirty[0].end(), idx.begin(), idx.end());
        }
        if (p.steps & (B200_EPOCH_REWARDS_AND_PENALTIES | B200_EPOCH_SLASHINGS | B200_EPOCH_EFFECTIVE_BALANCE_UPDATES))
            h->rehash[1] = 1;
        if (p.steps & B200_EPOCH_INACTIVITY_UPDATES) h->rehash[4] = 1;
    }
    if ((steps & B200_EPOCH_PARTICIPATION_FLAG_UPDATES) && n) {   // process_participation_flag_updates (:1231-1262)
        B200_CUDA_TRY(cudaMemcpyAsync(dev[2], dev[3], n, cudaMemcpyDeviceToDevice, e.stream));
        B200_CUDA_TRY(cudaMemsetAsync(dev[3], 0, n, e.stream));
        h->rehash[2] = h->rehash[3] = 1;
    }
    B200_CUDA_TRY(cudaEventRecord(e.ev1, e.stream));
    B200_CUDA_TRY(cudaEventSynchronize(e.ev1));
    float ms = 0;
    B200_CUDA_TRY(cudaEventElapsedTime(&ms, e.ev0, e.ev1));

    // ---- the small fields, through the paths b200_state_update_bytes and the reshaping calls take ----
    if (run_jf) {
        rc = update_bytes(e, h, h->so.justification_bits, jf, sizeof(jf));
        if (rc) return rc;
    }
    if ((steps & B200_EPOCH_ETH1_DATA_RESET) && next % P.epochs_per_eth1_voting_period == 0) {   // :1298-1328
        rc = set_small(e, h, 1, nullptr, 0);
        if (rc) return rc;
    }
    if (steps & B200_EPOCH_SLASHINGS_RESET) {   // :1371-1400
        const uint8_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        rc = update_bytes(e, h, h->so.slashings + 8 * (next % P.epochs_per_slashings_vector), zero, 8);
        if (rc) return rc;
    }
    if (steps & B200_EPOCH_RANDAO_MIXES_RESET) {   // :1401-1430
        uint8_t mix[32];
        memcpy(mix, h->shadow + h->so.randao_mixes + 32 * (cur % P.epochs_per_historical_vector), 32);
        rc = update_bytes(e, h, h->so.randao_mixes + 32 * (next % P.epochs_per_historical_vector), mix, 32);
        if (rc) return rc;
    }
    if (run_summary) {   // :929-964: hash_tree_root of block_roots and state_roots, pushed as one HistoricalSummary
        SszPlan sp;
        const uint64_t sphr = P.slots_per_historical_root;
        std::vector<uint32_t> outs{sp.wide_chunks(sp.stage_field(h->shadow + h->so.block_roots, 32 * sphr), sphr, depth_for(sphr)),
                                   sp.wide_chunks(sp.stage_field(h->shadow + h->so.state_roots, 32 * sphr), sphr, depth_for(sphr))};
        const size_t old_bytes = n_summaries * 64;
        std::vector<uint8_t> buf(old_bytes + 64);
        memcpy(buf.data(), h->shadow + h->so.var[8], old_bytes);
        rc = run_oneshot(e, sp, outs, buf.data() + old_bytes);
        if (rc) return rc;
        rc = set_small(e, h, 8, buf.data(), buf.size());
        if (rc) return rc;
    }
    if (run_sync) {   // last: a failed aggregation leaves every earlier sub-step applied
        int32_t rotated = 0;
        rc = sync_committee_updates(e, h, &rotated, out_code);
        if (rc) return rc;
        ms += e.last_kernel_ms;
    }
    e.last_kernel_ms = ms;
    return B200_SUCCESS;
}

int32_t b200_state_epoch_deltas(b200_state* h, uint64_t* out, size_t n_out) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || (n_out && !out)) return B200_ERR_BAD_ARG;
    const Preset& P = preset_of(h->preset);
    const uint64_t n = chain(h, 0).len;
    if (n_out != n) { e.last_error = "epoch_deltas: n is not the validator count"; return B200_ERR_BAD_ARG; }
    for (int f = 1; f < 5; f++)
        if (chain(h, f).len != n) { e.last_error = "epoch_deltas: the five big lists differ in length"; return B200_ERR_BAD_ARG; }
    if (!n) {
        e.last_kernel_ms = 0.f;
        return B200_SUCCESS;
    }
    const uint64_t cur = shadow_slot(h) / P.slots_per_epoch, prev = cur ? cur - 1 : 0;
    // get_unslashed_participating_indices(flag, prev) reads current_epoch_participation when prev == current (epoch 0)
    const uint8_t* part = chain_dev(h, cur ? 2 : 3);
    if ((rc = begin_timed(e))) return rc;
    EpochTotals T;
    rc = epoch_totals_on_device(e, chain_dev(h, 0), part, chain_dev(h, 3), n, cur, prev, P.ejection_balance, &T);
    if (rc) return rc;
    EpochParams p{};
    if ((rc = reward_scalars(e, T, P, 0xfu, "epoch_deltas", &p))) return rc;   // the active and the three flag sums
    p.cur = cur; p.prev = prev;
    p.leak = inactivity_leak(P, prev, le64(h->shadow + h->so.justification_bits + 81));   // finalized_checkpoint.epoch
    const uint64_t* d = nullptr;
    rc = epoch_deltas_on_device(e, chain_dev(h, 0), reinterpret_cast<const uint64_t*>(chain_dev(h, 4)), part, n, p, &d);
    if (rc) return rc;
    if ((rc = end_timed(e))) return rc;   // the device time of the kernels; the lists then go to the host
    B200_CUDA_TRY(cudaMemcpyAsync(out, d, size_t(n) * 64, cudaMemcpyDeviceToHost, e.stream));
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    return B200_SUCCESS;
}

int32_t b200_state_serialized_len(b200_state* h, uint64_t* out_len) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || !out_len) return B200_ERR_BAD_ARG;
    *out_len = h->len;
    return B200_SUCCESS;
}

int32_t b200_state_read_bytes(b200_state* h, uint64_t ssz_offset, uint8_t* out, size_t n) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!resident(h) || (n && !out) || ssz_offset > h->len || n > h->len - ssz_offset) return B200_ERR_BAD_ARG;
    for (const Piece& p : split_range(h, ssz_offset, ssz_offset + n)) {
        uint8_t* to = out + (p.x - ssz_offset);
        if (p.chain < 0) memcpy(to, h->shadow + p.x, p.y - p.x);
        else if (p.chain < 5)   // the big lists from HBM (the shadow holds the vectors)
            B200_CUDA_TRY(cudaMemcpyAsync(to, chain_dev(h, p.chain) + p.at, p.y - p.x, cudaMemcpyDeviceToHost, e.stream));
    }
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    return B200_SUCCESS;
}

// A state resident across the ranks of the communicator: every rank keeps its slices of the five big lists (and all small
// fields) in HBM; b200_state_root on such a handle is kernels + one ncclAllGather, no PCIe traffic.  Root only: the
// update / incremental entry points apply to single-GPU handles.
int32_t b200_state_upload_deneb_sharded(const uint8_t* ssz, size_t len, int32_t preset, b200_state** out_handle) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!ssz || !out_handle) return B200_ERR_BAD_ARG;
    const Comm& c = comm();
    if (!c.ready) { e.last_error = "b200_comm_init has not been called"; return B200_ERR_NOT_INITIALIZED; }
    std::unique_ptr<b200_state> h(new b200_state());
    rc = build_beacon_state_sharded_plan(h->plan, ssz, len, preset, c.rank, c.world, h->outputs);
    if (rc) { e.last_error = "sharded state upload: malformed SSZ or world not a power of two"; return rc; }
    uint8_t root[32];
    rc = h->plan.run(e, h->arena, h->fields, h->planbuf, COPY_ALL, h->outputs, root);   // uploads + first (collective) hash
    if (rc) return rc;
    h->len = len; h->preset = preset;
    h->sharded = true;
    *out_handle = h.release();
    return B200_SUCCESS;
}

// One call, all ranks: slices + small fields -> ncclAllGather of 5 x 32 B on the engine stream -> finisher.
int32_t b200_htr_beacon_state_deneb_sharded(const uint8_t* ssz, size_t len, int32_t preset, uint8_t out[32]) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!ssz || !out) return B200_ERR_BAD_ARG;
    const Comm& c = comm();
    if (!c.ready) { e.last_error = "b200_comm_init has not been called"; return B200_ERR_NOT_INITIALIZED; }
    SszPlan p;
    std::vector<uint32_t> outs;
    rc = build_beacon_state_sharded_plan(p, ssz, len, preset, c.rank, c.world, outs);
    if (rc) { e.last_error = "sharded hash_tree_root: malformed SSZ or world not a power of two"; return rc; }
    return run_oneshot(e, p, outs, out);
}

}  // extern "C"
