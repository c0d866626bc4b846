// extern "C" entry points — the BLS half of include/b200_consensus.h — and the host orchestration of the batch
// pipeline.  Every function below is a drop-in for one body in
// ethereum-consensus/src/crypto/bls.rs (line ranges in the header); all curve arithmetic runs in
// the kernels of bls_g1.cu / bls_g2.cu / bls_vm.cu / bls_rlc.cu.  The host only stages bytes and index arrays.
//
// Flow for T tuples with NK public keys in total (strict mode):
//   stream A: H2D offsets, keys (100 MB) ........ wait(B,C) | K1 key_validate (NK threads) | K2 per-tuple aggregate
//   stream B: H2D sigs | K3 sig decompress + subgroup check (T threads)   } under the key copy, before K1
//   stream C: H2D msgs | K4 hash_to_G2 (2T + T threads)                   }
//   stream A: K5 Miller loops (2T teams of 8 lanes) | K6 Gt product + final exponentiation (T teams) | D2H codes
// Registry mode skips K1: validated affine keys stay resident in HBM and K2 gathers them by validator index.
//
// Every entry point describes its work as one Batch; run_verify() runs it through these phases, in this order:
//   reserve_buffers  grow-only device buffers
//   stage_small      the small index arrays, built on the host, one pinned copy to the device (stream A)
//   key_phase        the key copy and K1 (two launches when big strict batches split the key copy), K3 / K4 right behind
//                    K1's first launch, K2
//   pairing_tail     K5 / K6 per tuple                                          | or rlc_tail: the whole-batch check
//   readback         verdicts to the host, event times; then the B200_BLS_TRACE line
#include <algorithm>
#include <cctype>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <random>
#include <string>
#include <type_traits>
#include <vector>

#include "bls_kernels.cuh"
#include "comm.h"
#include "engine.h"

namespace b200 {

struct BlsState {
    cudaStream_t sb = nullptr, sc = nullptr;  // signatures / messages: run under the per-key kernel
    cudaStream_t se = nullptr;   // split key copy: the second part of the keys and their per-key launch (ev_e: done)
    cudaEvent_t ev_e = nullptr;
    cudaEvent_t ev_in = nullptr, ev_b = nullptr, ev_c = nullptr, ev_k0 = nullptr, ev_k1 = nullptr, ev_d0 = nullptr, ev_d1 = nullptr;
    DevBuf keys, key_aff, key_code, g1pts, g1pre, pk_code, flags, sigs, g2pts, sig_code, msgs, small, f, out, h2c_tmp, gath;
    // RLC whole-batch check (bls_rlc.cu): Jacobian aggregates, scaled points, reduction ping-pong, zeros, indices, exchange
    DevBuf rlc_jac, rlc_g1, rlc_q, rlc_fa, rlc_fb, rlc_qa, rlc_qb, rlc_zero, rlc_idx, rlc_misc, rlc_xch;
    // batch aggregation: per-chunk partial sums and codes of the signature groups
    DevBuf agg_part;
    // aggregate_verify batches: the segmented Gt product's ping-pong levels
    DevBuf fold_a, fold_b;
    PinnedBuf stage;
    G1Pre* d_negg1_pre = nullptr;
    // registry (validated keys resident on the device)
    DevBuf reg_aff, reg_code;
    size_t reg_n = 0;
    float last_dominant_ms = 0.f;
    bool trace = false;          // B200_BLS_TRACE=1: per-phase CUDA-event timings on stderr
    cudaEvent_t ev_t[8] = {nullptr};
    // The signature / message kernels run under the per-key kernel K1 on high-priority streams.  With the call-based per-key
    // kernel (a fifth of the code, 12 warps/SM) that overlap beats running them before K1, with 128-thread CTAs at
    // T = 4096 and 32-thread CTAs at T = 256.  B200_BLS_SMALL_CTA overrides the CTA size (default: 32 up to 1 024 tuples, else 128).
    int small_cta_override = 0;

    // only a bls_state() that fails part-way destroys one: a completed state lives as long as the process
    ~BlsState() {
        for (cudaStream_t st : {sb, sc, se}) if (st) cudaStreamDestroy(st);
        for (cudaEvent_t ev : ev_t) if (ev) cudaEventDestroy(ev);
        for (cudaEvent_t ev : {ev_e, ev_in, ev_b, ev_c, ev_k0, ev_k1, ev_d0, ev_d1}) if (ev) cudaEventDestroy(ev);
        cudaFree(d_negg1_pre);
    }
};

// Launch-shape knobs: b200_tune(name, value), and at first use the environment variable B200_<NAME> (the name upper-cased),
// both through the row's setter.
struct Knob {
    const char* name;
    void (*set)(BlsState&, int64_t);
};
static const Knob kKnobs[] = {
    {"bls_small_cta", [](BlsState& s, int64_t v) { s.small_cta_override = int(v); }},
    {"vm_team16_max", [](BlsState&, int64_t v) { set_vm_team16_max(uint32_t(std::max<int64_t>(0, v))); }},
    {"vm_cta", [](BlsState&, int64_t v) { set_vm_cta(int(v)); }},
};

// The knobs' environment variables, then the settings b200_tune does not take: the per-key launch size up to which
// k_g1_validate goes out as 128-thread CTAs, and tracing, are fixed for the process at first use.
static void read_env(BlsState& s) {
    for (const Knob& k : kKnobs) {
        std::string var = "B200_";
        for (const char* c = k.name; *c; c++) var += char(toupper(static_cast<unsigned char>(*c)));
        if (const char* v = getenv(var.c_str())) k.set(s, atoll(v));
    }
    if (const char* v = getenv("B200_G1_SMALL_N")) set_g1_small_n(uint32_t(atol(v)));
    if (const char* v = getenv("B200_BLS_TRACE")) s.trace = atoi(v) != 0;
}

static int32_t bls_state(Engine& e, BlsState** out) {
    if (!e.bls) {
        std::unique_ptr<BlsState> s(new BlsState());   // freed if a step below fails; the next call starts over
        for (auto& ev : s->ev_t) B200_CUDA_TRY(cudaEventCreate(&ev));
        read_env(*s);
        // signatures / messages at the highest priority: their CTAs dispatch under the per-key kernel as its CTAs retire
        int prio_lo = 0, prio = 0;
        B200_CUDA_TRY(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio));
        B200_CUDA_TRY(cudaStreamCreateWithPriority(&s->sb, cudaStreamNonBlocking, prio));
        B200_CUDA_TRY(cudaStreamCreateWithPriority(&s->sc, cudaStreamNonBlocking, prio));
        B200_CUDA_TRY(cudaStreamCreateWithPriority(&s->se, cudaStreamNonBlocking, prio_lo));
        B200_CUDA_TRY(cudaEventCreateWithFlags(&s->ev_e, cudaEventDisableTiming));
        B200_CUDA_TRY(cudaEventCreateWithFlags(&s->ev_c, cudaEventDisableTiming));
        B200_CUDA_TRY(cudaEventCreateWithFlags(&s->ev_in, cudaEventDisableTiming));
        B200_CUDA_TRY(cudaEventCreateWithFlags(&s->ev_b, cudaEventDisableTiming));
        B200_CUDA_TRY(cudaEventCreate(&s->ev_k0));
        B200_CUDA_TRY(cudaEventCreate(&s->ev_k1));
        B200_CUDA_TRY(cudaEventCreate(&s->ev_d0));
        B200_CUDA_TRY(cudaEventCreate(&s->ev_d1));
        B200_CUDA_TRY(cudaMalloc(&s->d_negg1_pre, sizeof(G1Pre)));
        launch_neg_g1(s->d_negg1_pre, e.stream);
        e.launches++;
        if (vm_init(e.stream) != 0) { e.last_error = "pairing VM initialisation failed"; return B200_ERR_CUDA; }
        e.launches++;
        B200_CUDA_TRY(cudaGetLastError());
        B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
        e.bls = s.release();
    }
    *out = static_cast<BlsState*>(e.bls);
    return B200_SUCCESS;
}

enum PairMode { MODE_FAST_AGGREGATE = 0, MODE_AGGREGATE_BATCH = 1 };
// message offsets travel as uint32 (32 bytes per tuple on the batch paths): 32 * T must not wrap
constexpr size_t kMaxBatchTuples = size_t(1) << 26;
// keys a `..._batch_mixed` call may bring along (a block carries <= 16 deposits + 16 bls-to-execution changes)
constexpr size_t kRegistryExtraKeys = size_t(1) << 16;
constexpr size_t kRlcPart = sizeof(Fp12) + 16;   // one rank's exchanged RLC partial: Gt | bad flag (and 12 zero bytes)

// whole-batch RLC request: when passed, the pairing phase answers ONE boolean for all tuples instead of T codes
struct RlcReq {
    const uint8_t* seed32;  // scalars r_t = H(seed || t0 + t)
    uint64_t t0;            // global index of this call's first tuple (sharded batches)
    bool exchange;          // all-gather the per-rank Gt partials and bad flags over the library's communicator
    int32_t all_ok;         // out
};

// One call's work: T tuples.  MODE_FAST_AGGREGATE: tuple t sums keys [key_off[t], key_off[t+1]) and checks
// e(sum, H(msg_t)) e(-g1, sig_t) == 1.  MODE_AGGREGATE_BATCH: tuple t pairs keys [key_off[t], ..) with messages
// [msg_group[t], ..), (key_i, H(msg_i)) for each, plus (-g1, sig_t).
struct Batch {
    PairMode mode = MODE_FAST_AGGREGATE;
    // host key bytes (strict); with `index` as well: n_keys EXTRA keys (deposits, bls-to-execution changes) validated by this
    // call into the registry arrays' spare tail, named by indices reg_n + j
    const uint8_t* keys = nullptr;
    uint32_t n_keys = 0;
    const uint32_t* index = nullptr;   // non-null: registry gather by validator index
    uint32_t n_index = 0;
    const uint32_t* key_off = nullptr;
    const uint8_t* msgs = nullptr;     // host bytes + offsets (n_msgs + 1)
    const uint32_t* msg_off = nullptr;
    uint32_t n_msgs = 0;
    const uint32_t* msg_group = nullptr;   // MODE_AGGREGATE_BATCH: T + 1 offsets into the messages
    const uint8_t* sigs = nullptr;
    uint32_t T = 0;
    RlcReq* rlc = nullptr;
};

// aggregate_verify batches: tuple t has a pairing to check iff it has keys and as many messages as keys; the others are
// flagged EMPTY (VERIFY_FAIL after the key and signature decoding checks, as crypto/bls.rs:102-104)
static bool av_shape_ok(const Batch& b, uint32_t t) {
    const uint32_t nk = b.key_off[t + 1] - b.key_off[t];
    return nk != 0 && nk == b.msg_group[t + 1] - b.msg_group[t];
}
static uint32_t av_pairs(const Batch& b) {   // n + 1 pairs per tuple with a pairing
    uint32_t n = 0;
    for (uint32_t t = 0; t < b.T; t++)
        if (av_shape_ok(b, t)) n += b.key_off[t + 1] - b.key_off[t] + 1;
    return n;
}

// One level of the segmented Gt product (launch_fold_segments); o_*: word offsets of its arrays in the staged small array,
// o_out == kFinalLevel for the level that writes two values per segment
struct FoldLevel {
    size_t o_map, o_in, o_out;
    uint32_t n_in, n_out;
};
constexpr size_t kFinalLevel = ~size_t(0);

// Plans the segmented product of T segments whose T + 1 offsets are words[o_off ..]: each level's value -> segment map
// (level 0's at o_map0 unless that is kFinalLevel) and output offsets are appended to `words`.  Levels follow until every
// segment is in at most two pieces; with skip_pairs no level at all when every segment already holds two values or none.
static std::vector<FoldLevel> plan_fold(std::vector<uint32_t>& words, size_t o_off, uint32_t T, size_t o_map0, bool skip_pairs) {
    std::vector<FoldLevel> lv;
    auto len = [&](size_t o, uint32_t t) { return words[o + t + 1] - words[o + t]; };
    if (skip_pairs) {
        bool pairs = true;
        for (uint32_t t = 0; t < T && pairs; t++) pairs = len(o_off, t) == 0 || len(o_off, t) == 2;
        if (pairs) return lv;
    }
    auto pieces = [&](size_t o, uint32_t t) { return len(o, t) ? (words[o + t + 1] - 1) / 32 - words[o + t] / 32 + 1 : 0u; };
    size_t o_in = o_off, o_map = o_map0;
    for (;;) {
        const uint32_t n_in = words[o_in + T];
        if (o_map == kFinalLevel) {
            o_map = words.size();
            words.resize(o_map + n_in);
            for (uint32_t t = 0; t < T; t++)
                for (uint32_t i = words[o_in + t]; i < words[o_in + t + 1]; i++) words[o_map + i] = t;
        }
        uint32_t most = 0;
        for (uint32_t t = 0; t < T; t++) most = std::max(most, pieces(o_in, t));
        if (most <= 2) {
            lv.push_back({o_map, o_in, kFinalLevel, n_in, 2 * T});
            return lv;
        }
        const size_t o_out = words.size();
        words.resize(o_out + T + 1);
        words[o_out] = 0;
        for (uint32_t t = 0; t < T; t++) words[o_out + t + 1] = words[o_out + t] + pieces(o_in, t);
        lv.push_back({o_map, o_in, o_out, n_in, words[o_out + T]});
        o_in = o_out;
        o_map = kFinalLevel;
    }
}

// One run_verify call in phases.  The members are the sizes every phase derives from the batch, set once here, and where
// stage_small put the index arrays.
struct VerifyRun {
    Engine& e;
    BlsState& s;
    const Batch& b;
    const uint32_t T = b.T, n_keys = b.n_keys, n_msgs = b.n_msgs;
    const bool fa = b.mode == MODE_FAST_AGGREGATE, registry = b.index != nullptr;
    const uint32_t n_ops = registry ? b.n_index : n_keys;   // MODE_AGGREGATE_BATCH: one G1 operand per key of the call
    const uint32_t n_g1 = (fa ? T : n_ops) + 1;  // + (-g1)
    const uint32_t n_pairs = fa ? 2 * T : av_pairs(b);
    const uint32_t n_g2 = n_msgs + T;
    const uint32_t msg_bytes = b.msg_off[n_msgs];
    const uint32_t rlc_world = b.rlc && b.rlc->exchange ? uint32_t(comm().world) : 1u;
    const cudaStream_t sa = e.stream;
    // set by stage_small: word offsets in s.small, the pair arrays on the device, the pinned area results come back to
    size_t o_koff = 0, o_index = 0, o_moff = 0, o_tflags = 0, o_two = 0;
    std::vector<FoldLevel> fold;   // MODE_AGGREGATE_BATCH: the levels of the segmented Gt product
    const uint32_t *d_small = nullptr, *d_g1i = nullptr, *d_g2i = nullptr, *d_ptu = nullptr, *d_poff = nullptr;
    int32_t* h_out = nullptr;

    int32_t run(int32_t* out_codes);
    int32_t reserve_buffers();
    int32_t stage_small();
    int32_t key_phase();
    int32_t launch_small();
    void pairing_tail();
    int32_t rlc_tail();
    int32_t readback(void* h_dst, const void* d_src, size_t bytes);
};

int32_t VerifyRun::run(int32_t* out_codes) {
    if (b.rlc && !fa) return B200_ERR_BAD_ARG;
    int32_t rc;
    if ((rc = reserve_buffers()) || (rc = stage_small()) || (rc = key_phase())) return rc;
    if (b.rlc) return rlc_tail();
    pairing_tail();
    if ((rc = readback(h_out + 4, s.out.p, size_t(T) * 4))) return rc;
    if (s.trace) {
        float a = 0, b1 = 0, c = 0, d = 0, f2 = 0, g2 = 0;
        cudaEventElapsedTime(&a, s.ev_k0, s.ev_d0); cudaEventElapsedTime(&b1, s.ev_t[0], s.ev_t[1]);
        cudaEventElapsedTime(&c, s.ev_t[1], s.ev_t[2]); cudaEventElapsedTime(&d, s.ev_t[2], s.ev_t[3]);
        cudaEventElapsedTime(&f2, s.ev_t[3], s.ev_k1); cudaEventElapsedTime(&g2, s.ev_k0, s.ev_k1);
        fprintf(stderr, "[b200 bls] pre-K1 %.2f | K1 %.2f | K2 %.2f | wait(streamB) %.2f | miller %.2f | final %.2f | total %.2f ms\n",
                a, s.last_dominant_ms, b1, c, d, f2, g2);
    }
    for (uint32_t t = 0; t < T; t++) out_codes[t] = h_out[4 + t];
    return B200_SUCCESS;
}

int32_t VerifyRun::reserve_buffers() {
    B200_CUDA_TRY(s.keys.reserve(size_t(n_keys) * 48 + 64));
    B200_CUDA_TRY(s.key_aff.reserve(size_t(n_keys) * sizeof(G1Aff)));
    B200_CUDA_TRY(s.key_code.reserve(size_t(n_keys + 1) * 4));
    B200_CUDA_TRY(s.g1pre.reserve(size_t(n_g1) * sizeof(G1Pre)));
    B200_CUDA_TRY(s.pk_code.reserve(size_t(T + 1) * 4));
    B200_CUDA_TRY(s.flags.reserve(size_t(T + 1) * 4));
    B200_CUDA_TRY(s.sigs.reserve(size_t(T) * 96 + 64));
    B200_CUDA_TRY(s.g2pts.reserve(size_t(n_g2 + 1) * sizeof(G2Aff)));
    B200_CUDA_TRY(s.sig_code.reserve(size_t(T + 1) * 4));
    B200_CUDA_TRY(s.msgs.reserve(size_t(msg_bytes) + 64));
    B200_CUDA_TRY(s.f.reserve(size_t(n_pairs + 1) * sizeof(Fp12)));
    B200_CUDA_TRY(s.out.reserve(size_t(T + 1) * 4));
    B200_CUDA_TRY(s.h2c_tmp.reserve(size_t(2 * n_msgs + 2) * sizeof(G2Jac)));
    if (!b.rlc) return B200_SUCCESS;
    const uint32_t rlc_part = (T + 31) / 32 + rlc_world + 2;   // capacity of one reduction level (+ gathered partials)
    B200_CUDA_TRY(s.rlc_jac.reserve(size_t(T + 1) * sizeof(G1Jac)));
    B200_CUDA_TRY(s.rlc_g1.reserve(size_t(T + 2) * sizeof(G1Pre)));
    B200_CUDA_TRY(s.rlc_q.reserve(size_t(T + 1) * sizeof(G2Jac)));
    B200_CUDA_TRY(s.rlc_fa.reserve(size_t(rlc_part) * sizeof(Fp12)));
    B200_CUDA_TRY(s.rlc_fb.reserve(size_t(rlc_part) * sizeof(Fp12)));
    B200_CUDA_TRY(s.rlc_qa.reserve(size_t(rlc_part) * sizeof(G2Jac)));
    B200_CUDA_TRY(s.rlc_qb.reserve(size_t(rlc_part) * sizeof(G2Jac)));
    B200_CUDA_TRY(s.rlc_zero.reserve(size_t(T + 8) * 4));
    B200_CUDA_TRY(s.rlc_idx.reserve(size_t(2 * (T + 1)) * 4));
    B200_CUDA_TRY(s.rlc_misc.reserve(256));
    B200_CUDA_TRY(s.rlc_xch.reserve(size_t(rlc_world + 1) * kRlcPart));
    return B200_SUCCESS;
}

// small host-built arrays, one staged copy on stream A: [key_off | index | msg_off | g1_idx | g2_idx | pair_tuple | pair_off],
// then for MODE_AGGREGATE_BATCH [tuple flags | 0, 2, .., 2T | the fold levels' maps and offsets]
int32_t VerifyRun::stage_small() {
    std::vector<uint32_t> small;
    small.reserve(size_t(T) + 1 + b.n_index + n_msgs + 1 + 3 * size_t(n_pairs) + T + 1 + 8);
    o_koff = small.size();
    small.insert(small.end(), b.key_off, b.key_off + T + 1);
    o_index = small.size();
    if (registry) small.insert(small.end(), b.index, b.index + b.n_index);
    o_moff = small.size();
    small.insert(small.end(), b.msg_off, b.msg_off + n_msgs + 1);
    const size_t o_g1i = small.size();
    small.resize(small.size() + 3 * size_t(n_pairs) + T + 1);
    uint32_t* g1i = small.data() + o_g1i;
    uint32_t* g2i = g1i + n_pairs;
    uint32_t* ptu = g2i + n_pairs;
    uint32_t* poff = ptu + n_pairs;
    if (fa) {
        for (uint32_t t = 0; t < T; t++) {
            g1i[2 * t] = t;          g2i[2 * t] = t;          // (agg_t, H(msg_t))
            g1i[2 * t + 1] = T;      g2i[2 * t + 1] = n_msgs + t;  // (-g1, sig_t)
            ptu[2 * t] = ptu[2 * t + 1] = t;
            poff[t] = 2 * t;
        }
        poff[T] = 2 * T;
    } else {   // tuple t: (key_i, H(msg_i)) for its n keys and messages, then (-g1, sig_t); none without a pairing
        uint32_t p = 0;
        for (uint32_t t = 0; t < T; t++) {
            poff[t] = p;
            if (!av_shape_ok(b, t)) continue;
            for (uint32_t k = b.key_off[t], m = b.msg_group[t]; k < b.key_off[t + 1]; k++, m++, p++) { g1i[p] = k; g2i[p] = m; ptu[p] = t; }
            g1i[p] = n_ops; g2i[p] = n_msgs + t; ptu[p] = t;
            p++;
        }
        poff[T] = p;
        o_tflags = small.size();
        for (uint32_t t = 0; t < T; t++) small.push_back(av_shape_ok(b, t) ? 0u : uint32_t(TUPLE_FLAG_EMPTY));
        o_two = small.size();
        for (uint32_t t = 0; t <= T; t++) small.push_back(2 * t);
        // level 0 reads the Miller values, with pair_tuple as its map
        fold = plan_fold(small, o_g1i + 3 * size_t(n_pairs), T, o_g1i + 2 * size_t(n_pairs), true);
        uint32_t most = 0;
        for (const FoldLevel& l : fold) most = std::max(most, l.n_out);
        B200_CUDA_TRY(s.fold_a.reserve((size_t(most) + 1) * sizeof(Fp12)));
        B200_CUDA_TRY(s.fold_b.reserve((size_t(most) + 1) * sizeof(Fp12)));
    }
    const size_t small_bytes = small.size() * 4;
    B200_CUDA_TRY(s.stage.reserve(small_bytes + size_t(T + 1) * 4 + 64 +
                                  (b.rlc ? 256 + size_t(rlc_world) * kRlcPart + size_t(8 + 2 * (T + 1)) * 4 : 0)));
    B200_CUDA_TRY(s.small.reserve(small_bytes + 64));
    memcpy(s.stage.p, small.data(), small_bytes);
    h_out = reinterpret_cast<int32_t*>(static_cast<uint8_t*>(s.stage.p) + ((small_bytes + 15) & ~size_t(15)));
    d_small = static_cast<const uint32_t*>(s.small.p);
    d_g1i = d_small + o_g1i;
    d_g2i = d_g1i + n_pairs;
    d_ptu = d_g2i + n_pairs;
    d_poff = d_ptu + n_pairs;
    B200_CUDA_TRY(cudaMemcpyAsync(s.small.p, s.stage.p, small_bytes, cudaMemcpyHostToDevice, sa));
    B200_CUDA_TRY(cudaEventRecord(s.ev_in, sa));
    return B200_SUCCESS;
}

// Key copy and K1, the signature / message kernels right behind K1's first launch, K2, and the join
int32_t VerifyRun::key_phase() {
    const bool have_k1 = n_keys != 0;
    // Big strict batches: the first kSplitWaves full waves of the per-key kernel start as soon as THEIR keys have arrived; the rest of
    // the key bytes (~90 MB at T = 4096) cross PCIe on stream E under that first launch, and the second launch follows them there
    // (two streams, so its CTAs fill the first launch's draining tail).
    // The split point is a fixed key count (4 x 148 x 384), not whole waves of this GPU: on an H100 (132 SMs) sizing it and the
    // thresholds below from the SM count made the T = 4096 step ~1 % slower.
    constexpr uint32_t kSplitWaves = 4, kSplitKeys = kSplitWaves * 148u * 384u;
    const uint32_t k_split = (have_k1 && !registry && n_keys >= 4u * kSplitKeys) ? kSplitKeys : n_keys;
    if (n_keys) B200_CUDA_TRY(cudaMemcpyAsync(s.keys.p, b.keys, size_t(k_split) * 48, cudaMemcpyHostToDevice, sa));
    B200_CUDA_TRY(cudaEventRecord(s.ev_k0, sa));
    // packed CTAs only when there is a big per-key kernel to run under; alone (registry mode, small batches) they spread
    set_small_cta(s.small_cta_override ? s.small_cta_override : ((have_k1 && n_keys >= 148u * 384u && T > 1024) ? 128 : 32));
    // ---- stream A: public keys
    B200_CUDA_TRY(cudaEventRecord(s.ev_d0, sa));
    const G1Aff* key_aff = registry ? static_cast<const G1Aff*>(s.reg_aff.p) : static_cast<const G1Aff*>(s.key_aff.p);
    const int32_t* key_code = registry ? static_cast<const int32_t*>(s.reg_code.p) : static_cast<const int32_t*>(s.key_code.p);
    // where the per-key kernel writes: the call's own arrays, or (registry + extra keys) the tail behind the reg_n resident keys
    G1Aff* k1_aff = registry ? static_cast<G1Aff*>(s.reg_aff.p) + s.reg_n : static_cast<G1Aff*>(s.key_aff.p);
    int32_t* k1_code = registry ? static_cast<int32_t*>(s.reg_code.p) + s.reg_n : static_cast<int32_t*>(s.key_code.p);
    if (have_k1) {
        // the first launch of a split copy, the one the signature / message kernels run under, in 128-thread CTAs: as three
        // CTAs per SM a side kernel's CTA displaces a third of an SM's per-key work instead of all of it
        launch_g1_validate(static_cast<const uint8_t*>(s.keys.p), k_split, k1_aff, k1_code, sa, k_split < n_keys ? 128 : 0);
        e.launches++;
    }
    int32_t rc = launch_small();
    if (rc) return rc;
    if (k_split < n_keys) {   // the remaining keys: copy strictly after the first part's (one PCIe link), then their launch
        B200_CUDA_TRY(cudaStreamWaitEvent(s.se, s.ev_k0, 0));
        B200_CUDA_TRY(cudaMemcpyAsync(static_cast<uint8_t*>(s.keys.p) + size_t(k_split) * 48, b.keys + size_t(k_split) * 48,
                                      size_t(n_keys - k_split) * 48, cudaMemcpyHostToDevice, s.se));
        launch_g1_validate(static_cast<const uint8_t*>(s.keys.p) + size_t(k_split) * 48, n_keys - k_split, k1_aff + k_split,
                           k1_code + k_split, s.se, 384);
        e.launches++;
        B200_CUDA_TRY(cudaEventRecord(s.ev_e, s.se));
        B200_CUDA_TRY(cudaStreamWaitEvent(sa, s.ev_e, 0));
    }
    B200_CUDA_TRY(cudaEventRecord(s.ev_d1, sa));
    if (s.trace) cudaEventRecord(s.ev_t[0], sa);
    launch_g1_aggregate(key_aff, key_code, registry ? d_small + o_index : nullptr, d_small + o_koff, T,
                        nullptr, fa ? static_cast<G1Pre*>(s.g1pre.p) : nullptr,
                        static_cast<int32_t*>(s.pk_code.p), static_cast<uint32_t*>(s.flags.p),
                        0u, sa, b.rlc ? static_cast<G1Jac*>(s.rlc_jac.p) : nullptr, fa ? nullptr : d_small + o_tflags);
    e.launches++;
    if (!fa) {   // every key's pair operand for the VM
        launch_g1_pair_operands(key_aff, registry ? d_small + o_index : nullptr, n_ops, static_cast<G1Pre*>(s.g1pre.p), sa);
        if (n_ops) e.launches++;
    }
    // -g1 behind the tuples' aggregates or the keys' operands
    B200_CUDA_TRY(cudaMemcpyAsync(static_cast<G1Pre*>(s.g1pre.p) + n_g1 - 1, s.d_negg1_pre, sizeof(G1Pre), cudaMemcpyDeviceToDevice, sa));
    // ---- join, pairing
    if (s.trace) cudaEventRecord(s.ev_t[1], sa);
    B200_CUDA_TRY(cudaStreamWaitEvent(sa, s.ev_b, 0));
    B200_CUDA_TRY(cudaStreamWaitEvent(sa, s.ev_c, 0));
    if (s.trace) cudaEventRecord(s.ev_t[2], sa);
    return B200_SUCCESS;
}

// signatures on stream B, messages on stream C, both behind the small arrays (ev_in); done: ev_b, ev_c
int32_t VerifyRun::launch_small() {
    cudaStream_t sb = s.sb, sc = s.sc;
    B200_CUDA_TRY(cudaStreamWaitEvent(sb, s.ev_in, 0));
    B200_CUDA_TRY(cudaStreamWaitEvent(sc, s.ev_in, 0));
    if (T) B200_CUDA_TRY(cudaMemcpyAsync(s.sigs.p, b.sigs, size_t(T) * 96, cudaMemcpyHostToDevice, sb));
    if (msg_bytes) B200_CUDA_TRY(cudaMemcpyAsync(s.msgs.p, b.msgs, msg_bytes, cudaMemcpyHostToDevice, sc));
    launch_g2_sig_decode(static_cast<const uint8_t*>(s.sigs.p), T, static_cast<G2Aff*>(s.g2pts.p) + n_msgs, static_cast<int32_t*>(s.sig_code.p), sb);
    launch_hash_to_g2(static_cast<const uint8_t*>(s.msgs.p), d_small + o_moff, n_msgs, static_cast<G2Aff*>(s.g2pts.p), s.h2c_tmp.p, sc);
    e.launches += (T ? 1 : 0) + (n_msgs ? 2 : 0);
    B200_CUDA_TRY(cudaEventRecord(s.ev_b, sb));
    B200_CUDA_TRY(cudaEventRecord(s.ev_c, sc));
    return B200_SUCCESS;
}

// Miller loops and final exponentiations per tuple on stream A, on the lane-parallel VM.  An aggregate_verify tuple's
// n + 1 Miller values are folded level by level to the two the final exponentiation reads; fast-aggregate tuples have
// two already (no fold levels).
void VerifyRun::pairing_tail() {
    const G2Aff* d_g2 = static_cast<const G2Aff*>(s.g2pts.p);
    const int32_t* d_pk = static_cast<const int32_t*>(s.pk_code.p);
    const uint32_t* d_fl = static_cast<const uint32_t*>(s.flags.p);
    const int32_t* d_sc = static_cast<const int32_t*>(s.sig_code.p);
    launch_vm_miller(static_cast<const G1Pre*>(s.g1pre.p), d_g1i, d_g2, d_g2i, d_ptu, d_pk, d_fl, d_sc, n_pairs, static_cast<Fp12*>(s.f.p), sa);
    if (s.trace) cudaEventRecord(s.ev_t[3], sa);
    const Fp12* fin = static_cast<const Fp12*>(s.f.p);
    Fp12* const buf[2] = {static_cast<Fp12*>(s.fold_a.p), static_cast<Fp12*>(s.fold_b.p)};
    for (size_t k = 0; k < fold.size(); k++) {
        const FoldLevel& l = fold[k];
        launch_fold_segments(fin, l.n_in, d_small + l.o_map, d_small + l.o_in, l.o_out == kFinalLevel ? nullptr : d_small + l.o_out,
                             d_pk, d_fl, d_sc, buf[k & 1], sa);
        if (l.n_in) e.launches++;
        fin = buf[k & 1];
    }
    launch_vm_final(fin, fold.empty() ? d_poff : d_small + o_two, d_pk, d_fl, d_sc, T, static_cast<int32_t*>(s.out.p), sa);
    e.launches += (n_pairs ? 1 : 0) + (T ? 1 : 0);
}

// `bytes` of results into the pinned area once every stream has finished; the call's kernel and per-key times
int32_t VerifyRun::readback(void* h_dst, const void* d_src, size_t bytes) {
    B200_CUDA_TRY(cudaEventRecord(s.ev_k1, sa));
    B200_CUDA_TRY(cudaGetLastError());
    B200_CUDA_TRY(cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, sa));
    B200_CUDA_TRY(cudaStreamSynchronize(sa));
    B200_CUDA_TRY(cudaStreamSynchronize(s.sb));
    B200_CUDA_TRY(cudaStreamSynchronize(s.sc));
    B200_CUDA_TRY(cudaEventElapsedTime(&e.last_kernel_ms, s.ev_k0, s.ev_k1));
    B200_CUDA_TRY(cudaEventElapsedTime(&s.last_dominant_ms, s.ev_d0, s.ev_d1));
    return B200_SUCCESS;
}

// Warp-shuffle folds (k_rlc_reduce, 32 -> 1 per launch) until one value is left: the Gt product of n Fp12 values or the
// sum of n G2 points.  The launches alternate between buf[pp] and buf[pp ^ 1] (each holding at least ceil(n / 32)
// values); returns the buffer with the result, and pp then names the other one.
template <class T>
static const T* rlc_fold(Engine& e, const T* in, uint32_t n, T* const buf[2], int& pp, cudaStream_t st) {
    do {
        if constexpr (std::is_same_v<T, Fp12>) n = launch_rlc_reduce(in, nullptr, n, buf[pp], nullptr, st);
        else n = launch_rlc_reduce(nullptr, in, n, nullptr, buf[pp], st);
        e.launches++;
        in = buf[pp]; pp ^= 1;
    } while (n > 1);
    return in;
}

// ---- RLC whole-batch check (bls_rlc.cu): T Miller loops + ONE final exponentiation
int32_t VerifyRun::rlc_tail() {
    RlcReq* rlc = b.rlc;
    G2Aff* d_g2 = static_cast<G2Aff*>(s.g2pts.p);
    const size_t kPart = kRlcPart;
    uint8_t* h_x = reinterpret_cast<uint8_t*>(h_out + 16);                    // gathered partials (their bad flags are read on the host)
    uint32_t* d_zero = static_cast<uint32_t*>(s.rlc_zero.p);  // "every tuple alive" code arrays for the VM kernels
    uint32_t* d_idx = static_cast<uint32_t*>(s.rlc_idx.p);   // [0..T] identity (g1 / tuple index) | [0..T-1, n_g2] (H_t, then S)
    uint8_t* d_misc = static_cast<uint8_t*>(s.rlc_misc.p);    // [0,32) seed words | [32,36) bad flag | [64,68) final code
    G1Pre* d_rg1 = static_cast<G1Pre*>(s.rlc_g1.p);
    G2Jac* d_rq = static_cast<G2Jac*>(s.rlc_q.p);
    B200_CUDA_TRY(cudaMemsetAsync(d_zero, 0, size_t(T + 8) * 4, sa));
    B200_CUDA_TRY(cudaMemsetAsync(d_misc + 32, 0, 96, sa));
    {   // seed words + index arrays through the pinned staging area (behind the small arrays and the code slots)
        uint32_t* h = reinterpret_cast<uint32_t*>(h_x + ((size_t(rlc_world) * kPart + 63) & ~size_t(63)));
        for (int i = 0; i < 8; i++)
            h[i] = (uint32_t(rlc->seed32[4 * i]) << 24) | (uint32_t(rlc->seed32[4 * i + 1]) << 16) | (uint32_t(rlc->seed32[4 * i + 2]) << 8) | rlc->seed32[4 * i + 3];
        uint32_t* hi = h + 8;
        for (uint32_t t = 0; t <= T; t++) { hi[t] = t; hi[T + 1 + t] = t < T ? t : n_g2; }
        B200_CUDA_TRY(cudaMemcpyAsync(d_misc, h, 32, cudaMemcpyHostToDevice, sa));
        B200_CUDA_TRY(cudaMemcpyAsync(d_idx, hi, size_t(2 * (T + 1)) * 4, cudaMemcpyHostToDevice, sa));
    }
    launch_rlc_scale(static_cast<const G1Jac*>(s.rlc_jac.p), d_g2 + n_msgs, static_cast<const int32_t*>(s.pk_code.p),
                     static_cast<const uint32_t*>(s.flags.p), static_cast<const int32_t*>(s.sig_code.p),
                     reinterpret_cast<const uint32_t*>(d_misc), rlc->t0, T, d_rg1, d_rq, reinterpret_cast<int32_t*>(d_misc + 32), sa);
    B200_CUDA_TRY(cudaMemcpyAsync(d_rg1 + T, s.d_negg1_pre, sizeof(G1Pre), cudaMemcpyDeviceToDevice, sa));
    if (s.trace) cudaEventRecord(s.ev_t[3], sa);
    Fp12* fbuf[2] = {static_cast<Fp12*>(s.rlc_fa.p), static_cast<Fp12*>(s.rlc_fb.p)};
    G2Jac* qbuf[2] = {static_cast<G2Jac*>(s.rlc_qa.p), static_cast<G2Jac*>(s.rlc_qb.p)};
    // S = sum_t r_t sig_t first (warp-shuffle folds T -> T/32 -> ... -> 1): its pair (-g1, S) then rides in the SAME
    // Miller launch as the T tuple pairs instead of costing a second, latency-bound launch of one team
    int pp = 0;
    const G2Jac* qi = rlc_fold(e, d_rq, T, qbuf, pp, sa);
    launch_rlc_finish(qi, d_g2 + n_g2, sa);
    // T + 1 Miller loops on the lane-parallel VM: (r_t agg_t, H_t) for every tuple and (-g1, S)
    launch_vm_miller(d_rg1, d_idx, d_g2, d_idx + T + 1, d_zero, reinterpret_cast<const int32_t*>(d_zero), d_zero,
                     reinterpret_cast<const int32_t*>(d_zero), T + 1, static_cast<Fp12*>(s.f.p), sa);
    // Gt product of the T + 1 Miller values, again by warp-shuffle folds
    pp = 0;
    const Fp12* fi = rlc_fold(e, static_cast<const Fp12*>(s.f.p), T + 1, fbuf, pp, sa);
    if (rlc->exchange && rlc_world > 1) {
        // the path's one exchange step: e(-g1, sum over ranks) = product over ranks, so every rank has already paired
        // its own partial sum and only the Gt partial (576 B) and the bad flag travel; then the same fold on all ranks
        uint8_t* x = static_cast<uint8_t*>(s.rlc_xch.p);
        B200_CUDA_TRY(cudaMemcpyAsync(x, fi, sizeof(Fp12), cudaMemcpyDeviceToDevice, sa));
        B200_CUDA_TRY(cudaMemcpyAsync(x + sizeof(Fp12), d_misc + 32, 16, cudaMemcpyDeviceToDevice, sa));
        int32_t rcx = comm_all_gather(e, x, x + kPart, kPart, sa);
        if (rcx) return rcx;
        for (uint32_t r = 0; r < rlc_world; r++)   // unpack into the fold's input array (world <= a few dozen)
            B200_CUDA_TRY(cudaMemcpyAsync(fbuf[pp] + r, x + kPart * (1 + r), sizeof(Fp12), cudaMemcpyDeviceToDevice, sa));
        B200_CUDA_TRY(cudaMemcpyAsync(h_x, x + kPart, size_t(rlc_world) * kPart, cudaMemcpyDeviceToHost, sa));   // for the ranks' bad flags
        fi = fbuf[pp]; pp ^= 1;
        fi = rlc_fold(e, fi, rlc_world, fbuf, pp, sa);
    }
    // the single final exponentiation: (Gt product) * 1
    Fp12* d_fin = fbuf[pp];
    B200_CUDA_TRY(cudaMemcpyAsync(d_fin, fi, sizeof(Fp12), cudaMemcpyDeviceToDevice, sa));
    launch_fp12_one(d_fin + 1, sa);
    launch_vm_final(d_fin, d_zero, reinterpret_cast<const int32_t*>(d_zero), d_zero, reinterpret_cast<const int32_t*>(d_zero), 1,
                    reinterpret_cast<int32_t*>(d_misc + 64), sa);
    e.launches += 5;
    int32_t rc = readback(h_out, d_misc + 32, 64);   // [0] bad, [8] final code
    if (rc) return rc;
    bool bad = h_out[0] != 0;
    if (rlc->exchange && rlc_world > 1)
        for (uint32_t r = 0; r < rlc_world; r++) {
            int32_t flag;
            memcpy(&flag, h_x + size_t(r) * kPart + sizeof(Fp12), 4);
            bad = bad || flag != 0;
        }
    rlc->all_ok = (!bad && h_out[8] == BLS_SUCCESS) ? 1 : 0;
    if (s.trace) {
        float a = 0, g2 = 0;
        cudaEventElapsedTime(&a, s.ev_t[2], s.ev_k1); cudaEventElapsedTime(&g2, s.ev_k0, s.ev_k1);
        fprintf(stderr, "[b200 bls rlc] K1 %.2f | scale + T Miller loops + folds + 1 final exponentiation %.2f | total %.2f ms\n",
                s.last_dominant_ms, a, g2);
    }
    return B200_SUCCESS;
}

// An early error return must not leave work queued on the side streams (they read the caller's host buffers and the
// engine's grow-only device buffers): drain all of them before handing the error back.
static int32_t run_verify(Engine& e, BlsState& s, const Batch& b, int32_t* out_codes) {
    const int32_t rc = VerifyRun{e, s, b}.run(out_codes);
    if (rc != B200_SUCCESS) {
        cudaStreamSynchronize(e.stream);
        cudaStreamSynchronize(s.sb);
        cudaStreamSynchronize(s.sc);
        cudaStreamSynchronize(s.se);
        cudaGetLastError();
    }
    return rc;
}

// ---- argument checks and set-up shared by the batch entry points

// T + 1 non-decreasing offsets; *count: the last one (keys, or registry indices, of the batch)
static int32_t check_offsets(const uint32_t* off, size_t n_tuples, uint32_t* count) {
    for (size_t t = 0; t < n_tuples; t++)
        if (off[t] > off[t + 1]) return B200_ERR_BAD_ARG;
    *count = off[n_tuples];
    return B200_SUCCESS;
}

// offsets of T 32-byte messages
static std::vector<uint32_t> msg32_offsets(size_t n_tuples) {
    std::vector<uint32_t> moff(n_tuples + 1);
    for (size_t t = 0; t <= n_tuples; t++) moff[t] = uint32_t(32 * t);
    return moff;
}

// contiguous block of tuples per rank, balanced to within one (parallel.tuple_shard in the Python mirror)
struct TupleRange {
    size_t lo, cnt;
};
static TupleRange tuple_shard(size_t n_tuples, size_t world, size_t rank) {
    const size_t base = n_tuples / world, rem = n_tuples % world;
    return {rank * base + std::min(rank, rem), base + (rank < rem ? 1 : 0)};
}

// the rank's block of a strict batch as a batch of its own; koff / moff receive its rebased key and message offsets
static Batch shard_batch(const uint8_t* pks_flat, const uint32_t* pk_offsets, const uint8_t* msgs32, const uint8_t* sigs, TupleRange r,
                         std::vector<uint32_t>& koff, std::vector<uint32_t>& moff) {
    koff.resize(r.cnt + 1);
    for (size_t t = 0; t <= r.cnt; t++) koff[t] = pk_offsets[r.lo + t] - pk_offsets[r.lo];
    moff = msg32_offsets(r.cnt);
    return {.keys = pks_flat ? pks_flat + size_t(pk_offsets[r.lo]) * 48 : nullptr, .n_keys = koff[r.cnt], .key_off = koff.data(),
            .msgs = msgs32 + 32 * r.lo, .msg_off = moff.data(), .n_msgs = uint32_t(r.cnt), .sigs = sigs + 96 * r.lo, .T = uint32_t(r.cnt)};
}

// Registry entries beyond reg_n reserved when its arrays are (re)allocated: the resident state lists' rule, 2^16 or a
// sixteenth of the registry, so that appends of a block's deposits validate in place for many blocks
static size_t registry_headroom(size_t n) { return std::max<size_t>(size_t(1) << 16, n / 16); }

// Validate n keys into registry entries [at, at + n) and make the registry at + n keys long: at = 0 replaces it,
// at = reg_n appends.  The keys come from the host (`host_keys`) or from n Validator records in HBM (`records`).  The
// arrays always hold reg_n keys, then the extra-key tail `..._batch_mixed` validates into; an append past that grows them
// (entries [0, at) copied on the device) before any key is validated.  last_kernel_ms: the gather and K1.
static int32_t registry_fill(Engine& e, BlsState& s, size_t at, const uint8_t* host_keys, const uint8_t* records, size_t n) {
    const size_t need = at + n + kRegistryExtraKeys + 1;
    if (s.reg_aff.cap < need * sizeof(G1Aff) || s.reg_code.cap < need * 4) {
        const size_t want = at + n + registry_headroom(at + n) + kRegistryExtraKeys + 1;
        DevBuf na, nc;
        cudaError_t ce = na.reserve(want * sizeof(G1Aff));
        if (ce == cudaSuccess) ce = nc.reserve(want * 4);
        if (ce == cudaSuccess && at) ce = cudaMemcpyAsync(na.p, s.reg_aff.p, at * sizeof(G1Aff), cudaMemcpyDeviceToDevice, e.stream);
        if (ce == cudaSuccess && at) ce = cudaMemcpyAsync(nc.p, s.reg_code.p, at * 4, cudaMemcpyDeviceToDevice, e.stream);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(e.stream);
        if (ce != cudaSuccess) {
            na.release(); nc.release();
            e.last_error = std::string("registry growth: ") + cudaGetErrorString(ce);
            return B200_ERR_CUDA;
        }
        s.reg_aff.release(); s.reg_code.release();
        s.reg_aff = na; s.reg_code = nc;
    }
    B200_CUDA_TRY(s.keys.reserve(n * 48 + 64));
    if (host_keys && n) B200_CUDA_TRY(cudaMemcpyAsync(s.keys.p, host_keys, n * 48, cudaMemcpyHostToDevice, e.stream));
    B200_CUDA_TRY(cudaEventRecord(s.ev_k0, e.stream));
    if (records) {
        launch_gather_validator_keys(records, uint32_t(n), static_cast<uint8_t*>(s.keys.p), e.stream);
        e.launches += n ? 1 : 0;
    }
    launch_g1_validate(static_cast<const uint8_t*>(s.keys.p), uint32_t(n), static_cast<G1Aff*>(s.reg_aff.p) + at,
                       static_cast<int32_t*>(s.reg_code.p) + at, e.stream);
    e.launches += n ? 1 : 0;
    B200_CUDA_TRY(cudaEventRecord(s.ev_k1, e.stream));
    B200_CUDA_TRY(cudaGetLastError());
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    B200_CUDA_TRY(cudaEventElapsedTime(&e.last_kernel_ms, s.ev_k0, s.ev_k1));
    s.last_dominant_ms = e.last_kernel_ms;
    s.reg_n = at + n;
    return B200_SUCCESS;
}

// the registry calls on a resident state: its Validator records in HBM and their count
static int32_t registry_state_records(Engine& e, b200_state* h, const uint8_t** records, uint64_t* n) {
    if (state_validator_records(h, records, n)) {
        e.last_error = "registry: the state handle is NULL or sharded";
        return B200_ERR_BAD_ARG;
    }
    if (*n > 0x7fffffffu) { e.last_error = "registry: more validators than the registry holds"; return B200_ERR_BAD_ARG; }
    return B200_SUCCESS;
}

// every validator index names a resident registry key or one of the call's n_extra extra keys
static int32_t check_indices(Engine& e, const BlsState& s, const uint32_t* index, uint32_t n, size_t n_extra) {
    for (uint32_t i = 0; i < n; i++)
        if (index[i] >= s.reg_n + n_extra) {
            e.last_error = n_extra ? "validator index outside the loaded registry (+ extra keys)" : "validator index outside the loaded registry";
            return B200_ERR_BAD_ARG;
        }
    return B200_SUCCESS;
}

// ---- aggregation of T groups (aggregate / eth_aggregate_public_keys)

// the batch aggregation entry points' checks; n_groups == 0 passes (and sets last_kernel_ms); *n: the item count
static int32_t check_aggregate_args(Engine& e, const uint32_t* off, size_t n_groups, const uint8_t* out, const int32_t* codes,
                                    uint32_t* n) {
    e.last_kernel_ms = 0.f;
    *n = 0;
    if (n_groups == 0) return B200_SUCCESS;
    if (!off || !out || !codes || n_groups > kMaxBatchTuples) return B200_ERR_BAD_ARG;
    int32_t rc = check_offsets(off, n_groups, n);
    if (rc) return rc;
    if (*n > 0x3fffffffu) { e.last_error = "aggregate: more than 0x3fffffff items"; return B200_ERR_BAD_ARG; }
    return B200_SUCCESS;
}

// device results of T groups (codes, then `bytes` per group) to the caller; last_kernel_ms from ev_k0 / ev_k1
static int32_t aggregate_readback(Engine& e, BlsState& s, const void* d_codes, const void* d_bytes, uint32_t T, size_t bytes,
                                  uint8_t* out, int32_t* out_codes) {
    cudaStream_t sa = e.stream;
    B200_CUDA_TRY(s.stage.reserve(size_t(T) * (4 + bytes)));
    uint8_t* h = static_cast<uint8_t*>(s.stage.p);
    B200_CUDA_TRY(cudaMemcpyAsync(h, d_codes, size_t(T) * 4, cudaMemcpyDeviceToHost, sa));
    B200_CUDA_TRY(cudaMemcpyAsync(h + size_t(T) * 4, d_bytes, size_t(T) * bytes, cudaMemcpyDeviceToHost, sa));
    B200_CUDA_TRY(cudaStreamSynchronize(sa));
    B200_CUDA_TRY(cudaEventElapsedTime(&e.last_kernel_ms, s.ev_k0, s.ev_k1));
    memcpy(out_codes, h, size_t(T) * 4);
    memcpy(out, h + size_t(T) * 4, size_t(T) * bytes);
    return B200_SUCCESS;
}

// n signatures (host), T groups by `off` (host): K3 over all n, then the chunked sum and the per-group finish
static int32_t aggregate_sigs(Engine& e, BlsState& s, const uint8_t* sigs, uint32_t n, const uint32_t* off, uint32_t T,
                              uint8_t* out96, int32_t* out_codes) {
    const uint32_t chunk = g2_aggregate_chunk(n);
    // small array: offsets (T + 1) | chunk_off (T + 1) | chunk_group (n_chunks)
    std::vector<uint32_t> small(off, off + T + 1);
    small.push_back(0);
    auto chunks_of = [&](uint32_t g) { return std::max<uint32_t>(1u, (off[g + 1] - off[g] + chunk - 1) / chunk); };
    for (uint32_t g = 0; g < T; g++) small.push_back(small.back() + chunks_of(g));
    const uint32_t n_chunks = small.back();
    for (uint32_t g = 0; g < T; g++) small.insert(small.end(), chunks_of(g), g);
    B200_CUDA_TRY(s.sigs.reserve(size_t(n) * 96 + 64));
    B200_CUDA_TRY(s.g2pts.reserve((size_t(n) + 1) * sizeof(G2Aff)));
    B200_CUDA_TRY(s.sig_code.reserve((size_t(n) + 1) * 4));
    B200_CUDA_TRY(s.small.reserve(small.size() * 4 + 64));
    B200_CUDA_TRY(s.agg_part.reserve((size_t(n_chunks) + 1) * (sizeof(G2Jac) + 4) + size_t(T) * 4));
    B200_CUDA_TRY(s.out.reserve(size_t(T) * (96 + 4) + 64));
    cudaStream_t sa = e.stream;
    uint32_t* d_small = static_cast<uint32_t*>(s.small.p);
    B200_CUDA_TRY(cudaMemcpyAsync(d_small, small.data(), small.size() * 4, cudaMemcpyHostToDevice, sa));
    if (n) B200_CUDA_TRY(cudaMemcpyAsync(s.sigs.p, sigs, size_t(n) * 96, cudaMemcpyHostToDevice, sa));
    G2Jac* part = static_cast<G2Jac*>(s.agg_part.p);
    int32_t* part_code = reinterpret_cast<int32_t*>(part + n_chunks);
    uint32_t* done = reinterpret_cast<uint32_t*>(part_code + n_chunks);
    B200_CUDA_TRY(cudaMemsetAsync(done, 0, size_t(T) * 4, sa));
    int32_t* d_codes = static_cast<int32_t*>(s.out.p);
    uint8_t* d_out96 = static_cast<uint8_t*>(s.out.p) + size_t(T) * 4;
    B200_CUDA_TRY(cudaEventRecord(s.ev_k0, sa));
    launch_g2_sig_decode(static_cast<const uint8_t*>(s.sigs.p), n, static_cast<G2Aff*>(s.g2pts.p), static_cast<int32_t*>(s.sig_code.p), sa);
    launch_g2_aggregate(static_cast<const G2Aff*>(s.g2pts.p), static_cast<const int32_t*>(s.sig_code.p), d_small, d_small + 2 * T + 2,
                        d_small + T + 1, n_chunks, chunk, part, part_code, done, d_out96, d_codes, sa);
    e.launches += (n ? 1 : 0) + 1;
    B200_CUDA_TRY(cudaEventRecord(s.ev_k1, sa));
    B200_CUDA_TRY(cudaGetLastError());
    return aggregate_readback(e, s, d_codes, d_out96, T, 96, out96, out_codes);
}

// n keys, T groups by `off` (host): strict (`keys`: K1 over all n, then K2 over the call's points) or from the registry
// (`index`: K2 gathers the resident points and codes), then one compression thread per group.  Strict keys come from the
// host, or (`records`) from the Validator records rec_index[0 .. n) in HBM, packed into K1's staging buffer on the device.
static int32_t aggregate_keys(Engine& e, BlsState& s, bool registry, const uint8_t* keys, const uint32_t* index, uint32_t n,
                              const uint32_t* off, uint32_t T, uint8_t* out48, int32_t* out_codes,
                              const uint8_t* records = nullptr, const uint64_t* rec_index = nullptr) {
    const bool strict = !registry;
    const size_t n_small = size_t(T) + 1 + (registry ? n : 0);
    B200_CUDA_TRY(s.small.reserve(n_small * 4 + 64));
    B200_CUDA_TRY(s.g1pts.reserve(size_t(T) * sizeof(G1Aff) + 64));
    B200_CUDA_TRY(s.pk_code.reserve(size_t(T) * 4 + 64));
    B200_CUDA_TRY(s.flags.reserve(size_t(T) * 4 + 64));
    B200_CUDA_TRY(s.out.reserve(size_t(T) * (48 + 4) + 64));
    if (strict) {
        B200_CUDA_TRY(s.keys.reserve(size_t(n) * 48 + 64));
        B200_CUDA_TRY(s.key_aff.reserve((size_t(n) + 1) * sizeof(G1Aff)));
        B200_CUDA_TRY(s.key_code.reserve((size_t(n) + 1) * 4));
    }
    cudaStream_t sa = e.stream;
    uint32_t* d_off = static_cast<uint32_t*>(s.small.p);
    B200_CUDA_TRY(cudaMemcpyAsync(d_off, off, (size_t(T) + 1) * 4, cudaMemcpyHostToDevice, sa));
    if (registry && n) B200_CUDA_TRY(cudaMemcpyAsync(d_off + T + 1, index, size_t(n) * 4, cudaMemcpyHostToDevice, sa));
    if (strict && n && !records) B200_CUDA_TRY(cudaMemcpyAsync(s.keys.p, keys, size_t(n) * 48, cudaMemcpyHostToDevice, sa));
    int32_t* d_codes = static_cast<int32_t*>(s.out.p);
    uint8_t* d_out48 = static_cast<uint8_t*>(s.out.p) + size_t(T) * 4;
    B200_CUDA_TRY(cudaEventRecord(s.ev_k0, sa));
    if (records) {
        launch_gather_validator_keys(records, n, static_cast<uint8_t*>(s.keys.p), sa, rec_index);
        e.launches += n ? 1 : 0;
    }
    if (strict) {
        launch_g1_validate(static_cast<const uint8_t*>(s.keys.p), n, static_cast<G1Aff*>(s.key_aff.p), static_cast<int32_t*>(s.key_code.p), sa);
        e.launches += n ? 1 : 0;
    }
    launch_g1_aggregate(static_cast<const G1Aff*>(strict ? s.key_aff.p : s.reg_aff.p), static_cast<const int32_t*>(strict ? s.key_code.p : s.reg_code.p),
                        registry ? d_off + T + 1 : nullptr, d_off, T, static_cast<G1Aff*>(s.g1pts.p), nullptr,
                        static_cast<int32_t*>(s.pk_code.p), static_cast<uint32_t*>(s.flags.p), 0u, sa);
    launch_g1_compress_groups(static_cast<const G1Aff*>(s.g1pts.p), static_cast<const int32_t*>(s.pk_code.p),
                              static_cast<const uint32_t*>(s.flags.p), T, d_out48, d_codes, sa);
    e.launches += 2;
    B200_CUDA_TRY(cudaEventRecord(s.ev_k1, sa));
    B200_CUDA_TRY(cudaGetLastError());
    return aggregate_readback(e, s, d_codes, d_out48, T, 48, out48, out_codes);
}

// get_next_sync_committee's public keys and aggregate_pubkey (deneb/spec/mod.rs:2014-2060): the keys of Validator records
// index[0 .. n) (device) gathered in HBM, then eth_aggregate_public_keys' strict path over them.  keys48 (host) receives the
// n gathered keys, out48 the aggregate and *code its code.  The caller holds the engine lock.
int32_t aggregate_record_keys(const uint8_t* records, const uint64_t* index, uint32_t n, uint8_t* keys48, uint8_t out48[48],
                              int32_t* code) {
    Engine& e = engine();
    BlsState* s;
    int32_t rc = bls_state(e, &s);
    if (rc) return rc;
    const uint32_t off[2] = {0, n};
    rc = aggregate_keys(e, *s, false, nullptr, nullptr, n, off, 1, out48, code, records, index);
    if (rc) return rc;
    B200_CUDA_TRY(cudaMemcpy(keys48, s->keys.p, size_t(n) * 48, cudaMemcpyDeviceToHost));
    return B200_SUCCESS;
}

// ---- aggregate_verify over T tuples

// T + 1 offsets from 0, non-decreasing; *count: the last one
static int32_t check_offsets0(const uint32_t* off, size_t n, uint32_t* count) {
    if (off[0] != 0) return B200_ERR_BAD_ARG;
    return check_offsets(off, n, count);
}

// the checks of both aggregate_verify batch entry points (n_tuples > 0): key (or index) offsets, message groups, message
// byte offsets; *n_keys: keys (indices) of the call, *n_msgs: its messages
static int32_t check_aggregate_verify_args(Engine& e, const uint32_t* key_off, const uint8_t* msgs, const uint32_t* msg_offsets,
                                           const uint32_t* msg_group, const uint8_t* sigs, size_t n_tuples, const int32_t* out_codes,
                                           uint32_t* n_keys, uint32_t* n_msgs) {
    if (!key_off || !msg_offsets || !msg_group || !sigs || !out_codes || n_tuples > kMaxBatchTuples) return B200_ERR_BAD_ARG;
    int32_t rc;
    uint32_t n_bytes;
    if ((rc = check_offsets0(key_off, n_tuples, n_keys)) || (rc = check_offsets0(msg_group, n_tuples, n_msgs))) return rc;
    if (*n_keys > 0x3fffffffu || *n_msgs > 0x3fffffffu) { e.last_error = "aggregate_verify_batch: more than 0x3fffffff keys or messages"; return B200_ERR_BAD_ARG; }
    if ((rc = check_offsets0(msg_offsets, *n_msgs, &n_bytes))) return rc;   // n_msgs + 1 byte offsets
    if (n_bytes && !msgs) return B200_ERR_BAD_ARG;
    return B200_SUCCESS;
}

static void rlc_seed(const uint8_t* seed32, uint8_t out[32]) {
    if (seed32) { memcpy(out, seed32, 32); return; }
    std::random_device rd;   // the scalars must be unpredictable to whoever produced the signatures
    for (int i = 0; i < 8; i++) { const uint32_t v = rd(); memcpy(out + 4 * i, &v, 4); }
}

// the whole-batch entry points after their checks: `b` as one RLC check, scalars from the caller's seed (or one from the OS)
static int32_t verify_all(Engine& e, BlsState& s, Batch b, const uint8_t* seed32, uint64_t t0, bool exchange, int32_t* all_ok) {
    uint8_t seed[32];
    rlc_seed(seed32, seed);
    RlcReq req{seed, t0, exchange, 0};
    b.rlc = &req;
    const int32_t rc = run_verify(e, s, b, nullptr);
    if (rc) return rc;
    *all_ok = req.all_ok;
    return B200_SUCCESS;
}

}  // namespace b200

using namespace b200;

extern "C" {

// Knobs are the rows of kKnobs; an environment value takes the same rule as b200_tune's (see the header).
int32_t b200_tune(const char* knob, int64_t value) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    if (!knob) return B200_ERR_BAD_ARG;
    for (const Knob& k : kKnobs)
        if (strcmp(k.name, knob) == 0) { k.set(*s, value); return B200_SUCCESS; }
    return B200_ERR_BAD_ARG;
}

int32_t b200_vm_load_programs(const uint32_t* blob, size_t n_words) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    if (vm_load_programs(blob, n_words, e.stream) != 0) { e.last_error = "malformed pairing-VM program blob"; return B200_ERR_BAD_ARG; }
    return B200_SUCCESS;
}

float b200_last_dominant_kernel_ms(void) {
    Engine& e = engine();
    return e.bls ? static_cast<BlsState*>(e.bls)->last_dominant_ms : 0.f;
}

int32_t b200_fp_selftest(uint32_t n, uint32_t seed, uint32_t* mismatches) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!mismatches) return B200_ERR_BAD_ARG;
    uint32_t* d = nullptr;
    B200_CUDA_TRY(cudaMalloc(&d, 4));
    B200_CUDA_TRY(cudaMemsetAsync(d, 0, 4, e.stream));
    launch_fp_selftest(n, seed, d, e.stream);
    e.launches++;
    B200_CUDA_TRY(cudaGetLastError());
    B200_CUDA_TRY(cudaMemcpyAsync(mismatches, d, 4, cudaMemcpyDeviceToHost, e.stream));
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    cudaFree(d);
    return B200_SUCCESS;
}

int32_t b200_fp_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    const bool fp2 = op >= FP2_EVAL_MUL && op < FP2_EVAL_END;
    if (!(fp2 || (op >= 0 && op < FP_EVAL_N_OPS) || (op >= FPL_EVAL_SQRT_CHAIN && op < FPL_EVAL_END) ||
          (op >= FPD_EVAL_MUL && op < FPD_EVAL_END)) || n > (1u << 24))
        return B200_ERR_BAD_ARG;
    if (n == 0) return B200_SUCCESS;
    if (!a || !b || !out) return B200_ERR_BAD_ARG;
    const size_t in_bytes = size_t(n) * kFpEvalIn * 4, out_bytes = size_t(n) * kFpEvalOut * 4;
    uint32_t* d = nullptr;
    B200_CUDA_TRY(cudaMalloc(&d, 2 * in_bytes + out_bytes));
    uint32_t* da = d;
    uint32_t* db = d + size_t(n) * kFpEvalIn;
    uint32_t* dout = db + size_t(n) * kFpEvalIn;
    cudaMemcpyAsync(da, a, in_bytes, cudaMemcpyHostToDevice, e.stream);
    cudaMemcpyAsync(db, b, in_bytes, cudaMemcpyHostToDevice, e.stream);
    if (fp2) launch_fp2_eval(op, n, da, db, dout, e.stream);
    else launch_fp_eval(op, n, da, db, dout, e.stream);
    e.launches++;
    cudaError_t ce = cudaGetLastError();
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(out, dout, out_bytes, cudaMemcpyDeviceToHost, e.stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(e.stream);
    cudaFree(d);
    if (ce != cudaSuccess) { e.last_error = cudaGetErrorString(ce); return B200_ERR_CUDA; }
    return B200_SUCCESS;
}

int32_t b200_curve_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    const bool g2 = op >= CURVE_G2_ADD && op < CURVE_G2_END;
    if (!(g2 || (op >= 0 && op < CURVE_G1_N_OPS) || op == CURVE_G1L_DOUBLE || op == CURVE_G1_IN_SUBGROUP_ISO) || n > (1u << 24))
        return B200_ERR_BAD_ARG;
    if (n == 0) return B200_SUCCESS;
    if (!a || !b || !out) return B200_ERR_BAD_ARG;
    const size_t bytes = size_t(n) * kCurveEvalWords * 4;
    uint32_t* d = nullptr;
    B200_CUDA_TRY(cudaMalloc(&d, 3 * bytes));
    uint32_t* da = d;
    uint32_t* db = d + size_t(n) * kCurveEvalWords;
    uint32_t* dout = db + size_t(n) * kCurveEvalWords;
    cudaMemcpyAsync(da, a, bytes, cudaMemcpyHostToDevice, e.stream);
    cudaMemcpyAsync(db, b, bytes, cudaMemcpyHostToDevice, e.stream);
    if (g2) launch_curve2_eval(op, n, da, db, dout, e.stream);
    else launch_curve_eval(op, n, da, db, dout, e.stream);
    e.launches++;
    cudaError_t ce = cudaGetLastError();
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(out, dout, bytes, cudaMemcpyDeviceToHost, e.stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(e.stream);
    cudaFree(d);
    if (ce != cudaSuccess) { e.last_error = cudaGetErrorString(ce); return B200_ERR_CUDA; }
    return B200_SUCCESS;
}

// The one-thread ops run on the records themselves (bls_pairing.cu); the VM kernels and the folds take the engine's structs,
// packed here from the records' leading words, and run exactly as the batch paths launch them.
int32_t b200_pairing_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    const bool vm = op >= PAIRING_EVAL_VM_MILLER8 && op < PAIRING_EVAL_VM_END;
    const bool fold = op >= PAIRING_EVAL_FOLD_FP12 && op < PAIRING_EVAL_FOLD_END;
    if (!(vm || fold || (op >= 0 && op < PAIRING_EVAL_END)) || n > (1u << 24)) return B200_ERR_BAD_ARG;
    if (n == 0) return B200_SUCCESS;
    if (!a || !b || !out) return B200_ERR_BAD_ARG;
    if (op == PAIRING_EVAL_FOLD_SEGMENTS) {   // T segments over at most n values, two result records each
        uint32_t last;
        if (b[0] == 0 || 2 * size_t(b[0]) > n || check_offsets0(b + 1, b[0], &last) || last > n) return B200_ERR_BAD_ARG;
    }
    BlsState* s;
    if ((rc = bls_state(e, &s))) return rc;   // the VM's programs and constants
    constexpr size_t W = kPairingEvalWords;
    const size_t rec_bytes = size_t(n) * W * 4;
    cudaStream_t st = e.stream;
    std::vector<uint32_t> h_out(size_t(n) * W, 0);
    const int team = (op == PAIRING_EVAL_VM_MILLER16 || op == PAIRING_EVAL_VM_FINAL16) ? 16 : 8;
    // device scratch: records, or the structs and index arrays of the VM / fold launches
    uint8_t* d = nullptr;
    const size_t scratch = 3 * rec_bytes + size_t(n) * (sizeof(Fp12) * 3 + sizeof(G2Jac) + sizeof(G1Pre) + sizeof(G2Aff) + 12) + 4096;
    B200_CUDA_TRY(cudaMalloc(&d, scratch));
    auto carve = [&, off = size_t(0)](size_t bytes) mutable { uint8_t* p = d + off; off += (bytes + 255) & ~size_t(255); return p; };
    auto fp12_of = [&](const uint32_t* rec) { Fp12 v; memcpy(&v, rec, sizeof(Fp12)); return v; };
    auto put = [&](size_t i, const void* v, size_t bytes, uint32_t flag) {
        memcpy(&h_out[i * W], v, bytes);
        h_out[i * W + 144] = flag;
    };
    static_assert(sizeof(Fp12) == 144 * 4 && sizeof(G2Jac) == 72 * 4, "records hold the structs' words in order");
    cudaError_t ce = cudaSuccess;
    if (!vm && !fold) {
        uint32_t* da = reinterpret_cast<uint32_t*>(carve(rec_bytes));
        uint32_t* db = reinterpret_cast<uint32_t*>(carve(rec_bytes));
        uint32_t* dout = reinterpret_cast<uint32_t*>(carve(rec_bytes));
        cudaMemcpyAsync(da, a, rec_bytes, cudaMemcpyHostToDevice, st);
        cudaMemcpyAsync(db, b, rec_bytes, cudaMemcpyHostToDevice, st);
        launch_pairing_eval(op, n, da, db, dout, st);
        e.launches++;
        ce = cudaGetLastError();
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(h_out.data(), dout, rec_bytes, cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    } else if (op == PAIRING_EVAL_VM_MILLER8 || op == PAIRING_EVAL_VM_MILLER16) {
        std::vector<G1Pre> g1(n);
        std::vector<G2Aff> g2(n);
        std::vector<uint32_t> idx(n);
        for (uint32_t i = 0; i < n; i++) {
            memcpy(&g1[i], a + i * W, 3 * sizeof(Fp)); g1[i].inf = a[i * W + 144];
            memcpy(&g2[i], b + i * W, 2 * sizeof(Fp2)); g2[i].inf = b[i * W + 144];
            idx[i] = i;
        }
        G1Pre* dg1 = reinterpret_cast<G1Pre*>(carve(n * sizeof(G1Pre)));
        G2Aff* dg2 = reinterpret_cast<G2Aff*>(carve(n * sizeof(G2Aff)));
        uint32_t* didx = reinterpret_cast<uint32_t*>(carve(n * 4));
        uint32_t* dzero = reinterpret_cast<uint32_t*>(carve(n * 4));
        Fp12* df = reinterpret_cast<Fp12*>(carve(n * sizeof(Fp12)));
        std::vector<Fp12> f(n);
        cudaMemcpyAsync(dg1, g1.data(), n * sizeof(G1Pre), cudaMemcpyHostToDevice, st);
        cudaMemcpyAsync(dg2, g2.data(), n * sizeof(G2Aff), cudaMemcpyHostToDevice, st);
        cudaMemcpyAsync(didx, idx.data(), n * 4, cudaMemcpyHostToDevice, st);
        cudaMemsetAsync(dzero, 0, n * 4, st);
        launch_vm_miller_team(team, dg1, didx, dg2, dzero, n, df, st);
        e.launches++;
        ce = cudaGetLastError();
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(f.data(), df, n * sizeof(Fp12), cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
        for (uint32_t i = 0; i < n; i++) put(i, &f[i], sizeof(Fp12), 0);
    } else if (vm) {   // VM final: f0 from a, f1 from b -> one tuple each
        std::vector<Fp12> f(2 * size_t(n));
        std::vector<uint32_t> off(n);
        for (uint32_t i = 0; i < n; i++) { f[2 * i] = fp12_of(a + i * W); f[2 * i + 1] = fp12_of(b + i * W); off[i] = 2 * i; }
        Fp12* df = reinterpret_cast<Fp12*>(carve(2 * n * sizeof(Fp12)));
        Fp12* dfo = reinterpret_cast<Fp12*>(carve(n * sizeof(Fp12)));
        uint32_t* doff = reinterpret_cast<uint32_t*>(carve(n * 4));
        uint32_t* dzero = reinterpret_cast<uint32_t*>(carve(n * 4));
        int32_t* dcodes = reinterpret_cast<int32_t*>(carve(n * 4));
        std::vector<Fp12> fo(n);
        std::vector<int32_t> codes(n);
        cudaMemcpyAsync(df, f.data(), 2 * n * sizeof(Fp12), cudaMemcpyHostToDevice, st);
        cudaMemcpyAsync(doff, off.data(), n * 4, cudaMemcpyHostToDevice, st);
        cudaMemsetAsync(dzero, 0, n * 4, st);
        launch_vm_final_team(team, df, doff, dzero, n, dfo, dcodes, st);
        e.launches++;
        ce = cudaGetLastError();
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(fo.data(), dfo, n * sizeof(Fp12), cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(codes.data(), dcodes, n * 4, cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
        for (uint32_t i = 0; i < n; i++) put(i, &fo[i], sizeof(Fp12), codes[i] == BLS_SUCCESS ? 1u : 0u);
    } else if (op == PAIRING_EVAL_FOLD_FP12) {   // the product of the n values of a, through rlc_tail's fold
        std::vector<Fp12> f(n);
        for (uint32_t i = 0; i < n; i++) f[i] = fp12_of(a + i * W);
        Fp12* df = reinterpret_cast<Fp12*>(carve(n * sizeof(Fp12)));
        Fp12* buf[2] = {reinterpret_cast<Fp12*>(carve(n * sizeof(Fp12))), reinterpret_cast<Fp12*>(carve(n * sizeof(Fp12)))};
        cudaMemcpyAsync(df, f.data(), n * sizeof(Fp12), cudaMemcpyHostToDevice, st);
        int pp = 0;
        const Fp12* r = rlc_fold(e, static_cast<const Fp12*>(df), n, buf, pp, st);
        Fp12 v;
        ce = cudaGetLastError();
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(&v, r, sizeof(Fp12), cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
        put(0, &v, sizeof(Fp12), 0);
    } else if (op == PAIRING_EVAL_FOLD_SEGMENTS) {   // the aggregate_verify batches' levels, from the values of a
        const uint32_t T = b[0];
        std::vector<uint32_t> words(b + 1, b + 2 + T);
        const std::vector<FoldLevel> lv = plan_fold(words, 0, T, kFinalLevel, false);
        std::vector<Fp12> f(n);
        for (uint32_t i = 0; i < n; i++) f[i] = fp12_of(a + i * W);
        Fp12* df = reinterpret_cast<Fp12*>(carve(n * sizeof(Fp12)));
        Fp12* buf[2] = {reinterpret_cast<Fp12*>(carve(n * sizeof(Fp12))), reinterpret_cast<Fp12*>(carve(n * sizeof(Fp12)))};
        uint32_t* dw = reinterpret_cast<uint32_t*>(carve(words.size() * 4));
        cudaMemcpyAsync(df, f.data(), n * sizeof(Fp12), cudaMemcpyHostToDevice, st);
        cudaMemcpyAsync(dw, words.data(), words.size() * 4, cudaMemcpyHostToDevice, st);
        const Fp12* in = df;
        for (size_t k = 0; k < lv.size(); k++) {
            const FoldLevel& l = lv[k];
            if (l.o_out == kFinalLevel) cudaMemsetAsync(buf[k & 1], 0, 2 * size_t(T) * sizeof(Fp12), st);   // empty segments: zero
            launch_fold_segments(in, l.n_in, dw + l.o_map, dw + l.o_in, l.o_out == kFinalLevel ? nullptr : dw + l.o_out, nullptr, nullptr,
                                 nullptr, buf[k & 1], st);
            if (l.n_in) e.launches++;
            in = buf[k & 1];
        }
        std::vector<Fp12> fo(2 * size_t(T));
        ce = cudaGetLastError();
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(fo.data(), in, 2 * size_t(T) * sizeof(Fp12), cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
        for (uint32_t i = 0; i < 2 * T; i++) put(i, &fo[i], sizeof(Fp12), 0);
    } else {   // the sum of the n Jacobian points of a, through rlc_tail's fold and k_rlc_finish
        std::vector<G2Jac> q(n);
        for (uint32_t i = 0; i < n; i++) memcpy(&q[i], a + i * W, sizeof(G2Jac));
        G2Jac* dq = reinterpret_cast<G2Jac*>(carve(n * sizeof(G2Jac)));
        G2Jac* buf[2] = {reinterpret_cast<G2Jac*>(carve(n * sizeof(G2Jac))), reinterpret_cast<G2Jac*>(carve(n * sizeof(G2Jac)))};
        G2Aff* daff = reinterpret_cast<G2Aff*>(carve(sizeof(G2Aff)));
        cudaMemcpyAsync(dq, q.data(), n * sizeof(G2Jac), cudaMemcpyHostToDevice, st);
        int pp = 0;
        launch_rlc_finish(rlc_fold(e, static_cast<const G2Jac*>(dq), n, buf, pp, st), daff, st);
        e.launches++;
        G2Aff v;
        ce = cudaGetLastError();
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(&v, daff, sizeof(G2Aff), cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
        put(0, &v, 2 * sizeof(Fp2), v.inf);
    }
    cudaFree(d);
    if (ce != cudaSuccess) { e.last_error = cudaGetErrorString(ce); return B200_ERR_CUDA; }
    memcpy(out, h_out.data(), rec_bytes);
    return B200_SUCCESS;
}

int32_t b200_fast_aggregate_verify_batch(const uint8_t* pks_flat, const uint32_t* pk_offsets, const uint8_t* msgs32,
                                         const uint8_t* sigs, size_t n_tuples, int32_t* out_codes) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (n_tuples == 0) return B200_SUCCESS;
    if (!pk_offsets || !msgs32 || !sigs || !out_codes || n_tuples > kMaxBatchTuples) return B200_ERR_BAD_ARG;
    uint32_t nk;
    if ((rc = check_offsets(pk_offsets, n_tuples, &nk))) return rc;
    if (nk && !pks_flat) return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    const std::vector<uint32_t> moff = msg32_offsets(n_tuples);
    return run_verify(e, *s, {.keys = pks_flat, .n_keys = nk, .key_off = pk_offsets, .msgs = msgs32, .msg_off = moff.data(),
                              .n_msgs = uint32_t(n_tuples), .sigs = sigs, .T = uint32_t(n_tuples)}, out_codes);
}

// BASELINE configs[4]: the batch sharded over the communicator's ranks; verdicts exchanged with one ncclAllGather.
int32_t b200_fast_aggregate_verify_batch_sharded(const uint8_t* pks_flat, const uint32_t* pk_offsets, const uint8_t* msgs32,
                                                 const uint8_t* sigs, size_t n_tuples, int32_t* out_codes) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    const Comm& c = comm();
    if (!c.ready) { e.last_error = "b200_comm_init has not been called"; return B200_ERR_NOT_INITIALIZED; }
    if (n_tuples == 0) return B200_SUCCESS;
    if (!pk_offsets || !msgs32 || !sigs || !out_codes || n_tuples > kMaxBatchTuples) return B200_ERR_BAD_ARG;
    uint32_t nk;
    if ((rc = check_offsets(pk_offsets, n_tuples, &nk))) return rc;
    if (nk && !pks_flat) return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    const size_t world = size_t(c.world);
    const TupleRange mine = tuple_shard(n_tuples, world, size_t(c.rank));
    const size_t per = (n_tuples + world - 1) / world;  // padded shard length: equal contributions to the all-gather
    B200_CUDA_TRY(s->out.reserve((per + 1) * 4));
    B200_CUDA_TRY(s->gath.reserve(world * per * 4 + 16));
    if (mine.cnt) {
        std::vector<uint32_t> koff, moff;
        std::vector<int32_t> local(mine.cnt);
        rc = run_verify(e, *s, shard_batch(pks_flat, pk_offsets, msgs32, sigs, mine, koff, moff), local.data());
        if (rc) return rc;
    }
    cudaStream_t sa = e.stream;
    int32_t* d_out = static_cast<int32_t*>(s->out.p);
    if (per > mine.cnt) B200_CUDA_TRY(cudaMemsetAsync(d_out + mine.cnt, 0xff, (per - mine.cnt) * 4, sa));
    rc = comm_all_gather(e, d_out, s->gath.p, per * 4, sa);   // the path's one exchange step
    if (rc) return rc;
    B200_CUDA_TRY(s->stage.reserve(world * per * 4 + 64));
    B200_CUDA_TRY(cudaMemcpyAsync(s->stage.p, s->gath.p, world * per * 4, cudaMemcpyDeviceToHost, sa));
    B200_CUDA_TRY(cudaStreamSynchronize(sa));
    const int32_t* h = static_cast<const int32_t*>(s->stage.p);
    for (size_t r = 0; r < world; r++) {
        const TupleRange theirs = tuple_shard(n_tuples, world, r);
        memcpy(out_codes + theirs.lo, h + r * per, theirs.cnt * 4);
    }
    return B200_SUCCESS;
}

// ---- RLC whole-batch entry points (bls_rlc.cu) --------------------------------------------------------------------
int32_t b200_fast_aggregate_verify_batch_all(const uint8_t* pks_flat, const uint32_t* pk_offsets, const uint8_t* msgs32,
                                             const uint8_t* sigs, size_t n_tuples, const uint8_t* seed32, int32_t* all_ok) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!all_ok) return B200_ERR_BAD_ARG;
    if (n_tuples == 0) { *all_ok = 1; return B200_SUCCESS; }
    if (!pk_offsets || !msgs32 || !sigs || n_tuples > kMaxBatchTuples) return B200_ERR_BAD_ARG;
    uint32_t nk;
    if ((rc = check_offsets(pk_offsets, n_tuples, &nk))) return rc;
    if (nk && !pks_flat) return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    const std::vector<uint32_t> moff = msg32_offsets(n_tuples);
    return verify_all(e, *s, {.keys = pks_flat, .n_keys = nk, .key_off = pk_offsets, .msgs = msgs32, .msg_off = moff.data(),
                              .n_msgs = uint32_t(n_tuples), .sigs = sigs, .T = uint32_t(n_tuples)}, seed32, 0, false, all_ok);
}

int32_t b200_fast_aggregate_verify_batch_indexed_all(const uint32_t* indices, const uint32_t* offsets, const uint8_t* msgs32,
                                                     const uint8_t* sigs, size_t n_tuples, const uint8_t* seed32, int32_t* all_ok) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!all_ok) return B200_ERR_BAD_ARG;
    if (n_tuples == 0) { *all_ok = 1; return B200_SUCCESS; }
    if (!offsets || !msgs32 || !sigs || n_tuples > kMaxBatchTuples) return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    uint32_t ni;
    if ((rc = check_offsets(offsets, n_tuples, &ni))) return rc;
    if (ni && !indices) return B200_ERR_BAD_ARG;
    if ((rc = check_indices(e, *s, indices, ni, 0))) return rc;
    const std::vector<uint32_t> moff = msg32_offsets(n_tuples);
    static const uint32_t dummy = 0;
    return verify_all(e, *s, {.index = indices ? indices : &dummy, .n_index = ni, .key_off = offsets, .msgs = msgs32, .msg_off = moff.data(),
                              .n_msgs = uint32_t(n_tuples), .sigs = sigs, .T = uint32_t(n_tuples)}, seed32, 0, false, all_ok);
}

// every rank passes the same batch AND the same seed; each verifies its block, the Gt partials and bad flags are
// all-gathered and every rank finishes the same single final exponentiation
int32_t b200_fast_aggregate_verify_batch_all_sharded(const uint8_t* pks_flat, const uint32_t* pk_offsets, const uint8_t* msgs32,
                                                     const uint8_t* sigs, size_t n_tuples, const uint8_t seed32[32], int32_t* all_ok) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    const Comm& c = comm();
    if (!c.ready) { e.last_error = "b200_comm_init has not been called"; return B200_ERR_NOT_INITIALIZED; }
    if (!all_ok || !seed32) return B200_ERR_BAD_ARG;   // the ranks must agree on the scalars: the caller supplies the seed
    if (n_tuples == 0) { *all_ok = 1; return B200_SUCCESS; }
    if (!pk_offsets || !msgs32 || !sigs || n_tuples > kMaxBatchTuples) return B200_ERR_BAD_ARG;
    if (n_tuples < size_t(c.world)) { e.last_error = "fewer tuples than ranks"; return B200_ERR_BAD_ARG; }
    uint32_t nk;
    if ((rc = check_offsets(pk_offsets, n_tuples, &nk))) return rc;
    if (nk && !pks_flat) return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    const TupleRange mine = tuple_shard(n_tuples, size_t(c.world), size_t(c.rank));
    std::vector<uint32_t> koff, moff;
    return verify_all(e, *s, shard_batch(pks_flat, pk_offsets, msgs32, sigs, mine, koff, moff), seed32, uint64_t(mine.lo), true, all_ok);
}

int32_t b200_registry_load(const uint8_t* pks_flat, size_t n) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if ((!pks_flat && n) || n > 0x7fffffffu) return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    return registry_fill(e, *s, 0, pks_flat, nullptr, n);
}

int32_t b200_registry_append(const uint8_t* pks_flat, size_t n) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (!pks_flat && n) return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    if (n > 0x7fffffffu - s->reg_n) { e.last_error = "registry_append: more than 2^31 - 1 keys"; return B200_ERR_BAD_ARG; }
    if (n == 0) { e.last_kernel_ms = 0.f; return B200_SUCCESS; }
    return registry_fill(e, *s, s->reg_n, pks_flat, nullptr, n);
}

int32_t b200_registry_load_state(b200_state* h) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    const uint8_t* records;
    uint64_t n;
    if ((rc = registry_state_records(e, h, &records, &n))) return rc;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    return registry_fill(e, *s, 0, nullptr, records, size_t(n));
}

int32_t b200_registry_sync_state(b200_state* h) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    const uint8_t* records;
    uint64_t n;
    if ((rc = registry_state_records(e, h, &records, &n))) return rc;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    if (n < s->reg_n) { e.last_error = "registry_sync_state: the state has fewer validators than the registry"; return B200_ERR_BAD_ARG; }
    if (n == s->reg_n) { e.last_kernel_ms = 0.f; return B200_SUCCESS; }
    return registry_fill(e, *s, s->reg_n, nullptr, records + s->reg_n * 121, size_t(n) - s->reg_n);
}

int32_t b200_registry_key_codes(int32_t* out_codes, size_t n) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    if (!out_codes || n > s->reg_n) return B200_ERR_BAD_ARG;
    if (n) B200_CUDA_TRY(cudaMemcpy(out_codes, s->reg_code.p, n * 4, cudaMemcpyDeviceToHost));
    return B200_SUCCESS;
}

static int32_t verify_batch_indexed(const uint8_t* extra_pks, size_t n_extra, const uint32_t* indices, const uint32_t* offsets,
                                    const uint8_t* msgs32, const uint8_t* sigs, size_t n_tuples, int32_t* out_codes) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (n_tuples == 0) return B200_SUCCESS;
    if (!offsets || !msgs32 || !sigs || !out_codes || n_tuples > kMaxBatchTuples) return B200_ERR_BAD_ARG;
    if ((n_extra && !extra_pks) || n_extra > kRegistryExtraKeys) return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    if (n_extra && !s->reg_aff.p) { e.last_error = "no registry loaded"; return B200_ERR_BAD_ARG; }
    uint32_t ni;
    if ((rc = check_offsets(offsets, n_tuples, &ni))) return rc;
    if (ni && !indices) return B200_ERR_BAD_ARG;
    if ((rc = check_indices(e, *s, indices, ni, n_extra))) return rc;
    const std::vector<uint32_t> moff = msg32_offsets(n_tuples);
    static const uint32_t dummy = 0;
    return run_verify(e, *s, {.keys = n_extra ? extra_pks : nullptr, .n_keys = uint32_t(n_extra), .index = indices ? indices : &dummy,
                              .n_index = ni, .key_off = offsets, .msgs = msgs32, .msg_off = moff.data(), .n_msgs = uint32_t(n_tuples),
                              .sigs = sigs, .T = uint32_t(n_tuples)}, out_codes);
}

int32_t b200_fast_aggregate_verify_batch_indexed(const uint32_t* indices, const uint32_t* offsets, const uint8_t* msgs32,
                                                 const uint8_t* sigs, size_t n_tuples, int32_t* out_codes) {
    return verify_batch_indexed(nullptr, 0, indices, offsets, msgs32, sigs, n_tuples, out_codes);
}

int32_t b200_fast_aggregate_verify_batch_mixed(const uint8_t* extra_pks, size_t n_extra, const uint32_t* indices,
                                               const uint32_t* offsets, const uint8_t* msgs32, const uint8_t* sigs,
                                               size_t n_tuples, int32_t* out_codes) {
    return verify_batch_indexed(extra_pks, n_extra, indices, offsets, msgs32, sigs, n_tuples, out_codes);
}

// crypto/bls.rs:114-132 — `public_keys: &[&PublicKey]` is an array of pointers into the validator registry
int32_t b200_fast_aggregate_verify(const uint8_t* const* pks, size_t k, const uint8_t* msg, size_t msg_len,
                                   const uint8_t sig[96]) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if ((!pks && k) || (!msg && msg_len) || !sig || k > 0x7fffffffu || msg_len > 0x7fffffffu) return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    std::vector<uint8_t> flat(k * 48);
    for (size_t i = 0; i < k; i++) memcpy(flat.data() + 48 * i, pks[i], 48);
    const uint32_t koff[2] = {0, uint32_t(k)}, moff[2] = {0, uint32_t(msg_len)};
    int32_t code = B200_ERR_CUDA;
    rc = run_verify(e, *s, {.keys = flat.data(), .n_keys = uint32_t(k), .key_off = koff, .msgs = msg, .msg_off = moff, .n_msgs = 1,
                            .sigs = sig, .T = 1}, &code);
    return rc ? rc : code;
}

// crypto/bls.rs:150-160
int32_t b200_eth_fast_aggregate_verify(const uint8_t* const* pks, size_t k, const uint8_t* msg, size_t msg_len,
                                       const uint8_t sig[96]) {
    if (k == 0 && sig) {
        bool inf = sig[0] == 0xc0;
        for (int i = 1; i < 96 && inf; i++) inf = sig[i] == 0;
        if (inf) return B200_SUCCESS;  // G2_POINT_AT_INFINITY with no participants (byte comparison, bls.rs:343-347)
    }
    return b200_fast_aggregate_verify(pks, k, msg, msg_len, sig);
}

// crypto/bls.rs:64-77
int32_t b200_verify_signature(const uint8_t pk[48], const uint8_t* msg, size_t msg_len, const uint8_t sig[96]) {
    if (!pk) return B200_ERR_BAD_ARG;
    const uint8_t* one[1] = {pk};
    return b200_fast_aggregate_verify(one, 1, msg, msg_len, sig);
}

// crypto/bls.rs:95-112
int32_t b200_aggregate_verify(const uint8_t* pks_flat, size_t n_pks, const uint8_t* const* msgs, const size_t* msg_lens,
                              size_t n_msgs, const uint8_t sig[96]) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if ((!pks_flat && n_pks) || ((!msgs || !msg_lens) && n_msgs) || !sig || n_pks > 0x3fffffffu || n_msgs > 0x3fffffffu)
        return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    const bool shape_fail = (n_pks == 0 || n_pks != n_msgs);
    std::vector<uint32_t> moff(1, 0);
    std::vector<uint8_t> flat;
    if (!shape_fail) {
        size_t total = 0;
        for (size_t i = 0; i < n_msgs; i++) {
            if (msg_lens[i] > 0xffffffffu - total) { e.last_error = "aggregate_verify: messages exceed 4 GiB in total"; return B200_ERR_BAD_ARG; }
            total += msg_lens[i];
        }
        for (size_t i = 0; i < n_msgs; i++) {
            flat.insert(flat.end(), msgs[i], msgs[i] + msg_lens[i]);
            moff.push_back(uint32_t(flat.size()));
        }
    }
    // a batch of one tuple; with a bad shape it has no messages, so av_shape_ok flags it EMPTY
    const uint32_t key_off[2] = {0, uint32_t(n_pks)}, msg_group[2] = {0, uint32_t(moff.size() - 1)};
    int32_t code = B200_ERR_CUDA;
    rc = run_verify(e, *s, {.mode = MODE_AGGREGATE_BATCH, .keys = pks_flat, .n_keys = uint32_t(n_pks), .key_off = key_off, .msgs = flat.data(),
                            .msg_off = moff.data(), .n_msgs = msg_group[1], .msg_group = msg_group, .sigs = sig, .T = 1}, &code);
    return rc ? rc : code;
}

// crypto/bls.rs:95-112 over T tuples: the same codes as T calls of b200_aggregate_verify
int32_t b200_aggregate_verify_batch(const uint8_t* pks_flat, const uint32_t* pk_offsets, const uint8_t* msgs, const uint32_t* msg_offsets,
                                    const uint32_t* msg_group, const uint8_t* sigs, size_t n_tuples, int32_t* out_codes) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (n_tuples == 0) return B200_SUCCESS;
    uint32_t nk, nm;
    if ((rc = check_aggregate_verify_args(e, pk_offsets, msgs, msg_offsets, msg_group, sigs, n_tuples, out_codes, &nk, &nm))) return rc;
    if (nk && !pks_flat) return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    return run_verify(e, *s, {.mode = MODE_AGGREGATE_BATCH, .keys = pks_flat, .n_keys = nk, .key_off = pk_offsets, .msgs = msgs,
                              .msg_off = msg_offsets, .n_msgs = nm, .msg_group = msg_group, .sigs = sigs, .T = uint32_t(n_tuples)},
                      out_codes);
}

int32_t b200_aggregate_verify_batch_indexed(const uint32_t* indices, const uint32_t* offsets, const uint8_t* msgs,
                                            const uint32_t* msg_offsets, const uint32_t* msg_group, const uint8_t* sigs,
                                            size_t n_tuples, int32_t* out_codes) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    if (n_tuples == 0) return B200_SUCCESS;
    uint32_t ni, nm;
    if ((rc = check_aggregate_verify_args(e, offsets, msgs, msg_offsets, msg_group, sigs, n_tuples, out_codes, &ni, &nm))) return rc;
    if (ni && !indices) return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    if (!s->reg_aff.p) { e.last_error = "no registry loaded"; return B200_ERR_BAD_ARG; }
    if ((rc = check_indices(e, *s, indices, ni, 0))) return rc;
    static const uint32_t dummy = 0;
    return run_verify(e, *s, {.mode = MODE_AGGREGATE_BATCH, .index = indices ? indices : &dummy, .n_index = ni, .key_off = offsets,
                              .msgs = msgs, .msg_off = msg_offsets, .n_msgs = nm, .msg_group = msg_group, .sigs = sigs,
                              .T = uint32_t(n_tuples)}, out_codes);
}

// crypto/bls.rs:79-93: the batch path with one group
int32_t b200_aggregate(const uint8_t* sigs_flat, size_t n, uint8_t out[96]) {
    if (n == 0) {
        Engine& e = engine();
        Guard g(e);
        const int32_t rc = check_ready(e);
        return rc ? rc : B200_EMPTY_AGGREGATE;
    }
    if (!sigs_flat || !out || n > 0x3fffffffu) return B200_ERR_BAD_ARG;
    const uint32_t off[2] = {0, uint32_t(n)};
    uint8_t agg[96];
    int32_t code = B200_ERR_CUDA;
    const int32_t rc = b200_aggregate_batch(sigs_flat, off, 1, agg, &code);
    if (rc) return rc;
    if (code == B200_SUCCESS) memcpy(out, agg, 96);
    return code;
}

// crypto/bls.rs:135-148: the batch path with one group
int32_t b200_eth_aggregate_public_keys(const uint8_t* pks_flat, size_t n, uint8_t out[48]) {
    if (n == 0) {
        Engine& e = engine();
        Guard g(e);
        const int32_t rc = check_ready(e);
        return rc ? rc : B200_EMPTY_AGGREGATE;
    }
    if (!pks_flat || !out || n > 0x3fffffffu) return B200_ERR_BAD_ARG;
    const uint32_t off[2] = {0, uint32_t(n)};
    uint8_t agg[48];
    int32_t code = B200_ERR_CUDA;
    const int32_t rc = b200_eth_aggregate_public_keys_batch(pks_flat, off, 1, agg, &code);
    if (rc) return rc;
    if (code == B200_SUCCESS) memcpy(out, agg, 48);
    return code;
}

int32_t b200_aggregate_batch(const uint8_t* sigs_flat, const uint32_t* offsets, size_t n_groups, uint8_t* out96, int32_t* out_codes) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    uint32_t n;
    if ((rc = check_aggregate_args(e, offsets, n_groups, out96, out_codes, &n))) return rc;
    if (n_groups == 0) return B200_SUCCESS;
    if (n && !sigs_flat) return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    return aggregate_sigs(e, *s, sigs_flat, n, offsets, uint32_t(n_groups), out96, out_codes);
}

int32_t b200_eth_aggregate_public_keys_batch(const uint8_t* pks_flat, const uint32_t* offsets, size_t n_groups, uint8_t* out48,
                                             int32_t* out_codes) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    uint32_t n;
    if ((rc = check_aggregate_args(e, offsets, n_groups, out48, out_codes, &n))) return rc;
    if (n_groups == 0) return B200_SUCCESS;
    if (n && !pks_flat) return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    return aggregate_keys(e, *s, false, pks_flat, nullptr, n, offsets, uint32_t(n_groups), out48, out_codes);
}

int32_t b200_registry_aggregate_public_keys(const uint32_t* indices, const uint32_t* offsets, size_t n_groups, uint8_t* out48,
                                            int32_t* out_codes) {
    Engine& e = engine();
    Guard g(e);
    int32_t rc = check_ready(e);
    if (rc) return rc;
    uint32_t n;
    if ((rc = check_aggregate_args(e, offsets, n_groups, out48, out_codes, &n))) return rc;
    if (n_groups == 0) return B200_SUCCESS;
    if (n && !indices) return B200_ERR_BAD_ARG;
    BlsState* s;
    rc = bls_state(e, &s);
    if (rc) return rc;
    if ((rc = check_indices(e, *s, indices, n, 0))) return rc;
    return aggregate_keys(e, *s, true, nullptr, indices, n, offsets, uint32_t(n_groups), out48, out_codes);
}

}  // extern "C"
