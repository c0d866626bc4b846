// Host planner + executor for device-side SSZ hash_tree_root (see ssz_plan.h).
#include "ssz_plan.h"
#include "comm.h"

#include <cstdlib>

#include <algorithm>

namespace b200 {

static constexpr uint32_t kSmallBase = 65;
static constexpr uint32_t kSmallCap = 8192;

// smallest d with 2^d >= n; n above 2^63 saturates at 64 (the zero-subtree table has 65 levels, 0..64) — the shift
// below never reaches 64, so an absurd caller-supplied limit can neither invoke undefined behaviour nor spin.
int depth_for(uint64_t n) {
    int d = 0;
    while (d < 64 && (uint64_t(1) << d) < n) d++;
    return d;
}

static inline uint32_t be32(const uint8_t* p) {
    return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | p[3];
}

// ------------------------------------------------------------------------------------------------ building
uint32_t SszPlan::leaf(const uint8_t chunk[32]) {
    uint32_t i = uint32_t(small_words_.size() / 8);
    for (int k = 0; k < 8; k++) small_words_.push_back(be32(chunk + 4 * k));
    return kSmallBase + i;
}
uint32_t SszPlan::leaf_u64(uint64_t v) {
    uint8_t c[32] = {0};
    for (int i = 0; i < 8; i++) c[i] = uint8_t(v >> (8 * i));
    return leaf(c);
}
uint32_t SszPlan::leaf_bytes(const uint8_t* p, size_t n) {
    uint8_t c[32] = {0};
    memcpy(c, p, n > 32 ? 32 : n);
    return leaf(c);
}
int SszPlan::ready_wave(uint32_t idx) const {
    auto it = ready_.find(idx);
    return it == ready_.end() ? 0 : it->second;
}
uint32_t SszPlan::hash2(uint32_t a, uint32_t b) {
    uint32_t dst = uint32_t(arena_alloc(1));
    int w = std::max(ready_wave(a), ready_wave(b));
    ops_.push_back(FinOp{a, b, dst, FIN_HASH});
    op_wave_.push_back(w);
    ready_[dst] = w + 1;
    return dst;
}
uint32_t SszPlan::exchange(const std::vector<uint32_t>& local, int world) {
    xch_n_ = uint32_t(local.size());
    xch_world_ = world;
    xch_send_ = uint32_t(arena_alloc(xch_n_));
    xch_recv_ = uint32_t(arena_alloc(uint64_t(xch_n_) * uint64_t(world)));
    for (uint32_t i = 0; i < xch_n_; i++) {   // gather the local nodes into the contiguous send region
        const int w = ready_wave(local[i]);
        ops_.push_back(FinOp{local[i], local[i], xch_send_ + i, FIN_COPY});
        op_wave_.push_back(w);
    }
    for (uint32_t i = 0; i < xch_n_ * uint32_t(world); i++) ready_[xch_recv_ + i] = kRemoteWave;
    return xch_recv_;
}
uint32_t SszPlan::merkle_small(std::vector<uint32_t> nodes, int level, int depth_target) {
    if (nodes.empty()) return zero(depth_target);
    while (level < depth_target) {
        if (nodes.size() & 1) nodes.push_back(zero(level));
        std::vector<uint32_t> up(nodes.size() / 2);
        for (size_t i = 0; i < up.size(); i++) up[i] = hash2(nodes[2 * i], nodes[2 * i + 1]);
        nodes.swap(up);
        level++;
    }
    return nodes[0];
}
uint32_t SszPlan::container(const std::vector<uint32_t>& field_roots) {
    return merkle_small(field_roots, 0, depth_for(field_roots.size()));
}
uint64_t SszPlan::stage_field(const uint8_t* src, size_t nbytes) {
    uint64_t off = (field_next_ + 255) & ~uint64_t(255);
    size_t padded = ((nbytes + 31) & ~size_t(31)) + 32;
    field_next_ = off + padded;
    if (nbytes) {
        copies_.push_back(HostCopy{src, nbytes, off, padded - nbytes, false, cur_chain_});
        if (cur_chain_ >= 0) chains_[size_t(cur_chain_)].copy = int(copies_.size()) - 1;
    }
    return off;
}
void SszPlan::add_job(size_t stage, const PJob& j) {
    if (stages_.size() <= stage) stages_.resize(stage + 1);
    stages_[stage].push_back(j);
    stages_[stage].back().chain = cur_chain_;
    stages_[stage].back().copy = cur_copy_;
    if (cur_chain_ >= 0) chains_[size_t(cur_chain_)].jobs.emplace_back(int(stage), stages_[stage].size() - 1);
}
int SszPlan::copy_of(uint64_t field_off) const {
    for (size_t i = 0; i < copies_.size(); i++)
        if (copies_[i].field_off == field_off) return int(i);
    return -1;
}
bool SszPlan::chain_field(int c, uint64_t* field_off, size_t* nbytes) const {
    if (c < 0 || size_t(c) >= chains_.size() || chains_[size_t(c)].copy < 0) return false;
    const HostCopy& hc = copies_[size_t(chains_[size_t(c)].copy)];
    *field_off = hc.field_off; *nbytes = hc.nbytes;
    return true;
}

uint32_t SszPlan::wide_nodes(PSrc src, bool raw, uint64_t n, int level, int depth_target, size_t s) {
    if (n == 0) return zero(depth_target);
    while (n > kHandoff && level < depth_target) {
        uint32_t nlev = uint32_t(std::min(3, depth_target - level));
        uint64_t n_out = (n + (uint64_t(1) << nlev) - 1) >> nlev;
        PJob j;
        j.type = JOB_REDUCE; j.src = src; j.dst = arena_alloc(n_out); j.n_in = n;
        j.level = uint32_t(level); j.nlev = nlev; j.raw = raw ? 1 : 0;
        add_job(s++, j);
        src.in_arena = true; src.off = j.dst; raw = false;
        n = n_out; level += int(nlev);
    }
    if (!src.in_arena) {  // small raw input: convert to word form on the device
        PJob j;
        j.type = JOB_REDUCE; j.src = src; j.dst = arena_alloc(n); j.n_in = n;
        j.level = uint32_t(level); j.nlev = 0; j.raw = raw ? 1 : 0;
        add_job(s++, j);
        src.in_arena = true; src.off = j.dst;
    }
    // n > kHandoff can only remain if level == depth_target, which means n == 1 by the limit check upstream
    std::vector<uint32_t> nodes;
    for (uint64_t i = 0; i < n; i++) nodes.push_back(uint32_t(src.off + i));
    return merkle_small(nodes, level, depth_target);
}
uint32_t SszPlan::wide_chunks(uint64_t field_off, uint64_t n_chunks, int depth_target) {
    PSrc s; s.in_arena = false; s.off = field_off;
    cur_copy_ = copy_of(field_off);
    const uint32_t r = wide_nodes(s, true, n_chunks, 0, depth_target, 0);
    cur_copy_ = -1;
    return r;
}
uint32_t SszPlan::wide_records(uint32_t type, uint64_t field_off, uint64_t n, int depth_target) {
    if (n == 0) return zero(depth_target);
    cur_copy_ = copy_of(field_off);
    PJob j;
    j.type = type; j.src.in_arena = false; j.src.off = field_off; j.dst = arena_alloc(n); j.n_in = n;
    j.copy = cur_copy_;
    if (type == JOB_VALIDATORS) {
        j.chain = cur_chain_;
        validator_jobs_.push_back(j);
        if (cur_chain_ >= 0) chains_[size_t(cur_chain_)].jobs.emplace_back(-1, validator_jobs_.size() - 1);
        for (auto& c : copies_) if (c.field_off == field_off) c.validators = true;
    } else add_job(0, j);
    PSrc s; s.in_arena = true; s.off = j.dst;
    const uint32_t r = wide_nodes(s, false, n, 0, depth_target, 1);
    cur_copy_ = -1;
    return r;
}
uint32_t SszPlan::wide_pubkeys_with_extra(uint64_t field_off, uint64_t n, int depth_target, uint32_t* extra) {
    cur_copy_ = copy_of(field_off);
    PJob j;
    j.type = JOB_PUBKEY48; j.src.in_arena = false; j.src.off = field_off; j.dst = arena_alloc(n + 1); j.n_in = n + 1;
    add_job(0, j);
    *extra = uint32_t(j.dst + n);
    PSrc s; s.in_arena = true; s.off = j.dst;
    const uint32_t r = wide_nodes(s, false, n, 0, depth_target, 1);
    cur_copy_ = -1;
    return r;
}
uint64_t SszPlan::h2d_bytes() const {
    uint64_t b = small_words_.size() * 4 + ops_.size() * sizeof(FinOp);
    for (auto& c : copies_) b += c.nbytes;
    return b;
}

// ------------------------------------------------------------------------------------------------ execution
int32_t ensure_zero_nodes(Engine& e) {
    if (e.d_zero) return B200_SUCCESS;
    // zero[i+1] = H(zero[i], zero[i]) computed on the device with the finisher (64 one-op waves)
    uint32_t* d = nullptr;
    B200_CUDA_TRY(cudaMalloc(&d, 65 * 32));
    B200_CUDA_TRY(cudaMemsetAsync(d, 0, 65 * 32, e.stream));
    std::vector<FinOp> ops(64);
    std::vector<uint32_t> wend(64);
    for (uint32_t i = 0; i < 64; i++) { ops[i] = FinOp{i, i, i + 1, FIN_HASH}; wend[i] = i + 1; }
    FinOp* dops = nullptr; uint32_t* dw = nullptr;
    B200_CUDA_TRY(cudaMalloc(&dops, sizeof(FinOp) * 64));
    B200_CUDA_TRY(cudaMalloc(&dw, 4 * 64));
    B200_CUDA_TRY(cudaMemcpyAsync(dops, ops.data(), sizeof(FinOp) * 64, cudaMemcpyHostToDevice, e.stream));
    B200_CUDA_TRY(cudaMemcpyAsync(dw, wend.data(), 4 * 64, cudaMemcpyHostToDevice, e.stream));
    launch_finisher(d, dops, dw, 64, e.stream);
    e.launches++;
    B200_CUDA_TRY(cudaGetLastError());
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    cudaFree(dops); cudaFree(dw);
    e.d_zero = d;
    return B200_SUCCESS;
}

int32_t SszPlan::run(Engine& e, DevBuf& arena, DevBuf& fields, DevBuf& planbuf, CopyMode copy,
                     const std::vector<uint32_t>& outputs, uint8_t* out,
                     const std::vector<std::vector<uint32_t>>* dirty, DevBuf* selbuf,
                     const std::vector<std::pair<const uint8_t*, const uint8_t*>>* changed_host_ranges) {
    const bool sparse = dirty != nullptr;
    if (sparse && (dirty->size() != chains_.size() || !selbuf || copy == COPY_ALL)) return B200_ERR_BAD_ARG;
    if (small_words_.size() / 8 > kSmallCap) { e.last_error = "ssz plan: too many small leaves"; return B200_ERR_BAD_ARG; }
    int32_t rc = ensure_zero_nodes(e);
    if (rc) return rc;
    B200_CUDA_TRY(arena.reserve(arena_next_ * 32));
    B200_CUDA_TRY(fields.reserve(field_next_ + 256));
    uint32_t* d_arena = static_cast<uint32_t*>(arena.p);
    uint8_t* d_fields = static_cast<uint8_t*>(fields.p);

    // order finisher ops by wave; ops that depend on a remote node (wave >= kRemoteWave) form pass 2, numbered after
    // the local waves so that one cumulative wave_end table serves both finisher launches
    int n_local_waves = 0, n_remote_waves = 0;
    for (int w : op_wave_) {
        if (w >= kRemoteWave) n_remote_waves = std::max(n_remote_waves, w - kRemoteWave + 1);
        else n_local_waves = std::max(n_local_waves, w + 1);
    }
    if (xch_n_ && sparse) return B200_ERR_BAD_ARG;
    if (n_remote_waves && !xch_n_) return B200_ERR_BAD_ARG;
    std::vector<int> wave_of(op_wave_);   // (a resident plan runs many times: never renumber op_wave_ itself)
    for (int& w : wave_of) if (w >= kRemoteWave) w = n_local_waves + (w - kRemoteWave);
    const int nwaves = n_local_waves + n_remote_waves;
    std::vector<uint32_t> order(ops_.size());
    for (size_t i = 0; i < order.size(); i++) order[i] = uint32_t(i);
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return wave_of[a] < wave_of[b]; });
    std::vector<uint32_t> wave_end(size_t(nwaves), 0);
    for (size_t i = 0; i < order.size(); i++) wave_end[size_t(wave_of[order[i]])] = uint32_t(i + 1);
    for (int w = 1; w < nwaves; w++) wave_end[size_t(w)] = std::max(wave_end[size_t(w)], wave_end[size_t(w - 1)]);

    // dirty-path selection lists (host only): per chain, the outputs of job k that lie above the dirty inputs of job k
    std::vector<uint32_t> sel;           // all selection lists back to back
    struct Launch { const PJob* pj; size_t off; uint32_t n; size_t level; };
    std::vector<Launch> launches;
    if (sparse) {
        for (size_t c = 0; c < chains_.size(); c++) {
            std::vector<uint32_t> cur = (*dirty)[c];
            size_t level = 0;
            for (auto& ref : chains_[c].jobs) {
                if (cur.empty()) break;
                const PJob& pj = ref.first < 0 ? validator_jobs_[ref.second] : stages_[size_t(ref.first)][ref.second];
                if (pj.type == JOB_REDUCE && pj.nlev) {
                    size_t w = 0;
                    for (size_t i = 0; i < cur.size(); i++) {
                        const uint32_t o = cur[i] >> pj.nlev;
                        if (w == 0 || cur[w - 1] != o) cur[w++] = o;
                    }
                    cur.resize(w);
                } else if (pj.type != JOB_REDUCE && pj.type != JOB_VALIDATORS) {
                    return B200_ERR_BAD_ARG;
                }
                launches.push_back(Launch{&pj, sel.size(), uint32_t(cur.size()), level++});
                sel.insert(sel.end(), cur.begin(), cur.end());
            }
        }
        if (!sel.empty()) B200_CUDA_TRY(selbuf->reserve(sel.size() * 4));
    }

    // pinned staging image: [small words | ops | wave_end | out(32 B x outputs) | selection lists]
    size_t sz_small = small_words_.size() * 4;
    size_t sz_ops = ops_.size() * sizeof(FinOp);
    size_t sz_wend = wave_end.size() * 4;
    size_t off_ops = (sz_small + 15) & ~size_t(15);
    size_t off_wend = off_ops + ((sz_ops + 15) & ~size_t(15));
    size_t off_out = off_wend + ((sz_wend + 15) & ~size_t(15));
    size_t off_sel = (off_out + 32 * outputs.size() + 15) & ~size_t(15);
    size_t total = off_sel + sel.size() * 4;
    B200_CUDA_TRY(e.staging.reserve(total));
    B200_CUDA_TRY(planbuf.reserve(off_out + 64));
    uint8_t* st = static_cast<uint8_t*>(e.staging.p);
    if (sz_small) memcpy(st, small_words_.data(), sz_small);
    FinOp* hops = reinterpret_cast<FinOp*>(st + off_ops);
    for (size_t i = 0; i < order.size(); i++) hops[i] = ops_[order[i]];
    if (sz_wend) memcpy(st + off_wend, wave_end.data(), sz_wend);
    if (!sel.empty()) memcpy(st + off_sel, sel.data(), sel.size() * 4);

    cudaStream_t s = e.stream;
    uint8_t* d_plan = static_cast<uint8_t*>(planbuf.p);
    B200_CUDA_TRY(cudaMemcpyAsync(d_arena, e.d_zero, 65 * 32, cudaMemcpyDeviceToDevice, s));
    if (sz_small) B200_CUDA_TRY(cudaMemcpyAsync(d_arena + kSmallBase * 8, st, sz_small, cudaMemcpyHostToDevice, s));
    if (sz_ops + sz_wend)
        B200_CUDA_TRY(cudaMemcpyAsync(d_plan + off_ops, st + off_ops, off_out - off_ops, cudaMemcpyHostToDevice, s));
    auto materialize = [&](const PJob& pj) {
        Job j{};
        j.src = pj.src.in_arena ? static_cast<const void*>(d_arena + pj.src.off * 8)
                                : static_cast<const void*>(d_fields + pj.src.off);
        j.dst = d_arena + pj.dst * 8;
        j.n_in = pj.n_in; j.type = pj.type; j.level = pj.level; j.nlev = pj.nlev; j.raw = pj.raw;
        return j;
    };
    B200_CUDA_TRY(cudaEventRecord(e.ev0, s));
    static const bool trace = getenv("B200_SSZ_TRACE") && atoi(getenv("B200_SSZ_TRACE"));
    static cudaEvent_t tev[4] = {nullptr, nullptr, nullptr, nullptr};
    if (trace && !tev[0]) for (auto& ev : tev) cudaEventCreate(&ev);
    bool validators_launched = false;
    // stage launches over the jobs `pick` accepts (at most kMaxJobsPerStage jobs per launch).  Once a list is down to
    // kCoopMaxInputs nodes its remaining reduce jobs are latency-bound (7 dependent pair-hashes per thread and launch): up to
    // three consecutive ones are folded into ONE cooperative launch (k_merkle_coop: a pair-hash per thread per level), which
    // writes the same nodes to the same arena slots — the dirty-path re-hash still finds every level.  B200_SSZ_FOLD=0: off.
    static const bool fold = !(getenv("B200_SSZ_FOLD") && atoi(getenv("B200_SSZ_FOLD")) == 0);
    constexpr uint64_t kCoopMaxInputs = uint64_t(1) << 17;
    auto launch_stages = [&](auto&& pick, cudaStream_t on) {
        std::vector<std::vector<char>> folded(stages_.size());
        for (size_t si = 0; si < stages_.size(); si++) folded[si].assign(stages_[si].size(), 0);
        for (size_t si = 0; si < stages_.size(); si++) {
            auto& stage_all = stages_[si];
            std::vector<PJob> stage;
            std::vector<CoopJob> coop;
            std::vector<uint32_t> coop_levels;
            for (size_t k = 0; k < stage_all.size(); k++) {
                const PJob& pj = stage_all[k];
                if (folded[si][k] || !pick(pj)) continue;
                if (!(fold && pj.type == JOB_REDUCE && pj.nlev > 0 && pj.n_in <= kCoopMaxInputs)) { stage.push_back(pj); continue; }
                const Job j0 = materialize(pj);
                CoopJob cj{};
                cj.src = j0.src; cj.dst[0] = j0.dst; cj.n_in = pj.n_in; cj.level = pj.level; cj.nlev[0] = pj.nlev; cj.raw = pj.raw;
                uint32_t L = pj.nlev;
                uint32_t prev_dst = pj.dst;
                int slot = 1;
                for (size_t s2 = si + 1; s2 < stages_.size() && slot < 3; s2++) {
                    int found = -1;
                    for (size_t k2 = 0; k2 < stages_[s2].size(); k2++) {
                        const PJob& nx = stages_[s2][k2];
                        if (!folded[s2][k2] && nx.type == JOB_REDUCE && nx.nlev > 0 && !nx.raw && nx.src.in_arena && nx.src.off == prev_dst &&
                            L + nx.nlev <= 9 && pick(nx)) { found = int(k2); break; }
                    }
                    if (found < 0) break;
                    const PJob& nx = stages_[s2][size_t(found)];
                    cj.dst[slot] = d_arena + nx.dst * 8; cj.nlev[slot] = nx.nlev;
                    L += nx.nlev; prev_dst = nx.dst; folded[s2][size_t(found)] = 1; slot++;
                }
                coop.push_back(cj);
                coop_levels.push_back(L);
            }
            for (size_t b0 = 0; b0 < stage.size(); b0 += kMaxJobsPerStage) {
                StageDesc sd{};
                sd.zero_nodes = d_arena;
                uint32_t nb = 0;
                const size_t eidx = std::min(stage.size(), b0 + kMaxJobsPerStage);
                for (size_t k = b0; k < eidx; k++) {
                    Job j = materialize(stage[k]);
                    const uint64_t work = (j.type == JOB_REDUCE) ? ((j.n_in + (uint64_t(1) << j.nlev) - 1) >> j.nlev) : j.n_in;
                    j.block_begin = nb;
                    nb += uint32_t((work + kStageThreads - 1) / kStageThreads);
                    sd.jobs[sd.njobs++] = j;
                }
                sd.nblocks = nb;
                launch_stage(sd, on);
                e.launches++;
            }
            for (size_t b0 = 0; b0 < coop.size(); b0 += kMaxCoopJobs) {
                CoopDesc cd{};
                cd.zero_nodes = d_arena;
                uint32_t nb = 0;
                const size_t eidx = std::min(coop.size(), b0 + kMaxCoopJobs);
                for (size_t k = b0; k < eidx; k++) {
                    CoopJob cj = coop[k];
                    cj.block_begin = nb;
                    nb += uint32_t((cj.n_in + (uint64_t(1) << coop_levels[k]) - 1) >> coop_levels[k]);
                    cd.jobs[cd.njobs++] = cj;
                }
                cd.nblocks = nb;
                launch_coop(cd, on);
                e.launches++;
            }
        }
    };
    auto from_validators = [&](const PJob& pj) { return pj.copy >= 0 && copies_[size_t(pj.copy)].validators; };
    // One-shot call with a big Validator list: everything else is copied FIRST (a few MB) and hashed while the list
    // streams in behind it in slices, each slice hashed as soon as it has landed — the kernels hide under the PCIe
    // transfer (and, in a multi-GPU shard, the small fields under the rank's slice of the list).
    bool pipelined = false;
    if (copy == COPY_ALL && !sparse && validator_jobs_.size() == 1)
        for (auto& c : copies_) pipelined = pipelined || c.validators;
    if (copy != COPY_NONE) {
        cudaStream_t cs = e.copy_stream;
        B200_CUDA_TRY(cudaEventRecord(e.ev_copy[16], s));
        B200_CUDA_TRY(cudaStreamWaitEvent(cs, e.ev_copy[16], 0));  // buffers may still be in use by the previous call
        for (auto& c : copies_) {
            if (c.validators && pipelined) continue;
            if (copy == COPY_SMALL_ONLY && c.chain >= 0) continue;
            if (copy == COPY_SMALL_ONLY && changed_host_ranges) {
                bool hit = false;
                for (auto& r : *changed_host_ranges) hit = hit || (r.first < c.src + c.nbytes && c.src < r.second);
                if (!hit) continue;
            }
            B200_CUDA_TRY(cudaMemcpyAsync(d_fields + c.field_off, c.src, c.nbytes, cudaMemcpyHostToDevice, cs));
            if (c.nbytes % 32)
                B200_CUDA_TRY(cudaMemsetAsync(d_fields + c.field_off + c.nbytes, 0, c.zero_tail, cs));
        }
        B200_CUDA_TRY(cudaEventRecord(e.ev_copy[16], cs));
        B200_CUDA_TRY(cudaStreamWaitEvent(s, e.ev_copy[16], 0));
        if (pipelined) {
            launch_stages([&](const PJob& pj) { return !from_validators(pj); }, s);
            for (auto& c : copies_) {
                if (!c.validators) continue;
                const PJob& pj = validator_jobs_[0];
                const uint64_t n = pj.n_in;
                // up to 16 slices, none smaller than 32 768 records (a multi-GPU shard is 1/world of the list: slices
                // that cannot fill the SMs would cost more in launches than the overlap buys)
                const uint64_t n_slices = std::min<uint64_t>(16, std::max<uint64_t>(1, n / 32768));
                const uint64_t per = ((n + n_slices - 1) / n_slices + kStageThreads - 1) / kStageThreads * kStageThreads;  // whole CTAs per slice
                int k = 0;
                for (uint64_t lo = 0; lo < n; lo += per, k++) {
                    const uint64_t cnt = std::min(per, n - lo);
                    B200_CUDA_TRY(cudaMemcpyAsync(d_fields + c.field_off + lo * 121, c.src + lo * 121, cnt * 121, cudaMemcpyHostToDevice, cs));
                    B200_CUDA_TRY(cudaEventRecord(e.ev_copy[k], cs));
                    B200_CUDA_TRY(cudaStreamWaitEvent(s, e.ev_copy[k], 0));
                    Job j = materialize(pj);
                    j.src = d_fields + c.field_off + lo * 121;
                    j.dst = d_arena + (pj.dst + lo) * 8;
                    j.n_in = cnt;
                    launch_validators(j, s);
                    e.launches++;
                }
                if (c.nbytes % 32) {
                    B200_CUDA_TRY(cudaMemsetAsync(d_fields + c.field_off + c.nbytes, 0, c.zero_tail, cs));
                    B200_CUDA_TRY(cudaEventRecord(e.ev_copy[16], cs));
                    B200_CUDA_TRY(cudaStreamWaitEvent(s, e.ev_copy[16], 0));
                }
                validators_launched = true;
                break;
            }
        }
    }
    if (trace) cudaEventRecord(tev[0], s);
    if (sparse && !sel.empty()) {
        // dirty paths of the big lists: per chain, job k recomputes the outputs above the dirty inputs of job k
        B200_CUDA_TRY(cudaMemcpyAsync(selbuf->p, st + off_sel, sel.size() * 4, cudaMemcpyHostToDevice, s));
        const uint32_t* d_sel = static_cast<const uint32_t*>(selbuf->p);
        // job k of every chain reads only job k-1 of the SAME chain, so the k-th jobs of all chains share one launch:
        // the Validator records first (their own kernel), then one fused REDUCE launch per level over all lists
        size_t n_levels = 0;
        for (auto& l : launches) n_levels = std::max(n_levels, l.level + 1);
        for (size_t lev = 0; lev < n_levels; lev++) {
            SparseDesc sd{};
            sd.zero_nodes = d_arena; sd.sel = d_sel;
            uint32_t nb = 0;
            auto flush = [&]() {
                if (!sd.njobs) return;
                sd.block_begin[sd.njobs] = nb;
                launch_sparse_multi(sd, s); e.launches++;
                sd.njobs = 0; nb = 0;
            };
            for (auto& l : launches) {
                if (l.level != lev || l.n == 0) continue;
                if (l.pj->type == JOB_VALIDATORS) { launch_sparse(materialize(*l.pj), d_arena, d_sel + l.off, l.n, s); e.launches++; continue; }
                if (sd.njobs == kMaxSparseJobs) flush();
                sd.jobs[sd.njobs] = materialize(*l.pj);
                sd.sel_begin[sd.njobs] = uint32_t(l.off);
                sd.n_sel[sd.njobs] = l.n;
                sd.block_begin[sd.njobs] = nb;
                nb += (l.n + kStageThreads - 1) / kStageThreads;
                sd.njobs++;
            }
            flush();
        }
    }
    if (trace) cudaEventRecord(tev[1], s);
    // (Measured and dropped: running the non-Validator stage chains on the copy stream UNDER the Validator
    // kernel made the resident full re-hash slower — the chains' CTAs take SM slots from the kernel that
    // is the critical path, and the join adds two event waits.)
    if (!validators_launched)
        for (auto& pj : validator_jobs_) {
            if (sparse && pj.chain >= 0) continue;
            launch_validators(materialize(pj), s); e.launches++;
        }
    // incremental mode: the arena is the resident state's own, so the outputs of a dense job whose staged field did not
    // change since the previous root are still valid — only fields hit by `changed_host_ranges` are re-hashed
    std::vector<char> copy_changed(copies_.size(), sparse ? 0 : 1);
    if (sparse && changed_host_ranges)
        for (size_t ci = 0; ci < copies_.size(); ci++)
            for (auto& r : *changed_host_ranges)
                if (r.first < copies_[ci].src + copies_[ci].nbytes && copies_[ci].src < r.second) copy_changed[ci] = 1;
    launch_stages([&](const PJob& pj) {
        if (sparse && pj.chain >= 0) return false;
        if (sparse && pj.copy >= 0 && !copy_changed[size_t(pj.copy)]) return false;
        if (pipelined && !from_validators(pj)) return false;   // already launched, under the Validator list's transfer
        return true;
    }, s);
    if (trace) cudaEventRecord(tev[2], s);
    if (n_local_waves) {
        launch_finisher(d_arena, reinterpret_cast<const FinOp*>(d_plan + off_ops),
                        reinterpret_cast<const uint32_t*>(d_plan + off_wend), n_local_waves, s);
        e.launches++;
    }
    if (xch_n_) {   // the path's one exchange step, on the engine stream: slice roots -> every rank
        if (comm().world != xch_world_) { e.last_error = "ssz plan: communicator size changed"; return B200_ERR_BAD_ARG; }
        rc = comm_all_gather(e, d_arena + uint64_t(xch_send_) * 8, d_arena + uint64_t(xch_recv_) * 8, size_t(xch_n_) * 32, s);
        if (rc) return rc;
        if (n_remote_waves) {
            launch_finisher(d_arena, reinterpret_cast<const FinOp*>(d_plan + off_ops),
                            reinterpret_cast<const uint32_t*>(d_plan + off_wend) + n_local_waves, n_remote_waves, s,
                            n_local_waves ? wave_end[size_t(n_local_waves - 1)] : 0u);
            e.launches++;
        }
    }
    B200_CUDA_TRY(cudaEventRecord(e.ev1, s));
    B200_CUDA_TRY(cudaGetLastError());
    for (size_t i = 0; i < outputs.size(); i++)
        B200_CUDA_TRY(cudaMemcpyAsync(st + off_out + 32 * i, d_arena + uint64_t(outputs[i]) * 8, 32,
                                      cudaMemcpyDeviceToHost, s));
    B200_CUDA_TRY(cudaStreamSynchronize(s));
    B200_CUDA_TRY(cudaEventElapsedTime(&e.last_kernel_ms, e.ev0, e.ev1));
    if (trace) {
        float a = 0, b = 0, c = 0, d = 0;
        cudaEventElapsedTime(&a, e.ev0, tev[0]); cudaEventElapsedTime(&b, tev[0], tev[1]);
        cudaEventElapsedTime(&c, tev[1], tev[2]); cudaEventElapsedTime(&d, tev[2], e.ev1);
        fprintf(stderr, "[b200 ssz] uploads %.3f | dirty paths %.3f | dense stages %.3f | finisher %.3f | total %.3f ms (%s)\n",
                a, b, c, d, e.last_kernel_ms, sparse ? "incremental" : "full");
    }
    for (size_t i = 0; i < outputs.size(); i++) {
        const uint32_t* w = reinterpret_cast<const uint32_t*>(st + off_out + 32 * i);
        for (int k = 0; k < 8; k++) {
            out[32 * i + 4 * k + 0] = uint8_t(w[k] >> 24); out[32 * i + 4 * k + 1] = uint8_t(w[k] >> 16);
            out[32 * i + 4 * k + 2] = uint8_t(w[k] >> 8);  out[32 * i + 4 * k + 3] = uint8_t(w[k]);
        }
    }
    return B200_SUCCESS;
}

// ------------------------------------------------------------------------------------------------ BeaconState
namespace {
struct Preset {
    uint64_t slots_per_historical_root, historical_roots_limit, eth1_data_votes_bound, validator_registry_limit,
        epochs_per_historical_vector, epochs_per_slashings_vector, sync_committee_size;
};
// ethereum-consensus/src/phase0/presets/{mainnet.rs:5-36,82-83, minimal.rs:20-25},
// altair/presets/{mainnet,minimal}.rs:19
const Preset kPresets[2] = {
    {8192, 1ull << 24, 2048, 1ull << 40, 65536, 8192, 512},
    {64, 1ull << 24, 32, 1ull << 40, 64, 64, 32},
};
inline uint32_t le32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | (uint32_t(p[3]) << 24); }
inline uint64_t le64(const uint8_t* p) { return uint64_t(le32(p)) | (uint64_t(le32(p + 4)) << 32); }
}  // namespace

bool parse_beacon_state(const uint8_t* s, size_t len, int preset, StateOffsets& so) {
    if (preset < 0 || preset > 1) return false;
    const Preset& P = kPresets[preset];
    size_t fixed = 8 + 32 + 8 + 16 + 112 + 2 * 32 * P.slots_per_historical_root + 4 + 72 + 4 + 8 + 4 + 4 +
                   32 * P.epochs_per_historical_vector + 8 * P.epochs_per_slashings_vector + 4 + 4 + 1 + 3 * 40 + 4 +
                   2 * (48 * P.sync_committee_size + 48) + 4 + 8 + 8 + 4;
    if (len < fixed || len > 0xffffffffull) return false;
    size_t o = 8 + 32 + 8 + 16 + 112;
    so.block_roots = o; o += 32 * P.slots_per_historical_root;
    so.state_roots = o; o += 32 * P.slots_per_historical_root;
    so.var[0] = le32(s + o); o += 4;  // historical_roots
    so.eth1_data = o; o += 72;
    so.var[1] = le32(s + o); o += 4;  // eth1_data_votes
    so.eth1_deposit_index = o; o += 8;
    so.var[2] = le32(s + o); o += 4;  // validators
    so.var[3] = le32(s + o); o += 4;  // balances
    so.randao_mixes = o; o += 32 * P.epochs_per_historical_vector;
    so.slashings = o; o += 8 * P.epochs_per_slashings_vector;
    so.var[4] = le32(s + o); o += 4;  // previous_epoch_participation
    so.var[5] = le32(s + o); o += 4;  // current_epoch_participation
    so.justification_bits = o; o += 1;
    so.checkpoints = o; o += 120;
    so.var[6] = le32(s + o); o += 4;  // inactivity_scores
    so.current_sync_committee = o; o += 48 * P.sync_committee_size + 48;
    so.next_sync_committee = o; o += 48 * P.sync_committee_size + 48;
    so.var[7] = le32(s + o); o += 4;  // latest_execution_payload_header
    so.next_withdrawal_index = o; o += 8;
    so.next_withdrawal_validator_index = o; o += 8;
    so.var[8] = le32(s + o); o += 4;  // historical_summaries
    so.var[9] = uint32_t(len);
    so.fixed = fixed;
    if (o != fixed || so.var[0] != fixed) return false;
    for (int i = 0; i < 9; i++)
        if (so.var[i] > so.var[i + 1]) return false;
    auto sz = [&](int i) { return size_t(so.var[i + 1] - so.var[i]); };
    if (sz(0) % 32 || sz(1) % 72 || sz(1) / 72 > P.eth1_data_votes_bound || sz(2) % 121 || sz(3) % 8 || sz(6) % 8 ||
        sz(8) % 64 || sz(0) / 32 > P.historical_roots_limit || sz(8) / 64 > P.historical_roots_limit)
        return false;
    // ExecutionPayloadHeader: 584-byte fixed part whose only offset (extra_data) must equal 584; <= 32 bytes extra
    if (sz(7) < 584 || sz(7) > 584 + 32) return false;
    if (le32(s + so.var[7] + 436) != 584) return false;
    return true;
}

// Everything except the five big lists; `big[5]` = their roots (already length-mixed).
// `chain_vectors`: the four big fixed-size vectors become chains 5..8 (in this order: block_roots, state_roots,
// randao_mixes, slashings) so that a resident state can re-hash only their dirty paths too.
static uint32_t assemble_state(SszPlan& p, const uint8_t* s, const StateOffsets& so, const Preset& P,
                               const uint32_t big[5], bool chain_vectors = false) {
    std::vector<uint32_t> f(28);
    auto sz = [&](int i) { return size_t(so.var[i + 1] - so.var[i]); };
    f[0] = p.leaf_bytes(s + 0, 8);
    f[1] = p.leaf(s + 8);
    f[2] = p.leaf_bytes(s + 40, 8);
    f[3] = p.container({p.leaf_bytes(s + 48, 4), p.leaf_bytes(s + 52, 4), p.leaf_bytes(s + 56, 8)});
    f[4] = p.container({p.leaf_bytes(s + 64, 8), p.leaf_bytes(s + 72, 8), p.leaf(s + 80), p.leaf(s + 112), p.leaf(s + 144)});
    int d_hist = depth_for(P.slots_per_historical_root);
    if (chain_vectors) p.begin_chain();
    f[5] = p.wide_chunks(p.stage_field(s + so.block_roots, 32 * P.slots_per_historical_root), P.slots_per_historical_root, d_hist);
    if (chain_vectors) p.begin_chain();
    f[6] = p.wide_chunks(p.stage_field(s + so.state_roots, 32 * P.slots_per_historical_root), P.slots_per_historical_root, d_hist);
    if (chain_vectors) p.end_chain();
    f[7] = p.mix_in_length(p.wide_chunks(p.stage_field(s + so.var[0], sz(0)), sz(0) / 32, depth_for(P.historical_roots_limit)), sz(0) / 32);
    {
        const uint8_t* e = s + so.eth1_data;
        f[8] = p.container({p.leaf(e), p.leaf_bytes(e + 32, 8), p.leaf(e + 40)});
    }
    f[9] = p.mix_in_length(p.wide_records(JOB_ETH1DATA, p.stage_field(s + so.var[1], sz(1)), sz(1) / 72, depth_for(P.eth1_data_votes_bound)), sz(1) / 72);
    f[10] = p.leaf_bytes(s + so.eth1_deposit_index, 8);
    f[11] = big[0];
    f[12] = big[1];
    if (chain_vectors) p.begin_chain();
    f[13] = p.wide_chunks(p.stage_field(s + so.randao_mixes, 32 * P.epochs_per_historical_vector), P.epochs_per_historical_vector, depth_for(P.epochs_per_historical_vector));
    if (chain_vectors) p.begin_chain();
    f[14] = p.wide_chunks(p.stage_field(s + so.slashings, 8 * P.epochs_per_slashings_vector), P.epochs_per_slashings_vector / 4, depth_for(P.epochs_per_slashings_vector / 4));
    if (chain_vectors) p.end_chain();
    f[15] = big[2];
    f[16] = big[3];
    f[17] = p.leaf_bytes(s + so.justification_bits, 1);
    for (int i = 0; i < 3; i++) {
        const uint8_t* c = s + so.checkpoints + 40 * i;
        f[18 + i] = p.hash2(p.leaf_bytes(c, 8), p.leaf(c + 8));
    }
    f[21] = big[4];
    for (int k = 0; k < 2; k++) {
        const uint8_t* c = s + (k == 0 ? so.current_sync_committee : so.next_sync_committee);
        size_t n = P.sync_committee_size;
        // pubkeys vector and the aggregate key share one staged region: n + 1 records, hashed by one PUBKEY48 job
        uint64_t off = p.stage_field(c, 48 * (n + 1));
        uint32_t agg;
        uint32_t keys = p.wide_pubkeys_with_extra(off, n, depth_for(n), &agg);
        f[22 + k] = p.hash2(keys, agg);
    }
    {
        const uint8_t* h = s + so.var[7];
        size_t hl = sz(7);
        std::vector<uint32_t> l(17);
        l[0] = p.leaf(h + 0);
        l[1] = p.leaf_bytes(h + 32, 20);
        l[2] = p.leaf(h + 52);
        l[3] = p.leaf(h + 84);
        std::vector<uint32_t> bloom(8);
        for (int i = 0; i < 8; i++) bloom[i] = p.leaf(h + 116 + 32 * i);
        l[4] = p.merkle_small(bloom, 0, 3);
        l[5] = p.leaf(h + 372);
        for (int i = 0; i < 4; i++) l[6 + i] = p.leaf_bytes(h + 404 + 8 * i, 8);
        size_t extra = hl - 584;
        std::vector<uint32_t> ex;
        if (extra) ex.push_back(p.leaf_bytes(h + 584, extra));
        l[10] = p.mix_in_length(p.merkle_small(ex, 0, 0), extra);
        l[11] = p.leaf(h + 440);
        l[12] = p.leaf(h + 472);
        l[13] = p.leaf(h + 504);
        l[14] = p.leaf(h + 536);
        l[15] = p.leaf_bytes(h + 568, 8);
        l[16] = p.leaf_bytes(h + 576, 8);
        f[24] = p.container(l);
    }
    f[25] = p.leaf_bytes(s + so.next_withdrawal_index, 8);
    f[26] = p.leaf_bytes(s + so.next_withdrawal_validator_index, 8);
    f[27] = p.mix_in_length(p.wide_records(JOB_PAIR64, p.stage_field(s + so.var[8], sz(8)), sz(8) / 64, depth_for(P.historical_roots_limit)), sz(8) / 64);
    return p.container(f);
}

// slice [rank*S, (rank+1)*S) of a list whose dense part is split into `world` subtrees of 2^k leaves
static void slice_of(uint64_t n, int world, int rank, uint64_t* first, uint64_t* count, int* k) {
    uint64_t per = (n + uint64_t(world) - 1) / uint64_t(world);
    int kk = depth_for(per ? per : 1);
    uint64_t S = uint64_t(1) << kk;
    uint64_t lo = std::min(n, S * uint64_t(rank)), hi = std::min(n, S * uint64_t(rank + 1));
    *first = lo; *count = hi - lo; *k = kk;
}

int32_t build_beacon_state_plan(SszPlan& p, const uint8_t* s, size_t len, int preset, std::vector<uint32_t>& outputs) {
    StateOffsets so;
    if (!parse_beacon_state(s, len, preset, so)) return B200_ERR_SSZ_MALFORMED;
    const Preset& P = kPresets[preset];
    auto sz = [&](int i) { return size_t(so.var[i + 1] - so.var[i]); };
    uint32_t big[5];
    int d_reg = depth_for(P.validator_registry_limit);
    // the five big lists are chains 0..4 (B200_FIELD_* in the C ABI): their jobs can re-hash dirty paths only
    p.begin_chain();
    big[0] = p.mix_in_length(p.wide_records(JOB_VALIDATORS, p.stage_field(s + so.var[2], sz(2)), sz(2) / 121, d_reg), sz(2) / 121);
    p.begin_chain();
    big[1] = p.mix_in_length(p.wide_chunks(p.stage_field(s + so.var[3], sz(3)), (sz(3) + 31) / 32, d_reg - 2), sz(3) / 8);
    p.begin_chain();
    big[2] = p.mix_in_length(p.wide_chunks(p.stage_field(s + so.var[4], sz(4)), (sz(4) + 31) / 32, d_reg - 5), sz(4));
    p.begin_chain();
    big[3] = p.mix_in_length(p.wide_chunks(p.stage_field(s + so.var[5], sz(5)), (sz(5) + 31) / 32, d_reg - 5), sz(5));
    p.begin_chain();
    big[4] = p.mix_in_length(p.wide_chunks(p.stage_field(s + so.var[6], sz(6)), (sz(6) + 31) / 32, d_reg - 2), sz(6) / 8);
    p.end_chain();
    outputs.assign(1, assemble_state(p, s, so, P, big, true));
    return B200_SUCCESS;
}

int32_t build_beacon_state_shard_plan(SszPlan& p, const uint8_t* s, size_t len, int preset, int rank, int world,
                                      std::vector<uint32_t>& outputs) {
    StateOffsets so;
    if (!parse_beacon_state(s, len, preset, so)) return B200_ERR_SSZ_MALFORMED;
    if (world < 1 || (world & (world - 1)) || rank < 0 || rank >= world) return B200_ERR_BAD_ARG;
    auto sz = [&](int i) { return size_t(so.var[i + 1] - so.var[i]); };
    outputs.clear();
    uint64_t first, count; int k;
    // validators: records
    slice_of(sz(2) / 121, world, rank, &first, &count, &k);
    outputs.push_back(p.wide_records(JOB_VALIDATORS, p.stage_field(s + so.var[2] + 121 * first, 121 * count), count, k));
    // packed lists: chunk-granular slices (slice starts are multiples of 2^k chunks => 32-byte aligned)
    const int idx[4] = {3, 4, 5, 6};
    for (int q = 0; q < 4; q++) {
        size_t nb = sz(idx[q]);
        uint64_t nch = (nb + 31) / 32;
        slice_of(nch, world, rank, &first, &count, &k);
        size_t b0 = std::min(nb, size_t(first) * 32), b1 = std::min(nb, size_t(first + count) * 32);
        outputs.push_back(p.wide_chunks(p.stage_field(s + so.var[idx[q]] + b0, b1 - b0), count, k));
    }
    return B200_SUCCESS;
}

// One plan for the fused multi-GPU call: this rank's slices of the five big lists, ALL small fields, one exchange of
// the 5 slice roots, then the tops of the five lists and the 28-field tree on every rank.
int32_t build_beacon_state_sharded_plan(SszPlan& p, const uint8_t* s, size_t len, int preset, int rank, int world,
                                        std::vector<uint32_t>& outputs) {
    StateOffsets so;
    if (!parse_beacon_state(s, len, preset, so)) return B200_ERR_SSZ_MALFORMED;
    if (world < 1 || (world & (world - 1)) || rank < 0 || rank >= world) return B200_ERR_BAD_ARG;
    const Preset& P = kPresets[preset];
    auto sz = [&](int i) { return size_t(so.var[i + 1] - so.var[i]); };
    const int d_reg = depth_for(P.validator_registry_limit);
    const uint64_t n_elems[5] = {sz(2) / 121, (sz(3) + 31) / 32, (sz(4) + 31) / 32, (sz(5) + 31) / 32, (sz(6) + 31) / 32};
    const uint64_t lens[5] = {sz(2) / 121, sz(3) / 8, sz(4), sz(5), sz(6) / 8};
    const int depth[5] = {d_reg, d_reg - 2, d_reg - 5, d_reg - 5, d_reg - 2};
    const int var_of[5] = {2, 3, 4, 5, 6};
    std::vector<uint32_t> local(5);
    int kq[5];
    for (int q = 0; q < 5; q++) {
        uint64_t first, count;
        slice_of(n_elems[q], world, rank, &first, &count, &kq[q]);
        if (kq[q] > depth[q]) return B200_ERR_LIMIT;
        if (q == 0) {
            local[0] = p.wide_records(JOB_VALIDATORS, p.stage_field(s + so.var[2] + 121 * first, 121 * count), count, kq[0]);
        } else {   // chunk-granular slices: starts are multiples of 2^k chunks => 32-byte aligned
            const size_t nb = sz(var_of[q]);
            const size_t b0 = std::min(nb, size_t(first) * 32), b1 = std::min(nb, size_t(first + count) * 32);
            local[size_t(q)] = p.wide_chunks(p.stage_field(s + so.var[var_of[q]] + b0, b1 - b0), count, kq[q]);
        }
    }
    const uint32_t remote = p.exchange(local, world);
    uint32_t big[5];
    for (int q = 0; q < 5; q++) {
        std::vector<uint32_t> nodes;
        for (int r = 0; r < world; r++) nodes.push_back(remote + uint32_t(r) * 5u + uint32_t(q));
        big[q] = p.mix_in_length(p.merkle_small(nodes, kq[q], depth[q]), lens[q]);
    }
    outputs.assign(1, assemble_state(p, s, so, P, big));
    return B200_SUCCESS;
}

int32_t build_beacon_state_combine_plan(SszPlan& p, const uint8_t* s, size_t len, int preset, int world,
                                        const uint8_t* all_roots, std::vector<uint32_t>& outputs) {
    StateOffsets so;
    if (!parse_beacon_state(s, len, preset, so)) return B200_ERR_SSZ_MALFORMED;
    if (world < 1 || (world & (world - 1))) return B200_ERR_BAD_ARG;
    const Preset& P = kPresets[preset];
    auto sz = [&](int i) { return size_t(so.var[i + 1] - so.var[i]); };
    int d_reg = depth_for(P.validator_registry_limit);
    const uint64_t n_elems[5] = {sz(2) / 121, (sz(3) + 31) / 32, (sz(4) + 31) / 32, (sz(5) + 31) / 32, (sz(6) + 31) / 32};
    const uint64_t lens[5] = {sz(2) / 121, sz(3) / 8, sz(4), sz(5), sz(6) / 8};
    const int depth[5] = {d_reg, d_reg - 2, d_reg - 5, d_reg - 5, d_reg - 2};
    uint32_t big[5];
    for (int q = 0; q < 5; q++) {
        uint64_t first, count; int k;
        slice_of(n_elems[q], world, 0, &first, &count, &k);
        std::vector<uint32_t> nodes;
        for (int r = 0; r < world; r++) nodes.push_back(p.leaf(all_roots + (size_t(r) * 5 + q) * 32));
        big[q] = p.mix_in_length(p.merkle_small(nodes, k, depth[q]), lens[q]);
    }
    outputs.assign(1, assemble_state(p, s, so, P, big));
    return B200_SUCCESS;
}

}  // namespace b200
