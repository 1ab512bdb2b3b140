// hqsched.cu — H100 (sm_90a) task->worker assignment solver behind the C ABI of include/hqsched.h.
//
// Replaces, for the single-node hot path of HyperQueue's tako scheduler tick (v0.26.0):
//   create_task_batches        crates/tako/src/internal/scheduler/batches.rs:42-181   (priority histogram)
//   run_scheduling_solver      crates/tako/src/internal/scheduler/solver.rs:16-461    (who gets how many)
//   create_task_mapping        crates/tako/src/internal/scheduler/mapping.rs:23-154   (which task goes where)
//   TaskQueues                 crates/tako/src/internal/scheduler/taskqueue.rs        (ready set, device resident)
//   task_finished readiness    crates/tako/src/internal/server/reactor.rs:500-580     (DAG mode)
// It is NOT a port: the reference solves a MILP over (worker, class, variant) counts with HiGHS; this
// library runs a deterministic priority-ordered first-fit over the same aggregation, with the per-task
// work (histogram, stable ranking, emission) as streaming kernels over an SoA task table in HBM.
// See DESIGN.md for the data layout, the kernels and their rooflines.
//
// Device data (all SoA, indexed by dense task handle h):
//   key[h]   u32  bit31 READY | bit30 DONE (assigned by a tick) | bit29 VALID | bit28 PREFILLED | level(14) | class(14)
//   prio[h]  u64  tako Priority (only read when the level table changes)
//   deps[h]  u32  unfinished dependencies (DAG mode), cons_off/cons: CSR of consumers
// One tick = ONE cooperative kernel (tick_k, hqs_tick.cuh):
//   worker CTAs : per-chunk histogram of ready tasks by group g = level*Q + class (HBM streaming, 4 B/task), exclusive
//                 scan of the chunk table over chunks, on request the pack step (one warp fills one worker), then the
//                 stable rank of every ready task inside its group, rank -> (worker, variant) through the solver's count
//                 segments, compact write of 8-byte assignments, READY -> DONE
//   solver CTA  : stages the worker state in shared memory (read straight from the pinned host buffer while the others
//                 count), then one warp walks the non-empty groups in priority order: sparse first-fit over tiles of 32
//                 workers starting at the class's frontier tile (amounts gcd-scaled to 32 bits when the tick allows it)
// Sharded over several GPUs (one context per GPU, tasks block-sharded, workers replicated) the solver CTA stores the
// rank's count vector into every peer's exchange buffer over NVLink and acquires the peers' flags before it solves (no
// host collective).
// hqs_tick_fetch_grouped regroups the tick's records per worker at fetch time (hqs_group.cuh: three plain launches behind
// the tick; tick_k does not know about it).
// The algorithm has a sequential specification, tests/greedy_model.py, which the kernels equal bit for bit.
#include "../../include/hqsched.h"

#include <cuda_runtime.h>

#include <type_traits>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <numeric>
#include <vector>

namespace {

typedef uint32_t u32;
typedef uint64_t u64;

#include "hqs_ready_set.cuh"
#include "hqs_solver.cuh"
#include "hqs_tick.cuh"
#include "hqs_group.cuh"


// ================================================================================================
// host side
// ================================================================================================
thread_local std::string g_create_error;

}  // namespace

struct hqs_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    u32 R = 0;
    std::string err;
    // classes
    u32 Q = 0;
    std::vector<hqs_class> classes;
    unsigned char* d_classes = nullptr;   // ClassT<RT, u64>[Q]
    u32 d_classes_cap = 0;                // bytes
    unsigned char* d_classes32 = nullptr; // ClassT<RT, u32>[Q]: amounts / gscale[r] (valid when narrow_classes)
    u32 d_classes32_cap = 0;
    u32 class_bytes32 = 0;                // sizeof(ClassT<RT, u32>)
    u64 gscale[HQS_MAX_RESOURCES] = {};   // per-resource gcd of every requested amount (1 where nothing is requested)
    u64 narrow_limit[HQS_MAX_RESOURCES] = {};   // largest worker amount the narrow path can hold: gscale * (2^31 - 1)
    bool narrow_classes = false;          // every scaled class amount < 2^31
    // peer-to-peer sharded tick
    u32* d_xbuf = nullptr;                // my exchange buffer: [2][HQS_MAX_PEERS][HQS_MAX_GROUPS] counts + [2][HQS_MAX_PEERS] flags
    u32* x_peer[HQS_MAX_PEERS] = {};      // every rank's exchange buffer (own included), set by hqs_shard_attach
    std::vector<void*> x_opened;          // IPC mappings to close
    u32 x_world = 0, x_rank = 0, x_seq = 0;
    u32* d_xall = nullptr;                // [HQS_MAX_GROUPS] sum over ranks, written by the solver
    u32* d_xbefore = nullptr;             // [HQS_MAX_GROUPS] sum over lower ranks
    bool x_tick = false;                  // the tick being launched uses the exchange
    bool tick_narrow = false;             // this tick runs the narrow solver
    bool force_wide = false;              // hqs_create flag bit 1: always the 64-bit solver (tests)
    u32 RT = 4;                           // resource slots of the device class layout (4, 8 or 16)
    u32 class_bytes = 0;                  // sizeof(ClassT<RT>)
    // priority levels (descending)
    std::vector<u64> levels;      // exact distinct priorities seen, descending
    std::vector<u64> dev_levels;  // what the device uses (== levels, or bucket bounds when coarsened)
    bool coarse = false;
    bool levels_declared = false;   // hqs_levels_add was used: the caller numbers the levels (sharded ready set), no pruning
    size_t levels_pruned_at = 0;    // size of the level set after the last pruning
    u64* d_levels = nullptr;
    u32 d_levels_cap = 0;
    u64* d_prune_lv = nullptr;      // prune_levels scratch: the exact levels and their live flags
    u32* d_prune_live = nullptr;
    u32 prune_cap = 0;
    // task table
    u32 n_handles = 0, cap_handles = 0;
    u32* d_key = nullptr;
    u64* d_prio = nullptr;
    u32* d_deps = nullptr;
    u32* d_cons_off = nullptr;
    u32* d_cons = nullptr;
    bool dag = false;
    // push staging (device)
    u32* d_push_task = nullptr; u32* d_push_cls = nullptr; u64* d_push_prio = nullptr;
    u32 push_cap = 0;
    u32* d_newcnt = nullptr; u64* d_newprio = nullptr;
    // tick buffers
    u32 sm_count = 132;
    u32 grid_ctas = 132;                // CTAs of the cooperative tick kernel (solver CTA + worker CTAs)
    u32 G_cap = 0, P_cap = 0;
    u32* d_table = nullptr;
    u32* d_total = nullptr;
    GroupOut* d_gout = nullptr;
    TickSync* d_sync = nullptr;
    size_t smem_budget[2] = {0, 0};     // dynamic shared memory a tick kernel instance may use (narrow, wide)
    bool sync_dirty = true;             // the counters must be zeroed before the next launch (first tick / after a failed one)
    u64* d_pk_fr = nullptr; u32* d_pk_quota = nullptr; u32* d_pk_taken = nullptr; u32* d_pk_cand = nullptr; u32* d_pk_meta = nullptr;
    u32* d_rem_scratch = nullptr; uint8_t* d_excl = nullptr;
    // proactive filling
    u32 pf_reserve = 0, pf_max = 0;     // SchedulerConfig::proactive_filling_reserve / _max (state.rs:14-21); max == 0: off
    uint4* d_gout2 = nullptr; u32* d_pf_cum = nullptr; u32* d_pf_wk = nullptr;
    std::vector<uint8_t> prefilled_wc; u32 prefilled_W = 0;   // host mirror for the next tick: [W][Q]
    u32* d_seg_cum = nullptr; u32* d_seg_wv = nullptr;
    hqs_assignment* d_out = nullptr; u32 out_cap_dev = 0;
    TickHeaderOut* d_hdr = nullptr;
    u64* d_free_after = nullptr;
    unsigned char* d_tickin = nullptr; size_t tickin_cap = 0;   // device copy of the tick input (blocked mask; everything when zero-copy is off)
    unsigned char* h_tickin = nullptr;  // pinned + mapped: the solver CTA reads the worker state from here
    unsigned char* h_tickin_dev = nullptr;   // device-side address of h_tickin
    bool zero_copy = true;
    unsigned char* h_hdr = nullptr;     // pinned + mapped: TickHeaderOut + free_after, written by the kernel
    unsigned char* h_hdr_dev = nullptr;
    size_t h_hdr_cap = 0;
    u32* h_small = nullptr;             // pinned scratch (counters)
    u32* h_pw = nullptr;                // pinned [HQS_MAX_WORKERS]: per-worker task counts of the last query
    // per-worker grouping of the records (hqs_tick_fetch_grouped); nothing of it exists until the first grouped fetch or
    // hqs_grouped_reserve
    hqs_assignment* d_grp_out = nullptr; u32 grp_cap = 0;      // the grouped records
    u32* d_grp_hist = nullptr; size_t grp_hist_cap = 0;        // [2W + 1][tiles] counts, then their prefix over the tiles
    u32* d_grp_small = nullptr;         // key totals [GRP_KEYS_MAX], offset table [GRP_KEYS_MAX + 1], the scan's ticket
    u32* h_grp_off = nullptr;           // pinned mirror of the offset table
    float grp_ms = -1.f;                // device time of the last grouping (profiling on), < 0: none
    // last tick
    u32 last_W = 0, last_G = 0, last_L = 0;
    bool last_blocked = false;
    bool tick_pending = false;          // a tick or a query has been launched and not fetched
    bool query_pending = false;         // ... and it is a query (hqs_query_fetch)
    bool own_stream = true;
    bool profile = false;
    bool pack = true;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    bool ev_valid = false;
    float last_ms[4] = {0, 0, 0, 0};
    hqs_stats stats{};
    unsigned long long dbg[8] = {0};
};

namespace {

int fail(hqs_ctx* c, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (c) c->err = buf; else g_create_error = buf;
    return code;
}

#define CU(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess)                                                                     \
            return fail(ctx, HQS_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_),   \
                        __FILE__, __LINE__);                                                       \
    } while (0)

template <typename T>
int dev_realloc(hqs_ctx* ctx, T** p, size_t old_n, size_t new_n, bool keep, bool zero_new) {
    T* q = nullptr;
    CU(cudaMalloc(&q, new_n * sizeof(T)));
    if (zero_new) CU(cudaMemsetAsync(q, 0, new_n * sizeof(T), ctx->stream));
    if (keep && *p && old_n) CU(cudaMemcpyAsync(q, *p, old_n * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream));
    if (*p) {
        CU(cudaStreamSynchronize(ctx->stream));
        CU(cudaFree(*p));
    }
    *p = q;
    return HQS_OK;
}

int ensure_handles(hqs_ctx* ctx, u32 need) {
    if (need <= ctx->cap_handles) return HQS_OK;
    u32 cap = std::max<u32>(need, std::max<u32>(ctx->cap_handles * 2, 1u << 16));
    cap = (cap + 1023u) & ~1023u;
    int rc;
    if ((rc = dev_realloc(ctx, &ctx->d_key, ctx->cap_handles, cap, true, true))) return rc;
    if ((rc = dev_realloc(ctx, &ctx->d_prio, ctx->cap_handles, cap, true, true))) return rc;
    ctx->cap_handles = cap;
    return HQS_OK;
}

// (Re)builds the device level table from ctx->levels, coarsening when L * Q exceeds HQS_MAX_GROUPS.
int upload_levels(hqs_ctx* ctx) {
    const u32 q = std::max<u32>(ctx->Q, 1);
    const u32 max_levels = std::max<u32>(1, HQS_MAX_GROUPS / q);
    const u32 L = (u32)ctx->levels.size();
    ctx->dev_levels.clear();
    if (L <= max_levels) {
        ctx->dev_levels = ctx->levels;
        ctx->coarse = false;
    } else {
        // merge adjacent levels into max_levels buckets; entry i = lowest priority of bucket i
        ctx->coarse = true;
        for (u32 b = 0; b < max_levels; ++b) {
            const u64 last = ((u64)(b + 1) * L) / max_levels - 1;
            ctx->dev_levels.push_back(ctx->levels[last]);
        }
        ctx->dev_levels.back() = 0;  // the last bucket takes everything below
    }
    const u32 n = (u32)ctx->dev_levels.size();
    if (n > ctx->d_levels_cap) {
        if (ctx->d_levels) { CU(cudaStreamSynchronize(ctx->stream)); CU(cudaFree(ctx->d_levels)); ctx->d_levels = nullptr; }
        ctx->d_levels_cap = std::max<u32>(n * 2, 64);
        CU(cudaMalloc(&ctx->d_levels, ctx->d_levels_cap * sizeof(u64)));
    }
    if (n) {
        // pageable source: the copy is staged by the runtime before the call returns
        CU(cudaMemcpyAsync(ctx->d_levels, ctx->dev_levels.data(), n * sizeof(u64), cudaMemcpyHostToDevice, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
    }
    ctx->stats.coarsened = ctx->coarse ? 1 : 0;
    return HQS_OK;
}

// Re-keys every VALID task from the current table.  An empty table (nothing is registered) puts any VALID key at level 0.
int relevel_all(hqs_ctx* ctx) {
    if (!ctx->n_handles) return HQS_OK;
    relevel_k<<<(ctx->n_handles + 255) / 256, 256, 0, ctx->stream>>>(
        ctx->n_handles, ctx->d_key, ctx->d_prio, ctx->d_levels, (u32)ctx->dev_levels.size(), ctx->coarse ? 1 : 0);
    ctx->stats.kernel_launches++;
    CU(cudaGetLastError());
    return HQS_OK;
}

// Drops the priority levels no task of the table carries any more (tako priorities have a per-job component, so a
// long-running server sees one level per job ever submitted).  Called when the level set is about to exceed what the
// group limit allows, or has doubled since the last pruning.  Returns true if levels were dropped (the caller then
// uploads the table and re-keys the tasks).
int prune_levels(hqs_ctx* ctx, bool* changed) {
    *changed = false;
    const u32 L = (u32)ctx->levels.size();
    if (ctx->levels_declared || L == 0 || ctx->n_handles == 0) return HQS_OK;
    // scratch kept across calls: a coarse table is pruned on every push that brings a new priority, and cudaFree would
    // synchronise the device each time
    if (L > ctx->prune_cap) {
        CU(cudaStreamSynchronize(ctx->stream));
        if (ctx->d_prune_lv) { CU(cudaFree(ctx->d_prune_lv)); CU(cudaFree(ctx->d_prune_live)); }
        ctx->d_prune_lv = nullptr; ctx->d_prune_live = nullptr;
        ctx->prune_cap = std::max<u32>(L * 2, 4096);
        CU(cudaMalloc(&ctx->d_prune_lv, (size_t)ctx->prune_cap * 8));
        CU(cudaMalloc(&ctx->d_prune_live, (size_t)ctx->prune_cap * 4));
    }
    u64* d_lv = ctx->d_prune_lv;
    u32* d_live = ctx->d_prune_live;
    CU(cudaMemsetAsync(d_live, 0, (size_t)L * 4, ctx->stream));
    CU(cudaMemcpyAsync(d_lv, ctx->levels.data(), (size_t)L * 8, cudaMemcpyHostToDevice, ctx->stream));
    level_live_k<<<(ctx->n_handles + 255) / 256, 256, 0, ctx->stream>>>(ctx->n_handles, ctx->d_key, ctx->d_prio, d_lv, L, d_live);
    ctx->stats.kernel_launches++;
    std::vector<u32> live(L);
    CU(cudaMemcpyAsync(live.data(), d_live, (size_t)L * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    std::vector<u64> kept;
    kept.reserve(L);
    for (u32 i = 0; i < L; ++i)
        if (live[i]) kept.push_back(ctx->levels[i]);
    *changed = kept.size() != ctx->levels.size();
    ctx->levels.swap(kept);
    ctx->levels_pruned_at = ctx->levels.size();
    return HQS_OK;
}

// the level set outgrew the group budget, or doubled since it was last pruned
bool levels_need_pruning(const hqs_ctx* ctx) {
    const size_t max_levels = std::max<u32>(1, HQS_MAX_GROUPS / std::max<u32>(ctx->Q, 1));
    return !ctx->levels_declared && (ctx->levels.size() > max_levels || ctx->levels.size() > 2 * ctx->levels_pruned_at + 64);
}

// merges new distinct priorities into the level set; returns true if the set changed
bool merge_levels(hqs_ctx* ctx, std::vector<u64>& fresh) {
    std::sort(fresh.begin(), fresh.end(), std::greater<u64>());
    fresh.erase(std::unique(fresh.begin(), fresh.end()), fresh.end());
    std::vector<u64> merged;
    merged.reserve(ctx->levels.size() + fresh.size());
    std::merge(ctx->levels.begin(), ctx->levels.end(), fresh.begin(), fresh.end(), std::back_inserter(merged),
               std::greater<u64>());
    merged.erase(std::unique(merged.begin(), merged.end()), merged.end());
    const bool changed = merged.size() != ctx->levels.size();
    ctx->levels.swap(merged);
    return changed;
}

void distinct_priorities(const u64* p, u32 n, std::vector<u64>& out) {
    // small open-addressing set with a last-value fast path; distinct priorities are few
    std::vector<u64> slots(1024, 0);
    std::vector<unsigned char> used(1024, 0);
    size_t count = 0;
    u64 last = n ? ~p[0] : 0;
    for (u32 i = 0; i < n; ++i) {
        const u64 v = p[i];
        if (v == last) continue;
        last = v;
        if ((count + 1) * 2 > slots.size()) {
            std::vector<u64> ns(slots.size() * 4, 0);
            std::vector<unsigned char> nu(slots.size() * 4, 0);
            for (size_t s = 0; s < slots.size(); ++s)
                if (used[s]) {
                    size_t h = (slots[s] * 0x9E3779B97F4A7C15ull) >> 20 & (ns.size() - 1);
                    while (nu[h]) h = (h + 1) & (ns.size() - 1);
                    ns[h] = slots[s]; nu[h] = 1;
                }
            slots.swap(ns); used.swap(nu);
        }
        size_t h = (v * 0x9E3779B97F4A7C15ull) >> 20 & (slots.size() - 1);
        while (used[h] && slots[h] != v) h = (h + 1) & (slots.size() - 1);
        if (!used[h]) { used[h] = 1; slots[h] = v; ++count; }
    }
    for (size_t s = 0; s < slots.size(); ++s) if (used[s]) out.push_back(slots[s]);
}

int ensure_tick_buffers(hqs_ctx* ctx, u32 G, u32 P, u32 W, u32 out_cap) {
    if (G > ctx->G_cap || P > ctx->P_cap || (size_t)G * P > (size_t)ctx->G_cap * ctx->P_cap) {
        const u32 ng = std::max(G, ctx->G_cap), np = std::max(P, ctx->P_cap);
        CU(cudaStreamSynchronize(ctx->stream));
        if (ctx->d_table) CU(cudaFree(ctx->d_table));
        CU(cudaMalloc(&ctx->d_table, (size_t)ng * np * sizeof(u32)));
        if (ng > ctx->G_cap) {
            if (ctx->d_total) CU(cudaFree(ctx->d_total));
            if (ctx->d_gout) CU(cudaFree(ctx->d_gout));
            CU(cudaMalloc(&ctx->d_total, ng * sizeof(u32)));
            CU(cudaMemsetAsync(ctx->d_total, 0, ng * sizeof(u32), ctx->stream));
            CU(cudaMalloc(&ctx->d_gout, ng * sizeof(GroupOut)));
            CU(cudaMemsetAsync(ctx->d_gout, 0, ng * sizeof(GroupOut), ctx->stream));
            if (ctx->d_gout2) CU(cudaFree(ctx->d_gout2));
            CU(cudaMalloc(&ctx->d_gout2, ng * sizeof(uint4)));
            CU(cudaMemsetAsync(ctx->d_gout2, 0, ng * sizeof(uint4), ctx->stream));
        }
        ctx->G_cap = ng; ctx->P_cap = np;
    }
    if (!ctx->d_seg_cum) {
        CU(cudaMalloc(&ctx->d_seg_cum, SEG_CAP * sizeof(u32)));
        CU(cudaMalloc(&ctx->d_seg_wv, SEG_CAP * sizeof(u32)));
        CU(cudaMalloc(&ctx->d_hdr, sizeof(TickHeaderOut)));
        CU(cudaMalloc(&ctx->d_free_after, (size_t)HQS_MAX_WORKERS * HQS_MAX_RESOURCES * sizeof(u64)));
        CU(cudaMalloc(&ctx->d_sync, sizeof(TickSync)));
        CU(cudaMalloc(&ctx->d_pk_fr, (size_t)HQS_MAX_WORKERS * HQS_MAX_RESOURCES * sizeof(u64)));
        CU(cudaMalloc(&ctx->d_pk_quota, (size_t)HQS_MAX_WORKERS * PACK_MAX_CAND * sizeof(u32)));
        CU(cudaMalloc(&ctx->d_pk_taken, (size_t)HQS_MAX_WORKERS * PACK_MAX_CAND * sizeof(u32)));
        CU(cudaMalloc(&ctx->d_pk_cand, PACK_MAX_CAND * sizeof(u32)));
        CU(cudaMalloc(&ctx->d_pk_meta, 2 * sizeof(u32)));
        CU(cudaMalloc(&ctx->d_rem_scratch, (size_t)HQS_MAX_WORKERS * HQS_MAX_RESOURCES * sizeof(u64)));
        CU(cudaMalloc(&ctx->d_excl, HQS_MAX_WORKERS));
        CU(cudaMalloc(&ctx->d_pf_cum, PF_SEG_CAP * sizeof(u32)));
        CU(cudaMalloc(&ctx->d_pf_wk, PF_SEG_CAP * sizeof(u32)));
        ctx->sync_dirty = true;
    }
    if (!ctx->h_hdr) {
        ctx->h_hdr_cap = sizeof(TickHeaderOut) + (size_t)HQS_MAX_WORKERS * HQS_MAX_RESOURCES * 8;
        CU(cudaHostAlloc(&ctx->h_hdr, ctx->h_hdr_cap, cudaHostAllocMapped));
        memset(ctx->h_hdr, 0, ctx->h_hdr_cap);
        CU(cudaHostGetDevicePointer(reinterpret_cast<void**>(&ctx->h_hdr_dev), ctx->h_hdr, 0));
    }
    if (out_cap > ctx->out_cap_dev) {
        CU(cudaStreamSynchronize(ctx->stream));
        if (ctx->d_out) CU(cudaFree(ctx->d_out));
        ctx->out_cap_dev = std::max<u32>(out_cap, 1024);
        CU(cudaMalloc(&ctx->d_out, (size_t)ctx->out_cap_dev * sizeof(hqs_assignment)));
    }
    (void)W;
    return HQS_OK;
}

struct TickLayout {
    size_t off_free, off_total, off_rem, off_order, off_vorder, off_mu, off_blocked, off_pfwc, bytes;
};

TickLayout tick_layout(u32 W, u32 R, u32 Q, bool blocked, bool pfwc = false) {
    TickLayout l;
    size_t o = 0;
    l.off_free = o; o += (size_t)W * R * 8;
    l.off_total = o; o += (size_t)W * R * 8;
    l.off_rem = o; o += (size_t)W * 8;
    l.off_order = o; o += (size_t)Q * 4;
    l.off_mu = o; o += (size_t)W * 4;
    l.off_vorder = o; o += (size_t)Q * HQS_MAX_VARIANTS;
    o = (o + 15) & ~size_t(15);
    l.off_blocked = o; if (blocked) o += (size_t)W * Q;
    o = (o + 15) & ~size_t(15);
    l.off_pfwc = o; if (pfwc) o += (size_t)W * Q;
    l.bytes = (o + 15) & ~size_t(15);
    return l;
}

// Per-tick orders, both from S_r = sum over workers of free[r] (MAX counts as one unit):
//  order[]   classes inside one priority level by descending objective weight of one task, the greedy
//            analogue of the MILP coefficient of create_sn_var (solver.rs:520-549):
//            weight * sum_r amount_r / S_r
//  vorder[]  variants of a class by ascending dominant share max_r amount_r / S_r: the variant that costs
//            least of the scarcest thing it touches is tried first
void tick_orders(const hqs_ctx* ctx, u32 W, const u64* free_rw, const u64* total_rw, u32* order, uint8_t* vorder) {
    const u32 R = ctx->R, Q = ctx->Q;
    double S[HQS_MAX_RESOURCES], T[HQS_MAX_RESOURCES];
    for (u32 r = 0; r < R; ++r) { S[r] = 0; T[r] = 0; }
    for (u32 w = 0; w < W; ++w)
        for (u32 r = 0; r < R; ++r) {
            const u64 f = free_rw[(size_t)w * R + r];
            S[r] += f == HQS_AMOUNT_MAX ? 1.0 : (double)f / 10000.0;
            const u64 t = total_rw[(size_t)w * R + r];
            T[r] += t == HQS_AMOUNT_MAX ? 1.0 : (double)t / 10000.0;
        }
    std::vector<std::pair<double, u32>> sc(Q);
    for (u32 c = 0; c < Q; ++c) {
        double best = 0;
        const hqs_class& cl = ctx->classes[c];
        std::pair<double, u32> doms[HQS_MAX_VARIANTS];
        for (u32 v = 0; v < cl.n_variants; ++v) {
            double s = 0, dom = 0;
            for (u32 r = 0; r < R; ++r) {
                const bool all = (cl.variants[v].all_mask >> r) & 1;
                const u64 amt = all ? 0 : cl.variants[v].amount[r];
                if (amt) {
                    const double x = S[r] < 1e-6 ? INFINITY : ((double)amt / 10000.0) / S[r];
                    dom = x > dom ? x : dom;
                }
                if (S[r] < 1e-6) continue;
                if (all) s += (T[r] / std::max<u32>(W, 1)) / S[r];
                else s += ((double)amt / 10000.0) / S[r];
            }
            if (cl.variants[v].all_mask) dom = INFINITY;
            s *= (double)cl.variants[v].weight / 10000.0;
            best = std::max(best, s);
            doms[v] = {dom, v};
        }
        sc[c] = {best, c};
        std::stable_sort(doms, doms + cl.n_variants,
                         [](const std::pair<double, u32>& a, const std::pair<double, u32>& b) { return a.first < b.first; });
        for (u32 v = 0; v < HQS_MAX_VARIANTS; ++v) vorder[c * HQS_MAX_VARIANTS + v] = v < cl.n_variants ? (uint8_t)doms[v].second : 0;
    }
    std::stable_sort(sc.begin(), sc.end(), [](const std::pair<double, u32>& a, const std::pair<double, u32>& b) {
        return a.first > b.first;
    });
    for (u32 c = 0; c < Q; ++c) order[c] = sc[c].second;
}

// Chunk geometry of the streaming steps: every worker CTA of the tick kernel owns chunks b, b + nW, ...; an emit warp owns
// `rows` rows of 32 consecutive tasks of its chunk.  rows is chosen so that the table splits into (about) one chunk per
// worker CTA; large tables take several chunks per CTA.
struct TickGeom { u32 G, L, P, chunk, rows, emit_warps, g_smem, nbits, emit_stage; size_t worker_smem; };

TickGeom tick_geom(const hqs_ctx* ctx) {
    TickGeom t;
    t.L = std::max<u32>((u32)ctx->dev_levels.size(), 1);
    t.G = (t.L * std::max<u32>(ctx->Q, 1)) << (ctx->pf_max ? 1 : 0);      // proactive filling: waiting / prefilled sub-groups
    t.nbits = 1;
    while ((1u << t.nbits) < t.G) t.nbits++;
    const u32 n = std::max<u32>(ctx->n_handles, 1);
    const u32 nW = std::max<u32>(ctx->grid_ctas - 1, 1);
    // emit step shared memory: warps * G counters (+ G solver records) + the segment cache
    const size_t seg_cache = 2 * EMIT_SEG_SMEM * sizeof(u32);
    t.emit_warps = TICK_WARPS;
    while (t.emit_warps > 1 && (size_t)t.emit_warps * t.G * 4 > 128 * 1024) t.emit_warps /= 2;
    const u32 per_row = t.emit_warps * 32;
    t.rows = std::min<u32>(EMIT_ROWS_MAX, std::max<u32>(1, (u32)(((u64)n + (u64)nW * per_row - 1) / ((u64)nW * per_row))));
    t.chunk = per_row * t.rows;
    t.P = (n + t.chunk - 1) / t.chunk;
    t.g_smem = ((size_t)t.emit_warps * t.G * 4 + (size_t)t.G * sizeof(GroupOut) + seg_cache <= 192 * 1024) ? 1 : 0;
    size_t emit_smem = (size_t)t.emit_warps * t.G * 4 + (t.g_smem ? (size_t)t.G * sizeof(GroupOut) : 0) + seg_cache;
    // staged finishing pass (EmitSmem): + a 16-byte run record per group (+ one), a 4-byte slot and a 2-byte run place per
    // task of the chunk.  Read on every tick, so that a test can compare both passes in one process.
    const bool no_stage = getenv("HQS_DEBUG_EMIT_PER_TASK") != nullptr;     // measuring / testing aid: the per-task pass
    const size_t stage_smem = ((emit_smem + 15) & ~(size_t)15) + ((size_t)t.G + 1) * 16 + (size_t)t.chunk * 6;
    t.emit_stage = (t.g_smem && !no_stage && stage_smem <= 192 * 1024) ? 1 : 0;
    if (t.emit_stage) emit_smem = stage_smem;
    const size_t pack_smem = (size_t)TICK_WARPS * PACK_MAX_CAND * sizeof(double);
    t.worker_smem = std::max(std::max(emit_smem, pack_smem), (size_t)t.G * 4);
    return t;
}

int ensure_tickin(hqs_ctx* ctx, size_t bytes) {
    if (bytes <= ctx->tickin_cap) return HQS_OK;
    CU(cudaStreamSynchronize(ctx->stream));
    if (ctx->d_tickin) CU(cudaFree(ctx->d_tickin));
    if (ctx->h_tickin) CU(cudaFreeHost(ctx->h_tickin));
    ctx->d_tickin = nullptr; ctx->h_tickin = nullptr;
    ctx->tickin_cap = bytes * 2;
    CU(cudaMalloc(&ctx->d_tickin, ctx->tickin_cap));
    CU(cudaHostAlloc(&ctx->h_tickin, ctx->tickin_cap, cudaHostAllocMapped));
    CU(cudaHostGetDevicePointer(reinterpret_cast<void**>(&ctx->h_tickin_dev), ctx->h_tickin, 0));
    return HQS_OK;
}

// Fills the pinned staging buffer with the tick's worker state and orders.  The solver CTA reads it in place (mapped
// host memory, overlapped with the histogram of the worker CTAs); only the blocked mask, which the pack warps read
// with scattered byte loads, is copied to the device.
int upload_tick_input(hqs_ctx* ctx, u32 W, const hqs_worker* workers, const u64* free_rw, const u64* total_rw,
                      const uint8_t* blocked, TickLayout* lay_out, bool* has_mu, bool* any_time) {
    const u32 R = ctx->R, Q = ctx->Q;
    const bool pfwc = ctx->pf_max && ctx->prefilled_W == W && ctx->prefilled_wc.size() == (size_t)W * Q;
    const TickLayout lay = tick_layout(W, R, Q, blocked != nullptr, pfwc);
    int rc = ensure_tickin(ctx, lay.bytes);
    if (rc) return rc;
    unsigned char* h = ctx->h_tickin;
    memcpy(h + lay.off_free, free_rw, (size_t)W * R * 8);
    memcpy(h + lay.off_total, total_rw, (size_t)W * R * 8);
    // narrow solver: every worker amount of this tick must fit 31 bits after the per-resource scaling
    static const bool force_wide = getenv("HQS_DEBUG_WIDE") != nullptr;
    bool narrow = ctx->narrow_classes && !force_wide && !ctx->force_wide;
    if (narrow) {
        u64 over = 0;
        for (u32 w = 0; w < W; ++w)
            for (u32 r = 0; r < R; ++r) {
                const u64 f = free_rw[(size_t)w * R + r], t = total_rw[(size_t)w * R + r], lim = ctx->narrow_limit[r];
                over |= (u64)(f != HQS_AMOUNT_MAX && f > lim) | (u64)(t != HQS_AMOUNT_MAX && t > lim);
            }
        narrow = over == 0;
    }
    ctx->tick_narrow = narrow;
    ctx->stats.narrow_amounts = narrow ? 1 : 0;
    u64* rem = reinterpret_cast<u64*>(h + lay.off_rem);
    float* mu = reinterpret_cast<float*>(h + lay.off_mu);
    bool mu_any = false, time_any = false;
    for (u32 w = 0; w < W; ++w) {
        rem[w] = workers[w].remaining_time_ms;
        time_any |= rem[w] != HQS_TIME_INF;
        mu[w] = workers[w].min_utilization;
        mu_any |= mu[w] > 0.001f;
    }
    tick_orders(ctx, W, free_rw, total_rw, reinterpret_cast<u32*>(h + lay.off_order), h + lay.off_vorder);
    if (blocked) {
        // ABI bit index ((w*Q + c) * HQS_MAX_VARIANTS + v) with HQS_MAX_VARIANTS == 8: one byte per (w, c)
        memcpy(h + lay.off_blocked, blocked, (size_t)W * Q);
    }
    if (pfwc) memcpy(h + lay.off_pfwc, ctx->prefilled_wc.data(), (size_t)W * Q);
    ctx->h_small[11] = pfwc ? 1u : 0u;
    if (!ctx->zero_copy) CU(cudaMemcpyAsync(ctx->d_tickin, h, lay.bytes, cudaMemcpyHostToDevice, ctx->stream));
    else if (blocked || pfwc) CU(cudaMemcpyAsync(ctx->d_tickin + lay.off_blocked, h + lay.off_blocked, lay.bytes - lay.off_blocked, cudaMemcpyHostToDevice, ctx->stream));
    *lay_out = lay;
    *has_mu = mu_any;
    *any_time = time_any;
    ctx->h_small[9] = mu_any ? 1u : 0u;
    ctx->h_small[10] = time_any ? 1u : 0u;
    return HQS_OK;
}

int validate_workers(hqs_ctx* ctx, u32 W, const hqs_worker* workers, const u64* free_rw, const u64* total_rw) {
    if (!workers || !free_rw || !total_rw) return fail(ctx, HQS_E_INVALID, "null worker arrays");
    if (W == 0 || W > HQS_MAX_WORKERS) return fail(ctx, HQS_E_LIMIT, "n_workers=%u outside 1..%u", W, HQS_MAX_WORKERS);
    for (u32 w = 1; w < W; ++w)
        if (workers[w].worker_id <= workers[w - 1].worker_id)
            return fail(ctx, HQS_E_INVALID, "workers must be sorted by ascending unique worker_id");
    if (ctx->Q == 0) return fail(ctx, HQS_E_STATE, "hqs_classes_set has not been called");
    return HQS_OK;
}

// maxima of two u32 arrays, eight independent accumulators each (the compiler turns them into vector max)
void max_of_u32_pair(const u32* a, const u32* b, u32 n, u32* max_a, u32* max_b) {
    u32 ma[8] = {0, 0, 0, 0, 0, 0, 0, 0}, mb[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    u32 i = 0;
    for (; i + 8 <= n; i += 8)
        for (u32 j = 0; j < 8; ++j) {
            ma[j] = a[i + j] > ma[j] ? a[i + j] : ma[j];
            mb[j] = b[i + j] > mb[j] ? b[i + j] : mb[j];
        }
    for (; i < n; ++i) {
        ma[0] = a[i] > ma[0] ? a[i] : ma[0];
        mb[0] = b[i] > mb[0] ? b[i] : mb[0];
    }
    for (u32 j = 1; j < 8; ++j) { ma[0] = ma[j] > ma[0] ? ma[j] : ma[0]; mb[0] = mb[j] > mb[0] ? mb[j] : mb[0]; }
    *max_a = ma[0];
    *max_b = mb[0];
}

const void* tick_fn(u32 RT, bool narrow) {
#define HQS_PICK(AT) (RT == 4 ? (const void*)tick_k<4, AT> : RT == 8 ? (const void*)tick_k<8, AT> : (const void*)tick_k<16, AT>)
    return narrow ? HQS_PICK(u32) : HQS_PICK(u64);
#undef HQS_PICK
}

TickArgs base_args(hqs_ctx* ctx, const TickGeom& t, u32 W, const TickLayout& lay, bool blocked) {
    TickArgs a;
    memset(&a, 0, sizeof a);
    const unsigned char* in = ctx->zero_copy ? ctx->h_tickin_dev : ctx->d_tickin;
    a.free_rw = reinterpret_cast<const u64*>(in + lay.off_free);
    a.total_rw = reinterpret_cast<const u64*>(in + lay.off_total);
    a.rem_time = reinterpret_cast<const u64*>(in + lay.off_rem);
    a.order = reinterpret_cast<const u32*>(in + lay.off_order);
    a.vorder = in + lay.off_vorder;
    a.blocked = blocked ? ctx->d_tickin + lay.off_blocked : nullptr;
    a.min_util = ctx->h_small[9] ? reinterpret_cast<const float*>(in + lay.off_mu) : nullptr;
    a.any_time_limit = ctx->h_small[10];
    const bool narrow = ctx->tick_narrow;
    a.classes = narrow ? ctx->d_classes32 : ctx->d_classes;
    a.classes64 = ctx->d_classes;
    for (u32 r = 0; r < HQS_MAX_RESOURCES; ++r) a.gscale[r] = ctx->gscale[r] ? ctx->gscale[r] : 1;
    a.W = W; a.Q = ctx->Q; a.L = t.L; a.R = ctx->R; a.G = t.G;
    a.classes_bytes = ctx->Q * (narrow ? ctx->class_bytes32 : ctx->class_bytes);
    a.key = ctx->d_key; a.n_handles = ctx->n_handles; a.chunk = t.chunk; a.rows = t.rows; a.P = t.P; a.nbits = t.nbits;
    a.emit_warps = t.emit_warps; a.g_smem = t.g_smem; a.emit_stage = t.emit_stage;
    a.total_local = ctx->d_total;
    a.table = ctx->d_table;
    a.gout = ctx->d_gout;
    a.seg_cum = ctx->d_seg_cum; a.seg_wv = ctx->d_seg_wv;
    a.free_after = ctx->d_free_after;
    a.hdr = ctx->d_hdr;
    a.hdr_host = reinterpret_cast<TickHeaderOut*>(ctx->h_hdr_dev);
    a.out = ctx->d_out;
    a.rem_scratch = ctx->d_rem_scratch;
    a.sync = ctx->d_sync;
    a.pk.fr = ctx->d_pk_fr; a.pk.quota = ctx->d_pk_quota; a.pk.taken = ctx->d_pk_taken;
    a.pk.cand = ctx->d_pk_cand; a.pk.meta = ctx->d_pk_meta;
    a.excl_glob = ctx->d_excl;
    a.pf_shift = ctx->pf_max ? 1 : 0; a.pf_reserve = ctx->pf_reserve; a.pf_max = ctx->pf_max;
    a.prefilled_wc = ctx->h_small[11] ? ctx->d_tickin + lay.off_pfwc : nullptr;
    a.gout2 = ctx->d_gout2; a.pf_cum = ctx->d_pf_cum; a.pf_wk = ctx->d_pf_wk;
    return a;
}

// shared-memory layout of the solver CTA: mandatory arrays first, then the optional ones while they fit
size_t solver_layout(const hqs_ctx* ctx, TickArgs& a, size_t budget, bool sharded) {
    const u32 W = a.W, Q = a.Q, RT = ctx->RT;
    const size_t at = ctx->tick_narrow ? 4 : 8;
    const u32 n_pos = (a.L * Q) << a.pf_shift;
    size_t o = 0;
    auto put = [&](size_t bytes) { const size_t at_ = o; o = (o + bytes + 15) & ~size_t(15); return (u32)at_; };
    a.sm.fr = put((size_t)W * RT * at);
    a.sm.unt = put((size_t)W * 4);
    a.sm.remtime = put((size_t)W * 8);
    a.sm.excl = put(W);
    a.sm.touch = put(W);
    a.sm.td = put((size_t)W * 2);
    a.sm.frontier = put((size_t)Q * 2);
    a.sm.noresv = put(Q);
    a.sm.glist = put((size_t)n_pos * 8);
    a.sm.gcl = put((size_t)n_pos * 4);
    a.sm.kk = a.sm.top = a.sm.pflvl = SM_NONE;
    if (a.pf_shift) { a.sm.kk = put((size_t)n_pos * 4); a.sm.top = put((size_t)Q * 4); a.sm.pflvl = put((size_t)Q * 4); }
    auto opt = [&](size_t bytes, bool wanted) -> u32 {
        if (!wanted || o + bytes + 16 > budget) return SM_NONE;
        return put(bytes);
    };
    a.sm.classes = opt(a.classes_bytes, true);
    a.sm.vorder = opt((size_t)Q * HQS_MAX_VARIANTS, true);
    a.sm.rem = opt((size_t)W * RT * 8, ctx->tick_narrow);
    a.sm.blocked = opt((size_t)W * Q, a.blocked != nullptr);
    a.sm.bef = opt((size_t)n_pos * 4, sharded);
    a.sm.loc = a.sm.bef != SM_NONE ? opt((size_t)n_pos * 4, sharded) : SM_NONE;
    if (a.sm.loc == SM_NONE) a.sm.bef = SM_NONE;
    a.smem_solver = (u32)o;
    return o;
}

// Launches the tick kernel.  counts: nullptr (count inside the kernel), or host-provided totals (NCCL variant, the
// histogram was taken by hqs_shard_count).  emit = false: what-if query (nothing is emitted or consumed).
int launch_tick(hqs_ctx* ctx, const TickGeom& t, u32 W, const TickLayout& lay, bool blocked, const u32* d_counts_all,
                const u32* d_before, u32 out_cap, bool emit, bool exchange) {
    TickArgs a = base_args(ctx, t, W, lay, blocked);
    a.out_cap = out_cap;
    static const bool no_refresh = getenv("HQS_DEBUG_NO_REFRESH") != nullptr;   // measuring aid: frontiers are not refreshed after a pack
    static const bool no_wide = getenv("HQS_DEBUG_NO_WIDE") != nullptr;         // measuring aid: plain ticks use the one-warp lean loop
    a.flags = (d_counts_all ? 0u : TF_COUNT) | (emit ? TF_EMIT : 0u) | (ctx->pack ? TF_PACK : 0u) | (no_refresh ? TF_NO_REFRESH : 0u) |
              (no_wide ? TF_NO_WIDE : 0u);
    a.total_ext = d_counts_all;
    a.before_ext = d_before;
    if (exchange) {
        for (u32 r = 0; r < HQS_MAX_PEERS; ++r) a.x_peer[r] = r < ctx->x_world ? ctx->x_peer[r] : nullptr;
        a.x_world = ctx->x_world; a.x_rank = ctx->x_rank; a.x_seq = ctx->x_seq;
        a.x_all = ctx->d_xall; a.x_before = ctx->d_xbefore;
    }
    const void* fn = tick_fn(ctx->RT, ctx->tick_narrow);
    const size_t budget = ctx->smem_budget[ctx->tick_narrow ? 0 : 1];
    const size_t solver_smem = solver_layout(ctx, a, budget, exchange || d_before != nullptr);
    const size_t smem = std::max(solver_smem, t.worker_smem);
    if (smem > budget) return fail(ctx, HQS_E_LIMIT, "tick needs %zu bytes of shared memory, %zu available", smem, budget);
    if (ctx->sync_dirty) {
        CU(cudaMemsetAsync(ctx->d_sync, 0, sizeof(TickSync), ctx->stream));
        ctx->sync_dirty = false;
    }
    ctx->ev_valid = false;
    if (ctx->profile) CU(cudaEventRecord(ctx->ev[0], ctx->stream));
    void* kargs[] = {&a};
    static const bool no_coop = getenv("HQS_DEBUG_NO_COOP") != nullptr;   // profiling aid: some ncu versions skip cooperative launches
    if (no_coop) CU(cudaLaunchKernel(fn, dim3(ctx->grid_ctas), dim3(TICK_THREADS), kargs, smem, ctx->stream));
    else CU(cudaLaunchCooperativeKernel(fn, dim3(ctx->grid_ctas), dim3(TICK_THREADS), kargs, smem, ctx->stream));
    ctx->stats.kernel_launches++;
    CU(cudaGetLastError());
    if (ctx->profile) { CU(cudaEventRecord(ctx->ev[3], ctx->stream)); ctx->ev_valid = true; }
    ctx->last_W = W; ctx->last_G = t.G; ctx->last_L = t.L;
    return HQS_OK;
}

// waits for the tick kernel and reads the header the kernel wrote into the pinned mirror
int wait_header(hqs_ctx* ctx, TickHeaderOut* hdr) {
    CU(cudaStreamSynchronize(ctx->stream));
    memcpy(hdr, ctx->h_hdr, sizeof *hdr);
    ctx->stats.n_groups = hdr->n_groups;
    ctx->stats.n_levels = ctx->last_L;
    ctx->stats.n_assigned = hdr->n_assigned;
    ctx->stats.n_segments = hdr->n_segments;
    ctx->stats.solver_path = hdr->solver_path;
    memcpy(ctx->dbg, hdr->dbg, sizeof ctx->dbg);
    if (ctx->profile && ctx->ev_valid) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[3]) == cudaSuccess && hdr->dbg[5]) {
            const double cyc = (double)hdr->dbg[5];
            ctx->last_ms[0] = (float)(ms * (double)hdr->dbg[0] / cyc);
            ctx->last_ms[1] = (float)(ms * (double)(hdr->dbg[1] + hdr->dbg[2]) / cyc);
            ctx->last_ms[2] = (float)(ms * (double)hdr->dbg[3] / cyc);
            ctx->last_ms[3] = ms;
        }
    }
    if (hdr->error) ctx->sync_dirty = true;
    if (hdr->error == 2) {
        const u32 d = hdr->pad & 0xFFu, peer = hdr->pad >> 8;
        return fail(ctx, HQS_E_CUDA, "a grid synchronisation of the tick kernel timed out (%s%s%u; stage %llu, exchange+compact %llu cycles)",
                    d == 21 ? "the histogram of the worker CTAs" : d == 22 ? "count vector of peer rank " : d == 23 ? "the pack step" :
                    d == 24 ? "the emit step" : "a worker CTA waiting for the solver", d == 22 ? "" : ", code ", d == 22 ? peer : d,
                    (unsigned long long)hdr->dbg[0], (unsigned long long)hdr->dbg[1]);
    }
    if (hdr->error == 1) return fail(ctx, HQS_E_LIMIT, "count-segment overflow (> %u segments in one tick)", SEG_CAP);
    if (hdr->error == 4)
        return fail(ctx, HQS_E_STATE, "sharded tick: this rank has G=%u groups, rank %u has G=%u (the number of levels, the classes and "
                    "the proactive-filling setting must agree on every rank); nothing was scheduled", ctx->last_G, (hdr->pad2 >> 16) & 0x7FFFu,
                    hdr->pad2 & 0xFFFFu);
    return HQS_OK;
}

// What a query needs beyond a tick, set up by the first query or by hqs_tick_reserve (so ticks alone never pay for it): the
// pinned per-worker counters and seg_worker_totals_k.  A page-locked allocation and a kernel's lazy load at its first launch
// can synchronise the device, which would dead-lock a fused query waiting there for a peer context of this process: such
// contexts reserve before their first query, as before their first tick.
int ensure_query_buffers(hqs_ctx* ctx) {
    if (ctx->h_pw) return HQS_OK;
    cudaFuncAttributes fa;
    CU(cudaFuncGetAttributes(&fa, (const void*)seg_worker_totals_k));
    CU(cudaMallocHost(&ctx->h_pw, HQS_MAX_WORKERS * sizeof(u32)));
    return HQS_OK;
}

// What-if query: the tick kernel without its emit step (nothing is emitted or consumed), then the per-worker task counts of
// its count segments into the pinned buffer hqs_query_fetch reads.  Like a tick, the query is pending until it is fetched.
// counts_all / exchange as for launch_tick (a query has no local share, so no ranks_before).
int launch_query(hqs_ctx* ctx, const TickGeom& t, u32 W, const TickLayout& lay, bool blocked, const u32* d_counts_all,
                 bool exchange) {
    int rc = ensure_query_buffers(ctx);
    if (rc) return rc;
    rc = launch_tick(ctx, t, W, lay, blocked, d_counts_all, nullptr, 0, false, exchange);
    if (rc) return rc;
    u32* d_pw = ctx->d_pk_quota;    // scratch (pack is over): [W] counters
    CU(cudaMemsetAsync(d_pw, 0, W * sizeof(u32), ctx->stream));
    seg_worker_totals_k<<<(t.G + 127) / 128, 128, 0, ctx->stream>>>(ctx->d_gout, t.G, ctx->d_seg_cum, ctx->d_seg_wv, d_pw);
    ctx->stats.kernel_launches++;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(ctx->h_pw, d_pw, W * sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
    ctx->tick_pending = true;
    ctx->query_pending = true;
    return HQS_OK;
}

// shared body of hqs_query (exchange = false) and hqs_shard_query_launch: validation, tick input, launch
int query_launch_impl(hqs_ctx* ctx, u32 n_workers, const hqs_worker* workers, const u64* free_rw, const u64* total_rw,
                      const uint8_t* blocked_wcv, bool exchange) {
    int rc = validate_workers(ctx, n_workers, workers, free_rw, total_rw);
    if (rc) return rc;
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    CU(cudaSetDevice(ctx->device));
    const TickGeom t = tick_geom(ctx);
    if (t.G > HQS_MAX_GROUPS) return fail(ctx, HQS_E_LIMIT, "groups=%u > %u", t.G, HQS_MAX_GROUPS);
    if ((rc = ensure_tick_buffers(ctx, t.G, t.P, n_workers, 1024))) return rc;
    TickLayout lay;
    bool has_mu, any_time;
    if ((rc = upload_tick_input(ctx, n_workers, workers, free_rw, total_rw, blocked_wcv, &lay, &has_mu, &any_time))) return rc;
    // ticks and queries share one exchange sequence: every rank advances it in lockstep
    if (exchange) ctx->x_seq += 1;
    return launch_query(ctx, t, n_workers, lay, blocked_wcv != nullptr, nullptr, exchange);
}

// Per-worker grouping (hqs_group.cuh).  Like the query's extras, its buffers and kernels are set up by the first grouped fetch
// or by hqs_grouped_reserve, so a context that only fetches flat allocates and loads what it always did.
constexpr u32 GRP_KEYS_MAX = 2 * HQS_MAX_WORKERS + 1;

int ensure_group_buffers(hqs_ctx* ctx, u32 W, u32 cap) {
    if (!ctx->d_grp_small) {
        cudaFuncAttributes fa;
        CU(cudaFuncGetAttributes(&fa, (const void*)group_count_k));
        CU(cudaFuncGetAttributes(&fa, (const void*)group_scan_k));
        CU(cudaFuncGetAttributes(&fa, (const void*)group_scatter_k));
        CU(cudaFuncSetAttribute((const void*)group_scatter_k, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)group_scatter_smem(HQS_MAX_WORKERS)));
        CU(cudaMallocHost(&ctx->h_grp_off, (GRP_KEYS_MAX + 1) * sizeof(u32)));
        CU(cudaMalloc(&ctx->d_grp_small, (2 * GRP_KEYS_MAX + 2) * sizeof(u32)));
        CU(cudaMemsetAsync(ctx->d_grp_small, 0, (2 * GRP_KEYS_MAX + 2) * sizeof(u32), ctx->stream));   // the ticket starts at 0
    }
    if (cap > ctx->grp_cap) {
        CU(cudaStreamSynchronize(ctx->stream));
        if (ctx->d_grp_out) CU(cudaFree(ctx->d_grp_out));
        ctx->d_grp_out = nullptr;
        ctx->grp_cap = std::max<u32>(cap, 1024);
        CU(cudaMalloc(&ctx->d_grp_out, (size_t)ctx->grp_cap * sizeof(hqs_assignment)));
    }
    const size_t need = (size_t)(2 * W + 1) * ((ctx->grp_cap + GROUP_TILE - 1) / GROUP_TILE);
    if (need > ctx->grp_hist_cap) {
        CU(cudaStreamSynchronize(ctx->stream));
        if (ctx->d_grp_hist) CU(cudaFree(ctx->d_grp_hist));
        ctx->d_grp_hist = nullptr;
        ctx->grp_hist_cap = need;
        CU(cudaMalloc(&ctx->d_grp_hist, need * sizeof(u32)));
    }
    return HQS_OK;
}

// d_out[0..n) -> d_grp_out grouped by worker, offset table behind the key totals in d_grp_small
int launch_grouping(hqs_ctx* ctx, u32 n, u32 W) {
    const u32 K = 2 * W + 1, T = (n + GROUP_TILE - 1) / GROUP_TILE;
    u32* d_tot = ctx->d_grp_small;
    u32* d_off = d_tot + GRP_KEYS_MAX;
    u32* d_ticket = d_off + GRP_KEYS_MAX + 1;
    const bool timed = ctx->profile && ctx->ev[1];
    if (timed) CU(cudaEventRecord(ctx->ev[1], ctx->stream));
    group_count_k<<<T, GROUP_THREADS, K * sizeof(u32), ctx->stream>>>(ctx->d_out, n, W, T, ctx->d_grp_hist);
    group_scan_k<<<(K + GROUP_SCAN_THREADS / 32 - 1) / (GROUP_SCAN_THREADS / 32), GROUP_SCAN_THREADS, 0, ctx->stream>>>(
        ctx->d_grp_hist, K, T, d_tot, d_off, d_ticket);
    group_scatter_k<<<T, GROUP_THREADS, group_scatter_smem(W), ctx->stream>>>(ctx->d_out, n, W, T, ctx->d_grp_hist, d_off,
                                                                            ctx->d_grp_out);
    ctx->stats.kernel_launches += 3;
    CU(cudaGetLastError());
    if (timed) CU(cudaEventRecord(ctx->ev[2], ctx->stream));
    return HQS_OK;
}

// shared body of hqs_tick_fetch (worker_off == nullptr) and hqs_tick_fetch_grouped
int tick_fetch_impl(hqs_ctx* ctx, u32 out_cap, hqs_assignment* out, u32* out_n, u64* free_after, u32* worker_off) {
    if (out_n) *out_n = 0;
    CU(cudaSetDevice(ctx->device));
    ctx->tick_pending = false;
    ctx->prefilled_wc.clear(); ctx->prefilled_W = 0;             // the mirror is per tick, whether the tick succeeded or not
    TickHeaderOut hdr;
    int rc = wait_header(ctx, &hdr);
    if (rc) return rc;
    // error 3: the solver saw that out_cap is too small BEFORE the emit step: nothing was emitted, the ready set is intact
    const u32 n_rec = hdr.n_assigned + hdr.n_prefilled;           // assignments (kind 0 / 2), then prefills (kind 1)
    if (hdr.error == 3 || n_rec > out_cap || (n_rec && !out))
        return fail(ctx, HQS_E_OVERFLOW, "out_cap=%u too small for %u assignments + %u prefills", out_cap, hdr.n_assigned, hdr.n_prefilled);
    if (free_after) memcpy(free_after, ctx->h_hdr + sizeof(TickHeaderOut), (size_t)ctx->last_W * ctx->R * 8);
    const u32 W = ctx->last_W, n_off = 2 * W + 2;
    if (worker_off) memset(worker_off, 0, n_off * sizeof(u32));
    if (n_rec && !worker_off) {
        CU(cudaMemcpyAsync(out, ctx->d_out, (size_t)n_rec * sizeof(hqs_assignment), cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
    } else if (n_rec) {
        // n and the error word are known here, so the grids are exact and a failed tick never reaches this point
        ctx->grp_ms = -1.f;
        if ((rc = ensure_group_buffers(ctx, W, std::max(n_rec, ctx->out_cap_dev)))) return rc;
        if ((rc = launch_grouping(ctx, n_rec, W))) return rc;
        CU(cudaMemcpyAsync(out, ctx->d_grp_out, (size_t)n_rec * sizeof(hqs_assignment), cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaMemcpyAsync(ctx->h_grp_off, ctx->d_grp_small + GRP_KEYS_MAX, n_off * sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        memcpy(worker_off, ctx->h_grp_off, n_off * sizeof(u32));
        if (ctx->profile && ctx->ev[1] && cudaEventElapsedTime(&ctx->grp_ms, ctx->ev[1], ctx->ev[2]) != cudaSuccess) ctx->grp_ms = -1.f;
    }
    if (out_n) *out_n = n_rec;
    return HQS_OK;
}

}  // namespace

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" {

int hqs_abi_version(void) { return HQS_ABI_VERSION; }

const char* hqs_last_error(const hqs_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int hqs_create(hqs_ctx** out, int device, uint32_t n_resources, uint32_t flags) {
    hqs_ctx* ctx = nullptr;
    if (!out) return fail(nullptr, HQS_E_INVALID, "out is null");
    *out = nullptr;
    if (n_resources == 0 || n_resources > HQS_MAX_RESOURCES)
        return fail(nullptr, HQS_E_LIMIT, "n_resources=%u outside 1..%u", n_resources, HQS_MAX_RESOURCES);
    int n_dev = 0;
    cudaError_t e = cudaGetDeviceCount(&n_dev);
    if (e != cudaSuccess || n_dev == 0)
        return fail(nullptr, HQS_E_CUDA, "no CUDA device available (%s); this library has no CPU fallback",
                    cudaGetErrorString(e));
    if (device < 0 || device >= n_dev) return fail(nullptr, HQS_E_INVALID, "device %d out of range", device);
    ctx = new (std::nothrow) hqs_ctx();
    if (!ctx) return fail(nullptr, HQS_E_NOMEM, "out of memory");
    ctx->device = device;
    ctx->R = n_resources;
    ctx->RT = n_resources <= 4 ? 4 : n_resources <= 8 ? 8 : 16;
    ctx->class_bytes = ctx->RT == 4 ? sizeof(ClassT<4>) : ctx->RT == 8 ? sizeof(ClassT<8>) : sizeof(ClassT<16>);
    ctx->class_bytes32 = ctx->RT == 4 ? sizeof(ClassT<4, u32>) : ctx->RT == 8 ? sizeof(ClassT<8, u32>) : sizeof(ClassT<16, u32>);
    ctx->pack = !(flags & 1u);
    ctx->force_wide = (flags & 2u) != 0;
    e = cudaSetDevice(device);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
    int sms = 0;
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_newcnt, 2 * sizeof(u32));
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_newprio, NEWPRIO_CAP * sizeof(u64));
    if (e == cudaSuccess) e = cudaMallocHost(&ctx->h_small, 64 * sizeof(u32));
    {
        const void* fns[] = {(const void*)tick_k<4, u32>, (const void*)tick_k<8, u32>, (const void*)tick_k<16, u32>,
                             (const void*)tick_k<4, u64>, (const void*)tick_k<8, u64>, (const void*)tick_k<16, u64>};
        // dynamic + static shared memory of a CTA may not exceed 227 KB: allow each instance what its statics leave
        for (const void* f : fns) {
            cudaFuncAttributes fa;
            if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, f);
            if (e == cudaSuccess) {
                const size_t room = 227 * 1024 - fa.sharedSizeBytes;
                e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::min<size_t>(room, 216 * 1024));
            }
        }
    }
    if (e != cudaSuccess) {
        fail(nullptr, HQS_E_CUDA, "context setup failed: %s", cudaGetErrorString(e));
        delete ctx;
        return HQS_E_CUDA;
    }
    ctx->sm_count = sms > 0 ? (u32)sms : 132;
    // one CTA per SM (cooperative launch: all CTAs are co-resident).  HQS_CREATE_SHARE_DEVICE: half of the SMs, so
    // that two contexts whose ticks wait for each other on the device (peer exchange) can run side by side on one GPU
    ctx->grid_ctas = std::max<u32>(2, (flags & 4u) ? ctx->sm_count / 2 : ctx->sm_count);
    {
        static const bool copy_in = getenv("HQS_DEBUG_COPY_INPUT") != nullptr;   // debugging aid: H2D copy instead of reading pinned memory in place
        int can_map = 0;
        cudaDeviceGetAttribute(&can_map, cudaDevAttrCanMapHostMemory, device);
        ctx->zero_copy = can_map != 0 && !copy_in;
    }
    for (int nw = 0; nw < 2; ++nw) {
        cudaFuncAttributes fa;
        if (cudaFuncGetAttributes(&fa, tick_fn(ctx->RT, nw == 0)) == cudaSuccess) ctx->smem_budget[nw] = (size_t)fa.maxDynamicSharedSizeBytes;
    }
    *out = ctx;
    return HQS_OK;
}

void hqs_destroy(hqs_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    void* dev_ptrs[] = {ctx->d_classes, ctx->d_classes32, ctx->d_levels, ctx->d_key, ctx->d_prio, ctx->d_deps, ctx->d_cons_off,
                        ctx->d_cons, ctx->d_push_task, ctx->d_push_cls, ctx->d_push_prio, ctx->d_newcnt,
                        ctx->d_newprio, ctx->d_table, ctx->d_total, ctx->d_gout, ctx->d_rem_scratch, ctx->d_excl, ctx->d_gout2, ctx->d_pf_cum, ctx->d_pf_wk, ctx->d_seg_cum,
                        ctx->d_seg_wv, ctx->d_out, ctx->d_hdr, ctx->d_free_after, ctx->d_tickin, ctx->d_sync, ctx->d_pk_fr,
                        ctx->d_pk_quota, ctx->d_pk_taken, ctx->d_pk_cand, ctx->d_pk_meta, ctx->d_prune_lv, ctx->d_prune_live};
    for (void* p : dev_ptrs) if (p) cudaFree(p);
    for (void* p : ctx->x_opened) cudaIpcCloseMemHandle(p);
    if (ctx->d_xbuf) cudaFree(ctx->d_xbuf);
    if (ctx->d_xall) cudaFree(ctx->d_xall);
    if (ctx->d_xbefore) cudaFree(ctx->d_xbefore);
    if (ctx->h_tickin) cudaFreeHost(ctx->h_tickin);
    if (ctx->h_hdr) cudaFreeHost(ctx->h_hdr);
    if (ctx->h_small) cudaFreeHost(ctx->h_small);
    if (ctx->h_pw) cudaFreeHost(ctx->h_pw);
    if (ctx->d_grp_out) cudaFree(ctx->d_grp_out);
    if (ctx->d_grp_hist) cudaFree(ctx->d_grp_hist);
    if (ctx->d_grp_small) cudaFree(ctx->d_grp_small);
    if (ctx->h_grp_off) cudaFreeHost(ctx->h_grp_off);
    for (cudaEvent_t e : ctx->ev) if (e) cudaEventDestroy(e);
    if (ctx->stream && ctx->own_stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

int hqs_classes_set(hqs_ctx* ctx, uint32_t n_classes, const hqs_class* classes) {
    if (!ctx) return HQS_E_INVALID;
    if (!classes || n_classes == 0) return fail(ctx, HQS_E_INVALID, "empty class table");
    if (n_classes > HQS_MAX_CLASSES) return fail(ctx, HQS_E_LIMIT, "n_classes=%u > %u", n_classes, HQS_MAX_CLASSES);
    // device layout: ClassT<RT>[Q] with RT = 4 / 8 / 16 resource slots, built as raw bytes
    const u32 RT = ctx->RT;
    const size_t var_bytes = RT == 4 ? sizeof(VarT<4>) : RT == 8 ? sizeof(VarT<8>) : sizeof(VarT<16>), cls_bytes = ctx->class_bytes;
    std::vector<unsigned char> blob((size_t)n_classes * cls_bytes, 0);
    for (u32 c = 0; c < n_classes; ++c) {
        const hqs_class& sc = classes[c];
        if (sc.n_nodes != 0) return fail(ctx, HQS_E_INVALID, "class %u: multi-node requests are outside this path", c);
        if (sc.n_variants == 0 || sc.n_variants > HQS_MAX_VARIANTS)
            return fail(ctx, HQS_E_LIMIT, "class %u: n_variants=%u outside 1..%u", c, sc.n_variants, HQS_MAX_VARIANTS);
        unsigned char* cb = blob.data() + (size_t)c * cls_bytes;
        memcpy(cb, &sc.n_variants, 4);
        for (u32 v = 0; v < sc.n_variants; ++v) {
            const hqs_variant& hv = sc.variants[v];
            for (u32 r = ctx->R; r < HQS_MAX_RESOURCES; ++r)
                if (((hv.all_mask >> r) & 1) || hv.amount[r])
                    return fail(ctx, HQS_E_INVALID, "class %u variant %u uses resource %u >= n_resources", c, v, r);
            unsigned char* vb = cb + 8 + (size_t)v * var_bytes;
            u32 used;
            if (RT == 4) { pack_var64<4>(*reinterpret_cast<VarT<4>*>(vb), hv, ctx->R); used = reinterpret_cast<VarT<4>*>(vb)->used_mask; }
            else if (RT == 8) { pack_var64<8>(*reinterpret_cast<VarT<8>*>(vb), hv, ctx->R); used = reinterpret_cast<VarT<8>*>(vb)->used_mask; }
            else { pack_var64<16>(*reinterpret_cast<VarT<16>*>(vb), hv, ctx->R); used = reinterpret_cast<VarT<16>*>(vb)->used_mask; }
            if (!used) return fail(ctx, HQS_E_INVALID, "class %u variant %u: empty request (request.rs:191-194)", c, v);
            if (hv.weight == 0) return fail(ctx, HQS_E_INVALID, "class %u variant %u: zero weight", c, v);
        }
    }
    CU(cudaSetDevice(ctx->device));
    if (blob.size() > ctx->d_classes_cap) {
        CU(cudaStreamSynchronize(ctx->stream));
        if (ctx->d_classes) CU(cudaFree(ctx->d_classes));
        ctx->d_classes_cap = (u32)std::max<size_t>(blob.size() * 2, 4096);
        CU(cudaMalloc(&ctx->d_classes, ctx->d_classes_cap));
    }
    CU(cudaMemcpyAsync(ctx->d_classes, blob.data(), blob.size(), cudaMemcpyHostToDevice, ctx->stream));
    // narrow copy: amounts divided by the per-resource gcd of everything requested
    u64 gs[HQS_MAX_RESOURCES];
    for (u32 r = 0; r < HQS_MAX_RESOURCES; ++r) gs[r] = 0;
    for (u32 c = 0; c < n_classes; ++c)
        for (u32 v = 0; v < classes[c].n_variants; ++v)
            for (u32 r = 0; r < ctx->R; ++r)
                if (!((classes[c].variants[v].all_mask >> r) & 1) && classes[c].variants[v].amount[r])
                    gs[r] = std::gcd(gs[r], (u64)classes[c].variants[v].amount[r]);
    bool narrow_ok = true;
    const size_t var_bytes32 = RT == 4 ? sizeof(VarT<4, u32>) : RT == 8 ? sizeof(VarT<8, u32>) : sizeof(VarT<16, u32>), cls_bytes32 = ctx->class_bytes32;
    std::vector<unsigned char> blob32((size_t)n_classes * cls_bytes32, 0);
    for (u32 r = 0; r < HQS_MAX_RESOURCES; ++r) {
        if (gs[r] == 0) gs[r] = 1;
        ctx->gscale[r] = gs[r];
        ctx->narrow_limit[r] = gs[r] > HQS_AMOUNT_MAX / NARROW_LIMIT ? HQS_AMOUNT_MAX - 1 : gs[r] * NARROW_LIMIT;
    }
    for (u32 c = 0; c < n_classes && narrow_ok; ++c) {
        const hqs_class& sc = classes[c];
        unsigned char* cb = blob32.data() + (size_t)c * cls_bytes32;
        memcpy(cb, &sc.n_variants, 4);
        for (u32 v = 0; v < sc.n_variants; ++v) {
            unsigned char* vb = cb + 8 + (size_t)v * var_bytes32;
            const bool ok = RT == 4 ? pack_var32<4>(*reinterpret_cast<VarT<4, u32>*>(vb), sc.variants[v], ctx->R, gs)
                          : RT == 8 ? pack_var32<8>(*reinterpret_cast<VarT<8, u32>*>(vb), sc.variants[v], ctx->R, gs)
                                    : pack_var32<16>(*reinterpret_cast<VarT<16, u32>*>(vb), sc.variants[v], ctx->R, gs);
            narrow_ok &= ok;
        }
    }
    ctx->narrow_classes = narrow_ok;
    if (blob32.size() > ctx->d_classes32_cap) {
        CU(cudaStreamSynchronize(ctx->stream));
        if (ctx->d_classes32) CU(cudaFree(ctx->d_classes32));
        ctx->d_classes32_cap = (u32)std::max<size_t>(blob32.size() * 2, 4096);
        CU(cudaMalloc(&ctx->d_classes32, ctx->d_classes32_cap));
    }
    CU(cudaMemcpyAsync(ctx->d_classes32, blob32.data(), blob32.size(), cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    const bool q_changed = ctx->Q != n_classes;
    ctx->classes.assign(classes, classes + n_classes);
    ctx->Q = n_classes;
    if (q_changed && !ctx->levels.empty()) {
        // the level budget depends on Q: re-derive (possibly coarsened) levels and re-key the table
        const bool was_coarse = ctx->coarse;
        const size_t old_n = ctx->dev_levels.size();
        bool dropped = false;
        int rc = HQS_OK;
        if (levels_need_pruning(ctx) && (rc = prune_levels(ctx, &dropped))) return rc;
        if ((rc = upload_levels(ctx))) return rc;
        if (dropped || was_coarse || ctx->coarse || old_n != ctx->dev_levels.size())
            if ((rc = relevel_all(ctx))) return rc;
    }
    return HQS_OK;
}

namespace {
// shared body of hqs_ready_push / hqs_ready_push_range (task == nullptr: handles first_handle .. first_handle + n - 1)
int push_impl(hqs_ctx* ctx, u32 n, const u32* task, u32 first_handle, const u32* class_id, const u64* priority) {
    if (ctx->Q == 0) return fail(ctx, HQS_E_STATE, "hqs_classes_set has not been called");
    if (ctx->dag) return fail(ctx, HQS_E_STATE, "hqs_ready_push is not available after hqs_dag_load");
    CU(cudaSetDevice(ctx->device));
    if (n > ctx->push_cap) {
        CU(cudaStreamSynchronize(ctx->stream));
        if (ctx->d_push_task) { CU(cudaFree(ctx->d_push_task)); CU(cudaFree(ctx->d_push_cls)); CU(cudaFree(ctx->d_push_prio)); }
        ctx->push_cap = std::max<u32>(n, 1u << 16);
        CU(cudaMalloc(&ctx->d_push_task, (size_t)ctx->push_cap * 4));
        CU(cudaMalloc(&ctx->d_push_cls, (size_t)ctx->push_cap * 4));
        CU(cudaMalloc(&ctx->d_push_prio, (size_t)ctx->push_cap * 8));
    }
    if (task) CU(cudaMemcpyAsync(ctx->d_push_task, task, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->d_push_cls, class_id, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->d_push_prio, priority, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
    // the table must hold the largest handle before the kernel runs: a host pass over the handle array while the staging
    // copies are in flight (a range push knows it); class ids are validated on the device (push_validate_k)
    u32 max_h = first_handle + (n - 1);
    if (task) {
        u32 dummy = 0;
        max_of_u32_pair(task, task, n, &max_h, &dummy);
    } else if (max_h < first_handle) {
        max_h = ~0u;                                                  // the range wraps around
    }
    if (max_h == ~0u) {
        cudaStreamSynchronize(ctx->stream);      // the caller may free its arrays as soon as we return
        return fail(ctx, HQS_E_INVALID, "task handle 0xFFFFFFFF is reserved");
    }
    int rc = ensure_handles(ctx, max_h + 1);
    if (rc) { cudaStreamSynchronize(ctx->stream); return rc; }
    CU(cudaMemsetAsync(ctx->d_newcnt, 0, 2 * sizeof(u32), ctx->stream));
    push_validate_k<<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, ctx->d_push_cls, ctx->Q, ctx->d_newcnt);
    push_k<<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, task ? ctx->d_push_task : nullptr, first_handle, ctx->d_push_cls,
                                                     ctx->d_push_prio, ctx->d_key, ctx->d_prio, ctx->d_levels,
                                                     (u32)ctx->dev_levels.size(), ctx->coarse ? 1 : 0, ctx->d_newcnt, ctx->d_newprio);
    ctx->stats.kernel_launches += 2;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(ctx->h_small, ctx->d_newcnt, 2 * sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
    // a coarse table has a bucket for every priority, so push_k reports none as fresh: the batch's priorities are
    // collected here, while the kernels run, and registered like fresh ones (the level set keeps growing, gets pruned
    // and leaves coarse mode once the live priorities fit again).  Exact-mode pushes do not take this pass.
    std::vector<u64> fresh;
    if (ctx->coarse) distinct_priorities(priority, n, fresh);
    CU(cudaStreamSynchronize(ctx->stream));
    if (ctx->h_small[1]) return fail(ctx, HQS_E_INVALID, "a class id of the batch is >= n_classes %u (nothing was pushed)", ctx->Q);
    ctx->n_handles = std::max(ctx->n_handles, max_h + 1);
    ctx->stats.n_handles = ctx->n_handles;
    const u32 newcnt = ctx->h_small[0];
    bool grew = false;
    if (ctx->coarse) {
        grew = merge_levels(ctx, fresh);
    } else if (newcnt) {
        if (newcnt <= NEWPRIO_CAP) {
            fresh.resize(newcnt);
            CU(cudaMemcpy(fresh.data(), ctx->d_newprio, newcnt * sizeof(u64), cudaMemcpyDeviceToHost));
        } else {
            distinct_priorities(priority, n, fresh);
        }
        grew = merge_levels(ctx, fresh);
    }
    if (grew) {
        if (levels_need_pruning(ctx)) {
            bool dropped = false;
            if ((rc = prune_levels(ctx, &dropped))) return rc;
        }
        if ((rc = upload_levels(ctx))) return rc;
        if ((rc = relevel_all(ctx))) return rc;
    }
    return HQS_OK;
}
}  // namespace

int hqs_ready_push(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t* class_id,
                   const uint64_t* priority) {
    if (!ctx) return HQS_E_INVALID;
    if (n == 0) return HQS_OK;
    if (!task || !class_id || !priority) return fail(ctx, HQS_E_INVALID, "null task arrays");
    return push_impl(ctx, n, task, 0, class_id, priority);
}

int hqs_ready_push_range(hqs_ctx* ctx, uint32_t first_task, uint32_t n, const uint32_t* class_id, const uint64_t* priority) {
    if (!ctx) return HQS_E_INVALID;
    if (n == 0) return HQS_OK;
    if (!class_id || !priority) return fail(ctx, HQS_E_INVALID, "null task arrays");
    return push_impl(ctx, n, nullptr, first_task, class_id, priority);
}

int hqs_levels_add(hqs_ctx* ctx, uint32_t n, const uint64_t* priority) {
    if (!ctx) return HQS_E_INVALID;
    if (n == 0) return HQS_OK;
    if (!priority) return fail(ctx, HQS_E_INVALID, "null priority array");
    CU(cudaSetDevice(ctx->device));
    std::vector<u64> fresh;
    distinct_priorities(priority, n, fresh);
    ctx->levels_declared = true;
    if (!merge_levels(ctx, fresh)) return HQS_OK;
    int rc = upload_levels(ctx);
    if (rc) return rc;
    return relevel_all(ctx);
}

int hqs_ready_remove(hqs_ctx* ctx, uint32_t n, const uint32_t* task) {
    if (!ctx) return HQS_E_INVALID;
    if (n == 0) return HQS_OK;
    if (!task) return fail(ctx, HQS_E_INVALID, "null task array");
    CU(cudaSetDevice(ctx->device));
    if (n > ctx->push_cap) {
        CU(cudaStreamSynchronize(ctx->stream));
        if (ctx->d_push_task) { CU(cudaFree(ctx->d_push_task)); CU(cudaFree(ctx->d_push_cls)); CU(cudaFree(ctx->d_push_prio)); }
        ctx->push_cap = std::max<u32>(n, 1u << 16);
        CU(cudaMalloc(&ctx->d_push_task, (size_t)ctx->push_cap * 4));
        CU(cudaMalloc(&ctx->d_push_cls, (size_t)ctx->push_cap * 4));
        CU(cudaMalloc(&ctx->d_push_prio, (size_t)ctx->push_cap * 8));
    }
    CU(cudaMemcpyAsync(ctx->d_push_task, task, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    remove_k<<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, ctx->d_push_task, ctx->d_key, ctx->n_handles);
    ctx->stats.kernel_launches++;
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(ctx->stream));
    return HQS_OK;
}

int hqs_prefill_config(hqs_ctx* ctx, uint32_t reserve, uint32_t max_per_worker) {
    if (!ctx) return HQS_E_INVALID;
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    ctx->pf_reserve = reserve;
    ctx->pf_max = max_per_worker;
    return HQS_OK;
}

int hqs_prefill_state(hqs_ctx* ctx, uint32_t n_workers, const uint8_t* prefilled_wc) {
    if (!ctx) return HQS_E_INVALID;
    if (!prefilled_wc || n_workers == 0) { ctx->prefilled_wc.clear(); ctx->prefilled_W = 0; return HQS_OK; }
    if (ctx->Q == 0) return fail(ctx, HQS_E_STATE, "hqs_classes_set has not been called");
    ctx->prefilled_wc.assign(prefilled_wc, prefilled_wc + (size_t)n_workers * ctx->Q);
    ctx->prefilled_W = n_workers;
    return HQS_OK;
}

int hqs_prefill_dispose(hqs_ctx* ctx, uint32_t class_id) {
    if (!ctx) return HQS_E_INVALID;
    if (class_id >= ctx->Q) return fail(ctx, HQS_E_INVALID, "class id %u >= n_classes %u", class_id, ctx->Q);
    if (!ctx->n_handles) return HQS_OK;
    CU(cudaSetDevice(ctx->device));
    pf_dispose_k<<<(ctx->n_handles + 255) / 256, 256, 0, ctx->stream>>>(ctx->n_handles, ctx->d_key, class_id);
    ctx->stats.kernel_launches++;
    CU(cudaGetLastError());
    return HQS_OK;
}

int hqs_ready_rearm(hqs_ctx* ctx) {
    if (!ctx) return HQS_E_INVALID;
    if (!ctx->n_handles) return HQS_OK;
    CU(cudaSetDevice(ctx->device));
    rearm_k<<<(ctx->n_handles + 255) / 256, 256, 0, ctx->stream>>>(ctx->n_handles, ctx->d_key);
    ctx->stats.kernel_launches++;
    CU(cudaGetLastError());
    return HQS_OK;
}

int hqs_dag_load(hqs_ctx* ctx, uint32_t n_tasks, const uint32_t* class_id, const uint64_t* priority,
                 const uint32_t* n_deps, const uint32_t* cons_off, const uint32_t* cons) {
    if (!ctx) return HQS_E_INVALID;
    if (!n_tasks || !class_id || !priority || !n_deps || !cons_off) return fail(ctx, HQS_E_INVALID, "null DAG arrays");
    if (ctx->Q == 0) return fail(ctx, HQS_E_STATE, "hqs_classes_set has not been called");
    const u32 n_edges = cons_off[n_tasks];
    if (n_edges && !cons) return fail(ctx, HQS_E_INVALID, "null consumer array");
    for (u32 i = 0; i < n_tasks; ++i)
        if (class_id[i] >= ctx->Q) return fail(ctx, HQS_E_INVALID, "class id %u >= n_classes %u", class_id[i], ctx->Q);
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_handles(ctx, n_tasks);
    if (rc) return rc;
    CU(cudaStreamSynchronize(ctx->stream));
    if (ctx->d_deps) { CU(cudaFree(ctx->d_deps)); ctx->d_deps = nullptr; }
    if (ctx->d_cons_off) { CU(cudaFree(ctx->d_cons_off)); ctx->d_cons_off = nullptr; }
    if (ctx->d_cons) { CU(cudaFree(ctx->d_cons)); ctx->d_cons = nullptr; }
    u32* d_cls = nullptr;
    CU(cudaMalloc(&ctx->d_deps, (size_t)n_tasks * 4));
    CU(cudaMalloc(&ctx->d_cons_off, ((size_t)n_tasks + 1) * 4));
    CU(cudaMalloc(&ctx->d_cons, std::max<size_t>(n_edges, 1) * 4));
    CU(cudaMalloc(&d_cls, (size_t)n_tasks * 4));
    CU(cudaMemsetAsync(ctx->d_key, 0, (size_t)ctx->cap_handles * 4, ctx->stream));
    CU(cudaMemcpyAsync(ctx->d_deps, n_deps, (size_t)n_tasks * 4, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->d_cons_off, cons_off, ((size_t)n_tasks + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
    if (n_edges) CU(cudaMemcpyAsync(ctx->d_cons, cons, (size_t)n_edges * 4, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(d_cls, class_id, (size_t)n_tasks * 4, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->d_prio, priority, (size_t)n_tasks * 8, cudaMemcpyHostToDevice, ctx->stream));
    std::vector<u64> fresh;
    distinct_priorities(priority, n_tasks, fresh);
    ctx->levels.clear();
    merge_levels(ctx, fresh);
    if ((rc = upload_levels(ctx))) { cudaFree(d_cls); return rc; }
    ctx->n_handles = n_tasks;
    ctx->stats.n_handles = n_tasks;
    dag_init_k<<<(n_tasks + 255) / 256, 256, 0, ctx->stream>>>(n_tasks, d_cls, ctx->d_prio, ctx->d_deps, ctx->d_key,
                                                               ctx->d_levels, (u32)ctx->dev_levels.size(),
                                                               ctx->coarse ? 1 : 0);
    ctx->stats.kernel_launches++;
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(ctx->stream));
    CU(cudaFree(d_cls));
    ctx->dag = true;
    return HQS_OK;
}

int hqs_tasks_finished(hqs_ctx* ctx, uint32_t n, const uint32_t* task, uint32_t* n_new_ready) {
    if (!ctx) return HQS_E_INVALID;
    if (n_new_ready) *n_new_ready = 0;
    if (!ctx->dag) return fail(ctx, HQS_E_STATE, "hqs_tasks_finished needs hqs_dag_load");
    if (n == 0) return HQS_OK;
    if (!task) return fail(ctx, HQS_E_INVALID, "null task array");
    CU(cudaSetDevice(ctx->device));
    if (n > ctx->push_cap) {
        CU(cudaStreamSynchronize(ctx->stream));
        if (ctx->d_push_task) { CU(cudaFree(ctx->d_push_task)); CU(cudaFree(ctx->d_push_cls)); CU(cudaFree(ctx->d_push_prio)); }
        ctx->push_cap = std::max<u32>(n, 1u << 16);
        CU(cudaMalloc(&ctx->d_push_task, (size_t)ctx->push_cap * 4));
        CU(cudaMalloc(&ctx->d_push_cls, (size_t)ctx->push_cap * 4));
        CU(cudaMalloc(&ctx->d_push_prio, (size_t)ctx->push_cap * 8));
    }
    CU(cudaMemcpyAsync(ctx->d_push_task, task, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemsetAsync(ctx->d_newcnt, 0, sizeof(u32), ctx->stream));
    finished_k<<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, ctx->d_push_task, ctx->d_cons_off, ctx->d_cons, ctx->d_deps,
                                                         ctx->d_key, ctx->d_newcnt);
    ctx->stats.kernel_launches++;
    CU(cudaGetLastError());
    if (n_new_ready) {
        CU(cudaMemcpyAsync(ctx->h_small, ctx->d_newcnt, sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        *n_new_ready = ctx->h_small[0];
    }
    return HQS_OK;
}

int hqs_tick_launch(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
                    const uint64_t* total_rw, const uint8_t* blocked_wcv, uint32_t out_cap) {
    if (!ctx) return HQS_E_INVALID;
    int rc = validate_workers(ctx, n_workers, workers, free_rw, total_rw);
    if (rc) return rc;
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    CU(cudaSetDevice(ctx->device));
    const TickGeom t = tick_geom(ctx);
    if (t.G > HQS_MAX_GROUPS) return fail(ctx, HQS_E_LIMIT, "groups=%u > %u", t.G, HQS_MAX_GROUPS);
    if ((rc = ensure_tick_buffers(ctx, t.G, t.P, n_workers, out_cap))) return rc;
    TickLayout lay;
    bool has_mu, any_time;
    if ((rc = upload_tick_input(ctx, n_workers, workers, free_rw, total_rw, blocked_wcv, &lay, &has_mu, &any_time))) return rc;
    if ((rc = launch_tick(ctx, t, n_workers, lay, blocked_wcv != nullptr, nullptr, nullptr, out_cap, true, false))) return rc;
    ctx->tick_pending = true;
    ctx->stats.ticks++;
    return HQS_OK;
}

int hqs_tick_fetch(hqs_ctx* ctx, uint32_t out_cap, hqs_assignment* out, uint32_t* out_n, uint64_t* free_after) {
    if (!ctx) return HQS_E_INVALID;
    if (!ctx->tick_pending) return fail(ctx, HQS_E_STATE, "no tick in flight");
    if (ctx->query_pending) return fail(ctx, HQS_E_STATE, "a query is in flight: fetch it with hqs_query_fetch");
    return tick_fetch_impl(ctx, out_cap, out, out_n, free_after, nullptr);
}

int hqs_tick_fetch_grouped(hqs_ctx* ctx, uint32_t out_cap, hqs_assignment* out, uint32_t* out_n, uint32_t off_cap,
                           uint32_t* worker_off, uint64_t* free_after) {
    if (!ctx) return HQS_E_INVALID;
    if (!ctx->tick_pending) return fail(ctx, HQS_E_STATE, "no tick in flight");
    if (ctx->query_pending) return fail(ctx, HQS_E_STATE, "a query is in flight: fetch it with hqs_query_fetch");
    // checked before the tick is consumed: it stays fetchable
    if (!worker_off || off_cap < 2 * ctx->last_W + 2)
        return fail(ctx, HQS_E_INVALID, "worker_off needs 2 * n_workers + 2 = %u entries (off_cap=%u)", 2 * ctx->last_W + 2, off_cap);
    return tick_fetch_impl(ctx, out_cap, out, out_n, free_after, worker_off);
}

int hqs_tick_grouped(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
                     const uint64_t* total_rw, const uint8_t* blocked_wcv, uint32_t out_cap, hqs_assignment* out,
                     uint32_t* out_n, uint32_t off_cap, uint32_t* worker_off, uint64_t* free_after) {
    if (!ctx) return HQS_E_INVALID;
    if (!worker_off || (uint64_t)off_cap < 2 * (uint64_t)n_workers + 2)
        return fail(ctx, HQS_E_INVALID, "worker_off needs 2 * n_workers + 2 entries (off_cap=%u)", off_cap);
    int rc = hqs_tick_launch(ctx, n_workers, workers, free_rw, total_rw, blocked_wcv, out_cap);
    if (rc) return rc;
    return hqs_tick_fetch_grouped(ctx, out_cap, out, out_n, off_cap, worker_off, free_after);
}

int hqs_grouped_reserve(hqs_ctx* ctx, uint32_t n_workers, uint32_t out_cap) {
    if (!ctx) return HQS_E_INVALID;
    if (n_workers == 0 || n_workers > HQS_MAX_WORKERS) return fail(ctx, HQS_E_LIMIT, "n_workers=%u outside 1..%u", n_workers, HQS_MAX_WORKERS);
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_group_buffers(ctx, n_workers, std::max(out_cap, ctx->out_cap_dev));
    if (rc) return rc;
    CU(cudaStreamSynchronize(ctx->stream));
    return HQS_OK;
}

int hqs_grouped_kernel_ms(hqs_ctx* ctx, float* out_ms) {
    if (!ctx || !out_ms) return HQS_E_INVALID;
    if (ctx->grp_ms < 0) return fail(ctx, HQS_E_STATE, "no profiled grouped fetch available");
    *out_ms = ctx->grp_ms;
    return HQS_OK;
}

int hqs_tick(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
             const uint64_t* total_rw, const uint8_t* blocked_wcv, uint32_t out_cap, hqs_assignment* out,
             uint32_t* out_n, uint64_t* free_after) {
    int rc = hqs_tick_launch(ctx, n_workers, workers, free_rw, total_rw, blocked_wcv, out_cap);
    if (rc) return rc;
    return hqs_tick_fetch(ctx, out_cap, out, out_n, free_after);
}

int hqs_query(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
              const uint64_t* total_rw, const uint8_t* blocked_wcv, uint32_t* n_would_assign,
              uint32_t* per_worker_assigned, uint64_t* free_after) {
    if (!ctx) return HQS_E_INVALID;
    if (n_would_assign) *n_would_assign = 0;
    const int rc = query_launch_impl(ctx, n_workers, workers, free_rw, total_rw, blocked_wcv, false);
    if (rc) return rc;
    return hqs_query_fetch(ctx, n_would_assign, per_worker_assigned, free_after);
}

int hqs_query_fetch(hqs_ctx* ctx, uint32_t* n_would_assign, uint32_t* per_worker_assigned, uint64_t* free_after) {
    if (!ctx) return HQS_E_INVALID;
    if (n_would_assign) *n_would_assign = 0;
    if (!ctx->tick_pending) return fail(ctx, HQS_E_STATE, "no query in flight");
    if (!ctx->query_pending) return fail(ctx, HQS_E_STATE, "a tick is in flight: fetch it with hqs_tick_fetch");
    CU(cudaSetDevice(ctx->device));
    ctx->tick_pending = false;
    ctx->query_pending = false;
    TickHeaderOut hdr;
    const int rc = wait_header(ctx, &hdr);
    if (rc) return rc;
    if (free_after) memcpy(free_after, ctx->h_hdr + sizeof(TickHeaderOut), (size_t)ctx->last_W * ctx->R * 8);
    // the count segments cover every group's assigned ranks [0, k), so the per-worker counts sum to the tasks assigned over
    // all ranks; the header's n_assigned of a sharded launch is this rank's share only (the solver's local output offsets)
    u32 total = 0;
    for (u32 w = 0; w < ctx->last_W; ++w) total += ctx->h_pw[w];
    ctx->stats.n_assigned = total;
    if (n_would_assign) *n_would_assign = total;
    if (per_worker_assigned) memcpy(per_worker_assigned, ctx->h_pw, ctx->last_W * sizeof(u32));
    return HQS_OK;
}

int hqs_shard_count(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
                    const uint64_t* total_rw, const uint8_t* blocked_wcv, uint32_t* d_counts, uint32_t n_groups_cap,
                    uint32_t* n_groups) {
    if (!ctx) return HQS_E_INVALID;
    int rc = validate_workers(ctx, n_workers, workers, free_rw, total_rw);
    if (rc) return rc;
    if (!d_counts) return fail(ctx, HQS_E_INVALID, "null d_counts");
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    CU(cudaSetDevice(ctx->device));
    const TickGeom t = tick_geom(ctx);
    if (t.G > HQS_MAX_GROUPS) return fail(ctx, HQS_E_LIMIT, "groups=%u > %u", t.G, HQS_MAX_GROUPS);
    if (t.G > n_groups_cap) return fail(ctx, HQS_E_LIMIT, "groups=%u > n_groups_cap=%u", t.G, n_groups_cap);
    if ((rc = ensure_tick_buffers(ctx, t.G, t.P, n_workers, 1024))) return rc;
    TickLayout lay;
    bool has_mu, any_time;
    if ((rc = upload_tick_input(ctx, n_workers, workers, free_rw, total_rw, blocked_wcv, &lay, &has_mu, &any_time))) return rc;
    CU(cudaMemsetAsync(ctx->d_total, 0, (size_t)t.G * 4, ctx->stream));
    if (ctx->n_handles) {
        TickArgs a = base_args(ctx, t, n_workers, lay, blocked_wcv != nullptr);
        count_only_k<<<std::min<u32>(t.P, ctx->sm_count * 2), TICK_THREADS, t.G * sizeof(u32), ctx->stream>>>(a);
        ctx->stats.kernel_launches++;
        CU(cudaGetLastError());
    }
    CU(cudaMemsetAsync(d_counts, 0, (size_t)n_groups_cap * 4, ctx->stream));
    CU(cudaMemcpyAsync(d_counts, ctx->d_total, (size_t)t.G * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->last_W = n_workers;
    ctx->last_blocked = blocked_wcv != nullptr;
    if (n_groups) *n_groups = t.G;
    return HQS_OK;
}

int hqs_shard_solve_emit(hqs_ctx* ctx, const uint32_t* d_counts_all, const uint32_t* d_ranks_before, uint32_t out_cap) {
    if (!ctx) return HQS_E_INVALID;
    if (!d_counts_all || !d_ranks_before) return fail(ctx, HQS_E_INVALID, "null count vectors");
    if (!ctx->last_W) return fail(ctx, HQS_E_STATE, "hqs_shard_count has not been called");
    CU(cudaSetDevice(ctx->device));
    const TickGeom t = tick_geom(ctx);
    int rc = ensure_tick_buffers(ctx, t.G, t.P, ctx->last_W, out_cap);
    if (rc) return rc;
    // the tick input hqs_shard_count uploaded, prefill mask included (h_small[11] says whether it has one)
    const TickLayout lay = tick_layout(ctx->last_W, ctx->R, ctx->Q, ctx->last_blocked, ctx->h_small[11] != 0);
    if ((rc = launch_tick(ctx, t, ctx->last_W, lay, ctx->last_blocked, d_counts_all, d_ranks_before, out_cap, true, false))) return rc;
    ctx->tick_pending = true;
    ctx->stats.ticks++;
    return HQS_OK;
}

int hqs_tick_reserve(hqs_ctx* ctx, uint32_t n_workers, uint32_t out_cap, int with_blocked) {
    if (!ctx) return HQS_E_INVALID;
    if (n_workers == 0 || n_workers > HQS_MAX_WORKERS) return fail(ctx, HQS_E_LIMIT, "n_workers=%u outside 1..%u", n_workers, HQS_MAX_WORKERS);
    if (ctx->Q == 0) return fail(ctx, HQS_E_STATE, "hqs_classes_set has not been called");
    CU(cudaSetDevice(ctx->device));
    const TickGeom t = tick_geom(ctx);
    if (t.G > HQS_MAX_GROUPS) return fail(ctx, HQS_E_LIMIT, "groups=%u > %u", t.G, HQS_MAX_GROUPS);
    int rc = ensure_tick_buffers(ctx, t.G, t.P, n_workers, out_cap);
    if (rc) return rc;
    const TickLayout lay = tick_layout(n_workers, ctx->R, ctx->Q, with_blocked != 0, ctx->pf_max != 0);   // + the prefill mask
    if ((rc = ensure_tickin(ctx, lay.bytes))) return rc;
    if ((rc = ensure_query_buffers(ctx))) return rc;
    CU(cudaStreamSynchronize(ctx->stream));
    return HQS_OK;
}

// exchange buffer: count vectors [parity][rank][HQS_MAX_GROUPS], release flags [parity][rank], group counts G [parity][rank]
// (checked by the solver CTA: every rank runs the same library build, so the layout agrees)
static size_t xbuf_bytes() { return ((size_t)2 * HQS_MAX_PEERS * HQS_MAX_GROUPS + 4 * HQS_MAX_PEERS) * sizeof(u32); }

int hqs_shard_xbuf(hqs_ctx* ctx, void** d_xbuf, uint8_t ipc_handle[HQS_IPC_HANDLE_BYTES]) {
    if (!ctx) return HQS_E_INVALID;
    CU(cudaSetDevice(ctx->device));
    if (!ctx->d_xbuf) {
        CU(cudaMalloc(&ctx->d_xbuf, xbuf_bytes()));
        CU(cudaMemset(ctx->d_xbuf, 0, xbuf_bytes()));
        CU(cudaMalloc(&ctx->d_xall, HQS_MAX_GROUPS * sizeof(u32)));
        CU(cudaMalloc(&ctx->d_xbefore, HQS_MAX_GROUPS * sizeof(u32)));
    }
    if (d_xbuf) *d_xbuf = ctx->d_xbuf;
    if (ipc_handle) {
        static_assert(sizeof(cudaIpcMemHandle_t) == HQS_IPC_HANDLE_BYTES, "IPC handle size");
        cudaIpcMemHandle_t h;
        CU(cudaIpcGetMemHandle(&h, ctx->d_xbuf));
        memcpy(ipc_handle, &h, sizeof h);
    }
    return HQS_OK;
}

int hqs_ipc_open(hqs_ctx* ctx, const uint8_t ipc_handle[HQS_IPC_HANDLE_BYTES], void** d_ptr) {
    if (!ctx || !ipc_handle || !d_ptr) return HQS_E_INVALID;
    CU(cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, ipc_handle, sizeof h);
    void* p = nullptr;
    CU(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    ctx->x_opened.push_back(p);
    *d_ptr = p;
    return HQS_OK;
}

int hqs_shard_attach(hqs_ctx* ctx, uint32_t world, uint32_t rank, void* const* peer_xbufs) {
    if (!ctx || !peer_xbufs) return HQS_E_INVALID;
    if (world < 1 || world > HQS_MAX_PEERS || rank >= world) return fail(ctx, HQS_E_LIMIT, "world=%u rank=%u outside 1..%u", world, rank, HQS_MAX_PEERS);
    if (!ctx->d_xbuf) return fail(ctx, HQS_E_STATE, "hqs_shard_xbuf has not been called");
    if (peer_xbufs[rank] != ctx->d_xbuf) return fail(ctx, HQS_E_INVALID, "peer_xbufs[rank] must be this context's own buffer");
    CU(cudaSetDevice(ctx->device));
    for (u32 r = 0; r < world; ++r) {
        if (!peer_xbufs[r]) return fail(ctx, HQS_E_INVALID, "peer %u has no buffer", r);
        ctx->x_peer[r] = static_cast<u32*>(peer_xbufs[r]);
        // a buffer of another device of THIS process needs peer access (IPC mappings were opened with it)
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, peer_xbufs[r]) == cudaSuccess && at.type == cudaMemoryTypeDevice && at.device != ctx->device) {
            const cudaError_t e = cudaDeviceEnablePeerAccess(at.device, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
                return fail(ctx, HQS_E_CUDA, "no peer access from device %d to device %d: %s", ctx->device, at.device, cudaGetErrorString(e));
        }
        cudaGetLastError();
    }
    ctx->x_world = world; ctx->x_rank = rank; ctx->x_seq = 0;
    return HQS_OK;
}

int hqs_shard_tick_launch(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
                          const uint64_t* total_rw, const uint8_t* blocked_wcv, uint32_t out_cap) {
    if (!ctx) return HQS_E_INVALID;
    if (!ctx->x_world) return fail(ctx, HQS_E_STATE, "hqs_shard_attach has not been called");
    int rc = validate_workers(ctx, n_workers, workers, free_rw, total_rw);
    if (rc) return rc;
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    CU(cudaSetDevice(ctx->device));
    const TickGeom t = tick_geom(ctx);
    if (t.G > HQS_MAX_GROUPS) return fail(ctx, HQS_E_LIMIT, "groups=%u > %u", t.G, HQS_MAX_GROUPS);
    if ((rc = ensure_tick_buffers(ctx, t.G, t.P, n_workers, out_cap))) return rc;
    TickLayout lay;
    bool has_mu, any_time;
    if ((rc = upload_tick_input(ctx, n_workers, workers, free_rw, total_rw, blocked_wcv, &lay, &has_mu, &any_time))) return rc;
    // every rank advances the sequence number in lockstep (one sharded tick = one exchange)
    ctx->x_seq += 1;
    if ((rc = launch_tick(ctx, t, n_workers, lay, blocked_wcv != nullptr, nullptr, nullptr, out_cap, true, true))) return rc;
    ctx->tick_pending = true;
    ctx->stats.ticks++;
    return HQS_OK;
}

int hqs_shard_query_launch(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
                           const uint64_t* total_rw, const uint8_t* blocked_wcv) {
    if (!ctx) return HQS_E_INVALID;
    if (!ctx->x_world) return fail(ctx, HQS_E_STATE, "hqs_shard_attach has not been called");
    return query_launch_impl(ctx, n_workers, workers, free_rw, total_rw, blocked_wcv, true);
}

int hqs_shard_query_solve(hqs_ctx* ctx, const uint32_t* d_counts_all) {
    if (!ctx) return HQS_E_INVALID;
    if (!d_counts_all) return fail(ctx, HQS_E_INVALID, "null count vector");
    if (!ctx->last_W) return fail(ctx, HQS_E_STATE, "hqs_shard_count has not been called");
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    CU(cudaSetDevice(ctx->device));
    const TickGeom t = tick_geom(ctx);
    int rc = ensure_tick_buffers(ctx, t.G, t.P, ctx->last_W, 1024);
    if (rc) return rc;
    // the tick input hqs_shard_count uploaded
    const TickLayout lay = tick_layout(ctx->last_W, ctx->R, ctx->Q, ctx->last_blocked, ctx->h_small[11] != 0);
    return launch_query(ctx, t, ctx->last_W, lay, ctx->last_blocked, d_counts_all, false);
}

int hqs_device_result(hqs_ctx* ctx, const hqs_assignment** d_out, const uint32_t** d_out_n) {
    if (!ctx) return HQS_E_INVALID;
    if (d_out) *d_out = ctx->d_out;
    if (d_out_n) *d_out_n = ctx->d_hdr ? &ctx->d_hdr->n_assigned : nullptr;
    return HQS_OK;
}

void* hqs_stream(hqs_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

int hqs_set_stream(hqs_ctx* ctx, void* cuda_stream) {
    if (!ctx) return HQS_E_INVALID;
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(ctx->stream));
    if (ctx->own_stream && ctx->stream) CU(cudaStreamDestroy(ctx->stream));
    ctx->stream = (cudaStream_t)cuda_stream;
    ctx->own_stream = false;
    return HQS_OK;
}

int hqs_set_profile(hqs_ctx* ctx, int on) {
    if (!ctx) return HQS_E_INVALID;
    CU(cudaSetDevice(ctx->device));
    if (on && !ctx->ev[0])
        for (int i = 0; i < 4; ++i) CU(cudaEventCreate(&ctx->ev[i]));
    ctx->profile = on != 0;
    ctx->ev_valid = false;
    return HQS_OK;
}

int hqs_get_kernel_ms(hqs_ctx* ctx, float out_ms[4]) {
    if (!ctx || !out_ms) return HQS_E_INVALID;
    if (!ctx->profile || !ctx->ev_valid) return fail(ctx, HQS_E_STATE, "no profiled tick available");
    for (int i = 0; i < 4; ++i) out_ms[i] = ctx->last_ms[i];
    return HQS_OK;
}

int hqs_sync(hqs_ctx* ctx) {
    if (!ctx) return HQS_E_INVALID;
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(ctx->stream));
    return HQS_OK;
}

int hqs_debug_read(hqs_ctx* ctx, uint64_t out[8]) {
    if (!ctx || !out) return HQS_E_INVALID;
    for (int i = 0; i < 8; ++i) out[i] = ctx->dbg[i];
    return HQS_OK;
}

int hqs_debug_keys(hqs_ctx* ctx, uint32_t cap, uint32_t* keys, uint32_t* n_handles) {
    if (!ctx) return HQS_E_INVALID;
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    if (cap && !keys) return fail(ctx, HQS_E_INVALID, "null key array");
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(ctx->stream));
    const u32 n = std::min(cap, ctx->n_handles);
    if (n) {
        CU(cudaMemcpyAsync(keys, ctx->d_key, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
    }
    if (n_handles) *n_handles = ctx->n_handles;
    return HQS_OK;
}

int hqs_get_stats(hqs_ctx* ctx, hqs_stats* out) {
    if (!ctx || !out) return HQS_E_INVALID;
    *out = ctx->stats;
    out->n_levels = (u32)ctx->dev_levels.size();
    return HQS_OK;
}

}  // extern "C"
