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
//   gdeps[h], ggen[h], ghead[h] + an edge pool: task graphs grown by hqs_graph_push (hqs_graph.cuh); gwork[h]: the work
//            list of hqs_graph_cancel
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
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <new>
#include <string>
#include <numeric>
#include <vector>

namespace {

typedef uint32_t u32;
typedef uint64_t u64;

#include "hqs_ready_set.cuh"
#include "hqs_solver.cuh"
#include "hqs_graph.cuh"
#include "hqs_tick.cuh"
#include "hqs_group.cuh"


// ================================================================================================
// host side
// ================================================================================================
thread_local std::string g_create_error;

// One owned allocation of n elements of T: device memory (Mem::Dev), page-locked host memory (Mem::Host), or page-locked
// host memory mapped into the device's address space (Mem::Mapped, whose device alias is dev()).  Move-only: what it holds
// is freed when it is destroyed or assigned over.  It converts to T*, so kernel launches take it as a raw pointer.
enum class Mem { Dev, Host, Mapped };

template <typename T, Mem M = Mem::Dev>
class Buf {
    T* p_ = nullptr;
    T* dev_ = nullptr;
    size_t n_ = 0;

public:
    Buf() = default;
    Buf(Buf&& o) noexcept { swap(o); }
    Buf& operator=(Buf&& o) noexcept { Buf(std::move(o)).swap(*this); return *this; }
    ~Buf() {
        if (p_ && M == Mem::Dev) cudaFree(p_);
        else if (p_) cudaFreeHost(p_);
    }
    void swap(Buf& o) noexcept { std::swap(p_, o.p_); std::swap(dev_, o.dev_); std::swap(n_, o.n_); }
    operator T*() const { return p_; }
    T* operator->() const { return p_; }
    T* dev() const { return dev_; }
    size_t size() const { return n_; }

    // Replaces the allocation by one of n elements.  keep: the current elements are copied to its front; fill >= 0: the
    // elements not copied are set to that byte.  The old allocation is freed after `stream` has drained.  On failure the
    // buffer is left as it was.
    cudaError_t grow(size_t n, cudaStream_t stream, bool keep = false, int fill = -1) {
        void* raw = nullptr;
        cudaError_t e = M == Mem::Dev ? cudaMalloc(&raw, n * sizeof(T))
                                      : cudaHostAlloc(&raw, n * sizeof(T), M == Mem::Mapped ? cudaHostAllocMapped : cudaHostAllocDefault);
        if (e != cudaSuccess) return e;
        Buf q;
        q.p_ = static_cast<T*>(raw);
        q.n_ = n;
        const size_t kept = keep ? std::min(n_, n) : 0;
        if (M == Mem::Mapped) e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&q.dev_), raw, 0);
        if (e == cudaSuccess && fill >= 0 && kept < n) {
            if (M == Mem::Dev) e = cudaMemsetAsync(q.p_ + kept, fill, (n - kept) * sizeof(T), stream);
            else memset(q.p_ + kept, fill, (n - kept) * sizeof(T));
        }
        if (e == cudaSuccess && kept) e = cudaMemcpyAsync(q.p_, p_, kept * sizeof(T), cudaMemcpyDefault, stream);
        if (e == cudaSuccess && p_) e = cudaStreamSynchronize(stream);
        if (e == cudaSuccess) swap(q);
        return e;
    }
};

// the tick's fixed-size buffers, set up together by the first call that sizes a tick (ensure_tick_buffers)
struct TickBuffers {
    Buf<u32> seg_cum, seg_wv;                 // [SEG_CAP] count segments
    Buf<TickHeaderOut> hdr;
    Buf<u64> free_after;
    Buf<TickSync> sync;
    Buf<u64> pk_fr; Buf<u32> pk_quota, pk_taken, pk_cand, pk_meta;
    Buf<u32> rem_scratch; Buf<uint8_t> excl;
    Buf<u32> glist;                           // [4][HQS_MAX_GROUPS] the solver's group list when it does not fit shared memory
    Buf<u32> pf_cum, pf_wk;                   // [PF_SEG_CAP] prefill segments
    Buf<unsigned char, Mem::Mapped> h_hdr;    // TickHeaderOut + free_after, written by the kernel
};

struct TickLayout {
    size_t off_free, off_total, off_rem, off_order, off_vorder, off_mu, off_blocked, off_pfwc, bytes;
};

// the tick input upload_tick_input staged last, and what the launches read of it; only upload_tick_input writes it
struct TickInput {
    u32 W;
    TickLayout lay;
    bool blocked, pfwc;         // it has a blocked mask, a prefill mask (proactive filling: the previous tick's prefills)
    bool min_util, any_time;    // some worker has a minimum utilisation, a time limit
    bool narrow;                // the tick runs the narrow solver
};

// the counters the push and graph calls copy back from the device, in page-locked memory
struct HostCounters {
    u32 newcnt, reject;               // d_newcnt: a push's fresh priorities (hqs_tasks_finished: its newly ready tasks), rejection bits
    u32 ready;                        // tasks a graph push made ready at once
    u32 emitted;                      // handles graph_emit_bits emitted (newly ready or cancelled)
    u32 kept, live, own_lo, own_hi;   // a compaction's totals: survivors, live edges, a sharded compaction's new(lo) and new(hi)
};
static_assert(offsetof(HostCounters, reject) == offsetof(HostCounters, newcnt) + 4 &&
              offsetof(HostCounters, own_hi) == offsetof(HostCounters, kept) + 12, "multi-word copies land on adjacent fields");

}  // namespace

struct hqs_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    u32 R = 0;
    std::string err;
    // classes
    u32 Q = 0;
    std::vector<hqs_class> classes;
    Buf<unsigned char> d_classes;         // ClassT<RT, u64>[Q]
    Buf<unsigned char> d_classes32;       // ClassT<RT, u32>[Q]: amounts / gscale[r] (valid when narrow_classes)
    u32 class_bytes32 = 0;                // sizeof(ClassT<RT, u32>)
    u64 gscale[HQS_MAX_RESOURCES] = {};   // per-resource gcd of every requested amount (1 where nothing is requested)
    u64 narrow_limit[HQS_MAX_RESOURCES] = {};   // largest worker amount the narrow path can hold: gscale * (2^31 - 1)
    bool narrow_classes = false;          // every scaled class amount < 2^31
    // peer-to-peer sharded tick
    Buf<u32> d_xbuf;                      // my exchange buffer: [2][HQS_MAX_PEERS][HQS_MAX_GROUPS] counts + [2][HQS_MAX_PEERS] flags
    u32* x_peer[HQS_MAX_PEERS] = {};      // every rank's exchange buffer (own included), set by hqs_shard_attach
    std::vector<void*> x_opened;          // IPC mappings to close
    u32 x_world = 0, x_rank = 0, x_seq = 0;
    Buf<u32> d_xall;                      // [HQS_MAX_GROUPS] sum over ranks, written by the solver
    Buf<u32> d_xbefore;                   // [HQS_MAX_GROUPS] sum over lower ranks
    bool force_wide = false;              // hqs_create flag bit 1: always the 64-bit solver (tests)
    u32 RT = 4;                           // resource slots of the device class layout (4, 8 or 16)
    u32 class_bytes = 0;                  // sizeof(ClassT<RT>)
    // priority levels (descending)
    std::vector<u64> levels;      // exact distinct priorities seen, descending
    std::vector<u64> dev_levels;  // what the device uses (== levels, or bucket bounds when coarsened)
    bool coarse = false;
    bool levels_declared = false;   // hqs_levels_add was used: the caller numbers the levels (sharded ready set), no pruning
    size_t levels_pruned_at = 0;    // size of the level set after the last pruning
    Buf<u64> d_levels;
    Buf<u64> d_prune_lv;            // prune_levels scratch: the exact levels and their live flags
    Buf<u32> d_prune_live;
    // task table
    u32 n_handles = 0, cap_handles = 0;
    Buf<u32> d_key;
    Buf<u64> d_prio;
    Buf<u32> d_deps, d_cons_off, d_cons;
    bool dag = false;
    // task graph (hqs_graph_push / hqs_graph_finished, hqs_graph.cuh): nothing of it exists before the first graph call
    bool graph_storage = false;         // the per-handle arrays below exist and grow with the table
    bool graph = false;                 // a graph push was accepted: hqs_dag_load is refused
    Buf<u32> d_gdeps, d_ggen, d_ghead;
    Buf<u32> d_gbits;                   // [cap_handles / 32] ready bitmap of hqs_graph_finished (zero between calls)
    Buf<u32> d_gready;                  // [cap_handles] the newly ready handles, ascending
    Buf<u32> d_gblk;                    // [cap_handles / GRAPH_PER_BLOCK + 1] per-block sums of the ordered compactions
    Buf<u32> d_gsmall;                  // [4] n_ready of a push, n_new of a finish, live edges of a compaction
    Buf<GraphEdge> d_pool;
    u32 pool_cap = 0, pool_used = 0;    // edge slots; slots [0, pool_used) have been handed out since the last compaction
    u64 pool_compactions = 0;
    Buf<u32> d_gstage;                  // a push's dependency offsets [n + 1] and dependencies
    std::vector<u32> g_off, g_dep;      // host scratch of hqs_graph_push
    std::vector<std::pair<u32, u32>> g_pos;
    std::vector<u32> g_new_ready;       // what *new_ready of hqs_graph_finished / *cancelled of hqs_graph_cancel points to
    Buf<u32> d_gwork;                   // [cap_handles] work list of hqs_graph_cancel's marking (GRAPH_NIL between calls)
    Buf<GraphCancelSync> d_gcsync;
    // sharded graph (hqs_shard_graph_init): the graph arrays above are replicated over the global handles [0, g_total) and
    // keep that size; the key table holds the owned handles [g_lo, g_hi) at h - g_lo
    bool shard_graph = false;
    bool shard_graph_failed = false;    // a sharded graph call failed on the device: this replica may differ from the others
    u32 g_total = 0, g_lo = 0, g_hi = 0;
    Buf<u32> d_gvalid;                  // [g_total / 32] the graph's VALID bits
    // push staging (device)
    Buf<u32> d_push_task, d_push_cls; Buf<u64> d_push_prio;
    Buf<u32> d_newcnt; Buf<u64> d_newprio;
    // tick buffers
    u32 sm_count = 132;
    u32 grid_ctas = 132;                // CTAs of the cooperative tick kernel (solver CTA + worker CTAs)
    u32 G_cap = 0, P_cap = 0;
    Buf<u32> d_table;
    Buf<u32> d_total;
    Buf<GroupOut> d_gout;
    TickBuffers tick;
    size_t smem_budget[2] = {0, 0};     // dynamic shared memory a tick kernel instance may use (narrow, wide)
    bool sync_dirty = true;             // the counters must be zeroed before the next launch (first tick / after a failed one)
    // proactive filling
    u32 pf_reserve = 0, pf_max = 0;     // SchedulerConfig::proactive_filling_reserve / _max (state.rs:14-21); max == 0: off
    Buf<uint4> d_gout2;
    std::vector<uint8_t> prefilled_wc; u32 prefilled_W = 0;   // host mirror for the next tick: [W][Q]
    Buf<hqs_assignment> d_out;
    Buf<unsigned char> d_tickin;        // device copy of the tick input (blocked mask; everything when zero-copy is off)
    Buf<unsigned char, Mem::Mapped> h_tickin;   // the solver CTA reads the worker state from here
    bool zero_copy = true;
    Buf<HostCounters, Mem::Host> h_cnt;
    Buf<u32, Mem::Host> h_pw;           // [HQS_MAX_WORKERS]: per-worker task counts of the last query
    // per-worker grouping of the records (hqs_tick_fetch_grouped); nothing of it exists until the first grouped fetch or
    // hqs_grouped_reserve
    Buf<hqs_assignment> d_grp_out;      // the grouped records
    Buf<u32> d_grp_hist;                // [2W + 1][tiles] counts, then their prefix over the tiles
    Buf<u32> d_grp_small;               // key totals [GRP_KEYS_MAX], offset table [GRP_KEYS_MAX + 1], the scan's ticket
    Buf<u32, Mem::Host> h_grp_off;      // mirror of the offset table
    float grp_ms = -1.f;                // device time of the last grouping (profiling on), < 0: none
    // last tick
    TickInput staged{};
    u32 last_G = 0, last_L = 0;
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

    // the buffers free themselves after this, once the stream has drained
    ~hqs_ctx() {
        if (stream) cudaStreamSynchronize(stream);
        for (void* p : x_opened) cudaIpcCloseMemHandle(p);
        for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
        if (stream && own_stream) cudaStreamDestroy(stream);
    }
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

// The per-handle graph arrays at cap handles, one after the other (their old and new sizes are never all held at once).
// keep: the current entries stay; the new ones start with no dependencies, generation 0, an empty consumer list
// (GRAPH_NIL) and no ready bit.  The cancel work list is GRAPH_NIL throughout.
int size_graph_arrays(hqs_ctx* ctx, u32 cap, bool keep) {
    cudaStream_t s = ctx->stream;
    CU(ctx->d_gdeps.grow(cap, s, keep, 0));
    CU(ctx->d_ggen.grow(cap, s, keep, 0));
    CU(ctx->d_ghead.grow(cap, s, keep, 0xFF));
    CU(ctx->d_gbits.grow(cap / 32, s, keep, 0));
    CU(ctx->d_gready.grow(cap, s));
    CU(ctx->d_gblk.grow(cap / GRAPH_PER_BLOCK + 1, s));
    CU(ctx->d_gwork.grow(cap, s, false, 0xFF));
    return HQS_OK;
}

int ensure_handles(hqs_ctx* ctx, u32 need) {
    if (need <= ctx->cap_handles) return HQS_OK;
    u32 cap = std::max<u32>(need, std::max<u32>(ctx->cap_handles * 2, 1u << 16));
    cap = (cap + 1023u) & ~1023u;
    CU(ctx->d_key.grow(cap, ctx->stream, true, 0));
    CU(ctx->d_prio.grow(cap, ctx->stream, true, 0));
    if (ctx->graph_storage && !ctx->shard_graph)
        if (int rc = size_graph_arrays(ctx, cap, true)) return rc;
    ctx->cap_handles = cap;
    return HQS_OK;
}

// the per-handle graph arrays, at the table's current capacity (ensure_handles grows them from then on), or over the global
// handles of a sharded graph context
int ensure_graph_storage(hqs_ctx* ctx) {
    if (ctx->graph_storage) return HQS_OK;
    const u32 cap = ctx->shard_graph ? (ctx->g_total + 1023u) & ~1023u : ctx->cap_handles;
    if (!ctx->d_gsmall) CU(ctx->d_gsmall.grow(4, ctx->stream));
    if (!ctx->d_gcsync) CU(ctx->d_gcsync.grow(1, ctx->stream));
    if (int rc = size_graph_arrays(ctx, cap, false)) return rc;
    ctx->graph_storage = true;
    return HQS_OK;
}

// device staging of a batch's handles (and class ids / priorities) for the ready-set calls
int ensure_push_staging(hqs_ctx* ctx, u32 n) {
    const u32 cap = std::max<u32>(n, 1u << 16);
    if (n > ctx->d_push_task.size()) CU(ctx->d_push_task.grow(cap, ctx->stream));
    if (n > ctx->d_push_cls.size()) CU(ctx->d_push_cls.grow(cap, ctx->stream));
    if (n > ctx->d_push_prio.size()) CU(ctx->d_push_prio.grow(cap, ctx->stream));
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
    if (n > ctx->d_levels.size()) CU(ctx->d_levels.grow(std::max<u32>(n * 2, 64), ctx->stream));
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

// For every exact level of ctx->levels, whether a VALID key carries its priority (one level_live_k pass over the table).
int live_levels(hqs_ctx* ctx, std::vector<u32>& live) {
    const u32 L = (u32)ctx->levels.size();
    live.assign(L, 0);
    if (L == 0 || ctx->n_handles == 0) return HQS_OK;
    // scratch kept across calls: a coarse table is pruned on every push that brings a new priority, and freeing would
    // synchronise the device each time
    if (L > ctx->d_prune_lv.size()) CU(ctx->d_prune_lv.grow(std::max<u32>(L * 2, 4096), ctx->stream));
    if (L > ctx->d_prune_live.size()) CU(ctx->d_prune_live.grow(std::max<u32>(L * 2, 4096), ctx->stream));
    u64* d_lv = ctx->d_prune_lv;
    u32* d_live = ctx->d_prune_live;
    CU(cudaMemsetAsync(d_live, 0, (size_t)L * 4, ctx->stream));
    CU(cudaMemcpyAsync(d_lv, ctx->levels.data(), (size_t)L * 8, cudaMemcpyHostToDevice, ctx->stream));
    level_live_k<<<(ctx->n_handles + 255) / 256, 256, 0, ctx->stream>>>(ctx->n_handles, ctx->d_key, ctx->d_prio, d_lv, L, d_live);
    ctx->stats.kernel_launches++;
    CU(cudaMemcpyAsync(live.data(), d_live, (size_t)L * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return HQS_OK;
}

// Drops the priority levels no task of the table carries any more (tako priorities have a per-job component, so a
// long-running server sees one level per job ever submitted).  Called when the level set is about to exceed what the
// group limit allows, or has doubled since the last pruning.  Returns true if levels were dropped (the caller then
// uploads the table and re-keys the tasks).  Declared levels are pruned by the caller, over all ranks
// (hqs_levels_live / hqs_levels_retain).
int prune_levels(hqs_ctx* ctx, bool* changed) {
    *changed = false;
    const u32 L = (u32)ctx->levels.size();
    if (ctx->levels_declared || L == 0 || ctx->n_handles == 0) return HQS_OK;
    std::vector<u32> live;
    int rc = live_levels(ctx, live);
    if (rc) return rc;
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

int ensure_tick_buffers(hqs_ctx* ctx, u32 G, u32 P, u32 out_cap) {
    if (G > ctx->G_cap || P > ctx->P_cap || (size_t)G * P > (size_t)ctx->G_cap * ctx->P_cap) {
        const u32 ng = std::max(G, ctx->G_cap), np = std::max(P, ctx->P_cap);
        cudaStream_t s = ctx->stream;
        CU(ctx->d_table.grow((size_t)ng * np, s));
        if (ng > ctx->G_cap) {
            CU(ctx->d_total.grow(ng, s, false, 0));
            CU(ctx->d_gout.grow(ng, s, false, 0));
            CU(ctx->d_gout2.grow(ng, s, false, 0));
        }
        ctx->G_cap = ng; ctx->P_cap = np;
    }
    if (!ctx->tick.hdr) {
        const size_t wr = (size_t)HQS_MAX_WORKERS * HQS_MAX_RESOURCES;
        const size_t wc = (size_t)HQS_MAX_WORKERS * PACK_MAX_CAND;
        cudaStream_t s = ctx->stream;
        TickBuffers b;
        CU(b.seg_cum.grow(SEG_CAP, s));
        CU(b.seg_wv.grow(SEG_CAP, s));
        CU(b.hdr.grow(1, s));
        CU(b.free_after.grow(wr, s));
        CU(b.sync.grow(1, s));
        CU(b.pk_fr.grow(wr, s));
        CU(b.pk_quota.grow(wc, s));
        CU(b.pk_taken.grow(wc, s));
        CU(b.pk_cand.grow(PACK_MAX_CAND, s));
        CU(b.pk_meta.grow(2, s));
        CU(b.rem_scratch.grow(wr * sizeof(u64) / sizeof(u32), s));
        CU(b.excl.grow(HQS_MAX_WORKERS, s));
        CU(b.glist.grow((size_t)GLIST_GLOBAL_WORDS, s));
        CU(b.pf_cum.grow(PF_SEG_CAP, s));
        CU(b.pf_wk.grow(PF_SEG_CAP, s));
        CU(b.h_hdr.grow(sizeof(TickHeaderOut) + wr * 8, s, false, 0));
        ctx->tick = std::move(b);
        ctx->sync_dirty = true;
    }
    if (out_cap > ctx->d_out.size()) CU(ctx->d_out.grow(std::max<u32>(out_cap, 1024), ctx->stream));
    return HQS_OK;
}

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
    if (bytes > ctx->d_tickin.size()) CU(ctx->d_tickin.grow(bytes * 2, ctx->stream));
    if (bytes > ctx->h_tickin.size()) CU(ctx->h_tickin.grow(bytes * 2, ctx->stream));
    return HQS_OK;
}

// Fills the pinned staging buffer with the tick's worker state and orders.  The solver CTA reads it in place (mapped
// host memory, overlapped with the histogram of the worker CTAs); only the blocked mask, which the pack warps read
// with scattered byte loads, is copied to the device.  Records what it staged in ctx->staged.
int upload_tick_input(hqs_ctx* ctx, u32 W, const hqs_worker* workers, const u64* free_rw, const u64* total_rw,
                      const uint8_t* blocked) {
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
    if (!ctx->zero_copy) CU(cudaMemcpyAsync(ctx->d_tickin, h, lay.bytes, cudaMemcpyHostToDevice, ctx->stream));
    else if (blocked || pfwc) CU(cudaMemcpyAsync(ctx->d_tickin + lay.off_blocked, h + lay.off_blocked, lay.bytes - lay.off_blocked, cudaMemcpyHostToDevice, ctx->stream));
    ctx->staged = TickInput{W, lay, blocked != nullptr, pfwc, mu_any, time_any, narrow};
    return HQS_OK;
}

// The staging step of the calls that upload a tick input, after their own argument checks: no tick pending, G within
// HQS_MAX_GROUPS and groups_cap (~0u: no cap), tick buffers for out_cap records, then the upload.  *t: the tick's geometry.
int stage_tick(hqs_ctx* ctx, u32 W, const hqs_worker* workers, const u64* free_rw, const u64* total_rw, const uint8_t* blocked,
               u32 out_cap, u32 groups_cap, TickGeom* t) {
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    CU(cudaSetDevice(ctx->device));
    *t = tick_geom(ctx);
    if (t->G > HQS_MAX_GROUPS) return fail(ctx, HQS_E_LIMIT, "groups=%u > %u", t->G, HQS_MAX_GROUPS);
    if (t->G > groups_cap) return fail(ctx, HQS_E_LIMIT, "groups=%u > n_groups_cap=%u", t->G, groups_cap);
    if (int rc = ensure_tick_buffers(ctx, t->G, t->P, out_cap)) return rc;
    return upload_tick_input(ctx, W, workers, free_rw, total_rw, blocked);
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

TickArgs base_args(hqs_ctx* ctx, const TickGeom& t) {
    TickArgs a;
    memset(&a, 0, sizeof a);
    const TickInput& ti = ctx->staged;
    const TickLayout& lay = ti.lay;
    const unsigned char* in = ctx->zero_copy ? ctx->h_tickin.dev() : ctx->d_tickin;
    a.free_rw = reinterpret_cast<const u64*>(in + lay.off_free);
    a.total_rw = reinterpret_cast<const u64*>(in + lay.off_total);
    a.rem_time = reinterpret_cast<const u64*>(in + lay.off_rem);
    a.order = reinterpret_cast<const u32*>(in + lay.off_order);
    a.vorder = in + lay.off_vorder;
    a.blocked = ti.blocked ? ctx->d_tickin + lay.off_blocked : nullptr;
    a.min_util = ti.min_util ? reinterpret_cast<const float*>(in + lay.off_mu) : nullptr;
    a.any_time_limit = ti.any_time;
    a.classes = ti.narrow ? ctx->d_classes32 : ctx->d_classes;
    a.classes64 = ctx->d_classes;
    for (u32 r = 0; r < HQS_MAX_RESOURCES; ++r) a.gscale[r] = ctx->gscale[r] ? ctx->gscale[r] : 1;
    a.W = ti.W; a.Q = ctx->Q; a.L = t.L; a.R = ctx->R; a.G = t.G;
    a.classes_bytes = ctx->Q * (ti.narrow ? ctx->class_bytes32 : ctx->class_bytes);
    a.key = ctx->d_key; a.n_handles = ctx->n_handles; a.chunk = t.chunk; a.rows = t.rows; a.P = t.P; a.nbits = t.nbits;
    a.emit_warps = t.emit_warps; a.g_smem = t.g_smem; a.emit_stage = t.emit_stage;
    a.total_local = ctx->d_total;
    a.table = ctx->d_table;
    a.gout = ctx->d_gout;
    const TickBuffers& tb = ctx->tick;
    a.seg_cum = tb.seg_cum; a.seg_wv = tb.seg_wv;
    a.free_after = tb.free_after;
    a.hdr = tb.hdr;
    a.hdr_host = reinterpret_cast<TickHeaderOut*>(tb.h_hdr.dev());
    a.out = ctx->d_out;
    a.rem_scratch = tb.rem_scratch;
    a.glist_glob = tb.glist;
    a.sync = tb.sync;
    a.pk.fr = tb.pk_fr; a.pk.quota = tb.pk_quota; a.pk.taken = tb.pk_taken;
    a.pk.cand = tb.pk_cand; a.pk.meta = tb.pk_meta;
    a.excl_glob = tb.excl;
    a.pf_shift = ctx->pf_max ? 1 : 0; a.pf_reserve = ctx->pf_reserve; a.pf_max = ctx->pf_max;
    a.prefilled_wc = ti.pfwc ? ctx->d_tickin + lay.off_pfwc : nullptr;
    a.gout2 = ctx->d_gout2; a.pf_cum = tb.pf_cum; a.pf_wk = tb.pf_wk;
    return a;
}

// shared-memory layout of the solver CTA: mandatory arrays first, then the optional ones while they fit.  The group list
// (glist, gcl and, with proactive filling, kk: 12 or 16 B per entry) is mandatory unless the other mandatory arrays and it
// do not fit together (many workers x wide amounts x thousands of groups); then it lives in TickBuffers::glist, and every
// tick that fits keeps the layout it always had.
size_t solver_layout(const hqs_ctx* ctx, TickArgs& a, size_t budget, bool sharded) {
    const u32 W = a.W, Q = a.Q, RT = ctx->RT;
    const size_t at = ctx->staged.narrow ? 4 : 8;
    const u32 n_pos = (a.L * Q) << a.pf_shift;
    size_t o = 0;
    auto put = [&](size_t bytes) { const size_t at_ = o; o = (o + bytes + 15) & ~size_t(15); return (u32)at_; };
    auto mandatory = [&](bool groups) {
        o = 0;
        a.sm.fr = put((size_t)W * RT * at);
        a.sm.unt = put((size_t)W * 4);
        a.sm.remtime = put((size_t)W * 8);
        a.sm.excl = put(W);
        a.sm.touch = put(W);
        a.sm.td = put((size_t)W * 2);
        a.sm.frontier = put((size_t)Q * 2);
        a.sm.noresv = put(Q);
        a.sm.glist = groups ? put((size_t)n_pos * 8) : SM_NONE;
        a.sm.gcl = groups ? put((size_t)n_pos * 4) : SM_NONE;
        a.sm.kk = a.sm.top = a.sm.pflvl = SM_NONE;
        if (a.pf_shift) {
            if (groups) a.sm.kk = put((size_t)n_pos * 4);
            a.sm.top = put((size_t)Q * 4);
            a.sm.pflvl = put((size_t)Q * 4);
        }
    };
    mandatory(true);
    if (o > budget) mandatory(false);
    auto opt = [&](size_t bytes, bool wanted) -> u32 {
        if (!wanted || o + bytes + 16 > budget) return SM_NONE;
        return put(bytes);
    };
    a.sm.classes = opt(a.classes_bytes, true);
    a.sm.vorder = opt((size_t)Q * HQS_MAX_VARIANTS, true);
    a.sm.rem = opt((size_t)W * RT * 8, ctx->staged.narrow);
    a.sm.blocked = opt((size_t)W * Q, a.blocked != nullptr);
    a.sm.bef = opt((size_t)n_pos * 4, sharded);
    a.sm.loc = a.sm.bef != SM_NONE ? opt((size_t)n_pos * 4, sharded) : SM_NONE;
    if (a.sm.loc == SM_NONE) a.sm.bef = SM_NONE;
    a.smem_solver = (u32)o;
    return o;
}

// Launches the tick kernel over the staged input.  counts: nullptr (count inside the kernel), or host-provided totals (NCCL
// variant, the histogram was taken by hqs_shard_count).  emit = false: what-if query (nothing is emitted or consumed).
int launch_tick(hqs_ctx* ctx, const TickGeom& t, const u32* d_counts_all, const u32* d_before, u32 out_cap, bool emit,
                bool exchange) {
    TickArgs a = base_args(ctx, t);
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
    const void* fn = tick_fn(ctx->RT, ctx->staged.narrow);
    const size_t budget = ctx->smem_budget[ctx->staged.narrow ? 0 : 1];
    const size_t solver_smem = solver_layout(ctx, a, budget, exchange || d_before != nullptr);
    const size_t smem = std::max(solver_smem, t.worker_smem);
    if (smem > budget) return fail(ctx, HQS_E_LIMIT, "tick needs %zu bytes of shared memory, %zu available", smem, budget);
    if (ctx->sync_dirty) {
        CU(cudaMemsetAsync(ctx->tick.sync, 0, sizeof(TickSync), ctx->stream));
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
    ctx->last_G = t.G; ctx->last_L = t.L;
    return HQS_OK;
}

// waits for the tick kernel and reads the header the kernel wrote into the pinned mirror
int wait_header(hqs_ctx* ctx, TickHeaderOut* hdr) {
    CU(cudaStreamSynchronize(ctx->stream));
    memcpy(hdr, ctx->tick.h_hdr, sizeof *hdr);
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
    CU(ctx->h_pw.grow(HQS_MAX_WORKERS, ctx->stream));
    return HQS_OK;
}

// What-if query: the tick kernel without its emit step (nothing is emitted or consumed), then the per-worker task counts of
// its count segments into the pinned buffer hqs_query_fetch reads.  Like a tick, the query is pending until it is fetched.
// counts_all / exchange as for launch_tick (a query has no local share, so no ranks_before).
int launch_query(hqs_ctx* ctx, const TickGeom& t, const u32* d_counts_all, bool exchange) {
    int rc = ensure_query_buffers(ctx);
    if (rc) return rc;
    rc = launch_tick(ctx, t, d_counts_all, nullptr, 0, false, exchange);
    if (rc) return rc;
    const u32 W = ctx->staged.W;
    u32* d_pw = ctx->tick.pk_quota;    // scratch (pack is over): [W] counters
    CU(cudaMemsetAsync(d_pw, 0, W * sizeof(u32), ctx->stream));
    seg_worker_totals_k<<<(t.G + 127) / 128, 128, 0, ctx->stream>>>(ctx->d_gout, t.G, ctx->tick.seg_cum, ctx->tick.seg_wv, d_pw);
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
    TickGeom t;
    if ((rc = stage_tick(ctx, n_workers, workers, free_rw, total_rw, blocked_wcv, 1024, ~0u, &t))) return rc;
    // ticks and queries share one exchange sequence: every rank advances it in lockstep
    if (exchange) ctx->x_seq += 1;
    return launch_query(ctx, t, nullptr, exchange);
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
        Buf<u32, Mem::Host> off;
        Buf<u32> small;
        CU(off.grow(GRP_KEYS_MAX + 1, ctx->stream));
        CU(small.grow(2 * GRP_KEYS_MAX + 2, ctx->stream, false, 0));   // the ticket starts at 0
        ctx->h_grp_off = std::move(off);
        ctx->d_grp_small = std::move(small);
    }
    if (cap > ctx->d_grp_out.size()) CU(ctx->d_grp_out.grow(std::max<u32>(cap, 1024), ctx->stream));
    const size_t need = (2 * W + 1) * ((ctx->d_grp_out.size() + GROUP_TILE - 1) / GROUP_TILE);
    if (need > ctx->d_grp_hist.size()) CU(ctx->d_grp_hist.grow(need, ctx->stream));
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
    const u32 W = ctx->staged.W, n_off = 2 * W + 2;
    if (free_after) memcpy(free_after, ctx->tick.h_hdr + sizeof(TickHeaderOut), (size_t)W * ctx->R * 8);
    if (worker_off) memset(worker_off, 0, n_off * sizeof(u32));
    if (n_rec && !worker_off) {
        CU(cudaMemcpyAsync(out, ctx->d_out, (size_t)n_rec * sizeof(hqs_assignment), cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
    } else if (n_rec) {
        // n and the error word are known here, so the grids are exact and a failed tick never reaches this point
        ctx->grp_ms = -1.f;
        if ((rc = ensure_group_buffers(ctx, W, std::max(n_rec, (u32)ctx->d_out.size())))) return rc;
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
    if (e != cudaSuccess) ctx->stream = nullptr;   // not a stream after a failed create: nothing to destroy
    int sms = 0;
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (e == cudaSuccess) e = ctx->d_newcnt.grow(2, ctx->stream);
    if (e == cudaSuccess) e = ctx->d_newprio.grow(NEWPRIO_CAP, ctx->stream);
    if (e == cudaSuccess) e = ctx->h_cnt.grow(1, ctx->stream);
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
    if (blob.size() > ctx->d_classes.size()) CU(ctx->d_classes.grow(std::max<size_t>(blob.size() * 2, 4096), ctx->stream));
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
    if (blob32.size() > ctx->d_classes32.size())
        CU(ctx->d_classes32.grow(std::max<size_t>(blob32.size() * 2, 4096), ctx->stream));
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
// The dependencies of a graph push, staged by hqs_graph_push: d_gstage = dependency offsets [n + 1], then the dependency
// handles; the counted edges take the pool slots e0 + j.  task: the batch's n handles on the device on a sharded graph
// context (global; push_impl's own arrays are the owned part of the batch only); nullptr: push_impl's staged handles.
struct GraphBatch {
    u32 e0;
    u32 n;
    const u32* task;
};

// how the graph kernels see this context's keys (hqs_graph.cuh)
GraphKeys graph_keys(const hqs_ctx* ctx) {
    if (!ctx->shard_graph) return GraphKeys{ctx->d_key, nullptr, 0u, ~0u};
    return GraphKeys{ctx->d_key, ctx->d_gvalid, ctx->g_lo, ctx->g_lo + std::min(ctx->cap_handles, ctx->g_hi - ctx->g_lo)};
}

// the handles the graph calls accept: the table of one context, the global range of a sharded graph context
u32 graph_bound(const hqs_ctx* ctx) { return ctx->shard_graph ? ctx->g_total : ctx->n_handles; }

// shared body of hqs_ready_push / hqs_ready_push_range (task == nullptr: handles first_handle .. first_handle + n - 1) and
// hqs_graph_push (g != nullptr: the batch is also rejected if a pushed handle is VALID, and graph_link_k runs after push_k;
// h_cnt->ready receives the number of tasks ready at once).  A sharded graph push passes the owned part of its batch, which
// may be empty.
int push_impl(hqs_ctx* ctx, u32 n, const u32* task, u32 first_handle, const u32* class_id, const u64* priority,
              const GraphBatch* g = nullptr) {
    if (ctx->Q == 0) return fail(ctx, HQS_E_STATE, "hqs_classes_set has not been called");
    if (ctx->dag) return fail(ctx, HQS_E_STATE, "hqs_ready_push is not available after hqs_dag_load");
    if (!g && ctx->shard_graph)
        return fail(ctx, HQS_E_STATE, "hqs_ready_push is not available on a sharded graph context (hqs_shard_graph_push)");
    CU(cudaSetDevice(ctx->device));
    if (int rc_ = ensure_push_staging(ctx, n)) return rc_;
    if (n) {
        if (task) CU(cudaMemcpyAsync(ctx->d_push_task, task, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
        CU(cudaMemcpyAsync(ctx->d_push_cls, class_id, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
        CU(cudaMemcpyAsync(ctx->d_push_prio, priority, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
    }
    // the table must hold the largest handle before the kernel runs: a host pass over the handle array while the staging
    // copies are in flight (a range push knows it); class ids are validated on the device (push_validate_k)
    u32 max_h = n ? first_handle + (n - 1) : 0u;
    if (task && n) {
        u32 dummy = 0;
        max_of_u32_pair(task, task, n, &max_h, &dummy);
    } else if (max_h < first_handle) {
        max_h = ~0u;                                                  // the range wraps around
    }
    if (max_h == ~0u) {
        cudaStreamSynchronize(ctx->stream);      // the caller may free its arrays as soon as we return
        return fail(ctx, HQS_E_INVALID, "task handle 0xFFFFFFFF is reserved");
    }
    int rc = n ? ensure_handles(ctx, max_h + 1) : HQS_OK;
    if (rc) { cudaStreamSynchronize(ctx->stream); return rc; }
    CU(cudaMemsetAsync(ctx->d_newcnt, 0, 2 * sizeof(u32), ctx->stream));
    const GraphKeys gk = graph_keys(ctx);
    const u32* gtask = g && g->task ? g->task : ctx->d_push_task;     // after ensure_push_staging, which may move it
    if (n) push_validate_k<<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, ctx->d_push_cls, ctx->Q, ctx->d_newcnt);
    if (g)
        graph_dispatch(ctx->shard_graph, [&](auto S) {
            graph_validate_k<decltype(S)::value><<<(g->n + 255) / 256, 256, 0, ctx->stream>>>(g->n, gtask, gk, graph_bound(ctx),
                                                                                             ctx->d_newcnt);
        });
    if (n)
        push_k<<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, task ? (u32*)ctx->d_push_task : nullptr, first_handle, ctx->d_push_cls,
                                                         ctx->d_push_prio, ctx->d_key, ctx->d_prio, ctx->d_levels,
                                                         (u32)ctx->dev_levels.size(), ctx->coarse ? 1 : 0, ctx->d_newcnt, ctx->d_newprio);
    ctx->stats.kernel_launches += n ? 2 : 0;
    if (g) {
        CU(cudaMemsetAsync(ctx->d_gsmall, 0, sizeof(u32), ctx->stream));
        if (ctx->shard_graph) {
            graph_enter_k<<<(g->n + 255) / 256, 256, 0, ctx->stream>>>(g->n, gtask, ctx->d_newcnt, ctx->d_gvalid);
            ctx->stats.kernel_launches++;
        }
        graph_dispatch(ctx->shard_graph, [&](auto S) {
            graph_link_k<decltype(S)::value><<<(g->n + 255) / 256, 256, 0, ctx->stream>>>(
                g->n, gtask, ctx->d_gstage, ctx->d_gstage + g->n + 1, g->e0, ctx->d_newcnt, gk, ctx->d_gdeps, ctx->d_ggen,
                ctx->d_ghead, ctx->d_pool, ctx->d_gsmall);
        });
        CU(cudaMemcpyAsync(&ctx->h_cnt->ready, ctx->d_gsmall, sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
        ctx->stats.kernel_launches += 2;
    }
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(&ctx->h_cnt->newcnt, ctx->d_newcnt, 2 * sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
    // a coarse table has a bucket for every priority, so push_k reports none as fresh: the batch's priorities are
    // collected here, while the kernels run, and registered like fresh ones (the level set keeps growing, gets pruned
    // and leaves coarse mode once the live priorities fit again).  Exact-mode pushes do not take this pass.
    std::vector<u64> fresh;
    if (ctx->coarse) distinct_priorities(priority, n, fresh);
    CU(cudaStreamSynchronize(ctx->stream));
    if (ctx->h_cnt->reject & 1u) return fail(ctx, HQS_E_INVALID, "a class id of the batch is >= n_classes %u (nothing was pushed)", ctx->Q);
    if (ctx->h_cnt->reject) return fail(ctx, HQS_E_INVALID, "a handle of the batch is a live task (nothing was pushed)");
    if (n) ctx->n_handles = std::max(ctx->n_handles, max_h + 1);
    ctx->stats.n_handles = ctx->n_handles;
    const u32 newcnt = ctx->h_cnt->newcnt;
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

int hqs_levels_live(hqs_ctx* ctx, uint32_t cap, uint64_t* levels, uint8_t* live, uint32_t* n_levels) {
    if (!ctx) return HQS_E_INVALID;
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    if (cap && (!levels || !live)) return fail(ctx, HQS_E_INVALID, "null level arrays");
    const u32 L = (u32)ctx->levels.size();
    if (n_levels) *n_levels = L;
    if (!cap) return HQS_OK;
    if (cap < L) return fail(ctx, HQS_E_INVALID, "cap=%u < n_levels=%u", cap, L);
    CU(cudaSetDevice(ctx->device));
    std::vector<u32> lv;
    int rc = live_levels(ctx, lv);
    if (rc) return rc;
    for (u32 i = 0; i < L; ++i) {
        levels[i] = ctx->levels[i];
        live[i] = lv[i] ? 1 : 0;
    }
    return HQS_OK;
}

int hqs_levels_retain(hqs_ctx* ctx, uint32_t n, const uint8_t* keep) {
    if (!ctx) return HQS_E_INVALID;
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    const u32 L = (u32)ctx->levels.size();
    if (n != L) return fail(ctx, HQS_E_INVALID, "n=%u != n_levels=%u", n, L);
    if (L && !keep) return fail(ctx, HQS_E_INVALID, "null keep array");
    CU(cudaSetDevice(ctx->device));
    std::vector<u32> lv;
    int rc = live_levels(ctx, lv);
    if (rc) return rc;
    std::vector<u64> kept;
    kept.reserve(L);
    for (u32 i = 0; i < L; ++i) {
        if (keep[i]) kept.push_back(ctx->levels[i]);
        else if (lv[i]) return fail(ctx, HQS_E_INVALID, "level %u (priority %llu) is carried by a task of this context", i,
                                    (unsigned long long)ctx->levels[i]);
    }
    ctx->levels_pruned_at = kept.size();
    if (kept.size() == L) return HQS_OK;
    ctx->levels.swap(kept);
    if ((rc = upload_levels(ctx))) return rc;
    return relevel_all(ctx);
}

int hqs_ready_remove(hqs_ctx* ctx, uint32_t n, const uint32_t* task) {
    if (!ctx) return HQS_E_INVALID;
    if (n == 0) return HQS_OK;
    if (!task) return fail(ctx, HQS_E_INVALID, "null task array");
    if (ctx->shard_graph)
        return fail(ctx, HQS_E_STATE, "hqs_ready_remove is not available on a sharded graph context (hqs_shard_graph_remove)");
    CU(cudaSetDevice(ctx->device));
    if (int rc_ = ensure_push_staging(ctx, n)) return rc_;
    CU(cudaMemcpyAsync(ctx->d_push_task, task, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    remove_k<<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, ctx->d_push_task, ctx->d_key, ctx->n_handles);
    ctx->stats.kernel_launches++;
    if (ctx->graph_storage) {   // the removed tasks' consumer lists go (their consumers wait until the host cancels them)
        graph_unlink_k<<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, ctx->d_push_task, ctx->n_handles, ctx->d_ghead);
        ctx->stats.kernel_launches++;
    }
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
    if (ctx->graph) return fail(ctx, HQS_E_STATE, "hqs_dag_load is not available after hqs_graph_push");
    if (ctx->shard_graph) return fail(ctx, HQS_E_STATE, "hqs_dag_load is not available on a sharded graph context");
    const u32 n_edges = cons_off[n_tasks];
    if (n_edges && !cons) return fail(ctx, HQS_E_INVALID, "null consumer array");
    for (u32 i = 0; i < n_tasks; ++i)
        if (class_id[i] >= ctx->Q) return fail(ctx, HQS_E_INVALID, "class id %u >= n_classes %u", class_id[i], ctx->Q);
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_handles(ctx, n_tasks);
    if (rc) return rc;
    CU(cudaStreamSynchronize(ctx->stream));       // an earlier DAG's arrays are freed below
    Buf<u32> dev_deps, dev_off, dev_cons, d_cls;
    CU(dev_deps.grow(n_tasks, ctx->stream));
    CU(dev_off.grow((size_t)n_tasks + 1, ctx->stream));
    CU(dev_cons.grow(std::max<size_t>(n_edges, 1), ctx->stream));
    CU(d_cls.grow(n_tasks, ctx->stream));
    ctx->d_deps = std::move(dev_deps);
    ctx->d_cons_off = std::move(dev_off);
    ctx->d_cons = std::move(dev_cons);
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
    if ((rc = upload_levels(ctx))) return rc;
    ctx->n_handles = n_tasks;
    ctx->stats.n_handles = n_tasks;
    dag_init_k<<<(n_tasks + 255) / 256, 256, 0, ctx->stream>>>(n_tasks, d_cls, ctx->d_prio, ctx->d_deps, ctx->d_key,
                                                               ctx->d_levels, (u32)ctx->dev_levels.size(),
                                                               ctx->coarse ? 1 : 0);
    ctx->stats.kernel_launches++;
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->dag = true;
    return HQS_OK;
}

int hqs_tasks_finished(hqs_ctx* ctx, uint32_t n, const uint32_t* task, uint32_t* n_new_ready) {
    if (!ctx) return HQS_E_INVALID;
    if (n_new_ready) *n_new_ready = 0;
    if (!ctx->dag) return fail(ctx, HQS_E_STATE, "hqs_tasks_finished needs hqs_dag_load");
    if (n == 0) return HQS_OK;
    if (!task) return fail(ctx, HQS_E_INVALID, "null task array");
    for (u32 i = 0; i < n; ++i)
        if (task[i] >= ctx->n_handles) return fail(ctx, HQS_E_INVALID, "task %u >= n_tasks %u (nothing was finished)", task[i], ctx->n_handles);
    CU(cudaSetDevice(ctx->device));
    if (int rc_ = ensure_push_staging(ctx, n)) return rc_;
    CU(cudaMemcpyAsync(ctx->d_push_task, task, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemsetAsync(ctx->d_newcnt, 0, sizeof(u32), ctx->stream));
    finished_k<<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, ctx->d_push_task, ctx->d_cons_off, ctx->d_cons, ctx->d_deps,
                                                         ctx->d_key, ctx->d_newcnt);
    ctx->stats.kernel_launches++;
    CU(cudaGetLastError());
    if (n_new_ready) {
        CU(cudaMemcpyAsync(&ctx->h_cnt->newcnt, ctx->d_newcnt, sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        *n_new_ready = ctx->h_cnt->newcnt;
    }
    return HQS_OK;
}

}  // extern "C"

namespace {
// the context states in which the graph calls are refused
int graph_mode_check(hqs_ctx* ctx, const char* what) {
    if (ctx->dag) return fail(ctx, HQS_E_STATE, "%s is not available after hqs_dag_load", what);
    if (ctx->x_world) return fail(ctx, HQS_E_STATE, "%s is not available on a sharded ready set", what);
    if (ctx->shard_graph) return fail(ctx, HQS_E_STATE, "%s is not available on a sharded graph context (hqs_shard_graph_*)", what);
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    return HQS_OK;
}

// ... and the states in which the sharded graph calls are refused
int shard_graph_mode_check(hqs_ctx* ctx, const char* what) {
    if (!ctx->shard_graph) return fail(ctx, HQS_E_STATE, "%s needs hqs_shard_graph_init", what);
    if (ctx->shard_graph_failed)
        return fail(ctx, HQS_E_STATE, "%s: an earlier sharded graph call failed on the device, so this rank's replica may differ "
                    "from the others; the sharded graph must be set up again on new contexts", what);
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    return HQS_OK;
}

// A sharded graph call that failed on the device (HQS_E_CUDA: a CUDA error, an allocation, the cancel marking's time-out) may
// have changed this rank's replica and not the others', or the others' and not this one: the context refuses the sharded
// graph calls from then on.  The other failures are decided alike on every rank from the same arguments and change nothing.
int shard_graph_outcome(hqs_ctx* ctx, int rc) {
    if (rc == HQS_E_CUDA) ctx->shard_graph_failed = true;
    return rc;
}

// the body of hqs_shard_graph_remove, after the mode check
int shard_graph_remove_impl(hqs_ctx* ctx, u32 n, const u32* task) {
    if (n == 0) return HQS_OK;
    if (!task) return fail(ctx, HQS_E_INVALID, "null task array");
    for (u32 i = 0; i < n; ++i)
        if (task[i] >= ctx->g_total)
            return fail(ctx, HQS_E_INVALID, "task %u >= n_total %u (nothing was removed)", task[i], ctx->g_total);
    CU(cudaSetDevice(ctx->device));
    if (int rc = ensure_push_staging(ctx, n)) return rc;
    CU(cudaMemcpyAsync(ctx->d_push_task, task, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    // what hqs_ready_remove does, over the replica: the owner's keys and every rank's graph VALID bits and consumer lists go
    graph_leave_k<true><<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, ctx->d_push_task, graph_keys(ctx), ctx->d_push_cls);
    graph_unlink_k<<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, ctx->d_push_task, ctx->g_total, ctx->d_ghead);
    ctx->stats.kernel_launches += 2;
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(ctx->stream));
    return HQS_OK;
}

// Before a push whose edges do not fit: the pool keeps only the edges whose consumer still waits on their incarnation,
// rewritten list by list into a fresh pool of max(capacity, 2 * live + n_edges) slots.
int graph_compact(hqs_ctx* ctx, u32 n_edges) {
    const u32 nh = graph_bound(ctx), nb = (nh + GRAPH_PER_BLOCK - 1) / GRAPH_PER_BLOCK;
    const GraphKeys gk = graph_keys(ctx);
    u32 live = 0;
    if (nb) {
        graph_dispatch(ctx->shard_graph, [&](auto S) {
            graph_gc_count_k<decltype(S)::value><<<nb, GRAPH_NT, 0, ctx->stream>>>(nh, ctx->d_ghead, ctx->d_pool, gk, ctx->d_gdeps,
                                                                                  ctx->d_ggen, ctx->d_gblk);
        });
        graph_scan_k<<<1, 1024, 0, ctx->stream>>>(nb, ctx->d_gblk, ctx->d_gsmall + 2);
        ctx->stats.kernel_launches += 2;
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(&ctx->h_cnt->live, ctx->d_gsmall + 2, sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        live = ctx->h_cnt->live;
    }
    const u64 want = std::max<u64>(ctx->pool_cap, 2ull * live + n_edges);
    if (want >= GRAPH_NIL) return fail(ctx, HQS_E_LIMIT, "the edge pool would need %llu slots", (unsigned long long)want);
    Buf<GraphEdge> fresh;
    CU(fresh.grow(want, ctx->stream));
    if (nb) {
        graph_dispatch(ctx->shard_graph, [&](auto S) {
            graph_gc_move_k<decltype(S)::value><<<nb, GRAPH_NT, 0, ctx->stream>>>(nh, ctx->d_ghead, ctx->d_pool, fresh, gk,
                                                                                 ctx->d_gdeps, ctx->d_ggen, ctx->d_gblk);
        });
        ctx->stats.kernel_launches++;
        CU(cudaGetLastError());
    }
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->d_pool = std::move(fresh);
    ctx->pool_cap = (u32)want;
    ctx->pool_used = live;
    ctx->pool_compactions++;
    return HQS_OK;
}

// the device half of hqs_graph_push's validation on its own, before a compaction (a rejected batch changes nothing).  A
// sharded graph push has checked its class ids on the host and staged its handles at d_task.
int graph_prevalidate(hqs_ctx* ctx, u32 n, const u32* task, const u32* class_id, const u32* d_task) {
    if (int rc = ensure_push_staging(ctx, n)) return rc;
    CU(cudaMemsetAsync(ctx->d_newcnt, 0, 2 * sizeof(u32), ctx->stream));
    if (ctx->shard_graph) {
        graph_validate_k<true><<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, d_task, graph_keys(ctx), ctx->g_total, ctx->d_newcnt);
        ctx->stats.kernel_launches++;
    } else {
        CU(cudaMemcpyAsync(ctx->d_push_task, task, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
        CU(cudaMemcpyAsync(ctx->d_push_cls, class_id, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
        push_validate_k<<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, ctx->d_push_cls, ctx->Q, ctx->d_newcnt);
        graph_validate_k<false><<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, ctx->d_push_task, graph_keys(ctx), ctx->n_handles,
                                                                          ctx->d_newcnt);
        ctx->stats.kernel_launches += 2;
    }
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(&ctx->h_cnt->newcnt, ctx->d_newcnt, 2 * sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    if (ctx->h_cnt->reject & 1u) return fail(ctx, HQS_E_INVALID, "a class id of the batch is >= n_classes %u (nothing was pushed)", ctx->Q);
    if (ctx->h_cnt->reject) return fail(ctx, HQS_E_INVALID, "a handle of the batch is a live task (nothing was pushed)");
    return HQS_OK;
}

// duplicates among the k dependencies d[0..k)
bool has_duplicate(const u32* d, u32 k, std::vector<u32>& scratch) {
    if (k <= 16) {
        for (u32 a = 1; a < k; ++a)
            for (u32 b = 0; b < a; ++b)
                if (d[a] == d[b]) return true;
        return false;
    }
    scratch.assign(d, d + k);
    std::sort(scratch.begin(), scratch.end());
    return std::adjacent_find(scratch.begin(), scratch.end()) != scratch.end();
}
// The body of hqs_graph_push and hqs_shard_graph_push, after the mode check.  On a sharded graph context the handles are
// global: every rank checks and links the whole batch, and pushes the keys of the handles it owns.
int graph_push_impl(hqs_ctx* ctx, u32 n, const u32* task, const u32* class_id, const u64* priority, const u32* dep_off,
                    const u32* deps, u32* n_ready) {
    if (n == 0) return HQS_OK;
    if (!task || !class_id || !priority || !dep_off) return fail(ctx, HQS_E_INVALID, "null task arrays");
    if (ctx->Q == 0) return fail(ctx, HQS_E_STATE, "hqs_classes_set has not been called");
    const bool shard = ctx->shard_graph;
    const u32 bound = graph_bound(ctx);
    // host-knowable checks, then the batch's own dependency lists: the handle -> batch position map is a range test when
    // the handles are consecutive (a job's tasks), a sorted table otherwise
    if (dep_off[0] != 0) return fail(ctx, HQS_E_INVALID, "dep_off[0] = %u, not 0", dep_off[0]);
    for (u32 i = 0; i < n; ++i)
        if (dep_off[i + 1] < dep_off[i]) return fail(ctx, HQS_E_INVALID, "dep_off decreases at task %u", i);
    const u32 m = dep_off[n];
    if (m && !deps) return fail(ctx, HQS_E_INVALID, "null dependency array");
    bool range = true;
    for (u32 i = 0; i < n; ++i) {
        if (task[i] == GRAPH_NIL) return fail(ctx, HQS_E_INVALID, "task handle 0xFFFFFFFF is reserved");
        if (shard && task[i] >= bound) return fail(ctx, HQS_E_INVALID, "task %u >= n_total %u (nothing was pushed)", task[i], bound);
        range &= task[i] == task[0] + i;
    }
    if (shard) {
        // every rank must see the same rejections and number the levels alike: class ids here, declared priorities only
        for (u32 i = 0; i < n; ++i)
            if (class_id[i] >= ctx->Q) return fail(ctx, HQS_E_INVALID, "a class id of the batch is >= n_classes %u (nothing was pushed)", ctx->Q);
        std::vector<u64> pr;
        distinct_priorities(priority, n, pr);
        for (u64 p : pr)
            if (!std::binary_search(ctx->levels.begin(), ctx->levels.end(), p, std::greater<u64>()))
                return fail(ctx, HQS_E_INVALID, "priority %llu was not declared with hqs_levels_add (nothing was pushed)",
                            (unsigned long long)p);
    }
    std::vector<std::pair<u32, u32>>& pos = ctx->g_pos;
    if (!range) {
        pos.resize(n);
        for (u32 i = 0; i < n; ++i) pos[i] = {task[i], i};
        std::sort(pos.begin(), pos.end());
        for (u32 i = 1; i < n; ++i)
            if (pos[i].first == pos[i - 1].first) return fail(ctx, HQS_E_INVALID, "handle %u appears twice in the batch", pos[i].first);
    }
    auto batch_pos = [&](u32 h) -> u32 {      // position of h in the batch, GRAPH_NIL if it is not in it
        if (range) return h - task[0] < n ? h - task[0] : GRAPH_NIL;
        auto it = std::lower_bound(pos.begin(), pos.end(), std::make_pair(h, 0u));
        return it != pos.end() && it->first == h ? it->second : GRAPH_NIL;
    };
    std::vector<u32>& off = ctx->g_off;
    std::vector<u32>& dep = ctx->g_dep;
    std::vector<u32> scratch;
    off.resize((size_t)n + 1);
    dep.clear();
    dep.reserve(m);
    off[0] = 0;
    for (u32 i = 0; i < n; ++i) {
        const u32 lo = dep_off[i], hi = dep_off[i + 1];
        if (has_duplicate(deps + lo, hi - lo, scratch)) return fail(ctx, HQS_E_INVALID, "task %u names a dependency twice", task[i]);
        for (u32 j = lo; j < hi; ++j) {
            const u32 d = deps[j];
            if (d == task[i]) return fail(ctx, HQS_E_INVALID, "task %u depends on itself", d);
            const u32 p = batch_pos(d);
            if (p == GRAPH_NIL) {
                if (d >= bound) return fail(ctx, HQS_E_INVALID, "dependency %u of task %u is unknown", d, task[i]);
                dep.push_back(d);                // counts if VALID on the device
            } else if (p < i) {
                dep.push_back(d);                // an earlier task of the batch
            }                                    // a later one is dropped, as on_new_tasks does
        }
        off[i + 1] = (u32)dep.size();
    }
    const u32 me = (u32)dep.size();
    CU(cudaSetDevice(ctx->device));
    int rc;
    if ((rc = ensure_graph_storage(ctx))) return rc;
    // d_gstage: offsets, dependencies, then (sharded) the batch's global handles
    const size_t stage = (size_t)n + 1 + me + (shard ? n : 0);
    if (stage > ctx->d_gstage.size()) CU(ctx->d_gstage.grow(std::max<size_t>(stage * 2, 1u << 16), ctx->stream));
    // pageable sources: staged by the runtime before the calls return
    CU(cudaMemcpyAsync(ctx->d_gstage, off.data(), ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
    if (me) CU(cudaMemcpyAsync(ctx->d_gstage + n + 1, dep.data(), (size_t)me * 4, cudaMemcpyHostToDevice, ctx->stream));
    u32* d_task = nullptr;
    if (shard) {
        d_task = ctx->d_gstage + n + 1 + me;
        CU(cudaMemcpyAsync(d_task, task, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    }
    // a push that allocates or compacts the pool is validated on the device first, so that a rejected batch changes nothing
    if (!ctx->d_pool || (u64)ctx->pool_used + me > ctx->pool_cap)
        if ((rc = graph_prevalidate(ctx, n, task, class_id, d_task))) return rc;
    if (!ctx->d_pool) {
        const u64 cap = std::max<u64>(2ull * me, GRAPH_POOL_MIN);
        if (cap >= GRAPH_NIL) return fail(ctx, HQS_E_LIMIT, "the edge pool would need %llu slots", (unsigned long long)cap);
        CU(ctx->d_pool.grow(cap, ctx->stream));
        ctx->pool_cap = (u32)cap;
        ctx->pool_used = 0;
    } else if ((u64)ctx->pool_used + me > ctx->pool_cap) {
        if ((rc = graph_compact(ctx, me))) return rc;
    }
    const GraphBatch g{ctx->pool_used, n, d_task};
    if (shard) {
        // the owned part of the batch, as local handles
        std::vector<u32> ot, oc;
        std::vector<u64> op;
        for (u32 i = 0; i < n; ++i)
            if (task[i] >= ctx->g_lo && task[i] < ctx->g_hi) {
                ot.push_back(task[i] - ctx->g_lo);
                oc.push_back(class_id[i]);
                op.push_back(priority[i]);
            }
        rc = push_impl(ctx, (u32)ot.size(), ot.data(), 0, oc.data(), op.data(), &g);
    } else {
        rc = push_impl(ctx, n, task, 0, class_id, priority, &g);
    }
    if (rc) return rc;
    ctx->pool_used += me;
    ctx->graph = true;
    if (n_ready) *n_ready = ctx->h_cnt->ready;
    return HQS_OK;
}

// The newly ready (hqs_graph_finished) or cancelled (hqs_graph_cancel) handles flagged in d_gbits, ascending, into
// d_gready; *n into d_gsmall[1].  The bitmap is cleared.
void graph_emit_bits(hqs_ctx* ctx) {
    const u32 n_words = (graph_bound(ctx) + 31) / 32, nb = (n_words + GRAPH_PER_BLOCK - 1) / GRAPH_PER_BLOCK;
    graph_ready_count_k<<<nb, GRAPH_NT, 0, ctx->stream>>>(n_words, ctx->d_gbits, ctx->d_gblk);
    graph_scan_k<<<1, 1024, 0, ctx->stream>>>(nb, ctx->d_gblk, ctx->d_gsmall + 1);
    graph_ready_emit_k<<<nb, GRAPH_NT, 0, ctx->stream>>>(n_words, ctx->d_gbits, ctx->d_gblk, ctx->d_gready);
}

// the body of hqs_graph_finished and hqs_shard_graph_finished, after the mode check
int graph_finished_impl(hqs_ctx* ctx, u32 n, const u32* task, const u32** new_ready, u32* n_new_ready) {
    if (n == 0) return HQS_OK;
    if (!task) return fail(ctx, HQS_E_INVALID, "null task array");
    const u32 bound = graph_bound(ctx);
    for (u32 i = 0; i < n; ++i)
        if (task[i] >= bound) return fail(ctx, HQS_E_INVALID, "task %u >= n_handles %u (nothing was finished)", task[i], bound);
    CU(cudaSetDevice(ctx->device));
    int rc;
    if ((rc = ensure_graph_storage(ctx))) return rc;
    if ((rc = ensure_push_staging(ctx, n))) return rc;
    u32* win = ctx->d_push_cls;          // the staging of class ids is free during this call
    CU(cudaMemcpyAsync(ctx->d_push_task, task, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    const GraphKeys gk = graph_keys(ctx);
    graph_dispatch(ctx->shard_graph, [&](auto S) {
        constexpr bool s = decltype(S)::value;
        graph_leave_k<s><<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, ctx->d_push_task, gk, win);
        graph_release_k<s><<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, win, gk, ctx->d_gdeps, ctx->d_ggen, ctx->d_ghead,
                                                                     ctx->d_pool, ctx->d_gbits);
    });
    graph_emit_bits(ctx);
    ctx->stats.kernel_launches += 5;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(&ctx->h_cnt->emitted, ctx->d_gsmall + 1, sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    const u32 k = ctx->h_cnt->emitted;
    ctx->g_new_ready.resize(k);
    if (k) {
        CU(cudaMemcpyAsync(ctx->g_new_ready.data(), ctx->d_gready, (size_t)k * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
    }
    if (new_ready) *new_ready = ctx->g_new_ready.data();
    if (n_new_ready) *n_new_ready = k;
    return HQS_OK;
}

// the body of hqs_graph_cancel and hqs_shard_graph_cancel, after the mode check.  A sharded graph context marks, emits and
// applies the whole closure and returns the part it owns.
int graph_cancel_impl(hqs_ctx* ctx, u32 n, const u32* task, const u32** cancelled, u32* n_cancelled) {
    if (n == 0) return HQS_OK;
    if (!task) return fail(ctx, HQS_E_INVALID, "null task array");
    const u32 bound = graph_bound(ctx);
    for (u32 i = 0; i < n; ++i)
        if (task[i] >= bound) return fail(ctx, HQS_E_INVALID, "task %u >= n_handles %u (nothing was cancelled)", task[i], bound);
    CU(cudaSetDevice(ctx->device));
    int rc;
    if ((rc = ensure_graph_storage(ctx))) return rc;
    if ((rc = ensure_push_staging(ctx, n))) return rc;
    CU(cudaMemcpyAsync(ctx->d_push_task, task, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemsetAsync(ctx->d_gcsync, 0, sizeof(GraphCancelSync), ctx->stream));
    // the launches do not depend on the depth of the closure: seed, marking (the whole closure), ordered emit, apply
    GraphKeys gk = graph_keys(ctx);
    cudaError_t launched = cudaSuccess;
    graph_dispatch(ctx->shard_graph, [&](auto S) {
        constexpr bool s = decltype(S)::value;
        graph_cancel_seed_k<s><<<(n + 255) / 256, 256, 0, ctx->stream>>>(n, ctx->d_push_task, gk, ctx->d_gbits, ctx->d_gwork,
                                                                         ctx->d_gcsync);
        const u32* gdeps = ctx->d_gdeps; const u32* ggen = ctx->d_ggen; const u32* ghead = ctx->d_ghead;
        const GraphEdge* pool = ctx->d_pool;
        u32* bits = ctx->d_gbits; u32* work = ctx->d_gwork; GraphCancelSync* sync = ctx->d_gcsync;
        void* kargs[] = {&gk, &gdeps, &ggen, &ghead, &pool, &bits, &work, &sync};
        launched = cudaLaunchCooperativeKernel((const void*)graph_cancel_mark_k<s>, dim3(ctx->grid_ctas), dim3(GRAPH_CANCEL_NT),
                                               kargs, 0, ctx->stream);
    });
    CU(launched);
    graph_emit_bits(ctx);
    graph_dispatch(ctx->shard_graph, [&](auto S) {
        graph_cancel_apply_k<decltype(S)::value><<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(
            ctx->d_gwork, ctx->d_gcsync, ctx->d_gready, ctx->d_gsmall + 1, gk, ctx->d_ghead);
    });
    ctx->stats.kernel_launches += 6;
    CU(cudaGetLastError());
    GraphCancelSync hs;
    CU(cudaMemcpyAsync(&hs, ctx->d_gcsync, sizeof hs, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(&ctx->h_cnt->emitted, ctx->d_gsmall + 1, sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    if (hs.error || !hs.done)
        return fail(ctx, HQS_E_CUDA, "a wait of the cancel marking kernel timed out (%s; %u handles marked, nothing was cancelled)",
                    hs.error == 2 ? "a work-list slot that was never written" : "the work list made no progress", hs.tail);
    const u32 k = ctx->h_cnt->emitted;
    ctx->g_new_ready.resize(k);
    if (k) {
        CU(cudaMemcpyAsync(ctx->g_new_ready.data(), ctx->d_gready, (size_t)k * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
    }
    const u32* first = ctx->g_new_ready.data();
    const u32* last = first + k;
    if (ctx->shard_graph) {          // ascending: the owned handles are one run
        first = std::lower_bound(first, last, ctx->g_lo);
        last = std::lower_bound(first, last, ctx->g_hi);
    }
    if (cancelled) *cancelled = first;
    if (n_cancelled) *n_cancelled = (u32)(last - first);
    return HQS_OK;
}

// The body of hqs_handles_compact, after the checks (keep staged at d_push_task).  Nothing of the context is written
// before the end: the survivors are gathered into fresh arrays, the edges into a fresh pool, and these replace the
// context's arrays only once every kernel and copy has succeeded.
int handles_compact_impl(hqs_ctx* ctx, u32 n_keep) {
    const u32 nh = ctx->n_handles, cap = ctx->cap_handles;
    const u32 n_words = (nh + 31) / 32;
    const u32 nb_words = (n_words + GRAPH_PER_BLOCK - 1) / GRAPH_PER_BLOCK;   // ordered emit over the bitmap
    const u32 nb_lists = (nh + GRAPH_PER_BLOCK - 1) / GRAPH_PER_BLOCK;        // edge rewrite over the producers
    const bool graph = ctx->graph_storage;
    const bool edges = graph && ctx->d_pool;
    cudaStream_t s = ctx->stream;
    Buf<u32> bits, order, new_of_old, blk, key, gdeps, ggen, ghead;
    Buf<u64> prio;
    Buf<GraphEdge> pool;
    CU(bits.grow(n_words, s, false, 0));
    CU(order.grow(nh, s));
    CU(new_of_old.grow(nh, s));
    CU(blk.grow((size_t)std::max(nb_words, nb_lists) + 2, s));     // per-block sums, then the two totals
    CU(key.grow(cap, s, false, 0));
    CU(prio.grow(cap, s, false, 0));
    if (graph) {
        CU(gdeps.grow(cap, s, false, 0));
        CU(ggen.grow(cap, s, false, 0));
        CU(ghead.grow(cap, s, false, 0xFF));
    }
    if (edges) CU(pool.grow(ctx->pool_cap, s));
    u32* total = blk + std::max(nb_words, nb_lists);                // [0] survivors, [1] live edges
    CU(cudaMemsetAsync(total, 0, 2 * sizeof(u32), s));
    const u32 nt = std::max(nh, n_keep);
    compact_mark_k<<<(nt + 255) / 256, 256, 0, s>>>(nh, ctx->d_key, n_keep, ctx->d_push_task, bits);
    graph_ready_count_k<<<nb_words, GRAPH_NT, 0, s>>>(n_words, bits, blk);
    graph_scan_k<<<1, 1024, 0, s>>>(nb_words, blk, total);
    graph_ready_emit_k<<<nb_words, GRAPH_NT, 0, s>>>(n_words, bits, blk, order);
    ctx->stats.kernel_launches += 4;
    const GraphKeys gk = graph_keys(ctx);
    if (edges) {
        graph_gc_count_k<false><<<nb_lists, GRAPH_NT, 0, s>>>(nh, ctx->d_ghead, ctx->d_pool, gk, ctx->d_gdeps, ctx->d_ggen, blk);
        graph_scan_k<<<1, 1024, 0, s>>>(nb_lists, blk, total + 1);
        ctx->stats.kernel_launches += 2;
    }
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(&ctx->h_cnt->kept, total, 2 * sizeof(u32), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    const u32 n_kept = ctx->h_cnt->kept, live = ctx->h_cnt->live;
    if (n_kept) {
        compact_gather_k<<<(n_kept + 255) / 256, 256, 0, s>>>(n_kept, order, ctx->d_key, ctx->d_prio,
                                                              graph ? (u32*)ctx->d_gdeps : nullptr, ctx->d_ggen, key, prio,
                                                              gdeps, ggen, new_of_old);
        ctx->stats.kernel_launches++;
    }
    if (edges) {
        graph_gc_move_k<false, true><<<nb_lists, GRAPH_NT, 0, s>>>(nh, ctx->d_ghead, ctx->d_pool, pool, gk, ctx->d_gdeps,
                                                                    ctx->d_ggen, blk, new_of_old, ghead);
        ctx->stats.kernel_launches++;
    }
    CU(cudaGetLastError());
    ctx->g_new_ready.resize(n_kept);
    if (n_kept) CU(cudaMemcpyAsync(ctx->g_new_ready.data(), order, (size_t)n_kept * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->d_key = std::move(key);
    ctx->d_prio = std::move(prio);
    if (graph) {
        ctx->d_gdeps = std::move(gdeps);
        ctx->d_ggen = std::move(ggen);
        ctx->d_ghead = std::move(ghead);
    }
    if (edges) {
        ctx->d_pool = std::move(pool);
        ctx->pool_used = live;
    }
    ctx->n_handles = n_kept;
    ctx->stats.n_handles = n_kept;
    return HQS_OK;
}

// The body of hqs_shard_graph_compact, after the checks (keep staged at d_push_task).  Every rank runs the same kernels on
// the same replicated state and the same keep list, so the replicas stay equal and every rank derives the same renumbering;
// only the own keys differ.  As in handles_compact_impl, everything is gathered into fresh arrays that replace the context's
// only at the end.  range receives the new owned range.
int shard_graph_compact_impl(hqs_ctx* ctx, u32 n_keep, u32 range[2]) {
    const u32 nt = ctx->g_total, gcap = (nt + 1023u) & ~1023u;
    const u32 n_words = (nt + 31) / 32;
    const u32 nb_words = (n_words + GRAPH_PER_BLOCK - 1) / GRAPH_PER_BLOCK;
    const u32 nb_lists = (nt + GRAPH_PER_BLOCK - 1) / GRAPH_PER_BLOCK;
    const bool edges = ctx->d_pool;
    cudaStream_t s = ctx->stream;
    Buf<u32> bits, order, new_of_old, blk, gvalid, gdeps, ggen, ghead, key;
    Buf<u64> prio;
    Buf<GraphEdge> pool;
    CU(bits.grow(n_words, s, false, 0));
    CU(order.grow(nt, s));
    CU(new_of_old.grow(nt, s));
    CU(blk.grow((size_t)std::max(nb_words, nb_lists) + 4, s));     // per-block sums, then the four totals
    CU(gvalid.grow(gcap / 32, s, false, 0));
    CU(gdeps.grow(gcap, s, false, 0));
    CU(ggen.grow(gcap, s, false, 0));
    CU(ghead.grow(gcap, s, false, 0xFF));
    if (edges) CU(pool.grow(ctx->pool_cap, s));
    u32* total = blk + std::max(nb_words, nb_lists);                // [0] survivors, [1] live edges, [2] new(lo), [3] new(hi)
    CU(cudaMemsetAsync(total, 0, 4 * sizeof(u32), s));
    const u32 nm = std::max(n_words, n_keep);
    shard_compact_mark_k<<<(nm + 255) / 256, 256, 0, s>>>(n_words, ctx->d_gvalid, n_keep, ctx->d_push_task, bits);
    graph_ready_count_k<<<nb_words, GRAPH_NT, 0, s>>>(n_words, bits, blk);
    graph_scan_k<<<1, 1024, 0, s>>>(nb_words, blk, total);
    graph_ready_emit_k<<<nb_words, GRAPH_NT, 0, s>>>(n_words, bits, blk, order);
    shard_compact_range_k<<<1, 32, 0, s>>>(order, total, ctx->g_lo, ctx->g_hi, total + 2);
    ctx->stats.kernel_launches += 5;
    const GraphKeys gk = graph_keys(ctx);
    if (edges) {
        graph_gc_count_k<true><<<nb_lists, GRAPH_NT, 0, s>>>(nt, ctx->d_ghead, ctx->d_pool, gk, ctx->d_gdeps, ctx->d_ggen, blk);
        graph_scan_k<<<1, 1024, 0, s>>>(nb_lists, blk, total + 1);
        ctx->stats.kernel_launches += 2;
    }
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(&ctx->h_cnt->kept, total, 4 * sizeof(u32), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    const u32 n_kept = ctx->h_cnt->kept, live = ctx->h_cnt->live, own_lo = ctx->h_cnt->own_lo, own_hi = ctx->h_cnt->own_hi;
    // new(h) = survivors below h, except new(n_total) = n_total: the rank whose range ends at n_total takes the freed tail
    // (a rank with the empty range [n_total, n_total) keeps it), so the ranges still tile [0, n_total) in rank order
    const u32 new_lo = ctx->g_lo == nt ? nt : own_lo, new_hi = ctx->g_hi == nt ? nt : own_hi;
    const u32 n_own = own_hi - own_lo;
    const u32 cap = std::max(ctx->cap_handles, (n_own + 1023u) & ~1023u);
    if (cap) {
        CU(key.grow(cap, s, false, 0));
        CU(prio.grow(cap, s, false, 0));
    }
    if (n_kept) {
        shard_compact_gather_k<<<(n_kept + 255) / 256, 256, 0, s>>>(n_kept, order, ctx->d_gvalid, ctx->d_gdeps, ctx->d_ggen,
                                                                    ctx->g_lo, ctx->n_handles, own_lo, own_hi, ctx->d_key,
                                                                    ctx->d_prio, gvalid, gdeps, ggen, key, prio, new_of_old);
        ctx->stats.kernel_launches++;
    }
    if (edges) {
        graph_gc_move_k<true, true><<<nb_lists, GRAPH_NT, 0, s>>>(nt, ctx->d_ghead, ctx->d_pool, pool, gk, ctx->d_gdeps,
                                                                   ctx->d_ggen, blk, new_of_old, ghead);
        ctx->stats.kernel_launches++;
    }
    CU(cudaGetLastError());
    ctx->g_new_ready.resize(n_kept);
    if (n_kept) CU(cudaMemcpyAsync(ctx->g_new_ready.data(), order, (size_t)n_kept * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->d_gvalid = std::move(gvalid);
    ctx->d_gdeps = std::move(gdeps);
    ctx->d_ggen = std::move(ggen);
    ctx->d_ghead = std::move(ghead);
    ctx->d_key = std::move(key);
    ctx->d_prio = std::move(prio);
    ctx->cap_handles = cap;
    if (edges) {
        ctx->d_pool = std::move(pool);
        ctx->pool_used = live;
    }
    ctx->n_handles = n_own;
    ctx->stats.n_handles = n_own;
    ctx->g_lo = new_lo;
    ctx->g_hi = new_hi;
    range[0] = new_lo;
    range[1] = new_hi;
    return HQS_OK;
}
}  // namespace

extern "C" {

int hqs_graph_push(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t* class_id, const uint64_t* priority,
                   const uint32_t* dep_off, const uint32_t* deps, uint32_t* n_ready) {
    if (!ctx) return HQS_E_INVALID;
    if (n_ready) *n_ready = 0;
    if (int rc = graph_mode_check(ctx, "hqs_graph_push")) return rc;
    return graph_push_impl(ctx, n, task, class_id, priority, dep_off, deps, n_ready);
}

int hqs_graph_finished(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t** new_ready, uint32_t* n_new_ready) {
    if (!ctx) return HQS_E_INVALID;
    ctx->g_new_ready.clear();
    if (new_ready) *new_ready = ctx->g_new_ready.data();
    if (n_new_ready) *n_new_ready = 0;
    if (int rc = graph_mode_check(ctx, "hqs_graph_finished")) return rc;
    return graph_finished_impl(ctx, n, task, new_ready, n_new_ready);
}

int hqs_graph_cancel(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t** cancelled, uint32_t* n_cancelled) {
    if (!ctx) return HQS_E_INVALID;
    ctx->g_new_ready.clear();
    if (cancelled) *cancelled = ctx->g_new_ready.data();
    if (n_cancelled) *n_cancelled = 0;
    if (int rc = graph_mode_check(ctx, "hqs_graph_cancel")) return rc;
    return graph_cancel_impl(ctx, n, task, cancelled, n_cancelled);
}

int hqs_graph_debug(hqs_ctx* ctx, uint64_t out[4]) {
    if (!ctx || !out) return HQS_E_INVALID;
    if (int rc = ctx->shard_graph ? shard_graph_mode_check(ctx, "hqs_graph_debug") : graph_mode_check(ctx, "hqs_graph_debug"))
        return rc;
    CU(cudaSetDevice(ctx->device));
    Buf<unsigned long long> d_out;
    CU(d_out.grow(2, ctx->stream));
    unsigned long long h[2] = {0, 0};
    CU(cudaMemsetAsync(d_out, 0, sizeof h, ctx->stream));
    if (ctx->shard_graph) {
        // the replicated lists over the global handles, the waiting tasks over the own keys
        graph_debug_k<<<(ctx->g_total + 255) / 256, 256, 0, ctx->stream>>>(ctx->g_total, nullptr, ctx->d_ghead, ctx->d_pool, d_out);
        if (ctx->n_handles)
            graph_debug_k<<<(ctx->n_handles + 255) / 256, 256, 0, ctx->stream>>>(ctx->n_handles, ctx->d_key, nullptr, nullptr, d_out);
        ctx->stats.kernel_launches += ctx->n_handles ? 2 : 1;
        CU(cudaGetLastError());
    } else if (ctx->n_handles) {
        graph_debug_k<<<(ctx->n_handles + 255) / 256, 256, 0, ctx->stream>>>(ctx->n_handles, ctx->d_key,
                                                                           ctx->graph_storage ? (u32*)ctx->d_ghead : nullptr, ctx->d_pool, d_out);
        ctx->stats.kernel_launches++;
        CU(cudaGetLastError());
    }
    CU(cudaMemcpyAsync(h, d_out, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    out[0] = h[0];
    out[1] = ctx->pool_cap;
    out[2] = ctx->pool_compactions;
    out[3] = h[1];
    return HQS_OK;
}

int hqs_handles_compact(hqs_ctx* ctx, uint32_t n_keep, const uint32_t* keep, const uint32_t** old_of_new, uint32_t* n_kept) {
    if (!ctx) return HQS_E_INVALID;
    ctx->g_new_ready.clear();
    if (old_of_new) *old_of_new = ctx->g_new_ready.data();
    if (n_kept) *n_kept = 0;
    if (ctx->dag) return fail(ctx, HQS_E_STATE, "hqs_handles_compact is not available after hqs_dag_load");
    if (ctx->x_world) return fail(ctx, HQS_E_STATE, "hqs_handles_compact is not available on a sharded ready set");
    if (ctx->shard_graph) return fail(ctx, HQS_E_STATE, "hqs_handles_compact is not available on a sharded graph context");
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    if (n_keep && !keep) return fail(ctx, HQS_E_INVALID, "null keep array");
    for (u32 i = 0; i < n_keep; ++i)
        if (keep[i] >= ctx->n_handles)
            return fail(ctx, HQS_E_INVALID, "keep handle %u >= n_handles %u (nothing was compacted)", keep[i], ctx->n_handles);
    if (!ctx->n_handles) return HQS_OK;
    CU(cudaSetDevice(ctx->device));
    if (int rc = ensure_push_staging(ctx, n_keep)) return rc;
    if (n_keep) CU(cudaMemcpyAsync(ctx->d_push_task, keep, (size_t)n_keep * 4, cudaMemcpyHostToDevice, ctx->stream));
    const int rc = handles_compact_impl(ctx, n_keep);
    if (rc) {
        ctx->g_new_ready.clear();
        cudaStreamSynchronize(ctx->stream);       // the caller may free keep as soon as we return
        return rc;
    }
    if (old_of_new) *old_of_new = ctx->g_new_ready.data();
    if (n_kept) *n_kept = (u32)ctx->g_new_ready.size();
    return HQS_OK;
}

int hqs_shard_graph_compact(hqs_ctx* ctx, uint32_t n_keep, const uint32_t* keep, const uint32_t** old_of_new,
                            uint32_t* n_kept, uint32_t new_range[2]) {
    if (!ctx) return HQS_E_INVALID;
    ctx->g_new_ready.clear();
    if (old_of_new) *old_of_new = ctx->g_new_ready.data();
    if (n_kept) *n_kept = 0;
    if (new_range) {
        new_range[0] = ctx->g_lo;
        new_range[1] = ctx->g_hi;
    }
    if (int rc = shard_graph_mode_check(ctx, "hqs_shard_graph_compact")) return rc;
    if (n_keep && !keep) return fail(ctx, HQS_E_INVALID, "null keep array");
    for (u32 i = 0; i < n_keep; ++i)
        if (keep[i] >= ctx->g_total)
            return fail(ctx, HQS_E_INVALID, "keep handle %u >= n_total %u (nothing was compacted)", keep[i], ctx->g_total);
    if (!ctx->g_total) return HQS_OK;
    u32 range[2];
    const int rc = shard_graph_outcome(ctx, [&]() -> int {
        CU(cudaSetDevice(ctx->device));
        if (int r = ensure_push_staging(ctx, n_keep)) return r;
        if (n_keep) CU(cudaMemcpyAsync(ctx->d_push_task, keep, (size_t)n_keep * 4, cudaMemcpyHostToDevice, ctx->stream));
        return shard_graph_compact_impl(ctx, n_keep, range);
    }());
    if (rc) {
        ctx->g_new_ready.clear();
        cudaStreamSynchronize(ctx->stream);       // the caller may free keep as soon as we return
        return rc;
    }
    if (old_of_new) *old_of_new = ctx->g_new_ready.data();
    if (n_kept) *n_kept = (u32)ctx->g_new_ready.size();
    if (new_range) {
        new_range[0] = range[0];
        new_range[1] = range[1];
    }
    return HQS_OK;
}

int hqs_shard_graph_init(hqs_ctx* ctx, uint32_t n_total, uint32_t lo, uint32_t hi) {
    if (!ctx) return HQS_E_INVALID;
    if (ctx->shard_graph) return fail(ctx, HQS_E_STATE, "hqs_shard_graph_init was called before");
    if (ctx->dag) return fail(ctx, HQS_E_STATE, "hqs_shard_graph_init is not available after hqs_dag_load");
    if (ctx->graph) return fail(ctx, HQS_E_STATE, "hqs_shard_graph_init is not available after hqs_graph_push");
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    if (lo > hi || hi > n_total) return fail(ctx, HQS_E_INVALID, "owned range [%u, %u) is not inside [0, %u)", lo, hi, n_total);
    if (n_total > GRAPH_NIL - 1024u) return fail(ctx, HQS_E_LIMIT, "n_total %u is too large", n_total);
    CU(cudaSetDevice(ctx->device));
    if (ctx->n_handles) {            // the replica must see every live task: the table must hold none yet
        std::vector<u32> keys(ctx->n_handles);
        CU(cudaMemcpyAsync(keys.data(), ctx->d_key, (size_t)ctx->n_handles * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        for (u32 k : keys)
            if (k & KEY_VALID) return fail(ctx, HQS_E_STATE, "the task table already holds a live task");
    }
    const u32 cap = (n_total + 1023u) & ~1023u;
    CU(ctx->d_gvalid.grow(cap / 32, ctx->stream, false, 0));
    ctx->shard_graph = true;
    ctx->g_total = n_total;
    ctx->g_lo = lo;
    ctx->g_hi = hi;
    ctx->graph_storage = false;      // arrays a graph call on the empty table may have made are re-made at the global size
    int rc = ensure_graph_storage(ctx);
    if (!rc) CU(cudaStreamSynchronize(ctx->stream));
    return rc;
}

int hqs_shard_graph_push(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t* class_id, const uint64_t* priority,
                         const uint32_t* dep_off, const uint32_t* deps, uint32_t* n_ready) {
    if (!ctx) return HQS_E_INVALID;
    if (n_ready) *n_ready = 0;
    if (int rc = shard_graph_mode_check(ctx, "hqs_shard_graph_push")) return rc;
    return shard_graph_outcome(ctx, graph_push_impl(ctx, n, task, class_id, priority, dep_off, deps, n_ready));
}

int hqs_shard_graph_finished(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t** new_ready, uint32_t* n_new_ready) {
    if (!ctx) return HQS_E_INVALID;
    ctx->g_new_ready.clear();
    if (new_ready) *new_ready = ctx->g_new_ready.data();
    if (n_new_ready) *n_new_ready = 0;
    if (int rc = shard_graph_mode_check(ctx, "hqs_shard_graph_finished")) return rc;
    return shard_graph_outcome(ctx, graph_finished_impl(ctx, n, task, new_ready, n_new_ready));
}

int hqs_shard_graph_cancel(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t** cancelled, uint32_t* n_cancelled) {
    if (!ctx) return HQS_E_INVALID;
    ctx->g_new_ready.clear();
    if (cancelled) *cancelled = ctx->g_new_ready.data();
    if (n_cancelled) *n_cancelled = 0;
    if (int rc = shard_graph_mode_check(ctx, "hqs_shard_graph_cancel")) return rc;
    return shard_graph_outcome(ctx, graph_cancel_impl(ctx, n, task, cancelled, n_cancelled));
}

int hqs_shard_graph_remove(hqs_ctx* ctx, uint32_t n, const uint32_t* task) {
    if (!ctx) return HQS_E_INVALID;
    if (int rc = shard_graph_mode_check(ctx, "hqs_shard_graph_remove")) return rc;
    return shard_graph_outcome(ctx, shard_graph_remove_impl(ctx, n, task));
}

int hqs_tick_launch(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
                    const uint64_t* total_rw, const uint8_t* blocked_wcv, uint32_t out_cap) {
    if (!ctx) return HQS_E_INVALID;
    int rc = validate_workers(ctx, n_workers, workers, free_rw, total_rw);
    if (rc) return rc;
    TickGeom t;
    if ((rc = stage_tick(ctx, n_workers, workers, free_rw, total_rw, blocked_wcv, out_cap, ~0u, &t))) return rc;
    if ((rc = launch_tick(ctx, t, nullptr, nullptr, out_cap, true, false))) return rc;
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
    if (!worker_off || off_cap < 2 * ctx->staged.W + 2)
        return fail(ctx, HQS_E_INVALID, "worker_off needs 2 * n_workers + 2 = %u entries (off_cap=%u)", 2 * ctx->staged.W + 2, off_cap);
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
    int rc = ensure_group_buffers(ctx, n_workers, std::max(out_cap, (u32)ctx->d_out.size()));
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
    const u32 W = ctx->staged.W;
    if (free_after) memcpy(free_after, ctx->tick.h_hdr + sizeof(TickHeaderOut), (size_t)W * ctx->R * 8);
    // the count segments cover every group's assigned ranks [0, k), so the per-worker counts sum to the tasks assigned over
    // all ranks; the header's n_assigned of a sharded launch is this rank's share only (the solver's local output offsets)
    u32 total = 0;
    for (u32 w = 0; w < W; ++w) total += ctx->h_pw[w];
    ctx->stats.n_assigned = total;
    if (n_would_assign) *n_would_assign = total;
    if (per_worker_assigned) memcpy(per_worker_assigned, ctx->h_pw, W * sizeof(u32));
    return HQS_OK;
}

int hqs_shard_count(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
                    const uint64_t* total_rw, const uint8_t* blocked_wcv, uint32_t* d_counts, uint32_t n_groups_cap,
                    uint32_t* n_groups) {
    if (!ctx) return HQS_E_INVALID;
    int rc = validate_workers(ctx, n_workers, workers, free_rw, total_rw);
    if (rc) return rc;
    if (!d_counts) return fail(ctx, HQS_E_INVALID, "null d_counts");
    TickGeom t;
    if ((rc = stage_tick(ctx, n_workers, workers, free_rw, total_rw, blocked_wcv, 1024, n_groups_cap, &t))) return rc;
    CU(cudaMemsetAsync(ctx->d_total, 0, (size_t)t.G * 4, ctx->stream));
    if (ctx->n_handles) {
        TickArgs a = base_args(ctx, t);
        count_only_k<<<std::min<u32>(t.P, ctx->sm_count * 2), TICK_THREADS, t.G * sizeof(u32), ctx->stream>>>(a);
        ctx->stats.kernel_launches++;
        CU(cudaGetLastError());
    }
    CU(cudaMemsetAsync(d_counts, 0, (size_t)n_groups_cap * 4, ctx->stream));
    CU(cudaMemcpyAsync(d_counts, ctx->d_total, (size_t)t.G * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    if (n_groups) *n_groups = t.G;
    return HQS_OK;
}

int hqs_shard_solve_emit(hqs_ctx* ctx, const uint32_t* d_counts_all, const uint32_t* d_ranks_before, uint32_t out_cap) {
    if (!ctx) return HQS_E_INVALID;
    if (!d_counts_all || !d_ranks_before) return fail(ctx, HQS_E_INVALID, "null count vectors");
    if (!ctx->staged.W) return fail(ctx, HQS_E_STATE, "hqs_shard_count has not been called");
    CU(cudaSetDevice(ctx->device));
    const TickGeom t = tick_geom(ctx);
    int rc = ensure_tick_buffers(ctx, t.G, t.P, out_cap);
    if (rc) return rc;
    // over the tick input hqs_shard_count staged
    if ((rc = launch_tick(ctx, t, d_counts_all, d_ranks_before, out_cap, true, false))) return rc;
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
    int rc = ensure_tick_buffers(ctx, t.G, t.P, out_cap);
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
        Buf<u32> xbuf, xall, xbefore;
        CU(xbuf.grow(xbuf_bytes() / sizeof(u32), ctx->stream));
        CU(cudaMemset(xbuf, 0, xbuf_bytes()));
        CU(xall.grow(HQS_MAX_GROUPS, ctx->stream));
        CU(xbefore.grow(HQS_MAX_GROUPS, ctx->stream));
        ctx->d_xbuf = std::move(xbuf);
        ctx->d_xall = std::move(xall);
        ctx->d_xbefore = std::move(xbefore);
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
    TickGeom t;
    if ((rc = stage_tick(ctx, n_workers, workers, free_rw, total_rw, blocked_wcv, out_cap, ~0u, &t))) return rc;
    // every rank advances the sequence number in lockstep (one sharded tick = one exchange)
    ctx->x_seq += 1;
    if ((rc = launch_tick(ctx, t, nullptr, nullptr, out_cap, true, true))) return rc;
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
    if (!ctx->staged.W) return fail(ctx, HQS_E_STATE, "hqs_shard_count has not been called");
    if (ctx->tick_pending) return fail(ctx, HQS_E_STATE, "the previous tick has not been fetched");
    CU(cudaSetDevice(ctx->device));
    const TickGeom t = tick_geom(ctx);
    int rc = ensure_tick_buffers(ctx, t.G, t.P, 1024);
    if (rc) return rc;
    // over the tick input hqs_shard_count staged
    return launch_query(ctx, t, d_counts_all, false);
}

int hqs_device_result(hqs_ctx* ctx, const hqs_assignment** d_out, const uint32_t** d_out_n) {
    if (!ctx) return HQS_E_INVALID;
    if (d_out) *d_out = ctx->d_out;
    TickHeaderOut* hdr = ctx->tick.hdr;
    if (d_out_n) *d_out_n = hdr ? &hdr->n_assigned : nullptr;
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
