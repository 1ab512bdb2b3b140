// hqs_ready_set.cuh — task-table key encoding, per-tick device records and the ready-set maintenance kernels.
// Included by hqsched.cu inside its anonymous namespace (one translation unit; see the header of hqsched.cu).
#pragma once

constexpr u32 KEY_READY = 1u << 31;
constexpr u32 KEY_DONE = 1u << 30;
constexpr u32 KEY_VALID = 1u << 29;
constexpr u32 KEY_PF = 1u << 28;          // ready AND prefilled on a worker (mapping.rs:156-230): still assignable
constexpr u32 KEY_LEVEL_SHIFT = 14;
constexpr u32 KEY_LEVEL_MASK = 0x3FFFu;     // bits 14..27 (levels <= HQS_MAX_GROUPS); bit 28 is KEY_PF
constexpr u32 KEY_CLASS_MASK = 0x3FFFu;

constexpr u32 SEG_CAP = 1u << 20;         // (group, worker, variant) count segments per tick
constexpr u32 NEWPRIO_CAP = 4096;

__device__ __forceinline__ u32 key_level(u32 k) { return (k >> KEY_LEVEL_SHIFT) & KEY_LEVEL_MASK; }
__device__ __forceinline__ u32 key_class(u32 k) { return k & KEY_CLASS_MASK; }

// Per-group result of the solver, read by emit_k with one 16-byte load.
struct __align__(16) GroupOut {
    u32 k;        // tasks of this group assigned this tick (global count in sharded mode)
    u32 out_off;  // offset of the group's first assignment in the (local) output
    u32 seg_lo;   // first count segment
    u32 seg_n;    // number of count segments
};

struct TickHeaderOut {
    u32 n_assigned;  // local assignments
    u32 n_groups;
    u32 n_segments;
    u32 error;       // 1 = segment overflow, 2 = a grid wait timed out, 3 = out_cap too small (nothing was emitted),
                     // 4 = sharded tick: a peer has another group count G (nothing was solved or emitted)
    u32 n_prefilled; // prefill records (kind 1) behind the assignments (this rank's, in a sharded tick)
    u32 pad;         // detail of error 2: which wait timed out
    u32 solver_path; // HQS_PATH_* bits: which solve loops ran (hqs_stats.solver_path)
    u32 pad2;        // detail of error 4: 1 << 31 | peer rank << 16 | the peer's G
    unsigned long long dbg[8];   // clock64 phase lengths of the solver CTA (hqs_debug_read)
};

// ------------------------------------------------------------------------------------------------
// level lookup: levels[] sorted by DESCENDING priority.  exact mode: index of the entry equal to p
// (or ~0u if absent); coarse mode: levels[i] is the lowest priority of bucket i, index of the first
// bucket whose bound <= p (clamped to the last bucket).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ u32 find_level(const u64* __restrict__ levels, u32 n_levels, u64 p, bool coarse) {
    u32 lo = 0, hi = n_levels;  // first index with levels[i] <= p
    while (lo < hi) {
        u32 mid = (lo + hi) >> 1;
        if (__ldg(levels + mid) <= p) hi = mid; else lo = mid + 1;
    }
    if (coarse) return lo < n_levels ? lo : n_levels - 1;
    if (lo < n_levels && __ldg(levels + lo) == p) return lo;
    return ~0u;
}

// ready-set maintenance ---------------------------------------------------------------------------
// class ids of a push are validated on the device, in the same stream, BEFORE push_k touches the table: flag[1] != 0 makes
// push_k a no-op, so a rejected batch leaves the ready set unchanged (no host pass over the arrays, no host sync in between)
__global__ void push_validate_k(u32 n, const u32* __restrict__ cls, u32 n_classes, u32* __restrict__ flag) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool bad = i < n && cls[i] >= n_classes;
    if (__ballot_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicMax(&flag[1], 1u);
}

// task == nullptr: the handles are first_handle .. first_handle + n - 1 (a task array: no handle array crosses PCIe)
__global__ void push_k(u32 n, const u32* __restrict__ task, u32 first_handle, const u32* __restrict__ cls,
                       const u64* __restrict__ prio_in, u32* __restrict__ key, u64* __restrict__ prio,
                       const u64* __restrict__ levels, u32 n_levels, int coarse, u32* __restrict__ newcnt,
                       u64* __restrict__ newprio) {
    if (newcnt[1]) return;                  // push_validate_k rejected the batch
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < n;
    const u32 h = live ? (task ? task[i] : first_handle + i) : 0u;
    const u64 p = live ? prio_in[i] : 0ull;
    u32 lvl = (live && n_levels) ? find_level(levels, n_levels, p, coarse != 0) : ~0u;
    // unknown priority: report it to the host (one atomic per warp), key it provisionally to level 0;
    // relevel_k fixes every key once the host has merged the new priority
    const bool fresh = live && lvl == ~0u;
    const u32 fm = __ballot_sync(0xffffffffu, fresh);
    if (fm) {
        const u32 lane = threadIdx.x & 31;
        u32 slot0 = 0;
        if (lane == (u32)(__ffs(fm) - 1)) slot0 = atomicAdd(newcnt, (u32)__popc(fm));
        slot0 = __shfl_sync(0xffffffffu, slot0, __ffs(fm) - 1);
        if (fresh) {
            const u32 slot = slot0 + __popc(fm & ((1u << lane) - 1));
            if (slot < NEWPRIO_CAP) newprio[slot] = p;
            lvl = 0;
        }
    }
    if (!live) return;
    prio[h] = p;
    key[h] = KEY_READY | KEY_VALID | (lvl << KEY_LEVEL_SHIFT) | (cls[i] & KEY_CLASS_MASK);
}

__global__ void relevel_k(u32 n_handles, u32* __restrict__ key, const u64* __restrict__ prio,
                          const u64* __restrict__ levels, u32 n_levels, int coarse) {
    u32 h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n_handles) return;
    u32 k = key[h];
    if (!(k & KEY_VALID)) return;
    u32 lvl = find_level(levels, n_levels, prio[h], coarse != 0);
    if (lvl == ~0u) lvl = 0;
    key[h] = (k & ~(KEY_LEVEL_MASK << KEY_LEVEL_SHIFT)) | (lvl << KEY_LEVEL_SHIFT);
}

__global__ void remove_k(u32 n, const u32* __restrict__ task, u32* __restrict__ key, u32 n_handles) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    u32 h = task[i];
    // the task leaves the table: not ready, and it no longer pins its priority level (level_live_k)
    if (h < n_handles) key[h] &= ~(KEY_READY | KEY_VALID | KEY_DONE | KEY_PF);
}

// marks the (exact) priority levels that still have a task in the table
__global__ void level_live_k(u32 n_handles, const u32* __restrict__ key, const u64* __restrict__ prio,
                             const u64* __restrict__ levels, u32 n_levels, u32* __restrict__ live) {
    const u32 h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n_handles || !(key[h] & KEY_VALID)) return;
    const u32 lvl = find_level(levels, n_levels, prio[h], false);
    if (lvl != ~0u && !live[lvl]) live[lvl] = 1u;
}

// TaskQueue::check_dispose_prefill (taskqueue.rs:146-152): the prefilled tasks of one class go back to plain waiting
__global__ void pf_dispose_k(u32 n_handles, u32* __restrict__ key, u32 cls) {
    const u32 h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n_handles) return;
    const u32 k = key[h];
    if ((k & KEY_PF) && key_class(k) == cls) key[h] = k & ~KEY_PF;
}

__global__ void rearm_k(u32 n_handles, u32* __restrict__ key) {
    u32 h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n_handles) return;
    u32 k = key[h];
    if (k & KEY_DONE) key[h] = (k & ~KEY_DONE) | KEY_READY;
}

__global__ void dag_init_k(u32 n, const u32* __restrict__ cls, const u64* __restrict__ prio,
                           const u32* __restrict__ deps, u32* __restrict__ key,
                           const u64* __restrict__ levels, u32 n_levels, int coarse) {
    u32 h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n) return;
    u32 lvl = find_level(levels, n_levels, prio[h], coarse != 0);
    if (lvl == ~0u) lvl = 0;
    key[h] = KEY_VALID | (deps[h] == 0 ? KEY_READY : 0u) | (lvl << KEY_LEVEL_SHIFT) | (cls[h] & KEY_CLASS_MASK);
}

// task_finished (reactor.rs:545-571): one thread per (finished task, consumer) pair would need a
// segmented layout; out-degree is small (<= 8 in the benchmark DAG), so one thread per finished task.
__global__ void finished_k(u32 n, const u32* __restrict__ task, const u32* __restrict__ cons_off,
                           const u32* __restrict__ cons, u32* __restrict__ deps, u32* __restrict__ key,
                           u32* __restrict__ n_new) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    u32 made = 0;
    if (i < n) {
        u32 t = task[i];
        u32 lo = cons_off[t], hi = cons_off[t + 1];
        for (u32 e = lo; e < hi; ++e) {
            u32 c = cons[e];
            if (atomicSub(&deps[c], 1u) == 1u && (key[c] & KEY_VALID)) {  // decrease_unfinished_deps() hit zero (a removed consumer stays out)
                atomicOr(&key[c], KEY_READY);
                ++made;
            }
        }
        key[t] &= ~(KEY_VALID | KEY_DONE | KEY_READY | KEY_PF);      // finished for good: the handle no longer pins its priority level
    }
    made = __reduce_add_sync(0xffffffffu, made);
    if ((threadIdx.x & 31) == 0 && made) atomicAdd(n_new, made);
}
