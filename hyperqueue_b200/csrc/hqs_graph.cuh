// hqs_graph.cuh — task graphs that grow while the ready set runs: hqs_graph_push / hqs_graph_finished (on_new_tasks and
// task_finished, reactor.rs:188-220, 500-580) and hqs_graph_cancel (on_cancel_tasks / task_failed, reactor.rs:596-770).
// Included by hqsched.cu inside its anonymous namespace, after hqs_ready_set.cuh and hqs_solver.cuh.
//
// Per handle h (allocated at the first graph push, grown with the task table):
//   gdeps[h]  u32  unfinished counted dependencies of h's current incarnation
//   ggen[h]   u32  incarnation: +1 at every hqs_graph_push of h
//   ghead[h]  u32  first edge of h's consumer list, GRAPH_NIL = none
// Edge pool: GraphEdge {consumer, consumer's incarnation, next}.  A push takes its slots by the batch's dependency offsets
// (no atomics) and links each counted edge in front of its producer's list.  A list is emptied whenever its producer
// leaves the table (finished, removed or cancelled), so head[h] != GRAPH_NIL implies that h is VALID.
// hqs_graph_cancel also keeps gwork[h] (a work list of n_handles slots, GRAPH_NIL between calls).
//
// A sharded graph context (hqs_shard_graph_init) keeps all of the above replicated, indexed by the GLOBAL handle
// (0 .. n_total), plus gvalid[h], one bit per handle: h is VALID in the graph's view.  Its key table holds only the handles
// it owns, [lo, hi), at key[h - lo].  Every rank makes every graph call with the same arguments and runs the same kernels on
// the same replicated state, so the replicas stay equal; each rank writes only the keys it owns and reports only the
// handles it owns.  The kernels take both forms through GraphKeys and a template flag S (false: one context).
#pragma once

constexpr u32 GRAPH_NIL = ~0u;
constexpr u32 GRAPH_POOL_MIN = 4096;      // edge slots of a fresh pool
constexpr u32 GRAPH_NT = 256;             // threads of the counting / emitting kernels
constexpr u32 GRAPH_PER_THREAD = 8;       // consecutive words (ready bitmap) or handles (pool compaction) per thread
constexpr u32 GRAPH_PER_BLOCK = GRAPH_NT * GRAPH_PER_THREAD;

struct GraphEdge {
    u32 cons;   // consumer handle
    u32 gen;    // the consumer's incarnation the edge was made for
    u32 next;   // next edge of the producer's list
};

// Where the graph kernels read VALID and write keys.  S = false (one context): key[h] for every handle.  S = true (a sharded
// graph context): VALID is the replicated bit gvalid[h], a VALID task waits while it has unfinished dependencies (nothing
// but a release makes a task with dependencies READY there: hqs_ready_push is refused), and only the handles
// [lo, hi) have a key, key[h - lo] (hi is clipped to the key table's capacity: the keys beyond it are not VALID).
struct GraphKeys {
    u32* key;
    u32* gvalid;     // S only: [n_total / 32] bits
    u32 lo, hi;
};

template <bool S>
__device__ __forceinline__ bool graph_valid(const GraphKeys& k, u32 h) {
    if (S) return (k.gvalid[h >> 5] >> (h & 31)) & 1u;
    return k.key[h] & KEY_VALID;
}

// h is VALID and neither READY nor DONE
template <bool S>
__device__ __forceinline__ bool graph_waiting(const GraphKeys& k, const u32* gdeps, u32 h) {
    if (S) return graph_valid<true>(k, h) && gdeps[h] != 0u;
    return (k.key[h] & (KEY_VALID | KEY_READY | KEY_DONE)) == KEY_VALID;
}

// the key word of h if this context holds it, nullptr otherwise
template <bool S>
__device__ __forceinline__ u32* graph_own(const GraphKeys& k, u32 h) {
    if (!S) return k.key + h;
    return h - k.lo < k.hi - k.lo ? k.key + (h - k.lo) : nullptr;
}

// host: runs f(std::true_type) for a sharded graph context, f(std::false_type) otherwise (the kernel instance to launch)
template <typename F>
void graph_dispatch(bool shard, F&& f) {
    if (shard) f(std::true_type{});
    else f(std::false_type{});
}

// exclusive prefix sum over the block (NT <= 1024); *total receives the block's sum in every thread
template <u32 NT>
__device__ __forceinline__ u32 graph_block_scan(u32 v, u32* total) {
    __shared__ u32 warp_off[NT / 32];
    __shared__ u32 block_sum;
    const u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    u32 x = v;
    for (u32 o = 1; o < 32; o <<= 1) {
        const u32 y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_off[wid] = x;
    __syncthreads();
    if (wid == 0) {
        const u32 s = lane < NT / 32 ? warp_off[lane] : 0u;
        u32 t = s;
        for (u32 o = 1; o < 32; o <<= 1) {
            const u32 y = __shfl_up_sync(0xffffffffu, t, o);
            if (lane >= o) t += y;
        }
        if (lane < NT / 32) warp_off[lane] = t - s;
        if (lane == 31) block_sum = t;
    }
    __syncthreads();
    const u32 r = warp_off[wid] + x - v;
    *total = block_sum;
    __syncthreads();   // the shared words may be reused by the next call
    return r;
}

// single block: in-place exclusive scan of nb per-block sums; *total = their sum
__global__ void __launch_bounds__(1024) graph_scan_k(u32 nb, u32* __restrict__ blk, u32* __restrict__ total) {
    u32 carry = 0;
    for (u32 base = 0; base < nb; base += 1024) {
        const u32 i = base + threadIdx.x;
        const u32 v = i < nb ? blk[i] : 0u;
        u32 sum;
        const u32 ex = graph_block_scan<1024>(v, &sum);
        if (i < nb) blk[i] = carry + ex;
        carry += sum;
    }
    if (threadIdx.x == 0) *total = carry;
}

// a pushed handle that is still VALID rejects the batch (flag[1] bit 1; push_k and graph_link_k then write nothing).
// Handles >= n_handles have never been pushed.
template <bool S>
__global__ void graph_validate_k(u32 n, const u32* __restrict__ task, const GraphKeys k, u32 n_handles,
                                 u32* __restrict__ flag) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    const u32 h = i < n ? task[i] : GRAPH_NIL;
    const bool bad = h < n_handles && graph_valid<S>(k, h);
    if (__ballot_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(&flag[1], 2u);
}

// sharded graph context, after graph_validate_k: the batch becomes VALID in the graph's view (push_k's part for the replica)
__global__ void graph_enter_k(u32 n, const u32* __restrict__ task, const u32* __restrict__ flag, u32* __restrict__ gvalid) {
    if (flag[1]) return;                    // the batch was rejected
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) atomicOr(&gvalid[task[i] >> 5], 1u << (task[i] & 31));
}

// after push_k: task i's dependencies are dep[off[i] .. off[i+1]) (the host dropped those on later tasks of the batch).  One
// counts if its producer is VALID: a task of the table or an earlier task of the batch (push_k made those VALID).  Counted
// edges take slot e0 + j and are linked into the producer's list; a task with a counted dependency is waiting (READY
// cleared).  n_ready[0] += tasks ready at once (of this context's own handles).
template <bool S>
__global__ void graph_link_k(u32 n, const u32* __restrict__ task, const u32* __restrict__ off, const u32* __restrict__ dep,
                             u32 e0, const u32* __restrict__ flag, const GraphKeys k, u32* __restrict__ gdeps,
                             u32* __restrict__ ggen, u32* __restrict__ ghead, GraphEdge* __restrict__ pool,
                             u32* __restrict__ n_ready) {
    if (flag[1]) return;                    // the batch was rejected
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    bool ready = false;
    if (i < n) {
        const u32 h = task[i];
        const u32 g = ggen[h] + 1;
        ggen[h] = g;
        u32 cnt = 0;
        for (u32 j = off[i], hi = off[i + 1]; j < hi; ++j) {
            const u32 p = dep[j];
            if (!graph_valid<S>(k, p)) continue;            // finished, removed or never pushed: dropped
            const u32 e = e0 + j;
            pool[e].cons = h;
            pool[e].gen = g;
            pool[e].next = atomicExch(&ghead[p], e);
            ++cnt;
        }
        gdeps[h] = cnt;
        u32* kh = graph_own<S>(k, h);
        if (cnt && kh) *kh &= ~KEY_READY;   // only this thread writes key[h]; the others read its VALID bit
        ready = cnt == 0 && kh;
    }
    const u32 made = __popc(__ballot_sync(0xffffffffu, ready));
    if ((threadIdx.x & 31) == 0 && made) atomicAdd(n_ready, made);
}

// hqs_graph_finished, phase 1: every finished task leaves the table.  Only the thread that clears VALID keeps the handle
// (win[i]), so a handle named twice, or one that is not VALID, walks no list.  All tasks of the batch have left before any
// consumer is looked at (phase 2), so a consumer finished in the same batch is never released.
// On a sharded graph context the winner is the thread that clears the graph VALID bit, and the owner's key leaves with it.
template <bool S>
__global__ void graph_leave_k(u32 n, const u32* __restrict__ task, const GraphKeys k, u32* __restrict__ win) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u32 h = task[i];
    constexpr u32 gone = ~(KEY_READY | KEY_VALID | KEY_DONE | KEY_PF);
    bool won;
    if (S) {
        const u32 b = 1u << (h & 31);
        won = atomicAnd(&k.gvalid[h >> 5], ~b) & b;
        if (u32* kh = graph_own<S>(k, h); won && kh) *kh &= gone;
    } else {
        won = atomicAnd(&k.key[h], gone) & KEY_VALID;
    }
    win[i] = won ? h : GRAPH_NIL;
}

// the consumer of edge E still waits on the incarnation E was made for
template <bool S>
__device__ __forceinline__ bool graph_edge_waits(const GraphEdge& E, const GraphKeys& k, const u32* gdeps, const u32* ggen) {
    return ggen[E.cons] == E.gen && graph_waiting<S>(k, gdeps, E.cons);
}

// phase 2: each kept handle walks its consumers; the decrement that reaches zero makes the consumer READY and flags it in the
// ready bitmap (one bit per handle; on a sharded graph context only the handles it owns).  Then the list is emptied.
template <bool S>
__global__ void graph_release_k(u32 n, const u32* __restrict__ win, const GraphKeys k, u32* gdeps,
                                const u32* __restrict__ ggen, u32* __restrict__ ghead, const GraphEdge* __restrict__ pool,
                                u32* __restrict__ bits) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u32 h = win[i];
    if (h == GRAPH_NIL) return;
    for (u32 e = ghead[h]; e != GRAPH_NIL;) {
        const GraphEdge E = pool[e];
        if (graph_edge_waits<S>(E, k, gdeps, ggen) && atomicSub(&gdeps[E.cons], 1u) == 1u) {
            if (u32* kc = graph_own<S>(k, E.cons)) {
                atomicOr(kc, KEY_READY);
                atomicOr(&bits[E.cons >> 5], 1u << (E.cons & 31));
            }
        }
        e = E.next;
    }
    ghead[h] = GRAPH_NIL;
}

// phase 3: ordered compaction of the ready bitmap.  Thread t of block b owns the words [(b * NT + t) * 8, + 8).
__global__ void __launch_bounds__(GRAPH_NT) graph_ready_count_k(u32 n_words, const u32* __restrict__ bits,
                                                                 u32* __restrict__ blk) {
    const u32 w0 = (blockIdx.x * GRAPH_NT + threadIdx.x) * GRAPH_PER_THREAD;
    u32 c = 0;
#pragma unroll
    for (u32 k = 0; k < GRAPH_PER_THREAD; ++k)
        if (w0 + k < n_words) c += __popc(bits[w0 + k]);
    u32 sum;
    graph_block_scan<GRAPH_NT>(c, &sum);
    if (threadIdx.x == 0) blk[blockIdx.x] = sum;
}

// blk = exclusive scan of graph_ready_count_k's sums: the handles come out ascending, and the bitmap is cleared
__global__ void __launch_bounds__(GRAPH_NT) graph_ready_emit_k(u32 n_words, u32* __restrict__ bits,
                                                                const u32* __restrict__ blk, u32* __restrict__ out) {
    const u32 w0 = (blockIdx.x * GRAPH_NT + threadIdx.x) * GRAPH_PER_THREAD;
    u32 w[GRAPH_PER_THREAD];
    u32 c = 0;
#pragma unroll
    for (u32 k = 0; k < GRAPH_PER_THREAD; ++k) {
        w[k] = w0 + k < n_words ? bits[w0 + k] : 0u;
        c += __popc(w[k]);
    }
    u32 sum;
    u32 pos = blk[blockIdx.x] + graph_block_scan<GRAPH_NT>(c, &sum);
#pragma unroll
    for (u32 k = 0; k < GRAPH_PER_THREAD; ++k) {
        u32 x = w[k];
        if (!x) continue;
        bits[w0 + k] = 0u;
        while (x) {
            out[pos++] = (w0 + k) * 32u + (u32)(__ffs(x) - 1);
            x &= x - 1;
        }
    }
}

// hqs_ready_remove on a graph context: the removed producers' lists are emptied (their consumers stay waiting)
__global__ void graph_unlink_k(u32 n, const u32* __restrict__ task, u32 n_handles, u32* __restrict__ ghead) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u32 h = task[i];
    if (h < n_handles) ghead[h] = GRAPH_NIL;
}

// pool compaction, pass 1: edges whose consumer still waits on their incarnation, per block of 2048 producers
template <bool S>
__global__ void __launch_bounds__(GRAPH_NT) graph_gc_count_k(u32 n_handles, const u32* __restrict__ ghead,
                                                              const GraphEdge* __restrict__ pool, const GraphKeys k,
                                                              const u32* __restrict__ gdeps, const u32* __restrict__ ggen,
                                                              u32* __restrict__ blk) {
    const u32 h0 = (blockIdx.x * GRAPH_NT + threadIdx.x) * GRAPH_PER_THREAD;
    u32 c = 0;
    for (u32 j = 0; j < GRAPH_PER_THREAD; ++j) {
        if (h0 + j >= n_handles) break;
        for (u32 e = ghead[h0 + j]; e != GRAPH_NIL; e = pool[e].next) c += graph_edge_waits<S>(pool[e], k, gdeps, ggen) ? 1u : 0u;
    }
    u32 sum;
    graph_block_scan<GRAPH_NT>(c, &sum);
    if (threadIdx.x == 0) blk[blockIdx.x] = sum;
}

// pass 2 (blk scanned): every list is rewritten, in its order, into consecutive slots of the fresh pool.
// RN (hqs_handles_compact): the handles are renumbered as well.  Every consumer and every producer with a non-empty list is
// VALID, so it survives, and new_of_old[] holds its new handle: the edges take the new consumer handles, and each non-empty
// list's head goes to head_out[new handle] (a fresh array; ghead is only read).
template <bool S, bool RN = false>
__global__ void __launch_bounds__(GRAPH_NT) graph_gc_move_k(u32 n_handles, u32* __restrict__ ghead,
                                                             const GraphEdge* __restrict__ pool, GraphEdge* __restrict__ fresh,
                                                             const GraphKeys k, const u32* __restrict__ gdeps,
                                                             const u32* __restrict__ ggen, const u32* __restrict__ blk,
                                                             const u32* __restrict__ new_of_old = nullptr,
                                                             u32* __restrict__ head_out = nullptr) {
    const u32 h0 = (blockIdx.x * GRAPH_NT + threadIdx.x) * GRAPH_PER_THREAD;
    u32 c = 0;
    for (u32 j = 0; j < GRAPH_PER_THREAD; ++j) {
        if (h0 + j >= n_handles) break;
        for (u32 e = ghead[h0 + j]; e != GRAPH_NIL; e = pool[e].next) c += graph_edge_waits<S>(pool[e], k, gdeps, ggen) ? 1u : 0u;
    }
    u32 sum;
    u32 pos = blk[blockIdx.x] + graph_block_scan<GRAPH_NT>(c, &sum);
    for (u32 j = 0; j < GRAPH_PER_THREAD; ++j) {
        const u32 h = h0 + j;
        if (h >= n_handles) break;
        u32 first = GRAPH_NIL, prev = GRAPH_NIL;
        for (u32 e = ghead[h]; e != GRAPH_NIL; e = pool[e].next) {
            const GraphEdge E = pool[e];
            if (!graph_edge_waits<S>(E, k, gdeps, ggen)) continue;
            fresh[pos] = GraphEdge{RN ? new_of_old[E.cons] : E.cons, E.gen, GRAPH_NIL};
            if (prev == GRAPH_NIL) first = pos; else fresh[prev].next = pos;
            prev = pos++;
        }
        if (!RN) ghead[h] = first;
        else if (first != GRAPH_NIL) head_out[new_of_old[h]] = first;
    }
}

// hqs_graph_debug: out[0] += linked edges (ghead != nullptr), out[1] += waiting tasks (key != nullptr: VALID, neither READY
// nor DONE).  A sharded graph context counts the edges over its replicated lists and the waiting tasks over its own keys.
__global__ void graph_debug_k(u32 n_handles, const u32* __restrict__ key, const u32* __restrict__ ghead,
                              const GraphEdge* __restrict__ pool, unsigned long long* __restrict__ out) {
    const u32 h = blockIdx.x * blockDim.x + threadIdx.x;
    u32 edges = 0, waiting = 0;
    if (h < n_handles) {
        if (ghead)
            for (u32 e = ghead[h]; e != GRAPH_NIL; e = pool[e].next) ++edges;
        if (key) waiting = (key[h] & (KEY_VALID | KEY_READY | KEY_DONE)) == KEY_VALID ? 1u : 0u;
    }
    edges = __reduce_add_sync(0xffffffffu, edges);
    waiting = __reduce_add_sync(0xffffffffu, waiting);
    if ((threadIdx.x & 31) == 0) {
        if (edges) atomicAdd(&out[0], (unsigned long long)edges);
        if (waiting) atomicAdd(&out[1], (unsigned long long)waiting);
    }
}

// hqs_graph_cancel: the named VALID handles and, transitively, every consumer still waiting on its edge's incarnation are
// marked in the bitmap `bits` and appended to the work list `work` (a handle is admitted by winning its bit, so the list
// never holds a handle twice and never wraps).  The marking kernel's counters sit on separate lines: idle warps poll them.
struct GraphCancelSync {
    u32 tail, pad0[31];      // entries appended to the work list
    u32 head, pad1[31];      // entries taken from it
    u32 pending, pad2[31];   // entries admitted and not yet walked (queued or in a warp)
    u32 steps, pad3[31];     // entries walked so far: the progress the idle warps' time-outs watch
    u32 done, error, pad4[30];   // done: the marking drained the list; error: the wait that timed out (1 the list, 2 a slot)
};
constexpr u32 GRAPH_CANCEL_NT = 256;

// the named handles that are VALID seed the work list (host-checked: every handle < n_handles)
template <bool S>
__global__ void graph_cancel_seed_k(u32 n, const u32* __restrict__ task, const GraphKeys k, u32* __restrict__ bits,
                                    u32* __restrict__ work, GraphCancelSync* __restrict__ s) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
    u32 h = GRAPH_NIL;
    bool won = false;
    if (i < n) {
        h = task[i];
        const u32 b = 1u << (h & 31);
        won = graph_valid<S>(k, h) && !(atomicOr(&bits[h >> 5], b) & b);      // a handle named twice is admitted once
    }
    const u32 m = __ballot_sync(0xffffffffu, won);
    if (!m) return;
    const u32 lead = __ffs(m) - 1;
    u32 base = 0;
    if (lane == lead) {
        atomicAdd(&s->pending, __popc(m));
        base = atomicAdd(&s->tail, __popc(m));
    }
    base = __shfl_sync(0xffffffffu, base, lead);
    if (won) work[base + __popc(m & ((1u << lane) - 1))] = h;
}

// lane 0: the next entry of the work list, GRAPH_NIL once the list is drained (nothing queued, no warp walking) or a wait
// timed out.  The time-outs count time without progress (no entry appended or walked), so a long chain never trips them.
__device__ u32 graph_cancel_pop(const u32* work, GraphCancelSync* s) {
    long long t0 = clock64();
    u32 seen_tail = ld_acquire(&s->tail), seen_steps = ld_acquire(&s->steps);
    for (;;) {
        if (ld_acquire(&s->error)) return GRAPH_NIL;
        const u32 hd = ld_acquire(&s->head), tl = ld_acquire(&s->tail);
        if (hd < tl) {
            if (atomicCAS(&s->head, hd, hd + 1) != hd) continue;
            const long long t1 = clock64();      // the slot is reserved; its appender writes it next
            u32 v;
            while ((v = ld_acquire(&work[hd])) == GRAPH_NIL)
                if (clock64() - t1 > SPIN_TIMEOUT_CYCLES) { atomicCAS(&s->error, 0u, 2u); return GRAPH_NIL; }
            return v;
        }
        if (ld_acquire(&s->pending) == 0) {   // zero is final: only a warp holding an entry admits new ones
            s->done = 1u;
            return GRAPH_NIL;
        }
        const u32 st = ld_acquire(&s->steps);
        if (st != seen_steps || tl != seen_tail) {
            seen_steps = st;
            seen_tail = tl;
            t0 = clock64();
        } else if (clock64() - t0 > SPIN_TIMEOUT_CYCLES) {
            atomicCAS(&s->error, 0u, 1u);
            return GRAPH_NIL;
        }
        __nanosleep(100);
    }
}

// The marking: one cooperative launch, every warp a worker.  A warp walks its entry's consumer list (lane 0 follows the
// links, 32 edges at a time, and every lane tests one edge), admits each consumer that still waits on the edge's incarnation
// and wins its bit, keeps the first one it admits to walk next (a chain never goes through the list) and appends the rest.
// So the work list holds only part of the closure; the bitmap holds all of it.
// The keys, gvalid, gdeps, ggen, ghead and pool are only read: nothing leaves the table before graph_cancel_apply_k.  A
// sharded graph context marks the whole closure, whichever rank owns its handles.
template <bool S>
__global__ void __launch_bounds__(GRAPH_CANCEL_NT) graph_cancel_mark_k(const GraphKeys k, const u32* __restrict__ gdeps,
                                                                        const u32* __restrict__ ggen,
                                                                        const u32* __restrict__ ghead,
                                                                        const GraphEdge* __restrict__ pool, u32* bits, u32* work,
                                                                        GraphCancelSync* s) {
    __shared__ u32 s_cons[GRAPH_CANCEL_NT], s_gen[GRAPH_CANCEL_NT];
    const u32 lane = threadIdx.x & 31, w0 = threadIdx.x & ~31u;
    u32 h = GRAPH_NIL;                                  // warp-uniform: the entry being walked
    for (;;) {
        if (h == GRAPH_NIL) {
            if (lane == 0) h = graph_cancel_pop(work, s);
            h = __shfl_sync(0xffffffffu, h, 0);
            if (h == GRAPH_NIL) return;
        }
        u32 e = ghead[h], next = GRAPH_NIL;
        while (e != GRAPH_NIL) {
            u32 cnt = 0;
            if (lane == 0)
                for (; cnt < 32 && e != GRAPH_NIL; ++cnt) {
                    const GraphEdge E = pool[e];
                    s_cons[w0 + cnt] = E.cons;
                    s_gen[w0 + cnt] = E.gen;
                    e = E.next;
                }
            e = __shfl_sync(0xffffffffu, e, 0);
            cnt = __shfl_sync(0xffffffffu, cnt, 0);
            __syncwarp();
            bool won = false;
            u32 c = 0;
            if (lane < cnt) {
                c = s_cons[w0 + lane];
                const u32 b = 1u << (c & 31);
                won = ggen[c] == s_gen[w0 + lane] && graph_waiting<S>(k, gdeps, c) && !(atomicOr(&bits[c >> 5], b) & b);
            }
            __syncwarp();
            u32 m = __ballot_sync(0xffffffffu, won);
            if (m && next == GRAPH_NIL) {               // the first admitted consumer inherits this entry's pending count
                const u32 first = __ffs(m) - 1;
                next = __shfl_sync(0xffffffffu, c, first);
                m &= m - 1;
                won = won && lane != first;
            }
            if (m) {                                    // counted as pending before anyone can take them
                const u32 lead = __ffs(m) - 1;
                u32 base = 0;
                if (lane == lead) {
                    atomicAdd(&s->pending, __popc(m));
                    base = atomicAdd(&s->tail, __popc(m));
                }
                base = __shfl_sync(0xffffffffu, base, lead);
                if (won) st_release(&work[base + __popc(m & ((1u << lane) - 1))], c);
            }
        }
        if (lane == 0) {
            atomicAdd(&s->steps, 1u);
            if (next == GRAPH_NIL) atomicSub(&s->pending, 1u);
        }
        h = next;
    }
}

// After the ordered emit (graph_ready_emit_k wrote the marked handles ascending to out[0 .. *n_out) and cleared the bitmap),
// and only if the marking drained its list: every marked handle leaves the table (as graph_leave_k makes it leave) and its
// consumer list is emptied.  The work list returns to GRAPH_NIL either way.  A sharded graph context clears the graph VALID
// bit of every marked handle and the keys of the ones it owns.
template <bool S>
__global__ void graph_cancel_apply_k(u32* __restrict__ work, const GraphCancelSync* __restrict__ s, const u32* __restrict__ out,
                                     const u32* __restrict__ n_out, const GraphKeys k, u32* __restrict__ ghead) {
    const u32 stride = gridDim.x * blockDim.x, i0 = blockIdx.x * blockDim.x + threadIdx.x;
    for (u32 i = i0, n = s->tail; i < n; i += stride) work[i] = GRAPH_NIL;
    if (!s->done || s->error) return;
    for (u32 i = i0, n = *n_out; i < n; i += stride) {
        const u32 h = out[i];
        if (u32* kh = graph_own<S>(k, h)) *kh &= ~(KEY_READY | KEY_VALID | KEY_DONE | KEY_PF);
        if (S) atomicAnd(&k.gvalid[h >> 5], ~(1u << (h & 31)));
        ghead[h] = GRAPH_NIL;
    }
}

// hqs_handles_compact: the survivors (VALID keys, plus the handles named in keep) are marked in a zeroed bitmap of one bit
// per handle; the ordered compaction above then writes them out ascending.  One thread per handle (a warp covers one bitmap
// word) and one per keep entry.
__global__ void compact_mark_k(u32 n_handles, const u32* __restrict__ key, u32 n_keep, const u32* __restrict__ keep,
                               u32* __restrict__ bits) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    const u32 m = __ballot_sync(0xffffffffu, i < n_handles && (key[i] & KEY_VALID));
    if ((threadIdx.x & 31) == 0 && m) atomicOr(&bits[i >> 5], m);
    if (i < n_keep) atomicOr(&bits[keep[i] >> 5], 1u << (keep[i] & 31));      // host-checked: keep[i] < n_handles
}

// survivor i (old handle order[i]) becomes handle i: its key and priority, and on a graph context its dependency count and
// incarnation, move to slot i of the fresh arrays; new_of_old[old] = i for the edge rewrite (graph_gc_move_k<S, true>)
__global__ void compact_gather_k(u32 n_kept, const u32* __restrict__ order, const u32* __restrict__ key,
                                 const u64* __restrict__ prio, const u32* __restrict__ gdeps, const u32* __restrict__ ggen,
                                 u32* __restrict__ key_out, u64* __restrict__ prio_out, u32* __restrict__ gdeps_out,
                                 u32* __restrict__ ggen_out, u32* __restrict__ new_of_old) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_kept) return;
    const u32 o = order[i];
    key_out[i] = key[o];
    prio_out[i] = prio[o];
    new_of_old[o] = i;
    if (gdeps) {
        gdeps_out[i] = gdeps[o];
        ggen_out[i] = ggen[o];
    }
}

// hqs_shard_graph_compact: the survivors are the replicated graph VALID bits plus the handles named in keep, over the global
// handles, so every rank marks the same bitmap without reading a key.  One thread per bitmap word and one per keep entry,
// into a zeroed bitmap.
__global__ void shard_compact_mark_k(u32 n_words, const u32* __restrict__ gvalid, u32 n_keep, const u32* __restrict__ keep,
                                     u32* __restrict__ bits) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_words && gvalid[i]) atomicOr(&bits[i], gvalid[i]);
    if (i < n_keep) atomicOr(&bits[keep[i] >> 5], 1u << (keep[i] & 31));      // host-checked: keep[i] < n_total
}

// after the ordered emit: out[t] = the number of survivors below bound[t] (lo, then hi), by a binary search of the ascending
// order[0 .. *n_kept).  Two threads.
__global__ void shard_compact_range_k(const u32* __restrict__ order, const u32* __restrict__ n_kept, u32 lo, u32 hi,
                                      u32* __restrict__ out) {
    const u32 t = threadIdx.x;
    if (t >= 2) return;
    const u32 x = t ? hi : lo;
    u32 a = 0, b = *n_kept;
    while (a < b) {
        const u32 m = a + (b - a) / 2;
        if (order[m] < x) a = m + 1; else b = m;
    }
    out[t] = a;
}

// Survivor i (global old handle order[i]) becomes global handle i on every rank: its graph VALID bit, dependency count and
// incarnation move to slot i of the fresh replicated arrays, and new_of_old[old] = i for the edge rewrite
// (graph_gc_move_k<true, true>).  The rank's own survivors, i in [own_lo, own_hi), also move their key and priority from the
// local slot old - lo to the new local slot i - own_lo (a kept handle past the old table, n_handles, has neither).  The
// fresh bitmap is written a word per warp: blockDim is a multiple of 32, so a warp's survivors are one word's bits.
__global__ void shard_compact_gather_k(u32 n_kept, const u32* __restrict__ order, const u32* __restrict__ gvalid,
                                       const u32* __restrict__ gdeps, const u32* __restrict__ ggen, u32 lo, u32 n_handles,
                                       u32 own_lo, u32 own_hi, const u32* __restrict__ key, const u64* __restrict__ prio,
                                       u32* __restrict__ gvalid_out, u32* __restrict__ gdeps_out, u32* __restrict__ ggen_out,
                                       u32* __restrict__ key_out, u64* __restrict__ prio_out, u32* __restrict__ new_of_old) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    const u32 o = i < n_kept ? order[i] : 0u;
    const u32 m = __ballot_sync(0xffffffffu, i < n_kept && ((gvalid[o >> 5] >> (o & 31)) & 1u));
    if (i >= n_kept) return;
    if ((threadIdx.x & 31) == 0) gvalid_out[i >> 5] = m;
    gdeps_out[i] = gdeps[o];
    ggen_out[i] = ggen[o];
    new_of_old[o] = i;
    if (i >= own_lo && i < own_hi) {
        const u32 l = o - lo;
        key_out[i - own_lo] = l < n_handles ? key[l] : 0u;
        prio_out[i - own_lo] = l < n_handles ? prio[l] : 0ull;
    }
}
